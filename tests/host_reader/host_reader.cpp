// tests/host_reader/host_reader.cpp -- TEST INFRASTRUCTURE: drives abyss_b200/host/reads.h on the CPU.
//   host_reader serial FILE...                          one SeqReader after the other
//   host_reader stream THREADS BATCH PIECE FILE...      BatchStream (background, parallel parsing)
//   READER_TIME=1 ...                                   no output, reads/s on stderr (ingest throughput measurement)
// Both print "id<TAB>sequence" per read and a "# batch N" line per batch (stream mode), so that the
// test can compare the two record for record and check the batch sizes.
#include "../../abyss_b200/host/reads.h"
#include <chrono>

int main(int argc, char** argv)
{
	host::ReadOpts o;
	if (const char* q = getenv("READER_Q"))
		o.qualityThreshold = atoi(q);
	if (const char* q = getenv("READER_MASKQ"))
		o.internalQThreshold = atoi(q);
	if (getenv("READER_NO_CHASTITY"))
		o.chastityFilter = 0;
	if (getenv("READER_NO_TRIM_MASKED"))
		o.trimMasked = 0;
	if (const char* q = getenv("READER_QOFF"))
		o.qualityOffset = atoi(q);
	if (argc < 3)
		return 2;
	const bool timing = getenv("READER_TIME") != nullptr;
	const auto t0 = std::chrono::steady_clock::now();
	uint64_t n_reads = 0;
	auto report = [&]() {
		const double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
		if (timing)
			fprintf(stderr, "%llu reads in %.3f s: %.2f M reads/s\n", (unsigned long long)n_reads, s, n_reads / s / 1e6);
	};
	if (std::string(argv[1]) == "serial") {
		for (int i = 2; i < argc; ++i) {
			host::SeqReader in(argv[i], o);
			std::string id, seq;
			while (in.next(id, seq)) {
				++n_reads;
				if (!timing)
					printf("%s\t%s\n", id.c_str(), seq.c_str());
			}
		}
		report();
		return 0;
	}
	if (argc < 6)
		return 2;
	const unsigned threads = (unsigned)atoi(argv[2]);
	const uint64_t batch = strtoull(argv[3], nullptr, 10);
	const size_t piece = strtoull(argv[4], nullptr, 10);
	std::vector<std::string> files(argv + 5, argv + argc);
	host::BatchStream bs(files, o, batch, threads, false, piece);
	while (const host::ReadBatch* b = bs.next()) {
		n_reads += b->size();
		if (timing)
			continue;
		fprintf(stderr, "# batch %zu\n", b->size());
		for (size_t i = 0; i < b->size(); ++i)
			printf("%s\t%.*s\n", b->id(i).c_str(), (int)(b->offsets[i + 1] - b->offsets[i]), b->bases.data() + b->offsets[i]);
	}
	report();
	return 0;
}
