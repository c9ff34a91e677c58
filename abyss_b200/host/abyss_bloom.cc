// abyss-bloom (GPU) -- the `build` command of the reference's abyss-bloom for the ntHash filter
// family (Bloom/bloom.cc:584-622,625-800): `-t counting` (CountingBloomFilter<uint8_t>, the
// filter abyss-bloom-dbg loads with -i) and `-t rolling-hash [-l LEVELS]`
// (HashAgnosticCascadingBloom, last level serialised).  The Konnector filter family (`-t
// konnector`, city hash) and union/intersect/compare/graph/kmers/trim are out of scope
// (SURVEY.md section 2).  Output files are byte-compatible with the reference's.
//
//   abyss-bloom build [-v] -k K [-b SIZE] [-H N] [-l LEVELS] [-t counting|rolling-hash] OUT.bloom READS...
#include "../../include/abyss_b200.h"
#include "bloom_file.h"
#include "reads.h"
#include <getopt.h>
#include <cmath>
#include <iomanip>

#define PROGRAM "abyss-bloom"
using namespace host;

static void check(int rc, const char* what)
{
	if (rc != ABB_OK) {
		std::cerr << PROGRAM ": " << what << ": " << abb_last_error() << "\n";
		exit(EXIT_FAILURE);
	}
}
static void usage()
{
	std::cerr << "Usage: " PROGRAM " build [-v] -k K [-b SIZE] [-H N] [-l LEVELS] [-t counting|rolling-hash] <OUTPUT_BLOOM_FILE> <READS_FILE_1> [READS_FILE_2]...\n"
	             "Try `" PROGRAM " --help' for more information.\n";
	exit(EXIT_FAILURE);
}

/** `abyss-bloom info FILE`: printBloomStats (Bloom/bloom.cc:433-441,823-846) for the two ntHash-family file formats.
 *  (The reference's `info` reads the Konnector format only; the filters of this path are the BTL ones, so this command
 *  prints the same three lines for them, with the population counted on the GPU.) */
static int info(int argc, char** argv)
{
	int device = 0;
	std::string path;
	for (int i = 2; i < argc; ++i) {
		const std::string a = argv[i];
		if (a.rfind("--device=", 0) == 0)
			device = atoi(a.c_str() + 9);
		else if (a == "-v" || a == "--verbose")
			;
		else
			path = a;
	}
	if (path.empty()) {
		std::cerr << PROGRAM ": missing arguments\n";
		usage();
	}
	std::ifstream probe(path, std::ios::binary);
	std::string magic;
	std::getline(probe, magic);
	probe.close();
	BloomHeader h;
	std::vector<uint8_t> raw;
	abb_filter* f = nullptr;
	if (magic == "[BTLCountingBloomFilter_v1]") {
		read_counting_bloom(path, h, raw);
		check(abb_filter_create(&f, ABB_COUNTING, h.size, h.hashNum, h.kmerSize, 1, "", device), "filter");
	} else {
		read_bit_bloom(path, h, raw);
		check(abb_filter_create(&f, ABB_BIT, h.size, h.hashNum, h.kmerSize, 0, "", device), "filter");
	}
	check(abb_filter_upload(f, 0, raw.data(), raw.size()), "upload");
	uint64_t nz = 0;
	check(abb_filter_popcount(f, &nz, nullptr), "popcount");
	std::cerr << "Bloom size (bits): " << h.size << "\n"
	          << "Bloom popcount (bits): " << nz << "\n"
	          << "Bloom filter FPR: " << std::setprecision(3) << 100 * std::pow((double)nz / (double)h.size, (double)h.hashNum) << "%\n";
	abb_filter_destroy(f);
	return EXIT_SUCCESS;
}

int main(int argc, char** argv)
{
	if (argc >= 2 && std::string(argv[1]) == "info")
		return info(argc, argv);
	if (argc < 2 || std::string(argv[1]) != "build") {
		std::cerr << PROGRAM ": only the `build' (-t counting | rolling-hash) and `info' commands are implemented on the GPU\n";
		usage();
	}
	uint64_t bloomSize = 500ULL << 20; // [500M]
	unsigned k = 0, numHashes = 1, levels = 1, threads = 1;
	int verbose = 0, device = 0;
	uint64_t batchReads = 4000000;
	std::string type = "konnector";
	ReadOpts ropt;
	static int chastity = 1, trimMasked = 1, qualityOffset = 0; // 0 = the format's own offset
	static const struct option longopts[] = {
		{ "bloom-size", required_argument, NULL, 'b' }, { "kmer", required_argument, NULL, 'k' },
		{ "num-hashes", required_argument, NULL, 'H' }, { "levels", required_argument, NULL, 'l' },
		{ "bloom-type", required_argument, NULL, 't' }, { "threads", required_argument, NULL, 'j' },
		{ "trim-quality", required_argument, NULL, 'q' }, { "verbose", no_argument, NULL, 'v' },
		{ "chastity", no_argument, &chastity, 1 }, { "no-chastity", no_argument, &chastity, 0 },
		{ "trim-masked", no_argument, &trimMasked, 1 }, { "no-trim-masked", no_argument, &trimMasked, 0 },
		{ "standard-quality", no_argument, &qualityOffset, 33 }, { "illumina-quality", no_argument, &qualityOffset, 64 },
		{ "device", required_argument, NULL, 1000 }, { "batch-reads", required_argument, NULL, 1001 },
		{ NULL, 0, NULL, 0 }
	};
	optind = 2;
	for (int c; (c = getopt_long(argc, argv, "b:B:h:H:j:k:l:n:q:t:vw:", longopts, NULL)) != -1;) {
		switch (c) {
		case '?': usage(); break;
		case 'b':
			if (!si_to_bytes(optarg, &bloomSize)) {
				std::cerr << PROGRAM ": invalid option: `-b" << optarg << "'\n";
				exit(EXIT_FAILURE);
			}
			break;
		case 'k': k = (unsigned)atoi(optarg); break;
		case 'H': numHashes = (unsigned)atoi(optarg); break;
		case 'l': levels = (unsigned)atoi(optarg); break;
		case 'j': threads = (unsigned)atoi(optarg); break;
		case 'q': ropt.qualityThreshold = atoi(optarg); break;
		case 't': type = optarg; break;
		case 'v': ++verbose; break;
		case 1000: device = atoi(optarg); break;
		case 1001: batchReads = strtoull(optarg, nullptr, 10); break;
		case 'B': case 'h': case 'n': break; // I/O buffer, city-hash seed, lock count: no effect here
		case 'w':
			std::cerr << PROGRAM ": -w (Bloom windows) only applies to `-t konnector' filters\n";
			exit(EXIT_FAILURE);
		}
	}
	ropt.chastityFilter = chastity;
	ropt.trimMasked = trimMasked;
	ropt.qualityOffset = qualityOffset;
	if (k == 0) {
		std::cerr << PROGRAM ": missing mandatory option `-k'\n";
		usage();
	}
	if (type != "counting" && type != "rolling-hash") {
		std::cerr << PROGRAM ": `-t " << type << "' is not available on the GPU: use 'rolling-hash' or 'counting'\n";
		usage();
	}
	if (argc - optind < 2) {
		std::cerr << PROGRAM ": missing arguments\n";
		usage();
	}
	const std::string outputPath = argv[optind++];
	std::vector<std::string> files(argv + optind, argv + argc);

	abb_filter* f = nullptr;
	uint64_t levelBits = 0;
	if (type == "counting") {
		if (levels != 1)
			std::cerr << PROGRAM ": warning: -l option has no effect when using `-t counting'\n";
		/* buildCountingBloom (bloom.cc:604-622): CountingBloomFilter<uint8_t>(bytes, H, k, 0) */
		check(abb_filter_create(&f, ABB_COUNTING, bloomSize, numHashes, k, 0, "", device), "filter");
	} else {
		/* buildRollingHashBloom (bloom.cc:584-601): level size = roundUpToMultiple(bits / levels, 64) */
		levelBits = bloomSize * 8 / levels;
		if (levelBits % 64)
			levelBits += 64 - levelBits % 64;
		check(abb_filter_create(&f, ABB_CASCADING, levelBits, numHashes, k, levels, "", device), "filter");
	}
	uint64_t readCount = 0;
	{
		host::BatchStream stream(files, ropt, batchReads, threads > 1 ? threads : 0, verbose != 0);
		while (const ReadBatch* batch = stream.next()) {
			check(abb_insert_reads(f, batch->bases.data(), batch->offsets.data(), batch->size(), nullptr), "insert");
			readCount += batch->size();
			if (verbose)
				std::cerr << "Loaded " << readCount << " reads into Bloom filter\n";
		}
	}
	if (verbose) {
		uint64_t nz = 0, th = 0;
		check(abb_filter_popcount(f, &nz, &th), "popcount");
		std::cerr << "Bloom size: " << abb_filter_size(f) << "\nBloom popcount: " << nz << "\nBloom filter FPR: " << std::setprecision(3)
		          << 100 * std::pow((double)nz / (double)abb_filter_size(f), (double)numHashes) << "%\n"
		          << "Writing bloom filter to `" << outputPath << "'...\n";
	}
	std::vector<uint8_t> raw(abb_filter_size_in_bytes(f));
	check(abb_filter_download(f, -1, raw.data(), raw.size()), "download");
	std::ofstream out(outputPath, std::ios::binary);
	if (!out) {
		std::cerr << "error: `" << outputPath << "': cannot open for writing\n";
		exit(EXIT_FAILURE);
	}
	if (type == "counting") {
		BloomHeader h;
		h.size = abb_filter_size(f);
		h.sizeInBytes = abb_filter_size_in_bytes(f);
		h.hashNum = numHashes;
		h.kmerSize = k;
		write_counting_bloom(out, h, raw);
	} else
		write_bit_bloom(out, levelBits, numHashes, k, raw);
	out.flush();
	if (!out) {
		std::cerr << "error: `" << outputPath << "': write failed\n";
		exit(EXIT_FAILURE);
	}
	abb_filter_destroy(f);
	return EXIT_SUCCESS;
}
