// abyss-bloom-dbg (GPU) -- the reference's command line (BloomDBG/bloom-dbg.cc:44-558) over
// libabyssb200: same options, same AssemblyParams surface, same output, GPU underneath.
//
//   abyss-bloom-dbg -b <bloom_size> -H <bloom_hashes> -k <kmer_size> [options] <FASTQ>... > assembly.fasta
//
// Flow (countingBloomAssembly, bloom-dbg.cc:347-386): size the counting filter from -b, pass 1
// = abb_insert_reads over every input file in order, pass 2 = abb_assembler_process_reads over
// the same files again, FASTA records `>ID LEN COV read:READID` (printContig, bloom-dbg.h:455-487).
// -i FILE loads a [BTLCountingBloomFilter_v1] file instead of pass 1 (prebuiltBloomAssembly,
// :301-345).  -C FILE -R REF writes the 0/1 k-mer coverage track (writeCovTrack, bloom-dbg.h:1280-1334) with one GPU
// query per batch of reference records; -g FILE writes the GraphViz dump of the graph (outputGraph, :1171-1242): the breadth-first
// order is the reference's, the Bloom lookups of the frontier are GPU batches (abb_successors).
#include "../../include/abyss_b200.h"
#include "bloom_file.h"
#include "graph_dump.h"
#include "reads.h"
#include <getopt.h>
#include <climits>
#include <cmath>
#include <fstream>
#include <iomanip>
#include <iostream>
#include <sstream>
#include <thread>
#include <unordered_map>
#include <unordered_set>

#define PROGRAM "abyss-bloom-dbg"
#define MAX_KMER 192
#define MAX_HASHES 32

using namespace host;

/** BloomDBG::AssemblyParams (BloomDBG/AssemblyParams.h:13-121) */
struct AssemblyParams {
	uint64_t bloomSize = 0;
	uint64_t readsPerCheckpoint = UINT64_MAX;
	bool keepCheckpoint = false;
	std::string checkpointPathPrefix = "bloom-dbg-checkpoint";
	unsigned minCov = 2;
	std::string readLogPath, covTrackPath, graphPath;
	unsigned numHashes = 4;
	std::string bloomPath;
	unsigned threads = 1;
	unsigned k = 0, K = 0;
	std::string refPath;
	unsigned qrSeedLen = 0;
	std::string spacedSeed;
	unsigned trim = UINT_MAX;
	int verbose = 0;
	std::string outputPath, tracePath;
	int device = 0; // GPU extension: --device=N
	std::string devices; // GPU extension: --devices=LIST, several GPUs (one host thread per GPU)
	uint64_t batchReads = 4000000; // GPU extension: --batch-reads=N
	bool initialized() const { return bloomSize > 0 && k > 0 && trim != UINT_MAX; }
	void resetSpacedSeedParams()
	{
		spacedSeed.clear();
		K = 0;
		qrSeedLen = 0;
	}
};

static const char VERSION_MESSAGE[] = PROGRAM " (abyss-b200) 0.1.0, command-line compatible with " PROGRAM " (ABySS) 2.3.10\n";

static const char USAGE_MESSAGE[] =
    "Usage: " PROGRAM " -b <bloom_size> -H <bloom_hashes> -k <kmer_size> \\\n"
    "    [options] <FASTQ> [FASTQ]... > assembly.fasta\n"
    "\n"
    "Perform a de Bruijn graph assembly of the given FASTQ files on an NVIDIA H100 GPU.\n"
    "\n"
    "Basic Options:\n"
    "\n"
    "  -b  --bloom-size=N           overall memory budget for the assembly in bytes.\n"
    "                               Unit suffixes 'k', 'M', or 'G' may be used. [required]\n"
    "      --chastity               discard unchaste reads [default]\n"
    "      --no-chastity            do not discard unchaste reads\n"
    "      --help                   display this help and exit\n"
    "  -H  --num-hashes=N           number of Bloom filter hash functions [4]\n"
    "  -i  --input-bloom=FILE       load Bloom filter from FILE\n"
    "  -j, --threads=N              host threads that parse the input files [up to 8]\n"
    "      --trim-masked            trim masked bases from the ends of reads [default]\n"
    "      --no-trim-masked         do not trim masked bases from the ends of reads\n"
    "  -k, --kmer=N                 the size of a k-mer [<=192]\n"
    "      --kc=N                   ignore k-mers having a count < N [2]\n"
    "  -o, --out=FILE               write the contigs to FILE [STDOUT]\n"
    "  -q, --trim-quality=N         trim bases from the ends of reads whose quality is less than N\n"
    "  -Q, --mask-quality=N         mask all low quality bases as `N'\n"
    "      --standard-quality       zero quality is `!' (33) [default]\n"
    "      --illumina-quality       zero quality is `@' (64)\n"
    "  -t, --trim-length=N          max branch length to trim, in k-mers [k]\n"
    "  -v, --verbose                display verbose output\n"
    "      --version                output version information and exit\n"
    "      --read-log=FILE          write outcome of processing each read to FILE\n"
    "      --device=N               CUDA device to use [0]\n"
    "      --devices=LIST           several GPUs, e.g. 0-7 or 0,2,4: the counting Bloom\n"
    "                               filter is sharded by position range over them (same\n"
    "                               output as one GPU), one host thread per GPU\n"
    "      --batch-reads=N          reads per GPU batch [4000000]\n"
    "\n"
    "  -C, --cov-track=FILE         WIG track with 0/1 indicating k-mers with coverage\n"
    "                               above the --kc threshold; requires --ref\n"
    "  -R, --ref=FILE               reference genome for --cov-track\n"
    "\n"
    "  -g  --graph=FILE             write de Bruijn graph to FILE (GraphViz)\n"
    "\n"
    "Spaced seeds (-K, --qr-seed, -s), -T, --read-log, --checkpoint, -C/-R and -g work as in the reference\n"
    "(-g not together with a spaced seed).\n";

static AssemblyParams params;
static ReadOpts ropt;

enum { OPT_HELP = 1, OPT_VERSION, QR_SEED, MIN_KMER_COV, CHECKPOINT, KEEP_CHECKPOINT, CHECKPOINT_PREFIX, READ_LOG, OPT_DEVICE, OPT_DEVICES, OPT_BATCH };

static int chastity = 1, trimMasked = 1, qualityOffset = 0; // opt::qualityOffset (DataLayer/Options.h): 0 = the format's own
static const char shortopts[] = "b:C:g:H:i:j:k:K:o:q:Q:R:s:t:T:v";
static const struct option longopts[] = {
	{ "bloom-size", required_argument, NULL, 'b' },
	{ "min-coverage", required_argument, NULL, 'c' },
	{ "cov-track", required_argument, NULL, 'C' },
	{ "chastity", no_argument, &chastity, 1 },
	{ "no-chastity", no_argument, &chastity, 0 },
	{ "graph", required_argument, NULL, 'g' },
	{ "num-hashes", required_argument, NULL, 'H' },
	{ "help", no_argument, NULL, OPT_HELP },
	{ "input-bloom", required_argument, NULL, 'i' },
	{ "threads", required_argument, NULL, 'j' },
	{ "trim-masked", no_argument, &trimMasked, 1 },
	{ "no-trim-masked", no_argument, &trimMasked, 0 },
	{ "kmer", required_argument, NULL, 'k' },
	{ "kc", required_argument, NULL, MIN_KMER_COV },
	{ "single-kmer", required_argument, NULL, 'K' },
	{ "out", required_argument, NULL, 'o' },
	{ "trim-quality", required_argument, NULL, 'q' },
	{ "mask-quality", required_argument, NULL, 'Q' },
	{ "standard-quality", no_argument, &qualityOffset, 33 },
	{ "illumina-quality", no_argument, &qualityOffset, 64 },
	{ "qr-seed", required_argument, NULL, QR_SEED },
	{ "ref", required_argument, NULL, 'R' },
	{ "spaced-seed", required_argument, NULL, 's' },
	{ "trim-length", required_argument, NULL, 't' },
	{ "trace-file", required_argument, NULL, 'T' },
	{ "verbose", no_argument, NULL, 'v' },
	{ "version", no_argument, NULL, OPT_VERSION },
	{ "checkpoint", required_argument, NULL, CHECKPOINT },
	{ "keep-checkpoint", no_argument, NULL, KEEP_CHECKPOINT },
	{ "checkpoint-prefix", required_argument, NULL, CHECKPOINT_PREFIX },
	{ "read-log", required_argument, NULL, READ_LOG },
	{ "device", required_argument, NULL, OPT_DEVICE },
	{ "devices", required_argument, NULL, OPT_DEVICES },
	{ "batch-reads", required_argument, NULL, OPT_BATCH },
	{ NULL, 0, NULL, 0 }
};

static void check(int rc, const char* what)
{
	if (rc != ABB_OK) {
		std::cerr << PROGRAM ": " << what << ": " << abb_last_error() << "\n";
		exit(EXIT_FAILURE);
	}
}

/** printCountingBloomStats (bloom-dbg.cc:177-188) */
static void printCountingBloomStats(abb_filter* f, std::ostream& os)
{
	uint64_t nz = 0, th = 0;
	check(abb_filter_popcount(f, &nz, &th), "popcount");
	const double fpr = std::pow((double)th / (double)abb_filter_size(f), (double)abb_filter_hash_num(f));
	os << "Counting Bloom filter stats:"
	   << "\n\t#counters               = " << abb_filter_size(f)
	   << "\n\t#size (B)               = " << abb_filter_size_in_bytes(f)
	   << "\n\tthreshold               = " << abb_filter_threshold(f)
	   << "\n\tpopcount                = " << th
	   << "\n\tFPR                     = " << std::setprecision(3) << 100.f * fpr << "%"
	   << "\n";
}

/** batches of --batch-reads reads, parsed by background threads while the GPU works on the previous batch */
template <typename Fn>
static void for_each_batch(const std::vector<std::string>& files, Fn fn)
{
	// -j N (N > 1) sets the number of parsing threads; otherwise up to 8 of the host's cores
	host::BatchStream stream(files, ropt, params.batchReads, params.threads > 1 ? params.threads : 0, params.verbose != 0);
	while (const ReadBatch* batch = stream.next())
		fn(*batch);
}

/** --devices: "0-3", "0,2,5" or a mix */
static std::vector<int> parse_devices(const std::string& spec)
{
	std::vector<int> out;
	std::istringstream in(spec);
	std::string item;
	while (std::getline(in, item, ',')) {
		const size_t dash = item.find('-');
		const int a = atoi(item.substr(0, dash).c_str());
		const int b = dash == std::string::npos ? a : atoi(item.substr(dash + 1).c_str());
		for (int d = a; d <= b; ++d)
			out.push_back(d);
	}
	if (out.empty()) {
		std::cerr << PROGRAM ": invalid option: `--devices=" << spec << "'\n";
		exit(EXIT_FAILURE);
	}
	return out;
}

/** one host thread per GPU: run fn(rank) on every rank at once (the library's collectives meet inside) */
template <typename Fn>
static void on_all_ranks(size_t n, Fn fn)
{
	std::vector<std::thread> th;
	for (size_t r = 1; r < n; ++r)
		th.emplace_back([&fn, r] { fn(r); });
	fn((size_t)0);
	for (auto& t : th)
		t.join();
}

/** writeCovTrack (bloom-dbg.h:1280-1334): variableStep WIG blocks of equal 0/1 "k-mer is in the solid filter" values along every
 *  record of the reference; contains() of all k-mers of a batch of records is one GPU query (abb_contains_reads).  As in the
 *  reference, windows with a non-ACGT base are skipped by the iterator and simply do not interrupt a block. */
static void writeCovTrack(abb_filter* bloom)
{
	std::ofstream covTrack(params.covTrackPath.c_str());
	auto good = [&]() {
		if (!covTrack) {
			std::cerr << "error: `" << params.covTrackPath << "': " << strerror(errno) << "\n";
			exit(EXIT_FAILURE);
		}
	};
	good();
	if (params.verbose)
		std::cerr << "Writing 0/1 k-mer coverage track for `" << params.refPath << "` to `" << params.covTrackPath << "`\n";
	const unsigned k = abb_filter_kmer_size(bloom);
	SeqReader ref(params.refPath, ropt);
	ReadBatch b;
	std::vector<uint8_t> flag, valid;
	auto flush = [&]() {
		if (b.size() == 0)
			return;
		uint64_t slots = 0;
		for (size_t i = 0; i < b.size(); ++i) {
			const uint64_t len = b.offsets[i + 1] - b.offsets[i];
			slots += len >= k ? len - k + 1 : 0;
		}
		flag.resize(slots + 1);
		valid.resize(slots + 1);
		uint64_t n = 0;
		check(abb_contains_reads(bloom, b.bases.data(), b.offsets.data(), b.size(), flag.data(), valid.data(), slots + 1, &n), "coverage track");
		uint64_t s0 = 0;
		for (size_t i = 0; i < b.size(); ++i) {
			const uint64_t len = b.offsets[i + 1] - b.offsets[i];
			const uint64_t w = len >= k ? len - k + 1 : 0;
			const std::string chr = b.id(i);
			bool firstVal = true;
			uint64_t blockStart = 1, blockLength = 0;
			unsigned blockVal = 0;
			auto block = [&]() { // outputWigBlock (:1253-1266)
				covTrack << "variableStep chrom=" << chr << " span=" << blockLength << "\n" << blockStart << ' ' << blockVal << '\n';
				good();
			};
			for (uint64_t p = 0; p < w; ++p) {
				if (!valid[s0 + p])
					continue;
				const unsigned val = flag[s0 + p] ? 1 : 0;
				if (firstVal || val != blockVal) {
					if (!firstVal)
						block();
					firstVal = false;
					blockStart = p + 1; // WIG coordinates are 1-based
					blockLength = 1;
					blockVal = val;
				} else
					blockLength++;
			}
			if (blockLength > 0)
				block();
			s0 += w;
		}
		b.clear();
	};
	std::string id, seq;
	while (ref.next(id, seq)) {
		b.add(id, seq);
		if (b.bases.size() >= (256u << 20))
			flush();
	}
	flush();
	good();
	covTrack.close();
}

/** outputGraph (bloom-dbg.h:1171-1242) over the C ABI; the traversal itself is host/graph_dump.h */
static void outputGraph(const std::vector<std::string>& files, abb_filter* bloom, std::ostream& out)
{
	host::output_graph(
	    abb_filter_kmer_size(bloom), params.verbose, [&](auto fn) { for_each_batch(files, fn); },
	    [&](const char* bases, const uint64_t* offsets, uint64_t n, uint8_t* flag, uint8_t* valid, uint64_t cap) {
		    uint64_t slots = 0;
		    check(abb_contains_reads(bloom, bases, offsets, n, flag, valid, cap, &slots), "graph");
	    },
	    [&](const char* kmers, uint64_t n, unsigned max_chain, abb_succ_info* info, unsigned* len, uint64_t* self) {
		    check(abb_successors(bloom, kmers, n, max_chain, info, len, self), "graph");
	    },
	    out);
}

int main(int argc, char** argv)
{
	bool die = false;
	for (int c; (c = getopt_long(argc, argv, shortopts, longopts, NULL)) != -1;) {
		std::istringstream arg(optarg != NULL ? optarg : "");
		switch (c) {
		case '?': die = true; break;
		case 'b':
			if (!si_to_bytes(optarg, &params.bloomSize)) {
				std::cerr << PROGRAM ": invalid option: `-b" << optarg << "'\n";
				exit(EXIT_FAILURE);
			}
			arg.seekg(0, std::ios::end);
			arg.clear(std::ios::eofbit);
			break;
		case 'C': arg >> params.covTrackPath; break;
		case 'g': arg >> params.graphPath; break;
		case 'H': arg >> params.numHashes; break;
		case 'i': arg >> params.bloomPath; break;
		case 'j': arg >> params.threads; break;
		case 'k': arg >> params.k; break;
		case 'K': params.resetSpacedSeedParams(); arg >> params.K; break;
		case 'o': arg >> params.outputPath; break;
		case 'q': arg >> ropt.qualityThreshold; break;
		case 'R': arg >> params.refPath; break;
		case 's': params.resetSpacedSeedParams(); arg >> params.spacedSeed; break;
		case 't': arg >> params.trim; break;
		case 'T': arg >> params.tracePath; break;
		case 'Q': arg >> ropt.internalQThreshold; break;
		case 'v': ++params.verbose; break;
		case OPT_HELP: std::cout << USAGE_MESSAGE; exit(EXIT_SUCCESS);
		case MIN_KMER_COV: arg >> params.minCov; break;
		case OPT_VERSION: std::cout << VERSION_MESSAGE; exit(EXIT_SUCCESS);
		case QR_SEED: params.resetSpacedSeedParams(); arg >> params.qrSeedLen; break;
		case CHECKPOINT: arg >> params.readsPerCheckpoint; break;
		case KEEP_CHECKPOINT: params.keepCheckpoint = true; break;
		case CHECKPOINT_PREFIX: arg >> params.checkpointPathPrefix; break;
		case READ_LOG: arg >> params.readLogPath; break;
		case OPT_DEVICE: arg >> params.device; break;
		case OPT_DEVICES: arg >> params.devices; break;
		case OPT_BATCH: arg >> params.batchReads; break;
		}
		if (optarg != NULL && (!arg.eof() || arg.fail())) {
			std::cerr << PROGRAM ": invalid option: `-" << (char)c << optarg << "'\n";
			exit(EXIT_FAILURE);
		}
	}
	ropt.chastityFilter = chastity;
	ropt.trimMasked = trimMasked;
	ropt.qualityOffset = qualityOffset;

	if (params.bloomPath.empty() && params.bloomSize == 0) {
		std::cerr << PROGRAM ": missing mandatory option `-b'\n";
		die = true;
	}
	if (params.bloomPath.empty() && params.k == 0) {
		std::cerr << PROGRAM ": missing mandatory option `-k'\n";
		die = true;
	}
	if (params.k > 0 && params.K > 0 && params.K > params.k / 2) {
		std::cerr << PROGRAM ": value of `-K' must be <= k/2\n";
		die = true;
	}
	if (params.numHashes > MAX_HASHES) {
		std::cerr << PROGRAM ": number of hash functions (`-H`) must be <= " << MAX_HASHES << "\n";
		die = true;
	}
	if (params.k > MAX_KMER) {
		std::cerr << PROGRAM ": k-mer size (`-k`) must be <= " << MAX_KMER << "\n";
		die = true;
	}
	if (params.k > 0 && params.qrSeedLen > 0 && (params.qrSeedLen < 11 || params.qrSeedLen > params.k / 2)) {
		std::cerr << PROGRAM ": value of `--qr-seed' must be >= 11 and <= k/2\n";
		die = true;
	}
	if (!params.covTrackPath.empty() && params.refPath.empty()) {
		std::cerr << PROGRAM ": you must specify a reference with `-R' when using `-C'\n";
		die = true;
	}
	if (params.k > 0 && params.trim == UINT_MAX)
		params.trim = params.k;
	if (argc - optind < 1) {
		std::cerr << PROGRAM ": missing input file arguments\n";
		die = true;
	}
	if (die) {
		std::cerr << "Try `" << PROGRAM << " --help' for more information.\n";
		exit(EXIT_FAILURE);
	}
	if (!params.graphPath.empty() && (params.K > 0 || params.qrSeedLen > 0 || !params.spacedSeed.empty())) {
		std::cerr << PROGRAM ": -g is not supported together with a spaced seed by the GPU implementation\n";
		exit(EXIT_FAILURE);
	}
	/* initGlobals (bloom-dbg.cc:215-233) + MaskedKmer::setMask (BloomDBG/MaskedKmer.h:25-48), once k is known */
	auto spacedSeedMask = [&]() {
		std::string mask;
		const unsigned k = params.k;
		if (params.K > 0) { // SpacedSeed::kmerPair (BloomDBG/SpacedSeed.h:30-37)
			mask.assign(k, '0');
			std::fill(mask.begin(), mask.begin() + params.K, '1');
			std::fill(mask.rbegin(), mask.rbegin() + params.K, '1');
		} else if (params.qrSeedLen > 0) { // qrSeedPair (SpacedSeed.h:55-95): a quadratic-residue seed and its mirror image
			const unsigned len = params.qrSeedLen;
			std::string qr(len, '1');
			for (size_t i = 0; i < len; ++i)
				for (size_t j = 1; j < len; ++j)
					if (j * j % len == i) {
						qr[i] = '0';
						break;
					}
			mask.assign(k, '0');
			for (unsigned i = 0; i < len; ++i)
				mask[i] = mask[k - 1 - i] = qr[i];
		} else
			mask = params.spacedSeed;
		if (mask.empty())
			return mask;
		if (mask.size() != k) {
			std::cerr << "error: spaced seed must be exactly k bits long\n";
			exit(EXIT_FAILURE);
		} else if (mask.find_first_not_of("01") != std::string::npos) {
			std::cerr << "error: spaced seed must contain only '0's or '1's\n";
			exit(EXIT_FAILURE);
		} else if (mask.front() != '1' || mask.back() != '1') {
			std::cerr << "error: spaced seed must begin and end with '1's\n";
			exit(EXIT_FAILURE);
		}
		if (params.verbose)
			std::cerr << "Using spaced seed " << mask << "\n";
		return mask;
	};

	/* the `:' separator: files before it load the filter, files after it are assembled (BloomIO.h:104-113) */
	std::vector<std::string> loadFiles, asmFiles;
	{
		bool sep = false;
		std::vector<std::string> all(argv + optind, argv + argc);
		for (auto& a : all) {
			if (a == ":") {
				sep = true;
				continue;
			}
			(sep ? asmFiles : loadFiles).push_back(a);
		}
		if (!sep)
			asmFiles = loadFiles;
	}

	std::ofstream outputFile;
	if (!params.outputPath.empty()) {
		outputFile.open(params.outputPath.c_str());
		if (!outputFile) {
			std::cerr << "error: `" << params.outputPath << "': " << strerror(errno) << "\n";
			exit(EXIT_FAILURE);
		}
	}
	std::ostream& out = params.outputPath.empty() ? std::cout : outputFile;

	/* checkpoints (BloomDBG/Checkpoint.h): PREFIX.dbg.bloom, PREFIX.visited.bloom, PREFIX.counters.tsv, PREFIX.contigs.fa */
	const bool ckptOn = params.readsPerCheckpoint != UINT64_MAX && params.readsPerCheckpoint != 0;
	const std::string ckDbg = params.checkpointPathPrefix + ".dbg.bloom", ckVisited = params.checkpointPathPrefix + ".visited.bloom",
	                  ckCounters = params.checkpointPathPrefix + ".counters.tsv", ckFasta = params.checkpointPathPrefix + ".contigs.fa";
	auto readable = [](const std::string& p) { return std::ifstream(p.c_str()).good(); };
	const bool resume = ckptOn && readable(ckDbg) && readable(ckVisited) && readable(ckCounters) && readable(ckFasta); // checkpointExists
	if (resume) {
		if (params.verbose)
			std::cerr << "Resuming from last checkpoint...\n\tReading Bloom filter de Bruijn graph from `" << ckDbg << "'\n";
		params.bloomPath = ckDbg; // the solid filter comes from the checkpoint; pass 1 is skipped
	}
	if (ckptOn) { // batches must end on checkpoint boundaries: the largest divisor of N that is a reasonable batch
		uint64_t b = std::min<uint64_t>(params.readsPerCheckpoint, params.batchReads ? params.batchReads : 4000000);
		while (params.readsPerCheckpoint % b)
			--b;
		params.batchReads = b;
	}
	const std::vector<int> devs = params.devices.empty() ? std::vector<int>{ params.device } : parse_devices(params.devices);
	const size_t nd = devs.size();
	std::vector<abb_filter*> blooms(nd, nullptr);
	std::vector<abb_comm*> comms(nd, nullptr);
	if (nd > 1) { // the NCCL communicator of the sharded insert: rank r = r-th listed device
		uint8_t id[128];
		check(abb_comm_unique_id(id), "NCCL");
		on_all_ranks(nd, [&](size_t r) { check(abb_comm_create(&comms[r], (int)r, (int)nd, id, devs[r]), "NCCL communicator"); });
	}
	abb_filter*& bloom = blooms[0];
	if (!params.bloomPath.empty()) {
		/* prebuiltBloomAssembly (bloom-dbg.cc:301-345) */
		if (params.verbose)
			std::cerr << "Loading prebuilt Bloom filter from `" << params.bloomPath << "'\n";
		BloomHeader h;
		std::vector<uint8_t> raw;
		read_counting_bloom(params.bloomPath, h, raw);
		params.k = h.kmerSize;
		params.numHashes = h.hashNum;
		params.bloomSize = h.sizeInBytes;
		if (params.trim == UINT_MAX)
			params.trim = params.k;
		if (params.verbose)
			std::cerr << "Assembling with k-mer size " << params.k << "\n";
		const std::string mask = spacedSeedMask();
		on_all_ranks(nd, [&](size_t r) {
			check(abb_filter_create(&blooms[r], ABB_COUNTING, h.size, h.hashNum, h.kmerSize, params.minCov, mask.c_str(), devs[r]), "filter");
			check(abb_filter_upload(blooms[r], 0, raw.data(), raw.size()), "upload");
		});
		printCountingBloomStats(bloom, std::cerr);
	} else {
		/* countingBloomAssembly (bloom-dbg.cc:347-386) */
		if (params.verbose)
			std::cerr << "Assembling with k-mer size " << params.k << "\n";
		const double sz = (double)params.bloomSize / 1.125;
		uint64_t counters = (uint64_t)std::llround(sz);
		if (counters % 64)
			counters += 64 - counters % 64;
		const std::string mask = spacedSeedMask();
		on_all_ranks(nd, [&](size_t r) {
			check(abb_filter_create(&blooms[r], ABB_COUNTING, counters, params.numHashes, params.k, params.minCov, mask.c_str(), devs[r]), "filter");
		});
		uint64_t readCount = 0;
		for_each_batch(loadFiles, [&](const ReadBatch& b) {
			if (nd > 1) // every rank sees every batch and keeps the counters of its own position range (abb_shard.cuh)
				on_all_ranks(nd, [&](size_t r) {
					check(abb_insert_reads_sharded(blooms[r], comms[r], b.bases.data(), b.offsets.data(), b.size(), 0, nullptr), "insert");
				});
			else
				check(abb_insert_reads(bloom, b.bases.data(), b.offsets.data(), b.size(), nullptr), "insert");
			readCount += b.size();
			if (params.verbose)
				std::cerr << "Loaded " << readCount << " reads into Bloom filter\n";
		});
		if (nd > 1) // union of the shards: every GPU gets the whole filter for the extension stage
			on_all_ranks(nd, [&](size_t r) { check(abb_filter_allgather(blooms[r], comms[r]), "all-gather"); });
		if (params.verbose) {
			uint64_t nz = 0;
			check(abb_filter_popcount(bloom, &nz, nullptr), "popcount");
			std::cerr << "Bloom filter FPR: " << std::setprecision(3)
			          << 100 * std::pow((double)nz / (double)abb_filter_size(bloom), (double)params.numHashes) << "%\n";
			printCountingBloomStats(bloom, std::cerr);
		}
	}

	/* BloomDBG::assemble (bloom-dbg.h:900-1089) */
	if (params.verbose)
		std::cerr << "Trimming branches " << params.trim << " k-mers or shorter\n";
	abb_assembly_params ap = { params.trim, (unsigned)params.verbose, params.readLogPath.empty() ? 0u : 1u, params.tracePath.empty() ? 0u : 1u };
	std::vector<abb_assembler*> asms(nd, nullptr);
	on_all_ranks(nd, [&](size_t r) {
		check(abb_assembler_create(&asms[r], blooms[r], &ap), "assembler");
		if (nd > 1)
			check(abb_assembler_set_comm(asms[r], comms[r]), "assembler");
	});
	abb_assembler* as = asms[0];
	uint64_t contigID = 0, readBase = 0, skipReads = 0, sinceCheckpoint = 0;
	std::ofstream checkpointOut; // duplicate FASTA output (bloom-dbg.h:919-926)
	if (resume) { // resumeFromCheckpoint (Checkpoint.h:158-226)
		BloomHeader vh;
		std::vector<uint8_t> vraw;
		if (params.verbose)
			std::cerr << "\tReading reading visited k-mers Bloom from `" << ckVisited << "'\n";
		read_bit_bloom(ckVisited, vh, vraw);
		abb_assembly_counters cn = {};
		{
			std::ifstream cin_(ckCounters.c_str());
			std::string header;
			std::getline(cin_, header);
			unsigned long long a = 0, b = 0, c = 0, d = 0;
			cin_ >> a >> b >> c >> d;
			if (!cin_) {
				std::cerr << "error: `" << ckCounters << "': malformed counters\n";
				exit(EXIT_FAILURE);
			}
			cn.solid_reads = a;
			cn.reads_processed = b;
			cn.bases_assembled = c;
			cn.contig_id = d;
		}
		on_all_ranks(nd, [&](size_t r) {
			check(abb_filter_upload(abb_assembler_assembled_filter(asms[r]), 0, vraw.data(), vraw.size()), "visited filter");
			check(abb_assembler_set_counters(asms[r], &cn), "counters");
		});
		contigID = cn.contig_id;
		readBase = skipReads = cn.reads_processed;
		if (params.verbose)
			std::cerr << "\tAdvancing to read index " << cn.reads_processed << " in input reads...\n\tOutputting previously assembled contigs from `"
			          << ckFasta << "'\n";
		std::ifstream prev(ckFasta.c_str());
		out << prev.rdbuf();
		std::ifstream prev2(ckFasta.c_str());
		checkpointOut.open((ckFasta + ".tmp").c_str());
		checkpointOut << prev2.rdbuf();
	} else if (ckptOn)
		checkpointOut.open((ckFasta + ".tmp").c_str());
	bool dbgWritten = resume;
	auto createCheckpoint = [&]() { // createCheckpoint (Checkpoint.h:31-127); the solid filter does not change during pass 2
		checkpointOut.flush();
		if (params.verbose)
			std::cerr << "Writing checkpoint data...\n";
		if (!dbgWritten) {
			BloomHeader h;
			h.size = abb_filter_size(bloom);
			h.sizeInBytes = abb_filter_size_in_bytes(bloom);
			h.hashNum = abb_filter_hash_num(bloom);
			h.kmerSize = abb_filter_kmer_size(bloom);
			std::vector<uint8_t> raw(h.sizeInBytes);
			check(abb_filter_download(bloom, 0, raw.data(), raw.size()), "download");
			std::ofstream o((ckDbg + ".tmp").c_str(), std::ios::binary);
			write_counting_bloom(o, h, raw);
			o.close();
			rename((ckDbg + ".tmp").c_str(), ckDbg.c_str());
			dbgWritten = true;
		}
		{
			abb_filter* vis = abb_assembler_assembled_filter(as);
			std::vector<uint8_t> raw(abb_filter_size_in_bytes(vis));
			check(abb_filter_download(vis, 0, raw.data(), raw.size()), "download");
			std::ofstream o((ckVisited + ".tmp").c_str(), std::ios::binary);
			write_bit_bloom(o, abb_filter_size(vis), abb_filter_hash_num(vis), abb_filter_kmer_size(vis), raw);
			o.close();
		}
		{
			abb_assembly_counters cn;
			abb_assembler_counters(as, &cn);
			std::ofstream o((ckCounters + ".tmp").c_str());
			o << "solid_reads\tprocessed_reads\tbases_assembled\tnext_contig_id\n"
			  << cn.solid_reads << '\t' << cn.reads_processed << '\t' << cn.bases_assembled << '\t' << cn.contig_id << '\n';
		}
		{
			std::ifstream src((ckFasta + ".tmp").c_str(), std::ios::binary);
			std::ofstream dst(ckFasta.c_str(), std::ios::binary);
			dst << src.rdbuf();
		}
		rename((ckVisited + ".tmp").c_str(), ckVisited.c_str());
		rename((ckCounters + ".tmp").c_str(), ckCounters.c_str());
	};
	std::ofstream readLog;
	static const char* names[] = { "SHORTER_THAN_K", "NON_ACGT", "BLUNT_END", "NOT_SOLID", "ALL_KMERS_VISITED", "GENERATED_CONTIGS", "NA" };
	if (!params.readLogPath.empty()) {
		readLog.open(params.readLogPath.c_str());
		readLog << "read_id\tresult\n";
	}
	/* -T FILE: ContigRecord::printHeaders / operator<< (bloom-dbg.h:219-253) */
	std::ofstream traceOut;
	static const char* extNames[] = { "AMBI_IN", "AMBI_OUT", "DEAD_END", "CYCLE", "LENGTH_LIMIT" };
	if (!params.tracePath.empty()) {
		traceOut.open(params.tracePath.c_str());
		if (!traceOut) {
			std::cerr << "error: `" << params.tracePath << "': " << strerror(errno) << "\n";
			exit(EXIT_FAILURE);
		}
		traceOut << "contig_id\tlength\tredundant\tread_id\tleft_result\tleft_extension\tright_result\tright_extension\tseed_type\tseed_length\tseed\n";
	}
	for_each_batch(asmFiles, [&](const ReadBatch& b) {
		if (skipReads) { // resumed: these reads were processed before the checkpoint
			skipReads -= std::min<uint64_t>(skipReads, b.size());
			return;
		}
		const abb_contig* contigs = nullptr;
		uint64_t n = 0;
		const char* seqs = nullptr;
		if (nd > 1) // every rank runs the batch (sharded stages meet inside the library); rank 0's unitigs are printed
			on_all_ranks(nd, [&](size_t r) {
				if (r)
					check(abb_assembler_process_reads(asms[r], b.bases.data(), b.offsets.data(), b.size(), nullptr, nullptr, nullptr), "assemble");
				else
					check(abb_assembler_process_reads(as, b.bases.data(), b.offsets.data(), b.size(), &contigs, &n, &seqs), "assemble");
			});
		else
			check(abb_assembler_process_reads(as, b.bases.data(), b.offsets.data(), b.size(), &contigs, &n, &seqs), "assemble");
		for (uint64_t i = 0; i < n; ++i) {
			const abb_contig& c = contigs[i];
			/* printContig (bloom-dbg.h:455-487) */
			out << '>' << contigID << ' ' << c.length << ' ' << c.coverage << " read:" << b.id(c.seed_read - readBase) << '\n';
			out.write(seqs + c.seq_offset, c.length);
			out << '\n';
			if (checkpointOut.is_open()) {
				checkpointOut << '>' << contigID << ' ' << c.length << ' ' << c.coverage << " read:" << b.id(c.seed_read - readBase) << '\n';
				checkpointOut.write(seqs + c.seq_offset, c.length);
				checkpointOut << '\n';
			}
			++contigID;
		}
		if (traceOut.is_open()) {
			const abb_trace_row* rows = nullptr;
			uint64_t nr = 0;
			check(abb_assembler_trace(as, &rows, &nr), "trace");
			for (uint64_t i = 0; i < nr; ++i) {
				const abb_trace_row& t = rows[i];
				const uint64_t r = t.seed_read - readBase;
				if (t.redundant)
					traceOut << "NA\t";
				else
					traceOut << t.contig_id << '\t';
				traceOut << t.length << '\t' << (int)t.redundant << '\t' << b.id(r) << '\t';
				if (t.left_n > 0)
					traceOut << extNames[t.left_code > 4 ? 4 : t.left_code] << '\t' << t.left_n << '\t';
				else
					traceOut << "NA\tNA\t";
				if (t.right_n > 0)
					traceOut << extNames[t.right_code > 4 ? 4 : t.right_code] << '\t' << t.right_n << '\t';
				else
					traceOut << "NA\tNA\t";
				traceOut << "READ\t" << params.k << '\t';
				traceOut.write(b.bases.data() + b.offsets[r] + t.seed_pos, params.k);
				traceOut << '\n';
			}
		}
		if (readLog.is_open()) {
			const uint8_t* codes = nullptr;
			uint64_t nc = 0;
			check(abb_assembler_read_results(as, &codes, &nc), "read results");
			for (uint64_t i = 0; i < nc; ++i)
				readLog << b.id(i) << '\t' << names[codes[i] > 6 ? 6 : codes[i]] << '\n';
		}
		readBase += b.size();
		sinceCheckpoint += b.size();
		if (ckptOn && sinceCheckpoint == params.readsPerCheckpoint) {
			createCheckpoint();
			sinceCheckpoint = 0;
		}
		if (params.verbose) {
			abb_assembly_counters cn;
			abb_assembler_counters(as, &cn);
			std::cerr << "Processed " << cn.reads_processed << " reads, solid reads: " << cn.solid_reads
			          << ", visited reads: " << cn.visited_reads << "\nAssembled " << cn.bases_assembled << " bp in "
			          << cn.contig_id << " contigs\n";
		}
	});
	if (params.verbose)
		std::cerr << "Assembly complete\n";
	/* writeAuxiliaryFiles (bloom-dbg.cc:190-212) */
	if (!params.covTrackPath.empty() && !params.refPath.empty())
		writeCovTrack(bloom);
	if (!params.graphPath.empty()) {
		std::ofstream graphOut(params.graphPath.c_str());
		auto good = [&]() {
			if (!graphOut) {
				std::cerr << "error: `" << params.graphPath << "': " << strerror(errno) << "\n";
				exit(EXIT_FAILURE);
			}
		};
		good();
		std::vector<std::string> all = loadFiles; // outputGraph reads every file argument (bloom-dbg.cc:204-211)
		if (asmFiles != loadFiles)
			all.insert(all.end(), asmFiles.begin(), asmFiles.end());
		outputGraph(all, bloom, graphOut);
		good();
		graphOut.close();
		good();
	}
	if (ckptOn && !params.keepCheckpoint) { // removeCheckpointData (Checkpoint.h:229-247)
		checkpointOut.close();
		for (const std::string& f : { ckDbg, ckVisited, ckCounters, ckFasta, ckFasta + ".tmp" })
			remove(f.c_str());
	}
	for (size_t r = 0; r < nd; ++r) {
		abb_assembler_destroy(asms[r]);
		abb_filter_destroy(blooms[r]);
		abb_comm_destroy(comms[r]);
	}
	if (!params.outputPath.empty())
		outputFile.close();
	return EXIT_SUCCESS;
}
