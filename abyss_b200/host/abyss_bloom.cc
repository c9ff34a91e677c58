// abyss-bloom (GPU) -- the reference's abyss-bloom (Bloom/bloom.cc) over libabyssb200:
//   build -t konnector (default; CityHash, -l levels, -L N=FILE, -w M/N windows, -h seed), -t counting
//     (CountingBloomFilter<uint8_t>, the filter abyss-bloom-dbg loads with -i) and -t rolling-hash [-l LEVELS]
//     (HashAgnosticCascadingBloom, last level serialised);
//   union, intersect, info, compare, kmers (getKmers), trim on Konnector files, info on the two BTL formats, and graph on
//   rolling-hash (BTL bit) files.
// Output files and printed text are byte-compatible with the reference's.
//
//   abyss-bloom build [-v] -k K [-b SIZE] [-h SEED] [-l LEVELS] [-L N=FILE] [-w M/N] [-t konnector|counting|rolling-hash] OUT.bloom READS...
//   abyss-bloom union|intersect -k K OUT.bloom IN.bloom IN.bloom...
//   abyss-bloom info [-k K] IN.bloom
//   abyss-bloom compare -k K [-m jaccard|forbes|czekanowski] A.bloom B.bloom    (exits with status 1, as the reference does)
//   abyss-bloom kmers -k K [-r] [--fasta|--bed|--raw] IN.bloom READS
//   abyss-bloom trim [-v...] -k K [-q N] IN.bloom READS... > trimmed.fq
//   abyss-bloom graph [-v] -k K [-d N] (-R KMER | -f FASTA)... [-a ATTR:FASTA]... [-A ATTR:BLOOM]... IN.bloom > graph.dot
#include "../../include/abyss_b200.h"
#include "bloom_file.h"
#include "bloom_graph.h"
#include "max_kmer.h"
#include "reads.h"
#include "trim.h"
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
	std::cerr << "Try `" PROGRAM " --help' for more information.\n";
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

// ---- Konnector filters (Bloom/bloom.cc:520-581, 766-977, 1155-1231) --------------------------------------------------------

enum { FMT_BED, FMT_FASTA, FMT_RAW };
enum { OPT_HELP = 1, OPT_VERSION, OPT_BED, OPT_FASTA, OPT_RAW, OPT_DEVICE = 1000, OPT_BATCH_READS };
static int g_chastity = 1, g_trimMasked = 1, g_qualityOffset = 0; // 0 = the format's own offset
/** the reference's option table (bloom.cc:242-287) plus --device and --batch-reads */
static const char kShortOpts[] = "a:A:b:B:d:f:h:H:j:k:l:L:m:n:q:rR:vt:w:";
static const struct option kLongOpts[] = {
	{ "bloom-size", required_argument, NULL, 'b' }, { "bloom-type", required_argument, NULL, 't' },
	{ "buffer-size", required_argument, NULL, 'B' }, { "depth", required_argument, NULL, 'd' },
	{ "hash-seed", required_argument, NULL, 'h' }, { "num-hashes", required_argument, NULL, 'H' },
	{ "threads", required_argument, NULL, 'j' }, { "kmer", required_argument, NULL, 'k' },
	{ "levels", required_argument, NULL, 'l' }, { "init-level", required_argument, NULL, 'L' },
	{ "chastity", no_argument, &g_chastity, 1 }, { "no-chastity", no_argument, &g_chastity, 0 },
	{ "trim-masked", no_argument, &g_trimMasked, 1 }, { "no-trim-masked", no_argument, &g_trimMasked, 0 },
	{ "num-locks", required_argument, NULL, 'n' }, { "trim-quality", required_argument, NULL, 'q' },
	{ "standard-quality", no_argument, &g_qualityOffset, 33 }, { "illumina-quality", no_argument, &g_qualityOffset, 64 },
	{ "fasta-attr", required_argument, NULL, 'a' }, { "node-attr", required_argument, NULL, 'a' },
	{ "bloom-attr", required_argument, NULL, 'A' }, { "verbose", no_argument, NULL, 'v' },
	{ "help", no_argument, NULL, OPT_HELP }, { "version", no_argument, NULL, OPT_VERSION },
	{ "window", required_argument, NULL, 'w' }, { "method", required_argument, NULL, 'm' },
	{ "inverse", required_argument, NULL, 'r' }, { "root", required_argument, NULL, 'R' },
	{ "root-fasta", required_argument, NULL, 'f' }, { "bed", no_argument, NULL, OPT_BED },
	{ "fasta", no_argument, NULL, OPT_FASTA }, { "raw", no_argument, NULL, OPT_RAW },
	{ "device", required_argument, NULL, OPT_DEVICE }, { "batch-reads", required_argument, NULL, OPT_BATCH_READS },
	{ NULL, 0, NULL, 0 }
};

/** `arg >> value` with the reference's check (bloom.cc:330-333): the whole argument must be one number */
template <typename T>
static T parse_num(int c, const char* optarg)
{
	std::istringstream arg(optarg);
	T v = 0;
	arg >> v;
	if (!arg.eof() || arg.fail()) {
		std::cerr << PROGRAM ": invalid option: `-" << (char)c << optarg << "'\n";
		exit(EXIT_FAILURE);
	}
	return v;
}

/** the options of union / intersect / info / compare / kmers / trim */
struct KonOpts {
	unsigned k = 0;
	int verbose = 0, device = 0, format = FMT_FASTA, qualityThreshold = 0;
	bool inverse = false;
	std::string method = "jaccard";
	uint64_t batchReads = 4000000;
};

static KonOpts parse_kon_opts(int argc, char** argv, const std::string& cmd)
{
	KonOpts o;
	optind = 2;
	for (int c; (c = getopt_long(argc, argv, kShortOpts, kLongOpts, NULL)) != -1;) {
		switch (c) {
		case '?': usage(); break;
		case 'k': o.k = parse_num<unsigned>(c, optarg); break;
		case 'v': ++o.verbose; break;
		case 'q': o.qualityThreshold = atoi(optarg); break;
		case 'm':
			if (cmd == "compare") {
				o.method = optarg;
				if (o.method != "jaccard" && o.method != "czekanowski" && o.method != "forbes")
					std::cerr << "Invalid method: " << o.method << std::endl;
			}
			break;
		case 'r':
			// `--inverse' takes an argument that nothing reads, so the reference refuses it (bloom.cc:1168-1185)
			if (optarg) {
				std::cerr << PROGRAM ": invalid option: `-r" << optarg << "'\n";
				exit(EXIT_FAILURE);
			}
			o.inverse = true;
			break;
		case OPT_BED: o.format = FMT_BED; break;
		case OPT_FASTA: o.format = FMT_FASTA; break;
		case OPT_RAW: o.format = FMT_RAW; break;
		case OPT_DEVICE: o.device = atoi(optarg); break;
		case OPT_BATCH_READS: o.batchReads = strtoull(optarg, nullptr, 10); break;
		case OPT_HELP: case OPT_VERSION:
			std::cerr << PROGRAM ": see the reference's abyss-bloom --help\n";
			exit(EXIT_SUCCESS);
		default: break;
		}
	}
	if (o.k == 0) {
		std::cerr << PROGRAM ": missing mandatory option `-k'\n";
		usage();
	}
	return o;
}

static void check_alloc(int rc, const char* what)
{
	if (rc == ABB_ENOMEM) {
		std::cerr << PROGRAM ": " << what << ": " << abb_last_error()
		          << "\n" PROGRAM ": the filter does not fit in device memory: build it in windows (-w M/N) and join them with `union'\n";
		exit(EXIT_FAILURE);
	}
	check(rc, what);
}

/** Konnector::BloomFilter of the file's full size, the file's bits read in at its start bit (BloomFilter::read,
 *  Bloom/BloomFilter.h:111-139) */
static abb_filter* load_konnector(const std::string& path, unsigned k, int device, KonnectorHeader* hout = nullptr)
{
	std::vector<uint8_t> raw;
	const KonnectorHeader h = read_konnector_bloom(path, k, raw);
	abb_filter* f = nullptr;
	check_alloc(abb_konnector_create(&f, h.full, h.k, 1, h.seed, 0, h.full - 1, device), "filter");
	check(abb_filter_read_bits(f, 0, raw.data(), h.bits(), h.start, 0), "readBits");
	if (hout)
		*hout = h;
	return f;
}

/** printBloomStats (bloom.cc:434-441); the precision stays set on the stream, as in the reference */
static void print_bloom_stats(uint64_t size, uint64_t pop, const char* indent = "")
{
	std::cerr << indent << "Bloom size (bits): " << size << "\n"
	          << indent << "Bloom popcount (bits): " << pop << "\n"
	          << indent << "Bloom filter FPR: " << std::setprecision(3) << 100 * ((double)pop / (double)size) << "%\n";
}

static void write_konnector(const std::string& path, const KonnectorHeader& h, const std::vector<uint8_t>& raw)
{
	std::ofstream out(path, std::ios::binary);
	if (!out) {
		std::cerr << "error: `" << path << "': " << strerror(errno) << "\n";
		exit(EXIT_FAILURE);
	}
	write_konnector_bloom(out, h, raw.data());
	out.flush();
	if (!out) {
		std::cerr << "error: `" << path << "': " << strerror(errno) << "\n";
		exit(EXIT_FAILURE);
	}
}

/** buildKonnectorBloom (bloom.cc:520-581): `bits` = -b * 8 */
static int build_konnector(uint64_t bits, unsigned k, unsigned levels, uint64_t seed, unsigned windowIndex, unsigned windows,
                           const std::vector<std::vector<std::string>>& levelInitPaths, const std::string& outputPath,
                           const std::vector<std::string>& files, const ReadOpts& ropt, uint64_t batchReads, int verbose, int device)
{
	bits /= levels;
	KonnectorHeader h;
	h.k = k;
	h.full = bits;
	h.seed = seed;
	h.start = 0;
	h.end = bits - 1;
	if (windows != 0) {
		const uint64_t perWindow = bits / windows;
		h.start = (uint64_t)(windowIndex - 1) * perWindow;
		h.end = windowIndex < windows ? (uint64_t)windowIndex * perWindow - 1 : bits - 1;
	}
	abb_filter* f = nullptr;
	check_alloc(abb_konnector_create(&f, h.full, k, levels, seed, h.start, h.end, device), "filter");
	// -L N=FILE (initBloomFilterLevels, bloom.cc:382-403): the first file of a level overwrites it, later ones are ORed in.
	// Reading a file over a level adopts the file's seed for that level (BloomFilter::read, Bloom/BloomFilter.h:116-124), so
	// a file loaded into the last level sets the seed the output header carries.  The reference resizes a level to a file of
	// another size; a level of another size has no place in the cascade, so such a file is refused here.
	for (size_t i = 0; i < levelInitPaths.size(); ++i) {
		uint64_t levelSeed = seed;
		for (size_t j = 0; j < levelInitPaths[i].size(); ++j) {
			const std::string& path = levelInitPaths[i][j];
			std::cerr << "Loading `" << path << "' into level " << i + 1 << " of cascading bloom filter...\n";
			std::vector<uint8_t> raw;
			const KonnectorHeader lh = read_konnector_bloom(path, k, raw);
			if (lh.seed != levelSeed) {
				if (j == 0)
					levelSeed = lh.seed;
				else {
					std::cerr << "error: can't union/intersect bloom filters with different hash seed" << (windows ? " values" : "s") << "\n";
					exit(EXIT_FAILURE);
				}
			}
			// a level of a full filter takes the file at its start bit; a level of a window takes it at bit 0
			const bool fits = windows ? lh.full == h.full && lh.start == h.start && lh.end == h.end : lh.full == h.full;
			if (!fits) {
				std::cerr << PROGRAM ": `" << path << "' does not have the size of level " << i + 1 << "\n";
				exit(EXIT_FAILURE);
			}
			check(abb_filter_read_bits(f, (int)i, raw.data(), lh.bits(), windows ? 0 : lh.start, j > 0 ? 1 : 0), "readBits");
		}
		if (i + 1 == levels && !levelInitPaths[i].empty())
			h.seed = levelSeed;
	}
	for (const std::string& path : files) { // Bloom::loadFile (Bloom/Bloom.h:76-118), one file after the other
		if (verbose)
			std::cerr << "Reading `" << path << "'...\n";
		uint64_t count = 0;
		host::BatchStream stream({ path }, ropt, batchReads, 0, false);
		while (const ReadBatch* batch = stream.next()) {
			check(abb_insert_reads(f, batch->bases.data(), batch->offsets.data(), batch->size(), nullptr), "insert");
			for (uint64_t c = count / 100000 + 1; verbose && c <= (count + batch->size()) / 100000; ++c)
				std::cerr << "Loaded " << c * 100000 << " reads into bloom filter\n";
			count += batch->size();
		}
		if (verbose)
			std::cerr << "Loaded " << count << " reads from `" << path << "` into bloom filter\n";
	}
	if (verbose)
		std::cerr << "Successfully loaded bloom filter.\n";
	if (levels == 1) {
		uint64_t pop = 0;
		check(abb_filter_level_popcount(f, 0, &pop), "popcount");
		print_bloom_stats(h.bits(), pop);
	} else
		for (unsigned l = 0; l < levels; ++l) { // printCascadingBloomStats (bloom.cc:443-454)
			uint64_t pop = 0;
			check(abb_filter_level_popcount(f, (int)l, &pop), "popcount");
			std::cerr << "Stats for Bloom filter level " << l + 1 << ":\n";
			print_bloom_stats(h.bits(), pop, "\t");
		}
	if (verbose)
		std::cerr << "Writing bloom filter to `" << outputPath << "'...\n";
	std::vector<uint8_t> raw(abb_filter_size_in_bytes(f));
	check(abb_filter_download(f, -1, raw.data(), raw.size()), "download");
	abb_filter_destroy(f);
	write_konnector(outputPath, h, raw);
	return EXIT_SUCCESS;
}

/** union / intersect (combine, bloom.cc:766-820): the first file overwrites, the others are ORed / ANDed in at their start bit */
static int combine(int argc, char** argv, int op)
{
	const KonOpts o = parse_kon_opts(argc, argv, argv[1]);
	if (argc - optind < 3) {
		std::cerr << PROGRAM ": missing arguments\n";
		usage();
	}
	const std::string outputPath = argv[optind++];
	abb_filter* f = nullptr;
	KonnectorHeader out;
	for (int i = optind; i < argc; ++i) {
		const std::string path = argv[i];
		if (o.verbose)
			std::cerr << "Loading bloom filter from `" << path << "'...\n";
		std::vector<uint8_t> raw;
		const KonnectorHeader h = read_konnector_bloom(path, o.k, raw);
		if (i == optind) {
			out = h;
			out.start = 0;
			out.end = h.full - 1;
			check_alloc(abb_konnector_create(&f, h.full, h.k, 1, h.seed, 0, h.full - 1, o.device), "filter");
		} else if (h.seed != out.seed) {
			std::cerr << "error: can't union/intersect bloom filters with different hash seeds\n";
			exit(EXIT_FAILURE);
		} else if (h.full != out.full) {
			std::cerr << "error: can't union/intersect bloom filters with different sizes\n";
			exit(EXIT_FAILURE);
		}
		check(abb_filter_read_bits(f, 0, raw.data(), h.bits(), h.start, i == optind ? 0 : op), "readBits");
	}
	if (o.verbose) {
		std::cerr << "Successfully loaded bloom filter.\n";
		uint64_t pop = 0;
		check(abb_filter_level_popcount(f, 0, &pop), "popcount");
		print_bloom_stats(out.full, pop);
		std::cerr << (op == 1 ? "Writing union of bloom filters to `" : "Writing intersection of bloom filters to `") << outputPath << "'...\n";
	}
	std::vector<uint8_t> raw(abb_filter_size_in_bytes(f));
	check(abb_filter_download(f, -1, raw.data(), raw.size()), "download");
	abb_filter_destroy(f);
	write_konnector(outputPath, out, raw);
	return EXIT_SUCCESS;
}

/** info on a Konnector file (bloom.cc:822-847): the full size, its popcount and FPR = popcount / size */
static int info_konnector(int argc, char** argv)
{
	const KonOpts o = parse_kon_opts(argc, argv, "info");
	if (argc - optind < 1) {
		std::cerr << PROGRAM ": missing arguments\n";
		usage();
	}
	const std::string path = argv[optind];
	if (o.verbose)
		std::cerr << "Loading bloom filter from `" << path << "'...\n";
	KonnectorHeader h;
	abb_filter* f = load_konnector(path, o.k, o.device, &h);
	uint64_t pop = 0;
	check(abb_filter_level_popcount(f, 0, &pop), "popcount");
	print_bloom_stats(h.full, pop);
	abb_filter_destroy(f);
	return EXIT_SUCCESS;
}

/** compare (bloom.cc:849-977).  Counts exactly the bits of the two files; the reference counts whole 32 KiB buffers, so the
 *  two agree when the byte count of the files is a multiple of 32768.  Exits with status 1 on success, as the reference. */
static int compare(int argc, char** argv)
{
	const KonOpts o = parse_kon_opts(argc, argv, "compare");
	if (argc - optind < 2) {
		std::cerr << PROGRAM ": missing arguments\n";
		usage();
	}
	const std::string pathA = argv[optind], pathB = argv[optind + 1];
	if (o.verbose)
		std::cerr << "Computing distance for 2 samples...\n"
		          << "Loading bloom filters from " << pathA << " and " << pathB << "...\n";
	std::vector<uint8_t> rawA, rawB;
	const KonnectorHeader hA = read_konnector_bloom(pathA, o.k, rawA);
	const KonnectorHeader hB = read_konnector_bloom(pathB, o.k, rawB);
	if (hA.bits() != hB.bits()) {
		std::cerr << "Bit sizes of arrays not equal" << std::endl;
		exit(EXIT_FAILURE);
	}
	if (o.verbose)
		std::cerr << "Bits: " << hA.bits() << std::endl;
	abb_filter *fa = nullptr, *fb = nullptr;
	check_alloc(abb_konnector_create(&fa, hA.bits() < 2 ? 2 : hA.bits(), o.k, 1, 0, 0, hA.bits() - 1, o.device), "filter");
	check_alloc(abb_konnector_create(&fb, hB.bits() < 2 ? 2 : hB.bits(), o.k, 1, 0, 0, hB.bits() - 1, o.device), "filter");
	check(abb_filter_read_bits(fa, 0, rawA.data(), hA.bits(), 0, 0), "readBits");
	check(abb_filter_read_bits(fb, 0, rawB.data(), hB.bits(), 0, 0), "readBits");
	uint64_t n[4];
	check(abb_filter_compare(fa, fb, n), "compare");
	abb_filter_destroy(fa);
	abb_filter_destroy(fb);
	// the reference's types: unsigned long counts, float similarities
	const unsigned long a = n[0], b = n[1], c = n[2], d = n[3];
	std::cout << "1/1: " << a << "\n1/0: " << b << "\n0/1: " << c << "\n0/0: " << d << std::endl;
	if (o.method == "jaccard") {
		float Dist = (float)a / (float)(a + b + c);
		std::cout << "Jaccard similarity: " << Dist << std::endl;
	}
	if (o.method == "czekanowski") {
		float Dist = (2 * (float)a) / (float)((2 * a) + b + c);
		std::cout << "Czekanowski similarity: " << Dist << std::endl;
	}
	if (o.method == "forbes") {
		float nn = (float)(a + b + c + d);
		float Dist = (nn * a - ((a + b) * (a + c))) / (nn * std::min(a + b, a + c) - ((a + b) * (a + c)));
		std::cout << "Forbes similarity: " << Dist << std::endl;
	}
	return 1;
}

/** kmers / getKmers (memberOf, bloom.cc:1155-1231): every k-mer without a non-ACGT base whose membership differs from -r */
static int kmers(int argc, char** argv)
{
	const KonOpts o = parse_kon_opts(argc, argv, "kmers");
	if (argc - optind < 2) {
		std::cerr << PROGRAM ": missing arguments\n";
		usage();
	}
	const std::string path = argv[optind], fasta = argv[optind + 1];
	if (o.verbose)
		std::cerr << "Loading bloom filter from `" << path << "'...\n";
	abb_filter* f = load_konnector(path, o.k, o.device);
	if (o.verbose)
		std::cerr << "Reading `" << fasta << "'...\n";
	const unsigned k = o.k;
	ReadOpts ropt;
	ropt.chastityFilter = g_chastity;
	ropt.trimMasked = g_trimMasked;
	ropt.qualityOffset = g_qualityOffset;
	std::vector<uint8_t> flag, valid;
	std::string buf;
	uint64_t seqCount = 0;
	host::BatchStream stream({ fasta }, ropt, o.batchReads, 0, false);
	while (const ReadBatch* batch = stream.next()) {
		uint64_t slots = 0;
		for (size_t r = 0; r < batch->size(); ++r) {
			const uint64_t len = batch->offsets[r + 1] - batch->offsets[r];
			slots += len >= k ? len - k + 1 : 0;
		}
		flag.resize(slots);
		valid.resize(slots);
		check(abb_contains_reads(f, batch->bases.data(), batch->offsets.data(), batch->size(), flag.data(), valid.data(), slots, &slots),
		      "kmers");
		uint64_t slot = 0;
		for (size_t r = 0; r < batch->size(); ++r, ++seqCount) {
			const uint64_t len = batch->offsets[r + 1] - batch->offsets[r];
			const char* seq = batch->bases.data() + batch->offsets[r];
			const std::string id = batch->id(r);
			for (uint64_t i = 0; len >= k && i + k <= len; ++i, ++slot) {
				if (!valid[slot] || (flag[slot] != 0) == o.inverse)
					continue;
				if (o.format == FMT_FASTA)
					buf += ">" + id + ":seq:" + std::to_string(seqCount) + ":kmer:" + std::to_string(i) + "\n";
				else if (o.format == FMT_BED)
					buf += id + "\t" + std::to_string(i) + "\t" + std::to_string(i + k - 1) + "\t";
				for (unsigned j = 0; j < k; ++j)
					buf += (char)toupper((unsigned char)seq[i + j]);
				buf += '\n';
			}
			if (o.verbose && len >= k && seqCount % 1000 == 0) // memberOf prints before counting the record, not for short ones
				std::cerr << "processed " << seqCount << " sequences" << std::endl;
			if (buf.size() > (8u << 20)) {
				fwrite(buf.data(), 1, buf.size(), stdout);
				buf.clear();
			}
		}
	}
	fwrite(buf.data(), 1, buf.size(), stdout);
	fflush(stdout);
	if (o.verbose)
		std::cerr << "processed " << seqCount << " sequences" << std::endl;
	abb_filter_destroy(f);
	return EXIT_SUCCESS;
}

/** trim (bloom.cc:1292-1382): cut the read ends that are tips of the filter's de Bruijn graph; the scans run on the GPU
 *  (abb_trim_reads), the records are written in file order */
static int trim(int argc, char** argv)
{
	const KonOpts o = parse_kon_opts(argc, argv, "trim");
	if (argc - optind < 2) {
		std::cerr << PROGRAM ": missing arguments\n";
		usage();
	}
	if (o.k < 2) { // the reference's k - 2 wraps
		std::cerr << PROGRAM ": trim needs k >= 2\n";
		exit(EXIT_FAILURE);
	}
	const std::string path = argv[optind++];
	if (o.verbose)
		std::cerr << "Loading bloom filter from `" << path << "'...\n";
	KonnectorHeader h;
	abb_filter* f = load_konnector(path, o.k, o.device, &h);
	uint64_t pop = 0;
	check(abb_filter_level_popcount(f, 0, &pop), "popcount");
	if (o.verbose)
		print_bloom_stats(h.full, pop);
	uint64_t minBranchLen = 0;
	if (!trim_min_branch_len(pop, h.full, &minBranchLen) || minBranchLen > 0xffffffffULL) {
		// FPR = 1: the reference divides by log(1) = 0 and converts the infinity to size_t, which is undefined
		std::cerr << PROGRAM ": every bit of `" << path << "' is set: there is no branch length threshold for such a filter\n";
		exit(EXIT_FAILURE);
	}
	if (o.verbose >= 2)
		std::cerr << "min length threshold for true branches (k-mers): " << minBranchLen << std::endl;
	ReadOpts ropt;
	ropt.chastityFilter = g_chastity;
	ropt.trimMasked = g_trimMasked;
	ropt.qualityOffset = g_qualityOffset;
	ropt.qualityThreshold = o.qualityThreshold;
	ropt.keepText = true;
	std::vector<uint32_t> left, right;
	std::string buf;
	uint64_t readCount = 0;
	for (int i = optind; i < argc; ++i) {
		if (o.verbose)
			std::cerr << "Reading `" << argv[i] << "'..." << std::endl;
		host::BatchStream stream({ argv[i] }, ropt, o.batchReads, 0, false);
		while (const ReadBatch* batch = stream.next()) {
			left.resize(batch->size());
			right.resize(batch->size());
			const int rc = abb_trim_reads(f, batch->bases.data(), batch->offsets.data(), batch->size(), (unsigned)minBranchLen, left.data(), right.data());
			if (rc != ABB_OK) {
				std::cerr << PROGRAM ": trim: `" << argv[i] << "', batch starting at read " << readCount << ": " << abb_last_error() << "\n";
				exit(EXIT_FAILURE);
			}
			for (size_t r = 0; r < batch->size(); ++r, ++readCount) {
				const uint64_t b0 = batch->offsets[r], len = batch->offsets[r + 1] - b0;
				// the progress line is only reached by the reads that were printed after trimming (bloom.cc:1360-1370)
				const uint64_t i0 = batch->id_offsets[r];
				if (append_trimmed_record(buf, batch->id_chars.data() + i0, batch->id_offsets[r + 1] - i0, batch->comment(r), batch->comment_len(r),
				                          batch->bases.data() + b0, len, batch->qual(r), batch->qual_len(r), o.k, left[r], right[r]) &&
				    o.verbose && (readCount + 1) % 100000 == 0)
					std::cerr << "Processed " << (readCount + 1) << " reads" << std::endl;
				if (buf.size() > (8u << 20)) {
					fwrite(buf.data(), 1, buf.size(), stdout);
					buf.clear();
				}
			}
		}
	}
	fwrite(buf.data(), 1, buf.size(), stdout);
	fflush(stdout);
	if (o.verbose)
		std::cerr << "Processed " << readCount << " reads" << std::endl;
	abb_filter_destroy(f);
	return EXIT_SUCCESS;
}

/** the canonical hash, and whether `graph` contains it (null: not asked), of every k-mer window of a batch; valid[s] = 0 for a
 *  window RollingHashIterator skips */
static void hash_windows(unsigned k, abb_filter* graph, const ReadBatch& b, std::vector<uint64_t>& h0, std::vector<uint8_t>& valid,
                         std::vector<uint8_t>& flag, int device)
{
	uint64_t slots = 0;
	for (size_t r = 0; r < b.size(); ++r) {
		const uint64_t len = b.offsets[r + 1] - b.offsets[r];
		slots += len >= k ? len - k + 1 : 0;
	}
	h0.resize(slots);
	valid.resize(slots);
	flag.resize(slots);
	check(abb_hash_reads(k, "", b.bases.data(), b.offsets.data(), b.size(), h0.data(), valid.data(), &slots, device), "hash");
	if (graph)
		check(abb_contains_reads(graph, b.bases.data(), b.offsets.data(), b.size(), flag.data(), nullptr, slots, &slots), "contains");
}

/** graph (Bloom/bloom.cc:984-1153): the GraphViz dump of the rolling-hash Bloom de Bruijn graph of FILE within -d steps of the
 *  roots, in either direction; the search and its text are host::bloom_graph (bloom_graph.h), the lookups of each level one
 *  abb_graph_neighbors call.  Where the reference asserts or reads past an array -- a root whose length is not k, a -k that is
 *  not the file's, an -A filter with more hashes than the graph -- and for a root with a character other than A, C, G, T, this
 *  command says why and exits with status 1 (DESIGN.md, section 3, K7b). */
static int graph(int argc, char** argv)
{
	// parseGlobalOpts (bloom.cc:296-344): -k and -v up to the first option of the command
	unsigned k = 0;
	int verbose = 0, device = 0;
	optind = 2;
	for (int c, prev = optind; (c = getopt_long(argc, argv, kShortOpts, kLongOpts, NULL)) != -1; prev = optind) {
		if (c == '?')
			usage();
		else if (c == 'k')
			k = parse_num<unsigned>(c, optarg);
		else if (c == 'v')
			++verbose;
		else if (c == OPT_HELP || c == OPT_VERSION) {
			std::cerr << PROGRAM ": see the reference's abyss-bloom --help\n";
			exit(EXIT_SUCCESS);
		} else {
			optind = prev;
			break;
		}
	}
	if (k == 0) {
		std::cerr << PROGRAM ": missing mandatory option `-k'\n";
		usage();
	}
	uint64_t maxDepth = k;
	std::vector<std::pair<std::string, std::string>> fastaAttrs, bloomAttrs; // (attribute, file)
	std::vector<std::string> roots, rootFastas;
	for (int c; (c = getopt_long(argc, argv, kShortOpts, kLongOpts, NULL)) != -1;) {
		std::istringstream arg(optarg != NULL ? optarg : "");
		switch (c) {
		case '?': usage(); break;
		case 'a':
		case 'A': {
			std::string s;
			arg >> s;
			const size_t pos = s.find(':');
			if (pos < s.length())
				(c == 'a' ? fastaAttrs : bloomAttrs).emplace_back(s.substr(0, pos), s.substr(pos + 1));
			else
				arg.setstate(std::ios::failbit);
		} break;
		case 'd': arg >> maxDepth; break;
		case 'f': {
			std::string path;
			arg >> path;
			rootFastas.push_back(path);
		} break;
		case 'R': {
			std::string kmer;
			arg >> kmer;
			roots.push_back(kmer);
		} break;
		case OPT_DEVICE: arg >> device; break;
		default: break;
		}
		// any other option with an argument is refused here: its argument is left unread
		if (optarg != NULL && (!arg.eof() || arg.fail())) {
			std::cerr << PROGRAM ": invalid option: `-" << (char)c << optarg << "'\n";
			exit(EXIT_FAILURE);
		}
	}
	if (roots.empty() && rootFastas.empty()) {
		std::cerr << PROGRAM ": must specify either --root or --root-fasta\n";
		usage();
	}
	if (argc - optind != 1) {
		std::cerr << PROGRAM ": missing arguments\n";
		usage();
	}
	const std::string bloomPath = argv[optind];
	// -d is read as a size_t and kept in RollingBloomDBGVisitor's unsigned m_maxDepth (RollingBloomDBGVisitor.h:38,170):
	// 2^32 + d is d
	const unsigned depth = (unsigned)maxDepth;
	if (verbose)
		std::cerr << "Loading main Bloom filter from `" << bloomPath << "'..." << std::endl;
	BloomHeader h;
	std::vector<uint8_t> raw;
	read_bit_bloom(bloomPath, h, raw);
	if (h.kmerSize != k) {
		std::cerr << PROGRAM ": `" << bloomPath << "' holds " << h.kmerSize << "-mers, not the " << k << "-mers of -k\n";
		exit(EXIT_FAILURE);
	}
	abb_filter* g = nullptr;
	check(abb_filter_create(&g, ABB_BIT, h.size, h.hashNum, h.kmerSize, 0, "", device), "filter");
	check(abb_filter_upload(g, 0, raw.data(), raw.size()), "upload");
	ReadOpts ropt;
	ropt.chastityFilter = g_chastity;
	ropt.trimMasked = g_trimMasked;
	ropt.qualityOffset = g_qualityOffset;
	std::vector<uint64_t> h0;
	std::vector<uint8_t> valid, flag;
	// --fasta-attr: the k-mers of each file (bloom.cc:1060-1092)
	std::vector<FastaAttr> fastaSets;
	for (const auto& a : fastaAttrs) {
		if (verbose)
			std::cerr << "Loading k-mers from `" << a.second << "', to be annotated with '" << a.first << "'\n";
		fastaSets.emplace_back(a.first, std::unordered_set<uint64_t>());
		uint64_t count = 0, checkpoint = 0;
		host::BatchStream stream({ a.second }, ropt, 1 << 20, 0, false);
		while (const ReadBatch* b = stream.next()) {
			hash_windows(k, nullptr, *b, h0, valid, flag, device);
			uint64_t s = 0;
			for (size_t r = 0; r < b->size(); ++r) {
				const uint64_t len = b->offsets[r + 1] - b->offsets[r];
				for (uint64_t i = 0; len >= k && i + k <= len; ++i, ++s)
					if (valid[s]) {
						fastaSets.back().second.insert(h0[s]);
						++count;
					}
				for (; verbose && count >= checkpoint; checkpoint += 10000)
					std::cerr << "Loaded " << checkpoint << " k-mers\n";
			}
		}
		if (verbose)
			std::cerr << "Loaded " << count << " k-mers in total\n";
	}
	// --bloom-attr (bloom.cc:1094-1110)
	std::vector<abb_filter*> attrFilters;
	std::vector<std::string> attrNames;
	for (const auto& a : bloomAttrs) {
		if (verbose)
			std::cerr << "Loading Bloom filter from `" << a.second << "', to be annotated with '" << a.first << "'\n";
		BloomHeader ah;
		std::vector<uint8_t> araw;
		read_bit_bloom(a.second, ah, araw);
		if (ah.hashNum > h.hashNum) {
			std::cerr << PROGRAM ": `" << a.second << "' uses " << ah.hashNum << " hash functions, more than the " << h.hashNum
			          << " of the graph's filter\n";
			exit(EXIT_FAILURE);
		}
		abb_filter* f = nullptr;
		check(abb_filter_create(&f, ABB_BIT, ah.size, ah.hashNum, ah.kmerSize, 0, "", device), "filter");
		check(abb_filter_upload(f, 0, araw.data(), araw.size()), "upload");
		attrFilters.push_back(f);
		attrNames.push_back(a.first);
		if (verbose) { // printRollingBloomStats (bloom.cc:469-476)
			uint64_t nz = 0;
			check(abb_filter_popcount(f, &nz, nullptr), "popcount");
			std::cerr << "Bloom size (bits): " << ah.size << "\nBloom popcount (bits): " << nz << "\nBloom filter FPR: " << std::setprecision(3)
			          << 100 * std::pow((double)nz / (double)ah.size, (double)ah.hashNum) << "%\n";
		}
	}
	// -R, then -f (bloom.cc:1112-1137)
	GraphRoots rootSet;
	for (const std::string& r : roots) {
		if (r.size() != k) {
			std::cerr << PROGRAM ": root `" << r << "' is not a " << k << "-mer\n";
			exit(EXIT_FAILURE);
		}
		if (r.find_first_not_of("ACGTacgt") != std::string::npos) {
			std::cerr << PROGRAM ": root `" << r << "' has a character other than A, C, G, T\n";
			exit(EXIT_FAILURE);
		}
	}
	if (!roots.empty()) {
		ReadBatch b;
		for (const std::string& r : roots)
			b.add("", r);
		hash_windows(k, g, b, h0, valid, flag, device);
		for (size_t i = 0; i < roots.size(); ++i)
			if (flag[i])
				rootSet.add(h0[i], roots[i].data(), k);
	}
	for (const std::string& path : rootFastas) {
		host::BatchStream stream({ path }, ropt, 1 << 20, 0, false);
		while (const ReadBatch* b = stream.next()) {
			hash_windows(k, g, *b, h0, valid, flag, device);
			uint64_t s = 0;
			for (size_t r = 0; r < b->size(); ++r) {
				const uint64_t len = b->offsets[r + 1] - b->offsets[r];
				for (uint64_t i = 0; len >= k && i + k <= len; ++i, ++s)
					if (valid[s] && flag[s])
						rootSet.add(h0[s], b->bases.data() + b->offsets[r] + i, k);
			}
		}
	}
	std::ostringstream buf;
	host::bloom_graph(
	    k, depth, rootSet, fastaSets, attrNames,
	    [&](const char* kmers, uint64_t n, abb_nbr_info* out) {
		    check(abb_graph_neighbors(g, kmers, n, attrFilters.data(), (unsigned)attrFilters.size(), out), "graph");
		    if (buf.tellp() > (8 << 20)) {
			    std::cout << buf.str();
			    buf.str("");
		    }
	    },
	    buf);
	std::cout << buf.str() << std::flush;
	for (abb_filter* f : attrFilters)
		abb_filter_destroy(f);
	abb_filter_destroy(g);
	return EXIT_SUCCESS;
}

int main(int argc, char** argv)
{
	apply_max_kmer(PROGRAM);
	const std::string cmd = argc >= 2 ? argv[1] : "";
	if (cmd == "info") { // the first operand once getopt has skipped the options (and their arguments)
		optind = 2;
		opterr = 0;
		while (getopt_long(argc, argv, kShortOpts, kLongOpts, NULL) != -1)
			;
		opterr = 1;
		if (optind < argc && is_konnector_bloom(argv[optind]))
			return info_konnector(argc, argv);
		return info(argc, argv);
	}
	if (cmd == "union")
		return combine(argc, argv, 1);
	if (cmd == "intersect")
		return combine(argc, argv, 2);
	if (cmd == "compare")
		return compare(argc, argv);
	if (cmd == "kmers" || cmd == "getKmers")
		return kmers(argc, argv);
	if (cmd == "trim")
		return trim(argc, argv);
	if (cmd == "graph")
		return graph(argc, argv);
	if (cmd != "build") {
		std::cerr << PROGRAM ": unrecognized command: `" << cmd << "'" << std::endl;
		usage();
	}
	uint64_t bloomSize = 500ULL << 20; // [500M]
	unsigned k = 0, numHashes = 1, levels = 1, threads = 1;
	int verbose = 0, device = 0;
	uint64_t batchReads = 4000000;
	std::string type = "konnector";
	ReadOpts ropt;
	uint64_t seed = 0;
	unsigned windowIndex = 0, windows = 0;
	std::vector<std::vector<std::string>> levelInitPaths;
	optind = 2;
	for (int c; (c = getopt_long(argc, argv, kShortOpts, kLongOpts, NULL)) != -1;) {
		switch (c) {
		case '?': usage(); break;
		case 'b':
			if (!si_to_bytes(optarg, &bloomSize)) {
				std::cerr << PROGRAM ": invalid option: `-b" << optarg << "'\n";
				exit(EXIT_FAILURE);
			}
			break;
		case 'k': k = parse_num<unsigned>(c, optarg); break;
		case 'H': numHashes = (unsigned)atoi(optarg); break;
		case 'h': seed = parse_num<uint64_t>(c, optarg); break;
		case 'l': levels = (unsigned)atoi(optarg); break;
		case 'j': threads = (unsigned)atoi(optarg); break;
		case 'q': ropt.qualityThreshold = atoi(optarg); break;
		case 't': type = optarg; break;
		case 'v': ++verbose; break;
		case OPT_DEVICE: device = atoi(optarg); break;
		case OPT_BATCH_READS: batchReads = strtoull(optarg, nullptr, 10); break;
		case 'L': { // N=FILE
			const char* eq = strchr(optarg, '=');
			const unsigned level = (unsigned)atoi(optarg);
			if (!eq || level == 0 || !eq[1])
				break;
			if (level > levelInitPaths.size())
				levelInitPaths.resize(level);
			levelInitPaths[level - 1].push_back(eq + 1);
			break;
		}
		case 'w': {
			std::istringstream arg(optarg);
			char slash = 0;
			arg >> windowIndex >> slash >> windows;
			if (arg.fail() || !arg.eof() || slash != '/' || windowIndex < 1 || windows < 1 || windowIndex > windows) {
				std::cerr << PROGRAM ": invalid option: `-w" << optarg << "'\n";
				exit(EXIT_FAILURE);
			}
			break;
		}
		default: break; // I/O buffer, lock count, the options of the other commands: no effect here
		}
	}
	const int chastity = g_chastity, trimMasked = g_trimMasked, qualityOffset = g_qualityOffset;
	ropt.chastityFilter = chastity;
	ropt.trimMasked = trimMasked;
	ropt.qualityOffset = qualityOffset;
	if (k == 0) {
		std::cerr << PROGRAM ": missing mandatory option `-k'\n";
		usage();
	}
	if (!levelInitPaths.empty() && levels < 2) {
		std::cerr << PROGRAM ": -L can only be used with cascading bloom filters (-l >= 2)\n";
		usage();
	}
	if (levelInitPaths.size() > levels) {
		std::cerr << PROGRAM ": level arg to -L is greater than number of bloom filter levels (-l)\n";
		usage();
	}
	if (type != "konnector" && type != "counting" && type != "rolling-hash") {
		std::cerr << PROGRAM ": unrecognized argument to `-t' (should be 'konnector', 'rolling-hash' or 'counting')\n";
		usage();
	}
	if (type != "konnector" && windows != 0) {
		std::cerr << PROGRAM ": -w (Bloom windows) only applies to `-t konnector' filters\n";
		exit(EXIT_FAILURE);
	}
	if (type == "konnector" && numHashes != 1) {
		std::cerr << PROGRAM ": warning: -H option has no effect when using `-t konnector'\n";
		numHashes = 1;
	}
	if (windows != 0 && bloomSize * 8 / levels % windows != 0) {
		std::cerr << PROGRAM ": (b / l) % w == 0 must be true, where b is bloom filter size (-b), l is number of levels (-l), and w "
		             "is number of windows (-w)\n";
		usage();
	}
	if (argc - optind < 2) {
		std::cerr << PROGRAM ": missing arguments\n";
		usage();
	}
	const std::string outputPath = argv[optind++];
	std::vector<std::string> files(argv + optind, argv + argc);
	if (type == "konnector") {
		if (verbose)
			std::cerr << "Building a Bloom filter of type 'konnector' with " << levels << " level(s), " << numHashes
			          << " hash function(s), and a total size of " << bloomSize << " bytes" << std::endl;
		return build_konnector(bloomSize * 8, k, levels, seed, windowIndex, windows, levelInitPaths, outputPath, files, ropt, batchReads,
		                       verbose, device);
	}

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
