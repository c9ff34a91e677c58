// oracle/ref_arith.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// Thin command-line harness around the UNMODIFIED reference headers, compiled from
// the reference source tree where they lie (see oracle/Makefile). It exposes the reference's
// arithmetic for this path so that the C restatement (abyss_oracle.c) and the CUDA
// kernels can be pinned against it:
//
//   ref_arith hashes  K H [MASK]  < seqs   one line per valid k-mer: seqIdx pos h0 .. h{H-1}
//                                          (BloomDBG/RollingHashIterator.h:35-97)
//   ref_arith nthash  K H         < seqs   same through vendor/nthash/ntHashIterator.hpp
//   ref_arith count   K H M       < seqs   insert every k-mer into CountingBloomFilter<uint8_t>
//                                          of M counters (CountingBloomFilter.hpp:138-162) and
//                                          write the raw counter array to stdout
//   ref_arith bits    K H M       < seqs   same for BloomFilter (BloomFilter.hpp:182-200), M bits
//   ref_arith casc    K H M L     < seqs   HashAgnosticCascadingBloom with L levels of M bits;
//                                          writes all L level arrays, level 0 first
//   ref_arith seeds   k K | qr k N         SpacedSeed::kmerPair / qrSeedPair
#include "config.h"
#include "BloomDBG/RollingHashIterator.h"
#include "BloomDBG/MaskedKmer.h"
#include "BloomDBG/SpacedSeed.h"
#include "Bloom/HashAgnosticCascadingBloom.h"
#include "vendor/nthash/ntHashIterator.hpp"
#include "vendor/btl_bloomfilter/CountingBloomFilter.hpp"
#include "vendor/btl_bloomfilter/BloomFilter.hpp"
#include "DataLayer/FastaReader.h"
#include "DataLayer/Options.h"
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <sstream>
#include <string>

/* BloomFilter keeps its array private: serialise and strip the TOML header */
static void dumpRaw(const BloomFilter& bf)
{
	std::ostringstream ss;
	ss << bf;
	const std::string& s = ss.str();
	const std::string tag = "[HeaderEnd]\n";
	size_t p = s.find(tag);
	fwrite(s.data() + p + tag.size(), 1, s.size() - p - tag.size(), stdout);
}

static void usage() { fprintf(stderr, "usage: ref_arith hashes|nthash|count|bits|casc|seeds|reads ...\n"); exit(2); }

int main(int argc, char** argv)
{
	if (argc < 2) usage();
	std::string cmd = argv[1];
	if (cmd == "seeds") {
		if (argc < 5) usage();
		if (std::string(argv[2]) == "qr")
			std::cout << SpacedSeed::qrSeedPair(atoi(argv[3]), atoi(argv[4])) << "\n";
		else
			std::cout << SpacedSeed::kmerPair(atoi(argv[3]), atoi(argv[4])) << "\n";
		return 0;
	}
	if (cmd == "reads") {
		// ref_arith reads dump|time FILE...: the reference's own reader (DataLayer/FastaReader.cpp, FOLD_CASE as in
		// BloomIO.h:58 / bloom-dbg.h:917) -- "id<TAB>sequence" per record, or records/s
		if (argc < 4) usage();
		const bool dump = std::string(argv[2]) == "dump";
		// the reader's global options (DataLayer/Options.h), as abyss-bloom-dbg's -q / -Q / --illumina-quality / --no-chastity /
		// --no-trim-masked set them
		if (const char* e = getenv("REF_Q")) opt::qualityThreshold = atoi(e);
		if (const char* e = getenv("REF_MASKQ")) opt::internalQThreshold = atoi(e);
		if (const char* e = getenv("REF_QOFF")) opt::qualityOffset = atoi(e);
		if (getenv("REF_NO_CHASTITY")) opt::chastityFilter = 0;
		if (getenv("REF_NO_TRIM_MASKED")) opt::trimMasked = 0;
		size_t n = 0, bases = 0;
		auto t0 = std::chrono::steady_clock::now();
		for (int i = 3; i < argc; ++i) {
			FastaReader in(argv[i], FastaReader::FOLD_CASE);
			for (FastaRecord rec; in >> rec;) {
				++n;
				bases += rec.seq.size();
				if (dump)
					std::cout << rec.id << '\t' << rec.seq << '\n';
			}
		}
		double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
		fprintf(stderr, "%zu reads, %zu bases in %.3f s: %.2f M reads/s\n", n, bases, s, n / s / 1e6);
		return 0;
	}
	if (argc < 4) usage();
	unsigned k = atoi(argv[2]), H = atoi(argv[3]);
	Kmer::setLength(k);
	MaskedKmer::setLength(k);
	std::string seq;
	if (cmd == "hashes") {
		if (argc > 4) MaskedKmer::setMask(argv[4]);
		for (size_t idx = 0; std::getline(std::cin, seq); ++idx)
			for (RollingHashIterator it(seq, H, k); it != RollingHashIterator::end(); ++it) {
				printf("%zu %u", idx, it.pos());
				for (unsigned i = 0; i < H; ++i) printf(" %llu", (unsigned long long)(*it)[i]);
				printf("\n");
			}
	} else if (cmd == "nthash") {
		for (size_t idx = 0; std::getline(std::cin, seq); ++idx) {
			ntHashIterator it(seq, H, k);
			for (; it != it.end(); ++it) {
				printf("%zu %zu", idx, it.pos());
				for (unsigned i = 0; i < H; ++i) printf(" %llu", (unsigned long long)(*it)[i]);
				printf("\n");
			}
		}
	} else if (cmd == "count") {
		if (argc < 5) usage();
		size_t m = strtoull(argv[4], NULL, 10);
		CountingBloomFilter<uint8_t> bloom(m, H, k, 0);
		while (std::getline(std::cin, seq))
			for (RollingHashIterator it(seq, H, k); it != RollingHashIterator::end(); ++it)
				bloom.insert(*it);
		for (size_t i = 0; i < bloom.size(); ++i) putchar(bloom[i]);
	} else if (cmd == "bits") {
		if (argc < 5) usage();
		size_t m = strtoull(argv[4], NULL, 10);
		BloomFilter bloom(m, H, k);
		while (std::getline(std::cin, seq))
			for (RollingHashIterator it(seq, H, k); it != RollingHashIterator::end(); ++it)
				bloom.insert(*it);
		dumpRaw(bloom);
	} else if (cmd == "casc") {
		if (argc < 6) usage();
		size_t m = strtoull(argv[4], NULL, 10);
		unsigned L = atoi(argv[5]);
		HashAgnosticCascadingBloom bloom(m, H, L, k);
		while (std::getline(std::cin, seq))
			for (RollingHashIterator it(seq, H, k); it != RollingHashIterator::end(); ++it)
				bloom.insert(*it);
		for (unsigned l = 0; l < L; ++l)
			dumpRaw(bloom.getBloomFilter(l));
	} else
		usage();
	return 0;
}
