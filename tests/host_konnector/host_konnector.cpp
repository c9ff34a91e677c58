// tests/host_konnector/host_konnector.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libabyssb200).
//
// Single-thread CPU emulation of the Konnector kernels: the SAME __host__ __device__ code the GPU runs (abb_konnector.cuh:
// the rolling canonical k-mer, CityHash64WithSeed, the level walk, copyBits) on the product's reader and file writer.  Its
// files are compared with the unmodified reference's (tests/golden/make_golden_konnector.py).
//
//   host_konnector build K FULL_BITS LEVELS SEED START END OUT.bloom READS...     (abyss-bloom build -t konnector)
//   host_konnector union|intersect K OUT.bloom IN.bloom...                         (abyss-bloom union / intersect)
#include "../../abyss_b200/csrc/abb_konnector.cuh"
#include "../../abyss_b200/host/bloom_file.h"
#include "../../abyss_b200/host/reads.h"

using namespace abb;

static void write_file(const std::string& path, const host::KonnectorHeader& h, const std::vector<uint8_t>& level)
{
	std::ofstream out(path, std::ios::binary);
	host::write_konnector_bloom(out, h, level.data());
}

static int build(int argc, char** argv)
{
	host::KonnectorHeader h;
	h.k = atoi(argv[2]);
	h.full = strtoull(argv[3], nullptr, 10);
	const unsigned levels = atoi(argv[4]);
	h.seed = strtoull(argv[5], nullptr, 10);
	h.start = strtoull(argv[6], nullptr, 10);
	h.end = strtoull(argv[7], nullptr, 10);
	const uint64_t bits = h.bits(), bpl = h.bytes();
	std::vector<uint8_t> data(bpl * levels, 0);
	const KonGeom g = kon_geom(h.k);
	const FastMod full = make_fastmod(h.full);
	host::ReadOpts ropt;
	for (int a = 9; a < argc; ++a) {
		host::SeqReader in(argv[a], ropt);
		std::string id, seq;
		while (in.next(id, seq)) {
			KonKmer m;
			kon_clear(m);
			for (size_t i = 0; i < seq.size(); ++i) {
				kon_push(m, g, (unsigned char)seq[i]);
				if (i + 1 < h.k || m.run < h.k)
					continue;
				const uint64_t pos = fastmod_u64(kon_hash(m, g, h.seed), full);
				if (pos < h.start || pos - h.start >= bits)
					continue;
				const uint64_t bit = pos - h.start;
				for (unsigned l = 0; l < levels; ++l) { // the lowest level whose bit is unset
					uint8_t& b = data[l * bpl + bit / 8];
					const uint8_t mask = (uint8_t)(0x80u >> (bit % 8));
					if (!(b & mask)) {
						b |= mask;
						break;
					}
				}
			}
		}
	}
	write_file(argv[8], h, std::vector<uint8_t>(data.end() - bpl, data.end()));
	return 0;
}

static int combine(int argc, char** argv, int op)
{
	const unsigned k = atoi(argv[2]);
	host::KonnectorHeader out;
	std::vector<uint8_t> dest;
	for (int a = 4; a < argc; ++a) {
		std::vector<uint8_t> raw;
		const host::KonnectorHeader h = host::read_konnector_bloom(argv[a], k, raw);
		if (a == 4) {
			out = h;
			out.start = 0;
			out.end = h.full - 1;
			dest.assign(out.bytes(), 0);
		}
		const int o = a == 4 ? KON_OVERWRITE : op;
		std::vector<uint8_t> next(dest);
		for (uint64_t d = 0; d < dest.size(); ++d)
			next[d] = kon_copy_bits_byte(dest[d], raw.data(), h.bits(), h.start, o, d);
		dest.swap(next);
	}
	write_file(argv[3], out, dest);
	return 0;
}

int main(int argc, char** argv)
{
	const std::string cmd = argc > 1 ? argv[1] : "";
	if (cmd == "build" && argc >= 10)
		return build(argc, argv);
	if ((cmd == "union" || cmd == "intersect") && argc >= 5)
		return combine(argc, argv, cmd == "union" ? KON_OR : KON_AND);
	fprintf(stderr, "usage: host_konnector build K FULL_BITS LEVELS SEED START END OUT READS... | union|intersect K OUT IN...\n");
	return 2;
}
