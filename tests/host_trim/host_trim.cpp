// tests/host_trim/host_trim.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libabyssb200).
//
// `abyss-bloom trim` on one CPU thread: the SAME __host__ __device__ code the GPU runs (abb_konnector.cuh: KonVtx, kon_step,
// kon_left_trim; abb_walk.cuh: successor / trueBranch / lookAhead) over a one-lane context, on the product's reader and record
// writer.  Its output is compared with the unmodified reference's (tests/golden/make_golden_trim.py).
//
//   host_trim K [-q N] [--no-trim-masked] [--no-chastity] [--lengths FILE] IN.bloom READS...
// stdout: what `abyss-bloom trim -k K IN.bloom READS...` prints.  --lengths: one line "left right" per read (calcLeftTrim of
// the read and of its reverse complement; "0 0" for a read shorter than k, as abb_trim_reads gives).  stderr: minBranchLen and how many scans took
// each exit of calcLeftTrim.
#include "../../abyss_b200/csrc/abb_konnector.cuh"
#include "../../abyss_b200/host/bloom_file.h"
#include "../../abyss_b200/host/reads.h"
#include "../../abyss_b200/host/trim.h"

using namespace abb;

/** the Ctx of kon_left_trim and of the walk templates with one lane: every probe and search is a plain loop */
struct HostKonCtx {
	unsigned k, trim;
	KonGeom rt;
	KonView fv;
	Frame* frames;
	uint64_t* look;
	bool fail_ = false;
	mutable unsigned vertices = 0; // windows of the current scan that were in the filter
	unsigned probe(const KonVtx& v, unsigned lanes) const
	{
		unsigned m = 0;
		for (unsigned n = 0; n < 9; ++n)
			if (((lanes >> n) & 1u) && kon_test(fv, kon_neighbor_hash(v.m, rt, fv.seed, n)))
				m |= 1u << n;
		return m;
	}
	unsigned neighbors_self(const KonVtx& v) const
	{
		const unsigned m = probe(v, 0x1ffu);
		vertices += m >> 8;
		return m;
	}
	unsigned neighbors(const KonVtx& v) const { return probe(v, 0xffu); }
	unsigned neighbors_dir(const KonVtx& v, Dir d) const { return d == FWD ? probe(v, 0x0fu) : probe(v, 0xf0u) >> 4; }
	unsigned char base(const uint8_t* seq, unsigned, unsigned i) const { return seq[i]; }
	uint64_t rd64(const uint64_t* p) const { return *p; }
	void wr64(uint64_t* p, uint64_t v) const { *p = v; }
	void sync() const {}
	bool find64(const uint64_t* a, unsigned n, uint64_t key, unsigned stride) const
	{
		for (unsigned i = 0; i < n; ++i)
			if (a[(size_t)i * stride] == key)
				return true;
		return false;
	}
	void fail(unsigned) { fail_ = true; }
	bool failed() const { return fail_; }
};

int main(int argc, char** argv)
{
	if (argc < 4) {
		fprintf(stderr, "usage: host_trim K [-q N] [--no-trim-masked] [--no-chastity] [--lengths FILE] IN.bloom READS...\n");
		return 2;
	}
	const unsigned k = atoi(argv[1]);
	host::ReadOpts ropt;
	ropt.keepText = true;
	FILE* lengths = nullptr;
	int a = 2;
	for (; a < argc && argv[a][0] == '-'; ++a) {
		const std::string o = argv[a];
		if (o == "-q")
			ropt.qualityThreshold = atoi(argv[++a]);
		else if (o == "--no-trim-masked")
			ropt.trimMasked = 0;
		else if (o == "--no-chastity")
			ropt.chastityFilter = 0;
		else if (o == "--lengths")
			lengths = fopen(argv[++a], "w");
	}
	std::vector<uint8_t> raw;
	const host::KonnectorHeader h = host::read_konnector_bloom(argv[a++], k, raw);
	std::vector<uint8_t> data((h.full + 7) / 8, 0), next;
	if (h.start == 0)
		std::copy(raw.begin(), raw.end(), data.begin());
	else { // a window file: BloomFilter::read places its bits at the start bit
		next = data;
		for (uint64_t d = 0; d < data.size(); ++d)
			next[d] = kon_copy_bits_byte(data[d], raw.data(), h.bits(), h.start, KON_OVERWRITE, d);
		data.swap(next);
	}
	uint64_t pop = 0, mbl = 0;
	for (uint8_t b : data)
		pop += __builtin_popcount(b);
	if (!host::trim_min_branch_len(pop, h.full, &mbl)) {
		fprintf(stderr, "host_trim: full filter\n");
		return 1;
	}
	std::vector<Frame> frames(kFrameCap);
	std::vector<uint64_t> look(kLookCap);
	HostKonCtx c;
	c.k = k;
	c.trim = (unsigned)mbl;
	c.rt = kon_geom(k);
	c.fv = KonView{ data.data(), (uint64_t)data.size(), h.full, 0, 1, make_fastmod(h.full), h.seed };
	c.frames = frames.data();
	c.look = look.data();
	uint64_t exits[4] = { 0, 0, 0, 0 };
	std::string out;
	for (; a < argc; ++a) {
		host::SeqReader in(argv[a], ropt);
		std::string id, seq;
		while (in.next(id, seq)) {
			uint32_t lr[2] = { 0, 0 };
			if (seq.size() >= k) {
				for (int e = 0; e < 2; ++e) {
					c.vertices = 0;
					lr[e] = kon_left_trim(c, (const uint8_t*)seq.data(), (unsigned)seq.size(), e == 1);
					// how the scan ended: off the end (k - 2; a stop gives 0 or at least k) without meeting a vertex or after
					// a tip all the way, at the first vertex (not a tip) or at a later one (a fork)
					const unsigned kind = lr[e] == k - 2 ? (c.vertices == 0 ? 0 : 1) : (c.vertices == 1 ? 2 : 3);
					if (c.failed()) {
						fprintf(stderr, "host_trim: scratch overflow on read %s\n", id.c_str());
						return 1;
					}
					++exits[kind];
				}
			}
			if (lengths)
				fprintf(lengths, "%u %u\n", lr[0], lr[1]);
			const std::string& q = in.last_quality();
			const std::string& cm = in.last_comment();
			host::append_trimmed_record(out, id.data(), id.size(), cm.data(), cm.size(), seq.data(), seq.size(), q.data(), q.size(), k, lr[0], lr[1]);
		}
	}
	fwrite(out.data(), 1, out.size(), stdout);
	if (lengths)
		fclose(lengths);
	fprintf(stderr, "minBranchLen %llu exits end_no_vertex %llu end_tip %llu first_not_tip %llu fork %llu\n", (unsigned long long)mbl,
	        (unsigned long long)exits[0], (unsigned long long)exits[1], (unsigned long long)exits[2], (unsigned long long)exits[3]);
	return 0;
}
