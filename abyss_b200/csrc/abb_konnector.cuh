// abb_konnector.cuh -- the Konnector Bloom filter family of abyss-bloom (`-t konnector`, Bloom/BloomFilter.h,
// CascadingBloomFilter.h, BloomFilterWindow.h): one CityHash64WithSeed probe per canonical k-mer, MSB-first bit order,
// optional cascade levels and bit windows.  Everything above the kernels is __host__ __device__ so that the CPU harness
// tests/host_konnector runs the same arithmetic against the reference's files.
//
// K-mer bytes (Common/Kmer.cpp): A0 C1 G2 T3, base i in byte i/4 at bits 2*(3 - i%4), padding zero, (k+3)/4 bytes.  Here a
// k-mer is held as NW big-endian 64-bit words (base i at bit 62 - 2*(i%32) of word i/32), so byte j of the packed k-mer is
// byte 7 - j%8 of word j/8 and the byte string CityHash reads is the words' big-endian image.  NW is 6 for k <= 192 and 8
// for k = 193..256 (kon_words), one kernel instance per width, so that k <= 192 does not carry two more words per image.
#pragma once
#include "abb_device.cuh"
#include "abb_walk.cuh"

namespace abb {

constexpr unsigned kKonWords = 6;     // words of a k-mer up to k = 192
constexpr unsigned kKonWordsWide = 8; // k = 193..kMaxK
inline unsigned kon_words(unsigned k) { return k <= 32 * kKonWords ? kKonWords : kKonWordsWide; }

#if defined(__CUDA_ARCH__)
#define KON_UNROLL _Pragma("unroll")
#else
#define KON_UNROLL
#endif

// ---- CityHash64WithSeed (CityHash 1.0, Geoff Pike and Jyrki Alakuijala), inputs of 1..64 bytes ------------------------
constexpr uint64_t kCityK0 = 0xc3a5c85c97cb3127ULL;
constexpr uint64_t kCityK1 = 0xb492b66fbe98f273ULL;
constexpr uint64_t kCityK2 = 0x9ae16a3b2f90404fULL;
constexpr uint64_t kCityK3 = 0xc949d7c7509e6557ULL;
constexpr uint64_t kCityMul = 0x9ddfea08eb382d69ULL;

ABB_HD uint64_t city_rot(uint64_t v, unsigned s) { return s == 0 ? v : (v >> s) | (v << (64 - s)); }
ABB_HD uint64_t city_shift_mix(uint64_t v) { return v ^ (v >> 47); }
ABB_HD uint64_t city_bswap64(uint64_t v)
{
#if defined(__CUDA_ARCH__)
	const unsigned lo = (unsigned)v, hi = (unsigned)(v >> 32);
	return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
#else
	return __builtin_bswap64(v);
#endif
}
/** the 128-to-64-bit mix (Hash128to64) of (lo, hi) */
ABB_HD uint64_t city_hash16(uint64_t lo, uint64_t hi)
{
	uint64_t a = (lo ^ hi) * kCityMul;
	a ^= a >> 47;
	uint64_t b = (hi ^ a) * kCityMul;
	b ^= b >> 47;
	return b * kCityMul;
}

/** word i of a k-mer image, 0 past the end (a select chain keeps the words in registers) */
template <unsigned NW>
ABB_HD uint64_t kon_word(const uint64_t* w, unsigned i)
{
	uint64_t r = 0;
KON_UNROLL
	for (unsigned j = 0; j < NW; ++j)
		r = j == i ? w[j] : r;
	return r;
}
/** little-endian 64-bit load at byte offset o of the big-endian word image */
template <unsigned NW>
ABB_HD uint64_t kon_fetch64(const uint64_t* w, unsigned o)
{
	const unsigned s = 8 * (o % 8);
	const uint64_t hi = kon_word<NW>(w, o / 8), lo = kon_word<NW>(w, o / 8 + 1);
	return city_bswap64(s ? (hi << s) | (lo >> (64 - s)) : hi);
}
template <unsigned NW>
ABB_HD uint64_t kon_fetch32(const uint64_t* w, unsigned o) { return kon_fetch64<NW>(w, o) & 0xffffffffULL; }
template <unsigned NW>
ABB_HD unsigned kon_byte(const uint64_t* w, unsigned o) { return (unsigned)(kon_word<NW>(w, o / 8) >> (56 - 8 * (o % 8))) & 0xffu; }

/** CityHash64 of the first len (1..8 * NW, at most 64) bytes of an image of NW words */
template <unsigned NW>
ABB_HD uint64_t city64(const uint64_t* w, unsigned len)
{
	if (len > 32) { // 33..64 bytes
		uint64_t z = kon_fetch64<NW>(w, 24);
		uint64_t a = kon_fetch64<NW>(w, 0) + (len + kon_fetch64<NW>(w, len - 16)) * kCityK0;
		uint64_t b = city_rot(a + z, 52);
		uint64_t c = city_rot(a, 37);
		a += kon_fetch64<NW>(w, 8);
		c += city_rot(a, 7);
		a += kon_fetch64<NW>(w, 16);
		const uint64_t vf = a + z, vs = b + city_rot(a, 31) + c;
		a = kon_fetch64<NW>(w, 16) + kon_fetch64<NW>(w, len - 32);
		z = kon_fetch64<NW>(w, len - 8);
		b = city_rot(a + z, 52);
		c = city_rot(a, 37);
		a += kon_fetch64<NW>(w, len - 24);
		c += city_rot(a, 7);
		a += kon_fetch64<NW>(w, len - 16);
		const uint64_t wf = a + z, ws = b + city_rot(a, 31) + c;
		const uint64_t r = city_shift_mix((vf + ws) * kCityK2 + (wf + vs) * kCityK0);
		return city_shift_mix(r * kCityK0 + vs) * kCityK2;
	}
	if (len > 16) { // 17..32 bytes
		const uint64_t a = kon_fetch64<NW>(w, 0) * kCityK1, b = kon_fetch64<NW>(w, 8);
		const uint64_t c = kon_fetch64<NW>(w, len - 8) * kCityK2, d = kon_fetch64<NW>(w, len - 16) * kCityK0;
		return city_hash16(city_rot(a - b, 43) + city_rot(c, 30) + d, a + city_rot(b ^ kCityK3, 20) - c + len);
	}
	if (len > 8) {
		const uint64_t a = kon_fetch64<NW>(w, 0), b = kon_fetch64<NW>(w, len - 8);
		return city_hash16(a, city_rot(b + len, len)) ^ b;
	}
	if (len >= 4) {
		const uint64_t a = kon_fetch32<NW>(w, 0);
		return city_hash16(len + (a << 3), kon_fetch32<NW>(w, len - 4));
	}
	const uint32_t y = kon_byte<NW>(w, 0) + ((uint32_t)kon_byte<NW>(w, len >> 1) << 8);
	const uint32_t z = len + ((uint32_t)kon_byte<NW>(w, len - 1) << 2);
	return city_shift_mix(y * kCityK2 ^ z * kCityK3) * kCityK2;
}

/** Bloom::hash(kmer, seed) (Bloom/Bloom.h:63-71): CityHash64WithSeed of the canonical k-mer's (k+3)/4 bytes */
template <unsigned NW>
ABB_HD uint64_t city64_seed(const uint64_t* w, unsigned len, uint64_t seed)
{
	return city_hash16(city64<NW>(w, len) - kCityK2, seed);
}

// ---- the rolling canonical k-mer ---------------------------------------------------------------------------------------
/** forward and reverse-complement images of the current window, rolled one base at a time; `run` counts the ACGT bases
 *  since the last other character, so the window is a k-mer exactly when run >= k (Bloom::loadSeq skips the others) */
template <unsigned NW>
struct KonKmerN {
	uint64_t f[NW], r[NW];
	unsigned run;
};
using KonKmer = KonKmerN<kKonWords>;

struct KonGeom {
	unsigned k, nbytes;       // k, (k+3)/4
	unsigned last_word;       // word of base k-1
	unsigned last_shift;      // its bit shift, 62 - 2*((k-1) % 32)
	uint64_t last_mask;       // bits of bases 0..k-1 within the last word
};

inline KonGeom kon_geom(unsigned k) // host only
{
	KonGeom g;
	g.k = k;
	g.nbytes = (k + 3) / 4;
	g.last_word = (k - 1) / 32;
	g.last_shift = 62 - 2 * ((k - 1) % 32);
	g.last_mask = ~0ULL << g.last_shift;
	return g;
}

template <unsigned NW>
ABB_HD void kon_clear(KonKmerN<NW>& m)
{
KON_UNROLL
	for (unsigned j = 0; j < NW; ++j)
		m.f[j] = m.r[j] = 0;
	m.run = 0;
}

/** append character c (any case) to the window */
template <unsigned NW>
ABB_HD void kon_push(KonKmerN<NW>& m, const KonGeom& g, unsigned char c)
{
	unsigned code = base_code(c);
	if (code > 3) {
		m.run = 0;
		code = 0;
	} else
		++m.run;
KON_UNROLL
	for (unsigned j = 0; j < NW; ++j) // forward: shift left one base, the new base goes to position k-1
		m.f[j] = (m.f[j] << 2) | (j + 1 < NW ? m.f[j + 1] >> 62 : 0);
KON_UNROLL
	for (int j = NW - 1; j >= 0; --j) // reverse complement: shift right one base, the complement goes to position 0
		m.r[j] = (m.r[j] >> 2) | (j > 0 ? m.r[j - 1] << 62 : 0);
	m.r[0] |= (uint64_t)(3 - code) << 62;
KON_UNROLL
	for (unsigned j = 0; j < NW; ++j) {
		const uint64_t keep = j < g.last_word ? ~0ULL : j == g.last_word ? g.last_mask : 0ULL;
		m.f[j] &= keep;
		m.r[j] &= keep;
	}
KON_UNROLL
	for (unsigned j = 0; j < NW; ++j)
		if (j == g.last_word)
			m.f[j] |= (uint64_t)code << g.last_shift;
}

/** Bloom::hash of the current window: the forward image when it is not larger than its reverse complement
 *  (Kmer::isCanonical, Common/Kmer.cpp:297-310), else the reverse complement */
template <unsigned NW>
ABB_HD uint64_t kon_hash(const KonKmerN<NW>& m, const KonGeom& g, uint64_t seed)
{
	int cmp = 0;
KON_UNROLL
	for (unsigned j = 0; j < NW; ++j)
		if (cmp == 0 && m.f[j] != m.r[j])
			cmp = m.f[j] < m.r[j] ? -1 : 1;
	uint64_t c[NW];
KON_UNROLL
	for (unsigned j = 0; j < NW; ++j)
		c[j] = cmp <= 0 ? m.f[j] : m.r[j];
	return city64_seed<NW>(c, g.nbytes, seed);
}

// ---- filter geometry ---------------------------------------------------------------------------------------------------
/** one Konnector filter on the device: `levels` arrays of `bits` bits (bit i of a level: byte i/8, mask 0x80 >> i%8) that
 *  hold the positions [start, start + bits) of a filter of `full` bits (a window, BloomFilterWindow.h; start = 0 and
 *  bits = full without -w) */
struct KonView {
	uint8_t* data;
	uint64_t bytes_per_level, bits, start;
	unsigned levels;
	FastMod full;
	uint64_t seed;
};

// ---- readBits / copyBits (Common/BitUtil.h:69-158) ----------------------------------------------------------------------
enum { KON_OVERWRITE = 0, KON_OR = 1, KON_AND = 2 };

/** The value that byte d of dest ends up with when copyBits(src, dest, bits, bit_offset, op) runs over it: byte d is the
 *  "next" byte of source byte i - 1 and then the "this" byte of source byte i (i = d - bit_offset/8), and the two never read
 *  each other, so every destination byte is a function of its old value and two source bytes.  The source bytes are
 *  `char`, so a source byte with its top bit set sign-extends when it is shifted right and ORs ones into the top `shift`
 *  bits of its "this" byte; the reference does that, so does this.  The byte-aligned overwrite of readBits (a plain copy
 *  with a masked last byte) is the op == KON_OVERWRITE, shift == 0 case. */
ABB_HD uint8_t kon_copy_bits_byte(uint8_t old, const uint8_t* src, uint64_t bits, uint64_t bit_offset, int op, uint64_t d)
{
	const uint64_t bytes = (bits + 7) / 8, full_bytes = bits % 8 == 0 ? bytes : bytes - 1, bo = bit_offset / 8;
	const unsigned shift = (unsigned)(bit_offset % 8);
	if (d < bo || d > bo + bytes)
		return old;
	const uint64_t i = d - bo; // source byte whose "this" byte d is
	if (op == KON_OVERWRITE && shift == 0) {
		if (i < full_bytes)
			return src[i];
		if (i < bytes) {
			const uint8_t m = (uint8_t)(0xFF << (8 - bits % 8));
			return (uint8_t)((old & ~m) | (src[i] & m));
		}
		return old;
	}
	const uint8_t carry = (uint8_t)(0xFF << (8 - shift));
	int v = old;
	// as the "next" byte of source byte i - 1
	if (i >= 1 && i - 1 < full_bytes) {
		const int s = (int)(signed char)src[i - 1];
		if (op == KON_OVERWRITE)
			v &= ~carry;
		if (op == KON_AND)
			v &= (s << (8 - shift)) | ~(int)carry;
		else
			v |= s << (8 - shift);
	} else if (i >= 1 && i - 1 == full_bytes && full_bytes < bytes) { // after the partial last byte
		const uint8_t lmask = (uint8_t)(0xFF << (8 - bits % 8)), lcarry = (uint8_t)(lmask << (8 - shift));
		const int lb = (int)(signed char)(src[bytes - 1] & lmask);
		if (lcarry > 0) {
			if (op == KON_OVERWRITE)
				v &= ~lcarry;
			if (op == KON_AND)
				v &= (lb << (8 - shift)) | ~(int)lcarry;
			else
				v |= lb << (8 - shift);
		}
	}
	v &= 0xFF;
	// as the "this" byte of source byte i
	if (i < full_bytes) {
		const int s = (int)(signed char)src[i];
		if (op == KON_OVERWRITE)
			v &= carry;
		if (op == KON_AND)
			v &= (s >> shift) | carry;
		else
			v |= s >> shift;
	} else if (i < bytes) {
		const uint8_t lmask = (uint8_t)(0xFF << (8 - bits % 8));
		const int lb = (int)(signed char)(src[bytes - 1] & lmask);
		if (op == KON_OVERWRITE)
			v &= ~(int)(uint8_t)(lmask >> shift);
		if (op == KON_AND)
			v &= (lb >> shift) | ~(int)(lmask >> shift);
		else
			v |= lb >> shift;
	}
	return (uint8_t)(v & 0xFF);
}

// ---- the Konnector de Bruijn graph (Konnector/DBGBloom.h) and `abyss-bloom trim` (Bloom/bloom.cc:1233-1382) -------------
/** One step of a k-mer in place: FWD drops base 0 and appends b (Kmer::shift(SENSE) + setLastBase), REV drops base k-1 and
 *  prepends b; both images follow.  A step to the left of the forward image is a step to the right of the reverse
 *  complement with the complementary base, so one shift serves both directions.  Only the words that k uses are shifted:
 *  a step sits on the critical path of every graph move, where kon_push (a bulk scan) shifts all NW. */
template <unsigned NW>
ABB_HD void kon_step(KonKmerN<NW>& m, const KonGeom& g, Dir d, unsigned b)
{
	if (d == REV) {
KON_UNROLL
		for (unsigned j = 0; j < NW; ++j) {
			const uint64_t t = m.f[j];
			m.f[j] = m.r[j];
			m.r[j] = t;
		}
		b = 3 - b;
	}
KON_UNROLL
	for (unsigned j = 0; j < NW; ++j) { // shift left one base, b goes to position k-1
		if (j > g.last_word)
			break;
		m.f[j] = (m.f[j] << 2) | (j + 1 < NW && j < g.last_word ? m.f[j + 1 < NW ? j + 1 : j] >> 62 : 0);
		if (j == g.last_word)
			m.f[j] |= (uint64_t)b << g.last_shift;
	}
KON_UNROLL
	for (int j = NW - 1; j >= 0; --j) { // shift right one base, the complement goes to position 0
		if ((unsigned)j > g.last_word)
			continue;
		m.r[j] = (m.r[j] >> 2) | (j > 0 ? m.r[j > 0 ? j - 1 : 0] << 62 : 0);
		if ((unsigned)j == g.last_word)
			m.r[j] &= g.last_mask;
	}
	m.r[0] |= (uint64_t)(3 - b) << 62;
	if (d == REV) {
KON_UNROLL
		for (unsigned j = 0; j < NW; ++j) {
			const uint64_t t = m.f[j];
			m.f[j] = m.r[j];
			m.r[j] = t;
		}
	}
}

/** A vertex of DBGBloom: a k-mer AS GIVEN, not up to reverse complement (graph_traits<DBGBloom>::vertex_descriptor is Kmer,
 *  whose operator== compares the packed bytes), so `visited` in lookAhead / trueBranch and "source(*iei) == u" tell a k-mer
 *  from its reverse complement.  id stands for the forward image in those comparisons: the image itself for k <= 32
 *  (exact), a chain of CityHash's 128-to-64-bit mix over its words above that.  A walk compares a vertex with at most
 *  kFrameCap + kLookCap others, all within a few dozen steps of one read k-mer; two different k-mers among them sharing
 *  the 64-bit mix is a ~2^-64 event per comparison, the same order as the ntHash identity of the pass-2 walk. */
template <unsigned NW>
struct KonVtxN {
	KonKmerN<NW> m;
	uint64_t id;
	ABB_HD uint64_t canon() const { return id; }
};
using KonVtx = KonVtxN<kKonWords>;
template <unsigned NW>
ABB_HD uint64_t kon_identity(const KonKmerN<NW>& m, const KonGeom& g)
{
	uint64_t id = m.f[0];
KON_UNROLL
	for (unsigned j = 1; j < NW; ++j) {
		if (j > g.last_word)
			break;
		id = city_hash16(id, m.f[j]);
	}
	return id;
}
/** the vertex interface of the walk templates (abb_walk.cuh); returns the base that fell off */
template <unsigned NW>
ABB_HD unsigned vtx_step(KonVtxN<NW>& v, unsigned, const KonGeom& g, Dir d, unsigned b)
{
	const unsigned out = d == FWD ? (unsigned)(v.m.f[0] >> 62) : 3u - (unsigned)(v.m.r[0] >> 62);
	kon_step(v.m, g, d, b);
	v.id = kon_identity(v.m, g);
	return out;
}
template <unsigned NW>
ABB_HD void vtx_unstep(KonVtxN<NW>& v, unsigned k, const KonGeom& g, Dir d, unsigned out) { vtx_step(v, k, g, opposite(d), out); }

/** Bloom::hash of neighbour n of m: n = 0..3 the out-edges (append A, C, G, T: out_edge_iterator, DBGBloom.h:160-221),
 *  4..7 the in-edges (prepend A, C, G, T: in_edge_iterator, :224-285), 8 the k-mer itself */
template <unsigned NW>
ABB_HD uint64_t kon_neighbor_hash(const KonKmerN<NW>& m, const KonGeom& g, uint64_t seed, unsigned n)
{
	KonKmerN<NW> t = m;
	if (n < 8)
		kon_step(t, g, n < 4 ? FWD : REV, n & 3);
	return kon_hash(t, g, seed);
}
/** BloomFilter::operator[] on the last level: the level a cascading build writes to its file (vertex_exists, DBGBloom.h:294-299) */
ABB_HD bool kon_test(const KonView& fv, uint64_t hash)
{
	const uint64_t pos = fastmod_u64(hash, fv.full);
	if (pos < fv.start || pos - fv.start >= fv.bits)
		return false;
	const uint64_t bit = pos - fv.start;
	const uint8_t* level = fv.data + (uint64_t)(fv.levels - 1) * fv.bytes_per_level;
	return (level[bit / 8] >> (7 - bit % 8)) & 1;
}

constexpr uint32_t kKonTrimFailed = 0xffffffffu; // the walk scratch overflowed: no trim length for this task

/**
 * calcLeftTrim (bloom.cc:1236-1290) of seq[0, len), len >= k, or of its reverse complement (rc: read from the end of the
 * read, never materialised).  KmerIterator (Common/KmerIterator.h) skips the windows that hold a non-ACGT character; a
 * k-mer that is not in the filter is skipped; the first k-mer that is must be a tip -- (DEAD_END, LENGTH_LIMIT) or the
 * reverse -- for the scan to go on, and a later one stops it when either side is AMBI_OUT.  Stopping at window p gives
 * p == 0 ? 0 : k + p - 1.  When the scan runs off the end the reference's pos() is SIZE_MAX and its int result k - 2: kept.
 *
 * Ctx is the walk context of abb_walk.cuh (k, trim = minBranchLen, rt = the KonGeom, neighbors / neighbors_dir, the scratch
 * accessors) plus
 *   unsigned neighbors_self(const KonVtxN<NW>&)   neighbors() with bit 8 = the k-mer itself is in the filter: nine probes issued
 *                                            together, so a window costs one memory round trip whether or not it is a vertex
 *   unsigned char base(const uint8_t* seq, unsigned len, unsigned i)   seq[i]
 */
template <unsigned NW = kKonWords, class Ctx>
ABB_HD uint32_t kon_left_trim(Ctx& c, const uint8_t* seq, unsigned len, bool rc)
{
	const unsigned k = c.k;
	KonVtxN<NW> v;
	kon_clear(v.m);
	unsigned run = 0;
	bool first = true;
	for (unsigned i = 0; i < len; ++i) {
		unsigned code = base_code(c.base(seq, len, rc ? len - 1 - i : i));
		if (code > 3) { // the next k-mer starts after this character; the k bases pushed by then overwrite every position
			run = 0;
			continue;
		}
		kon_step(v.m, c.rt, FWD, rc ? 3 - code : code);
		if (++run < k)
			continue;
		const unsigned nb = c.neighbors_self(v);
		if (!(nb & 256u))
			continue;
		v.id = kon_identity(v.m, c.rt);
		unsigned vbase = 0;
		const ExtCode left = successor(c, v, nb & 255u, REV, &vbase);
		const ExtCode right = successor(c, v, nb & 255u, FWD, &vbase);
		if (c.failed())
			return kKonTrimFailed;
		const bool stop = first ? !((left == ER_DEAD_END && right == ER_LENGTH_LIMIT) || (left == ER_LENGTH_LIMIT && right == ER_DEAD_END))
		                        : (left == ER_AMBI_OUT || right == ER_AMBI_OUT); // this successor never returns AMBI_IN
		if (stop) {
			const unsigned pos = i + 1 - k;
			return pos == 0 ? 0 : k + pos - 1;
		}
		first = false;
	}
	return k - 2;
}

#if defined(__CUDACC__)
// ---- kernels -----------------------------------------------------------------------------------------------------------
constexpr unsigned kKonSlotsPerThread = 128; // windows one thread rolls through (the first k - 1 bases are the overhead)

/** first read whose slot range ends after `slot` (slot_offs: exclusive prefix sum of the window counts, n_reads + 1 entries) */
__device__ __forceinline__ uint64_t kon_read_of(const uint64_t* __restrict__ slot_offs, uint64_t n_reads, uint64_t slot)
{
	uint64_t lo = 0, hi = n_reads; // slot_offs[lo] <= slot < slot_offs[hi]
	while (hi - lo > 1) {
		const uint64_t mid = (lo + hi) / 2;
		if (slot_offs[mid] <= slot)
			lo = mid;
		else
			hi = mid;
	}
	return lo;
}

/** Each thread takes kKonSlotsPerThread consecutive window slots of the batch (crossing read boundaries), rolls the
 *  canonical k-mer along them and, for every valid window:
 *   kQuery = false: inserts it.  The level walk is CascadingBloomFilter::insert (CascadingBloomFilter.h:75-84): set the
 *     lowest level whose bit is unset.  atomicOr returns the old word, so a k-mer stops at the first level whose bit IT
 *     flipped; a bit is never cleared, so any interleaving leaves at each position the min(n, L) lowest unset levels set
 *     that n sequential inserts would -- the result does not depend on the order.  A position outside the window is
 *     dropped (BloomFilterWindow::insert).
 *   kQuery = true: writes the bit of the last level to flag[slot] and the window's validity to valid[slot].
 *  n_kmers (optional) counts the valid windows. */
template <bool kQuery, unsigned NW>
__global__ void __launch_bounds__(256) k_kon_walk(const uint8_t* __restrict__ bases, const uint64_t* __restrict__ offs,
                                                  const uint64_t* __restrict__ slot_offs, uint64_t n_reads, uint64_t n_slots,
                                                  KonGeom g, KonView fv, uint8_t* __restrict__ flag, uint8_t* __restrict__ valid,
                                                  unsigned long long* __restrict__ n_kmers)
{
	const uint64_t n_tasks = (n_slots + kKonSlotsPerThread - 1) / kKonSlotsPerThread;
	unsigned long long counted = 0;
	for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_tasks; t += (uint64_t)gridDim.x * blockDim.x) {
		const uint64_t s0 = t * kKonSlotsPerThread, s1 = min(n_slots, s0 + kKonSlotsPerThread);
		uint64_t r = kon_read_of(slot_offs, n_reads, s0);
		uint64_t s = s0;
		while (s < s1) {
			while (slot_offs[r + 1] <= s) // reads without windows
				++r;
			const uint64_t read_end = min(s1, slot_offs[r + 1]);
			const uint8_t* seq = bases + offs[r];
			const uint64_t p0 = s - slot_offs[r]; // first window of this read handled here
			KonKmerN<NW> m;
			kon_clear(m);
			for (unsigned i = 0; i + 1 < g.k; ++i)
				kon_push(m, g, seq[p0 + i]);
			for (uint64_t p = p0; s < read_end; ++s, ++p) {
				kon_push(m, g, seq[p + g.k - 1]);
				const bool ok = m.run >= g.k;
				uint8_t hit = 0;
				if (ok) {
					++counted;
					const uint64_t pos = fastmod_u64(kon_hash(m, g, fv.seed), fv.full);
					if (pos >= fv.start && pos - fv.start < fv.bits) {
						const uint64_t bit = pos - fv.start;
						if (kQuery) {
							hit = (fv.data[(uint64_t)(fv.levels - 1) * fv.bytes_per_level + bit / 8] >> (7 - bit % 8)) & 1;
						} else {
							for (unsigned l = 0; l < fv.levels; ++l) {
								const uint64_t byte = (uint64_t)l * fv.bytes_per_level + bit / 8;
								const unsigned mask = (0x80u >> (bit % 8)) << (8 * (byte % 4));
								unsigned* word = reinterpret_cast<unsigned*>(fv.data) + byte / 4;
								if (!(atomicOr(word, mask) & mask))
									break;
							}
						}
					}
				}
				if (kQuery) {
					flag[s] = hit;
					valid[s] = ok;
				}
			}
			++r;
		}
	}
	if (n_kmers) {
		for (int o = 16; o > 0; o >>= 1)
			counted += __shfl_down_sync(0xffffffffu, counted, o);
		if ((threadIdx.x & 31) == 0 && counted)
			atomicAdd(n_kmers, counted);
	}
}

/** readBits(in, dest, bits, bit_offset, op) with the source already on the device: one thread per destination byte */
__global__ void k_kon_read_bits(uint8_t* __restrict__ dest, uint64_t dest_bytes, const uint8_t* __restrict__ src, uint64_t bits,
                                uint64_t bit_offset, int op)
{
	const uint64_t bo = bit_offset / 8, last = min(dest_bytes, bo + (bits + 7) / 8 + 1);
	for (uint64_t d = bo + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; d < last; d += (uint64_t)gridDim.x * blockDim.x)
		dest[d] = kon_copy_bits_byte(dest[d], src, bits, bit_offset, op, d);
}

/** population of nbytes bytes at any alignment (cascade levels need not start on a word) */
__global__ void k_kon_popcount(const uint8_t* __restrict__ p, uint64_t nbytes, unsigned long long* __restrict__ out)
{
	const uint64_t align = (16 - ((uintptr_t)p & 15)) & 15, head = align < nbytes ? align : nbytes;
	const uint64_t nvec = (nbytes - head) / 16;
	const uint4* v = reinterpret_cast<const uint4*>(p + head);
	unsigned long long n = 0;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint4 x = v[i];
		n += __popc(x.x) + __popc(x.y) + __popc(x.z) + __popc(x.w);
	}
	if (blockIdx.x == 0 && threadIdx.x == 0) {
		for (uint64_t i = 0; i < head; ++i)
			n += __popc(p[i]);
		for (uint64_t i = head + nvec * 16; i < nbytes; ++i)
			n += __popc(p[i]);
	}
	for (int o = 16; o > 0; o >>= 1)
		n += __shfl_down_sync(0xffffffffu, n, o);
	if ((threadIdx.x & 31) == 0 && n)
		atomicAdd(out, n);
}

/** the 1/1, 1/0 and 0/1 bit counts of two arrays of nbytes bytes (0/0 is the rest of the bits); out[0..2] */
__global__ void k_kon_compare(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, uint64_t nbytes,
                              unsigned long long* __restrict__ out)
{
	unsigned long long n11 = 0, n10 = 0, n01 = 0;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nbytes; i += (uint64_t)gridDim.x * blockDim.x) {
		const unsigned x = a[i], y = b[i];
		n11 += __popc(x & y);
		n10 += __popc(x & ~y & 0xffu);
		n01 += __popc(~x & y & 0xffu);
	}
	for (int o = 16; o > 0; o >>= 1) {
		n11 += __shfl_down_sync(0xffffffffu, n11, o);
		n10 += __shfl_down_sync(0xffffffffu, n10, o);
		n01 += __shfl_down_sync(0xffffffffu, n01, o);
	}
	if ((threadIdx.x & 31) == 0) {
		atomicAdd(out + 0, n11);
		atomicAdd(out + 1, n10);
		atomicAdd(out + 2, n01);
	}
}

/** The walk context of one warp on a Konnector filter.  All 32 lanes run the graph logic with the same arguments; they part
 *  only in the probes, where lane n < 9 hashes neighbour n (kon_neighbor_hash) and loads its bit, and in the scratch
 *  accessors.  The scratch conventions are WarpCtx's (abb_assemble.cu): every lane stores the same value and reads back
 *  its own store. */
template <unsigned NW>
struct KonWarpCtx {
	unsigned k, trim;
	KonGeom rt;
	KonView fv;
	unsigned lane;
	Frame* frames;
	uint64_t* look;
	unsigned fail_;
	unsigned chunk;       // which 32 characters of the read `held` is
	unsigned char held;   // character 32 * chunk + lane

	__device__ unsigned probe(const KonVtxN<NW>& v, unsigned lanes) const
	{
		bool ok = false;
		if ((lanes >> lane) & 1u)
			ok = kon_test(fv, kon_neighbor_hash(v.m, rt, fv.seed, lane));
		return __ballot_sync(0xffffffffu, ok);
	}
	__device__ unsigned neighbors_self(const KonVtxN<NW>& v) const { return probe(v, 0x1ffu); }
	__device__ unsigned neighbors(const KonVtxN<NW>& v) const { return probe(v, 0xffu); }
	__device__ unsigned neighbors_dir(const KonVtxN<NW>& v, Dir d) const { return d == FWD ? probe(v, 0x0fu) : probe(v, 0xf0u) >> 4; }
	/** seq[i]: the warp keeps 32 characters in registers (one coalesced load per 32 windows instead of one load per window) */
	__device__ unsigned char base(const uint8_t* seq, unsigned len, unsigned i)
	{
		if (i / 32 != chunk) {
			chunk = i / 32;
			const unsigned j = chunk * 32 + lane;
			held = j < len ? seq[j] : 0;
		}
		return (unsigned char)__shfl_sync(0xffffffffu, (unsigned)held, i % 32);
	}
	__device__ uint64_t rd64(const uint64_t* p) const { return *(const volatile uint64_t*)p; }
	__device__ void wr64(uint64_t* p, uint64_t v) const { *(volatile uint64_t*)p = v; }
	__device__ void sync() const { __syncwarp(); }
	__device__ bool find64(const uint64_t* a, unsigned n, uint64_t key, unsigned stride) const
	{
		for (unsigned b0 = 0; b0 < n; b0 += 32) {
			const unsigned i = b0 + lane;
			const bool hit = i < n && *(const volatile uint64_t*)(a + (size_t)i * stride) == key;
			if (__any_sync(0xffffffffu, hit))
				return true;
		}
		return false;
	}
	__device__ void fail(unsigned why) { fail_ |= 1u << why; }
	__device__ bool failed() const { return fail_ != 0; }
};

constexpr unsigned kKonTrimThreads = 128;

/** `abyss-bloom trim`: task 2r is the left end of read r, task 2r + 1 its right end (the same scan over the reverse
 *  complement); each writes one trim length, kKonTrimFailed when the walk scratch overflowed, 0 for a read shorter than k
 *  (which the caller echoes).  One warp per task, tasks dealt round-robin to a grid that fills the device once: most tasks
 *  end at their first window after one probe round, a few walk tens of windows with a trueBranch search at each, and with
 *  hundreds of tasks per warp, the two ends of a read and neighbouring reads on different warps, the long ones spread out.
 *  frames / look: kFrameCap / kLookCap entries per warp of the grid. */
template <unsigned NW>
__global__ void __launch_bounds__(kKonTrimThreads) k_kon_trim(const uint8_t* __restrict__ bases, const uint64_t* __restrict__ offs,
                                                             uint64_t n_reads, KonGeom g, KonView fv, unsigned min_branch_len,
                                                             Frame* __restrict__ frames, uint64_t* __restrict__ look,
                                                             uint32_t* __restrict__ left, uint32_t* __restrict__ right)
{
	const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32, n_warps = (uint64_t)gridDim.x * blockDim.x / 32;
	KonWarpCtx<NW> c;
	c.k = g.k;
	c.trim = min_branch_len;
	c.rt = g;
	c.fv = fv;
	c.lane = threadIdx.x & 31;
	c.frames = frames + warp * kFrameCap;
	c.look = look + warp * kLookCap;
	for (uint64_t t = warp; t < 2 * n_reads; t += n_warps) {
		const uint64_t r = t / 2, b0 = offs[r], len = offs[r + 1] - b0;
		uint32_t out = 0;
		if (len >= g.k) {
			c.fail_ = 0;
			c.chunk = 0xffffffffu;
			out = kon_left_trim<NW>(c, bases + b0, (unsigned)len, (t & 1) != 0);
		}
		if (c.lane == 0)
			(t & 1 ? right : left)[r] = out;
		__syncwarp();
	}
}
#endif

} // namespace abb
