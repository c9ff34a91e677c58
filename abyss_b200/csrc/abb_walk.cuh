// abb_walk.cuh -- Bloom-backed de Bruijn graph traversal (pass 2), warp-uniform.
//
// Replaces, for the RollingBloomDBG<CountingBloomFilter> instantiation only:
//   RollingBloomDBG out/in_edge iterators + vertex_exists     BloomDBG/RollingBloomDBG.h:302-436
//   lookAhead / trueBranch / successor / ambiguous            Graph/ExtendPath.h:99-397
//   extendPathBySingleVertex / extendPath                     Graph/ExtendPath.h:403-459,621-720
//   getContigType / preprocessCircularContig / trimBranchKmers / isTip   BloomDBG/bloom-dbg.h:622-776
//   the per-read loop of processRead                          BloomDBG/bloom-dbg.h:837-879
//
// Execution model: ONE WARP walks one seed read.  Every function below is executed by all 32
// lanes with identical ("uniform") arguments and control flow; lanes only diverge inside the Ctx
// primitives:  Ctx::neighbors() probes the 8 neighbour k-mers x H hash functions of a vertex with
// one lane per (neighbour, hash) pair -- one HBM round trip per graph step -- and the scratch
// helpers let lane 0 write while everybody reads.  Because all graph logic is uniform scalar code
// over a Ctx, tests/host_walk instantiates the very same templates with a trivial single-thread
// Ctx to debug the logic without a GPU (test infrastructure; the library never runs it).
//
// Vertex identity: the reference compares vertices by canonical hash AND canonical string
// (RollingBloomDBG.h:92-100, RC-invariant).  Here identity is the 64-bit canonical ntHash alone;
// two distinct k-mers colliding inside one local traversal has probability ~2^-64 per comparison.
// With a spaced seed (MaskedKmer) a vertex carries the masked Bloom hash and a separate identity (see "Spaced seeds" in
// DESIGN.md section 3).  Two k-mers with the same identity can then differ at a don't-care position and continue
// differently, so tiles are named by the full k-mer instead (tile_key), while everything the walk compares by vertex
// identity stays on the identity.
#pragma once
#include "abb_device.cuh"

namespace abb {

enum Dir : unsigned { FWD = 0, REV = 1 };
ABB_HD Dir opposite(Dir d) { return d == FWD ? REV : FWD; }

/** PathExtensionResultCode (Graph/ExtendPath.h:45-57) */
enum ExtCode : unsigned { ER_AMBI_IN = 0, ER_AMBI_OUT = 1, ER_DEAD_END = 2, ER_CYCLE = 3, ER_LENGTH_LIMIT = 4 };

/** ReadResult (BloomDBG/bloom-dbg.h:256-266), compacted */
enum ReadCode : uint8_t {
	RC_SHORTER_THAN_K = 0, RC_NON_ACGT = 1, RC_BLUNT_END = 2, RC_NOT_SOLID = 3, RC_ALL_KMERS_VISITED = 4,
	RC_GENERATED_CONTIGS = 5, RC_CANDIDATE = 6 /* internal: solid, not blunt, not yet decided */
};

constexpr unsigned kFpTrim = 5; // hard-coded in the reference (bloom-dbg.h:500,550,661,741,847)

// ------------------------------------------------------------------------------------------
// 2-bit packed k-mer: base i (0 = leftmost) lives at bits [2(k-1-i), 2(k-1-i)+1] of a KW*64-bit
// integer, w[0] least significant.  Appending a base is a 2-bit left shift.
// ------------------------------------------------------------------------------------------
template <int KW>
struct Kmer {
	uint64_t w[KW];
};

template <int KW>
ABB_HD unsigned kmer_last(const Kmer<KW>& km) { return (unsigned)(km.w[0] & 3); }

template <int KW>
ABB_HD unsigned kmer_base(const Kmer<KW>& km, unsigned k, unsigned i)
{
	const unsigned p = 2 * (k - 1 - i);
	uint64_t word = 0;
#pragma unroll
	for (int j = 0; j < KW; ++j)
		if ((unsigned)j == (p >> 6))
			word = km.w[j];
	return (unsigned)((word >> (p & 63)) & 3);
}
template <int KW>
ABB_HD unsigned kmer_first(const Kmer<KW>& km, unsigned k) { return kmer_base(km, k, 0); }

/** drop the first base, append b */
template <int KW>
ABB_HD void kmer_append(Kmer<KW>& km, unsigned k, unsigned b)
{
#pragma unroll
	for (int j = KW - 1; j > 0; --j)
		km.w[j] = (km.w[j] << 2) | (km.w[j - 1] >> 62);
	km.w[0] = (km.w[0] << 2) | b;
	// clear everything at and above bit 2k
	const unsigned top = 2 * k;
#pragma unroll
	for (int j = 0; j < KW; ++j) {
		const unsigned lo = 64u * j;
		if (top <= lo)
			km.w[j] = 0;
		else if (top < lo + 64)
			km.w[j] &= (1ULL << (top - lo)) - 1;
	}
}
/** drop the last base, prepend b */
template <int KW>
ABB_HD void kmer_prepend(Kmer<KW>& km, unsigned k, unsigned b)
{
#pragma unroll
	for (int j = 0; j < KW - 1; ++j)
		km.w[j] = (km.w[j] >> 2) | (km.w[j + 1] << 62);
	km.w[KW - 1] >>= 2;
	const unsigned p = 2 * (k - 1);
#pragma unroll
	for (int j = 0; j < KW; ++j)
		if ((unsigned)j == (p >> 6))
			km.w[j] |= (uint64_t)b << (p & 63);
}
template <int KW>
ABB_HD bool kmer_equal(const Kmer<KW>& a, const Kmer<KW>& b)
{
	bool eq = true;
#pragma unroll
	for (int j = 0; j < KW; ++j)
		eq &= a.w[j] == b.w[j];
	return eq;
}
/** MaskedKmer equality (Common/MaskedKmer.h:100-118): don't-care positions are not compared */
template <int KW>
ABB_HD bool kmer_equal_masked(const Kmer<KW>& a, const Kmer<KW>& b, unsigned k, const RollTab& rt)
{
	if (rt.nmask == 0)
		return kmer_equal(a, b);
	Kmer<KW> x;
#pragma unroll
	for (int j = 0; j < KW; ++j)
		x.w[j] = a.w[j] ^ b.w[j];
	for (unsigned j = 0; j < rt.nmask; ++j) { // clear the differences at the masked positions
		const unsigned p = 2 * (k - 1 - rt.mpos[j]);
#pragma unroll
		for (int w = 0; w < KW; ++w)
			if ((unsigned)w == (p >> 6))
				x.w[w] &= ~(3ULL << (p & 63));
	}
	bool eq = true;
#pragma unroll
	for (int j = 0; j < KW; ++j)
		eq &= x.w[j] == 0;
	return eq;
}

/** XOR of the hash terms of the masked positions (maskHash, BloomDBG/MaskedKmer... RollingHash.h:207-218 via
 *  nthash.hpp:417-436): position i holds base km[i + shift] (shift = +1 / -1: the k-mer after a step right / left,
 *  whose inner positions are all still present in km). */
template <int KW>
ABB_HD HashPair mask_corr(const Kmer<KW>& km, unsigned k, const RollTab& rt, int shift)
{
	HashPair c;
	c.fh = c.rh = 0;
	for (unsigned j = 0; j < rt.nmask; ++j) {
		const unsigned i = rt.mpos[j];
		const unsigned b = kmer_base(km, k, (unsigned)((int)i + shift));
		c.fh ^= srol_n(seed_of(b), k - 1 - i);
		c.rh ^= srol_n(seed_of(3 - b), i);
	}
	return c;
}
ABB_HD bool mask_is_care(const RollTab& rt, unsigned p)
{
	for (unsigned j = 0; j < rt.nmask; ++j)
		if (rt.mpos[j] == p)
			return false;
	return true;
}
/** pathToSeq (bloom-dbg.h:131-158) writes only the '1' positions of each vertex, so with a spaced seed column c of
 *  an n-vertex path stays 'N' when no vertex has a '1' over it.  The mask begins and ends with '1': only the columns
 *  n..k-2 of a path shorter than k-1 vertices can be affected. */
ABB_HD bool column_written(const RollTab& rt, unsigned k, unsigned n, unsigned c)
{
	if (rt.nmask == 0 || c < n || c + 1 >= k)
		return true;
	for (unsigned i = 0; i < n; ++i)
		if (mask_is_care(rt, c - i))
			return true;
	return false;
}
ABB_HD uint64_t masked_canon(const HashPair& h, const HashPair& corr)
{
	const uint64_t f = h.fh ^ corr.fh, r = h.rh ^ corr.rh;
	return r < f ? r : f;
}

/** reverse the 2-bit groups of a word */
ABB_HD uint64_t rev2_u64(uint64_t x)
{
	x = ((x >> 2) & 0x3333333333333333ULL) | ((x & 0x3333333333333333ULL) << 2);
	x = ((x >> 4) & 0x0F0F0F0F0F0F0F0FULL) | ((x & 0x0F0F0F0F0F0F0F0FULL) << 4);
	x = ((x >> 8) & 0x00FF00FF00FF00FFULL) | ((x & 0x00FF00FF00FF00FFULL) << 8);
	x = ((x >> 16) & 0x0000FFFF0000FFFFULL) | ((x & 0x0000FFFF0000FFFFULL) << 16);
	return (x >> 32) | (x << 32);
}
/** packed reverse complement */
template <int KW>
ABB_HD Kmer<KW> kmer_revcomp(const Kmer<KW>& km, unsigned k)
{
	Kmer<KW> r;
#pragma unroll
	for (int j = 0; j < KW; ++j)
		r.w[j] = ~rev2_u64(km.w[KW - 1 - j]); // complement of code c is 3 - c == ~c on two bits
	// the k-mer now sits in the top 2k bits: shift it down
	unsigned sh = 64u * KW - 2u * k;
	while (sh >= 64) {
#pragma unroll
		for (int j = 0; j < KW - 1; ++j)
			r.w[j] = r.w[j + 1];
		r.w[KW - 1] = 0;
		sh -= 64;
	}
	if (sh) {
#pragma unroll
		for (int j = 0; j < KW - 1; ++j)
			r.w[j] = (r.w[j] >> sh) | (r.w[j + 1] << (64 - sh));
		r.w[KW - 1] >>= sh;
	}
	return r;
}
/** LightweightKmer::isCanonical (BloomDBG/LightweightKmer.h:88-101): the k-mer is <= its reverse complement */
template <int KW>
ABB_HD bool kmer_is_canonical(const Kmer<KW>& km, unsigned k)
{
	const Kmer<KW> r = kmer_revcomp(km, k);
	for (int j = KW - 1; j >= 0; --j)
		if (km.w[j] != r.w[j])
			return km.w[j] < r.w[j];
	return true;
}

/** A vertex: k-mer + rolling hash state (RollingBloomDBGVertex, RollingBloomDBG.h:33-159).
 *  mh is the value the Bloom filters are probed with (RollingHash::m_hash).  id is what vertex *identity* is decided
 *  on (operator==, RollingBloomDBG.h:92-158): without a spaced seed the canonical hash again; with one, operator==
 *  compares the '1' positions of the two k-mers after orienting each by its FULL k-mer (isCanonical looks at the
 *  don't-care positions too), so two k-mers that agree on every '1' position can still be different vertices.  That
 *  relation is exactly "equal masked forward hash of the full-canonical orientation", which is what id holds. */
template <int KW>
struct Vtx {
	Kmer<KW> km;
	HashPair h;  // unmasked rolling state
	uint64_t mh;
	uint64_t id;
	ABB_HD uint64_t canon() const { return id; }
	ABB_HD uint64_t bloom() const { return mh; }
};
/** spaced seed only; not inlined: the unmasked walk, which never gets here, stays as small as it was */
template <int KW>
ABB_HD_NOINLINE void vtx_rehash_masked(Vtx<KW>& v, unsigned k, const RollTab& rt)
{
	const HashPair c = mask_corr(v.km, k, rt, 0);
	const uint64_t f = v.h.fh ^ c.fh, r = v.h.rh ^ c.rh;
	v.mh = r < f ? r : f;
	v.id = kmer_is_canonical(v.km, k) ? f : r;
}
template <int KW>
ABB_HD void vtx_rehash(Vtx<KW>& v, unsigned k, const RollTab& rt)
{
	if (rt.nmask == 0)
		v.mh = v.id = v.h.canonical();
	else
		vtx_rehash_masked(v, k, rt);
}
/** Bloom hash of the neighbour of v in direction d with new base b, without building its k-mer */
template <int KW>
ABB_HD_NOINLINE uint64_t neighbor_bloom_masked(const HashPair& h, const Kmer<KW>& km, unsigned k, const RollTab& rt, int shift)
{
	return masked_canon(h, mask_corr(km, k, rt, shift));
}
template <int KW>
ABB_HD uint64_t neighbor_bloom(const Vtx<KW>& v, unsigned k, const RollTab& rt, Dir d, unsigned b)
{
	const HashPair h = d == FWD ? roll_right(v.h, rt, kmer_first(v.km, k), b) : roll_left(v.h, rt, kmer_last(v.km), b);
	if (rt.nmask == 0)
		return h.canonical();
	return neighbor_bloom_masked(h, v.km, k, rt, d == FWD ? 1 : -1);
}
template <int KW>
ABB_HD unsigned vtx_step(Vtx<KW>& v, unsigned k, const RollTab& rt, Dir d, unsigned b);
/** identity of that neighbour */
template <int KW>
ABB_HD uint64_t neighbor_canon(const Vtx<KW>& v, unsigned k, const RollTab& rt, Dir d, unsigned b)
{
	if (rt.nmask == 0)
		return neighbor_bloom(v, k, rt, d, b);
	Vtx<KW> t = v;
	vtx_step(t, k, rt, d, b);
	return t.id;
}

/** Move to the neighbour in direction d with new base b; returns the base that fell off.
 *  (vertex.shift + setLastBase, RollingBloomDBG.h:56-70; RollingHash.h:88-128,175-193) */
template <int KW>
ABB_HD unsigned vtx_step(Vtx<KW>& v, unsigned k, const RollTab& rt, Dir d, unsigned b)
{
	unsigned out;
	if (d == FWD) {
		out = kmer_first(v.km, k);
		v.h = roll_right(v.h, rt, out, b);
		kmer_append(v.km, k, b);
	} else {
		out = kmer_last(v.km);
		v.h = roll_left(v.h, rt, out, b);
		kmer_prepend(v.km, k, b);
	}
	vtx_rehash(v, k, rt);
	return out;
}
/** undo a vtx_step(d, .) that dropped `out` */
template <int KW>
ABB_HD void vtx_unstep(Vtx<KW>& v, unsigned k, const RollTab& rt, Dir d, unsigned out)
{
	vtx_step(v, k, rt, opposite(d), out);
}

/** vertex of the k bases at s[0..k) given as 2-bit codes (NTC64 from scratch, nthash.hpp:220-239) */
template <int KW>
ABB_HD Vtx<KW> vtx_from_codes(const uint8_t* s, unsigned k, bool ascii, const RollTab& rt)
{
	Vtx<KW> v;
#pragma unroll
	for (int j = 0; j < KW; ++j)
		v.km.w[j] = 0;
	v.h.fh = v.h.rh = 0;
	for (unsigned i = 0; i < k; ++i) {
		const unsigned c = ascii ? base_code(s[i]) : s[i];
		kmer_append(v.km, k, c & 3);
		v.h.fh = srol1(v.h.fh) ^ seed_of(c);
	}
	for (unsigned i = 0; i < k; ++i) {
		const unsigned c = ascii ? base_code(s[k - 1 - i]) : s[k - 1 - i];
		v.h.rh = srol1(v.h.rh) ^ seed_of(3 - c);
	}
	vtx_rehash(v, k, rt);
	return v;
}

/** reverse complement (RollingBloomDBGVertex::reverseComplement, RollingBloomDBG.h:72-76) */
template <int KW>
ABB_HD Vtx<KW> vtx_revcomp(const Vtx<KW>& v, unsigned k)
{
	Vtx<KW> r;
	r.km = kmer_revcomp(v.km, k);
	r.h.fh = v.h.rh;
	r.h.rh = v.h.fh;
	r.mh = v.mh; // the mask is symmetric
	r.id = v.id;
	return r;
}

// ------------------------------------------------------------------------------------------
// Scratch layouts (per warp, in global memory)
// ------------------------------------------------------------------------------------------
/** one active trueBranch() call (Graph/ExtendPath.h:173-244) */
struct Frame {
	uint64_t hv;   // canonical hash of this call's vertex v (the "visited" set is the stack)
	uint64_t meta; // see pack/unpack below
};
constexpr unsigned kFrameCap = 4096;  // trueBranch recursion depth bound per warp
constexpr unsigned kLookCap = 2048;   // lookAhead visited-list bound per warp (<= 1 + 4 + .. + 4^5 = 1365)

ABB_HD uint64_t frame_pack(unsigned dir, unsigned phase, unsigned depth, unsigned omask, unsigned imask, unsigned enter_dir,
                           unsigned dropped)
{
	return (uint64_t)dir | ((uint64_t)phase << 1) | ((uint64_t)omask << 3) | ((uint64_t)imask << 7) |
	       ((uint64_t)enter_dir << 11) | ((uint64_t)dropped << 12) | ((uint64_t)depth << 16);
}
struct FrameView {
	unsigned dir, phase, omask, imask, enter_dir, dropped, depth;
};
ABB_HD FrameView frame_unpack(uint64_t m)
{
	FrameView f;
	f.dir = (unsigned)(m & 1);
	f.phase = (unsigned)((m >> 1) & 3);
	f.omask = (unsigned)((m >> 3) & 15);
	f.imask = (unsigned)((m >> 7) & 15);
	f.enter_dir = (unsigned)((m >> 11) & 1);
	f.dropped = (unsigned)((m >> 12) & 3);
	f.depth = (unsigned)(m >> 16);
	return f;
}

ABB_HD unsigned ctz4(unsigned m) { return (m & 1) ? 0 : (m & 2) ? 1 : (m & 4) ? 2 : 3; }

/** Why a walk was abandoned: the value handed to Ctx::fail().  A context that reports to the host (WarpCtx, KonCtx) keeps
 *  the set of reasons as a mask of walk_fail_bit(); k_extend stores that mask as the read's status, 0 = walked to the end. */
enum WalkFail : unsigned {
	WALK_FAIL_NO_CODE = 0,     // k_extend only: the walk returned "not ok" although no fail() was recorded
	WALK_FAIL_LOOK_FULL = 1,   // lookAhead visited more than kLookCap vertices
	WALK_FAIL_FRAMES_FULL = 2, // trueBranch recursed deeper than kFrameCap frames
	WALK_FAIL_ARENA = 3,       // Ctx::alloc found the unitig arena exhausted
	WALK_FAIL_TILE_CYCLE = 4,  // the tile chain came back to a tile already spliced: walk this read vertex by vertex
};
ABB_HD constexpr unsigned walk_fail_bit(WalkFail why) { return 1u << why; }

/**
 * Ctx concept (device: WarpCtx in abb_assemble.cu; host emulation: tests/host_walk):
 *   unsigned k, trim; RollTab rt;
 *   template<int KW> unsigned neighbors(const Vtx<KW>&)   bits 0-3: out-neighbours A,C,G,T exist; 4-7: in-neighbours
 *   Probe neighbors_issue(v) / unsigned neighbors_finish(Probe)   the same, split so that other loads can be in flight
 *   unsigned neighbors_dir(v, dir)   4-bit mask of the neighbours in one direction only (half the probes; lookAhead)
 *   uint64_t rd64(const uint64_t*), void wr64(uint64_t*, uint64_t), uint8_t rd8(const uint8_t*), void wr8(uint8_t*, uint8_t)
 *   void sync()                      make lane-0 writes visible to the warp
 *   bool find64(const uint64_t* a, unsigned n, uint64_t key, unsigned stride_words)   cooperative linear search
 *   uint8_t* alloc(uint64_t bytes)   arena bump allocation, zero-filled iff zero==true; nullptr when exhausted
 *   void fail(unsigned why), bool failed()   record why (a WalkFail) the walk of this read is abandoned; the host retries it
 *   void copy8(dst, src, n), copy8_rev(dst, src, n)   cooperative byte copies (rev: dst[i] = src[n-1-i])
 *   void rehash(old, oldcap, new, newcap)              cooperative PathSet growth
 *   bool tiles_enabled(); const TileRec* tile_lookup(key, cls); const TileRec* tile_at(idx); void prefetch(const void*);
 *   uint32_t tile_index(const TileRec*); void wr32(uint32_t*, uint32_t)
 *   void mark_covered(ps, rh, cov, nk, contig)         cooperative: flag read k-mers that lie on the contig path
 *   Frame* frames; uint64_t* look;   per-warp scratch
 *
 * lookAhead / trueBranch / successor below are templates over the vertex type V as well: they reach a vertex only through
 * vtx_step / vtx_unstep (found by argument-dependent lookup), V::canon() (vertex identity) and the context's neighbors*;
 * `c.rt` is whatever the vertex's vtx_step takes as its third argument.  Vtx<KW> (ntHash, identity up to reverse
 * complement) is the vertex of abyss-bloom-dbg; KonVtx (abb_konnector.cuh: exact, strand-specific) that of abyss-bloom trim.
 */

// ------------------------------------------------------------------------------------------
// lookAhead (Graph/ExtendPath.h:99-161): bounded DFS with a permanent visited set
// ------------------------------------------------------------------------------------------
template <class V, class Ctx>
ABB_HD bool look_ahead(Ctx& c, const V& start, Dir dir, unsigned limit)
{
	unsigned nvis = 0;
	c.wr64(c.look + nvis++, start.canon()); // visited.insert(u)
	if (limit == 0)
		return true;
	V cur = start;
	// explicit stack, depth <= limit <= 8: remaining-neighbour mask and dropped base per level
	unsigned masks[8], dropped[8];
	unsigned sp = 0;
	{
		masks[0] = c.neighbors_dir(cur, dir);
		dropped[0] = 0;
		sp = 1;
	}
	c.sync();
	while (sp > 0) {
		unsigned& m = masks[sp - 1];
		if (m == 0) {
			--sp;
			if (sp > 0)
				vtx_unstep(cur, c.k, c.rt, dir, dropped[sp]);
			continue;
		}
		const unsigned b = ctz4(m);
		m &= m - 1;
		const unsigned out = vtx_step(cur, c.k, c.rt, dir, b);
		const uint64_t hv = cur.canon();
		if (c.find64(c.look, nvis, hv, 1)) { // already visited
			vtx_unstep(cur, c.k, c.rt, dir, out);
			continue;
		}
		if (nvis >= kLookCap) {
			c.fail(WALK_FAIL_LOOK_FULL);
			return true;
		}
		c.wr64(c.look + nvis++, hv);
		c.sync();
		if (sp >= limit) // depth of cur == sp
			return true;
		dropped[sp] = out;
		masks[sp] = c.neighbors_dir(cur, dir);
		++sp;
	}
	return false;
}

// ------------------------------------------------------------------------------------------
// trueBranch (Graph/ExtendPath.h:173-261), iterative; the DFS stack doubles as `visited`
// ------------------------------------------------------------------------------------------
template <class V, class Ctx>
ABB_HD bool true_branch(Ctx& c, const V& u, Dir dir, unsigned base, unsigned trim_i)
{
	if (trim_i == 0) // "depth >= trim" with an empty visited set
		return true;
	V cur = u;
	const uint64_t hu_top = u.canon();
	unsigned out = vtx_step(cur, c.k, c.rt, dir, base);
	unsigned sp = 0;
	{
		const unsigned m = c.neighbors(cur);
		c.wr64(&c.frames[0].hv, cur.canon());
		c.wr64(&c.frames[0].meta, frame_pack(dir, 0, 0, m & 15, m >> 4, dir, out));
		sp = 1;
		c.sync();
	}
	while (sp > 0) {
		Frame* F = &c.frames[sp - 1];
		FrameView f = frame_unpack(c.rd64(&F->meta));
		const Dir fdir = (Dir)f.dir;
		if (f.phase == 0) {
			unsigned m = fdir == FWD ? f.omask : f.imask;
			if (m != 0) {
				const unsigned b = ctz4(m);
				m &= m - 1;
				if (fdir == FWD)
					f.omask = m;
				else
					f.imask = m;
				c.wr64(&F->meta, frame_pack(f.dir, 0, f.depth, f.omask, f.imask, f.enter_dir, f.dropped));
				out = vtx_step(cur, c.k, c.rt, fdir, b);
				const uint64_t hv = cur.canon();
				// trueBranch(edge, depth + 1, same dir): visited? deep enough?
				if (c.find64(&c.frames[0].hv, sp, hv, 2) || f.depth + 1 >= trim_i)
					return true;
				if (sp >= kFrameCap) {
					c.fail(WALK_FAIL_FRAMES_FULL);
					return true;
				}
				const unsigned nm = c.neighbors(cur);
				c.wr64(&c.frames[sp].hv, hv);
				c.wr64(&c.frames[sp].meta, frame_pack(f.dir, 0, f.depth + 1, nm & 15, nm >> 4, f.dir, out));
				++sp;
				c.sync();
				continue;
			}
			// no more same-direction neighbours: decide whether to turn around (ExtendPath.h:206,227)
			const bool turn = f.depth >= kFpTrim || look_ahead(c, cur, fdir, kFpTrim);
			if (!turn) { // visited.erase(v); return false
				vtx_unstep(cur, c.k, c.rt, (Dir)f.enter_dir, f.dropped);
				--sp;
				continue;
			}
			f.phase = 2;
			c.wr64(&F->meta, frame_pack(f.dir, 2, f.depth, f.omask, f.imask, f.enter_dir, f.dropped));
			c.sync();
		}
		// phase 2: edges in the opposite direction, skipping the vertex we came from
		{
			const Dir od = opposite(fdir);
			unsigned m = od == FWD ? f.omask : f.imask;
			if (m == 0) { // visited.erase(v); return false
				vtx_unstep(cur, c.k, c.rt, (Dir)f.enter_dir, f.dropped);
				--sp;
				continue;
			}
			const unsigned b = ctz4(m);
			m &= m - 1;
			if (od == FWD)
				f.omask = m;
			else
				f.imask = m;
			c.wr64(&F->meta, frame_pack(f.dir, 2, f.depth, f.omask, f.imask, f.enter_dir, f.dropped));
			out = vtx_step(cur, c.k, c.rt, od, b);
			const uint64_t hv = cur.canon();
			const uint64_t hu = sp >= 2 ? c.rd64(&c.frames[sp - 2].hv) : hu_top;
			if (hv == hu) { // "if (source(*iei, g) == u) continue"
				vtx_unstep(cur, c.k, c.rt, od, out);
				c.sync();
				continue;
			}
			// trueBranch(edge, 0, opposite dir); trim_i >= 1 here
			if (c.find64(&c.frames[0].hv, sp, hv, 2))
				return true;
			if (sp >= kFrameCap) {
				c.fail(WALK_FAIL_FRAMES_FULL);
				return true;
			}
			const unsigned nm = c.neighbors(cur);
			c.wr64(&c.frames[sp].hv, hv);
			c.wr64(&c.frames[sp].meta, frame_pack(od, 0, 0, nm & 15, nm >> 4, od, out));
			++sp;
			c.sync();
		}
	}
	return false;
}

// ------------------------------------------------------------------------------------------
// successor (Graph/ExtendPath.h:314-362)
// ------------------------------------------------------------------------------------------
/** nbmask = c.neighbors(u).  Returns the result code; *vbase = base of the last true branch seen */
template <class V, class Ctx>
ABB_HD ExtCode successor(Ctx& c, const V& u, unsigned nbmask, Dir dir, unsigned* vbase)
{
	const unsigned m = dir == FWD ? (nbmask & 15) : (nbmask >> 4);
	// i = 0: every existing neighbour is a true branch (depth 0 >= trim 0), so the count is the degree
	if (m == 0)
		return ER_DEAD_END;
	if ((m & (m - 1)) == 0) {
		*vbase = ctz4(m);
		return ER_LENGTH_LIMIT;
	}
	if (c.trim == 0) {
		*vbase = ctz4(m & (m - 1)); // the second true branch is the one left in `v`
		return ER_AMBI_OUT;
	}
	for (unsigned i = 1;; i = (2 * i < c.trim ? 2 * i : c.trim)) {
		unsigned cnt = 0;
		for (unsigned mm = m; mm; mm &= mm - 1) {
			const unsigned b = ctz4(mm);
			if (true_branch(c, u, dir, b, i)) {
				*vbase = b;
				if (++cnt >= 2)
					break;
			}
		}
		if (cnt == 0)
			return ER_DEAD_END;
		if (cnt == 1)
			return ER_LENGTH_LIMIT;
		if (i == c.trim)
			return ER_AMBI_OUT;
	}
}

/** ambiguous(u, dir) (ExtendPath.h:368-375) */
template <int KW, class Ctx>
ABB_HD bool ambiguous(Ctx& c, const Vtx<KW>& u, Dir dir)
{
	unsigned b = 0;
	return successor(c, u, c.neighbors(u), dir, &b) == ER_AMBI_OUT;
}
/** ambiguous(u, expected, dir) (ExtendPath.h:384-397) */
template <int KW, class Ctx>
ABB_HD bool ambiguous_expected(Ctx& c, const Vtx<KW>& u, uint64_t expected_canon, Dir dir)
{
	unsigned b = 0;
	const ExtCode r = successor(c, u, c.neighbors(u), dir, &b);
	if (r == ER_AMBI_OUT)
		return true;
	if (r == ER_LENGTH_LIMIT) {
		Vtx<KW> v = u;
		vtx_step(v, c.k, c.rt, dir, b);
		return v.canon() != expected_canon;
	}
	return false;
}

// ------------------------------------------------------------------------------------------
// exact set of the canonical hashes of the path vertices (extendPath's `visited`, ExtendPath.h:699-703)
// open addressing in arena memory, doubled when more than 1/2 full; key 0 is tracked separately
// ------------------------------------------------------------------------------------------
struct PathSet {
	uint64_t* tab;
	unsigned cap; // power of two
	unsigned n;
	bool has_zero;
};

ABB_HD uint64_t pathset_slot(uint64_t key, unsigned cap) { return ((key * 0x9E3779B97F4A7C15ULL) >> 24) & (cap - 1); }

template <class Ctx>
ABB_HD bool pathset_init(Ctx& c, PathSet& ps, unsigned cap)
{
	ps.tab = (uint64_t*)c.alloc((uint64_t)cap * 8, true);
	ps.cap = cap;
	ps.n = 0;
	ps.has_zero = false;
	return ps.tab != nullptr;
}
template <class Ctx>
ABB_HD bool pathset_contains(Ctx& c, const PathSet& ps, uint64_t key)
{
	if (key == 0)
		return ps.has_zero;
	for (uint64_t s = pathset_slot(key, ps.cap);; s = (s + 1) & (ps.cap - 1)) {
		const uint64_t v = c.rd64(ps.tab + s);
		if (v == key)
			return true;
		if (v == 0)
			return false;
	}
}
/** returns true if newly inserted; *ok = false on arena exhaustion */
template <class Ctx>
ABB_HD bool pathset_insert(Ctx& c, PathSet& ps, uint64_t key, bool* ok)
{
	if (key == 0) {
		const bool fresh = !ps.has_zero;
		ps.has_zero = true;
		return fresh;
	}
	// every lane must read the slot before any lane writes the key there, or a late lane finds the key and reports a
	// cycle: extend_dir calls this between Ctx::neighbors_issue and neighbors_finish, where the lanes need not be
	// converged (with H < 4 some lanes issue no probe and run ahead)
	c.sync();
	if ((ps.n + 1) * 2 > ps.cap) { // grow: re-insert everything into a table twice the size
		PathSet big;
		if (!pathset_init(c, big, ps.cap * 2)) {
			*ok = false;
			return false;
		}
		big.has_zero = ps.has_zero;
		c.rehash(ps.tab, ps.cap, big.tab, big.cap); // cooperative re-insert of every non-zero entry
		big.n = ps.n;
		ps = big;
	}
	for (uint64_t s = pathset_slot(key, ps.cap);; s = (s + 1) & (ps.cap - 1)) {
		const uint64_t v = c.rd64(ps.tab + s);
		if (v == key)
			return false;
		if (v == 0) {
			c.wr64(ps.tab + s, key);
			c.sync();
			++ps.n;
			return true;
		}
	}
}

/** growable byte vector in arena memory (bases appended during an extension) */
struct ByteVec {
	uint8_t* p;
	unsigned cap, n;
};
template <class Ctx>
ABB_HD bool bytevec_push(Ctx& c, ByteVec& v, uint8_t x)
{
	if (v.n == v.cap) {
		const unsigned ncap = v.cap ? v.cap * 2 : 1024;
		uint8_t* np = c.alloc(ncap, false);
		if (!np)
			return false;
		c.copy8(np, v.p, v.n);
		v.p = np;
		v.cap = ncap;
	}
	c.wr8(v.p + v.n, x);
	++v.n;
	return true;
}

// ------------------------------------------------------------------------------------------
// Tiles: marker-to-marker path segments computed once, in parallel, and spliced by the walks.
//
// A unitig walk is a chain of dependent steps (Mbp-long unitigs = seconds of latency).  The step
// taken at a head h depends only on h and on the canonical hash of the previous head p:
//     look-behind  LB(h, d) = successor(h, opposite d)   must be (LENGTH_LIMIT, t) with t == p
//     next         NX(h, d) = successor(h, d)            must be (LENGTH_LIMIT, v); v becomes the head
// (extendPathBySingleVertex, ExtendPath.h:403-459; the start vertex of an extension skips LB).
// Vertices whose canonical hash has its low bits clear are MARKERS.  For every marker m, held
// orientation o and direction d, tile(m, o, d) is exactly the walk extendPath would do from the
// start vertex m -- no LB at m, LB at every later head -- cut when it pushes another marker (or
// stops for a graph reason, or after kTileCap pushes), together with LB(m, d) itself.  A walk that
// arrives at m from p applies the stored LB(m) to p, appends the tile, and continues at the tile's
// end marker with the tile's own last predecessor: by construction the result is what stepping
// vertex by vertex would have produced.  The visited set is not consulted while splicing; instead
// every finished path is checked for a repeated vertex afterwards and, if one is found (cycles,
// hairpins: rare), that read is walked again without tiles.
//
// Markers and tiles are named by tile_key(): the canonical hash of the FULL k-mer.  A walk from a
// vertex is a function of its full k-mer, the strand held, the direction and the read-only solid
// filter, so that name is exact (up to the ~2^-64 hash collision).  Without a spaced seed it is the
// vertex identity canon(); with one, canon() ignores the don't-care positions, and two k-mers that
// agree on every '1' position but continue differently would share a tile.  The look-behind
// hashes, the per-vertex hashes a tile stores and the path set stay canon().
// ------------------------------------------------------------------------------------------
constexpr uint64_t kMarkerMask = 255;   // 1 vertex in 256 is a marker
constexpr unsigned kTileCap = 4096;     // longest tile, in pushed vertices
enum TileStop : uint8_t { TS_MARKER = 0, TS_CODE = 1, TS_CAP = 2 };

ABB_HD bool is_marker(uint64_t key) { return (key & kMarkerMask) == 0; }

/** what tiles and markers are named by: the canonical ntHash of the full k-mer (see above) */
template <int KW>
ABB_HD uint64_t tile_key(const Vtx<KW>& v, const RollTab& rt)
{
	return rt.nmask == 0 ? v.id : v.h.canonical();
}

/** the set of markers that already have tiles: open addressing over mask + 1 entries of 64-bit keys, 0 = empty */
constexpr unsigned kMarkerProbes = 64; // probe bound: a full set answers MARKER_NO_ROOM instead of probing forever
enum MarkerInsert : unsigned { MARKER_SEEN = 0, MARKER_FRESH = 1, MARKER_NO_ROOM = 2 };

/** enter marker `canon` into the set.  Exactly one caller per key gets MARKER_FRESH (and makes its tiles).  A key that
 *  finds neither itself nor a free entry within kMarkerProbes probes gets MARKER_NO_ROOM and stays without tiles; walks
 *  pass it vertex by vertex.  Entries are never removed and a key is only ever stored within kMarkerProbes entries of
 *  its home slot, so the bound cannot hide a stored key: a key is fresh at most once. */
ABB_HD unsigned marker_set_insert(unsigned long long* set, unsigned mask, uint64_t canon)
{
	const unsigned long long key = canon ? canon : 1; // 0 marks an empty entry; 1 is no marker, so no marker collides with it
	uint64_t t = pathset_slot(key, mask + 1);
	for (unsigned i = 0; i < kMarkerProbes; ++i, t = (t + 1) & mask) {
#if defined(__CUDA_ARCH__)
		const unsigned long long old = atomicCAS(set + t, 0ULL, key);
#else
		unsigned long long old = 0;
		__atomic_compare_exchange_n(set + t, &old, key, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
#endif
		if (old == 0ULL)
			return MARKER_FRESH;
		if (old == key)
			return MARKER_SEEN;
	}
	return MARKER_NO_ROOM;
}

/** key, end_key, cls and end_orient name vertices as tiles do (tile_key: the full k-mer); lb_t, prev_last and hashes are
 *  vertex identities (canon()), compared with what the walk holds.  Without a spaced seed the two are the same value. */
struct TileRec {
	uint64_t key;        // tile_key of the marker
	uint64_t lb_t;       // canon() of LB's unique predecessor (valid if lb_code == ER_LENGTH_LIMIT)
	uint64_t prev_last;  // canon() of the vertex before the last pushed one (the marker itself if n == 1)
	uint64_t end_key;    // tile_key of the last pushed vertex
	uint8_t* bases;      // n pushed bases, in push order
	uint64_t* hashes;    // n canon() of the pushed vertices
	uint32_t n;
	uint32_t next;       // index + 1 of the tile that starts at this tile's end marker (same direction), 0 = look it up
	uint8_t cls;         // vtx_class of the marker as held: (strand of the full canonical k-mer) << 1 | direction
	uint8_t lb_code;     // ExtCode of LB(marker)
	uint8_t stop_kind;   // TileStop
	uint8_t stop_code;   // ExtCode when stop_kind == TS_CODE
	uint8_t end_orient;  // vtx_orient of the last pushed vertex
	uint8_t pad[3];
};

/** 1 if the held strand is the one whose unmasked forward hash is tile_key, i.e. the strand of the full canonical k-mer */
template <int KW>
ABB_HD unsigned vtx_orient(const Vtx<KW>& v) { return v.h.fh <= v.h.rh ? 1u : 0u; }
template <int KW>
ABB_HD unsigned vtx_class(const Vtx<KW>& v, Dir d) { return (vtx_orient(v) << 1) | (unsigned)d; }

/** growable vector of tile indices (arena memory) */
struct U32Vec {
	uint32_t* p;
	unsigned cap, n;
};
template <class Ctx>
ABB_HD bool u32vec_push(Ctx& c, U32Vec& v, uint32_t x)
{
	if (v.n == v.cap) {
		const unsigned ncap = v.cap ? v.cap * 2 : 256;
		uint32_t* np = (uint32_t*)c.alloc((uint64_t)ncap * 4, false);
		if (!np)
			return false;
		c.copy8((uint8_t*)np, (const uint8_t*)v.p, v.n * 4);
		v.p = np;
		v.cap = ncap;
	}
	c.wr32(v.p + v.n, x);
	++v.n;
	return true;
}
/** append n bytes */
template <class Ctx>
ABB_HD bool bytevec_append(Ctx& c, ByteVec& v, const uint8_t* src, unsigned n)
{
	if (v.n + n > v.cap) {
		unsigned ncap = v.cap ? v.cap : 1024;
		while (ncap < v.n + n)
			ncap *= 2;
		uint8_t* np = c.alloc(ncap, false);
		if (!np)
			return false;
		c.copy8(np, v.p, v.n);
		v.p = np;
		v.cap = ncap;
	}
	c.copy8(v.p + v.n, src, n);
	v.n += n;
	return true;
}

/** the end vertex of an extension that started at `start` and pushed the bases in `v` (direction d) */
template <int KW, class Ctx>
ABB_HD Vtx<KW> rebuild_head(Ctx& c, const Vtx<KW>& start, const ByteVec& v, unsigned from, Dir d)
{
	const unsigned k = c.k;
	Vtx<KW> h = start;
	const unsigned pushed = v.n - from;
	if (pushed >= k) {
		// the last k pushed bases spell the vertex (REV pushes prepend: newest base first)
		uint8_t tmp[KW > 6 ? 32 * KW : 192]; // the k bases; 192 bytes up to six words keeps those instances' stack frames
		for (unsigned i = 0; i < k; ++i)
			tmp[i] = d == FWD ? c.rd8(v.p + v.n - k + i) : c.rd8(v.p + v.n - 1 - i);
		return vtx_from_codes<KW>(tmp, k, false, c.rt);
	}
	for (unsigned i = from; i < v.n; ++i)
		vtx_step(h, k, c.rt, d, c.rd8(v.p + i));
	return h;
}

/**
 * tile(m, orientation of m as held, dir): see the block comment above.  bases/hashes are staging
 * buffers of kTileCap entries owned by the calling warp.
 */
template <int KW, class Ctx>
ABB_HD void make_tile(Ctx& c, const Vtx<KW>& m, Dir dir, TileRec* t, uint8_t* bases, uint64_t* hashes)
{
	Vtx<KW> head = m;
	unsigned nb = c.neighbors(head);
	unsigned b = 0;
	{ // LB(m, dir), consulted by whoever arrives at m
		const ExtCode lb = successor(c, head, nb, opposite(dir), &b);
		t->lb_code = (uint8_t)lb;
		t->lb_t = 0;
		if (lb == ER_LENGTH_LIMIT) {
			t->lb_t = neighbor_canon(head, c.k, c.rt, opposite(dir), b);
		}
	}
	t->key = tile_key(m, c.rt);
	t->next = 0;
	t->cls = (uint8_t)vtx_class(m, dir);
	unsigned n = 0;
	uint64_t prev_h = 0;
	bool look_behind = false;
	t->stop_kind = TS_CAP;
	t->stop_code = 0;
	for (;;) {
		if (look_behind) {
			const ExtCode r = successor(c, head, nb, opposite(dir), &b);
			if (r == ER_AMBI_OUT || r == ER_DEAD_END) {
				t->stop_kind = TS_CODE;
				t->stop_code = (uint8_t)ER_AMBI_IN;
				break;
			}
			if (neighbor_canon(head, c.k, c.rt, opposite(dir), b) != prev_h) {
				t->stop_kind = TS_CODE;
				t->stop_code = (uint8_t)ER_AMBI_IN;
				break;
			}
		}
		const ExtCode r = successor(c, head, nb, dir, &b);
		if (r != ER_LENGTH_LIMIT) {
			t->stop_kind = TS_CODE;
			t->stop_code = (uint8_t)r;
			break;
		}
		prev_h = head.canon();
		vtx_step(head, c.k, c.rt, dir, b);
		c.wr8(bases + n, (uint8_t)b);
		c.wr64(hashes + n, head.canon());
		++n;
		look_behind = true;
		if (is_marker(tile_key(head, c.rt))) {
			t->stop_kind = TS_MARKER;
			break;
		}
		if (n >= kTileCap || c.failed()) {
			t->stop_kind = TS_CAP;
			break;
		}
		nb = c.neighbors(head);
	}
	t->n = n;
	t->prev_last = prev_h;
	t->end_key = tile_key(head, c.rt);
	t->end_orient = (uint8_t)vtx_orient(head);
}

// ------------------------------------------------------------------------------------------
// extendPath in one direction (Graph/ExtendPath.h:403-459,621-681) with ExtendPathParams
// {trimLen = trim, fpTrim = 5, maxLen = NO_LIMIT, lookBehind = true, lookBehindStartVertex = false}
// (bloom-dbg.h:845-850).
//   head      in: the end vertex of the path in direction dir; out: the new end vertex
//   psize     in/out: number of vertices in the path
//   bases     receives the new base of every vertex pushed (in push order)
// ------------------------------------------------------------------------------------------
template <int KW, class Ctx>
ABB_HD ExtCode extend_dir(Ctx& c, Vtx<KW>& head, Dir dir, unsigned* psize, ByteVec& bases, PathSet& ps, bool* ok, U32Vec& tiles)
{
	bool look_behind = false; // lookBehindStartVertex
	uint64_t prev_h = 0;
	const Vtx<KW> start = head;
	// Brent cycle detection over the chain of spliced tiles (a circular unitig chains for ever)
	uint32_t brent_tortoise = 0xffffffffu;
	unsigned brent_power = 1, brent_lam = 0;
	unsigned nb = c.neighbors(head);
	for (;;) {
		unsigned b = 0;
		if (look_behind) { // extendPathBySingleVertex, ExtendPath.h:419-446
			const ExtCode r = successor(c, head, nb, opposite(dir), &b);
			if (r == ER_AMBI_OUT)
				return ER_AMBI_IN;
			if (*psize > 1) {
				if (r == ER_DEAD_END)
					return ER_AMBI_IN;
				// canonical hash of the unique predecessor t (hash only: no need to build its k-mer)
				if (neighbor_canon(head, c.k, c.rt, opposite(dir), b) != prev_h) // we are on a tip rejoining the graph
					return ER_AMBI_IN;
			}
		}
		const ExtCode r = successor(c, head, nb, dir, &b);
		if (r != ER_LENGTH_LIMIT)
			return r;
		const uint64_t old_h = head.canon();
		const unsigned out = vtx_step(head, c.k, c.rt, dir, b);
		// issue the Bloom probes of the new head before the visited-set probe so that the two
		// memory round trips of a step overlap
		const typename Ctx::Probe pr = c.neighbors_issue(head);
		if (!pathset_insert(c, ps, head.canon(), ok)) { // visited.insert(head) failed: ER_CYCLE, pop
			vtx_unstep(head, c.k, c.rt, dir, out);
			return *ok ? ER_CYCLE : ER_DEAD_END;
		}
		if (!bytevec_push(c, bases, (uint8_t)b)) { // FWD: the new last base; REV: the new first base
			*ok = false;
			return ER_DEAD_END;
		}
		++*psize;
		prev_h = old_h;
		look_behind = true; // params.lookBehind
		if (c.failed())
			return ER_DEAD_END;
		if (c.tiles_enabled() && is_marker(tile_key(head, c.rt))) {
			// splice marker-to-marker tiles for as long as they chain (see the Tiles comment above)
			uint64_t hk = tile_key(head, c.rt);
			unsigned cls = vtx_class(head, dir);
			bool moved = false;
			const TileRec* T = c.tile_lookup(hk, cls);
			while (T) {
				// extendPathBySingleVertex's look-behind at this marker, from the stored LB
				if (T->lb_code != ER_LENGTH_LIMIT || T->lb_t != prev_h) {
					if (moved)
						head = rebuild_head(c, start, bases, 0, dir);
					return ER_AMBI_IN;
				}
				const unsigned n = T->n;
				// where the chain goes next is known before the bases are copied: start fetching that record now
				const TileRec* Tn = nullptr;
				if (T->stop_kind == TS_MARKER && n) {
					Tn = T->next ? c.tile_at(T->next - 1) : c.tile_lookup(T->end_key, ((unsigned)T->end_orient << 1) | (unsigned)dir);
					c.prefetch(Tn);
				}
				if (n) {
					const uint32_t ti = c.tile_index(T);
					if (ti == brent_tortoise) { // the same tile again: a cycle the splice cannot see; walk this read without tiles
						c.fail(WALK_FAIL_TILE_CYCLE);
						*ok = false;
						return ER_DEAD_END;
					}
					if (++brent_lam == brent_power) {
						brent_tortoise = ti;
						brent_power *= 2;
						brent_lam = 0;
					}
					if (!bytevec_append(c, bases, T->bases, n) || !u32vec_push(c, tiles, ti)) {
						*ok = false;
						return ER_DEAD_END;
					}
					*psize += n;
					prev_h = T->prev_last;
					hk = T->end_key;
					cls = ((unsigned)T->end_orient << 1) | (unsigned)dir;
					moved = true;
				}
				if (T->stop_kind == TS_CODE) {
					if (moved)
						head = rebuild_head(c, start, bases, 0, dir);
					return (ExtCode)T->stop_code;
				}
				if (T->stop_kind == TS_CAP || !n)
					break;
				T = Tn;
			}
			if (moved) {
				head = rebuild_head(c, start, bases, 0, dir);
				nb = c.neighbors(head);
				continue;
			}
		}
		nb = c.neighbors_finish(pr);
	}
}

/** isTip (bloom-dbg.h:758-776) */
ABB_HD bool is_tip(unsigned length, ExtCode left, ExtCode right, unsigned trim)
{
	if (length > trim)
		return false;
	if (left == ER_DEAD_END && (right == ER_DEAD_END || right == ER_AMBI_IN))
		return true;
	if (right == ER_DEAD_END && (left == ER_DEAD_END || left == ER_AMBI_IN))
		return true;
	return false;
}

/** result of extending one seed k-mer */
struct ContigOut {
	uint8_t* seq;    // 2-bit codes, one per byte, after trimming (pathToSeq, bloom-dbg.h:132-158)
	unsigned len;    // bases
	unsigned psize;  // vertices before trimming (contigPath.size() as isTip sees it)
	ExtCode left, right;
	unsigned left_n, right_n; // vertices the two extendPath calls added (ContigRecord left/rightExtensionResult.first)
	const uint8_t* raw;       // pathToSeq of the UNTRIMMED path (reversed left + seed + right), raw_len = psize + k - 1 codes
	unsigned raw_len, seed_off; // the seed k-mer starts at raw[seed_off], in the orientation the read holds it
	bool tip;        // isTip: not output, but its k-mers still count as assembled for this read
	bool popped_front, popped_back; // a real path vertex (not a pushed duplicate) was trimmed off that end
	uint64_t front_h, back_h;       // canonical hashes of the trimmed-off vertices
	uint64_t front_b, back_b;       // their Bloom hashes (the repeat check hashes the contig the way the Bloom filters do)
	bool pushed_front, pushed_back; // preprocessCircularContig's duplicate vertex survives at that end of seq
	U32Vec tiles_left, tiles_right; // tiles spliced into the path (their vertices are not in the PathSet)
};

/**
 * Extend seed both ways, decide tip-ness, trim branch k-mers (bloom-dbg.h:852-869).
 * ps must be a fresh PathSet; it ends up holding every vertex of the untrimmed path.
 */
template <int KW, class Ctx>
ABB_HD bool extend_seed(Ctx& c, const Vtx<KW>& seed, PathSet& ps, ContigOut* o)
{
	const unsigned k = c.k;
	bool ok = true;
	pathset_insert(c, ps, seed.canon(), &ok);
	ByteVec left = { nullptr, 0, 0 }, right = { nullptr, 0, 0 };
	o->tiles_left = U32Vec{ nullptr, 0, 0 };
	o->tiles_right = U32Vec{ nullptr, 0, 0 };
	o->pushed_front = o->pushed_back = false;
	unsigned psize = 1;
	Vtx<KW> front = seed, back = seed;
	o->left = extend_dir(c, front, REV, &psize, left, ps, &ok, o->tiles_left);
	if (!ok || c.failed())
		return false;
	o->right = extend_dir(c, back, FWD, &psize, right, ps, &ok, o->tiles_right);
	if (!ok || c.failed())
		return false;
	o->psize = psize;
	o->left_n = left.n;
	o->right_n = right.n;
	o->tip = is_tip(psize, o->left, o->right, c.trim);
	o->popped_front = o->popped_back = false;
	o->front_h = o->back_h = 0;
	o->front_b = o->back_b = 0;

	// materialise pathToSeq(contigPath): reversed(left) + seed + right, with one spare byte each side
	// for the vertex preprocessCircularContig may push
	const unsigned n = psize + k - 1;
	uint8_t* buf = c.alloc((uint64_t)n + 2, false);
	if (!buf)
		return false;
	uint8_t* s = buf + 1;
	c.copy8_rev(s, left.p, left.n);
	for (unsigned i = 0; i < k; ++i)
		c.wr8(s + left.n + i, (uint8_t)kmer_base(seed.km, k, i));
	c.copy8(s + left.n + k, right.p, right.n);
	c.sync();
	o->seq = s;
	o->len = n;
	o->raw = s;
	o->raw_len = n;
	o->seed_off = left.n;
	if (o->tip || psize == 1) // trimBranchKmers returns immediately for a single vertex (bloom-dbg.h:727-728)
		return true;

	// ---- trimBranchKmers (bloom-dbg.h:720-756) ----
	unsigned l = psize;
	bool pushed_front = false, pushed_back = false;
	uint64_t second_id = 0, penult_id = 0;
	{ // getContigType (bloom-dbg.h:629-644): is there an edge back -> front?
		const unsigned om = c.neighbors(back) & 15;
		bool edge = false;
		for (unsigned mm = om; mm && !edge; mm &= mm - 1) {
			Vtx<KW> x = back;
			vtx_step(x, k, c.rt, FWD, ctz4(mm));
			edge = x.canon() == front.canon();
		}
		if (edge && psize > 2) { // preprocessCircularContig (bloom-dbg.h:648-697)
			Vtx<KW> v = front;
			vtx_step(v, k, c.rt, REV, kmer_first(back.km, k)); // v.shift(ANTISENSE, back.getBase(0))
			const bool circular = kmer_equal_masked(v.km, back.km, k, c.rt);
			const bool branch_start = ambiguous(c, front, FWD) || ambiguous(c, front, REV);
			const bool branch_end = ambiguous(c, back, FWD) || ambiguous(c, back, REV);
			if (branch_start && !branch_end) {
				// push_back(front) / push_back(rc(front)): pathToSeq lets the last k-mer overwrite its k columns
				const Vtx<KW> x = circular ? front : vtx_revcomp(front, k);
				// (with a spaced seed only its '1' positions are written; the others are columns of earlier vertices)
				for (unsigned i = 0; i < k; ++i)
					if (mask_is_care(c.rt, i))
						c.wr8(s + (l - 1) + 1 + i, (uint8_t)kmer_base(x.km, k, i));
				penult_id = back.canon();
				back = x;
				pushed_back = true;
				++l;
			} else if (!branch_start && branch_end) {
				// push_front(back) / push_front(rc(back)): only column 0 survives the later overwrites
				const Vtx<KW> x = circular ? back : vtx_revcomp(back, k);
				--s;
				c.wr8(s, (uint8_t)kmer_first(x.km, k));
				second_id = front.canon();
				front = x;
				pushed_front = true;
				++l;
			}
			c.sync();
		}
	}
	// path[1] and path[l-2]: the vertices next to a pushed one are the old ends; otherwise they are read back from
	// the string (a path of consecutive k-mers spells its vertices exactly, don't-care positions included)
	if (!pushed_front)
		second_id = vtx_from_codes<KW>(s + 1, k, false, c.rt).canon();
	if (!pushed_back)
		penult_id = vtx_from_codes<KW>(s + (l - 2), k, false, c.rt).canon();
	const bool amb1 = ambiguous_expected(c, front, second_id, FWD);
	const bool amb2 = ambiguous_expected(c, back, penult_id, REV);
	if (c.rt.nmask && pushed_front && !amb1) {
		// spaced seed, pathToSeq: a '1' position of the pushed front vertex survives where no later vertex writes the
		// column (columns <= l-1 are position 0 of a later vertex)
		for (unsigned p = l; p < k; ++p) {
			bool later = !mask_is_care(c.rt, p);
			for (unsigned j = 1; j < l && !later; ++j)
				later = mask_is_care(c.rt, p - j);
			if (!later)
				c.wr8(s + p, (uint8_t)kmer_base(front.km, k, p));
		}
		c.sync();
	}
	unsigned begin = 0, end = l + k - 1;
	if (amb1) {
		++begin;
		if (!pushed_front) {
			o->popped_front = true;
			o->front_h = front.canon();
			o->front_b = front.bloom();
		}
	} else
		o->pushed_front = pushed_front;
	if (amb2) {
		--end;
		if (!pushed_back) {
			o->popped_back = true;
			o->back_h = back.canon();
			o->back_b = back.bloom();
		}
	} else
		o->pushed_back = pushed_back;
	o->seq = s + begin;
	o->len = end - begin;
	return true;
}


// ------------------------------------------------------------------------------------------
// the extension loop of processRead (bloom-dbg.h:837-879) for one candidate read:
// every read k-mer not yet on a contig generated from this read seeds an extension.
// Emit::operator()(ctx, seed_index, contig) is called for every non-tip contig, in order.
// Returns false when scratch memory ran out (the host retries the read).
// ------------------------------------------------------------------------------------------
template <int KW, class Ctx, class Emit>
ABB_HD bool walk_read(Ctx& c, const uint8_t* read_ascii, unsigned L, Emit& emit)
{
	const unsigned k = c.k;
	const unsigned nk = L - k + 1;
	uint64_t* rh = (uint64_t*)c.alloc((uint64_t)nk * 8, false);
	uint8_t* cov = c.alloc(nk, true);
	if (!rh || !cov)
		return false;
	{ // seqToPath (bloom-dbg.h:115-125): canonical hash of every read k-mer
		Vtx<KW> v = vtx_from_codes<KW>(read_ascii, k, true, c.rt);
		c.wr64(rh, v.canon());
		for (unsigned i = 1; i < nk; ++i) {
			vtx_step(v, k, c.rt, FWD, base_code(read_ascii[i + k - 1]) & 3);
			c.wr64(rh + i, v.canon());
		}
		c.sync();
	}
	Vtx<KW> rv = vtx_from_codes<KW>(read_ascii, k, true, c.rt);
	unsigned ri = 0;
	for (unsigned i = 0; i < nk; ++i) {
		if (c.rd8(cov + i)) // assembledKmers.find(*it) != end
			continue;
		for (; ri < i; ++ri)
			vtx_step(rv, k, c.rt, FWD, base_code(read_ascii[ri + k]) & 3);
		PathSet ps;
		if (!pathset_init(c, ps, 1024))
			return false;
		ContigOut o;
		if (!extend_seed(c, rv, ps, &o) || c.failed())
			return false;
		if (!o.tip)
			emit(c, i, o);
		c.mark_covered(ps, rh, cov, nk, o, read_ascii, i);
	}
	return !c.failed();
}

} // namespace abb
