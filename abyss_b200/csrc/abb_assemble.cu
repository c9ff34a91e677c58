// abb_assemble.cu -- pass 2 (BloomDBG::assemble / processRead, bloom-dbg.h:783-882,972-1089)
// behind the C ABI.
//
// The reference processes reads strictly one after another at -j1; each read either is skipped
// (short / non-ACGT / blunt end / not solid / all k-mers already assembled) or seeds unitig
// extensions whose k-mers are then marked in the "assembled" bit Bloom filter.  Two facts make
// this parallel without changing a byte of the output:
//   (1) the classification tests and the extension of a seed k-mer are pure functions of the
//       read-only solid filter (Graph/ExtendPath.h takes a const Graph&);
//   (2) the assembled filter only ever gains bits, so "all k-mers assembled" is monotone: a read
//       that is covered now stays covered.
// Pipeline per batch of reads (file order):
//   K3a classify      warp per read, all reads at once            (pure)
//   loop over the candidate reads in file order:
//     K3b visited     warp per candidate vs the CURRENT assembled filter; covered reads are final
//     K4  extend      warp per not-yet-covered candidate, speculatively, many at once (pure)
//     K1  hash        ntHash of the produced unitigs
//     K5  replay      ONE CTA walks the speculated reads in file order doing exactly the
//                     reference's bookkeeping: re-test "all assembled" with the now-current filter,
//                     redundancy test, mark assembled, coverage = sum of minCount; 1024 threads
//                     share the k-mers of each unitig
// so every order-dependent decision is taken in file order with the same filter state the
// reference would have, while the expensive graph walks run thousands at a time.
#include "abb_common.h"
#include "abb_walk.cuh"
#include <cooperative_groups.h>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

namespace abb {
namespace cg = cooperative_groups;

// ------------------------------------------------------------------------------------------
// device context: the Ctx concept of abb_walk.cuh for one warp
// ------------------------------------------------------------------------------------------
__host__ __device__ inline uint64_t tile_slot(uint64_t key, unsigned cls, unsigned mask)
{
	return (((key ^ (0x9E3779B97F4A7C15ULL * (cls + 1))) * 0xD6E8FEB86659FD93ULL) >> 24) & mask;
}

struct WarpCtx {
	unsigned k, trim;
	RollTab rt;
	const HashCfg* cfg;
	const uint8_t* counters;
	unsigned threshold;
	unsigned lane;
	Frame* frames;
	uint64_t* look;
	uint8_t* arena;
	unsigned long long arena_size;
	unsigned long long* arena_top;
	unsigned fail_;
	// tiles (null table = disabled)
	const TileRec* tile_recs;
	const unsigned* tile_tab; // open addressing: tile index + 1, 0 = empty
	unsigned tile_mask;

	// profiling hook (ABB_ROUND_LOG): clock64 ticks between the stages of a walk, accumulated per speculated read
	unsigned long long* dbg = nullptr;
	long long t_last = 0;
	__device__ void tick(int slot)
	{
		if (!dbg)
			return;
		const long long now = clock64();
		if (slot >= 0 && lane == 0)
			dbg[slot] += (unsigned long long)(now - t_last);
		t_last = now;
	}
	__device__ bool tiles_enabled() const { return tile_tab != nullptr; }
	__device__ const TileRec* tile_lookup(uint64_t key, unsigned cls) const
	{
		for (uint64_t s = tile_slot(key, cls, tile_mask);; s = (s + 1) & tile_mask) {
			const unsigned v = __ldcg(tile_tab + s);
			if (v == 0)
				return nullptr;
			const TileRec* t = tile_recs + (v - 1);
			if (t->key == key && t->cls == cls)
				return t;
		}
	}
	__device__ uint32_t tile_index(const TileRec* t) const { return (uint32_t)(t - tile_recs); }
	__device__ const TileRec* tile_at(uint32_t idx) const { return tile_recs + idx; }
	__device__ void prefetch(const void* p) const
	{
		if (p)
			asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
	}
	__device__ void wr32(uint32_t* p, uint32_t v) const { *(volatile uint32_t*)p = v; }

	/** bits 0-3: out-neighbours (append A,C,G,T) present in the solid filter; bits 4-7: in-neighbours
	 *  (prepend).  Lane = 4 * neighbour + hash slot: 8 neighbours x 4 hash functions per round trip
	 *  (out/in_edge_iterator::next + vertex_exists, RollingBloomDBG.h:302-327,357-383,436-445). */
	struct Probe {
		bool ok;
	};
	template <int KW>
	__device__ Probe neighbors_issue(const Vtx<KW>& v) const
	{
		const unsigned n = lane >> 2, hs = lane & 3;
		const uint64_t h0 = neighbor_bloom(v, k, rt, n < 4 ? FWD : REV, n & 3);
		unsigned mn = 255;
		for (unsigned i = hs; i < cfg->H; i += 4)
			mn = min(mn, (unsigned)__ldcg(counters + nth_pos(h0, *cfg, i)));
		Probe p;
		p.ok = mn >= threshold;
		return p;
	}
	__device__ unsigned neighbors_finish(const Probe& p) const
	{
		unsigned b = __ballot_sync(0xffffffffu, p.ok);
		b &= b >> 1;
		b &= b >> 2; // bit 4n = AND of the four lanes of neighbour n
		unsigned r = 0;
#pragma unroll
		for (int j = 0; j < 8; ++j)
			r |= ((b >> (4 * j)) & 1u) << j;
		return r;
	}
	template <int KW>
	__device__ unsigned neighbors(const Vtx<KW>& v) const
	{
		return neighbors_finish(neighbors_issue(v));
	}
	/** neighbours in one direction only: 16 of the 32 lanes probe (lookAhead never turns around) */
	template <int KW>
	__device__ unsigned neighbors_dir(const Vtx<KW>& v, Dir d) const
	{
		const unsigned n = lane >> 2, hs = lane & 3;
		const bool mine = (n < 4) == (d == FWD);
		bool ok = true;
		if (mine) {
			const uint64_t h0 = neighbor_bloom(v, k, rt, n < 4 ? FWD : REV, n & 3);
			unsigned mn = 255;
			for (unsigned i = hs; i < cfg->H; i += 4)
				mn = min(mn, (unsigned)__ldcg(counters + nth_pos(h0, *cfg, i)));
			ok = mn >= threshold;
		}
		Probe p;
		p.ok = ok;
		const unsigned m = neighbors_finish(p);
		return d == FWD ? (m & 15) : (m >> 4);
	}
	// scratch accesses: every lane stores the same value to the same address and reads back its own
	// store, so no intra-warp synchronisation is needed for uniform data
	__device__ uint64_t rd64(const uint64_t* p) const { return *(const volatile uint64_t*)p; }
	__device__ void wr64(uint64_t* p, uint64_t v) const { *(volatile uint64_t*)p = v; }
	__device__ uint8_t rd8(const uint8_t* p) const { return *(const volatile uint8_t*)p; }
	__device__ void wr8(uint8_t* p, uint8_t v) const { *(volatile uint8_t*)p = v; }
	__device__ void sync() const { __syncwarp(); }
	__device__ bool find64(const uint64_t* a, unsigned n, uint64_t key, unsigned stride) const
	{
		for (unsigned base = 0; base < n; base += 32) {
			const unsigned i = base + lane;
			const bool hit = i < n && *(const volatile uint64_t*)(a + (size_t)i * stride) == key;
			if (__any_sync(0xffffffffu, hit))
				return true;
		}
		return false;
	}
	__device__ uint8_t* alloc(unsigned long long bytes, bool zero)
	{
		bytes = (bytes + 15) & ~15ULL;
		unsigned long long off = 0;
		if (lane == 0)
			off = atomicAdd(arena_top, bytes);
		off = __shfl_sync(0xffffffffu, off, 0);
		if (off + bytes > arena_size) {
			fail(3);
			return nullptr;
		}
		uint8_t* p = arena + off;
		if (zero) {
			uint4* q = reinterpret_cast<uint4*>(p);
			for (unsigned long long i = lane; i < bytes / 16; i += 32)
				q[i] = make_uint4(0, 0, 0, 0);
			__syncwarp();
		}
		return p;
	}
	__device__ void fail(unsigned why) { fail_ |= 1u << why; }
	__device__ bool failed() const { return fail_ != 0; }
	// cooperative byte copies.  Loads are issued in batches before the dependent stores: a naive
	// d[i] = s[i] loop pays one DRAM round trip per iteration (no restrict => no load hoisting), which made
	// splicing and vector growth the dominant cost of a tiled walk.
	__device__ void copy8(uint8_t* __restrict__ d, const uint8_t* __restrict__ s, unsigned n) const
	{
		unsigned done = 0;
		if (n >= 1024 && (((uintptr_t)d | (uintptr_t)s) & 15) == 0) { // big aligned copies (vector growth): 16 B per lane, 4 in flight
			const uint4* s4 = reinterpret_cast<const uint4*>(s);
			uint4* d4 = reinterpret_cast<uint4*>(d);
			const unsigned n16 = n / 16;
			unsigned i = lane;
			for (; i + 96 < n16; i += 128) {
				const uint4 a = s4[i], b = s4[i + 32], c2 = s4[i + 64], e = s4[i + 96];
				d4[i] = a;
				d4[i + 32] = b;
				d4[i + 64] = c2;
				d4[i + 96] = e;
			}
			for (; i < n16; i += 32)
				d4[i] = s4[i];
			done = n16 * 16;
		}
		for (unsigned base = done; base < n; base += 256) { // 8 bytes per lane in flight
			uint8_t v[8];
#pragma unroll
			for (int j = 0; j < 8; ++j) {
				const unsigned i = base + lane + 32 * j;
				v[j] = i < n ? s[i] : 0;
			}
#pragma unroll
			for (int j = 0; j < 8; ++j) {
				const unsigned i = base + lane + 32 * j;
				if (i < n)
					d[i] = v[j];
			}
		}
		__syncwarp();
	}
	__device__ void copy8_rev(uint8_t* __restrict__ d, const uint8_t* __restrict__ s, unsigned n) const
	{
		for (unsigned base = 0; base < n; base += 256) {
			uint8_t v[8];
#pragma unroll
			for (int j = 0; j < 8; ++j) {
				const unsigned i = base + lane + 32 * j;
				v[j] = i < n ? s[n - 1 - i] : 0;
			}
#pragma unroll
			for (int j = 0; j < 8; ++j) {
				const unsigned i = base + lane + 32 * j;
				if (i < n)
					d[i] = v[j];
			}
		}
		__syncwarp();
	}
	__device__ void rehash(const uint64_t* o, unsigned ocap, uint64_t* nt, unsigned ncap) const
	{
		for (unsigned s = lane; s < ocap; s += 32) {
			const uint64_t v = o[s];
			if (v == 0)
				continue;
			uint64_t t = pathset_slot(v, ncap);
			while (atomicCAS((unsigned long long*)(nt + t), 0ULL, (unsigned long long)v) != 0ULL)
				t = (t + 1) & (ncap - 1);
		}
		__syncwarp();
	}
	__device__ void mark_covered(const PathSet& ps, const uint64_t* rh, uint8_t* cov, unsigned nk, const ContigOut& o,
	                             const uint8_t* read_ascii, unsigned seed_i)
	{
		for (unsigned j = lane; j < nk; j += 32) {
			if (cov[j])
				continue;
			const uint64_t key = rh[j];
			if (!pathset_contains(*this, ps, key))
				continue;
			if ((o.popped_front && key == o.front_h) || (o.popped_back && key == o.back_h))
				continue;
			cov[j] = 1;
		}
		__syncwarp();
		if (o.tiles_left.n + o.tiles_right.n == 0)
			return;
		// The spliced tiles' vertices are not in the PathSet.  Fast path (no spaced seed): the contig string holds the
		// seed k-mer at raw[seed_off] in the read's orientation, so as long as the read and the contig agree base for base
		// away from the seed, the read's k-mers ARE the contig's vertices at those offsets.  A read that follows its unitig
		// (the normal case: every k-mer of a candidate read is solid) is settled by ~150 byte compares; only k-mers the
		// comparison does not reach fall through to the exact scan of all tile hashes below (it took 230 of the 266 ms of
		// the slowest walk of the 50 M-read job before this shortcut).
		if (!rt.nmask && o.raw) {
			const unsigned maxf = min(nk - 1 - seed_i, o.raw_len - (o.seed_off + k));
			unsigned mf = maxf;
			for (unsigned base = 0; base < maxf; base += 32) {
				const unsigned t = base + lane;
				const bool bad = t < maxf && base_code(read_ascii[seed_i + k + t]) != *(const volatile uint8_t*)(o.raw + o.seed_off + k + t);
				const unsigned m = __ballot_sync(0xffffffffu, bad);
				if (m) {
					mf = base + __ffs(m) - 1;
					break;
				}
			}
			const unsigned maxb = min(seed_i, o.seed_off);
			unsigned mb = maxb;
			for (unsigned base = 0; base < maxb; base += 32) {
				const unsigned t = base + lane;
				const bool bad = t < maxb && base_code(read_ascii[seed_i - 1 - t]) != *(const volatile uint8_t*)(o.raw + o.seed_off - 1 - t);
				const unsigned m = __ballot_sync(0xffffffffu, bad);
				if (m) {
					mb = base + __ffs(m) - 1;
					break;
				}
			}
			bool all = true;
			for (unsigned j = lane; j < nk; j += 32) {
				if (!cov[j] && j + mb >= seed_i && j <= seed_i + mf) {
					const uint64_t key = rh[j];
					if (!((o.popped_front && key == o.front_h) || (o.popped_back && key == o.back_h)))
						cov[j] = 1;
				}
				all &= cov[j] != 0;
			}
			__syncwarp(); // cov[] is read back by every lane (walk_read); a vote does not order the stores
			if (__all_sync(0xffffffffu, all))
				return;
		}
		// exact fallback: stream the tiles' hashes against a small table of the read's k-mer hashes
		unsigned cap = 64;
		while (cap < 2 * nk)
			cap <<= 1;
		uint64_t* keys = (uint64_t*)alloc((unsigned long long)cap * 8, true);
		uint8_t* hit = alloc(cap, true);
		if (!keys || !hit)
			return;
		for (unsigned j = lane; j < nk; j += 32) {
			const uint64_t key = rh[j] ? rh[j] : 1; // 0 marks an empty slot; hash 0 is remapped (2^-64)
			for (uint64_t t = pathset_slot(key, cap);; t = (t + 1) & (cap - 1)) {
				const unsigned long long old = atomicCAS((unsigned long long*)(keys + t), 0ULL, (unsigned long long)key);
				if (old == 0ULL || old == key)
					break;
			}
		}
		__syncwarp();
		for (int side = 0; side < 2; ++side) {
			const U32Vec& tv = side ? o.tiles_right : o.tiles_left;
			// the warp sweeps one tile at a time with coalesced loads (8 hashes per lane in flight); the next tile's record
			// and hashes are prefetched into L2 meanwhile, so a tile costs about one L2 round trip
			for (unsigned ti = 0; ti < tv.n; ++ti) {
				const TileRec* T = tile_recs + tv.p[ti];
				if (ti + 2 < tv.n && lane == 0)
					prefetch(tile_recs + tv.p[ti + 2]);
				if (ti + 1 < tv.n) {
					const TileRec* Tn = tile_recs + tv.p[ti + 1];
					const uint64_t* thn = Tn->hashes;
					if (lane * 16u < Tn->n)
						prefetch(thn + lane * 16u);
				}
				const uint64_t* __restrict__ th = T->hashes;
				const unsigned tn = T->n;
				for (unsigned i0 = 0; i0 < tn; i0 += 256) {
					uint64_t kv[8];
#pragma unroll
					for (int j = 0; j < 8; ++j) { // 8 independent coalesced loads before any probe
						const unsigned idx = i0 + lane + 32u * j;
						kv[j] = idx < tn ? th[idx] : 0;
					}
#pragma unroll
					for (int j = 0; j < 8; ++j) {
						uint64_t key = kv[j];
						if (i0 + lane + 32u * j >= tn)
							continue;
						if ((o.popped_front && key == o.front_h) || (o.popped_back && key == o.back_h))
							continue;
						key = key ? key : 1;
						for (uint64_t t = pathset_slot(key, cap);; t = (t + 1) & (cap - 1)) {
							const uint64_t v = keys[t];
							if (v == key) {
								hit[t] = 1;
								break;
							}
							if (v == 0)
								break;
						}
					}
				}
			}
		}
		__syncwarp();
		for (unsigned j = lane; j < nk; j += 32) {
			if (cov[j])
				continue;
			const uint64_t key = rh[j] ? rh[j] : 1;
			for (uint64_t t = pathset_slot(key, cap);; t = (t + 1) & (cap - 1)) {
				const uint64_t v = keys[t];
				if (v == key) {
					if (hit[t])
						cov[j] = 1;
					break;
				}
				if (v == 0)
					break;
			}
		}
		__syncwarp();
	}
};

/** one unitig produced by K4 */
struct ContigRec {
	unsigned long long seq; // device pointer to 2-bit codes, one per byte
	unsigned spec;          // index of the seeding read in the speculative set
	unsigned ordinal;       // n-th contig of that read
	unsigned len;
	unsigned seed_pos;
	unsigned psize;
	unsigned char left, right, flags, pad1; // flags: 1 pushed_front, 2 pushed_back, 4 popped_front, 8 popped_back
	unsigned long long front_h, back_h;     // canonical hashes of trimmed-off end vertices (flags 4 / 8)
	unsigned left_n, right_n;               // vertices added by the two extensions (-T trace)
};

struct DevEmit {
	ContigRec* recs;
	unsigned* nrecs;
	unsigned cap;
	unsigned spec, ordinal;
	__device__ void operator()(WarpCtx& c, unsigned seed_pos, const ContigOut& o)
	{
		if (c.lane == 0) {
			const unsigned idx = atomicAdd(nrecs, 1u);
			if (idx < cap) {
				ContigRec r;
				r.seq = (unsigned long long)o.seq;
				r.spec = spec;
				r.ordinal = ordinal;
				r.len = o.len;
				r.seed_pos = seed_pos;
				r.psize = o.psize;
				r.left = (unsigned char)o.left;
				r.right = (unsigned char)o.right;
				r.flags = (unsigned char)((o.pushed_front ? 1 : 0) | (o.pushed_back ? 2 : 0) | (o.popped_front ? 4 : 0) | (o.popped_back ? 8 : 0));
				r.pad1 = 0;
				r.front_h = o.front_h;
				r.back_h = o.back_h;
				r.left_n = o.left_n;
				r.right_n = o.right_n;
				recs[idx] = r;
			}
		}
		++ordinal;
	}
};

struct IsCandidate {
	const uint8_t* codes;
	__host__ __device__ bool operator()(unsigned r) const { return codes[r] == RC_CANDIDATE; }
};

struct WalkCfg {
	unsigned k, trim, threshold;
	RollTab rt;
	const uint8_t* counters;
};

/** device view of the tile store (tab == nullptr: tiles disabled) */
struct TileView {
	const TileRec* recs;
	const unsigned* tab;
	unsigned mask;
};

__device__ __forceinline__ WarpCtx make_ctx(const WalkCfg& w, const HashCfg* cfg, Frame* frames, uint64_t* look, unsigned gwarp,
                                            uint8_t* arena, unsigned long long arena_size, unsigned long long* arena_top)
{
	WarpCtx c;
	c.k = w.k;
	c.trim = w.trim;
	c.rt = w.rt;
	c.cfg = cfg;
	c.counters = w.counters;
	c.threshold = w.threshold;
	c.lane = threadIdx.x & 31;
	c.frames = frames ? frames + (size_t)gwarp * kFrameCap : nullptr;
	c.look = look + (size_t)gwarp * kLookCap;
	c.arena = arena;
	c.arena_size = arena_size;
	c.arena_top = arena_top;
	c.fail_ = 0;
	c.tile_recs = nullptr;
	c.tile_tab = nullptr;
	c.tile_mask = 0;
	return c;
}

constexpr int kWalkWarps = 4; // warps per CTA for the walking kernels

// ------------------------------------------------------------------------------------------
// K3a: classify every read of the batch (processRead's tests, bloom-dbg.h:803-817)
// ------------------------------------------------------------------------------------------
template <int KW>
__global__ void __launch_bounds__(kWalkWarps * 32)
k_classify(const uint8_t* __restrict__ bases, const uint64_t* __restrict__ offs, const uint64_t* __restrict__ slot_offs,
           const uint64_t* __restrict__ h0, const uint8_t* __restrict__ valid, uint64_t n_reads, WalkCfg w,
           const __grid_constant__ HashCfg cfg, uint64_t* look, int exact_codes, uint8_t* __restrict__ codes)
{
	const unsigned gwarp = blockIdx.x * kWalkWarps + (threadIdx.x >> 5);
	const unsigned nwarps = gridDim.x * kWalkWarps;
	WarpCtx c = make_ctx(w, &cfg, nullptr, look, gwarp, nullptr, 0, nullptr);
	const unsigned lane = c.lane;
	for (uint64_t r = gwarp; r < n_reads; r += nwarps) {
		const uint64_t beg = offs[r];
		const unsigned L = (unsigned)(offs[r + 1] - beg);
		uint8_t code;
		if (L < w.k) {
			code = RC_SHORTER_THAN_K;
		} else {
			const uint64_t s0 = slot_offs[r];
			const unsigned nk = L - w.k + 1;
			// allACGT(seq): every base of a read with L >= k lies in some window
			bool bad = false;
			if (w.rt.nmask) { // with a spaced seed the window flags only cover the '1' positions
				for (unsigned j = lane; j < L; j += 32)
					bad |= base_code(bases[beg + j]) >= 4;
			} else
				for (unsigned j = lane; j < nk; j += 32)
					bad |= valid[s0 + j] == 0;
			if (__any_sync(0xffffffffu, bad)) {
				code = RC_NON_ACGT;
			} else {
				// allKmersInBloom(seq, solidKmerSet) (bloom-dbg.h:60-78)
				bool solid = true;
				for (unsigned base = 0; base < nk && solid; base += 32) {
					const unsigned j = base + lane;
					bool ok = true;
					if (j < nk) {
						const uint64_t h = h0[s0 + j];
						for (unsigned i = 0; i < cfg.H; ++i)
							ok &= __ldcg(w.counters + nth_pos(h, cfg, i)) >= w.threshold;
					}
					solid = __all_sync(0xffffffffu, ok);
				}
				if (!solid && !exact_codes) {
					code = RC_NOT_SOLID;
				} else {
					// hasBluntEnd (bloom-dbg.h:494-532): lookAhead(first k-mer, REVERSE, 5) on the read and on
					// its reverse complement
					const Vtx<KW> first = vtx_from_codes<KW>(bases + beg, w.k, true, w.rt);
					bool blunt = !look_ahead(c, first, REV, kFpTrim);
					if (!blunt) {
						const Vtx<KW> last = vtx_from_codes<KW>(bases + beg + L - w.k, w.k, true, w.rt);
						blunt = !look_ahead(c, vtx_revcomp(last, w.k), REV, kFpTrim);
					}
					code = blunt ? RC_BLUNT_END : (solid ? RC_CANDIDATE : RC_NOT_SOLID);
				}
			}
		}
		if (lane == 0)
			codes[r] = code;
	}
}

// ------------------------------------------------------------------------------------------
// K3b: allKmersInBloom(seq, assembledKmerSet) for candidates cand[c0 .. c0+n) (bloom-dbg.h:823)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_visited(const unsigned* __restrict__ cand, unsigned c0, unsigned n, const uint64_t* __restrict__ slot_offs,
          const uint64_t* __restrict__ h0, const __grid_constant__ HashCfg cfg, const uint8_t* __restrict__ bits,
          uint8_t* __restrict__ out)
{
	const unsigned gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
	if (gwarp >= n)
		return;
	const unsigned r = cand[c0 + gwarp];
	const uint64_t s0 = slot_offs[r];
	const unsigned nk = (unsigned)(slot_offs[r + 1] - s0);
	bool all = true;
	for (unsigned base = 0; base < nk && all; base += 32) {
		const unsigned j = base + lane;
		bool ok = true;
		if (j < nk) {
			const uint64_t h = h0[s0 + j];
			for (unsigned i = 0; i < cfg.H; ++i) {
				const uint64_t p = nth_pos(h, cfg, i);
				ok &= (__ldcg(bits + (p >> 3)) >> (p & 7)) & 1;
			}
		}
		all = __all_sync(0xffffffffu, ok);
	}
	if (lane == 0)
		out[gwarp] = all;
}

// ------------------------------------------------------------------------------------------
// K4: extend -- one warp per speculated read runs processRead's extension loop
// ------------------------------------------------------------------------------------------
template <int KW>
__global__ void __launch_bounds__(kWalkWarps * 32)
k_extend(const uint8_t* __restrict__ bases, const uint64_t* __restrict__ offs, const unsigned* __restrict__ spec, unsigned n_spec,
         WalkCfg w, const __grid_constant__ HashCfg cfg, Frame* frames, uint64_t* look, uint8_t* arena,
         unsigned long long arena_size, unsigned long long* arena_top, ContigRec* recs, unsigned* nrecs, unsigned rec_cap,
         unsigned* __restrict__ status, TileView tv, unsigned long long* dbg)
{
	const unsigned gwarp = blockIdx.x * kWalkWarps + (threadIdx.x >> 5);
	if (gwarp >= n_spec)
		return;
	WarpCtx c = make_ctx(w, &cfg, frames, look, gwarp, arena, arena_size, arena_top);
	c.dbg = dbg ? dbg + 4ull * gwarp : nullptr;
	c.tile_recs = tv.recs;
	c.tile_tab = tv.tab;
	c.tile_mask = tv.mask;
	const unsigned r = spec[gwarp];
	const uint64_t beg = offs[r];
	const unsigned L = (unsigned)(offs[r + 1] - beg);
	DevEmit emit = { recs, nrecs, rec_cap, gwarp, 0 };
	const bool ok = walk_read<KW>(c, bases + beg, L, emit);
	if (c.lane == 0)
		status[gwarp] = ok ? 0u : (c.fail_ ? c.fail_ : 1u);
}


// ------------------------------------------------------------------------------------------
// Tiles (abb_walk.cuh): marker enumeration, production, and the repeat check that guards them
// ------------------------------------------------------------------------------------------
/** every valid, solid k-mer slot whose canonical hash is a marker and that is not yet in the marker
 *  set joins the list of new markers as (read, window) */
__global__ void __launch_bounds__(256)
k_find_markers(const uint64_t* __restrict__ h0, const uint8_t* __restrict__ valid, const uint64_t* __restrict__ slot_offs,
               uint64_t n_reads, uint64_t n_slots, WalkCfg w, const __grid_constant__ HashCfg cfg, unsigned long long* mset,
               unsigned mset_mask, unsigned long long* __restrict__ out /* packed (read << 24 | pos) */, unsigned* n_out,
               unsigned out_cap, unsigned world, unsigned rank)
{
	for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < n_slots; s += (uint64_t)gridDim.x * blockDim.x) {
		const uint64_t h = h0[s];
		if (!is_marker(h) || !valid[s])
			continue;
		if (world > 1 && (unsigned)((h >> 8) % world) != rank) // several GPUs: each marker is tiled by exactly one rank
			continue;
		bool solid = true;
		for (unsigned i = 0; i < cfg.H; ++i)
			solid &= __ldcg(w.counters + nth_pos(h, cfg, i)) >= w.threshold;
		if (!solid)
			continue;
		const unsigned long long key = h ? h : 1;
		bool fresh = false;
		for (uint64_t t = pathset_slot(key, mset_mask + 1);; t = (t + 1) & mset_mask) {
			const unsigned long long old = atomicCAS(mset + t, 0ULL, key);
			if (old == 0ULL) {
				fresh = true;
				break;
			}
			if (old == key)
				break;
		}
		if (!fresh)
			continue;
		// which read does slot s belong to? upper_bound over slot_offs
		uint64_t lo = 0, hi = n_reads;
		while (lo < hi) {
			const uint64_t mid = (lo + hi) / 2;
			if (slot_offs[mid + 1] <= s)
				lo = mid + 1;
			else
				hi = mid;
		}
		const unsigned idx = atomicAdd(n_out, 1u);
		if (idx < out_cap)
			out[idx] = (unsigned long long)lo << 24 | (unsigned long long)(s - slot_offs[lo]);
	}
}

struct TileStore { // device-side handles used while producing tiles
	TileRec* recs;
	unsigned* tab;
	unsigned mask;
	unsigned cap;          // capacity of recs
	unsigned* n_recs;
	uint8_t* pool;
	unsigned long long pool_size;
	unsigned long long* pool_top;
};

/** persistent warps: work item = (new marker, w) with w = 2 * use_revcomp + direction */
template <int KW>
__global__ void __launch_bounds__(kWalkWarps * 32)
k_make_tiles(const uint8_t* __restrict__ bases, const uint64_t* __restrict__ offs, const unsigned long long* __restrict__ markers,
             unsigned n_markers, unsigned* work, WalkCfg w, const __grid_constant__ HashCfg cfg, Frame* frames, uint64_t* look,
             uint8_t* stage_bases, uint64_t* stage_hashes, TileStore ts)
{
	const unsigned gwarp = blockIdx.x * kWalkWarps + (threadIdx.x >> 5);
	WarpCtx c = make_ctx(w, &cfg, frames, look, gwarp, nullptr, 0, nullptr);
	uint8_t* sb = stage_bases + (size_t)gwarp * kTileCap;
	uint64_t* sh = stage_hashes + (size_t)gwarp * kTileCap;
	const unsigned total = n_markers * 4;
	for (;;) {
		unsigned item = 0;
		if (c.lane == 0)
			item = atomicAdd(work, 1u);
		item = __shfl_sync(0xffffffffu, item, 0);
		if (item >= total)
			break;
		const unsigned long long mk = markers[item >> 2];
		const uint64_t r = mk >> 24;
		const unsigned pos = (unsigned)(mk & 0xffffff);
		Vtx<KW> v = vtx_from_codes<KW>(bases + offs[r] + pos, w.k, true, w.rt);
		if (item & 2)
			v = vtx_revcomp(v, w.k);
		TileRec t;
		c.fail_ = 0;
		make_tile(c, v, (item & 1) ? REV : FWD, &t, sb, sh);
		if (c.fail_)
			continue; // scratch overflow inside successor(): no tile, walks pass this marker vertex by vertex
		// store: hashes then bases, 16-byte aligned
		const unsigned long long bytes = ((unsigned long long)t.n * 9 + 15) & ~15ULL;
		unsigned long long off = 0;
		unsigned idx = 0;
		if (c.lane == 0) {
			off = atomicAdd(ts.pool_top, bytes);
			idx = atomicAdd(ts.n_recs, 1u);
		}
		off = __shfl_sync(0xffffffffu, off, 0);
		idx = __shfl_sync(0xffffffffu, idx, 0);
		if (off + bytes > ts.pool_size || idx >= ts.cap)
			continue; // store full: same graceful degradation
		uint64_t* dh = reinterpret_cast<uint64_t*>(ts.pool + off);
		uint8_t* db = ts.pool + off + 8ULL * t.n;
		for (unsigned i = c.lane; i < t.n; i += 32) {
			dh[i] = sh[i];
			db[i] = sb[i];
		}
		t.hashes = dh;
		t.bases = db;
		__syncwarp();
		if (c.lane == 0) {
			ts.recs[idx] = t;
			__threadfence();
			for (uint64_t s = tile_slot(t.key, t.cls, ts.mask);; s = (s + 1) & ts.mask) {
				const unsigned old = atomicCAS(ts.tab + s, 0u, idx + 1);
				if (old == 0u)
					break;
				const TileRec* o = ts.recs + (old - 1);
				if (o->key == t.key && o->cls == t.cls)
					break; // palindromic marker: the same (key, class) twice, keep the first
			}
		}
	}
}

/** tiles [first, first + n) as produced by THIS rank -> a copy whose pool pointers are offsets from pool_base (what
 *  travels to the other ranks) */
__global__ void __launch_bounds__(256)
k_export_tiles(const TileRec* __restrict__ recs, unsigned first, unsigned n, const uint8_t* pool_base, TileRec* __restrict__ out)
{
	const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n)
		return;
	TileRec t = recs[first + i];
	t.bases = reinterpret_cast<uint8_t*>(reinterpret_cast<const uint8_t*>(t.bases) - pool_base);
	t.hashes = reinterpret_cast<uint64_t*>(reinterpret_cast<const uint8_t*>(t.hashes) - pool_base);
	t.next = 0;
	out[i] = t;
}

/** received tiles [first, first + n) (pool offsets relative to the sender's segment, which now lives at seg_base):
 *  rebase the pointers and enter them into the (marker, class) table */
__global__ void __launch_bounds__(256)
k_import_tiles(TileRec* __restrict__ recs, unsigned first, unsigned n, uint8_t* seg_base, unsigned* __restrict__ tab, unsigned mask)
{
	const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n)
		return;
	TileRec* t = recs + first + i;
	t->bases = seg_base + reinterpret_cast<uintptr_t>(t->bases);
	t->hashes = reinterpret_cast<uint64_t*>(seg_base + reinterpret_cast<uintptr_t>(t->hashes));
	t->next = 0;
	for (uint64_t s = tile_slot(t->key, t->cls, mask);; s = (s + 1) & mask) {
		const unsigned old = atomicCAS(tab + s, 0u, first + i + 1);
		if (old == 0u)
			break;
		const TileRec* o = recs + (old - 1);
		if (o->key == t->key && o->cls == t->cls)
			break;
	}
}

/** resolve TileRec::next for every tile that ended on a marker (tiles of later batches link to earlier ones
 *  and vice versa, so this runs over the whole store after each production) */
__global__ void __launch_bounds__(256)
k_link_tiles(TileRec* recs, unsigned n, const unsigned* __restrict__ tab, unsigned mask)
{
	for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		TileRec* t = recs + i;
		if (t->next || t->stop_kind != TS_MARKER || t->n == 0)
			continue;
		const uint64_t key = t->end_key;
		const unsigned cls = ((unsigned)t->end_orient << 1) | (t->cls & 1u);
		for (uint64_t s = tile_slot(key, cls, mask);; s = (s + 1) & mask) {
			const unsigned v = tab[s];
			if (v == 0)
				break;
			const TileRec* o = recs + (v - 1);
			if (o->key == key && o->cls == cls) {
				t->next = v;
				break;
			}
		}
	}
}

/** a canonical hash occurring twice in one (untrimmed) path means the tile splice skipped an
 *  ER_CYCLE: flag the contig.  Every contig has its own open-addressing region
 *  [tab_off[c], tab_off[c+1]) keyed by the full 64-bit canonical hash, so a hit is a genuine repeat
 *  (a false alarm would cost a vertex-by-vertex walk of a possibly Mbp-long unitig). */
__global__ void __launch_bounds__(256)
k_repeat_check(const ContigRec* __restrict__ recs, unsigned n_contigs, const uint64_t* __restrict__ cslot,
               const uint64_t* __restrict__ ch0, unsigned long long* tab, const uint64_t* __restrict__ tab_off,
               uint8_t* __restrict__ flag)
{
	const uint64_t total = cslot[n_contigs];
	for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < total + 2ULL * n_contigs;
	     s += (uint64_t)gridDim.x * blockDim.x) {
		unsigned c;
		uint64_t h;
		if (s < total) {
			// contig of slot s
			unsigned lo = 0, hi = n_contigs;
			while (lo < hi) {
				const unsigned mid = (lo + hi) / 2;
				if (cslot[mid + 1] <= s)
					lo = mid + 1;
				else
					hi = mid;
			}
			c = lo;
			const uint64_t j = s - cslot[c], nk = cslot[c + 1] - cslot[c];
			const unsigned fl = recs[c].flags;
			if (((fl & 1) && j == 0) || ((fl & 2) && j == nk - 1))
				continue; // preprocessCircularContig's intentional duplicate
			h = ch0[s];
		} else {
			// the trimmed-off end vertices
			const uint64_t e = s - total;
			c = (unsigned)(e >> 1);
			const unsigned fl = recs[c].flags;
			if (e & 1) {
				if (!(fl & 8))
					continue;
				h = recs[c].back_h;
			} else {
				if (!(fl & 4))
					continue;
				h = recs[c].front_h;
			}
		}
		const unsigned long long key = h ? h : 1ULL; // 0 marks an empty slot
		const uint64_t base = tab_off[c], size = tab_off[c + 1] - base;
		uint64_t t = __umul64hi(key * 0xD6E8FEB86659FD93ULL, size);
		for (;;) {
			const unsigned long long old = atomicCAS(tab + base + t, 0ULL, key);
			if (old == 0ULL)
				break;
			if (old == key) {
				flag[c] = 1;
				break;
			}
			if (++t == size)
				t = 0;
		}
	}
}

/** dense ASCII copies of the ordered unitigs (pathToSeq output as characters) */
__global__ void __launch_bounds__(256)
k_gather(const ContigRec* __restrict__ recs, const unsigned* __restrict__ seg_contig, const uint64_t* __restrict__ seg_beg,
         const unsigned* __restrict__ seg_len, unsigned n_segs, const uint64_t* __restrict__ coffs, uint8_t* __restrict__ out,
         unsigned k, const __grid_constant__ RollTab rt)
{
	// one block per segment of a unitig (long unitigs are cut so that the copy uses the whole GPU);
	// seg_beg is the absolute offset in `out`, seg_len includes the k-1 overlap (harmlessly copied twice)
	for (unsigned sgi = blockIdx.x; sgi < n_segs; sgi += gridDim.x) {
		const unsigned c = seg_contig[sgi];
		const uint64_t rel = seg_beg[sgi] - coffs[c];
		const uint8_t* s = reinterpret_cast<const uint8_t*>(recs[c].seq) + rel;
		uint8_t* d = out + seg_beg[sgi];
		for (unsigned i = threadIdx.x; i < seg_len[sgi]; i += blockDim.x)
			d[i] = "ACGT"[s[i] & 3];
		if (rt.nmask && recs[c].len < 2 * k - 2) {
			// spaced seed: columns no vertex writes stay 'N' (pathToSeq, bloom-dbg.h:139-155); only paths of fewer than
			// k-1 vertices have any, and those are a single segment
			__syncthreads();
			const unsigned n = recs[c].len - k + 1;
			for (unsigned col = n + threadIdx.x; col + 1 < k; col += blockDim.x)
				if (!column_written(rt, k, n, col))
					d[col] = 'N';
		}
	}
}

// ------------------------------------------------------------------------------------------
// K5: ordered replay by one CTA (outputContig, bloom-dbg.h:538-620, and the "visited" test :823)
// ------------------------------------------------------------------------------------------
struct EndSet { // KmerHash contigEndKmers (bloom-dbg.h:37-47,992-993), keyed by canonical hash
	unsigned long long* tab;
	unsigned cap; // power of two
	unsigned* n;  // [0] entries, [1] has_zero
};
__device__ bool endset_contains(const EndSet& e, uint64_t key)
{
	if (key == 0)
		return e.n[1] != 0;
	for (uint64_t s = pathset_slot(key, e.cap);; s = (s + 1) & (e.cap - 1)) {
		const unsigned long long v = e.tab[s];
		if (v == key)
			return true;
		if (v == 0)
			return false;
	}
}
__device__ void endset_insert(const EndSet& e, uint64_t key)
{
	if (key == 0) {
		e.n[1] = 1;
		return;
	}
	for (uint64_t s = pathset_slot(key, e.cap);; s = (s + 1) & (e.cap - 1)) {
		const unsigned long long v = e.tab[s];
		if (v == key)
			return;
		if (v == 0) {
			e.tab[s] = key;
			++e.n[0];
			return;
		}
	}
}
__global__ void k_endset_rehash(const unsigned long long* o, unsigned ocap, unsigned long long* nt, unsigned ncap)
{
	for (unsigned s = blockIdx.x * blockDim.x + threadIdx.x; s < ocap; s += gridDim.x * blockDim.x) {
		const unsigned long long v = o[s];
		if (v == 0)
			continue;
		uint64_t t = pathset_slot(v, ncap);
		while (atomicCAS(nt + t, 0ULL, v) != 0ULL)
			t = (t + 1) & (ncap - 1);
	}
}

/** identity of outputContig's end vertices with a spaced seed (bloom-dbg.h:556-564): the k characters ('N' columns
 *  included; 'N' is its own complement and sorts between G and T) are put in their string-canonical orientation
 *  (Common/Sequence.h:39-44), and operator== then compares the '1' positions -- so the key is the masked forward hash
 *  of that orientation. */
__device__ uint64_t end_identity(const uint8_t* s, unsigned k, const uint8_t* care)
{
	bool use_rc = false;
	for (unsigned i = 0; i < k; ++i) {
		const uint8_t a = s[i], t = s[k - 1 - i];
		const uint8_t b = t == 'A' ? 'T' : t == 'C' ? 'G' : t == 'G' ? 'C' : t == 'T' ? 'A' : t;
		if (a != b) {
			use_rc = b < a;
			break;
		}
	}
	uint64_t f = 0;
	for (unsigned i = 0; i < k; ++i)
		if (care[i]) {
			const unsigned code = use_rc ? 3 - (base_code(s[k - 1 - i]) & 3) : (base_code(s[i]) & 3);
			f ^= srol_n(seed_of(code), k - 1 - i);
		}
	return f;
}

struct ReplayIO {
	// speculated reads, in file order
	const unsigned* spec;        // read index in the batch
	const unsigned* spec_cbeg;   // [n_spec + 1] first contig of each read
	unsigned n_spec;
	// reads
	const uint64_t* slot_offs;
	const uint64_t* h0;
	// contigs (ordered)
	const uint64_t* cslot;       // [n_contigs + 1] k-mer slot offsets into ch0
	const uint64_t* ch0;
	const unsigned* clen;
	// spaced seed only (care == nullptr otherwise): the unitig characters, for the identity of the end k-mers
	const uint8_t* cseq;
	const uint64_t* coffs;
	const uint8_t* care;
	// outputs
	uint8_t* rcode;              // per speculated read: RC_ALL_KMERS_VISITED or RC_GENERATED_CONTIGS
	uint8_t* caccept;            // per contig: 1 = printed
	unsigned* ccov;              // per contig: coverage
};

/** contigs with at least this many k-mers are replayed by whole-grid kernels (k_big_*) */
constexpr unsigned kBigContig = 1u << 15;

/**
 * Replays reads s0.. in file order with ONE CTA, starting at contig index cs and stopping before
 * contig index ce (a "big" contig that the host hands to k_big_check / k_big_apply, or the end).
 * A read whose first contig is >= cs has not been started: its "all k-mers assembled" test runs
 * here; otherwise its verdict is already in rcode[].
 */
__device__ void replay_segment(const ReplayIO& io, unsigned s0, unsigned cs, unsigned ce, const HashCfg& cfg, unsigned k,
                               const uint8_t* __restrict__ counters, uint8_t* bits, EndSet ends)
{
	__shared__ unsigned s_cov;
	__shared__ int s_flag;
	const unsigned tid = threadIdx.x, nt = blockDim.x;
	for (unsigned s = s0; s < io.n_spec; ++s) {
		const unsigned cb = io.spec_cbeg[s], cend = io.spec_cbeg[s + 1];
		if (cb > ce || (cb == ce && cs > cb))
			return;
		if (cb >= cs) {
			const unsigned r = io.spec[s];
			const uint64_t rs0 = io.slot_offs[r];
			const unsigned rnk = (unsigned)(io.slot_offs[r + 1] - rs0);
			// skip reads in previously assembled regions (bloom-dbg.h:823-827)
			int all = 1;
			for (unsigned base = 0; base < rnk && all; base += nt) {
				const unsigned j = base + tid;
				int ok = 1;
				if (j < rnk) {
					const uint64_t h = io.h0[rs0 + j];
					for (unsigned i = 0; i < cfg.H; ++i) {
						const uint64_t p = nth_pos(h, cfg, i);
						ok &= (__ldcg(bits + (p >> 3)) >> (p & 7)) & 1;
					}
				}
				all = __syncthreads_and(ok);
			}
			if (tid == 0)
				io.rcode[s] = all ? RC_ALL_KMERS_VISITED : RC_GENERATED_CONTIGS;
			if (all)
				continue;
		} else {
			if (__ldcg(io.rcode + s) == RC_ALL_KMERS_VISITED)
				continue;
		}
		for (unsigned c = cb > cs ? cb : cs; c < cend; ++c) {
			if (c >= ce)
				return;
			const uint64_t c0 = io.cslot[c];
			const unsigned nk = (unsigned)(io.cslot[c + 1] - c0);
			const unsigned len = io.clen[c];
			int redundant;
			if (len < k + kFpTrim - 1) {
				// very short contigs: exact table of end k-mers (bloom-dbg.h:576-586)
				if (tid == 0) {
					uint64_t v1 = io.ch0[c0], v2 = io.ch0[c0 + nk - 1];
					if (io.care) {
						const uint8_t* cs = io.cseq + io.coffs[c];
						v1 = end_identity(cs, k, io.care);
						v2 = end_identity(cs + len - k, k, io.care);
					}
					int red = endset_contains(ends, v1) && endset_contains(ends, v2);
					if (!red) {
						endset_insert(ends, v1);
						endset_insert(ends, v2);
					}
					s_flag = red;
				}
				__syncthreads();
				redundant = s_flag;
				__syncthreads();
			} else {
				redundant = 1; // allKmersInBloom(seq, assembledKmerSet) (bloom-dbg.h:588)
				for (unsigned base = 0; base < nk && redundant; base += nt) {
					const unsigned j = base + tid;
					int ok = 1;
					if (j < nk) {
						const uint64_t h = io.ch0[c0 + j];
						for (unsigned i = 0; i < cfg.H; ++i) {
							const uint64_t p = nth_pos(h, cfg, i);
							ok &= (__ldcg(bits + (p >> 3)) >> (p & 7)) & 1;
						}
					}
					redundant = __syncthreads_and(ok);
				}
			}
			if (redundant) {
				if (tid == 0)
					io.caccept[c] = 0;
				continue;
			}
			// addKmersToBloom(seq, assembledKmerSet) + getSeqAbsoluteKmerCoverage (bloom-dbg.h:83-109,594-602)
			if (tid == 0)
				s_cov = 0;
			__syncthreads();
			unsigned cov = 0;
			for (unsigned j = tid; j < nk; j += nt) {
				const uint64_t h = io.ch0[c0 + j];
				unsigned mn = 255;
				for (unsigned i = 0; i < cfg.H; ++i) {
					const uint64_t p = nth_pos(h, cfg, i);
					const uint64_t byte = p >> 3;
					atomicOr(reinterpret_cast<unsigned*>(bits + (byte & ~3ULL)), 1u << ((p & 7) + 8 * (byte & 3)));
					mn = min(mn, (unsigned)__ldcg(counters + p));
				}
				cov += mn;
			}
			for (int d = 16; d; d >>= 1)
				cov += __shfl_down_sync(0xffffffffu, cov, d);
			if ((tid & 31) == 0 && cov)
				atomicAdd(&s_cov, cov);
			__threadfence();
			__syncthreads();
			if (tid == 0) {
				io.caccept[c] = 1;
				io.ccov[c] = s_cov;
			}
			__syncthreads();
		}
	}
}

/** big contig c, step 1 (whole grid): redundant unless some k-mer is not yet assembled.
 *  caccept[c] was zeroed by the host; any thread that finds a missing k-mer sets it. */
__device__ void big_check(const ReplayIO& io, unsigned c, const HashCfg& cfg, const uint8_t* __restrict__ bits)
{
	const uint64_t c0 = io.cslot[c];
	const unsigned nk = (unsigned)(io.cslot[c + 1] - c0);
	bool missing = false;
	for (unsigned j = blockIdx.x * blockDim.x + threadIdx.x; j < nk; j += gridDim.x * blockDim.x) {
		const uint64_t h = io.ch0[c0 + j];
		bool ok = true;
		for (unsigned i = 0; i < cfg.H; ++i) {
			const uint64_t p = nth_pos(h, cfg, i);
			ok &= (__ldcg(bits + (p >> 3)) >> (p & 7)) & 1;
		}
		missing |= !ok;
	}
	if (__any_sync(0xffffffffu, missing) && (threadIdx.x & 31) == 0)
		io.caccept[c] = 1;
}
/** step 2 (whole grid): mark its k-mers assembled and sum their counts (ccov[c] zeroed by the host) */
__device__ void big_apply(const ReplayIO& io, unsigned c, const HashCfg& cfg, const uint8_t* __restrict__ counters, uint8_t* bits)
{
	const uint64_t c0 = io.cslot[c];
	const unsigned nk = (unsigned)(io.cslot[c + 1] - c0);
	unsigned cov = 0;
	for (unsigned j = blockIdx.x * blockDim.x + threadIdx.x; j < nk; j += gridDim.x * blockDim.x) {
		const uint64_t h = io.ch0[c0 + j];
		unsigned mn = 255;
		for (unsigned i = 0; i < cfg.H; ++i) {
			const uint64_t p = nth_pos(h, cfg, i);
			const uint64_t byte = p >> 3;
			atomicOr(reinterpret_cast<unsigned*>(bits + (byte & ~3ULL)), 1u << ((p & 7) + 8 * (byte & 3)));
			mn = min(mn, (unsigned)__ldcg(counters + p));
		}
		cov += mn;
	}
	for (int d = 16; d; d >>= 1)
		cov += __shfl_down_sync(0xffffffffu, cov, d);
	if ((threadIdx.x & 31) == 0 && cov)
		atomicAdd(io.ccov + c, cov);
}

/**
 * K5: the whole ordered replay of one speculation round in ONE cooperative launch (round 1: one launch of a
 * one-CTA kernel per stretch between big contigs plus two whole-grid launches per big contig, 5 400 launches per job).
 * CTA 0 walks the reads in file order exactly like processRead's bookkeeping (replay_segment) up to the next big
 * contig; there the whole grid checks and, if it is not redundant, applies it, between grid barriers.  big[b] = index
 * of the b-th big contig, big_s[b] = the speculated read it belongs to.
 */
__global__ void __launch_bounds__(1024)
k_replay_all(ReplayIO io, unsigned n_contigs, const unsigned* __restrict__ big, const unsigned* __restrict__ big_s, unsigned n_big,
             const __grid_constant__ HashCfg cfg, unsigned k, const uint8_t* __restrict__ counters, uint8_t* bits, EndSet ends)
{
	cg::grid_group grid = cg::this_grid();
	unsigned seg_s = 0, seg_c = 0;
	for (unsigned b = 0; b <= n_big; ++b) {
		const unsigned c_big = b < n_big ? big[b] : n_contigs;
		if (blockIdx.x == 0)
			replay_segment(io, seg_s, seg_c, c_big, cfg, k, counters, bits, ends);
		__threadfence();
		grid.sync();
		if (b == n_big)
			break;
		const unsigned s_of = big_s[b];
		if (__ldcg(io.rcode + s_of) == RC_GENERATED_CONTIGS) { // uniform over the grid
			big_check(io, c_big, cfg, bits);
			__threadfence();
			grid.sync();
			if (__ldcg(io.caccept + c_big) != 0) {
				big_apply(io, c_big, cfg, counters, bits);
				__threadfence();
				grid.sync();
			}
		}
		seg_s = s_of;
		seg_c = c_big + 1;
	}
}

} // namespace abb

using namespace abb;

// =============================================================================================
// host side
// =============================================================================================
struct abb_assembler {
	abb_filter* solid = nullptr;
	abb_filter* assembled = nullptr;
	abb_assembly_params params = {};
	abb_assembly_counters counters = {};
	cudaStream_t stream = nullptr;
	uint64_t reads_seen = 0;
	int kw = 0;
	RollTab rt; // per-k roll constants + spaced-seed positions
	uint8_t* d_mpos = nullptr;
	const uint8_t* ext_codes = nullptr; // classification supplied by the caller for the next batch (device)
	uint64_t ext_n = 0;
	abb_comm* comm = nullptr;           // multi-GPU: classification, candidate scans and tile production are sharded over it
	DevBuf<uint8_t> gather;             // all-gather staging (world x padded slice)
	const uint8_t* cur_bases = nullptr; // device reads of the batch being processed
	const uint64_t* cur_offs = nullptr;

	// batch state (device)
	DevBuf<uint8_t> bases, valid, codes, vis, scan_tmp, cseq, cvalid, rcode, caccept;
	DevBuf<uint64_t> offs, slot_offs, h0, coffs, cslot, ch0;
	DevBuf<unsigned> cand, spec, spec_cbeg, clen, ccov, status, seg_contig, seg_len, big_idx, big_spec;
	DevBuf<uint64_t> seg_beg, seg_slot, rep_off;
	DevBuf<ContigRec> recs, recs_sorted;
	DevBuf<Frame> frames;
	DevBuf<uint64_t> look;
	unsigned scratch_warps = 0;
	uint8_t* d_arena = nullptr;
	unsigned long long arena_size = 0;
	unsigned long long* d_arena_top = nullptr;
	unsigned* d_nrecs = nullptr;
	// contigEndKmers
	unsigned long long* d_ends = nullptr;
	unsigned ends_cap = 0;
	unsigned* d_ends_n = nullptr;
	uint64_t ends_upper = 0; // upper bound on entries

	// tile store (abb_walk.cuh "Tiles"); persistent across batches
	bool tiles_on = true;
	TileRec* d_tiles = nullptr;
	unsigned tile_cap = 0;
	unsigned* d_tile_tab = nullptr;
	unsigned tile_tab_mask = 0;
	unsigned* d_tile_n = nullptr;       // [0] tiles stored, [1] work counter, [2] new markers
	uint8_t* d_tile_pool = nullptr;
	unsigned long long tile_pool_size = 0;
	unsigned long long* d_tile_pool_top = nullptr;
	unsigned long long* d_marker_set = nullptr;
	unsigned marker_set_mask = 0;
	DevBuf<unsigned long long> new_markers, rep_tab, walk_dbg;
	DevBuf<TileRec> tile_export;
	DevBuf<uint8_t> stage_bases, rep_flag;
	DevBuf<uint64_t> stage_hashes;
	uint64_t st_markers = 0, st_tiles = 0, st_fallbacks = 0;
	float ms_tiles = 0, ms_walk = 0, ms_stage = 0, ms_repeat = 0, ms_total = 0, ms_cand = 0;

	// speculation control
	unsigned spec_target = 512;
	unsigned spec_fixed = 0;
	// host outputs of the last batch
	std::vector<abb_contig> out_contigs;
	std::vector<char> out_seqs;
	std::vector<uint8_t> out_codes;
	std::vector<abb_trace_row> out_trace; // one row per contig handed to outputContig (params.reserved & 1)
	// statistics
	uint64_t st_iterations = 0, st_speculated = 0, st_wasted = 0, st_launches = 0, st_candidates = 0, st_contigs_tried = 0;
	float ms_classify = 0, ms_visited = 0, ms_extend = 0, ms_replay = 0;
	cudaEvent_t ev[2] = { nullptr, nullptr }, ev2[2] = { nullptr, nullptr };
};

namespace {

struct PhaseTimer { // CUDA-event time of a phase on the assembler stream
	abb_assembler* a;
	float* acc;
	PhaseTimer(abb_assembler* a_, float* acc_) : a(a_), acc(acc_) { cudaEventRecord(a->ev[0], a->stream); }
	void stop()
	{
		cudaEventRecord(a->ev[1], a->stream);
		cudaEventSynchronize(a->ev[1]);
		float ms = 0;
		cudaEventElapsedTime(&ms, a->ev[0], a->ev[1]);
		*acc += ms;
	}
};

constexpr unsigned kMaxSpec = 1024;
constexpr unsigned kMinSpec = 256;   // with tiles a round costs about the same latency for 64 or 1024 walkers, and wasted walks are cheap
constexpr unsigned long long kArenaDefault = 4ULL << 30;
static unsigned long long g_arena_hint = 0; // the arena size the previous assembler of this process ended up needing
constexpr unsigned long long kArenaMax = 96ULL << 30;

int ensure_scratch(abb_assembler* a, unsigned warps)
{
	if (warps <= a->scratch_warps)
		return ABB_OK;
	ABB_CHECK(a->frames.reserve((size_t)warps * kFrameCap));
	ABB_CHECK(a->look.reserve((size_t)warps * kLookCap));
	a->scratch_warps = warps;
	return ABB_OK;
}

int ensure_arena(abb_assembler* a, unsigned long long bytes)
{
	if (a->d_arena && a->arena_size >= bytes)
		return ABB_OK;
	if (a->d_arena)
		cudaFree(a->d_arena);
	a->d_arena = nullptr;
	a->arena_size = 0;
	ABB_CUDA(cudaMalloc((void**)&a->d_arena, bytes));
	a->arena_size = bytes;
	return ABB_OK;
}

int ensure_endset(abb_assembler* a, uint64_t extra)
{
	const uint64_t need = (a->ends_upper + extra) * 2 + 16;
	if (a->d_ends && need <= a->ends_cap)
		return ABB_OK;
	uint64_t ncap = a->ends_cap ? a->ends_cap : 1024;
	while (ncap < need)
		ncap <<= 1;
	ABB_REQUIRE(ncap <= (1ULL << 31), "contigEndKmers table too large");
	unsigned long long* nt = nullptr;
	ABB_CUDA(cudaMalloc((void**)&nt, ncap * sizeof(unsigned long long)));
	ABB_CUDA(cudaMemsetAsync(nt, 0, ncap * sizeof(unsigned long long), a->stream));
	if (a->d_ends) {
		k_endset_rehash<<<256, 256, 0, a->stream>>>(a->d_ends, a->ends_cap, nt, (unsigned)ncap);
		ABB_CUDA(cudaGetLastError());
		ABB_CUDA(cudaStreamSynchronize(a->stream));
		cudaFree(a->d_ends);
	}
	a->d_ends = nt;
	a->ends_cap = (unsigned)ncap;
	return ABB_OK;
}

WalkCfg walk_cfg(const abb_assembler* a)
{
	WalkCfg w;
	w.k = a->solid->k;
	w.trim = a->params.trim;
	w.threshold = a->solid->threshold;
	w.rt = a->rt;
	w.counters = a->solid->d_data;
	return w;
}

#define ABB_DISPATCH_KW(kw, ...)              \
	do {                                      \
		switch (kw) {                         \
		case 1: { constexpr int KW = 1; __VA_ARGS__; } break; \
		case 2: { constexpr int KW = 2; __VA_ARGS__; } break; \
		case 3: { constexpr int KW = 3; __VA_ARGS__; } break; \
		case 4: { constexpr int KW = 4; __VA_ARGS__; } break; \
		default: { constexpr int KW = 6; __VA_ARGS__; } break; \
		}                                     \
	} while (0)

template <typename T>
int h2d(DevBuf<T>& d, const std::vector<T>& h, cudaStream_t s)
{
	ABB_CHECK(d.reserve(h.size() + 1));
	if (!h.empty())
		ABB_CUDA(cudaMemcpyAsync(d.p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, s));
	return ABB_OK;
}

/** rank r holds `mine` = n_r bytes (n_r = its slice of n_total split as [r*n/w, (r+1)*n/w)); afterwards `all` holds the
 *  n_total bytes of every rank's slice in rank order.  One ncclAllGather over slices padded to the longest. */
int allgather_slices(abb_assembler* a, const uint8_t* mine, uint64_t n_total, uint8_t* all)
{
	const unsigned world = (unsigned)abb_comm_world(a->comm), rank = (unsigned)abb_comm_rank(a->comm);
	cudaStream_t st = a->stream;
	uint64_t mx = 0;
	for (unsigned r = 0; r < world; ++r)
		mx = std::max<uint64_t>(mx, (r + 1) * n_total / world - r * n_total / world);
	mx = (mx + 15) & ~15ULL;
	ABB_CHECK(a->gather.reserve(world * mx));
	const uint64_t lo = rank * n_total / world, up = (rank + 1) * n_total / world;
	if (up > lo)
		ABB_CUDA(cudaMemcpyAsync(a->gather.p + rank * mx, mine, up - lo, cudaMemcpyDeviceToDevice, st));
	ABB_CHECK(abb_comm_allgather_bytes(a->comm, a->gather.p, mx, st));
	for (unsigned r = 0; r < world; ++r) {
		const uint64_t l = r * n_total / world, u = (r + 1) * n_total / world;
		if (u > l)
			ABB_CUDA(cudaMemcpyAsync(all + l, a->gather.p + r * mx, u - l, cudaMemcpyDeviceToDevice, st));
	}
	return ABB_OK;
}

TileView tile_view(const abb_assembler* a, bool on)
{
	TileView v = { nullptr, nullptr, 0 };
	if (on && a->tiles_on && a->d_tile_tab) {
		v.recs = a->d_tiles;
		v.tab = a->d_tile_tab;
		v.mask = a->tile_tab_mask;
	}
	return v;
}

/** allocate the tile store on first use, sized from the number of solid k-mers in the filter */
int ensure_tile_store(abb_assembler* a)
{
	if (a->d_tile_tab || !a->tiles_on)
		return ABB_OK;
	uint64_t nz = 0, th = 0;
	ABB_CHECK(abb_filter_popcount(a->solid, &nz, &th));
	const uint64_t solid = th / std::max(1u, a->solid->H) + 1024; // ~ distinct k-mers with count >= kc
	const uint64_t markers = solid / (kMarkerMask + 1) * 2 + 4096;
	size_t free_b = 0, total_b = 0;
	cudaMemGetInfo(&free_b, &total_b);
	a->tile_cap = (unsigned)std::min<uint64_t>(markers * 4, 1u << 30);
	unsigned long long pool = std::min<unsigned long long>(solid * 4 * 9 * 3 / 2 + (1 << 20), (unsigned long long)(free_b * 0.25));
	uint64_t tab = 1;
	while (tab < (uint64_t)a->tile_cap * 2)
		tab <<= 1;
	uint64_t mset = 1;
	while (mset < markers * 4)
		mset <<= 1;
	ABB_CUDA(cudaMalloc((void**)&a->d_tiles, (size_t)a->tile_cap * sizeof(TileRec)));
	ABB_CUDA(cudaMalloc((void**)&a->d_tile_tab, tab * sizeof(unsigned)));
	ABB_CUDA(cudaMemsetAsync(a->d_tile_tab, 0, tab * sizeof(unsigned), a->stream));
	a->tile_tab_mask = (unsigned)(tab - 1);
	ABB_CUDA(cudaMalloc((void**)&a->d_marker_set, mset * sizeof(unsigned long long)));
	ABB_CUDA(cudaMemsetAsync(a->d_marker_set, 0, mset * sizeof(unsigned long long), a->stream));
	a->marker_set_mask = (unsigned)(mset - 1);
	ABB_CUDA(cudaMalloc((void**)&a->d_tile_pool, pool));
	a->tile_pool_size = pool;
	ABB_CUDA(cudaMalloc((void**)&a->d_tile_n, 4 * sizeof(unsigned)));
	ABB_CUDA(cudaMemsetAsync(a->d_tile_n, 0, 4 * sizeof(unsigned), a->stream));
	ABB_CUDA(cudaMalloc((void**)&a->d_tile_pool_top, sizeof(unsigned long long)));
	ABB_CUDA(cudaMemsetAsync(a->d_tile_pool_top, 0, sizeof(unsigned long long), a->stream));
	return ABB_OK;
}

/** several GPUs: the tiles this rank has just produced ([n0, n1) of the store, pool bytes [p0, p1)) go to every other
 *  rank and theirs are appended here; afterwards every rank holds all tiles (indices differ between ranks, content not) */
int exchange_tiles(abb_assembler* a, unsigned n0, unsigned n1, unsigned long long p0, unsigned long long p1)
{
	cudaStream_t st = a->stream;
	const unsigned world = (unsigned)abb_comm_world(a->comm), rank = (unsigned)abb_comm_rank(a->comm);
	// 1. how much does everybody have?
	ABB_CHECK(a->gather.reserve(world * 16 + 16));
	unsigned long long mine[2] = { n1 - n0, p1 - p0 };
	ABB_CUDA(cudaMemcpyAsync(a->gather.p + rank * 16, mine, 16, cudaMemcpyHostToDevice, st));
	ABB_CHECK(abb_comm_allgather_bytes(a->comm, a->gather.p, 16, st));
	std::vector<unsigned long long> all(2 * world);
	ABB_CUDA(cudaMemcpyAsync(all.data(), a->gather.p, world * 16, cudaMemcpyDeviceToHost, st));
	ABB_CUDA(cudaStreamSynchronize(st));
	// 2. where the others' tiles and pool segments land in my store
	std::vector<uint64_t> rec_off(world, 0), rec_bytes(world, 0), pool_off(world, 0), pool_bytes(world, 0);
	unsigned long long nt = n1, pt = (p1 + 15) & ~15ULL;
	for (unsigned r = 0; r < world; ++r) {
		if (r == rank)
			continue;
		rec_off[r] = (uint64_t)nt * sizeof(TileRec);
		rec_bytes[r] = all[2 * r] * sizeof(TileRec);
		pool_off[r] = pt;
		pool_bytes[r] = all[2 * r + 1];
		nt += all[2 * r];
		pt += (all[2 * r + 1] + 15) & ~15ULL;
	}
	ABB_REQUIRE(nt <= a->tile_cap && pt <= a->tile_pool_size, "tile store too small for the merged tiles (%llu tiles, %llu pool bytes)", nt, pt);
	// 3. my records with pool-relative pointers, then the two exchanges
	ABB_CHECK(a->tile_export.reserve((size_t)(n1 - n0) + 1));
	if (n1 > n0)
		k_export_tiles<<<blocks_for(n1 - n0, 256), 256, 0, st>>>(a->d_tiles, n0, n1 - n0, a->d_tile_pool + p0, a->tile_export.p);
	ABB_CUDA(cudaGetLastError());
	ABB_CHECK(abb_comm_exchange_bytes(a->comm, a->tile_export.p, (uint64_t)(n1 - n0) * sizeof(TileRec), a->d_tiles, rec_off.data(), rec_bytes.data(), st));
	ABB_CHECK(abb_comm_exchange_bytes(a->comm, a->d_tile_pool + p0, p1 - p0, a->d_tile_pool, pool_off.data(), pool_bytes.data(), st));
	for (unsigned r = 0; r < world; ++r) {
		if (r == rank || all[2 * r] == 0)
			continue;
		const unsigned first = (unsigned)(rec_off[r] / sizeof(TileRec)), n = (unsigned)all[2 * r];
		k_import_tiles<<<blocks_for(n, 256), 256, 0, st>>>(a->d_tiles, first, n, a->d_tile_pool + pool_off[r], a->d_tile_tab, a->tile_tab_mask);
	}
	ABB_CUDA(cudaGetLastError());
	const unsigned nt32 = (unsigned)nt;
	ABB_CUDA(cudaMemcpyAsync(a->d_tile_n, &nt32, sizeof nt32, cudaMemcpyHostToDevice, st));
	ABB_CUDA(cudaMemcpyAsync(a->d_tile_pool_top, &pt, sizeof pt, cudaMemcpyHostToDevice, st));
	ABB_CUDA(cudaStreamSynchronize(st));
	a->st_launches += 2 + world;
	return ABB_OK;
}

/** markers among this batch's k-mers that have no tiles yet get their four tiles */
int produce_tiles(abb_assembler* a, uint64_t n_reads, uint64_t n_slots)
{
	if (!a->tiles_on || n_slots == 0)
		return ABB_OK;
	PhaseTimer tt(a, &a->ms_tiles);
	ABB_CHECK(ensure_tile_store(a));
	abb_filter* f = a->solid;
	cudaStream_t st = a->stream;
	const WalkCfg w = walk_cfg(a);
	const unsigned world = a->comm ? (unsigned)abb_comm_world(a->comm) : 1u, rank = a->comm ? (unsigned)abb_comm_rank(a->comm) : 0u;
	const unsigned out_cap = (unsigned)std::min<uint64_t>(n_slots / (kMarkerMask + 1) * 2 + 4096, a->marker_set_mask / 2 + 1);
	ABB_CHECK(a->new_markers.reserve(out_cap));
	ABB_CUDA(cudaMemsetAsync(a->d_tile_n + 1, 0, 2 * sizeof(unsigned), st));
	k_find_markers<<<sm_count() * 16, 256, 0, st>>>(a->h0.p, a->valid.p, a->slot_offs.p, n_reads, n_slots, w, f->cfg, a->d_marker_set,
	                                         a->marker_set_mask, a->new_markers.p, a->d_tile_n + 2, out_cap, world, rank);
	ABB_CUDA(cudaGetLastError());
	unsigned nm = 0, n0 = 0;
	unsigned long long p0 = 0;
	ABB_CUDA(cudaMemcpyAsync(&nm, a->d_tile_n + 2, sizeof nm, cudaMemcpyDeviceToHost, st));
	ABB_CUDA(cudaMemcpyAsync(&n0, a->d_tile_n, sizeof n0, cudaMemcpyDeviceToHost, st));
	ABB_CUDA(cudaMemcpyAsync(&p0, a->d_tile_pool_top, sizeof p0, cudaMemcpyDeviceToHost, st));
	ABB_CUDA(cudaStreamSynchronize(st));
	nm = std::min(nm, out_cap);
	n0 = std::min(n0, a->tile_cap);
	a->st_launches += 1;
	if (nm == 0 && world == 1) {
		tt.stop();
		return ABB_OK;
	}
	if (nm) {
		int sms = 132;
		cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, f->device);
		// persistent warps pulling (marker, orientation, direction) items from a counter: as many CTAs as fit
		static int tiles_per_sm = 0;
		if (tiles_per_sm == 0) {
			int n = 0;
			ABB_DISPATCH_KW(a->kw, (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_make_tiles<KW>, kWalkWarps * 32, 0)));
			tiles_per_sm = std::max(1, n);
		}
		const unsigned grid = (unsigned)std::min<uint64_t>(blocks_for((uint64_t)nm * 4, kWalkWarps), (uint64_t)sms * tiles_per_sm);
		const unsigned warps = grid * kWalkWarps;
		ABB_CHECK(ensure_scratch(a, warps));
		ABB_CHECK(a->stage_bases.reserve((size_t)warps * kTileCap));
		ABB_CHECK(a->stage_hashes.reserve((size_t)warps * kTileCap));
		TileStore ts = { a->d_tiles, a->d_tile_tab, a->tile_tab_mask, a->tile_cap, a->d_tile_n, a->d_tile_pool, a->tile_pool_size,
			             a->d_tile_pool_top };
		ABB_DISPATCH_KW(a->kw, (k_make_tiles<KW><<<grid, kWalkWarps * 32, 0, st>>>(a->cur_bases, a->cur_offs, a->new_markers.p, nm,
		                                                                          a->d_tile_n + 1, w, f->cfg, a->frames.p, a->look.p,
		                                                                          a->stage_bases.p, a->stage_hashes.p, ts)));
		ABB_CUDA(cudaGetLastError());
		a->st_launches += 1;
	}
	unsigned nt = 0;
	unsigned long long p1 = 0;
	ABB_CUDA(cudaMemcpyAsync(&nt, a->d_tile_n, sizeof nt, cudaMemcpyDeviceToHost, st));
	ABB_CUDA(cudaMemcpyAsync(&p1, a->d_tile_pool_top, sizeof p1, cudaMemcpyDeviceToHost, st));
	ABB_CUDA(cudaStreamSynchronize(st));
	nt = std::min(nt, a->tile_cap);
	p1 = std::min(p1, a->tile_pool_size);
	a->st_markers += nm;
	a->st_tiles = nt;
	if (world > 1) {
		ABB_CHECK(exchange_tiles(a, n0, nt, p0, p1));
		ABB_CUDA(cudaMemcpyAsync(&nt, a->d_tile_n, sizeof nt, cudaMemcpyDeviceToHost, st));
		ABB_CUDA(cudaStreamSynchronize(st));
		a->st_tiles = nt;
	}
	k_link_tiles<<<sm_count() * 8, 256, 0, st>>>(a->d_tiles, (unsigned)a->st_tiles, a->d_tile_tab, a->tile_tab_mask);
	ABB_CUDA(cudaGetLastError());
	a->st_launches += 1;
	tt.stop();
	return ABB_OK;
}

/** K4 over the reads listed in a->spec.p[0..n): returns the records (unsorted) and the per-read status.
 *  keep_arena: do not rewind the arena (results of an earlier launch of this round still live there). */
int run_extend(abb_assembler* a, unsigned n_spec, bool use_tiles, bool keep_arena, std::vector<ContigRec>& recs,
               std::vector<unsigned>& status)
{
	abb_filter* f = a->solid;
	cudaStream_t st = a->stream;
	ABB_CHECK(ensure_scratch(a, n_spec));
	ABB_CHECK(a->status.reserve(n_spec));
	unsigned rec_cap = std::max<unsigned>(n_spec * 8, 4096);
	status.assign(n_spec, 0);
	unsigned long long arena_mark = 0;
	if (keep_arena) {
		ABB_CUDA(cudaMemcpyAsync(&arena_mark, a->d_arena_top, sizeof arena_mark, cudaMemcpyDeviceToHost, st));
		ABB_CUDA(cudaStreamSynchronize(st));
	}
	for (;;) {
		ABB_CHECK(a->recs.reserve(rec_cap));
		unsigned long long* dbg = nullptr;
		if (getenv("ABB_ROUND_LOG")) {
			ABB_CHECK(a->walk_dbg.reserve(4ull * n_spec));
			ABB_CUDA(cudaMemsetAsync(a->walk_dbg.p, 0, 4ull * n_spec * sizeof(unsigned long long), st));
			dbg = a->walk_dbg.p;
		}
		ABB_CHECK(ensure_arena(a, a->arena_size ? a->arena_size : std::max(kArenaDefault, g_arena_hint)));
		ABB_CUDA(cudaMemcpyAsync(a->d_arena_top, &arena_mark, sizeof arena_mark, cudaMemcpyHostToDevice, st));
		ABB_CUDA(cudaMemsetAsync(a->d_nrecs, 0, sizeof(unsigned), st));
		const WalkCfg w = walk_cfg(a);
		const TileView tv = tile_view(a, use_tiles);
		cudaEventRecord(a->ev2[0], st);
		ABB_DISPATCH_KW(a->kw, (k_extend<KW><<<blocks_for(n_spec, kWalkWarps), kWalkWarps * 32, 0, st>>>(
		                           a->cur_bases, a->cur_offs, a->spec.p, n_spec, w, f->cfg, a->frames.p, a->look.p, a->d_arena, a->arena_size,
		                           a->d_arena_top, a->recs.p, a->d_nrecs, rec_cap, a->status.p, tv, dbg)));
		ABB_CUDA(cudaGetLastError());
		cudaEventRecord(a->ev2[1], st);
		++a->st_launches;
		unsigned nrecs = 0;
		ABB_CUDA(cudaMemcpyAsync(&nrecs, a->d_nrecs, sizeof nrecs, cudaMemcpyDeviceToHost, st));
		ABB_CUDA(cudaMemcpyAsync(status.data(), a->status.p, n_spec * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
		ABB_CUDA(cudaStreamSynchronize(st));
		{
			float ms = 0;
			cudaEventElapsedTime(&ms, a->ev2[0], a->ev2[1]);
			a->ms_walk += ms;
		}
		if (dbg) { // the slowest walk of this launch, by stage (SM clock ticks -> ms at 1.9 GHz)
			std::vector<unsigned long long> h(4ull * n_spec);
			cudaMemcpy(h.data(), dbg, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
			unsigned best = 0;
			unsigned long long bt = 0;
			for (unsigned i = 0; i < n_spec; ++i) {
				const unsigned long long t = h[4 * i] + h[4 * i + 1] + h[4 * i + 2] + h[4 * i + 3];
				if (t > bt) {
					bt = t;
					best = i;
				}
			}
			fprintf(stderr, "  k_extend %u walkers: slowest #%u extend-left %.1f extend-right %.1f materialise+trim %.1f mark_covered %.1f ms\n", n_spec, best,
			        h[4 * best] / 1.9e6, h[4 * best + 1] / 1.9e6, h[4 * best + 2] / 1.9e6, h[4 * best + 3] / 1.9e6);
		}
		if (nrecs > rec_cap) { // record buffer too small: rerun with room for everything
			rec_cap = nrecs + nrecs / 4 + 16;
			continue;
		}
		bool arena_fail = false;
		for (unsigned i = 0; i < n_spec; ++i)
			arena_fail |= (status[i] & (1u << 3)) != 0;
		if (arena_fail && !keep_arena) {
			// out of unitig scratch: grow the arena (free memory permitting) and rerun
			size_t free_b = 0, total_b = 0;
			cudaMemGetInfo(&free_b, &total_b);
			const unsigned long long room = a->arena_size + (unsigned long long)(free_b * 0.8);
			const unsigned long long bigger = std::min<unsigned long long>(std::min(kArenaMax, room), a->arena_size * 4);
			if (bigger > a->arena_size + (1ULL << 28)) {
				ABB_CHECK(ensure_arena(a, bigger));
				g_arena_hint = std::max(g_arena_hint, bigger);
				continue;
			}
		}
		recs.resize(nrecs);
		if (nrecs)
			ABB_CUDA(cudaMemcpyAsync(recs.data(), a->recs.p, nrecs * sizeof(ContigRec), cudaMemcpyDeviceToHost, st));
		ABB_CUDA(cudaStreamSynchronize(st));
		return ABB_OK;
	}
}

/** sort records by (read, ordinal) and build the per-read / per-contig index arrays */
struct RoundLayout {
	std::vector<unsigned> spec_cbeg, clen;
	std::vector<uint64_t> coffs, cslot;
};
void layout_records(std::vector<ContigRec>& recs, unsigned n_ok, unsigned k, RoundLayout& L)
{
	recs.erase(std::remove_if(recs.begin(), recs.end(), [&](const ContigRec& r) { return r.spec >= n_ok; }), recs.end());
	std::sort(recs.begin(), recs.end(), [](const ContigRec& x, const ContigRec& y) {
		return x.spec != y.spec ? x.spec < y.spec : x.ordinal < y.ordinal;
	});
	const unsigned nc = (unsigned)recs.size();
	L.spec_cbeg.assign(n_ok + 1, 0);
	L.clen.resize(nc);
	L.coffs.assign(nc + 1, 0);
	L.cslot.assign(nc + 1, 0);
	for (unsigned c = 0; c < nc; ++c) {
		++L.spec_cbeg[recs[c].spec + 1];
		L.clen[c] = recs[c].len;
		L.coffs[c + 1] = L.coffs[c] + recs[c].len;
		L.cslot[c + 1] = L.cslot[c] + (recs[c].len - k + 1);
	}
	for (unsigned s = 0; s < n_ok; ++s)
		L.spec_cbeg[s + 1] += L.spec_cbeg[s];
}

/** upload the layout, gather the unitigs as ASCII and hash them */
int stage_contigs(abb_assembler* a, const std::vector<ContigRec>& recs, const RoundLayout& L)
{
	abb_filter* f = a->solid;
	cudaStream_t st = a->stream;
	const unsigned nc = (unsigned)recs.size();
	ABB_CHECK(h2d(a->recs_sorted, recs, st));
	ABB_CHECK(h2d(a->spec_cbeg, L.spec_cbeg, st));
	ABB_CHECK(h2d(a->clen, L.clen, st));
	ABB_CHECK(h2d(a->coffs, L.coffs, st));
	ABB_CHECK(h2d(a->cslot, L.cslot, st));
	ABB_CHECK(a->cseq.reserve(L.coffs[nc] + 16));
	ABB_CHECK(a->ch0.reserve(L.cslot[nc] + 1));
	ABB_CHECK(a->cvalid.reserve(L.cslot[nc] + 1));
	if (nc) {
		// cut the unitigs into segments of kSegWindows k-mers (+ k-1 bases of overlap)
		constexpr unsigned kSegWindows = 8192;
		std::vector<unsigned> seg_contig, seg_len;
		std::vector<uint64_t> seg_beg, seg_slot;
		for (unsigned c = 0; c < nc; ++c) {
			const unsigned nk = recs[c].len - f->k + 1;
			for (unsigned j = 0; j < nk; j += kSegWindows) {
				const unsigned w = std::min(kSegWindows, nk - j);
				seg_contig.push_back(c);
				seg_beg.push_back(L.coffs[c] + j);
				seg_len.push_back(w + f->k - 1);
				seg_slot.push_back(L.cslot[c] + j);
			}
		}
		const unsigned ns = (unsigned)seg_contig.size();
		ABB_CHECK(h2d(a->seg_contig, seg_contig, st));
		ABB_CHECK(h2d(a->seg_len, seg_len, st));
		ABB_CHECK(h2d(a->seg_beg, seg_beg, st));
		ABB_CHECK(h2d(a->seg_slot, seg_slot, st));
		cudaEventRecord(a->ev2[0], st);
		k_gather<<<std::min<unsigned>(ns, sm_count() * 16), 256, 0, st>>>(a->recs_sorted.p, a->seg_contig.p, a->seg_beg.p, a->seg_len.p, ns, a->coffs.p,
		                                                          a->cseq.p, f->k, a->rt);
		ABB_CUDA(cudaGetLastError());
		ABB_CHECK(launch_hash_segments(f->k, f->d_care, a->cseq.p, a->seg_beg.p, a->seg_len.p, a->seg_slot.p, ns, a->ch0.p, a->cvalid.p, st));
		cudaEventRecord(a->ev2[1], st);
		cudaEventSynchronize(a->ev2[1]);
		float ms = 0;
		cudaEventElapsedTime(&ms, a->ev2[0], a->ev2[1]);
		a->ms_stage += ms;
		a->st_launches += 2;
	}
	return ABB_OK;
}

/** one speculation round over candidates starting at *cursor; appends accepted contigs */
int speculate_round(abb_assembler* a, const std::vector<unsigned>& cand, size_t* cursor, uint64_t n_reads)
{
	abb_filter* f = a->solid;
	cudaStream_t st = a->stream;
	const size_t ncand = cand.size();
	// ---- K3b over a chunk of candidates; pick the first spec_target uncovered ones
	std::vector<unsigned> spec;
	size_t pos = *cursor;
	size_t chunk = std::max<size_t>(a->spec_target, 1024);
	PhaseTimer tv(a, &a->ms_visited);
	while (pos < ncand && spec.size() < a->spec_target) {
		const unsigned n = (unsigned)std::min(chunk, ncand - pos);
		ABB_CHECK(a->vis.reserve(n));
		{
			// pure per candidate against the CURRENT assembled filter (identical on every rank: the replay is replicated)
			const unsigned world = a->comm ? (unsigned)abb_comm_world(a->comm) : 1u, rank = a->comm ? (unsigned)abb_comm_rank(a->comm) : 0u;
			const unsigned vlo = (unsigned)((uint64_t)rank * n / world), vup = (unsigned)((uint64_t)(rank + 1) * n / world);
			if (vup > vlo)
				k_visited<<<blocks_for((uint64_t)(vup - vlo) * 32, 256), 256, 0, st>>>(a->cand.p, (unsigned)pos + vlo, vup - vlo, a->slot_offs.p, a->h0.p,
				                                                                      f->cfg, a->assembled->d_data, a->vis.p + vlo);
			ABB_CUDA(cudaGetLastError());
			++a->st_launches;
			if (world > 1)
				ABB_CHECK(allgather_slices(a, a->vis.p + vlo, n, a->vis.p));
		}
		std::vector<uint8_t> vis(n);
		ABB_CUDA(cudaMemcpyAsync(vis.data(), a->vis.p, n, cudaMemcpyDeviceToHost, st));
		ABB_CUDA(cudaStreamSynchronize(st));
		size_t i = 0;
		for (; i < n && spec.size() < a->spec_target; ++i) {
			if (vis[i]) {
				a->out_codes[cand[pos + i]] = RC_ALL_KMERS_VISITED;
				++a->counters.visited_reads;
			} else
				spec.push_back(cand[pos + i]);
		}
		pos += i;
		chunk = std::min<size_t>(chunk * 4, 1u << 22);
	}
	*cursor = pos;
	tv.stop();
	if (spec.empty())
		return ABB_OK;
	++a->st_iterations;
	a->st_speculated += spec.size();
	const float round_walk0 = a->ms_walk, round_rep0 = a->ms_repeat, round_vis0 = a->ms_visited, round_replay0 = a->ms_replay;
	const auto round_t0 = std::chrono::steady_clock::now();

	// ---- K4: extend all speculated reads (tiles on), then the exact vertex-by-vertex fallback for
	// reads whose tiled walk cycled or produced a path with a repeated vertex
	const unsigned n_spec = (unsigned)spec.size();
	std::vector<ContigRec> recs;
	std::vector<unsigned> status;
	RoundLayout L;
	unsigned n_ok = n_spec;
	{
		PhaseTimer te(a, &a->ms_extend);
		ABB_CHECK(h2d(a->spec, spec, st));
		ABB_CHECK(run_extend(a, n_spec, true, false, recs, status));
		std::vector<unsigned> redo; // indices into spec
		for (unsigned i = 0; i < n_spec; ++i) {
			if (status[i] & (1u << 4)) { // tile chain cycled
				redo.push_back(i);
				status[i] = 0;
			}
		}
		for (unsigned i = 0; i < n_spec; ++i)
			if (status[i] != 0) {
				n_ok = i;
				break;
			}
		if (n_ok == 0) {
			if (status[0] & ((1u << 1) | (1u << 2)))
				set_error("graph traversal exceeded the per-warp scratch bounds (lookAhead %u / trueBranch %u frames)", kLookCap, kFrameCap);
			else
				set_error("unitig scratch arena exhausted at %llu bytes", a->arena_size);
			return ABB_ENOMEM;
		}
		// repeat check on everything that was produced with tiles
		if (a->tiles_on && a->d_tile_tab) {
			std::vector<ContigRec> keep;
			for (auto& r : recs)
				if (r.spec < n_ok && std::find(redo.begin(), redo.end(), r.spec) == redo.end())
					keep.push_back(r);
			recs.swap(keep);
			layout_records(recs, n_ok, f->k, L);
			ABB_CHECK(stage_contigs(a, recs, L));
			const unsigned nc = (unsigned)recs.size();
			if (nc) {
				std::vector<uint64_t> tab_off(nc + 1, 0);
				for (unsigned c = 0; c < nc; ++c)
					tab_off[c + 1] = tab_off[c] + 2 * (L.cslot[c + 1] - L.cslot[c]) + 8;
				const uint64_t tab = tab_off[nc];
				ABB_CHECK(h2d(a->rep_off, tab_off, st));
				ABB_CHECK(a->rep_tab.reserve(tab));
				ABB_CHECK(a->rep_flag.reserve(nc));
				cudaEventRecord(a->ev2[0], st);
				ABB_CUDA(cudaMemsetAsync(a->rep_tab.p, 0, tab * sizeof(unsigned long long), st));
				ABB_CUDA(cudaMemsetAsync(a->rep_flag.p, 0, nc, st));
				k_repeat_check<<<sm_count() * 8, 256, 0, st>>>(a->recs_sorted.p, nc, a->cslot.p, a->ch0.p, a->rep_tab.p, a->rep_off.p, a->rep_flag.p);
				ABB_CUDA(cudaGetLastError());
				cudaEventRecord(a->ev2[1], st);
				++a->st_launches;
				std::vector<uint8_t> flag(nc);
				ABB_CUDA(cudaMemcpyAsync(flag.data(), a->rep_flag.p, nc, cudaMemcpyDeviceToHost, st));
				ABB_CUDA(cudaStreamSynchronize(st));
				{
					float ms = 0;
					cudaEventElapsedTime(&ms, a->ev2[0], a->ev2[1]);
					a->ms_repeat += ms;
				}
				for (unsigned c = 0; c < nc; ++c)
					if (flag[c] && (redo.empty() || redo.back() != recs[c].spec) &&
					    std::find(redo.begin(), redo.end(), recs[c].spec) == redo.end())
						redo.push_back(recs[c].spec);
			}
		}
		redo.erase(std::remove_if(redo.begin(), redo.end(), [&](unsigned i) { return i >= n_ok; }), redo.end());
		if (!redo.empty()) {
			std::sort(redo.begin(), redo.end());
			a->st_fallbacks += redo.size();
			std::vector<unsigned> sub(redo.size());
			for (size_t i = 0; i < redo.size(); ++i)
				sub[i] = spec[redo[i]];
			ABB_CHECK(h2d(a->spec, sub, st));
			std::vector<ContigRec> recs2;
			std::vector<unsigned> status2;
			ABB_CHECK(run_extend(a, (unsigned)sub.size(), false, true, recs2, status2));
			for (size_t i = 0; i < sub.size(); ++i)
				if (status2[i] != 0) { // the serial walk itself ran out of scratch: end the round before this read
					n_ok = std::min(n_ok, redo[i]);
				}
			std::vector<ContigRec> merged;
			for (auto& r : recs)
				if (!std::binary_search(redo.begin(), redo.end(), r.spec))
					merged.push_back(r);
			for (auto& r : recs2) {
				r.spec = redo[r.spec];
				merged.push_back(r);
			}
			recs.swap(merged);
			ABB_CHECK(h2d(a->spec, spec, st)); // restore the full list for the replay
			if (n_ok == 0) {
				set_error("unitig scratch arena exhausted at %llu bytes", a->arena_size);
				return ABB_ENOMEM;
			}
		}
		layout_records(recs, n_ok, f->k, L);
		ABB_CHECK(stage_contigs(a, recs, L));
		te.stop();
	}
	if (n_ok < n_spec) {
		// reads from the first failure on go back to the queue; speculate less next time.
		// Candidates after the failed read that this round already labelled "visited" are re-examined
		// when the scan resumes there (monotone, so the label will be the same): undo the bookkeeping.
		const unsigned failed_read = spec[n_ok];
		const size_t p = std::lower_bound(cand.begin(), cand.end(), failed_read) - cand.begin();
		for (size_t i = p; i < *cursor; ++i)
			if (a->out_codes[cand[i]] == RC_ALL_KMERS_VISITED) {
				a->out_codes[cand[i]] = RC_CANDIDATE;
				--a->counters.visited_reads;
			}
		*cursor = p;
		a->spec_target = std::max(1u, n_ok);
		spec.resize(n_ok);
	}

	const unsigned nc = (unsigned)recs.size();
	const std::vector<unsigned>& spec_cbeg = L.spec_cbeg;
	const std::vector<unsigned>& clen = L.clen;
	const std::vector<uint64_t>& coffs = L.coffs;
	std::vector<uint8_t> rcode(n_ok), caccept(nc);
	std::vector<unsigned> ccov(nc);
	std::vector<uint64_t> hoff(nc + 1, 0); // where each accepted unitig lands in `seqs`
	std::vector<char> seqs;
	a->st_contigs_tried += nc;
	{
		PhaseTimer tr(a, &a->ms_replay);
		ABB_CHECK(a->rcode.reserve(n_ok));
		ABB_CHECK(a->caccept.reserve(nc + 1));
		ABB_CHECK(a->ccov.reserve(nc + 1));
		ABB_CHECK(ensure_endset(a, 2ull * nc));
		a->ends_upper += 2ull * nc;
		ReplayIO io;
		io.spec = a->spec.p;
		io.spec_cbeg = a->spec_cbeg.p;
		io.n_spec = n_ok;
		io.slot_offs = a->slot_offs.p;
		io.h0 = a->h0.p;
		io.cslot = a->cslot.p;
		io.ch0 = a->ch0.p;
		io.clen = a->clen.p;
		io.cseq = a->cseq.p;
		io.coffs = a->coffs.p;
		io.care = a->solid->d_care;
		io.rcode = a->rcode.p;
		io.caccept = a->caccept.p;
		io.ccov = a->ccov.p;
		EndSet ends = { a->d_ends, a->ends_cap, a->d_ends_n };
		if (nc) {
			ABB_CUDA(cudaMemsetAsync(a->caccept.p, 0, nc, st));
			ABB_CUDA(cudaMemsetAsync(a->ccov.p, 0, nc * sizeof(unsigned), st));
		}
		// one cooperative launch replays the whole round (k_replay_all)
		{
			std::vector<unsigned> big, big_s;
			unsigned s_of = 0;
			for (unsigned c = 0; c < nc; ++c) {
				if (clen[c] - f->k + 1 < kBigContig)
					continue;
				while (spec_cbeg[s_of + 1] <= c)
					++s_of;
				big.push_back(c);
				big_s.push_back(s_of);
			}
			ABB_CHECK(h2d(a->big_idx, big, st));
			ABB_CHECK(h2d(a->big_spec, big_s, st));
			static int replay_grid = 0;
			if (replay_grid == 0) {
				int per_sm = 0, sms = 0;
				ABB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_replay_all, 1024, 0));
				ABB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, f->device));
				replay_grid = std::max(1, per_sm) * sms;
			}
			unsigned n_big = (unsigned)big.size(), nc_arg = nc, k_arg = f->k;
			const unsigned* d_big = a->big_idx.p;
			const unsigned* d_big_s = a->big_spec.p;
			const uint8_t* d_counters = f->d_data;
			uint8_t* d_bits = a->assembled->d_data;
			void* params[] = { &io, &nc_arg, &d_big, &d_big_s, &n_big, &f->cfg, &k_arg, &d_counters, &d_bits, &ends };
			ABB_CUDA(cudaLaunchCooperativeKernel((void*)k_replay_all, dim3((unsigned)replay_grid), dim3(1024), params, 0, st));
			++a->st_launches;
		}
		ABB_CUDA(cudaGetLastError());
		ABB_CUDA(cudaMemcpyAsync(rcode.data(), a->rcode.p, n_ok, cudaMemcpyDeviceToHost, st));
		if (nc) {
			ABB_CUDA(cudaMemcpyAsync(caccept.data(), a->caccept.p, nc, cudaMemcpyDeviceToHost, st));
			ABB_CUDA(cudaMemcpyAsync(ccov.data(), a->ccov.p, nc * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
		}
		ABB_CUDA(cudaStreamSynchronize(st));
		// only the unitigs that were printed travel back to the host
		for (unsigned c = 0; c < nc; ++c)
			hoff[c + 1] = hoff[c] + (caccept[c] ? clen[c] : 0);
		seqs.resize(hoff[nc]);
		for (unsigned c = 0; c < nc; ++c)
			if (caccept[c])
				ABB_CUDA(cudaMemcpyAsync(seqs.data() + hoff[c], a->cseq.p + coffs[c], clen[c], cudaMemcpyDeviceToHost, st));
		ABB_CUDA(cudaStreamSynchronize(st));
		tr.stop();
	}

	// ---- collect
	unsigned wasted = 0;
	for (unsigned s = 0; s < n_ok; ++s) {
		a->out_codes[spec[s]] = rcode[s];
		if (rcode[s] == RC_ALL_KMERS_VISITED) {
			++a->counters.visited_reads;
			++wasted;
			continue;
		}
		for (unsigned c = spec_cbeg[s]; c < spec_cbeg[s + 1]; ++c) {
			if (a->params.reserved & 1u) { // ContigRecord (bloom-dbg.h:186-254): every contig that reached outputContig
				abb_trace_row tr;
				tr.contig_id = caccept[c] ? a->counters.contig_id : ~0ULL;
				tr.seed_read = a->reads_seen + spec[s];
				tr.length = clen[c];
				tr.seed_pos = recs[c].seed_pos;
				tr.left_n = recs[c].left_n;
				tr.right_n = recs[c].right_n;
				tr.left_code = recs[c].left;
				tr.right_code = recs[c].right;
				tr.redundant = caccept[c] ? 0 : 1;
				tr.pad = 0;
				a->out_trace.push_back(tr);
			}
			if (!caccept[c])
				continue;
			abb_contig oc;
			oc.seed_read = a->reads_seen + spec[s];
			oc.seq_offset = a->out_seqs.size();
			oc.length = clen[c];
			oc.coverage = ccov[c];
			a->out_contigs.push_back(oc);
			a->out_seqs.insert(a->out_seqs.end(), seqs.begin() + hoff[c], seqs.begin() + hoff[c] + clen[c]);
			a->out_seqs.push_back('\0');
			++a->counters.contig_id;
			a->counters.bases_assembled += clen[c];
		}
	}
	a->st_wasted += wasted;
	if (getenv("ABB_ROUND_LOG")) { // tuning aid: one line per speculation round
		unsigned long long longest = 0, accepted = 0;
		for (unsigned c = 0; c < nc; ++c) {
			longest = std::max<unsigned long long>(longest, clen[c]);
			accepted += caccept[c] ? 1 : 0;
		}
		fprintf(stderr, "round %llu: speculated %u wasted %u contigs %u accepted %llu longest %llu | visited %.1f walk %.1f repeat %.1f replay %.1f ms, wall %.1f ms\n",
		        (unsigned long long)a->st_iterations, n_ok, wasted, nc, accepted, longest, a->ms_visited - round_vis0, a->ms_walk - round_walk0,
		        a->ms_repeat - round_rep0, a->ms_replay - round_replay0,
		        std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - round_t0).count());
	}
	// adapt the amount of speculation: grow while most speculated reads were really needed
	if (n_ok == n_spec && !a->spec_fixed) {
		if (wasted * 2 <= n_ok)
			a->spec_target = std::min(kMaxSpec, a->spec_target * 2);
		else if (wasted * 20 > n_ok * 19)
			a->spec_target = std::max(kMinSpec, a->spec_target / 2);
	}
	(void)n_reads;
	return ABB_OK;
}

} // namespace

extern "C" {

int abb_assembler_create(abb_assembler** out, abb_filter* solid, const abb_assembly_params* params)
{
	ABB_REQUIRE(out && solid && params, "NULL argument");
	*out = nullptr;
	if (solid->kind != ABB_COUNTING) {
		set_error("the assembler needs a counting filter (CountingBloomFilter<uint8_t>), like abyss-bloom-dbg");
		return ABB_ESTATE;
	}
	if (!solid->mask.empty()) { // MaskedKmer::setMask / RollingBloomDBGVertex::compare (RollingBloomDBG.h:141-145)
		const std::string& m = solid->mask;
		ABB_REQUIRE(m.size() == solid->k, "spaced seed must be k characters long");
		ABB_REQUIRE(m.front() == '1' && m.back() == '1', "spaced seed must begin and end with '1's");
		ABB_REQUIRE(std::equal(m.begin(), m.end(), m.rbegin()), "spaced seed must be symmetric");
	}
	ABB_REQUIRE(solid->k >= 2, "k must be at least 2 for graph traversal");
	ABB_CUDA(cudaSetDevice(solid->device));
	abb_assembler* a = new (std::nothrow) abb_assembler();
	if (!a) {
		set_error("out of host memory");
		return ABB_ENOMEM;
	}
	a->solid = solid;
	a->params = *params;
	if (a->params.trim == 0xffffffffu)
		a->params.trim = solid->k; // bloom-dbg.cc:518-520
	a->kw = (int)((2 * solid->k + 63) / 64);
	a->rt = make_rolltab(solid->k);
	if (!solid->mask.empty()) {
		std::vector<uint8_t> mpos;
		for (unsigned i = 0; i < solid->k; ++i)
			if (solid->mask[i] == '0')
				mpos.push_back((uint8_t)i);
		if (!mpos.empty()) {
			if (cudaMalloc((void**)&a->d_mpos, mpos.size()) != cudaSuccess ||
			    cudaMemcpy(a->d_mpos, mpos.data(), mpos.size(), cudaMemcpyHostToDevice) != cudaSuccess) {
				set_error("cudaMalloc of the spaced-seed table failed");
				delete a;
				return ABB_ECUDA;
			}
			a->rt.nmask = (unsigned)mpos.size();
			a->rt.mpos = a->d_mpos;
		}
	}
	// tiles are keyed by vertex hash and assume that equal hashes continue identically; with a spaced seed two k-mers
	// can share the hash and differ on the don't-care positions, so those runs walk vertex by vertex
	a->tiles_on = getenv("ABB_NO_TILES") == nullptr && solid->mask.empty(); // env: debugging switch
	if (const char* sp = getenv("ABB_SPEC")) // tuning switch: fixed speculation width
		a->spec_fixed = a->spec_target = (unsigned)std::max(1, atoi(sp));
	// BloomFilter assembledKmerSet(solid.size(), solid.getHashNum(), solid.getKmerSize()) (bloom-dbg.h:910-911)
	int rc = abb_filter_create(&a->assembled, ABB_BIT, solid->size, solid->H, solid->k, 0, "", solid->device);
	if (rc != ABB_OK) {
		delete a;
		return rc;
	}
	auto fail = [&](cudaError_t e, const char* what) {
		set_error("%s: %s", what, cudaGetErrorString(e));
		abb_assembler_destroy(a);
		return e == cudaErrorMemoryAllocation ? ABB_ENOMEM : ABB_ECUDA;
	};
	cudaError_t e;
	a->stream = solid->stream; // one stream carries pass 1 and pass 2 of a filter
	if ((e = cudaEventCreate(&a->ev[0])) != cudaSuccess) return fail(e, "cudaEventCreate");
	if ((e = cudaEventCreate(&a->ev[1])) != cudaSuccess) return fail(e, "cudaEventCreate");
	if ((e = cudaEventCreate(&a->ev2[0])) != cudaSuccess) return fail(e, "cudaEventCreate");
	if ((e = cudaEventCreate(&a->ev2[1])) != cudaSuccess) return fail(e, "cudaEventCreate");
	if ((e = cudaMalloc((void**)&a->d_arena_top, sizeof(unsigned long long))) != cudaSuccess) return fail(e, "cudaMalloc");
	if ((e = cudaMalloc((void**)&a->d_nrecs, sizeof(unsigned))) != cudaSuccess) return fail(e, "cudaMalloc");
	if ((e = cudaMalloc((void**)&a->d_ends_n, 2 * sizeof(unsigned))) != cudaSuccess) return fail(e, "cudaMalloc");
	if ((e = cudaMemset(a->d_ends_n, 0, 2 * sizeof(unsigned))) != cudaSuccess) return fail(e, "cudaMemset");
	*out = a;
	return ABB_OK;
}

int abb_assembler_destroy(abb_assembler* a)
{
	if (!a)
		return ABB_OK;
	if (a->solid)
		cudaSetDevice(a->solid->device);
	if (a->stream)
		cudaStreamSynchronize(a->stream);
	abb_filter_destroy(a->assembled);
	a->bases.release(); a->valid.release(); a->codes.release(); a->vis.release(); a->scan_tmp.release();
	a->cseq.release(); a->cvalid.release(); a->rcode.release(); a->caccept.release();
	a->offs.release(); a->slot_offs.release(); a->h0.release(); a->coffs.release(); a->cslot.release(); a->ch0.release();
	a->cand.release(); a->spec.release(); a->spec_cbeg.release(); a->clen.release(); a->ccov.release(); a->status.release();
	a->recs.release(); a->recs_sorted.release(); a->frames.release(); a->look.release();
	cudaFree(a->d_mpos);
	cudaFree(a->d_tiles);
	cudaFree(a->d_tile_tab);
	cudaFree(a->d_tile_n);
	cudaFree(a->d_tile_pool);
	cudaFree(a->d_tile_pool_top);
	cudaFree(a->d_marker_set);
	a->rep_off.release();
	a->gather.release();
	a->walk_dbg.release();
	a->big_idx.release();
	a->big_spec.release();
	a->tile_export.release();
	a->seg_contig.release(); a->seg_len.release(); a->seg_beg.release(); a->seg_slot.release();
	a->new_markers.release(); a->rep_tab.release(); a->stage_bases.release(); a->rep_flag.release(); a->stage_hashes.release();
	cudaFree(a->d_arena);
	cudaFree(a->d_arena_top);
	cudaFree(a->d_nrecs);
	cudaFree(a->d_ends);
	cudaFree(a->d_ends_n);
	if (a->ev[0]) cudaEventDestroy(a->ev[0]);
	if (a->ev[1]) cudaEventDestroy(a->ev[1]);
	if (a->ev2[0]) cudaEventDestroy(a->ev2[0]);
	if (a->ev2[1]) cudaEventDestroy(a->ev2[1]);
	delete a;
	return ABB_OK;
}

/** slot offsets + K1 over the batch into a->h0 / a->valid, then (unless codes come from outside) K3a */
static int hash_and_classify(abb_assembler* a, const uint8_t* d_bases, const uint64_t* d_offs, uint64_t n_reads, bool classify,
                             uint64_t* total_out)
{
	abb_filter* f = a->solid;
	cudaStream_t st = a->stream;
	uint64_t total = 0;
	ABB_CHECK(compute_slot_offsets(f->k, d_offs, n_reads, a->slot_offs, a->scan_tmp, st, &total, &a->st_launches));
	ABB_CHECK(a->h0.reserve(total + 1));
	ABB_CHECK(a->valid.reserve(total + 1));
	ABB_CHECK(a->codes.reserve(n_reads));
	if (total)
		ABB_CHECK(launch_hash(nullptr, f->k, f->d_care, d_bases, d_offs, a->slot_offs.p, 0, n_reads, 0, a->h0.p, a->valid.p, st,
		                      &a->st_launches));
	*total_out = total;
	if (!classify)
		return ABB_OK;
	int sms = 132;
	cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, f->device);
	// K3a is pure per read: with a communicator every rank classifies its contiguous slice of the batch and the codes
	// are all-gathered
	const unsigned world = a->comm ? (unsigned)abb_comm_world(a->comm) : 1u, rank = a->comm ? (unsigned)abb_comm_rank(a->comm) : 0u;
	const uint64_t lo = rank * n_reads / world, up = (rank + 1) * n_reads / world;
	const unsigned grid = (unsigned)std::min<uint64_t>(blocks_for(std::max<uint64_t>(up - lo, 1), kWalkWarps), (uint64_t)sms * 8);
	ABB_CHECK(ensure_scratch(a, grid * kWalkWarps));
	const WalkCfg w = walk_cfg(a);
	if (up > lo)
		ABB_DISPATCH_KW(a->kw, (k_classify<KW><<<grid, kWalkWarps * 32, 0, st>>>(d_bases, d_offs + lo, a->slot_offs.p + lo, a->h0.p, a->valid.p,
		                                                                        up - lo, w, f->cfg, a->look.p, (int)a->params.read_log,
		                                                                        a->codes.p + lo)));
	ABB_CUDA(cudaGetLastError());
	++a->st_launches;
	if (world > 1)
		ABB_CHECK(allgather_slices(a, a->codes.p + lo, n_reads, a->codes.p));
	return ABB_OK;
}

static int process_batch(abb_assembler* a, const uint8_t* d_bases, const uint64_t* d_offs, uint64_t n_reads,
                         const abb_contig** contigs, uint64_t* n_contigs, const char** seqs)
{
	const auto t_begin = std::chrono::steady_clock::now();
	struct Total {
		abb_assembler* a;
		std::chrono::steady_clock::time_point t0;
		~Total() { a->ms_total += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
	} total_guard{ a, t_begin };
	abb_filter* f = a->solid;
	cudaStream_t st = a->stream;
	a->cur_bases = d_bases;
	a->cur_offs = d_offs;
	PhaseTimer tc(a, &a->ms_classify);
	uint64_t total = 0;
	const bool external = a->ext_codes != nullptr;
	ABB_CHECK(hash_and_classify(a, d_bases, d_offs, n_reads, !external, &total));
	if (external) { // classification done elsewhere (sharded over several GPUs): take it as is
		ABB_REQUIRE(a->ext_n == n_reads, "abb_assembler_set_codes: %llu codes for %llu reads", (unsigned long long)a->ext_n,
		            (unsigned long long)n_reads);
		ABB_CUDA(cudaMemcpyAsync(a->codes.p, a->ext_codes, n_reads, cudaMemcpyDeviceToDevice, st));
		a->ext_codes = nullptr;
	}
	ABB_CUDA(cudaMemcpyAsync(a->out_codes.data(), a->codes.p, n_reads, cudaMemcpyDeviceToHost, st));
	ABB_CUDA(cudaStreamSynchronize(st));
	tc.stop();

	const auto t_cand = std::chrono::steady_clock::now();
	// candidate list = indices of the reads classified RC_CANDIDATE, compacted on the device
	std::vector<unsigned> cand;
	{
		ABB_CHECK(a->cand.reserve(n_reads + 1));
		IsCandidate pred{ a->codes.p };
		thrust::counting_iterator<unsigned> first(0);
		size_t bytes = 0;
		ABB_CUDA(cub::DeviceSelect::If(nullptr, bytes, first, a->cand.p, a->d_nrecs, (int)n_reads, pred, st));
		ABB_CHECK(a->scan_tmp.reserve(bytes));
		ABB_CUDA(cub::DeviceSelect::If(a->scan_tmp.p, bytes, first, a->cand.p, a->d_nrecs, (int)n_reads, pred, st));
		unsigned nc = 0;
		ABB_CUDA(cudaMemcpyAsync(&nc, a->d_nrecs, sizeof nc, cudaMemcpyDeviceToHost, st));
		ABB_CUDA(cudaStreamSynchronize(st));
		cand.resize(nc);
		if (nc)
			ABB_CUDA(cudaMemcpyAsync(cand.data(), a->cand.p, (size_t)nc * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
		ABB_CUDA(cudaStreamSynchronize(st));
	}
	a->ms_cand += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_cand).count();
	a->counters.solid_reads += cand.size();
	a->st_candidates += cand.size();
	if (!cand.empty())
		ABB_CHECK(produce_tiles(a, n_reads, total));

	size_t cursor = 0;
	while (cursor < cand.size())
		ABB_CHECK(speculate_round(a, cand, &cursor, n_reads));

	a->counters.reads_processed += n_reads;
	a->reads_seen += n_reads;
	if (contigs) *contigs = a->out_contigs.data();
	if (n_contigs) *n_contigs = a->out_contigs.size();
	if (seqs) *seqs = a->out_seqs.data();
	return ABB_OK;
}

static int begin_batch(abb_assembler* a, uint64_t n_reads, const abb_contig** contigs, uint64_t* n_contigs, const char** seqs)
{
	ABB_REQUIRE(a, "NULL assembler");
	a->out_contigs.clear();
	a->out_seqs.clear();
	a->out_trace.clear();
	a->out_codes.assign(n_reads, RC_SHORTER_THAN_K);
	if (contigs) *contigs = nullptr;
	if (n_contigs) *n_contigs = 0;
	if (seqs) *seqs = nullptr;
	ABB_REQUIRE(n_reads < (1ULL << 31), "at most 2^31-1 reads per batch");
	ABB_CUDA(cudaSetDevice(a->solid->device));
	// the filters may have been written on their own streams
	ABB_CUDA(cudaStreamSynchronize(a->solid->stream));
	ABB_CUDA(cudaStreamSynchronize(a->assembled->stream));
	return ABB_OK;
}

int abb_assembler_process_reads(abb_assembler* a, const char* bases, const uint64_t* offsets, uint64_t n_reads,
                                const abb_contig** contigs, uint64_t* n_contigs, const char** seqs)
{
	ABB_CHECK(begin_batch(a, n_reads, contigs, n_contigs, seqs));
	if (n_reads == 0)
		return ABB_OK;
	ABB_REQUIRE(bases && offsets, "NULL read buffers");
	ABB_REQUIRE(offsets[0] == 0, "offsets[0] must be 0");
	const uint64_t n_bases = offsets[n_reads];
	ABB_CHECK(a->bases.reserve(n_bases + 16));
	ABB_CHECK(a->offs.reserve(n_reads + 1));
	ABB_CUDA(cudaMemcpyAsync(a->bases.p, bases, n_bases, cudaMemcpyHostToDevice, a->stream));
	ABB_CUDA(cudaMemcpyAsync(a->offs.p, offsets, (n_reads + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, a->stream));
	return process_batch(a, a->bases.p, a->offs.p, n_reads, contigs, n_contigs, seqs);
}

int abb_assembler_process_reads_dev(abb_assembler* a, const char* d_bases, const uint64_t* d_offsets, uint64_t n_reads,
                                    const abb_contig** contigs, uint64_t* n_contigs, const char** seqs)
{
	ABB_CHECK(begin_batch(a, n_reads, contigs, n_contigs, seqs));
	if (n_reads == 0)
		return ABB_OK;
	ABB_REQUIRE(d_bases && d_offsets, "NULL read buffers");
	return process_batch(a, (const uint8_t*)d_bases, d_offsets, n_reads, contigs, n_contigs, seqs);
}

int abb_assembler_stats(const abb_assembler* a, abb_assembly_stats* out)
{
	ABB_REQUIRE(a && out, "NULL argument");
	out->rounds = a->st_iterations;
	out->speculated_reads = a->st_speculated;
	out->wasted_reads = a->st_wasted;
	out->candidates = a->st_candidates;
	out->contigs_tried = a->st_contigs_tried;
	out->launches = a->st_launches;
	out->ms_classify = a->ms_classify;
	out->ms_visited = a->ms_visited;
	out->ms_extend = a->ms_extend;
	out->ms_replay = a->ms_replay;
	out->ms_tiles = a->ms_tiles;
	out->ms_walk = a->ms_walk;
	out->ms_total = a->ms_total;
	out->ms_cand = a->ms_cand;
	out->ms_stage = a->ms_stage;
	out->ms_repeat = a->ms_repeat;
	out->markers = a->st_markers;
	out->tiles = a->st_tiles;
	out->serial_fallbacks = a->st_fallbacks;
	return ABB_OK;
}

int abb_assembler_classify_dev(abb_assembler* a, const char* d_bases, const uint64_t* d_offsets, uint64_t n_reads, uint8_t* d_codes)
{
	ABB_REQUIRE(a, "NULL assembler");
	if (n_reads == 0)
		return ABB_OK;
	ABB_REQUIRE(d_bases && d_offsets && d_codes, "NULL buffer");
	ABB_CUDA(cudaSetDevice(a->solid->device));
	ABB_CUDA(cudaStreamSynchronize(a->solid->stream));
	PhaseTimer tc(a, &a->ms_classify);
	uint64_t total = 0;
	ABB_CHECK(hash_and_classify(a, (const uint8_t*)d_bases, d_offsets, n_reads, true, &total));
	ABB_CUDA(cudaMemcpyAsync(d_codes, a->codes.p, n_reads, cudaMemcpyDeviceToDevice, a->stream));
	ABB_CUDA(cudaStreamSynchronize(a->stream));
	tc.stop();
	return ABB_OK;
}

int abb_assembler_set_codes(abb_assembler* a, const uint8_t* d_codes, uint64_t n_reads)
{
	ABB_REQUIRE(a, "NULL assembler");
	a->ext_codes = d_codes;
	a->ext_n = n_reads;
	return ABB_OK;
}

int abb_assembler_reset(abb_assembler* a)
{
	ABB_REQUIRE(a, "NULL assembler");
	ABB_CUDA(cudaSetDevice(a->solid->device));
	cudaStream_t st = a->stream;
	ABB_CUDA(cudaStreamSynchronize(st));
	ABB_CHECK(abb_filter_clear(a->assembled));
	if (a->d_ends)
		ABB_CUDA(cudaMemsetAsync(a->d_ends, 0, (size_t)a->ends_cap * sizeof(unsigned long long), st));
	ABB_CUDA(cudaMemsetAsync(a->d_ends_n, 0, 2 * sizeof(unsigned), st));
	a->ends_upper = 0;
	if (a->d_tile_tab) { // the tiles describe the old contents of the solid filter: forget them, keep the memory
		ABB_CUDA(cudaMemsetAsync(a->d_tile_tab, 0, ((size_t)a->tile_tab_mask + 1) * sizeof(unsigned), st));
		ABB_CUDA(cudaMemsetAsync(a->d_marker_set, 0, ((size_t)a->marker_set_mask + 1) * sizeof(unsigned long long), st));
		ABB_CUDA(cudaMemsetAsync(a->d_tile_n, 0, 4 * sizeof(unsigned), st));
		ABB_CUDA(cudaMemsetAsync(a->d_tile_pool_top, 0, sizeof(unsigned long long), st));
	}
	ABB_CUDA(cudaStreamSynchronize(st));
	a->counters = abb_assembly_counters{};
	a->reads_seen = 0;
	a->spec_target = a->spec_fixed ? a->spec_fixed : 512;
	a->st_iterations = a->st_speculated = a->st_wasted = a->st_launches = a->st_candidates = a->st_contigs_tried = 0;
	a->st_markers = a->st_tiles = a->st_fallbacks = 0;
	a->ms_classify = a->ms_visited = a->ms_extend = a->ms_replay = a->ms_tiles = a->ms_walk = a->ms_stage = a->ms_repeat = a->ms_total = a->ms_cand = 0;
	a->out_contigs.clear();
	a->out_seqs.clear();
	a->out_codes.clear();
	return ABB_OK;
}

int abb_assembler_counters(const abb_assembler* a, abb_assembly_counters* out)
{
	ABB_REQUIRE(a && out, "NULL argument");
	*out = a->counters;
	return ABB_OK;
}

int abb_assembler_set_counters(abb_assembler* a, const abb_assembly_counters* in)
{
	ABB_REQUIRE(a && in, "NULL argument");
	a->counters = *in;
	a->reads_seen = in->reads_processed;
	return ABB_OK;
}

int abb_assembler_set_comm(abb_assembler* a, abb_comm* comm)
{
	ABB_REQUIRE(a, "NULL assembler");
	a->comm = comm && abb_comm_world(comm) > 1 ? comm : nullptr;
	return ABB_OK;
}

int abb_assembler_trace(const abb_assembler* a, const abb_trace_row** rows, uint64_t* n)
{
	ABB_REQUIRE(a && rows && n, "NULL argument");
	*rows = a->out_trace.data();
	*n = a->out_trace.size();
	return ABB_OK;
}

int abb_assembler_read_results(const abb_assembler* a, const uint8_t** codes, uint64_t* n)
{
	ABB_REQUIRE(a && codes && n, "NULL argument");
	*codes = a->out_codes.data();
	*n = a->out_codes.size();
	return ABB_OK;
}

abb_filter* abb_assembler_assembled_filter(abb_assembler* a) { return a ? a->assembled : nullptr; }

} // extern "C"
