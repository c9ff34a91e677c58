// abb_shard.cuh -- the ordered insert with the counter array sharded by position range over several GPUs.
//
// North star: "the Bloom bit array shards by hash-range across GPUs ... NCCL ... over NVLink to union per-GPU
// filters before extension" (BASELINE.json); SURVEY.md 8(e).  Rank r owns counters [r*chunk, (r+1)*chunk).  The
// result must be the sequential file-order insert (see abb_insert.cuh), so the ranks do NOT insert independent
// subsets: every rank walks the same global file-order windows and evaluates every slot, but touches only the
// positions it owns:
//   gather   for each lane (carried slot or new slot of the window): minimum of the OWN counters among its H
//            positions ("partial min", 255 if it owns none) and a veto flag (a conflict-map entry of an own
//            position was touched again / an own tag belongs to an older carried slot);
//   exchange ONE ncclAllReduce(min, uint8) per window over [partial mins | not-vetoed flags]: afterwards every
//            rank knows the true minimum of every slot and whether any rank vetoed it;
//   apply    a slot nobody vetoed has no pending neighbour on any rank: each rank bumps its own counters that
//            equal the minimum (CountingBloomFilter.hpp:138-162, split over the owners).  Vetoed slots are
//            carried, identically on every rank (the carry list is rebuilt in file order from a presence bitmap so
//            that lane i means the same slot everywhere).
// Counter traffic (the HBM-bound part) is divided by the number of ranks; hashing the window and the conflict
// marks of foreign positions are not needed.  After the last window the shards are all-gathered so that every
// rank holds the whole filter for the extension stage.
#pragma once
#include "abb_insert.cuh"

namespace abb {

struct Shard {
	uint64_t lo, hi; // own positions [lo, hi)
	ABB_D bool own(uint64_t p) const { return p >= lo && p < hi; }
};

/** control block of the sharded pipeline (device) */
struct ShardCtl {
	unsigned n_pending;          // slots vetoed in this window/iteration
	unsigned n_out;              // length of the carry list k_sh_compact wrote
	unsigned long long lo_pending; // smallest pending slot (bitmap enumeration starts there)
};

template <bool LITERAL, int MAXH>
__global__ void __launch_bounds__(256)
k_sh_mark_carry(const uint64_t* __restrict__ hashes, const uint64_t* __restrict__ carry, unsigned n_lanes, uint64_t w0, HashCfg cfg,
                TagTable tab, unsigned age_off, ConflictMap map, Shard sh)
{
	const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_lanes)
		return;
	const uint64_t s = carry[i];
	uint64_t pos[MAXH];
	slot_positions<LITERAL, MAXH>(hashes, s, cfg, pos);
	const uint64_t prio = s + age_off - w0;
#pragma unroll
	for (int j = 0; j < MAXH; ++j)
		if (j < (int)cfg.H && sh.own(pos[j])) {
			tag_reserve(tab, pos[j], prio);
			map_mark_carried(map, pos[j]);
		}
}

/** lanes [0, n_lanes) = the oldest carried slots, lane n_lanes + t = slot w0 + t.  pm[lane] = min of the own
 *  counters, ok[lane] = 0 if this rank vetoes the slot.  Also marks the own positions of slot w1 + t (next window). */
template <bool LITERAL, int MAXH>
__global__ void __launch_bounds__(256)
k_sh_gather(const uint64_t* __restrict__ hashes, const uint8_t* __restrict__ valid, uint64_t w0, unsigned n, uint64_t w1,
            unsigned n_next, HashCfg cfg, ConflictMap cur, ConflictMap next, TagTable tab,
            const uint8_t* __restrict__ counters, unsigned age_off, const uint64_t* __restrict__ carry_in, unsigned n_lanes, Shard sh,
            uint8_t* __restrict__ pm, uint8_t* __restrict__ ok)
{
	const unsigned id = blockIdx.x * blockDim.x + threadIdx.x;
	uint64_t pos[MAXH];
	if (id < n_lanes) {
		const uint64_t s = carry_in[id];
		const uint64_t prio = s + age_off - w0;
		slot_positions<LITERAL, MAXH>(hashes, s, cfg, pos);
		unsigned m = 255, good = 1;
#pragma unroll
		for (int i = 0; i < MAXH; ++i)
			if (i < (int)cfg.H && sh.own(pos[i])) {
				m = min(m, (unsigned)__ldcg(counters + pos[i]));
				good &= tag_owner(tab, pos[i]) == prio;
			}
		pm[id] = (uint8_t)m;
		ok[id] = (uint8_t)good;
		return;
	}
	const unsigned t = id - n_lanes;
	if (t < n) {
		const uint64_t s = w0 + t;
		unsigned m = 255, good = 1;
		if (!valid || valid[s]) {
			slot_positions<LITERAL, MAXH>(hashes, s, cfg, pos);
#pragma unroll
			for (int i = 0; i < MAXH; ++i)
				if (i < (int)cfg.H && sh.own(pos[i])) {
					m = min(m, (unsigned)__ldcg(counters + pos[i]));
					good &= !(map_get(cur, pos[i]) & 2u);
				}
		}
		pm[n_lanes + t] = (uint8_t)m;
		ok[n_lanes + t] = (uint8_t)good;
	}
	if (t < n_next) {
		const uint64_t s = w1 + t;
		if (!valid || valid[s]) {
			slot_positions<LITERAL, MAXH>(hashes, s, cfg, pos);
			unsigned old[MAXH];
#pragma unroll
			for (int i = 0; i < MAXH; ++i) // independent atomics first, their return values afterwards
				if (i < (int)cfg.H && sh.own(pos[i])) {
					const uint64_t e = pos[i] & next.mask;
					old[i] = atomicOr(&next.w[e >> 4], 1u << ((unsigned)(e & 15) * 2));
				}
#pragma unroll
			for (int i = 0; i < MAXH; ++i)
				if (i < (int)cfg.H && sh.own(pos[i])) {
					const uint64_t e = pos[i] & next.mask;
					const unsigned shf = (unsigned)(e & 15) * 2;
					if (((old[i] >> shf) & 3u) == 1u)
						atomicOr(&next.w[e >> 4], 2u << shf);
				}
		}
	}
}

/** after the all-reduce: pm = true minimum, ok = 0 if any rank vetoed.  Carried slots beyond n_lanes did not
 *  take part and stay pending.  Pending slots are recorded in the presence bitmap `bits` (bit = slot - lo_slot). */
template <bool LITERAL, int MAXH>
__global__ void __launch_bounds__(256)
k_sh_apply(const uint64_t* __restrict__ hashes, const uint8_t* __restrict__ valid, uint64_t w0, unsigned n, HashCfg cfg, TagTable tab,
           uint8_t* __restrict__ counters, const uint64_t* __restrict__ carry_in, unsigned n_in, unsigned n_lanes,
           Shard sh, const uint8_t* __restrict__ pm, const uint8_t* __restrict__ ok, unsigned* __restrict__ bits, uint64_t lo_slot,
           ShardCtl* __restrict__ ctl, unsigned long long* __restrict__ stats)
{
	const unsigned id = blockIdx.x * blockDim.x + threadIdx.x;
	uint64_t s;
	unsigned lane;
	bool carried;
	if (id < n_in) {
		s = carry_in[id];
		lane = id;
		carried = true;
	} else {
		const unsigned t = id - n_in;
		if (t >= n)
			return;
		s = w0 + t;
		if (valid && !valid[s])
			return;
		lane = n_lanes + t;
		carried = false;
	}
	const bool took_part = !carried || id < n_lanes;
	if (!took_part || !ok[lane]) {
		const uint64_t b = s - lo_slot;
		atomicOr(&bits[b >> 5], 1u << (b & 31));
		atomicAdd(&ctl->n_pending, 1u);
		atomicMin(&ctl->lo_pending, (unsigned long long)s);
		if (!carried)
			atomicAdd(&stats[kStatDeferred], 1ULL);
		return;
	}
	uint64_t pos[MAXH];
	slot_positions<LITERAL, MAXH>(hashes, s, cfg, pos);
	const unsigned mn = pm[lane];
#pragma unroll
	for (int i = 0; i < MAXH; ++i)
		if (i < (int)cfg.H && sh.own(pos[i])) {
			if (mn != 255 && __ldcg(counters + pos[i]) == mn)
				__stcg(counters + pos[i], (uint8_t)(mn + 1));
			if (carried)
				tag_release(tab, pos[i]);
		}
}

/** one CTA: the pending slots in file order (same list on every rank) -> carry_out; clears the bitmap and ctl */
__global__ void __launch_bounds__(kDrainThreads)
k_sh_compact(unsigned* __restrict__ bits, uint64_t lo_slot, uint64_t hi_slot, uint64_t* __restrict__ carry_out, ShardCtl* __restrict__ ctl,
             unsigned* __restrict__ n_out)
{
	__shared__ unsigned s_warp[32];
	__shared__ unsigned s_total;
	const unsigned n = ctl->n_pending;
	const unsigned long long lo = ctl->lo_pending;
	__syncthreads();
	if (n == 0) {
		if (threadIdx.x == 0)
			*n_out = 0;
		return;
	}
	const uint64_t base = (lo - lo_slot) & ~31ULL;
	const unsigned words = (unsigned)(((hi_slot - 1 - lo_slot) - base) / 32 + 1);
	const unsigned got = enumerate_presence(bits + base / 32, words, lo_slot + base, carry_out, s_warp, &s_total);
	if (threadIdx.x == 0) {
		*n_out = got;
		ctl->n_pending = 0;
		ctl->lo_pending = ~0ULL;
	}
}

} // namespace abb
