// abb_api.cu -- C ABI (include/abyss_b200.h): filter lifecycle, pass-1 insert, literal-hash
// interface, raw array transfer, statistics.  Host orchestration only; the arithmetic lives in
// abb_device.cuh and the kernels in abb_insert.cuh.
#include "abb_common.h"
#include "abb_insert.cuh"
#include "abb_shard.cuh"
#include <dlfcn.h>
#include <nccl.h>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

namespace abb {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof g_err, fmt, ap);
	va_end(ap);
}

constexpr uint64_t kChunkSlots = 1ULL << 27; // h0 staging: 128 Mi slots = 1 GiB + 128 MiB flags (one persistent launch + one forced drain per chunk)

static uint64_t next_pow2(uint64_t x)
{
	uint64_t p = 1;
	while (p < x)
		p <<= 1;
	return p;
}

int select_device(int device)
{
	int n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if (e != cudaSuccess || n <= 0) {
		set_error("no usable CUDA device (%s); libabyssb200 has no CPU fallback",
		          e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
		return ABB_ENODEV;
	}
	if (device < 0 || device >= n) {
		set_error("device %d out of range (0..%d)", device, n - 1);
		return ABB_EINVAL;
	}
	ABB_CUDA(cudaSetDevice(device));
	return ABB_OK;
}

static FilterView view_of(const abb_filter* f)
{
	FilterView v;
	v.data = f->d_data.p;
	v.level_stride = f->level_stride();
	v.levels = f->levels;
	return v;
}

/** conflict-map size: 2^25 two-bit entries (8 MiB per map; the three rotating maps are pinned in L2 while the insert
 *  runs, set_l2_policy), split into the two halves of 2^24 entries of a two-index map (ConflictMap2, abb_insert.cuh).
 *  Exact (no aliases) for filters of up to 2^24 positions. */
constexpr unsigned kMapLog2 = 25;
static_assert(kMapLog2 - 1 <= kMapHalfLog2Max, "half B of a conflict map cannot index more than 2^24 entries");
/** ordered-insert window (slots) when none was set.  A filter with more positions than a map half has entries aliases in
 *  the maps; there the two-index maps carry 1.7 % of the slots at 2^18 slots per window (bench job; one map of 2^25
 *  entries carried 6.4 % at 2^17), and the larger window halves the fixed cost per slot of the windows (two grid
 *  barriers, a map clear and the carried slots' reservations each).  2^19 carried 6.4 % again and measured slower (DESIGN
 *  §3 K2).  A filter the maps cover exactly has no false carries, only true ones, which grow with the window: it keeps
 *  2^17. */
constexpr uint64_t kDefaultWindow = 1ULL << 18;
constexpr uint64_t kExactMapWindow = 1ULL << 17;
static uint64_t default_window(uint64_t filter_size)
{
	return filter_size > (1ULL << (kMapLog2 - 1)) ? kDefaultWindow : kExactMapWindow;
}
/** the sharded insert's maps (one index): each rank marks window * H / world positions */
constexpr unsigned kShardMapLog2 = 27;

/** entries per conflict map of `halves` equal parts: 2^lg in all, or fewer when the filter has fewer positions (each part
 *  then still has an entry per position) */
static uint64_t map_entries_for(uint64_t filter_size, unsigned lg, unsigned halves)
{
	const uint64_t fit = std::max<uint64_t>(next_pow2(filter_size), 1024);
	return halves * std::min<uint64_t>((1ULL << lg) / halves, fit);
}

static unsigned age_windows_for(uint64_t window)
{
	return (unsigned)std::min<uint64_t>(kMaxAgeWindows, ((1ULL << kPrioBits) - 2) / window - 1);
}

/** make sure the ordered-insert workspace exists for `window` slots per window, conflict maps of 2^lg entries (at
 *  most) in `halves` parts and the current hash count */
static int ensure_workspace(abb_filter* f, uint64_t window, unsigned lg, unsigned halves)
{
	const uint64_t want_entries = map_entries_for(f->size, lg, halves);
	if (f->d_carry.p && f->ws_window == window && f->ws_H == f->H && f->map_entries == want_entries)
		return ABB_OK;
	// the old workspace is freed before the new one is allocated (peak memory), and it counts as valid again only once
	// every piece has been allocated
	f->ws_window = 0;
	f->d_map[0] = f->d_map[1] = f->d_map[2] = nullptr;
	f->maps.reset();
	f->d_tags2[0].reset();
	f->d_tags2[1].reset();
	f->d_carry.reset();
	f->d_slotbits.reset();
	const size_t map_words = std::max<size_t>(want_entries / 4, 256) / sizeof(unsigned);
	// at most kCarryLanes carried slots reserve H positions each; load factor <= 1/8.  Only a prefix sized to the
	// carried slots of a window is in use (tag_mask_for)
	f->tag_slots = next_pow2(8ULL * kCarryLanes * f->H);
	ABB_CHECK(f->maps.alloc(3 * map_words));
	ABB_CUDA(cudaMemsetAsync(f->maps.p, 0, 3 * map_words * sizeof(unsigned), f->stream));
	for (auto& tags : f->d_tags2) {
		ABB_CHECK(tags.alloc(f->tag_slots));
		ABB_CUDA(cudaMemsetAsync(tags.p, 0, f->tag_slots * sizeof(unsigned long long), f->stream));
	}
	// worst case everything defers: window slots + the carried lanes, twice, plus the drain's sorted copy
	ABB_CHECK(f->d_carry.alloc(3 * (window + kCarryLanes)));
	// presence bitmap of the drain: pending slots span at most age_off + 2 windows
	f->slotbit_words = ((uint64_t)age_windows_for(window) + 3) * window / 32 + 64;
	ABB_CHECK(f->d_slotbits.alloc(f->slotbit_words));
	ABB_CUDA(cudaMemsetAsync(f->d_slotbits.p, 0, f->slotbit_words * sizeof(unsigned), f->stream));
	for (int i = 0; i < 3; ++i)
		f->d_map[i] = f->maps.p + i * map_words;
	f->map_entries = want_entries;
	f->ws_window = window;
	f->ws_H = f->H;
	return ABB_OK;
}

#define ABB_DISPATCH_H(H, ...)            \
	do {                                  \
		if ((H) <= 4) {                   \
			constexpr int MAXH = 4;       \
			__VA_ARGS__;                  \
		} else if ((H) <= 8) {            \
			constexpr int MAXH = 8;       \
			__VA_ARGS__;                  \
		} else {                          \
			constexpr int MAXH = 32;      \
			__VA_ARGS__;                  \
		}                                 \
	} while (0)

/** While the insert runs, the two conflict maps are pinned in L2 (persisting access-policy window on the filter's stream)
 *  and everything else -- the random counter sectors, the hashes -- is treated as streaming, so that 30-60 MB of counter
 *  lines per window cannot push the maps out (ncu, round 2: without this 57 % of the map atomics missed L2 and the kernel
 *  moved 3x the algorithmic DRAM bytes). */
static void set_l2_policy(abb_filter* f, bool on, int n_maps = 3)
{
	cudaStreamAttrValue attr;
	memset(&attr, 0, sizeof attr);
	if (on) {
		int max_persist = 0, max_window = 0;
		cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, f->device);
		cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, f->device);
		const size_t bytes = (size_t)n_maps * std::max<size_t>(f->map_entries / 4, 256);
		if (max_persist <= 0 || max_window <= 0)
			return;
		cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, std::min<size_t>(bytes, (size_t)max_persist));
		attr.accessPolicyWindow.base_ptr = f->d_map[0];
		attr.accessPolicyWindow.num_bytes = std::min<size_t>(bytes, (size_t)max_window);
		attr.accessPolicyWindow.hitRatio = std::min(1.0f, (float)max_persist / (float)bytes);
		attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
		attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
	} else {
		attr.accessPolicyWindow.num_bytes = 0; // no window
		attr.accessPolicyWindow.hitProp = cudaAccessPropertyNormal;
		attr.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
	}
	cudaStreamSetAttribute(f->stream, cudaStreamAttributeAccessPolicyWindow, &attr);
	if (!on) { // hand the carve-out back to pass 2
		cudaCtxResetPersistingL2Cache();
		cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, 0);
	}
	cudaGetLastError(); // best effort: a device without the feature runs without the hint
}

/** Scope that holds the L2 policy.  Changing the persisting carve-out (cudaDeviceSetLimit, cudaCtxResetPersistingL2Cache)
 *  synchronises the whole device -- including a host-to-device copy running on another stream -- so a caller that overlaps
 *  a copy with the insert takes the hold once, before the copy starts; the per-chunk scopes inside then do nothing. */
struct PolicyHold {
	abb_filter* f;
	bool took;
	PolicyHold(abb_filter* f_, int n_maps) : f(f_), took(!f_->l2_policy_held && f_->d_map[0] != nullptr)
	{
		if (took) {
			set_l2_policy(f, true, n_maps);
			f->l2_policy_held = true;
		}
	}
	~PolicyHold()
	{
		if (took) {
			set_l2_policy(f, false);
			f->l2_policy_held = false;
		}
	}
	PolicyHold(const PolicyHold&) = delete;
	PolicyHold& operator=(const PolicyHold&) = delete;
};

/** cooperative launch of the persistent window kernel with as many CTAs as fit on the device */
template <int KIND, bool LITERAL, int MAXH>
static int launch_windows(const InsertArgs& args, int device, cudaStream_t st)
{
	static int grid_cache[64] = { 0 };
	int& grid = grid_cache[device & 63];
	if (grid == 0) {
		int per_sm = 0, sms = 0;
		ABB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_insert_windows<KIND, LITERAL, MAXH>, 256, 0));
		ABB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
		grid = std::max(1, per_sm) * sms;
	}
	void* params[] = { (void*)&args };
	ABB_CUDA(cudaLaunchCooperativeKernel((void*)k_insert_windows<KIND, LITERAL, MAXH>, dim3((unsigned)grid), dim3(256), params, 0, st));
	return ABB_OK;
}

/** fold the timed insert launches (event pairs in f->prof_ev) of one call into the statistics */
static int fold_profile(abb_filter* f)
{
	if (!f->profile || !f->prof_used)
		return ABB_OK;
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	for (size_t i = 0; i + 1 < f->prof_used; i += 2) {
		float ms = 0;
		cudaEventElapsedTime(&ms, f->prof_ev[i], f->prof_ev[i + 1]);
		f->st.ms_commit += ms;
		f->st.commit_launches += 1;
	}
	f->st.commit_slots += f->prof_slots;
	f->prof_used = 0;
	f->prof_slots = 0;
	return ABB_OK;
}

/** ordered insert of slots [0, n_slots) of `hashes` (h0 per slot, or literal H per slot); see abb_insert.cuh */
template <bool LITERAL>
static int ordered_insert(abb_filter* f, const uint64_t* d_hashes, const uint8_t* d_valid, uint64_t n_slots)
{
	if (n_slots == 0)
		return ABB_OK;
	if (f->kind == ABB_BIT) {
		ABB_DISPATCH_H(f->H, (k_bits_insert<LITERAL, MAXH><<<blocks_for(n_slots, 256), 256, 0, f->stream>>>(
		                         d_hashes, d_valid, n_slots, f->cfg, f->d_data.p)));
		f->st.launches += 1;
		ABB_CUDA(cudaGetLastError());
		return ABB_OK;
	}
	ABB_CHECK(ensure_workspace(f, f->window, kMapLog2, 2));
	cudaStream_t st = f->stream;
	const uint64_t W = f->window;
	const uint64_t n_windows = (n_slots + W - 1) / W;
	ABB_REQUIRE(n_windows < (1ULL << 31), "too many windows in one call");
	const uint64_t cap = W + kCarryLanes;
	InsertArgs a;
	a.hashes = d_hashes;
	a.valid = d_valid;
	a.n_slots = n_slots;
	a.window = (unsigned)W;
	a.w_begin = 0;
	a.n_windows = (unsigned)n_windows;
	a.cfg = f->cfg;
	for (int i = 0; i < 3; ++i)
		a.map[i].a = { f->d_map[i], f->map_entries / 2 - 1 }; // half B follows half A
	for (int i = 0; i < 2; ++i) {
		a.tags[i] = f->d_tags2[i].p;
		a.carry[i] = f->d_carry.p + (uint64_t)i * cap;
	}
	a.tag_cap = (unsigned)f->tag_slots;
	a.f = view_of(f);
	a.age_off = (unsigned)(age_windows_for(W) * W);
	a.drain_age = a.age_off / 3 * 2;
	a.ctl = f->d_ctl.p;
	a.stats = f->d_stats.p;
	uint64_t* sorted = f->d_carry.p + 2 * cap;
	// the maps, both tag tables and the control block start clean
	ABB_CUDA(cudaMemsetAsync(f->d_ctl.p, 0, sizeof(InsertCtl), st));
	ABB_CUDA(cudaMemsetAsync(f->d_map[0], 0, 3 * std::max<size_t>(f->map_entries / 4, 256), st));
	for (int i = 0; i < 2; ++i)
		ABB_CUDA(cudaMemsetAsync(f->d_tags2[i].p, 0, f->tag_slots * sizeof(unsigned long long), st));
	const bool counting = f->kind == ABB_COUNTING;
	PolicyHold policy(f, 3);
	while (a.w_begin < a.n_windows) {
		const bool timed = f->profile && f->prof_used + 2 <= f->prof_ev.size();
		if (timed)
			cudaEventRecord(f->prof_ev[f->prof_used++], st);
		ABB_DISPATCH_H(f->H, {
			if (counting)
				ABB_CHECK((launch_windows<0, LITERAL, MAXH>(a, f->device, st)));
			else
				ABB_CHECK((launch_windows<1, LITERAL, MAXH>(a, f->device, st)));
		});
		if (timed)
			cudaEventRecord(f->prof_ev[f->prof_used++], st);
		InsertCtl h;
		ABB_CUDA(cudaMemcpyAsync(&h, f->d_ctl.p, sizeof h, cudaMemcpyDeviceToHost, st));
		ABB_CUDA(cudaStreamSynchronize(st));
		ABB_REQUIRE(h.resume > a.w_begin && h.resume <= a.n_windows, "insert kernel made no progress (window %u of %u)", h.resume, a.n_windows);
		if (timed)
			f->prof_slots += std::min<uint64_t>(n_slots, (uint64_t)h.resume * W) - (uint64_t)a.w_begin * W;
		// the list the last processed window wrote: drained when the kernel stopped for it, and at the end of the call
		const int which = 1 - (int)((h.resume - 1) & 1);
		const uint64_t w0 = (uint64_t)(h.resume - 1) * W;
		const uint64_t lo_slot = w0 > (uint64_t)a.age_off + W ? w0 - a.age_off - W : 0;
		ABB_DISPATCH_H(f->H, {
			if (counting)
				k_drain<0, LITERAL, MAXH><<<1, kDrainThreads, 0, st>>>(d_hashes, f->cfg, a.f, a.carry[which], a.ctl, which, 0, 1, f->d_slotbits.p, lo_slot,
				                                                      sorted, f->d_stats.p);
			else
				k_drain<1, LITERAL, MAXH><<<1, kDrainThreads, 0, st>>>(d_hashes, f->cfg, a.f, a.carry[which], a.ctl, which, 0, 1, f->d_slotbits.p, lo_slot,
				                                                      sorted, f->d_stats.p);
		});
		f->st.launches += 2;
		f->st.windows += h.resume - a.w_begin;
		a.w_begin = h.resume;
	}
	ABB_CUDA(cudaGetLastError());
	return fold_profile(f);
}

/** single thread: cut reads into chunks of about `cap` slots (at least one read per chunk) */
__global__ void k_chunk_bounds(const uint64_t* __restrict__ slot_offs, uint64_t n_reads, uint64_t cap,
                               uint64_t* __restrict__ bounds, unsigned max_chunks, unsigned* __restrict__ n_chunks)
{
	uint64_t r = 0;
	unsigned c = 0;
	bounds[0] = 0;
	while (r < n_reads && c + 1 < max_chunks) {
		const uint64_t limit = slot_offs[r] + cap;
		// largest r1 in (r, n_reads] with slot_offs[r1] <= limit, but at least r + 1
		uint64_t lo = r + 1, hi = n_reads;
		while (lo < hi) {
			uint64_t mid = lo + (hi - lo + 1) / 2;
			if (slot_offs[mid] <= limit)
				lo = mid;
			else
				hi = mid - 1;
		}
		r = lo;
		bounds[++c] = r;
	}
	if (r < n_reads)
		bounds[++c] = n_reads;
	*n_chunks = c;
}

/** count valid flags (k-mers actually inserted) */
__global__ void __launch_bounds__(256)
k_count_valid(const uint8_t* __restrict__ valid, uint64_t n, unsigned long long* __restrict__ out)
{
	unsigned long long c = 0;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
		c += valid[i];
	for (int d = 16; d; d >>= 1)
		c += __shfl_down_sync(0xffffffffu, c, d);
	if ((threadIdx.x & 31) == 0 && c)
		atomicAdd(out, c);
}

/** the unmasked K1 over reads with the ring that holds k (see kRingWide) */
template <int RING>
static int launch_hash_tma(unsigned k, const uint8_t* d_bases, const uint64_t* d_offs, const uint64_t* d_slot_offs, uint64_t n,
                           uint64_t slot_base, uint64_t* d_h0, uint8_t* d_valid, cudaStream_t stream)
{
	// The opt-in to 16 KB of dynamic shared memory (56 KB in all) is a per-device attribute of the kernel: a process that
	// drives several GPUs (abyss-bloom-dbg --devices) sets it on each of them.
	static bool smem_opt_in[64] = {};
	int dev = 0;
	ABB_CUDA(cudaGetDevice(&dev));
	if (!smem_opt_in[dev & 63]) {
		ABB_CUDA(cudaFuncSetAttribute(k_hash_reads_tma<RING>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * kTmaStage));
		smem_opt_in[dev & 63] = true;
	}
	// read blocks staged into shared memory by the bulk-copy engine (cp.async.bulk), double buffered; the copy needs a
	// 16-byte aligned source, so reads at an unaligned base pointer are all hashed from global memory
	const bool may_stage = (reinterpret_cast<uintptr_t>(d_bases) & 15) == 0;
	const unsigned grid = (unsigned)std::min<uint64_t>((n + kTmaReads - 1) / kTmaReads, (uint64_t)sm_count() * 4);
	k_hash_reads_tma<RING><<<grid, ring_warps<RING>() * 32, 2 * kTmaStage, stream>>>(d_bases, d_offs, d_slot_offs, slot_base, n, k,
	                                                                               d_h0, d_valid, may_stage);
	return ABB_OK;
}

/** K1 launcher for reads [r0, r1): h0/valid index = slot_offs[r] + j - slot_base */
int launch_hash(unsigned k, const uint8_t* d_care, const uint8_t* d_bases, const uint64_t* d_offs, const uint64_t* d_slot_offs,
                uint64_t r0, uint64_t r1, uint64_t slot_base, uint64_t* d_h0, uint8_t* d_valid, cudaStream_t stream, uint64_t* launches)
{
	const uint64_t n = r1 - r0;
	if (n == 0)
		return ABB_OK;
	const uint64_t sms = sm_count();
	if (d_care) {
		const unsigned grid = (unsigned)std::min<uint64_t>((n + kHashWarps - 1) / kHashWarps, sms * 32);
		k_hash_reads_masked<<<grid, kHashWarps * 32, 0, stream>>>(d_bases, d_offs + r0, d_slot_offs + r0, slot_base, n, k, d_care,
		                                                          d_h0, d_valid);
	} else if (k <= kRingMaxK) {
		ABB_CHECK(launch_hash_tma<kRing>(k, d_bases, d_offs + r0, d_slot_offs + r0, n, slot_base, d_h0, d_valid, stream));
	} else {
		ABB_CHECK(launch_hash_tma<kRingWide>(k, d_bases, d_offs + r0, d_slot_offs + r0, n, slot_base, d_h0, d_valid, stream));
	}
	if (launches)
		*launches += 1;
	ABB_CUDA(cudaGetLastError());
	return ABB_OK;
}

/** K1 over explicit (possibly overlapping) segments, see k_hash_segments */
int launch_hash_segments(unsigned k, const uint8_t* d_care, const uint8_t* d_bases, const uint64_t* d_seg_beg,
                         const unsigned* d_seg_len, const uint64_t* d_seg_slot, uint64_t n_segs, uint64_t* d_h0, uint8_t* d_valid,
                         cudaStream_t stream)
{
	if (n_segs == 0)
		return ABB_OK;
	const unsigned grid = (unsigned)std::min<uint64_t>((n_segs + kHashWarps - 1) / kHashWarps, (uint64_t)sm_count() * 32);
	if (d_care)
		k_hash_segments_masked<<<grid, kHashWarps * 32, 0, stream>>>(d_bases, d_seg_beg, d_seg_len, d_seg_slot, n_segs, k, d_care,
		                                                             d_h0, d_valid);
	else if (k <= kRingMaxK)
		k_hash_segments<kRing><<<grid, kHashWarps * 32, 0, stream>>>(d_bases, d_seg_beg, d_seg_len, d_seg_slot, n_segs, k, d_h0, d_valid);
	else // half the warps per CTA: twice the CTAs for the same segments per launch
		k_hash_segments<kRingWide><<<2 * grid, ring_warps<kRingWide>() * 32, 0, stream>>>(d_bases, d_seg_beg, d_seg_len, d_seg_slot,
		                                                                                   n_segs, k, d_h0, d_valid);
	ABB_CUDA(cudaGetLastError());
	return ABB_OK;
}

/** slot_offs[0..n_reads] = exclusive prefix sum of per-read window counts; returns the total */
int compute_slot_offsets(unsigned k, const uint64_t* d_offs, uint64_t n_reads, DevBuf<uint64_t>& slot_offs,
                                DevBuf<uint8_t>& tmp, cudaStream_t stream, uint64_t* total, uint64_t* launches)
{
	ABB_CHECK(slot_offs.reserve(n_reads + 1));
	ABB_CUDA(cudaMemsetAsync(slot_offs.p + n_reads, 0, sizeof(uint64_t), stream));
	if (n_reads) {
		k_window_counts<<<blocks_for(n_reads, 256), 256, 0, stream>>>(d_offs, n_reads, k, slot_offs.p);
		ABB_CUDA(cudaGetLastError());
	}
	size_t bytes = 0;
	ABB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, slot_offs.p, slot_offs.p, n_reads + 1, stream));
	ABB_CHECK(tmp.reserve(bytes));
	ABB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, slot_offs.p, slot_offs.p, n_reads + 1, stream));
	ABB_CUDA(cudaMemcpyAsync(total, slot_offs.p + n_reads, sizeof(uint64_t), cudaMemcpyDeviceToHost, stream));
	ABB_CUDA(cudaStreamSynchronize(stream));
	if (launches)
		*launches += 3;
	return ABB_OK;
}

int check_read_batch(const char* bases, const uint64_t* offsets, uint64_t n_reads, const char* noun)
{
	if (n_reads == 0)
		return ABB_OK;
	ABB_REQUIRE(bases && offsets, "NULL %s buffers", noun);
	ABB_REQUIRE(offsets[0] == 0, "offsets[0] must be 0");
	return ABB_OK;
}

int stage_read_batch(const char* bases, const uint64_t* offsets, uint64_t n_reads, DevBuf<uint8_t>& d_bases, DevBuf<uint64_t>& d_offs,
                     cudaStream_t stream)
{
	if (n_reads == 0)
		return ABB_OK;
	const uint64_t n_bases = offsets[n_reads];
	ABB_CHECK(d_bases.reserve(n_bases + 16));
	ABB_CHECK(d_offs.reserve(n_reads + 1));
	ABB_CUDA(cudaMemcpyAsync(d_offs.p, offsets, (n_reads + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, stream));
	if (bases)
		ABB_CUDA(cudaMemcpyAsync(d_bases.p, bases, n_bases, cudaMemcpyHostToDevice, stream));
	return ABB_OK;
}

int resolve_level(const abb_filter* f, int level, unsigned* out)
{
	if (level < 0)
		level = (int)f->levels - 1;
	ABB_REQUIRE((unsigned)level < f->levels, "level %d out of range", level);
	*out = (unsigned)level;
	return ABB_OK;
}

static int sharded_ordered_insert(abb_filter* f, abb_comm* c, const uint64_t* d_h0, const uint8_t* d_valid, uint64_t n_slots);

/** a host-to-device copy of the bases that is still in flight, in pieces of `piece` bytes on f->copy_stream
 *  (f->copy_ev[i] fires when bytes [i * piece, (i + 1) * piece) have landed); h_offs are the caller's offsets */
struct PendingCopy {
	const uint64_t* h_offs = nullptr;
	uint64_t piece = 0;
	size_t n_pieces = 0;
	size_t waited = 0; // pieces the filter's stream already waits for
};

/** make the filter's stream wait until bases [0, end) are on the device */
static int wait_bases(abb_filter* f, PendingCopy* pc, uint64_t end)
{
	if (!pc || end == 0)
		return ABB_OK;
	const size_t need = std::min<size_t>(pc->n_pieces, (size_t)((end + pc->piece - 1) / pc->piece));
	if (need > pc->waited) {
		ABB_CUDA(cudaStreamWaitEvent(f->stream, f->copy_ev[need - 1], 0)); // pieces complete in order
		pc->waited = need;
	}
	return ABB_OK;
}

static int insert_reads_dev(abb_filter* f, const uint8_t* d_bases, const uint64_t* d_offs, uint64_t n_reads,
                            uint64_t* n_kmers_out, abb_comm* comm = nullptr, PendingCopy* pc = nullptr)
{
	uint64_t total = 0;
	ABB_CHECK(compute_slot_offsets(f->k, d_offs, n_reads, f->slot_offs, f->scan_tmp, f->stream, &total, &f->st.launches));
	if (n_kmers_out)
		*n_kmers_out = 0;
	if (total == 0)
		return ABB_OK;

	// chunk the reads so that the h0 staging buffer stays bounded
	std::vector<uint64_t> bounds;
	if (total <= kChunkSlots) {
		bounds = { 0, n_reads };
	} else {
		const unsigned max_chunks = (unsigned)(total / kChunkSlots + 3) * 2;
		// a member buffer: an allocation and free per call would synchronise the device, i.e. wait for the host-to-device copy
		// that abb_insert_reads runs next to this insert
		DevBuf<uint64_t>& d_bounds = f->bounds;
		ABB_CHECK(d_bounds.reserve(max_chunks + 2));
		k_chunk_bounds<<<1, 1, 0, f->stream>>>(f->slot_offs.p, n_reads, kChunkSlots, d_bounds.p, max_chunks,
		                                      (unsigned*)(d_bounds.p + max_chunks + 1));
		f->st.launches += 1;
		std::vector<uint64_t> h(max_chunks + 2);
		ABB_CUDA(cudaMemcpyAsync(h.data(), d_bounds.p, (max_chunks + 2) * sizeof(uint64_t), cudaMemcpyDeviceToHost, f->stream));
		ABB_CUDA(cudaStreamSynchronize(f->stream));
		unsigned nc = (unsigned)(h[max_chunks + 1] & 0xffffffffu);
		bounds.assign(h.begin(), h.begin() + nc + 1);
	}
	// per-chunk slot ranges need slot_offs at the chunk boundaries
	std::vector<uint64_t> slot_at(bounds.size());
	for (size_t i = 0; i < bounds.size(); ++i)
		ABB_CUDA(cudaMemcpyAsync(&slot_at[i], f->slot_offs.p + bounds[i], sizeof(uint64_t), cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));

	ABB_CUDA(cudaMemsetAsync(f->d_stats.p + kStatInsertKmers, 0, sizeof(unsigned long long), f->stream));
	for (size_t c = 0; c + 1 < bounds.size(); ++c) {
		const uint64_t r0 = bounds[c], r1 = bounds[c + 1];
		const uint64_t slots = slot_at[c + 1] - slot_at[c];
		if (slots == 0)
			continue;
		ABB_CHECK(f->h0.reserve(slots));
		ABB_CHECK(f->valid.reserve(slots));
		if (pc)
			ABB_CHECK(wait_bases(f, pc, pc->h_offs[r1]));
		ABB_CUDA(cudaEventRecord(f->ev0, f->stream));
		ABB_CHECK(launch_hash(f->k, f->d_care.p, d_bases, d_offs, f->slot_offs.p, r0, r1, slot_at[c], f->h0.p, f->valid.p, f->stream,
		                      &f->st.launches));
		k_count_valid<<<std::min<unsigned>(blocks_for(slots, 256), sm_count() * 8), 256, 0, f->stream>>>(f->valid.p, slots,
		                                                                                                  f->d_stats.p + kStatInsertKmers);
		f->st.launches += 1;
		ABB_CUDA(cudaEventRecord(f->ev1, f->stream));
		if (comm)
			ABB_CHECK(sharded_ordered_insert(f, comm, f->h0.p, f->valid.p, slots));
		else
			ABB_CHECK(ordered_insert<false>(f, f->h0.p, f->valid.p, slots));
		cudaEvent_t ev2 = f->ev0; // reuse: record end of insert after reading the hash time
		ABB_CUDA(cudaEventSynchronize(f->ev1));
		float ms = 0;
		ABB_CUDA(cudaEventElapsedTime(&ms, f->ev0, f->ev1));
		f->st.ms_hash += ms;
		ABB_CUDA(cudaEventRecord(ev2, f->stream));
		ABB_CUDA(cudaEventSynchronize(ev2));
		ABB_CUDA(cudaEventElapsedTime(&ms, f->ev1, ev2));
		f->st.ms_insert += ms;
		f->st.slots += slots;
	}
	unsigned long long nk = 0;
	ABB_CUDA(cudaMemcpyAsync(&nk, f->d_stats.p + kStatInsertKmers, sizeof nk, cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	f->st.kmers += nk;
	if (n_kmers_out)
		*n_kmers_out = nk;
	return ABB_OK;
}

// =============================================================================================
// multi-GPU: NCCL behind the C ABI (dlopen, no link-time dependency) and the sharded ordered insert
// =============================================================================================
struct NcclApi {
	void* h = nullptr;
	ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
	ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
	ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
	ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*GroupStart)() = nullptr;
	ncclResult_t (*GroupEnd)() = nullptr;
	const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi g_nccl;

static int load_nccl()
{
	if (g_nccl.h)
		return ABB_OK;
	const char* names[] = { getenv("ABB_NCCL_LIB"), "libnccl.so.2", "libnccl.so" };
	void* h = nullptr;
	for (const char* n : names)
		if (n && *n && (h = dlopen(n, RTLD_NOW | RTLD_GLOBAL)))
			break;
	if (!h) {
		set_error("cannot load NCCL (libnccl.so.2): %s", dlerror());
		return ABB_ENODEV;
	}
#define ABB_NCCL_SYM(field, name)                                        \
	do {                                                                 \
		*(void**)(&g_nccl.field) = dlsym(h, name);                       \
		if (!g_nccl.field) {                                             \
			set_error("NCCL library lacks %s", name);                    \
			return ABB_ENODEV;                                           \
		}                                                                \
	} while (0)
	ABB_NCCL_SYM(GetUniqueId, "ncclGetUniqueId");
	ABB_NCCL_SYM(CommInitRank, "ncclCommInitRank");
	ABB_NCCL_SYM(CommDestroy, "ncclCommDestroy");
	ABB_NCCL_SYM(AllReduce, "ncclAllReduce");
	ABB_NCCL_SYM(AllGather, "ncclAllGather");
	ABB_NCCL_SYM(Send, "ncclSend");
	ABB_NCCL_SYM(Recv, "ncclRecv");
	ABB_NCCL_SYM(GroupStart, "ncclGroupStart");
	ABB_NCCL_SYM(GroupEnd, "ncclGroupEnd");
	ABB_NCCL_SYM(GetErrorString, "ncclGetErrorString");
#undef ABB_NCCL_SYM
	g_nccl.h = h;
	return ABB_OK;
}

#define ABB_NCCL(call)                                                                                   \
	do {                                                                                                 \
		ncclResult_t r__ = (call);                                                                       \
		if (r__ != ncclSuccess) {                                                                        \
			abb::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #call, g_nccl.GetErrorString(r__)); \
			return ABB_ECUDA;                                                                            \
		}                                                                                                \
	} while (0)

} // namespace abb

struct abb_comm {
	ncclComm_t comm = nullptr;
	int rank = 0, world = 1, device = 0;
};

namespace abb {

static uint64_t shard_chunk(uint64_t size, unsigned world) { return ((size + world - 1) / world + 15) & ~15ULL; }

/** the window of the sharded pipeline: 2^18 slots per rank by default (twice the per-rank load of its one-index conflict
 *  maps at 2^17 slots), twice the filter's window per rank when one was set */
constexpr uint64_t kShardRankWindow = 1ULL << 18;
static uint64_t sharded_window(const abb_filter* f, unsigned world)
{
	const uint64_t per_rank = f->window == default_window(f->size) ? kShardRankWindow : 2 * f->window;
	return std::min<uint64_t>(std::max<uint64_t>(per_rank * world, 32), 1ULL << 21);
}

static int sharded_ordered_insert(abb_filter* f, abb_comm* c, const uint64_t* d_h0, const uint8_t* d_valid, uint64_t n_slots)
{
	if (n_slots == 0)
		return ABB_OK;
	const uint64_t W = sharded_window(f, (unsigned)c->world);
	ABB_CHECK(ensure_workspace(f, W, kShardMapLog2, 1));
	// carried slots served per step: the tag table holds only own positions, so world times the single-GPU number fit
	const unsigned max_lanes = (unsigned)std::min<uint64_t>((uint64_t)kCarryLanes * (unsigned)c->world, W / 2 + kCarryLanes);
	ABB_CHECK(f->sh_buf.reserve(2 * (W + (uint64_t)max_lanes) + 64));
	cudaStream_t st = f->stream;
	const uint64_t n_windows = (n_slots + W - 1) / W;
	const unsigned age_off = (unsigned)(age_windows_for(W) * W);
	const unsigned drain_age = age_off / 3 * 2;
	const uint64_t cap = 3 * (W + kCarryLanes) / 2; // two lists in the allocation of three (no drain list is needed here)
	uint64_t* carry[2] = { f->d_carry.p, f->d_carry.p + cap };
	ShardCtl* ctl = f->d_shard_ctl.p;
	const size_t map_bytes = std::max<size_t>(f->map_entries / 4, 256);
	ConflictMap maps[2] = { { f->d_map[0], f->map_entries - 1 }, { f->d_map[1], f->map_entries - 1 } };
	const uint64_t chunk = shard_chunk(f->size, (unsigned)c->world);
	Shard sh;
	sh.lo = std::min<uint64_t>(f->size, (uint64_t)c->rank * chunk);
	sh.hi = std::min<uint64_t>(f->size, sh.lo + chunk);
	{
		ShardCtl init;
		init.n_pending = 0;
		init.n_out = 0;
		init.lo_pending = ~0ULL;
		ABB_CUDA(cudaMemcpyAsync(ctl, &init, sizeof init, cudaMemcpyHostToDevice, st));
	}
	ABB_CUDA(cudaMemsetAsync(f->d_map[0], 0, 3 * map_bytes, st)); // the maps start clean
	unsigned n_in = 0; // host copy of the carry length (identical on every rank)
	uint64_t oldest = 0;
	int in = 0, p = 0;
	uint8_t* buf = f->sh_buf.p;
	// one step of the pipeline: the oldest carried slots + the n new slots of [w0, w0 + n); marks [w1, w1 + n_next)
	auto step = [&](uint64_t w0, unsigned n, uint64_t w1, unsigned n_next) -> int {
		const unsigned lanes_c = std::min<unsigned>(n_in, max_lanes);
		// the tag table prefix this step uses (a rank reserves only the positions it owns: 1/world of them), cleared first
		uint64_t tslots = 4096;
		while (tslots < 8ULL * lanes_c * f->H / (unsigned)c->world + 4096 && tslots < f->tag_slots)
			tslots <<= 1;
		const TagTable tab = { f->d_tags2[0].p, std::min<uint64_t>(tslots, f->tag_slots) - 1 };
		if (lanes_c)
			ABB_CUDA(cudaMemsetAsync(tab.e, 0, (tab.mask + 1) * sizeof(unsigned long long), st));
		const unsigned lanes = lanes_c + n;
		const uint64_t lo_slot = w0 > (uint64_t)age_off + W ? w0 - age_off - W : 0;
		uint8_t* pm = buf;
		uint8_t* ok = buf + lanes;
		const bool timed = f->profile && n && (f->st.windows % f->prof_stride) == 0 && f->prof_used + 2 <= f->prof_ev.size();
		ABB_DISPATCH_H(f->H, {
			if (lanes_c)
				k_sh_mark_carry<false, MAXH><<<blocks_for(lanes_c, 256), 256, 0, st>>>(d_h0, carry[in], lanes_c, w0, f->cfg, tab, age_off, maps[p], sh);
			if (timed)
				cudaEventRecord(f->prof_ev[f->prof_used++], st);
			k_sh_gather<false, MAXH><<<blocks_for((uint64_t)lanes_c + std::max(n, n_next), 256), 256, 0, st>>>(
			    d_h0, d_valid, w0, n, w1, n_next, f->cfg, maps[p], maps[1 - p], tab, f->d_data.p, age_off, carry[in], lanes_c, sh, pm, ok);
		});
		if (lanes) {
			ABB_NCCL(g_nccl.AllReduce(buf, buf, 2 * (size_t)lanes, ncclUint8, ncclMin, c->comm, st));
			ABB_DISPATCH_H(f->H, (k_sh_apply<false, MAXH><<<blocks_for((uint64_t)n_in + n, 256), 256, 0, st>>>(
			                         d_h0, d_valid, w0, n, f->cfg, tab, f->d_data.p, carry[in], n_in, lanes_c, sh, pm, ok, f->d_slotbits.p, lo_slot, ctl,
			                         f->d_stats.p)));
			if (timed) {
				cudaEventRecord(f->prof_ev[f->prof_used++], st);
				f->prof_slots += n;
			}
			k_sh_compact<<<1, kDrainThreads, 0, st>>>(f->d_slotbits.p, lo_slot, w0 + std::max<uint64_t>(n, 1), carry[1 - in], ctl, &ctl->n_out);
			unsigned h_n = 0;
			ABB_CUDA(cudaMemcpyAsync(&h_n, &ctl->n_out, sizeof h_n, cudaMemcpyDeviceToHost, st));
			// the oldest pending slot bounds the priorities
			ABB_CUDA(cudaMemcpyAsync(&oldest, carry[1 - in], sizeof oldest, cudaMemcpyDeviceToHost, st));
			ABB_CUDA(cudaStreamSynchronize(st));
			n_in = h_n;
			in = 1 - in;
			f->st.launches += 4;
		} else {
			if (timed)
				f->prof_used--; // nothing was applied
			f->st.launches += 1;
		}
		return ABB_OK;
	};
	// everything pending is retired by steps without new slots (the oldest kCarryLanes take part in each)
	auto drain = [&](uint64_t w0, unsigned until) -> int {
		while (n_in > until) {
			ABB_CHECK(step(w0, 0, w0, 0));
			f->sh_drains += 1;
		}
		return ABB_OK;
	};
	f->prof_stride = f->prof_ev.empty() ? 1 : std::max<uint64_t>(1, (2 * n_windows + f->prof_ev.size() - 1) / f->prof_ev.size());
	PolicyHold policy(f, 2); // this path alternates between the first two maps
	ABB_CHECK(step(0, 0, 0, (unsigned)std::min<uint64_t>(W, n_slots))); // marks of window 0
	p = 1 - p; // the marks went to maps[1 - p]
	for (uint64_t w = 0; w < n_windows; ++w) {
		const uint64_t w0 = w * W;
		const unsigned n = (unsigned)std::min<uint64_t>(W, n_slots - w0);
		const uint64_t w1 = w0 + W;
		const unsigned n_next = w + 1 < n_windows ? (unsigned)std::min<uint64_t>(W, n_slots - w1) : 0u;
		if (n_in > max_lanes)
			ABB_CHECK(drain(w0, max_lanes / 2));
		if (n_in && w0 - oldest > drain_age)
			ABB_CHECK(drain(w0, 0));
		ABB_CHECK(step(w0, n, w1, n_next));
		ABB_CUDA(cudaMemsetAsync(maps[p].w, 0, map_bytes, st));
		p = 1 - p;
		f->st.windows += 1;
	}
	ABB_CHECK(drain(n_slots, 0));
	ABB_CUDA(cudaGetLastError());
	return fold_profile(f);
}

} // namespace abb

using namespace abb;

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

int abb_version(void) { return ABB_VERSION; }
const char* abb_last_error(void) { return g_err; }

/* MAX_KMER of this process: k above it is refused by every entry point that takes a k, as the reference built with
 * configure --enable-maxk=<max_kmer> refuses it (Common/Kmer.h:44-56) */
static std::atomic<unsigned> g_max_kmer{ kDefaultMaxK };

int abb_set_max_kmer(unsigned max_k)
{
	ABB_REQUIRE(max_k >= 1 && max_k <= kMaxK, "the largest k-mer size must be in 1..%u", kMaxK);
	g_max_kmer.store(max_k);
	return ABB_OK;
}

unsigned abb_max_kmer(void) { return g_max_kmer.load(); }

int abb_device_count(void)
{
	int n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if (e != cudaSuccess) {
		set_error("cudaGetDeviceCount: %s", cudaGetErrorString(e));
		return ABB_ENODEV;
	}
	return n;
}

static int alloc_filter(std::unique_ptr<abb_filter> f, abb_filter** out);

int abb_filter_create(abb_filter** out, int kind, uint64_t size, unsigned num_hashes, unsigned k, unsigned arg,
                      const char* mask, int device)
{
	ABB_REQUIRE(out != nullptr, "abb_filter_create: out is NULL");
	*out = nullptr;
	ABB_REQUIRE(kind != ABB_KONNECTOR, "Konnector filters are created with abb_konnector_create");
	ABB_REQUIRE(kind == ABB_COUNTING || kind == ABB_BIT || kind == ABB_CASCADING, "unknown filter kind %d", kind);
	ABB_REQUIRE(num_hashes >= 1 && num_hashes <= kMaxHashes, "number of hash functions must be in 1..%u (MAX_HASHES)", kMaxHashes);
	ABB_REQUIRE(k >= 1 && k <= abb_max_kmer(), "k-mer size must be in 1..%u (MAX_KMER)", abb_max_kmer());
	if (kind == ABB_COUNTING) {
		// CountingBloomFilter ctor pads the byte size to a multiple of 8 (CountingBloomFilter.hpp:40-49)
		if (size % 8)
			size += 8 - size % 8;
	} else {
		// BloomFilter::initSize exits on this (BloomFilter.hpp:374-379)
		ABB_REQUIRE(size % 8 == 0, "ERROR: Filter Size \"%llu\" is not a multiple of 8.", (unsigned long long)size);
	}
	ABB_REQUIRE(size >= 8, "filter size must be at least 8");
	ABB_REQUIRE(size < (1ULL << kPosBits), "filter size %llu exceeds the supported maximum 2^%u", (unsigned long long)size, kPosBits);
	unsigned levels = 1;
	if (kind == ABB_CASCADING) {
		ABB_REQUIRE(arg >= 1 && arg <= 255, "cascading filter needs 1..255 levels");
		levels = arg;
	}
	std::string m = mask ? mask : "";
	if (!m.empty()) {
		// MaskedKmer::setMask (BloomDBG/MaskedKmer.h:38-55): k long, only 0/1
		ABB_REQUIRE(m.size() == k, "spaced seed must be exactly k=%u characters long", k);
		for (char c : m)
			ABB_REQUIRE(c == '0' || c == '1', "spaced seed must contain only '0' and '1'");
		if (m.find('0') == std::string::npos)
			m.clear(); // all ones == no mask
	}
	ABB_CHECK(select_device(device));

	std::unique_ptr<abb_filter> f(new (std::nothrow) abb_filter());
	if (!f) {
		set_error("out of host memory");
		return ABB_ENOMEM;
	}
	f->device = device;
	f->kind = kind;
	f->size = size;
	f->bytes_per_level = kind == ABB_COUNTING ? size : size / 8;
	f->H = num_hashes;
	f->k = k;
	f->threshold = kind == ABB_COUNTING ? arg : 0;
	f->levels = levels;
	f->mask = m;
	f->window = default_window(size);
	f->cfg.H = num_hashes;
	f->cfg.k = k;
	f->cfg.mod = make_fastmod(size);
	for (unsigned i = 0; i < kMaxHashes; ++i)
		f->cfg.mult[i] = (uint64_t)i ^ ((uint64_t)k * kMultiSeed); // nthash.hpp:339
	return alloc_filter(std::move(f), out);
}

/** the device side of a filter whose geometry is set: stream, events, the zeroed levels, control words */
static int alloc_filter(std::unique_ptr<abb_filter> f, abb_filter** out)
{
	const unsigned k = f->k, levels = f->levels;
	ABB_CUDA(cudaStreamCreateWithFlags(f->stream.out(), cudaStreamNonBlocking));
	ABB_CUDA(cudaEventCreate(f->ev0.out()));
	ABB_CUDA(cudaEventCreate(f->ev1.out()));
	// slack: the in-place all-gather of position shards rounds each shard up to 16 bytes (abb_filter_allgather)
	ABB_CHECK(f->d_data.alloc(f->level_stride() * levels + 4096));
	ABB_CUDA(cudaMemsetAsync(f->d_data.p, 0, f->level_stride() * levels, f->stream));
	ABB_CHECK(f->d_ctl.alloc(1));
	ABB_CUDA(cudaMemsetAsync(f->d_ctl.p, 0, sizeof(InsertCtl), f->stream));
	ABB_CHECK(f->d_shard_ctl.alloc(1));
	ABB_CHECK(f->d_stats.alloc(kStatWords));
	ABB_CUDA(cudaMemsetAsync(f->d_stats.p, 0, kStatWords * sizeof(unsigned long long), f->stream));
	if (!f->mask.empty()) {
		std::vector<uint8_t> care(k);
		for (unsigned i = 0; i < k; ++i)
			care[i] = f->mask[i] == '1';
		ABB_CHECK(f->d_care.alloc(k));
		ABB_CUDA(cudaMemcpyAsync(f->d_care.p, care.data(), k, cudaMemcpyHostToDevice, f->stream));
	}
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	return hand_over(f, out);
}

int abb_konnector_create(abb_filter** out, uint64_t full_bits, unsigned k, unsigned levels, uint64_t hash_seed, uint64_t start_bit,
                         uint64_t end_bit, int device)
{
	ABB_REQUIRE(out != nullptr, "abb_konnector_create: out is NULL");
	*out = nullptr;
	ABB_REQUIRE(k >= 1 && k <= abb_max_kmer(), "k-mer size must be in 1..%u (MAX_KMER)", abb_max_kmer());
	ABB_REQUIRE(full_bits >= 2, "a Konnector filter needs at least 2 bits");
	ABB_REQUIRE(start_bit <= end_bit && end_bit < full_bits, "window [%llu, %llu] is not inside a filter of %llu bits",
	            (unsigned long long)start_bit, (unsigned long long)end_bit, (unsigned long long)full_bits);
	ABB_REQUIRE(levels >= 1 && levels <= 255, "a Konnector filter needs 1..255 levels");
	ABB_CHECK(select_device(device));
	std::unique_ptr<abb_filter> f(new (std::nothrow) abb_filter());
	if (!f) {
		set_error("out of host memory");
		return ABB_ENOMEM;
	}
	f->device = device;
	f->kind = ABB_KONNECTOR;
	f->size = end_bit - start_bit + 1;
	f->bytes_per_level = (f->size + 7) / 8;
	f->H = 1;
	f->k = k;
	f->levels = levels;
	f->kon_full = full_bits;
	f->kon_start = start_bit;
	f->kon_seed = hash_seed;
	return alloc_filter(std::move(f), out);
}

int abb_filter_destroy(abb_filter* f)
{
	if (!f)
		return ABB_OK;
	cudaSetDevice(f->device);
	cudaStreamSynchronize(f->stream);
	if (f->copy_stream)
		cudaStreamSynchronize(f->copy_stream);
	delete f;
	return ABB_OK;
}

unsigned abb_filter_kmer_size(const abb_filter* f) { return f ? f->k : 0; }
unsigned abb_filter_hash_num(const abb_filter* f) { return f ? f->H : 0; }
uint64_t abb_filter_size(const abb_filter* f) { return f ? f->size : 0; }
uint64_t abb_filter_size_in_bytes(const abb_filter* f) { return f ? f->bytes_per_level : 0; }
unsigned abb_filter_threshold(const abb_filter* f) { return f ? f->threshold : 0; }
unsigned abb_filter_levels(const abb_filter* f) { return f ? f->levels : 0; }

int abb_filter_set_threshold(abb_filter* f, unsigned threshold)
{
	ABB_REQUIRE(f, "NULL filter");
	if (f->kind != ABB_COUNTING) {
		set_error("threshold only applies to counting filters");
		return ABB_ESTATE;
	}
	f->threshold = threshold;
	return ABB_OK;
}

int abb_filter_set_profiling(abb_filter* f, int on)
{
	ABB_REQUIRE(f, "NULL filter");
	ABB_CUDA(cudaSetDevice(f->device));
	f->profile = on != 0;
	if (f->profile && f->prof_ev.empty()) {
		std::vector<Event> ev(2048); // kept only if every create succeeds: an empty prof_ev is retried on the next call
		for (auto& e : ev)
			ABB_CUDA(cudaEventCreate(e.out()));
		f->prof_ev = std::move(ev);
	}
	return ABB_OK;
}

int abb_filter_set_window(abb_filter* f, uint64_t window_slots)
{
	ABB_REQUIRE(f, "NULL filter");
	if (window_slots == 0)
		window_slots = default_window(f->size);
	ABB_REQUIRE(window_slots >= 32 && window_slots <= (1ULL << 20) - 64, "window must be in [32, 2^20 - 64]");
	ABB_CUDA(cudaSetDevice(f->device));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	f->window = window_slots;
	return ABB_OK;
}

int abb_insert_reads_dev(abb_filter* f, const char* d_bases, const uint64_t* d_offsets, uint64_t n_reads,
                         uint64_t n_bases, uint64_t* n_kmers_out)
{
	(void)n_bases;
	ABB_REQUIRE(f, "NULL filter");
	ABB_REQUIRE(n_reads == 0 || (d_bases && d_offsets), "NULL read buffers");
	ABB_CUDA(cudaSetDevice(f->device));
	if (f->kind == ABB_KONNECTOR)
		return kon_insert_reads_dev(f, (const uint8_t*)d_bases, d_offsets, n_reads, n_kmers_out);
	return insert_reads_dev(f, (const uint8_t*)d_bases, d_offsets, n_reads, n_kmers_out);
}

int abb_insert_reads(abb_filter* f, const char* bases, const uint64_t* offsets, uint64_t n_reads, uint64_t* n_kmers_out)
{
	ABB_REQUIRE(f, "NULL filter");
	if (n_kmers_out)
		*n_kmers_out = 0;
	if (n_reads == 0)
		return ABB_OK;
	ABB_CHECK(check_read_batch(bases, offsets, n_reads));
	const uint64_t n_bases = offsets[n_reads];
	ABB_CUDA(cudaSetDevice(f->device));
	// The bases travel in pieces on a second stream; chunk c of the insert only waits for the pieces that hold its reads, so
	// the copy of the rest hides behind the hashing and inserting of the earlier chunks (with pinned host memory; a pageable
	// buffer makes cudaMemcpyAsync synchronous and the order is simply copy, then insert).  One piece: one copy up front.
	constexpr uint64_t kPiece = 256ULL << 20;
	const bool in_pieces = f->kind != ABB_KONNECTOR && n_bases > kPiece;
	ABB_CHECK(stage_read_batch(in_pieces ? nullptr : bases, offsets, n_reads, f->bases, f->offs, f->stream));
	f->resident_reads = n_reads;
	if (f->kind == ABB_KONNECTOR)
		return kon_insert_reads_dev(f, f->bases.p, f->offs.p, n_reads, n_kmers_out);
	if (!in_pieces)
		return insert_reads_dev(f, f->bases.p, f->offs.p, n_reads, n_kmers_out);
	if (!f->copy_stream)
		ABB_CUDA(cudaStreamCreateWithFlags(f->copy_stream.out(), cudaStreamNonBlocking));
	if (f->kind != ABB_BIT)
		ABB_CHECK(ensure_workspace(f, f->window, kMapLog2, 2)); // the maps exist before the policy that pins them is set
	PolicyHold policy(f, 3); // before the copy starts: setting it later would wait for the whole copy (see PolicyHold)
	PendingCopy pc;
	pc.h_offs = offsets;
	pc.piece = kPiece;
	pc.n_pieces = (size_t)((n_bases + kPiece - 1) / kPiece);
	while (f->copy_ev.size() < pc.n_pieces) {
		Event ev;
		ABB_CUDA(cudaEventCreateWithFlags(ev.out(), cudaEventDisableTiming));
		f->copy_ev.push_back(std::move(ev));
	}
	// the destination may still be read by work queued on the filter's stream (pass 2 of a previous job)
	ABB_CUDA(cudaEventRecord(f->ev0, f->stream));
	ABB_CUDA(cudaStreamWaitEvent(f->copy_stream, f->ev0, 0));
	for (size_t i = 0; i < pc.n_pieces; ++i) {
		const uint64_t b0 = (uint64_t)i * kPiece, b1 = std::min<uint64_t>(n_bases, b0 + kPiece);
		ABB_CUDA(cudaMemcpyAsync(f->bases.p + b0, bases + b0, b1 - b0, cudaMemcpyHostToDevice, f->copy_stream));
		ABB_CUDA(cudaEventRecord(f->copy_ev[i], f->copy_stream));
	}
	const int rc = insert_reads_dev(f, f->bases.p, f->offs.p, n_reads, n_kmers_out, nullptr, &pc);
	// The last chunk waited for the last piece, so normally everything has landed; after an early return (no k-mers, an
	// error) the copy may still be running, and the caller owns the host buffer again once this call returns.
	ABB_CUDA(cudaStreamSynchronize(f->copy_stream));
	return rc;
}

/** true: the counters are sharded over the ranks; false: every rank runs the whole insert (see abb_insert_reads_sharded_dev) */
static bool shard_policy(int world)
{
	static int min_world = -1;
	if (min_world < 0) {
		const char* e = getenv("ABB_SHARD_MIN_WORLD");
		min_world = e ? std::max(2, atoi(e)) : 4;
	}
	return world > 1 && world >= min_world;
}

int abb_insert_reads_sharded(abb_filter* f, abb_comm* c, const char* bases, const uint64_t* offsets, uint64_t n_reads, int finalize,
                             uint64_t* n_kmers_out)
{
	ABB_REQUIRE(f && c, "NULL argument");
	ABB_REQUIRE_NTHASH(f);
	if (!shard_policy(c->world)) { // replicated insert: the single-GPU host path, with its copy hidden behind the insert
		ABB_REQUIRE(f->kind == ABB_COUNTING, "the sharded insert is implemented for counting filters");
		ABB_REQUIRE(f->device == c->device, "filter and communicator live on different devices");
		f->replicated_insert = true;
		(void)finalize; // nothing to all-gather: every rank holds the whole filter
		return abb_insert_reads(f, bases, offsets, n_reads, n_kmers_out);
	}
	if (n_kmers_out)
		*n_kmers_out = 0;
	ABB_CHECK(check_read_batch(bases, offsets, n_reads));
	ABB_CUDA(cudaSetDevice(f->device));
	ABB_CHECK(stage_read_batch(bases, offsets, n_reads, f->bases, f->offs, f->stream));
	f->resident_reads = n_reads;
	return abb_insert_reads_sharded_dev(f, c, (const char*)f->bases.p, f->offs.p, n_reads, finalize, n_kmers_out);
}

int abb_filter_resident_reads(abb_filter* f, const char** d_bases, const uint64_t** d_offsets, uint64_t* n_reads)
{
	ABB_REQUIRE(f && d_bases && d_offsets && n_reads, "NULL argument");
	*d_bases = (const char*)f->bases.p;
	*d_offsets = f->offs.p;
	*n_reads = f->resident_reads;
	return ABB_OK;
}

int abb_insert_hashes(abb_filter* f, const uint64_t* hashes, uint64_t n)
{
	ABB_REQUIRE(f, "NULL filter");
	ABB_REQUIRE_NTHASH(f);
	if (n == 0)
		return ABB_OK;
	ABB_REQUIRE(hashes, "NULL hashes");
	ABB_CUDA(cudaSetDevice(f->device));
	ABB_CHECK(f->lit.reserve(n * f->H));
	ABB_CUDA(cudaMemcpyAsync(f->lit.p, hashes, n * f->H * sizeof(uint64_t), cudaMemcpyHostToDevice, f->stream));
	ABB_CHECK(ordered_insert<true>(f, f->lit.p, nullptr, n));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	f->st.kmers += n;
	return ABB_OK;
}

int abb_hash_reads_dev(abb_filter* f, const char* d_bases, const uint64_t* d_offsets, uint64_t n_reads, uint64_t* d_h0,
                       uint8_t* d_valid, uint64_t capacity, uint64_t* n_slots_out)
{
	ABB_REQUIRE(f, "NULL filter");
	ABB_REQUIRE_NTHASH(f);
	if (n_slots_out)
		*n_slots_out = 0;
	if (n_reads == 0)
		return ABB_OK;
	ABB_REQUIRE(d_bases && d_offsets, "NULL read buffers");
	ABB_CUDA(cudaSetDevice(f->device));
	uint64_t total = 0;
	ABB_CHECK(compute_slot_offsets(f->k, d_offsets, n_reads, f->slot_offs, f->scan_tmp, f->stream, &total, &f->st.launches));
	if (n_slots_out)
		*n_slots_out = total;
	if (total == 0 || !d_h0 || !d_valid)
		return ABB_OK;
	ABB_REQUIRE(capacity >= total, "output buffers hold %llu slots, %llu needed", (unsigned long long)capacity, (unsigned long long)total);
	ABB_CHECK(launch_hash(f->k, f->d_care.p, (const uint8_t*)d_bases, d_offsets, f->slot_offs.p, 0, n_reads, 0, d_h0, d_valid, f->stream,
	                      &f->st.launches));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	return ABB_OK;
}

int abb_comm_unique_id(uint8_t id_out[128])
{
	ABB_REQUIRE(id_out, "NULL id buffer");
	ABB_CHECK(load_nccl());
	static_assert(sizeof(ncclUniqueId) == 128, "NCCL unique id size");
	ncclUniqueId id;
	ABB_NCCL(g_nccl.GetUniqueId(&id));
	memcpy(id_out, &id, sizeof id);
	return ABB_OK;
}

int abb_comm_create(abb_comm** out, int rank, int world, const uint8_t id[128], int device)
{
	ABB_REQUIRE(out && id, "NULL argument");
	*out = nullptr;
	ABB_REQUIRE(world >= 1 && world <= 64 && rank >= 0 && rank < world, "rank %d / world %d out of range", rank, world);
	ABB_CHECK(load_nccl());
	ABB_CHECK(select_device(device));
	abb_comm* c = new (std::nothrow) abb_comm();
	if (!c) {
		set_error("out of host memory");
		return ABB_ENOMEM;
	}
	c->rank = rank;
	c->world = world;
	c->device = device;
	ncclUniqueId nid;
	memcpy(&nid, id, sizeof nid);
	ncclResult_t r = g_nccl.CommInitRank(&c->comm, world, nid, rank);
	if (r != ncclSuccess) {
		set_error("ncclCommInitRank failed: %s", g_nccl.GetErrorString(r));
		delete c;
		return ABB_ECUDA;
	}
	*out = c;
	return ABB_OK;
}

int abb_comm_destroy(abb_comm* c)
{
	if (!c)
		return ABB_OK;
	cudaSetDevice(c->device);
	if (c->comm && g_nccl.CommDestroy)
		g_nccl.CommDestroy(c->comm);
	delete c;
	return ABB_OK;
}

int abb_comm_rank(const abb_comm* c) { return c ? c->rank : 0; }
int abb_comm_world(const abb_comm* c) { return c ? c->world : 1; }

int abb_filter_allgather(abb_filter* f, abb_comm* c)
{
	ABB_REQUIRE(f && c, "NULL argument");
	ABB_REQUIRE_NTHASH(f);
	ABB_REQUIRE(f->levels == 1, "only single-level filters are sharded");
	ABB_CUDA(cudaSetDevice(f->device));
	if (c->world == 1 || f->replicated_insert)
		return ABB_OK;
	const uint64_t chunk = shard_chunk(f->bytes_per_level, (unsigned)c->world);
	ABB_REQUIRE(chunk * c->world <= f->bytes_per_level + 4096, "too many ranks for the all-gather slack");
	ABB_NCCL(g_nccl.AllGather(f->d_data.p + (uint64_t)c->rank * chunk, f->d_data.p, chunk, ncclUint8, c->comm, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	return ABB_OK;
}

int abb_comm_allgather_bytes(abb_comm* c, void* d_buf, uint64_t bytes_per_rank, void* cuda_stream)
{
	ABB_REQUIRE(c && (d_buf || bytes_per_rank == 0), "NULL argument");
	if (c->world == 1 || bytes_per_rank == 0)
		return ABB_OK;
	ABB_CUDA(cudaSetDevice(c->device));
	ABB_NCCL(g_nccl.AllGather((const uint8_t*)d_buf + (uint64_t)c->rank * bytes_per_rank, d_buf, bytes_per_rank, ncclUint8, c->comm,
	                          (cudaStream_t)cuda_stream));
	return ABB_OK;
}

int abb_comm_exchange_bytes(abb_comm* c, const void* d_send, uint64_t send_bytes, void* d_recv_base, const uint64_t* recv_offsets,
                            const uint64_t* recv_bytes, void* cuda_stream)
{
	ABB_REQUIRE(c && recv_offsets && recv_bytes, "NULL argument");
	if (c->world == 1)
		return ABB_OK;
	ABB_CUDA(cudaSetDevice(c->device));
	cudaStream_t st = (cudaStream_t)cuda_stream;
	ABB_NCCL(g_nccl.GroupStart());
	for (int r = 0; r < c->world; ++r) {
		if (r == c->rank)
			continue;
		if (send_bytes)
			ABB_NCCL(g_nccl.Send(d_send, send_bytes, ncclUint8, r, c->comm, st));
		if (recv_bytes[r])
			ABB_NCCL(g_nccl.Recv((uint8_t*)d_recv_base + recv_offsets[r], recv_bytes[r], ncclUint8, r, c->comm, st));
	}
	ABB_NCCL(g_nccl.GroupEnd());
	return ABB_OK;
}

int abb_insert_reads_sharded_dev(abb_filter* f, abb_comm* c, const char* d_bases, const uint64_t* d_offsets, uint64_t n_reads,
                                 int finalize, uint64_t* n_kmers_out)
{
	ABB_REQUIRE(f && c, "NULL argument");
	ABB_REQUIRE_NTHASH(f);
	ABB_REQUIRE(f->kind == ABB_COUNTING, "the sharded insert is implemented for counting filters");
	ABB_REQUIRE(n_reads == 0 || (d_bases && d_offsets), "NULL read buffers");
	ABB_REQUIRE(f->device == c->device, "filter and communicator live on different devices");
	ABB_CUDA(cudaSetDevice(f->device));
	// Policy: the position-sharded insert divides the counter traffic by the world size but every rank still evaluates every
	// lane and pays a collective per window, so with few ranks the collectives cost more than the divided traffic saves.
	// Below ABB_SHARD_MIN_WORLD ranks (default 4) every rank
	// therefore runs the whole insert itself -- same bytes, no communication -- and only pass 2 is divided.
	const bool shard = shard_policy(c->world);
	f->replicated_insert = !shard;
	ABB_CHECK(insert_reads_dev(f, (const uint8_t*)d_bases, d_offsets, n_reads, n_kmers_out, shard ? c : nullptr));
	if (finalize)
		ABB_CHECK(abb_filter_allgather(f, c));
	return ABB_OK;
}

void* abb_filter_device_ptr(abb_filter* f, int level)
{
	unsigned l = 0;
	if (!f || resolve_level(f, level, &l) != ABB_OK)
		return nullptr;
	cudaSetDevice(f->device);
	cudaStreamSynchronize(f->stream);
	return f->level_data(l);
}

static int query_hashes(abb_filter* f, const uint64_t* hashes, uint64_t n, uint8_t* out, bool want_min)
{
	ABB_REQUIRE(f, "NULL filter");
	ABB_REQUIRE_NTHASH(f);
	if (n == 0)
		return ABB_OK;
	ABB_REQUIRE(hashes && out, "NULL buffer");
	ABB_CUDA(cudaSetDevice(f->device));
	ABB_CHECK(f->lit.reserve(n * f->H));
	ABB_CHECK(f->out8.reserve(n));
	ABB_CUDA(cudaMemcpyAsync(f->lit.p, hashes, n * f->H * sizeof(uint64_t), cudaMemcpyHostToDevice, f->stream));
	const FilterView fv = view_of(f);
	if (f->kind == ABB_COUNTING)
		k_query<0><<<blocks_for(n, 256), 256, 0, f->stream>>>(f->lit.p, n, f->cfg, fv, f->threshold, want_min ? nullptr : f->out8.p,
		                                                       want_min ? f->out8.p : nullptr);
	else
		k_query<1><<<blocks_for(n, 256), 256, 0, f->stream>>>(f->lit.p, n, f->cfg, fv, 0, want_min ? nullptr : f->out8.p,
		                                                       want_min ? f->out8.p : nullptr);
	f->st.launches += 1;
	ABB_CUDA(cudaGetLastError());
	ABB_CUDA(cudaMemcpyAsync(out, f->out8.p, n, cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	return ABB_OK;
}

int abb_contains_hashes(abb_filter* f, const uint64_t* hashes, uint64_t n, uint8_t* out) { return query_hashes(f, hashes, n, out, false); }
int abb_mincount_hashes(abb_filter* f, const uint64_t* hashes, uint64_t n, uint8_t* out) { return query_hashes(f, hashes, n, out, true); }

int abb_contains_reads(abb_filter* f, const char* bases, const uint64_t* offsets, uint64_t n_reads, uint8_t* out_flag, uint8_t* out_valid,
                       uint64_t capacity, uint64_t* n_slots_out)
{
	ABB_REQUIRE(f, "NULL filter");
	if (n_slots_out)
		*n_slots_out = 0;
	if (n_reads == 0)
		return ABB_OK;
	ABB_CHECK(check_read_batch(bases, offsets, n_reads));
	ABB_CUDA(cudaSetDevice(f->device));
	// own staging buffers: the batch a previous insert left resident (abb_filter_resident_reads) stays valid
	DevBuf<uint8_t> d_bases;
	DevBuf<uint64_t> d_offs;
	const SyncOnExit sync = { f->stream }; // before the staging buffers are freed
	ABB_CHECK(stage_read_batch(bases, offsets, n_reads, d_bases, d_offs, f->stream));
	uint64_t total = 0;
	ABB_CHECK(compute_slot_offsets(f->k, d_offs.p, n_reads, f->slot_offs, f->scan_tmp, f->stream, &total, &f->st.launches));
	if (n_slots_out)
		*n_slots_out = total;
	if (total == 0 || (!out_flag && !out_valid))
		return ABB_OK;
	ABB_REQUIRE(capacity >= total, "output buffers hold %llu slots, %llu needed", (unsigned long long)capacity, (unsigned long long)total);
	ABB_CHECK(f->valid.reserve(total));
	ABB_CHECK(f->out8.reserve(total));
	if (f->kind == ABB_KONNECTOR)
		ABB_CHECK(kon_query_slots(f, d_bases.p, d_offs.p, n_reads, total));
	else {
		ABB_CHECK(f->h0.reserve(total));
		ABB_CHECK(launch_hash(f->k, f->d_care.p, d_bases.p, d_offs.p, f->slot_offs.p, 0, n_reads, 0, f->h0.p, f->valid.p, f->stream, &f->st.launches));
		const FilterView fv = view_of(f);
		const unsigned grid = std::min<unsigned>(blocks_for(total, 256), sm_count() * 16);
		if (f->kind == ABB_COUNTING)
			k_query_h0<0><<<grid, 256, 0, f->stream>>>(f->h0.p, f->valid.p, total, f->cfg, fv, f->threshold, f->out8.p);
		else
			k_query_h0<1><<<grid, 256, 0, f->stream>>>(f->h0.p, f->valid.p, total, f->cfg, fv, 0, f->out8.p);
		f->st.launches += 1;
		ABB_CUDA(cudaGetLastError());
	}
	if (out_flag)
		ABB_CUDA(cudaMemcpyAsync(out_flag, f->out8.p, total, cudaMemcpyDeviceToHost, f->stream));
	if (out_valid)
		ABB_CUDA(cudaMemcpyAsync(out_valid, f->valid.p, total, cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	return ABB_OK;
}

int abb_successors(abb_filter* f, const char* kmers, uint64_t n, unsigned max_chain, abb_succ_info* out, unsigned* out_len, uint64_t* self_hash)
{
	ABB_REQUIRE(f, "NULL filter");
	ABB_REQUIRE_NTHASH(f);
	if (n == 0)
		return ABB_OK;
	ABB_REQUIRE(kmers && out && out_len && self_hash, "NULL buffer");
	ABB_REQUIRE(max_chain >= 1 && max_chain <= 128, "max_chain must be in 1..128");
	ABB_REQUIRE(f->mask.empty(), "graph neighbourhood queries are not available with a spaced seed");
	ABB_REQUIRE(f->H <= 64, "too many hash functions");
	ABB_CUDA(cudaSetDevice(f->device));
	DevBuf<uint8_t>& d_k = f->gq_kmers;
	DevBuf<abb_succ_info>& d_info = f->gq_info;
	DevBuf<unsigned>& d_len = f->gq_len;
	DevBuf<uint64_t>& d_self = f->gq_self;
	const SyncOnExit sync = { f->stream };
	ABB_CHECK(d_k.reserve(n * f->k));
	ABB_CHECK(d_info.reserve(n * max_chain));
	ABB_CHECK(d_len.reserve(n));
	ABB_CHECK(d_self.reserve(n));
	ABB_CUDA(cudaMemcpyAsync(d_k.p, kmers, n * f->k, cudaMemcpyHostToDevice, f->stream));
	ABB_CUDA(cudaMemsetAsync(d_info.p, 0, n * max_chain * sizeof(abb_succ_info), f->stream));
	const FilterView fv = view_of(f);
	if (f->kind == ABB_COUNTING) {
		const FilterProbe<0> probe = { f->cfg, fv, f->threshold };
		k_successors<0><<<blocks_for(n, 128), 128, 0, f->stream>>>(d_k.p, n, f->k, max_chain, probe, d_info.p, d_len.p, d_self.p);
	} else {
		const FilterProbe<1> probe = { f->cfg, fv, 0 };
		k_successors<1><<<blocks_for(n, 128), 128, 0, f->stream>>>(d_k.p, n, f->k, max_chain, probe, d_info.p, d_len.p, d_self.p);
	}
	f->st.launches += 1;
	ABB_CUDA(cudaGetLastError());
	ABB_CUDA(cudaMemcpyAsync(out, d_info.p, n * max_chain * sizeof(abb_succ_info), cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaMemcpyAsync(out_len, d_len.p, n * sizeof(unsigned), cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaMemcpyAsync(self_hash, d_self.p, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	return ABB_OK;
}

/** k-mers per k_graph_neighbors launch of abb_graph_neighbors: bounds its staging to 12.5 MiB of k-mers (k = 192) and 5 MiB of
 *  results, reused from call to call */
constexpr uint64_t kNbrPiece = 1 << 16;

/** ABB_ESTATE unless f is a bit or cascading filter without a spaced seed */
static int require_bit_filter(const abb_filter* f, const char* what)
{
	if ((f->kind != ABB_BIT && f->kind != ABB_CASCADING) || !f->mask.empty()) {
		set_error("abb_graph_neighbors: the %s must be a bit or cascading filter without a spaced seed", what);
		return ABB_ESTATE;
	}
	return ABB_OK;
}

int abb_graph_neighbors(abb_filter* g, const char* kmers, uint64_t n, abb_filter* const* attr, unsigned n_attr, abb_nbr_info* out)
{
	ABB_CHECK(select_device(g ? g->device : 0));
	ABB_REQUIRE(g, "NULL filter");
	ABB_REQUIRE(n_attr <= kMaxAttrFilters, "at most %u attribute filters", kMaxAttrFilters);
	ABB_REQUIRE(n_attr == 0 || attr, "NULL attribute filter list");
	ABB_CHECK(require_bit_filter(g, "graph"));
	NbrQuery q;
	q.cfg = g->cfg;
	q.rt = make_rolltab(g->k);
	q.bits = g->level_data(g->levels - 1);
	q.n_attr = n_attr;
	for (unsigned a = 0; a < n_attr; ++a) {
		const abb_filter* f = attr[a];
		ABB_REQUIRE(f, "NULL attribute filter %u", a);
		ABB_CHECK(require_bit_filter(f, "attribute filter"));
		if (f->device != g->device || f->H > g->H) {
			set_error("abb_graph_neighbors: attribute filter %u must live on the graph's device and use at most its %u hashes", a, g->H);
			return ABB_ESTATE;
		}
		q.attr[a].bits = f->level_data(f->levels - 1);
		q.attr[a].mod = f->cfg.mod;
		q.attr[a].H = f->H;
		ABB_CUDA(cudaStreamSynchronize(f->stream)); // its bits are read on the graph's stream
	}
	if (n == 0)
		return ABB_OK;
	ABB_REQUIRE(kmers && out, "NULL buffer");
	const unsigned probes = nbr_lane_probes(q); // <= kMaxLaneProbes: H <= kMaxHashes, H_a <= H
	const SyncOnExit sync = { g->stream };
	ABB_CHECK(g->gq_kmers.reserve(std::min(n, kNbrPiece) * g->k));
	ABB_CHECK(g->gq_nbr.reserve(std::min(n, kNbrPiece)));
	for (uint64_t i0 = 0; i0 < n; i0 += kNbrPiece) {
		const uint64_t m = std::min(kNbrPiece, n - i0);
		ABB_CUDA(cudaMemcpyAsync(g->gq_kmers.p, kmers + i0 * g->k, m * g->k, cudaMemcpyHostToDevice, g->stream));
		{
			// with profiling on, the CUDA-event time of the launch alone (abb_insert_stats::ms_graph)
			std::unique_ptr<StreamTimer> timer;
			if (g->profile)
				timer.reset(new StreamTimer(g->ev0, g->ev1, g->stream, &g->st.ms_graph));
			const unsigned grid = std::min<unsigned>(blocks_for(m, 8), sm_count() * 8);
			with_lane_probes(probes, [&](auto P) {
				k_graph_neighbors<decltype(P)::value><<<grid, 256, 0, g->stream>>>(g->gq_kmers.p, m, q, g->gq_nbr.p);
			});
			ABB_CUDA(cudaGetLastError());
		}
		g->st.launches += 1;
		g->st.graph_launches += 1;
		ABB_CUDA(cudaMemcpyAsync(out + i0, g->gq_nbr.p, m * sizeof(abb_nbr_info), cudaMemcpyDeviceToHost, g->stream));
		ABB_CUDA(cudaStreamSynchronize(g->stream)); // the staging is reused by the next piece
	}
	return ABB_OK;
}

int abb_hash_reads(unsigned k, const char* mask, const char* bases, const uint64_t* offsets, uint64_t n_reads,
                   uint64_t* out_h0, uint8_t* out_valid, uint64_t* n_slots_out, int device)
{
	ABB_REQUIRE(k >= 1 && k <= abb_max_kmer(), "k-mer size must be in 1..%u", abb_max_kmer());
	if (n_slots_out)
		*n_slots_out = 0;
	if (n_reads == 0)
		return ABB_OK;
	ABB_CHECK(check_read_batch(bases, offsets, n_reads));
	ABB_CHECK(select_device(device));
	std::string m = mask ? mask : "";
	if (!m.empty()) {
		ABB_REQUIRE(m.size() == k, "spaced seed must be exactly k=%u characters long", k);
		if (m.find('0') == std::string::npos)
			m.clear();
	}
	DevBuf<uint8_t> d_bases, d_valid, tmp, d_care;
	DevBuf<uint64_t> d_offs, d_slot, d_h0;
	ABB_CHECK(stage_read_batch(bases, offsets, n_reads, d_bases, d_offs, 0));
	if (!m.empty()) {
		std::vector<uint8_t> care(k);
		for (unsigned i = 0; i < k; ++i)
			care[i] = m[i] == '1';
		ABB_CHECK(d_care.reserve(k));
		ABB_CUDA(cudaMemcpy(d_care.p, care.data(), k, cudaMemcpyHostToDevice));
	}
	uint64_t total = 0;
	ABB_CHECK(compute_slot_offsets(k, d_offs.p, n_reads, d_slot, tmp, 0, &total, nullptr));
	if (n_slots_out)
		*n_slots_out = total;
	if (total && out_h0 && out_valid) {
		ABB_CHECK(d_h0.reserve(total));
		ABB_CHECK(d_valid.reserve(total));
		ABB_CHECK(launch_hash(k, m.empty() ? nullptr : d_care.p, d_bases.p, d_offs.p, d_slot.p, 0, n_reads, 0, d_h0.p, d_valid.p, 0,
		                      nullptr));
		ABB_CUDA(cudaMemcpy(out_h0, d_h0.p, total * sizeof(uint64_t), cudaMemcpyDeviceToHost));
		ABB_CUDA(cudaMemcpy(out_valid, d_valid.p, total, cudaMemcpyDeviceToHost));
	}
	return ABB_OK;
}

static int level_ptr(abb_filter* f, int level, uint64_t nbytes, uint8_t** p)
{
	ABB_REQUIRE(f, "NULL filter");
	unsigned l = 0;
	ABB_CHECK(resolve_level(f, level, &l));
	ABB_REQUIRE(nbytes == f->bytes_per_level, "buffer is %llu bytes, the filter level is %llu", (unsigned long long)nbytes,
	            (unsigned long long)f->bytes_per_level);
	*p = f->level_data(l);
	return ABB_OK;
}

int abb_filter_download(abb_filter* f, int level, uint8_t* host, uint64_t nbytes)
{
	uint8_t* p = nullptr;
	ABB_CHECK(level_ptr(f, level, nbytes, &p));
	ABB_REQUIRE(host, "NULL buffer");
	ABB_CUDA(cudaSetDevice(f->device));
	ABB_CUDA(cudaMemcpyAsync(host, p, nbytes, cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	return ABB_OK;
}

int abb_filter_upload(abb_filter* f, int level, const uint8_t* host, uint64_t nbytes)
{
	uint8_t* p = nullptr;
	ABB_CHECK(level_ptr(f, level, nbytes, &p));
	ABB_REQUIRE(host, "NULL buffer");
	ABB_CUDA(cudaSetDevice(f->device));
	ABB_CUDA(cudaMemcpyAsync(p, host, nbytes, cudaMemcpyHostToDevice, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	return ABB_OK;
}

int abb_filter_clear(abb_filter* f)
{
	ABB_REQUIRE(f, "NULL filter");
	ABB_CUDA(cudaSetDevice(f->device));
	ABB_CUDA(cudaMemsetAsync(f->d_data.p, 0, f->level_stride() * f->levels, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	return ABB_OK;
}

int abb_filter_popcount(abb_filter* f, uint64_t* nonzero, uint64_t* at_or_above_threshold)
{
	ABB_REQUIRE(f, "NULL filter");
	if (f->kind == ABB_KONNECTOR) { // its levels need not start on a 16-byte boundary
		uint64_t n = 0;
		ABB_CHECK(abb_filter_level_popcount(f, -1, &n));
		if (nonzero)
			*nonzero = n;
		if (at_or_above_threshold)
			*at_or_above_threshold = n;
		return ABB_OK;
	}
	ABB_CUDA(cudaSetDevice(f->device));
	ABB_CUDA(cudaMemsetAsync(f->d_stats.p + kStatPopcount, 0, 2 * sizeof(unsigned long long), f->stream));
	// bit / cascading: population of the LAST level (the one contains() consults)
	const uint8_t* p = f->level_data(f->levels - 1);
	k_popcount<<<sm_count() * 8, 256, 0, f->stream>>>(p, f->bytes_per_level, f->kind == ABB_COUNTING, f->threshold,
	                                                  f->d_stats.p + kStatPopcount);
	f->st.launches += 1;
	ABB_CUDA(cudaGetLastError());
	unsigned long long h[2] = { 0, 0 };
	ABB_CUDA(cudaMemcpyAsync(h, f->d_stats.p + kStatPopcount, sizeof h, cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	if (nonzero)
		*nonzero = h[0];
	if (at_or_above_threshold)
		*at_or_above_threshold = f->kind == ABB_COUNTING ? h[1] : h[0];
	return ABB_OK;
}

void* abb_filter_stream(abb_filter* f) { return f ? (void*)f->stream : nullptr; }

int abb_filter_insert_stats(abb_filter* f, abb_insert_stats* out, int reset)
{
	ABB_REQUIRE(f, "NULL filter");
	ABB_CUDA(cudaSetDevice(f->device));
	unsigned long long h[kStatDrainedSlots + 1] = {}; // the words that accumulate over calls
	ABB_CUDA(cudaMemcpyAsync(h, f->d_stats.p, sizeof h, cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	f->st.deferred = h[kStatDeferred];
	f->st.drains = h[kStatDrains] + f->sh_drains;
	f->st.drained_slots = h[kStatDrainedSlots];
	if (out)
		*out = f->st;
	if (reset) {
		f->sh_drains = 0;
		f->st = abb_insert_stats{};
		ABB_CUDA(cudaMemsetAsync(f->d_stats.p, 0, sizeof h, f->stream));
	}
	return ABB_OK;
}

} // extern "C"
