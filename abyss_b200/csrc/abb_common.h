// abb_common.h -- host-side plumbing shared by the C-ABI translation units.
#pragma once
#include "../../include/abyss_b200.h"
#include "abb_device.cuh"
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdio>
#include <memory>
#include <string>
#include <utility>
#include <vector>

namespace abb {

void set_error(const char* fmt, ...);

#define ABB_CUDA(call)                                                                             \
	do {                                                                                           \
		cudaError_t e__ = (call);                                                                  \
		if (e__ != cudaSuccess) {                                                                  \
			cudaGetLastError(); /* returned here: a later launch check must not report it again */ \
			abb::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
			return (e__ == cudaErrorMemoryAllocation) ? ABB_ENOMEM                                 \
			       : (e__ == cudaErrorNoDevice || e__ == cudaErrorInsufficientDriver) ? ABB_ENODEV \
			                                                                          : ABB_ECUDA; \
		}                                                                                          \
	} while (0)

#define ABB_CHECK(expr)            \
	do {                           \
		int rc__ = (expr);         \
		if (rc__ != ABB_OK)        \
			return rc__;           \
	} while (0)

#define ABB_REQUIRE(cond, ...)         \
	do {                               \
		if (!(cond)) {                 \
			abb::set_error(__VA_ARGS__); \
			return ABB_EINVAL;         \
		}                              \
	} while (0)

/** entry points of the ntHash filter kinds (hash arrays, spaced seeds, the sharded insert, graph queries) */
#define ABB_REQUIRE_NTHASH(f)                                                                       \
	do {                                                                                            \
		if ((f)->kind == ABB_KONNECTOR) {                                                           \
			abb::set_error("%s: not available for Konnector (-t konnector) filters", __func__);     \
			return ABB_ESTATE;                                                                      \
		}                                                                                           \
	} while (0)

/** Device buffer that owns its allocation: freed by the destructor, moved but never copied.  Every owner lives in a
 *  handle or on the stack of a C-ABI call, never in static storage (its destructor would run after the runtime shut down). */
template <typename T>
struct DevBuf {
	T* p = nullptr;
	size_t cap = 0;
	DevBuf() = default;
	DevBuf(DevBuf&& o) noexcept { *this = std::move(o); }
	DevBuf& operator=(DevBuf&& o) noexcept
	{
		if (this != &o) {
			reset();
			std::swap(p, o.p);
			std::swap(cap, o.cap);
		}
		return *this;
	}
	~DevBuf() { reset(); }
	/** at least n elements, with slack for growing batches; the contents are not kept */
	int reserve(size_t n) { return n <= cap ? ABB_OK : alloc(n + n / 8 + 256); }
	/** exactly n elements, the old allocation freed first (peak memory); the contents are not kept */
	int alloc(size_t n)
	{
		reset();
		ABB_CUDA(cudaMalloc((void**)&p, n * sizeof(T)));
		cap = n;
		return ABB_OK;
	}
	void reset()
	{
		if (p)
			cudaFree(p);
		p = nullptr;
		cap = 0;
	}
};

/** A CUDA stream or event owned like DevBuf; it converts to the raw handle for the runtime calls that use it. */
template <typename H, cudaError_t (*Destroy)(H)>
struct Owned {
	H h = nullptr;
	Owned() = default;
	Owned(Owned&& o) noexcept { std::swap(h, o.h); }
	~Owned() { reset(); }
	operator H() const { return h; }
	/** for the create call: destroys the current handle and hands out the slot for the new one */
	H* out()
	{
		reset();
		return &h;
	}
	void reset()
	{
		if (h)
			Destroy(h);
		h = nullptr;
	}
};
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
using Event = Owned<cudaEvent_t, cudaEventDestroy>;

/** synchronises the stream when the scope ends, on every return path: no asynchronous copy into a caller's buffer
 *  outlives the C-ABI call that queued it */
struct SyncOnExit {
	cudaStream_t s;
	~SyncOnExit() { cudaStreamSynchronize(s); }
};

/** Adds the CUDA-event time of a stretch of a stream to *acc.  The stretch starts at construction and ends at end(), or
 *  where the scope is left, on every return path, if end() was not called.  The time is read when the scope is left,
 *  after waiting for the end event: a timer whose end() is followed by a stream synchronise waits for nothing. */
struct StreamTimer {
	cudaEvent_t e0, e1;
	cudaStream_t s;
	float* acc;
	bool ended = false;
	StreamTimer(cudaEvent_t e0_, cudaEvent_t e1_, cudaStream_t s_, float* acc_) : e0(e0_), e1(e1_), s(s_), acc(acc_) { cudaEventRecord(e0, s); }
	StreamTimer(const StreamTimer&) = delete;
	void end()
	{
		cudaEventRecord(e1, s);
		ended = true;
	}
	~StreamTimer()
	{
		if (!ended)
			end();
		float ms = 0;
		if (cudaEventSynchronize(e1) == cudaSuccess && cudaEventElapsedTime(&ms, e0, e1) == cudaSuccess)
			*acc += ms;
	}
};

/** hands a finished handle to the C caller, whose abb_*_destroy owns it from then on */
template <typename T>
int hand_over(std::unique_ptr<T>& h, T** out)
{
	*out = h.release();
	return ABB_OK;
}

inline unsigned blocks_for(uint64_t n, unsigned threads) { return (unsigned)((n + threads - 1) / threads); }

/** streaming multiprocessors of the current device (132 on an H100 SXM); grid-stride kernels are sized from it */
inline unsigned sm_count()
{
	int dev = 0, n = 0;
	cudaGetDevice(&dev);
	cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
	return n > 0 ? (unsigned)n : 132;
}

// host helpers implemented in abb_api.cu, shared with the other C-ABI translation units
int select_device(int device);
/** A host read batch (bases, offsets[n_reads + 1]) as the C ABI takes it: ABB_EINVAL unless the buffers are given and
 *  offsets[0] == 0; "NULL <noun> buffers" names them.  Host only, so a malformed batch is refused without a device.
 *  An empty batch needs no buffers. */
int check_read_batch(const char* bases, const uint64_t* offsets, uint64_t n_reads, const char* noun = "read");
/** Queues the copy of a checked host read batch to d_bases (16 bytes of slack) and d_offs on `stream`, growing them as
 *  needed.  With bases NULL only d_bases is sized: the caller copies the bases itself. */
int stage_read_batch(const char* bases, const uint64_t* offsets, uint64_t n_reads, DevBuf<uint8_t>& d_bases, DevBuf<uint64_t>& d_offs,
                     cudaStream_t stream);
/** slot_offs[0..n_reads] = exclusive prefix sum of per-read k-mer window counts; *total = sum */
int compute_slot_offsets(unsigned k, const uint64_t* d_offs, uint64_t n_reads, DevBuf<uint64_t>& slot_offs,
                         DevBuf<uint8_t>& tmp, cudaStream_t stream, uint64_t* total, uint64_t* launches);

} // namespace abb

struct abb_filter;
namespace abb {
/** device-resident control block of the ordered insert (abb_insert.cuh) */
struct InsertCtl {
	unsigned n_carry[2];  // lengths of the two carry lists
	unsigned old_flag;    // a slot carried again is older than the drain age
	unsigned resume;      // first window the kernel has NOT processed (it stops early when a drain is due)
	unsigned tag_mask[2]; // prefix of each tag table that is in use (to be cleared before its next use)
};
struct ShardCtl; // abb_shard.cuh

/** the words of abb_filter::d_stats; no two operations share one.  The first three accumulate over calls
 *  (abb_filter_insert_stats reads and resets them), each of the others is cleared by the call that uses it. */
enum StatWord : unsigned {
	kStatDeferred,                     // slots that did not commit in their own window
	kStatDrains,                       // drains that did work
	kStatDrainedSlots,                 // slots replayed by drains
	kStatInsertKmers,                  // valid k-mers of one insert (k_count_valid)
	kStatKonKmers,                     // k-mers of one Konnector insert
	kStatPopcount,                     // [2] abb_filter_popcount: nonzero, at or above the threshold
	kStatLevelPop = kStatPopcount + 2, // abb_filter_level_popcount
	kStatCompare,                      // [3] abb_filter_compare: the 1/1, 1/0 and 0/1 bit counts
	kStatWords = kStatCompare + 3
};

/** K1 for reads [r0, r1): h0/valid index = slot_offs[r] + j - slot_base */
int launch_hash(unsigned k, const uint8_t* d_care, const uint8_t* d_bases, const uint64_t* d_offs, const uint64_t* d_slot_offs,
                uint64_t r0, uint64_t r1, uint64_t slot_base, uint64_t* d_h0, uint8_t* d_valid, cudaStream_t stream, uint64_t* launches);
int launch_hash_segments(unsigned k, const uint8_t* d_care, const uint8_t* d_bases, const uint64_t* d_seg_beg, const unsigned* d_seg_len,
                         const uint64_t* d_seg_slot, uint64_t n_segs, uint64_t* d_h0, uint8_t* d_valid, cudaStream_t stream);
/** level -1 is the last one; ABB_EINVAL for a level the filter does not have */
int resolve_level(const abb_filter* f, int level, unsigned* out);
// abb_konnector.cu: the ABB_KONNECTOR paths of abb_insert_reads(_dev) and abb_contains_reads
int kon_insert_reads_dev(abb_filter* f, const uint8_t* d_bases, const uint64_t* d_offs, uint64_t n_reads, uint64_t* n_kmers_out);
/** membership of the last level and validity of every window slot (f->slot_offs already computed) into f->out8 / f->valid */
int kon_query_slots(abb_filter* f, const uint8_t* d_bases, const uint64_t* d_offs, uint64_t n_reads, uint64_t n_slots);
}

/** The filter handle (opaque in the C ABI). */
struct abb_filter {
	int device = 0;
	int kind = ABB_COUNTING;
	uint64_t size = 0;            // counters, or bits per level
	uint64_t bytes_per_level = 0; // bytes of one level
	unsigned H = 0, k = 0, threshold = 0, levels = 1;
	uint64_t kon_full = 0, kon_start = 0, kon_seed = 0; // ABB_KONNECTOR: filter size in bits, first bit held, hash seed
	std::string mask;
	abb::DevBuf<uint8_t> d_care; // k bytes (mask == '1'), only with a spaced seed
	abb::DevBuf<uint8_t> d_data;
	abb::HashCfg cfg;
	abb::Stream stream;
	abb::Event ev0, ev1;
	// host-buffer insert: the bases travel in pieces on their own stream while earlier chunks are hashed and inserted
	abb::Stream copy_stream;
	std::vector<abb::Event> copy_ev; // copy_ev[i]: piece i has landed

	// ordered-insert workspace (abb_insert.cuh K2)
	uint64_t window = 0;      // slots per window
	uint64_t ws_window = 0;   // window the workspace below was sized for
	unsigned ws_H = 0;
	uint64_t map_entries = 0; // two-bit entries per conflict map (power of two)
	abb::DevBuf<unsigned> maps;                         // the three maps in one allocation (one L2 access-policy window covers them)
	unsigned* d_map[3] = { nullptr, nullptr, nullptr }; // the maps within `maps`
	abb::DevBuf<unsigned long long> d_tags2[2];         // tag tables of the carried slots (alternating windows)
	uint64_t tag_slots = 0;
	abb::DevBuf<uint64_t> d_carry;    // two carry lists and the drain's sorted list, (window + kCarryLanes) slots each
	abb::DevBuf<unsigned> d_slotbits; // presence bitmap of the drain
	uint64_t slotbit_words = 0;
	abb::DevBuf<abb::InsertCtl> d_ctl;
	abb::DevBuf<abb::ShardCtl> d_shard_ctl;
	abb::DevBuf<unsigned long long> d_stats; // abb::kStatWords words, abb::StatWord

	// per-call buffers (bases/offs keep the device copy of the last host batch: abb_filter_resident_reads)
	uint64_t resident_reads = 0;
	bool l2_policy_held = false;    // an enclosing scope already pinned the conflict maps in L2 (abb_api.cu PolicyHold)
	bool replicated_insert = false; // the last "sharded" insert ran replicated (small worlds): nothing to all-gather
	abb::DevBuf<uint8_t> bases;
	abb::DevBuf<uint64_t> offs, slot_offs, h0, lit, bounds;
	abb::DevBuf<uint8_t> valid, scan_tmp, out8, sh_buf;
	// abb_trim_reads: the batch, its trim lengths and the walk scratch of the grid, kept from one batch to the next
	abb::DevBuf<uint8_t> trim_bases, trim_scratch;
	abb::DevBuf<uint64_t> trim_offs;
	abb::DevBuf<uint32_t> trim_out;
	// abb_successors staging (a graph dump issues thousands of small queries: no allocation per call)
	abb::DevBuf<uint8_t> gq_kmers;
	abb::DevBuf<abb_succ_info> gq_info;
	abb::DevBuf<unsigned> gq_len;
	abb::DevBuf<uint64_t> gq_self;
	abb::DevBuf<abb_nbr_info> gq_nbr; // abb_graph_neighbors (gq_kmers holds its k-mers)

	/** device bytes from one level to the next.  Bit and cascading levels start on 16-byte boundaries: bits_set ORs 4-byte words
	 *  and k_popcount loads uint4, while size / 8 need only be a multiple of 1.  Counting filters have one level, and the
	 *  Konnector kernels address a packed array of levels.  The padding is never part of a level: bytes_per_level is. */
	/** bits of one level: a Konnector filter holds `size` bits, the others a whole number of bytes */
	uint64_t bits_per_level() const { return kind == ABB_KONNECTOR ? size : bytes_per_level * 8; }
	uint64_t level_stride() const { return kind == ABB_BIT || kind == ABB_CASCADING ? (bytes_per_level + 15) & ~15ULL : bytes_per_level; }
	uint8_t* level_data(unsigned level) const { return d_data.p + (uint64_t)level * level_stride(); }

	// statistics
	abb_insert_stats st = {};
	bool profile = false; // time the k_window launches with CUDA events (every prof_stride-th window)
	uint64_t prof_stride = 1, prof_slots = 0, sh_drains = 0;
	std::vector<abb::Event> prof_ev;
	size_t prof_used = 0;
};
