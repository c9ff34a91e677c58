// abb_overlap.cu -- C ABI of the contig overlap graph (AdjList/AdjList.cpp; SURVEY.md section 8f.3): kernels over the
// per-item functions of abb_overlap.cuh, two-pass (count, scan, emit) hash joins, one final sort of the edges.
#include "abb_common.h"
#include "abb_overlap.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <new>

namespace abb {

__global__ void __launch_bounds__(256) k_ovl_keys(OvlSeqs s, uint64_t* key_p, uint32_t* val_p, uint64_t* key_s, unsigned* bad)
{
	const uint64_t n2 = 2 * s.n;
	for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n2; j += (uint64_t)gridDim.x * blockDim.x)
		ovl_keys_item(s, (uint32_t)j, key_p, val_p, key_s, bad);
}

/** contigs must be longer than k - 1 (AdjList.cpp:222 asserts it) */
__global__ void __launch_bounds__(256) k_ovl_check_len(OvlSeqs s, unsigned* bad)
{
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < s.n; i += (uint64_t)gridDim.x * blockDim.x)
		if (s.offs[i + 1] - s.offs[i] <= s.k1)
			bad[1] = 1;
}

/** EMIT = false: cnt[x] = out-degree of x from join (1); EMIT = true: edges written at off[x] */
template <bool EMIT>
__global__ void __launch_bounds__(256) k_ovl_join(OvlSeqs s, int ss, const uint64_t* key_s, const uint64_t* sorted_p, const uint32_t* sorted_t,
                                                 uint64_t* cnt_or_off, uint64_t* ekey, int* edist)
{
	const uint64_t n2 = 2 * s.n;
	for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < n2; x += (uint64_t)gridDim.x * blockDim.x) {
		if (EMIT)
			ovl_join_item(s, ss, (uint32_t)x, key_s, sorted_p, sorted_t, n2, ekey + cnt_or_off[x], edist + cnt_or_off[x]);
		else
			cnt_or_off[x] = ovl_join_item(s, ss, (uint32_t)x, key_s, sorted_p, sorted_t, n2, nullptr, nullptr);
	}
}

/** flag[x] = 1 for a vertex without out-edges after join (1) (cnt holds the exclusive scan of the degrees, n2 + 1 entries) */
__global__ void __launch_bounds__(256) k_ovl_flag_blunt(const uint64_t* off, uint64_t n2, uint64_t* flag)
{
	for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < n2; x += (uint64_t)gridDim.x * blockDim.x)
		flag[x] = off[x + 1] == off[x];
}

/** blunt[pos[x]] = x for the flagged vertices (pos = exclusive scan of the flags): ascending vertex order */
__global__ void __launch_bounds__(256) k_ovl_scatter_blunt(const uint64_t* off, const uint64_t* pos, uint64_t n2, uint32_t* blunt)
{
	for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < n2; x += (uint64_t)gridDim.x * blockDim.x)
		if (off[x + 1] == off[x])
			blunt[pos[x]] = (uint32_t)x;
}

__global__ void __launch_bounds__(256) k_ovl_sub_keys(OvlSeqs s, const uint32_t* blunt, uint64_t n_blunt, unsigned n_q, uint64_t* key, uint64_t* val)
{
	const uint64_t n = n_blunt * n_q;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
		ovl_sub_keys_item(s, blunt, i / n_q, (unsigned)(i % n_q), n_q, key, val);
}

template <bool EMIT>
__global__ void __launch_bounds__(256) k_ovl_sub_join(OvlSeqs s, int ss, const uint32_t* blunt, uint64_t n_blunt, unsigned n_q, const uint64_t* sorted_key,
                                                     const uint64_t* sorted_val, uint64_t* cnt_or_off, uint64_t* ekey, int* edist)
{
	for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; b < n_blunt; b += (uint64_t)gridDim.x * blockDim.x) {
		if (EMIT)
			ovl_sub_join_item(s, ss, blunt, b, n_q, sorted_key, sorted_val, n_blunt * n_q, ekey + cnt_or_off[b], edist + cnt_or_off[b]);
		else
			cnt_or_off[b] = ovl_sub_join_item(s, ss, blunt, b, n_q, sorted_key, sorted_val, n_blunt * n_q, nullptr, nullptr);
	}
}

__global__ void __launch_bounds__(256) k_ovl_unpack(const uint64_t* ekey, const int* edist, uint64_t n, abb_overlap_edge* out)
{
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		abb_overlap_edge e;
		e.u = (uint32_t)(ekey[i] >> 32);
		e.v = (uint32_t)(ekey[i] & 0xffffffffu) ^ 1u;
		e.distance = edist[i];
		out[i] = e;
	}
}

} // namespace abb

using namespace abb;

struct abb_overlap {
	int device = 0;
	Stream stream;
	DevBuf<uint8_t> bases, tmp;
	DevBuf<uint64_t> offs, key_p, key_p2, key_s, cnt, pos, sub_key, sub_key2, sub_val, sub_val2, ekey, ekey2;
	DevBuf<uint32_t> val_p, val_p2, blunt;
	DevBuf<int> edist, edist2;
	DevBuf<abb_overlap_edge> d_edges;
	std::vector<abb_overlap_edge> edges;
	DevBuf<unsigned> d_bad;
	abb_overlap_stats st = {};
};

namespace abb {

static unsigned ovl_grid(uint64_t n) { return (unsigned)std::min<uint64_t>(std::max<uint64_t>(blocks_for(n, 256), 1), sm_count() * 16); }

/** exclusive sum of n + 1 entries in place (entry n is the total), total copied to the host */
static int ovl_scan(abb_overlap* h, uint64_t* d, uint64_t n, uint64_t* total)
{
	ABB_CUDA(cudaMemsetAsync(d + n, 0, sizeof(uint64_t), h->stream));
	size_t bytes = 0;
	ABB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, d, d, n + 1, h->stream));
	ABB_CHECK(h->tmp.reserve(bytes));
	ABB_CUDA(cub::DeviceScan::ExclusiveSum(h->tmp.p, bytes, d, d, n + 1, h->stream));
	ABB_CUDA(cudaMemcpyAsync(total, d + n, sizeof(uint64_t), cudaMemcpyDeviceToHost, h->stream));
	ABB_CUDA(cudaStreamSynchronize(h->stream));
	return ABB_OK;
}

template <typename K, typename V>
static int ovl_sort(abb_overlap* h, const K* k_in, K* k_out, const V* v_in, V* v_out, uint64_t n)
{
	size_t bytes = 0;
	ABB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, k_in, k_out, v_in, v_out, n, 0, (int)sizeof(K) * 8, h->stream));
	ABB_CHECK(h->tmp.reserve(bytes));
	ABB_CUDA(cub::DeviceRadixSort::SortPairs(h->tmp.p, bytes, k_in, k_out, v_in, v_out, n, 0, (int)sizeof(K) * 8, h->stream));
	return ABB_OK;
}

static int overlap_build(abb_overlap* h, const char* bases, const uint64_t* offsets, uint64_t n, unsigned k, unsigned min_overlap, int ss)
{
	cudaStream_t st = h->stream;
	h->edges.clear();
	h->st = abb_overlap_stats{};
	h->st.vertices = 2 * n;
	if (n == 0)
		return ABB_OK;
	const uint64_t n2 = 2 * n;
	const unsigned k1 = k - 1;
	ABB_CHECK(stage_read_batch(bases, offsets, n, h->bases, h->offs, st));
	ABB_CUDA(cudaMemsetAsync(h->d_bad.p, 0, 2 * sizeof(unsigned), st));
	OvlSeqs s = { h->bases.p, h->offs.p, n, k1 };
	k_ovl_check_len<<<ovl_grid(n), 256, 0, st>>>(s, h->d_bad.p);
	unsigned bad[2] = { 0, 0 };
	ABB_CUDA(cudaMemcpyAsync(bad, h->d_bad.p, sizeof bad, cudaMemcpyDeviceToHost, st));
	ABB_CUDA(cudaStreamSynchronize(st));
	ABB_REQUIRE(!bad[1], "a contig is not longer than k-1 = %u bases (AdjList asserts seq.length() > overlap)", k1);
	// join (1): exact k-1 overlaps
	ABB_CHECK(h->key_p.reserve(n2));
	ABB_CHECK(h->key_p2.reserve(n2));
	ABB_CHECK(h->val_p.reserve(n2));
	ABB_CHECK(h->val_p2.reserve(n2));
	ABB_CHECK(h->key_s.reserve(n2));
	ABB_CHECK(h->cnt.reserve(n2 + 1));
	k_ovl_keys<<<ovl_grid(n2), 256, 0, st>>>(s, h->key_p.p, h->val_p.p, h->key_s.p, h->d_bad.p);
	ABB_CUDA(cudaGetLastError());
	ABB_CHECK(ovl_sort(h, h->key_p.p, h->key_p2.p, h->val_p.p, h->val_p2.p, n2)); // stable: equal keys stay in ascending t ^ 1
	k_ovl_join<false><<<ovl_grid(n2), 256, 0, st>>>(s, ss, h->key_s.p, h->key_p2.p, h->val_p2.p, h->cnt.p, nullptr, nullptr);
	ABB_CUDA(cudaGetLastError());
	uint64_t e1 = 0;
	ABB_CHECK(ovl_scan(h, h->cnt.p, n2, &e1));
	ABB_CUDA(cudaMemcpyAsync(bad, h->d_bad.p, sizeof bad, cudaMemcpyDeviceToHost, st));
	ABB_CUDA(cudaStreamSynchronize(st));
	ABB_REQUIRE(!bad[0], "a contig end holds a character that is not a nucleotide (the reference's Kmer constructor aborts on it)");
	h->st.launches += 5;
	// join (2): overlaps of min_overlap .. k-2 bases between blunt vertices
	uint64_t n_blunt = 0, e2 = 0;
	const unsigned n_q = min_overlap < k1 ? k1 - min_overlap : 0;
	if (n_q) {
		ABB_CHECK(h->pos.reserve(n2 + 1));
		k_ovl_flag_blunt<<<ovl_grid(n2), 256, 0, st>>>(h->cnt.p, n2, h->pos.p);
		ABB_CHECK(ovl_scan(h, h->pos.p, n2, &n_blunt));
		h->st.launches += 2;
	}
	ABB_CHECK(h->ekey.reserve(e1 + 1));
	ABB_CHECK(h->edist.reserve(e1 + 1));
	if (e1) {
		k_ovl_join<true><<<ovl_grid(n2), 256, 0, st>>>(s, ss, h->key_s.p, h->key_p2.p, h->val_p2.p, h->cnt.p, h->ekey.p, h->edist.p);
		ABB_CUDA(cudaGetLastError());
		h->st.launches += 1;
	}
	if (n_q && n_blunt) {
		const uint64_t n_rec = n_blunt * n_q;
		ABB_CHECK(h->blunt.reserve(n_blunt));
		ABB_CHECK(h->sub_key.reserve(n_rec));
		ABB_CHECK(h->sub_key2.reserve(n_rec));
		ABB_CHECK(h->sub_val.reserve(n_rec));
		ABB_CHECK(h->sub_val2.reserve(n_rec));
		k_ovl_scatter_blunt<<<ovl_grid(n2), 256, 0, st>>>(h->cnt.p, h->pos.p, n2, h->blunt.p);
		k_ovl_sub_keys<<<ovl_grid(n_rec), 256, 0, st>>>(s, h->blunt.p, n_blunt, n_q, h->sub_key.p, h->sub_val.p);
		ABB_CUDA(cudaGetLastError());
		ABB_CHECK(ovl_sort(h, h->sub_key.p, h->sub_key2.p, h->sub_val.p, h->sub_val2.p, n_rec));
		// the degrees of join (1) are no longer needed: reuse pos for the per-query counts
		k_ovl_sub_join<false><<<ovl_grid(n_blunt), 256, 0, st>>>(s, ss, h->blunt.p, n_blunt, n_q, h->sub_key2.p, h->sub_val2.p, h->pos.p, nullptr, nullptr);
		ABB_CUDA(cudaGetLastError());
		ABB_CHECK(ovl_scan(h, h->pos.p, n_blunt, &e2));
		h->st.launches += 5;
		if (e2) {
			// grow the edge arrays, keeping the edges of join (1)
			DevBuf<uint64_t> nk;
			DevBuf<int> nd;
			ABB_CHECK(nk.reserve(e1 + e2));
			ABB_CHECK(nd.reserve(e1 + e2));
			ABB_CUDA(cudaMemcpyAsync(nk.p, h->ekey.p, e1 * sizeof(uint64_t), cudaMemcpyDeviceToDevice, st));
			ABB_CUDA(cudaMemcpyAsync(nd.p, h->edist.p, e1 * sizeof(int), cudaMemcpyDeviceToDevice, st));
			ABB_CUDA(cudaStreamSynchronize(st));
			h->ekey = std::move(nk);
			h->edist = std::move(nd);
			k_ovl_sub_join<true><<<ovl_grid(n_blunt), 256, 0, st>>>(s, ss, h->blunt.p, n_blunt, n_q, h->sub_key2.p, h->sub_val2.p, h->pos.p, h->ekey.p + e1,
			                                                       h->edist.p + e1);
			ABB_CUDA(cudaGetLastError());
			h->st.launches += 1;
		}
	}
	const uint64_t e = e1 + e2;
	h->st.exact_edges = e1;
	h->st.short_edges = e2;
	h->st.blunt_vertices = n_blunt;
	if (e == 0)
		return ABB_OK;
	// every out-list in ascending (v ^ 1), vertices in ascending order: one sort by (u, v ^ 1)
	ABB_CHECK(h->ekey2.reserve(e));
	ABB_CHECK(h->edist2.reserve(e));
	ABB_CHECK(ovl_sort(h, h->ekey.p, h->ekey2.p, h->edist.p, h->edist2.p, e));
	ABB_CHECK(h->d_edges.reserve(e));
	k_ovl_unpack<<<ovl_grid(e), 256, 0, st>>>(h->ekey2.p, h->edist2.p, e, h->d_edges.p);
	ABB_CUDA(cudaGetLastError());
	h->st.launches += 2;
	h->edges.resize(e);
	ABB_CUDA(cudaMemcpyAsync(h->edges.data(), h->d_edges.p, e * sizeof(abb_overlap_edge), cudaMemcpyDeviceToHost, st));
	ABB_CUDA(cudaStreamSynchronize(st));
	return ABB_OK;
}

} // namespace abb

extern "C" {

int abb_overlap_create(abb_overlap** out, int device)
{
	ABB_REQUIRE(out != nullptr, "abb_overlap_create: out is NULL");
	*out = nullptr;
	ABB_CHECK(select_device(device));
	std::unique_ptr<abb_overlap> h(new (std::nothrow) abb_overlap());
	if (!h) {
		set_error("out of host memory");
		return ABB_ENOMEM;
	}
	h->device = device;
	ABB_CUDA(cudaStreamCreateWithFlags(h->stream.out(), cudaStreamNonBlocking));
	ABB_CHECK(h->d_bad.alloc(2));
	return hand_over(h, out);
}

int abb_overlap_destroy(abb_overlap* h)
{
	if (!h)
		return ABB_OK;
	cudaSetDevice(h->device);
	cudaStreamSynchronize(h->stream);
	delete h;
	return ABB_OK;
}

int abb_overlap_build(abb_overlap* h, const char* bases, const uint64_t* offsets, uint64_t n_contigs, unsigned k, unsigned min_overlap, int ss,
                      const abb_overlap_edge** edges, uint64_t* n_edges)
{
	ABB_REQUIRE(h, "NULL handle");
	if (edges)
		*edges = nullptr;
	if (n_edges)
		*n_edges = 0;
	ABB_REQUIRE(k >= 2, "k must be at least 2");
	ABB_CHECK(check_read_batch(bases, offsets, n_contigs, "contig"));
	ABB_REQUIRE(n_contigs < (1ULL << 31), "too many contigs");
	// AdjList.cpp:386-388: 0 means k-1, never more than k-1
	if (min_overlap == 0 || min_overlap > k - 1)
		min_overlap = k - 1;
	ABB_REQUIRE(k - 1 - min_overlap < 256, "at most 255 overlap lengths below k-1 are searched (k-1 - min_overlap = %u)", k - 1 - min_overlap);
	ABB_CUDA(cudaSetDevice(h->device));
	ABB_CHECK(overlap_build(h, bases, offsets, n_contigs, k, min_overlap, ss));
	if (edges)
		*edges = h->edges.data();
	if (n_edges)
		*n_edges = h->edges.size();
	return ABB_OK;
}

int abb_overlap_get_stats(const abb_overlap* h, abb_overlap_stats* out)
{
	ABB_REQUIRE(h && out, "NULL argument");
	*out = h->st;
	return ABB_OK;
}

} // extern "C"
