// abb_konnector.cu -- the C ABI of the Konnector filter family (abb_konnector.cuh): insert and membership of the k-mers of a
// batch of reads, readBits, compare and per-level population.  abb_konnector_create lives in abb_api.cu with the other
// constructors.
#include "abb_common.h"
#include "abb_konnector.cuh"
#include <algorithm>

using namespace abb;

static KonView kon_view(const abb_filter* f)
{
	KonView v;
	v.data = f->d_data.p;
	v.bytes_per_level = f->bytes_per_level;
	v.bits = f->size;
	v.start = f->kon_start;
	v.levels = f->levels;
	v.full = make_fastmod(f->kon_full);
	v.seed = f->kon_seed;
	return v;
}

static unsigned kon_grid(uint64_t n_slots)
{
	const uint64_t tasks = (n_slots + kKonSlotsPerThread - 1) / kKonSlotsPerThread;
	return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(blocks_for(tasks, 256), sm_count() * 16));
}

namespace abb {

int kon_insert_reads_dev(abb_filter* f, const uint8_t* d_bases, const uint64_t* d_offs, uint64_t n_reads, uint64_t* n_kmers_out)
{
	if (n_kmers_out)
		*n_kmers_out = 0;
	if (n_reads == 0)
		return ABB_OK;
	uint64_t total = 0;
	ABB_CHECK(compute_slot_offsets(f->k, d_offs, n_reads, f->slot_offs, f->scan_tmp, f->stream, &total, &f->st.launches));
	if (total == 0)
		return ABB_OK;
	unsigned long long* d_count = f->d_stats.p + kStatKonKmers;
	ABB_CUDA(cudaMemsetAsync(d_count, 0, sizeof(unsigned long long), f->stream));
	ABB_CUDA(cudaEventRecord(f->ev0, f->stream));
	if (kon_words(f->k) == kKonWords)
		k_kon_walk<false, kKonWords><<<kon_grid(total), 256, 0, f->stream>>>(d_bases, d_offs, f->slot_offs.p, n_reads, total, kon_geom(f->k),
		                                                                     kon_view(f), nullptr, nullptr, d_count);
	else
		k_kon_walk<false, kKonWordsWide><<<kon_grid(total), 256, 0, f->stream>>>(d_bases, d_offs, f->slot_offs.p, n_reads, total,
		                                                                         kon_geom(f->k), kon_view(f), nullptr, nullptr, d_count);
	ABB_CUDA(cudaGetLastError());
	ABB_CUDA(cudaEventRecord(f->ev1, f->stream));
	unsigned long long n = 0;
	ABB_CUDA(cudaMemcpyAsync(&n, d_count, sizeof n, cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	float ms = 0;
	cudaEventElapsedTime(&ms, f->ev0, f->ev1);
	f->st.ms_insert += ms;
	f->st.launches += 1;
	f->st.slots += total;
	f->st.kmers += n;
	if (n_kmers_out)
		*n_kmers_out = n;
	return ABB_OK;
}

int kon_query_slots(abb_filter* f, const uint8_t* d_bases, const uint64_t* d_offs, uint64_t n_reads, uint64_t n_slots)
{
	if (kon_words(f->k) == kKonWords)
		k_kon_walk<true, kKonWords><<<kon_grid(n_slots), 256, 0, f->stream>>>(d_bases, d_offs, f->slot_offs.p, n_reads, n_slots, kon_geom(f->k),
		                                                                      kon_view(f), f->out8.p, f->valid.p, nullptr);
	else
		k_kon_walk<true, kKonWordsWide><<<kon_grid(n_slots), 256, 0, f->stream>>>(d_bases, d_offs, f->slot_offs.p, n_reads, n_slots,
		                                                                          kon_geom(f->k), kon_view(f), f->out8.p, f->valid.p, nullptr);
	f->st.launches += 1;
	ABB_CUDA(cudaGetLastError());
	return ABB_OK;
}

} // namespace abb

extern "C" {

int abb_filter_read_bits(abb_filter* f, int level, const uint8_t* host, uint64_t bits, uint64_t bit_offset, int op)
{
	ABB_REQUIRE(f, "NULL filter");
	ABB_REQUIRE(f->kind != ABB_COUNTING, "readBits applies to bit filters");
	ABB_REQUIRE(op == KON_OVERWRITE || op == KON_OR || op == KON_AND, "op must be 0 (overwrite), 1 (or) or 2 (and)");
	unsigned l = 0;
	ABB_CHECK(resolve_level(f, level, &l));
	const uint64_t size = f->bits_per_level();
	ABB_REQUIRE(bit_offset <= size && bits <= size - bit_offset, "%llu bits at bit %llu do not fit in %llu bits", (unsigned long long)bits,
	            (unsigned long long)bit_offset, (unsigned long long)size);
	if (bits == 0)
		return ABB_OK;
	ABB_REQUIRE(host, "NULL buffer");
	ABB_CUDA(cudaSetDevice(f->device));
	const uint64_t nbytes = (bits + 7) / 8;
	DevBuf<uint8_t>& src = f->sh_buf;
	ABB_CHECK(src.reserve(nbytes));
	ABB_CUDA(cudaMemcpyAsync(src.p, host, nbytes, cudaMemcpyHostToDevice, f->stream));
	const uint64_t dest_bytes = bit_offset / 8 + nbytes + 1;
	k_kon_read_bits<<<std::min<unsigned>(blocks_for(dest_bytes, 256), sm_count() * 16), 256, 0, f->stream>>>(
	    f->level_data(l), f->bytes_per_level, src.p, bits, bit_offset, op);
	f->st.launches += 1;
	ABB_CUDA(cudaGetLastError());
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	return ABB_OK;
}

int abb_filter_level_popcount(abb_filter* f, int level, uint64_t* n)
{
	ABB_REQUIRE(f && n, "NULL argument");
	ABB_REQUIRE(f->kind != ABB_COUNTING, "the level population applies to bit filters");
	unsigned l = 0;
	ABB_CHECK(resolve_level(f, level, &l));
	ABB_CUDA(cudaSetDevice(f->device));
	unsigned long long* d_n = f->d_stats.p + kStatLevelPop;
	ABB_CUDA(cudaMemsetAsync(d_n, 0, sizeof(unsigned long long), f->stream));
	k_kon_popcount<<<sm_count() * 8, 256, 0, f->stream>>>(f->level_data(l), f->bytes_per_level, d_n);
	f->st.launches += 1;
	ABB_CUDA(cudaGetLastError());
	unsigned long long h = 0;
	ABB_CUDA(cudaMemcpyAsync(&h, d_n, sizeof h, cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	*n = h;
	return ABB_OK;
}

int abb_trim_reads(abb_filter* f, const char* bases, const uint64_t* offsets, uint64_t n_reads, unsigned min_branch_len, uint32_t* left,
                   uint32_t* right)
{
	ABB_REQUIRE(f, "NULL filter");
	if (f->kind != ABB_KONNECTOR) {
		set_error("abb_trim_reads: only Konnector (-t konnector) filters have the trim graph");
		return ABB_ESTATE;
	}
	if (n_reads == 0)
		return ABB_OK;
	ABB_REQUIRE(left && right, "NULL buffer");
	ABB_CHECK(check_read_batch(bases, offsets, n_reads));
	ABB_REQUIRE(f->k >= 2, "k must be at least 2");
	for (uint64_t r = 0; r < n_reads; ++r)
		ABB_REQUIRE(offsets[r + 1] - offsets[r] < (1ULL << 31), "read %llu is too long", (unsigned long long)r);
	ABB_CUDA(cudaSetDevice(f->device));
	const bool wide = kon_words(f->k) != kKonWords;
	int per_sm = 0; // a grid that is resident all at once: the walk scratch is sized per warp of the grid
	if (wide)
		ABB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_kon_trim<kKonWordsWide>, kKonTrimThreads, 0));
	else
		ABB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_kon_trim<kKonWords>, kKonTrimThreads, 0));
	const unsigned blocks =
	    (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(blocks_for(2 * n_reads * 32, kKonTrimThreads), (uint64_t)sm_count() * std::max(per_sm, 1)));
	const uint64_t n_warps = (uint64_t)blocks * kKonTrimThreads / 32;
	DevBuf<uint8_t>& d_bases = f->trim_bases;
	DevBuf<uint64_t>& d_offs = f->trim_offs;
	DevBuf<uint32_t>& d_out = f->trim_out;
	const size_t frame_bytes = n_warps * kFrameCap * sizeof(Frame);
	ABB_CHECK(f->trim_scratch.reserve(frame_bytes + n_warps * kLookCap * sizeof(uint64_t)));
	ABB_CHECK(d_out.reserve(2 * n_reads));
	Frame* d_frames = reinterpret_cast<Frame*>(f->trim_scratch.p);
	uint64_t* d_look = reinterpret_cast<uint64_t*>(f->trim_scratch.p + frame_bytes);
	const SyncOnExit sync = { f->stream };
	ABB_CHECK(stage_read_batch(bases, offsets, n_reads, d_bases, d_offs, f->stream));
	if (wide)
		k_kon_trim<kKonWordsWide><<<blocks, kKonTrimThreads, 0, f->stream>>>(d_bases.p, d_offs.p, n_reads, kon_geom(f->k), kon_view(f),
		                                                                     min_branch_len, d_frames, d_look, d_out.p, d_out.p + n_reads);
	else
		k_kon_trim<kKonWords><<<blocks, kKonTrimThreads, 0, f->stream>>>(d_bases.p, d_offs.p, n_reads, kon_geom(f->k), kon_view(f),
		                                                                 min_branch_len, d_frames, d_look, d_out.p, d_out.p + n_reads);
	ABB_CUDA(cudaGetLastError());
	f->st.launches += 1;
	ABB_CUDA(cudaMemcpyAsync(left, d_out.p, n_reads * sizeof(uint32_t), cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaMemcpyAsync(right, d_out.p + n_reads, n_reads * sizeof(uint32_t), cudaMemcpyDeviceToHost, f->stream));
	ABB_CUDA(cudaStreamSynchronize(f->stream));
	for (uint64_t r = 0; r < n_reads; ++r)
		if (left[r] == kKonTrimFailed || right[r] == kKonTrimFailed) {
			set_error("abb_trim_reads: read %llu of the batch: the branch search outgrew its scratch (%u frames, %u visited vertices)",
			          (unsigned long long)r, kFrameCap, kLookCap);
			return ABB_ESTATE;
		}
	return ABB_OK;
}

int abb_filter_compare(abb_filter* a, abb_filter* b, uint64_t counts[4])
{
	ABB_REQUIRE(a && b && counts, "NULL argument");
	ABB_REQUIRE(a->kind != ABB_COUNTING && b->kind != ABB_COUNTING, "compare applies to bit filters");
	const uint64_t bits_a = a->bits_per_level();
	ABB_REQUIRE(bits_a == b->bits_per_level(), "Bit sizes of arrays not equal");
	ABB_REQUIRE(a->device == b->device, "the two filters are on different devices");
	ABB_CUDA(cudaSetDevice(a->device));
	ABB_CUDA(cudaStreamSynchronize(b->stream));
	unsigned long long* d_c = a->d_stats.p + kStatCompare;
	ABB_CUDA(cudaMemsetAsync(d_c, 0, 3 * sizeof(unsigned long long), a->stream));
	const uint64_t nbytes = a->bytes_per_level;
	k_kon_compare<<<std::min<unsigned>(blocks_for(nbytes, 256), sm_count() * 8), 256, 0, a->stream>>>(
	    a->level_data(a->levels - 1), b->level_data(b->levels - 1), nbytes, d_c);
	a->st.launches += 1;
	ABB_CUDA(cudaGetLastError());
	unsigned long long h[3] = { 0, 0, 0 };
	ABB_CUDA(cudaMemcpyAsync(h, d_c, sizeof h, cudaMemcpyDeviceToHost, a->stream));
	ABB_CUDA(cudaStreamSynchronize(a->stream));
	counts[0] = h[0];
	counts[1] = h[1];
	counts[2] = h[2];
	counts[3] = bits_a - h[0] - h[1] - h[2]; // the bits past the size are 0 in both
	return ABB_OK;
}

} // extern "C"
