// microbench_sorted.cu -- does ordering the Bloom counter accesses by address lift the random-access
// ceiling of H100 HBM?  N byte accesses over a 7.6 GB
// array: in random order, fully sorted by address, and sorted only down to bins (random inside a bin).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o microbench_sorted microbench_sorted.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1);} } while (0)

__device__ __forceinline__ uint64_t mix(uint64_t z) {
	z += 0x9E3779B97F4A7C15ULL; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL; return z ^ (z >> 31);
}
__global__ void k_fill(uint8_t* a, uint64_t m) {
	for (uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * 16; i < m; i += (uint64_t)gridDim.x * blockDim.x * 16) {
		uint64_t x = mix(i), y = mix(i + 7);
		if (i + 16 <= m) *reinterpret_cast<uint4*>(a + i) = make_uint4((unsigned)x & 0x3f3f3f3f, (unsigned)(x >> 32) & 0x3f3f3f3f, (unsigned)y & 0x3f3f3f3f, (unsigned)(y >> 32) & 0x3f3f3f3f);
	}
}
__global__ void k_gen(uint64_t* p, uint64_t n, uint64_t m, uint64_t salt) {
	uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) p[i] = mix(i ^ (salt << 40)) % m;
}
/** permute inside blocks of `blk` elements (blk a power of two): bin-sorted order */
__global__ void k_shuffle(const uint64_t* in, uint64_t* out, uint64_t n, uint64_t blk) {
	uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	uint64_t b = i & ~(blk - 1), o = i & (blk - 1);
	// odd multiplier + xor = bijection on [0, blk)
	uint64_t q = ((o * 0x9E3779B1ULL) ^ (b >> 3)) & (blk - 1);
	q = (q ^ (q >> 7)) & (blk - 1);
	out[b + q] = in[i]; // not a bijection after the second xor-shift? (x ^ x>>7 is a bijection) ok
}
template <int MODE, int PER>
__global__ void __launch_bounds__(256) k_access(uint8_t* a, const uint64_t* __restrict__ p, uint64_t n, uint8_t* __restrict__ out) {
	// thread t of the grid handles records t, t + T, ... (consecutive threads = consecutive records)
	const uint64_t T = (uint64_t)gridDim.x * blockDim.x;
	uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	uint64_t q[PER]; unsigned v[PER];
#pragma unroll
	for (int u = 0; u < PER; ++u) q[u] = i + u * T < n ? p[i + u * T] : 0;
#pragma unroll
	for (int u = 0; u < PER; ++u) v[u] = __ldcg(a + q[u]);
#pragma unroll
	for (int u = 0; u < PER; ++u) {
		if (i + u * T >= n) break;
		if (MODE == 0) out[i + u * T] = (uint8_t)v[u];
		else if (MODE == 1) { if (v[u] & 1) __stcg(a + q[u], (uint8_t)(v[u] + 1)); } // ~half of the accesses write back
		else __stcg(a + q[u], (uint8_t)(v[u] + 1));
	}
}
/** store-only (the update sweep when the values are already known) */
__global__ void __launch_bounds__(256) k_store(uint8_t* a, const uint64_t* __restrict__ p, uint64_t n, const uint8_t* __restrict__ val) {
	uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) { unsigned v = val[i]; if (v & 1) __stcg(a + p[i], (uint8_t)(v + 1)); }
}
template <int MODE, int PER>
float run(uint8_t* a, const uint64_t* p, uint64_t n, uint8_t* out) {
	cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
	unsigned grid = (unsigned)((n / PER + 255) / 256);
	float best = 1e9;
	for (int it = 0; it < 3; ++it) {
		CK(cudaEventRecord(e0)); k_access<MODE, PER><<<grid, 256>>>(a, p, n, out); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
		float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
	}
	CK(cudaGetLastError());
	return best;
}
float run_store(uint8_t* a, const uint64_t* p, uint64_t n, uint8_t* val) {
	cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
	float best = 1e9;
	for (int it = 0; it < 3; ++it) {
		CK(cudaEventRecord(e0)); k_store<<<(unsigned)((n + 255) / 256), 256>>>(a, p, n, val); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
		float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
	}
	return best;
}
void report(const char* order, uint64_t n, uint8_t* a, const uint64_t* p, uint8_t* out) {
	float g1 = run<0, 1>(a, p, n, out), g4 = run<0, 4>(a, p, n, out);
	float h4 = run<1, 4>(a, p, n, out), w4 = run<2, 4>(a, p, n, out);
	float st = run_store(a, p, n, out);
	printf("%-22s n=2^%2d  gather %7.3f ms (%6.1f G/s) per4 %7.3f ms (%6.1f G/s) | rmw50%% %7.3f ms (%6.1f G/s) | rmw100%% %7.3f ms (%6.1f G/s) | store50%% %7.3f ms (%6.1f G/s)\n",
	       order, (int)(63 - __builtin_clzll(n)), g1, n / g1 / 1e6, g4, n / g4 / 1e6, h4, n / h4 / 1e6, w4, n / w4 / 1e6, st, n / st / 1e6);
	fflush(stdout);
}
int main(int argc, char** argv) {
	uint64_t m = argc > 1 ? strtoull(argv[1], 0, 10) : 7635497472ULL;
	if (const char* env = getenv("L2FETCH"))
		CK(cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)atoi(env)));
	size_t gran = 0;
	CK(cudaDeviceGetLimit(&gran, cudaLimitMaxL2FetchGranularity));
	printf("cudaLimitMaxL2FetchGranularity = %zu, array %.2f GB\n", gran, m / 1e9);
	uint8_t *a, *out; uint64_t *p, *ps, *pb; void* tmp = nullptr; size_t tmp_bytes = 0;
	const uint64_t nmax = 1ULL << 27;
	CK(cudaMalloc(&a, m)); CK(cudaMalloc(&out, nmax)); CK(cudaMalloc(&p, nmax * 8)); CK(cudaMalloc(&ps, nmax * 8)); CK(cudaMalloc(&pb, nmax * 8));
	k_fill<<<132 * 16, 256>>>(a, m); CK(cudaDeviceSynchronize());
	cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, p, ps, (int)nmax);
	CK(cudaMalloc(&tmp, tmp_bytes));
	for (int lg = 21; lg <= 27; lg += 2) {
		uint64_t n = 1ULL << lg;
		k_gen<<<(unsigned)((n + 255) / 256), 256>>>(p, n, m, lg);
		CK(cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, p, ps, (int)n));
		CK(cudaDeviceSynchronize());
		report("random", n, a, p, out);
		report("sorted", n, a, ps, out);
		for (uint64_t blk = 1 << 10; blk <= (1 << 16) && blk < n; blk <<= 3) {
			k_shuffle<<<(unsigned)((n + 255) / 256), 256>>>(ps, pb, n, blk);
			CK(cudaDeviceSynchronize());
			char name[64]; snprintf(name, sizeof name, "bins of %llu", (unsigned long long)blk);
			report(name, n, a, pb, out);
		}
	}
	return 0;
}
