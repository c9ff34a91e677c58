// microbench_random.cu -- what does H100 HBM deliver for the Bloom access pattern?
// Uniform-random 1-byte reads / read-modify-writes over an array much larger than L2, H per "k-mer".
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o microbench_random microbench_random.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1);} } while (0)

__device__ __forceinline__ uint64_t mix(uint64_t z) {
	z += 0x9E3779B97F4A7C15ULL; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL; return z ^ (z >> 31);
}
template <int H, int MODE, int PER>
__global__ void k(uint8_t* a, uint64_t m, uint64_t n, unsigned long long* sink) {
	uint64_t i0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * PER;
	unsigned acc = 0;
#pragma unroll
	for (int u = 0; u < PER; ++u) {
		uint64_t i = i0 + u;
		if (i >= n) break;
		uint64_t p[H]; unsigned v[H];
#pragma unroll
		for (int j = 0; j < H; ++j) p[j] = mix(i * H + j) % m;
#pragma unroll
		for (int j = 0; j < H; ++j) v[j] = __ldcg(a + p[j]);
		unsigned mn = 255;
#pragma unroll
		for (int j = 0; j < H; ++j) mn = min(mn, v[j]);
		if (MODE == 1) {
#pragma unroll
			for (int j = 0; j < H; ++j) if (v[j] == mn && mn < 255) __stcg(a + p[j], (uint8_t)(mn + 1));
		} else if (MODE == 2) {
#pragma unroll
			for (int j = 0; j < H; ++j) { unsigned* w = (unsigned*)(a + (p[j] & ~3ULL)); atomicOr(w, 1u << (p[j] & 31)); }
		}
		acc += mn;
	}
	if (acc == 0xffffffffu) *sink = acc;
}
template <int H, int MODE, int PER>
void run(const char* name, uint8_t* a, uint64_t m, uint64_t n, unsigned long long* sink) {
	cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
	unsigned grid = (unsigned)((n / PER + 255) / 256);
	k<H, MODE, PER><<<grid, 256>>>(a, m, n, sink);
	CK(cudaDeviceSynchronize());
	float best = 1e9;
	for (int it = 0; it < 3; ++it) {
		CK(cudaEventRecord(e0)); k<H, MODE, PER><<<grid, 256>>>(a, m, n, sink); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
		float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
	}
	double kps = n / (best * 1e-3);
	printf("%-28s H=%d per=%d  %8.3f ms  %7.2f G kmers/s  sector-bytes %7.1f GB/s (rd%s)\n", name, H, PER, best, kps / 1e9,
	       kps * H * 32 * (MODE ? 2 : 1) / 1e9, MODE ? "+wr" : "");
}
int main(int argc, char** argv) {
	uint64_t m = argc > 1 ? strtoull(argv[1], 0, 10) : 7635497472ULL;
	uint64_t n = argc > 2 ? strtoull(argv[2], 0, 10) : (1ULL << 28);
	uint8_t* a; unsigned long long* sink;
	if (const char* env = getenv("L2FETCH")) // cudaLimitMaxL2FetchGranularity: 32, 64 or 128
		CK(cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)atoi(env)));
	size_t gran = 0;
	CK(cudaDeviceGetLimit(&gran, cudaLimitMaxL2FetchGranularity));
	printf("cudaLimitMaxL2FetchGranularity = %zu\n", gran);
	CK(cudaMalloc(&a, m)); CK(cudaMemset(a, 0, m)); CK(cudaMalloc(&sink, 8));
	printf("array %.2f GB, %llu k-mers per launch\n", m / 1e9, (unsigned long long)n);
	run<4, 0, 1>("read-only", a, m, n, sink);
	run<4, 0, 4>("read-only", a, m, n, sink);
	run<4, 1, 1>("min-increment (plain st)", a, m, n, sink);
	run<4, 1, 4>("min-increment (plain st)", a, m, n, sink);
	run<4, 2, 1>("atomicOr bit set", a, m, n, sink);
	run<4, 2, 4>("atomicOr bit set", a, m, n, sink);
	// L2-resident table for comparison (64 MB)
	run<4, 0, 4>("read-only 64MB (L2)", a, 64ULL << 20, n, sink);
	run<4, 1, 4>("min-inc 64MB (L2)", a, 64ULL << 20, n, sink);
	return 0;
}
