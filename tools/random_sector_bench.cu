// How fast can this device serve dependent random 32-byte sector reads — the access pattern of FM-index seeding (every backward
// extension reads the rank blocks its previous result names)?  Each thread walks M independent chains of random 32-B reads over a
// table of the given size; the sweep over resident warps and chains per thread gives the ceiling `k_smem_bwd` is to be held against
// (bench.py's `roofline.peak` stays the data-sheet HBM bandwidth).  Each 32-B sector is read with two 128-bit loads, as
// load_blk32() in ssq_dev.cuh does on sm_90.
// build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/random_sector_bench tools/random_sector_bench.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

__device__ __forceinline__ uint32_t ld32B(const void *p)
{
	uint32_t a, b, c, d, e, f, g, h;
	asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8];\n\tld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d), "=r"(e), "=r"(f), "=r"(g), "=r"(h) : "l"(p));
	return a ^ b ^ c ^ d ^ e ^ f ^ g ^ h;
}
__device__ __forceinline__ uint64_t mix(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; return x ^ (x >> 33); }

template<int M> __global__ void k_chase(const uint8_t *tab, uint64_t n_sect, int iters, uint32_t *sink)
{
	uint64_t x[M];
	const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
#pragma unroll
	for (int m = 0; m < M; ++m) x[m] = mix(t * M + m + 1);
	for (int i = 0; i < iters; ++i) {
		uint32_t v[M];
#pragma unroll
		for (int m = 0; m < M; ++m) v[m] = ld32B(tab + (x[m] % n_sect) * 32);
#pragma unroll
		for (int m = 0; m < M; ++m) x[m] = mix(x[m] + v[m]);
	}
	uint64_t s = 0;
#pragma unroll
	for (int m = 0; m < M; ++m) s ^= x[m];
	if (s == 0x1234567) sink[0] = 1;
}
__global__ void k_fill(uint64_t *p, size_t n) { for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = mix(i + 7); }

template<int M> static double run(const uint8_t *tab, uint64_t n_sect, int blocks, int threads, int iters, uint32_t *sink)
{
	cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
	k_chase<M><<<blocks, threads>>>(tab, n_sect, iters / 8, sink);
	CK(cudaEventRecord(a)); k_chase<M><<<blocks, threads>>>(tab, n_sect, iters, sink); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
	float ms; CK(cudaEventElapsedTime(&ms, a, b));
	return (double)blocks * threads * M * iters * 32 / (ms * 1e-3) / 1e9;
}

int main(int argc, char **argv)
{
	int n_sm; CK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, 0));
	uint32_t *sink; CK(cudaMalloc(&sink, 4));
	const double sizes_gb[] = {0.064, 1.0, 4.0};
	printf("# random dependent 32-B sector reads, GB/s (sectors x 32 B / time); %d SMs\n# table_GB warps/SM chains/thread GB/s\n", n_sm);
	for (double gb : sizes_gb) {
		const size_t bytes = (size_t)(gb * (1ull << 30)) & ~(size_t)31;
		uint8_t *tab; CK(cudaMalloc(&tab, bytes));
		k_fill<<<n_sm * 8, 256>>>((uint64_t*)tab, bytes / 8); CK(cudaDeviceSynchronize());
		double best = 0; int bw = 0, bm = 0;
		for (int wps : {8, 16, 24, 32, 48, 64}) {
			const int threads = 256, blocks = n_sm * wps * 32 / threads, iters = 512;
			const double r1 = run<1>(tab, bytes / 32, blocks, threads, iters, sink), r2 = run<2>(tab, bytes / 32, blocks, threads, iters, sink), r4 = run<4>(tab, bytes / 32, blocks, threads, iters / 2, sink);
			printf("%.3f %d 1 %.0f\n%.3f %d 2 %.0f\n%.3f %d 4 %.0f\n", gb, wps, r1, gb, wps, r2, gb, wps, r4);
			if (r1 > best) best = r1, bw = wps, bm = 1;
			if (r2 > best) best = r2, bw = wps, bm = 2;
			if (r4 > best) best = r4, bw = wps, bm = 4;
		}
		printf("# table %.3f GB: best %.0f GB/s at %d warps/SM, %d chains/thread\n", gb, best, bw, bm);
		CK(cudaFree(tab));
	}
	return 0;
}
