// warpmap.cu — diagnostics: which hardware warp slot (%warpid) each warp of each co-resident CTA gets, for the CTA shapes the
// fused kernels use.  The sub-partition (scheduler) of a warp is %warpid % 4 on this architecture; the table tells whether two
// co-resident CTAs put their warp w on the same scheduler.   nvcc -arch=sm_90a -o warpmap warpmap.cu && ./warpmap
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <vector>

struct Rec { unsigned smid, cta, warp, warpid; };

__global__ void probe(Rec *out, unsigned long long spin) {
	extern __shared__ unsigned char smem[];
	unsigned smid, warpid;
	asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
	asm volatile("mov.u32 %0, %%warpid;" : "=r"(warpid));
	if ((threadIdx.x & 31) == 0) {
		Rec r{smid, blockIdx.x, threadIdx.x >> 5, warpid};
		out[blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)] = r;
	}
	smem[threadIdx.x] = 1;
	unsigned long long t0 = clock64();
	while (clock64() - t0 < spin) {}
}

static void run(int threads, int smem_kb, int ctas_per_sm) {
	int dev = 0, sms = 0;
	cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
	const int grid = sms * ctas_per_sm, nw = threads / 32;
	cudaFuncSetAttribute(probe, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_kb * 1024);
	Rec *d;
	cudaMalloc(&d, sizeof(Rec) * grid * nw);
	probe<<<grid, threads, smem_kb * 1024>>>(d, 2000000ull);
	cudaError_t e = cudaDeviceSynchronize();
	if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); exit(1); }
	std::vector<Rec> h(grid * nw);
	cudaMemcpy(h.data(), d, sizeof(Rec) * grid * nw, cudaMemcpyDeviceToHost);
	cudaFree(d);
	printf("== threads %d, smem %d KiB, %d CTAs/SM, grid %d\n", threads, smem_kb, ctas_per_sm, grid);
	// per SM: list CTAs with the warp slots of their warps
	for (int sm = 0; sm < 4; ++sm) {
		for (int c = 0; c < grid; ++c) {
			if (h[c * nw].smid != (unsigned)sm) continue;
			printf("  sm %d cta %3d  warpid:", sm, c);
			for (int w = 0; w < nw; ++w) printf(" %2u", h[c * nw + w].warpid);
			printf("   sched:");
			for (int w = 0; w < nw; ++w) printf(" %u", h[c * nw + w].warpid & 3);
			printf("\n");
		}
	}
	// histogram over all SMs: for warp index w of a CTA, which scheduler; and per SM the number of (cta,warp) pairs per scheduler
	std::vector<int> hist(nw * 4, 0);
	for (auto &r : h) hist[r.warp * 4 + (r.warpid & 3)]++;
	for (int w = 0; w < nw; ++w) printf("  warp %2d -> sched counts %d %d %d %d\n", w, hist[w * 4], hist[w * 4 + 1], hist[w * 4 + 2], hist[w * 4 + 3]);
	// how many SMs have both CTAs' warp 0 on the same scheduler
	std::vector<std::vector<unsigned>> w0(sms + 64);
	for (int c = 0; c < grid; ++c) w0[h[c * nw].smid].push_back(h[c * nw].warpid & 3);
	int same = 0, total = 0;
	for (auto &v : w0) if (v.size() == 2) { ++total; same += v[0] == v[1]; }
	printf("  SMs with 2 CTAs: %d, of which warp 0 of both on the same scheduler: %d\n", total, same);
}

int main() {
	run(288, 110, 2);
	run(256, 110, 2);
	run(320, 110, 2);
	run(192, 72, 3);
	run(288, 200, 1);
	return 0;
}
