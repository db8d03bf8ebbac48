/* warp_slots.cu -- which hardware warp slot (%warpid) does warp w of a CTA get when two
 * 8-warp CTAs with ~107 KB of shared memory share an SM?  (sub-partition = %warpid % 4) */
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k(int *out, int spin)
{
	extern __shared__ int sm[];
	unsigned smid, wid;
	asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
	asm volatile("mov.u32 %0, %%warpid;" : "=r"(wid));
	if ((threadIdx.x & 31) == 0) {
		int *o = out + (blockIdx.x * 8 + threadIdx.x / 32) * 2;
		o[0] = smid;
		o[1] = wid;
	}
	long long t0 = clock64();
	while (clock64() - t0 < spin)
		;
	sm[threadIdx.x] = 0;
}
int main()
{
	int n = 132 * 2 * 3; /* H100: 132 SMs */
	int *d, *h = new int[n * 16];
	cudaMalloc(&d, n * 16 * 4);
	cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 107 * 1024);
	k<<<n, 256, 107 * 1024>>>(d, 200000);
	cudaMemcpy(h, d, n * 16 * 4, cudaMemcpyDeviceToHost);
	for (int b = 0; b < n; b++) {
		if (h[b * 16] > 1)
			continue;
		printf("cta %4d sm %3d warpids:", b, h[b * 16]);
		for (int w = 0; w < 8; w++)
			printf(" %2d", h[b * 16 + w * 2 + 1]);
		printf("\n");
	}
	return 0;
}
