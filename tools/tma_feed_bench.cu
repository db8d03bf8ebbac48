/* tma_feed_bench.cu -- how fast can cp.async.bulk row segments feed an SM?
 * The fused thumbnail kernel's access pattern without its arithmetic: every CTA owns a
 * band of COLS pixel columns of one 4096x4096 RGBA frame and streams it top to bottom,
 * ROWS rows per stage through an S-deep mbarrier ring; consumer warps only touch one word
 * per row and release the stage.  Prints GB/s for a sweep of (COLS, ROWS, S, CTAs/SM).
 *   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tma_feed_bench tma_feed_bench.cu
 *
 * `tma_feed_bench headline FRAMES BOXW NBOX HINT c_lo...` copies the feed of the headline thumbnail kernel instead:
 * one CTA per SM, one band per blockIdx.x at input column c_lo (as many bands as c_lo values), frames on blockIdx.z,
 * stages of 8 rows (2 VS, VS = 4) in a 4-deep ring, each stage row NBOX tiled-TMA boxes of BOXW pixels.  HINT 0 loads
 * every box with the default L2 policy; 1 loads the boxes that no neighbouring band reads (all but a band's first and
 * last, bands 0 and n - 1 have one seam) with an evict_first policy; 2 adds evict_last on the seam boxes; 3 loads
 * every box with evict_first.  Prints
 * algorithmic GB/s: FRAMES x 4096 x 4096 x 4 bytes over the kernel time.
 */
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>

__device__ __forceinline__ unsigned smem_addr(const void *p) { return (unsigned) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity)
{
	unsigned done;
	do {
		asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
	} while (!done);
}
__device__ __forceinline__ void mbar_arrive(unsigned bar) { asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) { asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void bulk_copy_g2s(unsigned dst, const void *src, unsigned bytes, unsigned bar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

template <int MODE, int ROWS>
__global__ void feed(const uint8_t *in, int W, int H, int cols, int rows_, int S, int nwarps, unsigned *sink)
{
	extern __shared__ __align__(128) unsigned char smem[];
	const int rows = ROWS;
	const unsigned pitch = cols * 4;
	const unsigned stage_bytes = rows * pitch;
	uint64_t *bars = (uint64_t *) (smem + (size_t) S * stage_bytes);
	const unsigned full_s = smem_addr(bars), empty_s = full_s + 8u * S, stages_s = smem_addr(smem);
	const int t = threadIdx.x;
	if (t == 0) {
		for (int i = 0; i < S; i++) {
			mbar_init(full_s + 8u * i, 1);
			mbar_init(empty_s + 8u * i, nwarps);
		}
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();
	const uint8_t *fin = in + (size_t) blockIdx.y * W * H * 4 + (size_t) blockIdx.x * cols * 4;
	const int nst = H / rows;
	if (t >= nwarps * 32) {
		const int lane = t - nwarps * 32;
		int s = 0;
		unsigned phase = 0;
		for (int p = 0; p < nst; p++) {
			mbar_wait(empty_s + 8u * s, phase ^ 1u);
			if (lane == 0)
				mbar_expect_tx(full_s + 8u * s, stage_bytes);
			__syncwarp();
			if (MODE == 0) {
				if (lane < rows)
					bulk_copy_g2s(stages_s + s * stage_bytes + lane * pitch, fin + (size_t) (p * rows + lane) * W * 4, pitch, full_s + 8u * s);
			}
			else {
				/* warp-uniform addresses, one elected lane issues: the copies stay in the uniform datapath */
				unsigned pred;
				asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
				if (pred) {
#pragma unroll
					for (int r = 0; r < ROWS; r++)
						bulk_copy_g2s(stages_s + s * stage_bytes + r * pitch, fin + (size_t) (p * rows + r) * W * 4, pitch, full_s + 8u * s);
				}
			}
			if (++s == S) {
				s = 0;
				phase ^= 1u;
			}
		}
		return;
	}
	int s = 0;
	unsigned phase = 0, acc = 0;
	for (int p = 0; p < nst; p++) {
		mbar_wait(full_s + 8u * s, phase);
		for (int r = 0; r < rows; r++)
			acc += *(const unsigned *) (smem + (size_t) s * stage_bytes + r * pitch + (t % cols) * 4);
		__syncwarp();
		if ((t & 31) == 0)
			mbar_arrive(empty_s + 8u * s);
		if (++s == S) {
			s = 0;
			phase ^= 1u;
		}
	}
	if (acc == 0x12345678u)
		sink[0] = acc;
}

__global__ void __launch_bounds__(160, 1)
feed_headline(const __grid_constant__ CUtensorMap tm, int H, const int *c_lo, int boxw, int nbox, int hint, unsigned *sink)
{
	extern __shared__ __align__(128) unsigned char smem[];
	constexpr int S = 4, ROWS = 8, NW = 4;
	const unsigned box_bytes = ((unsigned) ROWS * boxw * 4 + 127u) & ~127u;
	const unsigned stage_bytes = nbox * box_bytes;
	uint64_t *bars = (uint64_t *) (smem + (size_t) S * stage_bytes);
	const unsigned full_s = smem_addr(bars), empty_s = full_s + 8u * S, stages_s = smem_addr(smem);
	const int t = threadIdx.x;
	if (t == 0) {
		for (int i = 0; i < S; i++) {
			mbar_init(full_s + 8u * i, 1);
			mbar_init(empty_s + 8u * i, NW);
		}
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();
	const int nst = H / ROWS;
	if (t >= NW * 32) {
		if (t != NW * 32)
			return;
		const int c0 = c_lo[blockIdx.x], band = blockIdx.x, nb = gridDim.x;
		uint64_t pol_first, pol_last;
		asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_first));
		asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol_last));
		int s = 0;
		unsigned phase = 0;
		for (int p = 0; p < nst; p++) {
			mbar_wait(empty_s + 8u * s, phase ^ 1u);
			mbar_expect_tx(full_s + 8u * s, (unsigned) nbox * ROWS * boxw * 4);
			for (int h = 0; h < nbox; h++) {
				const unsigned dst = stages_s + s * stage_bytes + h * box_bytes, bar = full_s + 8u * s;
				const int x = (c0 + h * boxw) >> 1, y = p * ROWS, z = blockIdx.z;
				const bool seam = (h == 0 && band > 0) || (h == nbox - 1 && band < nb - 1);
				if (hint == 0 || (seam && hint == 1))
					asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
								 ::"r"(dst), "l"(&tm), "r"(x), "r"(y), "r"(z), "r"(bar) : "memory");
				else
					asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3, %4}], [%5], %6;"
								 ::"r"(dst), "l"(&tm), "r"(x), "r"(y), "r"(z), "r"(bar), "l"(seam && hint == 2 ? pol_last : pol_first) : "memory");
			}
			if (++s == S) {
				s = 0;
				phase ^= 1u;
			}
		}
		return;
	}
	int s = 0;
	unsigned phase = 0, acc = 0;
	for (int p = 0; p < nst; p++) {
		mbar_wait(full_s + 8u * s, phase);
		for (int r = 0; r < ROWS; r++)
			acc += *(const unsigned *) (smem + (size_t) s * stage_bytes + (t % nbox) * box_bytes + r * boxw * 4 + (t % boxw) * 4);
		__syncwarp();
		if ((t & 31) == 0)
			mbar_arrive(empty_s + 8u * s);
		if (++s == S) {
			s = 0;
			phase ^= 1u;
		}
	}
	if (acc == 0x12345678u)
		sink[0] = acc;
}

static int headline(int argc, char **argv)
{
	const int W = 4096, H = 4096, frames = atoi(argv[2]), boxw = atoi(argv[3]), nbox = atoi(argv[4]), hint = atoi(argv[5]);
	const int nb = argc - 6;
	int c_lo[64];
	for (int b = 0; b < nb && b < 64; b++)
		c_lo[b] = atoi(argv[6 + b]);
	typedef CUresult (*encode_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
		const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
	void *fn = nullptr;
	cudaDriverEntryPointQueryResult q;
	if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn)
		return fprintf(stderr, "no cuTensorMapEncodeTiled\n"), 1;
	uint8_t *in;
	int *d_clo;
	unsigned *sink;
	if (cudaMalloc(&in, (size_t) frames * W * H * 4) != cudaSuccess)
		return fprintf(stderr, "cudaMalloc failed\n"), 1;
	cudaMemset(in, 1, (size_t) frames * W * H * 4);
	cudaMalloc(&d_clo, sizeof(c_lo));
	cudaMemcpy(d_clo, c_lo, sizeof(c_lo), cudaMemcpyHostToDevice);
	cudaMalloc(&sink, 4);
	CUtensorMap tm;
	const cuuint64_t dims[3] = {(cuuint64_t) W / 2, (cuuint64_t) H, (cuuint64_t) frames};
	const cuuint64_t strides[2] = {(cuuint64_t) W * 4, (cuuint64_t) W * H * 4};
	const cuuint32_t box[3] = {(cuuint32_t) boxw / 2, 8, 1}, estr[3] = {1, 1, 1};
	if (((encode_fn) fn)(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT64, 3, in, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
			CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
		return fprintf(stderr, "tensor map rejected\n"), 1;
	const size_t smem = (size_t) 4 * nbox * (((size_t) 8 * boxw * 4 + 127) & ~(size_t) 127) + 64;
	const size_t use = smem > 120 * 1024 ? smem : 120 * 1024; /* one CTA per SM, as the kernel */
	cudaFuncSetAttribute(feed_headline, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) use);
	cudaEvent_t e0, e1;
	cudaEventCreate(&e0);
	cudaEventCreate(&e1);
	float best = 1e9f, sum = 0;
	const int reps = 4;
	for (int it = 0; it <= reps; it++) {
		cudaEventRecord(e0);
		feed_headline<<<dim3(nb, 1, frames), 160, use>>>(tm, H, d_clo, boxw, nbox, hint, sink);
		cudaEventRecord(e1);
		cudaEventSynchronize(e1);
		float ms;
		cudaEventElapsedTime(&ms, e0, e1);
		if (it > 0) {
			best = ms < best ? ms : best;
			sum += ms;
		}
	}
	cudaError_t e = cudaGetLastError();
	printf("headline frames %d bands %d box %dx%d hint %d: loaded %d cols/frame  best %.2f ms  mean %.2f ms  %.1f GB/s algorithmic %s\n",
		frames, nb, nbox, boxw, hint, nb * nbox * boxw, best, sum / reps, (double) frames * W * H * 4 / best / 1e6,
		e == cudaSuccess ? "" : cudaGetErrorString(e));
	return e != cudaSuccess;
}

int main(int argc, char **argv)
{
	if (argc > 6 && !strcmp(argv[1], "headline"))
		return headline(argc, argv);
	const int W = 4096, H = 4096, frames = argc > 1 ? atoi(argv[1]) : 64;
	uint8_t *in;
	unsigned *sink;
	cudaMalloc(&in, (size_t) frames * W * H * 4);
	cudaMemset(in, 1, (size_t) frames * W * H * 4);
	cudaMalloc(&sink, 4);
	cudaEvent_t e0, e1;
	cudaEventCreate(&e0);
	cudaEventCreate(&e1);
	const int colsv[] = {256, 384, 512, 1024};
	const int rowsv[] = {8};
	const int Sv[] = {2, 3, 4, 6, 8};
	const int persm[] = {1, 2, 3, 4};
	for (int cols : colsv)
		for (int rows : rowsv)
			for (int S : Sv)
				for (int per : persm) for (int mode = 0; mode < 2; mode++) {
					size_t smem = (size_t) S * rows * cols * 4 + 2 * S * 8 + 64;
					size_t budget = (size_t) 227 * 1024 / per - 1024;
					if (smem > budget)
						continue;
					/* pad so that exactly `per` CTAs fit */
					size_t pad = per < 4 ? (size_t) 227 * 1024 / (per + 1) : 0;
					size_t use = smem > pad ? smem : pad;
					if (use > budget)
						use = budget;
					auto kern = mode ? feed<1, 8> : feed<0, 8>;
					cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) use);
					const int nwarps = 4;
					dim3 grid(W / cols, frames);
					float best = 1e9f;
					for (int it = 0; it < 3; it++) {
						cudaEventRecord(e0);
						kern<<<grid, (nwarps + 1) * 32, use>>>(in, W, H, cols, rows, S, nwarps, sink);
						cudaEventRecord(e1);
						cudaEventSynchronize(e1);
						float ms;
						cudaEventElapsedTime(&ms, e0, e1);
						if (it > 0 && ms < best)
							best = ms;
					}
					cudaError_t e = cudaGetLastError();
					printf("mode %d cols %4d rows %2d S %d ctas/sm %d  in-flight/SM %6.1f KB  %7.1f GB/s %s\n", mode, cols, rows, S, per,
						per * (double) S * rows * cols * 4 / 1024, (double) frames * (W / cols * cols) * H * 4 / best / 1e6,
						e == cudaSuccess ? "" : cudaGetErrorString(e));
				}
	return 0;
}
