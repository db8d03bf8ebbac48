/* resample_kernels.cu -- leaf resample kernels (one per reference generate
 * function) for every real band format except double, on device-resident
 * images.  The headline uchar RGBA thumbnail chain has its own fused kernel
 * (thumbnail_fused.cu); these are the general-format / general-band path and
 * the building blocks of vb200_resize().
 *
 * reference arithmetic:
 *   shrinkv   resample/shrinkv.c:158-266   (ADD, UCHAR_AVG, USHORT_AVG, IAVG, FAVG)
 *   shrinkh   resample/shrinkh.c:78-152    (UCHAR_SHRINK, USHORT_SHRINK, ISHRINK, FSHRINK)
 *   reducev   resample/reducev.cpp:420-496 (reducev_block + *_tab finalizers)
 *   reduceh   resample/reduceh.cpp:145-193 (reduce_sum per band + finalizers)
 *   pre/unpre conversion/premultiply.c:86-166, unpremultiply.c:85-222
 * Edge pixels: every vips_embed(..., EXTEND_COPY) in front of these ops
 * (conversion/embed.c:300-336) is clamp addressing here.
 *
 * Float paths accumulate in double with explicit round-to-nearest mul/add
 * (__dmul_rn/__dadd_rn) so nvcc cannot contract them into FMAs: the reference
 * build (x86-64 baseline) has none.
 */
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <utility>
#include <vector>

#include "vb200_internal.h"

namespace vb200 {

namespace {

template <typename T> struct Acc { typedef int type; };
template <> struct Acc<uint32_t> { typedef long long type; };
template <> struct Acc<int32_t> { typedef long long type; };
template <> struct Acc<float> { typedef double type; };

template <typename T> struct Limits;
template <> struct Limits<uint8_t> { static constexpr long long lo = 0, hi = 255; static constexpr bool sgn = false; };
template <> struct Limits<int8_t> { static constexpr long long lo = -128, hi = 127; static constexpr bool sgn = true; };
template <> struct Limits<uint16_t> { static constexpr long long lo = 0, hi = 65535; static constexpr bool sgn = false; };
template <> struct Limits<int16_t> { static constexpr long long lo = -32768, hi = 32767; static constexpr bool sgn = true; };
template <> struct Limits<uint32_t> { static constexpr long long lo = 0, hi = 4294967295LL; static constexpr bool sgn = false; };
template <> struct Limits<int32_t> { static constexpr long long lo = -2147483648LL, hi = 2147483647LL; static constexpr bool sgn = true; };

__device__ __forceinline__ int
clampi(int v, int lo, int hi)
{
	return max(lo, min(v, hi));
}

/* unsigned_fixed_round / signed_fixed_round + VIPS_CLIP, templates.h:150-210 */
template <typename T, typename IT>
__device__ __forceinline__ T
fixed_finalize(IT sum)
{
	IT v;
	if (Limits<T>::sgn) {
		const int round_by = sum >= 0 ? (VB200_INTERPOLATE_SCALE >> 1) : -(VB200_INTERPOLATE_SCALE >> 1);
		v = (sum + round_by) >> VB200_INTERPOLATE_SHIFT;
	}
	else
		v = (sum + (VB200_INTERPOLATE_SCALE >> 1)) >> VB200_INTERPOLATE_SHIFT;
	long long w = v;
	w = w < Limits<T>::lo ? Limits<T>::lo : (w > Limits<T>::hi ? Limits<T>::hi : w);
	return (T) w;
}

/* ------------------------------------------------------------------ shrinkv */

template <typename T>
__global__ void __launch_bounds__(256)
shrinkv_kernel(const T *__restrict__ in, size_t in_bpl, int in_h, T *__restrict__ out, size_t out_bpl, int out_h,
	int ne, int vshrink, unsigned int mult8, unsigned long long mult16)
{
	typedef typename Acc<T>::type ACC;
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= ne)
		return;

	const char *base = (const char *) in;
	for (int y = blockIdx.y; y < out_h; y += gridDim.y) {
		ACC sum = 0;
		for (int k = 0; k < vshrink; k++) {
			const int row = min(y * vshrink + k, in_h - 1);
			const T v = ((const T *) (base + (size_t) row * in_bpl))[x];
			sum += (ACC) v;
		}

		T *q = (T *) ((char *) out + (size_t) y * out_bpl) + x;
		const int amend = vshrink / 2;
		if constexpr (sizeof(T) == 1 && !Limits<T>::sgn)
			*q = (T) ((((unsigned int) ((int) sum + amend)) * mult8) >> 24);
		else if constexpr (sizeof(T) == 2 && !Limits<T>::sgn)
			*q = (T) (((unsigned long long) ((int) sum + amend) * mult16) >> 32);
		else
			*q = (T) ((sum + (ACC) amend) / (ACC) vshrink);
	}
}

template <>
__global__ void __launch_bounds__(256)
shrinkv_kernel<float>(const float *__restrict__ in, size_t in_bpl, int in_h, float *__restrict__ out, size_t out_bpl,
	int out_h, int ne, int vshrink, unsigned int, unsigned long long)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= ne)
		return;
	const char *base = (const char *) in;
	for (int y = blockIdx.y; y < out_h; y += gridDim.y) {
		double sum = 0.0;
		for (int k = 0; k < vshrink; k++) {
			const int row = min(y * vshrink + k, in_h - 1);
			sum = __dadd_rn(sum, (double) ((const float *) (base + (size_t) row * in_bpl))[x]);
		}
		const double inv = 1.0 / vshrink;
		((float *) ((char *) out + (size_t) y * out_bpl))[x] = (float) __dmul_rn(sum, inv);
	}
}

/* uchar, 4 elements per thread: one 32-bit load per row, two 16-bit lanes per
 * accumulator word (a lane holds at most 255 * vshrink <= 65535).
 */
__global__ void __launch_bounds__(256)
shrinkv_u8x4_kernel(const uint8_t *__restrict__ in, size_t in_bpl, int in_h, uint8_t *__restrict__ out,
	size_t out_bpl, int out_h, int nwords, int vshrink, unsigned int mult8)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= nwords)
		return;
	for (int y = blockIdx.y; y < out_h; y += gridDim.y) {
		unsigned int lo = 0, hi = 0; /* bytes 0,2 and bytes 1,3 */
		for (int k = 0; k < vshrink; k++) {
			const int row = min(y * vshrink + k, in_h - 1);
			const unsigned int v = __ldg((const unsigned int *) (in + (size_t) row * in_bpl) + x);
			lo += v & 0x00ff00ffu;
			hi += (v >> 8) & 0x00ff00ffu;
		}
		const unsigned int amend = vshrink / 2;
		const unsigned int b0 = (((lo & 0xffffu) + amend) * mult8) >> 24;
		const unsigned int b2 = (((lo >> 16) + amend) * mult8) >> 24;
		const unsigned int b1 = (((hi & 0xffffu) + amend) * mult8) >> 24;
		const unsigned int b3 = (((hi >> 16) + amend) * mult8) >> 24;
		((unsigned int *) (out + (size_t) y * out_bpl))[x] = (b0 & 0xff) | ((b1 & 0xff) << 8) | ((b2 & 0xff) << 16) | (b3 << 24);
	}
}

/* ------------------------------------------------------------------ shrinkh */

template <typename T>
__global__ void __launch_bounds__(256)
shrinkh_kernel(const T *__restrict__ in, size_t in_bpl, int in_w, T *__restrict__ out, size_t out_bpl, int out_w,
	int bands, int rows, int hshrink, unsigned int mult8, unsigned long long mult16)
{
	typedef typename Acc<T>::type ACC;
	const int e = blockIdx.x * blockDim.x + threadIdx.x; /* output element on the row */
	if (e >= out_w * bands)
		return;
	const int x = e / bands;
	const int b = e - x * bands;
	const int amend = hshrink / 2;
	for (int y = blockIdx.y; y < rows; y += gridDim.y) {
		const T *p = (const T *) ((const char *) in + (size_t) y * in_bpl);
		T *q = (T *) ((char *) out + (size_t) y * out_bpl) + e;

		if constexpr (sizeof(T) <= 2) {
			int sum = amend;
			for (int k = 0; k < hshrink; k++)
				sum += p[(size_t) min(x * hshrink + k, in_w - 1) * bands + b];
			if constexpr (sizeof(T) == 1 && !Limits<T>::sgn)
				*q = (T) (((unsigned int) sum * mult8) >> 24);
			else if constexpr (sizeof(T) == 2 && !Limits<T>::sgn)
				*q = (T) (((unsigned long long) sum * mult16) >> 32);
			else
				*q = (T) (sum / hshrink);
		}
		else {
			long long sum = amend;
			for (int k = 0; k < hshrink; k++)
				sum += p[(size_t) min(x * hshrink + k, in_w - 1) * bands + b];
			*q = (T) (sum / hshrink);
		}
	}
}

template <>
__global__ void __launch_bounds__(256)
shrinkh_kernel<float>(const float *__restrict__ in, size_t in_bpl, int in_w, float *__restrict__ out, size_t out_bpl,
	int out_w, int bands, int rows, int hshrink, unsigned int, unsigned long long)
{
	const int e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= out_w * bands)
		return;
	const int x = e / bands;
	const int b = e - x * bands;
	for (int y = blockIdx.y; y < rows; y += gridDim.y) {
		const float *p = (const float *) ((const char *) in + (size_t) y * in_bpl);
		double sum = 0.0;
		for (int k = 0; k < hshrink; k++)
			sum = __dadd_rn(sum, (double) p[(size_t) min(x * hshrink + k, in_w - 1) * bands + b]);
		const double inv = 1.0 / hshrink;
		((float *) ((char *) out + (size_t) y * out_bpl))[e] = (float) __dmul_rn(sum, inv);
	}
}

/* ------------------------------------------------------------------ reducev */

struct AxisDev {
	const int *first;
	const int *phase;
	const short *ms;
	const double *mf;
	const unsigned *mp; /* [65][npairs] s16 x 2: taps (2k, 2k + 1) of each phase, the odd tail paired with 0 (dp2a kernels) */
	int n_point;
	int embed;
	int npairs; /* (n_point + 1) / 2 */
};

__device__ __forceinline__ int
dp2a_lo_(unsigned coef, unsigned bytes, int acc)
{
	int d;
	asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(coef), "r"(bytes), "r"(acc));
	return d;
}

__device__ __forceinline__ int
dp2a_hi_(unsigned coef, unsigned bytes, int acc)
{
	int d;
	asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(coef), "r"(bytes), "r"(acc));
	return d;
}

template <typename T>
__global__ void __launch_bounds__(256)
reducev_kernel(const T *__restrict__ in, size_t in_bpl, int in_h, T *__restrict__ out, size_t out_bpl, int out_rows,
	int ne, AxisDev t)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= ne)
		return;
	const int n = t.n_point;
	const char *base = (const char *) in;
	for (int y = blockIdx.y; y < out_rows; y += gridDim.y) {
		const int py = t.first[y] - t.embed;
		T *q = (T *) ((char *) out + (size_t) y * out_bpl) + x;

		if constexpr (sizeof(T) == 4) {
			/* 32-bit ints: int64 sum */
			const short *c = t.ms + (size_t) t.phase[y] * n;
			long long sum = 0;
			for (int i = 0; i < n; i++) {
				const int row = clampi(py + i, 0, in_h - 1);
				sum += (long long) c[i] * (long long) ((const T *) (base + (size_t) row * in_bpl))[x];
			}
			*q = fixed_finalize<T, long long>(sum);
		}
		else {
			const short *c = t.ms + (size_t) t.phase[y] * n;
			int sum = 0;
			for (int i = 0; i < n; i++) {
				const int row = clampi(py + i, 0, in_h - 1);
				sum += (int) c[i] * (int) ((const T *) (base + (size_t) row * in_bpl))[x];
			}
			*q = fixed_finalize<T, int>(sum);
		}
	}
}

template <>
__global__ void __launch_bounds__(256)
reducev_kernel<float>(const float *__restrict__ in, size_t in_bpl, int in_h, float *__restrict__ out, size_t out_bpl,
	int out_rows, int ne, AxisDev t)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= ne)
		return;
	const int n = t.n_point;
	const char *base = (const char *) in;
	for (int y = blockIdx.y; y < out_rows; y += gridDim.y) {
		const int py = t.first[y] - t.embed;
		const double *c = t.mf + (size_t) t.phase[y] * n;
		double sum = 0.0;
		for (int i = 0; i < n; i++) {
			const int row = clampi(py + i, 0, in_h - 1);
			sum = __dadd_rn(sum, __dmul_rn(c[i], (double) ((const float *) (base + (size_t) row * in_bpl))[x]));
		}
		((float *) ((char *) out + (size_t) y * out_bpl))[x] = (float) sum;
	}
}

/* uchar, 4 bytes per thread */
__global__ void __launch_bounds__(256)
reducev_u8x4_kernel(const uint8_t *__restrict__ in, size_t in_bpl, int in_h, uint8_t *__restrict__ out,
	size_t out_bpl, int out_rows, int nwords, AxisDev t)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= nwords)
		return;
	const int n = t.n_point;
	for (int y = blockIdx.y; y < out_rows; y += gridDim.y) {
		const int py = t.first[y] - t.embed;
		const short *c = t.ms + (size_t) t.phase[y] * n;
		int s0 = 2048, s1 = 2048, s2 = 2048, s3 = 2048;
		for (int i = 0; i < n; i++) {
			const int row = clampi(py + i, 0, in_h - 1);
			const unsigned int v = __ldg((const unsigned int *) (in + (size_t) row * in_bpl) + x);
			const int ci = c[i];
			s0 += ci * (int) (v & 0xff);
			s1 += ci * (int) ((v >> 8) & 0xff);
			s2 += ci * (int) ((v >> 16) & 0xff);
			s3 += ci * (int) (v >> 24);
		}
		const unsigned int b0 = clampi(s0 >> 12, 0, 255), b1 = clampi(s1 >> 12, 0, 255);
		const unsigned int b2 = clampi(s2 >> 12, 0, 255), b3 = clampi(s3 >> 12, 0, 255);
		((unsigned int *) (out + (size_t) y * out_bpl))[x] = b0 | (b1 << 8) | (b2 << 16) | (b3 << 24);
	}
}

/* uchar, register-blocked: one thread owns a 4-byte column of kRvRows consecutive output rows and walks the
 * union of their tap windows ONCE, two input rows at a time.  The two words are interleaved by PRMT into
 * [b0 b0' b1 b1'] / [b2 b2' b3 b3'] and each output row takes them with four IDP.2A against its coefficient pair
 * (c[u], c[u + 1]) for that pair of rows -- zero where a row lies outside the output row's window.  The pair table
 * of the block's rows is built in shared memory from the phase masks (the rows of a block may have any first tap
 * and any phase: the per-rect stepping of build_axis_table is kept).  Same integer sum as reducev_u8x4_kernel
 * (reducev.cpp:461-471), 12 instead of ~60 instructions per input word: config 1's 49-tap pass went 93 -> 47 us under ncu.
 */
constexpr int kRvRows = 4;
constexpr int kRvThreads = 128;

__global__ void __launch_bounds__(kRvThreads)
reducev_u8_dp2a_kernel(const uint8_t *__restrict__ in, size_t in_bpl, int in_h, uint8_t *__restrict__ out,
	size_t out_bpl, int nwords, int out_rows, AxisDev t)
{
	extern __shared__ __align__(16) unsigned s_c2[]; /* [pairs][kRvRows] */
	const int n = t.n_point;
	const int x = blockIdx.x * kRvThreads + threadIdx.x;
	/* the whole CTA walks its groups of kRvRows output rows together: the pair table is shared */
	for (int y0 = blockIdx.y * kRvRows; y0 < out_rows; y0 += gridDim.y * kRvRows) {
		if (y0 != (int) blockIdx.y * kRvRows)
			__syncthreads(); /* the previous group's pair table has been read */
		int u0 = 0x7fffffff, u1 = -0x7fffffff;
#pragma unroll
		for (int j = 0; j < kRvRows; j++) {
			const int py = __ldg(t.first + min(y0 + j, out_rows - 1)) - t.embed;
			u0 = min(u0, py);
			u1 = max(u1, py + n - 1);
		}
		const int npairs = (u1 - u0 + 2) >> 1;
		for (int idx = threadIdx.x; idx < npairs * kRvRows; idx += kRvThreads) {
			const int k = idx / kRvRows, j = idx - k * kRvRows;
			const int yj = min(y0 + j, out_rows - 1);
			const short *c = t.ms + (size_t) __ldg(t.phase + yj) * n;
			const int i0 = u0 + 2 * k - (__ldg(t.first + yj) - t.embed);
			const unsigned lo = i0 >= 0 && i0 < n ? (unsigned short) c[i0] : 0u;
			const unsigned hi = i0 + 1 >= 0 && i0 + 1 < n ? (unsigned short) c[i0 + 1] : 0u;
			s_c2[idx] = lo | (hi << 16);
		}
		__syncthreads();
		if (x >= nwords)
			continue;
		int acc[kRvRows][4];
#pragma unroll
		for (int j = 0; j < kRvRows; j++)
#pragma unroll
			for (int c = 0; c < 4; c++)
				acc[j][c] = VB200_INTERPOLATE_SCALE >> 1;
#pragma unroll 8
		for (int k = 0; k < npairs; k++) {
			const int ra = clampi(u0 + 2 * k, 0, in_h - 1), rb = clampi(u0 + 2 * k + 1, 0, in_h - 1);
			const unsigned va = __ldg((const unsigned *) (in + (size_t) ra * in_bpl) + x);
			const unsigned vb = __ldg((const unsigned *) (in + (size_t) rb * in_bpl) + x);
			const unsigned w0 = __byte_perm(va, vb, 0x5140), w1 = __byte_perm(va, vb, 0x7362);
			const uint4 c4 = *(const uint4 *) (s_c2 + k * kRvRows);
			const unsigned cj[4] = {c4.x, c4.y, c4.z, c4.w};
#pragma unroll
			for (int j = 0; j < kRvRows; j++) {
				acc[j][0] = dp2a_lo_(cj[j], w0, acc[j][0]);
				acc[j][1] = dp2a_hi_(cj[j], w0, acc[j][1]);
				acc[j][2] = dp2a_lo_(cj[j], w1, acc[j][2]);
				acc[j][3] = dp2a_hi_(cj[j], w1, acc[j][3]);
			}
		}
#pragma unroll
		for (int j = 0; j < kRvRows; j++)
			if (y0 + j < out_rows) {
				const unsigned b0 = clampi(acc[j][0] >> VB200_INTERPOLATE_SHIFT, 0, 255), b1 = clampi(acc[j][1] >> VB200_INTERPOLATE_SHIFT, 0, 255);
				const unsigned b2 = clampi(acc[j][2] >> VB200_INTERPOLATE_SHIFT, 0, 255), b3 = clampi(acc[j][3] >> VB200_INTERPOLATE_SHIFT, 0, 255);
				((unsigned *) (out + (size_t) (y0 + j) * out_bpl))[x] = b0 | (b1 << 8) | (b2 << 16) | (b3 << 24);
			}
	}
}

/* The same kernel with the block's whole tap window staged in shared memory by bulk copies (cp.async.bulk, one per
 * input row, all in flight at once behind one mbarrier) instead of being walked with dependent global loads: the
 * register-blocked kernel above spends its time waiting on row loads from L2 (long_scoreboard 13.5 per issue), here the
 * walk reads shared memory.  Needs 16-byte aligned rows and a window that fits (rows x 512 B <= kRvsMaxRows).
 */
constexpr int kRvsMaxRows = 160; /* 80 KB of staged rows per CTA: two CTAs per SM */

__device__ __forceinline__ unsigned
rv_smem_addr(const void *p)
{
	return (unsigned) __cvta_generic_to_shared(p);
}

template <bool LOOP>
__global__ void __launch_bounds__(kRvThreads)
reducev_u8_dp2a_staged_kernel(const uint8_t *__restrict__ in, size_t in_bpl, int in_h, uint8_t *__restrict__ out, size_t out_bpl, int nwords,
	int out_rows, AxisDev t, int max_pairs)
{
	extern __shared__ __align__(128) unsigned char s_raw[];
	unsigned *s_c2 = (unsigned *) s_raw;								  /* [max_pairs][kRvRows] */
	unsigned long long *bar = (unsigned long long *) (s_c2 + (size_t) max_pairs * kRvRows);
	unsigned *s_rows = (unsigned *) (((uintptr_t) (bar + 1) + 127) & ~(uintptr_t) 127); /* [2 * npairs][kRvThreads] */
	const int n = t.n_point;
	const int x0 = blockIdx.x * kRvThreads;
	const unsigned row_bytes = (unsigned) min(kRvThreads, nwords - x0) * 4u;
	const unsigned bar_s = rv_smem_addr(bar);
	if (threadIdx.x == 0) {
		asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar_s), "r"(1));
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();
	/* the whole CTA walks its groups of kRvRows output rows together; the barrier completes one phase per group */
	unsigned parity = 0;
	int y0 = blockIdx.y * kRvRows;
	do {
		if (y0 != (int) blockIdx.y * kRvRows) {
			/* the previous group's rows and pair table have been read before the copies overwrite them */
			asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
			__syncthreads();
		}
		int u0 = 0x7fffffff, u1 = -0x7fffffff;
#pragma unroll
		for (int j = 0; j < kRvRows; j++) {
			const int py = __ldg(t.first + min(y0 + j, out_rows - 1)) - t.embed;
			u0 = min(u0, py);
			u1 = max(u1, py + n - 1);
		}
		const int npairs = (u1 - u0 + 2) >> 1;
		if (threadIdx.x == 0)
			asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(bar_s),
						 "r"(row_bytes * (unsigned) (2 * npairs))
						 : "memory");
		__syncthreads();
		/* one bulk copy per window row, issued by as many threads as there are rows */
		for (int r = threadIdx.x; r < 2 * npairs; r += kRvThreads) {
			const int row = clampi(u0 + r, 0, in_h - 1);
			asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
							 rv_smem_addr(s_rows + (size_t) r * kRvThreads)),
						 "l"(in + (size_t) row * in_bpl + (size_t) x0 * 4), "r"(row_bytes), "r"(bar_s)
						 : "memory");
		}
		/* the coefficient pairs of the block's rows, while the copies fly */
		for (int idx = threadIdx.x; idx < npairs * kRvRows; idx += kRvThreads) {
			const int k = idx / kRvRows, j = idx - k * kRvRows;
			const int yj = min(y0 + j, out_rows - 1);
			const short *c = t.ms + (size_t) __ldg(t.phase + yj) * n;
			const int i0 = u0 + 2 * k - (__ldg(t.first + yj) - t.embed);
			const unsigned lo = i0 >= 0 && i0 < n ? (unsigned short) c[i0] : 0u;
			const unsigned hi = i0 + 1 >= 0 && i0 + 1 < n ? (unsigned short) c[i0 + 1] : 0u;
			s_c2[idx] = lo | (hi << 16);
		}
		__syncthreads();
		{
			unsigned done;
			do {
				asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, 0x989680;\n\tselp.u32 %0, 1, 0, p;\n\t}"
							 : "=r"(done)
							 : "r"(bar_s), "r"(parity)
							 : "memory");
			} while (!done);
		}
		const int x = x0 + threadIdx.x;
		if (x >= nwords)
			continue;
		int acc[kRvRows][4];
#pragma unroll
		for (int j = 0; j < kRvRows; j++)
#pragma unroll
			for (int c = 0; c < 4; c++)
				acc[j][c] = VB200_INTERPOLATE_SCALE >> 1;
		const unsigned *mine = s_rows + threadIdx.x;
#pragma unroll 4
		for (int k = 0; k < npairs; k++) {
			const unsigned va = mine[(size_t) (2 * k) * kRvThreads], vb = mine[(size_t) (2 * k + 1) * kRvThreads];
			const unsigned w0 = __byte_perm(va, vb, 0x5140), w1 = __byte_perm(va, vb, 0x7362);
			const uint4 c4 = *(const uint4 *) (s_c2 + k * kRvRows);
			const unsigned cj[4] = {c4.x, c4.y, c4.z, c4.w};
#pragma unroll
			for (int j = 0; j < kRvRows; j++) {
				acc[j][0] = dp2a_lo_(cj[j], w0, acc[j][0]);
				acc[j][1] = dp2a_hi_(cj[j], w0, acc[j][1]);
				acc[j][2] = dp2a_lo_(cj[j], w1, acc[j][2]);
				acc[j][3] = dp2a_hi_(cj[j], w1, acc[j][3]);
			}
		}
#pragma unroll
		for (int j = 0; j < kRvRows; j++)
			if (y0 + j < out_rows) {
				const unsigned b0 = clampi(acc[j][0] >> VB200_INTERPOLATE_SHIFT, 0, 255), b1 = clampi(acc[j][1] >> VB200_INTERPOLATE_SHIFT, 0, 255);
				const unsigned b2 = clampi(acc[j][2] >> VB200_INTERPOLATE_SHIFT, 0, 255), b3 = clampi(acc[j][3] >> VB200_INTERPOLATE_SHIFT, 0, 255);
				((unsigned *) (out + (size_t) (y0 + j) * out_bpl))[x] = b0 | (b1 << 8) | (b2 << 16) | (b3 << 24);
			}
	} while (LOOP && (parity ^= 1u, y0 += gridDim.y * kRvRows) < out_rows);
}

/* uchar RGBA rows: a CTA stages the span of input pixels its kRhThreads output pixels read (clamp addressing =
 * the reference's EXTEND_COPY embed) into shared memory, padded one word in eight so that the stride-shrink reads
 * of a warp spread over the banks, then every thread runs its taps two pixels at a time: PRMT to [r r' g g'] /
 * [b b' a a'], four IDP.2A against the phase's coefficient pair (t.mp, built on the host).  reduceh.cpp:145-160.
 */
constexpr int kRhThreads = 128;

__device__ __forceinline__ int
rh_pad(int i)
{
	return i + (i >> 3);
}

template <bool LOOP>
__global__ void __launch_bounds__(kRhThreads)
reduceh_u8x4_dp2a_kernel(const uint8_t *__restrict__ in, size_t in_bpl, int in_w, uint8_t *__restrict__ out,
	size_t out_bpl, int out_w, int rows, AxisDev t)
{
	extern __shared__ __align__(16) unsigned s_px[];
	__shared__ int s_lo, s_hi;
	const int x = blockIdx.x * kRhThreads + threadIdx.x;
	const bool live = x < out_w;
	const int ix = __ldg(t.first + min(x, out_w - 1)) - t.embed;
	if (threadIdx.x == 0) {
		s_lo = 0x7fffffff;
		s_hi = -0x7fffffff;
	}
	__syncthreads();
	{
		int lo = ix, hi = ix;
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) {
			lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
			hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
		}
		if ((threadIdx.x & 31) == 0) {
			atomicMin(&s_lo, lo);
			atomicMax(&s_hi, hi);
		}
	}
	__syncthreads();
	const int p0 = s_lo, span = s_hi - s_lo + 2 * t.npairs; /* an odd tap count reads one word past its window (coefficient 0) */
	const int rel = ix - p0;
	/* the span depends on the columns only; the whole CTA walks its rows together through the staged row */
	int y = blockIdx.y;
	do {
		if (y != (int) blockIdx.y)
			__syncthreads(); /* the previous row has been read */
		const unsigned *row = (const unsigned *) (in + (size_t) y * in_bpl);
		for (int i = threadIdx.x; i < span; i += kRhThreads)
			s_px[rh_pad(i)] = __ldg(row + clampi(p0 + i, 0, in_w - 1));
		__syncthreads();
		if (!live)
			continue;
		const unsigned *cp = t.mp + (size_t) __ldg(t.phase + x) * t.npairs;
		int r = VB200_INTERPOLATE_SCALE >> 1, g = r, b = r, a = r;
#pragma unroll 5
		for (int k = 0; k < t.npairs; k++) {
			const unsigned pa = s_px[rh_pad(rel + 2 * k)], pb = s_px[rh_pad(rel + 2 * k + 1)];
			const unsigned w0 = __byte_perm(pa, pb, 0x5140), w1 = __byte_perm(pa, pb, 0x7362);
			const unsigned c = __ldg(cp + k);
			r = dp2a_lo_(c, w0, r);
			g = dp2a_hi_(c, w0, g);
			b = dp2a_lo_(c, w1, b);
			a = dp2a_hi_(c, w1, a);
		}
		const unsigned b0 = clampi(r >> VB200_INTERPOLATE_SHIFT, 0, 255), b1 = clampi(g >> VB200_INTERPOLATE_SHIFT, 0, 255);
		const unsigned b2 = clampi(b >> VB200_INTERPOLATE_SHIFT, 0, 255), b3 = clampi(a >> VB200_INTERPOLATE_SHIFT, 0, 255);
		((unsigned *) (out + (size_t) y * out_bpl))[x] = b0 | (b1 << 8) | (b2 << 16) | (b3 << 24);
	} while (LOOP && (y += gridDim.y) < rows);
}

/* ------------------------------------------------------------------ reduceh */

template <typename T>
__global__ void __launch_bounds__(256)
reduceh_kernel(const T *__restrict__ in, size_t in_bpl, int in_w, T *__restrict__ out, size_t out_bpl, int out_w,
	int bands, int rows, AxisDev t)
{
	const int e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= out_w * bands)
		return;
	const int x = e / bands;
	const int z = e - x * bands;
	const int ix = t.first[x] - t.embed;
	const int n = t.n_point;
	const short *c = t.ms + (size_t) t.phase[x] * n;
	for (int y = blockIdx.y; y < rows; y += gridDim.y) {
		const T *p = (const T *) ((const char *) in + (size_t) y * in_bpl) + z;
		T *q = (T *) ((char *) out + (size_t) y * out_bpl) + e;

		if constexpr (sizeof(T) == 4) {
			long long sum = 0;
			for (int i = 0; i < n; i++)
				sum += (long long) c[i] * (long long) p[(size_t) clampi(ix + i, 0, in_w - 1) * bands];
			*q = fixed_finalize<T, long long>(sum);
		}
		else {
			int sum = 0;
			for (int i = 0; i < n; i++)
				sum += (int) c[i] * (int) p[(size_t) clampi(ix + i, 0, in_w - 1) * bands];
			*q = fixed_finalize<T, int>(sum);
		}
	}
}

template <>
__global__ void __launch_bounds__(256)
reduceh_kernel<float>(const float *__restrict__ in, size_t in_bpl, int in_w, float *__restrict__ out, size_t out_bpl,
	int out_w, int bands, int rows, AxisDev t)
{
	const int e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= out_w * bands)
		return;
	const int x = e / bands;
	const int z = e - x * bands;
	const int ix = t.first[x] - t.embed;
	const int n = t.n_point;
	const double *c = t.mf + (size_t) t.phase[x] * n;
	for (int y = blockIdx.y; y < rows; y += gridDim.y) {
		const float *p = (const float *) ((const char *) in + (size_t) y * in_bpl) + z;
		double sum = 0.0;
		for (int i = 0; i < n; i++)
			sum = __dadd_rn(sum, __dmul_rn(c[i], (double) p[(size_t) clampi(ix + i, 0, in_w - 1) * bands]));
		((float *) ((char *) out + (size_t) y * out_bpl))[e] = (float) sum;
	}
}

/* ------------------------------------------------- premultiply / unpremultiply */

/* uchar -> uchar 8.8 LUT path.  The LUT is built in the prologue with IEEE
 * double mul/div (correctly rounded on host and device alike):
 *   pre:   scale[i] = (int) (256 * clip(i) / max_alpha)          premultiply.c:253-259
 *   unpre: scale[i] = clip == 0 ? 0 : (int) (256 * max_alpha / clip)  unpremultiply.c:313-324
 * out = (in * scale[alpha] + 128) >> 8 stored as a byte (no clip).
 * words: 4-band pixels as one 32-bit load and store; only when both images' bases and strides are multiples of 4.
 */
template <bool UNPRE>
__global__ void __launch_bounds__(256)
premul_u8_kernel(const uint8_t *__restrict__ in, size_t in_bpl, uint8_t *__restrict__ out, size_t out_bpl, int w,
	int h, int bands, double max_alpha, bool words)
{
	__shared__ int scale[256];
	{
		const int i = threadIdx.x;
		const double clip = fmax(0.0, fmin(max_alpha, (double) i));
		if (UNPRE)
			scale[i] = clip == 0 ? 0 : (int) __ddiv_rn(__dmul_rn(256.0, max_alpha), clip);
		else
			scale[i] = (int) __ddiv_rn(__dmul_rn(256.0, clip), max_alpha);
	}
	__syncthreads();
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= w)
		return;
	for (int y = blockIdx.y; y < h; y += gridDim.y) {
		const uint8_t *p = in + (size_t) y * in_bpl + (size_t) x * bands;
		uint8_t *q = out + (size_t) y * out_bpl + (size_t) x * bands;
		if (words) {
			const unsigned int v = *(const unsigned int *) p;
			const int s = scale[v >> 24];
			const unsigned int r = (((v & 0xff) * s + 128) >> 8) & 0xff;
			const unsigned int g = ((((v >> 8) & 0xff) * s + 128) >> 8) & 0xff;
			const unsigned int b = ((((v >> 16) & 0xff) * s + 128) >> 8) & 0xff;
			*(unsigned int *) q = r | (g << 8) | (b << 16) | (v & 0xff000000u);
			continue;
		}
		const uint8_t alpha = p[bands - 1];
		const int s = scale[alpha];
		int i;
		for (i = 0; i < bands - 1; i++)
			q[i] = (uint8_t) ((p[i] * s + 128) >> 8);
		q[i] = alpha;
	}
}

/* PRE_* : OUT nalpha = (OUT) clip_alpha / max_alpha; q = p * nalpha  (premultiply.c:86-122) */
template <typename IN>
__global__ void __launch_bounds__(256, 8) /* the row loop must not cost occupancy */
premul_float_kernel(const IN *__restrict__ in, size_t in_bpl, float *__restrict__ out, size_t out_bpl, int w,
	int h, int bands, double max_alpha)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= w)
		return;
	for (int y = blockIdx.y; y < h; y += gridDim.y) {
		const IN *p = (const IN *) ((const char *) in + (size_t) y * in_bpl) + (size_t) x * bands;
		float *q = (float *) ((char *) out + (size_t) y * out_bpl) + (size_t) x * bands;
		const IN alpha = p[bands - 1];
		/* VIPS_CLIP(0, alpha, max_alpha) is evaluated in double, assigned to IN */
		const IN clip_alpha = (IN) fmax(0.0, fmin(max_alpha, (double) alpha));
		const float nalpha = (float) __ddiv_rn((double) (float) clip_alpha, max_alpha);
		int i;
		for (i = 0; i < bands - 1; i++)
			q[i] = __fmul_rn((float) p[i], nalpha);
		q[i] = (float) alpha;
	}
}

/* UNPRE_* / FUNPRE_*  (unpremultiply.c:85-183), alpha_band = bands - 1 */
template <typename IN, bool FP>
__global__ void __launch_bounds__(256, 8) /* the row loop must not cost occupancy */
unpremul_float_kernel(const IN *__restrict__ in, size_t in_bpl, float *__restrict__ out, size_t out_bpl, int w,
	int h, int bands, double max_alpha)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= w)
		return;
	for (int y = blockIdx.y; y < h; y += gridDim.y) {
		const IN *p = (const IN *) ((const char *) in + (size_t) y * in_bpl) + (size_t) x * bands;
		float *q = (float *) ((char *) out + (size_t) y * out_bpl) + (size_t) x * bands;
		const IN alpha = p[bands - 1];
		float factor;
		if (FP)
			factor = fabs((double) alpha) < 0.01 ? 0.0f : (float) __ddiv_rn(max_alpha, (double) alpha);
		else
			factor = alpha == 0 ? 0.0f : (float) __ddiv_rn(max_alpha, (double) alpha);
		for (int i = 0; i < bands - 1; i++)
			q[i] = __fmul_rn(factor, (float) p[i]);
		q[bands - 1] = (float) fmax(0.0, fmin(max_alpha, (double) alpha));
	}
}

bool
aligned4(const void *p, size_t bpl)
{
	return (((uintptr_t) p) & 3) == 0 && (bpl & 3) == 0;
}

/* premul_u8_kernel's 32-bit word path: 4 bands, both images on the word grid */
bool
premul_words(const DevImage &in, const DevImage &out)
{
	return in.bands == 4 && aligned4(in.data, in.bpl) && aligned4(out.data, out.bpl);
}

/* An AxisTable packed into one block: the AxisDev points into it (host image `host`, `total` bytes). */
void
pack_axis(const AxisTable &t, std::vector<char> &host, AxisDev *d)
{
	const int npairs = (t.n_point + 1) / 2;
	std::vector<unsigned> mp((size_t) 65 * npairs);
	for (int ph = 0; ph < 65 && t.ms.size() >= (size_t) 65 * t.n_point; ph++)
		for (int k = 0; k < npairs; k++) {
			const unsigned lo = (unsigned short) t.ms[(size_t) ph * t.n_point + 2 * k];
			const unsigned hi = 2 * k + 1 < t.n_point ? (unsigned short) t.ms[(size_t) ph * t.n_point + 2 * k + 1] : 0u;
			mp[(size_t) ph * npairs + k] = lo | (hi << 16);
		}
	const size_t n_first = t.first.size() * sizeof(int);
	const size_t n_ms = t.ms.size() * sizeof(short);
	const size_t n_mf = t.mf.size() * sizeof(double);
	const size_t n_mp = mp.size() * sizeof(unsigned);
	const size_t off_mf = 0;
	const size_t off_first = off_mf + n_mf;
	const size_t off_phase = off_first + n_first;
	const size_t off_mp = off_phase + n_first;
	const size_t off_ms = off_mp + n_mp;
	host.resize(off_ms + n_ms);
	memcpy(&host[off_mf], t.mf.data(), n_mf);
	memcpy(&host[off_first], t.first.data(), n_first);
	memcpy(&host[off_phase], t.phase.data(), n_first);
	memcpy(&host[off_mp], mp.data(), n_mp);
	memcpy(&host[off_ms], t.ms.data(), n_ms);
	/* offsets; rebased onto the device block by the caller */
	d->mf = (const double *) off_mf;
	d->first = (const int *) off_first;
	d->phase = (const int *) off_phase;
	d->mp = (const unsigned *) off_mp;
	d->ms = (const short *) off_ms;
	d->n_point = t.n_point;
	d->embed = t.embed;
	d->npairs = npairs;
}

void
rebase_axis(AxisDev *d, const void *block)
{
	const char *b = (const char *) block;
	d->mf = (const double *) (b + (size_t) d->mf);
	d->first = (const int *) (b + (size_t) d->first);
	d->phase = (const int *) (b + (size_t) d->phase);
	d->mp = (const unsigned *) (b + (size_t) d->mp);
	d->ms = (const short *) (b + (size_t) d->ms);
}

/* Upload an AxisTable as one packed block from the stream-ordered pool; the AxisDev points into it. */
int
upload_axis(const char *domain, const AxisTable &t, AxisDev *d, void **block, cudaStream_t s)
{
	std::vector<char> host;
	pack_axis(t, host, d);
	if (dev_alloc(domain, block, host.size(), s))
		return -1;
	VB200_CUDA(domain, cudaMemcpyAsync(*block, host.data(), host.size(), cudaMemcpyHostToDevice, s));
	/* pageable source: the copy has been staged when the call returns */
	rebase_axis(d, *block);
	return 0;
}

int
check_launch(const char *domain, const char *what)
{
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
		return cuda_fail(domain, e, what);
	count_launch();
	return 0;
}

/* shared memory the dp2a kernels need for this table (0: not usable) */
size_t
reducev_dp2a_smem(const AxisTable &t, int out_rows)
{
	int pairs = 0;
	for (int y0 = 0; y0 < out_rows; y0 += kRvRows) {
		int u0 = 0x7fffffff, u1 = -0x7fffffff;
		for (int j = 0; j < kRvRows; j++) {
			const int py = t.first[std::min(y0 + j, out_rows - 1)];
			u0 = std::min(u0, py);
			u1 = std::max(u1, py + t.n_point - 1);
		}
		pairs = std::max(pairs, (u1 - u0 + 2) >> 1);
	}
	return (size_t) pairs * kRvRows * sizeof(unsigned);
}

size_t
reduceh_dp2a_smem(const AxisTable &t, int out_cols)
{
	int span = 0;
	for (int x0 = 0; x0 < out_cols; x0 += kRhThreads) {
		int lo = 0x7fffffff, hi = -0x7fffffff;
		for (int x = x0; x < std::min(x0 + kRhThreads, out_cols); x++) {
			lo = std::min(lo, t.first[x]);
			hi = std::max(hi, t.first[x]);
		}
		span = std::max(span, hi - lo + 2 * ((t.n_point + 1) / 2));
	}
	return (size_t) (span + (span >> 3) + 2) * sizeof(unsigned);
}

int
run_reducev(const char *domain, const void *in, size_t in_bpl, int in_h, void *out, size_t out_bpl, int ne, int out_rows,
	int fmt, const AxisDev &d, size_t dp2a_smem, cudaStream_t s)
{
#define RV(T) reducev_kernel<T><<<row_grid(ne, out_rows), 256, 0, s>>>((const T *) in, in_bpl, in_h, (T *) out, out_bpl, out_rows, ne, d)
	switch (fmt) {
	case VB200_FORMAT_UCHAR:
		if ((ne & 3) == 0 && aligned4(in, in_bpl) && aligned4(out, out_bpl)) {
			const int max_pairs = (int) (dp2a_smem / (kRvRows * sizeof(unsigned)));
			static const bool no_staged = getenv("VB200_NO_REDUCEV_STAGED") != nullptr;
			if (dp2a_smem > 0 && 2 * max_pairs <= kRvsMaxRows && !no_staged && (((uintptr_t) in | in_bpl) & 15) == 0 && (ne & 15) == 0) {
				const size_t smem = dp2a_smem + 8 + 128 + (size_t) 2 * max_pairs * kRvThreads * 4;
				static bool attr_done = false;
				if (!attr_done) {
					cudaFuncSetAttribute(reducev_u8_dp2a_staged_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
					cudaFuncSetAttribute(reducev_u8_dp2a_staged_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
					attr_done = true;
				}
				(rows_loop((out_rows + kRvRows - 1) / kRvRows) ? reducev_u8_dp2a_staged_kernel<true> : reducev_u8_dp2a_staged_kernel<false>)<<<row_grid(ne / 4, (out_rows + kRvRows - 1) / kRvRows, kRvThreads), kRvThreads, smem,
					s>>>((const uint8_t *) in, in_bpl, in_h, (uint8_t *) out, out_bpl, ne / 4, out_rows, d, max_pairs);
			}
			else if (dp2a_smem > 0 && dp2a_smem <= 40 * 1024 && out_rows >= 1)
				reducev_u8_dp2a_kernel<<<row_grid(ne / 4, (out_rows + kRvRows - 1) / kRvRows, kRvThreads), kRvThreads,
					dp2a_smem, s>>>((const uint8_t *) in, in_bpl, in_h, (uint8_t *) out, out_bpl, ne / 4, out_rows, d);
			else
				reducev_u8x4_kernel<<<row_grid(ne / 4, out_rows), 256, 0, s>>>((const uint8_t *) in, in_bpl, in_h,
					(uint8_t *) out, out_bpl, out_rows, ne / 4, d);
		}
		else
			RV(uint8_t);
		break;
	case VB200_FORMAT_CHAR: RV(int8_t); break;
	case VB200_FORMAT_USHORT: RV(uint16_t); break;
	case VB200_FORMAT_SHORT: RV(int16_t); break;
	case VB200_FORMAT_UINT: RV(uint32_t); break;
	case VB200_FORMAT_INT: RV(int32_t); break;
	case VB200_FORMAT_FLOAT: RV(float); break;
	default:
		error(domain, "band format %d not supported on the device path", fmt);
		return -1;
	}
#undef RV
	return check_launch(domain, "reducev kernel");
}

int
run_reduceh(const char *domain, const void *in, size_t in_bpl, int in_w, void *out, size_t out_bpl, int bands, int out_cols,
	int rows, int fmt, const AxisDev &d, size_t dp2a_smem, cudaStream_t s)
{
#define RH(T) reduceh_kernel<T><<<row_grid(out_cols * bands, rows), 256, 0, s>>>((const T *) in, in_bpl, in_w, (T *) out, out_bpl, out_cols, bands, rows, d)
	switch (fmt) {
	case VB200_FORMAT_UCHAR:
		if (bands == 4 && aligned4(in, in_bpl) && aligned4(out, out_bpl) && dp2a_smem > 0 && dp2a_smem <= 40 * 1024)
			(rows_loop(rows) ? reduceh_u8x4_dp2a_kernel<true> : reduceh_u8x4_dp2a_kernel<false>)<<<row_grid(out_cols, rows, kRhThreads), kRhThreads, dp2a_smem, s>>>(
				(const uint8_t *) in, in_bpl, in_w, (uint8_t *) out, out_bpl, out_cols, rows, d);
		else
			RH(uint8_t);
		break;
	case VB200_FORMAT_CHAR: RH(int8_t); break;
	case VB200_FORMAT_USHORT: RH(uint16_t); break;
	case VB200_FORMAT_SHORT: RH(int16_t); break;
	case VB200_FORMAT_UINT: RH(uint32_t); break;
	case VB200_FORMAT_INT: RH(int32_t); break;
	case VB200_FORMAT_FLOAT: RH(float); break;
	default:
		error(domain, "band format %d not supported on the device path", fmt);
		return -1;
	}
#undef RH
	return check_launch(domain, "reduceh kernel");
}

/* Tables of whole-image passes, cached: building one costs 65 x n sin() evaluations plus the per-rect stepping, and
 * uploading it a staged copy -- together several times the kernel on a single 4096 x 4096 frame (config 1).  The key
 * is everything build_axis_table() reads; the device block lives until the entry is evicted (cudaFree waits for the
 * device, so a kernel still reading it is safe).
 */
struct AxisPlan {
	AxisTable t;
	AxisDev d;
	void *block = nullptr;
	size_t v_smem = 0, h_smem = 0;
	~AxisPlan()
	{
		if (block)
			cudaFree(block);
	}
};

struct AxisKey {
	int out_size, n_point, kernel, rect;
	double residual, offset;
	bool
	operator==(const AxisKey &o) const
	{
		return out_size == o.out_size && n_point == o.n_point && kernel == o.kernel && rect == o.rect &&
			memcmp(&residual, &o.residual, sizeof(double)) == 0 && memcmp(&offset, &o.offset, sizeof(double)) == 0;
	}
};

std::mutex g_axis_lock;
std::vector<std::pair<AxisKey, std::shared_ptr<AxisPlan>>> g_axis_cache; /* most recent last */
constexpr size_t kAxisCacheEntries = 24;

std::shared_ptr<AxisPlan>
axis_plan(const char *domain, const ReduceGeom &g, int kernel, int rect, bool vertical)
{
	const AxisKey key = {g.out_size, g.n_point, kernel, rect, g.residual, g.offset};
	{
		std::lock_guard<std::mutex> lock(g_axis_lock);
		for (size_t i = 0; i < g_axis_cache.size(); i++)
			if (g_axis_cache[i].first == key) {
				auto hit = g_axis_cache[i];
				g_axis_cache.erase(g_axis_cache.begin() + i);
				g_axis_cache.push_back(hit);
				return hit.second;
			}
	}
	auto pl = std::make_shared<AxisPlan>();
	build_axis_table(pl->t, g.out_size, g.residual, g.offset, g.n_point, kernel, rect);
	std::vector<char> host;
	pack_axis(pl->t, host, &pl->d);
	if (cudaMalloc(&pl->block, host.size()) != cudaSuccess) {
		pl->block = nullptr;
		cuda_fail(domain, cudaGetLastError(), "cudaMalloc (axis tables)");
		return nullptr;
	}
	if (cudaMemcpy(pl->block, host.data(), host.size(), cudaMemcpyHostToDevice) != cudaSuccess) {
		cuda_fail(domain, cudaGetLastError(), "cudaMemcpy (axis tables)");
		return nullptr;
	}
	rebase_axis(&pl->d, pl->block);
	pl->v_smem = reducev_dp2a_smem(pl->t, g.out_size);
	pl->h_smem = reduceh_dp2a_smem(pl->t, g.out_size);
	(void) vertical;
	std::lock_guard<std::mutex> lock(g_axis_lock);
	if (g_axis_cache.size() >= kAxisCacheEntries)
		g_axis_cache.erase(g_axis_cache.begin());
	g_axis_cache.push_back(std::make_pair(key, pl));
	return pl;
}

} // namespace

void
resample_cache_clear()
{
	std::lock_guard<std::mutex> lock(g_axis_lock);
	g_axis_cache.clear();
}

/* ------------------------------------------------------------- launchers */

int
launch_reducev(const char *domain, const void *in, size_t in_bpl, int in_h, void *out, size_t out_bpl, int ne,
	int out_rows, int fmt, const AxisTable &t, cudaStream_t s)
{
	AxisDev d;
	void *block = nullptr;
	if (upload_axis(domain, t, &d, &block, s))
		return -1;
	const int r = run_reducev(domain, in, in_bpl, in_h, out, out_bpl, ne, out_rows, fmt, d,
		fmt == VB200_FORMAT_UCHAR ? reducev_dp2a_smem(t, out_rows) : 0, s);
	dev_free(block, s);
	return r;
}

int
launch_reduceh(const char *domain, const void *in, size_t in_bpl, int in_w, void *out, size_t out_bpl, int bands,
	int out_cols, int rows, int fmt, const AxisTable &t, cudaStream_t s)
{
	AxisDev d;
	void *block = nullptr;
	if (upload_axis(domain, t, &d, &block, s))
		return -1;
	const int r = run_reduceh(domain, in, in_bpl, in_w, out, out_bpl, bands, out_cols, rows, fmt, d,
		fmt == VB200_FORMAT_UCHAR && bands == 4 ? reduceh_dp2a_smem(t, out_cols) : 0, s);
	dev_free(block, s);
	return r;
}

/* ------------------------------------------------------------- device ops */

int
dev_shrinkv(const char *domain, const DevImage &in, DevImage *out, int vshrink, int ceil_mode, cudaStream_t s)
{
	if (vshrink < 1) {
		error(domain, "shrink factors should be >= 1");
		return -1;
	}
	if (!format_is_supported(in.fmt)) {
		error(domain, "band format %d not supported on the device path", in.fmt);
		return -1;
	}
	if (vshrink == 1) {
		*out = in;
		out->owned = false;
		return 0;
	}
	const int oh = shrink_size(in.h, vshrink, ceil_mode);
	if (oh <= 0) {
		error(domain, "image has shrunk to nothing");
		return -1;
	}
	if (dev_image_new(domain, out, in.w, oh, in.bands, in.fmt, in.type, s))
		return -1;
	const int ne = in.w * in.bands;
	const unsigned int mult8 = (unsigned int) ((1LL << 32) / ((1 << 8) * (long long) vshrink));
	const unsigned long long mult16 = ((1ULL << 32) + vshrink - 1) / vshrink;

#define SV(T) shrinkv_kernel<T><<<row_grid(ne, oh), 256, 0, s>>>((const T *) in.data, in.bpl, in.h, (T *) out->data, out->bpl, oh, ne, vshrink, mult8, mult16)
	switch (in.fmt) {
	case VB200_FORMAT_UCHAR:
		if ((ne & 3) == 0 && aligned4(in.data, in.bpl) && aligned4(out->data, out->bpl) && vshrink <= 257)
			shrinkv_u8x4_kernel<<<row_grid(ne / 4, oh), 256, 0, s>>>((const uint8_t *) in.data, in.bpl, in.h,
				(uint8_t *) out->data, out->bpl, oh, ne / 4, vshrink, mult8);
		else
			SV(uint8_t);
		break;
	case VB200_FORMAT_CHAR: SV(int8_t); break;
	case VB200_FORMAT_USHORT: SV(uint16_t); break;
	case VB200_FORMAT_SHORT: SV(int16_t); break;
	case VB200_FORMAT_UINT: SV(uint32_t); break;
	case VB200_FORMAT_INT: SV(int32_t); break;
	case VB200_FORMAT_FLOAT: SV(float); break;
	}
#undef SV
	return check_launch(domain, "shrinkv kernel");
}

int
dev_shrinkh(const char *domain, const DevImage &in, DevImage *out, int hshrink, int ceil_mode, cudaStream_t s)
{
	if (hshrink < 1) {
		error(domain, "shrink factors should be >= 1");
		return -1;
	}
	if (!format_is_supported(in.fmt)) {
		error(domain, "band format %d not supported on the device path", in.fmt);
		return -1;
	}
	if (hshrink == 1) {
		*out = in;
		out->owned = false;
		return 0;
	}
	const int ow = shrink_size(in.w, hshrink, ceil_mode);
	if (ow <= 0) {
		error(domain, "image has shrunk to nothing");
		return -1;
	}
	if (dev_image_new(domain, out, ow, in.h, in.bands, in.fmt, in.type, s))
		return -1;
	const unsigned int mult8 = (unsigned int) ((1LL << 32) / ((1 << 8) * (long long) hshrink));
	const unsigned long long mult16 = ((1ULL << 32) + hshrink - 1) / hshrink;

#define SH(T) shrinkh_kernel<T><<<row_grid(ow * in.bands, in.h), 256, 0, s>>>((const T *) in.data, in.bpl, in.w, (T *) out->data, out->bpl, ow, in.bands, in.h, hshrink, mult8, mult16)
	switch (in.fmt) {
	case VB200_FORMAT_UCHAR: SH(uint8_t); break;
	case VB200_FORMAT_CHAR: SH(int8_t); break;
	case VB200_FORMAT_USHORT: SH(uint16_t); break;
	case VB200_FORMAT_SHORT: SH(int16_t); break;
	case VB200_FORMAT_UINT: SH(uint32_t); break;
	case VB200_FORMAT_INT: SH(int32_t); break;
	case VB200_FORMAT_FLOAT: SH(float); break;
	}
#undef SH
	return check_launch(domain, "shrinkh kernel");
}

int
dev_reducev_pass(const char *domain, const DevImage &in, DevImage *out, const ReduceGeom &g, int kernel, int rect_h,
	cudaStream_t s)
{
	const std::shared_ptr<AxisPlan> ap = axis_plan(domain, g, kernel, rect_h, true);
	if (!ap)
		return -1;
	if (dev_image_new(domain, out, in.w, g.out_size, in.bands, in.fmt, in.type, s))
		return -1;
	return run_reducev(domain, in.data, in.bpl, in.h, out->data, out->bpl, in.w * in.bands, g.out_size, in.fmt, ap->d, ap->v_smem, s);
}

int
dev_reduceh_pass(const char *domain, const DevImage &in, DevImage *out, const ReduceGeom &g, int kernel, int rect_w,
	cudaStream_t s)
{
	const std::shared_ptr<AxisPlan> ap = axis_plan(domain, g, kernel, rect_w, false);
	if (!ap)
		return -1;
	if (dev_image_new(domain, out, g.out_size, in.h, in.bands, in.fmt, in.type, s))
		return -1;
	return run_reduceh(domain, in.data, in.bpl, in.w, out->data, out->bpl, in.bands, g.out_size, in.h, in.fmt, ap->d, ap->h_smem, s);
}

int
dev_reducev(const char *domain, const DevImage &in, DevImage *out, double vshrink, int kernel, double gap, int rect_h,
	cudaStream_t s)
{
	if (!format_is_supported(in.fmt)) {
		error(domain, "band format %d not supported on the device path", in.fmt);
		return -1;
	}
	ReduceGeom g;
	if (reduce_geometry(domain, in.h, vshrink, kernel, gap, &g))
		return -1;
	DevImage box;
	if (dev_shrinkv(domain, in, &box, g.int_shrink, 1, s))
		return -1;
	if (g.n_point == 0) {
		*out = box;
		return 0;
	}
	int r = dev_reducev_pass(domain, box, out, g, kernel, rect_h, s);
	dev_image_release(&box, s);
	return r;
}

int
dev_reduceh(const char *domain, const DevImage &in, DevImage *out, double hshrink, int kernel, double gap, int rect_w,
	cudaStream_t s)
{
	if (!format_is_supported(in.fmt)) {
		error(domain, "band format %d not supported on the device path", in.fmt);
		return -1;
	}
	ReduceGeom g;
	if (reduce_geometry(domain, in.w, hshrink, kernel, gap, &g))
		return -1;
	DevImage box;
	if (dev_shrinkh(domain, in, &box, g.int_shrink, 1, s))
		return -1;
	if (g.n_point == 0) {
		*out = box;
		return 0;
	}
	int r = dev_reduceh_pass(domain, box, out, g, kernel, rect_w, s);
	dev_image_release(&box, s);
	return r;
}

int
dev_premultiply(const char *domain, const DevImage &in, DevImage *out, double max_alpha, int uchar_mode, cudaStream_t s)
{
	if (!format_is_supported(in.fmt)) {
		error(domain, "band format %d not supported on the device path", in.fmt);
		return -1;
	}
	if (in.bands == 1) {
		*out = in;
		out->owned = false;
		return 0;
	}
	if (max_alpha <= 0)
		max_alpha = interpretation_max_alpha(in.type);
	const bool lut = uchar_mode && in.fmt == VB200_FORMAT_UCHAR;
	if (dev_image_new(domain, out, in.w, in.h, in.bands, lut ? VB200_FORMAT_UCHAR : VB200_FORMAT_FLOAT, in.type, s))
		return -1;
	const dim3 grid = row_grid(in.w, in.h);
#define PM(T) premul_float_kernel<T><<<grid, 256, 0, s>>>((const T *) in.data, in.bpl, (float *) out->data, out->bpl, in.w, in.h, in.bands, max_alpha)
	if (lut)
		premul_u8_kernel<false><<<grid, 256, 0, s>>>((const uint8_t *) in.data, in.bpl, (uint8_t *) out->data,
			out->bpl, in.w, in.h, in.bands, max_alpha, premul_words(in, *out));
	else
		switch (in.fmt) {
		case VB200_FORMAT_UCHAR: PM(uint8_t); break;
		case VB200_FORMAT_CHAR: PM(int8_t); break;
		case VB200_FORMAT_USHORT: PM(uint16_t); break;
		case VB200_FORMAT_SHORT: PM(int16_t); break;
		case VB200_FORMAT_UINT: PM(uint32_t); break;
		case VB200_FORMAT_INT: PM(int32_t); break;
		case VB200_FORMAT_FLOAT: PM(float); break;
		}
#undef PM
	return check_launch(domain, "premultiply kernel");
}

int
dev_unpremultiply(const char *domain, const DevImage &in, DevImage *out, double max_alpha, int uchar_mode,
	cudaStream_t s)
{
	if (!format_is_supported(in.fmt)) {
		error(domain, "band format %d not supported on the device path", in.fmt);
		return -1;
	}
	if (in.bands == 1) {
		*out = in;
		out->owned = false;
		return 0;
	}
	if (max_alpha <= 0)
		max_alpha = interpretation_max_alpha(in.type);
	const bool lut = uchar_mode && in.fmt == VB200_FORMAT_UCHAR;
	if (dev_image_new(domain, out, in.w, in.h, in.bands, lut ? VB200_FORMAT_UCHAR : VB200_FORMAT_FLOAT, in.type, s))
		return -1;
	const dim3 grid = row_grid(in.w, in.h);
#define UPM(T, FP) unpremul_float_kernel<T, FP><<<grid, 256, 0, s>>>((const T *) in.data, in.bpl, (float *) out->data, out->bpl, in.w, in.h, in.bands, max_alpha)
	if (lut)
		premul_u8_kernel<true><<<grid, 256, 0, s>>>((const uint8_t *) in.data, in.bpl, (uint8_t *) out->data,
			out->bpl, in.w, in.h, in.bands, max_alpha, premul_words(in, *out));
	else
		switch (in.fmt) {
		case VB200_FORMAT_UCHAR: UPM(uint8_t, false); break;
		case VB200_FORMAT_CHAR: UPM(int8_t, false); break;
		case VB200_FORMAT_USHORT: UPM(uint16_t, false); break;
		case VB200_FORMAT_SHORT: UPM(int16_t, false); break;
		case VB200_FORMAT_UINT: UPM(uint32_t, false); break;
		case VB200_FORMAT_INT: UPM(int32_t, false); break;
		case VB200_FORMAT_FLOAT: UPM(float, true); break;
		}
#undef UPM
	return check_launch(domain, "unpremultiply kernel");
}

/* vips_resize, downsizing half: resize.c:150-231.  Upsizing (affine) is in
 * affine.cu.
 */
int
dev_resize(const char *domain, const DevImage &in, DevImage *out, double hscale, double vscale, int kernel, double gap,
	cudaStream_t s)
{
	hscale = std::max(hscale, 1.0 / in.w);
	vscale = std::max(vscale, 1.0 / in.h);
	if (hscale > 1.0 || vscale > 1.0) {
		if (hscale < 1.0 || vscale < 1.0) {
			/* reduce on one axis feeding an affine on the other: the reduce pass would see
			 * the rects the affine asks for, which the whole-image passes here do not model
			 */
			error(domain, "mixed up/down resize is not on the device path");
			return -1;
		}
		return dev_resize_up(domain, in, out, hscale, vscale, kernel, s);
	}
	if (kernel == VB200_KERNEL_NEAREST) {
		/* resize.c:167-205: VIPS_KERNEL_NEAREST first drops whole pixels with vips_subsample (the integer part of the
		 * shrink over gap), then reduces the residual.  The subsample step is not on the device path: when it would
		 * run, decline -- a direct nearest reduce by the whole factor picks different pixels and another size.
		 */
		int xfac, yfac;
		if (gap < 1.0) {
			xfac = (int) floor(1.0 / hscale);
			yfac = (int) floor(1.0 / vscale);
		}
		else {
			const int target_width = VB200_ROUND_UINT(in.w * hscale), target_height = VB200_ROUND_UINT(in.h * vscale);
			xfac = target_width > 0 ? (int) floor((double) in.w / target_width / gap) : 1;
			yfac = target_height > 0 ? (int) floor((double) in.h / target_height / gap) : 1;
		}
		if (xfac > 1 || yfac > 1) {
			error(domain, "nearest-neighbour resize with a subsample step (%d x %d) is not on the device path", xfac, yfac);
			return -1;
		}
	}
	const double vs = vscale < 1.0 ? 1.0 / vscale : 1.0;
	const double hs = hscale < 1.0 ? 1.0 / hscale : 1.0;
	return dev_reduce_chain(domain, in, out, hs, vs, kernel, gap, s);
}

/* reducev(vshrink) then reduceh(hshrink) with the caller's doubles: the downsizing half of
 * vips_resize (resize.c:215-231) and the whole of vips_reduce (reduce.c:106-114).  A factor of
 * exactly 1.0 skips its pass, as both builds do.
 */
int
dev_reduce_chain(const char *domain, const DevImage &in, DevImage *out, double hs, double vs, int kernel, double gap,
	cudaStream_t s)
{
	ReduceGeom gv, gh;
	gv.int_shrink = gh.int_shrink = 1;
	gh.out_size = in.w;
	if (vs != 1.0 && reduce_geometry(domain, in.h, vs, kernel, gap, &gv))
		return -1;
	if (hs != 1.0 && reduce_geometry(domain, in.w, hs, kernel, gap, &gh))
		return -1;

	/* Sink tile geometry from the pipeline's demand hint: the minimum over
	 * all ops (iofuncs/generate.c:275-293); shrinkv asks SMALLTILE
	 * (shrinkv.c:553), reducev/reduceh FATSTRIP.  vips_get_tile_size,
	 * iofuncs/thread.c:288-325.
	 */
	const TileGeometry tg = tile_geometry();
	int tile_w, tile_h;
	if (gv.int_shrink > 1) {
		tile_w = tg.tile_width;
		tile_h = tg.tile_height;
	}
	else {
		tile_w = gh.out_size;
		tile_h = tg.fatstrip_height;
	}
	/* shrinkh chunks its requests into fatstrip-height strips (shrinkh.c:247-272):
	 * that is the rect height reducev sees when a shrinkh sits downstream.
	 */
	int rect_h = tile_h;
	if (gh.int_shrink > 1)
		rect_h = std::min(rect_h, tg.fatstrip_height);

	DevImage mid = in;
	mid.owned = false;
	if (vs != 1.0 && dev_reducev(domain, in, &mid, vs, kernel, gap, rect_h, s))
		return -1;
	if (hs != 1.0) {
		int r = dev_reduceh(domain, mid, out, hs, kernel, gap, tile_w, s);
		dev_image_release(&mid, s);
		return r;
	}
	*out = mid;
	return 0;
}

} // namespace vb200
