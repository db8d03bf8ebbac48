/* jpeg_common.cuh -- what the JPEG decoder (jpeg.cu) and encoder (jpeg_encode.cu) share: the zig-zag order, the
 * fixed-point constants of libjpeg's integer DCTs and the one-CTA prefix scan.
 */
#pragma once

#define HD __host__ __device__ __forceinline__

namespace vb200 {

/* T.81 Figure A.6: the natural (row-major) position of the k-th coefficient in zig-zag order */
constexpr unsigned char kZigzag[64] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7,
	14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

/* jidctint.c / jfdctint.c: the DCT constants as FIX(x) at CONST_BITS 13 */
#define FIXC(name, v) constexpr int name = v
FIXC(F_0_211164243, 1730);
FIXC(F_0_298631336, 2446);
FIXC(F_0_390180644, 3196);
FIXC(F_0_509795579, 4176);
FIXC(F_0_541196100, 4433);
FIXC(F_0_601344887, 4926);
FIXC(F_0_720959822, 5906);
FIXC(F_0_765366865, 6270);
FIXC(F_0_850430095, 6967);
FIXC(F_0_899976223, 7373);
FIXC(F_1_061594337, 8697);
FIXC(F_1_175875602, 9633);
FIXC(F_1_272758580, 10426);
FIXC(F_1_451774981, 11893);
FIXC(F_1_501321110, 12299);
FIXC(F_1_847759065, 15137);
FIXC(F_1_961570560, 16069);
FIXC(F_2_053119869, 16819);
FIXC(F_2_172734803, 17799);
FIXC(F_2_562915447, 20995);
FIXC(F_3_072711026, 25172);
FIXC(F_3_624509785, 29692);
constexpr int CB = 13, P1 = 2; /* CONST_BITS, PASS1_BITS */

HD int
descale(int x, int n)
{
	return (x + (1 << (n - 1))) >> n;
}

/* Exclusive prefix sum over items 0 .. n - 1 in one CTA: each thread sums a contiguous chunk of val(i), the chunk sums
 * are scanned in s_part[blockDim.x] (shared memory), then put(i, the sum of the items before i) is called for every item
 * in order, each after its val(i).  Returns the sum of all items.
 */
template <typename T, typename Val, typename Put>
__device__ __forceinline__ T
cta_exclusive_scan(unsigned n, T *s_part, Val val, Put put)
{
	const unsigned per = (n + blockDim.x - 1) / blockDim.x;
	const unsigned a = min(n, threadIdx.x * per), e = min(n, a + per);
	T sum = 0;
	for (unsigned i = a; i < e; i++)
		sum += val(i);
	s_part[threadIdx.x] = sum;
	__syncthreads();
	for (unsigned o = 1; o < blockDim.x; o <<= 1) {
		const T v = threadIdx.x >= o ? s_part[threadIdx.x - o] : 0;
		__syncthreads();
		s_part[threadIdx.x] += v;
		__syncthreads();
	}
	T run = s_part[threadIdx.x] - sum;
	for (unsigned i = a; i < e; i++) {
		const T v = val(i);
		put(i, run);
		run += v;
	}
	return s_part[blockDim.x - 1];
}

} // namespace vb200
