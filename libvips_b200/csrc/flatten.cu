/* flatten.cu -- vips_flatten on the device, SURVEY 8f rank 3 (conversion ops that share the pixel-wise kernel shape).
 *
 * reference: conversion/flatten.c:421-529 (vips_flatten_build) and its generate functions
 *   :170-225  vips_flatten_black_gen_uchar   q = p * lut[a],  lut[i] = (float) ((double) i / max_alpha)
 *   :293-354  vips_flatten_gen_uchar         q = p * fa[a] + ink * fn[a],  fn[i] = (float) ((max_alpha - i) / max_alpha)
 *   :227-288, :358-419 the per-format loops (:88-166): double arithmetic for the wider formats,
 *                                            q = ((double) p * alpha + (double) ink * nalpha) / max_alpha
 *   :463-470, :519-523 integer images whose max_alpha is below the format's range are cast to double, flattened
 *             there and cast back (cast.c:123-131, 231-238: clip in double, truncate)
 * and vips__vector_to_ink (conversion/insert.c:244-359) for the background pixel: (float) bg through vips_linear, then
 * vips_cast to the working format.
 *
 * Pixel-wise, HBM-bound: bands elements in, bands - 1 out.  One thread per pixel in the general kernel; 4-band uchar
 * rows (the RGBA case) go four pixels per thread, one 128-bit load and three 32-bit stores.  The uchar LUTs are built
 * per CTA in shared memory with IEEE double divisions (the same values the reference's host loop computes), so nothing
 * is uploaded.  Every float / double operation is an explicit round-to-nearest intrinsic: no FMA contraction.
 * Algorithmic bytes: w * h * (2 * bands - 1) * sizeof(element).
 *
 * Declined (-1, the host keeps its C path): the integer loops where the reference itself converts an out-of-range double
 * to an integer type (`TYPE nalpha = max_alpha - alpha` with max_alpha beyond the format, flatten.c:134, undefined in C):
 * char / short / uint / int outside the double detour, ushort unless max_alpha is 65535; double images; > 17 bands.
 *
 * The per-pixel code is __host__ __device__: vb200_debug_flatten_host runs it on the CPU (tests/test_widen_flatten.py).
 */
#include <climits>
#include <cstring>
#include <vector>

#include "vb200_internal.h"

namespace vb200 {

namespace {

constexpr int kFlattenMaxBands = 17;

enum FlattenMode { FM_UCHAR = 0, FM_DOUBLE_LOOPS = 1, FM_WIDE = 2 };

struct FlattenDev {
	int w, h, bands, black;
	size_t in_bpl, out_bpl;
	double max_alpha;
	double ink[kFlattenMaxBands - 1]; /* the background in the working format (exact in a double) */
};

#ifdef __CUDA_ARCH__
#define FL_FMUL(a, b) __fmul_rn((a), (b))
#define FL_FADD(a, b) __fadd_rn((a), (b))
#define FL_DMUL(a, b) __dmul_rn((a), (b))
#define FL_DADD(a, b) __dadd_rn((a), (b))
#define FL_DSUB(a, b) __dsub_rn((a), (b))
#define FL_DDIV(a, b) __ddiv_rn((a), (b))
#define FL_D2F(a) __double2float_rn(a)
#else
/* host twin: this translation unit's host code is compiled without FMA contraction (x86-64 baseline) */
#define FL_FMUL(a, b) ((float) (a) * (float) (b))
#define FL_FADD(a, b) ((float) (a) + (float) (b))
#define FL_DMUL(a, b) ((double) (a) * (double) (b))
#define FL_DADD(a, b) ((double) (a) + (double) (b))
#define FL_DSUB(a, b) ((double) (a) - (double) (b))
#define FL_DDIV(a, b) ((double) (a) / (double) (b))
#define FL_D2F(a) ((float) (a))
#endif

/* CAST_FLOAT_INT(double -> T): VIPS_CLIP in double, then C truncation (cast.c:123-131, 231-238) */
template <typename T> struct FlattenLimits;
template <> struct FlattenLimits<uint8_t> { static constexpr double lo = 0, hi = UCHAR_MAX; };
template <> struct FlattenLimits<int8_t> { static constexpr double lo = SCHAR_MIN, hi = SCHAR_MAX; };
template <> struct FlattenLimits<uint16_t> { static constexpr double lo = 0, hi = USHRT_MAX; };
template <> struct FlattenLimits<int16_t> { static constexpr double lo = SHRT_MIN, hi = SHRT_MAX; };
template <> struct FlattenLimits<uint32_t> { static constexpr double lo = 0, hi = UINT_MAX; };
template <> struct FlattenLimits<int32_t> { static constexpr double lo = INT_MIN, hi = INT_MAX; };

template <typename T>
__host__ __device__ __forceinline__ T
flatten_cast(double v)
{
	const double lo = FlattenLimits<T>::lo, hi = FlattenLimits<T>::hi;
	v = v < lo ? lo : (v > hi ? hi : v);
	return (T) v;
}
template <>
__host__ __device__ __forceinline__ float
flatten_cast<float>(double v)
{
	return FL_D2F(v);
}

/* entry i of the two uchar LUTs */
__host__ __device__ __forceinline__ void
flatten_lut_entry(double max_alpha, int i, float *fa, float *fn)
{
	*fa = FL_D2F(FL_DDIV((double) i, max_alpha));
	*fn = FL_D2F(FL_DDIV(FL_DSUB(max_alpha, (double) i), max_alpha));
}

/* one pixel: p[nb + 1] -> q[nb], nb = bands - 1 */
template <typename T, int MODE>
__host__ __device__ __forceinline__ void
flatten_pixel(const FlattenDev &P, const float *lut_a, const float *lut_n, const T *p, T *q, const int nb)
{
	if constexpr (MODE == FM_UCHAR) {
		const int a = (int) p[nb];
		const float fa = lut_a[a], fn = lut_n[a];
		for (int b = 0; b < nb; b++) {
			float v = FL_FMUL((float) (int) p[b], fa);
			if (!P.black)
				v = FL_FADD(v, FL_FMUL((float) P.ink[b], fn));
			q[b] = (T) (int) v;
		}
	}
	else if constexpr (MODE == FM_DOUBLE_LOOPS) {
		/* VIPS_FLATTEN[_BLACK]_FLOAT(TYPE): TYPE alpha; TYPE nalpha = max_alpha - alpha */
		const T alpha = p[nb];
		const T nalpha = (T) FL_DSUB(P.max_alpha, (double) alpha);
		for (int b = 0; b < nb; b++) {
			double v = FL_DMUL((double) p[b], (double) alpha);
			if (!P.black)
				v = FL_DADD(v, FL_DMUL(P.ink[b], (double) nalpha));
			v = FL_DDIV(v, P.max_alpha);
			if constexpr (sizeof(T) == 2)
				q[b] = (T) (int) v; /* ushort: 0 <= v <= 65535, C truncation */
			else
				q[b] = flatten_cast<float>(v);
		}
	}
	else {
		/* cast to double, VIPS_FLATTEN[_BLACK]_FLOAT(double), cast back */
		const double alpha = (double) p[nb];
		const double nalpha = FL_DSUB(P.max_alpha, alpha);
		for (int b = 0; b < nb; b++) {
			double v = FL_DMUL((double) p[b], alpha);
			if (!P.black)
				v = FL_DADD(v, FL_DMUL(P.ink[b], nalpha));
			q[b] = flatten_cast<T>(FL_DDIV(v, P.max_alpha));
		}
	}
}

/* four RGBA uchar pixels held in four little-endian words -> three words of RGB */
__host__ __device__ __forceinline__ void
flatten_quad(const FlattenDev &P, const float *lut_a, const float *lut_n, const uint32_t in[4], uint32_t out[3])
{
	uint8_t q[12];
	for (int k = 0; k < 4; k++) {
		const uint8_t p[4] = {(uint8_t) in[k], (uint8_t) (in[k] >> 8), (uint8_t) (in[k] >> 16), (uint8_t) (in[k] >> 24)};
		flatten_pixel<uint8_t, FM_UCHAR>(P, lut_a, lut_n, p, q + 3 * k, 3);
	}
	for (int k = 0; k < 3; k++)
		out[k] = (uint32_t) q[4 * k] | ((uint32_t) q[4 * k + 1] << 8) | ((uint32_t) q[4 * k + 2] << 16) | ((uint32_t) q[4 * k + 3] << 24);
}

template <typename T, int MODE>
__global__ void __launch_bounds__(256)
flatten_kernel(const __grid_constant__ FlattenDev P, const unsigned char *__restrict__ in, unsigned char *__restrict__ out)
{
	__shared__ float lut_a[256], lut_n[256];
	if (MODE == FM_UCHAR) {
		for (int i = threadIdx.x; i < 256; i += blockDim.x)
			flatten_lut_entry(P.max_alpha, i, lut_a + i, lut_n + i);
		__syncthreads();
	}
	for (int y = blockIdx.y; y < P.h; y += gridDim.y) {
		const T *p = reinterpret_cast<const T *>(in + (size_t) y * P.in_bpl);
		T *q = reinterpret_cast<T *>(out + (size_t) y * P.out_bpl);
		for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < P.w; x += gridDim.x * blockDim.x)
			flatten_pixel<T, MODE>(P, lut_a, lut_n, p + (size_t) x * P.bands, q + (size_t) x * (P.bands - 1), P.bands - 1);
	}
}

/* RGBA uchar rows of 4 n pixels, 16-byte aligned: four pixels per thread */
__global__ void __launch_bounds__(256)
flatten_u8x4_kernel(const __grid_constant__ FlattenDev P, const unsigned char *__restrict__ in, unsigned char *__restrict__ out)
{
	__shared__ float lut_a[256], lut_n[256];
	for (int i = threadIdx.x; i < 256; i += blockDim.x)
		flatten_lut_entry(P.max_alpha, i, lut_a + i, lut_n + i);
	__syncthreads();
	const int quads = P.w / 4;
	for (int y = blockIdx.y; y < P.h; y += gridDim.y) {
		const uint4 *p = reinterpret_cast<const uint4 *>(in + (size_t) y * P.in_bpl);
		uint32_t *q = reinterpret_cast<uint32_t *>(out + (size_t) y * P.out_bpl);
		for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < quads; t += gridDim.x * blockDim.x) {
			const uint4 v = __ldg(p + t);
			const uint32_t w[4] = {v.x, v.y, v.z, v.w};
			uint32_t o[3];
			flatten_quad(P, lut_a, lut_n, w, o);
			q[3 * t] = o[0];
			q[3 * t + 1] = o[1];
			q[3 * t + 2] = o[2];
		}
	}
}

double
format_max(int fmt)
{
	/* vips_image_get_format_max, iofuncs/header.c:440-473 */
	switch (fmt) {
	case VB200_FORMAT_UCHAR: return UCHAR_MAX;
	case VB200_FORMAT_CHAR: return SCHAR_MAX;
	case VB200_FORMAT_USHORT: return USHRT_MAX;
	case VB200_FORMAT_SHORT: return SHRT_MAX;
	case VB200_FORMAT_UINT: return UINT_MAX;
	case VB200_FORMAT_INT: return INT_MAX;
	default: return 3.40282346638528859812e+38;
	}
}

/* everything vips_flatten_build decides before a pixel moves: mode, black, max_alpha, ink.  -1 with the error set */
int
flatten_plan(const char *domain, int bands, int fmt, int type, const double *background, int n, double max_alpha, FlattenDev *P,
	int *mode)
{
	if (bands < 2 || bands > kFlattenMaxBands) {
		error(domain, "%d bands not supported on the device path", bands);
		return -1;
	}
	if (fmt < VB200_FORMAT_UCHAR || fmt > VB200_FORMAT_FLOAT) {
		error(domain, "band format %d not supported on the device path", fmt);
		return -1;
	}
	if (max_alpha <= 0)
		max_alpha = interpretation_max_alpha(type); /* flatten.c:454-455 */
	static const double zero = 0.0;
	if (!background || n < 1) {
		background = &zero; /* vips_flatten_init: background = {0} */
		n = 1;
	}
	P->black = 1;
	for (int i = 0; i < n; i++)
		if (background[i] != 0.0)
			P->black = 0;
	if (!P->black && n != 1 && n != bands - 1) {
		error(domain, "vector must have 1 or %d elements", bands - 1); /* vips_linear's check under vips__vector_to_ink */
		return -1;
	}
	P->bands = bands;
	P->max_alpha = max_alpha;
	const bool isint = fmt != VB200_FORMAT_FLOAT;
	if (isint && max_alpha < format_max(fmt))
		*mode = FM_WIDE;
	else if (fmt == VB200_FORMAT_UCHAR)
		*mode = FM_UCHAR;
	else if (fmt == VB200_FORMAT_FLOAT || (fmt == VB200_FORMAT_USHORT && max_alpha == 65535.0))
		*mode = FM_DOUBLE_LOOPS;
	else {
		error(domain, "band format %d with max_alpha %g not supported on the device path", fmt, max_alpha);
		return -1;
	}
	for (int b = 0; b < bands - 1; b++) {
		/* vips__vector_to_ink: black -> vips_linear (float output: (float) bg) -> vips_cast to the working format */
		const double f = (double) (float) background[n == 1 ? 0 : b];
		double v = f;
		if (*mode == FM_UCHAR)
			v = (double) flatten_cast<uint8_t>(f);
		else if (*mode == FM_DOUBLE_LOOPS && fmt == VB200_FORMAT_USHORT)
			v = (double) flatten_cast<uint16_t>(f);
		P->ink[b] = v; /* FM_WIDE: double; float images: the float itself */
	}
	return 0;
}

bool
flatten_can_x4(const FlattenDev &P, int mode, const void *in, const void *out)
{
	return mode == FM_UCHAR && P.bands == 4 && P.w % 4 == 0 && P.in_bpl % 16 == 0 && P.out_bpl % 4 == 0 &&
		(uintptr_t) in % 16 == 0 && (uintptr_t) out % 4 == 0;
}

#define FLATTEN_WIDE_SWITCH(FMT, CALL) \
	switch (FMT) { \
	case VB200_FORMAT_UCHAR: CALL(uint8_t, FM_WIDE); break; \
	case VB200_FORMAT_CHAR: CALL(int8_t, FM_WIDE); break; \
	case VB200_FORMAT_USHORT: CALL(uint16_t, FM_WIDE); break; \
	case VB200_FORMAT_SHORT: CALL(int16_t, FM_WIDE); break; \
	case VB200_FORMAT_UINT: CALL(uint32_t, FM_WIDE); break; \
	default: CALL(int32_t, FM_WIDE); break; \
	}

template <typename T, int MODE>
void
flatten_host_rows(const FlattenDev &P, const unsigned char *in, unsigned char *out)
{
	float lut_a[256], lut_n[256];
	for (int i = 0; i < 256; i++)
		flatten_lut_entry(P.max_alpha, i, lut_a + i, lut_n + i);
	for (int y = 0; y < P.h; y++) {
		const T *p = reinterpret_cast<const T *>(in + (size_t) y * P.in_bpl);
		T *q = reinterpret_cast<T *>(out + (size_t) y * P.out_bpl);
		for (int x = 0; x < P.w; x++)
			flatten_pixel<T, MODE>(P, lut_a, lut_n, p + (size_t) x * P.bands, q + (size_t) x * (P.bands - 1), P.bands - 1);
	}
}

void
flatten_host_x4(const FlattenDev &P, const unsigned char *in, unsigned char *out)
{
	float lut_a[256], lut_n[256];
	for (int i = 0; i < 256; i++)
		flatten_lut_entry(P.max_alpha, i, lut_a + i, lut_n + i);
	for (int y = 0; y < P.h; y++)
		for (int t = 0; t < P.w / 4; t++) {
			uint32_t w[4], o[3];
			memcpy(w, in + (size_t) y * P.in_bpl + 16 * (size_t) t, 16);
			flatten_quad(P, lut_a, lut_n, w, o);
			memcpy(out + (size_t) y * P.out_bpl + 12 * (size_t) t, o, 12);
		}
}

} // namespace

int
dev_flatten(const char *domain, const DevImage &in, DevImage *out, const double *background, int n, double max_alpha, cudaStream_t s)
{
	if (in.bands == 1) {
		/* flatten.c:445-446: a copy */
		if (dev_image_new(domain, out, in.w, in.h, 1, in.fmt, in.type, s))
			return -1;
		VB200_CUDA(domain, cudaMemcpy2DAsync(out->data, out->bpl, in.data, in.bpl, (size_t) in.w * format_sizeof(in.fmt), in.h,
			cudaMemcpyDeviceToDevice, s));
		return 0;
	}
	FlattenDev P;
	int mode = 0;
	if (flatten_plan(domain, in.bands, in.fmt, in.type, background, n, max_alpha, &P, &mode))
		return -1;
	if (dev_image_new(domain, out, in.w, in.h, in.bands - 1, in.fmt, in.type, s))
		return -1;
	P.w = in.w;
	P.h = in.h;
	P.in_bpl = in.bpl;
	P.out_bpl = out->bpl;
	const unsigned char *pi = (const unsigned char *) in.data;
	unsigned char *po = (unsigned char *) out->data;
	const int rows = in.h < 1184 ? in.h : 1184; /* 8 CTAs of rows per SM at most; the kernels stride over the rest */
	if (flatten_can_x4(P, mode, pi, po)) {
		const dim3 grid((in.w / 4 + 255) / 256, rows);
		flatten_u8x4_kernel<<<grid, 256, 0, s>>>(P, pi, po);
	}
	else {
		const dim3 grid((in.w + 255) / 256, rows);
#define CALL(T, M) flatten_kernel<T, M><<<grid, 256, 0, s>>>(P, pi, po)
		if (mode == FM_WIDE) {
			FLATTEN_WIDE_SWITCH(in.fmt, CALL)
		}
		else if (mode == FM_UCHAR)
			CALL(uint8_t, FM_UCHAR);
		else if (in.fmt == VB200_FORMAT_USHORT)
			CALL(uint16_t, FM_DOUBLE_LOOPS);
		else
			CALL(float, FM_DOUBLE_LOOPS);
#undef CALL
	}
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
		return cuda_fail(domain, e, "flatten_kernel");
	count_launch();
	return 0;
}

} // namespace vb200

using namespace vb200;

/* test hook, host only: flatten.cu's per-pixel code on the CPU over packed host arrays; x4 != 0 asks for the
 * four-pixels-per-thread form (-1 if the image does not qualify)
 */
extern "C" int
vb200_debug_flatten_host(const void *in, int width, int height, int bands, int band_format, int interpretation, const double *background,
	int n, double max_alpha, int x4, void *out)
{
	const char *domain = "flatten";
	if (!in || !out) {
		error(domain, "null argument");
		return -1;
	}
	const size_t es = format_sizeof(band_format);
	if (bands == 1) {
		memcpy(out, in, (size_t) width * height * es);
		return 0;
	}
	FlattenDev P;
	int mode = 0;
	if (flatten_plan(domain, bands, band_format, interpretation, background, n, max_alpha, &P, &mode))
		return -1;
	P.w = width;
	P.h = height;
	P.in_bpl = (size_t) width * bands * es;
	P.out_bpl = (size_t) width * (bands - 1) * es;
	const unsigned char *pi = (const unsigned char *) in;
	unsigned char *po = (unsigned char *) out;
	if (x4) {
		if (!flatten_can_x4(P, mode, nullptr, nullptr)) {
			error(domain, "not a four-pixel case");
			return -1;
		}
		flatten_host_x4(P, pi, po);
		return 0;
	}
#define CALL(T, M) flatten_host_rows<T, M>(P, pi, po)
	if (mode == FM_WIDE) {
		FLATTEN_WIDE_SWITCH(band_format, CALL)
	}
	else if (mode == FM_UCHAR)
		CALL(uint8_t, FM_UCHAR);
	else if (band_format == VB200_FORMAT_USHORT)
		CALL(uint16_t, FM_DOUBLE_LOOPS);
	else
		CALL(float, FM_DOUBLE_LOOPS);
#undef CALL
	return 0;
}
