/* affine.cu -- the upsizing half of vips_resize: a scale-only vips_affine with the
 * nearest / bilinear / bicubic interpolators.
 *
 * reference:
 *   resample/resize.c:116-132,233-307   interpolator per kernel, idx/idy = 0.5 * (1 - 1 / scale), the affine calls
 *   resample/affine.c:412-605           transform, oarea = ROUND_INT(forward rect), embed by window + 1, idx -= 1
 *   resample/affine.c:227-410           vips_affine_gen: ix advanced by repeated addition of ddx along each rect row
 *   resample/transform.c:48-70          inverse: tmp = 1 / det; ia = tmp * d; id = tmp * a
 *   resample/interpolate.c:334-349      nearest;  :433-482 bilinear (12-bit fixed point for 8/16-bit ints, double else)
 *   resample/bicubic.cpp:106-405,487-645, templates.h:150-305   bicubic (fixed point for 8-bit, double tables else)
 *
 * A scale-only affine (b = c = 0) separates: the column coordinate depends only
 * on x (and on the rect it starts in: FATSTRIP rects are full width, so it is
 * one sequence per row starting at x = 0) and the row coordinate only on y.
 * The host builds both sequences with the reference's own double additions and
 * uploads them; one thread interpolates one output pixel.
 */
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "vb200_internal.h"

namespace vb200 {

namespace {

enum { INTERP_NEAREST = 0, INTERP_BILINEAR = 1, INTERP_BICUBIC = 2 };

struct AffineDev {
	const double *ixs; /* [OW] column coordinate in the embedded image */
	const double *iys; /* [OH] */
	const double *cf;  /* [65][4] bicubic, double */
	const int *ci;	   /* [65][4] bicubic, 12-bit fixed point */
	int w, h, bands, pad; /* source; pad = window_offset + 1 */
	int OW, OH;
	size_t in_bpl, out_bpl;
	int ile, iri, ito, ibo; /* clip against iarea, affine.c:318-323 */
	int interp;
};

template <typename T> struct Kind;
template <> struct Kind<uint8_t> { static constexpr int k = 0; static constexpr double lo = 0, hi = 255; };
template <> struct Kind<int8_t> { static constexpr int k = 1; static constexpr double lo = -128, hi = 127; };
template <> struct Kind<uint16_t> { static constexpr int k = 2; static constexpr double lo = 0, hi = 65535; };
template <> struct Kind<int16_t> { static constexpr int k = 2; static constexpr double lo = -32768, hi = 32767; };
template <> struct Kind<uint32_t> { static constexpr int k = 3; static constexpr double lo = 0, hi = 2147483647.0; };
template <> struct Kind<int32_t> { static constexpr int k = 3; static constexpr double lo = -2147483648.0, hi = 2147483647.0; };
template <> struct Kind<float> { static constexpr int k = 4; };

__device__ __forceinline__ int
ufr(int v)
{
	return (v + (VB200_INTERPOLATE_SCALE >> 1)) >> VB200_INTERPOLATE_SHIFT;
}

__device__ __forceinline__ int
sfr(int v)
{
	const int round_by = v >= 0 ? (VB200_INTERPOLATE_SCALE >> 1) : -(VB200_INTERPOLATE_SCALE >> 1);
	return (v + round_by) >> VB200_INTERPOLATE_SHIFT;
}

/* The common upsize: uchar, 4 bands, bicubic.  One thread per output pixel, all four channels at
 * once: the 4 x 4 window is 16 32-bit loads through 4 clamped column offsets and 4 clamped row
 * pointers, pixels are byte-transposed pairwise (PRMT) so that dp2a does two taps of one channel
 * per instruction.  Same two-stage fixed-point sums as bicubic_unsigned_int_tab (bicubic.cpp:106-166).
 */
/* vips_zoom: out(x, y) = in(x / xfac, y / yfac), pixels of ps bytes */
__global__ void __launch_bounds__(256)
zoom_kernel(const char *__restrict__ in, size_t in_bpl, char *__restrict__ out, size_t out_bpl, int ow, int oh, int ps, int xf,
	int yf)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= ow)
		return;
	for (int y = blockIdx.y; y < oh; y += gridDim.y) {
		const char *p = in + (size_t) (y / yf) * in_bpl + (size_t) (x / xf) * ps;
		char *q = out + (size_t) y * out_bpl + (size_t) x * ps;
		for (int i = 0; i < ps; i++)
			q[i] = p[i];
	}
}

__device__ __forceinline__ int
dp2a_lo_s(unsigned coef, unsigned bytes, int acc)
{
	int d;
	asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(coef), "r"(bytes), "r"(acc));
	return d;
}
__device__ __forceinline__ int
dp2a_hi_s(unsigned coef, unsigned bytes, int acc)
{
	int d;
	asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(coef), "r"(bytes), "r"(acc));
	return d;
}

__device__ __forceinline__ void
affine_bicubic_u8x4_px(const AffineDev &P, const uint8_t *__restrict__ in, uint8_t *__restrict__ out, int x, int y)
{
	const double ix = P.ixs[x];
	const double iy = P.iys[y];
	unsigned *q = (unsigned *) ((char *) out + (size_t) y * P.out_bpl) + x;
	const int fx = (int) floor(ix);
	const int fy = (int) floor(iy);
	if (!(fx >= P.ile && fx <= P.iri && fy >= P.ito && fy <= P.ibo)) {
		*q = 0;
		return;
	}
	const int xi = (int) ix, yi = (int) iy;
	const int sx = (int) __dmul_rn(__dmul_rn(ix, (double) VB200_TRANSFORM_SCALE), 2.0);
	const int sy = (int) __dmul_rn(__dmul_rn(iy, (double) VB200_TRANSFORM_SCALE), 2.0);
	const int tx = ((sx & (VB200_TRANSFORM_SCALE * 2 - 1)) + 1) >> 1;
	const int ty = ((sy & (VB200_TRANSFORM_SCALE * 2 - 1)) + 1) >> 1;
	const int4 cx = __ldg((const int4 *) (P.ci + tx * 4));
	const int4 cy = __ldg((const int4 *) (P.ci + ty * 4));
	const unsigned cx01 = ((unsigned) cx.y << 16) | ((unsigned) cx.x & 0xffffu);
	const unsigned cx23 = ((unsigned) cx.w << 16) | ((unsigned) cx.z & 0xffffu);
	int col[4];
#pragma unroll
	for (int i = 0; i < 4; i++)
		col[i] = max(0, min(xi - 1 + i - P.pad, P.w - 1));
	const int cyv[4] = {cy.x, cy.y, cy.z, cy.w};
	int acc[4] = {0, 0, 0, 0};
#pragma unroll
	for (int j = 0; j < 4; j++) {
		const int sy2 = max(0, min(yi - 1 + j - P.pad, P.h - 1));
		const unsigned *row = (const unsigned *) (in + (size_t) sy2 * P.in_bpl);
		const unsigned p0 = __ldg(row + col[0]), p1 = __ldg(row + col[1]), p2 = __ldg(row + col[2]), p3 = __ldg(row + col[3]);
		const unsigned a01 = __byte_perm(p0, p1, 0x5140); /* [p0.c0 p1.c0 p0.c1 p1.c1] */
		const unsigned b01 = __byte_perm(p0, p1, 0x7362); /* [p0.c2 p1.c2 p0.c3 p1.c3] */
		const unsigned a23 = __byte_perm(p2, p3, 0x5140);
		const unsigned b23 = __byte_perm(p2, p3, 0x7362);
		const int r0 = ufr(dp2a_lo_s(cx23, a23, dp2a_lo_s(cx01, a01, 0)));
		const int r1 = ufr(dp2a_hi_s(cx23, a23, dp2a_hi_s(cx01, a01, 0)));
		const int r2 = ufr(dp2a_lo_s(cx23, b23, dp2a_lo_s(cx01, b01, 0)));
		const int r3 = ufr(dp2a_hi_s(cx23, b23, dp2a_hi_s(cx01, b01, 0)));
		acc[0] += cyv[j] * r0;
		acc[1] += cyv[j] * r1;
		acc[2] += cyv[j] * r2;
		acc[3] += cyv[j] * r3;
	}
	unsigned v = 0;
#pragma unroll
	for (int c = 0; c < 4; c++)
		v |= (unsigned) max(0, min(ufr(acc[c]), 255)) << (8 * c);
	*q = v;
}

__global__ void __launch_bounds__(256)
affine_bicubic_u8x4_kernel(const __grid_constant__ AffineDev P, const uint8_t *__restrict__ in, uint8_t *__restrict__ out)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= P.OW)
		return;
	for (int y = blockIdx.y; y < P.OH; y += gridDim.y)
		affine_bicubic_u8x4_px(P, in, out, x, y);
}

/* The same pixels, separably.  vips_interpolate_bicubic's integer path is two-stage -- four horizontal sums
 * rounded to integers, then the vertical sum of those (bicubic_unsigned_int_tab, bicubic.cpp:106-166) -- so
 * the horizontal stage of an input row is shared by every output row that samples it (two of them at x2).
 * One CTA owns a 64 x 32 output tile: it runs the horizontal stage once per input row the tile touches
 * (at most 32 + 3 when the vertical scale is >= 1) into shared memory as short4, then each output pixel
 * is four 64-bit shared loads and sixteen multiply-adds.  ~65 instead of ~225 instructions per output pixel.
 */
constexpr int kSepTW = 64, kSepTH = 32, kSepRows = kSepTH + 4;

template <bool LOOP>
__global__ void __launch_bounds__(256)
affine_bicubic_u8x4_sep_kernel(const __grid_constant__ AffineDev P, const uint8_t *__restrict__ in, uint8_t *__restrict__ out)
{
	__shared__ short4 sh[kSepRows][kSepTW];
	const int t = threadIdx.x;
	const int lx = t & (kSepTW - 1), ly = t >> 6; /* 64 columns x 4 row phases */
	const int x0 = blockIdx.x * kSepTW;
	const int x = min(x0 + lx, P.OW - 1);

	/* this thread's column: the horizontal coordinates never change down the tile */
	const double ix = P.ixs[x];
	const int fx = (int) floor(ix);
	const bool x_in = fx >= P.ile && fx <= P.iri;
	const int xi = (int) ix;
	const int sx = (int) __dmul_rn(__dmul_rn(ix, (double) VB200_TRANSFORM_SCALE), 2.0);
	const int tx = ((sx & (VB200_TRANSFORM_SCALE * 2 - 1)) + 1) >> 1;
	const int4 cx = __ldg((const int4 *) (P.ci + tx * 4));
	const unsigned cx01 = ((unsigned) cx.y << 16) | ((unsigned) cx.x & 0xffffu);
	const unsigned cx23 = ((unsigned) cx.w << 16) | ((unsigned) cx.z & 0xffffu);
	int col[4];
#pragma unroll
	for (int i = 0; i < 4; i++)
		col[i] = max(0, min(xi - 1 + i - P.pad, P.w - 1));

	/* the whole CTA walks its tiles down the image together through the staged rows */
	int y0 = blockIdx.y * kSepTH;
	do {
		if (y0 != (int) blockIdx.y * kSepTH)
			__syncthreads(); /* the previous tile's rows have been read */
		const int y_last = min(y0 + kSepTH, P.OH) - 1;

		/* the input rows this tile samples */
		const int r_lo = (int) P.iys[y0] - 1;
		const int nrows = min((int) P.iys[y_last] + 2 - r_lo + 1, kSepRows);
		for (int rr = ly; rr < nrows; rr += 4) {
			const int sy2 = max(0, min(r_lo + rr - P.pad, P.h - 1));
			const unsigned *row = (const unsigned *) (in + (size_t) sy2 * P.in_bpl);
			const unsigned p0 = __ldg(row + col[0]), p1 = __ldg(row + col[1]), p2 = __ldg(row + col[2]), p3 = __ldg(row + col[3]);
			const unsigned a01 = __byte_perm(p0, p1, 0x5140); /* [p0.c0 p1.c0 p0.c1 p1.c1] */
			const unsigned b01 = __byte_perm(p0, p1, 0x7362); /* [p0.c2 p1.c2 p0.c3 p1.c3] */
			const unsigned a23 = __byte_perm(p2, p3, 0x5140);
			const unsigned b23 = __byte_perm(p2, p3, 0x7362);
			short4 r;
			r.x = (short) ufr(dp2a_lo_s(cx23, a23, dp2a_lo_s(cx01, a01, 0)));
			r.y = (short) ufr(dp2a_hi_s(cx23, a23, dp2a_hi_s(cx01, a01, 0)));
			r.z = (short) ufr(dp2a_lo_s(cx23, b23, dp2a_lo_s(cx01, b01, 0)));
			r.w = (short) ufr(dp2a_hi_s(cx23, b23, dp2a_hi_s(cx01, b01, 0)));
			sh[rr][lx] = r;
		}
		__syncthreads();

		if (x0 + lx >= P.OW)
			continue;
		for (int y = y0 + ly; y <= y_last; y += 4) {
			unsigned *q = (unsigned *) ((char *) out + (size_t) y * P.out_bpl) + x;
			const double iy = P.iys[y];
			const int fy = (int) floor(iy);
			if (!(x_in && fy >= P.ito && fy <= P.ibo)) {
				*q = 0;
				continue;
			}
			const int yi = (int) iy;
			const int sy = (int) __dmul_rn(__dmul_rn(iy, (double) VB200_TRANSFORM_SCALE), 2.0);
			const int ty = ((sy & (VB200_TRANSFORM_SCALE * 2 - 1)) + 1) >> 1;
			const int4 cy = __ldg((const int4 *) (P.ci + ty * 4));
			const int cyv[4] = {cy.x, cy.y, cy.z, cy.w};
			const int base = yi - 1 - r_lo;
			int acc[4] = {0, 0, 0, 0};
#pragma unroll
			for (int j = 0; j < 4; j++) {
				const short4 r = sh[base + j][lx];
				acc[0] += cyv[j] * r.x;
				acc[1] += cyv[j] * r.y;
				acc[2] += cyv[j] * r.z;
				acc[3] += cyv[j] * r.w;
			}
			unsigned v = 0;
#pragma unroll
			for (int c = 0; c < 4; c++)
				v |= (unsigned) max(0, min(ufr(acc[c]), 255)) << (8 * c);
			*q = v;
		}
	} while (LOOP && (y0 += gridDim.y * kSepTH) < P.OH);
}

template <typename T>
__device__ __forceinline__ void
affine_scale_px(const AffineDev &P, const T *__restrict__ in, T *__restrict__ out, int x, int y)
{
	const double ix = P.ixs[x];
	const double iy = P.iys[y];
	T *q = (T *) ((char *) out + (size_t) y * P.out_bpl) + (size_t) x * P.bands;
	const int fx = (int) floor(ix);
	const int fy = (int) floor(iy);
	if (!(fx >= P.ile && fx <= P.iri && fy >= P.ito && fy <= P.ibo)) {
		for (int z = 0; z < P.bands; z++)
			q[z] = (T) 0;
		return;
	}

	auto at = [&](int X, int Y, int z) -> T {
		const int sx = max(0, min(X - P.pad, P.w - 1));
		const int sy = max(0, min(Y - P.pad, P.h - 1));
		return ((const T *) ((const char *) in + (size_t) sy * P.in_bpl))[(size_t) sx * P.bands + z];
	};

	const int xi = (int) ix, yi = (int) iy;
	if (P.interp == INTERP_NEAREST) {
		for (int z = 0; z < P.bands; z++)
			q[z] = at(xi, yi, z);
		return;
	}
	if (P.interp == INTERP_BILINEAR) {
		if constexpr (Kind<T>::k <= 2) {
			/* BILINEAR_INT */
			const int X = (int) __dmul_rn(__dsub_rn(ix, (double) xi), (double) VB200_INTERPOLATE_SCALE);
			const int Y = (int) __dmul_rn(__dsub_rn(iy, (double) yi), (double) VB200_INTERPOLATE_SCALE);
			const int Yd = VB200_INTERPOLATE_SCALE - Y;
			const int c4 = (Y * X) >> VB200_INTERPOLATE_SHIFT;
			const int c2 = (Yd * X) >> VB200_INTERPOLATE_SHIFT;
			const int c3 = Y - c4;
			const int c1 = Yd - c2;
			for (int z = 0; z < P.bands; z++)
				q[z] = (T) ((c1 * (int) at(xi, yi, z) + c2 * (int) at(xi + 1, yi, z) + c3 * (int) at(xi, yi + 1, z) +
								c4 * (int) at(xi + 1, yi + 1, z) + (1 << VB200_INTERPOLATE_SHIFT) / 2) >>
					VB200_INTERPOLATE_SHIFT);
		}
		else {
			/* BILINEAR_FLOAT: coefficients and sum in double, evaluation order as written */
			const double X = __dsub_rn(ix, (double) xi);
			const double Y = __dsub_rn(iy, (double) yi);
			const double Yd = __dsub_rn(1.0, Y);
			const double c4 = __dmul_rn(Y, X);
			const double c2 = __dmul_rn(Yd, X);
			const double c3 = __dsub_rn(Y, c4);
			const double c1 = __dsub_rn(Yd, c2);
			for (int z = 0; z < P.bands; z++) {
				double v = __dmul_rn(c1, (double) at(xi, yi, z));
				v = __dadd_rn(v, __dmul_rn(c2, (double) at(xi + 1, yi, z)));
				v = __dadd_rn(v, __dmul_rn(c3, (double) at(xi, yi + 1, z)));
				v = __dadd_rn(v, __dmul_rn(c4, (double) at(xi + 1, yi + 1, z)));
				q[z] = (T) v;
			}
		}
		return;
	}

	/* bicubic */
	const int sx = (int) __dmul_rn(__dmul_rn(ix, (double) VB200_TRANSFORM_SCALE), 2.0);
	const int sy = (int) __dmul_rn(__dmul_rn(iy, (double) VB200_TRANSFORM_SCALE), 2.0);
	const int tx = ((sx & (VB200_TRANSFORM_SCALE * 2 - 1)) + 1) >> 1;
	const int ty = ((sy & (VB200_TRANSFORM_SCALE * 2 - 1)) + 1) >> 1;
	for (int z = 0; z < P.bands; z++) {
		if constexpr (Kind<T>::k <= 1) {
			const int *cx = P.ci + tx * 4, *cy = P.ci + ty * 4;
			int r[4];
			for (int j = 0; j < 4; j++) {
				const int sum = cx[0] * (int) at(xi - 1, yi - 1 + j, z) + cx[1] * (int) at(xi, yi - 1 + j, z) +
					cx[2] * (int) at(xi + 1, yi - 1 + j, z) + cx[3] * (int) at(xi + 2, yi - 1 + j, z);
				r[j] = Kind<T>::k == 0 ? ufr(sum) : sfr(sum);
			}
			const int sum = cy[0] * r[0] + cy[1] * r[1] + cy[2] * r[2] + cy[3] * r[3];
			int v = Kind<T>::k == 0 ? ufr(sum) : sfr(sum);
			v = max((int) Kind<T>::lo, min(v, (int) Kind<T>::hi));
			q[z] = (T) v;
		}
		else {
			const double *cx = P.cf + tx * 4, *cy = P.cf + ty * 4;
			double r[4];
			for (int j = 0; j < 4; j++) {
				double v = __dmul_rn(cx[0], (double) at(xi - 1, yi - 1 + j, z));
				v = __dadd_rn(v, __dmul_rn(cx[1], (double) at(xi, yi - 1 + j, z)));
				v = __dadd_rn(v, __dmul_rn(cx[2], (double) at(xi + 1, yi - 1 + j, z)));
				v = __dadd_rn(v, __dmul_rn(cx[3], (double) at(xi + 2, yi - 1 + j, z)));
				/* bicubic_float<float>: every cubic_float<T> returns T */
				r[j] = Kind<T>::k == 4 ? (double) (float) v : v;
			}
			double v = __dmul_rn(cy[0], r[0]);
			v = __dadd_rn(v, __dmul_rn(cy[1], r[1]));
			v = __dadd_rn(v, __dmul_rn(cy[2], r[2]));
			v = __dadd_rn(v, __dmul_rn(cy[3], r[3]));
			if constexpr (Kind<T>::k == 4)
				q[z] = (T) (float) v;
			else {
				/* VIPS_CLIP in double, then the C conversion */
				const double m = Kind<T>::hi < v ? Kind<T>::hi : v;
				v = Kind<T>::lo > m ? Kind<T>::lo : m;
				q[z] = (T) v;
			}
		}
	}
}

template <typename T, bool LOOP>
__global__ void __launch_bounds__(256)
affine_scale_kernel(const __grid_constant__ AffineDev P, const T *__restrict__ in, T *__restrict__ out)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= P.OW)
		return;
	int y = blockIdx.y;
	do
		affine_scale_px<T>(P, in, out, x, y);
	while (LOOP && (y += gridDim.y) < P.OH);
}

#define VB200_ROUND_INT(R) ((int) ((R) > 0 ? ((R) + 0.5) : ((R) -0.5)))

struct AffineKey {
	int dev, OW, OH, ol, ot, window_offset;
	double ia, id, tidx, tidy;
};
struct AffineEntry {
	AffineKey key;
	void *block;
	size_t nd;
	unsigned long long stamp;
};
std::mutex g_affine_lock;
std::vector<AffineEntry> g_affine_cache;
unsigned long long g_affine_clock = 0;

} // namespace

/* vips_affine(in, a, 0, 0, d, interpolate, idx, idy, extend COPY, premultiplied TRUE) */
int
dev_affine_scale(const char *domain, const DevImage &in, DevImage *out, double a, double d, int interp, double idx,
	double idy, cudaStream_t s)
{
	if (!format_is_supported(in.fmt)) {
		error(domain, "band format %d not supported on the device path", in.fmt);
		return -1;
	}
	/* vips__transform_calc_inverse */
	const double det = a * d;
	if (fabs(det) < 2.0 * 2.2250738585072014e-308) {
		error(domain, "singular or near-singular matrix");
		return -1;
	}
	const double tmp = 1.0 / det;
	const double ia = tmp * d, id = tmp * a;
	/* vips__transform_set_area: forward rect of (0, 0, w, h) with idx = idy = 0 */
	const double xs[2] = {a * 0.0 + 0.0 * 0.0 + 0.0, a * in.w + 0.0 * 0.0 + 0.0};
	const double ys[2] = {0.0 * 0.0 + d * 0.0 + 0.0, 0.0 * 0.0 + d * in.h + 0.0};
	const double left = std::min(xs[0], xs[1]), right = std::max(xs[0], xs[1]);
	const double top = std::min(ys[0], ys[1]), bottom = std::max(ys[0], ys[1]);
	const int ol = VB200_ROUND_INT(left), ot = VB200_ROUND_INT(top);
	const int OW = VB200_ROUND_INT(right - left), OH = VB200_ROUND_INT(bottom - top);
	if (OW <= 0 || OH <= 0) {
		error(domain, "image has shrunk to nothing");
		return -1;
	}
	const int window_size = interp == INTERP_BICUBIC ? 4 : (interp == INTERP_BILINEAR ? 2 : 1);
	const int window_offset = std::max(0, window_size / 2 - 1);
	const double tidx = idx - 1, tidy = idy - 1; /* the embed's one-pixel border, affine.c:533-534 */

	/* The coordinate and coefficient tables depend on the geometry only: a server resizing same-shaped frames
	 * builds and uploads them once (host loops + a pageable copy were as long as the kernel itself at 4K x2).
	 */
	void *block = nullptr;
	size_t nd = 0;
	{
		int dev = 0;
		VB200_CUDA(domain, cudaGetDevice(&dev));
		const AffineKey key{dev, OW, OH, ol, ot, window_offset, ia, id, tidx, tidy};
		std::lock_guard<std::mutex> lock(g_affine_lock);
		for (auto &e : g_affine_cache)
			if (memcmp(&e.key, &key, sizeof(key)) == 0) {
				block = e.block;
				nd = e.nd;
				e.stamp = ++g_affine_clock;
			}
		if (!block) {
		/* the coordinate sequences of vips_affine_gen (affine.c:325-400), ib = ic = 0, odx = ody = 0 */
		std::vector<double> host((((size_t) OW + OH + 65 * 4) + 1) & ~(size_t) 1); /* even: the int table after it stays 16-byte aligned */
		{
			const double ox = 0 + ol - 0.0;
			double ix = ia * ox + 0.0 * (0 + ot - 0.0);
			ix -= tidx;
			ix += window_offset;
			for (int x = 0; x < OW; x++) {
				host[x] = ix;
				ix += ia; /* ddx */
			}
			for (int y = 0; y < OH; y++) {
				const double oy = y + ot - 0.0;
				double iy = 0.0 * ox + id * oy;
				iy -= tidy;
				iy += window_offset;
				host[OW + y] = iy;
			}
		}
		/* bicubic tables: calculate_coefficients_catmull (templates.h:281-305), bicubic.cpp:636-644 */
		std::vector<int> ci(65 * 4);
		for (int t = 0; t <= VB200_TRANSFORM_SCALE; t++) {
			const double x = (float) t / VB200_TRANSFORM_SCALE;
			const double cr1 = 1. - x;
			const double cr2 = -.5 * x;
			const double cr3 = cr1 * cr2;
			const double cone = cr1 * cr3;
			const double cfou = x * cr3;
			const double cr4 = cfou - cone;
			const double ctwo = cr1 - cone + cr4;
			const double cthr = x - cfou - cr4;
			double *c = &host[(size_t) OW + OH + t * 4];
			c[0] = cone;
			c[1] = ctwo;
			c[2] = cthr;
			c[3] = cfou;
			for (int i = 0; i < 4; i++)
				ci[t * 4 + i] = c[i] * VB200_INTERPOLATE_SCALE;
		}

		nd = host.size() * sizeof(double);
		const size_t ni = ci.size() * sizeof(int);
		VB200_CUDA(domain, cudaMalloc(&block, nd + ni));
		/* synchronous copies: the entry may be used from any stream afterwards */
		VB200_CUDA(domain, cudaMemcpy(block, host.data(), nd, cudaMemcpyHostToDevice));
		VB200_CUDA(domain, cudaMemcpy((char *) block + nd, ci.data(), ni, cudaMemcpyHostToDevice));
		if (g_affine_cache.size() >= 16) {
			/* evict the least recently used (cudaFree waits for kernels still reading it) */
			size_t victim = 0;
			for (size_t i = 1; i < g_affine_cache.size(); i++)
				if (g_affine_cache[i].stamp < g_affine_cache[victim].stamp)
					victim = i;
			cudaFree(g_affine_cache[victim].block);
			g_affine_cache.erase(g_affine_cache.begin() + victim);
		}
		AffineEntry e;
		memset(&e.key, 0, sizeof(e.key));
		e.key = key;
		e.block = block;
		e.nd = nd;
		e.stamp = ++g_affine_clock;
		g_affine_cache.push_back(e);
		}
	}


	if (dev_image_new(domain, out, OW, OH, in.bands, in.fmt, in.type, s))
		return -1;
	AffineDev P;
	P.ixs = (const double *) block;
	P.iys = P.ixs + OW;
	P.cf = P.iys + OH;
	P.ci = (const int *) ((char *) block + nd);
	P.w = in.w;
	P.h = in.h;
	P.bands = in.bands;
	P.pad = window_offset + 1;
	P.OW = OW;
	P.OH = OH;
	P.in_bpl = in.bpl;
	P.out_bpl = out->bpl;
	P.ile = 0 + window_offset;
	P.ito = 0 + window_offset;
	P.iri = P.ile + in.w;
	P.ibo = P.ito + in.h;
	P.interp = interp;
	const dim3 grid = row_grid(OW, OH);
	const bool loop = rows_loop(OH);
#define AF(T) (loop ? affine_scale_kernel<T, true> : affine_scale_kernel<T, false>)<<<grid, 256, 0, s>>>(P, (const T *) in.data, (T *) out->data)
	const bool u8x4 = in.fmt == VB200_FORMAT_UCHAR && in.bands == 4 && interp == INTERP_BICUBIC && (in.bpl & 3) == 0 &&
		((uintptr_t) in.data & 3) == 0 && getenv("VB200_NO_AFFINE_X4") == nullptr;
	/* vertical scale >= 1: a tile of 32 output rows touches at most 35 input rows (the separable kernel's budget) */
	const bool sep = u8x4 && id <= 1.0 && getenv("VB200_NO_AFFINE_SEP") == nullptr;
	if (sep)
		(rows_loop((OH + kSepTH - 1) / kSepTH) ? affine_bicubic_u8x4_sep_kernel<true> : affine_bicubic_u8x4_sep_kernel<false>)<<<
			row_grid(OW, (OH + kSepTH - 1) / kSepTH, kSepTW), 256, 0, s>>>(P,
			(const uint8_t *) in.data, (uint8_t *) out->data);
	else if (u8x4)
		affine_bicubic_u8x4_kernel<<<grid, 256, 0, s>>>(P, (const uint8_t *) in.data, (uint8_t *) out->data);
	else
	switch (in.fmt) {
	case VB200_FORMAT_UCHAR: AF(uint8_t); break;
	case VB200_FORMAT_CHAR: AF(int8_t); break;
	case VB200_FORMAT_USHORT: AF(uint16_t); break;
	case VB200_FORMAT_SHORT: AF(int16_t); break;
	case VB200_FORMAT_UINT: AF(uint32_t); break;
	case VB200_FORMAT_INT: AF(int32_t); break;
	case VB200_FORMAT_FLOAT: AF(float); break;
	}
#undef AF
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
		return cuda_fail(domain, e, "affine kernel");
	count_launch();
	return 0;
}

/* the upsizing tail of vips_resize for a pure enlargement, resize.c:233-307 */
int
dev_resize_up(const char *domain, const DevImage &in, DevImage *out, double hscale, double vscale, int kernel,
	cudaStream_t s)
{
	const int interp = kernel == VB200_KERNEL_NEAREST ? INTERP_NEAREST
		: (kernel == VB200_KERNEL_LINEAR ? INTERP_BILINEAR : INTERP_BICUBIC);
	if (kernel == VB200_KERNEL_NEAREST && hscale == floor(hscale) && vscale == floor(vscale)) {
		/* vips_zoom (resize.c:263-271, conversion/zoom.c:95-227): every input pixel becomes an
		 * xfac x yfac block -- exact replication, not the nearest affine (whose coordinate is
		 * built by repeated addition of 1 / scale and can land one pixel low for scales like 3)
		 */
		const int xf = (int) floor(hscale), yf = (int) floor(vscale);
		if ((long long) in.w * xf > 100000000LL || (long long) in.h * yf > 100000000LL) {
			error(domain, "zoom factors too large");
			return -1;
		}
		if (dev_image_new(domain, out, in.w * xf, in.h * yf, in.bands, in.fmt, in.type, s))
			return -1;
		const int ps = (int) (format_sizeof(in.fmt) * in.bands);
		const dim3 grid = row_grid(out->w, out->h);
		zoom_kernel<<<grid, 256, 0, s>>>((const char *) in.data, in.bpl, (char *) out->data, out->bpl, out->w, out->h, ps, xf, yf);
		const cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess)
			return cuda_fail(domain, e, "zoom_kernel");
		count_launch();
		return 0;
	}
	const double idx = kernel == VB200_KERNEL_NEAREST ? 0.0 : 0.5 * (1.0 - 1.0 / hscale);
	const double idy = kernel == VB200_KERNEL_NEAREST ? 0.0 : 0.5 * (1.0 - 1.0 / vscale);
	double a, d;
	if (hscale > 1.0 && vscale > 1.0) {
		a = hscale;
		d = vscale;
	}
	else if (hscale > 1.0) {
		a = hscale;
		d = 1.0;
	}
	else {
		a = 1.0;
		d = vscale;
	}
	return dev_affine_scale(domain, in, out, a, d, interp, idx, idy, s);
}

} // namespace vb200
