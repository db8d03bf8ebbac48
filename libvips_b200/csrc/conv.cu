/* conv.cu -- vips_conv / vips_convsep / vips_gaussblur / vips_sharpen on the device.
 *
 * Arithmetic restated from the reference's generate functions:
 *   convf   convolution/convf.c:163-180     double sum = offset; sum += coeff[i] * p[off[i]]  (coeff = mask / scale,
 *                                           zeros squeezed, row-major tap order); float store
 *   convi   convolution/convi.c:698-717     int64 sum; ((sum + scale / 2) / scale) + offset, C truncating division, clip
 *           convolution/convi.c:721-739     float input through convi: double sum of int coefficients, / scale + offset
 *   convi (vector semantics, uchar)  convi_hwy.cpp:265-273   int32 sum = 1 << (exp - 1); sum += p * mant;
 *                                           clip((sum >> exp) + offset)   with the 8-bit-mantissa mask of
 *                                           vips_convi_intize (convi.c:931-1119)
 *   sharpen convolution/sharpen.c:116-168   out = clip(v1 + lut[(v1 & 0x7fff) - (v2 & 0x7fff) + 32768], 0, 32767)
 * Mask preparation (vips__image_intize convi.c:859-923, gaussmat create/gaussmat.c:93-170, the sharpen LUT
 * sharpen.c:227-257) runs on the host exactly as the reference's build() does.
 * The vips_embed(EXTEND_COPY) in front of every conv (convf.c:335-341) is clamp addressing.
 */
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <vector>

#include "vb200_internal.h"

namespace vb200 {

namespace {

static std::atomic<bool> g_vector_convi{false};

struct Tap {
	int dx, dy; /* relative to the output pixel, already minus M / 2 */
};

struct ConvDev {
	const Tap *taps;
	const double *fcoeff; /* convf */
	const int *icoeff;	  /* convi C path, or mantissas for the vector path */
	int nnz;
	int w, h, bands;
	size_t in_bpl, out_bpl;
	double offset;		/* convf */
	int iscale, ioffset; /* convi */
	int exp;			/* vector path */
};

__device__ __forceinline__ int
clampi(int v, int lo, int hi)
{
	return max(lo, min(v, hi));
}

template <typename T>
__global__ void __launch_bounds__(256)
convf_kernel(const __grid_constant__ ConvDev P, const T *__restrict__ in, float *__restrict__ out)
{
	const int e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= P.w * P.bands)
		return;
	const int x = e / P.bands;
	const int b = e - x * P.bands;
	for (int y = blockIdx.y; y < P.h; y += gridDim.y) {
		double sum = P.offset;
		for (int i = 0; i < P.nnz; i++) {
			const Tap t = P.taps[i];
			const int sx = clampi(x + t.dx, 0, P.w - 1);
			const int sy = clampi(y + t.dy, 0, P.h - 1);
			const T v = ((const T *) ((const char *) in + (size_t) sy * P.in_bpl))[sx * P.bands + b];
			sum = __dadd_rn(sum, __dmul_rn(P.fcoeff[i], (double) v));
		}
		((float *) ((char *) out + (size_t) y * P.out_bpl))[e] = (float) sum;
	}
}

/* 1-D masks (the two passes of convsep / gaussblur): taps in shared memory, an
 * interior fast path without clamping, unit-stride (coalesced) loads per tap.
 * Same accumulation order and rounding as convf_kernel.
 */
template <typename T, bool VERT>
__global__ void __launch_bounds__(256)
convf_line_kernel(const __grid_constant__ ConvDev P, const T *__restrict__ in, float *__restrict__ out)
{
	__shared__ double sc[64];
	__shared__ int sd[64];
	if (threadIdx.x < P.nnz) {
		sc[threadIdx.x] = P.fcoeff[threadIdx.x];
		sd[threadIdx.x] = VERT ? P.taps[threadIdx.x].dy : P.taps[threadIdx.x].dx;
	}
	__syncthreads();
	const int e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= P.w * P.bands)
		return;
	const int nnz = P.nnz;
	for (int y = blockIdx.y; y < P.h; y += gridDim.y) {
		double sum = P.offset;
		if (VERT) {
			const size_t stride = P.in_bpl;
			const char *col = (const char *) in + (size_t) e * sizeof(T);
			if (y + sd[0] >= 0 && y + sd[nnz - 1] < P.h) {
				const char *p = col + (size_t) y * stride;
				for (int i = 0; i < nnz; i++)
					sum = __dadd_rn(sum, __dmul_rn(sc[i], (double) *(const T *) (p + (ptrdiff_t) sd[i] * (ptrdiff_t) stride)));
			}
			else
				for (int i = 0; i < nnz; i++) {
					const int sy = clampi(y + sd[i], 0, P.h - 1);
					sum = __dadd_rn(sum, __dmul_rn(sc[i], (double) *(const T *) (col + (size_t) sy * stride)));
				}
		}
		else {
			const T *row = (const T *) ((const char *) in + (size_t) y * P.in_bpl);
			const int x = e / P.bands;
			if (x + sd[0] >= 0 && x + sd[nnz - 1] < P.w) {
				const T *p = row + e;
				for (int i = 0; i < nnz; i++)
					sum = __dadd_rn(sum, __dmul_rn(sc[i], (double) p[sd[i] * P.bands]));
			}
			else {
				const int b = e - x * P.bands;
				for (int i = 0; i < nnz; i++)
					sum = __dadd_rn(sum, __dmul_rn(sc[i], (double) row[clampi(x + sd[i], 0, P.w - 1) * P.bands + b]));
			}
		}
		((float *) ((char *) out + (size_t) y * P.out_bpl))[e] = (float) sum;
	}
}

/* 1-D masks again, register-blocked: R outputs per thread along the mask axis, so each input
 * is loaded and widened to double once per R outputs instead of once per tap, and the
 * coefficients of an R x R block of multiply-adds sit in registers.  Every accumulator still
 * takes its taps in ascending mask order with a separately rounded multiply and add
 * (convf.c:175-199 compiled without contraction), and absent (zero) taps are skipped, not
 * multiplied, exactly like the reference's squeezed tap list.
 */
struct LineMask {
	double c[64];			   /* dense: c[i] for mask position i (0 where absent) */
	unsigned long long present; /* bit i: position i is a tap */
	int n;					   /* mask length */
};

template <typename T, bool VERT, int R, bool LOOP>
__global__ void __launch_bounds__(128)
convf_block_kernel(const __grid_constant__ ConvDev P, const __grid_constant__ LineMask M, const T *__restrict__ in,
	float *__restrict__ out)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	const int n = M.n;
	const int d0 = -(n / 2);
	int e, y_first, y_step, x0 = 0, b = 0;
	if (VERT) {
		e = idx;
		if (e >= P.w * P.bands)
			return;
		y_first = blockIdx.y * R;
		y_step = gridDim.y * R;
	}
	else {
		const int groups = (P.w + R - 1) / R;
		if (idx >= groups * P.bands)
			return;
		const int pg = idx / P.bands;
		b = idx - pg * P.bands;
		x0 = pg * R;
		y_first = blockIdx.y;
		y_step = gridDim.y;
		e = 0;
	}
	int y0 = y_first;
	do {
		double acc[R];
#pragma unroll
		for (int r = 0; r < R; r++)
			acc[r] = P.offset;
		const char *base = (const char *) in;
		const T *row = (const T *) (base + (size_t) y0 * P.in_bpl); /* HORIZ */

		for (int j0 = 0; j0 < n + R - 1; j0 += R) {
			double cc[2 * R - 1];
			unsigned vm = 0;
#pragma unroll
			for (int k = 0; k < 2 * R - 1; k++) {
				const int i = j0 - (R - 1) + k;
				const bool ok = (unsigned) i < (unsigned) n && ((M.present >> i) & 1ull);
				cc[k] = ok ? M.c[i] : 0.0;
				vm |= ok ? (1u << k) : 0u;
			}
#pragma unroll
			for (int jj = 0; jj < R; jj++) {
				const int j = j0 + jj;
				if (j < n + R - 1) {
					double v;
					if (VERT) {
						const int sy = clampi(y0 + d0 + j, 0, P.h - 1);
						v = (double) ((const T *) (base + (size_t) sy * P.in_bpl))[e];
					}
					else {
						const int sx = clampi(x0 + d0 + j, 0, P.w - 1);
						v = (double) row[sx * P.bands + b];
					}
#pragma unroll
					for (int r = 0; r < R; r++) {
						const int k = jj - r + R - 1;
						if (vm & (1u << k))
							acc[r] = __dadd_rn(acc[r], __dmul_rn(cc[k], v));
					}
				}
			}
		}
#pragma unroll
		for (int r = 0; r < R; r++) {
			if (VERT) {
				if (y0 + r < P.h)
					((float *) ((char *) out + (size_t) (y0 + r) * P.out_bpl))[e] = (float) acc[r];
			}
			else if (x0 + r < P.w)
				((float *) ((char *) out + (size_t) y0 * P.out_bpl))[(x0 + r) * P.bands + b] = (float) acc[r];
		}
	} while (LOOP && (y0 += y_step) < P.h);
}

/* The dense case of the above (every mask position is a tap, n >= R: Gaussians): the
 * (row, output) pairs that exist form a head triangle, a band of full rows and a tail
 * triangle, so nothing is predicated and no multiply-add is issued for a tap that does
 * not exist.  Same arithmetic, same order.
 */
template <typename T, bool VERT, int R, bool LOOP>
__global__ void __launch_bounds__(128)
convf_dense_kernel(const __grid_constant__ ConvDev P, const __grid_constant__ LineMask M, const T *__restrict__ in,
	float *__restrict__ out)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	const int n = M.n;
	const int d0 = -(n / 2);
	int e = 0, y_first, y_step, x0 = 0, b = 0;
	if (VERT) {
		e = idx;
		if (e >= P.w * P.bands)
			return;
		y_first = blockIdx.y * R;
		y_step = gridDim.y * R;
	}
	else {
		const int groups = (P.w + R - 1) / R;
		if (idx >= groups * P.bands)
			return;
		const int pg = idx / P.bands;
		b = idx - pg * P.bands;
		x0 = pg * R;
		y_first = blockIdx.y;
		y_step = gridDim.y;
	}
	int y0 = y_first;
	do {
		const char *base = (const char *) in;
		const T *row = (const T *) (base + (size_t) y0 * P.in_bpl); /* HORIZ */
		const bool interior = VERT ? (y0 + d0 >= 0 && y0 + d0 + n + R - 2 < P.h) : (x0 + d0 >= 0 && x0 + d0 + n + R - 2 < P.w);
		const T *p0 = VERT ? (const T *) (base + (size_t) (y0 + d0) * P.in_bpl) + e : row + (size_t) (x0 + d0) * P.bands + b;
		const size_t step = VERT ? P.in_bpl / sizeof(T) : (size_t) P.bands;
		double acc[R];
#pragma unroll
		for (int r = 0; r < R; r++)
			acc[r] = P.offset;

		/* the body twice: interior tiles read through one pointer + a constant step, so the loads of a
		 * group of rows can be issued together; edge tiles clamp every coordinate (VIPS_EXTEND_COPY)
		 */
		auto body = [&](auto load) {
			/* head: rows 0 .. R - 2, outputs r <= row */
#pragma unroll
			for (int j = 0; j < R - 1; j++) {
				const double v = load(j);
#pragma unroll
				for (int r = 0; r <= j; r++)
					acc[r] = __dadd_rn(acc[r], __dmul_rn(M.c[j - r], v));
			}
			/* full rows R - 1 .. n - 1, R at a time with their 2R - 1 coefficients in registers */
			int j = R - 1;
			for (; j + R <= n; j += R) {
				double cc[2 * R - 1];
#pragma unroll
				for (int k = 0; k < 2 * R - 1; k++)
					cc[k] = M.c[j - (R - 1) + k];
#pragma unroll
				for (int jj = 0; jj < R; jj++) {
					const double v = load(j + jj);
#pragma unroll
					for (int r = 0; r < R; r++)
						acc[r] = __dadd_rn(acc[r], __dmul_rn(cc[jj - r + R - 1], v));
				}
			}
			for (; j < n; j++) {
				const double v = load(j);
#pragma unroll
				for (int r = 0; r < R; r++)
					acc[r] = __dadd_rn(acc[r], __dmul_rn(M.c[j - r], v));
			}
			/* tail: rows n .. n + R - 2, outputs r > row - n */
			double ct[R - 1];
#pragma unroll
			for (int k = 0; k < R - 1; k++)
				ct[k] = M.c[n - R + 1 + k];
#pragma unroll
			for (int jt = 0; jt < R - 1; jt++) {
				const double v = load(n + jt);
#pragma unroll
				for (int r = jt + 1; r < R; r++)
					acc[r] = __dadd_rn(acc[r], __dmul_rn(ct[jt - r + R - 1], v));
			}
		};
		if (interior)
			body([&](int j) -> double { return (double) p0[(size_t) j * step]; });
		else if (VERT)
			body([&](int j) -> double { return (double) ((const T *) (base + (size_t) clampi(y0 + d0 + j, 0, P.h - 1) * P.in_bpl))[e]; });
		else
			body([&](int j) -> double { return (double) row[clampi(x0 + d0 + j, 0, P.w - 1) * P.bands + b]; });
#pragma unroll
		for (int r = 0; r < R; r++) {
			if (VERT) {
				if (y0 + r < P.h)
					((float *) ((char *) out + (size_t) (y0 + r) * P.out_bpl))[e] = (float) acc[r];
			}
			else if (x0 + r < P.w)
				((float *) ((char *) out + (size_t) y0 * P.out_bpl))[(x0 + r) * P.bands + b] = (float) acc[r];
		}
	} while (LOOP && (y0 += y_step) < P.h);
}

template <typename T>
__global__ void __launch_bounds__(256)
convi_kernel(const __grid_constant__ ConvDev P, const T *__restrict__ in, T *__restrict__ out, long long lo,
	long long hi, int clip)
{
	const int e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= P.w * P.bands)
		return;
	const int x = e / P.bands;
	const int b = e - x * P.bands;
	for (int y = blockIdx.y; y < P.h; y += gridDim.y) {
		long long sum = 0;
		for (int i = 0; i < P.nnz; i++) {
			const Tap t = P.taps[i];
			const int sx = clampi(x + t.dx, 0, P.w - 1);
			const int sy = clampi(y + t.dy, 0, P.h - 1);
			const T v = ((const T *) ((const char *) in + (size_t) sy * P.in_bpl))[sx * P.bands + b];
			sum += (long long) P.icoeff[i] * (long long) v;
		}
		sum = ((sum + P.iscale / 2) / P.iscale) + P.ioffset;
		if (clip)
			sum = sum < lo ? lo : (sum > hi ? hi : sum);
		((T *) ((char *) out + (size_t) y * P.out_bpl))[e] = (T) sum;
	}
}

__global__ void __launch_bounds__(256)
convi_float_kernel(const __grid_constant__ ConvDev P, const float *__restrict__ in, float *__restrict__ out)
{
	const int e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= P.w * P.bands)
		return;
	const int x = e / P.bands;
	const int b = e - x * P.bands;
	for (int y = blockIdx.y; y < P.h; y += gridDim.y) {
		double sum = 0;
		for (int i = 0; i < P.nnz; i++) {
			const Tap t = P.taps[i];
			const int sx = clampi(x + t.dx, 0, P.w - 1);
			const int sy = clampi(y + t.dy, 0, P.h - 1);
			const float v = ((const float *) ((const char *) in + (size_t) sy * P.in_bpl))[sx * P.bands + b];
			sum = __dadd_rn(sum, __dmul_rn((double) P.icoeff[i], (double) v));
		}
		sum = __dadd_rn(__ddiv_rn(sum, (double) P.iscale), (double) P.ioffset);
		((float *) ((char *) out + (size_t) y * P.out_bpl))[e] = (float) sum;
	}
}

__global__ void __launch_bounds__(256)
convi_vector_u8_kernel(const __grid_constant__ ConvDev P, const uint8_t *__restrict__ in, uint8_t *__restrict__ out)
{
	const int e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= P.w * P.bands)
		return;
	const int x = e / P.bands;
	const int b = e - x * P.bands;
	for (int y = blockIdx.y; y < P.h; y += gridDim.y) {
		int sum = 1 << (P.exp - 1);
		for (int i = 0; i < P.nnz; i++) {
			const Tap t = P.taps[i];
			const int sx = clampi(x + t.dx, 0, P.w - 1);
			const int sy = clampi(y + t.dy, 0, P.h - 1);
			sum += (int) (in + (size_t) sy * P.in_bpl)[sx * P.bands + b] * P.icoeff[i];
		}
		(out + (size_t) y * P.out_bpl)[e] = (uint8_t) clampi((sum >> P.exp) + P.ioffset, 0, 255);
	}
}

/* band 0 of a short image -> packed 1-band image, and the sharpen merge */
__global__ void __launch_bounds__(256)
extract_band0_short_kernel(const short *__restrict__ in, size_t in_bpl, int bands, short *__restrict__ out,
	size_t out_bpl, int w, int h)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= w)
		return;
	for (int y = blockIdx.y; y < h; y += gridDim.y)
		((short *) ((char *) out + (size_t) y * out_bpl))[x] = ((const short *) ((const char *) in + (size_t) y * in_bpl))[x * bands];
}

__global__ void __launch_bounds__(256)
sharpen_kernel(short *__restrict__ labs, size_t labs_bpl, int bands, const short *__restrict__ blur, size_t blur_bpl,
	const int *__restrict__ lut, int w, int h)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= w)
		return;
	for (int y = blockIdx.y; y < h; y += gridDim.y) {
		short *p = (short *) ((char *) labs + (size_t) y * labs_bpl) + x * bands;
		const int v1 = *p;
		const int v2 = ((const short *) ((const char *) blur + (size_t) y * blur_bpl))[x];
		const int diff = (v1 & 0x7fff) - (v2 & 0x7fff);
		int o = v1 + __ldg(lut + diff + 32768);
		o = max(0, min(o, 32767));
		*p = (short) o;
	}
}

/* vips__image_intize, convi.c:859-923 */
void
image_intize(const double *mask, int n, double scale, double offset, std::vector<int> &coeff, int *iscale, int *ioffset)
{
	double double_result = 0;
	for (int i = 0; i < n; i++)
		double_result += mask[i];
	double_result /= scale;
	coeff.resize(n);
	int int_result = 0;
	for (int i = 0; i < n; i++) {
		const double r = rint(mask[i]);
		coeff[i] = r;
		int_result += r;
	}
	/* vips__image_intize goes on to adjust the scale of its int copy, but
	 * vips_convi_gen reads scale / offset from convolution->M, the ORIGINAL
	 * matrix (convi.c:760-763): the adjustment never reaches the pixels.
	 */
	(void) int_result;
	(void) double_result;
	*iscale = rint(scale);
	*ioffset = rint(offset);
}

/* vips_convi_intize (HAVE_HWY), convi.c:931-1119 */
bool
intize8(const double *mask, int n_point, double scale, std::vector<int> &mant, std::vector<int> &pos, int *exp_out)
{
	std::vector<double> scaled(n_point);
	for (int i = 0; i < n_point; i++)
		scaled[i] = mask[i] / scale;
	double mx = scaled[0];
	for (int i = 1; i < n_point; i++)
		mx = std::max(mx, scaled[i]);
	const int shift = ceil(log2(mx) + 1);
	if (shift > 6 || shift < -24)
		return false;
	if (ceil(log2(n_point)) > 10)
		return false;
	const int exp = 7 - shift;
	mant.clear();
	pos.clear();
	for (int i = 0; i < n_point; i++) {
		const short m = rint(128 * scaled[i] * pow(2, -shift));
		if (m < -128 || m > 127)
			return false;
		if (m) {
			mant.push_back(m);
			pos.push_back(i);
		}
	}
	if (mant.empty()) {
		mant.push_back(0);
		pos.push_back(0);
	}
	double true_sum = 0.0;
	int int_sum = 0;
	for (size_t i = 0; i < mant.size(); i++) {
		true_sum += 128 * scaled[pos[i]];
		int_sum += 128 * mant[i];
	}
	const int true_value = std::max(0.0, std::min(255.0, true_sum));
	int int_value = (int_sum + (1 << (exp - 1))) >> exp;
	int_value = std::max(0, std::min(255, int_value));
	if (abs(true_value - int_value) > 2)
		return false;
	*exp_out = exp;
	return true;
}

struct Uploaded {
	void *block = nullptr;
};

int
upload_taps(const char *domain, const std::vector<int> &pos, int mw, int mh, const std::vector<double> *fc,
	const std::vector<int> *ic, ConvDev *P, Uploaded *u, cudaStream_t s)
{
	const int nnz = (int) pos.size();
	std::vector<Tap> taps(nnz);
	for (int i = 0; i < nnz; i++) {
		taps[i].dx = pos[i] % mw - mw / 2;
		taps[i].dy = pos[i] / mw - mh / 2;
	}
	const size_t n_f = fc ? nnz * sizeof(double) : 0;
	const size_t n_t = nnz * sizeof(Tap);
	const size_t n_i = ic ? nnz * sizeof(int) : 0;
	std::vector<char> host(n_f + n_t + n_i);
	if (fc)
		memcpy(&host[0], fc->data(), n_f);
	memcpy(&host[n_f], taps.data(), n_t);
	if (ic)
		memcpy(&host[n_f + n_t], ic->data(), n_i);
	if (dev_alloc(domain, &u->block, host.size(), s))
		return -1;
	VB200_CUDA(domain, cudaMemcpyAsync(u->block, host.data(), host.size(), cudaMemcpyHostToDevice, s));
	P->fcoeff = (const double *) u->block;
	P->taps = (const Tap *) ((char *) u->block + n_f);
	P->icoeff = (const int *) ((char *) u->block + n_f + n_t);
	P->nnz = nnz;
	return 0;
}

} // namespace

int
dev_conv(const char *domain, const DevImage &in, DevImage *out, const double *mask, int mw, int mh, double scale,
	double offset, int precision, cudaStream_t s, bool allow_vector)
{
	if (!format_is_supported(in.fmt)) {
		error(domain, "band format %d not supported on the device path", in.fmt);
		return -1;
	}
	if (mw <= 0 || mh <= 0 || !mask) {
		error(domain, "bad mask");
		return -1;
	}
	const int n = mw * mh;
	ConvDev P;
	memset(&P, 0, sizeof(P));
	P.w = in.w;
	P.h = in.h;
	P.bands = in.bands;
	P.in_bpl = in.bpl;
	Uploaded u;
	const dim3 grid = row_grid(in.w * in.bands, in.h);

	if (precision == VB200_PRECISION_FLOAT) {
		/* convf.c:303-331: bake the scale in, squeeze zeros */
		std::vector<double> coeff;
		std::vector<int> pos;
		for (int i = 0; i < n; i++) {
			const double c = mask[i] / scale;
			if (c) {
				coeff.push_back(c);
				pos.push_back(i);
			}
		}
		if (coeff.empty()) {
			coeff.push_back(0);
			pos.push_back(0);
		}
		P.offset = offset;
		if (dev_image_new(domain, out, in.w, in.h, in.bands, VB200_FORMAT_FLOAT, in.type, s))
			return -1;
		P.out_bpl = out->bpl;
		/* taps arrive sorted by mask position, so sd[0] / sd[nnz - 1] bound the stencil */
		const bool line_h = mh == 1 && coeff.size() <= 64, line_v = mw == 1 && coeff.size() <= 64;
		constexpr int RB = 8; /* outputs per thread of convf_block_kernel */
		LineMask lm;
		bool block_ok = (line_h || line_v) && n <= 64 && getenv("VB200_NO_CONV_BLOCK") == nullptr;
		if (block_ok) {
			memset(&lm, 0, sizeof(lm));
			lm.n = n;
			for (int i = 0; i < n; i++) {
				const double c = mask[i] / scale;
				if (c) {
					lm.c[i] = c;
					lm.present |= 1ull << i;
				}
			}
		}
		if (block_ok && lm.present == 0)
			block_ok = false; /* the all-zero mask keeps one 0 * pixel term (convf.c:321-325): the generic kernels do that */
		const bool dense_ok = block_ok && n >= RB && lm.present == (n == 64 ? ~0ull : (1ull << n) - 1) &&
			getenv("VB200_NO_CONV_DENSE") == nullptr;
		/* the 1-D kernels take their mask as a kernel parameter: no table upload (a pageable
		 * cudaMemcpyAsync is a host-side stall as long as the kernel itself on a big image)
		 */
		if (!block_ok && upload_taps(domain, pos, mw, mh, &coeff, nullptr, &P, &u, s))
			return -1;
		const dim3 grid_h = row_grid((in.w + RB - 1) / RB * in.bands, in.h, 128);
		const dim3 grid_v = row_grid(in.w * in.bands, (in.h + RB - 1) / RB, 128);
		const bool loop_h = rows_loop(in.h), loop_v = rows_loop((in.h + RB - 1) / RB);
#define CF(T) \
	do { \
		if (dense_ok && line_h) \
			(loop_h ? convf_dense_kernel<T, false, RB, true> : convf_dense_kernel<T, false, RB, false>)<<<grid_h, 128, 0, s>>>(P, lm, (const T *) in.data, (float *) out->data); \
		else if (dense_ok && line_v) \
			(loop_v ? convf_dense_kernel<T, true, RB, true> : convf_dense_kernel<T, true, RB, false>)<<<grid_v, 128, 0, s>>>(P, lm, (const T *) in.data, (float *) out->data); \
		else if (block_ok && line_h) \
			(loop_h ? convf_block_kernel<T, false, RB, true> : convf_block_kernel<T, false, RB, false>)<<<grid_h, 128, 0, s>>>(P, lm, (const T *) in.data, (float *) out->data); \
		else if (block_ok && line_v) \
			(loop_v ? convf_block_kernel<T, true, RB, true> : convf_block_kernel<T, true, RB, false>)<<<grid_v, 128, 0, s>>>(P, lm, (const T *) in.data, (float *) out->data); \
		else if (line_h) \
			convf_line_kernel<T, false><<<grid, 256, 0, s>>>(P, (const T *) in.data, (float *) out->data); \
		else if (line_v) \
			convf_line_kernel<T, true><<<grid, 256, 0, s>>>(P, (const T *) in.data, (float *) out->data); \
		else \
			convf_kernel<T><<<grid, 256, 0, s>>>(P, (const T *) in.data, (float *) out->data); \
	} while (0)
		switch (in.fmt) {
		case VB200_FORMAT_UCHAR: CF(uint8_t); break;
		case VB200_FORMAT_CHAR: CF(int8_t); break;
		case VB200_FORMAT_USHORT: CF(uint16_t); break;
		case VB200_FORMAT_SHORT: CF(int16_t); break;
		case VB200_FORMAT_UINT: CF(uint32_t); break;
		case VB200_FORMAT_INT: CF(int32_t); break;
		case VB200_FORMAT_FLOAT: CF(float); break;
		}
#undef CF
	}
	else if (precision == VB200_PRECISION_INTEGER) {
		if (dev_image_new(domain, out, in.w, in.h, in.bands, in.fmt, in.type, s))
			return -1;
		P.out_bpl = out->bpl;
		std::vector<int> mant, pos;
		int exp = 0;
		if (allow_vector && g_vector_convi.load() && in.fmt == VB200_FORMAT_UCHAR && intize8(mask, n, scale, mant, pos, &exp)) {
			/* the Highway arithmetic (convi.c:1152-1160 picks it for uchar when intize succeeds) */
			P.exp = exp;
			P.ioffset = rint(offset);
			if (upload_taps(domain, pos, mw, mh, nullptr, &mant, &P, &u, s))
				return -1;
			convi_vector_u8_kernel<<<grid, 256, 0, s>>>(P, (const uint8_t *) in.data, (uint8_t *) out->data);
		}
		else {
			std::vector<int> all, coeff;
			image_intize(mask, n, scale, offset, all, &P.iscale, &P.ioffset);
			if (P.iscale == 0) {
				/* the reference divides by it (convi.c:711) */
				error(domain, "mask scale rounds to zero");
				dev_image_release(out, s);
				return -1;
			}
			pos.clear();
			for (int i = 0; i < n; i++)
				if (all[i]) {
					coeff.push_back(all[i]);
					pos.push_back(i);
				}
			if (coeff.empty()) {
				coeff.push_back(0);
				pos.push_back(0);
			}
			if (upload_taps(domain, pos, mw, mh, nullptr, &coeff, &P, &u, s))
				return -1;
#define CI(T, LO, HI, CLIP) convi_kernel<T><<<grid, 256, 0, s>>>(P, (const T *) in.data, (T *) out->data, LO, HI, CLIP)
			switch (in.fmt) {
			case VB200_FORMAT_UCHAR: CI(uint8_t, 0, 255, 1); break;
			case VB200_FORMAT_CHAR: CI(int8_t, -128, 127, 1); break;
			case VB200_FORMAT_USHORT: CI(uint16_t, 0, 65535, 1); break;
			case VB200_FORMAT_SHORT: CI(int16_t, -32768, 32767, 1); break;
			case VB200_FORMAT_UINT: CI(uint32_t, 0, 0, 0); break;
			case VB200_FORMAT_INT: CI(int32_t, 0, 0, 0); break;
			case VB200_FORMAT_FLOAT:
				convi_float_kernel<<<grid, 256, 0, s>>>(P, (const float *) in.data, (float *) out->data);
				break;
			}
#undef CI
		}
	}
	else {
		error(domain, "precision %d (approximate: conva) is not on the device path", precision);
		return -1;
	}
	cudaError_t e = cudaGetLastError();
	dev_free(u.block, s);
	if (e != cudaSuccess)
		return cuda_fail(domain, e, "conv kernel");
	count_launch();
	return 0;
}

/* 0 = done, -1 = error, 1 = this mask / image is not eligible (defined below) */
int dev_convsep_fused(const char *domain, const DevImage &in, DevImage *out, const double *first, const double *second, int mw,
	int mh, double scale, double offset, cudaStream_t s);

/* vips_convsep, convsep.c:61-114: conv(M) as given, with its offset, then conv(rot90(M)) with offset 0
 * and the same scale.  vips_rot90 (conversion/rot.c:100-156) maps out(x, y) = in(y, Ysize - 1 - x): an
 * n x 1 mask becomes the 1 x n column in the same order; a 1 x n mask becomes the n x 1 row REVERSED.
 */
int
dev_convsep(const char *domain, const DevImage &in, DevImage *out, const double *mask, int mw, int mh, double scale,
	double offset, int precision, cudaStream_t s, bool allow_vector)
{
	const int n = mw * mh;
	std::vector<double> rot(mask, mask + n);
	if (mw == 1)
		std::reverse(rot.begin(), rot.end());
	/* the dense float pair as ONE kernel: the intermediate never leaves shared memory */
	if (precision == VB200_PRECISION_FLOAT) {
		const int fused = dev_convsep_fused(domain, in, out, mask, rot.data(), mw, mh, scale, offset, s);
		if (fused <= 0)
			return fused; /* 0 done, -1 failed; 1 = not eligible */
	}
	DevImage mid;
	if (dev_conv(domain, in, &mid, mask, mw, mh, scale, offset, precision, s, allow_vector))
		return -1;
	int r = dev_conv(domain, mid, out, rot.data(), mh, mw, scale, 0.0, precision, s, allow_vector);
	dev_image_release(&mid, s);
	return r;
}

int
dev_convsep_fused(const char *domain, const DevImage &in, DevImage *out, const double *first, const double *second, int mw,
	int mh, double scale, double offset, cudaStream_t s)
{
	return 1;
}

/* vips_gaussmat, create/gaussmat.c:93-170 */
void
host_gaussmat(double sigma, double min_ampl, bool separable, bool integer_precision, std::vector<double> &coeff, int *width,
	int *height, double *scale)
{
	const double sig2 = 2. * sigma * sigma;
	const int max_x = (int) std::max(0.0, std::min(5000.0, 8 * sigma));
	int x;
	for (x = 0; x < max_x; x++) {
		const double v = exp(-((double) (x * x)) / sig2);
		if (v < min_ampl)
			break;
	}
	const int w = 2 * std::max(x - 1, 0) + 1;
	const int h = separable ? 1 : w;
	coeff.resize((size_t) w * h);
	double sum = 0.0;
	for (int y = 0; y < h; y++)
		for (int xx = 0; xx < w; xx++) {
			const int xo = xx - w / 2;
			const int yo = y - h / 2;
			const double distance = xo * xo + yo * yo;
			double v = exp(-distance / sig2);
			if (integer_precision)
				v = rint(20 * v);
			coeff[(size_t) y * w + xx] = v;
			sum += v;
		}
	if (sum == 0)
		sum = 1;
	*width = w;
	*height = h;
	*scale = sum;
}

int
dev_gaussblur(const char *domain, const DevImage &in, DevImage *out, double sigma, double min_ampl, int precision,
	cudaStream_t s)
{
	if (sigma < 0.2) {
		/* gaussblur.c:83-86: a copy */
		*out = in;
		out->owned = false;
		return 0;
	}
	std::vector<double> m;
	int w, h;
	double scale;
	host_gaussmat(sigma, min_ampl, true, precision != VB200_PRECISION_FLOAT, m, &w, &h, &scale);
	return dev_convsep(domain, in, out, m.data(), w, h, scale, 0.0, precision, s, true);
}

/* sharpen_fused.cu */
int dev_sharpen_fused(const char *domain, const void *in, size_t in_bpl, size_t in_frame_stride, void *out, size_t out_bpl,
	size_t out_frame_stride, int n_frames, int w, int h, int bands, double sigma, double x1, double y2, double y3, double m1,
	double m2, cudaStream_t s);

/* vips_sharpen, sharpen.c:171-303 */
int
dev_sharpen(const char *domain, const DevImage &in, DevImage *out, double sigma, double x1, double y2, double y3,
	double m1, double m2, cudaStream_t s)
{
	/* 8-bit sRGB, 3 or 4 bands: the whole graph as one kernel (sharpen_fused.cu) */
	if (in.fmt == VB200_FORMAT_UCHAR && in.type == VB200_INTERPRETATION_sRGB && (in.bands == 3 || in.bands == 4)) {
		DevImage res;
		if (dev_image_new(domain, &res, in.w, in.h, in.bands, in.fmt, in.type, s))
			return -1;
		const int rc = dev_sharpen_fused(domain, in.data, in.bpl, 0, res.data, res.bpl, 0, 1, in.w, in.h, in.bands, sigma, x1, y2,
			y3, m1, m2, s);
		if (rc == 0) {
			*out = res;
			return 0;
		}
		dev_image_release(&res, s);
		if (rc < 0)
			return -1;
	}
	DevImage labs;
	if (dev_colourspace(domain, in, &labs, VB200_INTERPRETATION_LABS, in.type, s))
		return -1;
	if (labs.bands < 3) {
		dev_image_release(&labs, s);
		error(domain, "image must have at least 3 bands");
		return -1;
	}
	if (labs.data == in.data) {
		/* already LABS: work on a private copy, sharpen_kernel writes in place */
		DevImage copy;
		if (dev_image_new(domain, &copy, in.w, in.h, in.bands, in.fmt, in.type, s))
			return -1;
		cudaMemcpy2DAsync(copy.data, copy.bpl, in.data, in.bpl, copy.bpl, in.h, cudaMemcpyDeviceToDevice, s);
		labs = copy;
	}

	std::vector<double> m;
	int mw, mh;
	double scale;
	host_gaussmat(sigma, 0.1, true, true, m, &mw, &mh, &scale);

	std::vector<int> lut(65536);
	for (int i = 0; i < 65536; i++) {
		const double v = (i - 32767) / 327.67;
		double y;
		if (v < -x1)
			y = (v + x1) * m2 + -x1 * m1;
		else if (v < x1)
			y = v * m1;
		else
			y = (v - x1) * m2 + x1 * m1;
		if (y < -y3)
			y = -y3;
		if (y > y2)
			y = y2;
		lut[i] = rint(y * 327.67);
	}
	void *dlut = nullptr;
	int rc = dev_alloc(domain, &dlut, lut.size() * sizeof(int), s);
	if (!rc && cudaMemcpyAsync(dlut, lut.data(), lut.size() * sizeof(int), cudaMemcpyHostToDevice, s) != cudaSuccess)
		rc = -1;

	DevImage L, blur;
	if (!rc)
		rc = dev_image_new(domain, &L, labs.w, labs.h, 1, VB200_FORMAT_SHORT, VB200_INTERPRETATION_B_W, s);
	const dim3 grid = row_grid(labs.w, labs.h);
	if (!rc) {
		extract_band0_short_kernel<<<grid, 256, 0, s>>>((const short *) labs.data, labs.bpl, labs.bands, (short *) L.data,
			L.bpl, labs.w, labs.h);
		count_launch();
		/* short input: always the exact C path, never the vector one */
		rc = dev_convsep(domain, L, &blur, m.data(), mw, mh, scale, 0.0, VB200_PRECISION_INTEGER, s, false);
	}
	if (!rc) {
		sharpen_kernel<<<grid, 256, 0, s>>>((short *) labs.data, labs.bpl, labs.bands, (const short *) blur.data, blur.bpl,
			(const int *) dlut, labs.w, labs.h);
		count_launch();
		rc = dev_colourspace(domain, labs, out, in.type, VB200_INTERPRETATION_LABS, s);
		if (!rc)
			adopt_pass_through(&labs, out);
	}
	dev_image_release(&L, s);
	dev_image_release(&blur, s);
	dev_image_release(&labs, s);
	dev_free(dlut, s);
	return rc;
}

} // namespace vb200

using namespace vb200;

extern "C" void
vb200_set_vector_convi(int on)
{
	g_vector_convi = on != 0;
}

extern "C" int
vb200_gaussmat(VB200Mask *out, double sigma, double min_ampl, int separable, int precision)
{
	if (!out) {
		error("gaussmat", "null argument");
		return -1;
	}
	std::vector<double> m;
	int w, h;
	double scale;
	host_gaussmat(sigma, min_ampl, separable != 0, precision != VB200_PRECISION_FLOAT, m, &w, &h, &scale);
	double *c = (double *) malloc(m.size() * sizeof(double));
	if (!c) {
		error("gaussmat", "out of memory");
		return -1;
	}
	memcpy(c, m.data(), m.size() * sizeof(double));
	out->width = w;
	out->height = h;
	out->coeff = c;
	out->scale = scale;
	out->offset = 0.0;
	return 0;
}

extern "C" void
vb200_mask_free(VB200Mask *mask)
{
	if (mask && mask->coeff) {
		free((void *) mask->coeff);
		mask->coeff = nullptr;
	}
}
