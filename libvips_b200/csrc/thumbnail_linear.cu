/* thumbnail_linear.cu -- the linear-light thumbnail (vips_thumbnail_image(..., linear = TRUE)) of an
 * 8-bit sRGB frame as TWO kernels instead of the reference's nine image-sized float passes.
 *
 * The reference chain (resample/thumbnail.c:757-806, 848-902, 971-987; SURVEY 3.1b), every link a
 * separate operation with a float image (16 bytes per RGBA pixel) in between:
 *     sRGB -> scRGB (uchar LUT -> float; alpha * (1 / 255) in float)            sRGB2scRGB.c:71-107, colour.c:252-291
 *     premultiply, float                 q = p * (clip(alpha) / 1.0)            premultiply.c:104-122
 *     shrinkv, float                     (float) (sum_double * (1.0 / vshrink)) shrinkv.c:198-199, 258-266
 *     reducev, float                     (float) sum_i cy[i] * (double) in[i]   reducev.cpp:487-496, templates.h:565-578
 *     shrinkh, float                     FSHRINK                                shrinkh.c:134-152
 *     reduceh, float                                                            reduceh.cpp:182-193
 *     unpremultiply, float               fabs(alpha) < 0.01 ? 0 : 1.0 / alpha   unpremultiply.c:137-176
 *     scRGB -> sRGB                      LUT + lerp + rintf; alpha * 255, cast  scRGB2sRGB.c:83-131, LabQ2sRGB.c:290-361
 *
 * Kernel V (linear_v_kernel): one thread per input COLUMN streams down the frame.  Per box-shrunk row it
 * reads VS uchar pixels, linearises and premultiplies them in registers, box-sums them in double, rounds
 * to float as shrinkv does, and feeds the result to the (at most 8) output rows whose Lanczos window it
 * lies in: each in-flight output row owns a double accumulator that receives its taps in tap order
 * (accumulation order is the reference's, so the sums are bit-identical).  A finished row is rounded to
 * float and written to the intermediate [OH][W] image -- the only intermediate, 1/8 of the input's pixel
 * count at 4K -> 512.  No thread ever needs another thread's data: no shared-memory exchange, no halo.
 * Kernel H (linear_h_kernel): one CTA per output row box-shrinks the row into shared memory, then one
 * thread per output pixel runs reduceh, unpremultiply and scRGB -> sRGB and stores the uchar pixel.
 *
 * What bounds it: not HBM.  Bit-exactness with the reference's `double` sums costs, per input pixel, four
 * float -> double conversions and ~18 separately rounded FP64 multiplies / adds (reducev alone is 2 x 13 taps
 * x 4 channels per 2 x 4 input pixels); the 64-bit conversion unit (16 lanes / clk / SM) and the FP64 pipe
 * (64 lanes / clk / SM) each need ~20 us per 4096 x 4096 frame, against 10 us of HBM time.  See DESIGN 4.6.
 *
 * Algorithmic bytes per frame: W * H * bands in + OW * OH * bands out (the fused-ideal figure); the
 * intermediate adds 2 * OH * W * bands * 4.
 */
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "colour_steps.cuh"
#include "vb200_internal.h"

namespace vb200 {

namespace {

constexpr int kSlots = 8;	  /* output rows in flight per column */
constexpr int kVThreads = 256; /* columns per CTA of kernel V */
constexpr int kDepth = 6;	  /* box-shrunk rows each thread keeps in flight (cp.async groups) */
constexpr int kMaxBox = 8;	  /* rows of a box the cp.async ring holds; larger boxes load directly */

struct LinVParams {
	int W, H, OH, VS, Hs, vembed, nv;
	size_t in_bpl, in_frame_stride;
	const int *vfirst, *vphase;
	const double *vcoef; /* [65][nv] */
	float *mid;
	size_t mid_frame_stride; /* floats */
	int RPC;				 /* output rows per CTA */
	double inv_v;
	StepInfo fwd[2];
	int n_fwd;
	const float *v2Y_8;
	/* the residual-2.0 schedule (linear_v2_kernel): first[y] = f0 + 2 y, one phase, 13 taps */
	int f0;
	double c2[13];
};

struct LinHParams {
	int W, OW, OH, HS, Ws, hembed, nh, Wse;
	const int *hfirst, *hphase;
	const double *hcoef; /* [65][nh] */
	const float *mid;
	size_t mid_frame_stride;
	size_t out_bpl, out_frame_stride;
	double inv_h;
	StepInfo bwd[2];
	int n_bwd;
	const int *Y2v_8;
};

template <int NCH, bool PREMUL, int VST>
__global__ void __launch_bounds__(kVThreads, 2)
linear_v_kernel(const __grid_constant__ LinVParams P, const uint8_t *__restrict__ in, int frame0)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	double *s_vc = (double *) smem_raw;			  /* [65 * nv] */
	float *s_lin = (float *) (s_vc + 65 * P.nv);  /* vips_v2Y_8 */
	float *s_al = s_lin + 256;					  /* alpha byte -> scRGB alpha (x 1 / 255, float) */
	float *s_nal = s_al + 256;					  /* alpha byte -> premultiply factor */
	/* [kDepth + 1][box rows][kVThreads] pixels in flight: every thread copies (cp.async) and later reads
	 * ONLY its own words, so the ring needs no barrier -- cp.async.wait_group orders a thread's own copies.
	 * One 128-byte request per warp and row is latency-bound on its own (8 KB in flight per SM); kDepth
	 * boxes ahead put ~50 KB per SM in flight.
	 */
	unsigned *s_ring = (unsigned *) (s_nal + 256);

	const int t = threadIdx.x;
	for (int i = t; i < 65 * P.nv; i += kVThreads)
		s_vc[i] = P.vcoef[i];
	for (int i = t; i < 256; i += kVThreads) {
		s_lin[i] = P.v2Y_8[i];
		/* the 4th band through sRGB -> scRGB as vips_colour_build carries it, then PRE_RGBA's
		 * nalpha = (float) clip(alpha) / max_alpha with max_alpha = 1.0 (premultiply.c:104-111)
		 */
		const float A = (float) carry_extra_band((double) i, P.fwd, P.n_fwd);
		s_al[i] = A;
		const float clip_alpha = (float) fmax(0.0, fmin(1.0, (double) A));
		s_nal[i] = (float) __ddiv_rn((double) clip_alpha, 1.0);
	}
	__syncthreads();

	const int xi = blockIdx.x * kVThreads + t;
	const bool live = xi < P.W;
	const int x = min(xi, P.W - 1);
	const int y_begin = blockIdx.y * P.RPC, y_end = min(y_begin + P.RPC, P.OH);
	const int frame = frame0 + blockIdx.z;
	const uint8_t *col = in + (size_t) frame * P.in_frame_stride + (size_t) x * NCH;
	float *mcol = P.mid + (size_t) frame * P.mid_frame_stride + (size_t) x * NCH;
	const int VS = VST ? VST : P.VS;
	const int nv = P.nv;

	double acc[kSlots][NCH];
	int s_first[kSlots], s_phase[kSlots], s_y[kSlots]; /* uniform across the CTA */
	unsigned active = 0;
#pragma unroll
	for (int J = 0; J < kSlots; J++) {
		s_first[J] = s_phase[J] = s_y[J] = 0;
#pragma unroll
		for (int c = 0; c < NCH; c++)
			acc[J][c] = 0.0;
	}
	int y_next = y_begin;
	const int e0 = __ldg(P.vfirst + y_begin), e1 = __ldg(P.vfirst + y_end - 1) + nv - 1;

	const bool ring = NCH == 4 && VS <= kMaxBox;
	auto prefetch = [&](int ee) {
		if (ring && ee <= e1) {
			const int srr = max(0, min(ee - P.vembed, P.Hs - 1));
			unsigned *dst = s_ring + (size_t) ((ee - e0) % (kDepth + 1)) * kMaxBox * kVThreads + t;
			for (int k = 0; k < VS; k++) {
				const int row = min(srr * VS + k, P.H - 1);
				const unsigned d = (unsigned) __cvta_generic_to_shared(dst + k * kVThreads);
				asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(col + (size_t) row * P.in_bpl) : "memory");
			}
		}
		asm volatile("cp.async.commit_group;" ::: "memory");
	};
	for (int d = 0; d < kDepth; d++)
		prefetch(e0 + d);

	for (int e = e0; e <= e1; e++) {
		/* ---- one box-shrunk row of this column: sRGB -> scRGB, premultiply, shrinkv */
		prefetch(e + kDepth);
		asm volatile("cp.async.wait_group %0;" ::"n"(kDepth) : "memory");
		const unsigned *mine = s_ring + (size_t) ((e - e0) % (kDepth + 1)) * kMaxBox * kVThreads + t;
		const int sr = max(0, min(e - P.vembed, P.Hs - 1));
		double sum[NCH];
#pragma unroll
		for (int c = 0; c < NCH; c++)
			sum[c] = 0.0;
#pragma unroll
		for (int k = 0; k < (VST ? VST : 1); k++) {
			for (int kk = 0; kk < (VST ? 1 : VS); kk++) {
				const int row = min(sr * VS + k + kk, P.H - 1);
				const uint8_t *p = col + (size_t) row * P.in_bpl;
				float q[NCH];
				if (NCH == 4) {
					const unsigned px = ring ? mine[(k + kk) * kVThreads] : __ldg((const unsigned *) p);
					const float r = s_lin[px & 255], g = s_lin[(px >> 8) & 255], b = s_lin[(px >> 16) & 255];
					if (PREMUL) {
						const float n = s_nal[px >> 24];
						q[0] = __fmul_rn(r, n);
						q[1] = __fmul_rn(g, n);
						q[2] = __fmul_rn(b, n);
					}
					else {
						q[0] = r;
						q[1] = g;
						q[2] = b;
					}
					q[NCH - 1] = s_al[px >> 24];
				}
				else {
#pragma unroll
					for (int c = 0; c < NCH; c++)
						q[c] = s_lin[__ldg(p + c)];
				}
#pragma unroll
				for (int c = 0; c < NCH; c++)
					sum[c] = __dadd_rn(sum[c], (double) q[c]);
			}
		}
		double sv[NCH];
#pragma unroll
		for (int c = 0; c < NCH; c++)
			sv[c] = (double) (float) __dmul_rn(sum[c], P.inv_v);

		/* ---- output rows whose window starts here */
		while (y_next < y_end && __ldg(P.vfirst + y_next) <= e) {
			const int j = y_next & (kSlots - 1);
			const int f = __ldg(P.vfirst + y_next), ph = __ldg(P.vphase + y_next);
#pragma unroll
			for (int J = 0; J < kSlots; J++)
				if (J == j) {
					s_first[J] = f;
					s_phase[J] = ph;
					s_y[J] = y_next;
#pragma unroll
					for (int c = 0; c < NCH; c++)
						acc[J][c] = 0.0;
				}
			active |= 1u << j;
			y_next++;
		}

		/* ---- reducev: this row is tap (e - first) of every row in flight; taps arrive in order */
#pragma unroll
		for (int J = 0; J < kSlots; J++) {
			if (active & (1u << J)) {
				const int tap = e - s_first[J];
				const double cf = s_vc[s_phase[J] * nv + tap];
#pragma unroll
				for (int c = 0; c < NCH; c++)
					acc[J][c] = __dadd_rn(acc[J][c], __dmul_rn(cf, sv[c]));
				if (tap == nv - 1) {
					if (live) {
						float *q = mcol + (size_t) s_y[J] * P.W * NCH;
						if (NCH == 4)
							*(float4 *) q = make_float4((float) acc[J][0], (float) acc[J][1], (float) acc[J][2], (float) acc[J][NCH - 1]);
						else {
#pragma unroll
							for (int c = 0; c < NCH; c++)
								q[c] = (float) acc[J][c];
						}
					}
					active &= ~(1u << J);
				}
			}
		}
	}
}


/* Kernel V for the commonest geometry: a total shrink that is an even integer (4096 -> 512, 3840 -> 640 ...)
 * leaves vips_resize a residual of exactly 2.0 after the box, so every output row has the same 13
 * coefficients and its window starts two box-shrunk rows after its predecessor's.  The schedule is then
 * static: per iteration one output row starts (tap 0), seven rows receive an even tap from shrunk row A
 * (the oldest completes with tap 12 and is stored), six receive an odd tap from row B.  The seven
 * accumulators rotate through registers by unrolling seven iterations; coefficients are kernel-parameter
 * constants.  Same sums in the same order as the general kernel -- 42 instead of 93 instructions per pixel.
 */
template <bool PREMUL, int VST>
__global__ void __launch_bounds__(kVThreads, 2)
linear_v2_kernel(const __grid_constant__ LinVParams P, const uint8_t *__restrict__ in, int frame0)
{
	constexpr int NCH = 4;
	constexpr int ROWS = 2 * VST;						   /* input rows per iteration */
	constexpr int CAP = (kDepth + 1) * kMaxBox;			   /* ring capacity in rows */
	constexpr int NST = CAP / ROWS < 7 ? CAP / ROWS : 7;   /* ring stages */
	constexpr int D2 = NST - 1;							   /* iterations in flight */
	extern __shared__ __align__(16) unsigned char smem_raw[];
	double *s_vc = (double *) smem_raw; /* unused here; keeps the layout of linear_v_kernel */
	float *s_lin = (float *) (s_vc + 65 * P.nv);
	/* alpha byte -> (premultiply factor, scRGB alpha): one 64-bit lookup.  (Holding the alpha as a double to
	 * save its conversion was measured: the 8-byte random gather costs more shared-memory wavefronts than the
	 * conversion it saves -- 57.7 vs 45.4 us per frame.)
	 */
	float2 *s_aln = (float2 *) (s_lin + 256);
	unsigned *s_ring = (unsigned *) (s_lin + 4 * 256);

	const int t = threadIdx.x;
	for (int i = t; i < 256; i += kVThreads) {
		s_lin[i] = P.v2Y_8[i];
		const float A = (float) carry_extra_band((double) i, P.fwd, P.n_fwd);
		const float clip_alpha = (float) fmax(0.0, fmin(1.0, (double) A));
		s_aln[i] = make_float2((float) __ddiv_rn((double) clip_alpha, 1.0), A);
	}
	__syncthreads();

	const int xi = blockIdx.x * kVThreads + t;
	const bool live = xi < P.W;
	const int x = min(xi, P.W - 1);
	const int y_begin = blockIdx.y * P.RPC, y_end = min(y_begin + P.RPC, P.OH);
	const int frame = frame0 + blockIdx.z;
	const uint8_t *col = in + (size_t) frame * P.in_frame_stride + (size_t) x * NCH;
	float *mcol = P.mid + (size_t) frame * P.mid_frame_stride + (size_t) x * NCH;
	const int m_end = y_end + 6; /* iterations: output row mm starts at iteration mm, completes at mm + 6 */

	/* iteration mm reads box-shrunk rows e = f0 + 2 mm (A) and e + 1 (B) */
	/* ring stage of iteration mm: (mm - y_begin) mod NST -- the unrolled loop below passes it as a constant
	 * when NST is 7 (the loop advances seven iterations at a time)
	 */
	auto prefetch = [&](int mm, int stage) {
		if (mm < m_end) {
			unsigned *dst = s_ring + stage * (ROWS * kVThreads) + t;
#pragma unroll
			for (int h = 0; h < 2; h++) {
				const int sr = max(0, min(P.f0 + 2 * mm + h - P.vembed, P.Hs - 1));
#pragma unroll
				for (int k = 0; k < VST; k++) {
					const int row = min(sr * VST + k, P.H - 1);
					const unsigned d = (unsigned) __cvta_generic_to_shared(dst + (h * VST + k) * kVThreads);
					asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(col + (size_t) row * P.in_bpl) : "memory");
				}
			}
		}
		asm volatile("cp.async.commit_group;" ::: "memory");
	};
#pragma unroll
	for (int d = 0; d < D2; d++)
		prefetch(y_begin + d, d % NST);

	double a[7][NCH];
#pragma unroll
	for (int J = 0; J < 7; J++)
#pragma unroll
		for (int c = 0; c < NCH; c++)
			a[J][c] = 0.0;

	for (int m = y_begin; m < m_end; m += 7) {
#pragma unroll
		for (int u = 0; u < 7; u++) {
			const int mm = m + u;
			if (mm < m_end) {
				const int stage = NST == 7 ? u : (mm - y_begin) % NST;
				prefetch(mm + D2, NST == 7 ? (u + D2) % NST : (mm + D2 - y_begin) % NST);
				asm volatile("cp.async.wait_group %0;" ::"n"(D2) : "memory");
				const unsigned *mine = s_ring + stage * (ROWS * kVThreads) + t;
				double sv[2][NCH];
#pragma unroll
				for (int h = 0; h < 2; h++) {
					double sum[NCH];
#pragma unroll
					for (int c = 0; c < NCH; c++)
						sum[c] = 0.0;
#pragma unroll
					for (int k = 0; k < VST; k++) {
						const unsigned px = mine[(h * VST + k) * kVThreads];
						const float r = s_lin[px & 255], g = s_lin[(px >> 8) & 255], b = s_lin[(px >> 16) & 255];
						const float2 an = s_aln[px >> 24];
						float q0 = r, q1 = g, q2 = b;
						if (PREMUL) {
							q0 = __fmul_rn(r, an.x);
							q1 = __fmul_rn(g, an.x);
							q2 = __fmul_rn(b, an.x);
						}
						sum[0] = __dadd_rn(sum[0], (double) q0);
						sum[1] = __dadd_rn(sum[1], (double) q1);
						sum[2] = __dadd_rn(sum[2], (double) q2);
						sum[3] = __dadd_rn(sum[3], (double) an.y);
					}
#pragma unroll
					for (int c = 0; c < NCH; c++)
						sv[h][c] = (double) (float) __dmul_rn(sum[c], P.inv_v);
				}
				/* row A: even taps.  Output row mm - j sits in slot (u - j) mod 7; slot u starts here */
#pragma unroll
				for (int c = 0; c < NCH; c++)
					a[u][c] = 0.0;
#pragma unroll
				for (int j = 0; j < 7; j++) {
					const int sl = (u - j + 7) % 7;
#pragma unroll
					for (int c = 0; c < NCH; c++)
						a[sl][c] = __dadd_rn(a[sl][c], __dmul_rn(P.c2[2 * j], sv[0][c]));
				}
				{
					const int y = mm - 6, sl = (u + 1) % 7;
					if (live && y >= y_begin)
						*(float4 *) (mcol + (size_t) y * P.W * NCH) =
							make_float4((float) a[sl][0], (float) a[sl][1], (float) a[sl][2], (float) a[sl][3]);
				}
				/* row B: odd taps */
#pragma unroll
				for (int j = 0; j < 6; j++) {
					const int sl = (u - j + 7) % 7;
#pragma unroll
					for (int c = 0; c < NCH; c++)
						a[sl][c] = __dadd_rn(a[sl][c], __dmul_rn(P.c2[2 * j + 1], sv[1][c]));
				}
			}
		}
	}
}

template <int NCH, bool PREMUL>
__global__ void __launch_bounds__(256)
linear_h_kernel(const __grid_constant__ LinHParams P, uint8_t *__restrict__ out, int frame0)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	float *s_row = (float *) smem_raw;								 /* [OW][NCH] the reduceh result */
	float *s_shr = s_row + ((P.OW * NCH + 3) & ~3);					 /* [Wse][NCH] the box-shrunk, embedded row */
	double *s_hc = (double *) (s_shr + ((P.Wse * NCH + 3) & ~3));	 /* [65 * nh] */
	float *s_Y2v = (float *) (s_hc + 65 * P.nh);					 /* [257], integers as floats */

	const int t = threadIdx.x;
	for (int i = t; i < 65 * P.nh; i += 256)
		s_hc[i] = P.hcoef[i];
	for (int i = t; i < 257; i += 256)
		s_Y2v[i] = (float) P.Y2v_8[i];

	const int y = blockIdx.x;
	const int frame = frame0 + blockIdx.y;
	const float *row = P.mid + (size_t) frame * P.mid_frame_stride + (size_t) y * P.W * NCH;

	/* ---- shrinkh (FSHRINK, shrinkh.c:134-152) over the embedded row: vips_embed(EXTEND_COPY) = clamp.
	 * One (column, band) per thread straight from the intermediate image: the NCH lanes of a column read
	 * NCH consecutive floats, a warp covers 32 / NCH boxes, and over the HS steps of the box every sector is
	 * used in full -- no staging of the 64 KB row, so many CTAs fit an SM and hide the loads' latency.
	 */
	__syncthreads();
	for (int i = t; i < P.Wse * NCH; i += 256) {
		const int j = NCH == 4 ? i >> 2 : i / NCH, c = i - j * NCH;
		const int sc = max(0, min(j - P.hembed, P.Ws - 1));
		double sum = 0.0;
		for (int k = 0; k < P.HS; k++)
			sum = __dadd_rn(sum, (double) __ldg(row + (size_t) min(sc * P.HS + k, P.W - 1) * NCH + c));
		s_shr[i] = (float) __dmul_rn(sum, P.inv_h);
	}
	__syncthreads();

	/* ---- reduceh (reduceh.cpp:182-193): one (pixel, band) per thread */
	for (int i = t; i < P.OW * NCH; i += 256) {
		const int x = NCH == 4 ? i >> 2 : i / NCH, c = i - x * NCH;
		const float *win = s_shr + __ldg(P.hfirst + x) * NCH + c;
		const double *cf = s_hc + __ldg(P.hphase + x) * P.nh;
		double sum = 0.0;
		for (int k = 0; k < P.nh; k++)
			sum = __dadd_rn(sum, __dmul_rn(cf[k], (double) win[k * NCH]));
		s_row[i] = (float) sum;
	}
	__syncthreads();

	/* ---- unpremultiply, scRGB -> sRGB: one pixel per thread */
	uint8_t *orow = out + (size_t) frame * P.out_frame_stride + (size_t) y * P.out_bpl;
	for (int x = t; x < P.OW; x += 256) {
		float v[NCH];
#pragma unroll
		for (int c = 0; c < NCH; c++)
			v[c] = s_row[x * NCH + c];
		if (PREMUL) {
			/* FUNPRE_RGBA with max_alpha 1.0, unpremultiply.c:160-176 */
			const float alpha = v[NCH - 1];
			const float factor = fabs((double) alpha) < 0.01 ? 0.0f : (float) __ddiv_rn(1.0, (double) alpha);
			v[0] = __fmul_rn(factor, v[0]);
			v[1] = __fmul_rn(factor, v[1]);
			v[2] = __fmul_rn(factor, v[2]);
			v[NCH - 1] = (float) fmax(0.0, fmin(1.0, (double) alpha));
		}
		unsigned R = 0, G = 0, B = 0;
		if (!(isnan(v[0]) || isnan(v[1]) || isnan(v[2]))) {
			R = (unsigned) scRGB2sRGB_channel_f(s_Y2v, 255.0f, v[0]) & 255u;
			G = (unsigned) scRGB2sRGB_channel_f(s_Y2v, 255.0f, v[1]) & 255u;
			B = (unsigned) scRGB2sRGB_channel_f(s_Y2v, 255.0f, v[2]) & 255u;
		}
		if (NCH == 4) {
			const unsigned A = (unsigned) (uint8_t) carry_extra_band((double) v[NCH - 1], P.bwd, P.n_bwd);
			*(unsigned *) (orow + (size_t) x * 4) = R | (G << 8) | (B << 16) | (A << 24);
		}
		else {
			orow[(size_t) x * 3] = (uint8_t) R;
			orow[(size_t) x * 3 + 1] = (uint8_t) G;
			orow[(size_t) x * 3 + 2] = (uint8_t) B;
		}
	}
}

} // namespace

struct LinearThumb {
	int W = 0, H = 0, OW = 0, OH = 0, bands = 0;
	bool premul = false;
	LinVParams v{};
	LinHParams h{};
	void *tables = nullptr;
	size_t smem_v = 0, smem_h = 0;
	int vst = 0;
	bool static2 = false; /* linear_v2_kernel: residual exactly 2.0, 13 taps, one phase */
};

/* 0 = ready, 1 = this geometry is not on the two-kernel path (the caller chains the leaf kernels), -1 = error */
int
linear_thumb_new(const char *domain, int W, int H, int bands, bool premul, const ReduceGeom &gv, const ReduceGeom &gh,
	const AxisTable &tv, const AxisTable &th, LinearThumb **out)
{
	*out = nullptr;
	if (getenv("VB200_NO_LINEAR_FUSED") != nullptr)
		return 1;
	if ((bands != 3 && bands != 4) || gv.n_point <= 0 || gh.n_point <= 0)
		return 1;
	if (bands == 4 && !premul)
		return 1; /* a 4th band that is not alpha (or an axis left alone): the general chain */
	const int OH = gv.out_size, OW = gh.out_size;
	if ((int) tv.first.size() < OH || (int) th.first.size() < OW)
		return 1;
	/* the column stream needs the windows to start in order and at most kSlots rows in flight */
	for (int y = 0; y + 1 < OH; y++)
		if (tv.first[y + 1] < tv.first[y])
			return 1;
	for (int y = 0; y + kSlots < OH; y++)
		if (tv.first[y + kSlots] < tv.first[y] + gv.n_point)
			return 1;
	int wse = 0;
	for (int x = 0; x < OW; x++)
		wse = std::max(wse, th.first[x] + gh.n_point);
	const size_t smem_v = (size_t) 65 * gv.n_point * 8 + 4 * 256 * 4 + (size_t) (kDepth + 1) * kMaxBox * kVThreads * 4;
	const size_t smem_h = (size_t) 65 * gh.n_point * 8 + 260 * 4 + (size_t) ((wse * bands + 3) & ~3) * 4 +
		(size_t) ((OW * bands + 3) & ~3) * 4;
	if (smem_v > 100 * 1024 || smem_h > 200 * 1024)
		return 1;

	RouteParams fwd, bwd;
	if (colour_route_params(domain, VB200_INTERPRETATION_sRGB, VB200_INTERPRETATION_scRGB, &fwd) ||
		colour_route_params(domain, VB200_INTERPRETATION_scRGB, VB200_INTERPRETATION_sRGB, &bwd))
		return -1;
	if (fwd.n_steps > 2 || bwd.n_steps > 2)
		return 1;

	LinearThumb *lt = new LinearThumb();
	lt->W = W;
	lt->H = H;
	lt->OW = OW;
	lt->OH = OH;
	lt->bands = bands;
	lt->premul = premul;
	lt->smem_v = smem_v;
	lt->smem_h = smem_h;
	lt->vst = gv.int_shrink == 2 || gv.int_shrink == 4 || gv.int_shrink == 8 ? gv.int_shrink : 0;

	/* one device block: vfirst | vphase | hfirst | hphase | vcoef | hcoef */
	const size_t n_vi = (size_t) OH * 4, n_hi = (size_t) OW * 4;
	const size_t n_vc = (size_t) 65 * gv.n_point * 8, n_hc = (size_t) 65 * gh.n_point * 8;
	size_t off_vc = 2 * n_vi + 2 * n_hi;
	off_vc = (off_vc + 7) & ~(size_t) 7;
	std::vector<char> host(off_vc + n_vc + n_hc);
	memcpy(&host[0], tv.first.data(), n_vi);
	memcpy(&host[n_vi], tv.phase.data(), n_vi);
	memcpy(&host[2 * n_vi], th.first.data(), n_hi);
	memcpy(&host[2 * n_vi + n_hi], th.phase.data(), n_hi);
	memcpy(&host[off_vc], tv.mf.data(), n_vc);
	memcpy(&host[off_vc + n_vc], th.mf.data(), n_hc);
	if (cudaMalloc(&lt->tables, host.size()) != cudaSuccess ||
		cudaMemcpy(lt->tables, host.data(), host.size(), cudaMemcpyHostToDevice) != cudaSuccess) {
		cuda_fail(domain, cudaGetLastError(), "linear thumbnail tables");
		delete lt;
		return -1;
	}
	char *b = (char *) lt->tables;

	LinVParams &v = lt->v;
	v.W = W;
	v.H = H;
	v.OH = OH;
	v.VS = gv.int_shrink;
	v.Hs = gv.shrunk_size;
	v.vembed = tv.embed;
	v.nv = gv.n_point;
	v.in_bpl = (size_t) W * bands;
	v.vfirst = (const int *) b;
	v.vphase = (const int *) (b + n_vi);
	v.vcoef = (const double *) (b + off_vc);
	v.inv_v = 1.0 / gv.int_shrink;
	memcpy(v.fwd, fwd.steps, sizeof(v.fwd));
	v.n_fwd = fwd.n_steps;
	v.v2Y_8 = fwd.t.v2Y_8;
	/* the static schedule: every window two box-shrunk rows after the last, one set of 13 coefficients */
	lt->static2 = bands == 4 && lt->vst != 0 && gv.n_point == 13 && getenv("VB200_NO_LINEAR_STATIC") == nullptr;
	for (int y = 0; y < OH && lt->static2; y++)
		if (tv.first[y] != tv.first[0] + 2 * y || tv.phase[y] != tv.phase[0])
			lt->static2 = false;
	if (lt->static2) {
		v.f0 = tv.first[0];
		for (int i = 0; i < 13; i++)
			v.c2[i] = tv.mf[(size_t) tv.phase[0] * 13 + i];
	}

	LinHParams &h = lt->h;
	h.W = W;
	h.OW = OW;
	h.OH = OH;
	h.HS = gh.int_shrink;
	h.Ws = gh.shrunk_size;
	h.hembed = th.embed;
	h.nh = gh.n_point;
	h.Wse = wse;
	h.hfirst = (const int *) (b + 2 * n_vi);
	h.hphase = (const int *) (b + 2 * n_vi + n_hi);
	h.hcoef = (const double *) (b + off_vc + n_vc);
	h.out_bpl = (size_t) OW * bands;
	h.inv_h = 1.0 / gh.int_shrink;
	memcpy(h.bwd, bwd.steps, sizeof(h.bwd));
	h.n_bwd = bwd.n_steps;
	h.Y2v_8 = bwd.t.Y2v_8;
	*out = lt;
	return 0;
}

void
linear_thumb_free(LinearThumb *lt)
{
	if (!lt)
		return;
	if (lt->tables)
		cudaFree(lt->tables);
	delete lt;
}

namespace {

template <int NCH, bool PREMUL>
int
launch_v(const char *domain, const LinearThumb *lt, const LinVParams &v, const void *in, dim3 grid, int f0, cudaStream_t s)
{
#define LV(VST_) \
	do { \
		auto kern = linear_v_kernel<NCH, PREMUL, VST_>; \
		VB200_CUDA(domain, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) lt->smem_v)); \
		kern<<<grid, kVThreads, lt->smem_v, s>>>(v, (const uint8_t *) in, f0); \
	} while (0)
	switch (lt->vst) {
	case 2: LV(2); break;
	case 4: LV(4); break;
	case 8: LV(8); break;
	default: LV(0); break;
	}
#undef LV
	return 0;
}

int
launch_v2(const char *domain, const LinearThumb *lt, const LinVParams &v, const void *in, dim3 grid, cudaStream_t s)
{
#define LV2(PM_, VST_) \
	do { \
		auto kern = linear_v2_kernel<PM_, VST_>; \
		VB200_CUDA(domain, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) lt->smem_v)); \
		kern<<<grid, kVThreads, lt->smem_v, s>>>(v, (const uint8_t *) in, 0); \
	} while (0)
	if (lt->premul) {
		switch (lt->vst) {
		case 2: LV2(true, 2); break;
		case 4: LV2(true, 4); break;
		default: LV2(true, 8); break;
		}
	}
	else {
		switch (lt->vst) {
		case 2: LV2(false, 2); break;
		case 4: LV2(false, 4); break;
		default: LV2(false, 8); break;
		}
	}
#undef LV2
	return 0;
}

} // namespace

/* frames: packed uchar, `bands` per pixel; queued on s.  The float intermediate ([OH][W][bands] per frame)
 * comes from the stream-ordered pool, at most kSub frames of it at a time.
 */
int
linear_thumb_run(const char *domain, LinearThumb *lt, const void *in, size_t in_stride, void *out, size_t out_stride, int n,
	cudaStream_t s)
{
	if (n <= 0)
		return 0;
	if (lt->bands == 4 && ((((uintptr_t) in) | in_stride | ((uintptr_t) out) | out_stride) & 3) != 0) {
		error(domain, "RGBA frames must be 4-byte aligned");
		return -1;
	}
	const size_t mid_frame = (size_t) lt->OH * lt->W * lt->bands; /* floats */
	/* sub-batches keep the scratch near 2 GiB (33.5 MB per 4K frame) and, at small sizes, inside L2 */
	const int sub = (int) std::max<size_t>(1, std::min<size_t>((size_t) n, ((size_t) 2 << 30) / (mid_frame * 4)));
	float *mid = nullptr;
	if (dev_alloc(domain, (void **) &mid, mid_frame * 4 * sub, s))
		return -1;
	int rc = 0;
	for (int f0 = 0; f0 < n && !rc; f0 += sub) {
		const int nf = std::min(sub, n - f0);
		LinVParams v = lt->v;
		v.in_frame_stride = in_stride;
		v.mid = mid;
		v.mid_frame_stride = mid_frame;
		/* rows per CTA: the whole height when there are enough frames to fill the machine */
		const int col_blocks = (lt->W + kVThreads - 1) / kVThreads;
		int splits = 1;
		while ((long) col_blocks * splits * nf < 4 * sm_count() && lt->OH / (splits * 2) >= 16)
			splits *= 2;
		v.RPC = (lt->OH + splits - 1) / splits;
		const dim3 gv(col_blocks, (lt->OH + v.RPC - 1) / v.RPC, nf);
		const char *fin = (const char *) in + (size_t) f0 * in_stride;
		if (lt->static2)
			rc = launch_v2(domain, lt, v, fin, gv, s);
		else if (lt->bands == 4)
			rc = lt->premul ? launch_v<4, true>(domain, lt, v, fin, gv, 0, s) : launch_v<4, false>(domain, lt, v, fin, gv, 0, s);
		else
			rc = launch_v<3, false>(domain, lt, v, fin, gv, 0, s);
		cudaError_t e = cudaGetLastError();
		if (!rc && e != cudaSuccess)
			rc = cuda_fail(domain, e, "linear_v_kernel launch");
		if (rc)
			break;
		count_launch();

		LinHParams h = lt->h;
		h.mid = mid;
		h.mid_frame_stride = mid_frame;
		h.out_frame_stride = out_stride;
		const dim3 gh(lt->OH, nf);
		uint8_t *fout = (uint8_t *) out + (size_t) f0 * out_stride;
		if (lt->bands == 4) {
			auto kern = lt->premul ? linear_h_kernel<4, true> : linear_h_kernel<4, false>;
			cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) lt->smem_h);
			kern<<<gh, 256, lt->smem_h, s>>>(h, fout, 0);
		}
		else {
			auto kern = linear_h_kernel<3, false>;
			cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) lt->smem_h);
			kern<<<gh, 256, lt->smem_h, s>>>(h, fout, 0);
		}
		e = cudaGetLastError();
		if (e != cudaSuccess)
			rc = cuda_fail(domain, e, "linear_h_kernel launch");
		else
			count_launch();
	}
	dev_free(mid, s);
	return rc;
}

size_t
linear_thumb_scratch_bytes_per_frame(const LinearThumb *lt)
{
	return (size_t) lt->OH * lt->W * lt->bands * 4;
}

} // namespace vb200
