/* thumbnail_fused.cu -- ONE kernel for the whole uchar RGBA thumbnail chain
 *
 *   premultiply(uchar) -> shrinkv(box) -> reducev(kernel) -> shrinkh(box) -> reduceh(kernel) -> unpremultiply(uchar)
 *
 * i.e. what vips_thumbnail_image() builds for an 8-bit image with alpha
 * (reference: resample/thumbnail.c:848-902 -> resize.c:213-231 ->
 * reducev.cpp:898-922 / reduceh.cpp:436-460), with every intermediate uchar
 * rounding of the unfused reference chain reproduced bit for bit.
 *
 * Work decomposition (HBM-bound design: each input byte is read once from
 * DRAM, the 13-tap windows live in shared memory, nothing but the final
 * thumbnail is written back):
 *
 *   CTA      = a band of TW output columns x RPC output rows of one frame.
 *   thread   = one INPUT pixel column of the band (incl. the reduceh halo).  It
 *              streams down the rows with coalesced 32-bit loads (a warp reads
 *              128 contiguous bytes per row), premultiplies, box-sums vshrink
 *              rows in 16-bit SIMD lanes, and keeps its private window of
 *              box-shrunk rows in a shared-memory column, stored as
 *              byte-transposed ROW PAIRS so that one dp2a does two taps.
 *   per chunk of K output rows:
 *     stage V  every thread: produce the row pairs the chunk needs, then K
 *              reducev outputs (dp2a over the pair window) -> rv[K][cols]
 *     stage H1 box-sum hshrink adjacent columns of rv -> column PAIRS sh[K][..]
 *     stage H2 one thread per output pixel: reduceh (dp2a over column pairs),
 *              unpremultiply, 32-bit coalesced store.
 *
 * Sampling positions come from host tables built by the same sequential
 * double additions as the reference's generate functions (see
 * build_axis_table), so fractional shrinks and tile-dependent phases match.
 */
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <vector>

#include <cuda.h> /* CUtensorMap + the cuTensorMapEncodeTiled prototype; resolved at run time, libcuda is not linked */

#include "vb200_internal.h"

namespace vb200 {

namespace {

constexpr int kChunkRows = 8; /* K */
constexpr int kMaxThreads = 576; /* 18 consumer warps (+1 producer in v2): 2 CTAs per SM at 48 registers */

struct FusedParams {
	/* input frame geometry */
	int W, H;
	size_t in_bpl;
	/* vertical */
	int VS;		  /* box shrink */
	int Hs;		  /* rows after the box shrink */
	int vembed;	  /* ceil(n_v / 2) - 1 */
	int NPv;	  /* coefficient pairs per vertical set */
	unsigned vmul8; /* ((1 << 32) / (256 * VS)) << 8, for umulhi */
	int vshift;	  /* log2(VS) if VS is a power of two, else -1 */
	unsigned accmul; /* v4: 256 / VS when VS is a power of two (box sums scaled by it before the byte pick), else 1 */
	/* horizontal */
	int HS, Ws, hembed, NPh;
	unsigned hmul8;
	int hshift;
	int OW, OH;
	size_t out_bpl;
	/* decomposition */
	int TW;	 /* output columns per CTA */
	int RPC; /* output rows per CTA */
	int NT;	 /* threads per CTA == pair-buffer column stride */
	int NEmax; /* max embedded shrinkh columns per band (even) */
	int slots;	/* pair slots per column */
	int stage_pitch; /* v2: bytes between rows of a TMA stage (multiple of 16) */
	int vgrid, hgrid; /* pair p covers embedded rows / columns 2p + grid, 2p + grid + 1 */
	/* tables */
	const int2 *vrow;  /* [OH] {first pair (embedded rows >> 1), coefficient set} */
	const int2 *hcol;  /* [OW] {first pair (embedded cols >> 1), coefficient set} */
	const int *vcoef;  /* [nvsets][NPv] packed s16x2 */
	const int *hcoef;  /* [nhsets][NPh] */
	int nvsets, nhsets;
	/* v4 (thumbnail_fused_mma.cuh) */
	const int2 *vchunk;	 /* [ceil(OH / 8)] {first quad, last quad} of each 8-row chunk */
	const uint4 *vbfrag; /* [chunks][32] B fragments {hi b0, hi b1, lo b0, lo b1} */
	int mma_rows;		 /* output rows per chunk (4 .. 8) */
	/* alpha */
	int premul;		  /* 1: premultiply/unpremultiply with max_alpha */
	const unsigned char *opaque_hint; /* v4: [frames of the launch] 1 = arm the V warps' opaque-stage vote for this frame; nullptr = never */
	double max_alpha; /* LUTs are derived from it in the prologue */
};

/* One band of the tensor-pipe kernel: output columns [xa, xb), ne embedded shrinkh columns, and the input columns
 * [c_lo, c_hi) its stage rows load (c_lo on the layout's box alignment, c_hi on 16 bytes) -- what
 * thumbnail_fused_mma.cuh derives from column_of
 */
struct MmaBand {
	int xa, xb, ne, c_lo, c_hi;
};

__device__ __forceinline__ int
dp2a_lo(unsigned coef, unsigned bytes, int acc)
{
	int d;
	asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(coef), "r"(bytes), "r"(acc));
	return d;
}

__device__ __forceinline__ int
dp2a_hi(unsigned coef, unsigned bytes, int acc)
{
	int d;
	asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(coef), "r"(bytes), "r"(acc));
	return d;
}

__device__ __forceinline__ unsigned
ld_stream(const unsigned *p)
{
	unsigned v;
	asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
	return v;
}

/* Box-sum VS premultiplied rows of one pixel column into 16-bit lanes:
 * rb = r | b << 16, ga = g | a << 16, both pre-loaded with the rounding amend.
 */
template <int VS, bool PREMUL>
__device__ __forceinline__ void
box_rows(const unsigned (&px)[VS], int vs, const int *pscale, bool lut, unsigned amend2, unsigned &rb, unsigned &ga)
{
	rb = amend2;
	ga = amend2;
#pragma unroll
	for (int k = 0; k < VS; k++) {
		const unsigned x = px[k];
		if (PREMUL) {
			/* out = (in * scale[alpha] + 128) >> 8, premultiply.c:152-166;
			 * for max_alpha 255 scale[a] = a + (a == 255).
			 */
			const unsigned a = x >> 24;
			const unsigned s = lut ? (unsigned) pscale[a] : a + (a == 255u);
			const unsigned prb = (((x & 0x00ff00ffu) * s + 0x00800080u) >> 8) & 0x00ff00ffu;
			const unsigned pg = ((((x >> 8) & 0xffu) * s + 128u) >> 8) & 0xffu;
			rb += prb;
			ga += pg + (a << 16);
		}
		else {
			rb += x & 0x00ff00ffu;
			ga += (x >> 8) & 0x00ff00ffu;
		}
	}
}

/* ((sum + amend) * multiplier) >> 24 per 16-bit lane (shrinkv.c:218-227),
 * amend already inside; result lanes are bytes.
 */
__device__ __forceinline__ unsigned
box_average(unsigned lanes, unsigned mul8, int shift)
{
	if (shift >= 0)
		return (lanes >> shift) & 0x00ff00ffu;
	const unsigned lo = __umulhi(lanes & 0xffffu, mul8);
	const unsigned hi = __umulhi(lanes >> 16, mul8);
	return lo | (hi << 16);
}

template <int VS, bool PREMUL>
__global__ void __launch_bounds__(kMaxThreads, 2)
thumbnail_fused_kernel(const __grid_constant__ FusedParams P, const uint8_t *__restrict__ in, size_t in_frame_stride,
	uint8_t *__restrict__ out, size_t out_frame_stride, int frame0)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];

	const int NT = P.NT;
	const int t = threadIdx.x;
	const int vs = VS > 0 ? VS : P.VS;

	/* shared memory carve-up */
	uint2 *pairbuf = (uint2 *) smem_raw;							  /* [slots][NT] */
	unsigned *rv = (unsigned *) (pairbuf + (size_t) P.slots * NT); /* [K][NT] */
	uint2 *sh = (uint2 *) (rv + (size_t) kChunkRows * NT);		  /* [K][NEmax / 2] column pairs */
	int *vcoef = (int *) (sh + (size_t) kChunkRows * (P.NEmax / 2));
	int *hcoef = vcoef + P.nvsets * P.NPv;
	int *pscale = hcoef + P.nhsets * P.NPh; /* [256] premultiply LUT */
	int *uscale = pscale + 256;				/* [256] unpremultiply LUT */

	for (int i = t; i < P.nvsets * P.NPv; i += NT)
		vcoef[i] = P.vcoef[i];
	for (int i = t; i < P.nhsets * P.NPh; i += NT)
		hcoef[i] = P.hcoef[i];
	if (PREMUL)
		for (int i = t; i < 256; i += NT) {
			/* premultiply.c:253-259, unpremultiply.c:313-324 (IEEE double, exact on device) */
			const double clip = fmax(0.0, fmin(P.max_alpha, (double) i));
			pscale[i] = (int) __ddiv_rn(__dmul_rn(256.0, clip), P.max_alpha);
			uscale[i] = clip == 0 ? 0 : (int) __ddiv_rn(__dmul_rn(256.0, P.max_alpha), clip);
		}
	const bool lut = PREMUL && P.max_alpha != 255.0;

	/* which band / rows / frame */
	const int xa = blockIdx.x * P.TW;
	const int xb = min(xa + P.TW, P.OW);
	const int y_begin = blockIdx.y * P.RPC;
	const int y_end = min(y_begin + P.RPC, P.OH);
	const int frame = frame0 + blockIdx.z;
	const uint8_t *fin = in + (size_t) frame * in_frame_stride;
	uint8_t *fout = out + (size_t) frame * out_frame_stride;

	/* embedded shrinkh columns of this band: [E0, E0 + NE), E0 even */
	const int pair_h0 = __ldg(&P.hcol[xa]).x;
	const int E0 = 2 * pair_h0 + P.hgrid;
	const int NE = 2 * (__ldg(&P.hcol[xb - 1]).x + P.NPh - pair_h0);

	/* this thread's input pixel column (clamped: the two EXTEND_COPY embeds of
	 * reduceh.cpp:515-521 and shrinkh.c:383)
	 */
	const bool col_active = t < NE * P.HS;
	int in_col;
	{
		const int e = E0 + t / P.HS;
		const int k = t - (t / P.HS) * P.HS;
		const int sc = max(0, min(e - P.hembed, P.Ws - 1));
		in_col = min(sc * P.HS + k, P.W - 1);
	}
	const unsigned *col_ptr = (const unsigned *) fin + in_col;

	const unsigned amend2 = (unsigned) (vs / 2) * 0x00010001u;

	__syncthreads();

	int pdone = INT_MIN; /* pairs < pdone are in the buffer */
	int P0_prev = 0;

	for (int ya = y_begin; ya < y_end; ya += kChunkRows) {
		const int yb = min(ya + kChunkRows, y_end);
		const int P0 = __ldg(&P.vrow[ya]).x;
		const int P1 = __ldg(&P.vrow[yb - 1]).x + P.NPv - 1;

		if (col_active) {
			/* -------- stage V.a: carry the window over from the last chunk */
			int pfirst = P0;
			if (pdone > P0) {
				const int shift = P0 - P0_prev;
				if (shift > 0)
					for (int p = P0; p < pdone; p++)
						pairbuf[(size_t) (p - P0) * NT + t] = pairbuf[(size_t) (p - P0 + shift) * NT + t];
				pfirst = pdone;
			}

			/* -------- stage V.b: produce row pairs pfirst..P1 */
			for (int p = pfirst; p <= P1; p++) {
				unsigned rbA, gaA, rbB, gaB;
				/* embedded reducev rows 2p, 2p+1 -> box-shrunk rows (EXTEND_COPY
				 * embed of reducev.cpp:975-981) -> VS input rows each (the
				 * round-up embed of shrinkv.c:501)
				 */
				const int sA = max(0, min(2 * p + P.vgrid - P.vembed, P.Hs - 1));
				const int sB = max(0, min(2 * p + P.vgrid + 1 - P.vembed, P.Hs - 1));
				if (VS > 0) {
					unsigned pa[VS > 0 ? VS : 1], pb[VS > 0 ? VS : 1];
#pragma unroll
					for (int k = 0; k < VS; k++) {
						const int ra = min(sA * VS + k, P.H - 1);
						const int rb_ = min(sB * VS + k, P.H - 1);
						pa[k] = ld_stream((const unsigned *) ((const char *) col_ptr + (size_t) ra * P.in_bpl));
						pb[k] = ld_stream((const unsigned *) ((const char *) col_ptr + (size_t) rb_ * P.in_bpl));
					}
					box_rows<(VS > 0 ? VS : 1), PREMUL>(pa, vs, pscale, lut, amend2, rbA, gaA);
					box_rows<(VS > 0 ? VS : 1), PREMUL>(pb, vs, pscale, lut, amend2, rbB, gaB);
				}
				else {
					/* generic box height: one row at a time */
					rbA = gaA = rbB = gaB = amend2;
					for (int k = 0; k < vs; k++) {
						unsigned one[1], rb1, ga1;
						one[0] = ld_stream((const unsigned *) ((const char *) col_ptr + (size_t) min(sA * vs + k, P.H - 1) * P.in_bpl));
						box_rows<1, PREMUL>(one, 1, pscale, lut, 0u, rb1, ga1);
						rbA += rb1;
						gaA += ga1;
						one[0] = ld_stream((const unsigned *) ((const char *) col_ptr + (size_t) min(sB * vs + k, P.H - 1) * P.in_bpl));
						box_rows<1, PREMUL>(one, 1, pscale, lut, 0u, rb1, ga1);
						rbB += rb1;
						gaB += ga1;
					}
				}
				rbA = box_average(rbA, P.vmul8, P.vshift);
				gaA = box_average(gaA, P.vmul8, P.vshift);
				rbB = box_average(rbB, P.vmul8, P.vshift);
				gaB = box_average(gaB, P.vmul8, P.vshift);
				/* byte-transpose the pair: w.x = [rA rB bA bB], w.y = [gA gB aA aB] */
				uint2 w;
				w.x = __byte_perm(rbA, rbB, 0x6240);
				w.y = __byte_perm(gaA, gaB, 0x6240);
				pairbuf[(size_t) (p - P0) * NT + t] = w;
			}

			/* -------- stage V.c: reducev for the chunk's rows */
			for (int y = ya; y < yb; y++) {
				const int2 vr = __ldg(&P.vrow[y]);
				const uint2 *win = pairbuf + (size_t) (vr.x - P0) * NT + t;
				const int *cf = vcoef + vr.y * P.NPv;
				int r = VB200_INTERPOLATE_SCALE >> 1, g = r, b = r, a = r;
#pragma unroll 7
				for (int k = 0; k < P.NPv; k++) {
					const uint2 w = win[(size_t) k * NT];
					const unsigned c = (unsigned) cf[k];
					r = dp2a_lo(c, w.x, r);
					b = dp2a_hi(c, w.x, b);
					g = dp2a_lo(c, w.y, g);
					a = dp2a_hi(c, w.y, a);
				}
				/* unsigned_fixed_round + VIPS_CLIP(0, v, 255), reducev.cpp:461-471 */
				r = max(0, min(r >> VB200_INTERPOLATE_SHIFT, 255));
				g = max(0, min(g >> VB200_INTERPOLATE_SHIFT, 255));
				b = max(0, min(b >> VB200_INTERPOLATE_SHIFT, 255));
				a = max(0, min(a >> VB200_INTERPOLATE_SHIFT, 255));
				rv[(size_t) (y - ya) * NT + t] = (unsigned) r | ((unsigned) g << 8) | ((unsigned) b << 16) | ((unsigned) a << 24);
			}
		}
		pdone = P1 + 1;
		P0_prev = P0;

		__syncthreads();

		/* -------- stage H1: box-sum HS adjacent columns, emit column pairs
		 * q = ((amend + sum) * multiplier) >> 24, shrinkh.c:78-93
		 */
		const int rows = yb - ya;
		const int npairs = NE / 2;
		const unsigned hamend2 = (unsigned) (P.HS / 2) * 0x00010001u;
		for (int idx = t; idx < rows * npairs; idx += NT) {
			const int k = idx / npairs;
			const int j = idx - k * npairs;
			const unsigned *src = rv + (size_t) k * NT + (size_t) (2 * j) * P.HS;
			unsigned rbA = hamend2, gaA = hamend2, rbB = hamend2, gaB = hamend2;
			for (int i = 0; i < P.HS; i++) {
				const unsigned wA = src[i];
				const unsigned wB = src[P.HS + i];
				rbA += wA & 0x00ff00ffu;
				gaA += (wA >> 8) & 0x00ff00ffu;
				rbB += wB & 0x00ff00ffu;
				gaB += (wB >> 8) & 0x00ff00ffu;
			}
			rbA = box_average(rbA, P.hmul8, P.hshift);
			gaA = box_average(gaA, P.hmul8, P.hshift);
			rbB = box_average(rbB, P.hmul8, P.hshift);
			gaB = box_average(gaB, P.hmul8, P.hshift);
			uint2 w;
			w.x = __byte_perm(rbA, rbB, 0x6240);
			w.y = __byte_perm(gaA, gaB, 0x6240);
			sh[(size_t) k * (P.NEmax / 2) + j] = w;
		}

		__syncthreads();

		/* -------- stage H2: reduceh + unpremultiply + store */
		const int bw = xb - xa;
		for (int idx = t; idx < rows * bw; idx += NT) {
			const int k = idx / bw;
			const int x = xa + (idx - k * bw);
			const int2 hc = __ldg(&P.hcol[x]);
			const uint2 *win = sh + (size_t) k * (P.NEmax / 2) + (hc.x - pair_h0);
			const int *cf = hcoef + hc.y * P.NPh;
			int r = VB200_INTERPOLATE_SCALE >> 1, g = r, b = r, a = r;
#pragma unroll 7
			for (int kk = 0; kk < P.NPh; kk++) {
				const uint2 w = win[kk];
				const unsigned c = (unsigned) cf[kk];
				r = dp2a_lo(c, w.x, r);
				b = dp2a_hi(c, w.x, b);
				g = dp2a_lo(c, w.y, g);
				a = dp2a_hi(c, w.y, a);
			}
			r = max(0, min(r >> VB200_INTERPOLATE_SHIFT, 255));
			g = max(0, min(g >> VB200_INTERPOLATE_SHIFT, 255));
			b = max(0, min(b >> VB200_INTERPOLATE_SHIFT, 255));
			a = max(0, min(a >> VB200_INTERPOLATE_SHIFT, 255));
			if (PREMUL) {
				/* unpremultiply.c:209-222: byte store without clip */
				const int s = uscale[a];
				r = ((r * s + 128) >> 8) & 0xff;
				g = ((g * s + 128) >> 8) & 0xff;
				b = ((b * s + 128) >> 8) & 0xff;
			}
			*(unsigned *) (fout + (size_t) (ya + k) * P.out_bpl + (size_t) x * 4) =
				(unsigned) r | ((unsigned) g << 8) | ((unsigned) b << 16) | ((unsigned) a << 24);
		}
		/* the next chunk's stage V writes pairbuf/rv (not read after H1) and its
		 * H1 writes sh only after its own barrier: no third barrier needed.
		 */
	}
}

/* ======================================================================
 * v2: the same chain with the input rows brought on chip by the TMA engine.
 *
 * A producer warp (one elected lane) streams the band's input rows into a
 * shared-memory ring with cp.async.bulk (one bulk copy per row, completion
 * counted on an mbarrier per stage); the consumer threads never form a global
 * address: each pixel costs them one LDS.  A stage holds the 2 * VS input rows
 * of one box-shrunk ROW PAIR.  full[] / empty[] mbarriers hand the stages back
 * and forth; the consumers' block barrier is a named barrier that excludes the
 * producer warp.  Arithmetic is identical to v1 (and to the reference).
 * ====================================================================== */

constexpr int kStages = 3;
constexpr int kChunkRowsTma = 4;
constexpr int kColsPerThread = 2;
/* bytes between rows of a stage: a compile-time constant so the 2 * VS row
 * reads of a pair are LDS with immediate offsets (band width <= kMaxThreads + 6 columns)
 */
constexpr int kStagePitch = (kMaxThreads + 8) * 4;

__device__ __forceinline__ unsigned
smem_addr(const void *p)
{
	return (unsigned) __cvta_generic_to_shared(p);
}

__device__ __forceinline__ void
mbar_init(unsigned bar, unsigned count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}

__device__ __forceinline__ void
mbar_wait(unsigned bar, unsigned parity)
{
	unsigned done;
	do {
		asm volatile("{\n\t.reg .pred p;\n\t"
					 "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, 0x989680;\n\t"
					 "selp.u32 %0, 1, 0, p;\n\t}"
					 : "=r"(done)
					 : "r"(bar), "r"(parity)
					 : "memory");
	} while (!done);
}

__device__ __forceinline__ void
mbar_arrive(unsigned bar)
{
	asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}

__device__ __forceinline__ void
mbar_expect_tx(unsigned bar, unsigned bytes)
{
	asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(bar), "r"(bytes)
				 : "memory");
}

__device__ __forceinline__ void
bulk_copy_g2s(unsigned dst, const void *src, unsigned bytes, unsigned bar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
				 "l"(src), "r"(bytes), "r"(bar)
				 : "memory");
}

/* idx / d for 0 <= idx < 4096 and 1 <= d: exact via a float reciprocal + one correction */
__device__ __forceinline__ int
fast_div(int idx, int d)
{
	int q = (int) (__int2float_rn(idx) * __frcp_rn(__int2float_rn(d)));
	const int r = idx - q * d;
	q += (r >= d) - (r < 0);
	return q;
}

__device__ __forceinline__ void
consumer_barrier(int n_threads)
{
	asm volatile("bar.sync 1, %0;" ::"r"(n_threads) : "memory");
}

/* one pixel: premultiply (max_alpha 255) and add into the 16-bit-lane accumulators */
template <bool PREMUL>
__device__ __forceinline__ void
accumulate_pixel(unsigned x, unsigned &rb, unsigned &ga)
{
	if (PREMUL) {
		/* out = (in * scale[alpha] + 128) >> 8 with scale[a] = (int) (256 * a / 255.0)
		 * = a + (a == 255) = (a * 257 + 1) >> 8      premultiply.c:152-166, 253-259
		 */
		const unsigned a = x >> 24;
		const unsigned s = (a * 257u + 1u) >> 8;
		const unsigned trb = (x & 0x00ff00ffu) * s + 0x00800080u;
		const unsigned tg = __byte_perm(x, 0, 0x4441) * s + 128u; /* bytes [lo, g', 0, 0] */
		rb += __byte_perm(trb, 0, 0x4341);						  /* [r', 0, b', 0] */
		ga += __byte_perm(tg, x, 0x3731);						  /* [g', 0, a, 0] */
	}
	else {
		rb += x & 0x00ff00ffu;
		ga += __byte_perm(x, 0, 0x4341);
	}
}

/* box average of both rows of a pair + byte transposition: [A0 B0 A2 B2] */
__device__ __forceinline__ unsigned
average_pair(unsigned lanesA, unsigned lanesB, unsigned mul8, int shift)
{
	if (shift >= 0)
		/* bytes 0 and 2 of (lanes >> shift) are exact: no masking needed */
		return __byte_perm(lanesA >> shift, lanesB >> shift, 0x6240);
	const unsigned a = __umulhi(lanesA & 0xffffu, mul8) | (__umulhi(lanesA >> 16, mul8) << 16);
	const unsigned b = __umulhi(lanesB & 0xffffu, mul8) | (__umulhi(lanesB >> 16, mul8) << 16);
	return __byte_perm(a, b, 0x6240);
}

/* Box sums on the half2 adder.  A 16-bit lane holding an integer below 1024 IS an fp16
 * denormal (value n * 2^-24), denormals and the first normal binade share one spacing, so
 * add.f16x2 (no .ftz) adds the lanes as integers, exactly, while a lane stays below 2048 --
 * and a box of up to 8 bytes + its rounding amend does.  HADD2 keeps the accumulation off
 * both the alu pipe and the IMAD half of the fma pipe.
 */
__device__ __forceinline__ unsigned
hadd2_lanes(unsigned a, unsigned b)
{
	unsigned d;
	asm("add.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
	return d;
}

template <bool PREMUL>
__device__ __forceinline__ void
accumulate_pixel_h(unsigned x, unsigned k16, unsigned &rb, unsigned &ga)
{
	if (PREMUL) {
		/* s = (a * 257 + 1) >> 8 = hi32((a << 24 | 1 << 16) * 257); k16 = 1 << 16 held in a register so that the
		 * mask-and-or is ONE LOP3 (it encodes a single immediate)
		 */
		unsigned t0;
		asm("lop3.b32 %0, %1, 0xff000000, %2, 0xea;" : "=r"(t0) : "r"(x), "r"(k16)); /* (x & 0xff000000) | k16 */
		const unsigned s = __umulhi(t0, 257u);
		const unsigned trb = (x & 0x00ff00ffu) * s + 0x00800080u; /* 16-bit lanes r * s + 128, b * s + 128 */
		const unsigned tg = (x & 0x0000ff00u) * s + 0x00008000u;	  /* (g * s + 128) << 8: byte 2 = g', byte 3 = 0 */
		rb = hadd2_lanes(rb, __byte_perm(trb, 0, 0x4341));
		ga = hadd2_lanes(ga, __byte_perm(tg, x, 0x3732));
	}
	else {
		rb = hadd2_lanes(rb, x & 0x00ff00ffu);
		ga = hadd2_lanes(ga, __byte_perm(x, 0, 0x4341));
	}
}

__device__ __forceinline__ unsigned
finalize_pack(int r, int g, int b, int a)
{
	/* unsigned_fixed_round + VIPS_CLIP(0, v, 255), reducev.cpp:461-471 */
	r = max(0, min(r >> VB200_INTERPOLATE_SHIFT, 255));
	g = max(0, min(g >> VB200_INTERPOLATE_SHIFT, 255));
	b = max(0, min(b >> VB200_INTERPOLATE_SHIFT, 255));
	a = max(0, min(a >> VB200_INTERPOLATE_SHIFT, 255));
	return (unsigned) r + (unsigned) g * 256u + (unsigned) b * 65536u + (unsigned) a * 16777216u;
}

/* NP > 0: both axes use exactly NP coefficient pairs (unrolled, vertical
 * coefficients in registers); NP == 0: run-time pair counts.
 * CPT: adjacent input pixel columns per consumer thread.  Two columns halve
 * every per-thread overhead (barrier waits, loop control, window addressing,
 * coefficient loads) and turn the window traffic into 128-bit LDS / STS.
 */
template <int VS, int NP, bool PREMUL, int CPT>
__global__ void __launch_bounds__(kMaxThreads / CPT + 32, 2)
thumbnail_fused_tma_kernel(const __grid_constant__ FusedParams P, const uint8_t *__restrict__ in, size_t in_frame_stride,
	uint8_t *__restrict__ out, size_t out_frame_stride, int frame0)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];

	constexpr int K = kChunkRowsTma;
	constexpr int NPR = NP > 0 ? NP : 1;
	constexpr int VSR = VS > 0 ? VS : 1;
	const int NT = P.NT;	   /* consumer threads; the producer warp is threads NT..NT+31 */
	const int NC = NT * CPT; /* columns: the stride of pairbuf / rv */
	const int t = threadIdx.x;
	const int vs = VS > 0 ? VS : P.VS;
	const int NPv = NP > 0 ? NP : P.NPv;
	const int NPh = NP > 0 ? NP : P.NPh;
	const int rows_per_stage = 2 * vs;
	const unsigned stage_bytes = (unsigned) rows_per_stage * kStagePitch;

	unsigned char *stages = smem_raw; /* [kStages][2 * vs][kStagePitch] */
	uint64_t *bars = (uint64_t *) (smem_raw + kStages * stage_bytes);
	uint2 *pairbuf = (uint2 *) (bars + 2 * kStages);			  /* [slots][NC] */
	unsigned *rv = (unsigned *) (pairbuf + (size_t) P.slots * NC); /* [K][NC] */
	uint2 *sh = (uint2 *) (rv + (size_t) K * NC);				  /* [K][NEmax / 2] */
	int *vcoef = (int *) (sh + (size_t) K * (P.NEmax / 2));
	int *hcoef = vcoef + P.nvsets * P.NPv;
	int *uscale = hcoef + P.nhsets * P.NPh; /* [256] unpremultiply LUT */

	const unsigned stages_s = smem_addr(stages);
	const unsigned full_s = smem_addr(bars);		   /* full[i] at + 8 * i */
	const unsigned empty_s = full_s + 8u * kStages; /* empty[i] at + 8 * i */

	if (t == 0) {
		for (int i = 0; i < kStages; i++) {
			mbar_init(full_s + 8u * i, 1);
			mbar_init(empty_s + 8u * i, NT / 32);
		}
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	for (int i = t; i < P.nvsets * P.NPv; i += blockDim.x)
		vcoef[i] = P.vcoef[i];
	for (int i = t; i < P.nhsets * P.NPh; i += blockDim.x)
		hcoef[i] = P.hcoef[i];
	if (PREMUL)
		for (int i = t; i < 256; i += blockDim.x)
			/* unpremultiply.c:313-324 with max_alpha 255 (IEEE double, exact on device) */
			uscale[i] = i == 0 ? 0 : (int) __ddiv_rn(__dmul_rn(256.0, 255.0), (double) i);

	const int xa = blockIdx.x * P.TW;
	const int xb = min(xa + P.TW, P.OW);
	const int y_begin = blockIdx.y * P.RPC;
	const int y_end = min(y_begin + P.RPC, P.OH);
	const int frame = frame0 + blockIdx.z;
	const uint8_t *fin = in + (size_t) frame * in_frame_stride;
	uint8_t *fout = out + (size_t) frame * out_frame_stride;

	const int pair_h0 = __ldg(&P.hcol[xa]).x;
	const int E0 = 2 * pair_h0 + P.hgrid;
	const int NE = 2 * (__ldg(&P.hcol[xb - 1]).x + P.NPh - pair_h0);

	/* input columns of the band: [c_lo, c_hi), 16-byte aligned for the bulk copies */
	auto column_of = [&](int tt) {
		const int e = E0 + tt / P.HS;
		const int k = tt - (tt / P.HS) * P.HS;
		const int sc = max(0, min(e - P.hembed, P.Ws - 1));
		return min(sc * P.HS + k, P.W - 1);
	};
	const int c_lo = column_of(0) & ~3;
	const int c_hi = min(P.W, (column_of(NE * P.HS - 1) + 4) & ~3);
	const unsigned row_bytes = (unsigned) (c_hi - c_lo) * 4u;

	__syncthreads();

	if (t >= NT) {
		/* ---------------- producer warp: lane L copies row L of each stage */
		const int lane = t - NT;
		const uint8_t *src0 = fin + (size_t) c_lo * 4;
		const int j = lane / vs, k = lane - j * vs; /* lane -> (row of the pair, row of the box) */
		const bool copier = lane < rows_per_stage;
		int s = 0;
		unsigned phase = 0;
		int pdone = INT_MIN;
		for (int ya = y_begin; ya < y_end; ya += K) {
			const int yb = min(ya + K, y_end);
			const int P0 = __ldg(&P.vrow[ya]).x;
			const int P1 = __ldg(&P.vrow[yb - 1]).x + P.NPv - 1;
			for (int p = max(pdone, P0); p <= P1; p++) {
				mbar_wait(empty_s + 8u * s, phase ^ 1u);
				if (lane == 0)
					mbar_expect_tx(full_s + 8u * s, (unsigned) rows_per_stage * row_bytes);
				__syncwarp();
				if (copier) {
					/* embedded reducev row -> box-shrunk row -> input row, all EXTEND_COPY */
					const int sr = max(0, min(2 * p + P.vgrid + j - P.vembed, P.Hs - 1));
					const int row = min(sr * vs + k, P.H - 1);
					bulk_copy_g2s(stages_s + (unsigned) s * stage_bytes + (unsigned) lane * kStagePitch,
						src0 + (size_t) row * P.in_bpl, row_bytes, full_s + 8u * s);
				}
				if (++s == kStages) {
					s = 0;
					phase ^= 1u;
				}
			}
			pdone = P1 + 1;
		}
		return;
	}

	/* ---------------- consumers */
	/* columns beyond the band shadow the last one */
	/* generic pointers into the ring: with the compile-time pitch the 2 * VS row
	 * reads of a pair become LDS [reg + immediate]
	 */
	const unsigned char *my_col[CPT];
#pragma unroll
	for (int i = 0; i < CPT; i++)
		my_col[i] = stages + (size_t) (column_of(min(t * CPT + i, NE * P.HS - 1)) - c_lo) * 4u;
	const unsigned amend2 = (unsigned) (vs / 2) * 0x00010001u;
	const bool lane0 = (t & 31) == 0;
	const unsigned vmul8 = P.vmul8;
	/* box height a power of two: the average is a compile-time shift */
	const int vshift = VS == 1 ? 0 : VS == 2 ? 1 : VS == 4 ? 2 : VS == 8 ? 3 : P.vshift;
	const int tc = t * CPT; /* first column of this thread */

	int s = 0;
	unsigned phase = 0;
	int pdone = INT_MIN;
	int P0_prev = 0;
	int cset = -1;
	unsigned cf[NPR];

	for (int ya = y_begin; ya < y_end; ya += K) {
		const int yb = min(ya + K, y_end);
		const int P0 = __ldg(&P.vrow[ya]).x;
		const int P1 = __ldg(&P.vrow[yb - 1]).x + P.NPv - 1;

		/* stage V.a: carry the window over */
		int pfirst = P0;
		if (pdone > P0) {
			const int shift = P0 - P0_prev;
			if (shift > 0) {
				const int cnt = pdone - P0;
				uint2 *dstp = pairbuf + tc;
				const uint2 *srcp = pairbuf + shift * NC + tc;
#pragma unroll 4
				for (int i = 0; i < cnt; i++) {
					if (CPT == 2)
						*(uint4 *) (dstp + i * NC) = *(const uint4 *) (srcp + i * NC);
					else
						dstp[i * NC] = srcp[i * NC];
				}
			}
			pfirst = pdone;
		}

		/* stage V.b: consume one ring stage per row pair */
		uint2 *pdst = pairbuf + (pfirst - P0) * NC + tc;
		for (int p = pfirst; p <= P1; p++, pdst += NC) {
			const unsigned soff = (unsigned) s * stage_bytes;
			unsigned rbA[CPT], gaA[CPT], rbB[CPT], gaB[CPT];
#pragma unroll
			for (int i = 0; i < CPT; i++)
				rbA[i] = gaA[i] = rbB[i] = gaB[i] = amend2;
			mbar_wait(full_s + 8u * s, phase);
			if (VS > 0) {
				unsigned pa[CPT][VSR], pb[CPT][VSR];
#pragma unroll
				for (int i = 0; i < CPT; i++)
#pragma unroll
					for (int k = 0; k < VSR; k++) {
						pa[i][k] = *(const unsigned *) (my_col[i] + soff + k * kStagePitch);
						pb[i][k] = *(const unsigned *) (my_col[i] + soff + (VSR + k) * kStagePitch);
					}
				__syncwarp();
				if (lane0)
					mbar_arrive(empty_s + 8u * s);
#pragma unroll
				for (int i = 0; i < CPT; i++)
#pragma unroll
					for (int k = 0; k < VSR; k++) {
						accumulate_pixel<PREMUL>(pa[i][k], rbA[i], gaA[i]);
						accumulate_pixel<PREMUL>(pb[i][k], rbB[i], gaB[i]);
					}
			}
			else {
				for (int k = 0; k < vs; k++)
#pragma unroll
					for (int i = 0; i < CPT; i++) {
						accumulate_pixel<PREMUL>(*(const unsigned *) (my_col[i] + soff + k * kStagePitch), rbA[i], gaA[i]);
						accumulate_pixel<PREMUL>(*(const unsigned *) (my_col[i] + soff + (vs + k) * kStagePitch), rbB[i], gaB[i]);
					}
				__syncwarp();
				if (lane0)
					mbar_arrive(empty_s + 8u * s);
			}
			if (++s == kStages) {
				s = 0;
				phase ^= 1u;
			}
			uint2 w[CPT];
#pragma unroll
			for (int i = 0; i < CPT; i++) {
				w[i].x = average_pair(rbA[i], rbB[i], vmul8, vshift); /* [rA rB bA bB] */
				w[i].y = average_pair(gaA[i], gaB[i], vmul8, vshift); /* [gA gB aA aB] */
			}
			if (CPT == 2)
				*(uint4 *) pdst = make_uint4(w[0].x, w[0].y, w[CPT - 1].x, w[CPT - 1].y);
			else
				*pdst = w[0];
		}

		/* stage V.c: reducev */
		unsigned *rvp = rv + tc;
		for (int y = ya; y < yb; y++, rvp += NC) {
			const int2 vr = __ldg(&P.vrow[y]);
			const uint2 *win = pairbuf + (vr.x - P0) * NC + tc;
			int acc[CPT][4];
#pragma unroll
			for (int i = 0; i < CPT; i++)
				acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = VB200_INTERPOLATE_SCALE >> 1;
			if (NP > 0) {
				if (vr.y != cset) {
					cset = vr.y;
#pragma unroll
					for (int k = 0; k < NPR; k++)
						cf[k] = (unsigned) vcoef[cset * NPR + k];
				}
#pragma unroll
				for (int k = 0; k < NPR; k++) {
					uint2 w[CPT];
					if (CPT == 2) {
						const uint4 q = *(const uint4 *) (win + k * NC);
						w[0] = make_uint2(q.x, q.y);
						w[CPT - 1] = make_uint2(q.z, q.w);
					}
					else
						w[0] = win[k * NC];
#pragma unroll
					for (int i = 0; i < CPT; i++) {
						acc[i][0] = dp2a_lo(cf[k], w[i].x, acc[i][0]);
						acc[i][2] = dp2a_hi(cf[k], w[i].x, acc[i][2]);
						acc[i][1] = dp2a_lo(cf[k], w[i].y, acc[i][1]);
						acc[i][3] = dp2a_hi(cf[k], w[i].y, acc[i][3]);
					}
				}
			}
			else {
				const int *cfp = vcoef + vr.y * NPv;
				for (int k = 0; k < NPv; k++) {
					const unsigned c = (unsigned) cfp[k];
#pragma unroll
					for (int i = 0; i < CPT; i++) {
						const uint2 w = win[k * NC + i];
						acc[i][0] = dp2a_lo(c, w.x, acc[i][0]);
						acc[i][2] = dp2a_hi(c, w.x, acc[i][2]);
						acc[i][1] = dp2a_lo(c, w.y, acc[i][1]);
						acc[i][3] = dp2a_hi(c, w.y, acc[i][3]);
					}
				}
			}
			if (CPT == 2)
				*(uint2 *) rvp = make_uint2(finalize_pack(acc[0][0], acc[0][1], acc[0][2], acc[0][3]),
					finalize_pack(acc[CPT - 1][0], acc[CPT - 1][1], acc[CPT - 1][2], acc[CPT - 1][3]));
			else
				*rvp = finalize_pack(acc[0][0], acc[0][1], acc[0][2], acc[0][3]);
		}
		pdone = P1 + 1;
		P0_prev = P0;

		consumer_barrier(NT);

		/* stage H1: box-sum HS adjacent columns -> column pairs */
		const int rows = yb - ya;
		const int npairs = NE / 2;
		const unsigned hamend2 = (unsigned) (P.HS / 2) * 0x00010001u;
		for (int idx = t; idx < rows * npairs; idx += NT) {
			const int k = fast_div(idx, npairs);
			const int j = idx - k * npairs;
			const unsigned *src = rv + k * NC + (2 * j) * P.HS;
			unsigned rbA = hamend2, gaA = hamend2, rbB = hamend2, gaB = hamend2;
			if (P.HS == 4) {
				const uint4 A = *(const uint4 *) src;
				const uint4 B = *(const uint4 *) (src + 4);
				rbA += (A.x & 0x00ff00ffu) + (A.y & 0x00ff00ffu) + (A.z & 0x00ff00ffu) + (A.w & 0x00ff00ffu);
				gaA += __byte_perm(A.x, 0, 0x4341) + __byte_perm(A.y, 0, 0x4341) + __byte_perm(A.z, 0, 0x4341) +
					__byte_perm(A.w, 0, 0x4341);
				rbB += (B.x & 0x00ff00ffu) + (B.y & 0x00ff00ffu) + (B.z & 0x00ff00ffu) + (B.w & 0x00ff00ffu);
				gaB += __byte_perm(B.x, 0, 0x4341) + __byte_perm(B.y, 0, 0x4341) + __byte_perm(B.z, 0, 0x4341) +
					__byte_perm(B.w, 0, 0x4341);
			}
			else
				for (int i = 0; i < P.HS; i++) {
					const unsigned wA = src[i];
					const unsigned wB = src[P.HS + i];
					rbA += wA & 0x00ff00ffu;
					gaA += __byte_perm(wA, 0, 0x4341);
					rbB += wB & 0x00ff00ffu;
					gaB += __byte_perm(wB, 0, 0x4341);
				}
			uint2 w;
			w.x = average_pair(rbA, rbB, P.hmul8, P.hshift);
			w.y = average_pair(gaA, gaB, P.hmul8, P.hshift);
			sh[k * (P.NEmax / 2) + j] = w;
		}

		consumer_barrier(NT);

		/* stage H2: reduceh + unpremultiply + store */
		const int bw = xb - xa;
		for (int idx = t; idx < rows * bw; idx += NT) {
			const int k = fast_div(idx, bw);
			const int x = xa + (idx - k * bw);
			const int2 hc = __ldg(&P.hcol[x]);
			const uint2 *win = sh + k * (P.NEmax / 2) + (hc.x - pair_h0);
			const int *cfp = hcoef + hc.y * NPh;
			int r = VB200_INTERPOLATE_SCALE >> 1, g = r, b = r, a = r;
			if (NP > 0) {
#pragma unroll
				for (int kk = 0; kk < NPR; kk++) {
					const uint2 w = win[kk];
					const unsigned c = (unsigned) cfp[kk];
					r = dp2a_lo(c, w.x, r);
					b = dp2a_hi(c, w.x, b);
					g = dp2a_lo(c, w.y, g);
					a = dp2a_hi(c, w.y, a);
				}
			}
			else
				for (int kk = 0; kk < NPh; kk++) {
					const uint2 w = win[kk];
					const unsigned c = (unsigned) cfp[kk];
					r = dp2a_lo(c, w.x, r);
					b = dp2a_hi(c, w.x, b);
					g = dp2a_lo(c, w.y, g);
					a = dp2a_hi(c, w.y, a);
				}
			r = max(0, min(r >> VB200_INTERPOLATE_SHIFT, 255));
			g = max(0, min(g >> VB200_INTERPOLATE_SHIFT, 255));
			b = max(0, min(b >> VB200_INTERPOLATE_SHIFT, 255));
			a = max(0, min(a >> VB200_INTERPOLATE_SHIFT, 255));
			if (PREMUL) {
				/* unpremultiply.c:209-222: byte store without clip */
				const int sc = uscale[a];
				r = ((r * sc + 128) >> 8) & 0xff;
				g = ((g * sc + 128) >> 8) & 0xff;
				b = ((b * sc + 128) >> 8) & 0xff;
			}
			*(unsigned *) (fout + (size_t) (ya + k) * P.out_bpl + (size_t) x * 4) =
				(unsigned) r | ((unsigned) g << 8) | ((unsigned) b << 16) | ((unsigned) a << 24);
		}
	}
}

#include "thumbnail_fused_mma.cuh"

/* The tensor-pipe kernel's instantiations, (VS, NP, HS): boxes that are powers of two freely mixed but for (8, 2), and
 * boxes 2 .. 8 that differ by at most one (what a uniform shrink gives).  The plan chooses the kernel only for a (VS, HS)
 * pair listed here, and a launch dispatches on the same list.
 */
#define VB200_V4_LIST(X) \
	X(4, 6, 4) X(4, 7, 4) X(2, 6, 2) X(2, 7, 2) X(8, 6, 8) X(8, 7, 8) \
	X(4, 0, 4) X(2, 0, 2) X(4, 0, 2) X(2, 0, 4) X(4, 0, 8) X(2, 0, 8) X(8, 0, 8) X(8, 0, 4) \
	X(3, 0, 3) X(5, 0, 5) X(6, 0, 6) X(7, 0, 7) X(2, 0, 3) X(3, 0, 2) X(3, 0, 4) X(4, 0, 3) \
	X(4, 0, 5) X(5, 0, 4) X(5, 0, 6) X(6, 0, 5) X(6, 0, 7) X(7, 0, 6) X(7, 0, 8) X(8, 0, 7)

/* The NP of the v4 instantiation that runs boxes (vs, hs) with nph horizontal coefficient pairs: nph where (vs, nph, hs)
 * is listed, else 0 (the generic instantiation, which reads P.NPh at run time); -1 when (vs, hs) is not listed.
 */
int
v4_np(int vs, int nph, int hs)
{
	int np = -1;
#define X(VS_, NP_, HS_) \
	if (vs == VS_ && hs == HS_ && (NP_ == nph || (NP_ == 0 && np < 0))) \
		np = NP_;
	VB200_V4_LIST(X)
#undef X
	return np;
}

/* Pack a 65 x n table of short coefficients into parity-aligned s16x2 pairs:
 * set (phase, parity) holds pairs k = 0..NP-1 = (c[2k - parity], c[2k + 1 - parity]).
 */
struct PairSets {
	int NP = 0;
	std::vector<int> coef;			   /* [nsets][NP] */
	std::map<std::pair<int, int>, int> ids; /* (phase, parity) -> set */

	int
	get(const AxisTable &t, int phase, int parity)
	{
		auto key = std::make_pair(phase, parity);
		auto it = ids.find(key);
		if (it != ids.end())
			return it->second;
		const int id = (int) ids.size();
		ids[key] = id;
		const short *c = &t.ms[(size_t) phase * t.n_point];
		for (int k = 0; k < NP; k++) {
			const int i0 = 2 * k - parity, i1 = 2 * k + 1 - parity;
			const int c0 = (i0 >= 0 && i0 < t.n_point) ? c[i0] : 0;
			const int c1 = (i1 >= 0 && i1 < t.n_point) ? c[i1] : 0;
			coef.push_back((int) (((unsigned) (c0 & 0xffff)) | ((unsigned) (c1 & 0xffff) << 16)));
		}
		return id;
	}

	/* Drop trailing pairs that are zero in EVERY set in use (e.g. Lanczos3 at
	 * shrink 2, phase 0: the 13th tap is 0, so 6 pairs carry the 12 live taps).
	 * Zero taps contribute nothing to the integer sum, so results are unchanged.
	 */
	void
	trim()
	{
		const int nsets = (int) ids.size();
		int keep = 1;
		for (int s = 0; s < nsets; s++)
			for (int k = 0; k < NP; k++)
				if (coef[(size_t) s * NP + k] != 0)
					keep = std::max(keep, k + 1);
		if (keep == NP)
			return;
		std::vector<int> packed;
		for (int s = 0; s < nsets; s++)
			for (int k = 0; k < keep; k++)
				packed.push_back(coef[(size_t) s * NP + k]);
		coef.swap(packed);
		NP = keep;
	}
};

} // namespace

/* ------------------------------------------------------------------ plan */

/* thumbnail_linear.cu */
struct LinearThumb;
int linear_thumb_new(const char *domain, int W, int H, int bands, bool premul, const ReduceGeom &gv, const ReduceGeom &gh,
	const AxisTable &tv, const AxisTable &th, LinearThumb **out);
int linear_thumb_run(const char *domain, LinearThumb *lt, const void *in, size_t in_stride, void *out, size_t out_stride, int n,
	cudaStream_t s, const IccBatch *icc = nullptr, int out_bands = 0);
void linear_thumb_free(LinearThumb *lt);

/* The fused kernel a plan runs, chosen once by plan_build_fused */
enum class FusedKernel {
	Ldg, /* v1: thumbnail_fused_kernel */
	Tma, /* v2: thumbnail_fused_tma_kernel */
	Mma, /* v4: thumbnail_fused_mma_kernel */
};

struct ThumbnailPlanImpl {
	/* request */
	int W = 0, H = 0, bands = 0, fmt = 0, has_alpha = 0;
	int target_w = 0, target_h = 0, size = 0, linear = 0;
	/* a page strip: H / page_h pages of page_h rows stacked vertically; 0 = one page */
	int page_h = 0;
	/* derived */
	double hshrink = 1, vshrink = 1;
	int OW = 0, OH = 0;
	int out_page_h = 0; /* vips_image_get_page_height of the result: OH for one page */
	ReduceGeom gv{}, gh{};
	bool premul = false;
	bool fused = false;
	int device = -1;
	/* fused path: v1's parameters, which every fused plan can run */
	FusedKernel kernel = FusedKernel::Ldg;
	FusedParams fp{};
	void *tables = nullptr; /* one device block */
	size_t smem = 0;
	/* v2 (TMA-fed) variant of the same kernel: its own chunking and smem */
	int slots_tma = 0;
	size_t smem_tma = 0;
	/* v4: reducev on the integer tensor pipe */
	int mma_tw = 0, mma_nt = 0, mma_nemax = 0;
	std::vector<MmaBand> mma_bands; /* the bands of mma_tw over a frame row */
	size_t smem_mma = 0;
	/* plan the geometry only: no device tables (vb200_debug_thumbnail_bands) */
	bool geometry_only = false;
	void *tables_mma = nullptr;
	/* host pump */
	static constexpr int kStreams = 3;
	cudaStream_t streams[kStreams] = {nullptr, nullptr, nullptr};
	void *stage_in[kStreams] = {nullptr, nullptr, nullptr};
	void *stage_out[kStreams] = {nullptr, nullptr, nullptr};
	cudaEvent_t drained[kStreams] = {nullptr, nullptr, nullptr};
	int stage_frames = 0;
	std::mutex pump_lock;
	/* the opaque-stage vote of the tensor-pipe kernel (thumbnail_fused_mma.cuh): per-launch counts of hinted frames
	 * come back through pinned memory, a few launches late; opaque_mode picks the instantiation of the NEXT launch
	 */
	static constexpr int kHintSlots = 4;
	std::mutex hint_lock;
	int *hint_counts = nullptr; /* pinned [kHintSlots] */
	cudaEvent_t hint_done[kHintSlots] = {nullptr, nullptr, nullptr, nullptr};
	bool hint_pending[kHintSlots] = {false, false, false, false};
	unsigned hint_slot_seq[kHintSlots] = {0, 0, 0, 0};
	unsigned hint_seq = 0, hint_seen = 0;
	bool opaque_mode = false;
	/* 3-band frames (what a JPEG decodes to) on the fused RGBA kernels: expanded to RGBX on the device */
	bool rgb_expand = false;
	/* linear = TRUE: the two-kernel linear-light path (thumbnail_linear.cu), or null = the leaf chain */
	LinearThumb *lin = nullptr;
	/* vips_sharpen appended to every batch (vb200_thumbnail_plan_set_sharpen) */
	bool sharpen = false;
	double sh_sigma = 0.5, sh_x1 = 2.0, sh_y2 = 10.0, sh_y3 = 20.0, sh_m1 = 0.0, sh_m2 = 3.0;
	/* colour management (vb200_thumbnail_plan_set_icc / _set_linear_icc), null = off: in the stage's linear mode when the plan
	 * is linear (import / export inside the linear thumbnail), else between the thumbnail and the sharpen stage
	 */
	IccStage *icc = nullptr;
	int icc_bands = 0;			 /* output bands with the stage on */
	size_t stage_out_frame = 0; /* the host pump's output slots are sized for frames of this many bytes */
	int out_bands() const { return icc ? icc_bands : bands; }
};

/* sharpen_fused.cu */
int dev_sharpen_fused(const char *domain, const void *in, size_t in_bpl, size_t in_frame_stride, void *out, size_t out_bpl,
	size_t out_frame_stride, int n_frames, int w, int h, int bands, double sigma, double x1, double y2, double y3, double m1,
	double m2, cudaStream_t s);

namespace {

/* vips_thumbnail_calculate_shrink, thumbnail.c:413-466 (no crop, no rotate) */
void
thumbnail_shrink(int w, int h, int tw, int th, int size, double *hshrink, double *vshrink)
{
	double hs = (double) w / tw;
	double vs = (double) h / th;
	const bool horizontal = !(hs < vs);
	if (size != VB200_SIZE_FORCE) {
		if (horizontal)
			vs = hs;
		else
			hs = vs;
	}
	if (size == VB200_SIZE_UP) {
		hs = std::min(1.0, hs);
		vs = std::min(1.0, vs);
	}
	else if (size == VB200_SIZE_DOWN) {
		hs = std::max(1.0, hs);
		vs = std::max(1.0, vs);
	}
	*hshrink = std::min(hs, (double) w);
	*vshrink = std::min(vs, (double) h);
}

/* The error check and launch count after a fused kernel's launch */
int
launch_status(const char *domain, const char *what)
{
	const cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
		return cuda_fail(domain, e, what);
	count_launch();
	return 0;
}

/* Rows per CTA: the whole height in chunks of k rows, halved (on whole chunks, down to min_chunks of them) while the
 * batch gives fewer than `ctas` CTAs
 */
int
rows_per_cta(int OH, int k, int min_chunks, int bands_x, int n, int ctas)
{
	int rpc = ((OH + k - 1) / k) * k;
	while ((long long) bands_x * ((OH + rpc - 1) / rpc) * n < ctas && rpc > min_chunks * k)
		rpc = ((rpc / 2 + k - 1) / k) * k;
	return rpc;
}

/* v1: frames f0 .. f0 + grid.z - 1 */
template <int VS, bool PREMUL>
int
launch_ldg_t(const char *domain, const FusedParams &fp, size_t smem, const void *in, size_t in_stride, void *out,
	size_t out_stride, int f0, dim3 grid, cudaStream_t s)
{
	auto kern = thumbnail_fused_kernel<VS, PREMUL>;
	VB200_CUDA(domain, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
	kern<<<grid, fp.NT, smem, s>>>(fp, (const uint8_t *) in, in_stride, (uint8_t *) out, out_stride, f0);
	return launch_status(domain, "thumbnail_fused_kernel launch");
}

template <bool PREMUL>
int
launch_ldg_vs(const char *domain, const FusedParams &fp, size_t smem, const void *in, size_t is, void *out, size_t os, int f0,
	dim3 grid, cudaStream_t s)
{
	switch (fp.VS) {
	case 1: return launch_ldg_t<1, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	case 2: return launch_ldg_t<2, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	case 3: return launch_ldg_t<3, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	case 4: return launch_ldg_t<4, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	case 5: return launch_ldg_t<5, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	case 6: return launch_ldg_t<6, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	case 8: return launch_ldg_t<8, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	default: return launch_ldg_t<0, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	}
}

/* v1 over frames f0 .. f0 + nf - 1 of an n-frame batch: enough CTAs to fill the machine, rows split when the batch is small */
int
launch_ldg(const char *domain, const ThumbnailPlanImpl *pl, const void *in, size_t is, void *out, size_t os, int n, int f0,
	int nf, cudaStream_t s)
{
	FusedParams fp = pl->fp;
	const int bands_x = (pl->OW + fp.TW - 1) / fp.TW;
	fp.RPC = rows_per_cta(pl->OH, kChunkRows, 2, bands_x, n, 2 * sm_count());
	const dim3 grid(bands_x, (pl->OH + fp.RPC - 1) / fp.RPC, nf);
	return pl->premul ? launch_ldg_vs<true>(domain, fp, pl->smem, in, is, out, os, f0, grid, s)
					  : launch_ldg_vs<false>(domain, fp, pl->smem, in, is, out, os, f0, grid, s);
}

/* v2: the v1 grid, one extra (producer) warp per CTA */
template <int VS, int NP, bool PREMUL>
int
launch_tma_t(const char *domain, const FusedParams &fp, size_t smem, const void *in, size_t in_stride, void *out,
	size_t out_stride, int f0, dim3 grid, cudaStream_t s)
{
	auto kern = thumbnail_fused_tma_kernel<VS, NP, PREMUL, kColsPerThread>;
	VB200_CUDA(domain, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
	kern<<<grid, fp.NT + 32, smem, s>>>(fp, (const uint8_t *) in, in_stride, (uint8_t *) out, out_stride, f0);
	return launch_status(domain, "thumbnail_fused_tma_kernel launch");
}

template <int NP, bool PREMUL>
int
launch_tma_vs(const char *domain, const FusedParams &fp, size_t smem, const void *in, size_t is, void *out, size_t os, int f0,
	dim3 grid, cudaStream_t s)
{
	switch (fp.VS) {
	case 1: return launch_tma_t<1, NP, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	case 2: return launch_tma_t<2, NP, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	case 3: return launch_tma_t<3, NP, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	case 4: return launch_tma_t<4, NP, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	case 8: return launch_tma_t<8, NP, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	default: return launch_tma_t<0, NP, PREMUL>(domain, fp, smem, in, is, out, os, f0, grid, s);
	}
}

int
launch_tma(const char *domain, const ThumbnailPlanImpl *pl, const void *in, size_t is, void *out, size_t os, int n, int f0,
	int nf, cudaStream_t s)
{
	FusedParams fp = pl->fp;
	fp.slots = pl->slots_tma;
	/* consumer threads: kColsPerThread columns each (pl->fp.NT counts columns, rounded to 32) */
	fp.NT = ((pl->fp.NT / kColsPerThread + 31) / 32) * 32;
	const int bands_x = (pl->OW + fp.TW - 1) / fp.TW;
	fp.RPC = rows_per_cta(pl->OH, kChunkRowsTma, 4, bands_x, n, 2 * sm_count());
	const dim3 grid(bands_x, (pl->OH + fp.RPC - 1) / fp.RPC, nf);
	const size_t smem = pl->smem_tma;
	const int np = fp.NPv == fp.NPh ? fp.NPv : 0;
	if (np == 6)
		return pl->premul ? launch_tma_vs<6, true>(domain, fp, smem, in, is, out, os, f0, grid, s)
						  : launch_tma_vs<6, false>(domain, fp, smem, in, is, out, os, f0, grid, s);
	if (np == 7)
		return pl->premul ? launch_tma_vs<7, true>(domain, fp, smem, in, is, out, os, f0, grid, s)
						  : launch_tma_vs<7, false>(domain, fp, smem, in, is, out, os, f0, grid, s);
	return pl->premul ? launch_tma_vs<0, true>(domain, fp, smem, in, is, out, os, f0, grid, s)
					  : launch_tma_vs<0, false>(domain, fp, smem, in, is, out, os, f0, grid, s);
}

/* A tiled tensor map over the batch: u64 elements (2 pixels), dims {W / 2, H, frames}, box
 * {v4_boxw(HS) / 2, rows, 1}: one cp.async.bulk.tensor per TMA stage.  Returns false when
 * the driver entry point or the geometry is not usable; the kernel then copies row by row.
 */
bool
make_stage_tensor_map(CUtensorMap *tm, const void *in, int W, int H, size_t in_bpl, size_t frame_stride, int frames,
	int box_cols, int box_rows)
{
	typedef CUresult (*encode_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
		const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
		CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
	static encode_fn encode = nullptr;
	static bool tried = false;
	if (!tried) {
		tried = true;
		void *fn = nullptr;
		cudaDriverEntryPointQueryResult qres;
		if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess &&
			qres == cudaDriverEntryPointSuccess)
			encode = (encode_fn) fn;
		cudaGetLastError();
	}
	if (!encode || getenv("VB200_NO_TENSORMAP"))
		return false;
	if ((W & 1) || (in_bpl % 16) || (frame_stride % 16) || ((uintptr_t) in % 16) || box_cols / 2 > 256 || box_rows > 256)
		return false;
	const cuuint64_t dims[3] = {(cuuint64_t) W / 2, (cuuint64_t) H, (cuuint64_t) frames};
	const cuuint64_t strides[2] = {(cuuint64_t) in_bpl, (cuuint64_t) frame_stride};
	const cuuint32_t box[3] = {(cuuint32_t) box_cols / 2, (cuuint32_t) box_rows, 1};
	const cuuint32_t estr[3] = {1, 1, 1};
	return encode(tm, CU_TENSOR_MAP_DATA_TYPE_UINT64, 3, const_cast<void *>(in), dims, strides, box, estr,
			   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
			   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

/* Arms the tensor-pipe kernel's opaque-stage vote per frame: 128 threads sample 2 pixels each, spread over the
 * frame by a multiplicative hash; the hint is set where at least a quarter of the samples have alpha 255, and
 * *count receives the number of hinted frames.  A hint, not a promise: the V warps still vote on every stage they
 * skip the premultiply for.
 */
constexpr int kHintThreads = 128, kHintSamples = 2;

__global__ void __launch_bounds__(kHintThreads)
alpha_hint_kernel(const uint8_t *__restrict__ in, size_t in_frame_stride, size_t in_bpl, int W, int H, unsigned char *__restrict__ hint,
	int *__restrict__ count)
{
	const uint8_t *f = in + (size_t) blockIdx.x * in_frame_stride;
	const unsigned npix = (unsigned) W * (unsigned) H;
	int opaque = 0;
#pragma unroll
	for (int i = 0; i < kHintSamples; i++) {
		const unsigned k = (unsigned) (threadIdx.x * kHintSamples + i);
		const unsigned p = (unsigned) (((unsigned long long) (k * 2654435761u) * npix) >> 32); /* 0 .. npix - 1 */
		const unsigned y = p / (unsigned) W, x = p - y * (unsigned) W;
		opaque += f[(size_t) y * in_bpl + (size_t) x * 4 + 3] == 255;
	}
	__shared__ int s_sum;
	if (threadIdx.x == 0)
		s_sum = 0;
	__syncthreads();
	opaque = __reduce_add_sync(0xffffffffu, opaque);
	if ((threadIdx.x & 31) == 0)
		atomicAdd(&s_sum, opaque);
	__syncthreads();
	if (threadIdx.x == 0) {
		const int h = s_sum * 4 >= kHintThreads * kHintSamples ? 1 : 0;
		hint[blockIdx.x] = (unsigned char) h;
		if (h)
			atomicAdd(count, 1);
	}
}

/* Before a launch: harvest the counts of earlier launches that have completed (never waits), decide the
 * instantiation, and run the hint kernel for this launch's frames.  *hint = nullptr when the vote is off.
 */
int
opaque_hint_begin(const char *domain, ThumbnailPlanImpl *pl, const FusedParams &fp, const void *in, size_t in_stride, int n,
	cudaStream_t s, void **hint, bool *use_opq)
{
	*hint = nullptr;
	*use_opq = false;
	const char *probe_env = getenv("VB200_OPAQUE_PROBE"); /* 0: never (A/B timing); 2: always use the voting instantiation */
	if (!pl->premul || (probe_env && probe_env[0] == '0'))
		return 0;
	{
		std::lock_guard<std::mutex> lock(pl->hint_lock);
		if (!pl->hint_counts) {
			if (cudaHostAlloc((void **) &pl->hint_counts, sizeof(int) * ThumbnailPlanImpl::kHintSlots, cudaHostAllocDefault) != cudaSuccess) {
				cudaGetLastError();
				pl->hint_counts = nullptr;
				return 0; /* no vote, same pixels */
			}
			for (int i = 0; i < ThumbnailPlanImpl::kHintSlots; i++)
				cudaEventCreateWithFlags(&pl->hint_done[i], cudaEventDisableTiming);
		}
		for (int i = 0; i < ThumbnailPlanImpl::kHintSlots; i++)
			if (pl->hint_pending[i] && cudaEventQuery(pl->hint_done[i]) == cudaSuccess) {
				pl->hint_pending[i] = false;
				if (pl->hint_slot_seq[i] + 1 > pl->hint_seen) {
					pl->hint_seen = pl->hint_slot_seq[i] + 1;
					pl->opaque_mode = pl->hint_counts[i] > 0;
				}
			}
		cudaGetLastError(); /* cudaErrorNotReady from the queries */
		*use_opq = pl->opaque_mode || (probe_env && probe_env[0] == '2');
	}
	const size_t count_off = ((size_t) n + 3) & ~(size_t) 3;
	if (dev_alloc(domain, hint, count_off + sizeof(int), s))
		return -1;
	int *count = (int *) ((char *) *hint + count_off);
	VB200_CUDA(domain, cudaMemsetAsync(count, 0, sizeof(int), s));
	alpha_hint_kernel<<<n, kHintThreads, 0, s>>>((const uint8_t *) in, in_stride, fp.in_bpl, fp.W, fp.H, (unsigned char *) *hint, count);
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) {
		dev_free(*hint, s);
		*hint = nullptr;
		return cuda_fail(domain, e, "alpha_hint_kernel launch");
	}
	count_launch();
	return 0;
}

/* After the launch: send this launch's count home and release the hint buffer (stream-ordered). */
void
opaque_hint_end(ThumbnailPlanImpl *pl, void *hint, int n, cudaStream_t s)
{
	if (!hint)
		return;
	{
		std::lock_guard<std::mutex> lock(pl->hint_lock);
		const int slot = (int) (pl->hint_seq % ThumbnailPlanImpl::kHintSlots);
		if (!pl->hint_pending[slot]) {
			const int *count = (const int *) ((const char *) hint + (((size_t) n + 3) & ~(size_t) 3));
			if (cudaMemcpyAsync(&pl->hint_counts[slot], count, sizeof(int), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
				cudaEventRecord(pl->hint_done[slot], s) == cudaSuccess) {
				pl->hint_pending[slot] = true;
				pl->hint_slot_seq[slot] = pl->hint_seq;
			}
			cudaGetLastError();
		}
		pl->hint_seq++;
	}
	dev_free(hint, s);
}

template <int VS, int NP, bool PREMUL, int HSQ, bool OPQ>
int
launch_mma_k(const char *domain, const ThumbnailPlanImpl *pl, const FusedParams &fp, const CUtensorMap &tm, int use_tmap, const void *in,
	size_t in_stride, void *out, size_t out_stride, int f0, dim3 grid, cudaStream_t s)
{
	auto kern = thumbnail_fused_mma_kernel<VS, NP, PREMUL, HSQ, OPQ>;
	VB200_CUDA(domain, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) pl->smem_mma));
	kern<<<grid, fp.NT + 32 * kV4HWarps + 32, pl->smem_mma, s>>>(fp, tm, use_tmap, (const uint8_t *) in, in_stride,
		(uint8_t *) out, out_stride, f0);
	return launch_status(domain, "thumbnail_fused_mma_kernel launch");
}

/* v4 over frames f0 .. f0 + grid.z - 1 of an n-frame batch (the stage tensor map spans the batch) */
template <int VS, int NP, bool PREMUL, int HSQ>
int
launch_mma_t(const char *domain, ThumbnailPlanImpl *pl, FusedParams fp, const void *in, size_t in_stride, void *out,
	size_t out_stride, int n, int f0, dim3 grid, cudaStream_t s)
{
	CUtensorMap tm;
	memset(&tm, 0, sizeof(tm));
	const int use_tmap = make_stage_tensor_map(&tm, in, fp.W, fp.H, fp.in_bpl, in_stride, n, v4_boxw(HSQ), 2 * VS) ? 1 : 0;
	void *hint = nullptr;
	bool use_opq = false;
	if (PREMUL && opaque_hint_begin(domain, pl, fp, (const uint8_t *) in + (size_t) f0 * in_stride, in_stride, (int) grid.z, s, &hint, &use_opq))
		return -1;
	fp.opaque_hint = (const unsigned char *) hint;
	int rc;
	if constexpr (PREMUL)
		rc = use_opq ? launch_mma_k<VS, NP, PREMUL, HSQ, true>(domain, pl, fp, tm, use_tmap, in, in_stride, out, out_stride, f0, grid, s)
					 : launch_mma_k<VS, NP, PREMUL, HSQ, false>(domain, pl, fp, tm, use_tmap, in, in_stride, out, out_stride, f0, grid, s);
	else
		rc = launch_mma_k<VS, NP, PREMUL, HSQ, false>(domain, pl, fp, tm, use_tmap, in, in_stride, out, out_stride, f0, grid, s);
	opaque_hint_end(pl, hint, (int) grid.z, s);
	return rc;
}

template <bool PREMUL>
int
launch_mma_list(const char *domain, ThumbnailPlanImpl *pl, const FusedParams &fp, const void *in, size_t is, void *out, size_t os,
	int n, int f0, dim3 grid, cudaStream_t s)
{
	const int np = v4_np(fp.VS, fp.NPh, fp.HS);
#define X(VS_, NP_, HS_) \
	if (fp.VS == VS_ && np == NP_ && fp.HS == HS_) \
		return launch_mma_t<VS_, NP_, PREMUL, HS_>(domain, pl, fp, in, is, out, os, n, f0, grid, s);
	VB200_V4_LIST(X)
#undef X
	error(domain, "the tensor-pipe kernel has no instantiation for VS %d, HS %d", fp.VS, fp.HS);
	return -1;
}

int
launch_mma(const char *domain, ThumbnailPlanImpl *pl, const void *in, size_t is, void *out, size_t os, int n, int f0, int nf,
	cudaStream_t s)
{
	FusedParams fp = pl->fp;
	fp.TW = pl->mma_tw;
	fp.NT = pl->mma_nt;
	fp.NEmax = pl->mma_nemax;
	const int bands_x = (pl->OW + fp.TW - 1) / fp.TW;
	fp.RPC = rows_per_cta(pl->OH, fp.mma_rows, 4, bands_x, n, sm_count());
	const dim3 grid(bands_x, (pl->OH + fp.RPC - 1) / fp.RPC, nf);
	return pl->premul ? launch_mma_list<true>(domain, pl, fp, in, is, out, os, n, f0, grid, s)
					  : launch_mma_list<false>(domain, pl, fp, in, is, out, os, n, f0, grid, s);
}

/* The per-row / per-column sampling tables of the plan's vips_resize, stepped per rect exactly as the
 * reference's sink would call reducev / reduceh (demand hints: shrinkv forces SMALLTILE, shrinkh chunks
 * into fatstrip-height strips; see dev_reduce_chain).
 */
void
plan_axis_tables(const ThumbnailPlanImpl *pl, AxisTable &tv, AxisTable &th)
{
	const TileGeometry tg = tile_geometry();
	int tile_w, tile_h;
	if (pl->gv.int_shrink > 1) {
		tile_w = tg.tile_width;
		tile_h = tg.tile_height;
	}
	else {
		tile_w = pl->OW;
		tile_h = tg.fatstrip_height;
	}
	int rect_h = tile_h;
	if (pl->gh.int_shrink > 1)
		rect_h = std::min(rect_h, tg.fatstrip_height);
	build_axis_table(tv, pl->OH, pl->gv.residual, pl->gv.offset, pl->gv.n_point, VB200_KERNEL_LANCZOS3, rect_h);
	build_axis_table(th, pl->OW, pl->gh.residual, pl->gh.offset, pl->gh.n_point, VB200_KERNEL_LANCZOS3, tile_w);
}

/* The bands of a fused kernel at band width tw (the last one shorter), with the input columns each loads: c_lo rounded
 * down to clo_align pixels (v2: 4; v4: v4_clo_align)
 */
std::vector<MmaBand>
mma_bands_of(const FusedParams &fp, const std::vector<int2> &hcol, int tw, int clo_align)
{
	auto column_of = [&](int E0, int tt) {
		const int e = E0 + tt / fp.HS;
		const int k = tt % fp.HS;
		const int sc = std::max(0, std::min(e - fp.hembed, fp.Ws - 1));
		return std::min(sc * fp.HS + k, fp.W - 1);
	};
	std::vector<MmaBand> bands;
	for (int xa = 0; xa < fp.OW; xa += tw) {
		MmaBand b;
		b.xa = xa;
		b.xb = std::min(xa + tw, fp.OW);
		const int E0 = 2 * hcol[xa].x + fp.hgrid;
		b.ne = 2 * (hcol[b.xb - 1].x + fp.NPh - hcol[xa].x);
		b.c_lo = column_of(E0, 0) & ~(clo_align - 1);
		b.c_hi = std::min(fp.W, (column_of(E0, b.ne * fp.HS - 1) + 4) & ~3);
		bands.push_back(b);
	}
	return bands;
}

int
plan_build_fused(const char *domain, ThumbnailPlanImpl *pl)
{
	AxisTable tv, th;
	plan_axis_tables(pl, tv, th);

	/* Pair grid: pair p covers embedded positions (2p + grid, 2p + grid + 1).  Pick
	 * the grid phase (0 / 1) that needs fewer coefficient pairs once all-zero
	 * trailing pairs are trimmed: at shrink 2 the first tap sits on an odd
	 * position, so grid 1 packs the 12 live Lanczos3 taps into 6 pairs, not 7.
	 */
	auto build_sets = [](const AxisTable &t, int count, int grid, PairSets &sets, std::vector<int2> &idx) {
		sets = PairSets();
		sets.NP = (t.n_point + 2) / 2;
		idx.resize(count);
		for (int i = 0; i < count; i++) {
			const int rel = t.first[i] - grid;
			idx[i].x = rel >> 1; /* floor */
			idx[i].y = sets.get(t, t.phase[i], rel & 1);
		}
		sets.trim();
	};
	PairSets sv, shh;
	std::vector<int2> vrow, hcol;
	int vgrid = 0, hgrid = 0;
	{
		PairSets alt;
		std::vector<int2> alt_idx;
		build_sets(tv, pl->OH, 0, sv, vrow);
		build_sets(tv, pl->OH, 1, alt, alt_idx);
		if (alt.NP < sv.NP) {
			sv = alt;
			vrow = alt_idx;
			vgrid = 1;
		}
		build_sets(th, pl->OW, 0, shh, hcol);
		build_sets(th, pl->OW, 1, alt, alt_idx);
		if (alt.NP < shh.NP) {
			shh = alt;
			hcol = alt_idx;
			hgrid = 1;
		}
	}

	FusedParams &fp = pl->fp;
	fp.W = pl->W;
	fp.H = pl->H;
	fp.in_bpl = (size_t) pl->W * 4;
	fp.VS = pl->gv.int_shrink;
	fp.Hs = pl->gv.shrunk_size;
	fp.vembed = tv.embed;
	fp.NPv = sv.NP;
	fp.vgrid = vgrid;
	fp.hgrid = hgrid;
	fp.vmul8 = (unsigned) (((1LL << 32) / (256LL * fp.VS)) << 8);
	fp.vshift = -1;
	fp.accmul = 1;
	for (int sft = 0; sft < 9; sft++)
		if ((1 << sft) == fp.VS) {
			fp.vshift = sft;
			fp.accmul = 256u >> sft;
		}
	fp.HS = pl->gh.int_shrink;
	fp.Ws = pl->gh.shrunk_size;
	fp.hembed = th.embed;
	fp.NPh = shh.NP;
	fp.hmul8 = (unsigned) (((1LL << 32) / (256LL * fp.HS)) << 8);
	fp.hshift = -1;
	for (int sft = 0; sft < 9; sft++)
		if ((1 << sft) == fp.HS)
			fp.hshift = sft;
	fp.OW = pl->OW;
	fp.OH = pl->OH;
	fp.out_bpl = (size_t) pl->OW * 4;
	fp.premul = pl->premul;
	fp.max_alpha = 255.0;
	fp.opaque_hint = nullptr; /* set per launch (launch_mma_t) */
	fp.nvsets = (int) sv.ids.size();
	fp.nhsets = (int) shh.ids.size();
	if (fp.VS > 256 || fp.HS > 256)
		return 1; /* 16-bit lanes would overflow: use the unfused path */

	/* band width: as wide as the thread budget allows */
	int TW = 64;
	auto band_threads = [&](int tw, int *nemax) {
		int worst = 0;
		for (int xa = 0; xa < pl->OW; xa += tw) {
			const int xb = std::min(xa + tw, pl->OW);
			const int ne = 2 * (hcol[xb - 1].x + fp.NPh) - 2 * hcol[xa].x;
			worst = std::max(worst, ne);
		}
		*nemax = worst;
		return worst * fp.HS;
	};
	int nemax = 0;
	while (TW > 4 && band_threads(TW, &nemax) > kMaxThreads)
		TW /= 2;
	if (band_threads(TW, &nemax) > kMaxThreads)
		return 1;
	fp.TW = TW;
	fp.NEmax = nemax;
	fp.NT = std::min(kMaxThreads, ((nemax * fp.HS + 31) / 32) * 32);
	fp.NT = std::max(fp.NT, 64);

	/* pair slots: worst chunk */
	int slots = 0;
	for (int ya = 0; ya < pl->OH; ya += kChunkRows) {
		const int yb = std::min(ya + kChunkRows, pl->OH);
		slots = std::max(slots, vrow[yb - 1].x + fp.NPv - 1 - vrow[ya].x + 1);
	}
	fp.slots = slots;

	pl->smem = (size_t) slots * fp.NT * 8 + (size_t) kChunkRows * fp.NT * 4 + (size_t) kChunkRows * (nemax / 2) * 8 +
		(size_t) (fp.nvsets * fp.NPv + fp.nhsets * fp.NPh + 512) * 4;
	if (pl->smem > 200 * 1024)
		return 1;

	/* The kernel: v4 where its tables, bands and shared memory fit and its (VS, HS) is instantiated, else v2 where the
	 * rows are 16-byte aligned (cp.async.bulk) and the band fits a stage, else v1.
	 */
	pl->kernel = FusedKernel::Ldg;
	if ((fp.in_bpl % 16) == 0 && fp.VS <= 16) {
		int slots2 = 0;
		for (int ya = 0; ya < pl->OH; ya += kChunkRowsTma) {
			const int yb = std::min(ya + kChunkRowsTma, pl->OH);
			slots2 = std::max(slots2, vrow[yb - 1].x + fp.NPv - 1 - vrow[ya].x + 1);
		}
		/* widest band, in input columns rounded out to 4-pixel (16-byte) bounds */
		int max_cols = 0;
		for (const MmaBand &b : mma_bands_of(fp, hcol, TW, 4))
			max_cols = std::max(max_cols, b.c_hi - b.c_lo);
		fp.stage_pitch = kStagePitch;
		pl->slots_tma = slots2;
		const int nc = ((fp.NT / kColsPerThread + 31) / 32) * 32 * kColsPerThread; /* buffer columns of the v2 kernel */
		pl->smem_tma = (size_t) kStages * 2 * fp.VS * kStagePitch + 2 * kStages * 8 + (size_t) slots2 * nc * 8 +
			(size_t) kChunkRowsTma * nc * 4 + (size_t) kChunkRowsTma * (nemax / 2) * 8 +
			(size_t) (fp.nvsets * fp.NPv + fp.nhsets * fp.NPh + 256) * 4;
		if (max_cols * 4 <= kStagePitch && pl->smem_tma <= 113 * 1024 && fp.max_alpha == 255.0)
			pl->kernel = FusedKernel::Tma;
	}

	/* v4: reducev as u8 x s8 MMAs over a ring of 8 quads (32 box-shrunk rows) per 8 output rows.  Not gated on v2: v2's
	 * shared-memory bound fails for box 8, this kernel's does not.
	 */
	const bool hpow2 = fp.HS == 2 || fp.HS == 4 || fp.HS == 8;
	/* with a power-of-two horizontal box a V thread loads its two columns as one 8-byte word: not where the last box
	 * runs past the frame's edge (W = 8k + 4 at box 8) and its columns replicate the odd last one
	 */
	const bool pairs_aligned = !hpow2 || fp.Ws * fp.HS <= fp.W;
	if ((fp.in_bpl % 16) == 0 && fp.max_alpha == 255.0 && pairs_aligned && v4_np(fp.VS, fp.NPh, fp.HS) >= 0) {
		std::vector<int> vchunk_flat;
		std::vector<unsigned> bfrag_flat;
		const int K = pick_mma_rows(tv, pl->OH, vchunk_flat, bfrag_flat); /* 0: no chunking fits the ring */
		bool ok = K > 0;
		fp.mma_rows = K;
		const int chunks = ok ? (pl->OH + K - 1) / K : 0;
		std::vector<int2> vchunk(chunks);
		std::vector<uint4> bfrag((size_t) chunks * 32);
		if (ok) {
			memcpy(vchunk.data(), vchunk_flat.data(), vchunk.size() * sizeof(int2));
			memcpy(bfrag.data(), bfrag_flat.data(), bfrag.size() * sizeof(uint4));
		}
		/* logical columns a V warp covers: 64, or 2 * floor(32 / HS) * HS when the horizontal box is not a
		 * power of two (V4Group in thumbnail_fused_mma.cuh)
		 */
		const int warp_cols = hpow2 ? 0 : 2 * (32 / fp.HS) * fp.HS;
		const int pitch = v4_nbox(fp.HS) * v4_boxw(fp.HS) * 4;
		/* band width: the one that needs the fewest V warps over a frame row (warps past a band's last
		 * column exit at once, so a narrow last band is cheap); ties go to the wider band
		 */
		int tw4 = 0, nemax4 = 0;
		long best_cost = LONG_MAX;
		const int cols_per_warp = warp_cols ? warp_cols : 32 * kV4Cpt;
		const int col_budget = warp_cols ? (kV4Cols / (32 * kV4Cpt)) * warp_cols : kV4Cols;
		for (int tw = std::min(pl->OW, 256); tw >= 2 && ok; tw--) {
			int worst = 0, max_cols = 0;
			long cost = 0;
			for (const MmaBand &b : mma_bands_of(fp, hcol, tw, v4_clo_align(fp.HS))) {
				worst = std::max(worst, b.ne);
				max_cols = std::max(max_cols, b.c_hi - b.c_lo);
				cost += (b.ne * fp.HS + cols_per_warp - 1) / cols_per_warp + 1; /* + the H / P warps' share */
			}
			if (worst * fp.HS <= col_budget && max_cols * 4 <= pitch && cost < best_cost) {
				best_cost = cost;
				tw4 = tw;
				nemax4 = worst;
			}
		}
		if (ok && tw4 > 0) {
			pl->mma_tw = tw4;
			pl->mma_nemax = nemax4;
			pl->mma_nt = warp_cols ? std::max(64, ((nemax4 * fp.HS + warp_cols - 1) / warp_cols) * 32)
								   : std::max(64, ((nemax4 * fp.HS / kV4Cpt + 31) / 32) * 32);
			const int stages = fp.VS <= 2 ? 2 * VB200_V4_STAGES
				: (fp.VS >= 7 ? VB200_V4_STAGES / 2 : (fp.VS >= 5 ? (3 * VB200_V4_STAGES) / 4 : VB200_V4_STAGES));
			const int logical_cols = warp_cols ? (pl->mma_nt / 32) * warp_cols : pl->mma_nt * kV4Cpt;
			pl->mma_bands = mma_bands_of(fp, hcol, tw4, v4_clo_align(fp.HS));
			const int nbox = v4_nbox(fp.HS);
			const size_t box_bytes = ((size_t) 2 * fp.VS * (pitch / nbox) + 127) & ~(size_t) 127;
			pl->smem_mma = (size_t) stages * nbox * box_bytes + (2 * stages + 4) * 8 +
				(size_t) kV4Quads * ((size_t) pl->mma_nt * kV4Cpt * 16 + 16) +
				(size_t) 2 * kV4Rows * ((logical_cols / fp.HS + 1) / 2) * 8 +
				(size_t) (fp.nhsets * fp.NPh + 256) * 4;
			const size_t n_ch = vchunk.size() * sizeof(int2), n_bf = bfrag.size() * sizeof(uint4);
			if (pl->smem_mma <= 226 * 1024) {
				if (!pl->geometry_only) {
					VB200_CUDA(domain, cudaMalloc(&pl->tables_mma, n_bf + n_ch));
					VB200_CUDA(domain, cudaMemcpy(pl->tables_mma, bfrag.data(), n_bf, cudaMemcpyHostToDevice));
					VB200_CUDA(domain, cudaMemcpy((char *) pl->tables_mma + n_bf, vchunk.data(), n_ch, cudaMemcpyHostToDevice));
					fp.vbfrag = (const uint4 *) pl->tables_mma;
					fp.vchunk = (const int2 *) ((char *) pl->tables_mma + n_bf);
				}
				pl->kernel = FusedKernel::Mma;
			}
		}
	}
	if (pl->geometry_only)
		return 0;

	/* upload tables as one block */
	const size_t n_vrow = vrow.size() * sizeof(int2), n_hcol = hcol.size() * sizeof(int2);
	const size_t n_vc = sv.coef.size() * 4, n_hc = shh.coef.size() * 4;
	std::vector<char> host(n_vrow + n_hcol + n_vc + n_hc);
	memcpy(&host[0], vrow.data(), n_vrow);
	memcpy(&host[n_vrow], hcol.data(), n_hcol);
	memcpy(&host[n_vrow + n_hcol], sv.coef.data(), n_vc);
	memcpy(&host[n_vrow + n_hcol + n_vc], shh.coef.data(), n_hc);
	VB200_CUDA(domain, cudaMalloc(&pl->tables, host.size()));
	VB200_CUDA(domain, cudaMemcpy(pl->tables, host.data(), host.size(), cudaMemcpyHostToDevice));
	char *b = (char *) pl->tables;
	fp.vrow = (const int2 *) b;
	fp.hcol = (const int2 *) (b + n_vrow);
	fp.vcoef = (const int *) (b + n_vrow + n_hcol);
	fp.hcoef = (const int *) (b + n_vrow + n_hcol + n_vc);
	return 0;
}

} // namespace

namespace {

/* packed RGB -> RGBX (X = 255) and back: four pixels (three words <-> four words) per thread */
__global__ void __launch_bounds__(256)
rgb_expand_kernel(const uint8_t *__restrict__ in, size_t in_stride, uint8_t *__restrict__ out, size_t out_stride, size_t quads)
{
	const size_t q = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
	if (q >= quads)
		return;
	const unsigned *p = (const unsigned *) (in + (size_t) blockIdx.y * in_stride) + q * 3;
	const unsigned w0 = __ldg(p), w1 = __ldg(p + 1), w2 = __ldg(p + 2);
	uint4 o;
	o.x = (w0 & 0x00ffffffu) | 0xff000000u;
	o.y = (w0 >> 24) | ((w1 & 0xffffu) << 8) | 0xff000000u;
	o.z = (w1 >> 16) | ((w2 & 0xffu) << 16) | 0xff000000u;
	o.w = (w2 >> 8) | 0xff000000u;
	((uint4 *) (out + (size_t) blockIdx.y * out_stride))[q] = o;
}

__global__ void __launch_bounds__(256)
rgbx_compact_kernel(const uint8_t *__restrict__ in, size_t in_stride, uint8_t *__restrict__ out, size_t out_stride, size_t pixels)
{
	const size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= pixels)
		return;
	const unsigned px = __ldg((const unsigned *) (in + (size_t) blockIdx.y * in_stride) + i);
	uint8_t *q = out + (size_t) blockIdx.y * out_stride + i * 3;
	q[0] = (uint8_t) px;
	q[1] = (uint8_t) (px >> 8);
	q[2] = (uint8_t) (px >> 16);
}

} // namespace

/* The largest page strip a plan takes, in input bytes: every kernel a plan can pick keeps its row and byte offsets in
 * size_t, but pixel counts (alpha_hint_kernel) and the gridDim.x of the RGB expansion in 32 bits; 2^31 - 1 bytes keeps
 * all of them far from overflow.
 */
constexpr size_t kMaxStripBytes = 0x7fffffff;

/* vips_thumbnail_build's shrink for a page strip (thumbnail.c:825-839): vips_thumbnail_calculate_shrink of one page, then
 * vshrink adjusted so that every page lands on a whole number of rows.  One page: the shrink of the whole frame.
 */
static int
plan_page_shrink(const char *domain, ThumbnailPlanImpl *pl)
{
	const int ph = pl->page_h > 0 && pl->page_h < pl->H && pl->H % pl->page_h == 0 ? pl->page_h : pl->H; /* header.c:889-901 */
	pl->page_h = ph < pl->H ? ph : 0;
	thumbnail_shrink(pl->W, ph, pl->target_w, pl->target_h, pl->size, &pl->hshrink, &pl->vshrink);
	if (!pl->page_h)
		return 0;
	if ((size_t) pl->W * pl->H * pl->bands > kMaxStripBytes) {
		error(domain, "page strips over 2^31 - 1 bytes (%d x %d x %d) are not on the device path", pl->W, pl->H, pl->bands);
		return -1;
	}
	const int n_loaded_pages = pl->H / ph; /* thumbnail.c:238-239 */
	const int target_page_height = (int) rint(ph / pl->vshrink);
	pl->vshrink = (double) pl->H / ((double) target_page_height * n_loaded_pages);
	return 0;
}

/* thumbnail.c:904-917: page-height = rint(page_height / vshrink) on a result of more than one page, read back as
 * vips_image_get_page_height does
 */
static int
plan_out_page_height(const ThumbnailPlanImpl &pl)
{
	if (!pl.page_h)
		return pl.OH;
	const int oph = (int) rint(pl.page_h / pl.vshrink);
	return oph > 0 && oph < pl.OH && pl.OH % oph == 0 ? oph : pl.OH;
}

int
thumbnail_plan_init(const char *domain, ThumbnailPlanImpl *pl)
{
	if (pl->fmt != VB200_FORMAT_UCHAR) {
		error(domain, "only uchar frames are on the batched device path");
		return -1;
	}
	if (plan_page_shrink(domain, pl))
		return -1;
	if (pl->linear && (pl->bands < 3 || pl->hshrink < 1.0 || pl->vshrink < 1.0)) {
		error(domain, pl->bands < 3 ? "linear thumbnails on the device path need an 8-bit image with 3+ bands"
									: "upsizing is not on the device path yet");
		return -1;
	}
	if (pl->hshrink < 1.0 || pl->vshrink < 1.0) {
		/* enlarging thumbnail: premultiply / vips_resize (affine) / unpremultiply, unfused */
		const double hscale = std::max(1.0 / pl->hshrink, 1.0 / pl->W);
		const double vscale = std::max(1.0 / pl->vshrink, 1.0 / pl->H);
		if (hscale < 1.0 || vscale < 1.0) {
			error(domain, "mixed up/down resize is not on the device path");
			return -1;
		}
		/* oarea of the scale-only affine, affine.c:466-481 */
		const double rw = (hscale > 1.0 ? hscale : 1.0) * pl->W, rh = (vscale > 1.0 ? vscale : 1.0) * pl->H;
		pl->OW = (int) (rw > 0 ? rw + 0.5 : rw - 0.5);
		pl->OH = (int) (rh > 0 ? rh + 0.5 : rh - 0.5);
		pl->premul = pl->has_alpha && pl->hshrink != 1.0 && pl->vshrink != 1.0;
		pl->fused = false;
		return 0;
	}
	/* vips_resize: scale = 1 / shrink, then reducev(1 / vscale) -- keep the double rounding */
	double hscale = std::max(1.0 / pl->hshrink, 1.0 / pl->W);
	double vscale = std::max(1.0 / pl->vshrink, 1.0 / pl->H);
	const double vs = vscale < 1.0 ? 1.0 / vscale : 1.0;
	const double hs = hscale < 1.0 ? 1.0 / hscale : 1.0;
	pl->gv = ReduceGeom{pl->H, pl->H, 1, pl->H, 0, 1.0, 0.0};
	pl->gh = ReduceGeom{pl->W, pl->W, 1, pl->W, 0, 1.0, 0.0};
	if (vs > 1.0 && reduce_geometry(domain, pl->H, vs, VB200_KERNEL_LANCZOS3, 2.0, &pl->gv))
		return -1;
	if (hs > 1.0 && reduce_geometry(domain, pl->W, hs, VB200_KERNEL_LANCZOS3, 2.0, &pl->gh))
		return -1;
	pl->OW = pl->gh.out_size;
	pl->OH = pl->gv.out_size;
	/* thumbnail.c:848-861 */
	pl->premul = pl->has_alpha && pl->hshrink != 1.0 && pl->vshrink != 1.0;

	pl->fused = false;
	if (pl->linear) {
		/* thumbnail.c:766-806: sRGB -> scRGB first; the float chain as two kernels where the geometry allows */
		AxisTable tv, th;
		if (pl->gv.n_point > 0 && pl->gh.n_point > 0) {
			plan_axis_tables(pl, tv, th);
			if (linear_thumb_new(domain, pl->W, pl->H, pl->bands, pl->premul, pl->gv, pl->gh, tv, th, &pl->lin) < 0)
				return -1;
		}
		pl->fused = pl->lin != nullptr;
		return 0;
	}
	/* 3-band 8-bit frames: the channels of the uchar chain never mix without a premultiply, so RGB through the RGBA
	 * kernels (X = 255, no premultiply) gives the reference's RGB bytes; needs frames whose pixel count is a
	 * multiple of four (word-wise expansion)
	 */
	pl->rgb_expand = pl->bands == 3 && ((size_t) pl->W * pl->H) % 4 == 0 && getenv("VB200_NO_RGB_EXPAND") == nullptr;
	if ((pl->bands == 4 || pl->rgb_expand) && pl->gv.n_point > 0 && pl->gh.n_point > 0) {
		int r = plan_build_fused(domain, pl);
		if (r < 0)
			return -1;
		pl->fused = r == 0;
	}
	if (!pl->fused)
		pl->rgb_expand = false;
	return 0;
}

static int thumbnail_plan_run_fused(const char *domain, ThumbnailPlanImpl *pl, const void *in, size_t in_stride, void *out,
	size_t out_stride, int n, cudaStream_t s);

double
thumbnail_common_shrink(int w, int h, int tw, int th, int size)
{
	double hs, vs;
	thumbnail_shrink(w, h, tw, th, size, &hs, &vs);
	return std::min(hs, vs);
}

/* One frame through the leaf kernels (upsizing plans, 1- and 2-band plans, one-axis shrinks, and the linear geometries the
 * two-kernel path declines): enter the working space, premultiply, vips_resize, unpremultiply, leave the working space.
 *   uchar plan:   no working space; premultiply with the 8-bit LUT (thumbnail.c:848-902)
 *   linear plan:  sRGB -> scRGB ... scRGB -> sRGB, float premultiply at 1.0 (thumbnail.c:766-806, 971-987)
 *   LIN_XYZ:      sRGB -> scRGB ... scRGB -> XYZ -> the export job (:790-805, 957-970)
 *   LIN_IMPORT:   the import job ... the export job, float premultiply at 255 on XYZ (:766-789, 929-942; header.c:195-206)
 * fr / jobs: the frame's colour management and the batch's host job table (fr null: none).  `out` takes the last step's bands.
 */
static int
thumbnail_leaf_chain(const char *domain, const ThumbnailPlanImpl *pl, const IccFrame *fr, const IccJob *jobs, const void *in,
	void *out, cudaStream_t s)
{
	const int kind = fr ? fr->kind : LIN_PLAIN;
	DevImage din, lin, pre, res, unpre, xyz, fin;
	din.w = pl->W;
	din.h = pl->H;
	din.bands = pl->bands;
	din.fmt = VB200_FORMAT_UCHAR;
	din.type = pl->bands < 3 ? VB200_INTERPRETATION_B_W : VB200_INTERPRETATION_sRGB;
	din.bpl = (size_t) pl->W * pl->bands;
	din.data = const_cast<void *>(in);
	const double max_alpha = pl->linear && kind != LIN_IMPORT ? 1.0 : 255.0;
	const int uchar_mode = !pl->linear;
	const DevImage *cur = &din;
	int rc = 0;
	if (kind == LIN_IMPORT)
		rc = icc_job_apply(domain, jobs, fr->imp, din, &lin, s);
	else if (pl->linear)
		rc = dev_colourspace(domain, din, &lin, VB200_INTERPRETATION_scRGB, VB200_INTERPRETATION_sRGB, s);
	if (pl->linear)
		cur = &lin;
	if (!rc && pl->premul) {
		rc = dev_premultiply(domain, *cur, &pre, max_alpha, uchar_mode, s);
		cur = &pre;
	}
	if (!rc)
		rc = dev_resize(domain, *cur, &res, 1.0 / pl->hshrink, 1.0 / pl->vshrink, VB200_KERNEL_LANCZOS3, 2.0, s);
	cur = &res;
	if (!rc && pl->premul) {
		rc = dev_unpremultiply(domain, res, &unpre, max_alpha, uchar_mode, s);
		cur = &unpre;
	}
	if (!rc && pl->linear && kind != LIN_IMPORT) {
		rc = dev_colourspace(domain, *cur, &xyz, kind == LIN_XYZ ? VB200_INTERPRETATION_XYZ : VB200_INTERPRETATION_sRGB,
			VB200_INTERPRETATION_scRGB, s);
		cur = &xyz;
	}
	if (!rc && kind != LIN_PLAIN) {
		rc = icc_job_apply(domain, jobs, fr->exp, *cur, &fin, s);
		cur = &fin;
	}
	if (!rc) {
		const size_t line = (size_t) cur->w * cur->bands;
		if (cudaMemcpy2DAsync(out, line, cur->data, cur->bpl, line, cur->h, cudaMemcpyDeviceToDevice, s) != cudaSuccess)
			rc = cuda_fail(domain, cudaGetLastError(), "leaf thumbnail copy");
	}
	for (DevImage *d : {&lin, &pre, &res, &unpre, &xyz, &fin})
		dev_image_release(d, s);
	return rc;
}

/* The resize stage: the two-kernel linear path, the fused kernels (RGB frames expanded to RGBX around them) or, where they
 * decline, the leaf chain frame by frame.  icc: the batch's jobs of a linear plan's colour management (null: none), which the
 * linear path and the leaf chain run around the resize; `out` then takes the plan's output bands.
 */
static int
thumbnail_plan_run_thumbnail(const char *domain, ThumbnailPlanImpl *pl, const void *in, size_t in_stride, void *out,
	size_t out_stride, int n, cudaStream_t s, const IccBatch *icc)
{
	if (pl->lin) {
		const int rc = linear_thumb_run(domain, pl->lin, in, in_stride, out, out_stride, n, s, icc, pl->out_bands());
		if (rc != 1)
			return rc;
	}
	else if (pl->fused && pl->rgb_expand && pl->bands == 3) {
		/* sub-batches of RGBX scratch (~1 GiB): expand, fused kernel, compact */
		if ((((uintptr_t) in) | in_stride) & 3) {
			error(domain, "RGB frames must be 4-byte aligned for the fused path");
			return -1;
		}
		const size_t px_in = (size_t) pl->W * pl->H, px_out = (size_t) pl->OW * pl->OH;
		/* the frames of a sub-batch are gridDim.y of the expand / compact kernels: at most kMaxBatchFrames */
		const int sub = (int) std::max<size_t>(1,
			std::min<size_t>(std::min<size_t>((size_t) n, kMaxBatchFrames), ((size_t) 1 << 30) / (px_in * 4)));
		void *xin = nullptr, *xout = nullptr;
		if (dev_alloc(domain, &xin, px_in * 4 * sub, s) || dev_alloc(domain, &xout, px_out * 4 * sub, s)) {
			dev_free(xin, s);
			return -1;
		}
		int rc = 0;
		for (int f0 = 0; f0 < n && !rc; f0 += sub) {
			const int nf = std::min(sub, n - f0);
			rgb_expand_kernel<<<dim3((unsigned) ((px_in / 4 + 255) / 256), nf), 256, 0, s>>>(
				(const uint8_t *) in + (size_t) f0 * in_stride, in_stride, (uint8_t *) xin, px_in * 4, px_in / 4);
			cudaError_t e = cudaGetLastError();
			if (e != cudaSuccess) {
				rc = cuda_fail(domain, e, "rgb_expand_kernel");
				break;
			}
			count_launch();
			rc = thumbnail_plan_run_fused(domain, pl, xin, px_in * 4, xout, px_out * 4, nf, s);
			if (!rc) {
				rgbx_compact_kernel<<<dim3((unsigned) ((px_out + 255) / 256), nf), 256, 0, s>>>((const uint8_t *) xout, px_out * 4,
					(uint8_t *) out + (size_t) f0 * out_stride, out_stride, px_out);
				e = cudaGetLastError();
				if (e != cudaSuccess)
					rc = cuda_fail(domain, e, "rgbx_compact_kernel");
				else
					count_launch();
			}
		}
		dev_free(xin, s);
		dev_free(xout, s);
		return rc;
	}
	else if (pl->fused)
		return thumbnail_plan_run_fused(domain, pl, in, in_stride, out, out_stride, n, s);
	for (int i = 0; i < n; i++)
		if (thumbnail_leaf_chain(domain, pl, icc ? &icc->h_frames[i] : nullptr, icc ? icc->h_jobs : nullptr,
				(const char *) in + (size_t) i * in_stride, (char *) out + (size_t) i * out_stride, s))
			return -1;
	return 0;
}

/* The plan's stages over a device batch: the resize stage (on a linear plan with colour management, its import and export
 * inside it) -> the ICC stage (if set on a plan that is not linear) -> the sharpen stage (if set).  Every stage but the last
 * writes a scratch batch from the stream-ordered pool; the last writes `out`.  embedded / embedded_lens: each frame's embedded
 * ICC profile for colour management (NULL: none); frame0: the first frame's index in the caller's batch, for errors.
 */
int
thumbnail_plan_run_device(const char *domain, ThumbnailPlanImpl *pl, const void *in, size_t in_stride, void *out,
	size_t out_stride, int n, cudaStream_t s, const void *const *embedded = nullptr, const size_t *embedded_lens = nullptr,
	int frame0 = 0)
{
	if (n <= 0)
		return 0;
	const int ob = pl->out_bands();
	if (pl->sharpen && ob != 3 && ob != 4) {
		error(domain, "the sharpen stage needs 3- or 4-band frames, the output profile gives %d bands", ob);
		return -1;
	}
	const bool icc_stage = pl->icc && !pl->linear;
	const size_t pixels = (size_t) pl->OW * pl->OH, frame = pixels * (icc_stage ? pl->bands : ob), oframe = pixels * ob;
	void *mid = nullptr, *mid2 = nullptr; /* the resize stage's output, the ICC stage's before sharpen */
	if ((icc_stage || pl->sharpen) && dev_alloc(domain, &mid, frame * n, s))
		return -1;
	if (icc_stage && pl->sharpen && dev_alloc(domain, &mid2, oframe * n, s)) {
		dev_free(mid, s);
		return -1;
	}
	void *dst = mid ? mid : out;
	const size_t dst_stride = mid ? frame : out_stride;
	int rc;
	if (pl->icc && pl->linear)
		rc = icc_stage_batch(domain, pl->icc, n, embedded, embedded_lens, s, frame0, [&](const IccBatch &b) {
			return thumbnail_plan_run_thumbnail(domain, pl, in, in_stride, dst, dst_stride, n, s, &b);
		});
	else
		rc = thumbnail_plan_run_thumbnail(domain, pl, in, in_stride, dst, dst_stride, n, s, nullptr);
	if (!rc && icc_stage)
		rc = icc_stage_run(domain, pl->icc, mid, frame, mid2 ? mid2 : out, mid2 ? oframe : out_stride, n, pixels, embedded,
			embedded_lens, s, frame0);
	if (!rc && pl->sharpen) {
		rc = dev_sharpen_fused(domain, mid2 ? mid2 : mid, (size_t) pl->OW * ob, oframe, out, (size_t) pl->OW * ob, out_stride, n, pl->OW,
			pl->OH, ob, pl->sh_sigma, pl->sh_x1, pl->sh_y2, pl->sh_y3, pl->sh_m1, pl->sh_m2, s);
		if (rc == 1) {
			error(domain, "sharpen parameters are not on the fused path (mask too wide)");
			rc = -1;
		}
	}
	if (mid)
		dev_free(mid, s);
	if (mid2)
		dev_free(mid2, s);
	return rc;
}

/* the fused kernels over RGBA frames: the plan's kernel, but v1 when the base pointer or the frame stride of a batch
 * is off 16 bytes (the TMA-fed kernels copy whole 16-byte units); frames in chunks of at most kMaxBatchFrames (gridDim.z)
 */
static int
thumbnail_plan_run_fused(const char *domain, ThumbnailPlanImpl *pl, const void *in, size_t in_stride, void *out,
	size_t out_stride, int n, cudaStream_t s)
{
	const bool aligned = (((uintptr_t) in) & 15) == 0 && (n == 1 || (in_stride & 15) == 0);
	const FusedKernel kernel = aligned ? pl->kernel : FusedKernel::Ldg;
	for (int f0 = 0; f0 < n; f0 += kMaxBatchFrames) {
		const int nf = std::min(kMaxBatchFrames, n - f0);
		int rc = 0;
		switch (kernel) {
		case FusedKernel::Ldg: rc = launch_ldg(domain, pl, in, in_stride, out, out_stride, n, f0, nf, s); break;
		case FusedKernel::Tma: rc = launch_tma(domain, pl, in, in_stride, out, out_stride, n, f0, nf, s); break;
		case FusedKernel::Mma: rc = launch_mma(domain, pl, in, in_stride, out, out_stride, n, f0, nf, s); break;
		}
		if (rc)
			return rc;
	}
	return 0;
}

/* vb200_thumbnail_plan_kernel's name of the kernel a plan runs, in buf or a static string */
static const char *
plan_kernel_name(const ThumbnailPlanImpl &pl, char *buf, size_t cap)
{
	if (!pl.fused)
		return "leaf kernels";
	if (pl.linear)
		return "linear_v_kernel + linear_h_kernel";
	const FusedParams &fp = pl.fp;
	const char *alpha = pl.premul ? "premul" : "plain";
	/* v1 / v2: the box their switch instantiates (launch_ldg_vs, launch_tma_vs), else VS=0, the run-time form, and the box */
	char vs[24];
	const bool listed = (fp.VS >= 1 && fp.VS <= 4) || fp.VS == 8 || (pl.kernel == FusedKernel::Ldg && (fp.VS == 5 || fp.VS == 6));
	if (listed)
		snprintf(vs, sizeof(vs), "%d", fp.VS);
	else
		snprintf(vs, sizeof(vs), "0(%d)", fp.VS);
	const int np_tma = fp.NPv == fp.NPh && (fp.NPv == 6 || fp.NPv == 7) ? fp.NPv : 0; /* launch_tma */
	switch (pl.kernel) {
	case FusedKernel::Mma:
		snprintf(buf, cap, "thumbnail_fused_mma_kernel<VS=%d,NP=%d,%s,HS=%d,cols=%d,cpt=%d>", fp.VS, v4_np(fp.VS, fp.NPh, fp.HS), alpha,
			fp.HS, kV4Cols, kV4Cpt);
		break;
	case FusedKernel::Tma: snprintf(buf, cap, "thumbnail_fused_tma_kernel<VS=%s,NP=%d,%s>", vs, np_tma, alpha); break;
	case FusedKernel::Ldg: snprintf(buf, cap, "thumbnail_fused_kernel<VS=%s,%s>", vs, alpha); break;
	}
	return buf;
}

void
thumbnail_plan_destroy(ThumbnailPlanImpl *pl)
{
	if (pl->tables)
		cudaFree(pl->tables);
	if (pl->tables_mma)
		cudaFree(pl->tables_mma);
	if (pl->lin)
		linear_thumb_free(pl->lin);
	pl->lin = nullptr;
	icc_stage_free(pl->icc);
	pl->icc = nullptr;
	for (int i = 0; i < ThumbnailPlanImpl::kHintSlots; i++)
		if (pl->hint_done[i]) {
			cudaEventSynchronize(pl->hint_done[i]);
			cudaEventDestroy(pl->hint_done[i]);
		}
	if (pl->hint_counts)
		cudaFreeHost(pl->hint_counts);
	for (int i = 0; i < ThumbnailPlanImpl::kStreams; i++) {
		if (pl->stage_in[i])
			cudaFree(pl->stage_in[i]);
		if (pl->stage_out[i])
			cudaFree(pl->stage_out[i]);
		if (pl->drained[i])
			cudaEventDestroy(pl->drained[i]);
		if (pl->streams[i])
			cudaStreamDestroy(pl->streams[i]);
	}
}

} // namespace vb200

/* ------------------------------------------------------------------ C ABI */

using namespace vb200;

struct VB200ThumbnailPlan {
	ThumbnailPlanImpl impl;
};

/* a plan's request: frames of n_pages pages of page_height rows, 8-bit unless the caller says otherwise; -1 for a geometry no
 * plan takes
 */
static int
plan_request(ThumbnailPlanImpl *pl, int width, int page_height, int n_pages, int bands, int has_alpha, int target_width,
	int target_height, int size, int linear)
{
	if (width <= 0 || page_height <= 0 || n_pages <= 0 || (long long) page_height * n_pages > INT_MAX || bands <= 0 || target_width <= 0)
		return -1;
	pl->W = width;
	pl->H = page_height * n_pages;
	pl->page_h = n_pages > 1 ? page_height : 0;
	pl->bands = bands;
	pl->fmt = VB200_FORMAT_UCHAR;
	pl->has_alpha = has_alpha;
	pl->target_w = target_width;
	pl->target_h = target_height > 0 ? target_height : target_width;
	pl->size = size;
	pl->linear = linear;
	return 0;
}

extern "C" VB200ThumbnailPlan *
vb200_thumbnail_plan_new(int width, int height, int bands, int band_format, int has_alpha, int target_width,
	int target_height, int size, int linear)
{
	return vb200_thumbnail_plan_new_pages(width, height, 1, bands, band_format, has_alpha, target_width, target_height, size, linear);
}

/* See vb200.h: a plan for strips of n_pages pages of page_height rows (thumbnail.c:825-839, 904-917) */
extern "C" VB200ThumbnailPlan *
vb200_thumbnail_plan_new_pages(int width, int page_height, int n_pages, int bands, int band_format, int has_alpha, int target_width,
	int target_height, int size, int linear)
{
	const char *domain = "thumbnail_plan";
	if (ensure_init(domain))
		return nullptr;
	auto *plan = new VB200ThumbnailPlan();
	ThumbnailPlanImpl &pl = plan->impl;
	if (plan_request(&pl, width, page_height, n_pages, bands, has_alpha, target_width, target_height, size, linear)) {
		error(domain, "bad frame geometry");
		delete plan;
		return nullptr;
	}
	pl.fmt = band_format;
	if (thumbnail_plan_init(domain, &pl)) {
		thumbnail_plan_destroy(&pl);
		delete plan;
		return nullptr;
	}
	pl.out_page_h = plan_out_page_height(pl);
	return plan;
}

extern "C" int
vb200_thumbnail_plan_page_height(const VB200ThumbnailPlan *plan)
{
	return plan ? plan->impl.out_page_h : -1;
}

extern "C" void
vb200_thumbnail_plan_free(VB200ThumbnailPlan *plan)
{
	if (!plan)
		return;
	thumbnail_plan_destroy(&plan->impl);
	delete plan;
}

extern "C" int
vb200_thumbnail_plan_output(const VB200ThumbnailPlan *plan, int *out_width, int *out_height)
{
	if (!plan)
		return -1;
	if (out_width)
		*out_width = plan->impl.OW;
	if (out_height)
		*out_height = plan->impl.OH;
	return 0;
}

extern "C" size_t
vb200_thumbnail_plan_bytes_per_frame(const VB200ThumbnailPlan *plan)
{
	const ThumbnailPlanImpl &pl = plan->impl;
	return (size_t) pl.W * pl.H * pl.bands + (size_t) pl.OW * pl.OH * pl.bands;
}

extern "C" int
vb200_thumbnail_plan_set_sharpen(VB200ThumbnailPlan *plan, double sigma, double x1, double y2, double y3, double m1, double m2)
{
	const char *domain = "thumbnail_plan_set_sharpen";
	if (!plan) {
		error(domain, "null plan");
		return -1;
	}
	ThumbnailPlanImpl &pl = plan->impl;
	if (sigma <= 0) {
		pl.sharpen = false;
		return 0;
	}
	if ((pl.bands != 3 && pl.bands != 4) || pl.fmt != VB200_FORMAT_UCHAR) {
		error(domain, "the sharpen stage needs 3- or 4-band 8-bit frames");
		return -1;
	}
	if (sigma < 0.000001 || sigma > 10.0) { /* sharpen.c: the "sigma" argument's range */
		error(domain, "parameter sigma out of range [0.000001, 10]");
		return -1;
	}
	pl.sh_sigma = sigma;
	pl.sh_x1 = x1;
	pl.sh_y2 = y2;
	pl.sh_y3 = y3;
	pl.sh_m1 = m1;
	pl.sh_m2 = m2;
	pl.sharpen = true;
	return 0;
}

extern "C" int
vb200_thumbnail_plan_is_fused(const VB200ThumbnailPlan *plan)
{
	return plan && plan->impl.fused;
}

/* See vb200.h: the plan's kernel, which a batch call runs unless its frames are off 16 bytes */
extern "C" const char *
vb200_thumbnail_plan_kernel(const VB200ThumbnailPlan *plan)
{
	static thread_local char name[160];
	if (!plan)
		return "leaf kernels";
	return plan_kernel_name(plan->impl, name, sizeof(name));
}

extern "C" int
vb200_thumbnail_batch_device(VB200ThumbnailPlan *plan, const void *in, size_t in_frame_stride, void *out,
	size_t out_frame_stride, int n_frames)
{
	return vb200_thumbnail_batch_device_icc(plan, in, in_frame_stride, out, out_frame_stride, n_frames, nullptr, nullptr);
}

extern "C" int
vb200_thumbnail_batch_device_icc(VB200ThumbnailPlan *plan, const void *in, size_t in_frame_stride, void *out,
	size_t out_frame_stride, int n_frames, const void *const *embedded, const size_t *embedded_lens)
{
	const char *domain = "thumbnail_batch_device";
	if (!plan || !in || !out) {
		error(domain, "null argument");
		return -1;
	}
	if (ensure_init(domain))
		return -1;
	return thumbnail_plan_run_device(domain, &plan->impl, in, in_frame_stride, out, out_frame_stride, n_frames,
		current_stream(), embedded, embedded_lens);
}

/* the body of the ICC setters: the plan's stage, in the plan's mode, replaced by one for icc (NULL: off) */
static int
plan_set_icc(const char *domain, ThumbnailPlanImpl &pl, const VB200ThumbnailIcc *icc)
{
	IccStage *st = nullptr;
	int ob = 0;
	if (icc) {
		st = icc_stage_new();
		if (icc_stage_set(domain, st, icc, pl.bands, pl.linear, &ob)) {
			icc_stage_free(st);
			return -1;
		}
	}
	icc_stage_free(pl.icc);
	pl.icc = st;
	pl.icc_bands = ob;
	return 0;
}

extern "C" int
vb200_thumbnail_plan_set_icc(VB200ThumbnailPlan *plan, const VB200ThumbnailIcc *icc)
{
	const char *domain = "thumbnail_plan_set_icc";
	if (!plan) {
		error(domain, "null plan");
		return -1;
	}
	const bool off = !icc || !icc->output_profile;
	if (plan->impl.linear) {
		/* a linear plan's stage is vb200_thumbnail_plan_set_linear_icc's, and this setter's "off" leaves it alone.
		 * thumbnail.c:766-806, 957-970: an ICC import into the linear V kernel and an export from the H kernel, not built here
		 */
		if (off)
			return 0;
		error(domain, "linear thumbnails with an output profile are not supported on the device path");
		return -1;
	}
	return plan_set_icc(domain, plan->impl, off ? nullptr : icc);
}

extern "C" int
vb200_thumbnail_plan_set_linear_icc(VB200ThumbnailPlan *plan, const VB200ThumbnailIcc *icc)
{
	const char *domain = "thumbnail_plan_set_linear_icc";
	if (!plan) {
		error(domain, "null plan");
		return -1;
	}
	if (!plan->impl.linear) {
		error(domain, "the plan is not linear: use vb200_thumbnail_plan_set_icc");
		return -1;
	}
	return plan_set_icc(domain, plan->impl, icc);
}

extern "C" int
vb200_thumbnail_plan_output_bands(const VB200ThumbnailPlan *plan)
{
	return plan ? plan->impl.out_bands() : -1;
}

/* reference: vips_thumbnail_buffer(buf, len, &out, width, "height", height, "size", size, NULL), resample/thumbnail.c:
 * 583-613 (open with the load-time shrink vips_thumbnail_find_jpegshrink picks) then :848-902 on what was loaded.
 * JPEG, PNG, GIF or TIFF streams; everything between the compressed bytes and the thumbnail stays on the device.  A TIFF
 * loads the subifd or page of a pyramid that vips_thumbnail_find_pyrlevel picks (vb200_thumbnail_tiff_level).
 */
extern "C" int
vb200_thumbnail_buffer(const void *buf, size_t len, VB200Image *out, int width, int height, int size)
{
	return vb200_thumbnail_buffer_icc(buf, len, out, width, height, size, nullptr);
}

static int thumbnail_image_run(const VB200Image *in, int page_height, VB200Image *out, int width, int height, int size, int linear,
	const VB200ThumbnailIcc *icc, const void *embedded, size_t embedded_len, int *out_page_height);

/* linear: decoded at full size (thumbnail.c:496-499) and thumbnailed by vb200_thumbnail_image_linear_icc.  A GIF's pages
 * page .. page + n - 1 decode to a strip with nsgifload's page-height, set when more than one page loaded
 * (nsgifload.c:279-280), and are thumbnailed as one (vb200_thumbnail_image_pages).
 */
static int
thumbnail_buffer_run(const void *buf, size_t len, VB200Image *out, int width, int height, int size, const VB200ThumbnailIcc *icc,
	bool linear, int page = 0, int n_pages = 1, int *out_page_height = nullptr, bool webp = false)
{
	const char *domain = "thumbnail_buffer";
	if (!buf || !out) {
		error(domain, "null argument");
		return -1;
	}
	DecodeRequest req{stream_kind(buf, len), 1, page, n_pages};
	if (req.kind == STREAM_WEBP && !webp) {
		/* thumbnail.c:627-636, 1524-1532 load WebP at scale = 1 / factor: libwebp's own rescaler, not the full-size decode */
		error(domain, "WebP shrink-on-load (libwebp's scaled decode) is not built on the device path; vb200_thumbnail_webp_buffer takes WebP streams");
		return -1;
	}
	if (webp && req.kind != STREAM_WEBP) {
		error(domain, "not a WebP stream (no RIFF / WEBP signature)");
		return -1;
	}
	if (ensure_init(domain))
		return -1;
	if (req.kind == STREAM_TIFF) {
		/* the level vips_thumbnail_open picks: a subifd or page of a pyramid, else page 0 (thumbnail.c:562-581, 1552-1576) */
		if (page != 0 || n_pages != 1) {
			error(domain, "TIFF page strips are not thumbnailed on the device (page %d, n %d)", page, n_pages);
			return -1;
		}
		if (tiff_thumbnail_level(domain, (const unsigned char *) buf, len, width, height, size, &req.subifd, &req.page))
			return -1;
	}
	const bool want_profile = icc && (icc->output_profile || linear);
	std::vector<unsigned char> embedded;
	if ((req.kind == STREAM_PNG || req.kind == STREAM_TIFF || want_profile) && stream_profile(domain, req, (const unsigned char *) buf, len, &embedded))
		return -1;
	if (!want_profile)
		embedded.clear();
	cudaStream_t s = current_stream();
	if (req.kind == STREAM_JPEG && !linear) {
		int w0, h0, b0;
		if (dev_decode_batch(domain, req, &buf, &len, 1, nullptr, 0, 0, &w0, &h0, &b0, nullptr, s))
			return -1;
		req.shrink = vb200_thumbnail_jpegshrink(w0, h0, width, height, size);
	}
	if (req.kind == STREAM_WEBP) {
		/* linear or not: only find_jpegshrink declines in linear mode (thumbnail.c:496-499) */
		int w0, h0, b0;
		if (dev_decode_batch(domain, req, &buf, &len, 1, nullptr, 0, 0, &w0, &h0, &b0, nullptr, s) ||
			vb200_thumbnail_webp_scale(w0, h0, width, height, size, &req.scale, nullptr, nullptr))
			return -1;
	}
	DevImage dec;
	int page_height;
	if (dev_load(domain, req, buf, len, &dec, &page_height, s))
		return -1;
	VB200Image din;
	memset(&din, 0, sizeof(din));
	din.Xsize = dec.w;
	din.Ysize = dec.h;
	din.Bands = dec.bands;
	din.BandFmt = VB200_FORMAT_UCHAR;
	din.Type = dec.type;
	din.where = VB200_DEVICE;
	din.data = dec.data;
	din.bpl = dec.bpl;
	const int where = out->where;
	VB200Image tmp;
	memset(&tmp, 0, sizeof(tmp));
	tmp.where = VB200_DEVICE;
	int rc = thumbnail_image_run(&din, page_height, &tmp, width, height, size, linear, icc, embedded.data(), embedded.size(), out_page_height);
	if (!rc) {
		/* deliver where the caller asked (allocate-or-fill) */
		DevImage dt;
		dt.w = tmp.Xsize;
		dt.h = tmp.Ysize;
		dt.bands = tmp.Bands;
		dt.fmt = tmp.BandFmt;
		dt.type = tmp.Type;
		dt.data = tmp.data;
		dt.bpl = tmp.bpl;
		dt.owned = true;
		VB200Image like = *out;
		like.where = where;
		rc = deliver(domain, &dt, &like, out, s);
	}
	dev_image_release(&dec, s);
	return rc;
}

extern "C" int
vb200_thumbnail_buffer_icc(const void *buf, size_t len, VB200Image *out, int width, int height, int size, const VB200ThumbnailIcc *icc)
{
	return thumbnail_buffer_run(buf, len, out, width, height, size, icc, false);
}

extern "C" int
vb200_thumbnail_buffer_linear_icc(const void *buf, size_t len, VB200Image *out, int width, int height, int size,
	const VB200ThumbnailIcc *icc)
{
	return thumbnail_buffer_run(buf, len, out, width, height, size, icc, true);
}

/* reference: vips_thumbnail_buffer of a WebP stream: loaded at scale = 1 / vips_thumbnail_open's factor (thumbnail.c:627-636,
 * 1524-1532) through the device's scaled decode, the stream's ICCP as the embedded profile, then thumbnail_image_run */
extern "C" int
vb200_thumbnail_webp_buffer(const void *buf, size_t len, VB200Image *out, int width, int height, int size, const VB200ThumbnailIcc *icc, int linear)
{
	return thumbnail_buffer_run(buf, len, out, width, height, size, icc, linear != 0, 0, 1, nullptr, true);
}

/* reference: vips_thumbnail_open's WebP factor, max(1, the common shrink) (thumbnail.c:627-636), as webpload's scale and the
 * frame size it loads at (webp2vips.c:513-514) */
extern "C" int
vb200_thumbnail_webp_scale(int width, int height, int target_width, int target_height, int size, double *scale, int *scaled_width,
	int *scaled_height)
{
	if (width < 1 || height < 1 || target_width < 1 || !scale) {
		error("thumbnail_webp_scale", "bad arguments (%d x %d to width %d)", width, height, target_width);
		return -1;
	}
	const double factor = std::max(1.0, thumbnail_common_shrink(width, height, target_width, target_height > 0 ? target_height : target_width, size));
	*scale = 1.0 / factor;
	if (scaled_width)
		*scaled_width = (int) rint(width * *scale);
	if (scaled_height)
		*scaled_height = (int) rint(height * *scale);
	return 0;
}

/* See vb200.h: vips_thumbnail_buffer(..., option_string = "page=..,n=..") */
extern "C" int
vb200_thumbnail_buffer_pages(const void *buf, size_t len, VB200Image *out, int width, int height, int size, const VB200ThumbnailIcc *icc,
	int linear, int page, int n, int *out_page_height)
{
	if (buf && stream_kind(buf, len) == STREAM_TIFF) {
		error("thumbnail_buffer", "TIFF page strips are not thumbnailed on the device: use vb200_thumbnail_buffer");
		return -1;
	}
	return thumbnail_buffer_run(buf, len, out, width, height, size, icc, linear != 0, page, n, out_page_height);
}

/* Decode staging feeding the plan (SURVEY 8f rank 1): compressed bytes up, decoded on the device (jpeg.cu at `shrink`,
 * png.cu and gif.cu at full size), thumbnailed by the plan's kernels -- the decoded frames never exist in host memory.  What
 * vips_thumbnail_buffer() does with the loader + vips_thumbnail_image (thumbnail.c:583-613, 848-902).
 */
static int
plan_run_streams(const char *domain, const DecodeRequest &req, VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, void *out,
	int out_location, size_t out_frame_stride)
{
	if (!plan || !bufs || !lens || !out || n < 1) {
		error(domain, "null argument");
		return -1;
	}
	if (ensure_init(domain))
		return -1;
	ThumbnailPlanImpl &pl = plan->impl;
	cudaStream_t s = current_stream();
	const size_t in_frame = (size_t) pl.W * pl.H * pl.bands, out_frame = (size_t) pl.OW * pl.OH * pl.out_bands();
	if (out_frame_stride == 0)
		out_frame_stride = out_frame;
	/* with colour management on, each stream's embedded profile (jpeg2vips.c:699-799, spngload.c:244-246) goes to the ICC
	 * stage; PNG streams are read for eXIf either way
	 */
	const bool managed = pl.icc != nullptr;
	std::vector<std::vector<unsigned char>> profiles(managed || req.kind == STREAM_PNG || req.kind == STREAM_TIFF ? n : 0);
	std::vector<const void *> emb(profiles.size());
	std::vector<size_t> emb_len(profiles.size());
	for (size_t i = 0; i < profiles.size(); i++) {
		if (stream_profile(domain, req, (const unsigned char *) bufs[i], lens[i], &profiles[i])) {
			error(domain, "stream %d", (int) i);
			return -1;
		}
		emb[i] = profiles[i].empty() ? nullptr : profiles[i].data();
		emb_len[i] = profiles[i].size();
	}
	const void *const *embedded = managed ? emb.data() : nullptr;
	const size_t *embedded_lens = managed ? emb_len.data() : nullptr;
	void *dec = nullptr, *res = nullptr;
	if (dev_alloc(domain, &dec, in_frame * n, s))
		return -1;
	int rc = -1;
	do {
		int w, h, b, page_h;
		if (dev_decode_batch(domain, req, bufs, lens, n, dec, (size_t) pl.W * pl.bands, in_frame, &w, &h, &b, &page_h, s))
			break;
		/* a GIF strip is the plan's only if its pages are: the screen must be one page high */
		if ((req.kind == STREAM_GIF || req.kind == STREAM_TIFF) && (page_h ? page_h : h) != (pl.page_h ? pl.page_h : pl.H)) {
			error(domain, "the plan is for pages of %d rows, the streams' screen is %d rows", pl.page_h ? pl.page_h : pl.H, page_h ? page_h : h);
			break;
		}
		if (w != pl.W || h != pl.H || b != pl.bands) {
			error(domain, "the plan is for %d x %d x %d frames, the streams decode to %d x %d x %d", pl.W, pl.H, pl.bands, w, h, b);
			break;
		}
		if (out_location == VB200_DEVICE) {
			rc = thumbnail_plan_run_device(domain, &pl, dec, in_frame, out, out_frame_stride, n, s, embedded, embedded_lens);
			break;
		}
		if (dev_alloc(domain, &res, out_frame * n, s))
			break;
		if (thumbnail_plan_run_device(domain, &pl, dec, in_frame, res, out_frame, n, s, embedded, embedded_lens))
			break;
		if (cudaMemcpy2DAsync(out, out_frame_stride, res, out_frame, out_frame, n, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
			cudaStreamSynchronize(s) != cudaSuccess) {
			cuda_fail(domain, cudaGetLastError(), "copy to host");
			break;
		}
		rc = 0;
	} while (0);
	dev_free(dec, s);
	if (res)
		dev_free(res, s);
	return rc;
}

extern "C" int
vb200_thumbnail_plan_run_jpeg(VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, int shrink, void *out,
	int out_location, size_t out_frame_stride)
{
	return plan_run_streams("thumbnail_plan_run_jpeg", {STREAM_JPEG, shrink}, plan, bufs, lens, n, out, out_location, out_frame_stride);
}

extern "C" int
vb200_thumbnail_plan_run_png(VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, void *out, int out_location,
	size_t out_frame_stride)
{
	return plan_run_streams("thumbnail_plan_run_png", {STREAM_PNG}, plan, bufs, lens, n, out, out_location, out_frame_stride);
}

extern "C" int
vb200_thumbnail_plan_run_gif(VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, void *out, int out_location,
	size_t out_frame_stride)
{
	return plan_run_streams("thumbnail_plan_run_gif", {STREAM_GIF}, plan, bufs, lens, n, out, out_location, out_frame_stride);
}

extern "C" int
vb200_thumbnail_plan_run_gif_pages(VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, int page, int n_pages,
	void *out, int out_location, size_t out_frame_stride)
{
	return plan_run_streams("thumbnail_plan_run_gif", {STREAM_GIF, 1, page, n_pages}, plan, bufs, lens, n, out, out_location, out_frame_stride);
}

/* See vb200.h: the WebP streams decoded at webpload's scale, then the plan (made for the scaled geometry) */
extern "C" int
vb200_thumbnail_plan_run_webp(VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, double scale, void *out, int out_location,
	size_t out_frame_stride)
{
	DecodeRequest req{STREAM_WEBP};
	req.scale = scale;
	return plan_run_streams("thumbnail_plan_run_webp", req, plan, bufs, lens, n, out, out_location, out_frame_stride);
}

/* See vb200.h: the TIFF streams' pages page .. page + n_pages - 1 at subifd, then the plan */
extern "C" int
vb200_thumbnail_plan_run_tiff(VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, int page, int n_pages, int subifd,
	void *out, int out_location, size_t out_frame_stride)
{
	DecodeRequest req{STREAM_TIFF, 1, page, n_pages};
	req.subifd = subifd;
	return plan_run_streams("thumbnail_plan_run_tiff", req, plan, bufs, lens, n, out, out_location, out_frame_stride);
}

/* The tile pump: a ring of kStreams device staging slots; for each slice of
 * frames  H2D (pinned or pageable source) -> fused kernel -> D2H  on its own
 * stream, so copy-in, compute and copy-out of consecutive slices overlap.
 * Replaces vips_sink_memory + the threadpool on this path
 * (reference: iofuncs/sinkmemory.c:171-274, threadpool.c:301-369).
 */
extern "C" int
vb200_thumbnail_batch_host(VB200ThumbnailPlan *plan, const void *in, size_t in_frame_stride, void *out,
	size_t out_frame_stride, int n_frames)
{
	return vb200_thumbnail_batch_host_icc(plan, in, in_frame_stride, out, out_frame_stride, n_frames, nullptr, nullptr);
}

extern "C" int
vb200_thumbnail_batch_host_icc(VB200ThumbnailPlan *plan, const void *in, size_t in_frame_stride, void *out,
	size_t out_frame_stride, int n_frames, const void *const *embedded, const size_t *embedded_lens)
{
	const char *domain = "thumbnail_batch_host";
	if (!plan || !in || !out) {
		error(domain, "null argument");
		return -1;
	}
	if (ensure_init(domain))
		return -1;
	ThumbnailPlanImpl &pl = plan->impl;
	std::lock_guard<std::mutex> lock(pl.pump_lock); /* one pump per plan at a time: the staging ring is the plan's */
	const size_t in_frame = (size_t) pl.W * pl.H * pl.bands;
	const size_t out_frame = (size_t) pl.OW * pl.OH * pl.out_bands();
	/* Slice size: ~64 MiB of input per slot (one 4K RGBA frame).  The pump is bound by the H2D copy
	 * (one such frame is 1.2 ms of PCIe against 14 us of kernel), so small slices cost nothing and
	 * shorten the pipeline fill; small frames are batched up to the same byte budget.
	 */
	const int per_slice = (int) std::max<size_t>(1, std::min<size_t>(n_frames, (64u << 20) / in_frame));
	if (pl.stage_frames < per_slice || pl.stage_out_frame != out_frame) { /* the ICC stage may change the output bands */
		for (int i = 0; i < ThumbnailPlanImpl::kStreams; i++) {
			if (pl.streams[i])
				cudaStreamSynchronize(pl.streams[i]);
			if (pl.stage_in[i])
				cudaFree(pl.stage_in[i]);
			if (pl.stage_out[i])
				cudaFree(pl.stage_out[i]);
			pl.stage_in[i] = pl.stage_out[i] = nullptr;
			VB200_CUDA(domain, cudaMalloc(&pl.stage_in[i], in_frame * std::max(per_slice, pl.stage_frames)));
			VB200_CUDA(domain, cudaMalloc(&pl.stage_out[i], out_frame * std::max(per_slice, pl.stage_frames)));
			if (!pl.streams[i])
				VB200_CUDA(domain, cudaStreamCreateWithFlags(&pl.streams[i], cudaStreamNonBlocking));
			if (!pl.drained[i])
				VB200_CUDA(domain, cudaEventCreateWithFlags(&pl.drained[i], cudaEventDisableTiming | cudaEventBlockingSync));
		}
		pl.stage_frames = std::max(per_slice, pl.stage_frames);
		pl.stage_out_frame = out_frame;
	}

	bool used[ThumbnailPlanImpl::kStreams] = {false, false, false};
	int slot = 0;
	for (int f = 0; f < n_frames; f += per_slice, slot = (slot + 1) % ThumbnailPlanImpl::kStreams) {
		const int n = std::min(per_slice, n_frames - f);
		cudaStream_t s = pl.streams[slot];
		/* the slot's previous slice must have drained (its D2H recorded the event) before its staging
		 * buffers are overwritten; the host sleeps on the event instead of spinning on the stream
		 */
		if (used[slot])
			VB200_CUDA(domain, cudaEventSynchronize(pl.drained[slot]));
		VB200_CUDA(domain, cudaMemcpy2DAsync(pl.stage_in[slot], in_frame, (const char *) in + (size_t) f * in_frame_stride,
							   in_frame_stride, in_frame, n, cudaMemcpyHostToDevice, s));
		if (thumbnail_plan_run_device(domain, &pl, pl.stage_in[slot], in_frame, pl.stage_out[slot], out_frame, n, s,
				embedded ? embedded + f : nullptr, embedded_lens ? embedded_lens + f : nullptr, f))
			return -1;
		VB200_CUDA(domain, cudaMemcpy2DAsync((char *) out + (size_t) f * out_frame_stride, out_frame_stride,
							   pl.stage_out[slot], out_frame, out_frame, n, cudaMemcpyDeviceToHost, s));
		VB200_CUDA(domain, cudaEventRecord(pl.drained[slot], s));
		used[slot] = true;
	}
	for (int i = 0; i < ThumbnailPlanImpl::kStreams; i++)
		if (used[i])
			VB200_CUDA(domain, cudaEventSynchronize(pl.drained[i]));
	return 0;
}

/* vips_thumbnail_image, with colour management when icc sets an output profile, or with linear = TRUE when icc is set at all
 * (vb200_thumbnail_plan_set_linear_icc).  page_height: the input's page-height metadata (0: none), read as
 * vips_image_get_page_height does; out_page_height (may be NULL) gets the result's.
 */
static int
thumbnail_image_run(const VB200Image *in, int page_height, VB200Image *out, int width, int height, int size, int linear,
	const VB200ThumbnailIcc *icc, const void *embedded, size_t embedded_len, int *out_page_height)
{
	const char *domain = "thumbnail";
	if (!in || !out) {
		error(domain, "null argument");
		return -1;
	}
	if (linear && icc && !(in->Type == VB200_INTERPRETATION_sRGB && in->Bands >= 3)) {
		/* thumbnail.c:766-789 imports other interpretations with a profile of their space, and 1- / 2-band frames with sGrey:
		 * not on the device path
		 */
		error(domain, "linear colour-managed thumbnails of interpretation %d with %d bands are not supported on the device path",
			in->Type, in->Bands);
		return -1;
	}
	if (linear && icc) {
		/* the profiles are checked before any pixel moves: the stage's own checks, on the host, on a stage of its own */
		IccStage *st = icc_stage_new();
		int ob = 0;
		const int rc = icc_stage_set(domain, st, icc, in->Bands, true, &ob);
		icc_stage_free(st);
		if (rc)
			return -1;
	}
	if (icc && icc->output_profile &&
		!((in->Type == VB200_INTERPRETATION_sRGB && in->Bands >= 3) || (in->Type == VB200_INTERPRETATION_B_W && in->Bands < 3))) {
		/* with a profile pair the reference keeps the image's own interpretation (thumbnail.c:807-823) and imports with a
		 * profile of that space (icc_transform.c:565-577, e.g. CMYK); the device stage takes 8-bit sRGB / B_W frames only
		 */
		error(domain, "colour-managed thumbnails of interpretation %d with %d bands are not supported on the device path", in->Type,
			in->Bands);
		return -1;
	}
	if (ensure_init(domain))
		return -1;
	if (linear && (in->BandFmt != VB200_FORMAT_UCHAR || in->Bands < 3)) {
		error(domain, "linear thumbnails on the device path need an 8-bit image with 3+ bands");
		return -1;
	}
	/* vips_image_hasalpha(): more bands than the interpretation implies (iofuncs/image.c:3113-3119) */
	const int has_alpha = image_hasalpha(in->Type, in->Bands);
	const int ph = page_height > 0 && page_height < in->Ysize && in->Ysize % page_height == 0 ? page_height : in->Ysize; /* header.c:889-901 */
	VB200ThumbnailPlan *plan = vb200_thumbnail_plan_new_pages(in->Xsize, ph, ph > 0 ? in->Ysize / ph : 1, in->Bands, in->BandFmt, has_alpha, width,
		height, size, linear);
	if (!plan)
		return -1;
	if (out_page_height)
		*out_page_height = plan->impl.out_page_h;
	if (icc && (linear ? vb200_thumbnail_plan_set_linear_icc(plan, icc) : vb200_thumbnail_plan_set_icc(plan, icc))) {
		vb200_thumbnail_plan_free(plan);
		return -1;
	}
	const int ob = plan->impl.out_bands();
	/* icc_transform.c:374-433: the output interpretation follows the output profile's colour bands */
	const int colour = ob - (in->Bands - (in->Bands < 3 ? 1 : 3));
	const int otype = !plan->impl.icc ? in->Type
		: colour == 1				  ? VB200_INTERPRETATION_B_W
		: colour == 3				  ? VB200_INTERPRETATION_sRGB
									  : VB200_INTERPRETATION_CMYK;
	cudaStream_t s = current_stream();
	DevImage din, dout;
	int rc = to_device(domain, in, &din, s);
	if (!rc && din.bpl != (size_t) din.w * din.bands) {
		error(domain, "device frames must be packed");
		rc = -1;
	}
	if (!rc)
		rc = dev_image_new(domain, &dout, plan->impl.OW, plan->impl.OH, ob, in->BandFmt, otype, s);
	if (!rc) {
		const void *emb[1] = {embedded};
		const size_t emb_len[1] = {embedded ? embedded_len : 0};
		rc = thumbnail_plan_run_device(domain, &plan->impl, din.data, 0, dout.data, 0, 1, s, emb, emb_len);
	}
	if (!rc)
		rc = deliver(domain, &dout, in, out, s);
	if (!rc && in->where == VB200_DEVICE)
		cudaStreamSynchronize(s); /* the plan's tables die with it */
	dev_image_release(&din, s);
	vb200_thumbnail_plan_free(plan);
	return rc;
}

/* reference: vips_thumbnail_image(), resample/thumbnail.c:2000 */
extern "C" int
vb200_thumbnail_image(const VB200Image *in, VB200Image *out, int width, int height, int size, int linear)
{
	return thumbnail_image_run(in, 0, out, width, height, size, linear, nullptr, nullptr, 0, nullptr);
}

/* vips_thumbnail_image with "input_profile" / "output_profile" / "intent"; `embedded`: the image's ICC blob */
extern "C" int
vb200_thumbnail_image_icc(const VB200Image *in, VB200Image *out, int width, int height, int size, const VB200ThumbnailIcc *icc,
	const void *embedded, size_t embedded_len)
{
	return thumbnail_image_run(in, 0, out, width, height, size, 0, icc, embedded, embedded_len, nullptr);
}

/* See vb200.h: vips_thumbnail_image of a page strip (thumbnail.c:825-839, 904-917) */
extern "C" int
vb200_thumbnail_image_pages(const VB200Image *in, int page_height, VB200Image *out, int width, int height, int size,
	const VB200ThumbnailIcc *icc, const void *embedded, size_t embedded_len, int linear, int *out_page_height)
{
	return thumbnail_image_run(in, page_height, out, width, height, size, linear != 0, icc, embedded, embedded_len, out_page_height);
}

/* vips_thumbnail_image(..., linear = TRUE) with "input_profile" / "output_profile" / "intent" (thumbnail.c:766-805, 929-987):
 * an embedded profile alone turns colour management on.  icc NULL: vb200_thumbnail_image(linear = 1).
 */
extern "C" int
vb200_thumbnail_image_linear_icc(const VB200Image *in, VB200Image *out, int width, int height, int size, const VB200ThumbnailIcc *icc,
	const void *embedded, size_t embedded_len)
{
	return thumbnail_image_run(in, 0, out, width, height, size, 1, icc, embedded, embedded_len, nullptr);
}

/* Test hook (tests/test_thumbnail_bands.py, CPU): the tensor-pipe kernel's bands of an RGBA thumbnail plan, planned
 * without a device.  See vb200.h.
 */
extern "C" int
vb200_debug_thumbnail_bands(int width, int height, int target_width, int *out_width, int *n_bands, int *xa, int *xb,
	int *c_lo, int *c_hi, int *seam, int cap, int *box_width, int *n_box)
{
	ThumbnailPlanImpl pl;
	if (cap <= 0 || plan_request(&pl, width, height, 1, 4, 1, target_width, target_width, VB200_SIZE_BOTH, 0))
		return -1;
	pl.geometry_only = true;
	if (thumbnail_plan_init("debug_thumbnail_bands", &pl))
		return -1;
	if (!pl.fused || pl.kernel != FusedKernel::Mma)
		return 1;
	const int nb = (int) pl.mma_bands.size();
	if (nb > cap)
		return -1;
	*out_width = pl.OW;
	*n_bands = nb;
	for (int b = 0; b < nb; b++) {
		const MmaBand &m = pl.mma_bands[b];
		xa[b] = m.xa;
		xb[b] = m.xb;
		c_lo[b] = m.c_lo;
		c_hi[b] = m.c_hi;
		seam[b] = b + 1 < nb ? std::max(0, m.c_hi - pl.mma_bands[b + 1].c_lo) : 0;
	}
	*n_box = v4_nbox(pl.fp.HS); /* the boxes launch_mma_t gives the stage tensor map */
	*box_width = v4_boxw(pl.fp.HS);
	return 0;
}

/* Test hook (tests/test_thumbnail_kernel_choice.py, CPU): vb200_thumbnail_plan_kernel's name for the plan
 * vb200_thumbnail_plan_new would build, planned without a device.  See vb200.h.
 */
extern "C" int
vb200_debug_thumbnail_kernel(int width, int height, int bands, int has_alpha, int target_width, int target_height, int size,
	char *name, int cap)
{
	return vb200_debug_thumbnail_pages_kernel(width, height, 1, bands, has_alpha, target_width, target_height, size, name, cap);
}

/* Test hook (tests/test_thumbnail_pages.py, CPU): vb200_debug_thumbnail_kernel for the plan vb200_thumbnail_plan_new_pages
 * would build.  See vb200.h.
 */
extern "C" int
vb200_debug_thumbnail_pages_kernel(int width, int page_height, int n_pages, int bands, int has_alpha, int target_width,
	int target_height, int size, char *name, int cap)
{
	ThumbnailPlanImpl pl;
	if (!name || cap <= 0 || plan_request(&pl, width, page_height, n_pages, bands, has_alpha, target_width, target_height, size, 0))
		return -1;
	pl.geometry_only = true;
	if (thumbnail_plan_init("debug_thumbnail_kernel", &pl))
		return -1;
	char buf[160];
	const char *k = plan_kernel_name(pl, buf, sizeof(buf));
	if ((int) strlen(k) >= cap)
		return -1;
	strcpy(name, k);
	return 0;
}

/* Test hook (tests/test_thumbnail_pages.py, CPU): the shrinks, output size and output page height of the plan
 * vb200_thumbnail_plan_new_pages would build, planned without a device.  See vb200.h.
 */
extern "C" int
vb200_debug_thumbnail_pages_size(int width, int page_height, int n_pages, int target_width, int target_height, int size, double *hshrink,
	double *vshrink, int *out_width, int *out_height, int *out_page_height)
{
	ThumbnailPlanImpl pl;
	if (plan_request(&pl, width, page_height, n_pages, 1, 0, target_width, target_height, size, 0))
		return -1;
	pl.geometry_only = true;
	if (thumbnail_plan_init("debug_thumbnail_pages_size", &pl))
		return -1;
	*hshrink = pl.hshrink;
	*vshrink = pl.vshrink;
	*out_width = pl.OW;
	*out_height = pl.OH;
	*out_page_height = plan_out_page_height(pl);
	return 0;
}
