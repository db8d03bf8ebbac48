/* histogram.cu -- vips_hist_find, vips_hist_equal and vips_hist_local on the device.
 *
 * reference:
 *   arithmetic/hist_find.c: uchar and ushort inputs (the format table :376-379 casts everything else to one of them, which
 *     is not built here), band -1 or one band (vips_check_bandno, :147-149), width mx + 1 where a uchar histogram of every
 *     band is always 256 wide (:361) and every other one is as wide as the largest value seen plus one (SCANOP :285-296,
 *     SCAN1 :323-339), format UINT, DOUBLE from 2^32 pixels on (:155-162, :176-177), interpretation HISTOGRAM.
 *   histogram/hist_equal.c:81-89: hist_find -> hist_cum -> hist_norm -> cast to the input's format -> maplut.
 *   histogram/hist_cum.c:72-85, 140-141: a uint histogram accumulates in unsigned int.
 *   histogram/hist_norm.c:98-127: a[b] = new_max / max[b] in double with new_max = the histogram's width - 1, through
 *     vips_linear; every band's max is the pixel count, so the constants are equal and linear.c:155-178 takes its
 *     single-element loop, LOOP1(unsigned int, float) :213-224: q = (float) a * (float) p + 0.0f.  The result is cast
 *     (cast.c:231-239, clip in double, then truncation) to uchar when new_max <= 255, else ushort, and then to the input's
 *     format.
 *   histogram/maplut.c:140-160 and siblings: an index past the table is clipped to its last entry (clp = sz - 1, :684-685);
 *     a one-band table maps every band (loop1), an n-band table band by band (loop).
 *   histogram/hist_local.c:133-250 (generate), :283-306 (build): uchar only, window no larger than the image, input
 *     embedded at (width / 2, height / 2) with VIPS_EXTEND_MIRROR (conversion/embed.c:398-430: period 2W, the edge pixel
 *     repeated), the 256-bin window histogram slid one column per output, and per element
 *         sum = sum_{i <= t} min(h[i], m) + (t + 1) * sum_over / 256,  sum_over = sum_i max(h[i] - m, 0)   (m > 0)
 *         sum = sum_{i <= t} h[i]                                                                         (m == 0)
 *         q = 255 * sum / (width * height)
 *     all in int (:237, :249).  255 * sum and (t + 1) * sum_over overflow int once width * height > 8 388 607, undefined
 *     behaviour in the reference: such windows are refused here.
 *
 * hist_find: per-CTA shared-memory sub-histograms merged into a uint32 table with global atomics; the largest value is a
 *   warp max then one atomicMax per warp.  uchar: 256 bins for up to 32 bands per CTA.  ushort: 65 536 uint32 bins per
 *   band do not fit in shared memory, so the bins are split in two passes of 32 768 (128 KiB): each (band, half) is a
 *   grid row of its own and reads the image once.  No bin can wrap: images of 2^32 pixels or more are declined (the
 *   reference's DOUBLE histogram is not built), so no count reaches 2^32.
 * hist_equal: the histogram, its cumulative sum and the LUT are built on the device from the device histogram (one CTA
 *   per LUT band scans the table), so neither the stand-alone call nor a chain step waits for the host; maplut reads the
 *   LUT from shared memory.
 * hist_local: one CTA per (16-row x 128-column output tile), 16 warps.  The CTA stages the mirrored input window of its
 *   tile in shared memory (addressing the mirror, no embedded copy).  Each warp owns an (output row, band) item, keeps its
 *   256-bin window histogram in shared memory and slides it: per output the 32 lanes remove `height` pixels and add
 *   `height` pixels (shared atomics), then each lane clips and sums its 8 bins and two warp reductions give sum and
 *   sum_over, O(height / 32 + 8) per lane instead of the reference's O(height + 256).  A window whose staged tile does not
 *   fit in shared memory reads the input through the same mirror addressing from global memory.
 *
 * The per-window update, the per-lane partial sums and the per-element arithmetic are __host__ __device__ functions of
 * (lane, nlanes): vb200_debug_hist_local_host runs the very same code on the CPU, tile by tile, and
 * vb200_debug_hist_equal_lut_host the LUT arithmetic (tests/test_histogram.py, no GPU needed).
 */
#include <cstring>
#include <vector>

#include "vb200_internal.h"

namespace vb200 {

namespace {

/* ------------------------------------------------------------------ hist_find */

constexpr int kFindThreads = 256;
constexpr int kUcharBandsPerCta = 32;
constexpr int kUshortSlice = 32768;

struct FindDev {
	int w, h, bands, band; /* band: -1 every band, else the one scanned */
	size_t in_stride;	   /* elements per line */
	int nout;			   /* output bands: bands or 1 */
	int size;			   /* bins per output band: 256 or 65 536 */
	int slices;			   /* value slices per output band (ushort: 2) */
	int ob_per_part;	   /* output bands per grid row */
};

/* grid row `part`: output bands [ob0, ob0 + nob), values [v0, v0 + nv) */
__host__ __device__ __forceinline__ void
find_part(const FindDev &P, int part, int *ob0, int *nob, int *v0, int *nv)
{
	const int group = part / P.slices, slice = part - group * P.slices;
	*ob0 = group * P.ob_per_part;
	*nob = min(P.ob_per_part, P.nout - *ob0);
	*nv = P.size / P.slices;
	*v0 = slice * *nv;
}

template <typename T>
__global__ void __launch_bounds__(kFindThreads)
hist_find_kernel(const __grid_constant__ FindDev P, const T *__restrict__ in, unsigned *__restrict__ counts, unsigned *__restrict__ mx)
{
	extern __shared__ __align__(16) unsigned find_smem[];
	int ob0, nob, v0, nv;
	find_part(P, blockIdx.y, &ob0, &nob, &v0, &nv);
	for (int i = threadIdx.x; i < nob * nv; i += blockDim.x)
		find_smem[i] = 0;
	__syncthreads();
	unsigned vmax = 0;
	/* band -1: every element of the row, output band = input band; else pixel x's element `band` */
	const int per_row = P.band < 0 ? P.w * P.bands : P.w;
	for (int y = blockIdx.x; y < P.h; y += gridDim.x) {
		const T *row = in + (size_t) y * P.in_stride;
		for (int i = threadIdx.x; i < per_row; i += blockDim.x) {
			int ob, v;
			if (P.band < 0) {
				v = row[i];
				ob = i % P.bands;
			}
			else {
				v = row[(size_t) i * P.bands + P.band];
				ob = 0;
			}
			vmax = max(vmax, (unsigned) v);
			if (ob >= ob0 && ob < ob0 + nob && v >= v0 && v < v0 + nv)
				atomicAdd(&find_smem[(ob - ob0) * nv + (v - v0)], 1u);
		}
	}
	if (P.size == 256 && P.band < 0)
		vmax = 255; /* hist_find.c:361: a uchar histogram of every band is 256 wide whatever the data */
	vmax = __reduce_max_sync(0xffffffffu, vmax);
	if ((threadIdx.x & 31) == 0 && blockIdx.y == 0)
		atomicMax(mx, vmax);
	__syncthreads();
	for (int i = threadIdx.x; i < nob * nv; i += blockDim.x) {
		const unsigned c = find_smem[i];
		if (c) {
			const int ob = i / nv, v = i - ob * nv;
			atomicAdd(&counts[(size_t) (ob0 + ob) * P.size + v0 + v], c);
		}
	}
}

/* the reference's refusals that need the image (hist_find.c:147-162), in its order */
int
find_plan(const char *domain, const DevImage &in, int band, FindDev *P)
{
	if (band < -1 || band > in.bands - 1) {
		error(domain, "bandno must be -1, or less than %d", in.bands); /* iofuncs/error.c:1013-1023 */
		return -1;
	}
	if (in.fmt != VB200_FORMAT_UCHAR && in.fmt != VB200_FORMAT_USHORT) {
		error(domain, "band format %d not supported on the device path: cast to uchar or ushort first", in.fmt);
		return -1;
	}
	if ((uint64_t) in.w * (uint64_t) in.h >= ((uint64_t) 1 << 32)) {
		error(domain, "image of 2^32 or more pixels: its DOUBLE histogram is not built on the device path");
		return -1;
	}
	P->w = in.w;
	P->h = in.h;
	P->bands = in.bands;
	P->band = band;
	P->in_stride = in.bpl / format_sizeof(in.fmt);
	P->nout = band < 0 ? in.bands : 1;
	if (in.fmt == VB200_FORMAT_UCHAR) {
		P->size = 256;
		P->slices = 1;
		P->ob_per_part = kUcharBandsPerCta;
	}
	else {
		P->size = 65536;
		P->slices = 65536 / kUshortSlice;
		P->ob_per_part = 1;
	}
	return 0;
}

/* counts: nout x size uint32 (zeroed here), *mx: the largest value seen (uchar band -1: 255, hist_find.c:361) */
int
find_launch(const char *domain, const FindDev &P, const void *in, unsigned *counts, unsigned *mx, cudaStream_t s)
{
	VB200_CUDA(domain, cudaMemsetAsync(counts, 0, (size_t) P.nout * P.size * sizeof(unsigned), s));
	VB200_CUDA(domain, cudaMemsetAsync(mx, 0, sizeof(unsigned), s));
	const int groups = (P.nout + P.ob_per_part - 1) / P.ob_per_part;
	const int parts = groups * P.slices;
	const size_t smem = (size_t) std::min(P.ob_per_part, P.nout) * (P.size / P.slices) * sizeof(unsigned);
	/* enough CTAs per grid row to fill the machine; each walks its rows of the image */
	const int per_part = std::max(1, std::min(P.h, 4 * sm_count() / std::max(1, std::min(parts, 4))));
	const dim3 grid(per_part, std::min(parts, kMaxGridY));
	if (parts > kMaxGridY) {
		error(domain, "too many bands for the device path");
		return -1;
	}
	cudaError_t e;
	if (P.size == 256) {
		hist_find_kernel<uint8_t><<<grid, kFindThreads, smem, s>>>(P, (const uint8_t *) in, counts, mx);
		e = cudaGetLastError();
	}
	else {
		VB200_CUDA(domain, cudaFuncSetAttribute(hist_find_kernel<uint16_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
		hist_find_kernel<uint16_t><<<grid, kFindThreads, smem, s>>>(P, (const uint16_t *) in, counts, mx);
		e = cudaGetLastError();
	}
	if (e != cudaSuccess)
		return cuda_fail(domain, e, "hist_find_kernel");
	count_launch();
	return 0;
}

/* out: the (mx + 1) x 1 nout-band UINT histogram, bands interleaved (hist_find.c:184-200) */
__global__ void
hist_interleave_kernel(const unsigned *__restrict__ counts, int size, int nout, int width, unsigned *__restrict__ out)
{
	const size_t total = (size_t) width * nout;
	for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t) gridDim.x * blockDim.x) {
		const size_t j = i / nout, ob = i - j * nout;
		out[i] = counts[ob * size + j];
	}
}

/* ------------------------------------------------------------------ hist_equal: the LUT */

/* One LUT entry from the cumulative count c: hist_norm's linear (LOOP1(unsigned int, float)), its cast to uchar or ushort
 * and the cast to the input's format (hist_equal.c:87).  width: the histogram's width, total: its cumulative maximum.
 */
__host__ __device__ __forceinline__ unsigned
equal_lut_entry(unsigned c, int width, unsigned total)
{
	const unsigned long long new_max = (unsigned long long) width - 1;
	const double a = (double) new_max / (double) total;
	const float a1 = (float) a;
	const float q = a1 * (float) c + 0.0f;
	const double top = new_max <= 255 ? 255.0 : 65535.0; /* hist_norm.c:117-122: uchar, else ushort (new_max < 65 536) */
	const double v = (double) q;
	const double clipped = v < 0.0 ? 0.0 : (v > top ? top : v); /* VIPS_CLIP(0, (double) p, MAX), cast.c:231-239 */
	return (unsigned) clipped;
}

constexpr int kLutThreads = 1024;

/* one CTA per LUT band: the cumulative sum of counts[band][0 .. width) (hist_cum.c, unsigned int) and the LUT entries */
template <typename T>
__global__ void __launch_bounds__(kLutThreads)
hist_equal_lut_kernel(const unsigned *__restrict__ counts, int size, const unsigned *__restrict__ mx, T *__restrict__ lut)
{
	__shared__ unsigned partial[kLutThreads];
	__shared__ unsigned total_s;
	const int width = (int) *mx + 1;
	const unsigned *c = counts + (size_t) blockIdx.x * size;
	T *l = lut + (size_t) blockIdx.x * size;
	const int per = (width + blockDim.x - 1) / blockDim.x;
	const int i0 = threadIdx.x * per, i1 = min(width, i0 + per);
	unsigned run = 0;
	for (int i = i0; i < i1; i++)
		run += c[i];
	partial[threadIdx.x] = run;
	__syncthreads();
	/* exclusive prefix of the per-thread sums (Hillis-Steele over the CTA) */
	for (int off = 1; off < (int) blockDim.x; off <<= 1) {
		const unsigned v = threadIdx.x >= (unsigned) off ? partial[threadIdx.x - off] : 0u;
		__syncthreads();
		partial[threadIdx.x] += v;
		__syncthreads();
	}
	if (threadIdx.x == blockDim.x - 1)
		total_s = partial[threadIdx.x];
	__syncthreads();
	const unsigned total = total_s;
	unsigned acc = partial[threadIdx.x] - run;
	for (int i = i0; i < i1; i++) {
		acc += c[i];
		l[i] = (T) equal_lut_entry(acc, width, total);
	}
}

/* ------------------------------------------------------------------ maplut */

struct MapDev {
	int w, h, bands;
	int lut_bands; /* 1: one table for every band; else one per band */
	int lut_size;  /* entries per table in memory */
	size_t in_stride, out_stride; /* elements per line */
	int band_per_part;			  /* ushort n-band: grid z = band; 0: every band in one grid plane */
};

constexpr int kMapThreads = 256;
constexpr int kMapVec = 4;

template <typename T>
__global__ void __launch_bounds__(kMapThreads)
maplut_kernel(const __grid_constant__ MapDev P, const T *__restrict__ in, const T *__restrict__ lut, const unsigned *__restrict__ mx,
	T *__restrict__ out)
{
	extern __shared__ __align__(16) unsigned char map_smem[];
	T *tab = reinterpret_cast<T *>(map_smem);
	const unsigned clp = *mx; /* the LUT is mx + 1 wide: maplut.c:684-685 */
	const int zb = P.band_per_part ? (int) blockIdx.z : 0;
	const int ntab = P.band_per_part ? 1 : P.lut_bands;
	for (int i = threadIdx.x; i < ntab * (int) (clp + 1); i += blockDim.x) {
		const int t = i / (int) (clp + 1), v = i - t * (int) (clp + 1);
		tab[t * (clp + 1) + v] = lut[(size_t) (zb + t) * P.lut_size + v];
	}
	__syncthreads();
	const int row_elems = P.w * P.bands;
	for (int y = blockIdx.y; y < P.h; y += gridDim.y) {
		const T *p = in + (size_t) y * P.in_stride;
		T *q = out + (size_t) y * P.out_stride;
		if (P.band_per_part) {
			/* one band of this plane, its own table */
			for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < P.w; x += gridDim.x * blockDim.x) {
				const size_t e = (size_t) x * P.bands + zb;
				q[e] = tab[min((unsigned) p[e], clp)];
			}
			continue;
		}
		const bool vec = sizeof(T) == 1 && ((uintptr_t) p % kMapVec) == 0 && ((uintptr_t) q % kMapVec) == 0;
		const int e0 = (blockIdx.x * blockDim.x + threadIdx.x) * kMapVec;
		for (int e = e0; e < row_elems; e += gridDim.x * blockDim.x * kMapVec) {
			if (vec && e + kMapVec <= row_elems) {
				const uchar4 v = *reinterpret_cast<const uchar4 *>(p + e);
				const unsigned char vv[4] = {v.x, v.y, v.z, v.w};
				unsigned char r[4];
#pragma unroll
				for (int k = 0; k < 4; k++) {
					const int t = P.lut_bands == 1 ? 0 : (e + k) % P.bands;
					r[k] = (unsigned char) tab[t * (clp + 1) + min((unsigned) vv[k], clp)];
				}
				*reinterpret_cast<uchar4 *>(q + e) = make_uchar4(r[0], r[1], r[2], r[3]);
			}
			else
				for (int k = e; k < min(e + kMapVec, row_elems); k++) {
					const int t = P.lut_bands == 1 ? 0 : k % P.bands;
					q[k] = tab[t * (clp + 1) + min((unsigned) p[k], clp)];
				}
		}
	}
}

/* ------------------------------------------------------------------ hist_local */

constexpr int kLocalWarps = 16;
constexpr int kLocalThreads = kLocalWarps * 32;
constexpr int kLocalBins = 256;
constexpr int kLocalMaxArea = 8388607; /* (t + 1) * sum_over <= 256 * area must fit in int */
constexpr size_t kLocalMaxSmem = 160 * 1024;

struct LocalDev {
	int w, h, bands, rw, rh, max_slope;
	size_t in_stride, out_stride; /* elements per line */
	int tx, ty;					  /* output tile: columns x rows */
	int staged;					  /* 1: the tile's window is staged in shared memory */
	int tile_pitch;				  /* staged bytes per line: (tx + rw - 1) * bands */
	int tile_rows;				  /* ty + rh - 1 */
};

/* embed.c's VIPS_EXTEND_MIRROR: period 2n, the edge pixel repeated */
__host__ __device__ __forceinline__ int
mirror(int s, int n)
{
	const int n2 = 2 * n;
	int u = s % n2;
	if (u < 0)
		u += n2;
	return u < n ? u : n2 - 1 - u;
}

/* The mirrored input around output tile (bx, by): tile column ex, row ey is embedded pixel (bx * tx + ex, by * ty + ey),
 * i.e. input pixel (mirror(bx * tx + ex - rw / 2), mirror(by * ty + ey - rh / 2)).
 */
struct LocalSrc {
	const uint8_t *base; /* staged tile, or the input */
	int pitch;			 /* staged: tile_pitch */
	int x0, y0;			 /* unstaged: the tile's embedded origin minus the embed offset */
	int w, h, bands;
	size_t stride;
	bool staged;

	__host__ __device__ __forceinline__ int
	at(int ex, int ey, int b) const
	{
		if (staged)
			return base[(size_t) ey * pitch + (size_t) ex * bands + b];
		return base[(size_t) mirror(y0 + ey, h) * stride + (size_t) mirror(x0 + ex, w) * bands + b];
	}
};

__host__ __device__ __forceinline__ LocalSrc
local_src(const LocalDev &P, const uint8_t *in, const uint8_t *tile, int bx, int by)
{
	LocalSrc S;
	S.staged = P.staged != 0;
	S.base = S.staged ? tile : in;
	S.pitch = P.tile_pitch;
	S.x0 = bx * P.tx - P.rw / 2;
	S.y0 = by * P.ty - P.rh / 2;
	S.w = P.w;
	S.h = P.h;
	S.bands = P.bands;
	S.stride = P.in_stride;
	return S;
}

/* the staged window of tile (bx, by): thread tid of nthreads */
__host__ __device__ __forceinline__ void
local_stage(const LocalDev &P, const uint8_t *__restrict__ in, uint8_t *tile, int bx, int by, int tid, int nthreads)
{
	const int x0 = bx * P.tx - P.rw / 2, y0 = by * P.ty - P.rh / 2;
	const int total = P.tile_pitch * P.tile_rows;
	for (int i = tid; i < total; i += nthreads) {
		const int r = i / P.tile_pitch, e = i - r * P.tile_pitch;
		const int px = e / P.bands, b = e - px * P.bands;
		tile[i] = in[(size_t) mirror(y0 + r, P.h) * P.in_stride + (size_t) mirror(x0 + px, P.w) * P.bands + b];
	}
}

#ifdef __CUDA_ARCH__
#define LOCAL_ADD(P, V) atomicAdd((P), (V))
#else
#define LOCAL_ADD(P, V) (*(P) += (V))
#endif

/* the window histogram of band b for the output at tile column lx, tile row ly: lane's share of its rows */
__host__ __device__ __forceinline__ void
local_hist_init(const LocalDev &P, const LocalSrc &S, unsigned *hist, int lx, int ly, int b, int lane, int nlanes)
{
	for (int i = lane; i < P.rw * P.rh; i += nlanes) {
		const int j = i / P.rw, x = i - j * P.rw;
		LOCAL_ADD(&hist[S.at(lx + x, ly + j, b)], 1u);
	}
}

/* slide from output column lx to lx + 1: remove column lx, add column lx + rw (hist_local.c:254-262) */
__host__ __device__ __forceinline__ void
local_hist_slide(const LocalDev &P, const LocalSrc &S, unsigned *hist, int lx, int ly, int b, int lane, int nlanes)
{
	for (int j = lane; j < P.rh; j += nlanes) {
		LOCAL_ADD(&hist[S.at(lx, ly + j, b)], 0u - 1u);
		LOCAL_ADD(&hist[S.at(lx + P.rw, ly + j, b)], 1u);
	}
}

/* lane's share of the sums of hist_local.c:205-243: its bins lane * (256 / nlanes) ... */
__host__ __device__ __forceinline__ void
local_partial(const unsigned *hist, int target, int max_slope, int lane, int nlanes, int *sum, int *sum_over)
{
	const int per = kLocalBins / nlanes;
	int s = 0, o = 0;
	for (int k = 0; k < per; k++) {
		const int i = lane * per + k;
		const unsigned c = hist[i];
		if (max_slope > 0) {
			if (c > (unsigned) max_slope) {
				o += (int) (c - (unsigned) max_slope);
				if (i <= target)
					s += max_slope;
			}
			else if (i <= target)
				s += (int) c;
		}
		else if (i <= target)
			s += (int) c;
	}
	*sum = s;
	*sum_over = o;
}

/* the output element from the reduced sums (hist_local.c:237, :249) */
__host__ __device__ __forceinline__ uint8_t
local_finish(int sum, int sum_over, int target, int max_slope, int area)
{
	if (max_slope > 0)
		sum += (target + 1) * sum_over / 256;
	return (uint8_t) (255 * sum / area);
}

template <bool LOOP>
__global__ void __launch_bounds__(kLocalThreads)
hist_local_kernel(const __grid_constant__ LocalDev P, const uint8_t *__restrict__ in, uint8_t *__restrict__ out)
{
	extern __shared__ __align__(16) unsigned local_smem[];
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	unsigned *hist = local_smem + warp * kLocalBins;
	uint8_t *tile = reinterpret_cast<uint8_t *>(local_smem + kLocalWarps * kLocalBins);
	const int nby = (P.h + P.ty - 1) / P.ty;
	const int area = P.rw * P.rh;
	int by = blockIdx.y;
	do {
		if (P.staged) {
			if (by != (int) blockIdx.y)
				__syncthreads(); /* the previous tile has been read */
			local_stage(P, in, tile, blockIdx.x, by, threadIdx.x, blockDim.x);
			__syncthreads();
		}
		const LocalSrc S = local_src(P, in, tile, blockIdx.x, by);
		const int ncols = min(P.tx, P.w - (int) blockIdx.x * P.tx);
		const int nrows = min(P.ty, P.h - by * P.ty);
		/* items: (tile row, band), one per warp at a time */
		for (int item = warp; item < nrows * P.bands; item += kLocalWarps) {
			const int ly = item / P.bands, b = item - ly * P.bands;
			for (int i = lane; i < kLocalBins; i += 32)
				hist[i] = 0;
			__syncwarp();
			local_hist_init(P, S, hist, 0, ly, b, lane, 32);
			uint8_t *q = out + (size_t) (by * P.ty + ly) * P.out_stride + (size_t) blockIdx.x * P.tx * P.bands + b;
			for (int lx = 0; lx < ncols; lx++) {
				__syncwarp();
				const int target = S.at(lx + P.rw / 2, ly + P.rh / 2, b);
				int s, o;
				local_partial(hist, target, P.max_slope, lane, 32, &s, &o);
				s = __reduce_add_sync(0xffffffffu, s);
				o = __reduce_add_sync(0xffffffffu, o);
				if (lane == 0)
					q[(size_t) lx * P.bands] = local_finish(s, o, target, P.max_slope, area);
				if (lx + 1 < ncols) {
					__syncwarp();
					local_hist_slide(P, S, hist, lx, ly, b, lane, 32);
				}
			}
			__syncwarp();
		}
	} while (LOOP && (by += gridDim.y) < nby);
}

/* the reference's refusals (hist_local.c:288-297) and the tile geometry: 128 x 16 outputs, shrunk until the staged
 * window fits in shared memory, else read through the mirror from global memory
 */
int
local_plan(const char *domain, int w, int h, int bands, int fmt, int rw, int rh, int max_slope, LocalDev *P, size_t *smem)
{
	if (fmt != VB200_FORMAT_UCHAR) {
		error(domain, "image must be uchar"); /* vips_check_format, iofuncs/error.c:741-751 */
		return -1;
	}
	if (rw > w || rh > h) {
		error(domain, "window too large"); /* hist_local.c:292-297 */
		return -1;
	}
	P->w = w;
	P->h = h;
	P->bands = bands;
	P->rw = rw;
	P->rh = rh;
	P->max_slope = max_slope;
	const size_t hist_bytes = (size_t) kLocalWarps * kLocalBins * sizeof(unsigned);
	for (int tx = 128, ty = 16;;) {
		P->tx = tx;
		P->ty = ty;
		P->tile_pitch = (tx + rw - 1) * bands;
		P->tile_rows = ty + rh - 1;
		const size_t tile = (size_t) P->tile_pitch * P->tile_rows;
		if (hist_bytes + tile <= kLocalMaxSmem) {
			P->staged = 1;
			*smem = hist_bytes + tile;
			return 0;
		}
		if (ty > 1)
			ty /= 2;
		else if (tx > 32)
			tx /= 2;
		else
			break;
	}
	P->tx = 128;
	P->ty = 16;
	P->staged = 0;
	P->tile_pitch = 0;
	P->tile_rows = 0;
	*smem = hist_bytes;
	return 0;
}

} // namespace

/* the refusals of the op's constructor: no image needed */
int
hist_local_check(const char *domain, int width, int height, int max_slope)
{
	if (width < 1 || height < 1) {
		error(domain, "window too large"); /* the arguments' range is 1 ... (hist_local.c:363-375) */
		return -1;
	}
	if ((long long) width * height > kLocalMaxArea) {
		error(domain, "window of %d x %d pixels: 255 * sum overflows int beyond %d pixels", width, height, kLocalMaxArea);
		return -1;
	}
	if (max_slope < 0) {
		error(domain, "max_slope should be >= 0");
		return -1;
	}
	return 0;
}

/* the refusals that need the image's descriptor but no pixels: the stand-alone call makes them before the upload */
int
hist_refuse(const char *domain, int kind, int w, int h, int bands, int fmt, int band, int width, int height)
{
	DevImage d;
	d.w = w;
	d.h = h;
	d.bands = bands;
	d.fmt = fmt;
	d.bpl = (size_t) w * bands * format_sizeof(fmt);
	if (kind == 2) {
		LocalDev P;
		size_t smem;
		return local_plan(domain, w, h, bands, fmt, width, height, 0, &P, &smem);
	}
	FindDev P;
	return find_plan(domain, d, band, &P);
}

int
dev_hist_find(const char *domain, const DevImage &in, DevImage *out, int band, cudaStream_t s)
{
	FindDev P;
	if (find_plan(domain, in, band, &P))
		return -1;
	void *scratch = nullptr;
	const size_t counts_bytes = (size_t) P.nout * P.size * sizeof(unsigned);
	if (dev_alloc(domain, &scratch, counts_bytes + sizeof(unsigned), s))
		return -1;
	unsigned *counts = (unsigned *) scratch, *mx = counts + (size_t) P.nout * P.size;
	int rc = find_launch(domain, P, in.data, counts, mx, s);
	/* the output's width is data: the one host sync of this op */
	unsigned mx_h = 0;
	if (!rc && cudaMemcpyAsync(&mx_h, mx, sizeof(unsigned), cudaMemcpyDeviceToHost, s) != cudaSuccess)
		rc = cuda_fail(domain, cudaGetLastError(), "hist_find max");
	if (!rc && cudaStreamSynchronize(s) != cudaSuccess)
		rc = cuda_fail(domain, cudaGetLastError(), "hist_find sync");
	if (!rc)
		rc = dev_image_new(domain, out, (int) mx_h + 1, 1, P.nout, VB200_FORMAT_UINT, VB200_INTERPRETATION_HISTOGRAM, s);
	if (!rc) {
		const int n = (int) (((size_t) (mx_h + 1) * P.nout + 255) / 256);
		hist_interleave_kernel<<<std::min(n, 4096), 256, 0, s>>>(counts, P.size, P.nout, (int) mx_h + 1, (unsigned *) out->data);
		cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess)
			rc = cuda_fail(domain, e, "hist_interleave_kernel");
		else
			count_launch();
	}
	dev_free(scratch, s);
	return rc;
}

int
dev_hist_equal(const char *domain, const DevImage &in, DevImage *out, int band, cudaStream_t s)
{
	FindDev P;
	if (find_plan(domain, in, band, &P))
		return -1;
	const size_t es = format_sizeof(in.fmt);
	const size_t counts_bytes = (size_t) P.nout * P.size * sizeof(unsigned);
	const size_t lut_bytes = (size_t) P.nout * P.size * es;
	void *scratch = nullptr;
	if (dev_alloc(domain, &scratch, counts_bytes + lut_bytes + 16, s))
		return -1;
	unsigned *counts = (unsigned *) scratch;
	unsigned char *lut = (unsigned char *) scratch + counts_bytes;
	unsigned *mx = (unsigned *) ((unsigned char *) scratch + counts_bytes + ((lut_bytes + 3) & ~(size_t) 3));
	int rc = find_launch(domain, P, in.data, counts, mx, s);
	if (!rc) {
		if (es == 1)
			hist_equal_lut_kernel<uint8_t><<<P.nout, kLutThreads, 0, s>>>(counts, P.size, mx, (uint8_t *) lut);
		else
			hist_equal_lut_kernel<uint16_t><<<P.nout, kLutThreads, 0, s>>>(counts, P.size, mx, (uint16_t *) lut);
		cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess)
			rc = cuda_fail(domain, e, "hist_equal_lut_kernel");
		else
			count_launch();
	}
	if (!rc)
		rc = dev_image_new(domain, out, in.w, in.h, in.bands, in.fmt, in.type, s);
	if (!rc) {
		MapDev M;
		M.w = in.w;
		M.h = in.h;
		M.bands = in.bands;
		M.lut_bands = P.nout;
		M.lut_size = P.size;
		M.in_stride = in.bpl / es;
		M.out_stride = out->bpl / es;
		/* every table fits in shared memory but a ushort one per band: then one grid plane per band */
		M.band_per_part = (es == 2 && P.nout > 1) ? 1 : 0;
		const size_t smem = (M.band_per_part ? 1 : (size_t) P.nout) * P.size * es;
		const int planes = M.band_per_part ? in.bands : 1;
		const int row_elems = M.band_per_part ? in.w : in.w * in.bands;
		const int per_cta = kMapThreads * (M.band_per_part ? 1 : kMapVec);
		/* the table is loaded once per CTA: a few CTAs per SM walk the rows */
		const int gx = (row_elems + per_cta - 1) / per_cta;
		const int gy = std::max(1, std::min({in.h, kMaxGridY, 4 * sm_count() / std::max(1, gx * planes)}));
		dim3 grid(gx, gy, planes);
		if (planes > kMaxGridY) {
			error(domain, "too many bands for the device path");
			rc = -1;
		}
		else if (smem > 200 * 1024) {
			error(domain, "%d-band LUT too large for the device path", P.nout);
			rc = -1;
		}
		else {
			cudaError_t e;
			if (es == 1) {
				if (smem > 48 * 1024)
					cudaFuncSetAttribute(maplut_kernel<uint8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
				maplut_kernel<uint8_t><<<grid, kMapThreads, smem, s>>>(M, (const uint8_t *) in.data, (const uint8_t *) lut, mx,
					(uint8_t *) out->data);
			}
			else {
				cudaFuncSetAttribute(maplut_kernel<uint16_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
				maplut_kernel<uint16_t><<<grid, kMapThreads, smem, s>>>(M, (const uint16_t *) in.data, (const uint16_t *) lut, mx,
					(uint16_t *) out->data);
			}
			e = cudaGetLastError();
			if (e != cudaSuccess)
				rc = cuda_fail(domain, e, "maplut_kernel");
			else
				count_launch();
		}
	}
	dev_free(scratch, s);
	return rc;
}

int
dev_hist_local(const char *domain, const DevImage &in, DevImage *out, int width, int height, int max_slope, cudaStream_t s)
{
	LocalDev P;
	size_t smem = 0;
	if (local_plan(domain, in.w, in.h, in.bands, in.fmt, width, height, max_slope, &P, &smem))
		return -1;
	if (dev_image_new(domain, out, in.w, in.h, in.bands, in.fmt, in.type, s))
		return -1;
	P.in_stride = in.bpl;
	P.out_stride = out->bpl;
	const int nby = (P.h + P.ty - 1) / P.ty;
	auto kern = rows_loop(nby) ? hist_local_kernel<true> : hist_local_kernel<false>;
	if (smem > 48 * 1024)
		VB200_CUDA(domain, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
	const dim3 grid = row_grid(P.w, nby, P.tx);
	kern<<<grid, kLocalThreads, smem, s>>>(P, (const uint8_t *) in.data, (uint8_t *) out->data);
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
		return cuda_fail(domain, e, "hist_local_kernel");
	count_launch();
	return 0;
}

} // namespace vb200

using namespace vb200;

/* test hook, host only: the kernel's staging, window update, lane sums and per-element arithmetic run tile by tile on
 * the CPU over packed host arrays, 32 "lanes" per window as a warp has.  staged: -1 the plan's choice, 0 / 1 forced.
 */
extern "C" int
vb200_debug_hist_local_host(const void *in, int width, int height, int bands, int rank_width, int rank_height, int max_slope,
	int staged, void *out)
{
	const char *domain = "hist_local";
	LocalDev P;
	size_t smem = 0;
	if (!in || !out || bands < 1) {
		error(domain, "null argument");
		return -1;
	}
	if (hist_local_check(domain, rank_width, rank_height, max_slope) ||
		local_plan(domain, width, height, bands, VB200_FORMAT_UCHAR, rank_width, rank_height, max_slope, &P, &smem))
		return -1;
	if (staged >= 0) {
		P.staged = staged;
		P.tile_pitch = (P.tx + P.rw - 1) * bands;
		P.tile_rows = P.ty + P.rh - 1;
	}
	P.in_stride = P.out_stride = (size_t) width * bands;
	const uint8_t *src = (const uint8_t *) in;
	uint8_t *dst = (uint8_t *) out;
	std::vector<uint8_t> tile(P.staged ? (size_t) P.tile_pitch * P.tile_rows : 1);
	std::vector<unsigned> hist(kLocalBins);
	const int area = P.rw * P.rh;
	for (int by = 0; by < (P.h + P.ty - 1) / P.ty; by++)
		for (int bx = 0; bx < (P.w + P.tx - 1) / P.tx; bx++) {
			if (P.staged)
				for (int t = 0; t < 7; t++)
					local_stage(P, src, tile.data(), bx, by, t, 7);
			const LocalSrc S = local_src(P, src, tile.data(), bx, by);
			const int ncols = std::min(P.tx, P.w - bx * P.tx), nrows = std::min(P.ty, P.h - by * P.ty);
			for (int item = 0; item < nrows * bands; item++) {
				const int ly = item / bands, b = item - ly * bands;
				std::fill(hist.begin(), hist.end(), 0u);
				for (int l = 0; l < 32; l++)
					local_hist_init(P, S, hist.data(), 0, ly, b, l, 32);
				uint8_t *q = dst + (size_t) (by * P.ty + ly) * P.out_stride + (size_t) bx * P.tx * bands + b;
				for (int lx = 0; lx < ncols; lx++) {
					const int target = S.at(lx + P.rw / 2, ly + P.rh / 2, b);
					int s = 0, o = 0;
					for (int l = 0; l < 32; l++) {
						int ls, lo;
						local_partial(hist.data(), target, P.max_slope, l, 32, &ls, &lo);
						s += ls;
						o += lo;
					}
					q[(size_t) lx * bands] = local_finish(s, o, target, P.max_slope, area);
					if (lx + 1 < ncols)
						for (int l = 0; l < 32; l++)
							local_hist_slide(P, S, hist.data(), lx, ly, b, l, 32);
				}
			}
		}
	return 0;
}

/* test hook, host only: hist_equal's LUT from a histogram (n_bands x width uint32, band-major), through the device's own
 * per-entry arithmetic; lut: n_bands x width entries of the input's format (uchar or ushort)
 */
extern "C" int
vb200_debug_hist_equal_lut_host(const unsigned *hist, int width, int n_bands, int band_format, void *lut)
{
	if (!hist || !lut || width < 1 || n_bands < 1 || (band_format != VB200_FORMAT_UCHAR && band_format != VB200_FORMAT_USHORT)) {
		error("hist_equal", "bad argument");
		return -1;
	}
	for (int b = 0; b < n_bands; b++) {
		const unsigned *c = hist + (size_t) b * width;
		unsigned total = 0;
		for (int i = 0; i < width; i++)
			total += c[i];
		unsigned acc = 0;
		for (int i = 0; i < width; i++) {
			acc += c[i];
			const unsigned v = equal_lut_entry(acc, width, total);
			if (band_format == VB200_FORMAT_UCHAR)
				((uint8_t *) lut)[(size_t) b * width + i] = (uint8_t) v;
			else
				((uint16_t *) lut)[(size_t) b * width + i] = (uint16_t) v;
		}
	}
	return 0;
}
