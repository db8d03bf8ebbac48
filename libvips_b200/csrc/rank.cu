/* rank.cu -- vips_rank / vips_median on the device, SURVEY 8f rank 4.
 *
 * reference: morphology/rank.c:458-525 (vips_rank_build: window within the image, 0 <= index < n, embed at
 * (width / 2, height / 2) with VIPS_EXTEND_COPY), :414-456 (vips_rank_generate), and its four inner loops -- uchar
 * histogram :165-232, Numerical-Recipes select :236-323, max :327-352, min :356-381.  All four return the same
 * thing, the index-th smallest element of the width x height window of every band, which is what is computed here.
 *
 * One CTA stages the (TX + width - 1) x (TY + height - 1) pixel window of a TX x TY output tile into shared memory,
 * edge pixels replicated while staging (the embed), elements stored as order-preserving unsigned keys (signed
 * integers with the sign bit flipped, floats with the usual sign-magnitude fold).  Each thread then owns output
 * elements of the tile.  min / max walk the window once; every other index is a radix select on the keys, most
 * significant bit first: with `res` the bits decided so far, count the window's keys <= res | (2^bit - 1); if that
 * is at most index, the bit is set.  BITS passes over the window, no data-dependent branches, no scratch per thread
 * (the reference's sort array), and the same loop for every format.
 * Algorithmic bytes: w * h * bands * sizeof(element), in and out.
 *
 * The tile staging and the per-element select are __host__ __device__ functions of (tid, nthreads):
 * vb200_debug_rank_host runs the very same code on the CPU, tile by tile (tests/test_widen_rank.py, no GPU needed).
 * Floats: NaNs order by their bit patterns (the reference's comparisons leave their place undefined); -0 < +0.
 */
#include <cstring>
#include <vector>

#include "vb200_internal.h"

namespace vb200 {

namespace {

struct RankDev {
	int w, h, bands, rw, rh, index;
	size_t in_stride, out_stride; /* elements per line */
	int tx, ty;					  /* output tile, pixels x rows */
	int tile_stride;			  /* elements per staged line: (tx + rw - 1) * bands */
	int tile_rows;				  /* ty + rh - 1 */
};

template <typename T> struct RankTraits;
template <> struct RankTraits<uint8_t> { typedef uint8_t Key; static constexpr int bits = 8; static constexpr unsigned flip = 0; };
template <> struct RankTraits<int8_t> { typedef uint8_t Key; static constexpr int bits = 8; static constexpr unsigned flip = 0x80u; };
template <> struct RankTraits<uint16_t> { typedef uint16_t Key; static constexpr int bits = 16; static constexpr unsigned flip = 0; };
template <> struct RankTraits<int16_t> { typedef uint16_t Key; static constexpr int bits = 16; static constexpr unsigned flip = 0x8000u; };
template <> struct RankTraits<uint32_t> { typedef uint32_t Key; static constexpr int bits = 32; static constexpr unsigned flip = 0; };
template <> struct RankTraits<int32_t> { typedef uint32_t Key; static constexpr int bits = 32; static constexpr unsigned flip = 0x80000000u; };
template <> struct RankTraits<float> { typedef uint32_t Key; static constexpr int bits = 32; };

template <typename T>
__host__ __device__ __forceinline__ typename RankTraits<T>::Key
rank_key(T v)
{
	typename RankTraits<T>::Key k;
	memcpy(&k, &v, sizeof(k));
	return (typename RankTraits<T>::Key)(k ^ RankTraits<T>::flip);
}
template <>
__host__ __device__ __forceinline__ uint32_t
rank_key<float>(float v)
{
	uint32_t k;
	memcpy(&k, &v, sizeof(k));
	return (k & 0x80000000u) ? ~k : (k | 0x80000000u);
}

template <typename T>
__host__ __device__ __forceinline__ T
rank_unkey(typename RankTraits<T>::Key k)
{
	k = (typename RankTraits<T>::Key)(k ^ RankTraits<T>::flip);
	T v;
	memcpy(&v, &k, sizeof(v));
	return v;
}
template <>
__host__ __device__ __forceinline__ float
rank_unkey<float>(uint32_t k)
{
	k = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
	float v;
	memcpy(&v, &k, sizeof(v));
	return v;
}

__host__ __device__ __forceinline__ int
rank_clamp(int v, int hi)
{
	return v < 0 ? 0 : (v > hi ? hi : v);
}

/* the window of output tile (bx, by), keyed, edges replicated: thread tid of nthreads */
template <typename T>
__host__ __device__ __forceinline__ void
rank_stage(const RankDev &P, const T *__restrict__ in, typename RankTraits<T>::Key *tile, int bx, int by, int tid, int nthreads)
{
	const int x0 = bx * P.tx - P.rw / 2, y0 = by * P.ty - P.rh / 2;
	const int total = P.tile_stride * P.tile_rows;
	for (int i = tid; i < total; i += nthreads) {
		const int r = i / P.tile_stride, e = i - r * P.tile_stride;
		const int px = e / P.bands, b = e - px * P.bands;
		const int sx = rank_clamp(x0 + px, P.w - 1), sy = rank_clamp(y0 + r, P.h - 1);
		tile[i] = rank_key<T>(in[(size_t) sy * P.in_stride + (size_t) sx * P.bands + b]);
	}
}

/* the output elements of tile (bx, by) this thread owns */
template <typename T>
__host__ __device__ __forceinline__ void
rank_select(const RankDev &P, const typename RankTraits<T>::Key *tile, T *__restrict__ out, int bx, int by, int tid, int nthreads)
{
	typedef typename RankTraits<T>::Key Key;
	const int row_elems = P.tx * P.bands;
	const int total = row_elems * P.ty;
	const int n = P.rw * P.rh;
	for (int o = tid; o < total; o += nthreads) {
		const int r = o / row_elems, e = o - r * row_elems;
		const int x = bx * P.tx + e / P.bands, y = by * P.ty + r;
		if (x >= P.w || y >= P.h)
			continue;
		const Key *win = tile + (size_t) r * P.tile_stride + e;
		Key res;
		if (P.index == 0 || P.index == n - 1) {
			const bool want_max = P.index != 0; /* n == 1: either */
			res = win[0];
			for (int j = 0; j < P.rh; j++)
				for (int i = 0; i < P.rw; i++) {
					const Key k = win[j * P.tile_stride + i * P.bands];
					res = want_max ? (k > res ? k : res) : (k < res ? k : res);
				}
		}
		else {
			unsigned acc = 0;
			for (int bit = RankTraits<T>::bits - 1; bit >= 0; bit--) {
				const unsigned t = acc | ((1u << bit) - 1u);
				int count = 0;
				for (int j = 0; j < P.rh; j++)
					for (int i = 0; i < P.rw; i++)
						count += (unsigned) win[j * P.tile_stride + i * P.bands] <= t;
				if (count <= P.index)
					acc |= 1u << bit;
			}
			res = (Key) acc;
		}
		out[(size_t) y * P.out_stride + (size_t) bx * row_elems + e] = rank_unkey<T>(res);
	}
}

template <typename T, bool LOOP>
__global__ void __launch_bounds__(256)
rank_kernel(const __grid_constant__ RankDev P, const T *__restrict__ in, T *__restrict__ out)
{
	extern __shared__ __align__(16) unsigned char rank_smem[];
	typename RankTraits<T>::Key *tile = reinterpret_cast<typename RankTraits<T>::Key *>(rank_smem);
	/* the whole CTA walks its rows of tiles together through the staged window */
	int by = blockIdx.y;
	do {
		if (by != (int) blockIdx.y)
			__syncthreads(); /* the previous tile has been read */
		rank_stage<T>(P, in, tile, blockIdx.x, by, threadIdx.x, blockDim.x);
		__syncthreads();
		rank_select<T>(P, tile, out, blockIdx.x, by, threadIdx.x, blockDim.x);
	} while (LOOP && (by += gridDim.y) < (P.h + P.ty - 1) / P.ty);
}

constexpr size_t kRankMaxSmem = 200 * 1024;

/* tile geometry: 32 x 8 pixels, shrunk until the staged window fits in shared memory */
int
rank_plan(const char *domain, int w, int h, int bands, int fmt, int rw, int rh, int index, RankDev *P, size_t *smem)
{
	if (rw < 1 || rh < 1 || rw > w || rh > h) {
		error(domain, "window too large"); /* rank.c:478-483 */
		return -1;
	}
	if (index < 0 || index > rw * rh - 1) {
		error(domain, "index out of range"); /* rank.c:485-489 */
		return -1;
	}
	if (fmt < VB200_FORMAT_UCHAR || fmt > VB200_FORMAT_FLOAT) {
		error(domain, "band format %d not supported on the device path", fmt);
		return -1;
	}
	P->w = w;
	P->h = h;
	P->bands = bands;
	P->rw = rw;
	P->rh = rh;
	P->index = index;
	const size_t es = format_sizeof(fmt);
	for (int tx = 32, ty = 8;;) {
		P->tx = tx;
		P->ty = ty;
		P->tile_stride = (tx + rw - 1) * bands;
		P->tile_rows = ty + rh - 1;
		*smem = (size_t) P->tile_stride * P->tile_rows * es;
		if (*smem <= kRankMaxSmem)
			return 0;
		if (ty > 1)
			ty /= 2;
		else if (tx > 1)
			tx /= 2;
		else
			break;
	}
	error(domain, "window too large for the device path");
	return -1;
}

template <typename T>
int
rank_launch(const char *domain, const RankDev &P, size_t smem, const void *in, void *out, cudaStream_t s)
{
	auto kern = rows_loop((P.h + P.ty - 1) / P.ty) ? rank_kernel<T, true> : rank_kernel<T, false>;
	if (smem > 48 * 1024)
		VB200_CUDA(domain, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
	const dim3 grid = row_grid(P.w, (P.h + P.ty - 1) / P.ty, P.tx);
	kern<<<grid, 256, smem, s>>>(P, (const T *) in, (T *) out);
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
		return cuda_fail(domain, e, "rank_kernel");
	count_launch();
	return 0;
}

template <typename T>
void
rank_host(const RankDev &P, const void *in, void *out)
{
	std::vector<typename RankTraits<T>::Key> tile((size_t) P.tile_stride * P.tile_rows);
	for (int by = 0; by < (P.h + P.ty - 1) / P.ty; by++)
		for (int bx = 0; bx < (P.w + P.tx - 1) / P.tx; bx++) {
			/* 7 "threads", as the kernel's 256 would: strided ownership */
			for (int t = 0; t < 7; t++)
				rank_stage<T>(P, (const T *) in, tile.data(), bx, by, t, 7);
			for (int t = 0; t < 7; t++)
				rank_select<T>(P, tile.data(), (T *) out, bx, by, t, 7);
		}
}

#define RANK_SWITCH(FMT, CALL) \
	switch (FMT) { \
	case VB200_FORMAT_UCHAR: CALL(uint8_t); break; \
	case VB200_FORMAT_CHAR: CALL(int8_t); break; \
	case VB200_FORMAT_USHORT: CALL(uint16_t); break; \
	case VB200_FORMAT_SHORT: CALL(int16_t); break; \
	case VB200_FORMAT_UINT: CALL(uint32_t); break; \
	case VB200_FORMAT_INT: CALL(int32_t); break; \
	default: CALL(float); break; \
	}

} // namespace

int
dev_rank(const char *domain, const DevImage &in, DevImage *out, int width, int height, int index, cudaStream_t s)
{
	RankDev P;
	size_t smem = 0;
	if (rank_plan(domain, in.w, in.h, in.bands, in.fmt, width, height, index, &P, &smem))
		return -1;
	if (dev_image_new(domain, out, in.w, in.h, in.bands, in.fmt, in.type, s))
		return -1;
	const size_t es = format_sizeof(in.fmt);
	P.in_stride = in.bpl / es;
	P.out_stride = out->bpl / es;
	int rc = 0;
#define CALL(T) rc = rank_launch<T>(domain, P, smem, in.data, out->data, s)
	RANK_SWITCH(in.fmt, CALL)
#undef CALL
	return rc;
}

} // namespace vb200

using namespace vb200;

/* test hook, host only: the kernel's staging and select code run tile by tile on the CPU over packed host arrays */
extern "C" int
vb200_debug_rank_host(const void *in, int width, int height, int bands, int band_format, int rank_width, int rank_height, int index,
	void *out)
{
	const char *domain = "rank";
	RankDev P;
	size_t smem = 0;
	if (!in || !out || bands < 1) {
		error(domain, "null argument");
		return -1;
	}
	if (rank_plan(domain, width, height, bands, band_format, rank_width, rank_height, index, &P, &smem))
		return -1;
	P.in_stride = P.out_stride = (size_t) width * bands;
#define CALL(T) rank_host<T>(P, in, out)
	RANK_SWITCH(band_format, CALL)
#undef CALL
	return 0;
}
