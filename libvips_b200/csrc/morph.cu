/* morph.cu -- vips_morph (binary erode / dilate) on the device, SURVEY 8f rank 4.
 *
 * reference: morphology/morph.c:657-739 (vips_dilate_gen), :744-826 (vips_erode_gen), :829-935 (build);
 * the Highway kernels morph_hwy.cpp compute the same bytes.  Per element
 *     dilate: OR  over the mask's non-128 elements of (coeff ? p : ~p)
 *     erode:  AND over them
 * on the image embedded by the mask with VIPS_EXTEND_COPY (clamp addressing here).  One thread per
 * output element, the mask's live elements as a {dx, dy, coeff} list; neighbouring threads read
 * neighbouring bytes, the window stays in L1.  (First version: correct and coalesced, not yet tuned --
 * the ops are bitwise, so a word-per-thread form with funnel shifts is the obvious next step.)
 * Algorithmic bytes: w * h * bands in + the same out.
 */
#include <cmath>
#include <cstring>
#include <vector>

#include "vb200_internal.h"

namespace vb200 {

namespace {

constexpr int kMaxMorph = 1024; /* mask elements that take part (e.g. 31 x 31) */

struct MorphDev {
	int w, h, bands, n;
	size_t in_bpl, out_bpl;
	const int *taps; /* n x {dx, dy, coeff} */
};

template <bool DILATE>
__global__ void __launch_bounds__(256)
morph_kernel(const __grid_constant__ MorphDev P, const uint8_t *__restrict__ in, uint8_t *__restrict__ out)
{
	const int e = blockIdx.x * blockDim.x + threadIdx.x; /* element (byte) of the row */
	const int ne = P.w * P.bands;
	if (e >= ne)
		return;
	const int x = e / P.bands, b = e - x * P.bands;
	for (int y = blockIdx.y; y < P.h; y += gridDim.y) {
		int result = DILATE ? 0 : 255;
		for (int i = 0; i < P.n; i++) {
			const int dx = __ldg(P.taps + 3 * i), dy = __ldg(P.taps + 3 * i + 1), co = __ldg(P.taps + 3 * i + 2);
			const int sx = max(0, min(x + dx, P.w - 1)), sy = max(0, min(y + dy, P.h - 1));
			const int p = in[(size_t) sy * P.in_bpl + (size_t) sx * P.bands + b];
			const int v = co ? p : ~p;
			result = DILATE ? (result | v) : (result & v);
		}
		out[(size_t) y * P.out_bpl + e] = (uint8_t) result;
	}
}

} // namespace

int
dev_morph(const char *domain, const DevImage &in, DevImage *out, const double *mask, int mw, int mh, int op, cudaStream_t s)
{
	if (in.fmt != VB200_FORMAT_UCHAR) {
		/* the reference casts to uchar first (morph.c:868); only uchar images are on the device path */
		error(domain, "band format %d not supported on the device path", in.fmt);
		return -1;
	}
	if (!mask || mw <= 0 || mh <= 0) {
		error(domain, "bad mask");
		return -1;
	}
	if (op != 0 && op != 1) {
		error(domain, "bad morphology operation %d", op);
		return -1;
	}
	std::vector<int> taps;
	for (int y = 0; y < mh; y++)
		for (int x = 0; x < mw; x++) {
			const double c = rint(mask[y * mw + x]); /* vips__image_intize */
			if (c != 0 && c != 128 && c != 255) {
				error(domain, "bad mask element (%f should be 0, 128 or 255)", c);
				return -1;
			}
			if (c == 128)
				continue;
			taps.push_back(x - mw / 2);
			taps.push_back(y - mh / 2);
			taps.push_back((int) c);
		}
	const int n = (int) taps.size() / 3;
	if (n > kMaxMorph) {
		error(domain, "mask too large for the device path");
		return -1;
	}
	void *dt = nullptr;
	if (dev_alloc(domain, &dt, std::max<size_t>(taps.size() * sizeof(int), 16), s))
		return -1;
	if (n && cudaMemcpyAsync(dt, taps.data(), taps.size() * sizeof(int), cudaMemcpyHostToDevice, s) != cudaSuccess) {
		dev_free(dt, s);
		return cuda_fail(domain, cudaGetLastError(), "morph mask upload");
	}
	if (dev_image_new(domain, out, in.w, in.h, in.bands, in.fmt, in.type, s)) {
		dev_free(dt, s);
		return -1;
	}
	MorphDev P;
	P.w = in.w;
	P.h = in.h;
	P.bands = in.bands;
	P.n = n;
	P.in_bpl = in.bpl;
	P.out_bpl = out->bpl;
	P.taps = (const int *) dt;
	const dim3 grid = row_grid(in.w * in.bands, in.h);
	if (op)
		morph_kernel<true><<<grid, 256, 0, s>>>(P, (const uint8_t *) in.data, (uint8_t *) out->data);
	else
		morph_kernel<false><<<grid, 256, 0, s>>>(P, (const uint8_t *) in.data, (uint8_t *) out->data);
	cudaError_t e = cudaGetLastError();
	cudaStreamSynchronize(s); /* the pageable upload above reads `taps` */
	dev_free(dt, s);
	if (e != cudaSuccess)
		return cuda_fail(domain, e, "morph_kernel");
	count_launch();
	return 0;
}

} // namespace vb200
