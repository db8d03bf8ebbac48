/* api_resample.cu -- the resample family's region and scanline seams: the generate()-shaped
 * vb200_*_gen entry points and the reference's Highway kernel signatures (the whole-image
 * entry points are in image_ops.cu).
 */
#include <algorithm>
#include <cmath>
#include <cstring>

#include "vb200_internal.h"
#include "vb200_vips_abi.h"

using namespace vb200;

/* ------------------------------------------------------ generate()-shaped */

namespace {

struct StagedRegion {
	void *dev = nullptr;
	size_t bpl = 0;
	size_t line = 0;
};

int
stage_in(const char *domain, const VB200Region *r, StagedRegion *st, cudaStream_t s)
{
	const size_t ps = format_sizeof(r->im.BandFmt) * r->im.Bands;
	st->line = ps * r->valid.width;
	st->bpl = st->line;
	if (dev_alloc(domain, &st->dev, st->line * r->valid.height, s))
		return -1;
	VB200_CUDA(domain, cudaMemcpy2DAsync(st->dev, st->bpl, r->data, r->bpl, st->line, r->valid.height,
						   cudaMemcpyHostToDevice, s));
	return 0;
}

int
stage_out(const char *domain, const VB200Region *r, StagedRegion *st, cudaStream_t s)
{
	VB200_CUDA(domain, cudaMemcpy2DAsync(r->data, r->bpl, st->dev, st->bpl, st->line, r->valid.height,
						   cudaMemcpyDeviceToHost, s));
	VB200_CUDA(domain, cudaStreamSynchronize(s));
	return 0;
}

int
check_regions(const char *domain, const VB200Region *out, const VB200Region *in)
{
	if (!out || !in || !out->data || !in->data) {
		error(domain, "null region");
		return -1;
	}
	if (!format_is_supported(in->im.BandFmt)) {
		error(domain, "band format %d not supported on the device path", in->im.BandFmt);
		return -1;
	}
	return ensure_init(domain);
}

} // namespace

extern "C" int
vb200_reducev_gen(const VB200Region *out, const VB200Region *in, const VB200ReduceParams *p)
{
	const char *domain = "reducev_gen";
	if (check_regions(domain, out, in))
		return -1;
	const VB200Rect *r = &out->valid;
	/* the rows the reference would prepare: reducev.cpp:539-544 */
	AxisTable t;
	build_axis_table(t, 0, p->residual_shrink, p->offset, p->n_point, p->kernel, 0, r->top, r->height);
	const int need_top = t.first[0];
	const int need_bottom = t.first[r->height - 1] + p->n_point;
	if (in->valid.left > r->left || in->valid.left + in->valid.width < r->left + r->width ||
		in->valid.top > need_top || in->valid.top + in->valid.height < need_bottom) {
		error(domain, "input region does not cover rows %d..%d of the embedded image", need_top, need_bottom);
		return -1;
	}
	cudaStream_t s = current_stream();
	StagedRegion si, so;
	if (stage_in(domain, in, &si, s))
		return -1;
	const size_t ps = format_sizeof(in->im.BandFmt) * in->im.Bands;
	so.line = so.bpl = ps * r->width;
	if (dev_alloc(domain, &so.dev, so.line * r->height, s))
		return -1;
	/* The region is on the EMBEDDED image: taps never clamp.  Shift the table
	 * into region-local rows and neutralise the embed offset.
	 */
	for (auto &f : t.first)
		f -= in->valid.top;
	t.embed = 0;
	const char *src = (const char *) si.dev + (size_t) (r->left - in->valid.left) * ps;
	int rc = launch_reducev(domain, src, si.bpl, in->valid.height, so.dev, so.bpl, r->width * in->im.Bands,
		r->height, in->im.BandFmt, t, s);
	if (!rc)
		rc = stage_out(domain, out, &so, s);
	dev_free(si.dev, s);
	dev_free(so.dev, s);
	return rc;
}

extern "C" int
vb200_reduceh_gen(const VB200Region *out, const VB200Region *in, const VB200ReduceParams *p)
{
	const char *domain = "reduceh_gen";
	if (check_regions(domain, out, in))
		return -1;
	const VB200Rect *r = &out->valid;
	AxisTable t;
	build_axis_table(t, 0, p->residual_shrink, p->offset, p->n_point, p->kernel, 0, r->left, r->width);
	const int need_left = t.first[0];
	const int need_right = t.first[r->width - 1] + p->n_point;
	if (in->valid.top > r->top || in->valid.top + in->valid.height < r->top + r->height ||
		in->valid.left > need_left || in->valid.left + in->valid.width < need_right) {
		error(domain, "input region does not cover columns %d..%d of the embedded image", need_left, need_right);
		return -1;
	}
	cudaStream_t s = current_stream();
	StagedRegion si, so;
	if (stage_in(domain, in, &si, s))
		return -1;
	const size_t ps = format_sizeof(in->im.BandFmt) * in->im.Bands;
	so.line = so.bpl = ps * r->width;
	if (dev_alloc(domain, &so.dev, so.line * r->height, s))
		return -1;
	for (auto &f : t.first)
		f -= in->valid.left;
	t.embed = 0;
	const char *src = (const char *) si.dev + (size_t) (r->top - in->valid.top) * si.bpl;
	int rc = launch_reduceh(domain, src, si.bpl, in->valid.width, so.dev, so.bpl, in->im.Bands, r->width, r->height,
		in->im.BandFmt, t, s);
	if (!rc)
		rc = stage_out(domain, out, &so, s);
	dev_free(si.dev, s);
	dev_free(so.dev, s);
	return rc;
}

extern "C" int
vb200_shrinkv_gen(const VB200Region *out, const VB200Region *in, int vshrink)
{
	const char *domain = "shrinkv_gen";
	if (check_regions(domain, out, in))
		return -1;
	const VB200Rect *r = &out->valid;
	/* rows r->top * vshrink .. of the (rounded-up, embedded) input: shrinkv.c:346-366 */
	if (in->valid.top > r->top * vshrink || in->valid.top + in->valid.height < (r->top + r->height) * vshrink ||
		in->valid.left > r->left || in->valid.left + in->valid.width < r->left + r->width) {
		error(domain, "input region too small");
		return -1;
	}
	cudaStream_t s = current_stream();
	StagedRegion si;
	if (stage_in(domain, in, &si, s))
		return -1;
	const size_t ps = format_sizeof(in->im.BandFmt) * in->im.Bands;
	DevImage d, o;
	d.w = r->width;
	d.h = r->height * vshrink;
	d.bands = in->im.Bands;
	d.fmt = in->im.BandFmt;
	d.type = in->im.Type;
	d.bpl = si.bpl;
	d.data = (char *) si.dev + (size_t) (r->top * vshrink - in->valid.top) * si.bpl + (size_t) (r->left - in->valid.left) * ps;
	int rc = dev_shrinkv(domain, d, &o, vshrink, 1, s);
	if (!rc) {
		StagedRegion so;
		so.dev = o.data;
		so.bpl = o.bpl;
		so.line = ps * r->width;
		rc = stage_out(domain, out, &so, s);
	}
	dev_image_release(&o, s);
	dev_free(si.dev, s);
	return rc;
}

extern "C" int
vb200_shrinkh_gen(const VB200Region *out, const VB200Region *in, int hshrink)
{
	const char *domain = "shrinkh_gen";
	if (check_regions(domain, out, in))
		return -1;
	const VB200Rect *r = &out->valid;
	if (in->valid.left > r->left * hshrink || in->valid.left + in->valid.width < (r->left + r->width) * hshrink ||
		in->valid.top > r->top || in->valid.top + in->valid.height < r->top + r->height) {
		error(domain, "input region too small");
		return -1;
	}
	cudaStream_t s = current_stream();
	StagedRegion si;
	if (stage_in(domain, in, &si, s))
		return -1;
	const size_t ps = format_sizeof(in->im.BandFmt) * in->im.Bands;
	DevImage d, o;
	d.w = r->width * hshrink;
	d.h = r->height;
	d.bands = in->im.Bands;
	d.fmt = in->im.BandFmt;
	d.type = in->im.Type;
	d.bpl = si.bpl;
	d.data = (char *) si.dev + (size_t) (r->top - in->valid.top) * si.bpl + (size_t) (r->left * hshrink - in->valid.left) * ps;
	int rc = dev_shrinkh(domain, d, &o, hshrink, 1, s);
	if (!rc) {
		StagedRegion so;
		so.dev = o.data;
		so.bpl = o.bpl;
		so.line = ps * r->width;
		rc = stage_out(domain, out, &so, s);
	}
	dev_image_release(&o, s);
	dev_free(si.dev, s);
	return rc;
}

/* ------------------------------------------------------ scanline kernel seam
 * reference: resample/presample.h:74-87 (the Highway kernels).  void
 * functions: on a CUDA failure they leave the output untouched and record the
 * error in the buffer.
 */

extern "C" void
vips_reducev_uchar_hwy(uint8_t *pout, uint8_t *pin, int n, int ne, int lskip, const short *k)
{
	const char *domain = "vips_reducev_uchar_hwy";
	if (ensure_init(domain))
		return;
	cudaStream_t s = current_stream();
	void *din = nullptr, *dout = nullptr;
	if (dev_alloc(domain, &din, (size_t) n * ne, s) || dev_alloc(domain, &dout, ne, s))
		return;
	cudaMemcpy2DAsync(din, ne, pin, lskip, ne, n, cudaMemcpyHostToDevice, s);
	AxisTable t;
	t.n_point = n;
	t.embed = 0;
	t.first.assign(1, 0);
	t.phase.assign(1, 0);
	t.ms.assign(k, k + n);
	t.mf.assign(n, 0.0);
	if (!launch_reducev(domain, din, ne, n, dout, ne, ne, 1, VB200_FORMAT_UCHAR, t, s)) {
		cudaMemcpyAsync(pout, dout, ne, cudaMemcpyDeviceToHost, s);
		cudaStreamSynchronize(s);
	}
	dev_free(din, s);
	dev_free(dout, s);
}

extern "C" void
vips_reduceh_uchar_hwy(uint8_t *pout, uint8_t *pin, int n, int width, int bands, short *cs[65], double X,
	double hshrink)
{
	const char *domain = "vips_reduceh_uchar_hwy";
	if (ensure_init(domain) || width <= 0)
		return;
	/* same stepping as reduceh_hwy.cpp:157-237: X advances by hshrink */
	AxisTable t;
	t.n_point = n;
	t.embed = 0;
	t.first.resize(width);
	t.phase.resize(width);
	t.ms.resize((size_t) 65 * n);
	t.mf.assign((size_t) 65 * n, 0.0);
	for (int p = 0; p < 65; p++)
		memcpy(&t.ms[(size_t) p * n], cs[p], n * sizeof(short));
	double pos = X;
	for (int x = 0; x < width; x++) {
		const int ix = (int) pos;
		const int sx = pos * VB200_TRANSFORM_SCALE * 2;
		const int six = sx & (VB200_TRANSFORM_SCALE * 2 - 1);
		t.first[x] = ix;
		t.phase[x] = (six + 1) >> 1;
		pos += hshrink;
	}
	/* pin is a VIRTUAL origin: the caller passes VIPS_REGION_ADDR(ir, ir->valid.left, y) - ir->valid.left * ps
	 * with X in absolute image coordinates (reduceh.cpp:379-386), so only pixels first[0] .. first[w - 1] + n - 1
	 * are inside the region.  Copy exactly those and rebase the table.
	 */
	const int x0 = t.first[0];
	const int in_w = t.first[width - 1] + n - x0;
	for (auto &f : t.first)
		f -= x0;
	cudaStream_t s = current_stream();
	void *din = nullptr, *dout = nullptr;
	if (dev_alloc(domain, &din, (size_t) in_w * bands, s) || dev_alloc(domain, &dout, (size_t) width * bands, s))
		return;
	cudaMemcpyAsync(din, pin + (ptrdiff_t) x0 * bands, (size_t) in_w * bands, cudaMemcpyHostToDevice, s);
	if (!launch_reduceh(domain, din, (size_t) in_w * bands, in_w, dout, (size_t) width * bands, bands, width, 1,
			VB200_FORMAT_UCHAR, t, s)) {
		cudaMemcpyAsync(pout, dout, (size_t) width * bands, cudaMemcpyDeviceToHost, s);
		cudaStreamSynchronize(s);
	}
	dev_free(din, s);
	dev_free(dout, s);
}

extern "C" void
vips_shrinkh_uchar_hwy(uint8_t *pout, uint8_t *pin, int width, int hshrink, int bands)
{
	const char *domain = "vips_shrinkh_uchar_hwy";
	if (ensure_init(domain))
		return;
	cudaStream_t s = current_stream();
	VB200Image in = {width * hshrink, 1, bands, VB200_FORMAT_UCHAR, 0, VB200_HOST, pin, 0};
	DevImage d, o;
	if (to_device(domain, &in, &d, s))
		return;
	if (!dev_shrinkh(domain, d, &o, hshrink, 1, s)) {
		cudaMemcpyAsync(pout, o.data, (size_t) width * bands, cudaMemcpyDeviceToHost, s);
		cudaStreamSynchronize(s);
	}
	dev_image_release(&o, s);
	dev_image_release(&d, s);
}

namespace {

__global__ void
add_line_kernel(const uint8_t *__restrict__ in, int ne, unsigned int *__restrict__ sum)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x < ne)
		sum[x] += in[x];
}

__global__ void
write_line_kernel(uint8_t *__restrict__ out, int ne, unsigned int amend, unsigned int multiplier,
	const unsigned int *__restrict__ sum)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x < ne)
		out[x] = (uint8_t) (((sum[x] + amend) * multiplier) >> 24);
}

} // namespace

extern "C" void
vips_shrinkv_add_line_uchar_hwy(uint8_t *pin, int ne, unsigned int *sum)
{
	const char *domain = "vips_shrinkv_add_line_uchar_hwy";
	if (ensure_init(domain) || ne <= 0)
		return;
	cudaStream_t s = current_stream();
	void *din = nullptr, *dsum = nullptr;
	if (dev_alloc(domain, &din, ne, s) || dev_alloc(domain, &dsum, (size_t) ne * 4, s))
		return;
	cudaMemcpyAsync(din, pin, ne, cudaMemcpyHostToDevice, s);
	cudaMemcpyAsync(dsum, sum, (size_t) ne * 4, cudaMemcpyHostToDevice, s);
	add_line_kernel<<<(ne + 255) / 256, 256, 0, s>>>((const uint8_t *) din, ne, (unsigned int *) dsum);
	count_launch();
	cudaMemcpyAsync(sum, dsum, (size_t) ne * 4, cudaMemcpyDeviceToHost, s);
	cudaStreamSynchronize(s);
	dev_free(din, s);
	dev_free(dsum, s);
}

extern "C" void
vips_shrinkv_write_line_uchar_hwy(uint8_t *pout, int ne, int vshrink, unsigned int *sum)
{
	const char *domain = "vips_shrinkv_write_line_uchar_hwy";
	if (ensure_init(domain) || ne <= 0)
		return;
	cudaStream_t s = current_stream();
	void *dout = nullptr, *dsum = nullptr;
	if (dev_alloc(domain, &dout, ne, s) || dev_alloc(domain, &dsum, (size_t) ne * 4, s))
		return;
	cudaMemcpyAsync(dsum, sum, (size_t) ne * 4, cudaMemcpyHostToDevice, s);
	const unsigned int multiplier = (unsigned int) ((1LL << 32) / ((1 << 8) * (long long) vshrink));
	write_line_kernel<<<(ne + 255) / 256, 256, 0, s>>>((uint8_t *) dout, ne, vshrink / 2, multiplier,
		(const unsigned int *) dsum);
	count_launch();
	cudaMemcpyAsync(pout, dout, ne, cudaMemcpyDeviceToHost, s);
	cudaStreamSynchronize(s);
	dev_free(dout, s);
	dev_free(dsum, s);
}

/* ------------------------------------------------------ vips_convi_uchar_hwy
 * reference: convolution/pconvolution.h:74-76, convi_hwy.cpp:93-276 (scalar statement :265-273).
 */
namespace {

__global__ void __launch_bounds__(256)
convi_hwy_kernel(const uint8_t *__restrict__ p0, int in_bpl, uint8_t *__restrict__ q0, int out_bpl, int ne, int nnz,
	const int *__restrict__ offsets, const short *__restrict__ mant, int exp, int offset)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= ne)
		return;
	const uint8_t *p = p0 + (size_t) blockIdx.y * in_bpl + x;
	int sum = 1 << (exp - 1);
	for (int i = 0; i < nnz; i++)
		sum += (int) p[__ldg(offsets + i)] * (int) __ldg(mant + i);
	q0[(size_t) blockIdx.y * out_bpl + x] = (uint8_t) max(0, min((sum >> exp) + offset, 255));
}

} // namespace

extern "C" int
vb200_convi_uchar_vector(uint8_t *q0, int out_bpl, const uint8_t *p0, int in_bpl, int in_line_bytes, int in_rows, int ne,
	int rows, int nnz, int offset, const int32_t *offsets, const int16_t *mant, int exp)
{
	const char *domain = "vips_convi_uchar_hwy";
	if (!q0 || !p0 || !offsets || !mant || ne <= 0 || rows <= 0 || nnz <= 0 || exp < 1 || exp > 31) {
		error(domain, "bad argument");
		return -1;
	}
	/* every read must stay inside the prepared input */
	for (int i = 0; i < nnz; i++) {
		const long last = (long) (rows - 1) * in_bpl + (ne - 1) + offsets[i];
		if (offsets[i] < 0 || last / in_bpl >= in_rows || (offsets[i] % in_bpl) + ne > in_line_bytes) {
			error(domain, "tap %d (offset %d) reads outside the input region", i, offsets[i]);
			return -1;
		}
	}
	if (ensure_init(domain))
		return -1;
	cudaStream_t s = current_stream();
	void *din = nullptr, *dout = nullptr, *dtab = nullptr;
	const size_t tab = (size_t) nnz * (sizeof(int) + sizeof(short));
	int rc = dev_alloc(domain, &din, (size_t) in_bpl * in_rows, s) || dev_alloc(domain, &dout, (size_t) ne * rows, s) ||
		dev_alloc(domain, &dtab, tab, s);
	if (!rc) {
		std::vector<char> host(tab);
		memcpy(host.data(), offsets, (size_t) nnz * sizeof(int));
		memcpy(host.data() + (size_t) nnz * sizeof(int), mant, (size_t) nnz * sizeof(short));
		/* same pitch on the device: the caller's element offsets stay valid */
		cudaMemcpy2DAsync(din, in_bpl, p0, in_bpl, in_line_bytes, in_rows, cudaMemcpyHostToDevice, s);
		cudaMemcpyAsync(dtab, host.data(), tab, cudaMemcpyHostToDevice, s);
		cudaStreamSynchronize(s); /* host staging vector dies with this scope */
		convi_hwy_kernel<<<dim3((ne + 255) / 256, rows), 256, 0, s>>>((const uint8_t *) din, in_bpl, (uint8_t *) dout, ne, ne, nnz,
			(const int *) dtab, (const short *) ((char *) dtab + (size_t) nnz * sizeof(int)), exp, offset);
		count_launch();
		cudaError_t e = cudaGetLastError();
		if (e == cudaSuccess)
			e = cudaMemcpy2DAsync(q0, out_bpl, dout, ne, ne, rows, cudaMemcpyDeviceToHost, s);
		if (e == cudaSuccess)
			e = cudaStreamSynchronize(s);
		if (e != cudaSuccess)
			rc = cuda_fail(domain, e, "convi_hwy_kernel");
	}
	dev_free(din, s);
	dev_free(dout, s);
	dev_free(dtab, s);
	return rc ? -1 : 0;
}

extern "C" void
vips_convi_uchar_hwy(VB200VipsRegionHead *out_region, VB200VipsRegionHead *ir, VB200Rect *r, int32_t ne, int32_t nnz,
	int32_t offset, const int32_t *offsets, const int16_t *mant, int32_t exp)
{
	if (!out_region || !ir || !r || !ir->im || !out_region->im)
		return;
	/* VIPS_REGION_ADDR, include/vips/region.h:230-233 (uchar: sizeof pel = Bands) */
	const int ips = ir->im->Bands, ops = out_region->im->Bands;
	const uint8_t *p0 = ir->data + (size_t) (r->top - ir->valid.top) * ir->bpl + (size_t) (r->left - ir->valid.left) * ips;
	uint8_t *q0 = out_region->data + (size_t) (r->top - out_region->valid.top) * out_region->bpl +
		(size_t) (r->left - out_region->valid.left) * ops;
	const int in_rows = ir->valid.top + ir->valid.height - r->top;
	const int in_line = (ir->valid.left + ir->valid.width - r->left) * ips;
	vb200_convi_uchar_vector(q0, out_region->bpl, p0, ir->bpl, in_line, in_rows, ne, r->height, nnz, offset, offsets, mant, exp);
}
