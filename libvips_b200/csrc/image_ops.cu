/* image_ops.cu -- the whole-image ops of the C ABI: one record per op, one dispatch, and two ways to run them.
 *
 * Each op mirrors the libvips C API call named in include/vb200.h: same argument meaning, same error conditions and
 * messages where the reference has them.  An op's constructor takes its C arguments, applies their defaults and makes
 * every refusal that needs no image; vb200_<op>() and vb200_chain_add_<op>() call the same constructor, and
 * image_op_apply() runs the record on a device image.  Stand-alone, vb200_<op>() runs it through run_image().
 *
 * Chained (SURVEY 8f rank 2), what the reference does by pulling tiles through every op's generate() from a sink
 * (iofuncs/sinkmemory.c:324, threadpool.c:625) runs image by image: image i is uploaded on one of three streams, every
 * step runs on DEVICE images of that stream (intermediates come from the stream-ordered pool and never visit the host)
 * and the result is downloaded, while images i + 1 and i + 2 are in their own phases on the other streams.  Images of
 * one batch may differ in size and format.
 */
#include <mutex>
#include <vector>

#include "vb200_internal.h"

using namespace vb200;

namespace {

enum ImageOpKind {
	OP_SHRINKV, OP_SHRINKH, OP_REDUCEV, OP_REDUCEH, OP_REDUCE, OP_RESIZE, OP_PREMULTIPLY, OP_UNPREMULTIPLY, OP_CONV, OP_CONVSEP,
	OP_GAUSSBLUR, OP_SHARPEN, OP_COLOURSPACE, OP_FLATTEN, OP_MORPH, OP_RANK, OP_HIST_FIND, OP_HIST_EQUAL, OP_HIST_LOCAL
};

/* One op with its arguments, defaults applied.  Each kind reads the fields named beside it. */
struct ImageOp {
	ImageOpKind kind = OP_SHRINKV;
	int shrink = 1, ceil_mode = 0;	 /* shrinkv, shrinkh */
	double hshrink = 1, vshrink = 1; /* reduceh, reducev, reduce */
	double hscale = 1, vscale = 1;	 /* resize */
	int kernel = 0;					 /* reduce*, resize */
	double gap = 0;
	double max_alpha = 0; /* (un)premultiply, flatten */
	int uchar_mode = 0;	  /* (un)premultiply */
	std::vector<double> mask; /* conv, convsep, morph: mw x mh coefficients */
	int mw = 0, mh = 0;
	double scale = 1, offset = 0; /* conv, convsep */
	int precision = 0;			  /* conv, convsep, gaussblur */
	int morph = 0;				  /* morph: 0 erode, 1 dilate */
	double sigma = 0, min_ampl = 0;				   /* gaussblur; sharpen's sigma */
	double x1 = 0, y2 = 0, y3 = 0, m1 = 0, m2 = 0; /* sharpen */
	int space = 0;								   /* colourspace */
	std::vector<double> background;				   /* flatten: none if empty */
	int width = 0, height = 0, index = 0;		   /* rank; hist_local's window */
	int band = -1;								   /* hist_find, hist_equal */
	int max_slope = 0;							   /* hist_local */
};

/* ------------------------------------------------------------------ constructors */

ImageOp
op_shrink(ImageOpKind kind, int shrink, int ceil_mode)
{
	ImageOp op;
	op.kind = kind;
	op.shrink = shrink;
	op.ceil_mode = ceil_mode;
	return op;
}

/* reducev reads vshrink, reduceh hshrink, reduce both (reduce.c:97-119: the caller's doubles untouched) */
int
op_reduce(const char *domain, ImageOpKind kind, double hshrink, double vshrink, int kernel, double gap, ImageOp *op)
{
	if (hshrink < 1.0 || vshrink < 1.0) {
		error(domain, "reduce factor should be >= 1.0");
		return -1;
	}
	op->kind = kind;
	op->hshrink = hshrink;
	op->vshrink = vshrink;
	op->kernel = kernel;
	op->gap = gap;
	return 0;
}

ImageOp
op_resize(double scale, double vscale, int kernel, double gap)
{
	ImageOp op;
	op.kind = OP_RESIZE;
	op.hscale = scale;
	op.vscale = vscale > 0 ? vscale : scale;
	op.kernel = kernel;
	op.gap = gap < 0 ? 2.0 : gap; /* resize.c:352-357 */
	return op;
}

ImageOp
op_premultiply(ImageOpKind kind, double max_alpha, int uchar_mode)
{
	ImageOp op;
	op.kind = kind;
	op.max_alpha = max_alpha;
	op.uchar_mode = uchar_mode;
	return op;
}

/* conv, convsep (mode: the precision) and morph (mode: 0 erode, 1 dilate) */
int
op_mask(const char *domain, ImageOpKind kind, const VB200Mask *mask, int mode, ImageOp *op)
{
	if (!mask || !mask->coeff) {
		error(domain, "no mask");
		return -1;
	}
	if (mask->width <= 0 || mask->height <= 0) {
		error(domain, "bad mask");
		return -1;
	}
	/* vips_check_separable: one of the dimensions must be 1 */
	if (kind == OP_CONVSEP && mask->width != 1 && mask->height != 1) {
		error(domain, "mask must be 1xn or nx1 elements");
		return -1;
	}
	op->kind = kind;
	op->mask.assign(mask->coeff, mask->coeff + (size_t) mask->width * mask->height);
	op->mw = mask->width;
	op->mh = mask->height;
	op->scale = mask->scale;
	op->offset = mask->offset;
	if (kind == OP_MORPH)
		op->morph = mode;
	else
		op->precision = mode;
	return 0;
}

ImageOp
op_gaussblur(double sigma, double min_ampl, int precision)
{
	ImageOp op;
	op.kind = OP_GAUSSBLUR;
	op.sigma = sigma;
	op.min_ampl = min_ampl <= 0 ? 0.2 : min_ampl; /* gaussblur.c class default */
	op.precision = precision;
	return op;
}

ImageOp
op_sharpen(double sigma, double x1, double y2, double y3, double m1, double m2)
{
	ImageOp op;
	op.kind = OP_SHARPEN;
	op.sigma = sigma;
	op.x1 = x1;
	op.y2 = y2;
	op.y3 = y3;
	op.m1 = m1;
	op.m2 = m2;
	return op;
}

ImageOp
op_colourspace(int space)
{
	ImageOp op;
	op.kind = OP_COLOURSPACE;
	op.space = space;
	return op;
}

/* background: n = 1 or bands - 1 values (NULL or n < 1: black); max_alpha <= 0: the interpretation's default */
ImageOp
op_flatten(const double *background, int n, double max_alpha)
{
	ImageOp op;
	op.kind = OP_FLATTEN;
	if (background && n > 0)
		op.background.assign(background, background + n);
	op.max_alpha = max_alpha;
	return op;
}

ImageOp
op_rank(int width, int height, int index)
{
	ImageOp op;
	op.kind = OP_RANK;
	op.width = width;
	op.height = height;
	op.index = index;
	return op;
}

/* hist_find and hist_equal: band -1 (every band) or the band to scan, checked against the image (vips_check_bandno) */
ImageOp
op_hist(ImageOpKind kind, int band)
{
	ImageOp op;
	op.kind = kind;
	op.band = band;
	return op;
}

/* hist_local.c:283-306; the window's area is bounded so that the int sums cannot overflow */
int
op_hist_local(const char *domain, int width, int height, int max_slope, ImageOp *op)
{
	if (hist_local_check(domain, width, height, max_slope))
		return -1;
	op->kind = OP_HIST_LOCAL;
	op->width = width;
	op->height = height;
	op->max_slope = max_slope;
	return 0;
}

/* ------------------------------------------------------------------ dispatch */

int
image_op_apply(const char *domain, const ImageOp &op, const DevImage &in, DevImage *out, cudaStream_t s)
{
	switch (op.kind) {
	case OP_SHRINKV:
		return dev_shrinkv(domain, in, out, op.shrink, op.ceil_mode, s);
	case OP_SHRINKH:
		return dev_shrinkh(domain, in, out, op.shrink, op.ceil_mode, s);
	case OP_REDUCEV: {
		/* stand-alone vips_reducev: the output is FATSTRIP (reducev.cpp:1019) unless the gap pre-shrink adds a SMALLTILE shrinkv */
		ReduceGeom g;
		if (reduce_geometry(domain, in.h, op.vshrink, op.kernel, op.gap, &g))
			return -1;
		const TileGeometry tg = tile_geometry();
		const int rect_h = g.int_shrink > 1 ? tg.tile_height : tg.fatstrip_height;
		return dev_reducev(domain, in, out, op.vshrink, op.kernel, op.gap, rect_h, s);
	}
	case OP_REDUCEH:
		/* FATSTRIP (full-width tiles): one rect per scanline strip, left = 0 */
		return dev_reduceh(domain, in, out, op.hshrink, op.kernel, op.gap, 0, s);
	case OP_REDUCE:
		return dev_reduce_chain(domain, in, out, op.hshrink, op.vshrink, op.kernel, op.gap, s);
	case OP_RESIZE:
		return dev_resize(domain, in, out, op.hscale, op.vscale, op.kernel, op.gap, s);
	case OP_PREMULTIPLY:
		return dev_premultiply(domain, in, out, op.max_alpha, op.uchar_mode, s);
	case OP_UNPREMULTIPLY:
		return dev_unpremultiply(domain, in, out, op.max_alpha, op.uchar_mode, s);
	case OP_CONV:
		return dev_conv(domain, in, out, op.mask.data(), op.mw, op.mh, op.scale, op.offset, op.precision, s, true);
	case OP_CONVSEP:
		return dev_convsep(domain, in, out, op.mask.data(), op.mw, op.mh, op.scale, op.offset, op.precision, s, true);
	case OP_GAUSSBLUR:
		return dev_gaussblur(domain, in, out, op.sigma, op.min_ampl, op.precision, s);
	case OP_SHARPEN:
		return dev_sharpen(domain, in, out, op.sigma, op.x1, op.y2, op.y3, op.m1, op.m2, s);
	case OP_COLOURSPACE:
		/* the source space is the image's Type (the reference guesses it, vips_image_guess_interpretation) */
		return dev_colourspace(domain, in, out, op.space, in.type, s);
	case OP_FLATTEN:
		return dev_flatten(domain, in, out, op.background.empty() ? nullptr : op.background.data(), (int) op.background.size(),
			op.max_alpha, s);
	case OP_MORPH:
		return dev_morph(domain, in, out, op.mask.data(), op.mw, op.mh, op.morph, s);
	case OP_RANK:
		return dev_rank(domain, in, out, op.width, op.height, op.index, s);
	case OP_HIST_FIND:
		return dev_hist_find(domain, in, out, op.band, s);
	case OP_HIST_EQUAL:
		return dev_hist_equal(domain, in, out, op.band, s);
	case OP_HIST_LOCAL:
		return dev_hist_local(domain, in, out, op.width, op.height, op.max_slope, s);
	}
	return -1;
}

/* ------------------------------------------------------------------ stand-alone */

/* The bytes of a result line the op may write straight into a caller's device buffer (0: it never does, and deliver()
 * copies into such a buffer).
 */
size_t
preset_line(const ImageOp &op, const VB200Image &in)
{
	switch (op.kind) {
	case OP_CONV:
	case OP_CONVSEP:
	case OP_GAUSSBLUR:
		/* convolutions keep the geometry; convf widens to float */
		return (size_t) in.Xsize * in.Bands * std::max<size_t>(4, format_sizeof(in.BandFmt));
	case OP_COLOURSPACE: {
		/* colour ops keep the geometry and, but for B_W / GREY16 sources (two bands more), the band count; no output element
		 * is wider than a float
		 */
		const bool grey_source = in.Type == VB200_INTERPRETATION_B_W || in.Type == VB200_INTERPRETATION_GREY16;
		return (size_t) in.Xsize * (in.Bands + (grey_source ? 2 : 0)) * 4;
	}
	default:
		return 0;
	}
}

int
run_op(const char *domain, const ImageOp &op, const VB200Image *in, VB200Image *out)
{
	return run_image(domain, in, out,
		[&](size_t *line) {
			*line = preset_line(op, *in);
			/* the histogram ops refuse a band, format or window that the descriptor rules out before the upload */
			if (op.kind == OP_HIST_FIND || op.kind == OP_HIST_EQUAL || op.kind == OP_HIST_LOCAL)
				return hist_refuse(domain, op.kind - OP_HIST_FIND, in->Xsize, in->Ysize, in->Bands, in->BandFmt, op.band, op.width,
					op.height);
			return 0;
		},
		[&](const DevImage &d, DevImage *o, cudaStream_t s) { return image_op_apply(domain, op, d, o, s); });
}

} // namespace

namespace vb200 {

int
run_image(const char *domain, const VB200Image *in, VB200Image *out, const std::function<int(size_t *preset_line)> &prepare,
	const ImageApply &apply)
{
	if (!in) {
		error(domain, "no input image");
		return -1;
	}
	if (!out) {
		error(domain, "no output image");
		return -1;
	}
	size_t line = 0;
	if (ensure_init(domain) || prepare(&line))
		return -1;
	cudaStream_t s = current_stream();
	DevImage din, dout;
	if (to_device(domain, in, &din, s))
		return -1;
	if (line)
		preset_output(&dout, in, out, line, in->Ysize);
	int rc = apply(din, &dout, s);
	if (!rc)
		rc = deliver(domain, &dout, in, out, s);
	dev_image_release(&din, s);
	return rc;
}

} // namespace vb200

extern "C" int
vb200_shrinkv(const VB200Image *in, VB200Image *out, int vshrink, int ceil_mode)
{
	return run_op("shrinkv", op_shrink(OP_SHRINKV, vshrink, ceil_mode), in, out);
}

extern "C" int
vb200_shrinkh(const VB200Image *in, VB200Image *out, int hshrink, int ceil_mode)
{
	return run_op("shrinkh", op_shrink(OP_SHRINKH, hshrink, ceil_mode), in, out);
}

extern "C" int
vb200_reducev(const VB200Image *in, VB200Image *out, double vshrink, int kernel, double gap)
{
	ImageOp op;
	return op_reduce("reducev", OP_REDUCEV, 1.0, vshrink, kernel, gap, &op) ? -1 : run_op("reducev", op, in, out);
}

extern "C" int
vb200_reduceh(const VB200Image *in, VB200Image *out, double hshrink, int kernel, double gap)
{
	ImageOp op;
	return op_reduce("reduceh", OP_REDUCEH, hshrink, 1.0, kernel, gap, &op) ? -1 : run_op("reduceh", op, in, out);
}

extern "C" int
vb200_reduce(const VB200Image *in, VB200Image *out, double hshrink, double vshrink, int kernel, double gap)
{
	ImageOp op;
	return op_reduce("reduce", OP_REDUCE, hshrink, vshrink, kernel, gap, &op) ? -1 : run_op("reduce", op, in, out);
}

extern "C" int
vb200_resize(const VB200Image *in, VB200Image *out, double scale, double vscale, int kernel, double gap)
{
	return run_op("resize", op_resize(scale, vscale, kernel, gap), in, out);
}

extern "C" int
vb200_premultiply(const VB200Image *in, VB200Image *out, double max_alpha, int uchar_mode)
{
	return run_op("premultiply", op_premultiply(OP_PREMULTIPLY, max_alpha, uchar_mode), in, out);
}

extern "C" int
vb200_unpremultiply(const VB200Image *in, VB200Image *out, double max_alpha, int uchar_mode)
{
	return run_op("unpremultiply", op_premultiply(OP_UNPREMULTIPLY, max_alpha, uchar_mode), in, out);
}

extern "C" int
vb200_conv(const VB200Image *in, VB200Image *out, const VB200Mask *mask, int precision)
{
	ImageOp op;
	return op_mask("conv", OP_CONV, mask, precision, &op) ? -1 : run_op("conv", op, in, out);
}

extern "C" int
vb200_convsep(const VB200Image *in, VB200Image *out, const VB200Mask *mask, int precision)
{
	ImageOp op;
	return op_mask("convsep", OP_CONVSEP, mask, precision, &op) ? -1 : run_op("convsep", op, in, out);
}

extern "C" int
vb200_gaussblur(const VB200Image *in, VB200Image *out, double sigma, double min_ampl, int precision)
{
	return run_op("gaussblur", op_gaussblur(sigma, min_ampl, precision), in, out);
}

extern "C" int
vb200_sharpen(const VB200Image *in, VB200Image *out, double sigma, double x1, double y2, double y3, double m1, double m2)
{
	return run_op("sharpen", op_sharpen(sigma, x1, y2, y3, m1, m2), in, out);
}

/* reference: vips_colourspace(), colour/colourspace.c:551-617 */
extern "C" int
vb200_colourspace(const VB200Image *in, VB200Image *out, int space)
{
	return run_op("colourspace", op_colourspace(space), in, out);
}

/* reference: vips_flatten(), conversion/flatten.c:605-616 */
extern "C" int
vb200_flatten(const VB200Image *in, VB200Image *out, const double *background, int n, double max_alpha)
{
	return run_op("flatten", op_flatten(background, n, max_alpha), in, out);
}

/* reference: vips_morph(), morphology/morph.c:1030-1042.  morph: 0 = erode, 1 = dilate (VipsOperationMorphology). */
extern "C" int
vb200_morph(const VB200Image *in, VB200Image *out, const VB200Mask *mask, int morph)
{
	ImageOp op;
	return op_mask("morph", OP_MORPH, mask, morph, &op) ? -1 : run_op("morph", op, in, out);
}

/* reference: vips_rank(), morphology/rank.c:623-635; vips_median(in, out, size) is rank(size, size, size * size / 2), :651-664 */
extern "C" int
vb200_rank(const VB200Image *in, VB200Image *out, int width, int height, int index)
{
	return run_op("rank", op_rank(width, height, index), in, out);
}

extern "C" int
vb200_median(const VB200Image *in, VB200Image *out, int size)
{
	return run_op("rank", op_rank(size, size, (size * size) / 2), in, out);
}

/* reference: vips_hist_find(), arithmetic/hist_find.c:471-482 */
extern "C" int
vb200_hist_find(const VB200Image *in, VB200Image *out, int band)
{
	return run_op("hist_find", op_hist(OP_HIST_FIND, band), in, out);
}

/* reference: vips_hist_equal(), histogram/hist_equal.c:156-167 */
extern "C" int
vb200_hist_equal(const VB200Image *in, VB200Image *out, int band)
{
	return run_op("hist_equal", op_hist(OP_HIST_EQUAL, band), in, out);
}

/* reference: vips_hist_local(), histogram/hist_local.c:417-428 */
extern "C" int
vb200_hist_local(const VB200Image *in, VB200Image *out, int width, int height, int max_slope)
{
	ImageOp op;
	return op_hist_local("hist_local", width, height, max_slope, &op) ? -1 : run_op("hist_local", op, in, out);
}

/* ------------------------------------------------------------------ the chain pump */

namespace {

constexpr int kChainStreams = 3;

} // namespace

struct VB200Chain {
	std::vector<ImageOp> ops;
	cudaStream_t streams[kChainStreams] = {nullptr, nullptr, nullptr};
	std::mutex lock;
};

extern "C" VB200Chain *
vb200_chain_new(void)
{
	if (ensure_init("chain"))
		return nullptr;
	return new VB200Chain();
}

extern "C" void
vb200_chain_free(VB200Chain *chain)
{
	if (!chain)
		return;
	for (auto &s : chain->streams)
		if (s) {
			cudaStreamSynchronize(s);
			cudaStreamDestroy(s);
		}
	delete chain;
}

static int
chain_push(VB200Chain *chain, ImageOp &&op)
{
	if (!chain) {
		error("chain", "null chain");
		return -1;
	}
	chain->ops.push_back(std::move(op));
	return 0;
}

extern "C" int
vb200_chain_add_resize(VB200Chain *chain, double scale, double vscale, int kernel, double gap)
{
	return chain_push(chain, op_resize(scale, vscale, kernel, gap));
}

extern "C" int
vb200_chain_add_reduce(VB200Chain *chain, double hshrink, double vshrink, int kernel, double gap)
{
	ImageOp op;
	return op_reduce("chain", OP_REDUCE, hshrink, vshrink, kernel, gap, &op) ? -1 : chain_push(chain, std::move(op));
}

extern "C" int
vb200_chain_add_colourspace(VB200Chain *chain, int space)
{
	return chain_push(chain, op_colourspace(space));
}

extern "C" int
vb200_chain_add_conv(VB200Chain *chain, const VB200Mask *mask, int precision)
{
	ImageOp op;
	return op_mask("chain", OP_CONV, mask, precision, &op) ? -1 : chain_push(chain, std::move(op));
}

extern "C" int
vb200_chain_add_convsep(VB200Chain *chain, const VB200Mask *mask, int precision)
{
	ImageOp op;
	return op_mask("chain", OP_CONVSEP, mask, precision, &op) ? -1 : chain_push(chain, std::move(op));
}

extern "C" int
vb200_chain_add_morph(VB200Chain *chain, const VB200Mask *mask, int morph)
{
	ImageOp op;
	return op_mask("chain", OP_MORPH, mask, morph, &op) ? -1 : chain_push(chain, std::move(op));
}

extern "C" int
vb200_chain_add_flatten(VB200Chain *chain, const double *background, int n, double max_alpha)
{
	return chain_push(chain, op_flatten(background, n, max_alpha));
}

extern "C" int
vb200_chain_add_rank(VB200Chain *chain, int width, int height, int index)
{
	return chain_push(chain, op_rank(width, height, index));
}

extern "C" int
vb200_chain_add_gaussblur(VB200Chain *chain, double sigma, double min_ampl, int precision)
{
	return chain_push(chain, op_gaussblur(sigma, min_ampl, precision));
}

extern "C" int
vb200_chain_add_sharpen(VB200Chain *chain, double sigma, double x1, double y2, double y3, double m1, double m2)
{
	return chain_push(chain, op_sharpen(sigma, x1, y2, y3, m1, m2));
}

extern "C" int
vb200_chain_add_premultiply(VB200Chain *chain, double max_alpha, int uchar_mode)
{
	return chain_push(chain, op_premultiply(OP_PREMULTIPLY, max_alpha, uchar_mode));
}

extern "C" int
vb200_chain_add_unpremultiply(VB200Chain *chain, double max_alpha, int uchar_mode)
{
	return chain_push(chain, op_premultiply(OP_UNPREMULTIPLY, max_alpha, uchar_mode));
}

extern "C" int
vb200_chain_add_hist_find(VB200Chain *chain, int band)
{
	return chain_push(chain, op_hist(OP_HIST_FIND, band));
}

extern "C" int
vb200_chain_add_hist_equal(VB200Chain *chain, int band)
{
	return chain_push(chain, op_hist(OP_HIST_EQUAL, band));
}

extern "C" int
vb200_chain_add_hist_local(VB200Chain *chain, int width, int height, int max_slope)
{
	ImageOp op;
	return op_hist_local("chain", width, height, max_slope, &op) ? -1 : chain_push(chain, std::move(op));
}

/* in[i]: host images (pinned memory lets the three phases overlap; pageable memory is correct but its
 * copies are staged synchronously).  out[i]: data == NULL -> malloc'ed by the library (vb200_image_free),
 * else the caller's buffer (it must be large enough: run the chain once with NULL to learn the geometry).
 * Returns after the last result has landed.
 */
extern "C" int
vb200_chain_run_host(VB200Chain *chain, const VB200Image *in, VB200Image *out, int n_images)
{
	const char *domain = "chain_run_host";
	if (!chain || !in || !out || n_images < 0) {
		error(domain, "bad argument");
		return -1;
	}
	if (ensure_init(domain))
		return -1;
	std::lock_guard<std::mutex> lock(chain->lock);
	for (auto &s : chain->streams)
		if (!s)
			VB200_CUDA(domain, cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));

	int rc = 0;
	for (int i = 0; i < n_images && !rc; i++) {
		cudaStream_t s = chain->streams[i % kChainStreams];
		if (in[i].where != VB200_HOST) {
			error(domain, "image %d is not a host image", i);
			rc = -1;
			break;
		}
		DevImage cur;
		if (to_device(domain, &in[i], &cur, s)) { /* cudaMemcpy2DAsync on s */
			rc = -1;
			break;
		}
		for (const ImageOp &op : chain->ops) {
			DevImage next;
			if (image_op_apply(domain, op, cur, &next, s)) {
				dev_image_release(&cur, s);
				rc = -1;
				break;
			}
			adopt_pass_through(&cur, &next);
			dev_image_release(&cur, s);
			cur = next;
		}
		if (rc)
			break;
		/* download: async on s; the buffer is released to the pool in stream order */
		if (deliver_host(domain, &cur, &in[i], &out[i], s)) {
			dev_image_release(&cur, s);
			rc = -1;
		}
	}
	for (auto &s : chain->streams)
		if (s && cudaStreamSynchronize(s) != cudaSuccess && !rc)
			rc = cuda_fail(domain, cudaGetLastError(), "chain sync");
	return rc;
}
