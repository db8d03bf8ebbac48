/* vb200.h -- C ABI of libvb200.so, the sm_90a (H100) replacement for libvips'
 * per-tile pixel hot path (resample / convolution / colour generate callbacks).
 *
 * Plain C, plain pointers and sizes.  Every entry point returns 0 on success
 * and -1 on error with a message appended to a thread-local buffer read with
 * vb200_error_buffer() -- the convention of vips_error()/vips_error_buffer()
 * (reference: libvips/iofuncs/error.c:214,329).
 *
 * There is NO CPU fallback inside this library: every pixel is produced by a
 * CUDA kernel.  Unsupported formats return -1 so the host (libvips) keeps its
 * own C generate function for them, exactly as it does today behind
 * vips_vector_isenabled() (reference: resample/reducev.cpp:985-1016).
 *
 * "reference:" comments cite the libvips 8.19 interface each item replaces.
 */
#ifndef VB200_H
#define VB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ enums */

/* reference: VipsBandFormat, include/vips/image.h:121-132 (same values) */
typedef enum {
	VB200_FORMAT_UCHAR = 0,
	VB200_FORMAT_CHAR = 1,
	VB200_FORMAT_USHORT = 2,
	VB200_FORMAT_SHORT = 3,
	VB200_FORMAT_UINT = 4,
	VB200_FORMAT_INT = 5,
	VB200_FORMAT_FLOAT = 6,
	VB200_FORMAT_COMPLEX = 7,
	VB200_FORMAT_DOUBLE = 8,
	VB200_FORMAT_DPCOMPLEX = 9
} VB200BandFormat;

/* reference: VipsInterpretation, include/vips/image.h:94-117 (same values) */
typedef enum {
	VB200_INTERPRETATION_MULTIBAND = 0,
	VB200_INTERPRETATION_B_W = 1,
	VB200_INTERPRETATION_CMYK = 15,
	VB200_INTERPRETATION_XYZ = 12,
	VB200_INTERPRETATION_LAB = 13,
	VB200_INTERPRETATION_LCH = 19,
	VB200_INTERPRETATION_LABS = 21,
	VB200_INTERPRETATION_sRGB = 22,
	VB200_INTERPRETATION_YXY = 23,
	VB200_INTERPRETATION_RGB16 = 25,
	VB200_INTERPRETATION_GREY16 = 26,
	VB200_INTERPRETATION_scRGB = 28,
	VB200_INTERPRETATION_HSV = 29
} VB200Interpretation;

/* reference: VipsKernel, include/vips/resample.h:41-51 (same values) */
typedef enum {
	VB200_KERNEL_NEAREST = 0,
	VB200_KERNEL_LINEAR = 1,
	VB200_KERNEL_CUBIC = 2,
	VB200_KERNEL_MITCHELL = 3,
	VB200_KERNEL_LANCZOS2 = 4,
	VB200_KERNEL_LANCZOS3 = 5,
	VB200_KERNEL_MKS2013 = 6,
	VB200_KERNEL_MKS2021 = 7
} VB200Kernel;

/* reference: VipsSize, include/vips/resample.h:53-59 */
typedef enum {
	VB200_SIZE_BOTH = 0,
	VB200_SIZE_UP = 1,
	VB200_SIZE_DOWN = 2,
	VB200_SIZE_FORCE = 3
} VB200Size;

/* reference: VipsPrecision, include/vips/basic.h:106-111 */
typedef enum {
	VB200_PRECISION_INTEGER = 0,
	VB200_PRECISION_FLOAT = 1,
	VB200_PRECISION_APPROXIMATE = 2
} VB200Precision;

typedef enum {
	VB200_HOST = 0,	 /* data is host memory */
	VB200_DEVICE = 1 /* data is device memory on the current device */
} VB200Where;

/* ------------------------------------------------------------------ types */

/* reference: VipsRect, include/vips/rect.h:40-46 */
typedef struct {
	int left;
	int top;
	int width;
	int height;
} VB200Rect;

/* The header fields of VipsImage the pixel path reads (include/vips/image.h:189-260)
 * plus where the pixels are.  Pixels are row-major, band-interleaved; bpl is
 * the line stride in bytes (VIPS_REGION_LSKIP / VIPS_IMAGE_SIZEOF_LINE).
 */
typedef struct {
	int Xsize;
	int Ysize;
	int Bands;
	int BandFmt; /* VB200BandFormat */
	int Type;	 /* VB200Interpretation */
	int where;	 /* VB200Where */
	void *data;
	size_t bpl;
} VB200Image;

/* reference: VipsRegion {im, valid, data, bpl}, include/vips/region.h:96-130.
 * data points at pixel (valid.left, valid.top); VIPS_REGION_ADDR(reg, x, y) ==
 * data + (y - valid.top) * bpl + (x - valid.left) * sizeof_pel.
 */
typedef struct {
	VB200Image im; /* header of the image the region is on (im.data unused) */
	VB200Rect valid;
	void *data;
	int bpl;
} VB200Region;

/* ---------------------------------------------------------------- runtime */

/* reference: vips_init()/vips_shutdown(), iofuncs/init.c */
int vb200_init(int device);
void vb200_shutdown(void);
/* reference: vips_error_buffer()/vips_error_clear(), iofuncs/error.c:329,350 */
const char *vb200_error_buffer(void);
void vb200_error_clear(void);
/* reference: vips_vector_isenabled(), iofuncs/vector.cpp:98-110 */
int vb200_isenabled(void);
/* The CUDA stream (cudaStream_t) device-resident calls are queued on, per
 * calling thread; NULL = the legacy default stream.  Host-image calls use the
 * library's own staging streams.
 */
void vb200_set_stream(void *cuda_stream);
void *vb200_get_stream(void);
/* reference: --vips-tile-width/--vips-tile-height/--vips-fatstrip-height/
 * --vips-thinstrip-height, iofuncs/init.c:893-905, thread.c:74-77.  The tile
 * geometry decides the rects generate() sees and therefore the sequential
 * coordinate stepping of reducev/reduceh (reducev.cpp:548-611).
 */
void vb200_set_tile_geometry(int tile_width, int tile_height, int fatstrip_height, int thinstrip_height);
/* Number of kernels this library has launched in this process. */
uint64_t vb200_launch_count(void);
void vb200_image_free(VB200Image *image);
size_t vb200_format_sizeof(int band_format);

/* ------------------------------------------------- resample: whole-image ops
 *
 * in->where selects host or device pixels.  If out->data is NULL the library
 * allocates it in the same memory space (free with vb200_image_free); otherwise
 * out->data/out->bpl are used as given and must be large enough.  The rest of
 * *out is filled in.
 */

/* reference: vips_shrinkv()/vips_shrinkh(), resample/shrinkv.c:474, shrinkh.c:357 */
int vb200_shrinkv(const VB200Image *in, VB200Image *out, int vshrink, int ceil_mode);
int vb200_shrinkh(const VB200Image *in, VB200Image *out, int hshrink, int ceil_mode);
/* reference: vips_reducev()/vips_reduceh(), resample/reducev.cpp:859, reduceh.cpp:396 */
int vb200_reducev(const VB200Image *in, VB200Image *out, double vshrink, int kernel, double gap);
int vb200_reduceh(const VB200Image *in, VB200Image *out, double hshrink, int kernel, double gap);
/* reference: vips_reduce(), resample/reduce.c:97-119 (reducev then reduceh) */
int vb200_reduce(const VB200Image *in, VB200Image *out, double hshrink, double vshrink, int kernel, double gap);
/* reference: vips_resize(), resample/resize.c:135-311.  gap < 0 = default 2.0 */
int vb200_resize(const VB200Image *in, VB200Image *out, double scale, double vscale, int kernel, double gap);
/* reference: vips_premultiply()/vips_unpremultiply(), conversion/premultiply.c:215,
 * unpremultiply.c:272.  max_alpha <= 0 = vips_interpretation_max_alpha(in->Type).
 */
int vb200_premultiply(const VB200Image *in, VB200Image *out, double max_alpha, int uchar_mode);
int vb200_unpremultiply(const VB200Image *in, VB200Image *out, double max_alpha, int uchar_mode);
/* reference: vips_thumbnail_image(), resample/thumbnail.c:2000 (image source,
 * no ICC, no crop/rotate).  height <= 0 = width.
 */
int vb200_thumbnail_image(const VB200Image *in, VB200Image *out, int width, int height, int size, int linear);

/* ------------------------------------------------------------------ colour
 *
 * reference: vips_colourspace(), colour/colourspace.c:551-617.  The source
 * space is in->Type.  Routes among sRGB (uchar), RGB16 (ushort), scRGB, XYZ,
 * LAB, LCH, YXY (float) and LABS (short) run as ONE fused kernel; every reference step
 * (sRGB2scRGB, scRGB2XYZ, XYZ2Lab, Lab2LabS, LabS2Lab, Lab2XYZ, XYZ2scRGB,
 * scRGB2sRGB, Lab2LCh, LCh2Lab, XYZ2Yxy, Yxy2XYZ) keeps its own arithmetic (the two LCh steps call
 * atan / cosf / sinf: float results within 1 ULP of the reference's glibc; everything else is exact).  Bands beyond the third are carried
 * as vips_colour_build does (colour.c:196-291).  sRGB <-> RGB16 are the reference's two rows that are not colour
 * conversions (colourspace.c:85-110, 372, 420): a shifting vips_cast over every band, alpha included (cast.c:137-164).
 * B_W (uchar), GREY16 (ushort) and HSV (uchar) as source or target run the table's rows for them (BW2sRGB /
 * GREY162RGB16 / HSV2sRGB first, scRGB2BW / sRGB2HSV last: colour_ext.cu) as the leaf kernel(s) plus the fused route
 * kernel between; sRGB / RGB16 / scRGB -> B_W / GREY16 is a single launch.  B_W / GREY16 sources gain two bands,
 * targets lose two.  All exact.
 */
int vb200_colourspace(const VB200Image *in, VB200Image *out, int space);

/* ------------------------------------------------------------- convolution
 *
 * A mask is what the reference passes as a VipsImage matrix: width x height
 * doubles, row-major, plus the "scale" and "offset" metadata
 * (reference: vips_check_matrix, vips_image_get_scale/offset).
 */
typedef struct {
	int width;
	int height;
	const double *coeff;
	double scale;
	double offset;
} VB200Mask;

/* reference: vips_conv(), convolution/conv.c:60-121.  precision FLOAT ->
 * vips_convf (double accumulate, float out); INTEGER -> vips_convi (exact
 * int64 C path; see vb200_set_vector_convi).  APPROXIMATE (conva) returns -1.
 */
int vb200_conv(const VB200Image *in, VB200Image *out, const VB200Mask *mask, int precision);
/* reference: vips_convsep(), convolution/convsep.c:61-114 (mask is n x 1 or 1 x n) */
int vb200_convsep(const VB200Image *in, VB200Image *out, const VB200Mask *mask, int precision);
/* reference: vips_gaussblur(), convolution/gaussblur.c:70-114.  min_ampl <= 0 = 0.2 */
int vb200_gaussblur(const VB200Image *in, VB200Image *out, double sigma, double min_ampl, int precision);
/* reference: vips_gaussmat(), create/gaussmat.c:93-170.  Allocates out->coeff
 * (free with vb200_mask_free).
 */
int vb200_gaussmat(VB200Mask *out, double sigma, double min_ampl, int separable, int precision);
void vb200_mask_free(VB200Mask *mask);
/* reference: vips_sharpen(), convolution/sharpen.c:171-303
 * (defaults sigma 0.5, x1 2, y2 10, y3 20, m1 0, m2 3)
 */
int vb200_sharpen(const VB200Image *in, VB200Image *out, double sigma, double x1, double y2, double y3, double m1,
	double m2);
/* vips_sharpen over a batch of same-shaped packed 8-bit sRGB frames (3 or 4 bands) resident on the
 * device, as ONE fused kernel (sRGB -> LabS, separable integer blur of L, the sharpen LUT, LabS -> sRGB;
 * nothing but the input and the output touches HBM): the second stage of the thumbnail + sharpen stream.
 * Frame i at in + i * in_frame_stride; in and out must not overlap.  Queued on the caller's stream.
 */
int vb200_sharpen_batch_device(const void *in, size_t in_frame_stride, void *out, size_t out_frame_stride, int n_frames, int width,
	int height, int bands, double sigma, double x1, double y2, double y3, double m1, double m2);
/* 0 (default): uchar INTEGER convolutions use the exact C arithmetic
 * (vips_convi_gen, what a --vips-novector / non-Highway build runs).
 * 1: they use the Highway arithmetic (8-bit mantissa + shared exponent,
 * convi.c:931-1119, convi_hwy.cpp:265-273) whenever vips_convi_intize accepts
 * the mask, like a Highway build with vips_vector_isenabled().
 */
void vb200_set_vector_convi(int on);

/* ------------------------------------------- resample: generate()-shaped ops
 *
 * reference: VipsGenerateFn, include/vips/image.h:151-154.  Fill out->valid
 * from the input region, which must cover the rect the reference generate
 * function would vips_region_prepare() (reducev.cpp:539-544 etc.) on the
 * EMBEDDED input image.  Host pointers; staged through the device.
 */
typedef struct {
	int n_point;
	int kernel;
	double residual_shrink; /* residual_vshrink / residual_hshrink */
	double offset;			/* voffset / hoffset */
} VB200ReduceParams;

int vb200_reducev_gen(const VB200Region *out, const VB200Region *in, const VB200ReduceParams *params);
int vb200_reduceh_gen(const VB200Region *out, const VB200Region *in, const VB200ReduceParams *params);
int vb200_shrinkv_gen(const VB200Region *out, const VB200Region *in, int vshrink);
int vb200_shrinkh_gen(const VB200Region *out, const VB200Region *in, int hshrink);
/* convolution and colour in the same shape.  conv: regions are on the EMBEDDED image and `in`
 * covers {left, top, width + mask->width - 1, height + mask->height - 1} of out->valid
 * (replaces vips_convf_gen convf.c:185-282 / vips_convi_gen convi.c:752-852; the arithmetic is
 * vb200_conv's).  colour: `in` covers out->valid, in->im.Type is the source space (replaces
 * vips_colour_gen colour.c:119-156 over the route of vips_colourspace_build colourspace.c:551-617).
 */
int vb200_conv_gen(const VB200Region *out, const VB200Region *in, const VB200Mask *mask, int precision);
int vb200_colour_gen(const VB200Region *out, const VB200Region *in, int space);

/* -------------------------------------------- resample: scanline kernel seam
 *
 * reference: resample/presample.h:74-87.  Same names, same signatures: a
 * replacement .so can be linked in place of the Highway objects.  Host
 * pointers; each call stages its scanlines through the device.
 */
void vips_reducev_uchar_hwy(uint8_t *pout, uint8_t *pin, int n, int ne, int lskip, const short *k);
void vips_reduceh_uchar_hwy(uint8_t *pout, uint8_t *pin, int n, int width, int bands, short *cs[65], double X,
	double hshrink);
void vips_shrinkh_uchar_hwy(uint8_t *pout, uint8_t *pin, int width, int hshrink, int bands);
void vips_shrinkv_add_line_uchar_hwy(uint8_t *pin, int ne, unsigned int *sum);
void vips_shrinkv_write_line_uchar_hwy(uint8_t *pout, int ne, int vshrink, unsigned int *sum);

/* ------------------------------------------------ thumbnail: batched stream
 *
 * The CUDA-stream tile pump that replaces vips_sink_memory + vips_threadpool_run
 * (reference: iofuncs/sinkmemory.c:324, threadpool.c:625) for a batch of
 * same-shaped frames: one fused kernel per op chain
 * premultiply -> shrinkv -> reducev -> shrinkh -> reduceh -> unpremultiply.
 */
typedef struct VB200ThumbnailPlan VB200ThumbnailPlan;

VB200ThumbnailPlan *vb200_thumbnail_plan_new(int width, int height, int bands, int band_format, int has_alpha,
	int target_width, int target_height, int size, int linear);
void vb200_thumbnail_plan_free(VB200ThumbnailPlan *plan);
int vb200_thumbnail_plan_output(const VB200ThumbnailPlan *plan, int *out_width, int *out_height);
/* Frames are contiguous: frame i at in + i * in_frame_stride bytes. */
int vb200_thumbnail_batch_device(VB200ThumbnailPlan *plan, const void *in, size_t in_frame_stride, void *out,
	size_t out_frame_stride, int n_frames);
/* Host frames (pinned or pageable); H2D / kernel / D2H overlapped on the
 * library's streams.  Returns after the last output frame has landed.
 */
int vb200_thumbnail_batch_host(VB200ThumbnailPlan *plan, const void *in, size_t in_frame_stride, void *out,
	size_t out_frame_stride, int n_frames);
/* Append vips_sharpen (convolution/sharpen.c:171-303) to every batch call of the plan: the fused
 * thumbnail kernel writes into a device scratch batch, vb200_sharpen_batch_device's kernel reads it and
 * writes the caller's output -- BASELINE config 5's "thumbnail + sharpen + sRGB" stream, two kernels per
 * batch.  sigma <= 0 switches it off again.  Needs 3- or 4-band frames.
 */
int vb200_thumbnail_plan_set_sharpen(VB200ThumbnailPlan *plan, double sigma, double x1, double y2, double y3, double m1, double m2);
/* 1 if the plan runs the single fused kernel, 0 if it chains the leaf kernels
 * (other band counts, one-axis shrinks, or a window that does not fit on chip).
 */
int vb200_thumbnail_plan_is_fused(const VB200ThumbnailPlan *plan);
/* Algorithmic HBM bytes one frame moves through the fused kernel. */
size_t vb200_thumbnail_plan_bytes_per_frame(const VB200ThumbnailPlan *plan);
/* Which kernel a batch call of this plan launches (for bench / profile labels): a
 * static string such as "thumbnail_fused_mma_kernel<VS=4,NP=6,premul,HS=4,cols=384,cpt=1>",
 * or "leaf kernels" for an unfused plan.
 */
const char *vb200_thumbnail_plan_kernel(const VB200ThumbnailPlan *plan);

/* test hook, host only: the sRGB <-> HSV per-pixel code of colour_ext.cu on the CPU; n pixels of 3 bytes */
int vb200_debug_hsv_host(const void *in, size_t n, int to_hsv, void *out);

/* ------------------------------------------------------------ flatten (SURVEY 8f rank 3)
 * reference: vips_flatten(), conversion/flatten.c:605-616 (build :421-529; generate functions :170-419).  Blends the
 * last band (alpha) out against `background` (n = 1 or bands - 1 values; NULL / n = 0: black): bands - 1 bands out, same
 * format.  max_alpha <= 0: the interpretation's default (255, 65535 for RGB16 / GREY16, 1 for scRGB).  One-band images are
 * copied.  uchar .. float images; the integer cases where the reference's own arithmetic is undefined C (see flatten.cu)
 * return -1 and stay on the host.
 */
int vb200_flatten(const VB200Image *in, VB200Image *out, const double *background, int n, double max_alpha);
/* test hook, host only: flatten.cu's per-pixel code on the CPU (packed arrays); x4: the four-pixels-per-thread form */
int vb200_debug_flatten_host(const void *in, int width, int height, int bands, int band_format, int interpretation,
	const double *background, int n, double max_alpha, int x4, void *out);

/* ------------------------------------------------------------ morphology (SURVEY 8f rank 4)
 * reference: vips_morph(), morphology/morph.c:1030-1042 (generate functions :657-826; the Highway kernels
 * morph_hwy.cpp give the same bytes).  mask elements 0 / 128 (do not care) / 255; uchar images.
 */
enum { VB200_MORPHOLOGY_ERODE = 0, VB200_MORPHOLOGY_DILATE = 1 };
int vb200_morph(const VB200Image *in, VB200Image *out, const VB200Mask *mask, int morph);
/* reference: vips_rank(), morphology/rank.c:623-635 (build :458-525, generate :414-456: histogram / select / max / min
 * loops, all "the index-th smallest element of the width x height window", per band; the window is centred at
 * (width / 2, height / 2), edges replicated); vips_median(), :651-664 = rank(size, size, size * size / 2).
 * uchar .. float images.  Errors as the reference: "window too large", "index out of range".
 */
int vb200_rank(const VB200Image *in, VB200Image *out, int width, int height, int index);
int vb200_median(const VB200Image *in, VB200Image *out, int size);
/* test hook, host only: rank.cu's staging + select code run tile by tile on the CPU (packed arrays) */
int vb200_debug_rank_host(const void *in, int width, int height, int bands, int band_format, int rank_width, int rank_height,
	int index, void *out);

/* ------------------------------------------------- unfused graphs: the chain pump (SURVEY 8f rank 2)
 *
 * What vips_sink_memory + vips_threadpool_run (iofuncs/sinkmemory.c:324, threadpool.c:625) do for an
 * arbitrary graph of operations: a VB200Chain is a list of the operations above; vb200_chain_run_host
 * runs it over a batch of host images with upload / compute / download of consecutive images overlapped on
 * three streams, every intermediate staying on the device.  Each step is the stand-alone entry point's own
 * device function: same pixels as calling vb200_resize(), vb200_conv() ... one by one, without their
 * per-call host round trips.  in[i] / out[i] are arrays of n_images; out[i].data == NULL -> allocated
 * (vb200_image_free).  Pinned host memory (vb200_host_alloc) lets the phases overlap.
 */
typedef struct VB200Chain VB200Chain;
VB200Chain *vb200_chain_new(void);
void vb200_chain_free(VB200Chain *chain);
int vb200_chain_add_resize(VB200Chain *chain, double scale, double vscale, int kernel, double gap);
int vb200_chain_add_reduce(VB200Chain *chain, double hshrink, double vshrink, int kernel, double gap);
int vb200_chain_add_colourspace(VB200Chain *chain, int space);
int vb200_chain_add_conv(VB200Chain *chain, const VB200Mask *mask, int precision);
int vb200_chain_add_convsep(VB200Chain *chain, const VB200Mask *mask, int precision);
int vb200_chain_add_gaussblur(VB200Chain *chain, double sigma, double min_ampl, int precision);
int vb200_chain_add_sharpen(VB200Chain *chain, double sigma, double x1, double y2, double y3, double m1, double m2);
int vb200_chain_add_premultiply(VB200Chain *chain, double max_alpha, int uchar_mode);
int vb200_chain_add_unpremultiply(VB200Chain *chain, double max_alpha, int uchar_mode);
int vb200_chain_add_morph(VB200Chain *chain, const VB200Mask *mask, int morph);
int vb200_chain_add_rank(VB200Chain *chain, int width, int height, int index);
int vb200_chain_add_flatten(VB200Chain *chain, const double *background, int n, double max_alpha);
int vb200_chain_run_host(VB200Chain *chain, const VB200Image *in, VB200Image *out, int n_images);

/* ------------------------------------------------------------------ ICC (SURVEY 8a a20)
 * vips_icc_import / vips_icc_export / vips_icc_transform (colour/icc_transform.c:813-945, :995-1117,
 * :1166-1220) with the profile passed as a memory blob (what vips_icc_load_profile_blob hands lcms2).
 * The reference's arithmetic is lcms2's; this is a from-specification ICC evaluator whose parity is
 * pinned to lcms2 2.18 within a tolerance (tests/test_icc.py), not bit for bit.  Supported: RGB
 * matrix/TRC, grey TRC, lut8 / lut16 (e.g. CMYK) and v4 lutAtoB / lutBtoA profiles; intent VB200_INTENT_RELATIVE (the
 * reference's default), and PERCEPTUAL / SATURATION for matrix / grey profiles with a zero black point (where
 * lcms2's black point compensation is the identity), and ABSOLUTE for matrix / TRC profiles (lcms2's media-white scale,
 * folded into the colorant matrix); depth 8 or 16;
 * bands after the profile's channels ride along as in vips_colour_build.  Everything else (the other
 * intents, black point compensation) returns -1: keep the host path.
 */
enum { VB200_INTENT_PERCEPTUAL = 0, VB200_INTENT_RELATIVE = 1, VB200_INTENT_SATURATION = 2, VB200_INTENT_ABSOLUTE = 3 };
enum { VB200_PCS_LAB = 0, VB200_PCS_XYZ = 1 };
int vb200_icc_import(const VB200Image *in, VB200Image *out, const void *profile, size_t profile_len, int intent, int pcs);
int vb200_icc_export(const VB200Image *in, VB200Image *out, const void *profile, size_t profile_len, int intent, int depth,
	int pcs);
int vb200_icc_transform(const VB200Image *in, VB200Image *out, const void *in_profile, size_t in_len,
	const void *out_profile, size_t out_len, int intent, int depth);
/* Test hook, host only: the evaluator's per-pixel code on the CPU over n packed pixels
 * (mode 0 import, 1 export, 2 transform; pa / pb = the profile(s)); returns the output band count.
 */
int vb200_debug_icc_eval(int mode, const void *in, int in_fmt, int in_bands, void *out, int n, const void *pa, size_t la,
	const void *pb, size_t lb, int intent, int depth, int pcs);

/* Test hook, host only (no GPU, no CUDA call): the reducev geometry, sampling table and
 * tensor-pipe tables of a vertical thumbnail shrink exactly as a plan builds them, so that the CPU
 * test suite can replay the MMA arithmetic over them (tests/test_mma_tables.py).  Caller-sized arrays:
 * first / phase [cap_rows], mask65 [65 * n_point] shorts, vchunk [2 * chunks], bfrag [128 * chunks]
 * with chunks = ceil(out_size / *rows_per_chunk) (the largest of 8 .. 4 rows whose windows fit).  0 = ok, 1 = window does not fit the quad ring, -1 = bad arguments.
 */
int vb200_debug_mma_tables(int in_size, double shrink, int rect_size, int *int_shrink, int *shrunk_size, int *out_size,
	int *n_point, int *embed, int *first, int *phase, short *mask65, int *vchunk, unsigned *bfrag, int cap_rows,
	int *rows_per_chunk);

/* ------------------------------------------------------------------ JPEG decode staging (SURVEY 8f rank 1)
 * vips_jpegload_buffer(buf, len, &out, "shrink", shrink) (foreign/jpeg2vips.c:532-538, 631-640: scale_num = 1,
 * scale_denom = shrink, output cropped to floor(size / shrink)) with the decoder on the device: the compressed
 * bytes are all that crosses PCIe.  libjpeg(-turbo) itself is a third-party dependency outside the reference
 * tree; its algorithm for the reference's configuration (JDCT_ISLOW, 8-bit Huffman, sequential and progressive)
 * is restated in csrc/jpeg.cu and pinned bit for bit to the libjpeg-turbo inside this image's Pillow
 * (tests/test_jpeg.py).  Decoded: 8-bit Huffman streams, baseline / extended sequential and progressive, greyscale or
 * YCbCr at 4:4:4, 4:2:2 and 4:2:0, at shrink 1 / 2 / 4 / 8 (where libjpeg's upsampler has work left -- 4:2:0 at full
 * size, 4:2:2 -- its h2v2 / h2v1 "fancy" triangle filters, jdsample.c).  Arithmetic-coded, 12-bit, CMYK / RGB-coded and
 * 4:4:0 / 4:1:1 streams return -1 (host loader).  Baseline streams with restart markers decode one interval per GPU
 * thread, those without by self-synchronising subsequences; progressive streams one scan after the other.
 *
 * vb200_jpeg_decode_batch: n streams of ONE output geometry -> out[n][height][width][bands] uchar (bands 1 or 3),
 *   out in host or device memory (out_location VB200_HOST / VB200_DEVICE); out = NULL only reports the geometry.
 * vb200_jpegload_buffer: one stream into a VB200Image (allocate-or-fill like every op).
 * vb200_thumbnail_jpegshrink: the load-time shrink vips_thumbnail picks (resample/thumbnail.c:489-517).
 * vb200_thumbnail_plan_run_jpeg: decode at `shrink` + the plan's thumbnail chain, frames never leave the device;
 *   the plan must have been made for the decoded geometry (3 bands).
 * vb200_debug_jpeg_decode: test hook, host only -- the same per-block code on the CPU.
 */
int vb200_jpeg_decode_batch(const void *const *bufs, const size_t *lens, int n, int shrink, void *out, int out_location,
	size_t out_bpl, size_t out_frame_stride, int *width, int *height, int *bands);
int vb200_jpegload_buffer(const void *buf, size_t len, int shrink, VB200Image *out);
int vb200_thumbnail_jpegshrink(int width, int height, int target_width, int target_height, int size);
/* vips_thumbnail_buffer(buf, len, &out, width, "height", height, "size", size, NULL) for a JPEG stream (thumbnail.c:583-613,
 * 848-902): load-time shrink by vb200_thumbnail_jpegshrink, decode and thumbnail on the device; out: allocate-or-fill */
int vb200_thumbnail_buffer(const void *buf, size_t len, VB200Image *out, int width, int height, int size);
int vb200_thumbnail_plan_run_jpeg(VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, int shrink,
	void *out, int out_location, size_t out_frame_stride);
int vb200_debug_jpeg_decode(const void *buf, size_t len, int shrink, void *out, size_t out_bpl, int *width, int *height,
	int *bands);
/* test hook, host only: the self-synchronising decode of a scan without restart markers (subsequences of sub_bytes,
 * max_passes passes), *passes_used = the last pass that changed a record */
int vb200_debug_jpeg_decode_sync(const void *buf, size_t len, int shrink, int sub_bytes, int max_passes, void *out, size_t out_bpl,
	int *width, int *height, int *bands, int *passes_used);
/* vips_jpegsave_buffer (foreign/vips2jpeg.c:551-700: jpeg_set_quality(Q, TRUE), chroma subsampled 2 x 2 below Q 90 unless
 * subsample_mode says otherwise -- 0 auto, 1 on, 2 off --, baseline, standard Huffman tables, JFIF header) for n equally sized
 * 8-bit frames of 1 or 3 bands, encoded on the device (csrc/jpeg_encode.cu): the streams are libjpeg-turbo's byte for byte
 * (tests/test_jpeg_encode.py).  frames / out in host or device memory; stream i at out + i * out_stride, lengths[i] bytes
 * (host array); -1 when a stream does not fit its stride.
 */
int vb200_jpegsave_batch(const void *frames, int frames_location, size_t bpl, size_t frame_stride, int n, int width, int height, int bands,
	int Q, int subsample_mode, void *out, int out_location, size_t out_stride, size_t *lengths);
/* test hook, host only: vips_jpegsave_buffer's stream (csrc/jpeg_encode.cu) through the encoder's per-block code on the CPU.
 * subsample_mode: 0 auto (4:2:0 below Q 90, vips2jpeg.c:676-690), 1 on, 2 off.  *len = bytes written */
int vb200_debug_jpeg_encode(const void *pixels, size_t bpl, int width, int height, int bands, int quality, int subsample_mode, void *out,
	size_t cap, size_t *len);
/* with env VB200_JPEG_TIMING: CUDA-event times of jpeg_huffman_kernel / jpeg_idct_kernel over the calling thread's last decode */
void vb200_debug_jpeg_times(float *huffman_ms, float *idct_ms);

/* Pinned host memory for the pump: page-locked and, on a multi-socket machine, placed on the NUMA
 * node the current device hangs off (falls back to cudaHostAlloc).  vb200_device_numa_node():
 * that node, or -1 (unknown / single node).
 */
void *vb200_host_alloc(size_t bytes);
void vb200_host_free(void *p);
int vb200_device_numa_node(void);

#ifdef __cplusplus
}
#endif

#endif /* VB200_H */
