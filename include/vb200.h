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
	VB200_INTERPRETATION_HISTOGRAM = 10,
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
 *
 * Strides and alignment (every whole-image op below, colour, convolution, ICC,
 * flatten and morphology too): bpl = 0 means packed rows; a non-zero bpl smaller
 * than Xsize * Bands * vb200_format_sizeof(BandFmt) is an error.  A VB200_DEVICE
 * image is read in place, so its data and bpl must both be multiples of the
 * element size (any byte for uchar / char, 2 for ushort / short, 4 for uint / int
 * / float); otherwise the call fails before any launch.  Padded strides and bases
 * off a 4- or 16-byte grid are accepted and give the same pixels: the vector
 * kernels are used only where the layout allows them.  A caller's output buffer
 * may have any base and stride at least a line long; one off the result's element
 * grid is filled by a copy rather than written by the kernel.
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
 * no colour management (see vb200_thumbnail_image_icc), no crop/rotate).  height <= 0 = width.
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
 * static string such as "thumbnail_fused_mma_kernel<VS=4,NP=6,premul,HS=4,cols=768,cpt=2>",
 * or "leaf kernels" for an unfused plan.  The template arguments are those of the instantiation
 * that launches: "VS=0(13)" is the run-time-box form running box 13.  The plan chooses the kernel
 * once; the one exception is a batch whose base pointer, or whose frame stride (with more than
 * one frame), is not a multiple of 16 bytes: it runs thumbnail_fused_kernel (the ld.global kernel)
 * with the same pixels.
 */
const char *vb200_thumbnail_plan_kernel(const VB200ThumbnailPlan *plan);

/* ------------------------------------------------ thumbnail: colour management
 *
 * vips_thumbnail's "input_profile" / "output_profile" / "intent" in non-linear mode (resample/thumbnail.c:733-735,
 * 929-970).  With an output profile, each frame after the resize runs one of:
 *   - vips_icc_transform(output_profile, input_profile, embedded = TRUE, depth 8) when the frame embeds a profile or
 *     input_profile is set.  Its input profile is chosen as vips_icc_set_import does (colour/icc_transform.c:692-752):
 *     the embedded profile, then input_profile, then the built-in one for the frame's interpretation (sRGB for 3+ bands,
 *     grey below).  A profile lcms2 would not open, or whose colour space has the wrong band count, is skipped.
 *   - vips_colourspace(XYZ) then vips_icc_export(output_profile, depth 8) when there is neither.
 * Profiles are memory blobs (what vips_profile_load / vips_image_get_blob hand on).  The library ships no profile data:
 * the caller passes the built-in "srgb" / "sgrey" profiles, needed only when selection reaches them.  A transform the
 * device evaluator declines (see the ICC section) fails the call with -1, the error naming the frame: keep the host path.
 * Output bands follow the output profile (grey -> 1, RGB -> 3, CMYK -> 4) plus the frame's extra bands (alpha).
 * Frames are 8-bit sRGB (3+ bands) or B_W (1 / 2 bands), the thumbnail plan's interpretations: vb200_thumbnail_image_icc
 * returns -1 for an image of any other interpretation (a CMYK image, say, which the reference imports with its CMYK profile).
 */
typedef struct {
	const void *input_profile;	/* thumbnail "input_profile"; NULL = none */
	size_t input_len;
	const void *output_profile; /* thumbnail "output_profile"; NULL = colour management off */
	size_t output_len;
	const void *builtin_rgb; /* vips_profile_load("srgb"): last resort of the selection for 3+ band frames */
	size_t builtin_rgb_len;
	const void *builtin_grey; /* vips_profile_load("sgrey"): the same for 1 / 2 band frames */
	size_t builtin_grey_len;
	int intent; /* VB200_INTENT_*; vips_thumbnail's default is RELATIVE */
} VB200ThumbnailIcc;

/* The ICC stage runs after the thumbnail kernel and before the sharpen stage.  NULL, or a NULL output profile: off.
 * The profiles are copied.  Not available with linear = 1 (-1): see vb200_thumbnail_plan_set_linear_icc.
 */
int vb200_thumbnail_plan_set_icc(VB200ThumbnailPlan *plan, const VB200ThumbnailIcc *icc);
/* bands of an output frame: the plan's bands, or what the output profile makes of them */
int vb200_thumbnail_plan_output_bands(const VB200ThumbnailPlan *plan);
/* the batch calls with each frame's embedded profile (arrays of n_frames; NULL arrays or a NULL / 0-length entry: none) */
int vb200_thumbnail_batch_device_icc(VB200ThumbnailPlan *plan, const void *in, size_t in_frame_stride, void *out,
	size_t out_frame_stride, int n_frames, const void *const *embedded, const size_t *embedded_lens);
int vb200_thumbnail_batch_host_icc(VB200ThumbnailPlan *plan, const void *in, size_t in_frame_stride, void *out,
	size_t out_frame_stride, int n_frames, const void *const *embedded, const size_t *embedded_lens);
/* vips_thumbnail_image with colour management; icc NULL = vb200_thumbnail_image.  embedded: the image's ICC blob */
int vb200_thumbnail_image_icc(const VB200Image *in, VB200Image *out, int width, int height, int size, const VB200ThumbnailIcc *icc,
	const void *embedded, size_t embedded_len);
/* vips_thumbnail_buffer with colour management: the embedded profile comes from the stream's APP2 segments */
int vb200_thumbnail_buffer_icc(const void *buf, size_t len, VB200Image *out, int width, int height, int size,
	const VB200ThumbnailIcc *icc);
/* ------------------------------------------------ thumbnail: colour-managed linear-light thumbnails
 *
 * vips_thumbnail(..., linear = TRUE) with "input_profile" / "output_profile" / "intent" (resample/thumbnail.c:766-805, 929-987)
 * for 8-bit sRGB frames of 3+ bands.  Unlike the non-linear mode, an embedded profile alone turns colour management on.  Per frame:
 *   - a profile to import with (the embedded one, input_profile or the built-in sRGB profile, chosen as above): vips_icc_import
 *     to float XYZ, float premultiply / resize / unpremultiply with max_alpha 255, vips_icc_export(depth 8) to output_profile --
 *     or, with no output profile, to the profile the import used.  One that cannot serve as an output profile: -1, as the
 *     reference's "no output profile".
 *   - no embedded profile and no input_profile, but an output profile: the plain linear chain, vips_colourspace(scRGB -> XYZ),
 *     then vips_icc_export(output_profile, depth 8).
 *   - neither: the plain linear thumbnail, unchanged.
 * The import runs inside the linear thumbnail's vertical kernel and the export inside its horizontal kernel.  Output bands
 * follow the export's profile plus alpha.  1- / 2-band frames, 16-bit frames and other interpretations return -1.
 */
/* Linear plans only (-1 otherwise); NULL: off.  A struct with output_profile NULL: frames with a profile to import with export
 * to that profile, the others run the plain path.  The profiles are copied and checked here.
 */
int vb200_thumbnail_plan_set_linear_icc(VB200ThumbnailPlan *plan, const VB200ThumbnailIcc *icc);
/* vips_thumbnail_image(..., linear = TRUE) with colour management; icc NULL = vb200_thumbnail_image(linear = 1) */
int vb200_thumbnail_image_linear_icc(const VB200Image *in, VB200Image *out, int width, int height, int size,
	const VB200ThumbnailIcc *icc, const void *embedded, size_t embedded_len);
/* vips_thumbnail_buffer(..., linear = TRUE): decoded at full size (thumbnail.c:496-499), the embedded profile from the
 * stream's APP2 segments
 */
int vb200_thumbnail_buffer_linear_icc(const void *buf, size_t len, VB200Image *out, int width, int height, int size,
	const VB200ThumbnailIcc *icc);
/* Test hook, host only: one frame's linear-mode choice.  *branch 0 plain, 1 import + export, 2 XYZ export; *source as
 * vb200_debug_icc_select (-1: no import); *export_from 0 output_profile, 1 the import's profile, -1 no export.  -1: error.
 */
int vb200_debug_icc_select_linear(const VB200ThumbnailIcc *icc, int bands, const void *embedded, size_t embedded_len,
	int *branch, int *source, int *export_from);

/* vips_image_get_blob(VIPS_META_ICC_NAME) of a JPEG stream (foreign/jpeg2vips.c:699-799): the APP2 "ICC_PROFILE" chunks
 * before the first SOS, by sequence number 1 .. 100, concatenated up to the first missing one.  Host only, no GPU.
 * 0 with *profile_len = 0: no profile; out = NULL only reports the length; -1 when cap is too small or the stream is
 * not a JPEG.
 */
int vb200_jpeg_icc_profile(const void *buf, size_t len, void *out, size_t cap, size_t *profile_len);

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

/* ------------------------------------------------------------ histograms
 * reference: vips_hist_find(), arithmetic/hist_find.c:471-482 (band -1: every band; else that band alone).  uchar and
 * ushort images (others: cast first).  The result is (mx + 1) x 1, one band per scanned band, UINT, interpretation
 * HISTOGRAM: a uchar histogram of every band is 256 wide, every other one as wide as its largest value plus one.  Images
 * of 2^32 or more pixels (the reference's DOUBLE histogram) are refused.  A bad band: "bandno must be -1, or less than n".
 */
int vb200_hist_find(const VB200Image *in, VB200Image *out, int band);
/* reference: vips_hist_equal(), histogram/hist_equal.c:156-167: hist_find -> hist_cum -> hist_norm -> cast -> maplut, the
 * LUT built on the device.  uchar and ushort images; band as hist_find (a one-band LUT then maps every band).
 */
int vb200_hist_equal(const VB200Image *in, VB200Image *out, int band);
/* reference: vips_hist_local(), histogram/hist_local.c:417-428 (build :283-306, generate :133-250): contrast-limited local
 * equalisation over a width x height window (max_slope > 0: CLAHE; sharp's clahe()).  uchar images; errors as the
 * reference ("image must be uchar", "window too large"), and windows of more than 8 388 607 pixels, whose int sums
 * overflow in the reference, are refused.
 */
int vb200_hist_local(const VB200Image *in, VB200Image *out, int width, int height, int max_slope);
/* test hooks, host only: histogram.cu's hist_local staging, window update and element arithmetic run tile by tile on the
 * CPU (packed uchar arrays; staged -1: as planned, 0 / 1: forced), and hist_equal's LUT from an n_bands x width uint32
 * histogram (band-major) into n_bands x width entries of band_format (uchar or ushort)
 */
int vb200_debug_hist_local_host(const void *in, int width, int height, int bands, int window_width, int window_height,
	int max_slope, int staged, void *out);
int vb200_debug_hist_equal_lut_host(const unsigned *hist, int width, int n_bands, int band_format, void *lut);

/* ------------------------------------------------- unfused graphs: the chain pump (SURVEY 8f rank 2)
 *
 * What vips_sink_memory + vips_threadpool_run (iofuncs/sinkmemory.c:324, threadpool.c:625) do for an
 * arbitrary graph of operations: a VB200Chain is a list of the operations above; vb200_chain_run_host
 * runs it over a batch of host images with upload / compute / download of consecutive images overlapped on
 * three streams, every intermediate staying on the device.  vb200_chain_add_<op>() takes the arguments of
 * vb200_<op>(), applies the same defaults and refuses what it refuses without an image (a missing or empty mask,
 * a convsep mask that is not 1xn or nx1, a reduce factor below 1) with the same reason; the step then runs the
 * stand-alone op's own device code: same pixels as calling vb200_resize(), vb200_conv() ... one by one, without
 * their per-call host round trips.  in[i] / out[i] are arrays of n_images; out[i].data == NULL -> allocated
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
int vb200_chain_add_hist_find(VB200Chain *chain, int band);
int vb200_chain_add_hist_equal(VB200Chain *chain, int band);
int vb200_chain_add_hist_local(VB200Chain *chain, int width, int height, int max_slope);
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
 * (mode 0 import, 1 export, 2 transform, 3 vips_colourspace(XYZ) of 8-bit sRGB (3+ bands) or B_W (1 / 2 bands) then
 * export with the XYZ PCS -- the thumbnail's branch without an input profile; pa / pb = the profile(s));
 * returns the output band count.
 */
int vb200_debug_icc_eval(int mode, const void *in, int in_fmt, int in_bands, void *out, int n, const void *pa, size_t la,
	const void *pb, size_t lb, int intent, int depth, int pcs);
/* Test hooks, host only: the thumbnail's input-profile selection for one frame (0: transform with the profile *source names,
 * 0 embedded / 1 input_profile / 2 built-in; 1: no input profile, the XYZ export; -1: error), and its per-profile check
 * (0 usable, 1 skipped as the reference skips it, 2 kept by the reference with the header's intent instead).
 */
int vb200_debug_icc_select(const VB200ThumbnailIcc *icc, int bands, const void *embedded, size_t embedded_len, int *source);
int vb200_debug_icc_classify(const void *profile, size_t len, int want_bands, int intent);
/* with env VB200_ICC_TIMING set: CUDA-event milliseconds of the calling thread's last ICC stage of a thumbnail plan
 * (its icc_frames_kernel launches, from the first to the last); -1 when none was timed
 */
float vb200_debug_icc_stage_ms(void);
/* with env VB200_LINEAR_TIMING set: CUDA-event milliseconds of the calling thread's last two-kernel linear thumbnail call
 * (from before its first linear_v launch to after its last linear_h launch); -1 when none was timed
 */
float vb200_debug_linear_thumb_ms(void);

/* Test hook, host only (no GPU, no CUDA call): the reducev geometry, sampling table and
 * tensor-pipe tables of a vertical thumbnail shrink exactly as a plan builds them, so that the CPU
 * test suite can replay the MMA arithmetic over them (tests/test_mma_tables.py).  Caller-sized arrays:
 * first / phase [cap_rows], mask65 [65 * n_point] shorts, vchunk [2 * chunks], bfrag [128 * chunks]
 * with chunks = ceil(out_size / *rows_per_chunk) (the largest of 8 .. 4 rows whose windows fit).  0 = ok, 1 = window does not fit the quad ring, -1 = bad arguments.
 */
int vb200_debug_mma_tables(int in_size, double shrink, int rect_size, int *int_shrink, int *shrunk_size, int *out_size,
	int *n_point, int *embed, int *first, int *phase, short *mask65, int *vchunk, unsigned *bfrag, int cap_rows,
	int *rows_per_chunk);

/* Test hook, host only (no GPU, no CUDA call): the bands of the tensor-pipe thumbnail kernel for a width x height
 * RGBA uchar frame thumbnailed to target_width (VB200_SIZE_BOTH), exactly as a plan lays them out.  Band b writes
 * output columns [xa[b], xb[b]) and reads input columns [c_lo[b], c_hi[b]); seam[b] (b < n_bands - 1) is how many input
 * columns bands b and b + 1 both read.  A TMA stage row is *n_box boxes of *box_width pixels.  Caller-sized arrays
 * [cap].  0 = ok, 1 = the plan does not use the tensor-pipe kernel, -1 = bad arguments.
 */
int vb200_debug_thumbnail_bands(int width, int height, int target_width, int *out_width, int *n_bands, int *xa, int *xb,
	int *c_lo, int *c_hi, int *seam, int cap, int *box_width, int *n_box);
/* Test hook, host only (no GPU, no CUDA call): the name vb200_thumbnail_plan_kernel gives the plan
 * vb200_thumbnail_plan_new(width, height, bands, VB200_FORMAT_UCHAR, has_alpha, target_width, target_height, size, 0) would
 * build, written to name[cap] with its terminating NUL ("leaf kernels" for an unfused plan).  0 = ok, -1 = bad arguments,
 * a plan that fails, or a name longer than cap - 1.
 */
int vb200_debug_thumbnail_kernel(int width, int height, int bands, int has_alpha, int target_width, int target_height, int size,
	char *name, int cap);

/* ------------------------------------------------------------------ JPEG decode staging (SURVEY 8f rank 1)
 * vips_jpegload_buffer(buf, len, &out, "shrink", shrink) (foreign/jpeg2vips.c:532-538, 631-640: scale_num = 1,
 * scale_denom = shrink, output cropped to floor(size / shrink)) with the decoder on the device: the compressed
 * bytes are all that crosses PCIe.  libjpeg(-turbo) itself is a third-party dependency outside the reference
 * tree; its algorithm for the reference's configuration (JDCT_ISLOW, 8-bit Huffman, sequential and progressive)
 * is restated in csrc/jpeg.cu and pinned bit for bit to the libjpeg-turbo inside this image's Pillow
 * (tests/test_jpeg.py, tests/test_jpeg_layouts.py).  Decoded: 8-bit Huffman streams, baseline / extended sequential (one
 * interleaved scan) and progressive, greyscale (whatever sampling its frame header declares) or YCbCr with sampling
 * factors 1 or 2 in which Y has the largest factor both ways and each chroma component is at Y's resolution, halved
 * across, or halved both ways: 4:4:4, 4:2:2, 4:2:0, every component 2x1, every component 1x2, Y 2x2 over chroma 1x2 --
 * at shrink 1 / 2 / 4 / 8 (where libjpeg's upsampler has work left, its h2v2 / h2v1 "fancy" triangle filters,
 * jdsample.c).  At shrink 2 / 4 / 8 also Y 1x1 under 2x2 chroma, which libjpeg's scaled IDCT brings to Y's size.
 * Everything else returns -1 (host loader): arithmetic-coded, 12-bit, CMYK / RGB-coded streams, sequential streams with
 * a scan per component, factors above 2 (4:1:1), chroma halved only vertically (4:4:0: libjpeg's h1v2 upsampler), Y
 * that would need upsampling, and interleaved scans of more than 10 blocks per MCU (2x2 in all three components:
 * T.81 B.2.3, libjpeg refuses them too).  Baseline streams with restart markers decode one interval per GPU thread,
 * those without by self-synchronising subsequences; progressive streams one scan after the other.
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
 * 848-902): load-time shrink by vb200_thumbnail_jpegshrink, decode and thumbnail on the device; out: allocate-or-fill.
 * A PNG stream (by its signature) decodes at full size (no load-time shrink, thumbnail.c:609-660) with its iCCP profile as
 * the embedded profile; PNGs with eXIf return -1 (their orientation would need vips_autorot).  A GIF stream (GIF87a /
 * GIF89a) loads with nsgifload's defaults (page 0, n = 1) at full size and without a profile (nsgifload attaches none):
 * its first frame, RGB or RGBA, is an untagged input to colour management. */
int vb200_thumbnail_buffer(const void *buf, size_t len, VB200Image *out, int width, int height, int size);
int vb200_thumbnail_plan_run_jpeg(VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, int shrink,
	void *out, int out_location, size_t out_frame_stride);
int vb200_debug_jpeg_decode(const void *buf, size_t len, int shrink, void *out, size_t out_bpl, int *width, int *height,
	int *bands);
/* test hook, host only: the self-synchronising decode of a scan without restart markers (subsequences of sub_bytes,
 * max_passes passes), *passes_used = the last pass that changed a record */
int vb200_debug_jpeg_decode_sync(const void *buf, size_t len, int shrink, int sub_bytes, int max_passes, void *out, size_t out_bpl,
	int *width, int *height, int *bands, int *passes_used);

/* ------------------------------------------------------------------ PNG decode on the device (SURVEY 8f rank 1)
 * vips_pngload_buffer(buf, len, &out, NULL) (foreign/spngload.c, libspng over zlib, fail_on = none: CRCs and Adler-32 not
 * checked, :346-352) with inflate and unfilter on the device (csrc/png.cu): the IDAT payloads are all that crosses PCIe.
 * Decoded: non-interlaced 8-bit grey, grey + alpha, RGB and RGBA; palette at 1 / 2 / 4 / 8 bits, to RGB or, with tRNS,
 * RGBA; grey at 1 / 2 / 4 bits scaled to 8; tRNS on 8-bit grey and RGB as an alpha band, 0 where the sample equals the
 * key (SPNG_DECODE_TRNS, :592; formats :385-480).  Output is uchar [n][height][width][bands], bands 1 to 4, B_W below 3
 * bands and sRGB from 3.  Everything else returns -1 with its reason (the host keeps its loader): 16-bit samples, Adam7,
 * low-bit grey with tRNS, a missing PLTE or an index beyond it, IDAT chunks that are not consecutive, a zlib header with a
 * preset dictionary, another method or a bad FCHECK, a deflate stream zlib refuses, one that inflates to more or fewer
 * scanline bytes than IHDR implies, frames over 2^28 pixels.
 *
 * vb200_png_decode_batch: n streams of ONE output geometry; a stream that fails fails the batch with "frame i:" in the
 *   error, and with out in host memory nothing is written (in device memory, frames of earlier chunks of a batch larger
 *   than one chunk may be).  out = NULL only reports the geometry, without a device.
 * vb200_pngload_buffer: one stream into a VB200Image (allocate-or-fill).
 * vb200_png_icc_profile: the iCCP profile (spngload.c:244-246), inflated on the host; as vb200_jpeg_icc_profile.
 * vb200_thumbnail_plan_run_png: decode + the plan's thumbnail chain, frames never leave the device; PNG has no load-time
 *   shrink (thumbnail.c:609-660), so the plan is made for the full frame.  Streams with eXIf are declined, as by
 *   vb200_thumbnail_buffer: their orientation would need vips_autorot (thumbnail.c:989-996).
 * vb200_debug_png_decode / vb200_debug_inflate: test hooks, host only -- the same per-symbol, per-byte and per-pixel code
 *   on the CPU; vb200_debug_inflate takes raw deflate data and sets *out_len = cap + 1 when the output does not fit.
 * vb200_debug_png_set_budget: device bytes per chunk (0: an eighth of the device, at least 1 GiB); it bounds the PNG and
 *   GIF decoders and the JPEG and PNG encoders.
 */
int vb200_png_decode_batch(const void *const *bufs, const size_t *lens, int n, void *out, int out_location, size_t out_bpl,
	size_t out_frame_stride, int *width, int *height, int *bands);
int vb200_pngload_buffer(const void *buf, size_t len, VB200Image *out);
int vb200_png_icc_profile(const void *buf, size_t len, void *out, size_t cap, size_t *profile_len);
int vb200_thumbnail_plan_run_png(VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, void *out,
	int out_location, size_t out_frame_stride);
int vb200_debug_png_decode(const void *buf, size_t len, void *out, size_t out_bpl, int *width, int *height, int *bands);
int vb200_debug_inflate(const void *buf, size_t len, void *out, size_t cap, size_t *out_len);
void vb200_debug_png_set_budget(size_t bytes);
/* ------------------------------------------------------------------ WebP decode on the device
 * vips_webpload_buffer(buf, len, &out, NULL) (foreign/webp2vips.c through webpload.c: WebPDecode in MODE_RGBA with
 * fancy upsampling, the fourth band dropped without alpha, :600-645, 740-790) with the VP8 key frame decoded on the device
 * (csrc/webp.cu): the VP8 chunk payloads are all that crosses PCIe.  Decoded: the simple format and VP8X without the
 * ANIMATION and ALPHA flags, key frames up to 16383 x 16383 with every key-frame feature.  Output is uchar sRGB
 * [n][height][width][3], pixel for pixel libwebp's.  Everything else returns -1 with its reason (the host keeps
 * webpload): VP8L, ALPH or the ALPHA flag, ANIM / ANMF, non-key frames, a bad signature or chunk sizes that run past the
 * RIFF or the buffer, a VP8X canvas other than the frame.  A frame libwebp refuses while decoding (a header or partition
 * cut short, a bad partition table) fails the batch with "frame i:".
 *
 * vb200_webp_geometry: width, height and bands (3); host only.
 * vb200_webp_decode_batch: n streams of ONE geometry; a stream that fails fails the batch with "frame i:" in the error,
 *   and with out in host memory nothing is written (in device memory, frames of earlier chunks of a batch larger than one
 *   chunk may be).  out = NULL only reports the geometry, without a device.
 * vb200_webpload_buffer: one stream into a VB200Image (allocate-or-fill).
 * vb200_webp_icc_profile: the ICCP chunk of a VP8X stream; as vb200_png_icc_profile.
 * vb200_debug_webp_decode: test hook, host only -- the same per-symbol, per-block and per-pixel code on the CPU.
 * vb200_debug_webp_tables: test hook -- the decoder's constant tables, one after another (*len bytes; copied when cap holds
 *   them).
 * vb200_debug_webp_times: with VB200_WEBP_TIMING set in the environment, ms[4] = the last batch's device milliseconds in the
 *   header, token, reconstruction and RGB kernels on the calling thread (each chunk then waits for its events); -1 without.
 * vb200_thumbnail_buffer and the other thumbnail entries refuse WebP: thumbnail.c loads it at a non-integer scale through
 * libwebp's own rescaler, which only the WebP entries below take.  Chunks are bounded by vb200_debug_png_set_budget.
 *
 * WebP shrink-on-load: vips_webpload_buffer(buf, len, &out, "scale", scale, NULL).  scale != 1.0 is libwebp's scaled decode
 * (webp2vips.c:513-514, 630-634): the frame becomes rint(w * scale) x rint(h * scale), refused outside 1 .. 16383 on either
 * axis or for scale outside webpload's [0, 1024]; the loop filter is bypassed when both axes come out below three quarters
 * (w * 3 / 4, in integers); Y, U and V each go through libwebp's WebPRescaler (area average shrinking, linear interpolation
 * expanding, 32-bit fixed point) with no upsampler, then the same 14-bit YUV -> RGB.  Pixel for pixel libwebp's.
 * scale == 1.0 is exactly the plain decode above.
 *
 * vb200_webp_decode_batch_scaled: vb200_webp_decode_batch at scale; the streams must share one source size.
 * vb200_webpload_buffer_scaled: vb200_webpload_buffer at scale.
 * vb200_thumbnail_webp_scale: host only -- vips_thumbnail_open's WebP factor max(1, common shrink) (thumbnail.c:627-636)
 *   as *scale = 1 / factor and the size webpload loads at (*scaled_width / *scaled_height may be NULL).  Unlike JPEG's
 *   shrink it applies in linear mode too.
 * vb200_thumbnail_webp_buffer: vips_thumbnail_buffer of a WebP stream: loaded at vb200_thumbnail_webp_scale's scale on the
 *   device, its ICCP as the embedded profile, then what vb200_thumbnail_buffer_icc (linear = 0) or
 *   vb200_thumbnail_buffer_linear_icc (linear = 1) runs on the decode; icc NULL: no colour management.
 * vb200_thumbnail_plan_run_webp: the streams decoded at scale + the plan's thumbnail chain, frames never leave the device;
 *   the plan must have been made for the scaled geometry.
 * vb200_debug_webp_decode_scaled: test hook, host only -- the scaled decode on the CPU, its rescaler streaming rows in
 *   libwebp's order.
 * vb200_debug_webp_rescale: test hook, host only -- one plane of src_w x src_h rescaled to dst_w x dst_h, closed_form set by
 *   the device kernel's per-sample function, else by the host twin's row-streaming rescaler.
 */
int vb200_webp_geometry(const void *buf, size_t len, int *width, int *height, int *bands);
int vb200_webp_decode_batch(const void *const *bufs, const size_t *lens, int n, void *out, int out_location, size_t out_bpl,
	size_t out_frame_stride, int *width, int *height, int *bands);
int vb200_webpload_buffer(const void *buf, size_t len, VB200Image *out);
int vb200_webp_icc_profile(const void *buf, size_t len, void *out, size_t cap, size_t *profile_len);
int vb200_debug_webp_decode(const void *buf, size_t len, void *out, size_t out_bpl, int *width, int *height, int *bands);
int vb200_debug_webp_tables(void *out, size_t cap, size_t *len);
void vb200_debug_webp_times(float *ms);
int vb200_webp_decode_batch_scaled(const void *const *bufs, const size_t *lens, int n, double scale, void *out, int out_location,
	size_t out_bpl, size_t out_frame_stride, int *width, int *height, int *bands);
int vb200_webpload_buffer_scaled(const void *buf, size_t len, double scale, VB200Image *out);
int vb200_thumbnail_webp_scale(int width, int height, int target_width, int target_height, int size, double *scale, int *scaled_width,
	int *scaled_height);
int vb200_thumbnail_webp_buffer(const void *buf, size_t len, VB200Image *out, int width, int height, int size, const VB200ThumbnailIcc *icc,
	int linear);
int vb200_thumbnail_plan_run_webp(VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, double scale, void *out,
	int out_location, size_t out_frame_stride);
int vb200_debug_webp_decode_scaled(const void *buf, size_t len, double scale, void *out, size_t out_bpl, int *width, int *height,
	int *bands);
int vb200_debug_webp_rescale(const void *plane, size_t stride, int src_w, int src_h, int dst_w, int dst_h, int closed_form, void *out,
	size_t out_bpl);
/* ------------------------------------------------------------------ GIF decode on the device (SURVEY 8f rank 1)
 * vips_gifload_buffer(buf, len, &out, "page", page, "n", n, NULL) (foreign/nsgifload.c over libnsgif, fail_on = none)
 * with LZW and frame composition on the device (csrc/gif.cu): the LZW payloads, without their sub-block length bytes, and
 * one colour table per frame are all that crosses PCIe.  Output is uchar sRGB [n_streams][height * pages][width][bands]:
 * page k is the screen after frames 0 .. page + k composed by libnsgif's disposal rules, 4 bands if any frame of the
 * stream has transparency and 3 otherwise (nsgifload.c:262-280, 480-540).  n_pages = -1: every page from `page` on.
 * Declined (-1 with the reason; the host keeps nsgifload): a scan that is not NSGIF_OK, a truncated last frame (nsgifload
 * loads those only with a warning), no frames, screens over 65 535 on a side ("bad image dimensions") or over 2^28
 * pixels, page / n out of range ("bad page number").  A frame with a code libnsgif refuses fails the batch.
 *
 * vb200_gif_geometry: nsgif_get_info after the scan: screen width and height, bands, frame count; host only.
 * vb200_gif_decode_batch: n streams of ONE geometry (screen, bands and pages); a stream that fails fails the batch with
 *   "stream i:" in the error, and with out in host memory nothing is written (in device memory, streams of earlier chunks
 *   of a batch larger than one chunk may be).  out = NULL only reports the geometry (*height: all pages), without a device.
 * vb200_gifload_buffer: one stream into a VB200Image (allocate-or-fill), height * pages rows.
 * vb200_thumbnail_plan_run_gif: page 0 of each stream + the plan's thumbnail chain, frames never leave the device; GIF has
 *   no load-time shrink (thumbnail.c:609-660), so the plan is made for the full screen (3 or 4 bands).
 * vb200_debug_gif_decode / vb200_debug_lzw: test hooks, host only -- the same per-code and per-pixel code on the CPU;
 *   vb200_debug_lzw takes joined sub-block data and decodes at most `want` values (lenient: the complex path's rule that a
 *   bad code at a multiple of 4096 values ends the frame quietly).
 * Chunks are bounded by vb200_debug_png_set_budget, the PNG codecs' device budget.
 */
int vb200_gif_geometry(const void *buf, size_t len, int *width, int *height, int *bands, int *frames);
int vb200_gif_decode_batch(const void *const *bufs, const size_t *lens, int n, int page, int n_pages, void *out, int out_location,
	size_t out_bpl, size_t out_frame_stride, int *width, int *height, int *bands);
int vb200_gifload_buffer(const void *buf, size_t len, int page, int n, VB200Image *out);
int vb200_thumbnail_plan_run_gif(VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, void *out,
	int out_location, size_t out_frame_stride);
int vb200_debug_gif_decode(const void *buf, size_t len, int page, int n, void *out, size_t out_bpl, int *width, int *height,
	int *bands);
int vb200_debug_lzw(const void *data, size_t len, int min_code_size, unsigned want, int lenient, void *out, size_t *out_len);
/* ------------------------------------------------------------------ TIFF decode on the device
 * vips_tiffload_buffer(buf, len, &out, "page", page, "n", n, "subifd", subifd, NULL) (foreign/tiff2vips.c over libtiff) with
 * the strips or tiles decoded and placed on the device (csrc/tiff.cu).  Classic and BigTIFF, either byte order,
 * PlanarConfiguration 1, FillOrder 1, 8-bit unsigned samples: MINISBLACK / MINISWHITE with 1-2 samples load as B_W (the
 * first band of MINISWHITE inverted, rtiff_greyscale_line, tiff2vips.c:1359-1448), RGB with 3-4 as sRGB
 * (rtiff_parse_copy, :1723-1780); ExtraSamples 0 or 2, the extra band copied.  Compression none, PackBits, LZW and deflate
 * (8 and 32946), predictor 1 or 2; JPEG tiles, greyscale or YCbCr (to sRGB by libjpeg's YCbCr path), with or without
 * JPEGTables (rtiff_decompress_jpeg_run, :2082-2177).  Pages page .. page + n - 1 (n = -1: to the last) stack as a strip whose pages must agree
 * (rtiff_header_equal, :3364); subifd >= 0 loads that SubIFD of each page (rtiff_set_page, :798-846).
 * Declined from the IFD before any device work (-1 with the reason; the host keeps tiff2vips): other depths and sample
 * formats, PlanarConfiguration 2, FillOrder 2, palette / CIELAB / separated / LogLuv, YCbCr without JPEG, JPEG strips and
 * RGB-photometric JPEG, associated alpha, old-style JPEG and LZW, other compressions, predictor 3, segments outside the
 * stream, pages that differ, frames over 2^28 pixels, JPEG tiles the JPEG decoder declines ("tile k: ...").  A segment that
 * decodes short (libtiff's "Not enough data") or corrupt, or a deflate segment whose Adler-32 trailer zlib reads and
 * refuses, fails the batch.
 *
 * vb200_tiff_geometry: width, height and bands of the IFD page / subifd select, the stream's page count and the SubIFD
 *   count of that page's main IFD; host only.
 * vb200_tiff_decode_batch: n streams of ONE geometry -> out[n][h * pages][w][bands]; as vb200_gif_decode_batch, a stream
 *   that fails fails the batch with "frame i:", and out = NULL only reports the geometry without a device.
 * vb200_tiffload_buffer: one stream into a VB200Image (allocate-or-fill).
 * vb200_tiff_icc_profile: the ICCProfile tag (34675) of the IFD page / subifd select (*profile_len = 0: none).
 * vb200_thumbnail_plan_run_tiff: the streams' pages at subifd + the plan's thumbnail chain, frames never leave the device.
 * vb200_thumbnail_tiff_level: host only -- the subifd (-1: none) and page vips_thumbnail_buffer loads for a thumbnail of
 *   width / height / size: vips_thumbnail_get_tiff_pyramid_subifd (thumbnail.c:324-383) first, then
 *   vips_thumbnail_get_pyramid_page (:262-322), and vips_thumbnail_find_pyrlevel (:519-541) over the levels found.
 *   vb200_thumbnail_buffer (and _icc / _linear_icc) load that level; vb200_thumbnail_buffer_pages declines TIFF.
 *   A TIFF IFD whose Orientation is not 1 is declined for thumbnails (it would need vips_autorot).
 * vb200_debug_thumbnail_pyramid_level: test hook, host only -- the same level choice over given level geometries.
 * vb200_debug_tiff_decode / vb200_debug_tiff_lzw: test hooks, host only -- the same per-code and per-byte code on the CPU;
 *   vb200_debug_tiff_lzw decodes one LZW segment into exactly `want` bytes.
 * Chunks are bounded by vb200_debug_png_set_budget, the PNG codecs' device budget.
 */
int vb200_tiff_geometry(const void *buf, size_t len, int page, int subifd, int *width, int *height, int *bands, int *pages, int *subifds);
int vb200_tiff_decode_batch(const void *const *bufs, const size_t *lens, int n, int page, int n_pages, int subifd, void *out, int out_location,
	size_t out_bpl, size_t out_frame_stride, int *width, int *height, int *bands);
int vb200_tiffload_buffer(const void *buf, size_t len, int page, int n, int subifd, VB200Image *out);
int vb200_tiff_icc_profile(const void *buf, size_t len, int page, int subifd, void *out, size_t cap, size_t *profile_len);
int vb200_thumbnail_plan_run_tiff(VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, int page, int n_pages,
	int subifd, void *out, int out_location, size_t out_frame_stride);
int vb200_thumbnail_tiff_level(const void *buf, size_t len, int width, int height, int size, int *subifd, int *page);
int vb200_debug_thumbnail_pyramid_level(int in_w, int in_h, int n_pages, const int *page_w, const int *page_h, int n_subifds,
	const int *sub_w, const int *sub_h, int width, int height, int size, int *subifd, int *page);
int vb200_debug_tiff_decode(const void *buf, size_t len, int page, int n, int subifd, void *out, size_t out_bpl, int *width, int *height,
	int *bands);
int vb200_debug_tiff_lzw(const void *data, size_t len, size_t want, void *out, size_t *out_len);
/* ------------------------------------------------------------------ thumbnail: page strips (animated thumbnails)
 * vips_thumbnail of a multi-page image held as a strip: pages of page_height rows stacked vertically, with libvips'
 * "page-height" metadata (a GIF loaded with n = -1, a multi-page TIFF, an animated WebP).  As vips_thumbnail_build does
 * (resample/thumbnail.c:825-839, 848-861, 904-917):
 *   - the page height is read as vips_image_get_page_height does (iofuncs/header.c:889-901): <= 0, not less than the
 *     height, or not dividing it means one page;
 *   - hshrink / vshrink are vips_thumbnail_calculate_shrink's for one page (width x page_height), then, with more than one
 *     page, vshrink = height / (rint(page_height / vshrink) * n_pages) so that every page lands on whole rows;
 *   - premultiply when there is alpha and neither adjusted shrink is 1; vips_resize(1 / hshrink, vscale = 1 / vshrink)
 *     runs over the whole strip as one image, so shrink boxes and reduce windows straddle the page seams as in libvips;
 *   - the result's page height is rint(page_height / vshrink), reported as vips_image_get_page_height would read it back:
 *     the output height when it does not divide it, and for one page.
 * With one page every entry below computes what the single-image entry computes.  Strips over 2^31 - 1 input bytes are
 * declined (-1 with the reason).
 *
 * vb200_thumbnail_plan_new_pages: vb200_thumbnail_plan_new for strips of n_pages pages of page_height rows (frames of
 *   width x page_height * n_pages); vb200_thumbnail_plan_new is the n_pages = 1 case.
 * vb200_thumbnail_plan_page_height: the page height of the plan's output frames (vips_image_get_page_height of the result).
 * vb200_thumbnail_image_pages: vips_thumbnail_image of a strip with page_height (0: none); icc NULL = no colour
 *   management; linear selects vb200_thumbnail_image_linear_icc's path, otherwise vb200_thumbnail_image_icc's.
 *   *out_page_height (may be NULL): the result's page height.
 * vb200_thumbnail_plan_run_gif_pages: vb200_thumbnail_plan_run_gif of pages page .. page + n_pages - 1 (n_pages = -1: every
 *   page from `page` on).  The streams of a batch share screen, bands and page count (vb200_gif_decode_batch); the plan is
 *   made with vb200_thumbnail_plan_new_pages(screen width, screen height, pages, ...).
 * vb200_thumbnail_buffer_pages: vips_thumbnail_buffer(..., option_string = "page=..,n=..") (thumbnail.c:1486-1490,
 *   1585-1590), with the ICC and linear variants as vb200_thumbnail_image_pages.  A GIF loads pages page .. page + n - 1,
 *   with page-height set only when more than one page loaded (nsgifload.c:279-280).  JPEG and PNG streams with page != 0
 *   or n != 1 return -1: jpegload and spngload have no such options.
 * vb200_debug_thumbnail_pages_size: test hook, host only (no GPU, no CUDA call): the shrinks, output size and output page
 *   height vb200_thumbnail_plan_new_pages would plan.  -1: bad arguments or a plan that declines (mixed up / down).
 *   Each entry cites thumbnail.c where its rule comes from: :825-839 (shrink), :848-861 (premultiply), :904-917 (page-height).
 */
VB200ThumbnailPlan *vb200_thumbnail_plan_new_pages(int width, int page_height, int n_pages, int bands, int band_format, int has_alpha,
	int target_width, int target_height, int size, int linear);
int vb200_thumbnail_plan_page_height(const VB200ThumbnailPlan *plan);
int vb200_thumbnail_image_pages(const VB200Image *in, int page_height, VB200Image *out, int width, int height, int size,
	const VB200ThumbnailIcc *icc, const void *embedded, size_t embedded_len, int linear, int *out_page_height);
int vb200_thumbnail_plan_run_gif_pages(VB200ThumbnailPlan *plan, const void *const *bufs, const size_t *lens, int n, int page,
	int n_pages, void *out, int out_location, size_t out_frame_stride);
int vb200_thumbnail_buffer_pages(const void *buf, size_t len, VB200Image *out, int width, int height, int size,
	const VB200ThumbnailIcc *icc, int linear, int page, int n, int *out_page_height);
int vb200_debug_thumbnail_pages_size(int width, int page_height, int n_pages, int target_width, int target_height, int size,
	double *hshrink, double *vshrink, int *out_width, int *out_height, int *out_page_height);
/* test hook, host only: vb200_debug_thumbnail_kernel's kernel name for the plan vb200_thumbnail_plan_new_pages would build */
int vb200_debug_thumbnail_pages_kernel(int width, int page_height, int n_pages, int bands, int has_alpha, int target_width,
	int target_height, int size, char *name, int cap);
/* ------------------------------------------------------------------ PNG save on the device
 * vips_pngsave_buffer (foreign/spngsave.c, libspng over zlib) for uchar frames of 1-4 bands (grey, grey + alpha, RGB,
 * RGBA): bit depth 8 (:608-613), non-interlaced, filter NONE (:714-720, :769), IHDR from the bands (:405-439), pHYs of
 * rint(xres * 1000) pixels per metre on both axes (:455-456 reads Xres twice), iCCP named "icc" when a profile is given
 * (:176-230), compressed at the image's level (:447-448).  The frames are deflated on the device (csrc/png_encode.cu): the
 * zlib stream -- the IDAT payloads concatenated -- is zlib 1.3's at window bits 15 and memLevel 8 byte for byte
 * (tests/test_png_save.py).  Chunks: signature, IHDR, iCCP, pHYs, IDATs of at most 8192 payload bytes, IEND.  Whole-file
 * equality with libspng is not claimed: its IDAT split, its chunk order and the strategy it picks cannot be checked here.
 *
 * compression: zlib level (:700-705, default 6); 4-9 are built, 0-3 return -1 with the reason.  strategy: 0
 *   Z_DEFAULT_STRATEGY (libpng's choice for unfiltered images), 1 Z_FILTERED.  xres: pixels per millimetre (libvips' Xres,
 *   default 1.0).
 * filter (:714-720, :449-450): a VipsForeignPngFilter flag -- NONE 0x08, SUB 0x10, UP 0x20, AVG 0x40, PAETH 0x80 -- or 0
 *   for NONE; every scanline is filtered with that type (PNG 2nd edition 9.2) on the raw bytes.  interlace (:707-712,
 *   :439): non-zero writes Adam7 scanlines and IHDR interlace 1.  bitdepth (:743-748): 0 or 8, or 1 / 2 / 4 for one band,
 *   written as grey without a palette: each sample p >> (8 - bitdepth), packed MSB first as vips_foreign_save_spng_pack
 *   packs it (:295-324), its tail rule included (at depth 4 an odd-width row ends in v[w-2] << 4 | v[w-1]).  With all three
 *   0 the streams are what they were before these fields existed.
 * Declined (-1 with the reason; the host keeps spngsave): compression 0-3, another strategy, bands outside 1-4, frames over
 *   2^28 pixels, a format other than uchar (vb200_pngsave_buffer), unknown filter bits, more than one filter flag
 *   (libspng's adaptive choice, ALL = 0xF8), bitdepth 16 or other than 1 / 2 / 4 / 8, bitdepth below 8 with 2 bands (no
 *   low-bit grey + alpha in PNG) or 3-4 bands (spngsave palettises; quantisation is not built), bitdepth below 8 with a
 *   filter other than NONE or with interlace.  Palette output and metadata chunks other than iCCP are not written.
 * vb200_pngsave_batch: n frames of one geometry in host or device memory (frames_location); stream i at out + i *
 *   out_stride (out_location), lengths[i] bytes (host array, may be NULL).  A stream that does not fit out_stride returns -1
 *   with its frame before its chunk writes anything: with out in host memory nothing is written then, in device memory the
 *   frames of earlier chunks of a batch larger than one chunk (vb200_debug_png_set_budget) may be.  vb200_jpegsave_batch
 *   behaves the same.
 * vb200_pngsave_buffer: one image; *out is malloc()ed, free() it.
 * vb200_debug_png_encode: test hook, host only -- the whole stream through the kernels' per-position, per-symbol and
 *   per-block code compiled for the CPU.  out = NULL only reports *len.
 * vb200_debug_deflate: test hook, host only -- the zlib stream (header, deflate data, Adler-32) of buf[0, n) at a level
 *   and strategy, through the same code.  out = NULL only reports *len.
 * The struct grew by filter, interlace and bitdepth, its last members: C callers rebuild against this header.
 */
typedef struct {
	int compression;
	int strategy;
	double xres;
	int filter;
	int interlace;
	int bitdepth;
} VB200PngSaveOptions;
int vb200_pngsave_batch(const void *frames, int frames_location, size_t bpl, size_t frame_stride, int n, int width, int height, int bands,
	const VB200PngSaveOptions *options, const void *profile, size_t profile_len, void *out, int out_location, size_t out_stride, size_t *lengths);
int vb200_pngsave_buffer(const VB200Image *in, const VB200PngSaveOptions *options, const void *profile, size_t profile_len, void **out,
	size_t *len);
int vb200_debug_png_encode(const void *pixels, size_t bpl, int width, int height, int bands, const VB200PngSaveOptions *options,
	const void *profile, size_t profile_len, void *out, size_t cap, size_t *len);
int vb200_debug_deflate(const void *buf, size_t n, int level, int strategy, void *out, size_t cap, size_t *len);
/* vips_jpegsave_buffer (foreign/vips2jpeg.c:551-700: jpeg_set_quality(Q, TRUE), chroma subsampled 2 x 2 below Q 90 unless
 * subsample_mode says otherwise -- 0 auto, 1 on, 2 off --, baseline, standard Huffman tables, JFIF header) for n equally sized
 * 8-bit frames of 1 or 3 bands, encoded on the device (csrc/jpeg_encode.cu): the streams are libjpeg-turbo's byte for byte
 * (tests/test_jpeg_encode.py).  frames / out in host or device memory; stream i at out + i * out_stride, lengths[i] bytes
 * (host array, may be NULL).  Batches run in chunks bounded by vb200_debug_png_set_budget; a stream that does not fit
 * out_stride fails the call as in vb200_pngsave_batch.
 */
int vb200_jpegsave_batch(const void *frames, int frames_location, size_t bpl, size_t frame_stride, int n, int width, int height, int bands,
	int Q, int subsample_mode, void *out, int out_location, size_t out_stride, size_t *lengths);
/* vips_jpegsave's options that the device encoder takes.  Q, subsample_mode: as above.  optimize_coding
 * (jpegsave.c:227-232 -> vips2jpeg.c:590-591, cinfo.optimize_coding): non-zero builds each frame's Huffman tables from
 * its own symbol counts (jchuff.c jpeg_gen_optimal_table), so every frame carries its own DHT segments.
 * restart_interval (jpegsave.c:284-289 -> vips2jpeg.c:593-597, cinfo.restart_interval): an RSTn marker every that many
 * MCUs and a DRI segment; 0 for none.  Values above 65535 are refused (-1): libjpeg would write DRI modulo 65536 and a
 * stream no reader can follow.  interlace (jpegsave.c:234-238 -> vips2jpeg.c:670-673, jpeg_simple_progression):
 * non-zero writes a progressive stream (SOF2, libjpeg's 10-scan script for colour, 6 scans for greyscale); libjpeg forces
 * optimize_coding on in progressive mode, so every scan carries its own optimal Huffman table and optimize_coding makes
 * no difference; restart_interval counts MCUs in the interleaved DC scans and single blocks in the others.  With all
 * three 0 the streams are vb200_jpegsave_batch's.
 * The struct grew by interlace, its last member: C callers rebuild against this header.
 */
typedef struct {
	int Q;
	int subsample_mode;
	int optimize_coding;
	int restart_interval;
	int interlace;
} VB200JpegSaveOptions;
/* vb200_jpegsave_batch with VB200JpegSaveOptions; the streams are libjpeg-turbo's byte for byte with the same options
 * (tests/test_jpeg_encode_options.py) */
int vb200_jpegsave_batch_opts(const void *frames, int frames_location, size_t bpl, size_t frame_stride, int n, int width, int height,
	int bands, const VB200JpegSaveOptions *options, void *out, int out_location, size_t out_stride, size_t *lengths);
/* test hook, host only: vips_jpegsave_buffer's stream (csrc/jpeg_encode.cu) through the encoder's per-block code on the CPU.
 * subsample_mode: 0 auto (4:2:0 below Q 90, vips2jpeg.c:676-690), 1 on, 2 off.  *len = bytes written */
int vb200_debug_jpeg_encode(const void *pixels, size_t bpl, int width, int height, int bands, int quality, int subsample_mode, void *out,
	size_t cap, size_t *len);
/* test hook, host only: vb200_debug_jpeg_encode with every option of VB200JpegSaveOptions */
int vb200_debug_jpeg_encode_opts(const void *pixels, size_t bpl, int width, int height, int bands, const VB200JpegSaveOptions *options,
	void *out, size_t cap, size_t *len);
/* test hook, host only: what the host twin's progressive coder (jcphuff.c restated) reaches for an image: events[0] EOB runs
 * forced out at 0x7FFF blocks, [1] EOB runs forced out by the correction-bit buffer, [2] ZRLs in refinement scans */
int vb200_debug_jpeg_prog_events(const void *pixels, size_t bpl, int width, int height, int bands, const VB200JpegSaveOptions *options,
	unsigned long long *events);
/* test hook, host only: the encoder's restatement of jpeg_gen_optimal_table on symbol counts freq[256] -> bits[17]
 * (bits[0] unused) and huffval[256]; -1 when the counts add up to 10^9 or more */
int vb200_debug_jpeg_optimal_table(const unsigned *freq, unsigned char *bits, unsigned char *huffval);
/* with env VB200_JPEG_TIMING: CUDA-event times of jpeg_huffman_kernel / jpeg_idct_kernel over the calling thread's last decode */
void vb200_debug_jpeg_times(float *huffman_ms, float *idct_ms);

/* ------------------------------------------------------------------ Deep Zoom tile pyramids
 * vips_dzsave (foreign/dzsave.c) in its "dz" and "zoomify" layouts with JPEG or PNG tiles, on the device (csrc/dzsave.cu):
 * every level of the pyramid (strip_shrink :1761-1835 over region.c:1139-1156, each level the 2 x 2 rounded mean
 * (a + b + c + d + 2) >> 2 of the level above with its last column / row repeated when its size is odd,
 * level_generate_extras :1710-1754), every tile cut from it (image_strip_allocate :1106-1152) and every tile's
 * vips_jpegsave stream (write_image :369-404 -- the bytes vb200_jpegsave_batch_opts writes) is produced by CUDA kernels;
 * the finished streams and their index come back to the host.
 *
 * Options follow vips_foreign_save_dz_build (:2043-2113).  layout: the reference's VipsForeignDzLayout values; google,
 * iiif and iiif3 return -1.  tile_size 0 and overlap -1 take the layout's defaults (254 and 1 for dz, 256 and 0 for
 * zoomify); a tile_step (tile_size for dz, tile_size - overlap for zoomify) <= 0 is the reference's error "overlap too
 * large".  depth 0 is the layout's default (onepixel for dz, onetile for zoomify).  region_shrink, skip_blanks and
 * container are there to be refused: only the reference's defaults (mean, off, a directory tree) run here.  suffix NULL
 * is the layout's default (".jpeg" / ".jpg"); any other suffix must name a JPEG tile without [options].
 * Images are uchar with 1 or 3 bands, in host or device memory, any bpl; everything else returns -1 and keeps the host path.
 */
enum { VB200_DZ_LAYOUT_DZ = 0, VB200_DZ_LAYOUT_ZOOMIFY = 1, VB200_DZ_LAYOUT_GOOGLE = 2, VB200_DZ_LAYOUT_IIIF = 3, VB200_DZ_LAYOUT_IIIF3 = 4 };
enum { VB200_DZ_DEPTH_DEFAULT = 0, VB200_DZ_DEPTH_ONEPIXEL = 1, VB200_DZ_DEPTH_ONETILE = 2, VB200_DZ_DEPTH_ONE = 3 };
typedef struct {
	int layout;
	int tile_size;
	int overlap;
	int depth;
	int region_shrink; /* VipsRegionShrink: 0 mean; the others return -1 */
	int skip_blanks;   /* the reference's skip_blanks + 1, so that 0 is its default (off); anything else returns -1 */
	int container;	   /* VipsForeignDzContainer: 0 a directory tree; zip and szi return -1 */
	const char *suffix;
	VB200JpegSaveOptions jpeg; /* Q 0 = 75; the rest as vb200_jpegsave_batch_opts */
} VB200DzOptions;

/* a finished pyramid: the tile streams and their index, on the host */
typedef struct VB200DzPyramid VB200DzPyramid;

/* The whole save.  options NULL = every default.  On any error *out is NULL and nothing is left allocated. */
int vb200_dzsave(const VB200Image *in, const VB200DzOptions *options, VB200DzPyramid **out);
/* test hook, host only (no GPU, no CUDA call): the same pyramid, tiling and streams through the kernels' per-pixel code
 * and the encoder's host twin
 */
int vb200_debug_dzsave(const VB200Image *in, const VB200DzOptions *options, VB200DzPyramid **out);
/* The save with PNG tiles: the reference with suffix ".png", where every tile is vips_image_write_to_buffer(tile, ".png")
 * (write_image :369-402) -- spngsave with its defaults and keep NONE, so no iCCP -- and each stream is what
 * vb200_pngsave_batch writes for it.  Images are uchar with 1 to 4 bands, Type B_W for 1-2 bands and sRGB for 3-4 (any
 * other Type returns -1: spngsave's vips_colourspace or vips_image_hasalpha would change the pixels).  With 2 or 4 bands the
 * last is alpha and every level is vips_region_shrink_alpha's (region.c:1444-1482): with S the sum of the four alphas, each
 * colour band the alpha-weighted sum over S (truncated), alpha S >> 2, all 0 where S is 0 -- so an opaque RGBA image does
 * not get the RGB pyramid.  options: as vb200_dzsave, except suffix NULL = ".png", and any other suffix must be ".png" in
 * any case without [options]; options->jpeg is ignored.  png: the tiles' options as vb200_pngsave_batch takes them, with
 * the same declines; NULL = spngsave's defaults (compression 6, default strategy, xres 1.0, filter NONE, no interlace,
 * bitdepth 8).  Every decline happens before any device call.  The result is read with the vb200_dz_* calls below.
 */
int vb200_dzsave_png(const VB200Image *in, const VB200DzOptions *options, const VB200PngSaveOptions *png, VB200DzPyramid **out);
/* test hook, host only: vb200_dzsave_png through the kernels' per-pixel code and the PNG encoder's host twin */
int vb200_debug_dzsave_png(const VB200Image *in, const VB200DzOptions *options, const VB200PngSaveOptions *png, VB200DzPyramid **out);
void vb200_dz_free(VB200DzPyramid *pyramid);
/* levels are numbered as the reference numbers them (pyramid_build :441-577): n = 0 is the smallest */
int vb200_dz_levels(const VB200DzPyramid *pyramid);
int vb200_dz_level_geometry(const VB200DzPyramid *pyramid, int n, int *width, int *height, int *tiles_across, int *tiles_down);
/* tiles in the order zoomify numbers them (tile_name :1182-1191): level 0 first, then down, then across.  left, top,
 * width, height: the tile's rect in its level; stream: its JPEG or PNG, owned by the pyramid
 */
long vb200_dz_tiles(const VB200DzPyramid *pyramid);
int vb200_dz_tile(const VB200DzPyramid *pyramid, long i, int *level, int *x, int *y, int *left, int *top, int *width, int *height,
	const void **stream, size_t *len);
/* tile i's path relative to the directory the save is written in (tile_name :1156-1297): <basename>_files/<n>/<x>_<y>.jpeg,
 * or <basename>/TileGroup<N / 256>/<n>-<x>-<y>.jpg.  basename NULL = "untitled" (:2282)
 */
int vb200_dz_tile_name(const VB200DzPyramid *pyramid, long i, const char *basename, char *name, size_t cap);
/* the file beside the tiles: <basename>.dzi (write_dzi :579-620) or <basename>/ImageProperties.xml (write_properties
 * :622-655), byte for byte; *len = bytes of text (no terminating NUL is counted, one is written)
 */
int vb200_dz_sidecar(const VB200DzPyramid *pyramid, const char *basename, char *name, size_t ncap, char *text, size_t tcap, size_t *len);
/* The pixel pyramid alone: level n_from_top of the image (0 = the image itself, 1 = half size ...) through the same
 * kernels, into out (allocate-or-fill like every op).  -1 when the image has no such level (it stops at 1 x 1).  uchar,
 * 1 to 4 bands: 2 bands (Type B_W) and 4 bands (Type sRGB) are shrunk with their alpha, as vb200_dzsave_png does.
 */
int vb200_dz_pyramid_level(const VB200Image *in, int n_from_top, VB200Image *out);
/* test hook, host only: vb200_dz_pyramid_level through the per-pixel code on the CPU; out: packed, caller-sized.  It has no
 * Type: 2 and 4 bands are alpha images */
int vb200_debug_dz_pyramid_level(const void *pixels, size_t bpl, int width, int height, int bands, int n_from_top, void *out);
/* test hooks: the device memory one shape batch of tiles may take (pixels, encoder scratch and stream slots; 0 = the
 * default: 1 GiB for JPEG tiles, the PNG codecs' chunk budget for PNG tiles), and the bytes currently allocated from the
 * device's stream-ordered pool
 */
void vb200_debug_dz_set_budget(size_t bytes);
size_t vb200_debug_dz_pool_used(void);
/* with env VB200_DZ_TIMING set: CUDA-event milliseconds of the calling thread's last vb200_dzsave, split into
 * ms[0] pyramid kernels, [1] gather kernels, [2] encoder calls with the packed streams' device-to-host copies, [3] the
 * host-side placement of the tiles' streams
 */
void vb200_debug_dz_times(float *ms);

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
