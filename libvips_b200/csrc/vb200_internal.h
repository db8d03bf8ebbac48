/* vb200_internal.h -- shared declarations inside libvb200.so (not installed). */
#ifndef VB200_INTERNAL_H
#define VB200_INTERNAL_H

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <functional>
#include <thread>
#include <vector>

#include "vb200.h"

#define VB200_TRANSFORM_SHIFT 6 /* reference: include/vips/interpolate.h:109-118 */
#define VB200_TRANSFORM_SCALE (1 << VB200_TRANSFORM_SHIFT)
#define VB200_INTERPOLATE_SHIFT 12
#define VB200_INTERPOLATE_SCALE (1 << VB200_INTERPOLATE_SHIFT)
#define VB200_MAX_POINT 2000 /* reference: resample/presample.h:70 */
#define VB200_ROUND_UINT(R) ((int) ((R) + 0.5))

namespace vb200 {

/* vips_error(domain, fmt, ...): append to the thread-local buffer. */
void error(const char *domain, const char *fmt, ...);
/* drop what was appended to the thread's error buffer after its first len bytes (a probe whose failures are not errors) */
void error_truncate(size_t len);
int cuda_fail(const char *domain, cudaError_t e, const char *what);

#define VB200_CUDA(domain, call) \
	do { \
		cudaError_t e_ = (call); \
		if (e_ != cudaSuccess) \
			return vb200::cuda_fail(domain, e_, #call); \
	} while (0)

/* CUDA refuses a launch whose gridDim.y or gridDim.z exceeds 65 535.  Whole-image kernels take one CTA row per
 * `rows` unit (an image row, or a group of rows): row_grid() caps gridDim.y there and the kernels walk
 * for (y = blockIdx.y; y < rows; y += gridDim.y), so the row count is limited only by memory, and an image of up
 * to 65 535 units launches exactly one CTA row per unit.  Batches of frames in y / z go in chunks of kMaxBatchFrames.
 */
constexpr int kMaxGridY = 65535;
constexpr int kMaxBatchFrames = 32768;
inline dim3
row_grid(int elems, int rows, int threads = 256)
{
	return dim3((elems + threads - 1) / threads, rows < kMaxGridY ? rows : kMaxGridY);
}
/* Whether row_grid(.., rows) caps the grid.  Kernels whose registers grow when the compiler sees a row loop take a
 * template flag LOOP = rows_loop(rows): without it their loop advances straight to the end after one row, so an image of
 * up to kMaxGridY units runs the code it ran with one CTA row per unit.
 */
inline bool
rows_loop(int rows)
{
	return rows > kMaxGridY;
}

cudaStream_t current_stream();
void count_launch(int n = 1);
int sm_count(); /* SMs of the device vb200_init selected: grid sizing fills the machine */
int ensure_init(const char *domain);

struct TileGeometry {
	int tile_width, tile_height, fatstrip_height, thinstrip_height;
};
TileGeometry tile_geometry();

/* Device scratch, stream-ordered (cudaMallocAsync on the current stream). */
int dev_alloc(const char *domain, void **p, size_t bytes, cudaStream_t s);
void dev_free(void *p, cudaStream_t s);

/* A device-resident image: the working type of every op. */
struct DevImage {
	int w = 0, h = 0, bands = 0, fmt = 0, type = 0;
	void *data = nullptr;
	size_t bpl = 0;
	bool owned = false; /* free with dev_free on destruction of the holder */
	bool preset = false; /* data / bpl name the caller's output buffer: dev_image_new() adopts it instead of allocating */
};

size_t format_sizeof(int fmt);
bool format_is_supported(int fmt); /* the 8 real formats minus double */

/* Bring a VB200Image onto the device (no copy if it already is there). */
int to_device(const char *domain, const VB200Image *in, DevImage *d, cudaStream_t s);
/* Deliver a device image into *out following the allocate-or-fill contract, in like's memory (host or device), and
 * release it.  Returns once a host result has landed.
 */
int deliver(const char *domain, DevImage *d, const VB200Image *like, VB200Image *out, cudaStream_t s);
/* deliver()'s host branch without the synchronise: the download is queued on s, d released in stream order */
int deliver_host(const char *domain, DevImage *d, const VB200Image *like, VB200Image *out, cudaStream_t s);
/* After an op that may pass its input through (out->data == in->data, out->owned false): out takes over in's ownership,
 * so that releasing in leaves the buffer to out.
 */
void adopt_pass_through(DevImage *in, DevImage *out);
/* Allocate an owned packed device image. */
int dev_image_new(const char *domain, DevImage *d, int w, int h, int bands, int fmt, int type, cudaStream_t s);
/* Let the op write straight into a device buffer the caller supplied (no device-to-device copy in
 * deliver()), when it cannot alias the input.
 */
void preset_output(DevImage *dout, const VB200Image *in, const VB200Image *out, size_t out_line_bytes, int out_rows);
void dev_image_release(DevImage *d, cudaStream_t s);

/* image_ops.cu: the stand-alone form of a whole-image op (vb200_resize, vb200_conv ..., vb200_icc_import ...).  It checks
 * in and out, runs prepare on the host (refusals that need in's descriptor; *preset_line: the bytes of a result line the
 * op may write straight into a caller's device buffer, 0 never), brings in onto the device, runs apply, delivers the
 * result into *out and releases in.  The whole-image ops themselves, their records and the chain pump live there too.
 */
using ImageApply = std::function<int(const DevImage &in, DevImage *out, cudaStream_t s)>;
int run_image(const char *domain, const VB200Image *in, VB200Image *out, const std::function<int(size_t *preset_line)> &prepare,
	const ImageApply &apply);

/* ------------------------------------------------------------ resample host */

struct ReduceGeom {
	int in_size, out_size, int_shrink, shrunk_size, n_point;
	double residual, offset;
};
int reduce_get_points(int kernel, double shrink);
void reduce_make_mask(double *c, int kernel, int n_points, double shrink, double x);
int reduce_geometry(const char *domain, int in_size, double shrink, int kernel, double gap, ReduceGeom *g);
int shrink_size(int in_size, int shrink, int ceil_mode);

/* Per-output-row (or column) sampling table, built by the same sequential
 * double additions vips_reducev_gen / vips_reduceh_gen perform per rect.
 */
struct AxisTable {
	std::vector<int> first; /* (int) Y: first tap, in embedded coordinates */
	std::vector<int> phase; /* ty / tx, 0..64 */
	int n_point = 0;
	int embed = 0; /* ceil(n_point / 2) - 1 */
	std::vector<short> ms;	/* 65 x n_point, truncated x4096 */
	std::vector<double> mf; /* 65 x n_point */
};
void build_axis_table(AxisTable &t, int out_size, double residual, double offset, int n_point, int kernel,
	int rect_size, int rect_origin = 0, int count = -1);

/* Tables of the tensor-pipe reducev (thumbnail_fused_mma.cuh): per chunk of 8 output rows the
 * {first, last} quad (4 box-shrunk rows) of its window in a ring of 8, and the 32 B fragments
 * {hi b0, hi b1, lo b0, lo b1} of mma.m16n8k32 with the coefficients placed by ring slot.
 * false when a chunk's window does not fit the ring (the plan then uses the dp2a kernels).
 * Pure host code: tests/test_mma_tables.py replays the MMA arithmetic over these tables on the CPU.
 */
bool build_mma_tables(const AxisTable &t, int out_size, int rows, std::vector<int> &vchunk, std::vector<unsigned> &bfrag);
/* the largest rows-per-chunk in 8 .. 4 for which every chunk fits (0: none), with its tables */
int pick_mma_rows(const AxisTable &t, int out_size, std::vector<int> &vchunk, std::vector<unsigned> &bfrag);

/* ------------------------------------------------------- resample device ops */

int dev_shrinkv(const char *domain, const DevImage &in, DevImage *out, int vshrink, int ceil_mode, cudaStream_t s);
int dev_shrinkh(const char *domain, const DevImage &in, DevImage *out, int hshrink, int ceil_mode, cudaStream_t s);
int dev_reducev_pass(const char *domain, const DevImage &in, DevImage *out, const ReduceGeom &g, int kernel,
	int rect_h, cudaStream_t s);
int dev_reduceh_pass(const char *domain, const DevImage &in, DevImage *out, const ReduceGeom &g, int kernel,
	int rect_w, cudaStream_t s);
int dev_reducev(const char *domain, const DevImage &in, DevImage *out, double vshrink, int kernel, double gap,
	int rect_h, cudaStream_t s);
int dev_reduceh(const char *domain, const DevImage &in, DevImage *out, double hshrink, int kernel, double gap,
	int rect_w, cudaStream_t s);
int dev_premultiply(const char *domain, const DevImage &in, DevImage *out, double max_alpha, int uchar_mode,
	cudaStream_t s);
int dev_unpremultiply(const char *domain, const DevImage &in, DevImage *out, double max_alpha, int uchar_mode,
	cudaStream_t s);
int dev_resize(const char *domain, const DevImage &in, DevImage *out, double hscale, double vscale, int kernel,
	double gap, cudaStream_t s);

int dev_reduce_chain(const char *domain, const DevImage &in, DevImage *out, double hshrink, double vshrink, int kernel,
	double gap, cudaStream_t s);

double interpretation_max_alpha(int type);
/* vips_interpretation_bands / vips_image_hasalpha, iofuncs/header.c:217-249, image.c:3113-3119 */
int interpretation_bands(int type);
bool image_hasalpha(int type, int bands);

/* affine.cu */
int dev_resize_up(const char *domain, const DevImage &in, DevImage *out, double hscale, double vscale, int kernel,
	cudaStream_t s);

/* conv.cu */
int dev_conv(const char *domain, const DevImage &in, DevImage *out, const double *mask, int mw, int mh, double scale,
	double offset, int precision, cudaStream_t s, bool allow_vector);
int dev_convsep(const char *domain, const DevImage &in, DevImage *out, const double *mask, int mw, int mh, double scale,
	double offset, int precision, cudaStream_t s, bool allow_vector);
int dev_gaussblur(const char *domain, const DevImage &in, DevImage *out, double sigma, double min_ampl, int precision,
	cudaStream_t s);
int dev_sharpen(const char *domain, const DevImage &in, DevImage *out, double sigma, double x1, double y2, double y3,
	double m1, double m2, cudaStream_t s);

/* morph.cu */
int dev_morph(const char *domain, const DevImage &in, DevImage *out, const double *mask, int mw, int mh, int op, cudaStream_t s);

/* flatten.cu */
int dev_flatten(const char *domain, const DevImage &in, DevImage *out, const double *background, int n, double max_alpha,
	cudaStream_t s);

/* rank.cu */
int dev_rank(const char *domain, const DevImage &in, DevImage *out, int width, int height, int index, cudaStream_t s);
/* histogram.cu: vips_hist_find, vips_hist_equal, vips_hist_local */
int dev_hist_find(const char *domain, const DevImage &in, DevImage *out, int band, cudaStream_t s);
int dev_hist_equal(const char *domain, const DevImage &in, DevImage *out, int band, cudaStream_t s);
int dev_hist_local(const char *domain, const DevImage &in, DevImage *out, int width, int height, int max_slope, cudaStream_t s);
int hist_local_check(const char *domain, int width, int height, int max_slope);
/* kind 0 hist_find, 1 hist_equal, 2 hist_local: the refusals that need in's descriptor and no pixels */
int hist_refuse(const char *domain, int kind, int w, int h, int bands, int fmt, int band, int width, int height);

/* colour.cu */
int dev_colourspace(const char *domain, const DevImage &in, DevImage *out, int space, int source_space,
	cudaStream_t s);

/* colour_ext.cu: the B_W / GREY16 / HSV rows of the route table, composed of the route kernels and three leaf kernels */
bool colour_ext_space(int space);
int dev_colourspace_ext(const char *domain, const DevImage &in, DevImage *out, int space, int source_space, cudaStream_t s);

/* Launchers of the row/column-table kernels on raw device pointers (used by
 * the generate()-shaped and scanline seams too).
 */
/* decode.cu: the decoders' shared driver.  A stream's kind is its signature (PNG, GIF, TIFF, WebP), else JPEG. */
enum StreamKind { STREAM_JPEG, STREAM_PNG, STREAM_GIF, STREAM_TIFF, STREAM_WEBP };
StreamKind stream_kind(const void *buf, size_t len);
/* what to decode: shrink is JPEG's load-time shrink; page / n_pages GIF's and TIFF's pages (n_pages -1: to the last), 0 / 1
 * elsewhere; subifd TIFF's SubIFD of each page (-1: the page's main IFD), -1 elsewhere; scale webpload's scale (read only
 * for WebP: 1 is the plain decode, anything else libwebp's scaled decode) */
struct DecodeRequest {
	StreamKind kind;
	int shrink = 1, page = 0, n_pages = 1;
	int subifd = -1;
	double scale = 1.0;
};
/* A batch's geometry as the decoders report it: frames of h rows, or (pages > 0) strips of `pages` pages of h rows. */
struct StreamGeometry {
	int w = 0, h = 0, bands = 0, pages = 0;
	int rows() const { return h * std::max(1, pages); }
};
/* n streams of one geometry -> out[n][h][w][bands] on the device, out_frame_stride apart (out = nullptr: geometry only, no
 * device call).  *page_h: the page height of a strip of more than one page, else 0.  Outputs may be null. */
int dev_decode_batch(const char *domain, const DecodeRequest &req, const void *const *bufs, const size_t *lens, int n, void *out, size_t out_bpl,
	size_t out_frame_stride, int *w, int *h, int *bands, int *page_h, cudaStream_t s);
/* the body of vb200_{jpeg,png,gif,tiff,webp}_decode_batch: out in host or device memory, or null for the geometry */
int decode_batch_abi(const char *domain, const DecodeRequest &req, const void *const *bufs, const size_t *lens, int n, void *out, int out_location,
	size_t out_bpl, size_t out_frame_stride, int *width, int *height, int *bands);
/* one stream into a new packed device image, B_W below 3 bands and sRGB from 3 */
int dev_load(const char *domain, const DecodeRequest &req, const void *buf, size_t len, DevImage *out, int *page_h, cudaStream_t s);
/* the body of vb200_{jpeg,png,gif,tiff,webp}load_buffer: dev_load, then deliver into *out */
int load_abi(const char *domain, const DecodeRequest &req, const void *buf, size_t len, VB200Image *out);
/* the body of vb200_*_icc_profile: fetch(domain, &profile) (0, or -1 with the reason), *profile_len its length and, unless
 * out is null, its bytes in out[cap] */
int profile_abi(const char *domain, void *out, size_t cap, size_t *profile_len, const std::function<int(const char *, std::vector<unsigned char> *)> &fetch);
/* the body of a host twin's test hook: fn(domain), an exception it throws reported as domain's error */
int host_twin_abi(const char *domain, const std::function<int(const char *)> &fn);
/* the profile a stream embeds (empty: none): JPEG's APP2, PNG's iCCP, the ICCProfile of the TIFF IFD req selects, WebP's ICCP; -1 for a
 * PNG with eXIf or a TIFF IFD whose Orientation is not 1; GIF has none */
int stream_profile(const char *domain, const DecodeRequest &req, const unsigned char *d, size_t n, std::vector<unsigned char> *profile);
/* The pieces of the per-format batch decoders.  parse_streams runs parse(i) for the n streams on the host workers (0, or -1
 * with the reason in the worker's error buffer, restated as "<noun> i: reason") and checks that geometry(i) agrees. */
size_t align16(size_t v);
int parse_streams(const char *domain, const char *noun, int n, const std::function<int(int)> &parse,
	const std::function<StreamGeometry(int)> &geometry, StreamGeometry *g);
/* out_bpl and out_frame_stride hold frames of geometry g */
int check_out_strides(const char *domain, const StreamGeometry &g, size_t out_bpl, size_t out_frame_stride);
/* device bytes per chunk of the PNG, GIF, TIFF and WebP decoders and the JPEG and PNG encoders (vb200_debug_png_set_budget;
 * 0: an eighth of the device, at least 1 GiB) */
size_t chunk_budget();
/* chunk(c0, cn) for consecutive streams [c0, c0 + cn) whose device_bytes fit chunk_budget() (at least one: -1 when
 * that one alone does not), one decode at a time, so that chunk may use decode_staging(); returns once s has finished the
 * chunks' work.  what names the format in the labels of CUDA failures. */
int decode_chunks(const char *domain, const char *what, const char *noun, int n, const std::function<size_t(int)> &device_bytes,
	const std::function<int(int, int)> &chunk, cudaStream_t s);
/* the pinned staging block, grow-only, at least bytes long (nullptr: cudaMallocHost failed, with the reason) */
void *decode_staging(const char *domain, size_t bytes);
void decode_staging_release(); /* vb200_shutdown */
/* A chunk's one device block: [host_bytes that stage(pinned block) writes, copied up in one piece | scratch_bytes |
 * n_status ints, zeroed], each region starting 16-aligned (the scratch at align16(host_bytes)). */
struct DecodeBlock {
	size_t host_bytes = 0, scratch_bytes = 0;
	int n_status = 0;
};
/* One chunk of a PNG, GIF, TIFF or WebP batch on s, inside decode_chunks: the block staged and copied up, decode(dev, status)
 * (the kernels it launched, or -1 with the reason set), then, once they have finished, refuse(k, status[k]) for the first
 * nonzero status word (it sets the reason), else place(dev) (the kernels it launched that write the output, or -1). */
int decode_chunk(const char *domain, const char *what, const DecodeBlock &b, const std::function<void(unsigned char *)> &stage,
	const std::function<int(unsigned char *, int *)> &decode, const std::function<void(int, int)> &refuse,
	const std::function<int(unsigned char *)> &place, cudaStream_t s);

/* The five batch decoders dev_decode_batch switches over (n >= 1; out_frame_stride holds a frame whatever n is). */
/* jpeg.cu: n JPEG streams of one output geometry -> out[n][h][w][bands] on the device (out = nullptr: geometry only) */
int dev_jpeg_decode_batch(const char *domain, const void *const *bufs, const size_t *lens, int n, int shrink, void *out, size_t out_bpl,
	size_t out_frame_stride, StreamGeometry *g, cudaStream_t s);
int host_jpeg_decode(const char *domain, const void *buf, size_t len, int shrink, unsigned char *out, size_t out_bpl, int *out_w,
	int *out_h, int *bands, unsigned sub_bytes, int max_passes, int *passes_used);
/* jpeg_encode.cu: the encoder's host twins (the per-block code on the CPU), one stream appended to out */
int host_jpeg_encode(const char *domain, const unsigned char *img, size_t bpl, int w, int h, int bands, int quality, int subsample_mode, int optimize,
	int restart, std::vector<unsigned char> &out);
int host_jpeg_encode_progressive(const char *domain, const unsigned char *img, size_t bpl, int w, int h, int bands, int quality, int subsample_mode,
	int restart, std::vector<unsigned char> &out, unsigned long long *events);
/* png_encode.cu: the PNG encoder's host twin (the kernels' per-position, per-symbol and per-block code on the CPU), the
 * whole stream into out */
int host_png_encode(const char *domain, const unsigned char *img, size_t bpl, int w, int h, int bands, const VB200PngSaveOptions &o,
	const unsigned char *profile, size_t profile_len, std::vector<unsigned char> &out);
/* encode.cu: the encoders' shared driver.  place(lengths, length_stride, at, &out), which an encoder's chunk calls once its
 * kernels have the streams' lengths (device memory, an unsigned long long every length_stride bytes), reads them back,
 * fails the call for a stream longer than its slot, and stores where each stream goes: stream i at out + at[i] (at: the
 * encoder's device array of the chunk's frames).
 */
using EncodePlace = std::function<int(const void *lengths, size_t length_stride, unsigned long long *at, unsigned char **out)>;
struct Encoder {
	size_t scratch_bytes = 0; /* device scratch per frame of a chunk */
	size_t stream_bytes = 0;  /* a stream's bound: its device room when the streams go to the host */
	/* cn frames on the device (bpl, frame_stride apart): the kernels through the lengths, place, then the write kernel at the
	 * places given */
	std::function<int(const unsigned char *src, size_t bpl, size_t frame_stride, int cn, const EncodePlace &place, cudaStream_t s)> chunk;
};
/* the encoders: the option and geometry checks (0, or -1 with the reason) and, without a device call, *enc */
int jpeg_encoder(const char *domain, int w, int h, int bands, const VB200JpegSaveOptions &o, Encoder *enc);
int png_encoder(const char *domain, int w, int h, int bands, const VB200PngSaveOptions &o, const unsigned char *profile, size_t profile_len,
	Encoder *enc);
/* where the streams go: device slots (stream i at dev + i * slot), or packed host bytes appended to *bytes (stream i at
 * (*bytes)[at[i]]).  A stream longer than slot fails the call before its chunk writes anything. */
struct EncodeDest {
	size_t slot = SIZE_MAX;
	unsigned char *dev = nullptr;
	std::vector<unsigned char> *bytes = nullptr;
	std::vector<size_t> at;
};
/* n frames (host or device memory, rows of `line` bytes) -> n streams into dst, lengths[n], in chunks bounded by
 * chunk_budget() (a frame larger than the budget runs alone); returns with the chunks' work done */
int dev_encode_batch(const char *domain, const Encoder &enc, const void *frames, int frames_location, size_t bpl, size_t frame_stride, int n,
	size_t line, int h, EncodeDest &dst, size_t *lengths, cudaStream_t s);
/* the body of vb200_jpegsave_batch_opts and vb200_pngsave_batch: every argument checked, then make(&enc), before any device
 * call; streams for the host placed in out only once every chunk has succeeded (lengths may be null) */
int encode_batch_abi(const char *domain, const void *options, const std::function<int(Encoder *)> &make, const void *frames, int frames_location,
	size_t bpl, size_t frame_stride, int n, int w, int h, int bands, void *out, int out_location, size_t out_stride, size_t *lengths);
/* min(hshrink, vshrink) of vips_thumbnail_calculate_shrink, thumbnail.c:413-487 */
double thumbnail_common_shrink(int w, int h, int tw, int th, int size);
void jpeg_pump_release(); /* the JPEG pump's pinned / device slots (jpeg.cu); vb200_shutdown */
void resample_cache_clear(); /* cached axis tables (resample_kernels.cu); vb200_shutdown */
/* jpeg.cu: the ICC profile a JPEG stream embeds, as jpeg2vips.c:699-799 reassembles it (*len = 0: none) */
int jpeg_icc_profile(const char *domain, const unsigned char *d, size_t n, std::vector<unsigned char> *profile);
/* png.cu: n PNG streams of one output geometry -> out[n][h][w][bands] on the device (out = nullptr: geometry only, no
 * device call) */
int dev_png_decode_batch(const char *domain, const void *const *bufs, const size_t *lens, int n, void *out, size_t out_bpl, size_t out_frame_stride,
	StreamGeometry *g, cudaStream_t s);
bool png_signature(const void *buf, size_t len);
/* png.cu: the iCCP profile inflated (empty: none); *exif = whether the stream has an eXIf chunk (exif may be null) */
int png_icc_profile(const char *domain, const unsigned char *d, size_t n, std::vector<unsigned char> *profile, bool *exif);
/* gif.cu: n GIF streams of one geometry, pages page .. page + npages - 1 (npages -1: to the last) -> out[n][h * pages][w][bands]
 * on the device, g->h the screen height (out = nullptr: geometry only, no device call) */
int dev_gif_decode_batch(const char *domain, const void *const *bufs, const size_t *lens, int n, int page, int npages, void *out, size_t out_bpl,
	size_t out_frame_stride, StreamGeometry *g, cudaStream_t s);
bool gif_signature(const void *buf, size_t len); /* GIF87a or GIF89a */
/* tiff.cu: n TIFF streams of one geometry, pages page .. page + npages - 1 (npages -1: to the last) at subifd (-1: each
 * page's main IFD) -> out[n][h * pages][w][bands] on the device (out = nullptr: geometry only, no device call) */
int dev_tiff_decode_batch(const char *domain, const void *const *bufs, const size_t *lens, int n, int page, int npages, int subifd, void *out,
	size_t out_bpl, size_t out_frame_stride, StreamGeometry *g, cudaStream_t s);
bool tiff_signature(const void *buf, size_t len); /* II*\0, MM\0*, or BigTIFF's 43 in either order */
/* tiff.cu: the ICCProfile of the IFD page / subifd select (empty: none), and the first Orientation other than 1 among pages
 * page .. page + n_pages - 1 (n_pages -1: to the last; orientation may be null) */
int tiff_icc_profile(const char *domain, const unsigned char *d, size_t len, int page, int n_pages, int subifd, std::vector<unsigned char> *profile,
	int *orientation);
/* tiff.cu: the subifd / page vips_thumbnail_buffer loads for a thumbnail of width x height (thumbnail.c:562-581, 1552-1576) */
int tiff_thumbnail_level(const char *domain, const unsigned char *d, size_t len, int width, int height, int size, int *subifd, int *page);

/* webp.cu: n WebP streams (lossy, still, opaque) of one geometry -> out[n][h][w][3] on the device (out = nullptr: geometry
 * only, no device call); scale != 1: libwebp's scaled decode to rint(w * scale) x rint(h * scale) */
int dev_webp_decode_batch(const char *domain, const void *const *bufs, const size_t *lens, int n, double scale, void *out, size_t out_bpl,
	size_t out_frame_stride, StreamGeometry *g, cudaStream_t s);
bool webp_signature(const void *buf, size_t len); /* RIFF, 4 bytes, WEBP */
/* webp.cu: the ICCP chunk of a VP8X stream (empty: none) */
int webp_icc_profile(const char *domain, const unsigned char *d, size_t len, std::vector<unsigned char> *profile);

/* the decoders' host workers: VB200_JPEG_THREADS, else the CPUs this process may run on, at most 16 (jpeg.cu) */
int host_workers();
/* run fn(i) for i in [0, n) on up to `threads` host threads */
template <typename Fn>
void
parallel_for(int n, int threads, Fn fn)
{
	threads = std::max(1, std::min(threads, n));
	if (threads == 1) {
		for (int i = 0; i < n; i++)
			fn(i);
		return;
	}
	std::atomic<int> next(0);
	std::vector<std::thread> pool;
	for (int t = 0; t < threads; t++)
		pool.emplace_back([&] {
			for (;;) {
				const int i = next.fetch_add(1);
				if (i >= n)
					return;
				fn(i);
			}
		});
	for (auto &t : pool)
		t.join();
}

/* icc.cu: the colour-management stage of the thumbnail plan (vb200_thumbnail_plan_set_icc / _set_linear_icc).  Frames are
 * 8-bit, `bands` bands in, *out_bands out; each frame's input profile is chosen as vips_icc_set_import does.  The stage has
 * two modes, fixed by icc_stage_set:
 *   - after the thumbnail kernel (linear = false): one job per frame, the transform from its input profile or the XYZ export,
 *     run over a batch by icc_stage_run in one launch per kMaxBatchFrames frames;
 *   - linear (thumbnail.c:766-805, 929-987): the import runs inside the linear thumbnail's V kernel and the export inside its
 *     H kernel (thumbnail_linear.cu), or in the leaf chain around the float resize.  Each frame takes one of:
 *       LIN_PLAIN   sRGB -> scRGB ... scRGB -> sRGB, the linear thumbnail without a profile anywhere;
 *       LIN_IMPORT  vips_icc_import(XYZ PCS) ... vips_icc_export from XYZ (thumbnail.c:766-789, 929-942: a profile to import with);
 *       LIN_XYZ     sRGB -> scRGB ... scRGB -> XYZ, vips_icc_export from XYZ (:790-805, 957-970: only an output profile).
 */
struct IccStage;
IccStage *icc_stage_new();
void icc_stage_free(IccStage *st);
/* the stage's profiles (copied) and mode; refuses 1- and 2-band frames in linear mode, and needs an output profile outside it */
int icc_stage_set(const char *domain, IccStage *st, const VB200ThumbnailIcc *icc, int bands, bool linear, int *out_bands);
int icc_debug_select(const VB200ThumbnailIcc *icc, int bands, const void *embedded, size_t embedded_len, int *source);
int icc_debug_classify(const void *profile, size_t len, int want_bands, int intent);

enum { LIN_PLAIN = 0, LIN_IMPORT = 1, LIN_XYZ = 2 };
/* one frame's jobs, indices into the batch's job table: a linear frame's LIN_* kind and its import and export jobs (-1: none);
 * a frame of the other mode has its one job in exp
 */
struct IccFrame {
	int kind, imp, exp;
};
struct IccJob; /* icc_eval.cuh */
/* one batch's resolved jobs: device copies for the kernels, host copies (device pool pointers) for the leaf chain */
struct IccBatch {
	const IccJob *d_jobs;
	const IccFrame *d_frames;
	const IccJob *h_jobs;
	const IccFrame *h_frames;
};
/* resolves the n frames' jobs in the stage's mode (embedded / embedded_lens: each frame's embedded profile, NULL arrays or a NULL
 * entry: none), uploads them on s and calls body with them, the stage locked and its cache entries held until the launches body
 * queues have been recorded.  frame0: the index of the first frame in the caller's batch, for the errors that name a frame (the
 * host pump runs a batch in slices)
 */
int icc_stage_batch(const char *domain, IccStage *st, int n, const void *const *embedded, const size_t *embedded_lens,
	cudaStream_t s, int frame0, const std::function<int(const IccBatch &)> &body);
/* the stage after the thumbnail kernel: icc_stage_batch with icc_frames_kernel over n frames of `pixels` pixels */
int icc_stage_run(const char *domain, IccStage *st, const void *in, size_t in_stride, void *out, size_t out_stride, int n, size_t pixels,
	const void *const *embedded, const size_t *embedded_lens, cudaStream_t s, int frame0);
/* the leaf chain's ICC steps: jobs[k] over a packed device image (icc_kernel, as vb200_icc_import / _export launch it) */
int icc_job_apply(const char *domain, const IccJob *jobs, int k, const DevImage &in, DevImage *out, cudaStream_t s);
/* test hook: one frame's linear-mode choice (*branch LIN_*, *source as icc_debug_select or -1, *export_from 0 output_profile,
 * 1 the import's profile, -1 none) */
int icc_debug_select_linear(const VB200ThumbnailIcc *icc, int bands, const void *embedded, size_t embedded_len, int *branch,
	int *source, int *export_from);

int launch_reducev(const char *domain, const void *in, size_t in_bpl, int in_h, void *out, size_t out_bpl, int ne,
	int out_rows, int fmt, const AxisTable &t, cudaStream_t s);
int launch_reduceh(const char *domain, const void *in, size_t in_bpl, int in_w, void *out, size_t out_bpl, int bands,
	int out_cols, int rows, int fmt, const AxisTable &t, cudaStream_t s);

} // namespace vb200

#endif
