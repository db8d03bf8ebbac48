/* vb200_internal.h -- shared declarations inside libvb200.so (not installed). */
#ifndef VB200_INTERNAL_H
#define VB200_INTERNAL_H

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
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
int cuda_fail(const char *domain, cudaError_t e, const char *what);

#define VB200_CUDA(domain, call) \
	do { \
		cudaError_t e_ = (call); \
		if (e_ != cudaSuccess) \
			return vb200::cuda_fail(domain, e_, #call); \
	} while (0)

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
/* Deliver a device image into *out following the allocate-or-fill contract. */
int deliver(const char *domain, DevImage *d, const VB200Image *like, VB200Image *out, cudaStream_t s);
/* Allocate an owned packed device image. */
int dev_image_new(const char *domain, DevImage *d, int w, int h, int bands, int fmt, int type, cudaStream_t s);
/* Let the op write straight into a device buffer the caller supplied (no device-to-device copy in
 * deliver()), when it cannot alias the input.
 */
void preset_output(DevImage *dout, const VB200Image *in, const VB200Image *out, size_t out_line_bytes, int out_rows);
void dev_image_release(DevImage *d, cudaStream_t s);

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

/* colour.cu */
int dev_colourspace(const char *domain, const DevImage &in, DevImage *out, int space, int source_space,
	cudaStream_t s);

/* colour_ext.cu: the B_W / GREY16 / HSV rows of the route table, composed of the route kernels and three leaf kernels */
bool colour_ext_space(int space);
int dev_colourspace_ext(const char *domain, const DevImage &in, DevImage *out, int space, int source_space, cudaStream_t s);

/* Launchers of the row/column-table kernels on raw device pointers (used by
 * the generate()-shaped and scanline seams too).
 */
/* jpeg.cu: n JPEG streams of one output geometry -> out[n][h][w][bands] on the device (out = nullptr: geometry only) */
int dev_jpeg_decode_batch(const char *domain, const void *const *bufs, const size_t *lens, int n, int shrink, void *out, size_t out_bpl,
	size_t out_frame_stride, int *out_w, int *out_h, int *bands, cudaStream_t s);
int host_jpeg_decode(const char *domain, const void *buf, size_t len, int shrink, unsigned char *out, size_t out_bpl, int *out_w,
	int *out_h, int *bands, unsigned sub_bytes, int max_passes, int *passes_used);
/* min(hshrink, vshrink) of vips_thumbnail_calculate_shrink, thumbnail.c:413-487 */
double thumbnail_common_shrink(int w, int h, int tw, int th, int size);
void jpeg_pump_release(); /* the JPEG pump's pinned / device slots (jpeg.cu); vb200_shutdown */
void resample_cache_clear(); /* cached axis tables (resample_kernels.cu); vb200_shutdown */
int launch_reducev(const char *domain, const void *in, size_t in_bpl, int in_h, void *out, size_t out_bpl, int ne,
	int out_rows, int fmt, const AxisTable &t, cudaStream_t s);
int launch_reduceh(const char *domain, const void *in, size_t in_bpl, int in_w, void *out, size_t out_bpl, int bands,
	int out_cols, int rows, int fmt, const AxisTable &t, cudaStream_t s);

} // namespace vb200

#endif
