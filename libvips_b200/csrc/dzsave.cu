/* dzsave.cu -- vips_dzsave (foreign/dzsave.c) in its "dz" and "zoomify" layouts with JPEG or PNG tiles, on the device.
 *
 * What the reference does: pyramid_build (:441-577) makes a chain of levels, each half the size of the one above, rounded
 * up; vips_sink_disc feeds the top level strips of rows (pyramid_strip :1942-2014); a level that has a line of tiles
 * writes them (strip_save :1653-1703, one vips_jpegsave per tile: image_strip_allocate :1106-1152, write_image :369-404)
 * and shrinks the strip into the level below (strip_shrink :1761-1835) after level_generate_extras (:1710-1754) has
 * repeated the last column / row of a level of odd size; the shrink is vips_region_shrink_uncoded_mean
 * (iofuncs/region.c:1139-1156), (p00 + p01 + p10 + p11 + 2) >> 2 per band.  With PNG tiles (vb200_dzsave_png) the
 * tiles are vips_image_write_to_buffer(tile, ".png") (write_image :369-402, spngsave's defaults) and an image with alpha
 * (vips_image_hasalpha: more bands than its Type has, iofuncs/image.c:3113-3119) is shrunk by vips_region_shrink_alpha
 * instead (region.c:1444-1482, 1551-1573, whatever region_shrink says): dz_shrink_alpha.
 *
 * Stated over whole images, which is what runs here: level k - 1 is the 2 x 2 rounded mean of level k with its last column /
 * row read twice when its width / height is odd, and tile (x, y) of a level is the rect [x * step - margin, y * step -
 * margin, size + 2 * margin, size + 2 * margin] clipped to the level.  tests/test_dzsave.py holds this against a loop for
 * loop restatement of the strip walk (oracle/pydz.py) at every size that takes a different branch there.
 *
 * Device pipeline, nothing but the finished streams crossing back to the host:
 *   dz_pyramid_kernel   a CTA loads a 64 x 64 block of level L once (16-byte loads when the rows allow) and reduces it in
 *                       shared memory to levels L-1 .. L-4, so four levels cost one read of the largest; the rounding is
 *                       per level, so the levels cannot be folded into one wide box, and each level applies its own
 *                       odd-edge rule from its own size.  All levels stay in device memory: 4/3 of the input.
 *                       With alpha (2 or 4 bands) a thread makes one output pixel from all the bands of its four.
 *   dz_gather_kernel    the tiles of one shape (w, h), from every level, copied into one batch [n][h][w][bands], driven by
 *                       a table of source pointers built on the host
 *   the encoder         the encoders' batch driver per shape batch (encode.cu), device in: the streams packed end to end
 *                       on the device, so the one device-to-host copy per chunk moves their bytes and not their slots
 * With the defaults a 16384 x 16384 image is 5 730 tiles in 45 shapes, 5 214 of them 256 x 256.
 */
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include <strings.h>

#include "../../include/vb200.h"
#include "vb200_internal.h"

namespace vb200 {

struct DzLevel {
	int w, h, across, down;
};

struct DzTile {
	int level, x, y, left, top, w, h;
	size_t off, len; /* its stream in VB200DzPyramid::bytes */
};

} // namespace vb200

struct VB200DzPyramid {
	int layout = 0, tile_size = 0, overlap = 0, bands = 0;
	std::string suffix;
	std::vector<vb200::DzLevel> levels; /* by the reference's n: 0 is the smallest */
	std::vector<vb200::DzTile> tiles;	/* level 0 first, then down, then across */
	std::vector<unsigned char> bytes;
};

namespace vb200 {

namespace {

#define HD __host__ __device__ __forceinline__

/* region.c:1146-1149 */
HD int
dz_mean(int a, int b, int c, int d)
{
	return (a + b + c + d + 2) >> 2;
}

/* SHRINK_ALPHA_TYPE (region.c:1446-1482) for uchar, the last band alpha: in double there, a = (a1 + a2 + a3 + a4) / 4.0,
 * each colour band (a1 p1 + a2 p2 + a3 p3 + a4 p4) / (4.0 a), alpha a, every band 0 when a == 0, each truncated to uchar.
 * With S = a1 + a2 + a3 + a4 that is integer arithmetic: 4.0 a == S exactly, so alpha is S >> 2; the numerator is below
 * 2^18, exact in double, and a quotient that is not an integer is at least 1 / S >= 1 / 1020 from one, far more than the
 * division's rounding error, so truncating it is the integer quotient.
 */
HD void
dz_shrink_alpha(const unsigned char *p00, const unsigned char *p01, const unsigned char *p10, const unsigned char *p11, int bands,
	unsigned char *q)
{
	const unsigned a1 = p00[bands - 1], a2 = p01[bands - 1], a3 = p10[bands - 1], a4 = p11[bands - 1], S = a1 + a2 + a3 + a4;
	if (S == 0) {
		for (int b = 0; b < bands; b++)
			q[b] = 0;
		return;
	}
	for (int b = 0; b < bands - 1; b++)
		q[b] = (unsigned char) ((a1 * p00[b] + a2 * p01[b] + a3 * p10[b] + a4 * p11[b]) / S);
	q[bands - 1] = (unsigned char) (S >> 2);
}

/* vips_image_hasalpha of the images the device path takes: 2 and 4 bands are B_W / sRGB with alpha */
HD bool
dz_alpha(int bands)
{
	return bands == 2 || bands == 4;
}

/* one level from the one above, whole image: pixel (x, y) from columns 2x and 2x + 1 (2x again when that is past the
 * level's own last column: level_generate_extras), rows likewise
 */
void
host_shrink_level(const unsigned char *src, size_t bpl, int w, int h, int bands, unsigned char *dst)
{
	const int ow = (w + 1) / 2, oh = (h + 1) / 2;
	for (int y = 0; y < oh; y++) {
		const unsigned char *r0 = src + (size_t) (2 * y) * bpl, *r1 = src + (size_t) std::min(2 * y + 1, h - 1) * bpl;
		unsigned char *q = dst + (size_t) y * ow * bands;
		for (int x = 0; x < ow; x++) {
			const int c0 = 2 * x * bands, c1 = std::min(2 * x + 1, w - 1) * bands;
			if (dz_alpha(bands))
				dz_shrink_alpha(r0 + c0, r0 + c1, r1 + c0, r1 + c1, bands, q + x * bands);
			else
				for (int b = 0; b < bands; b++)
					q[x * bands + b] = (unsigned char) dz_mean(r0[c0 + b], r0[c1 + b], r1[c0 + b], r1[c1 + b]);
		}
	}
}

constexpr int kDzBlock = 64;  /* pixels of level L a CTA loads, each way */
constexpr int kDzFuse = 4;	  /* levels one launch writes */
constexpr int kDzThreads = 256;

struct DzPyramidArgs {
	const unsigned char *src;
	size_t src_bpl;
	int w, h; /* of src */
	int n;	  /* levels to write, 1 .. kDzFuse */
	int blocks_y;
	unsigned char *dst[kDzFuse];
	size_t dst_bpl[kDzFuse]; /* multiples of 16, on 16-byte aligned bases: a block's rows start on a word */
};

template <int BANDS>
__global__ void __launch_bounds__(kDzThreads)
dz_pyramid_kernel(const DzPyramidArgs A)
{
	constexpr int kSrcPitch = kDzBlock * BANDS;
	constexpr int kChunks = kSrcPitch / 16;
	/* the block of level L, then levels L-1 .. L-4 of it: 32 x 32, 16 x 16, 8 x 8, 4 x 4 pixels */
	__shared__ __align__(16) unsigned char s_src[kDzBlock * kSrcPitch];
	__shared__ __align__(16) unsigned char s_out[(32 * 32 + 16 * 16 + 8 * 8 + 4 * 4) * BANDS];
	const int tid = threadIdx.x;
	/* RGB rows are not pixel aligned: rows are loaded as bytes, 16 at a time when the image's base and stride allow */
	const bool vec = (((size_t) A.src | A.src_bpl) & 15) == 0;
	for (int by = blockIdx.y; by < A.blocks_y; by += gridDim.y) {
		const int x0 = blockIdx.x * kDzBlock, y0 = by * kDzBlock;
		const int rows = min(kDzBlock, A.h - y0), valid = min(kDzBlock, A.w - x0) * BANDS;
		const unsigned char *g = A.src + (size_t) y0 * A.src_bpl + (size_t) x0 * BANDS;
		for (int i = tid; i < rows * kChunks; i += kDzThreads) {
			const int r = i / kChunks, b0 = (i - r * kChunks) * 16;
			if (b0 >= valid)
				continue;
			const unsigned char *p = g + (size_t) r * A.src_bpl + b0;
			unsigned char *q = s_src + r * kSrcPitch + b0;
			if (vec && b0 + 16 <= valid)
				*(uint4 *) q = __ldg((const uint4 *) p);
			else
				for (int k = 0; k < 16 && b0 + k < valid; k++)
					q[k] = p[k];
		}
		__syncthreads();
		const unsigned char *from = s_src;
		unsigned char *to = s_out;
		int fpitch = kSrcPitch, fw = A.w, fh = A.h, fx0 = x0, fy0 = y0, n = kDzBlock / 2;
		for (int l = 0; l < A.n; l++) {
			/* this level's size and this block's origin in it; the edge rule comes from the size of the level read */
			const int ow = (fw + 1) >> 1, oh = (fh + 1) >> 1, ox0 = fx0 >> 1, oy0 = fy0 >> 1, pitch = n * BANDS;
			if (dz_alpha(BANDS))
				/* one thread per output pixel: the alpha weights every band of it */
				for (int i = tid; i < n * n; i += kDzThreads) {
					const int y = i / n, x = i - y * n;
					if (ox0 + x >= ow || oy0 + y >= oh)
						continue;
					const int c0 = 2 * x * BANDS, c1 = (2 * (ox0 + x) + 1 < fw ? 2 * x + 1 : 2 * x) * BANDS;
					const unsigned char *r0 = from + 2 * y * fpitch, *r1 = from + (2 * (oy0 + y) + 1 < fh ? 2 * y + 1 : 2 * y) * fpitch;
					dz_shrink_alpha(r0 + c0, r0 + c1, r1 + c0, r1 + c1, BANDS, to + y * pitch + x * BANDS);
				}
			else
				for (int i = tid; i < n * pitch; i += kDzThreads) {
					const int y = i / pitch, xb = i - y * pitch, x = xb / BANDS, b = xb - x * BANDS;
					if (ox0 + x >= ow || oy0 + y >= oh)
						continue;
					const int c0 = 2 * x * BANDS + b, c1 = (2 * (ox0 + x) + 1 < fw ? 2 * x + 1 : 2 * x) * BANDS + b;
					const int r0 = 2 * y * fpitch, r1 = (2 * (oy0 + y) + 1 < fh ? 2 * y + 1 : 2 * y) * fpitch;
					to[i] = (unsigned char) dz_mean(from[r0 + c0], from[r0 + c1], from[r1 + c0], from[r1 + c1]);
				}
			__syncthreads();
			const int orows = min(n, oh - oy0), ovalid = min(n, ow - ox0) * BANDS, words = pitch / 4;
			unsigned char *d = A.dst[l] + (size_t) oy0 * A.dst_bpl[l] + (size_t) ox0 * BANDS;
			for (int i = tid; i < orows * words; i += kDzThreads) {
				const int r = i / words, c = (i - r * words) * 4;
				if (c >= ovalid)
					continue;
				unsigned char *q = d + (size_t) r * A.dst_bpl[l] + c;
				const unsigned char *p = to + r * pitch + c;
				if (c + 4 <= ovalid)
					*(unsigned *) q = *(const unsigned *) p;
				else
					for (int k = 0; c + k < ovalid; k++)
						q[k] = p[k];
			}
			from = to;
			fpitch = pitch;
			fw = ow;
			fh = oh;
			fx0 = ox0;
			fy0 = oy0;
			to += n * pitch;
			n >>= 1;
		}
		__syncthreads();
	}
}

/* where a tile's pixels start in its level */
struct DzGatherTile {
	const unsigned char *src;
	size_t bpl;
};

/* tile blockIdx.y of the batch: h rows of row_bytes from its level into out + tile * frame_stride, packed.  A thread
 * writes one word of the packed tile from four byte loads: a tile's left edge falls on any byte of its level's row.
 */
__global__ void __launch_bounds__(kDzThreads)
dz_gather_kernel(const DzGatherTile *__restrict__ tiles, int row_bytes, int h, unsigned char *__restrict__ out, size_t frame_stride)
{
	const DzGatherTile t = tiles[blockIdx.y];
	const int total = row_bytes * h, words = (total + 3) / 4;
	unsigned *o = (unsigned *) (out + (size_t) blockIdx.y * frame_stride);
	for (int j = blockIdx.x * kDzThreads + threadIdx.x; j < words; j += gridDim.x * kDzThreads) {
		int r = (4 * j) / row_bytes, c = 4 * j - r * row_bytes;
		unsigned v = 0;
		for (int k = 0; k < 4 && 4 * j + k < total; k++) {
			v |= (unsigned) t.src[(size_t) r * t.bpl + c] << (8 * k);
			if (++c == row_bytes) {
				c = 0;
				r++;
			}
		}
		o[j] = v;
	}
}

/* device scratch of one call: everything still held is freed when the call leaves, whichever way */
struct DzScratch {
	cudaStream_t s;
	std::vector<void *> held;
	explicit DzScratch(cudaStream_t s_) : s(s_) {}
	~DzScratch()
	{
		for (void *p : held)
			dev_free(p, s);
	}
	int
	alloc(const char *domain, void **p, size_t bytes)
	{
		if (dev_alloc(domain, p, bytes, s))
			return -1;
		held.push_back(*p);
		return 0;
	}
	void
	release(void *p)
	{
		held.erase(std::remove(held.begin(), held.end(), p), held.end());
		dev_free(p, s);
	}
};

struct DevLevel {
	unsigned char *p;
	size_t bpl;
	int w, h;
};

/* levels[0] = the image as given; `count` - 1 more below it, each allocated from sc with 16-byte aligned rows */
int
dev_pyramid(const char *domain, const unsigned char *top, size_t bpl, int w, int h, int bands, int count, std::vector<DevLevel> &L, DzScratch &sc)
{
	L.clear();
	L.push_back({(unsigned char *) top, bpl, w, h});
	for (int k = 1; k < count; k++) {
		const int lw = (L[k - 1].w + 1) / 2, lh = (L[k - 1].h + 1) / 2;
		DevLevel l = {nullptr, ((size_t) lw * bands + 15) & ~(size_t) 15, lw, lh};
		if (sc.alloc(domain, (void **) &l.p, l.bpl * lh))
			return -1;
		L.push_back(l);
	}
	for (int k = 0; k + 1 < count; k += kDzFuse) {
		DzPyramidArgs A;
		A.src = L[k].p;
		A.src_bpl = L[k].bpl;
		A.w = L[k].w;
		A.h = L[k].h;
		A.n = std::min(kDzFuse, count - 1 - k);
		for (int l = 0; l < kDzFuse; l++) {
			A.dst[l] = l < A.n ? L[k + 1 + l].p : nullptr;
			A.dst_bpl[l] = l < A.n ? L[k + 1 + l].bpl : 0;
		}
		A.blocks_y = (A.h + kDzBlock - 1) / kDzBlock;
		const dim3 grid((A.w + kDzBlock - 1) / kDzBlock, std::min(A.blocks_y, kMaxGridY));
		if (bands == 1)
			dz_pyramid_kernel<1><<<grid, kDzThreads, 0, sc.s>>>(A);
		else if (bands == 2)
			dz_pyramid_kernel<2><<<grid, kDzThreads, 0, sc.s>>>(A);
		else if (bands == 3)
			dz_pyramid_kernel<3><<<grid, kDzThreads, 0, sc.s>>>(A);
		else
			dz_pyramid_kernel<4><<<grid, kDzThreads, 0, sc.s>>>(A);
		VB200_CUDA(domain, cudaGetLastError());
		count_launch();
	}
	return 0;
}

const char *const kLayoutNames[] = {"dz", "zoomify", "google", "iiif", "iiif3"};

/* what every tile is written as: vb200_dzsave's JPEG, or vb200_dzsave_png's PNG */
struct DzCodec {
	bool png = false;
	VB200JpegSaveOptions jpeg;
	VB200PngSaveOptions pngo;
};

/* the device encoder of one tile shape (no device call) */
int
tile_encoder(const char *domain, const DzCodec &c, int w, int h, int bands, Encoder *enc)
{
	return c.png ? png_encoder(domain, w, h, bands, c.pngo, nullptr, 0, enc) : jpeg_encoder(domain, w, h, bands, c.jpeg, enc);
}

/* one tile's stream through the encoder's host twin, appended to out */
int
host_tile_encode(const char *domain, const DzCodec &c, const unsigned char *p, size_t bpl, int w, int h, int bands, std::vector<unsigned char> &out)
{
	if (c.png) {
		std::vector<unsigned char> one;
		if (host_png_encode(domain, p, bpl, w, h, bands, c.pngo, nullptr, 0, one))
			return -1;
		out.insert(out.end(), one.begin(), one.end());
		return 0;
	}
	const VB200JpegSaveOptions &j = c.jpeg;
	unsigned long long events[3]; /* the progressive coder's counters, a test hook of its own */
	return j.interlace ? host_jpeg_encode_progressive(domain, p, bpl, w, h, bands, j.Q, j.subsample_mode, j.restart_interval, out, events)
					   : host_jpeg_encode(domain, p, bpl, w, h, bands, j.Q, j.subsample_mode, j.optimize_coding != 0, j.restart_interval, out);
}

/* options and geometry: vips_foreign_save_dz_build :2043-2113, pyramid_build :441-577, image_strip_allocate :1132-1145.
 * c->png on entry picks the tiles; png: their options (NULL: spngsave's defaults).
 */
int
dz_plan(const char *domain, const VB200Image *in, const VB200DzOptions *options, const VB200PngSaveOptions *png, VB200DzPyramid *P, DzCodec *c)
{
	if (!in || !in->data) {
		error(domain, "no input image");
		return -1;
	}
	if (in->Xsize < 1 || in->Ysize < 1) {
		error(domain, "bad image dimensions %d x %d", in->Xsize, in->Ysize);
		return -1;
	}
	if (in->BandFmt != VB200_FORMAT_UCHAR) {
		/* the reference casts to uchar first (:2020-2023): the host keeps that */
		error(domain, "band format %d not supported on the device path (uchar only)", in->BandFmt);
		return -1;
	}
	if (!c->png && in->Bands != 1 && in->Bands != 3) {
		error(domain, "%d-band images not supported on the device path (1 or 3 bands: the JPEG saver would flatten or drop the others)", in->Bands);
		return -1;
	}
	if (c->png && (in->Bands < 1 || in->Bands > 4)) {
		error(domain, "%d-band images not supported on the device path (1 to 4 bands with PNG tiles)", in->Bands);
		return -1;
	}
	/* spngsave runs vips_colourspace to B_W below 3 bands and to sRGB from 3 (spngsave.c:621-641), and hasalpha reads the
	 * Type: with any other Type the pixels saved would not be these
	 */
	const int want_type = in->Bands < 3 ? VB200_INTERPRETATION_B_W : VB200_INTERPRETATION_sRGB;
	if (c->png && in->Type != want_type) {
		error(domain, "interpretation %d with %d bands not supported on the device path (PNG tiles take B_W with 1-2 bands, sRGB with 3-4)",
			in->Type, in->Bands);
		return -1;
	}
	if (in->bpl && in->bpl < (size_t) in->Xsize * in->Bands) {
		error(domain, "line stride %zu too small for %d x %d", in->bpl, in->Xsize, in->Bands);
		return -1;
	}
	VB200DzOptions o;
	memset(&o, 0, sizeof(o));
	o.overlap = -1;
	if (options)
		o = *options;
	if (o.layout != VB200_DZ_LAYOUT_DZ && o.layout != VB200_DZ_LAYOUT_ZOOMIFY) {
		if (o.layout > 0 && o.layout <= VB200_DZ_LAYOUT_IIIF3)
			error(domain, "layout %s not supported on the device path", kLayoutNames[o.layout]);
		else
			error(domain, "unknown layout %d", o.layout);
		return -1;
	}
	if (o.region_shrink != 0) {
		error(domain, "region_shrink other than mean not supported on the device path");
		return -1;
	}
	if (o.skip_blanks != 0) {
		error(domain, "skip_blanks not supported on the device path");
		return -1;
	}
	if (o.container != 0) {
		error(domain, "zip containers not supported on the device path");
		return -1;
	}
	const bool dz = o.layout == VB200_DZ_LAYOUT_DZ;
	P->suffix = o.suffix ? o.suffix : c->png ? ".png" : (dz ? ".jpeg" : ".jpg");
	if (P->suffix.find('[') != std::string::npos) {
		error(domain, "suffix options not supported on the device path");
		return -1;
	}
	if (c->png && strcasecmp(P->suffix.c_str(), ".png") != 0) {
		error(domain, "suffix %s not supported on the device path (PNG tiles here; vb200_dzsave takes JPEG suffixes)", P->suffix.c_str());
		return -1;
	}
	if (!c->png && strcasecmp(P->suffix.c_str(), ".jpg") != 0 && strcasecmp(P->suffix.c_str(), ".jpeg") != 0) {
		error(domain, "suffix %s not supported on the device path (JPEG tiles only%s)", P->suffix.c_str(),
			strcasecmp(P->suffix.c_str(), ".png") == 0 ? "; vb200_dzsave_png takes PNG tiles" : "");
		return -1;
	}
	P->layout = o.layout;
	P->bands = in->Bands;
	P->tile_size = o.tile_size ? o.tile_size : (dz ? 254 : 256);
	P->overlap = o.overlap == -1 ? (dz ? 1 : 0) : o.overlap;
	/* the reference's argument ranges (:2595-2605) */
	if (P->tile_size < 1 || P->tile_size > 8192 || P->overlap < 0 || P->overlap > 8192) {
		error(domain, "tile_size %d / overlap %d out of range", P->tile_size, P->overlap);
		return -1;
	}
	const int margin = dz ? P->overlap : 0, step = dz ? P->tile_size : P->tile_size - P->overlap;
	if (step <= 0) {
		error(domain, "overlap too large");
		return -1;
	}
	/* The reference's strips hold one line of tiles (an even number of rows), and at the bottom of a level strip_flush
	 * (:1925-1937) writes one more line at most; with steps this short the image can end more than one line of tiles
	 * before the strip does, and the reference leaves those tiles out.  Not worth matching: the host keeps it.
	 */
	if (2 * step < P->tile_size + (P->tile_size & 1)) {
		error(domain, "an overlap above half the tile size is not supported on the device path");
		return -1;
	}
	if (o.depth < VB200_DZ_DEPTH_DEFAULT || o.depth > VB200_DZ_DEPTH_ONE) {
		error(domain, "unknown depth %d", o.depth);
		return -1;
	}
	const int depth = o.depth ? o.depth : (dz ? VB200_DZ_DEPTH_ONEPIXEL : VB200_DZ_DEPTH_ONETILE);
	int w = in->Xsize, h = in->Ysize;
	const int limit = depth == VB200_DZ_DEPTH_ONEPIXEL ? 1 : depth == VB200_DZ_DEPTH_ONETILE ? P->tile_size : std::max(w, h);
	for (;;) {
		P->levels.push_back({w, h, (w + step - 1) / step, (h + step - 1) / step});
		if (w <= limit && h <= limit)
			break;
		w = (w + 1) / 2;
		h = (h + 1) / 2;
	}
	std::reverse(P->levels.begin(), P->levels.end());
	const int full = P->tile_size + 2 * margin;
	for (int n = 0; n < (int) P->levels.size(); n++) {
		const DzLevel &l = P->levels[n];
		for (int y = 0; y < l.down; y++)
			for (int x = 0; x < l.across; x++) {
				DzTile t;
				t.level = n;
				t.x = x;
				t.y = y;
				t.left = std::max(0, x * step - margin);
				t.top = std::max(0, y * step - margin);
				t.w = std::min(l.w, x * step - margin + full) - t.left;
				t.h = std::min(l.h, y * step - margin + full) - t.top;
				t.off = t.len = 0;
				P->tiles.push_back(t);
			}
	}
	if (!c->png) {
		c->jpeg = o.jpeg;
		if (c->jpeg.Q == 0)
			c->jpeg.Q = 75;
		return 0;
	}
	/* spngsave's defaults (spngsave.c:700-748): compression 6, filter NONE, no interlace, 8 bits, Xres 1 */
	const VB200PngSaveOptions defaults = {6, 0, 1.0, 0, 0, 8};
	c->pngo = png ? *png : defaults;
	/* the encoder's own checks, once, before any device call: its geometry limit grows with the tile, so the largest shape */
	const DzLevel &top = P->levels.back();
	Encoder enc;
	return png_encoder(domain, std::min(top.w, full), std::min(top.h, full), in->Bands, c->pngo, nullptr, 0, &enc);
}

std::atomic<size_t> g_budget{0};
/* JPEG tiles' default batch bound.  PNG tiles take chunk_budget(), the PNG codecs' own: at ~20 bytes of deflate scratch a
 * scanline byte, 1 GiB holds only ~180 RGBA tiles of 256 x 256, and the parse kernel runs one warp a tile. */
constexpr size_t kDzBudget = (size_t) 1 << 30;

struct DzTimer {
	bool on;
	cudaEvent_t a = nullptr, b = nullptr;
	float ms[4] = {0, 0, 0, 0};
	cudaStream_t s;
	explicit DzTimer(cudaStream_t s_) : s(s_)
	{
		const char *e = getenv("VB200_DZ_TIMING");
		on = e && *e && cudaEventCreate(&a) == cudaSuccess && cudaEventCreate(&b) == cudaSuccess;
	}
	~DzTimer()
	{
		if (a)
			cudaEventDestroy(a);
		if (b)
			cudaEventDestroy(b);
	}
	void
	begin()
	{
		if (on)
			cudaEventRecord(a, s);
	}
	void
	end(int k)
	{
		float t = 0;
		if (on && cudaEventRecord(b, s) == cudaSuccess && cudaEventSynchronize(b) == cudaSuccess && cudaEventElapsedTime(&t, a, b) == cudaSuccess)
			ms[k] += t;
	}
};
thread_local float t_dz_ms[4] = {-1, -1, -1, -1};

int
dev_dzsave(const char *domain, const VB200Image *in, VB200DzPyramid *P, const DzCodec &codec, cudaStream_t s)
{
	DzScratch sc(s);
	DzTimer timer(s);
	const int bands = in->Bands, nl = (int) P->levels.size();
	const size_t line = (size_t) in->Xsize * bands;
	const unsigned char *top = (const unsigned char *) in->data;
	size_t top_bpl = in->bpl ? in->bpl : line;
	if (in->where != VB200_DEVICE) {
		void *d = nullptr;
		top_bpl = (line + 15) & ~(size_t) 15;
		if (sc.alloc(domain, &d, top_bpl * in->Ysize))
			return -1;
		VB200_CUDA(domain, cudaMemcpy2DAsync(d, top_bpl, in->data, in->bpl ? in->bpl : line, line, in->Ysize, cudaMemcpyHostToDevice, s));
		top = (const unsigned char *) d;
	}
	std::vector<DevLevel> L; /* from the top */
	timer.begin();
	if (dev_pyramid(domain, top, top_bpl, in->Xsize, in->Ysize, bands, nl, L, sc))
		return -1;
	timer.end(0);

	std::map<std::pair<int, int>, std::vector<long>> shapes;
	for (long i = 0; i < (long) P->tiles.size(); i++)
		shapes[{P->tiles[i].w, P->tiles[i].h}].push_back(i);
	const size_t budget = g_budget.load() ? g_budget.load() : codec.png ? chunk_budget() : kDzBudget;
	std::vector<DzGatherTile> table;
	std::vector<size_t> lens;
	for (const auto &sh : shapes) {
		const int w = sh.first.first, h = sh.first.second;
		const std::vector<long> &idx = sh.second;
		const size_t frame_stride = ((size_t) w * h * bands + 15) & ~(size_t) 15;
		Encoder enc;
		if (tile_encoder(domain, codec, w, h, bands, &enc))
			return -1;
		const size_t per_tile = frame_stride + enc.scratch_bytes + enc.stream_bytes;
		if (per_tile > budget) {
			error(domain, "a %d x %d tile takes %zu bytes of device memory, more than the %zu allowed for a batch", w, h, per_tile, budget);
			return -1;
		}
		const size_t chunk = std::min<size_t>(std::min<size_t>(budget / per_tile, (size_t) kMaxBatchFrames), idx.size());
		void *d_table = nullptr, *d_pix = nullptr;
		if (sc.alloc(domain, &d_table, chunk * sizeof(DzGatherTile)) || sc.alloc(domain, &d_pix, chunk * frame_stride))
			return -1;
		for (size_t c0 = 0; c0 < idx.size(); c0 += chunk) {
			const int cn = (int) std::min(chunk, idx.size() - c0);
			table.resize(cn);
			for (int i = 0; i < cn; i++) {
				const DzTile &t = P->tiles[idx[c0 + i]];
				const DevLevel &l = L[nl - 1 - t.level];
				table[i] = {l.p + (size_t) t.top * l.bpl + (size_t) t.left * bands, l.bpl};
			}
			timer.begin();
			/* from pageable memory: staged by the driver before the call returns, so the table can be refilled */
			VB200_CUDA(domain, cudaMemcpyAsync(d_table, table.data(), cn * sizeof(DzGatherTile), cudaMemcpyHostToDevice, s));
			const int words = (w * h * bands + 3) / 4;
			dz_gather_kernel<<<dim3(std::min((words + kDzThreads - 1) / kDzThreads, 64), cn), kDzThreads, 0, s>>>((const DzGatherTile *) d_table,
				w * bands, h, (unsigned char *) d_pix, frame_stride);
			VB200_CUDA(domain, cudaGetLastError());
			count_launch();
			timer.end(1);
			timer.begin();
			EncodeDest dst;
			dst.bytes = &P->bytes;
			lens.assign(cn, 0);
			if (dev_encode_batch(domain, enc, d_pix, VB200_DEVICE, (size_t) w * bands, frame_stride, cn, (size_t) w * bands, h, dst, lens.data(), s)) {
				const DzTile &t = P->tiles[idx[c0]];
				error(domain, "encoding the %d x %d tiles failed; frame 0 there is level %d tile %d_%d, the rest follow in index order", w, h, t.level,
					t.x, t.y);
				return -1;
			}
			timer.end(2);
			timer.begin();
			for (int i = 0; i < cn; i++) {
				DzTile &t = P->tiles[idx[c0 + i]];
				t.off = dst.at[i];
				t.len = lens[i];
			}
			timer.end(3);
		}
		sc.release(d_table);
		sc.release(d_pix);
	}
	if (timer.on)
		memcpy(t_dz_ms, timer.ms, sizeof(t_dz_ms));
	return 0;
}

int
host_dzsave(const char *domain, const VB200Image *in, VB200DzPyramid *P, const DzCodec &codec)
{
	const int bands = in->Bands, nl = (int) P->levels.size();
	struct HostLevel {
		const unsigned char *p;
		size_t bpl;
	};
	std::vector<std::vector<unsigned char>> store(nl);
	std::vector<HostLevel> L; /* from the top */
	L.push_back({(const unsigned char *) in->data, in->bpl ? in->bpl : (size_t) in->Xsize * bands});
	for (int k = 1; k < nl; k++) {
		const DzLevel &above = P->levels[nl - k], &l = P->levels[nl - 1 - k];
		store[k].resize((size_t) l.w * l.h * bands);
		host_shrink_level(L[k - 1].p, L[k - 1].bpl, above.w, above.h, bands, store[k].data());
		L.push_back({store[k].data(), (size_t) l.w * bands});
	}
	std::vector<unsigned char> one;
	for (DzTile &t : P->tiles) {
		const HostLevel &l = L[nl - 1 - t.level];
		const unsigned char *p = l.p + (size_t) t.top * l.bpl + (size_t) t.left * bands;
		one.clear();
		if (host_tile_encode(domain, codec, p, l.bpl, t.w, t.h, bands, one)) {
			error(domain, "level %d tile %d_%d", t.level, t.x, t.y);
			return -1;
		}
		t.off = P->bytes.size();
		t.len = one.size();
		P->bytes.insert(P->bytes.end(), one.begin(), one.end());
	}
	return 0;
}

int
dzsave_entry(const char *domain, const VB200Image *in, const VB200DzOptions *options, bool png, const VB200PngSaveOptions *pngo,
	VB200DzPyramid **out, bool device)
{
	if (!out) {
		error(domain, "null argument");
		return -1;
	}
	*out = nullptr;
	VB200DzPyramid *P = new VB200DzPyramid;
	DzCodec codec;
	codec.png = png;
	int rc = dz_plan(domain, in, options, pngo, P, &codec);
	if (!rc && device)
		rc = ensure_init(domain) ? -1 : dev_dzsave(domain, in, P, codec, current_stream());
	else if (!rc) {
		if (in->where != VB200_HOST) {
			error(domain, "the host twin takes host memory");
			rc = -1;
		}
		else
			rc = host_dzsave(domain, in, P, codec);
	}
	if (rc) {
		delete P;
		return -1;
	}
	*out = P;
	return 0;
}

int
copy_text(const char *domain, const std::string &s, char *dst, size_t cap)
{
	if (!dst || cap < s.size() + 1) {
		error(domain, "buffer too small: %zu bytes needed", s.size() + 1);
		return -1;
	}
	memcpy(dst, s.c_str(), s.size() + 1);
	return 0;
}

/* the reference strips a ".dz" the caller left on the name (:2304-2310; ".zip" / ".szi" would pick a container) */
std::string
image_name(const char *basename)
{
	std::string n = basename && *basename ? basename : "untitled";
	const size_t dot = n.rfind('.');
	if (dot != std::string::npos && strcasecmp(n.c_str() + dot + 1, "dz") == 0)
		n.resize(dot);
	return n;
}

} // namespace

} // namespace vb200

using namespace vb200;

extern "C" int
vb200_dzsave(const VB200Image *in, const VB200DzOptions *options, VB200DzPyramid **out)
{
	return dzsave_entry("dzsave", in, options, false, nullptr, out, true);
}

extern "C" int
vb200_debug_dzsave(const VB200Image *in, const VB200DzOptions *options, VB200DzPyramid **out)
{
	return dzsave_entry("dzsave", in, options, false, nullptr, out, false);
}

extern "C" int
vb200_dzsave_png(const VB200Image *in, const VB200DzOptions *options, const VB200PngSaveOptions *png, VB200DzPyramid **out)
{
	return dzsave_entry("dzsave_png", in, options, true, png, out, true);
}

extern "C" int
vb200_debug_dzsave_png(const VB200Image *in, const VB200DzOptions *options, const VB200PngSaveOptions *png, VB200DzPyramid **out)
{
	return dzsave_entry("dzsave_png", in, options, true, png, out, false);
}

extern "C" void
vb200_dz_free(VB200DzPyramid *pyramid)
{
	delete pyramid;
}

extern "C" int
vb200_dz_levels(const VB200DzPyramid *pyramid)
{
	return pyramid ? (int) pyramid->levels.size() : 0;
}

extern "C" int
vb200_dz_level_geometry(const VB200DzPyramid *pyramid, int n, int *width, int *height, int *tiles_across, int *tiles_down)
{
	if (!pyramid || n < 0 || n >= (int) pyramid->levels.size()) {
		error("dzsave", "no level %d", n);
		return -1;
	}
	const DzLevel &l = pyramid->levels[n];
	if (width)
		*width = l.w;
	if (height)
		*height = l.h;
	if (tiles_across)
		*tiles_across = l.across;
	if (tiles_down)
		*tiles_down = l.down;
	return 0;
}

extern "C" long
vb200_dz_tiles(const VB200DzPyramid *pyramid)
{
	return pyramid ? (long) pyramid->tiles.size() : 0;
}

extern "C" int
vb200_dz_tile(const VB200DzPyramid *pyramid, long i, int *level, int *x, int *y, int *left, int *top, int *width, int *height, const void **stream,
	size_t *len)
{
	if (!pyramid || i < 0 || i >= (long) pyramid->tiles.size()) {
		error("dzsave", "no tile %ld", i);
		return -1;
	}
	const DzTile &t = pyramid->tiles[i];
	int *dst[7] = {level, x, y, left, top, width, height};
	const int val[7] = {t.level, t.x, t.y, t.left, t.top, t.w, t.h};
	for (int k = 0; k < 7; k++)
		if (dst[k])
			*dst[k] = val[k];
	if (stream)
		*stream = pyramid->bytes.data() + t.off;
	if (len)
		*len = t.len;
	return 0;
}

extern "C" int
vb200_dz_tile_name(const VB200DzPyramid *pyramid, long i, const char *basename, char *name, size_t cap)
{
	if (!pyramid || i < 0 || i >= (long) pyramid->tiles.size()) {
		error("dzsave", "no tile %ld", i);
		return -1;
	}
	const DzTile &t = pyramid->tiles[i];
	char buf[128];
	if (pyramid->layout == VB200_DZ_LAYOUT_DZ)
		snprintf(buf, sizeof(buf), "_files/%d/%d_%d", t.level, t.x, t.y);
	else {
		/* tile_name :1182-1193: the tiles of the smaller levels first, then this level's in reading order -- the index */
		snprintf(buf, sizeof(buf), "/TileGroup%ld/%d-%d-%d", i / 256, t.level, t.x, t.y);
	}
	return copy_text("dzsave", image_name(basename) + buf + pyramid->suffix, name, cap);
}

extern "C" int
vb200_dz_sidecar(const VB200DzPyramid *pyramid, const char *basename, char *name, size_t ncap, char *text, size_t tcap, size_t *len)
{
	if (!pyramid || pyramid->levels.empty()) {
		error("dzsave", "null argument");
		return -1;
	}
	const DzLevel &top = pyramid->levels.back();
	char buf[512];
	std::string file = image_name(basename);
	if (pyramid->layout == VB200_DZ_LAYOUT_DZ) {
		file += ".dzi";
		snprintf(buf, sizeof(buf),
			"<?xml version=\"1.0\" encoding=\"UTF-8\"?>\n"
			"<Image xmlns=\"http://schemas.microsoft.com/deepzoom/2008\"\n"
			"  Format=\"%s\"\n"
			"  Overlap=\"%d\"\n"
			"  TileSize=\"%d\"\n"
			"  >\n"
			"  <Size \n"
			"    Height=\"%d\"\n"
			"    Width=\"%d\"\n"
			"  />\n"
			"</Image>\n",
			pyramid->suffix.c_str() + 1, pyramid->overlap, pyramid->tile_size, top.h, top.w);
	}
	else {
		file += "/ImageProperties.xml";
		snprintf(buf, sizeof(buf), "<IMAGE_PROPERTIES WIDTH=\"%d\" HEIGHT=\"%d\" NUMTILES=\"%ld\" NUMIMAGES=\"1\" VERSION=\"1.8\" TILESIZE=\"%d\" />\n",
			top.w, top.h, (long) pyramid->tiles.size(), pyramid->tile_size);
	}
	if (len)
		*len = strlen(buf);
	if (copy_text("dzsave", file, name, ncap) || copy_text("dzsave", buf, text, tcap))
		return -1;
	return 0;
}

extern "C" int
vb200_dz_pyramid_level(const VB200Image *in, int n_from_top, VB200Image *out)
{
	const char *domain = "dz_pyramid_level";
	if (!in || !in->data || !out) {
		error(domain, "null argument");
		return -1;
	}
	if (in->BandFmt != VB200_FORMAT_UCHAR || in->Bands < 1 || in->Bands > 4 || in->Xsize < 1 || in->Ysize < 1) {
		error(domain, "uchar images of 1 to 4 bands only");
		return -1;
	}
	/* 2 and 4 bands are shrunk with alpha: that is what the reference does for B_W and sRGB (vips_image_hasalpha) */
	if ((in->Bands == 2 && in->Type != VB200_INTERPRETATION_B_W) || (in->Bands == 4 && in->Type != VB200_INTERPRETATION_sRGB)) {
		error(domain, "a %d-band image takes interpretation %s (its last band alpha)", in->Bands, in->Bands == 2 ? "B_W" : "sRGB");
		return -1;
	}
	int w = in->Xsize, h = in->Ysize;
	for (int k = 0; k < std::abs(n_from_top); k++) {
		if (n_from_top < 0 || (w == 1 && h == 1)) {
			error(domain, "a %d x %d image has no level %d", in->Xsize, in->Ysize, n_from_top);
			return -1;
		}
		w = (w + 1) / 2;
		h = (h + 1) / 2;
	}
	if (ensure_init(domain))
		return -1;
	cudaStream_t s = current_stream();
	DzScratch sc(s);
	DevImage din;
	if (to_device(domain, in, &din, s))
		return -1;
	if (din.owned)
		sc.held.push_back(din.data);
	std::vector<DevLevel> L;
	if (dev_pyramid(domain, (const unsigned char *) din.data, din.bpl, din.w, din.h, din.bands, n_from_top + 1, L, sc))
		return -1;
	DevImage d;
	d.w = L.back().w;
	d.h = L.back().h;
	d.bands = din.bands;
	d.fmt = din.fmt;
	d.type = din.type;
	d.data = L.back().p;
	d.bpl = L.back().bpl;
	d.owned = false; /* sc frees it, after the copy deliver() queues on the same stream */
	return deliver(domain, &d, in, out, s);
}

extern "C" int
vb200_debug_dz_pyramid_level(const void *pixels, size_t bpl, int width, int height, int bands, int n_from_top, void *out)
{
	const char *domain = "dz_pyramid_level (host twin)";
	if (!pixels || !out || width < 1 || height < 1 || bands < 1 || bands > 4 || n_from_top < 0) {
		error(domain, "bad argument");
		return -1;
	}
	std::vector<unsigned char> a, b;
	const unsigned char *p = (const unsigned char *) pixels;
	size_t pbpl = bpl ? bpl : (size_t) width * bands;
	int w = width, h = height;
	for (int k = 0; k < n_from_top; k++) {
		if (w == 1 && h == 1) {
			error(domain, "a %d x %d image has no level %d", width, height, n_from_top);
			return -1;
		}
		b.resize((size_t) ((w + 1) / 2) * ((h + 1) / 2) * bands);
		host_shrink_level(p, pbpl, w, h, bands, b.data());
		a.swap(b);
		w = (w + 1) / 2;
		h = (h + 1) / 2;
		p = a.data();
		pbpl = (size_t) w * bands;
	}
	for (int y = 0; y < h; y++)
		memcpy((unsigned char *) out + (size_t) y * w * bands, p + (size_t) y * pbpl, (size_t) w * bands);
	return 0;
}

extern "C" void
vb200_debug_dz_set_budget(size_t bytes)
{
	g_budget.store(bytes);
}

extern "C" size_t
vb200_debug_dz_pool_used(void)
{
	if (ensure_init("dz_pool_used"))
		return 0;
	int device = 0;
	cudaMemPool_t pool;
	uint64_t used = 0;
	if (cudaGetDevice(&device) != cudaSuccess || cudaDeviceGetDefaultMemPool(&pool, device) != cudaSuccess ||
		cudaDeviceSynchronize() != cudaSuccess || cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemCurrent, &used) != cudaSuccess)
		return 0;
	return (size_t) used;
}

extern "C" void
vb200_debug_dz_times(float *ms)
{
	if (ms)
		memcpy(ms, t_dz_ms, sizeof(t_dz_ms));
}
