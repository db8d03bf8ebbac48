/* png.cu -- SURVEY 8(f) rank 1, the PNG half: vips_pngload_buffer's 8-bit frames inflated and unfiltered on the device.
 *
 * What the reference does (foreign/spngload.c, libspng over zlib, fail_on = none): CRCs and the Adler-32 are not
 * checked (:346-352); palette images expand to RGB8, or RGBA8 with a tRNS chunk; 1 / 2 / 4-bit grey expands to G8 by
 * scaling; tRNS on grey or RGB adds an alpha band, 0 where the sample equals the key and 255 elsewhere
 * (SPNG_DECODE_TRNS, :592); the interpretation is B_W or sRGB by band count (:385-480); iCCP becomes the ICC profile
 * (:244-246) and eXIf the EXIF (:273-276).  Decoding is lossless and exactly specified (RFC 1950 / 1951, PNG 2nd
 * edition), so the pixels are bit-exact by definition.
 *
 * Scope: non-interlaced 8-bit grey, grey + alpha, RGB and RGBA; palette at 1 / 2 / 4 / 8 bits with or without tRNS;
 * grey at 1 / 2 / 4 bits without tRNS; tRNS on 8-bit grey and RGB.  Everything else returns -1 with its reason and the
 * host keeps its loader: 16-bit samples, Adam7, low-bit grey with tRNS, a missing PLTE or a palette index beyond it,
 * IDAT chunks that are not consecutive, a zlib header with a preset dictionary / another method / a bad FCHECK, a deflate
 * stream that zlib refuses, a stream that inflates to more or fewer scanline bytes than IHDR implies, frames over 2^28
 * pixels.
 *
 * Device pipeline per chunk of frames (the IDAT payloads, without chunk framing and zlib header, are all that crosses
 * PCIe):
 *   png_inflate_kernel    one warp per frame: lane 0 decodes symbols and writes literals, the warp copies every match
 *                         and stored block with 32 lanes; out: the frame's filtered scanlines
 *   png_unfilter_kernel   one CTA per frame, in place: each warp runs 32 rows as a diagonal wavefront (lane r one byte
 *                         behind lane r - 1, neighbours passed by shuffle), row bands chained warp to warp through
 *                         progress words in shared memory; palette indices are range-checked here
 *   png_expand_kernel     one thread per pixel, only once every frame of the chunk has decoded clean: palette lookup,
 *                         low-bit unpacking and scaling, tRNS alpha, written at the caller's stride
 * The per-symbol, per-byte and per-pixel code is __host__ __device__: vb200_debug_png_decode runs it on the CPU so that
 * the CPU test-suite pins it against Pillow and Python's zlib without a GPU.
 */
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <vector>

#include "../../include/vb200.h"
#include "png_common.cuh"
#include "vb200_internal.h"

#define VB_HD __host__ __device__ __forceinline__

#include "inflate.cuh"

namespace vb200 {

namespace {

enum { ERR_FEWER = 4, ERR_FILTER = 8, ERR_PALETTE = 16 };

/* ------------------------------------------------------------------ scanlines: unfilter and expand, host and device */

/* one frame as the kernels see it; offsets are into the chunk's pools */
struct PngFrameDev {
	unsigned long long data_off, data_len; /* the raw deflate bytes */
	unsigned long long scan_off;		   /* h rows of 1 + rb bytes */
	int w, h, rb, bpp;					   /* bpp: bytes per complete pixel, at least 1 (the filters' unit) */
	int depth, ct, bands, trns;
	int pal_off, pal_n; /* into the palette pool (256 RGBA entries each), -1: none */
	unsigned short key[3];
};

/* the reconstructed byte from the filtered one, a = left, b = up, c = up-left */
VB_HD unsigned char
unfilter_byte(int ft, int raw, int a, int b, int c)
{
	switch (ft) {
	case 1:
		return (unsigned char) (raw + a);
	case 2:
		return (unsigned char) (raw + b);
	case 3:
		return (unsigned char) (raw + ((a + b) >> 1));
	case 4:
		return (unsigned char) (raw + paeth(a, b, c));
	default:
		return (unsigned char) raw;
	}
}

/* whether byte x of a palette row holds an index beyond PLTE (padding bits after the last pixel are not indices) */
VB_HD bool
palette_bad(const PngFrameDev &F, int x, unsigned v)
{
	if (F.ct != 3)
		return false;
	const int spb = 8 / F.depth, mask = (1 << F.depth) - 1;
	for (int k = 0; k < spb; k++) {
		const int px = x * spb + k;
		if (px < F.w && (int) ((v >> (8 - F.depth * (k + 1))) & mask) >= F.pal_n)
			return true;
	}
	return false;
}

/* pixel x of an unfiltered row (its bytes after the filter byte) in spngload's layout */
VB_HD void
expand_pixel(const PngFrameDev &F, const unsigned char *row, const unsigned char *pal, int x, unsigned char *o)
{
	if (F.depth < 8) {
		const int bit = x * F.depth, mask = (1 << F.depth) - 1;
		const int v = (row[bit >> 3] >> (8 - F.depth - (bit & 7))) & mask;
		if (F.ct == 3) {
			const unsigned char *e = pal + 4 * v;
			o[0] = e[0], o[1] = e[1], o[2] = e[2];
			if (F.trns)
				o[3] = e[3];
		}
		else
			o[0] = (unsigned char) (v * (255 / mask));
		return;
	}
	const unsigned char *s = row + (size_t) x * F.bpp;
	switch (F.ct) {
	case 0:
		o[0] = s[0];
		if (F.trns)
			o[1] = s[0] == F.key[0] ? 0 : 255;
		break;
	case 2:
		o[0] = s[0], o[1] = s[1], o[2] = s[2];
		if (F.trns)
			o[3] = (s[0] == F.key[0] && s[1] == F.key[1] && s[2] == F.key[2]) ? 0 : 255;
		break;
	case 3: {
		const unsigned char *e = pal + 4 * s[0];
		o[0] = e[0], o[1] = e[1], o[2] = e[2];
		if (F.trns)
			o[3] = e[3];
		break;
	}
	case 4:
		o[0] = s[0], o[1] = s[1];
		break;
	default:
		o[0] = s[0], o[1] = s[1], o[2] = s[2], o[3] = s[3];
	}
}

/* ------------------------------------------------------------------ kernels */

constexpr int kInflateWarps = 4;

__global__ void __launch_bounds__(kInflateWarps * 32)
png_inflate_kernel(const PngFrameDev *__restrict__ frames, int n, const unsigned char *__restrict__ bytes, unsigned char *scan, int *status)
{
	__shared__ InflateTables tabs[kInflateWarps];
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	for (int f = blockIdx.x * kInflateWarps + warp; f < n; f += gridDim.x * kInflateWarps) {
		const PngFrameDev F = frames[f];
		const unsigned char *src = bytes + F.data_off;
		unsigned char *out = scan + F.scan_off;
		const unsigned long long want = (unsigned long long) F.h * (F.rb + 1);
		Inflate z;
		inflate_init(z, src, F.data_len, want, &tabs[warp]);
		const int op = inflate_warp(z, src, out, lane);
		if (lane == 0 && (op == OP_ERR || z.pos != want))
			status[f] = op == OP_ERR ? z.err : ERR_FEWER;
		__syncwarp();
	}
}

constexpr int kUnfilterWarps = 8;

/* One CTA per frame.  Band k (rows 32k .. 32k + 31) runs on warp k mod 8, lane r on row 32k + r at byte t - r of step t:
 * up and up-left come from lane r - 1's results of the last steps (shuffled up), left and up-left from the lane's own
 * history.  Lane 0 reads the row above from memory, after the warp of band k - 1 has published that it passed those
 * bytes (progress[warp] = band << 32 | bytes done of its last row).
 */
template <int BPP>
__global__ void __launch_bounds__(kUnfilterWarps * 32)
png_unfilter_kernel(const PngFrameDev *__restrict__ frames, int n, unsigned char *scan, int *status)
{
	__shared__ volatile long long progress[kUnfilterWarps];
	__shared__ int skip;
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	for (int f = blockIdx.x; f < n; f += gridDim.x) {
		const PngFrameDev F = frames[f];
		if (F.bpp != BPP) /* another launch's unit */
			continue;
		if (threadIdx.x < kUnfilterWarps)
			progress[threadIdx.x] = -1;
		if (threadIdx.x == 0)
			skip = status[f]; /* read once: a warp that finishes early ORs its verdict in */
		__syncthreads();
		if (skip == 0) {
			unsigned char *img = scan + F.scan_off;
			const size_t stride = (size_t) F.rb + 1;
			const int bands = (F.h + 31) / 32;
			int bad = 0;
			for (int band = warp; band < bands; band += kUnfilterWarps) {
				const int y = band * 32 + lane;
				const bool active = y < F.h;
				unsigned char *row = img + (size_t) y * stride;
				const unsigned char *up = img + ((size_t) y - 1) * stride; /* lane 0's row above */
				int ft = active ? row[0] : 0;
				if (ft > 4) {
					bad |= ERR_FILTER;
					ft = 0;
				}
				int ah[BPP], ch[BPP]; /* own results and the row above's, the last BPP bytes (newest first) */
				for (int k = 0; k < BPP; k++)
					ah[k] = ch[k] = 0;
				int mine = 0;
				const volatile long long &pred = progress[(warp + kUnfilterWarps - 1) % kUnfilterWarps];
				for (int t = 0; t < F.rb + 31; t++) {
					if (band > 0 && (t & 31) == 0 && t < F.rb) {
						const long long need = ((long long) (band - 1) << 32) | (long long) min(t + 32, F.rb);
						while (pred < need)
							;
						__threadfence_block();
					}
					const int x = t - lane;
					int b = __shfl_up_sync(0xffffffffu, mine, 1);
					if (lane == 0)
						b = (y > 0 && x >= 0 && x < F.rb) ? up[1 + x] : 0;
					const int c = ch[BPP - 1], a = ah[BPP - 1];
					for (int k = BPP - 1; k > 0; k--)
						ch[k] = ch[k - 1];
					ch[0] = x >= 0 ? b : 0;
					if (active && x >= 0 && x < F.rb) {
						mine = unfilter_byte(ft, row[1 + x], a, b, c);
						row[1 + x] = (unsigned char) mine;
						if (palette_bad(F, x, (unsigned) mine))
							bad |= ERR_PALETTE;
						if (lane == 31 && (((x + 1) & 31) == 0 || x + 1 == F.rb)) {
							__threadfence_block();
							progress[warp] = ((long long) band << 32) | (long long) (x + 1);
						}
					}
					else
						mine = 0;
					for (int k = BPP - 1; k > 0; k--)
						ah[k] = ah[k - 1];
					ah[0] = mine;
				}
				__syncwarp();
			}
			if (bad)
				atomicOr(status + f, bad);
		}
		__syncthreads();
	}
}

__global__ void __launch_bounds__(256)
png_expand_kernel(const PngFrameDev *__restrict__ frames, const unsigned char *__restrict__ scan, const unsigned char *__restrict__ pals,
	unsigned char *out, size_t out_bpl, size_t out_frame_stride)
{
	const PngFrameDev &F = frames[blockIdx.z];
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= F.w)
		return;
	const unsigned char *pal = F.pal_off >= 0 ? pals + (size_t) F.pal_off * 1024 : nullptr;
	unsigned char *o = out + (size_t) blockIdx.z * out_frame_stride + (size_t) x * F.bands;
	for (int y = blockIdx.y; y < F.h; y += gridDim.y)
		expand_pixel(F, scan + F.scan_off + (size_t) y * (F.rb + 1) + 1, pal, x, o + (size_t) y * out_bpl);
}

/* ------------------------------------------------------------------ host: the chunk walk */

const unsigned char kSignature[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};

unsigned
be32(const unsigned char *p)
{
	return ((unsigned) p[0] << 24) | ((unsigned) p[1] << 16) | ((unsigned) p[2] << 8) | p[3];
}

struct PngHeader {
	int w = 0, h = 0, depth = 0, ct = 0, bands = 0;
	int pal_n = 0;
	unsigned char pal[256][4];
	bool trns = false, exif = false;
	unsigned short key[3] = {0, 0, 0};
	std::vector<std::pair<const unsigned char *, size_t>> idat;
	size_t idat_bytes = 0;
	const unsigned char *iccp = nullptr;
	size_t iccp_len = 0;
	int rb = 0, bpp = 0;
};

/* Walk the chunks (CRCs not read) and check what the decoder relies on.  -1 with the reason as the error. */
int
parse_png(const char *domain, const unsigned char *d, size_t len, PngHeader *H)
{
	if (!d || len < 8 || memcmp(d, kSignature, 8) != 0) {
		error(domain, "not a PNG stream");
		return -1;
	}
	size_t p = 8;
	bool have_plte = false, idat_done = false, first = true;
	for (;;) {
		if (len - p < 8) {
			error(domain, "PNG stream ends before its IEND chunk");
			return -1;
		}
		const size_t n = be32(d + p);
		const unsigned char *type = d + p + 4, *c = d + p + 8;
		if (n > 0x7fffffffu || len - p - 8 < n + 4) {
			error(domain, "PNG chunk %.4s runs past the end of the stream", (const char *) type);
			return -1;
		}
		const bool is_idat = memcmp(type, "IDAT", 4) == 0;
		if (first != (memcmp(type, "IHDR", 4) == 0)) {
			error(domain, first ? "PNG stream does not begin with IHDR" : "PNG stream has a second IHDR");
			return -1;
		}
		if (!is_idat && !H->idat.empty())
			idat_done = true;
		if (first) {
			first = false;
			if (n != 13) {
				error(domain, "bad IHDR length");
				return -1;
			}
			const unsigned w = be32(c), h = be32(c + 4);
			const int depth = c[8], ct = c[9];
			if (w < 1 || h < 1 || w > 0x7fffffffu || h > 0x7fffffffu) {
				error(domain, "bad PNG dimensions %u x %u", w, h);
				return -1;
			}
			const bool ok = (ct == 0 && (depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16)) ||
							(ct == 3 && (depth == 1 || depth == 2 || depth == 4 || depth == 8)) ||
							((ct == 2 || ct == 4 || ct == 6) && (depth == 8 || depth == 16));
			if (!ok || c[10] != 0 || c[11] != 0 || c[12] > 1) {
				error(domain, "bad IHDR (colour type %d, bit depth %d, methods %d %d %d)", ct, depth, c[10], c[11], c[12]);
				return -1;
			}
			if (depth == 16) {
				error(domain, "16-bit PNG not supported");
				return -1;
			}
			if (c[12] == 1) {
				error(domain, "Adam7-interlaced PNG not supported");
				return -1;
			}
			if ((unsigned long long) w * h > (1ull << 28)) {
				error(domain, "%u x %u: frames over 2^28 pixels are not supported", w, h);
				return -1;
			}
			H->w = (int) w;
			H->h = (int) h;
			H->depth = depth;
			H->ct = ct;
			const int spp = ct == 2 ? 3 : ct == 4 ? 2 : ct == 6 ? 4 : 1;
			H->bpp = spp;
			H->rb = (int) (((unsigned long long) w * spp * depth + 7) / 8);
		}
		else if (memcmp(type, "PLTE", 4) == 0) {
			if (have_plte || !H->idat.empty() || H->ct == 0 || H->ct == 4 || n == 0 || n % 3 || n > 768) {
				error(domain, "bad PLTE chunk");
				return -1;
			}
			have_plte = true;
			H->pal_n = (int) n / 3;
			for (int i = 0; i < 256; i++) {
				for (int k = 0; k < 3; k++)
					H->pal[i][k] = i < H->pal_n ? c[3 * i + k] : 0;
				H->pal[i][3] = 255;
			}
		}
		else if (memcmp(type, "tRNS", 4) == 0) {
			const bool ok = !H->trns && H->idat.empty() &&
							((H->ct == 0 && n == 2) || (H->ct == 2 && n == 6) || (H->ct == 3 && have_plte && (int) n <= H->pal_n));
			if (!ok) {
				error(domain, "bad tRNS chunk");
				return -1;
			}
			if (H->ct == 0 && H->depth < 8) {
				error(domain, "low-bit grey with tRNS not supported");
				return -1;
			}
			H->trns = true;
			if (H->ct == 3)
				for (size_t i = 0; i < n; i++)
					H->pal[i][3] = c[i];
			else
				for (size_t i = 0; i < n / 2; i++)
					H->key[i] = (unsigned short) ((c[2 * i] << 8) | c[2 * i + 1]);
		}
		else if (memcmp(type, "iCCP", 4) == 0) {
			if (H->iccp || !H->idat.empty()) {
				error(domain, "bad iCCP chunk");
				return -1;
			}
			H->iccp = c;
			H->iccp_len = n;
		}
		else if (memcmp(type, "eXIf", 4) == 0)
			H->exif = true;
		else if (is_idat) {
			if (idat_done) {
				error(domain, "IDAT chunks are not consecutive");
				return -1;
			}
			H->idat.emplace_back(c, n);
			H->idat_bytes += n;
		}
		else if (memcmp(type, "IEND", 4) == 0)
			break;
		else if (!(type[0] & 0x20)) {
			error(domain, "unknown critical PNG chunk %.4s", (const char *) type);
			return -1;
		}
		p += 12 + n;
	}
	if (H->idat.empty()) {
		error(domain, "PNG stream has no IDAT chunk");
		return -1;
	}
	if (H->ct == 3 && !have_plte) {
		error(domain, "palette image without PLTE");
		return -1;
	}
	H->bands = H->ct == 0 ? 1 + H->trns : H->ct == 4 ? 2 : H->ct == 6 ? 4 : 3 + H->trns;
	/* RFC 1950 2.2: the zlib header, which may straddle IDAT chunks */
	unsigned char zh[2];
	size_t got = 0;
	for (size_t i = 0; i < H->idat.size() && got < 2; i++)
		for (size_t k = 0; k < H->idat[i].second && got < 2; k++)
			zh[got++] = H->idat[i].first[k];
	if (got < 2) {
		error(domain, "IDAT data too short for a zlib header");
		return -1;
	}
	if ((zh[0] & 15) != 8 || (zh[0] >> 4) > 7) {
		error(domain, "zlib header: method %d, window 2^%d: not deflate", zh[0] & 15, (zh[0] >> 4) + 8);
		return -1;
	}
	if ((zh[0] * 256 + zh[1]) % 31) {
		error(domain, "zlib header: bad FCHECK");
		return -1;
	}
	if (zh[1] & 0x20) {
		error(domain, "zlib header: preset dictionary not supported");
		return -1;
	}
	return 0;
}

/* the raw deflate bytes: the IDAT payloads after the 2-byte zlib header, concatenated */
void
stage_idat(const PngHeader &H, unsigned char *dst)
{
	size_t skip = 2;
	for (const auto &c : H.idat) {
		const size_t k = std::min(skip, c.second);
		skip -= k;
		memcpy(dst, c.first + k, c.second - k);
		dst += c.second - k;
	}
}

size_t
deflate_bytes(const PngHeader &H)
{
	return H.idat_bytes - 2;
}

size_t
scan_bytes(const PngHeader &H)
{
	return (size_t) H.h * ((size_t) H.rb + 1);
}

PngFrameDev
frame_record(const PngHeader &H)
{
	PngFrameDev F;
	memset(&F, 0, sizeof(F));
	F.data_len = deflate_bytes(H);
	F.w = H.w;
	F.h = H.h;
	F.rb = H.rb;
	F.bpp = H.depth < 8 ? 1 : H.bpp;
	F.depth = H.depth;
	F.ct = H.ct;
	F.bands = H.bands;
	F.trns = H.trns;
	F.pal_off = -1;
	F.pal_n = H.pal_n;
	for (int k = 0; k < 3; k++)
		F.key[k] = H.key[k];
	return F;
}

const char *
status_text(int st)
{
	if (st & ERR_CORRUPT)
		return "corrupt deflate stream (zlib refuses it)";
	if (st & ERR_MORE)
		return "the stream inflates to more scanline bytes than IHDR implies";
	if (st & ERR_FEWER)
		return "the stream inflates to fewer scanline bytes than IHDR implies";
	if (st & ERR_FILTER)
		return "bad PNG filter type";
	return "palette index beyond PLTE";
}

/* device bytes a frame takes in a chunk: its staged deflate bytes and its scanlines */
size_t
frame_device_bytes(const PngHeader &H)
{
	return align16(deflate_bytes(H)) + align16(scan_bytes(H));
}

} // namespace

bool
png_signature(const void *buf, size_t len)
{
	return buf && len >= 8 && memcmp(buf, kSignature, 8) == 0;
}

/* the iCCP profile, inflated by the host twin's inflate (profile empty: none); exif: whether the stream has eXIf */
int
png_icc_profile(const char *domain, const unsigned char *d, size_t len, std::vector<unsigned char> *profile, bool *exif)
{
	profile->clear();
	PngHeader H;
	if (parse_png(domain, d, len, &H))
		return -1;
	if (exif)
		*exif = H.exif;
	if (!H.iccp)
		return 0;
	/* name (1-79 bytes), NUL, compression method 0, zlib stream */
	const unsigned char *z = (const unsigned char *) memchr(H.iccp, 0, std::min<size_t>(H.iccp_len, 80));
	if (!z || z == H.iccp || (size_t) (z - H.iccp) + 4 > H.iccp_len || z[1] != 0 || (z[2] & 15) != 8 || (z[2] >> 4) > 7 ||
		(z[2] * 256 + z[3]) % 31 || (z[3] & 0x20)) {
		error(domain, "bad iCCP chunk");
		return -1;
	}
	const unsigned char *src = z + 4;
	const size_t n = H.iccp_len - (size_t) (z + 4 - H.iccp);
	for (size_t cap = 1 << 16;; cap *= 2) {
		profile->resize(cap);
		size_t got = 0;
		int err = 0;
		if (inflate_host(src, n, profile->data(), cap, &got, &err) == 0) {
			profile->resize(got);
			return 0;
		}
		if (err != ERR_MORE || cap >= ((size_t) 1 << 28)) {
			profile->clear();
			error(domain, "iCCP chunk: corrupt deflate stream");
			return -1;
		}
	}
}

/* Decode n PNG streams (host memory) of one output geometry into out[n][h][w][bands] on the device (out = nullptr: only
 * report the geometry).  Headers are walked on the host workers; the frames go up in chunks bounded by device memory,
 * each one pinned block (frame records, palettes, raw deflate bytes) copied to the device and decoded on s.  Every
 * frame of a chunk must decode clean before its pixels are expanded into out; the call returns when they are.
 */
int
dev_png_decode_batch(const char *domain, const void *const *bufs, const size_t *lens, int n, void *out, size_t out_bpl, size_t out_frame_stride,
	StreamGeometry *g, cudaStream_t s)
{
	std::vector<PngHeader> hdr(n);
	if (parse_streams(
			domain, "frame", n, [&](int i) { return parse_png(domain, (const unsigned char *) bufs[i], lens[i], &hdr[i]); },
			[&](int i) { return StreamGeometry{hdr[i].w, hdr[i].h, hdr[i].bands, 0}; }, g))
		return -1;
	if (!out)
		return 0;
	if (check_out_strides(domain, *g, out_bpl, out_frame_stride))
		return -1;
	const int W = g->w, Hh = g->h;
	return decode_chunks(domain, "png", "frame", n, [&](int i) { return frame_device_bytes(hdr[i]); }, [&](int c0, int cn) {
		/* the block: records, palettes, deflate bytes staged; the scanlines as scratch */
		std::vector<PngFrameDev> F(cn);
		size_t n_pal = 0, data = 0, scan = 0;
		for (int i = 0; i < cn; i++) {
			const PngHeader &H = hdr[c0 + i];
			F[i] = frame_record(H);
			if (H.ct == 3)
				F[i].pal_off = (int) n_pal++;
			F[i].data_off = data;
			data += align16(deflate_bytes(H));
			F[i].scan_off = scan;
			scan += align16(scan_bytes(H));
		}
		const size_t off_pal = align16(cn * sizeof(PngFrameDev)), off_data = off_pal + n_pal * 1024, total = off_data + data;
		return decode_chunk(
			domain, "png", {total, scan, cn},
			[&](unsigned char *hst) {
				memcpy(hst, F.data(), cn * sizeof(PngFrameDev));
				parallel_for(cn, host_workers(), [&](int i) {
					const PngHeader &H = hdr[c0 + i];
					if (F[i].pal_off >= 0)
						memcpy(hst + off_pal + (size_t) F[i].pal_off * 1024, H.pal, 1024);
					stage_idat(H, hst + off_data + F[i].data_off);
				});
			},
			[&](unsigned char *dev, int *status) {
				const PngFrameDev *dF = (const PngFrameDev *) dev;
				png_inflate_kernel<<<(cn + kInflateWarps - 1) / kInflateWarps, kInflateWarps * 32, 0, s>>>(dF, cn, dev + off_data, dev + align16(total),
					status);
				int launches = 1;
				/* frames of one geometry may still differ in their filter unit (a palette frame's is 1 byte, an RGB frame's 3):
				 * one launch per unit present, each skipping the others' frames
				 */
				bool unit[5] = {false, false, false, false, false};
				for (const PngFrameDev &f : F)
					unit[f.bpp] = true;
				void (*const unfilter[5])(const PngFrameDev *, int, unsigned char *, int *) = {nullptr, png_unfilter_kernel<1>, png_unfilter_kernel<2>,
					png_unfilter_kernel<3>, png_unfilter_kernel<4>};
				for (int u = 1; u <= 4; u++)
					if (unit[u]) {
						unfilter[u]<<<cn, kUnfilterWarps * 32, 0, s>>>(dF, cn, dev + align16(total), status);
						launches++;
					}
				return launches;
			},
			[&](int i, int st) { error(domain, "frame %d: %s", c0 + i, status_text(st)); },
			[&](unsigned char *dev) {
				png_expand_kernel<<<dim3((W + 255) / 256, std::min(Hh, kMaxGridY), cn), 256, 0, s>>>((const PngFrameDev *) dev, dev + align16(total),
					dev + off_pal, (unsigned char *) out + (size_t) c0 * out_frame_stride, out_bpl, out_frame_stride);
				return 1;
			},
			s);
	}, s);
}

/* the same decode on the CPU through the same per-symbol, per-byte and per-pixel code: the test-suite's host twin */
int
host_png_decode(const char *domain, const void *buf, size_t len, unsigned char *out, size_t out_bpl, int *out_w, int *out_h, int *out_bands)
{
	PngHeader H;
	if (parse_png(domain, (const unsigned char *) buf, len, &H))
		return -1;
	if (out_w)
		*out_w = H.w;
	if (out_h)
		*out_h = H.h;
	if (out_bands)
		*out_bands = H.bands;
	if (!out)
		return 0;
	const PngFrameDev F = frame_record(H);
	std::vector<unsigned char> data(deflate_bytes(H)), scan(scan_bytes(H));
	stage_idat(H, data.data());
	size_t got = 0;
	int err = 0;
	if (inflate_host(data.data(), data.size(), scan.data(), scan.size(), &got, &err) || got != scan.size()) {
		error(domain, "%s", status_text(err ? err : ERR_FEWER));
		return -1;
	}
	const size_t stride = (size_t) F.rb + 1;
	for (int y = 0; y < F.h; y++) {
		unsigned char *row = scan.data() + (size_t) y * stride;
		const unsigned char *up = y > 0 ? row - stride : nullptr;
		if (row[0] > 4) {
			error(domain, "%s", status_text(ERR_FILTER));
			return -1;
		}
		for (int x = 0; x < F.rb; x++) {
			const int a = x >= F.bpp ? row[1 + x - F.bpp] : 0, b = up ? up[1 + x] : 0, c = up && x >= F.bpp ? up[1 + x - F.bpp] : 0;
			row[1 + x] = unfilter_byte(row[0], row[1 + x], a, b, c);
			if (palette_bad(F, x, row[1 + x])) {
				error(domain, "%s", status_text(ERR_PALETTE));
				return -1;
			}
		}
	}
	for (int y = 0; y < F.h; y++)
		for (int x = 0; x < F.w; x++)
			expand_pixel(F, scan.data() + (size_t) y * stride + 1, &H.pal[0][0], x, out + (size_t) y * out_bpl + (size_t) x * F.bands);
	return 0;
}

} // namespace vb200

/* ------------------------------------------------------------------ C ABI */

using namespace vb200;

extern "C" int
vb200_png_decode_batch(const void *const *bufs, const size_t *lens, int n, void *out, int out_location, size_t out_bpl, size_t out_frame_stride,
	int *width, int *height, int *bands)
{
	return decode_batch_abi("png_decode_batch", {STREAM_PNG}, bufs, lens, n, out, out_location, out_bpl, out_frame_stride, width, height, bands);
}

/* reference: vips_pngload_buffer(buf, len, &out, NULL), foreign/spngload.c */
extern "C" int
vb200_pngload_buffer(const void *buf, size_t len, VB200Image *out)
{
	return load_abi("pngload_buffer", {STREAM_PNG}, buf, len, out);
}

extern "C" int
vb200_png_icc_profile(const void *buf, size_t len, void *out, size_t cap, size_t *profile_len)
{
	return profile_abi("png_icc_profile", out, cap, profile_len,
		[&](const char *domain, std::vector<unsigned char> *prof) { return png_icc_profile(domain, (const unsigned char *) buf, len, prof, nullptr); });
}

extern "C" int
vb200_debug_png_decode(const void *buf, size_t len, void *out, size_t out_bpl, int *width, int *height, int *bands)
{
	return host_twin_abi("png_decode (host twin)",
		[&](const char *domain) { return host_png_decode(domain, buf, len, (unsigned char *) out, out_bpl, width, height, bands); });
}

/* raw deflate data (no zlib header) through the host twin's inflate: 0 and *out_len bytes, or -1 (refused, or more than
 * cap bytes: *out_len = cap + 1) */
extern "C" int
vb200_debug_inflate(const void *buf, size_t len, void *out, size_t cap, size_t *out_len)
{
	size_t got = 0;
	int err = 0;
	const int rc = inflate_host((const unsigned char *) buf, len, (unsigned char *) out, cap, &got, &err);
	if (out_len)
		*out_len = rc == 0 ? got : err == ERR_MORE ? cap + 1 : got;
	if (rc)
		error("inflate (host twin)", "%s", err == ERR_MORE ? "more output than the buffer holds" : "corrupt deflate stream");
	return rc;
}
