/* gif.cu -- the GIF half of SURVEY 8(f) rank 1: vips_gifload_buffer's frames decoded on the device, pixel for pixel
 * what libnsgif gives nsgifload.
 *
 * What the reference does (foreign/nsgifload.c over its vendored libnsgif, foreign/libnsgif/gif.c and lzw.c):
 * nsgif_data_scan walks the whole stream (:357-460); the image is width x height * n uchar sRGB pixels with 4 bands if any
 * frame has transparency and 3 otherwise (:262-280); every output line copies the RGBA bitmap nsgif_frame_decode(page)
 * left, dropping the fourth byte without alpha (:480-540).  Page k of an animation is the screen after frames 0 .. k have
 * been composed by libnsgif's rules, restated here with their lines in gif.c:
 *   - the logical screen: 640x480 and the other "broken" sizes, 0 and anything over 2048 become 1 x 1 (:1656-1671); the
 *     first frame may grow the screen (:1046-1054); the bitmap is at most 65 535 on a side (nsgifload.c:642-650)
 *   - the global table, or black and white without one; entries past a table are 0 (transparent black) and a local table
 *     only overwrites its own entries of the one local table libnsgif keeps (:1071-1190, :1693-1738)
 *   - before frame 0 the screen is cleared to transparent (:704-706); then the previous frame's disposal: background sets
 *     its rect, clipped to the screen, to transparent if that frame has transparency and to the background colour
 *     otherwise (:639-684); previous restores the screen recorded before that frame was drawn (:294-342, :713-724)
 *   - a frame draws through its table, leaving its transparent index alone, clipped to the screen; interlaced rows come
 *     in the four-pass order of its clipped height (:357-394); a full-width frame at x = 0 that is not interlaced takes
 *     the "simple" path, every other one the "complex" path (:597-630)
 *   - LZW (lzw.c): LSB-first codes of 3-12 bits, clear and EOI codes, a full table of 4096 entries stops growing, the
 *     KwKwK case; a code past the table or a first code past the clear code fails the frame (LZW_BAD_CODE / _BAD_ICODE).
 *     Data that ends, or an EOI, before the rect is full leaves the rest of the rect as it was (:489-594).  A code ends
 *     the data when its last bit is the last bit of the frame's sub-blocks (lzw.c:163-220 needs the byte after it).
 *     The complex path takes a failing code quietly when it falls at a multiple of 4096 values: lzw_decode fills its
 *     4096-value stack and an empty fill ends the frame without looking at the error (:501-506).
 * Declined (-1 with the reason; the host keeps nsgifload): a scan that does not return NSGIF_OK, a truncated last frame
 * that nsgif_data_complete would promote, no frames, screens over 65 535 on a side ("bad image dimensions") or 2^28
 * pixels, a page / n out of range ("bad page number").  A frame libnsgif fails on fails the batch.
 *
 * Device pipeline per chunk of streams (the LZW payloads without their sub-block length bytes, one 256-entry RGBA table
 * per frame and the frame records are all that crosses PCIe):
 *   gif_lzw_kernel      one warp per frame: lane 0 reads the codes and keeps every table entry as the (position, length)
 *                       of a string already written; a string goes out as a copy from earlier output, by lane 0 when it
 *                       is short and by the 32 lanes otherwise (the self-overlapping KwKwK copy repeats its period, as
 *                       png_inflate_kernel's matches do); out: the frame's index plane in stored row order and the
 *                       number of indices decoded; a bad code sets the frame's status word
 *   gif_compose_kernel  one thread per screen pixel per stream, only once every frame of the chunk decoded clean: walks
 *                       frames 0 .. page + n - 1 applying disposal and drawing, and writes each requested page
 * The per-code and per-pixel code is __host__ __device__: vb200_debug_gif_decode / vb200_debug_lzw run it on the CPU so
 * the CPU test-suite pins it to libnsgif itself.
 */
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <vector>

#include "../../include/vb200.h"
#include "vb200_internal.h"

#define VB_HD __host__ __device__ __forceinline__

namespace vb200 {

namespace {

/* ------------------------------------------------------------------ LZW (lzw.c), host and device */

constexpr int kCodeMax = 12; /* LZW_CODE_MAX */
constexpr int kTable = 1 << kCodeMax;
constexpr int kPad = 4; /* zero bytes after each staged payload: the code reader loads 3 bytes */
constexpr unsigned long long kMaxValues = 1ull << 28; /* index values one frame may need */

enum { OP_COPY = 0, OP_DONE = 1 };
enum { ERR_CODE = 1 };

struct Lzw {
	const unsigned char *src;
	unsigned long long nbits, bit;
	unsigned at, want; /* values produced so far (full strings), values the frame needs */
	int clear, eoi, initial, code_size, code_max, table_size;
	unsigned prev_at, prev_len; /* where the last code's string went, its full length */
	int lenient, started, err;
	unsigned *tpos;
	unsigned short *tlen;
};

VB_HD void
lzw_init(Lzw &z, const unsigned char *src, unsigned len, unsigned want, int min_code, int lenient, unsigned *tpos, unsigned short *tlen)
{
	z.src = src;
	z.nbits = 8ull * len;
	z.bit = 0;
	z.at = 0;
	z.want = want;
	z.clear = 1 << min_code;
	z.eoi = z.clear + 1;
	z.initial = min_code + 1;
	z.code_size = z.initial;
	z.code_max = (1 << z.initial) - 1;
	z.table_size = z.eoi + 1;
	z.prev_at = z.prev_len = 0;
	z.lenient = lenient;
	z.started = 0;
	z.err = 0;
	z.tpos = tpos;
	z.tlen = tlen;
}

/* lzw__read_code: a code is there only if the byte after its last bit is (the slow path reads byte_advance + 1 bytes) */
VB_HD bool
lzw_read(Lzw &z, int *code)
{
	if (z.bit + (unsigned) z.code_size >= z.nbits)
		return false;
	const unsigned long long b = z.bit >> 3;
	const unsigned v = (unsigned) z.src[b] | ((unsigned) z.src[b + 1] << 8) | ((unsigned) z.src[b + 2] << 16);
	*code = (int) ((v >> (z.bit & 7)) & ((1u << z.code_size) - 1));
	z.bit += (unsigned) z.code_size;
	return true;
}

/* lzw__handle_clear: 0 with the first code after the clear codes, 1 the data ended, 2 LZW_BAD_ICODE */
VB_HD int
lzw_clear(Lzw &z, int *code)
{
	z.code_size = z.initial;
	z.code_max = (1 << z.initial) - 1;
	z.table_size = z.eoi + 1;
	do {
		if (!lzw_read(z, code))
			return 1;
	} while (*code == z.clear);
	return *code > z.clear ? 2 : 0;
}

/* a bad code after `at` values: the complex path's empty 4096-value fill ends the frame quietly, else the frame fails */
VB_HD int
lzw_bad(Lzw &z)
{
	if (!(z.lenient && z.at % 4096u == 0))
		z.err = ERR_CODE;
	return OP_DONE;
}

/* Decode until the next string that is a copy of earlier output (OP_COPY: *len bytes to *at from *src, clipped to the
 * frame's need) or the end (OP_DONE, z.err set if the frame fails).  Root codes are written here.
 */
VB_HD int
lzw_step(Lzw &z, unsigned char *out, unsigned *at, unsigned *src, unsigned *len)
{
	for (;;) {
		if (z.at >= z.want)
			return OP_DONE;
		int code;
		if (!z.started) {
			/* lzw_decode_init: a failure here is not subject to the 4096 rule */
			z.started = 1;
			const int r = lzw_clear(z, &code);
			if (r == 2)
				z.err = ERR_CODE;
			if (r)
				return OP_DONE;
		}
		else {
			if (!lzw_read(z, &code) || code == z.eoi)
				return OP_DONE;
			if (code > z.table_size)
				return lzw_bad(z);
			if (code == z.clear) {
				const int r = lzw_clear(z, &code);
				if (r == 1)
					return OP_DONE;
				if (r == 2)
					return lzw_bad(z);
			}
			else if (z.table_size < kTable) {
				/* the previous string plus the first value of this one: the output from prev_at on */
				const int size = z.table_size;
				z.tpos[size] = z.prev_at;
				z.tlen[size] = (unsigned short) (z.prev_len + 1);
				if (size == z.code_max && z.code_size < kCodeMax) {
					z.code_size++;
					z.code_max = (1 << z.code_size) - 1;
				}
				z.table_size++;
			}
		}
		const unsigned a = z.at;
		z.prev_at = a;
		if (code < z.clear) {
			out[a] = (unsigned char) code; /* table[i].value = i, a uint8_t */
			z.prev_len = 1;
			z.at = a + 1;
			continue;
		}
		const unsigned n = z.tlen[code];
		z.prev_len = n;
		z.at = a + n;
		*at = a;
		*src = z.tpos[code];
		*len = min(n, z.want - a);
		return OP_COPY;
	}
}

/* the whole frame on one thread: the host twin's LZW.  Returns the values decoded (at most want); *err as z.err */
unsigned
lzw_host(const unsigned char *src, unsigned len, unsigned want, int min_code, int lenient, unsigned char *out, int *err)
{
	std::vector<unsigned> tpos(kTable);
	std::vector<unsigned short> tlen(kTable);
	Lzw z;
	lzw_init(z, src, len, want, min_code, lenient, tpos.data(), tlen.data());
	unsigned at = 0, from = 0, n = 0;
	while (lzw_step(z, out, &at, &from, &n) == OP_COPY)
		for (unsigned i = 0; i < n; i++)
			out[at + i] = out[from + i];
	*err = z.err;
	return min(z.at, want);
}

/* ------------------------------------------------------------------ composition, host and device */

/* one frame as the kernels see it; offsets are into the chunk's pools */
struct GifFrameDev {
	unsigned long long data_off, idx_off;
	unsigned data_len, want; /* LZW payload bytes; index values the frame needs (0: it draws nothing) */
	int min_code, lenient;	 /* lenient: the complex path */
	int x0, y0, w;			 /* rect origin and stored row length */
	int wc, hc;				 /* drawn columns and rows, clipped to the screen */
	int bx1, by1;			 /* end of the rect the background disposal sets, clipped (bx1 <= x0: none) */
	int interlaced, trans, transparency, disposal, pal;
};

/* a stream: frames f0 .. f0 + nf - 1 of the chunk's records, pages page .. nf - 1 written */
struct GifStreamDev {
	int f0, nf, page;
	unsigned bg; /* info.background, RGBA bytes */
};

/* the stored row of image row y of an interlaced frame of h rows (nsgif__deinterlace's four passes, inverted) */
VB_HD int
interlace_row(int y, int h)
{
	const int n1 = (h + 7) / 8, n2 = (h + 3) / 8, n3 = (h + 1) / 4;
	if (y % 8 == 0)
		return y / 8;
	if (y % 8 == 4)
		return n1 + y / 8;
	if (y % 4 == 2)
		return n1 + n2 + y / 4;
	return n1 + n2 + n3 + y / 2;
}

/* Pixel (x, y) through frame F: the previous frame P's disposal (nsgif__update_bitmap :704-719), the record of a frame
 * whose own disposal is "previous" (:721-724), then F's index at that pixel if it was decoded and is not transparent.
 * cur / saved: the pixel's screen and recorded values, RGBA bytes.
 */
VB_HD void
gif_pixel(const GifFrameDev &F, const GifFrameDev *P, unsigned count, const unsigned char *idx, const unsigned *pals, unsigned bg, int x, int y,
	unsigned &cur, unsigned &saved)
{
	if (!P)
		cur = 0;
	else if (P->disposal == 2) {
		if (x >= P->x0 && x < P->bx1 && y >= P->y0 && y < P->by1)
			cur = P->transparency ? 0u : bg;
	}
	else if (P->disposal == 3)
		cur = saved;
	if (F.disposal == 3)
		saved = cur;
	if (F.want && x >= F.x0 && x < F.x0 + F.wc && y >= F.y0 && y < F.y0 + F.hc) {
		const int r = F.interlaced ? interlace_row(y - F.y0, F.hc) : y - F.y0;
		const unsigned long long i = (unsigned long long) r * (unsigned) F.w + (unsigned) (x - F.x0);
		if (i < count) {
			const int v = idx[F.idx_off + i];
			if (v != F.trans)
				cur = pals[(size_t) F.pal * 256 + v];
		}
	}
}

VB_HD void
put_pixel(unsigned char *o, unsigned v, int bands)
{
	o[0] = (unsigned char) v;
	o[1] = (unsigned char) (v >> 8);
	o[2] = (unsigned char) (v >> 16);
	if (bands == 4)
		o[3] = (unsigned char) (v >> 24);
}

/* ------------------------------------------------------------------ kernels */

constexpr unsigned kShortCopy = 16; /* strings up to this long are copied by lane 0 without waking the warp */

__global__ void __launch_bounds__(32)
gif_lzw_kernel(const GifFrameDev *__restrict__ frames, int n, const unsigned char *__restrict__ bytes, unsigned char *idx, unsigned *counts, int *status)
{
	__shared__ unsigned tpos[kTable];
	__shared__ unsigned short tlen[kTable];
	const int lane = threadIdx.x;
	for (int f = blockIdx.x; f < n; f += gridDim.x) {
		const GifFrameDev &F = frames[f];
		if (!F.want) {
			if (lane == 0)
				counts[f] = 0;
			continue;
		}
		unsigned char *out = idx + F.idx_off;
		Lzw z;
		lzw_init(z, bytes + F.data_off, F.data_len, F.want, F.min_code, F.lenient, tpos, tlen);
		for (;;) {
			int op = OP_DONE;
			unsigned at = 0, src = 0, len = 0;
			if (lane == 0)
				for (;;) {
					op = lzw_step(z, out, &at, &src, &len);
					if (op != OP_COPY || len > kShortCopy)
						break;
					for (unsigned i = 0; i < len; i++)
						out[at + i] = out[src + i];
				}
			op = __shfl_sync(0xffffffffu, op, 0);
			at = __shfl_sync(0xffffffffu, at, 0);
			src = __shfl_sync(0xffffffffu, src, 0);
			len = __shfl_sync(0xffffffffu, len, 0);
			__syncwarp(); /* lane 0's output is visible to the warp */
			if (op != OP_COPY)
				break;
			/* every source byte lies before `at`: the KwKwK copy (d = len - 1) repeats its period */
			const unsigned d = at - src;
			for (unsigned i = lane; i < len; i += 32)
				out[at + i] = out[src + (d >= len ? i : i % d)];
			__syncwarp();
		}
		if (lane == 0) {
			counts[f] = min(z.at, F.want);
			status[f] = z.err;
		}
		__syncwarp();
	}
}

__global__ void __launch_bounds__(256)
gif_compose_kernel(const GifFrameDev *__restrict__ frames, const GifStreamDev *__restrict__ streams, const unsigned *__restrict__ counts,
	const unsigned char *__restrict__ idx, const unsigned *__restrict__ pals, int W, int H, int bands, unsigned char *out, size_t out_bpl,
	size_t out_stride)
{
	const GifStreamDev S = streams[blockIdx.z];
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= W)
		return;
	unsigned char *o = out + (size_t) blockIdx.z * out_stride + (size_t) x * bands;
	for (int y = blockIdx.y; y < H; y += gridDim.y) {
		unsigned cur = 0, saved = 0;
		for (int k = 0; k < S.nf; k++) {
			const GifFrameDev *F = frames + S.f0 + k;
			gif_pixel(*F, k ? F - 1 : nullptr, counts[S.f0 + k], idx, pals, S.bg, x, y, cur, saved);
			if (k >= S.page)
				put_pixel(o + ((size_t) (k - S.page) * H + y) * out_bpl, cur, bands);
		}
	}
}

/* ------------------------------------------------------------------ host: the block walk (nsgif_data_scan) */

struct GifFrameInfo {
	unsigned x, y, w, h;
	int flags, interlaced, transparency, trans, disposal;
	size_t pal_pos;	 /* the local table, if flags say there is one */
	size_t data_pos; /* the minimum code size byte; sub-blocks follow */
	size_t lzw_bytes;
};

struct GifInfo {
	int W = 0, H = 0, bands = 3;
	unsigned global[256];
	unsigned bg = 0;
	std::vector<GifFrameInfo> fr;
	const unsigned char *d = nullptr;
};

GifFrameDev frame_record(const GifInfo &G, int k);

unsigned
rgba(const unsigned char *c)
{
	return (unsigned) c[0] | ((unsigned) c[1] << 8) | ((unsigned) c[2] << 16) | 0xff000000u;
}

/* What nsgif_data_scan + nsgif_data_complete leave (gif.c:1536-1786, with :748-1263 for each frame), or -1 with the
 * reason when nsgifload would not give what the decoder gives.
 */
int
parse_gif(const char *domain, const unsigned char *d, size_t len, GifInfo *G)
{
	enum { OK = 0, END = 1, DATA = 2 };
	if (!d || len < 6) {
		error(domain, "GIF stream too short");
		return -1;
	}
	if (memcmp(d, "GIF", 3) != 0) {
		error(domain, "not a GIF stream");
		return -1;
	}
	if (len - 6 < 7) {
		error(domain, "truncated GIF stream: %s", "the scan ends before the logical screen");
		return -1;
	}
	G->d = d;
	unsigned W = d[6] | (d[7] << 8), H = d[8] | (d[9] << 8);
	const bool gp = d[10] & 0x80;
	size_t cts = (size_t) 2 << (d[10] & 7);
	const unsigned bg_index = d[11];
	size_t pos = 13;
	if ((W == 640 && H == 480) || (W == 640 && H == 512) || (W == 800 && H == 600) || (W == 1024 && H == 768) || (W == 1280 && H == 1024) ||
		(W == 1600 && H == 1200) || W == 0 || H == 0 || W > 2048 || H > 2048)
		W = H = 1;
	if (len == pos + 1 && d[pos] == 0x3b) {
		error(domain, "no frames in GIF");
		return -1;
	}
	memset(G->global, 0, sizeof(G->global));
	if (gp) {
		if (len - pos < cts * 3) {
			error(domain, "truncated GIF stream: %s", "the global colour table runs past the end");
			return -1;
		}
		for (size_t i = 0; i < cts; i++)
			G->global[i] = rgba(d + pos + 3 * i);
		pos += cts * 3;
	}
	else {
		G->global[0] = 0xff000000u;
		G->global[1] = 0xffffffffu;
		cts = 2;
	}
	G->bg = gp && bg_index < cts ? G->global[bg_index] : G->global[0];
	/* nsgif__process_frame (decode = false) until a frame is not counted */
	int ret = OK;
	size_t partial_lzw = 0;
	bool partial = false;
	for (;;) {
		const size_t nfr = G->fr.size();
		GifFrameInfo F;
		memset(&F, 0, sizeof(F));
		F.trans = -1;
		if (pos < len && d[pos] == 0x3b)
			break;
		/* extensions (:888-982) */
		size_t p = pos;
		long long bytes = (long long) len - (long long) p;
		while (bytes > 0 && d[p] == 0x21) {
			p++;
			bytes--;
			if (bytes == 0) {
				ret = END;
				break;
			}
			bool step = true;
			if (d[p] == 0xf9) {
				if (bytes < 6) {
					ret = END;
					break;
				}
				if (d[p + 2] & 1) {
					F.transparency = 1;
					F.trans = d[p + 5];
				}
				F.disposal = (d[p + 2] & 0x1c) >> 2;
				if (F.disposal == 4)
					F.disposal = 3;
			}
			else if (d[p] == 0xff) {
				if (bytes < 17) {
					ret = END;
					break;
				}
			}
			else if (d[p] == 0xfe) {
				p++;
				step = false;
			}
			if (step) {
				if (bytes < 2) {
					ret = END;
					break;
				}
				p += 2 + d[p + 1];
			}
			while (p < len && d[p] != 0) {
				p += d[p] + 1;
				if (p >= len) {
					ret = END;
					break;
				}
			}
			if (ret)
				break;
			p++;
			bytes = (long long) len - (long long) p;
		}
		if (ret)
			break;
		if (p > len)
			p = len;
		/* image descriptor (:1007-1061) */
		if (len - p < 10) {
			ret = END;
			break;
		}
		if (d[p] != 0x2c) {
			ret = DATA;
			break;
		}
		F.x = d[p + 1] | (d[p + 2] << 8);
		F.y = d[p + 3] | (d[p + 4] << 8);
		F.w = d[p + 5] | (d[p + 6] << 8);
		F.h = d[p + 7] | (d[p + 8] << 8);
		F.flags = d[p + 9];
		F.interlaced = (F.flags & 0x40) != 0;
		if (nfr == 0) {
			W = std::max(W, F.x + F.w);
			H = std::max(H, F.y + F.h);
		}
		p += 10;
		/* local colour table (:1140-1179) */
		if (F.flags & 0x80) {
			const size_t n = (size_t) 2 << (F.flags & 7);
			if (len - p < n * 3) {
				ret = END;
				break;
			}
			F.pal_pos = p;
			p += n * 3;
		}
		/* image data (:1192-1263) */
		partial = true;
		partial_lzw = 0;
		const size_t rem0 = len - p;
		if (rem0 <= 2) {
			const bool trailer = (rem0 == 2 && (d[p + 1] == 0x3b || d[p] == 0x3b)) || (rem0 == 1 && d[p] == 0x3b);
			ret = trailer ? OK : END;
			break;
		}
		if (d[p] == 0x3b)
			break;
		if (d[p] >= kCodeMax) {
			ret = DATA;
			break;
		}
		F.data_pos = p;
		size_t rem = rem0 - 1, bs = 0;
		p++;
		while (bs != 1) {
			if (rem < 1) {
				ret = END;
				break;
			}
			bs = (size_t) d[p] + 1;
			if (bs > rem) {
				partial_lzw += rem;
				ret = END;
				break;
			}
			rem -= bs;
			p += bs;
			partial_lzw += bs;
			F.lzw_bytes += bs - 1;
		}
		if (ret)
			break;
		partial = false;
		pos = p;
		G->fr.push_back(F);
	}
	if (ret == END && !G->fr.empty())
		ret = OK;
	if (ret != OK) {
		error(domain, ret == END ? "truncated GIF stream (%s)" : "bad GIF stream (%s)", ret == END ? "Unexpected end of GIF source data" : "Invalid frame data");
		return -1;
	}
	if (partial && partial_lzw > 0) {
		error(domain, "truncated GIF stream: frame %d's data runs past the end", (int) G->fr.size());
		return -1;
	}
	if (G->fr.empty()) {
		error(domain, "no frames in GIF");
		return -1;
	}
	if (W > 65535 || H > 65535) {
		error(domain, "bad image dimensions");
		return -1;
	}
	if ((unsigned long long) W * H > (1ull << 28)) {
		error(domain, "%u x %u: screens over 2^28 pixels are not supported", W, H);
		return -1;
	}
	G->W = (int) W;
	G->H = (int) H;
	G->bands = 3;
	for (const GifFrameInfo &F : G->fr)
		if (F.transparency)
			G->bands = 4;
	for (size_t k = 0; k < G->fr.size(); k++)
		if (frame_record(*G, (int) k).want > kMaxValues) {
			error(domain, "frame %d needs more than 2^28 LZW values", (int) k);
			return -1;
		}
	return 0;
}

/* nsgifload's page / n rules (nsgifload.c:440-450): the pages to write, or -1 */
int
resolve_pages(const char *domain, const GifInfo &G, int page, int n, int *gif_n)
{
	const int fc = (int) G.fr.size();
	*gif_n = n == -1 ? fc - page : n;
	if (page < 0 || *gif_n <= 0 || page + *gif_n > fc) {
		error(domain, "bad page number");
		return -1;
	}
	return 0;
}

/* frame k's record (offsets and palette left to the caller): nsgif__decode's choice of path and its clipping */
GifFrameDev
frame_record(const GifInfo &G, int k)
{
	const GifFrameInfo &I = G.fr[k];
	GifFrameDev F;
	memset(&F, 0, sizeof(F));
	const unsigned W = (unsigned) G.W, H = (unsigned) G.H;
	F.data_len = (unsigned) I.lzw_bytes;
	F.min_code = G.d[I.data_pos];
	F.x0 = (int) I.x;
	F.y0 = (int) I.y;
	F.w = (int) I.w;
	F.interlaced = I.interlaced;
	F.trans = I.trans;
	F.transparency = I.transparency;
	F.disposal = I.disposal;
	F.bx1 = I.x < W && I.y < H ? (int) std::min(I.x + I.w, W) : F.x0;
	F.by1 = (int) std::min(I.y + I.h, H);
	const bool simple = !I.interlaced && I.x == 0 && I.w == W;
	if (I.x >= W || I.y >= H)
		return F;
	const unsigned wc = I.w - (I.x + I.w > W ? I.x + I.w - W : 0), hc = I.h - (I.y + I.h > H ? I.y + I.h - H : 0);
	if (wc == 0 || hc == 0)
		return F;
	F.wc = (int) wc;
	F.hc = (int) hc;
	F.lenient = !simple;
	/* the simple path decodes W x hc values; the complex one stops after the last drawn value of its last row.  A frame
	 * far wider than the screen could need more than 2^32: parse_gif declines past kMaxValues
	 */
	const unsigned long long want = simple ? (unsigned long long) W * hc : (unsigned long long) (hc - 1) * I.w + wc;
	F.want = (unsigned) std::min(want, kMaxValues + 1);
	return F;
}

/* the frame's LZW payload, its sub-blocks without their length bytes, and kPad zero bytes */
void
stage_lzw(const GifInfo &G, int k, unsigned char *dst)
{
	const unsigned char *p = G.d + G.fr[k].data_pos + 1;
	while (*p) {
		memcpy(dst, p + 1, *p);
		dst += *p;
		p += *p + 1;
	}
	memset(dst, 0, kPad);
}

/* every frame's table as nsgif__parse_colour_table leaves gif->colour_table: the global one, or the one local table
 * libnsgif keeps (zeroed by calloc) with this frame's entries written over it
 */
void
stage_palettes(const GifInfo &G, int nf, unsigned *pals)
{
	unsigned local[256];
	memset(local, 0, sizeof(local));
	for (int k = 0; k < nf; k++) {
		const GifFrameInfo &I = G.fr[k];
		if (I.flags & 0x80) {
			const int n = 2 << (I.flags & 7);
			for (int i = 0; i < n; i++)
				local[i] = rgba(G.d + I.pal_pos + 3 * i);
			memcpy(pals + (size_t) k * 256, local, sizeof(local));
		}
		else
			memcpy(pals + (size_t) k * 256, G.global, sizeof(local));
	}
}

/* device bytes a stream takes in a chunk: per frame its record, table, payload and index plane */
size_t
stream_device_bytes(const GifInfo &G, int nf)
{
	size_t b = sizeof(GifStreamDev);
	for (int k = 0; k < nf; k++) {
		const GifFrameDev F = frame_record(G, k);
		b += sizeof(GifFrameDev) + 1024 + align16(F.data_len + kPad) + align16(F.want) + 2 * sizeof(int);
	}
	return b;
}

} // namespace

bool
gif_signature(const void *buf, size_t len)
{
	return buf && len >= 6 && (memcmp(buf, "GIF87a", 6) == 0 || memcmp(buf, "GIF89a", 6) == 0);
}

/* Decode n GIF streams (host memory) of one output geometry into out[n][h * pages][w][bands] on the device (out = nullptr:
 * only report the geometry).  Streams are walked on the host workers; they go up in chunks bounded by
 * chunk_budget(), each one pinned block (stream and frame records, tables, LZW payloads) copied to the device.
 * Every frame of a chunk must decode clean before its pixels are composed into out.
 */
int
dev_gif_decode_batch(const char *domain, const void *const *bufs, const size_t *lens, int n, int page, int npages, void *out, size_t out_bpl,
	size_t out_frame_stride, StreamGeometry *g, cudaStream_t s)
{
	std::vector<GifInfo> info(n);
	std::vector<int> pages(n, 0);
	if (parse_streams(
			domain, "stream", n,
			[&](int i) {
				return parse_gif(domain, (const unsigned char *) bufs[i], lens[i], &info[i]) || resolve_pages(domain, info[i], page, npages, &pages[i]) ? -1 : 0;
			},
			[&](int i) { return StreamGeometry{info[i].W, info[i].H, info[i].bands, pages[i]}; }, g))
		return -1;
	if (!out)
		return 0;
	if (check_out_strides(domain, *g, out_bpl, out_frame_stride))
		return -1;
	const int W = g->w, H = g->h, B = g->bands;
	const int nf_stream = page + g->pages; /* frames 0 .. page + n - 1 of every stream */
	return decode_chunks(domain, "gif", "stream", n, [&](int i) { return stream_device_bytes(info[i], nf_stream); }, [&](int c0, int cn) {
		/* the block: stream records, frame records, tables and payloads staged; the index planes and counts as scratch */
		const int nf = cn * nf_stream;
		std::vector<GifStreamDev> S(cn);
		std::vector<GifFrameDev> F(nf);
		size_t data = 0, planes = 0;
		for (int i = 0; i < cn; i++) {
			S[i].f0 = i * nf_stream;
			S[i].nf = nf_stream;
			S[i].page = page;
			S[i].bg = info[c0 + i].bg;
			for (int k = 0; k < nf_stream; k++) {
				GifFrameDev &f = F[S[i].f0 + k];
				f = frame_record(info[c0 + i], k);
				f.pal = S[i].f0 + k;
				f.data_off = data;
				data += align16(f.data_len + kPad);
				f.idx_off = planes;
				planes += align16(f.want);
			}
		}
		const size_t off_fr = align16(cn * sizeof(GifStreamDev)), off_pal = off_fr + align16(nf * sizeof(GifFrameDev)),
					 off_data = off_pal + (size_t) nf * 1024, total = off_data + data;
		const size_t off_planes = align16(total), off_counts = off_planes + align16(planes);
		return decode_chunk(
			domain, "gif", {total, align16(planes) + nf * sizeof(unsigned), nf},
			[&](unsigned char *hst) {
				memcpy(hst, S.data(), cn * sizeof(GifStreamDev));
				memcpy(hst + off_fr, F.data(), nf * sizeof(GifFrameDev));
				parallel_for(cn, host_workers(), [&](int i) {
					const GifInfo &G = info[c0 + i];
					stage_palettes(G, nf_stream, (unsigned *) (hst + off_pal) + (size_t) S[i].f0 * 256);
					for (int k = 0; k < nf_stream; k++)
						stage_lzw(G, k, hst + off_data + F[S[i].f0 + k].data_off);
				});
			},
			[&](unsigned char *dev, int *status) {
				gif_lzw_kernel<<<std::min(nf, sm_count() * 16), 32, 0, s>>>((const GifFrameDev *) (dev + off_fr), nf, dev + off_data, dev + off_planes,
					(unsigned *) (dev + off_counts), status);
				return 1;
			},
			[&](int i, int) { error(domain, "stream %d: frame %d: bad LZW code (libnsgif: Invalid frame data)", c0 + i / nf_stream, i % nf_stream); },
			[&](unsigned char *dev) {
				gif_compose_kernel<<<dim3((W + 255) / 256, std::min(H, kMaxGridY), cn), 256, 0, s>>>((const GifFrameDev *) (dev + off_fr),
					(const GifStreamDev *) dev, (const unsigned *) (dev + off_counts), dev + off_planes, (const unsigned *) (dev + off_pal), W, H, B,
					(unsigned char *) out + (size_t) c0 * out_frame_stride, out_bpl, out_frame_stride);
				return 1;
			},
			s);
	}, s);
}

/* the same decode on the CPU through the same per-code and per-pixel code: the test-suite's host twin */
int
host_gif_decode(const char *domain, const void *buf, size_t len, int page, int npages, unsigned char *out, size_t out_bpl, int *out_w, int *out_h,
	int *out_bands)
{
	GifInfo G;
	int P = 0;
	if (parse_gif(domain, (const unsigned char *) buf, len, &G) || resolve_pages(domain, G, page, npages, &P))
		return -1;
	if (out_w)
		*out_w = G.W;
	if (out_h)
		*out_h = G.H * P;
	if (out_bands)
		*out_bands = G.bands;
	if (!out)
		return 0;
	const int nf = page + P;
	std::vector<GifFrameDev> F(nf);
	std::vector<unsigned> pals((size_t) nf * 256), counts(nf);
	size_t planes = 0;
	for (int k = 0; k < nf; k++) {
		F[k] = frame_record(G, k);
		F[k].pal = k;
		F[k].idx_off = planes;
		planes += F[k].want;
	}
	stage_palettes(G, nf, pals.data());
	std::vector<unsigned char> idx(planes + 1);
	for (int k = 0; k < nf; k++) {
		if (!F[k].want)
			continue;
		std::vector<unsigned char> data(F[k].data_len + kPad);
		stage_lzw(G, k, data.data());
		int err = 0;
		counts[k] = lzw_host(data.data(), F[k].data_len, F[k].want, F[k].min_code, F[k].lenient, idx.data() + F[k].idx_off, &err);
		if (err) {
			error(domain, "frame %d: bad LZW code (libnsgif: Invalid frame data)", k);
			return -1;
		}
	}
	for (int y = 0; y < G.H; y++)
		for (int x = 0; x < G.W; x++) {
			unsigned cur = 0, saved = 0;
			for (int k = 0; k < nf; k++) {
				gif_pixel(F[k], k ? &F[k - 1] : nullptr, counts[k], idx.data(), pals.data(), G.bg, x, y, cur, saved);
				if (k >= page)
					put_pixel(out + ((size_t) (k - page) * G.H + y) * out_bpl + (size_t) x * G.bands, cur, G.bands);
			}
		}
	return 0;
}

} // namespace vb200

/* ------------------------------------------------------------------ C ABI */

using namespace vb200;

/* reference: nsgif_data_scan + nsgif_get_info as nsgifload's header reads them (nsgifload.c:364-474) */
extern "C" int
vb200_gif_geometry(const void *buf, size_t len, int *width, int *height, int *bands, int *frames)
{
	GifInfo G;
	if (parse_gif("gif_geometry", (const unsigned char *) buf, len, &G))
		return -1;
	if (width)
		*width = G.W;
	if (height)
		*height = G.H;
	if (bands)
		*bands = G.bands;
	if (frames)
		*frames = (int) G.fr.size();
	return 0;
}

extern "C" int
vb200_gif_decode_batch(const void *const *bufs, const size_t *lens, int n, int page, int n_pages, void *out, int out_location, size_t out_bpl,
	size_t out_frame_stride, int *width, int *height, int *bands)
{
	return decode_batch_abi("gif_decode_batch", {STREAM_GIF, 1, page, n_pages}, bufs, lens, n, out, out_location, out_bpl, out_frame_stride, width,
		height, bands);
}

/* reference: vips_gifload_buffer(buf, len, &out, "page", page, "n", n, NULL), foreign/nsgifload.c */
extern "C" int
vb200_gifload_buffer(const void *buf, size_t len, int page, int n, VB200Image *out)
{
	return load_abi("gifload_buffer", {STREAM_GIF, 1, page, n}, buf, len, out);
}

extern "C" int
vb200_debug_gif_decode(const void *buf, size_t len, int page, int n, void *out, size_t out_bpl, int *width, int *height, int *bands)
{
	return host_twin_abi("gif_decode (host twin)",
		[&](const char *domain) { return host_gif_decode(domain, buf, len, page, n, (unsigned char *) out, out_bpl, width, height, bands); });
}

/* LZW data (sub-blocks already joined) through the host twin's decoder: 0 and *out_len values (at most want), or -1 for
 * a code libnsgif refuses.  lenient: the complex path's rule for a bad code at a multiple of 4096 values
 */
extern "C" int
vb200_debug_lzw(const void *data, size_t len, int min_code_size, unsigned want, int lenient, void *out, size_t *out_len)
{
	const char *domain = "lzw (host twin)";
	if (min_code_size < 0 || min_code_size >= kCodeMax) {
		error(domain, "minimum code size %d (libnsgif: Invalid frame data)", min_code_size);
		return -1;
	}
	if (len > 0xffffffffu - kPad) {
		error(domain, "too much data");
		return -1;
	}
	std::vector<unsigned char> src(len + kPad, 0);
	if (len)
		memcpy(src.data(), data, len);
	int err = 0;
	const unsigned got = lzw_host(src.data(), (unsigned) len, want, min_code_size, lenient, (unsigned char *) out, &err);
	if (out_len)
		*out_len = got;
	if (err) {
		error(domain, "bad LZW code after %u values (libnsgif: Invalid frame data)", got);
		return -1;
	}
	return 0;
}
