/* tiff.cu -- vips_tiffload_buffer's 8-bit strips and tiles decoded on the device, and the pyramid level vips_thumbnail
 * loads from a TIFF.
 *
 * What the reference does (foreign/tiff2vips.c over libtiff, fail_on = none): rtiff_header_read (:3008-3360) reads the
 * IFD that `page` / `n` / `subifd` select (rtiff_set_page, :798-846); the pages of an n > 1 strip must agree
 * (rtiff_header_equal, :3364); greyscale images load as B_W with MINISWHITE's first band inverted for uint samples
 * (rtiff_parse_greyscale / rtiff_greyscale_line, :1359-1448), RGB as sRGB with every sample copied (rtiff_parse_copy,
 * :1723-1780).  libtiff itself decodes the segments: none, PackBits, LZW (MSB-first codes, early change), deflate (zlib
 * streams), each followed by predictor 2's horizontal accumulation over a segment row when the Predictor tag asks.
 *
 * Scope: classic and BigTIFF, either byte order, PlanarConfiguration 1, FillOrder 1, 8-bit unsigned samples; MINISBLACK
 * and MINISWHITE with 1-2 samples, RGB with 3-4; ExtraSamples 0 or 2; compression 1, 5, 8, 32946 and 32773 in strips or
 * tiles; predictor 1 or 2; JPEG (7) tiles, greyscale or YCbCr, with or without JPEGTables, which tiff2vips decodes with
 * its own libjpeg calls (rtiff_decompress_jpeg_run, :2082-2177).  Everything else returns -1 with its reason from the IFD
 * (and, for JPEG, the tiles' headers), before any device work, and the host keeps tiff2vips: other bit depths and sample
 * formats, separate planes, FillOrder 2, palette / CIELAB / separated / LogLuv photometrics, YCbCr without JPEG, JPEG
 * strips (libtiff's own JPEG codec decodes those) and RGB-photometric JPEG, associated alpha, old-style JPEG and LZW, any
 * other compression, predictor 3, segments outside the stream, pages of a strip whose headers differ, frames over 2^28
 * pixels, and every JPEG tile the JPEG decoder declines ("tile k: ...").  A segment that decodes to fewer bytes than its
 * rows need fails the batch, as libtiff's "Not enough data" does.  Deflate runs as zlib does under libtiff's ZIPDecode:
 * it stops once the segment's rows are full (a padded last strip loads), and when the last block ends with them full it
 * checks the Adler-32 trailer and refuses a mismatch.
 *
 * Device pipeline per chunk of streams (the compressed segments, deflate's without their 2-byte zlib header, are all that
 * crosses PCIe; uncompressed segments are placed straight from their staged bytes):
 *   tiff_inflate_kernel   one warp per deflate segment: inflate.cuh's inflate_warp, the loop png_inflate_kernel runs
 *   tiff_lzw_kernel       one warp per LZW segment: lane 0 reads the codes and writes short strings, the warp copies
 *                         long ones; the string table (where each code's string begins in the output and its length) in
 *                         shared memory
 *   tiff_packbits_kernel  one thread per PackBits segment
 *   JPEG tiles            no new kernel: each tile with JPEGTables' DQT / DHT spliced in front of its SOF, one
 *                         dev_jpeg_decode_batch at shrink 1 per run of tiles of one geometry
 *   tiff_place_kernel     one CTA per segment, only once every segment of the chunk decoded clean: one warp per row undoes
 *                         predictor 2 as a per-band warp scan, inverts MINISWHITE and writes the clipped row into
 *                         out[n][rows][w][bands] at the caller's strides
 * The per-code and per-byte code is __host__ __device__: vb200_debug_tiff_decode runs it on the CPU so that the CPU
 * test-suite pins it against the oracle and libtiff without a GPU.
 */
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <functional>
#include <string>
#include <vector>

#include "../../include/vb200.h"
#include "vb200_internal.h"

#define VB_HD __host__ __device__ __forceinline__

#include "inflate.cuh"

namespace vb200 {

namespace {

/* ------------------------------------------------------------------ segment codecs, host and device */

enum { C_NONE = 0, C_PACKBITS = 1, C_LZW = 2, C_DEFLATE = 3, C_JPEG = 4 };
enum { ERR_FEWER = 4, ERR_CHECK = 8 }; /* above inflate.cuh's ERR_CORRUPT / ERR_MORE */
constexpr int kCheckTrailer = -1;

/* libtiff's ZIPDecode over a clip-mode inflate that has stopped: 0, an ERR_* status, or kCheckTrailer when zlib goes on to
 * read the trailer (the last block ended with the rows exactly full and 4 bytes follow), *trailer its value
 */
VB_HD int
deflate_status(const Inflate &z, int op, unsigned long long want, unsigned *trailer)
{
	if (op == OP_ERR)
		return z.err;
	if (z.pos != want)
		return ERR_FEWER; /* "Not enough data" */
	if (!z.full && inflate_trailer(z, trailer))
		return kCheckTrailer;
	return 0;
}

constexpr unsigned kAdlerMod = 65521;

/* adler32 (RFC 1950 8.2) of n bytes on one thread */
inline unsigned
adler32_host(const unsigned char *p, unsigned long long n)
{
	unsigned long long a = 1, b = 0;
	for (unsigned long long i = 0; i < n; i++) {
		a = (a + p[i]) % kAdlerMod;
		b = (b + a) % kAdlerMod;
	}
	return (unsigned) ((b << 16) | a);
}

#ifdef __CUDACC__
/* the same on a warp: lane l sums its slice (S = the bytes, T = the sum of its running sums), and each slice's T is shifted
 * by S times the bytes after it: adler = (1 + sum S) | (n + sum over slices of T + S * after) << 16, every sum mod 65521
 */
__device__ unsigned
adler32_warp(const unsigned char *p, unsigned long long n, int lane)
{
	const unsigned long long per = (n + 31) / 32, lo = min(n, per * lane), hi = min(n, lo + per);
	unsigned long long S = 0, T = 0;
	for (unsigned long long i = lo; i < hi; i++) {
		S += p[i];
		T += S;
		if ((i - lo) % 4096 == 4095) {
			S %= kAdlerMod;
			T %= kAdlerMod;
		}
	}
	S %= kAdlerMod;
	T = (T + S * ((n - hi) % kAdlerMod)) % kAdlerMod;
	for (int o = 16; o > 0; o >>= 1) {
		S = (S + __shfl_xor_sync(0xffffffffu, S, o)) % kAdlerMod;
		T = (T + __shfl_xor_sync(0xffffffffu, T, o)) % kAdlerMod;
	}
	const unsigned long long a = (1 + S) % kAdlerMod, b = (n % kAdlerMod + T) % kAdlerMod;
	return (unsigned) ((b << 16) | a);
}
#endif

/* one segment as the kernels see it; offsets are into the chunk's device block */
struct TiffSeg {
	unsigned long long src, src_len; /* the staged compressed bytes */
	unsigned long long dec;			 /* the decoded bytes (the staged bytes themselves when uncompressed) */
	unsigned long long dec_len;		 /* rows * seg_w * spp */
	int frame;						 /* the stream's index in the chunk */
	int row0, col0;					 /* where the segment's first pixel goes in the frame (rows of every page) */
	int seg_w, clip_w, clip_h;		 /* pixels per decoded row; pixels and rows inside the image */
	unsigned char comp, pred, invert, spp;
};

/* libtiff's LZWDecode (tif_lzw.c): MSB-first codes of 9-12 bits, 256 clear, 257 end; a code widens when the next free
 * entry reaches 2^bits - 1 (early change), the table holds 5119 entries before anything but clear or end is refused.
 * Entry k's string is the previous code's string followed by the first byte of the code after it: in the output, the
 * previous code's bytes and the one after them.  So the table keeps where that string begins and how long it is, and
 * every code past 257 is a copy from earlier output.
 */
constexpr int kLzwClear = 256, kLzwEoi = 257, kLzwFirst = 258, kLzwTable = 4095 + 1024;
constexpr unsigned kLzwShort = 16; /* strings lane 0 copies itself; longer ones go to the warp */

struct Lzw {
	const unsigned char *src;
	unsigned long long len, bit; /* input bytes, bits consumed */
	unsigned long long pos, cap; /* output */
	unsigned *start;			 /* kLzwTable entries each */
	unsigned short *length;
	unsigned long long old_pos;
	unsigned old_len;
	int nbits, free_ent, have_old, err;
};

VB_HD void
lzw_init(Lzw &z, const unsigned char *src, unsigned long long len, unsigned long long cap, unsigned *start, unsigned short *length)
{
	z.src = src;
	z.len = len;
	z.bit = 0;
	z.pos = 0;
	z.cap = cap;
	z.start = start;
	z.length = length;
	z.old_pos = 0;
	z.old_len = 0;
	z.nbits = 9;
	z.free_ent = kLzwFirst;
	z.have_old = 0; /* LZWPreDecode's dec_oldcodep = &dec_codetab[-1]: a first code that is not clear is refused */
	z.err = 0;
}

/* GetNextCode: a code that needs bits past the end reads as the end code (libtiff warns "not terminated with EOI") */
VB_HD int
lzw_code(Lzw &z)
{
	if (z.len * 8 - z.bit < (unsigned long long) z.nbits)
		return kLzwEoi;
	const unsigned long long b = z.bit >> 3;
	unsigned w = (unsigned) z.src[b] << 16;
	if (b + 1 < z.len)
		w |= (unsigned) z.src[b + 1] << 8;
	if (b + 2 < z.len)
		w |= z.src[b + 2];
	const int code = (int) ((w >> (24 - (int) (z.bit & 7) - z.nbits)) & ((1u << z.nbits) - 1));
	z.bit += z.nbits;
	return code;
}

/* Run until a string longer than kLzwShort (*at, *len, *dist: a copy from at - dist), the end or an error; literals and
 * short strings are written here.  Stops once cap bytes are out, as LZWDecode's loop does.
 */
VB_HD int
lzw_step(Lzw &z, unsigned char *out, unsigned long long *at, unsigned *len, unsigned long long *dist)
{
	while (z.pos < z.cap) {
		int code = lzw_code(z);
		if (code == kLzwEoi)
			break;
		if (code == kLzwClear) {
			do {
				z.free_ent = kLzwFirst;
				z.nbits = 9;
				code = lzw_code(z);
			} while (code == kLzwClear);
			if (code == kLzwEoi)
				break;
			if (code > kLzwClear) {
				z.err = ERR_CORRUPT; /* "Corrupted LZW table" */
				return OP_ERR;
			}
			z.old_pos = z.pos;
			z.old_len = 1;
			z.have_old = 1;
			out[z.pos++] = (unsigned char) code;
			continue;
		}
		/* the new entry first (the previous string plus this code's first byte), then this code */
		if (!z.have_old || z.free_ent >= kLzwTable || (code >= kLzwFirst && code > z.free_ent)) {
			z.err = ERR_CORRUPT;
			return OP_ERR;
		}
		z.start[z.free_ent] = (unsigned) z.old_pos;
		z.length[z.free_ent] = (unsigned short) (z.old_len + 1);
		if (++z.free_ent > (1 << z.nbits) - 2 && z.nbits < 12)
			z.nbits++;
		if (code < 256) {
			z.old_pos = z.pos;
			z.old_len = 1;
			out[z.pos++] = (unsigned char) code;
			continue;
		}
		const unsigned long long s = z.start[code];
		const unsigned l = z.length[code];
		const unsigned n = (unsigned) (z.cap - z.pos < l ? z.cap - z.pos : l);
		z.old_pos = z.pos;
		z.old_len = l;
		if (n > kLzwShort) {
			*at = z.pos;
			*len = n;
			*dist = z.pos - s;
			z.pos += n;
			return OP_MATCH;
		}
		for (unsigned i = 0; i < n; i++)
			out[z.pos + i] = out[s + i];
		z.pos += n;
	}
	return z.pos == z.cap ? OP_DONE : (z.err = ERR_FEWER, OP_ERR);
}

/* the whole segment on one thread (the host twin); -1 with z.err set */
int
lzw_host(Lzw &z, unsigned char *out)
{
	for (;;) {
		unsigned long long at = 0, dist = 0;
		unsigned n = 0;
		const int op = lzw_step(z, out, &at, &n, &dist);
		if (op != OP_MATCH)
			return op == OP_DONE ? 0 : -1;
		for (unsigned i = 0; i < n; i++)
			out[at + i] = out[at - dist + i];
	}
}

/* libtiff's PackBitsDecode (tif_packbits.c): runs and literals clipped to the output, "Not enough data" if it is not full */
VB_HD int
packbits_decode(const unsigned char *src, unsigned long long cc, unsigned char *out, unsigned long long occ)
{
	unsigned long long o = 0;
	while (cc > 0 && o < occ) {
		long long n = *src++;
		cc--;
		if (n >= 128)
			n -= 256;
		if (n < 0) {
			if (n == -128)
				continue;
			n = -n + 1;
			if ((long long) (occ - o) < n)
				n = (long long) (occ - o);
			if (cc == 0)
				break;
			const unsigned char b = *src++;
			cc--;
			for (long long i = 0; i < n; i++)
				out[o++] = b;
		}
		else {
			if ((long long) (occ - o) < n + 1)
				n = (long long) (occ - o) - 1;
			if ((long long) cc < n + 1)
				break;
			for (long long i = 0; i <= n; i++)
				out[o++] = src[i];
			src += n + 1;
			cc -= (unsigned long long) n + 1;
		}
	}
	return o == occ ? 0 : ERR_FEWER;
}

/* ------------------------------------------------------------------ kernels */

constexpr int kInflateWarps = 4;

__global__ void __launch_bounds__(kInflateWarps * 32)
tiff_inflate_kernel(const TiffSeg *__restrict__ segs, const int *__restrict__ list, int n, unsigned char *block, int *status)
{
	__shared__ InflateTables tabs[kInflateWarps];
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	for (int i = blockIdx.x * kInflateWarps + warp; i < n; i += gridDim.x * kInflateWarps) {
		const int k = list[i];
		const TiffSeg S = segs[k];
		const unsigned char *src = block + S.src;
		unsigned char *out = block + S.dec;
		Inflate z;
		inflate_init(z, src, S.src_len, S.dec_len, &tabs[warp]);
		z.clip = 1;
		const int op = inflate_warp(z, src, out, lane);
		int st = 0;
		unsigned trailer = 0;
		if (lane == 0)
			st = deflate_status(z, op, S.dec_len, &trailer);
		st = __shfl_sync(0xffffffffu, st, 0);
		if (st == kCheckTrailer) {
			/* the last block ended with the rows full: zlib reads the Adler-32 trailer (RFC 1950) and refuses a mismatch */
			trailer = __shfl_sync(0xffffffffu, trailer, 0);
			st = adler32_warp(out, S.dec_len, lane) == trailer ? 0 : ERR_CHECK;
		}
		if (lane == 0 && st)
			status[k] = st;
		__syncwarp();
	}
}

__global__ void __launch_bounds__(32)
tiff_lzw_kernel(const TiffSeg *__restrict__ segs, const int *__restrict__ list, int n, unsigned char *block, int *status)
{
	__shared__ unsigned start[kLzwTable];
	__shared__ unsigned short length[kLzwTable];
	const int lane = threadIdx.x;
	for (int i = blockIdx.x; i < n; i += gridDim.x) {
		const int k = list[i];
		const TiffSeg S = segs[k];
		unsigned char *out = block + S.dec;
		Lzw z;
		lzw_init(z, block + S.src, S.src_len, S.dec_len, start, length);
		int op = OP_DONE;
		for (;;) {
			unsigned long long at = 0, dist = 0;
			unsigned len = 0;
			if (lane == 0)
				op = lzw_step(z, out, &at, &len, &dist);
			op = __shfl_sync(0xffffffffu, op, 0);
			at = __shfl_sync(0xffffffffu, at, 0);
			dist = __shfl_sync(0xffffffffu, dist, 0);
			len = __shfl_sync(0xffffffffu, len, 0);
			__syncwarp(); /* lane 0's bytes are visible to the warp */
			if (op != OP_MATCH)
				break;
			/* an overlapping copy (the code just added) repeats its period */
			const unsigned d = (unsigned) dist;
			for (unsigned j = lane; j < len; j += 32)
				out[at + j] = out[at - d + (d >= len ? j : j % d)];
			__syncwarp();
		}
		if (lane == 0 && op == OP_ERR)
			status[k] = z.err;
		__syncwarp();
	}
}

__global__ void __launch_bounds__(128)
tiff_packbits_kernel(const TiffSeg *__restrict__ segs, const int *__restrict__ list, int n, unsigned char *block, int *status)
{
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const int k = list[i];
		const TiffSeg S = segs[k];
		const int st = packbits_decode(block + S.src, S.src_len, block + S.dec, S.dec_len);
		if (st)
			status[k] = st;
	}
}

constexpr int kPlaceWarps = 8;

/* One CTA per segment, one warp per row.  Predictor 2 (tif_predict.c horAcc8) is a running sum per band along the row:
 * the warp takes 32 - 32 % spp bytes at a time, scans each band with shuffles spp, 2 spp, 4 spp .. lanes up, and carries
 * every band's last sum into the next step.
 */
__global__ void __launch_bounds__(kPlaceWarps * 32)
tiff_place_kernel(const TiffSeg *__restrict__ segs, int n, const unsigned char *__restrict__ block, unsigned char *out, size_t out_bpl,
	size_t out_frame_stride)
{
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	for (int k = blockIdx.x; k < n; k += gridDim.x) {
		const TiffSeg S = segs[k];
		const int spp = S.spp, clip = S.clip_w * spp, chunk = 32 - 32 % spp;
		const size_t row_bytes = (size_t) S.seg_w * spp;
		for (int r = warp; r < S.clip_h; r += kPlaceWarps) {
			const unsigned char *src = block + S.dec + (size_t) r * row_bytes;
			unsigned char *dst = out + (size_t) S.frame * out_frame_stride + (size_t) (S.row0 + r) * out_bpl + (size_t) S.col0 * spp;
			if (!S.pred) {
				for (int i = lane; i < clip; i += 32) {
					const unsigned char v = src[i];
					dst[i] = S.invert && i % spp == 0 ? (unsigned char) (255 - v) : v;
				}
				continue;
			}
			const int band = lane % spp;
			unsigned carry = 0; /* sums mod 256: only the low byte is ever kept */
			for (int i0 = 0; i0 < clip; i0 += chunk) {
				const int i = i0 + lane;
				const bool mine = lane < chunk && i < clip;
				unsigned v = mine ? src[i] : 0;
				for (int off = spp; off < 32; off <<= 1) {
					const unsigned u = __shfl_up_sync(0xffffffffu, v, off);
					if (lane >= off)
						v = (v + u) & 255;
				}
				v = (v + carry) & 255;
				carry = __shfl_sync(0xffffffffu, v, chunk - spp + band);
				if (mine)
					dst[i] = S.invert && band == 0 ? (unsigned char) (255 - v) : (unsigned char) v;
			}
		}
	}
}

/* ------------------------------------------------------------------ host: the IFD walk */

const int kMaxPages = 1 << 16; /* IFDs followed along a chain before it counts as a loop */

struct TiffFile {
	const unsigned char *d = nullptr;
	size_t len = 0;
	bool le = true, big = false;
	std::vector<unsigned long long> pages; /* the main IFD of each page */

	unsigned long long u(size_t at, int bytes) const
	{
		unsigned long long v = 0;
		for (int i = 0; i < bytes; i++)
			v |= (unsigned long long) d[at + (le ? i : bytes - 1 - i)] << (8 * i);
		return v;
	}
};

struct TiffIfd {
	long long w = -1, h = -1;
	int spp = 1, bps = 1, photometric = -1, compression = 1, planar = 1, fill = 1, predictor = 1, sample_format = 1, orientation = 1;
	int extra = 0;
	bool tiled = false;
	long long tw = 0, th = 0, rps = 0xffffffffll;
	std::vector<unsigned long long> offsets, counts, subifds;
	const unsigned char *icc = nullptr;
	size_t icc_len = 0;
	const unsigned char *tables = nullptr; /* JPEGTables (347) */
	size_t tables_len = 0;
	/* the decode's view, set by check_ifd */
	int comp = C_NONE, seg_w = 0, seg_h = 0, across = 0, segs = 0;
	bool pred = false, invert = false;
};

int
type_size(int type)
{
	switch (type) {
	case 1: case 2: case 6: case 7:
		return 1;
	case 3: case 8:
		return 2;
	case 4: case 9: case 11: case 13:
		return 4;
	case 5: case 10: case 12: case 16: case 17: case 18:
		return 8;
	default:
		return 0;
	}
}

int
parse_header(const char *domain, const unsigned char *d, size_t len, TiffFile *F)
{
	if (!d || len < 8 || !((d[0] == 'I' && d[1] == 'I') || (d[0] == 'M' && d[1] == 'M'))) {
		error(domain, "not a TIFF stream");
		return -1;
	}
	F->d = d;
	F->len = len;
	F->le = d[0] == 'I';
	const unsigned magic = (unsigned) F->u(2, 2);
	unsigned long long first;
	if (magic == 42)
		first = F->u(4, 4);
	else if (magic == 43 && len >= 16 && F->u(4, 2) == 8 && F->u(6, 2) == 0) {
		F->big = true;
		first = F->u(8, 8);
	}
	else {
		error(domain, "not a TIFF stream");
		return -1;
	}
	/* the IFD chain: every IFD must hold its entry count, its entries and its next offset */
	for (unsigned long long off = first; off;) {
		if ((int) F->pages.size() >= kMaxPages) {
			error(domain, "IFD chain longer than %d pages (a loop?)", kMaxPages);
			return -1;
		}
		const int cb = F->big ? 8 : 2, eb = F->big ? 20 : 12, nb = F->big ? 8 : 4;
		if (off > len || len - off < (size_t) cb) {
			error(domain, "IFD %d lies outside the stream", (int) F->pages.size());
			return -1;
		}
		const unsigned long long ne = F->u(off, cb);
		if (ne > (len - off - cb) / eb || len - off - cb - ne * eb < (size_t) nb) {
			error(domain, "IFD %d lies outside the stream", (int) F->pages.size());
			return -1;
		}
		F->pages.push_back(off);
		off = F->u(off + cb + ne * eb, nb);
	}
	if (F->pages.empty()) {
		error(domain, "TIFF stream has no IFD");
		return -1;
	}
	return 0;
}

/* one entry's values as unsigned integers */
int
entry_values(const char *domain, const TiffFile &F, size_t e, std::vector<unsigned long long> *v, int tag)
{
	const int type = (int) F.u(e + 2, 2), sz = type_size(type);
	const unsigned long long count = F.u(e + 4, F.big ? 8 : 4);
	const int inl = F.big ? 8 : 4;
	if (!(type == 1 || type == 3 || type == 4 || type == 13 || type == 16 || type == 18)) {
		error(domain, "tag %d has type %d, not an unsigned integer", tag, type);
		return -1;
	}
	if (count > F.len / sz) {
		error(domain, "tag %d's values lie outside the stream", tag);
		return -1;
	}
	size_t at = e + (F.big ? 12 : 8);
	if (count * sz > (unsigned long long) inl) {
		const unsigned long long off = F.u(at, inl);
		if (off > F.len || F.len - off < count * sz) {
			error(domain, "tag %d's values lie outside the stream", tag);
			return -1;
		}
		at = (size_t) off;
	}
	v->resize((size_t) count);
	for (size_t i = 0; i < count; i++)
		(*v)[i] = F.u(at + i * sz, sz);
	return 0;
}

/* an UNDEFINED / BYTE blob (ICCProfile) */
int
entry_blob(const char *domain, const TiffFile &F, size_t e, const unsigned char **p, size_t *n, int tag)
{
	const int type = (int) F.u(e + 2, 2), sz = type_size(type);
	const unsigned long long count = F.u(e + 4, F.big ? 8 : 4);
	const int inl = F.big ? 8 : 4;
	if (sz != 1 || count > F.len) {
		error(domain, "tag %d is not a byte string", tag);
		return -1;
	}
	size_t at = e + (F.big ? 12 : 8);
	if (count > (unsigned long long) inl) {
		const unsigned long long off = F.u(at, inl);
		if (off > F.len || F.len - off < count) {
			error(domain, "tag %d's values lie outside the stream", tag);
			return -1;
		}
		at = (size_t) off;
	}
	*p = F.d + at;
	*n = (size_t) count;
	return 0;
}

/* the IFD at off: the fields tiff2vips reads for this subset; the chain walk has bounded the entries */
int
parse_ifd(const char *domain, const TiffFile &F, unsigned long long off, TiffIfd *I)
{
	const int cb = F.big ? 8 : 2, eb = F.big ? 20 : 12;
	const unsigned long long ne = F.u(off, cb);
	std::vector<unsigned long long> v;
	for (unsigned long long k = 0; k < ne; k++) {
		const size_t e = (size_t) (off + cb + k * eb);
		const int tag = (int) F.u(e, 2);
		switch (tag) {
		case 256: case 257: case 258: case 259: case 262: case 266: case 274: case 277: case 278: case 284: case 317: case 322: case 323:
		case 338: case 339:
			if (entry_values(domain, F, e, &v, tag))
				return -1;
			if (v.empty()) {
				error(domain, "tag %d has no value", tag);
				return -1;
			}
			break;
		case 273: case 279: case 324: case 325: case 330:
			if (entry_values(domain, F, e, &v, tag))
				return -1;
			break;
		case 34675:
			if (entry_blob(domain, F, e, &I->icc, &I->icc_len, tag))
				return -1;
			continue;
		case 347:
			if (entry_blob(domain, F, e, &I->tables, &I->tables_len, tag))
				return -1;
			continue;
		default:
			continue;
		}
		const long long v0 = v.empty() ? 0 : (long long) std::min<unsigned long long>(v[0], 0x7fffffffffffll);
		switch (tag) {
		case 256: I->w = v0; break;
		case 257: I->h = v0; break;
		case 258:
			I->bps = (int) std::min<long long>(v0, 1 << 16);
			for (unsigned long long x : v)
				if ((long long) x != v0)
					I->bps = -1; /* samples of different depths */
			break;
		case 259: I->compression = (int) std::min<long long>(v0, 1 << 20); break;
		case 262: I->photometric = (int) std::min<long long>(v0, 1 << 20); break;
		case 266: I->fill = (int) std::min<long long>(v0, 1 << 16); break;
		case 274: I->orientation = (int) std::min<long long>(v0, 1 << 16); break;
		case 277: I->spp = (int) std::min<long long>(v0, 1 << 16); break;
		case 278: I->rps = v0; break;
		case 284: I->planar = (int) std::min<long long>(v0, 1 << 16); break;
		case 317: I->predictor = (int) std::min<long long>(v0, 1 << 16); break;
		case 322: I->tw = v0; I->tiled = true; break;
		case 323: I->th = v0; I->tiled = true; break;
		case 338: I->extra = (int) std::min<long long>(v0, 1 << 16); break;
		case 339:
			I->sample_format = (int) std::min<long long>(v0, 1 << 16);
			break;
		case 273: case 324: I->offsets = v; break;
		case 279: case 325: I->counts = v; break;
		case 330: I->subifds = v; break;
		}
	}
	if (I->w < 1 || I->h < 1) {
		error(domain, "TIFF IFD without ImageWidth / ImageLength");
		return -1;
	}
	if (I->w > 0x7fffffff || I->h > 0x7fffffff) {
		error(domain, "bad TIFF dimensions %lld x %lld", I->w, I->h);
		return -1;
	}
	return 0;
}

/* The IFD that page / subifd name (subifd -1: the page's main IFD), rtiff_set_page (tiff2vips.c:798-846) */
int
select_ifd(const char *domain, const TiffFile &F, int page, int subifd, TiffIfd *I)
{
	if (page < 0 || page >= (int) F.pages.size()) {
		error(domain, "bad page number %d (the stream has %d)", page, (int) F.pages.size());
		return -1;
	}
	if (parse_ifd(domain, F, F.pages[page], I))
		return -1;
	if (subifd < 0)
		return 0;
	if (subifd >= (int) I->subifds.size()) {
		error(domain, "subifd %d out of range (page %d has %d)", subifd, page, (int) I->subifds.size());
		return -1;
	}
	const unsigned long long off = I->subifds[subifd];
	const int cb = F.big ? 8 : 2, eb = F.big ? 20 : 12;
	if (off > F.len || F.len - off < (size_t) cb || F.u(off, cb) > (F.len - off - cb) / eb) {
		error(domain, "subifd %d lies outside the stream", subifd);
		return -1;
	}
	*I = TiffIfd();
	return parse_ifd(domain, F, off, I);
}

const char *
photometric_name(int p)
{
	switch (p) {
	case 3: return "palette";
	case 4: return "transparency mask";
	case 5: return "separated (CMYK)";
	case 6: return "YCbCr";
	case 8: case 9: case 10: return "CIELAB";
	case 32844: case 32845: return "LogLuv";
	default: return "unknown";
	}
}

/* what the device decodes, checked from the IFD alone (the segments' first bytes for LZW and deflate's headers) */
int
check_ifd(const char *domain, const TiffFile &F, TiffIfd *I)
{
	if (I->bps != 8) {
		error(domain, "%d-bit samples not supported", I->bps);
		return -1;
	}
	if (I->sample_format != 1) {
		error(domain, "sample format %d not supported (unsigned integers only)", I->sample_format);
		return -1;
	}
	if (I->planar != 1) {
		error(domain, "PlanarConfiguration %d (separate planes) not supported", I->planar);
		return -1;
	}
	if (I->fill != 1) {
		error(domain, "FillOrder %d not supported", I->fill);
		return -1;
	}
	const int ph = I->photometric;
	if (ph < 0) {
		error(domain, "TIFF IFD without PhotometricInterpretation");
		return -1;
	}
	if (ph == 0 || ph == 1) {
		if (I->spp < 1 || I->spp > 2) {
			error(domain, "greyscale with %d samples not supported", I->spp);
			return -1;
		}
	}
	else if (ph == 2) {
		if (I->spp < 3 || I->spp > 4) {
			error(domain, "RGB with %d samples not supported", I->spp);
			return -1;
		}
	}
	else if (ph == 6 && I->compression != 7) {
		error(domain, "YCbCr without JPEG compression not supported");
		return -1;
	}
	else if (ph == 6 && I->spp != 3) {
		error(domain, "YCbCr with %d samples not supported", I->spp);
		return -1;
	}
	else if (ph != 6) {
		error(domain, "photometric %d (%s) not supported", ph, photometric_name(ph));
		return -1;
	}
	if (I->extra == 1) {
		error(domain, "associated alpha not supported (it would need vips_unpremultiply)");
		return -1;
	}
	if (I->extra != 0 && I->extra != 2) {
		error(domain, "ExtraSamples %d not supported", I->extra);
		return -1;
	}
	switch (I->compression) {
	case 1: I->comp = C_NONE; break;
	case 32773: I->comp = C_PACKBITS; break;
	case 5: I->comp = C_LZW; break;
	case 8: case 32946: I->comp = C_DEFLATE; break;
	case 6:
		error(domain, "old-style JPEG compression not supported");
		return -1;
	case 7:
		/* tiff2vips decodes JPEG tiles itself (tiff2vips.c:274-283, 2082-2177); strips go through libtiff's JPEG codec */
		if (!I->tiled) {
			error(domain, "JPEG-compressed strips not supported (libtiff's JPEG codec decodes them)");
			return -1;
		}
		if (ph == 2) {
			error(domain, "RGB-photometric JPEG not supported (libjpeg's JCS_RGB path is not on the device)");
			return -1;
		}
		I->comp = C_JPEG;
		break;
	default:
		error(domain, "compression %d not supported", I->compression);
		return -1;
	}
	if (I->predictor != 1 && I->predictor != 2) {
		error(domain, "predictor %d not supported", I->predictor);
		return -1;
	}
	/* libtiff's predictor belongs to the LZW and deflate codecs: none and PackBits ignore the tag */
	I->pred = I->predictor == 2 && (I->comp == C_LZW || I->comp == C_DEFLATE);
	I->invert = ph == 0; /* WhiteIsZero */
	if ((unsigned long long) I->w * I->h > (1ull << 28)) {
		error(domain, "%lld x %lld: frames over 2^28 pixels are not supported", I->w, I->h);
		return -1;
	}
	if (I->tiled) {
		if (I->tw < 1 || I->th < 1 || I->tw > 65536 || I->th > 65536) {
			error(domain, "bad tile size %lld x %lld", I->tw, I->th);
			return -1;
		}
		I->seg_w = (int) I->tw;
		I->seg_h = (int) I->th;
		I->across = (int) ((I->w + I->tw - 1) / I->tw);
		I->segs = I->across * (int) ((I->h + I->th - 1) / I->th);
	}
	else {
		const long long rps = std::max(1ll, std::min(I->rps, I->h));
		I->seg_w = (int) I->w;
		I->seg_h = (int) rps;
		I->across = 1;
		I->segs = (int) ((I->h + rps - 1) / rps);
	}
	if (I->offsets.size() < (size_t) I->segs || I->counts.size() < (size_t) I->segs) {
		error(domain, "%zu %s offsets and %zu byte counts for %d %s", I->offsets.size(), I->tiled ? "tile" : "strip", I->counts.size(), I->segs,
			I->tiled ? "tiles" : "strips");
		return -1;
	}
	if ((unsigned long long) I->seg_w * I->seg_h * I->spp > (1ull << 31)) {
		error(domain, "%s of %d x %d pixels not supported", I->tiled ? "tiles" : "strips", I->seg_w, I->seg_h);
		return -1;
	}
	for (int k = 0; k < I->segs; k++) {
		const unsigned long long o = I->offsets[k], c = I->counts[k];
		if (o > F.len || F.len - o < c) {
			error(domain, "%s %d (offset %llu, %llu bytes) lies outside the stream", I->tiled ? "tile" : "strip", k, o, c);
			return -1;
		}
		const unsigned char *s = F.d + o;
		if (I->comp == C_LZW && c >= 2 && s[0] == 0 && (s[1] & 1)) {
			error(domain, "old-style LZW not supported");
			return -1;
		}
		if (I->comp == C_DEFLATE && (c < 2 || (s[0] & 15) != 8 || (s[0] >> 4) > 7 || (s[0] * 256 + s[1]) % 31 || (s[1] & 0x20))) {
			error(domain, "%s %d: not a zlib stream libtiff inflates", I->tiled ? "tile" : "strip", k);
			return -1;
		}
	}
	return 0;
}

/* rtiff_header_equal (tiff2vips.c:3364) over the fields this subset reads */
bool
ifd_equal(const TiffIfd &a, const TiffIfd &b)
{
	if (a.w != b.w || a.h != b.h || a.spp != b.spp || a.bps != b.bps || a.photometric != b.photometric || a.sample_format != b.sample_format ||
		a.compression != b.compression || a.planar != b.planar || a.tiled != b.tiled || a.orientation != b.orientation)
		return false;
	if (a.tiled)
		return a.tw == b.tw && a.th == b.th;
	return a.seg_h == b.seg_h && a.segs == b.segs;
}

/* one stream's load: pages page .. page + n - 1, each at `subifd` */
struct TiffLoad {
	TiffFile F;
	std::vector<TiffIfd> ifd;
	size_t src_bytes = 0, dec_bytes = 0; /* staged and decoded bytes, each segment 16-aligned */
	std::vector<std::vector<unsigned char>> jpeg; /* the JPEG segments, page after page, as spliced_tile made them */
};

/* The stream libjpeg has seen once rtiff_decompress_jpeg_run's tables-only pass over JPEGTables is done (tiff2vips.c:
 * 2097-2109): the tables' DQT and DHT segments after the tile's SOI.  Nothing else in the tables outlives that pass:
 * get_soi resets the restart interval, the arithmetic conditioning and the JFIF / Adobe flags for the tile.
 */
int
spliced_tile(const char *domain, const TiffIfd &I, const unsigned char *tile, size_t n, std::vector<unsigned char> *out)
{
	out->clear();
	if (!I.tables) {
		out->assign(tile, tile + n);
		return 0;
	}
	const unsigned char *t = I.tables;
	const size_t tn = I.tables_len;
	if (tn < 4 || t[0] != 0xFF || t[1] != 0xD8 || n < 2) {
		error(domain, "bad JPEGTables");
		return -1;
	}
	out->reserve(n + tn);
	out->insert(out->end(), tile, tile + 2);
	for (size_t p = 2;;) {
		if (tn - p < 2 || t[p] != 0xFF) {
			error(domain, "bad JPEGTables");
			return -1;
		}
		const unsigned char m = t[p + 1];
		if (m == 0xD9)
			break;
		if (tn - p < 4) {
			error(domain, "bad JPEGTables");
			return -1;
		}
		const size_t l = ((size_t) t[p + 2] << 8) | t[p + 3];
		if (l < 2 || tn - p - 2 < l) {
			error(domain, "bad JPEGTables");
			return -1;
		}
		if (m == 0xDB || m == 0xC4)
			out->insert(out->end(), t + p, t + p + 2 + l);
		p += 2 + l;
	}
	out->insert(out->end(), tile + 2, tile + n);
	return 0;
}

/* the errors appended to the thread's buffer after its first `before` bytes, taken out of it: "reason" of "domain: reason" */
std::string
take_errors(size_t before)
{
	std::string e = vb200_error_buffer() + before;
	error_truncate(before);
	const size_t at = e.find(": ");
	e = e.substr(at == std::string::npos ? 0 : at + 2);
	return e.substr(0, e.find('\n'));
}

/* "frame i: reason" of the JPEG batch decoder -> i and the reason (i = -1: no frame named) */
int
jpeg_frame_error(const std::string &e, std::string *reason)
{
	int i = -1, used = 0;
	if (sscanf(e.c_str(), "frame %d: %n", &i, &used) == 1 && used > 0) {
		*reason = e.substr(used);
		return i;
	}
	*reason = e;
	return -1;
}

size_t
seg_src_len(const TiffIfd &I, int k)
{
	const size_t c = (size_t) I.counts[k];
	return I.comp == C_DEFLATE ? c - 2 : I.comp == C_NONE ? (size_t) I.seg_w * I.seg_h * I.spp : I.comp == C_JPEG ? 0 : c;
}

int
seg_rows(const TiffIfd &I, int k)
{
	if (I.tiled)
		return I.seg_h;
	return (int) std::min<long long>(I.seg_h, I.h - (long long) k * I.seg_h);
}

int
parse_tiff(const char *domain, const unsigned char *d, size_t len, int page, int n, int subifd, TiffLoad *L)
{
	if (parse_header(domain, d, len, &L->F))
		return -1;
	const int np = (int) L->F.pages.size();
	if (page < 0 || page >= np) {
		error(domain, "bad page number %d (the stream has %d)", page, np);
		return -1;
	}
	if (n == -1)
		n = np - page;
	if (n < 1 || page + n > np) {
		error(domain, "bad number of pages %d from page %d (the stream has %d)", n, page, np);
		return -1;
	}
	L->ifd.resize(n);
	for (int p = 0; p < n; p++) {
		if (select_ifd(domain, L->F, page + p, subifd, &L->ifd[p]) || check_ifd(domain, L->F, &L->ifd[p]))
			return -1;
		if (p > 0 && !ifd_equal(L->ifd[0], L->ifd[p])) {
			error(domain, "page %d's header differs from page %d's: the pages cannot load as one strip", page + p, page);
			return -1;
		}
		const TiffIfd &I = L->ifd[p];
		if (I.comp == C_JPEG) {
			/* every tile spliced, and its header checked by the JPEG decoder (no device call): it must decode to the tile */
			const size_t j0 = L->jpeg.size();
			L->jpeg.resize(j0 + I.segs);
			std::vector<const void *> ptr(I.segs);
			std::vector<size_t> len(I.segs);
			for (int k = 0; k < I.segs; k++) {
				if (spliced_tile(domain, I, d + I.offsets[k], (size_t) I.counts[k], &L->jpeg[j0 + k]))
					return -1;
				ptr[k] = L->jpeg[j0 + k].data();
				len[k] = L->jpeg[j0 + k].size();
			}
			const size_t before = strlen(vb200_error_buffer());
			StreamGeometry g;
			if (dev_jpeg_decode_batch(domain, ptr.data(), len.data(), I.segs, 1, nullptr, 0, 0, &g, nullptr)) {
				std::string reason;
				const int t = jpeg_frame_error(take_errors(before), &reason);
				if (t >= 0)
					error(domain, "tile %d: %s", t, reason.c_str());
				else
					error(domain, "JPEG tiles: %s", reason.c_str());
				return -1;
			}
			if (g.w != I.seg_w || g.h != I.seg_h || g.bands != I.spp) {
				error(domain, "JPEG tiles decode to %d x %d x %d, the IFD's tiles are %d x %d x %d", g.w, g.h, g.bands, I.seg_w, I.seg_h, I.spp);
				return -1;
			}
		}
		for (int k = 0; k < I.segs; k++) {
			const size_t dec = (size_t) seg_rows(I, k) * I.seg_w * I.spp;
			if (I.comp == C_NONE && I.counts[k] < dec) {
				error(domain, "%s %d holds %llu bytes, its rows need %zu", I.tiled ? "tile" : "strip", k, I.counts[k], dec);
				return -1;
			}
			L->src_bytes += align16(I.comp == C_NONE ? dec : seg_src_len(I, k));
			if (I.comp != C_NONE)
				L->dec_bytes += align16(dec);
		}
	}
	return 0;
}

StreamGeometry
load_geometry(const TiffLoad &L)
{
	const TiffIfd &I = L.ifd[0];
	return StreamGeometry{(int) I.w, (int) I.h, I.spp, (int) L.ifd.size()};
}

/* the records of one stream's segments, appended; src / dec are offsets from *src_at / *dec_at, which advance.  A JPEG
 * segment stages nothing (jpeg: its spliced stream, nullptr for the other kinds) and gets its dec slot from the caller */
void
stream_records(const TiffLoad &L, int frame, size_t *src_at, size_t *dec_at, std::vector<TiffSeg> &out,
	std::vector<const std::vector<unsigned char> *> &jpeg)
{
	size_t j = 0;
	for (size_t p = 0; p < L.ifd.size(); p++) {
		const TiffIfd &I = L.ifd[p];
		for (int k = 0; k < I.segs; k++) {
			TiffSeg S;
			memset(&S, 0, sizeof(S));
			const int rows = seg_rows(I, k);
			const int x0 = (k % I.across) * I.seg_w, y0 = (k / I.across) * I.seg_h;
			S.dec_len = (unsigned long long) rows * I.seg_w * I.spp;
			S.src = *src_at;
			S.src_len = I.comp == C_NONE ? S.dec_len : seg_src_len(I, k);
			*src_at += align16((size_t) S.src_len);
			if (I.comp == C_NONE)
				S.dec = S.src;
			else if (I.comp == C_JPEG)
				S.dec = 0; /* the caller's JPEG slots */
			else {
				S.dec = *dec_at;
				*dec_at += align16((size_t) S.dec_len);
			}
			S.frame = frame;
			S.row0 = (int) (p * I.h) + y0;
			S.col0 = x0;
			S.seg_w = I.seg_w;
			S.clip_w = (int) std::min<long long>(I.seg_w, I.w - x0);
			S.clip_h = (int) std::min<long long>(rows, I.h - y0);
			S.comp = (unsigned char) I.comp;
			S.pred = I.pred;
			S.invert = I.invert;
			S.spp = (unsigned char) I.spp;
			out.push_back(S);
			jpeg.push_back(I.comp == C_JPEG ? &L.jpeg[j++] : nullptr);
		}
	}
}

/* the bytes a segment stages: deflate's without the zlib header, uncompressed ones only as far as its rows go */
void
stage_segments(const TiffLoad &L, const TiffSeg *S, unsigned char *base)
{
	for (const TiffIfd &I : L.ifd)
		for (int k = 0; k < I.segs; k++, S++)
			memcpy(base + S->src, L.F.d + I.offsets[k] + (I.comp == C_DEFLATE ? 2 : 0), (size_t) S->src_len);
}

const char *
status_text(int st)
{
	if (st & ERR_CORRUPT)
		return "corrupt compressed data (libtiff refuses it)";
	if (st & ERR_MORE)
		return "the segment inflates to more bytes than its rows hold";
	if (st & ERR_CHECK)
		return "incorrect data check (the zlib trailer does not match)";
	return "not enough data for the segment's rows";
}

/* the host twin's placement: tif_predict.c's horAcc8 over each decoded row, then rtiff_greyscale_line / memcpy_line */
void
place_host(const TiffSeg &S, const unsigned char *dec, unsigned char *out, size_t out_bpl)
{
	const int spp = S.spp;
	std::vector<unsigned char> row((size_t) S.seg_w * spp);
	for (int r = 0; r < S.clip_h; r++) {
		memcpy(row.data(), dec + (size_t) r * row.size(), row.size());
		if (S.pred)
			for (size_t i = spp; i < row.size(); i++)
				row[i] = (unsigned char) (row[i] + row[i - spp]);
		unsigned char *dst = out + (size_t) (S.row0 + r) * out_bpl + (size_t) S.col0 * spp;
		for (int i = 0; i < S.clip_w * spp; i++)
			dst[i] = S.invert && i % spp == 0 ? (unsigned char) (255 - row[i]) : row[i];
	}
}

/* ------------------------------------------------------------------ thumbnail.c's pyramid level */

constexpr int kMaxLevels = 256; /* MAX_LEVELS */

/* vips_thumbnail_get_tiff_pyramid_subifd (thumbnail.c:324-383), vips_thumbnail_get_pyramid_page (:262-322) and
 * vips_thumbnail_find_pyrlevel (:519-541), as vips_thumbnail_open (:562-581) and vips_thumbnail_buffer_open's TIFF branch
 * (:1552-1576) run them: a subifd pyramid first, then a page pyramid; the level's geometry from geom(kind, i, &w, &h)
 * (false: that IFD does not open, so no pyramid).  *subifd = -1 and *page = 0 without a pyramid.
 */
void
pyramid_level(int in_w, int in_h, int n_pages, int n_subifds, const std::function<bool(bool, int, int *, int *)> &geom, int width, int height,
	int size, int *subifd, int *page)
{
	int lw[kMaxLevels], lh[kMaxLevels];
	auto detect = [&](bool sub, int count) {
		for (int i = 0; i < count; i++) {
			int w, h;
			if (!geom(sub, i, &w, &h))
				return 0;
			/* the main image is size 1, subifd 0 is half that; page i is 1 / 2^i */
			const int ew = sub ? in_w / (2 << i) : in_w / (1 << i), eh = sub ? in_h / (2 << i) : in_h / (1 << i);
			if (abs(w - ew) > 5 || w < 2 || abs(h - eh) > 5 || h < 2)
				return 0;
			lw[i] = w;
			lh[i] = h;
		}
		return count;
	};
	*subifd = -1;
	*page = 0;
	if (height <= 0) /* vips_thumbnail's height defaults to its width */
		height = width;
	bool sub = true;
	int levels = n_subifds >= 1 && n_subifds <= 28 ? detect(true, n_subifds) : 0;
	if (!levels) {
		sub = false;
		levels = n_pages >= 2 && n_pages <= 29 ? detect(false, n_pages) : 0;
	}
	if (!levels)
		return;
	int level = 0;
	for (int l = levels - 1; l >= 0; l--)
		if (thumbnail_common_shrink(lw[l], lh[l], width, height, size) > 1.0) { /* not >=, shrink can clip to 1.0 */
			level = l;
			break;
		}
	if (sub)
		*subifd = level;
	else
		*page = level;
}

} // namespace

bool
tiff_signature(const void *buf, size_t len)
{
	const unsigned char *d = (const unsigned char *) buf;
	if (!d || len < 4)
		return false;
	return (d[0] == 'I' && d[1] == 'I' && (d[2] == 42 || d[2] == 43) && d[3] == 0) || (d[0] == 'M' && d[1] == 'M' && d[2] == 0 && (d[3] == 42 || d[3] == 43));
}

/* the ICCProfile (tag 34675) of the IFD page / subifd select, and the first Orientation other than 1 among pages page ..
 * page + n_pages - 1 (n_pages -1: to the last; 1 when every page is upright)
 */
int
tiff_icc_profile(const char *domain, const unsigned char *d, size_t len, int page, int n_pages, int subifd, std::vector<unsigned char> *profile,
	int *orientation)
{
	profile->clear();
	TiffFile F;
	TiffIfd I;
	if (parse_header(domain, d, len, &F) || select_ifd(domain, F, page, subifd, &I))
		return -1;
	if (I.icc)
		profile->assign(I.icc, I.icc + I.icc_len);
	if (!orientation)
		return 0;
	*orientation = I.orientation;
	const int last = n_pages == -1 ? (int) F.pages.size() : std::min((int) F.pages.size(), page + std::max(1, n_pages));
	for (int p = page + 1; p < last && *orientation == 1; p++) {
		TiffIfd P;
		if (select_ifd(domain, F, p, subifd, &P))
			return -1;
		*orientation = P.orientation;
	}
	return 0;
}

/* the subifd / page vips_thumbnail_buffer loads (thumbnail.c:562-581, 1552-1576) */
int
tiff_thumbnail_level(const char *domain, const unsigned char *d, size_t len, int width, int height, int size, int *subifd, int *page)
{
	TiffFile F;
	TiffIfd I0;
	if (parse_header(domain, d, len, &F) || parse_ifd(domain, F, F.pages[0], &I0))
		return -1;
	/* a level that does not open ends the search quietly, as class->open failing does: its errors are not the call's */
	const size_t before = strlen(vb200_error_buffer());
	pyramid_level((int) I0.w, (int) I0.h, (int) F.pages.size(), (int) I0.subifds.size(),
		[&](bool sub, int i, int *w, int *h) {
			TiffIfd I;
			if (select_ifd(domain, F, sub ? 0 : i, sub ? i : -1, &I))
				return false;
			*w = (int) I.w;
			*h = (int) I.h;
			return true;
		},
		width, height, size, subifd, page);
	error_truncate(before);
	return 0;
}


/* Decode n TIFF streams (host memory) of one output geometry into out[n][h * pages][w][bands] on the device (out = nullptr:
 * only report the geometry).  IFDs are walked on the host workers; the streams go up in chunks bounded by device memory,
 * each one pinned block (segment records, kind lists, staged segments) copied to the device and decoded on s.  Every segment
 * of a chunk must decode clean before any is placed into out; the call returns when they are.
 */
int
dev_tiff_decode_batch(const char *domain, const void *const *bufs, const size_t *lens, int n, int page, int npages, int subifd, void *out,
	size_t out_bpl, size_t out_frame_stride, StreamGeometry *g, cudaStream_t s)
{
	std::vector<TiffLoad> ld(n);
	if (parse_streams(
			domain, "frame", n, [&](int i) { return parse_tiff(domain, (const unsigned char *) bufs[i], lens[i], page, npages, subifd, &ld[i]); },
			[&](int i) { return load_geometry(ld[i]); }, g))
		return -1;
	if (!out)
		return 0;
	if (check_out_strides(domain, *g, out_bpl, out_frame_stride))
		return -1;
	auto seg_count = [&](int i) {
		size_t c = 0;
		for (const TiffIfd &I : ld[i].ifd)
			c += I.segs;
		return c;
	};
	return decode_chunks(
		domain, "tiff", "frame", n, [&](int i) { return ld[i].src_bytes + ld[i].dec_bytes + seg_count(i) * (sizeof(TiffSeg) + 2 * sizeof(int)); },
		[&](int c0, int cn) {
			std::vector<TiffSeg> S;
			std::vector<const std::vector<unsigned char> *> J;
			std::vector<size_t> first(cn + 1);
			size_t src = 0, dec = 0;
			for (int i = 0; i < cn; i++) {
				first[i] = S.size();
				stream_records(ld[c0 + i], i, &src, &dec, S, J);
			}
			first[cn] = S.size();
			const int ns = (int) S.size();
			std::vector<int> list[5];
			for (int k = 0; k < ns; k++)
				list[S[k].comp].push_back(k);
			/* JPEG segments in runs of one tile geometry, each run's slots one stride apart: one JPEG batch per run */
			std::vector<int> &jk = list[C_JPEG];
			std::stable_sort(jk.begin(), jk.end(), [&](int a, int b) { return S[a].seg_w != S[b].seg_w ? S[a].seg_w < S[b].seg_w : S[a].dec_len < S[b].dec_len; });
			size_t jpg = 0;
			for (int k : jk) {
				S[k].dec = jpg;
				jpg += align16((size_t) S[k].dec_len);
			}
			/* the block: records, the kind lists and staged bytes; decoded bytes and JPEG-decoded tiles as scratch */
			const size_t off_list = align16(ns * sizeof(TiffSeg)), off_src = off_list + align16(ns * sizeof(int)), off_dec = off_src + src,
						 off_jpg = off_dec + dec;
			for (TiffSeg &r : S) {
				r.src += off_src;
				r.dec += r.comp == C_NONE ? off_src : r.comp == C_JPEG ? off_jpg : off_dec;
			}
			int li[4], at = 0;
			for (int c = 1; c < 4; c++) {
				li[c] = at;
				at += (int) list[c].size();
			}
			return decode_chunk(
				domain, "tiff", {off_src + src, dec + jpg, ns},
				[&](unsigned char *hst) {
					memcpy(hst, S.data(), ns * sizeof(TiffSeg));
					for (int c = 1; c < 4; c++)
						if (!list[c].empty())
							memcpy(hst + off_list + li[c] * sizeof(int), list[c].data(), list[c].size() * sizeof(int));
					parallel_for(cn, host_workers(), [&](int i) { stage_segments(ld[c0 + i], S.data() + first[i], hst); });
				},
				[&](unsigned char *dB, int *status) {
					const TiffSeg *dS = (const TiffSeg *) dB;
					const int *dL = (const int *) (dB + off_list);
					int launches = 0;
					const int nb = std::max(1, std::min(sm_count() * 64, 1 << 20));
					if (!list[C_DEFLATE].empty()) {
						const int m = (int) list[C_DEFLATE].size();
						tiff_inflate_kernel<<<std::min((m + kInflateWarps - 1) / kInflateWarps, nb), kInflateWarps * 32, 0, s>>>(dS, dL + li[C_DEFLATE], m,
							dB, status);
						launches++;
					}
					if (!list[C_LZW].empty()) {
						const int m = (int) list[C_LZW].size();
						tiff_lzw_kernel<<<std::min(m, nb), 32, 0, s>>>(dS, dL + li[C_LZW], m, dB, status);
						launches++;
					}
					if (!list[C_PACKBITS].empty()) {
						const int m = (int) list[C_PACKBITS].size();
						tiff_packbits_kernel<<<std::min((m + 127) / 128, nb), 128, 0, s>>>(dS, dL + li[C_PACKBITS], m, dB, status);
						launches++;
					}
					/* JPEG tiles: dev_jpeg_decode_batch at shrink 1 over each run of one geometry, into their slots (no new kernel);
					 * it counts its own launches */
					for (size_t a = 0; a < jk.size();) {
						size_t b = a + 1;
						while (b < jk.size() && S[jk[b]].seg_w == S[jk[a]].seg_w && S[jk[b]].dec_len == S[jk[a]].dec_len)
							b++;
						const TiffSeg &R = S[jk[a]];
						std::vector<const void *> ptr(b - a);
						std::vector<size_t> len(b - a);
						for (size_t q = a; q < b; q++) {
							ptr[q - a] = J[jk[q]]->data();
							len[q - a] = J[jk[q]]->size();
						}
						const size_t before = strlen(vb200_error_buffer());
						StreamGeometry jg;
						if (dev_jpeg_decode_batch(domain, ptr.data(), len.data(), (int) (b - a), 1, dB + R.dec, (size_t) R.seg_w * R.spp,
								align16((size_t) R.dec_len), &jg, s)) {
							std::string reason;
							const int t = jpeg_frame_error(take_errors(before), &reason);
							if (t >= 0) {
								const int k = jk[a + t];
								error(domain, "frame %d: tile %d: %s", c0 + S[k].frame, k - (int) first[S[k].frame], reason.c_str());
							}
							else
								error(domain, "JPEG tiles: %s", reason.c_str());
							count_launch(launches);
							return -1;
						}
						a = b;
					}
					return launches;
				},
				[&](int k, int st) { error(domain, "frame %d: segment %d: %s", c0 + S[k].frame, k - (int) first[S[k].frame], status_text(st)); },
				[&](unsigned char *dB) {
					tiff_place_kernel<<<std::min(ns, 1 << 20), kPlaceWarps * 32, 0, s>>>((const TiffSeg *) dB, ns, dB,
						(unsigned char *) out + (size_t) c0 * out_frame_stride, out_bpl, out_frame_stride);
					return 1;
				},
				s);
		}, s);
}

/* the same decode on the CPU through the same per-code and per-byte code: the test-suite's host twin */
int
host_tiff_decode(const char *domain, const void *buf, size_t len, int page, int npages, int subifd, unsigned char *out, size_t out_bpl, int *out_w,
	int *out_h, int *out_bands)
{
	TiffLoad L;
	if (parse_tiff(domain, (const unsigned char *) buf, len, page, npages, subifd, &L))
		return -1;
	const StreamGeometry g = load_geometry(L);
	if (out_w)
		*out_w = g.w;
	if (out_h)
		*out_h = g.rows();
	if (out_bands)
		*out_bands = g.bands;
	if (!out)
		return 0;
	std::vector<TiffSeg> S;
	std::vector<const std::vector<unsigned char> *> J;
	size_t src = 0, dec = 0;
	stream_records(L, 0, &src, &dec, S, J);
	for (TiffSeg &r : S)
		if (r.comp == C_JPEG) {
			r.dec = dec;
			dec += align16((size_t) r.dec_len);
		}
	std::vector<unsigned char> staged(src + 16), decoded(dec + 16);
	stage_segments(L, S.data(), staged.data());
	std::vector<unsigned> start(kLzwTable);
	std::vector<unsigned short> length(kLzwTable);
	for (size_t k = 0; k < S.size(); k++) {
		const TiffSeg &R = S[k];
		const unsigned char *in = staged.data() + R.src;
		unsigned char *o = R.comp == C_NONE ? staged.data() + R.dec : decoded.data() + R.dec;
		int st = 0;
		if (R.comp == C_DEFLATE) {
			size_t got = 0;
			Inflate z;
			const int op = inflate_host(in, R.src_len, o, R.dec_len, &got, &st, true, &z) ? OP_ERR : OP_DONE;
			unsigned trailer = 0;
			st = deflate_status(z, op, R.dec_len, &trailer);
			if (st == kCheckTrailer)
				st = adler32_host(o, R.dec_len) == trailer ? 0 : ERR_CHECK;
		}
		else if (R.comp == C_JPEG) {
			int w, h, b;
			const size_t before = strlen(vb200_error_buffer());
			if (host_jpeg_decode(domain, J[k]->data(), J[k]->size(), 1, o, (size_t) R.seg_w * R.spp, &w, &h, &b, 0, 0, nullptr)) {
				std::string reason = take_errors(before);
				error(domain, "tile %d: %s", (int) k, reason.c_str());
				return -1;
			}
		}
		else if (R.comp == C_LZW) {
			Lzw z;
			lzw_init(z, in, R.src_len, R.dec_len, start.data(), length.data());
			if (lzw_host(z, o))
				st = z.err;
		}
		else if (R.comp == C_PACKBITS)
			st = packbits_decode(in, R.src_len, o, R.dec_len);
		if (st) {
			error(domain, "segment %d: %s", (int) k, status_text(st));
			return -1;
		}
		place_host(R, o, out, out_bpl);
	}
	return 0;
}

int
debug_tiff_lzw(const char *domain, const unsigned char *data, size_t len, size_t want, unsigned char *out, size_t *out_len)
{
	std::vector<unsigned> start(kLzwTable);
	std::vector<unsigned short> length(kLzwTable);
	Lzw z;
	lzw_init(z, data, len, want, start.data(), length.data());
	const int rc = lzw_host(z, out);
	if (out_len)
		*out_len = (size_t) z.pos;
	if (rc)
		error(domain, "%s", status_text(z.err));
	return rc;
}

void
debug_pyramid_level(int in_w, int in_h, int n_pages, const int *page_w, const int *page_h, int n_subifds, const int *sub_w, const int *sub_h,
	int width, int height, int size, int *subifd, int *page)
{
	pyramid_level(in_w, in_h, n_pages, n_subifds,
		[&](bool sub, int i, int *w, int *h) {
			*w = sub ? sub_w[i] : page_w[i];
			*h = sub ? sub_h[i] : page_h[i];
			return true;
		},
		width, height, size, subifd, page);
}

} // namespace vb200

/* ------------------------------------------------------------------ C ABI */

using namespace vb200;

/* reference: rtiff_header_read (tiff2vips.c:3008-3360) on the IFD rtiff_set_page selects (:798-846); n-pages is the IFD
 * chain's length and n-subifds the SubIFDs count of the selected page's main IFD
 */
extern "C" int
vb200_tiff_geometry(const void *buf, size_t len, int page, int subifd, int *width, int *height, int *bands, int *pages, int *subifds)
{
	const char *domain = "tiff_geometry";
	TiffFile F;
	TiffIfd I, M;
	if (parse_header(domain, (const unsigned char *) buf, len, &F) || select_ifd(domain, F, page, -1, &M) ||
		(subifd >= 0 ? select_ifd(domain, F, page, subifd, &I) : (I = M, 0)))
		return -1;
	if (width)
		*width = (int) I.w;
	if (height)
		*height = (int) I.h;
	if (bands)
		*bands = I.spp;
	if (pages)
		*pages = (int) F.pages.size();
	if (subifds)
		*subifds = (int) M.subifds.size();
	return 0;
}

/* reference: vips_tiffload_buffer(buf, len, &out, "page", page, "n", n, "subifd", subifd, NULL), foreign/tiff2vips.c */
extern "C" int
vb200_tiff_decode_batch(const void *const *bufs, const size_t *lens, int n, int page, int n_pages, int subifd, void *out, int out_location,
	size_t out_bpl, size_t out_frame_stride, int *width, int *height, int *bands)
{
	DecodeRequest req{STREAM_TIFF, 1, page, n_pages};
	req.subifd = subifd;
	return decode_batch_abi("tiff_decode_batch", req, bufs, lens, n, out, out_location, out_bpl, out_frame_stride, width, height, bands);
}

extern "C" int
vb200_tiffload_buffer(const void *buf, size_t len, int page, int n, int subifd, VB200Image *out)
{
	DecodeRequest req{STREAM_TIFF, 1, page, n};
	req.subifd = subifd;
	return load_abi("tiffload_buffer", req, buf, len, out);
}

/* reference: rtiff_header_read's ICC profile (tiff2vips.c, TIFFTAG_ICCPROFILE) of the IFD page / subifd select */
extern "C" int
vb200_tiff_icc_profile(const void *buf, size_t len, int page, int subifd, void *out, size_t cap, size_t *profile_len)
{
	return profile_abi("tiff_icc_profile", out, cap, profile_len, [&](const char *domain, std::vector<unsigned char> *prof) {
		return tiff_icc_profile(domain, (const unsigned char *) buf, len, page, 1, subifd, prof, nullptr);
	});
}

/* reference: vips_thumbnail_open (thumbnail.c:562-581, 615-626) and vips_thumbnail_buffer_open's TIFF branch (:1552-1576) */
extern "C" int
vb200_thumbnail_tiff_level(const void *buf, size_t len, int width, int height, int size, int *subifd, int *page)
{
	const char *domain = "thumbnail_tiff_level";
	if (!subifd || !page) {
		error(domain, "null argument");
		return -1;
	}
	return tiff_thumbnail_level(domain, (const unsigned char *) buf, len, width, height, size, subifd, page);
}

extern "C" int
vb200_debug_thumbnail_pyramid_level(int in_w, int in_h, int n_pages, const int *page_w, const int *page_h, int n_subifds, const int *sub_w,
	const int *sub_h, int width, int height, int size, int *subifd, int *page)
{
	if (!subifd || !page || (n_pages > 0 && (!page_w || !page_h)) || (n_subifds > 0 && (!sub_w || !sub_h)) || n_pages > kMaxLevels ||
		n_subifds > kMaxLevels) {
		error("thumbnail_pyramid_level", "bad argument");
		return -1;
	}
	debug_pyramid_level(in_w, in_h, n_pages, page_w, page_h, n_subifds, sub_w, sub_h, width, height, size, subifd, page);
	return 0;
}

extern "C" int
vb200_debug_tiff_decode(const void *buf, size_t len, int page, int n, int subifd, void *out, size_t out_bpl, int *width, int *height, int *bands)
{
	return host_twin_abi("tiff_decode (host twin)",
		[&](const char *domain) { return host_tiff_decode(domain, buf, len, page, n, subifd, (unsigned char *) out, out_bpl, width, height, bands); });
}

/* one LZW segment (libtiff's new-style codes) through the decoder's LZW on the host: 0 and *out_len = want, or -1 (refused,
 * or fewer than want bytes: *out_len the bytes it got) */
extern "C" int
vb200_debug_tiff_lzw(const void *data, size_t len, size_t want, void *out, size_t *out_len)
{
	return host_twin_abi("tiff_lzw (host twin)",
		[&](const char *domain) { return debug_tiff_lzw(domain, (const unsigned char *) data, len, want, (unsigned char *) out, out_len); });
}
