/* png_encode.cu -- vips_pngsave_buffer's uchar frames on the device: scanlines built and deflated by CUDA kernels.
 *
 * What the reference does (foreign/spngsave.c, libspng over zlib, defaults): compression 6 (:700-705, :768), filter NONE
 * (:714-720, :769: every scanline is its filter byte 0 and the raw row), bit depth 8 for uchar frames (:608-613), IHDR from
 * the bands (:405-439), pHYs with rint(Xres * 1000) on both axes (:455-456 uses Xres twice), iCCP named "icc" compressed
 * at the image's level (:176-230, :447-448).  libspng feeds zlib one row at a time (:367); zlib's stream fed row by row
 * equals the stream fed in one shot (tests/test_png_save.py asserts it on its corpus), so the target is zlib's one-shot
 * deflate at window bits 15, memLevel 8.  The zlib stream (the IDAT payloads concatenated) is zlib 1.3's byte for byte at
 * levels 4-9 with Z_DEFAULT_STRATEGY or Z_FILTERED.  Not claimed: whole-file equality with libvips + libspng.  libspng's
 * IDAT split size, the order it writes iCCP and pHYs in, and the strategy it picks for unfiltered images cannot be read
 * from its source here; this encoder writes IHDR, iCCP, pHYs, IDATs of at most 8192 payload bytes and IEND, and uses
 * Z_DEFAULT_STRATEGY unless asked (libpng's choice without filtering, vipspng.c:1380-1384).
 *
 * The scanlines (scan_byte) follow the options that change them without quantisation:
 *   filter (:449-450, SPNG_FILTER_CHOICE; VipsForeignPngFilter, include/vips/foreign.h:744-748): 0 or NONE 0x08, SUB 0x10,
 *     UP 0x20, AVG 0x40 or PAETH 0x80 filters every scanline with that type (PNG 2nd edition 9.2) on the raw bytes: a is
 *     the byte bpp to the left, b the byte above in the same pass, c the byte left of b, each 0 where it does not exist,
 *     bpp the bands at 8 bits.  More than one flag (ALL = 0xF8) is libspng's adaptive choice: declined.
 *   interlace (:707-712, :439: IHDR interlace 1): Adam7 (8.2), passes (x0, y0, dx, dy) = (0,0,8,8) (4,0,8,8) (0,4,4,8) (2,0,4,4)
 *     (0,2,2,4) (1,0,2,2) (0,1,1,2), each ceil((w - x0) / dx) x ceil((h - y0) / dy); an empty pass has no scanlines.
 *   bitdepth 1 / 2 / 4 on one band (:400-441, :606-653): grey without a palette, each sample p >> (8 - bitdepth) packed
 *     MSB first by vips_foreign_save_spng_pack (:295-324), whose tail takes the last 8 / bitdepth samples and shifts them
 *     left by 8 - (leftover << (bitdepth - 1)): right at depths 1 and 2, 0 at depth 4, so an odd-width row at depth 4 ends
 *     in v[w-2] << 4 | v[w-1].  Only NONE, not interlaced, is built at these depths.
 * Every scanline byte is a function of at most four raw bytes, so one thread builds each.
 *
 * Why an exact deflate can be parallel.  Levels 4-9 run zlib's deflate_slow, which inserts every position into the hash
 * chains; the 3-byte hash (15 bits, shift 5) is a pure function of the data, so the candidates of a position -- earlier
 * positions with its hash, newest first, the first at most MAX_DIST = 32506 back and the later ones less -- do not depend
 * on the parse.  The lazy parse
 * needs two answers per position: the longest match under max_chain, and under max_chain >> 2 (used when prev_length >=
 * good_match); the shorter walk is a prefix of the longer one.  A search that starts at best_len = prev_length returns
 * the candidate a search from 2 returns whenever that one is longer than prev_length, and otherwise leads to the same
 * decision, so the parse reads answers computed ahead of it.
 *
 * Device pipeline per chunk of frames (all frames of a batch share one geometry, so one scanline count N):
 *   png_scan_kernel         frames (any bpl / frame stride) -> the scanlines in pool memory, one thread per byte
 *   png_adler_kernel        one CTA per frame: per-thread sums, combined in order
 *   deflate_last_kernel     per 32 KiB tile: the last position of every hash (shared-memory atomicMax)
 *   deflate_chain_kernel    one warp per tile: the previous position of the same hash for every position, 32 positions
 *                           per step (__match_any_sync), seeded by the tile before (MAX_DIST < 32 KiB)
 *   deflate_match_kernel    one thread per position: the chain walk, (length, distance) at both budgets
 *   deflate_parse_kernel    one warp per frame: zlib's lazy state machine, records prefetched 32 at a time; emits
 *                           symbols and cuts blocks where zlib's symbol buffer fills (16383 at memLevel 8)
 *   deflate_block_kernel    one warp per block: histograms, trees.c's build_tree / gen_bitlen / gen_codes, the
 *                           stored / fixed / dynamic choice of _tr_flush_block
 *   deflate_offsets_kernel  one thread per frame: block bit offsets (stored blocks byte-aligned), the zlib header and
 *                           trailer, the PNG length
 *   deflate_emit_kernel     one warp per block: header and symbols OR-ed into the stream at prefix-sum bit offsets
 *   png_frame_kernel        one warp per IDAT chunk: payload, length and CRC-32; the header chunks and IEND; each stream
 *                           at its own offset, so that streams for the host land packed and go back in one copy
 * The per-position, per-symbol and per-block code is __host__ __device__: vb200_debug_png_encode runs it on the CPU.
 */
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <exception>
#include <memory>
#include <string>
#include <vector>

#include "../../include/vb200.h"
#include "png_common.cuh"
#include "vb200_internal.h"

#define VB_HD __host__ __device__ __forceinline__

namespace vb200 {

namespace {

constexpr unsigned kWSize = 32768, kMaxDist = kWSize - 262, kTooFar = 4096, kMaxSyms = 16383, kIdat = 8192;
constexpr int kHashMask = 0x7fff, kLCodes = 286, kDCodes = 30, kBlCodes = 19, kHeap = 2 * kLCodes + 1;

struct Level {
	int good, lazy, nice, chain;
};

/* deflate.c configuration_table, levels 4-9 (deflate_slow) */
VB_HD Level
level_params(int level)
{
	switch (level) {
	case 4: return {4, 4, 16, 16};
	case 5: return {8, 16, 32, 32};
	case 6: return {8, 16, 128, 128};
	case 7: return {8, 32, 128, 256};
	case 8: return {32, 128, 258, 1024};
	default: return {32, 258, 258, 4096};
	}
}

VB_HD int
ilog2(unsigned x)
{
#ifdef __CUDA_ARCH__
	return 31 - __clz(x);
#else
	return 31 - __builtin_clz(x);
#endif
}

VB_HD unsigned
hash3(const unsigned char *d, size_t p)
{
	return (((unsigned) d[p] << 10) ^ ((unsigned) d[p + 1] << 5) ^ d[p + 2]) & kHashMask;
}

/* 4 bytes at any offset (the buffers are padded by 8 bytes) */
VB_HD unsigned
ld32(const unsigned char *d, size_t i)
{
#ifdef __CUDA_ARCH__
	const unsigned *w = (const unsigned *) (d + (i & ~(size_t) 3));
	return __funnelshift_r(__ldg(w), __ldg(w + 1), 8 * (unsigned) (i & 3));
#else
	unsigned v;
	memcpy(&v, d + i, 4);
	return v;
#endif
}

/* The byte zlib's match loop sees at frame position q.  Past the input it compares what its window still holds: zeros
 * (WIN_INIT) while the window has never slid, and the data 32 KiB back once it has -- which it has at the last positions
 * exactly when p >= wsize + MAX_DIST (fill_window slides there once the input is exhausted). */
VB_HD unsigned
window_byte(const unsigned char *d, size_t n, size_t q, bool slid)
{
	return q < n ? d[q] : slid ? d[q - kWSize] : 0;
}

/* longest_match's length for candidate m at position p: 0 unless the first two bytes agree (the third agrees through the
 * hash), else the first index in 3..258 that differs, or 258 */
VB_HD int
match_len(const unsigned char *d, size_t n, size_t p, size_t m)
{
	if (d[m] != d[p] || d[m + 1] != d[p + 1])
		return 0;
	if (p + 258 <= n) {
		for (int k = 3; k < 258; k += 4) {
			const unsigned x = ld32(d, p + k) ^ ld32(d, m + k);
			if (x) {
#ifdef __CUDA_ARCH__
				const int b = (__ffs(x) - 1) >> 3;
#else
				const int b = __builtin_ctz(x) >> 3;
#endif
				return k + b < 258 ? k + b : 258;
			}
		}
		return 258;
	}
	const bool slid = p >= kWSize + kMaxDist;
	for (int k = 3; k < 258; k++)
		if (window_byte(d, n, p + k, slid) != window_byte(d, n, m + k, slid))
			return k;
	return 258;
}

/* the two answers of position p: .x under max_chain, .y under max_chain >> 2; each (length clipped to the input left)
 * | distance << 16, 0 when nothing of length 3 or more */
VB_HD uint2
match_records(const unsigned char *d, const unsigned *prev, size_t n, size_t p, const Level &L)
{
	uint2 r = make_uint2(0, 0);
	if (p + 3 > n)
		return r;
	size_t m = prev[p];
	if (m == 0 || p - m > kMaxDist)
		return r;
	const int left = (int) std::min<size_t>(n - p, 258), nice = L.nice < left ? L.nice : left, qa = L.chain >> 2;
	int best = 2, count = 0;
	unsigned bestd = 0;
	for (;;) {
		const int len = match_len(d, n, p, m);
		count++;
		bool stop = false;
		if (len > best) {
			best = len;
			bestd = (unsigned) (p - m);
			stop = len >= nice;
		}
		if (count == qa)
			r.y = best >= 3 ? (unsigned) (best < left ? best : left) | bestd << 16 : 0;
		if (stop)
			break;
		/* deflate_slow takes the first candidate up to MAX_DIST back; longest_match walks on only while cur_match >
		 * strstart - MAX_DIST, so a later candidate exactly MAX_DIST back ends the walk */
		m = prev[m];
		if (m == 0 || p - m >= kMaxDist || count >= L.chain)
			break;
	}
	r.x = best >= 3 ? (unsigned) (best < left ? best : left) | bestd << 16 : 0;
	if (count < qa)
		r.y = r.x;
	return r;
}

struct BlockRec {
	unsigned sym0, nsym, byte0, nbytes, last, stored_ok;
	unsigned long long bit0; /* the block's first bit in the zlib stream (deflate_offsets_kernel) */
};

/* deflate_slow (zlib 1.3) over precomputed match records.  Src: rec(p) -> uint2, byte(p); Out: sym(v) with v = dist << 8
 * | (length - 3), or the literal with dist 0; block(rec).  fill_window is emulated by its window base B: it slides when
 * it is called (lookahead < MIN_LOOKAHEAD) with strstart >= wsize + MAX_DIST, and a stored block needs its start still
 * inside the window (block_start >= 0). */
#pragma nv_exec_check_disable
template <class Out>
VB_HD void
block_out(Out &out, const BlockRec &b)
{
	out.block(b);
}

#pragma nv_exec_check_disable
template <class Src, class Out>
VB_HD void
deflate_parse(Src &src, Out &out, unsigned n, const Level &L, bool filtered)
{
	unsigned strstart = 0, block_start = 0, B = 0, nsym = 0, sym0 = 0, match_start = 0, prev_match = 0;
	int match_length = 2, prev_length = 2;
	bool match_available = false;
	auto flush = [&](unsigned last) {
		block_out(out, BlockRec{sym0, nsym - sym0, block_start, strstart - block_start, last, block_start >= B, 0});
		block_start = strstart;
		sym0 = nsym;
	};
	for (;;) {
		unsigned lookahead = std::min(n, B + 2 * kWSize) - strstart;
		if (lookahead < 262) {
			if (strstart >= B + kWSize + kMaxDist)
				B += kWSize;
			lookahead = std::min(n, B + 2 * kWSize) - strstart;
			if (lookahead == 0)
				break;
		}
		prev_length = match_length;
		prev_match = match_start;
		match_length = 2;
		if (lookahead >= 3 && prev_length < L.lazy) {
			const uint2 r = src.rec(strstart);
			const unsigned v = prev_length >= L.good ? r.y : r.x;
			const int len = (int) (v & 0xffff);
			if (len > prev_length) {
				match_length = len;
				match_start = strstart - (v >> 16);
				if (len <= 5 && (filtered || (len == 3 && (v >> 16) > kTooFar)))
					match_length = 2;
			}
		}
		if (prev_length >= 3 && match_length <= prev_length) {
			out.sym((strstart - 1 - prev_match) << 8 | (unsigned) (prev_length - 3));
			nsym++;
			strstart += prev_length - 1;
			match_available = false;
			match_length = 2;
			if (nsym - sym0 == kMaxSyms)
				flush(0);
		}
		else if (match_available) {
			out.sym(src.byte(strstart - 1));
			nsym++;
			if (nsym - sym0 == kMaxSyms)
				flush(0);
			strstart++;
		}
		else {
			match_available = true;
			strstart++;
		}
	}
	if (match_available) {
		out.sym(src.byte(strstart - 1));
		nsym++;
	}
	flush(1);
}

/* ------------------------------------------------------------------ trees.c, restated */

VB_HD int
length_code(unsigned lc)
{
	return lc < 8 ? (int) lc : lc == 255 ? 28 : 4 * (ilog2(lc) - 2) + 4 + (int) ((lc >> (ilog2(lc) - 2)) & 3);
}
VB_HD int
length_extra(int code)
{
	return code < 8 || code == 28 ? 0 : (code - 4) / 4;
}
VB_HD unsigned
length_base(int code)
{
	return code < 8 ? (unsigned) code : code == 28 ? 255u : (unsigned) (4 + (code & 3)) << ((code - 4) / 4);
}
VB_HD int
dist_code(unsigned d)
{
	return d < 4 ? (int) d : 2 * (ilog2(d) - 1) + 2 + (int) ((d >> (ilog2(d) - 1)) & 1);
}
VB_HD int
dist_extra(int code)
{
	return code < 4 ? 0 : (code - 2) / 2;
}
VB_HD unsigned
dist_base(int code)
{
	return code < 4 ? (unsigned) code : (unsigned) (2 + (code & 1)) << ((code - 2) / 2);
}
VB_HD int
bl_extra(int n)
{
	return n == 16 ? 2 : n == 17 ? 3 : n == 18 ? 7 : 0;
}
VB_HD int
bl_order(int i)
{
	const unsigned char o[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
	return o[i];
}
VB_HD int
static_llen(int n)
{
	return n < 144 ? 8 : n < 256 ? 9 : n < 280 ? 7 : 8;
}

VB_HD unsigned
bi_reverse(unsigned code, int len)
{
	unsigned r = 0;
	do {
		r |= code & 1;
		code >>= 1;
		r <<= 1;
	} while (--len > 0);
	return r >> 1;
}

/* a block's codes: kind 0 stored, 1 fixed, 2 dynamic; bits = tree header + symbols + END_BLOCK (not the 3-bit block
 * header, nor a stored block's alignment and contents) */
struct DeflatePlan {
	int kind, lcodes, dcodes, blcodes;
	unsigned bits;
	unsigned short lcode[288], dcode[32], blcode[kBlCodes];
	unsigned char llen[288], dlen[32], bllen[kBlCodes];
};

/* build_tree's scratch: one per warp in shared memory on the device */
struct TreeWork {
	unsigned freq[kHeap];
	unsigned short dad[kHeap], len[kHeap];
	unsigned char depth[kHeap];
	short heap[kHeap];
	int heap_len, heap_max;
	unsigned short bl_count[16];
	unsigned long long opt_len, static_len;
	unsigned blfreq[kBlCodes];
};

VB_HD bool
smaller(const TreeWork &w, int n, int m)
{
	return w.freq[n] < w.freq[m] || (w.freq[n] == w.freq[m] && w.depth[n] <= w.depth[m]);
}

VB_HD void
pqdownheap(TreeWork &w, int k)
{
	const int v = w.heap[k];
	int j = k << 1;
	while (j <= w.heap_len) {
		if (j < w.heap_len && smaller(w, w.heap[j + 1], w.heap[j]))
			j++;
		if (smaller(w, v, w.heap[j]))
			break;
		w.heap[k] = w.heap[j];
		k = j;
		j <<= 1;
	}
	w.heap[k] = (short) v;
}

/* build_tree + gen_bitlen + gen_codes for a tree of `elems` leaves whose counts are in w.freq[0, elems): lengths to
 * len_out, codes to code_out; which: 0 literal/length (static lengths, extra bits from 257), 1 distance, 2 bit lengths */
VB_HD int
build_tree(TreeWork &w, int elems, int which, unsigned char *len_out, unsigned short *code_out)
{
	const int max_length = which == 2 ? 7 : 15;
	auto xbits = [&](int n) { return which == 0 ? (n >= 257 ? length_extra(n - 257) : 0) : which == 1 ? dist_extra(n) : bl_extra(n); };
	auto slen = [&](int n) { return which == 0 ? static_llen(n) : 5; };
	int max_code = -1;
	w.heap_len = 0;
	w.heap_max = kHeap;
	for (int n = 0; n < elems; n++) {
		if (w.freq[n]) {
			w.heap[++w.heap_len] = (short) (max_code = n);
			w.depth[n] = 0;
		}
		else
			w.len[n] = 0;
	}
	while (w.heap_len < 2) {
		const int node = w.heap[++w.heap_len] = (short) (max_code < 2 ? ++max_code : 0);
		w.freq[node] = 1;
		w.depth[node] = 0;
		w.opt_len--;
		if (which != 2)
			w.static_len -= slen(node);
	}
	for (int n = w.heap_len / 2; n >= 1; n--)
		pqdownheap(w, n);
	int node = elems;
	do {
		const int n = w.heap[1];
		w.heap[1] = w.heap[w.heap_len--];
		pqdownheap(w, 1);
		const int m = w.heap[1];
		w.heap[--w.heap_max] = (short) n;
		w.heap[--w.heap_max] = (short) m;
		w.freq[node] = w.freq[n] + w.freq[m];
		w.depth[node] = (unsigned char) ((w.depth[n] >= w.depth[m] ? w.depth[n] : w.depth[m]) + 1);
		w.dad[n] = w.dad[m] = (unsigned short) node;
		w.heap[1] = (short) node++;
		pqdownheap(w, 1);
	} while (w.heap_len >= 2);
	w.heap[--w.heap_max] = w.heap[1];

	/* gen_bitlen */
	for (int b = 0; b <= 15; b++)
		w.bl_count[b] = 0;
	w.len[w.heap[w.heap_max]] = 0;
	int overflow = 0, h;
	for (h = w.heap_max + 1; h < kHeap; h++) {
		const int n = w.heap[h];
		int bits = w.len[w.dad[n]] + 1;
		if (bits > max_length)
			bits = max_length, overflow++;
		w.len[n] = (unsigned short) bits;
		if (n > max_code)
			continue;
		w.bl_count[bits]++;
		const int xb = xbits(n);
		const unsigned f = w.freq[n];
		w.opt_len += (unsigned long long) f * (unsigned) (bits + xb);
		if (which != 2)
			w.static_len += (unsigned long long) f * (unsigned) (slen(n) + xb);
	}
	if (overflow) {
		do {
			int bits = max_length - 1;
			while (w.bl_count[bits] == 0)
				bits--;
			w.bl_count[bits]--;
			w.bl_count[bits + 1] += 2;
			w.bl_count[max_length]--;
			overflow -= 2;
		} while (overflow > 0);
		for (int bits = max_length; bits != 0; bits--) {
			int n = w.bl_count[bits];
			while (n != 0) {
				const int m = w.heap[--h];
				if (m > max_code)
					continue;
				if (w.len[m] != (unsigned) bits) {
					w.opt_len += ((unsigned long long) bits - w.len[m]) * w.freq[m];
					w.len[m] = (unsigned short) bits;
				}
				n--;
			}
		}
	}
	/* gen_codes */
	unsigned short next[16];
	unsigned code = 0;
	for (int bits = 1; bits <= 15; bits++) {
		code = (code + w.bl_count[bits - 1]) << 1;
		next[bits] = (unsigned short) code;
	}
	for (int n = 0; n <= max_code; n++) {
		len_out[n] = (unsigned char) w.len[n];
		code_out[n] = w.len[n] ? (unsigned short) bi_reverse(next[w.len[n]]++, w.len[n]) : 0;
	}
	return max_code;
}

/* scan_tree (the bit-length counts, into w.blfreq) and send_tree (emit != nullptr) share the run walk */
template <class Emit>
VB_HD void
walk_tree(const unsigned char *len, int max_code, Emit emit)
{
	int prevlen = -1, nextlen = len[0], count = 0, max_count = 7, min_count = 4;
	if (nextlen == 0)
		max_count = 138, min_count = 3;
	for (int n = 0; n <= max_code; n++) {
		const int curlen = nextlen;
		nextlen = n + 1 <= max_code ? len[n + 1] : 0xffff;
		if (++count < max_count && curlen == nextlen)
			continue;
		else if (count < min_count)
			emit(curlen, 0, count);
		else if (curlen != 0) {
			if (curlen != prevlen) {
				emit(curlen, 0, 1);
				count--;
			}
			emit(16, count - 3, 1);
		}
		else if (count <= 10)
			emit(17, count - 3, 1);
		else
			emit(18, count - 11, 1);
		count = 0;
		prevlen = curlen;
		if (nextlen == 0)
			max_count = 138, min_count = 3;
		else if (curlen == nextlen)
			max_count = 6, min_count = 3;
		else
			max_count = 7, min_count = 4;
	}
}

/* an LSB-first bit sink ORing into little-endian 32-bit words, which must start zeroed */
struct WordSink {
	unsigned *W;
	unsigned long long o;
	VB_HD void orw(unsigned long long i, unsigned v)
	{
#ifdef __CUDA_ARCH__
		if (v)
			atomicOr(&W[i], v);
#else
		W[i] |= v;
#endif
	}
	VB_HD void put(unsigned v, int nb)
	{
		if (!nb)
			return;
		const int sh = (int) (o & 31);
		orw(o >> 5, v << sh);
		if (sh + nb > 32)
			orw((o >> 5) + 1, v >> (32 - sh));
		o += nb;
	}
};

/* send_all_trees */
template <class Sink>
VB_HD void
send_trees(const DeflatePlan &P, Sink &s)
{
	s.put(P.lcodes - 257, 5);
	s.put(P.dcodes - 1, 5);
	s.put(P.blcodes - 4, 4);
	for (int r = 0; r < P.blcodes; r++)
		s.put(P.bllen[bl_order(r)], 3);
	auto emit = [&](int sym, int extra, int times) {
		for (int t = 0; t < times; t++) {
			s.put(P.blcode[sym], P.bllen[sym]);
			if (sym >= 16)
				s.put((unsigned) extra, bl_extra(sym));
		}
	};
	walk_tree(P.llen, P.lcodes - 1, emit);
	walk_tree(P.dlen, P.dcodes - 1, emit);
}

struct CountSink {
	unsigned long long o = 0;
	VB_HD void put(unsigned, int nb) { o += nb; }
};

/* one symbol's bits: the literal / length code and its extra bits (*v1, *n1), the distance code and its extra (*v2, *n2) */
VB_HD void
sym_bits(const DeflatePlan &P, unsigned sym, unsigned *v1, int *n1, unsigned *v2, int *n2)
{
	const unsigned dist = sym >> 8, lc = sym & 255;
	if (!dist) {
		*v1 = P.lcode[lc];
		*n1 = P.llen[lc];
		*n2 = 0;
		*v2 = 0;
		return;
	}
	const int c = length_code(lc), le = length_extra(c);
	*v1 = P.lcode[257 + c] | (lc - length_base(c)) << P.llen[257 + c];
	*n1 = P.llen[257 + c] + le;
	const unsigned d = dist - 1;
	const int dc = dist_code(d), de = dist_extra(dc);
	*v2 = P.dcode[dc] | (d - dist_base(dc)) << P.dlen[dc];
	*n2 = P.dlen[dc] + de;
}

/* _tr_flush_block's choice for a block with symbol counts lf[286] / df[30] (lf[256] = 1 for END_BLOCK) */
VB_HD void
plan_block(const unsigned *lf, const unsigned *df, const BlockRec &b, TreeWork &w, DeflatePlan &P)
{
	w.opt_len = w.static_len = 0;
	for (int i = 0; i < kLCodes; i++)
		w.freq[i] = lf[i];
	for (int i = kLCodes; i < 288; i++)
		P.llen[i] = 0, P.lcode[i] = 0;
	const int lmax = build_tree(w, kLCodes, 0, P.llen, P.lcode);
	for (int i = lmax + 1; i < kLCodes; i++)
		P.llen[i] = 0, P.lcode[i] = 0;
	for (int i = 0; i < kDCodes; i++)
		w.freq[i] = df[i];
	const int dmax = build_tree(w, kDCodes, 1, P.dlen, P.dcode);
	for (int i = dmax + 1; i < 32; i++)
		P.dlen[i] = 0, P.dcode[i] = 0;
	/* build_bl_tree */
	for (int i = 0; i < kBlCodes; i++)
		w.blfreq[i] = 0;
	auto count = [&](int sym, int, int times) { w.blfreq[sym] += times; };
	walk_tree(P.llen, lmax, count);
	walk_tree(P.dlen, dmax, count);
	for (int i = 0; i < kBlCodes; i++)
		w.freq[i] = w.blfreq[i];
	const int blmax = build_tree(w, kBlCodes, 2, P.bllen, P.blcode);
	for (int i = blmax + 1; i < kBlCodes; i++)
		P.bllen[i] = 0, P.blcode[i] = 0;
	int max_blindex;
	for (max_blindex = kBlCodes - 1; max_blindex >= 3; max_blindex--)
		if (P.bllen[bl_order(max_blindex)] != 0)
			break;
	w.opt_len += 3 * ((unsigned long long) max_blindex + 1) + 5 + 5 + 4;
	unsigned long long opt_lenb = (w.opt_len + 3 + 7) >> 3;
	const unsigned long long static_lenb = (w.static_len + 3 + 7) >> 3;
	if (static_lenb <= opt_lenb)
		opt_lenb = static_lenb;
	P.lcodes = lmax + 1;
	P.dcodes = dmax + 1;
	P.blcodes = max_blindex + 1;
	if ((unsigned long long) b.nbytes + 4 <= opt_lenb && b.stored_ok) {
		P.kind = 0;
		P.bits = 0;
		return;
	}
	if (static_lenb == opt_lenb) {
		P.kind = 1;
		/* static_ltree / static_dtree */
		unsigned short bl_count[16] = {0};
		for (int n = 0; n < 288; n++)
			bl_count[static_llen(n)]++;
		unsigned short next[16];
		unsigned code = 0;
		for (int bits = 1; bits <= 15; bits++) {
			code = (code + bl_count[bits - 1]) << 1;
			next[bits] = (unsigned short) code;
		}
		for (int n = 0; n < 288; n++) {
			P.llen[n] = (unsigned char) static_llen(n);
			P.lcode[n] = (unsigned short) bi_reverse(next[P.llen[n]]++, P.llen[n]);
		}
		for (int n = 0; n < kDCodes; n++) {
			P.dlen[n] = 5;
			P.dcode[n] = (unsigned short) bi_reverse(n, 5);
		}
	}
	else
		P.kind = 2;
	unsigned long long bits = 0;
	if (P.kind == 2) {
		CountSink c;
		send_trees(P, c);
		bits = c.o;
	}
	for (int n = 0; n < kLCodes; n++)
		if (lf[n])
			bits += (unsigned long long) lf[n] * (P.llen[n] + (n >= 257 ? length_extra(n - 257) : 0));
	for (int n = 0; n < kDCodes; n++)
		if (df[n])
			bits += (unsigned long long) df[n] * (P.dlen[n] + dist_extra(n));
	P.bits = (unsigned) bits;
}

VB_HD void
count_symbol(unsigned sym, unsigned *lf, unsigned *df)
{
	if (!(sym >> 8))
		lf[sym & 255]++;
	else {
		lf[257 + length_code(sym & 255)]++;
		df[dist_code((sym >> 8) - 1)]++;
	}
}

/* the bit after the block, from its first bit (a stored block: 3 header bits, byte alignment, LEN, NLEN, the bytes) */
VB_HD unsigned long long
block_end(const BlockRec &b, const DeflatePlan &P, unsigned long long o)
{
	if (P.kind == 0)
		return ((o + 3 + 7) & ~7ull) + 32 + 8ull * b.nbytes;
	return o + 3 + P.bits;
}

/* the block's header; a stored block's also aligns and writes LEN / NLEN (its bytes follow) */
VB_HD void
emit_block_head(const BlockRec &b, const DeflatePlan &P, WordSink &s)
{
	s.put((unsigned) (P.kind == 0 ? 0 : P.kind == 1 ? 2 : 4) + b.last, 3);
	if (P.kind == 2)
		send_trees(P, s);
	if (P.kind == 0) {
		s.o = (s.o + 7) & ~7ull;
		s.put(b.nbytes & 0xffff, 16);
		s.put(~b.nbytes & 0xffff, 16);
	}
}

VB_HD unsigned
zlib_header(int level)
{
	const unsigned flags = level < 6 ? 1 : level == 6 ? 2 : 3;
	unsigned h = (0x78u << 8) | (flags << 6);
	return h + 31 - (h % 31);
}

constexpr unsigned kAdlerBase = 65521;

VB_HD unsigned
crc_update(unsigned crc, const unsigned char *p, size_t n, const unsigned *tab)
{
	for (size_t i = 0; i < n; i++)
		crc = tab[(crc ^ p[i]) & 255] ^ (crc >> 8);
	return crc;
}

/* ------------------------------------------------------------------ device kernels */

/* a non-empty pass: its first column and row, their steps, its size, row bytes and first scanline byte */
struct ScanPass {
	unsigned x0, y0, dx, dy, w, h;
	size_t rb, off;
};

/* the scanlines of a frame: what png_scan_kernel alone reads */
struct ScanGeom {
	int bands, depth, filter; /* depth: bits per sample; filter: PNG filter type 0-4 */
	int npass;		  /* non-empty passes: 1 without interlace, up to 7 with */
	ScanPass pass[7];
	size_t n; /* scanline bytes: every pass's rows of rb + 1 */
};

struct EncGeom {
	int w, h, bands, level, filtered;
	size_t n;		/* scanline bytes of a frame (ScanGeom::n) */
	size_t scan_stride; /* per frame in the scanline pool (n + 8, aligned) */
	int tiles;		/* 32 KiB tiles per frame */
	int maxblk;		/* block records per frame */
	size_t zcap;		/* zlib stream words' bytes per frame */
	size_t prefix;		/* signature .. pHYs */
	int maxchunks;		/* IDAT chunks per frame at most */
};

struct FrameOut {
	unsigned long long zlen, len;
	unsigned adler, nblk;
};

/* byte k of row y of pass P as spngsave hands it to libspng: the pass's samples at 8 bits, or packed MSB first at 1 / 2 / 4
 * bits with vips_foreign_save_spng_pack's tail rule (see the top of the file).  rd(row, byte): a byte of the frame. */
#pragma nv_exec_check_disable
template <class Rd>
VB_HD unsigned
raw_byte(const ScanGeom &g, const ScanPass &P, size_t y, size_t k, Rd &rd)
{
	const size_t row = P.y0 + y * P.dy;
	if (g.depth == 8)
		return rd(row, P.dx == 1 ? k : (P.x0 + k / g.bands * P.dx) * g.bands + k % g.bands);
	const int per = 8 / g.depth;
	const long long e = (long long) std::min<size_t>((k + 1) * per, P.w);
	unsigned u = 0;
	for (int j = per; j >= 1; j--)
		u = u << g.depth | (e - j >= 0 ? rd(row, P.x0 + (size_t) (e - j) * P.dx) >> (8 - g.depth) : 0);
	const size_t left = P.w - k * per;
	return left >= (size_t) per ? u : (u << (8 - ((int) left << (g.depth - 1)))) & 255;
}

/* scanline byte i of a frame: the filter type at the start of each row, then the row's bytes filtered */
#pragma nv_exec_check_disable
template <class Rd>
VB_HD unsigned
scan_byte(const ScanGeom &g, size_t i, Rd &rd)
{
	int p = 0;
	while (p + 1 < g.npass && i >= g.pass[p + 1].off)
		p++;
	const ScanPass &P = g.pass[p];
	const size_t q = i - P.off, y = q / (P.rb + 1), x = q - y * (P.rb + 1);
	if (x == 0)
		return (unsigned) g.filter;
	const size_t k = x - 1, bpp = g.depth == 8 ? g.bands : 1;
	const unsigned raw = raw_byte(g, P, y, k, rd);
	if (g.filter == 0)
		return raw;
	const unsigned a = g.filter != 2 && k >= bpp ? raw_byte(g, P, y, k - bpp, rd) : 0;
	const unsigned b = g.filter != 1 && y ? raw_byte(g, P, y - 1, k, rd) : 0;
	const unsigned c = g.filter == 4 && y && k >= bpp ? raw_byte(g, P, y - 1, k - bpp, rd) : 0;
	const unsigned pred = g.filter == 1 ? a : g.filter == 2 ? b : g.filter == 3 ? (a + b) >> 1 : (unsigned) paeth((int) a, (int) b, (int) c);
	return (raw - pred) & 255;
}

__global__ void
png_scan_kernel(const unsigned char *__restrict__ src, size_t bpl, size_t frame_stride, ScanGeom sg, size_t scan_stride, unsigned char *scan)
{
	const size_t f = blockIdx.y;
	const unsigned char *s = src + f * frame_stride;
	unsigned char *dst = scan + f * scan_stride;
	auto rd = [&](size_t row, size_t col) -> unsigned { return s[row * bpl + col]; };
	for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < scan_stride; i += (size_t) gridDim.x * blockDim.x)
		dst[i] = i < sg.n ? (unsigned char) scan_byte(sg, i, rd) : 0;
}

__global__ void __launch_bounds__(256)
png_adler_kernel(const unsigned char *__restrict__ scan, EncGeom g, FrameOut *fo)
{
	const unsigned char *d = scan + (size_t) blockIdx.x * g.scan_stride;
	const size_t per = (g.n + 255) / 256, s0 = std::min(g.n, per * threadIdx.x), s1 = std::min(g.n, s0 + per);
	unsigned long long a = 0, b = 0;
	for (size_t i = s0; i < s1; i++) {
		a += d[i];
		b += (unsigned long long) (s1 - i) * d[i] % kAdlerBase;
		if ((i & 4095) == 4095)
			a %= kAdlerBase, b %= kAdlerBase;
	}
	__shared__ unsigned long long A[256], Bs[256];
	A[threadIdx.x] = a % kAdlerBase;
	Bs[threadIdx.x] = (b + (unsigned long long) ((g.n - s1) % kAdlerBase) * (a % kAdlerBase)) % kAdlerBase;
	__syncthreads();
	if (threadIdx.x == 0) {
		unsigned long long s1s = 1, s2s = g.n % kAdlerBase;
		for (int t = 0; t < 256; t++)
			s1s = (s1s + A[t]) % kAdlerBase, s2s = (s2s + Bs[t]) % kAdlerBase;
		fo[blockIdx.x].adler = (unsigned) (s2s << 16 | s1s);
	}
}

/* last position + 1 of every hash in a tile (0: none) */
__global__ void __launch_bounds__(1024)
deflate_last_kernel(const unsigned char *__restrict__ scan, EncGeom g, unsigned short *last)
{
	extern __shared__ unsigned tab[];
	const size_t f = blockIdx.y, t0 = (size_t) blockIdx.x * kWSize;
	const unsigned char *d = scan + f * g.scan_stride;
	for (int i = threadIdx.x; i < (int) kWSize; i += blockDim.x)
		tab[i] = 0;
	__syncthreads();
	for (int i = threadIdx.x; i < (int) kWSize; i += blockDim.x)
		if (t0 + i + 3 <= g.n)
			atomicMax(&tab[hash3(d, t0 + i)], (unsigned) i + 1);
	__syncthreads();
	unsigned short *o = last + (f * g.tiles + blockIdx.x) * kWSize;
	for (int i = threadIdx.x; i < (int) kWSize; i += blockDim.x)
		o[i] = (unsigned short) tab[i];
}

/* prev[p]: the last position before p with p's hash, 0 when none within reach.  The head table holds positions relative
 * to the start of the previous tile (0: none; that tile's first position is more than MAX_DIST from every position here). */
__global__ void __launch_bounds__(32)
deflate_chain_kernel(const unsigned char *__restrict__ scan, EncGeom g, const unsigned short *__restrict__ last, unsigned *prev)
{
	extern __shared__ unsigned short head[];
	const size_t f = blockIdx.y, t0 = (size_t) blockIdx.x * kWSize, base = t0 - kWSize;
	const unsigned char *d = scan + f * g.scan_stride;
	const unsigned lane = threadIdx.x;
	const unsigned short *seed = blockIdx.x ? last + (f * g.tiles + blockIdx.x - 1) * kWSize : nullptr;
	for (int i = lane; i < (int) kWSize; i += 32) {
		const unsigned v = seed ? seed[i] : 0;
		head[i] = (unsigned short) (v > 1 ? v - 1 : 0);
	}
	__syncwarp();
	unsigned *pv = prev + f * g.n;
	const size_t end = std::min(g.n, t0 + kWSize);
	for (size_t s = t0; s < end; s += 32) {
		const size_t p = s + lane;
		const bool ok = p + 3 <= g.n;
		const unsigned h = ok ? hash3(d, p) : 0x10000u + lane;
		const unsigned peers = __match_any_sync(0xffffffffu, h);
		const unsigned lower = peers & ((1u << lane) - 1);
		if (ok) {
			unsigned v;
			if (lower)
				v = (unsigned) (s + 31 - __clz(lower));
			else {
				const unsigned r = head[h];
				v = r ? (unsigned) (base + r) : 0;
			}
			pv[p] = v;
		}
		__syncwarp();
		if (ok && lane == 31 - __clz(peers))
			head[h] = (unsigned short) (p - base);
		__syncwarp();
	}
}

__global__ void __launch_bounds__(128)
deflate_match_kernel(const unsigned char *__restrict__ scan, EncGeom g, const unsigned *__restrict__ prev, uint2 *rec)
{
	const size_t f = blockIdx.y;
	const Level L = level_params(g.level);
	for (size_t p = (size_t) blockIdx.x * blockDim.x + threadIdx.x; p < g.n; p += (size_t) gridDim.x * blockDim.x)
		rec[f * g.n + p] = match_records(scan + f * g.scan_stride, prev + f * g.n, g.n, p, L);
}

/* the parse's inputs, 32 records and 128 bytes per coalesced load, shared by shuffle (every lane runs the parse) */
struct WarpSrc {
	const uint2 *rec;
	const unsigned char *d;
	size_t n;
	unsigned lane, rbase = 0, bbase = 0;
	bool rset = false, bset = false;
	uint2 r;
	unsigned b;
	__device__ uint2 rec_at(unsigned p)
	{
		if (!rset || p - rbase >= 32) {
			rset = true;
			rbase = p;
			r = p + lane < n ? rec[p + lane] : make_uint2(0, 0);
		}
		return make_uint2(__shfl_sync(0xffffffffu, r.x, p - rbase), __shfl_sync(0xffffffffu, r.y, p - rbase));
	}
	__device__ unsigned byte_at(unsigned p)
	{
		if (!bset || p - bbase >= 128) {
			bset = true;
			bbase = p;
			b = 0;
			for (int k = 3; k >= 0; k--)
				b = b << 8 | (p + 4 * lane + k < n ? d[p + 4 * lane + k] : 0);
		}
		const unsigned o = p - bbase;
		return (__shfl_sync(0xffffffffu, b, o >> 2) >> (8 * (o & 3))) & 255;
	}
};
struct WarpSrcAdapter {
	WarpSrc *s;
	__device__ uint2 rec(unsigned p) { return s->rec_at(p); }
	__device__ unsigned byte(unsigned p) { return s->byte_at(p); }
};
struct DevOut {
	unsigned *sym;
	BlockRec *blk;
	unsigned ns = 0, nb = 0;
	bool lead;
	__device__ void sym_(unsigned v)
	{
		if (lead)
			sym[ns] = v;
		ns++;
	}
};
struct DevOutAdapter {
	DevOut *o;
	__device__ void sym(unsigned v) { o->sym_(v); }
	__device__ void block(const BlockRec &b)
	{
		if (o->lead)
			o->blk[o->nb] = b;
		o->nb++;
	}
};

constexpr int kParseWarps = 4;

__global__ void __launch_bounds__(kParseWarps * 32)
deflate_parse_kernel(const unsigned char *__restrict__ scan, EncGeom g, int nframes, const uint2 *__restrict__ rec, unsigned *sym, BlockRec *blk,
	FrameOut *fo)
{
	const int f = blockIdx.x * kParseWarps + threadIdx.x / 32;
	if (f >= nframes)
		return;
	WarpSrc src;
	src.rec = rec + (size_t) f * g.n;
	src.d = scan + (size_t) f * g.scan_stride;
	src.n = g.n;
	src.lane = threadIdx.x & 31;
	DevOut out;
	out.sym = sym + (size_t) f * g.n;
	out.blk = blk + (size_t) f * g.maxblk;
	out.lead = src.lane == 0;
	WarpSrcAdapter sa{&src};
	DevOutAdapter oa{&out};
	deflate_parse(sa, oa, (unsigned) g.n, level_params(g.level), g.filtered != 0);
	if (out.lead)
		fo[f].nblk = out.nb;
}

constexpr int kBlockWarps = 4;

__global__ void __launch_bounds__(kBlockWarps * 32)
deflate_block_kernel(EncGeom g, const unsigned *__restrict__ sym, BlockRec *blk, DeflatePlan *plans, const FrameOut *__restrict__ fo)
{
	__shared__ TreeWork work[kBlockWarps];
	__shared__ unsigned lf[kBlockWarps][kLCodes], df[kBlockWarps][kDCodes];
	const int wi = threadIdx.x / 32, lane = threadIdx.x & 31;
	const size_t f = blockIdx.y;
	const int b = blockIdx.x * kBlockWarps + wi;
	if (b >= (int) fo[f].nblk)
		return;
	for (int i = lane; i < kLCodes; i += 32)
		lf[wi][i] = i == 256;
	for (int i = lane; i < kDCodes; i += 32)
		df[wi][i] = 0;
	__syncwarp();
	const BlockRec B = blk[f * g.maxblk + b];
	const unsigned *s = sym + f * g.n + B.sym0;
	for (unsigned i = lane; i < B.nsym; i += 32) {
		const unsigned v = s[i];
		if (!(v >> 8))
			atomicAdd(&lf[wi][v & 255], 1u);
		else {
			atomicAdd(&lf[wi][257 + length_code(v & 255)], 1u);
			atomicAdd(&df[wi][dist_code((v >> 8) - 1)], 1u);
		}
	}
	__syncwarp();
	if (lane == 0)
		plan_block(lf[wi], df[wi], B, work[wi], plans[f * g.maxblk + b]);
}

/* block bit offsets, the zlib header and Adler-32, the PNG length */
__global__ void
deflate_offsets_kernel(EncGeom g, int nframes, BlockRec *blk, const DeflatePlan *__restrict__ plans, unsigned *zs, FrameOut *fo)
{
	const int f = blockIdx.x * blockDim.x + threadIdx.x;
	if (f >= nframes)
		return;
	unsigned long long o = 16;
	for (unsigned b = 0; b < fo[f].nblk; b++) {
		BlockRec &B = blk[(size_t) f * g.maxblk + b];
		B.bit0 = o;
		o = block_end(B, plans[(size_t) f * g.maxblk + b], o);
	}
	const unsigned long long z = (o + 7) / 8 + 4;
	unsigned char *zb = (unsigned char *) (zs + (size_t) f * (g.zcap / 4));
	const unsigned hdr = zlib_header(g.level), ad = fo[f].adler;
	zb[0] = (unsigned char) (hdr >> 8);
	zb[1] = (unsigned char) hdr;
	for (int k = 0; k < 4; k++)
		zb[z - 4 + k] = (unsigned char) (ad >> (24 - 8 * k));
	const unsigned long long chunks = (z + kIdat - 1) / kIdat, len = g.prefix + z + 12 * chunks + 12;
	fo[f].zlen = z;
	fo[f].len = len;
}

__global__ void __launch_bounds__(kBlockWarps * 32)
deflate_emit_kernel(EncGeom g, const unsigned char *__restrict__ scan, const unsigned *__restrict__ sym, const BlockRec *__restrict__ blk,
	const DeflatePlan *__restrict__ plans, const FrameOut *__restrict__ fo, unsigned *zs)
{
	const int wi = threadIdx.x / 32, lane = threadIdx.x & 31;
	const size_t f = blockIdx.y;
	const int b = blockIdx.x * kBlockWarps + wi;
	if (b >= (int) fo[f].nblk)
		return;
	const BlockRec B = blk[f * g.maxblk + b];
	const DeflatePlan &P = plans[f * g.maxblk + b];
	unsigned *W = zs + f * (g.zcap / 4);
	WordSink head{W, B.bit0};
	if (lane == 0)
		emit_block_head(B, P, head);
	/* every lane advances its own copy of the header sink to the same offset */
	WordSink cnt{W, B.bit0};
	{
		CountSink c;
		c.o = B.bit0 + 3;
		if (P.kind == 2)
			send_trees(P, c);
		if (P.kind == 0)
			c.o = ((c.o + 7) & ~7ull) + 32;
		cnt.o = c.o;
	}
	const unsigned char *d = scan + f * g.scan_stride;
	if (P.kind == 0) {
		/* the bytes, byte-aligned from cnt.o */
		const unsigned long long byte0 = cnt.o >> 3;
		const unsigned long long w0 = byte0 >> 2, w1 = (byte0 + B.nbytes + 3) >> 2;
		for (unsigned long long wd = w0 + lane; wd < w1; wd += 32) {
			unsigned v = 0;
			for (int k = 0; k < 4; k++) {
				const unsigned long long at = wd * 4 + k;
				if (at >= byte0 && at < byte0 + B.nbytes)
					v |= (unsigned) d[B.byte0 + (at - byte0)] << (8 * k);
			}
			if (v)
				atomicOr(&W[wd], v);
		}
		return;
	}
	const unsigned *s = sym + f * g.n + B.sym0;
	unsigned long long o = cnt.o;
	for (unsigned i0 = 0; i0 < B.nsym; i0 += 32) {
		const unsigned i = i0 + lane;
		unsigned v1 = 0, v2 = 0;
		int n1 = 0, n2 = 0;
		if (i < B.nsym)
			sym_bits(P, s[i], &v1, &n1, &v2, &n2);
		unsigned x = n1 + n2;
		for (int k = 1; k < 32; k <<= 1) {
			const unsigned y = __shfl_up_sync(0xffffffffu, x, k);
			if (lane >= k)
				x += y;
		}
		const unsigned total = __shfl_sync(0xffffffffu, x, 31);
		WordSink w{W, o + x - (n1 + n2)};
		w.put(v1, n1);
		w.put(v2, n2);
		o += total;
	}
	if (lane == 0) {
		WordSink w{W, o};
		w.put(P.lcode[256], P.llen[256]);
	}
}

/* one warp per IDAT chunk of a frame: length, "IDAT", payload, CRC; chunk 0 also writes the header chunks, the last one
 * IEND.  Frame f's stream starts at out + at[f]. */
__global__ void __launch_bounds__(256)
png_frame_kernel(EncGeom g, const unsigned char *__restrict__ prefix, const unsigned *__restrict__ zs, const FrameOut *__restrict__ fo,
	const unsigned long long *__restrict__ at_out, unsigned char *out)
{
	__shared__ unsigned tab[256];
	for (unsigned v = threadIdx.x; v < 256; v += blockDim.x) {
		unsigned c = v;
		for (int k = 0; k < 8; k++)
			c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1;
		tab[v] = c;
	}
	__syncthreads();
	const size_t f = blockIdx.y;
	const int k = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
	const unsigned long long z = fo[f].zlen, chunks = (z + kIdat - 1) / kIdat;
	if ((unsigned long long) k >= chunks)
		return;
	unsigned char *o = out + at_out[f];
	const unsigned char *zb = (const unsigned char *) (zs + f * (g.zcap / 4));
	if (k == 0)
		for (size_t i = lane; i < g.prefix; i += 32)
			o[i] = prefix[i];
	const unsigned long long at = (unsigned long long) k * kIdat, len = std::min<unsigned long long>(kIdat, z - at);
	unsigned char *c = o + g.prefix + (size_t) k * (kIdat + 12);
	for (unsigned long long i = lane; i < len; i += 32)
		c[8 + i] = zb[at + i];
	if (lane == 0) {
		const unsigned char hd[8] = {(unsigned char) (len >> 24), (unsigned char) (len >> 16), (unsigned char) (len >> 8), (unsigned char) len, 'I', 'D',
			'A', 'T'};
		for (int i = 0; i < 8; i++)
			c[i] = hd[i];
		const unsigned crc = ~crc_update(crc_update(~0u, hd + 4, 4, tab), zb + at, len, tab);
		for (int i = 0; i < 4; i++)
			c[8 + len + i] = (unsigned char) (crc >> (24 - 8 * i));
		if ((unsigned long long) k == chunks - 1) {
			const unsigned char iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
			for (int i = 0; i < 12; i++)
				c[12 + len + i] = iend[i];
		}
	}
}

/* ------------------------------------------------------------------ host side */

struct CrcTable {
	unsigned t[256];
	CrcTable()
	{
		for (unsigned n = 0; n < 256; n++) {
			unsigned c = n;
			for (int k = 0; k < 8; k++)
				c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1;
			t[n] = c;
		}
	}
};
const CrcTable g_crc;

void
put_be32(std::vector<unsigned char> &v, unsigned x)
{
	for (int i = 0; i < 4; i++)
		v.push_back((unsigned char) (x >> (24 - 8 * i)));
}

void
put_chunk(std::vector<unsigned char> &v, const char *type, const std::vector<unsigned char> &data)
{
	put_be32(v, (unsigned) data.size());
	const size_t at = v.size();
	v.insert(v.end(), type, type + 4);
	v.insert(v.end(), data.begin(), data.end());
	put_be32(v, ~crc_update(~0u, v.data() + at, 4 + data.size(), g_crc.t));
}

/* host chains, records, parse, plans and emission: the same functions the kernels run */
struct HostSrc {
	const std::vector<uint2> *rec;
	const unsigned char *d;
	uint2 rec_(unsigned p) const { return (*rec)[p]; }
};
struct HostSrcAdapter {
	const HostSrc *s;
	uint2 rec(unsigned p) { return s->rec_(p); }
	unsigned byte(unsigned p) { return s->d[p]; }
};
struct HostOut {
	std::vector<unsigned> sym;
	std::vector<BlockRec> blk;
	void block(const BlockRec &b) { blk.push_back(b); }
};
struct HostOutAdapter {
	HostOut *o;
	void sym(unsigned v) { o->sym.push_back(v); }
	void block(const BlockRec &b) { o->block(b); }
};

/* the zlib stream of d[0, n) (n + 8 bytes readable) */
void
host_deflate(const unsigned char *d, size_t n, int level, int filtered, std::vector<unsigned char> &z)
{
	const Level L = level_params(level);
	std::vector<unsigned> prev(n + 1, 0), head(kHashMask + 1, 0);
	for (size_t p = 0; p + 3 <= n; p++) {
		const unsigned h = hash3(d, p);
		prev[p] = head[h];
		head[h] = (unsigned) p;
	}
	std::vector<uint2> rec(n);
	for (size_t p = 0; p < n; p++)
		rec[p] = match_records(d, prev.data(), n, p, L);
	HostSrc hs{&rec, d};
	HostSrcAdapter sa{&hs};
	HostOut ho;
	HostOutAdapter oa{&ho};
	deflate_parse(sa, oa, (unsigned) n, L, filtered != 0);
	std::vector<DeflatePlan> plans(ho.blk.size());
	std::unique_ptr<TreeWork> work(new TreeWork);
	unsigned long long o = 16;
	for (size_t b = 0; b < ho.blk.size(); b++) {
		unsigned lf[kLCodes] = {0}, df[kDCodes] = {0};
		lf[256] = 1;
		for (unsigned i = 0; i < ho.blk[b].nsym; i++)
			count_symbol(ho.sym[ho.blk[b].sym0 + i], lf, df);
		plan_block(lf, df, ho.blk[b], *work, plans[b]);
		ho.blk[b].bit0 = o;
		o = block_end(ho.blk[b], plans[b], o);
	}
	const size_t zlen = (o + 7) / 8 + 4;
	std::vector<unsigned> W((zlen + 7) / 4 + 2, 0);
	for (size_t b = 0; b < ho.blk.size(); b++) {
		const BlockRec &B = ho.blk[b];
		const DeflatePlan &P = plans[b];
		WordSink s{W.data(), B.bit0};
		emit_block_head(B, P, s);
		if (P.kind == 0) {
			for (unsigned i = 0; i < B.nbytes; i++)
				s.put(d[B.byte0 + i], 8);
			continue;
		}
		for (unsigned i = 0; i < B.nsym; i++) {
			unsigned v1, v2;
			int n1, n2;
			sym_bits(P, ho.sym[B.sym0 + i], &v1, &n1, &v2, &n2);
			s.put(v1, n1);
			s.put(v2, n2);
		}
		s.put(P.lcode[256], P.llen[256]);
	}
	z.assign((const unsigned char *) W.data(), (const unsigned char *) W.data() + zlen);
	const unsigned hdr = zlib_header(level);
	z[0] = (unsigned char) (hdr >> 8);
	z[1] = (unsigned char) hdr;
	unsigned long long a = 1, b2 = 0;
	for (size_t i = 0; i < n; i++) {
		a = (a + d[i]) % kAdlerBase;
		b2 = (b2 + a) % kAdlerBase;
	}
	const unsigned ad = (unsigned) (b2 << 16 | a);
	for (int k = 0; k < 4; k++)
		z[zlen - 4 + k] = (unsigned char) (ad >> (24 - 8 * k));
}

/* the options and geometry checks every entry point shares: 0, or -1 with the reason */
int
check_save(const char *domain, int w, int h, int bands, const VB200PngSaveOptions &o)
{
	if (o.compression < 4 || o.compression > 9) {
		error(domain, "compression %d is not built on the device (levels 4-9; 1-3 are zlib's deflate_fast, whose hash chains depend on "
			"the parse, and 0 writes stored blocks sized by zlib's buffers)", o.compression);
		return -1;
	}
	if (o.strategy != 0 && o.strategy != 1) {
		error(domain, "strategy %d is not built (0: Z_DEFAULT_STRATEGY, 1: Z_FILTERED)", o.strategy);
		return -1;
	}
	if (bands < 1 || bands > 4) {
		error(domain, "%d bands: PNG save takes 1 to 4 bands", bands);
		return -1;
	}
	if (w < 1 || h < 1 || (size_t) w * h > ((size_t) 1 << 28)) {
		error(domain, "a %d x %d frame: PNG save takes 1 to 2^28 pixels", w, h);
		return -1;
	}
	if (!(o.xres >= 0) || !std::isfinite(o.xres) || std::rint(o.xres * 1000.0) > 4294967295.0) {
		error(domain, "bad xres %g", o.xres);
		return -1;
	}
	if (o.filter & ~0xF8) {
		error(domain, "filter 0x%x: unknown flag bits (NONE 0x08, SUB 0x10, UP 0x20, AVG 0x40, PAETH 0x80)", (unsigned) o.filter);
		return -1;
	}
	if (o.filter & (o.filter - 1)) {
		error(domain, "filter 0x%x: more than one flag is libspng's adaptive filter choice, which is not built (one flag or 0)",
			(unsigned) o.filter);
		return -1;
	}
	const int depth = o.bitdepth ? o.bitdepth : 8;
	if (depth == 16) {
		error(domain, "bitdepth 16 is not built (uchar frames only, bit depth 1, 2, 4 or 8)");
		return -1;
	}
	if (depth != 1 && depth != 2 && depth != 4 && depth != 8) {
		error(domain, "bitdepth %d: PNG save takes bit depth 1, 2, 4 or 8", depth);
		return -1;
	}
	if (depth < 8 && bands == 2) {
		error(domain, "bitdepth %d with 2 bands: PNG has no low-bit grey + alpha", depth);
		return -1;
	}
	if (depth < 8 && bands > 2) {
		error(domain, "bitdepth %d with %d bands: spngsave writes a palette, and quantisation is not built", depth, bands);
		return -1;
	}
	if (depth < 8 && ((o.filter && o.filter != 0x08) || o.interlace)) {
		error(domain, "bitdepth %d with a filter other than NONE or with interlace is not built (libspng's sub-byte filter unit and "
			"pass packing cannot be checked)", depth);
		return -1;
	}
	return 0;
}

/* the PNG filter type of a checked filter flag */
int
filter_type(int flags)
{
	return flags == 0x10 ? 1 : flags == 0x20 ? 2 : flags == 0x40 ? 3 : flags == 0x80 ? 4 : 0;
}

/* signature, IHDR, iCCP (profile non-empty), pHYs */
std::vector<unsigned char>
png_prefix(int w, int h, int bands, const VB200PngSaveOptions &o, const unsigned char *profile, size_t profile_len)
{
	static const unsigned char sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
	std::vector<unsigned char> v(sig, sig + 8), c;
	put_be32(c, (unsigned) w);
	put_be32(c, (unsigned) h);
	const unsigned char ct[5] = {0, 0, 4, 2, 6};
	c.insert(c.end(), {(unsigned char) (o.bitdepth ? o.bitdepth : 8), ct[bands], 0, 0, (unsigned char) (o.interlace ? 1 : 0)});
	put_chunk(v, "IHDR", c);
	if (profile && profile_len) {
		c.assign({'i', 'c', 'c', 0, 0});
		std::vector<unsigned char> pad(profile, profile + profile_len), z;
		pad.resize(profile_len + 8, 0);
		host_deflate(pad.data(), profile_len, o.compression, o.strategy, z);
		c.insert(c.end(), z.begin(), z.end());
		put_chunk(v, "iCCP", c);
	}
	c.clear();
	const unsigned ppm = (unsigned) std::rint(o.xres * 1000.0);
	put_be32(c, ppm);
	put_be32(c, ppm);
	c.push_back(1);
	put_chunk(v, "pHYs", c);
	return v;
}

ScanGeom
scan_geom(int w, int h, int bands, const VB200PngSaveOptions &o)
{
	ScanGeom g;
	g.bands = bands;
	g.depth = o.bitdepth ? o.bitdepth : 8;
	g.filter = filter_type(o.filter);
	static const unsigned adam7[7][4] = {{0, 0, 8, 8}, {4, 0, 8, 8}, {0, 4, 4, 8}, {2, 0, 4, 4}, {0, 2, 2, 4}, {1, 0, 2, 2}, {0, 1, 1, 2}};
	static const unsigned whole[1][4] = {{0, 0, 1, 1}};
	const unsigned(*steps)[4] = o.interlace ? adam7 : whole;
	g.npass = 0;
	g.n = 0;
	for (int p = 0; p < (o.interlace ? 7 : 1); p++) {
		ScanPass P;
		P.x0 = steps[p][0], P.y0 = steps[p][1], P.dx = steps[p][2], P.dy = steps[p][3];
		P.w = (unsigned) w > P.x0 ? (w - P.x0 + P.dx - 1) / P.dx : 0;
		P.h = (unsigned) h > P.y0 ? (h - P.y0 + P.dy - 1) / P.dy : 0;
		if (!P.w || !P.h)
			continue;
		P.rb = ((size_t) P.w * bands * g.depth + 7) / 8;
		P.off = g.n;
		g.n += P.h * (P.rb + 1);
		g.pass[g.npass++] = P;
	}
	return g;
}

EncGeom
enc_geom(int w, int h, int bands, const VB200PngSaveOptions &o, size_t prefix)
{
	EncGeom g;
	g.w = w, g.h = h, g.bands = bands, g.level = o.compression, g.filtered = o.strategy == 1;
	g.n = scan_geom(w, h, bands, o).n;
	g.scan_stride = (g.n + 8 + 15) & ~(size_t) 15;
	g.tiles = (int) ((g.n + kWSize - 1) / kWSize);
	g.maxblk = (int) (g.n / kMaxSyms + 2);
	/* fixed codes cost at most 9 bits a byte; every block adds at most its header */
	g.zcap = ((g.n + g.n / 8 + 400 * (size_t) g.maxblk + 64) + 15) & ~(size_t) 15;
	g.prefix = prefix;
	g.maxchunks = (int) ((g.zcap + kIdat - 1) / kIdat);
	return g;
}

size_t
align256(size_t v)
{
	return (v + 255) & ~(size_t) 255;
}

/* the kernels of cn frames at src (device memory): scanlines, deflate, then place and png_frame_kernel */
int
png_chunk(const char *domain, const EncGeom &g, const ScanGeom &sg, const std::vector<unsigned char> &prefix, const unsigned char *src, size_t bpl,
	size_t frame_stride, int cn, const EncodePlace &place, cudaStream_t s)
{
	VB200_CUDA(domain, cudaFuncSetAttribute(deflate_last_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWSize * 4));
	VB200_CUDA(domain, cudaFuncSetAttribute(deflate_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWSize * 2));
	unsigned char *dev = nullptr;
	const size_t off_prev = align256(g.scan_stride * cn), off_last = off_prev + align256(4 * g.n * cn),
				 off_rec = off_last + align256((size_t) 2 * kWSize * g.tiles * cn), off_sym = off_rec + align256(8 * g.n * cn),
				 off_blk = off_sym + align256(4 * g.n * cn), off_plan = off_blk + align256(sizeof(BlockRec) * g.maxblk * cn),
				 off_zs = off_plan + align256(sizeof(DeflatePlan) * g.maxblk * cn), off_fo = off_zs + align256(g.zcap * cn),
				 off_at = off_fo + align256(sizeof(FrameOut) * cn), off_pre = off_at + align256(sizeof(unsigned long long) * cn),
				 total = off_pre + align256(prefix.size());
	if (dev_alloc(domain, (void **) &dev, total, s))
		return -1;
	unsigned char *scan = dev;
	unsigned *prev = (unsigned *) (dev + off_prev), *sym = (unsigned *) (dev + off_sym), *zs = (unsigned *) (dev + off_zs);
	unsigned short *last = (unsigned short *) (dev + off_last);
	uint2 *rec = (uint2 *) (dev + off_rec);
	BlockRec *blk = (BlockRec *) (dev + off_blk);
	DeflatePlan *plans = (DeflatePlan *) (dev + off_plan);
	FrameOut *fo = (FrameOut *) (dev + off_fo);
	unsigned long long *at_out = (unsigned long long *) (dev + off_at);
	unsigned char *dpre = dev + off_pre, *out = nullptr;
	int rc = -1;
	do {
		if (cudaMemsetAsync(zs, 0, g.zcap * cn, s) != cudaSuccess ||
			cudaMemcpyAsync(dpre, prefix.data(), prefix.size(), cudaMemcpyHostToDevice, s) != cudaSuccess) {
			cuda_fail(domain, cudaGetLastError(), "png save staging");
			break;
		}
		const unsigned gx = (unsigned) std::min<size_t>((g.scan_stride + 255) / 256, 4096);
		png_scan_kernel<<<dim3(gx, cn), 256, 0, s>>>(src, bpl, frame_stride, sg, g.scan_stride, scan);
		png_adler_kernel<<<cn, 256, 0, s>>>(scan, g, fo);
		deflate_last_kernel<<<dim3(g.tiles, cn), 1024, kWSize * 4, s>>>(scan, g, last);
		deflate_chain_kernel<<<dim3(g.tiles, cn), 32, kWSize * 2, s>>>(scan, g, last, prev);
		const unsigned mx = (unsigned) std::min<size_t>((g.n + 127) / 128, 1 << 20);
		deflate_match_kernel<<<dim3(mx, cn), 128, 0, s>>>(scan, g, prev, rec);
		deflate_parse_kernel<<<(cn + kParseWarps - 1) / kParseWarps, kParseWarps * 32, 0, s>>>(scan, g, cn, rec, sym, blk, fo);
		const unsigned bx = (unsigned) ((g.maxblk + kBlockWarps - 1) / kBlockWarps);
		deflate_block_kernel<<<dim3(bx, cn), kBlockWarps * 32, 0, s>>>(g, sym, blk, plans, fo);
		deflate_offsets_kernel<<<(cn + 127) / 128, 128, 0, s>>>(g, cn, blk, plans, zs, fo);
		deflate_emit_kernel<<<dim3(bx, cn), kBlockWarps * 32, 0, s>>>(g, scan, sym, blk, plans, fo, zs);
		count_launch(9);
		cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess) {
			cuda_fail(domain, e, "png save kernels");
			break;
		}
		if (place(&fo->len, sizeof(FrameOut), at_out, &out))
			break;
		png_frame_kernel<<<dim3((g.maxchunks + 7) / 8, cn), 256, 0, s>>>(g, dpre, zs, fo, at_out, out);
		count_launch(1);
		e = cudaGetLastError();
		if (e != cudaSuccess) {
			cuda_fail(domain, e, "png_frame_kernel");
			break;
		}
		rc = 0;
	} while (0);
	dev_free(dev, s);
	return rc;
}

} // namespace

int
png_encoder(const char *domain, int w, int h, int bands, const VB200PngSaveOptions &o, const unsigned char *profile, size_t profile_len,
	Encoder *enc)
{
	if (check_save(domain, w, h, bands, o))
		return -1;
	const std::vector<unsigned char> prefix = png_prefix(w, h, bands, o, profile, profile_len);
	const EncGeom g = enc_geom(w, h, bands, o, prefix.size());
	const ScanGeom sg = scan_geom(w, h, bands, o);
	enc->scratch_bytes = g.scan_stride + align256(4 * g.n) + align256((size_t) 2 * kWSize * g.tiles) + align256(8 * g.n) + align256(4 * g.n) +
		align256(g.maxblk * (sizeof(BlockRec) + sizeof(DeflatePlan))) + g.zcap + sizeof(FrameOut) + sizeof(unsigned long long);
	enc->stream_bytes = g.prefix + g.zcap + 12 * (size_t) g.maxchunks + 12;
	enc->chunk = [domain, g, sg, prefix](const unsigned char *src, size_t bpl, size_t frame_stride, int cn, const EncodePlace &place,
				 cudaStream_t s) {
		return png_chunk(domain, g, sg, prefix, src, bpl, frame_stride, cn, place, s);
	};
	return 0;
}

/* the whole PNG stream on the CPU through the kernels' per-position, per-symbol and per-block code */
int
host_png_encode(const char *domain, const unsigned char *img, size_t bpl, int w, int h, int bands, const VB200PngSaveOptions &o,
	const unsigned char *profile, size_t profile_len, std::vector<unsigned char> &out)
{
	if (check_save(domain, w, h, bands, o))
		return -1;
	out = png_prefix(w, h, bands, o, profile, profile_len);
	const ScanGeom sg = scan_geom(w, h, bands, o);
	std::vector<unsigned char> scan(sg.n + 8, 0), z;
	auto rd = [&](size_t row, size_t col) -> unsigned { return img[row * bpl + col]; };
	for (size_t i = 0; i < sg.n; i++)
		scan[i] = (unsigned char) scan_byte(sg, i, rd);
	host_deflate(scan.data(), sg.n, o.compression, o.strategy, z);
	for (size_t at = 0; at < z.size(); at += kIdat)
		put_chunk(out, "IDAT", std::vector<unsigned char>(z.begin() + at, z.begin() + std::min(z.size(), at + kIdat)));
	put_chunk(out, "IEND", {});
	return 0;
}

} // namespace vb200

/* ------------------------------------------------------------------ C ABI */

using namespace vb200;

extern "C" int
vb200_pngsave_batch(const void *frames, int frames_location, size_t bpl, size_t frame_stride, int n, int width, int height, int bands,
	const VB200PngSaveOptions *options, const void *profile, size_t profile_len, void *out, int out_location, size_t out_stride, size_t *lengths)
{
	const char *domain = "pngsave_batch";
	return encode_batch_abi(domain, options,
		[&](Encoder *enc) { return png_encoder(domain, width, height, bands, *options, (const unsigned char *) profile, profile_len, enc); }, frames,
		frames_location, bpl, frame_stride, n, width, height, bands, out, out_location, out_stride, lengths);
}

/* reference: vips_pngsave_buffer(in, &buf, &len, "compression", .., NULL), foreign/spngsave.c */
extern "C" int
vb200_pngsave_buffer(const VB200Image *in, const VB200PngSaveOptions *options, const void *profile, size_t profile_len, void **out, size_t *len)
{
	const char *domain = "pngsave_buffer";
	if (!in || !options || !out || !len || !in->data) {
		error(domain, "null argument");
		return -1;
	}
	if (in->BandFmt != VB200_FORMAT_UCHAR) {
		error(domain, "format %d: PNG save on the device takes uchar frames (bit depth 8; 16-bit is not built)", in->BandFmt);
		return -1;
	}
	const size_t line = (size_t) in->Xsize * in->Bands;
	if (in->bpl < line) {
		error(domain, "frame strides too small for %d x %d x %d", in->Xsize, in->Ysize, in->Bands);
		return -1;
	}
	Encoder enc;
	if (png_encoder(domain, in->Xsize, in->Ysize, in->Bands, *options, (const unsigned char *) profile, profile_len, &enc) || ensure_init(domain))
		return -1;
	std::vector<unsigned char> bytes;
	EncodeDest dst;
	dst.bytes = &bytes;
	size_t got = 0;
	if (dev_encode_batch(domain, enc, in->data, in->where, in->bpl, in->bpl * in->Ysize, 1, line, in->Ysize, dst, &got, current_stream()))
		return -1;
	void *buf = malloc(got);
	if (!buf) {
		error(domain, "out of memory");
		return -1;
	}
	memcpy(buf, bytes.data(), got);
	*out = buf;
	*len = got;
	return 0;
}

extern "C" int
vb200_debug_png_encode(const void *pixels, size_t bpl, int width, int height, int bands, const VB200PngSaveOptions *options, const void *profile,
	size_t profile_len, void *out, size_t cap, size_t *len)
{
	const char *domain = "png_encode (host twin)";
	if (!pixels || !options || !len) {
		error(domain, "null argument");
		return -1;
	}
	try {
		std::vector<unsigned char> v;
		if (host_png_encode(domain, (const unsigned char *) pixels, bpl, width, height, bands, *options, (const unsigned char *) profile, profile_len, v))
			return -1;
		*len = v.size();
		if (out) {
			if (cap < v.size()) {
				error(domain, "the stream is %zu bytes, the buffer %zu", v.size(), cap);
				return -1;
			}
			memcpy(out, v.data(), v.size());
		}
		return 0;
	}
	catch (const std::exception &e) {
		error(domain, "%s", e.what());
		return -1;
	}
}

extern "C" int
vb200_debug_deflate(const void *buf, size_t n, int level, int strategy, void *out, size_t cap, size_t *len)
{
	const char *domain = "deflate (host twin)";
	const VB200PngSaveOptions o = {level, strategy, 1.0};
	if (!len || (!buf && n) || check_save(domain, 1, 1, 1, o))
		return -1;
	try {
		std::vector<unsigned char> d(n + 8, 0), z;
		if (n)
			memcpy(d.data(), buf, n);
		host_deflate(d.data(), n, level, strategy, z);
		*len = z.size();
		if (out) {
			if (cap < z.size()) {
				error(domain, "the stream is %zu bytes, the buffer %zu", z.size(), cap);
				return -1;
			}
			memcpy(out, z.data(), z.size());
		}
		return 0;
	}
	catch (const std::exception &e) {
		error(domain, "%s", e.what());
		return -1;
	}
}
