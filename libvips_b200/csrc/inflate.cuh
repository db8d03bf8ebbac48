/* inflate.cuh -- raw deflate (RFC 1951) on the host and the device, shared by the PNG decoder (png.cu) and the TIFF
 * decoder's deflate segments (tiff.cu).  inflate_step runs on one thread; inflate_warp is the warp loop around it: lane 0
 * decodes symbols and writes literals, the warp copies every match and stored block with 32 lanes.
 */
#ifndef VB200_INFLATE_CUH
#define VB200_INFLATE_CUH

#include <cstring>

#ifndef VB_HD
#define VB_HD __host__ __device__ __forceinline__
#endif

namespace vb200 {

namespace {

/* ------------------------------------------------------------------ inflate (RFC 1951), host and device */

constexpr int kFastBits = 9;

/* a canonical Huffman code: a 2^9 lookup of the short codes ((symbol << 4) | length, 0 = longer or no code) and the
 * per-length counts and symbols of puff.c's slow decode
 */
struct Huff {
	unsigned short fast[1 << kFastBits];
	unsigned short count[16];
	unsigned short sym[288];
};

struct InflateTables {
	Huff lit, dist;
	unsigned char lens[320]; /* a dynamic block's 286 + 30 code lengths (or the 19 of the code-length code) */
};

__host__ __device__ inline unsigned
bit_reverse(unsigned code, int len)
{
	unsigned r = 0;
	for (int i = 0; i < len; i++, code >>= 1)
		r = (r << 1) | (code & 1);
	return r;
}

/* inftrees.c's rules: an over-subscribed set is refused; an incomplete one too, except a single code of length 1 in a
 * literal / length or distance set (codes = false).  An empty distance set is accepted (every use of it is an error).
 */
__host__ __device__ inline int
build_huff(Huff *h, const unsigned char *len, int n, bool codes)
{
	for (int i = 0; i < 16; i++)
		h->count[i] = 0;
	for (int i = 0; i < n; i++)
		h->count[len[i]]++;
	h->count[0] = 0;
	int max = 15;
	while (max >= 1 && !h->count[max])
		max--;
	int left = 1;
	for (int l = 1; l <= 15; l++) {
		left = (left << 1) - h->count[l];
		if (left < 0)
			return -1;
	}
	if (max == 0)
		return codes ? -1 : 0; /* zlib takes an empty code-length code, and then always fails: no end-of-block code */
	if (left > 0 && (codes || max != 1))
		return -1;
	unsigned short offs[16];
	offs[1] = 0;
	for (int l = 1; l < 15; l++)
		offs[l + 1] = offs[l] + h->count[l];
	for (int i = 0; i < n; i++)
		if (len[i])
			h->sym[offs[len[i]]++] = (unsigned short) i;
	for (int i = 0; i < (1 << kFastBits); i++)
		h->fast[i] = 0;
	unsigned code = 0;
	int k = 0;
	for (int l = 1; l <= kFastBits; l++) {
		for (int j = 0; j < h->count[l]; j++, k++, code++) {
			const unsigned r = bit_reverse(code, l);
			for (unsigned f = r; f < (1u << kFastBits); f += 1u << l)
				h->fast[f] = (unsigned short) ((h->sym[k] << 4) | l);
		}
		code <<= 1;
	}
	return 0;
}

/* LSB-first bit reader over len bytes; reads past the end see zeros, and over() says whether any were consumed */
struct BitIn {
	const unsigned char *src;
	unsigned long long len, p;
	unsigned long long bb;
	int nb;

	VB_HD void refill()
	{
		while (nb <= 56) {
			bb |= (unsigned long long) (p < len ? src[p] : 0) << nb;
			p++;
			nb += 8;
		}
	}
	VB_HD unsigned bits(int n)
	{
		if (nb < n)
			refill();
		const unsigned v = (unsigned) (bb & ((1ull << n) - 1));
		bb >>= n;
		nb -= n;
		return v;
	}
	VB_HD bool over() const { return 8 * p - (unsigned long long) nb > 8 * len; }
};

__host__ __device__ inline int
decode_sym(const Huff *h, BitIn &in)
{
	if (in.nb < 15)
		in.refill();
	const unsigned e = h->fast[in.bb & ((1u << kFastBits) - 1)];
	if (e) {
		in.bb >>= e & 15;
		in.nb -= e & 15;
		return (int) (e >> 4);
	}
	/* puff.c's canonical decode, one bit at a time */
	int code = 0, first = 0, index = 0;
	unsigned long long b = in.bb;
	for (int l = 1; l <= 15; l++) {
		code |= (int) (b & 1);
		b >>= 1;
		const int c = h->count[l];
		if (code - first < c) {
			in.bb >>= l;
			in.nb -= l;
			return h->sym[index + code - first];
		}
		index += c;
		first = (first + c) << 1;
		code <<= 1;
	}
	return -1;
}

/* RFC 1951 3.2.5 and 3.2.7: length and distance bases and extra bits, the order of the code-length code's lengths */
struct InflateConsts {
	unsigned short lbase[29], dbase[30];
	unsigned char lext[29], dext[30], order[19];
};
#define INFLATE_CONSTS_INIT                                                                                                                              \
	{                                                                                                                                                    \
		{3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258},                             \
			{1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, \
				24577},                                                                                                                                  \
			{0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0},                                                     \
			{0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13},                                          \
			{16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15},                                                                          \
	}
__constant__ InflateConsts d_inflate_consts = INFLATE_CONSTS_INIT;
[[maybe_unused]] const InflateConsts h_inflate_consts = INFLATE_CONSTS_INIT;
#ifdef __CUDA_ARCH__
#define INFLATE_CONSTS d_inflate_consts
#else
#define INFLATE_CONSTS h_inflate_consts
#endif

enum { OP_MATCH = 0, OP_STORED = 1, OP_DONE = 2, OP_ERR = 3 };
enum { ERR_CORRUPT = 1, ERR_MORE = 2 }; /* the decoders' own status bits start at 4 */

struct Inflate {
	BitIn in;
	InflateTables *t;
	unsigned long long pos, cap;
	int in_block, last, err;
	int clip; /* stop once cap bytes are out, as zlib does with a full output buffer (libtiff's ZIPDecode), instead of ERR_MORE */
	int full; /* clip mode: the output filled before the last block ended */
};

__host__ __device__ inline void
inflate_init(Inflate &z, const unsigned char *src, unsigned long long len, unsigned long long cap, InflateTables *t)
{
	z.in.src = src;
	z.in.len = len;
	z.in.p = 0;
	z.in.bb = 0;
	z.in.nb = 0;
	z.t = t;
	z.pos = 0;
	z.cap = cap;
	z.in_block = 0;
	z.last = 0;
	z.err = 0;
	z.clip = 0;
	z.full = 0;
}

/* clip mode's stop: nothing more is read, and the stream counts as done */
__host__ __device__ inline void
inflate_stop_full(Inflate &z)
{
	z.in_block = 0;
	z.last = 1;
	z.full = 1;
}

__host__ __device__ inline int
inflate_fail(Inflate &z, int err)
{
	z.err = err;
	return OP_ERR;
}

/* RFC 1951 3.2.7: a dynamic block's code lengths, then its two codes (zlib's checks, inflate.c:1000-1100) */
__host__ __device__ inline int
read_dynamic(Inflate &z)
{
	const unsigned char *order = INFLATE_CONSTS.order;
	const int nlen = (int) z.in.bits(5) + 257, ndist = (int) z.in.bits(5) + 1, ncode = (int) z.in.bits(4) + 4;
	if (nlen > 286 || ndist > 30)
		return -1;
	unsigned char *lens = z.t->lens;
	for (int i = 0; i < 19; i++)
		lens[i] = 0;
	for (int i = 0; i < ncode; i++)
		lens[order[i]] = (unsigned char) z.in.bits(3);
	if (z.in.over() || build_huff(&z.t->lit, lens, 19, true))
		return -1;
	int i = 0;
	while (i < nlen + ndist) {
		const int sym = decode_sym(&z.t->lit, z.in);
		if (sym < 0)
			return -1;
		if (sym < 16)
			lens[i++] = (unsigned char) sym;
		else {
			int rep, v = 0;
			if (sym == 16) {
				if (i == 0)
					return -1;
				v = lens[i - 1];
				rep = 3 + (int) z.in.bits(2);
			}
			else if (sym == 17)
				rep = 3 + (int) z.in.bits(3);
			else
				rep = 11 + (int) z.in.bits(7);
			if (i + rep > nlen + ndist)
				return -1;
			while (rep--)
				lens[i++] = (unsigned char) v;
		}
		if (z.in.over())
			return -1;
	}
	if (lens[256] == 0)
		return -1;
	/* the distance lengths first: the literal table is built over the lengths it came from */
	if (build_huff(&z.t->dist, lens + nlen, ndist, false) || build_huff(&z.t->lit, lens, nlen, false))
		return -1;
	return 0;
}

/* Run until the next match or stored block (*at: where it goes; *len; *arg: the distance, or the stored bytes' input
 * offset), the end of the stream or an error.  Literals are written here.  Refuses exactly what zlib's raw inflate
 * refuses, and any stream that needs bits past its end (zlib would wait for more input).
 */
__host__ __device__ inline int
inflate_step(Inflate &z, unsigned char *out, unsigned long long *at, unsigned *len, unsigned long long *arg)
{
	const InflateConsts &K = INFLATE_CONSTS;
	const unsigned short *lbase = K.lbase, *dbase = K.dbase;
	const unsigned char *lext = K.lext, *dext = K.dext;
	for (;;) {
		if (!z.in_block) {
			if (z.last)
				return OP_DONE;
			z.last = (int) z.in.bits(1);
			const unsigned type = z.in.bits(2);
			if (type == 0) {
				z.in.bits(z.in.nb & 7);
				const unsigned n = z.in.bits(16), nn = z.in.bits(16);
				if (z.in.over() || n != (~nn & 0xffff))
					return inflate_fail(z, ERR_CORRUPT);
				/* back to the byte the bit buffer has reached */
				z.in.p -= (unsigned long long) (z.in.nb >> 3);
				z.in.bb = 0;
				z.in.nb = 0;
				if (z.in.p + n > z.in.len)
					return inflate_fail(z, ERR_CORRUPT);
				unsigned n_out = n;
				if (z.pos + n > z.cap) {
					if (!z.clip)
						return inflate_fail(z, ERR_MORE);
					n_out = (unsigned) (z.cap - z.pos);
					inflate_stop_full(z);
				}
				if (n_out == 0)
					continue;
				*at = z.pos;
				*len = n_out;
				*arg = z.in.p;
				z.in.p += n;
				z.pos += n_out;
				return OP_STORED;
			}
			if (type == 1) {
				unsigned char *l = z.t->lens;
				for (int i = 0; i < 288; i++)
					l[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
				build_huff(&z.t->lit, l, 288, false);
				for (int i = 0; i < 32; i++)
					l[i] = 5;
				build_huff(&z.t->dist, l, 32, false);
			}
			else if (type == 3 || read_dynamic(z))
				return inflate_fail(z, ERR_CORRUPT);
			if (z.in.over())
				return inflate_fail(z, ERR_CORRUPT);
			z.in_block = 1;
		}
		const int sym = decode_sym(&z.t->lit, z.in);
		if (sym < 0 || z.in.over())
			return inflate_fail(z, ERR_CORRUPT);
		if (sym < 256) {
			if (z.pos >= z.cap) {
				if (!z.clip)
					return inflate_fail(z, ERR_MORE);
				inflate_stop_full(z);
				return OP_DONE;
			}
			out[z.pos++] = (unsigned char) sym;
			continue;
		}
		if (sym == 256) {
			z.in_block = 0;
			continue;
		}
		if (sym > 285) /* 286 / 287: in a fixed block only */
			return inflate_fail(z, ERR_CORRUPT);
		const unsigned n = lbase[sym - 257] + z.in.bits(lext[sym - 257]);
		const int ds = decode_sym(&z.t->dist, z.in);
		if (ds < 0 || ds >= 30) /* 30 / 31: in a fixed block only */
			return inflate_fail(z, ERR_CORRUPT);
		const unsigned d = dbase[ds] + z.in.bits(dext[ds]);
		if (z.in.over() || d > z.pos)
			return inflate_fail(z, ERR_CORRUPT);
		unsigned n_out = n;
		if (z.pos + n > z.cap) {
			if (!z.clip)
				return inflate_fail(z, ERR_MORE);
			n_out = (unsigned) (z.cap - z.pos);
			inflate_stop_full(z);
		}
		*at = z.pos;
		*len = n_out;
		*arg = d;
		z.pos += n_out;
		return OP_MATCH;
	}
}

/* after OP_DONE of a stream whose last block ended: the big-endian 32-bit word at the next byte boundary (RFC 1950's
 * Adler-32 trailer), false when fewer than 4 bytes are left (zlib then waits for input and checks nothing)
 */
__host__ __device__ inline bool
inflate_trailer(const Inflate &z, unsigned *word)
{
	const unsigned long long at = (8 * z.in.p - (unsigned long long) z.in.nb + 7) / 8;
	if (at > z.in.len || z.in.len - at < 4)
		return false;
	const unsigned char *t = z.in.src + at;
	*word = ((unsigned) t[0] << 24) | ((unsigned) t[1] << 16) | ((unsigned) t[2] << 8) | t[3];
	return true;
}

/* the whole stream on one thread: the host twin's inflate.  *out_len = the bytes written; -1 with z.err set.  clip: stop once
 * cap bytes are out (Inflate::clip); end: the decoder's state when it stopped */
int
inflate_host(const unsigned char *src, size_t len, unsigned char *out, size_t cap, size_t *out_len, int *err, bool clip = false,
	Inflate *end = nullptr)
{
	InflateTables t;
	Inflate z;
	inflate_init(z, src, len, cap, &t);
	z.clip = clip;
	for (;;) {
		unsigned long long at = 0, arg = 0;
		unsigned n = 0;
		const int op = inflate_step(z, out, &at, &n, &arg);
		if (op == OP_MATCH)
			for (unsigned i = 0; i < n; i++)
				out[at + i] = out[at - arg + i];
		else if (op == OP_STORED)
			memcpy(out + at, src + arg, n);
		else {
			*out_len = (size_t) z.pos;
			*err = z.err;
			if (end)
				*end = z;
			return op == OP_DONE ? 0 : -1;
		}
	}
}

#ifdef __CUDACC__
/* One warp runs z over src into out: lane 0 steps the decoder, the warp copies each match and stored block.  Returns OP_DONE
 * or OP_ERR on every lane; z.pos and z.err are lane 0's.
 */
__device__ __forceinline__ int
inflate_warp(Inflate &z, const unsigned char *src, unsigned char *out, int lane)
{
	int op = OP_DONE;
	for (;;) {
		unsigned long long at = 0, arg = 0;
		unsigned len = 0;
		if (lane == 0)
			op = inflate_step(z, out, &at, &len, &arg);
		op = __shfl_sync(0xffffffffu, op, 0);
		at = __shfl_sync(0xffffffffu, at, 0);
		arg = __shfl_sync(0xffffffffu, arg, 0);
		len = __shfl_sync(0xffffffffu, len, 0);
		__syncwarp(); /* lane 0's literals are visible to the warp */
		if (op == OP_MATCH) {
			/* every source byte lies before `at`: an overlapping copy repeats its period */
			const unsigned d = (unsigned) arg;
			for (unsigned i = lane; i < len; i += 32)
				out[at + i] = out[at - d + (d >= len ? i : i % d)];
		}
		else if (op == OP_STORED) {
			for (unsigned i = lane; i < len; i += 32)
				out[at + i] = src[arg + i];
		}
		else
			return op;
		__syncwarp();
	}
}
#endif

} // namespace

} // namespace vb200

#endif
