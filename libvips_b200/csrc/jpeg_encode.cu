/* jpeg_encode.cu -- the other half of SURVEY 8(f) rank 1: vips_jpegsave_buffer() on the device.
 *
 * What the reference does (foreign/vips2jpeg.c:551-700): jpeg_set_defaults, jpeg_set_quality(Q, TRUE), chroma
 * subsampled 2x2 unless Q >= 90 (subsample_mode AUTO, :676-690), optimize_coding and progressive off by default, a JFIF
 * header, then jpeg_write_scanlines.  As with the loader, the codec is libjpeg(-turbo), a third-party dependency outside
 * the reference tree; this file restates its published baseline algorithm for that configuration:
 *     RGB -> YCbCr                 jccolor.c: 16-bit fixed-point tables (FIX(0.29900) ... ), Cb / Cr offset 128 + rounding
 *     2x2 chroma downsampling      jcsample.c h2v2_downsample: (a + b + c + d + bias) >> 2, bias alternating 1, 2 along a
 *                                  row; edges replicated to whole MCUs (jcprepct.c, expand_right_edge)
 *     forward DCT                  jfdctint.c "islow": CONST_BITS 13, PASS1_BITS 2, output scaled by 8
 *     quantisation                 jcdctmgr.c: (|x| + q / 2) / q with the sign restored, q = table << 3;
 *                                  tables = T.81 Annex K scaled by jpeg_quality_scaling, forced to 1..255
 *     entropy coding               jchuff.c with the T.81 Annex K.3 tables: DC difference category + bits, AC (run, size)
 *                                  + bits, ZRL, EOB; FF byte stuffing; the last byte padded with 1-bits
 * Parity: tests/test_jpeg_encode.py holds the stream to libjpeg-turbo's (the one inside this image's Pillow): the same
 * quantisation tables and, byte for byte, the same entropy-coded segment, on the CPU twin and on the GPU.
 *
 * Device pipeline per batch of equally sized frames, no host involvement between the pixels and the finished streams:
 *   jpeg_fdct_kernel       one thread per MCU: colour conversion, downsampling, FDCT + quantisation of its blocks
 *   jpeg_count_kernel      one thread per block: the number of bits its Huffman code takes (DC difference against the
 *                          previous block of its component: the coefficients are all there, nothing is sequential)
 *   (prefix sum)           bit offset of every block
 *   jpeg_emit_kernel       one thread per block: its bits OR-ed into the frame's bit buffer
 *   jpeg_stuff_kernel      FF -> FF00 and the markers around the scan: per 256-byte span count, prefix sum, copy
 */
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/vb200.h"
#include "vb200_internal.h"

namespace vb200 {

namespace {

#define HD __host__ __device__ __forceinline__

/* ITU T.81 Annex K.1 / K.3, as jcparam.c holds them (natural order) */
const unsigned char kStdLumQ[64] = {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51,
	87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
const unsigned char kStdChrQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99,
	99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
const unsigned char kBitsDcLum[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
const unsigned char kBitsDcChr[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
const unsigned char kValDc[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
const unsigned char kBitsAcLum[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125};
const unsigned char kValAcLum[162] = {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
	0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a,
	0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56,
	0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87,
	0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5,
	0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
	0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
const unsigned char kBitsAcChr[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119};
const unsigned char kValAcChr[162] = {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
	0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17,
	0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55,
	0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85,
	0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3,
	0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
	0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
const unsigned char kZz[64] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35,
	42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

/* everything the kernels need about one geometry / quality */
struct EncodeTables {
	unsigned short q[2][64];		  /* natural order, the file's values (1..255) */
	unsigned ehufco[4][256];		  /* code per symbol: dc lum, ac lum, dc chr, ac chr */
	unsigned char ehufsi[4][256];	  /* code length per symbol (0: not in the table) */
	unsigned char zz[64];
};

struct EncodeGeom {
	int w, h, bands, ncomp;
	int sub;			 /* 1: 4:2:0, 0: 4:4:4 (always 0 for greyscale) */
	int mcus_x, mcus_y, blocks_per_mcu;
	int blocks;			 /* per frame */
};

/* jcparam.c jpeg_quality_scaling + jpeg_add_quant_table(force_baseline = TRUE) */
void
scaled_quant(int quality, const unsigned char *base, unsigned short *out)
{
	quality = std::max(1, std::min(100, quality));
	const int scale = quality < 50 ? 5000 / quality : 200 - quality * 2;
	for (int i = 0; i < 64; i++) {
		long t = ((long) base[i] * scale + 50L) / 100L;
		t = std::max(1L, std::min(255L, t));
		out[i] = (unsigned short) t;
	}
}

/* jchuff.c jpeg_make_c_derived_tbl: canonical codes from (bits, values) */
void
derive_codes(const unsigned char bits[16], const unsigned char *vals, unsigned *co, unsigned char *si)
{
	memset(co, 0, 256 * sizeof(unsigned));
	memset(si, 0, 256);
	unsigned code = 0;
	int k = 0;
	for (int l = 1; l <= 16; l++) {
		for (int i = 0; i < bits[l - 1]; i++, k++, code++) {
			co[vals[k]] = code;
			si[vals[k]] = (unsigned char) l;
		}
		code <<= 1;
	}
}

void
make_tables(int quality, EncodeTables *T)
{
	scaled_quant(quality, kStdLumQ, T->q[0]);
	scaled_quant(quality, kStdChrQ, T->q[1]);
	derive_codes(kBitsDcLum, kValDc, T->ehufco[0], T->ehufsi[0]);
	derive_codes(kBitsAcLum, kValAcLum, T->ehufco[1], T->ehufsi[1]);
	derive_codes(kBitsDcChr, kValDc, T->ehufco[2], T->ehufsi[2]);
	derive_codes(kBitsAcChr, kValAcChr, T->ehufco[3], T->ehufsi[3]);
	memcpy(T->zz, kZz, 64);
}

/* ------------------------------------------------------------------ pixels -> quantised blocks (host + device) */

HD int
clampi_(int v, int lo, int hi)
{
	return v < lo ? lo : (v > hi ? hi : v);
}

/* jccolor.c rgb_ycc_convert, the tables written out */
HD void
rgb_to_ycc(int r, int g, int b, int *y, int *cb, int *cr)
{
	*y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
	*cb = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
	*cr = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

HD int
min_(int a, int b)
{
	return a < b ? a : b;
}

HD int
fdescale(int x, int n)
{
	return (x + (1 << (n - 1))) >> n;
}

/* jfdctint.c jpeg_fdct_islow on d[64] (samples already centred on 0), in place */
HD void
fdct_islow(int *d)
{
	constexpr int CB = 13, P1 = 2;
	constexpr int F_0_298631336 = 2446, F_0_390180644 = 3196, F_0_541196100 = 4433, F_0_765366865 = 6270, F_0_899976223 = 7373, F_1_175875602 = 9633,
				  F_1_501321110 = 12299, F_1_847759065 = 15137, F_1_961570560 = 16069, F_2_053119869 = 16819, F_2_562915447 = 20995,
				  F_3_072711026 = 25172;
	for (int pass = 0; pass < 2; pass++) {
		const int step = pass == 0 ? 1 : 8, next = pass == 0 ? 8 : 1;
		for (int i = 0; i < 8; i++) {
			int *p = d + i * next;
			const int tmp0 = p[0] + p[7 * step], tmp7 = p[0] - p[7 * step];
			const int tmp1 = p[1 * step] + p[6 * step], tmp6 = p[1 * step] - p[6 * step];
			const int tmp2 = p[2 * step] + p[5 * step], tmp5 = p[2 * step] - p[5 * step];
			const int tmp3 = p[3 * step] + p[4 * step], tmp4 = p[3 * step] - p[4 * step];
			const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
			if (pass == 0) {
				p[0] = (int) ((unsigned) (tmp10 + tmp11) << P1);
				p[4 * step] = (int) ((unsigned) (tmp10 - tmp11) << P1);
			}
			else {
				p[0] = fdescale(tmp10 + tmp11, P1);
				p[4 * step] = fdescale(tmp10 - tmp11, P1);
			}
			const int sh = pass == 0 ? CB - P1 : CB + P1;
			int z1 = (tmp12 + tmp13) * F_0_541196100;
			p[2 * step] = fdescale(z1 + tmp13 * F_0_765366865, sh);
			p[6 * step] = fdescale(z1 + tmp12 * (-F_1_847759065), sh);
			z1 = tmp4 + tmp7;
			int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
			const int z5 = (z3 + z4) * F_1_175875602;
			const int t4 = tmp4 * F_0_298631336, t5 = tmp5 * F_2_053119869, t6 = tmp6 * F_3_072711026, t7 = tmp7 * F_1_501321110;
			z1 *= -F_0_899976223;
			z2 *= -F_2_562915447;
			z3 *= -F_1_961570560;
			z4 *= -F_0_390180644;
			z3 += z5;
			z4 += z5;
			p[7 * step] = fdescale(t4 + z1 + z3, sh);
			p[5 * step] = fdescale(t5 + z2 + z4, sh);
			p[3 * step] = fdescale(t6 + z2 + z3, sh);
			p[1 * step] = fdescale(t7 + z1 + z4, sh);
		}
	}
}

/* jcdctmgr.c quantize: divisor = table value << 3 (the islow FDCT scales by 8) */
HD short
quantise(int v, int q)
{
	const int qv = q << 3;
	int t = v < 0 ? -v : v;
	t += qv >> 1;
	t = t >= qv ? t / qv : 0;
	return (short) (v < 0 ? -t : t);
}

/* sample (x, y) of the frame with the edges replicated to whole MCUs */
HD void
pixel_ycc(const unsigned char *img, size_t bpl, int w, int h, int bands, int x, int y, int *yy, int *cb, int *cr)
{
	const unsigned char *p = img + (size_t) clampi_(y, 0, h - 1) * bpl + (size_t) clampi_(x, 0, w - 1) * bands;
	if (bands == 1) {
		*yy = p[0];
		*cb = *cr = 128;
	}
	else
		rgb_to_ycc(p[0], p[1], p[2], yy, cb, cr);
}

/* all blocks of MCU (mx, my) into coef[blocks_per_mcu][64] (natural order) */
HD void
encode_mcu(const EncodeGeom &G, const unsigned short (*q)[64], const unsigned char *img, size_t bpl, int mx, int my, short *coef)
{
	int d[64];
	if (G.ncomp == 1 || !G.sub) {
		/* one 8 x 8 block per component */
		const int x0 = mx * 8, y0 = my * 8;
		for (int c = 0; c < G.ncomp; c++) {
			for (int y = 0; y < 8; y++)
				for (int x = 0; x < 8; x++) {
					int v[3];
					pixel_ycc(img, bpl, G.w, G.h, G.bands, x0 + x, y0 + y, &v[0], &v[1], &v[2]);
					d[y * 8 + x] = v[c] - 128;
				}
			fdct_islow(d);
			for (int i = 0; i < 64; i++)
				coef[c * 64 + i] = quantise(d[i], q[c ? 1 : 0][i]);
		}
		return;
	}
	/* 4:2:0: four luma blocks, then Cb, Cr of the 16 x 16 area downsampled 2 x 2 (jcsample.c h2v2_downsample: the bias
	 * alternates 1, 2 along an output row, starting at 1)
	 */
	const int x0 = mx * 16, y0 = my * 16;
	/* luma blocks past the component's own block grid (an odd number of block columns / rows) are DUMMY blocks, not
	 * encoded pixels: all zero but for a DC copied from a neighbour (jccoefct.c compress_data: at the right edge the block
	 * before it; a dummy bottom row takes the last block of the row above it in the MCU)
	 */
	const int wb = (G.w + 7) / 8, hb = (G.h + 7) / 8;
	for (int b = 0; b < 4; b++) {
		const int bx = x0 + (b & 1) * 8, by = y0 + (b >> 1) * 8;
		const bool dummy_row = my * 2 + (b >> 1) >= hb, dummy_col = mx * 2 + (b & 1) >= wb;
		if (dummy_row || dummy_col) {
			for (int i = 0; i < 64; i++)
				coef[b * 64 + i] = 0;
			coef[b * 64] = coef[(dummy_row ? 1 : b - 1) * 64];
			continue;
		}
		for (int y = 0; y < 8; y++)
			for (int x = 0; x < 8; x++) {
				int yy, cb, cr;
				pixel_ycc(img, bpl, G.w, G.h, G.bands, bx + x, by + y, &yy, &cb, &cr);
				d[y * 8 + x] = yy - 128;
			}
		fdct_islow(d);
		for (int i = 0; i < 64; i++)
			coef[b * 64 + i] = quantise(d[i], q[0][i]);
	}
	for (int c = 1; c < 3; c++) {
		for (int y = 0; y < 8; y++)
			for (int x = 0; x < 8; x++) {
				/* rows: the colour buffer is padded to a whole row GROUP by repeating the last input row, but the rest
				 * of the iMCU by repeating the last DOWNSAMPLED row (jcprepct.c pre_process_data); columns: the input
				 * is padded (expand_right_edge)
				 */
				const int ry = min_(my * 8 + y, (G.h + 1) / 2 - 1);
				int sum = 0;
				for (int dy = 0; dy < 2; dy++)
					for (int dx = 0; dx < 2; dx++) {
						int v[3];
						pixel_ycc(img, bpl, G.w, G.h, G.bands, x0 + 2 * x + dx, 2 * ry + dy, &v[0], &v[1], &v[2]);
						sum += v[c];
					}
				/* the bias of output column (mx * 8 + x): 1, 2, 1, 2 ... from the row's first column */
				d[y * 8 + x] = ((sum + 1 + ((mx * 8 + x) & 1)) >> 2) - 128;
			}
		fdct_islow(d);
		for (int i = 0; i < 64; i++)
			coef[(3 + c) * 64 + i] = quantise(d[i], q[1][i]);
	}
}

/* ------------------------------------------------------------------ entropy coding (host + device) */

HD int
bit_size(int v)
{
	/* jchuff.c: the number of bits needed for |v| */
	int a = v < 0 ? -v : v, n = 0;
	while (a) {
		n++;
		a >>= 1;
	}
	return n;
}

/* component of block b of an MCU, and the index of the previous block of the same component in scan order (or -1) */
HD int
block_comp(const EncodeGeom &G, int bi)
{
	if (G.ncomp == 1)
		return 0;
	if (!G.sub)
		return bi;
	return bi < 4 ? 0 : bi - 3;
}

/* Walk one block's symbols: emit(code, length) for every Huffman code and its extra bits; returns the bit count */
template <typename Emit>
HD unsigned
code_block(const EncodeTables &T, const short *blk, int comp, int prev_dc, Emit emit)
{
	const int dt = comp ? 2 : 0, at = dt + 1;
	unsigned bits = 0;
	int diff = blk[0] - prev_dc;
	int t2 = diff;
	if (diff < 0) {
		diff = -diff;
		t2--; /* one's complement of the magnitude for negative values (F.1.2.1) */
	}
	int nb = bit_size(diff);
	emit(T.ehufco[dt][nb], T.ehufsi[dt][nb]);
	bits += T.ehufsi[dt][nb];
	if (nb) {
		emit((unsigned) t2 & ((1u << nb) - 1), nb);
		bits += nb;
	}
	int run = 0;
	for (int k = 1; k < 64; k++) {
		int v = blk[T.zz[k]];
		if (v == 0) {
			run++;
			continue;
		}
		while (run > 15) {
			emit(T.ehufco[at][0xF0], T.ehufsi[at][0xF0]);
			bits += T.ehufsi[at][0xF0];
			run -= 16;
		}
		t2 = v;
		if (v < 0) {
			v = -v;
			t2--;
		}
		nb = bit_size(v);
		const int sym = (run << 4) + nb;
		emit(T.ehufco[at][sym], T.ehufsi[at][sym]);
		emit((unsigned) t2 & ((1u << nb) - 1), nb);
		bits += T.ehufsi[at][sym] + nb;
		run = 0;
	}
	if (run > 0) {
		emit(T.ehufco[at][0], T.ehufsi[at][0]);
		bits += T.ehufsi[at][0];
	}
	return bits;
}

/* the DC value the block's difference is taken against: the previous block of its component in scan order */
HD int
previous_dc(const EncodeGeom &G, const short *coef, unsigned blk)
{
	const int nb = G.blocks_per_mcu;
	const unsigned mcu = blk / (unsigned) nb;
	const int bi = (int) (blk - mcu * (unsigned) nb);
	if (G.ncomp == 3 && G.sub && bi >= 1 && bi <= 3)
		return coef[(size_t) (blk - 1) * 64]; /* luma blocks 1..3 follow luma block bi - 1 */
	if (mcu == 0)
		return 0;
	/* the last block of the component in the previous MCU */
	const int last = (G.ncomp == 3 && G.sub && bi == 0) ? 3 : bi;
	return coef[((size_t) (mcu - 1) * nb + last) * 64];
}

/* ------------------------------------------------------------------ stream assembly (host) */

void
put16(std::vector<unsigned char> &o, unsigned v)
{
	o.push_back((unsigned char) (v >> 8));
	o.push_back((unsigned char) v);
}

/* everything up to and including SOS, in libjpeg's order: SOI, JFIF APP0, DQT per table, SOF0, DHT per table, SOS */
void
write_headers(const EncodeGeom &G, const EncodeTables &T, std::vector<unsigned char> &o)
{
	o.clear();
	put16(o, 0xFFD8);
	put16(o, 0xFFE0);
	put16(o, 16);
	const unsigned char jfif[14] = {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
	o.insert(o.end(), jfif, jfif + 14);
	for (int t = 0; t < (G.ncomp == 1 ? 1 : 2); t++) {
		put16(o, 0xFFDB);
		put16(o, 67);
		o.push_back((unsigned char) t);
		for (int i = 0; i < 64; i++)
			o.push_back((unsigned char) T.q[t][kZz[i]]);
	}
	put16(o, 0xFFC0);
	put16(o, 8 + 3 * G.ncomp);
	o.push_back(8);
	put16(o, (unsigned) G.h);
	put16(o, (unsigned) G.w);
	o.push_back((unsigned char) G.ncomp);
	for (int c = 0; c < G.ncomp; c++) {
		o.push_back((unsigned char) (c + 1));
		o.push_back((unsigned char) (c == 0 && G.sub && G.ncomp == 3 ? 0x22 : 0x11));
		o.push_back((unsigned char) (c ? 1 : 0));
	}
	const unsigned char *bits[4] = {kBitsDcLum, kBitsAcLum, kBitsDcChr, kBitsAcChr};
	const unsigned char *vals[4] = {kValDc, kValAcLum, kValDc, kValAcChr};
	const int nvals[4] = {12, 162, 12, 162};
	for (int t = 0; t < (G.ncomp == 1 ? 2 : 4); t++) {
		put16(o, 0xFFC4);
		put16(o, 19 + nvals[t]);
		o.push_back((unsigned char) (((t & 1) << 4) | (t >> 1)));
		o.insert(o.end(), bits[t], bits[t] + 16);
		o.insert(o.end(), vals[t], vals[t] + nvals[t]);
	}
	put16(o, 0xFFDA);
	put16(o, 6 + 2 * G.ncomp);
	o.push_back((unsigned char) G.ncomp);
	for (int c = 0; c < G.ncomp; c++) {
		o.push_back((unsigned char) (c + 1));
		o.push_back((unsigned char) (c ? 0x11 : 0x00));
	}
	o.push_back(0);
	o.push_back(63);
	o.push_back(0);
}

int
make_geom(const char *domain, int w, int h, int bands, int quality, int subsample_mode, EncodeGeom *G)
{
	if (w < 1 || h < 1 || w > 65535 || h > 65535) {
		error(domain, "image size %d x %d outside what JPEG can hold", w, h);
		return -1;
	}
	if (bands != 1 && bands != 3) {
		error(domain, "JPEG save on the device path takes 1- or 3-band uchar images");
		return -1;
	}
	G->w = w;
	G->h = h;
	G->bands = bands;
	G->ncomp = bands;
	/* vips2jpeg.c:676-690: AUTO subsamples chroma below Q 90 */
	G->sub = bands == 3 && (subsample_mode == 1 || (subsample_mode == 0 && quality < 90));
	const int ms = G->sub ? 16 : 8;
	G->mcus_x = (w + ms - 1) / ms;
	G->mcus_y = (h + ms - 1) / ms;
	G->blocks_per_mcu = bands == 1 ? 1 : (G->sub ? 6 : 3);
	G->blocks = G->mcus_x * G->mcus_y * G->blocks_per_mcu;
	return 0;
}

/* ------------------------------------------------------------------ kernels */

constexpr int kStuffChunk = 256; /* bytes of raw scan per thread of the stuffing kernels */
constexpr int kMaxBlockBytes = 208; /* 64 coefficients x (16-bit code + 10 bits): the bit buffer's bound per block */

/* one thread per MCU; blockIdx.y = frame */
__global__ void __launch_bounds__(128)
jpeg_fdct_kernel(const EncodeGeom G, const EncodeTables *__restrict__ T, const unsigned char *__restrict__ img, size_t bpl, size_t frame_stride,
	short *__restrict__ coef)
{
	__shared__ unsigned short s_q[2][64];
	for (int i = threadIdx.x; i < 128; i += blockDim.x)
		s_q[i >> 6][i & 63] = T->q[i >> 6][i & 63];
	__syncthreads();
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= G.mcus_x * G.mcus_y)
		return;
	const int my = i / G.mcus_x, mx = i - my * G.mcus_x;
	__align__(16) short local[6 * 64];
	encode_mcu(G, s_q, img + (size_t) blockIdx.y * frame_stride, bpl, mx, my, local);
	short *dst = coef + ((size_t) blockIdx.y * G.blocks + (size_t) i * G.blocks_per_mcu) * 64;
	for (int j = 0; j < G.blocks_per_mcu * 64; j += 8)
		*(uint4 *) (dst + j) = *(const uint4 *) (local + j);
}

/* one thread per block: how many bits its code takes */
__global__ void __launch_bounds__(128)
jpeg_count_kernel(const EncodeGeom G, const EncodeTables *__restrict__ T, const short *__restrict__ coef, unsigned *__restrict__ bits)
{
	const unsigned b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= (unsigned) G.blocks)
		return;
	const short *fc = coef + (size_t) blockIdx.y * G.blocks * 64;
	bits[(size_t) blockIdx.y * G.blocks + b] = code_block(*T, fc + (size_t) b * 64, block_comp(G, (int) (b % (unsigned) G.blocks_per_mcu)),
		previous_dc(G, fc, b), [](unsigned, int) {});
}

/* exclusive prefix sum of a frame's per-block bit counts (in place), total into totals[frame]: one CTA per frame */
__global__ void __launch_bounds__(1024)
jpeg_bitscan_kernel(int blocks, unsigned *__restrict__ bits, unsigned long long *__restrict__ totals)
{
	__shared__ unsigned long long s_part[1024];
	unsigned *b = bits + (size_t) blockIdx.x * blocks;
	const unsigned per = ((unsigned) blocks + blockDim.x - 1) / blockDim.x;
	const unsigned a = min((unsigned) blocks, threadIdx.x * per), e = min((unsigned) blocks, a + per);
	unsigned long long sum = 0;
	for (unsigned i = a; i < e; i++)
		sum += b[i];
	s_part[threadIdx.x] = sum;
	__syncthreads();
	for (unsigned o = 1; o < blockDim.x; o <<= 1) {
		const unsigned long long v = threadIdx.x >= o ? s_part[threadIdx.x - o] : 0;
		__syncthreads();
		s_part[threadIdx.x] += v;
		__syncthreads();
	}
	unsigned long long run = s_part[threadIdx.x] - sum;
	for (unsigned i = a; i < e; i++) {
		const unsigned n = b[i];
		b[i] = (unsigned) run; /* a frame's scan stays far below 2^32 bits (65535 x 65535 would not, and is refused) */
		run += n;
	}
	if (threadIdx.x == blockDim.x - 1)
		totals[blockIdx.x] = s_part[threadIdx.x];
}

/* one thread per block: its bits into the frame's (zeroed) raw bit buffer, whole bytes OR-ed in (neighbouring blocks share
 * their boundary bytes); the thread that ends the frame also pads the last byte with 1-bits
 */
__global__ void __launch_bounds__(128)
jpeg_emit_kernel(const EncodeGeom G, const EncodeTables *__restrict__ T, const short *__restrict__ coef, const unsigned *__restrict__ offs,
	const unsigned long long *__restrict__ totals, unsigned *__restrict__ raw, size_t raw_words)
{
	const unsigned b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= (unsigned) G.blocks)
		return;
	const short *fc = coef + (size_t) blockIdx.y * G.blocks * 64;
	unsigned *out = raw + (size_t) blockIdx.y * raw_words;
	unsigned pos = offs[(size_t) blockIdx.y * G.blocks + b]; /* bit index */
	unsigned long long acc = 0;
	int nacc = (int) (pos & 7u); /* the bits of the first byte that belong to the block before: zeros here, OR-ed there */
	unsigned byte = pos >> 3;
	auto put = [&](unsigned code, int len) {
		acc = (acc << len) | code;
		nacc += len;
		while (nacc >= 8) {
			const unsigned v = (unsigned) (acc >> (nacc - 8)) & 0xffu;
			if (v)
				atomicOr(out + (byte >> 2), v << (8 * (byte & 3u)));
			byte++;
			nacc -= 8;
		}
	};
	code_block(*T, fc + (size_t) b * 64, block_comp(G, (int) (b % (unsigned) G.blocks_per_mcu)), previous_dc(G, fc, b), put);
	if (nacc > 0) {
		unsigned v = (unsigned) (acc << (8 - nacc)) & 0xffu;
		if (b == (unsigned) G.blocks - 1)
			v |= (1u << (8 - nacc)) - 1; /* jchuff.c flush_bits: pad the last byte with ones */
		if (v)
			atomicOr(out + (byte >> 2), v << (8 * (byte & 3u)));
	}
	(void) totals;
}

/* stuffing, pass 1: 0xFF bytes per kStuffChunk-byte span of each frame's raw scan */
__global__ void __launch_bounds__(128)
jpeg_ffcount_kernel(const unsigned long long *__restrict__ totals, const unsigned char *__restrict__ raw, size_t raw_bytes, int max_chunks,
	unsigned *__restrict__ counts)
{
	const int c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= max_chunks)
		return;
	const unsigned long long nbytes = (totals[blockIdx.y] + 7) >> 3;
	const unsigned char *p = raw + (size_t) blockIdx.y * raw_bytes;
	unsigned n = 0;
	const unsigned long long a = (unsigned long long) c * kStuffChunk, e = min(nbytes, a + kStuffChunk);
	for (unsigned long long i = a; i < e; i++)
		n += p[i] == 0xFF;
	counts[(size_t) blockIdx.y * max_chunks + c] = n;
}

/* stuffing, pass 2: prefix sum of the spans' counts, one CTA per frame; lengths[frame] = header + scan + stuffed zeros + EOI */
__global__ void __launch_bounds__(1024)
jpeg_ffscan_kernel(const unsigned long long *__restrict__ totals, int max_chunks, unsigned *__restrict__ counts, unsigned header_len,
	unsigned long long *__restrict__ lengths)
{
	__shared__ unsigned s_part[1024];
	unsigned *cnt = counts + (size_t) blockIdx.x * max_chunks;
	const unsigned per = ((unsigned) max_chunks + blockDim.x - 1) / blockDim.x;
	const unsigned a = min((unsigned) max_chunks, threadIdx.x * per), e = min((unsigned) max_chunks, a + per);
	unsigned sum = 0;
	for (unsigned i = a; i < e; i++)
		sum += cnt[i];
	s_part[threadIdx.x] = sum;
	__syncthreads();
	for (unsigned o = 1; o < blockDim.x; o <<= 1) {
		const unsigned v = threadIdx.x >= o ? s_part[threadIdx.x - o] : 0;
		__syncthreads();
		s_part[threadIdx.x] += v;
		__syncthreads();
	}
	unsigned run = s_part[threadIdx.x] - sum;
	for (unsigned i = a; i < e; i++) {
		const unsigned n = cnt[i];
		cnt[i] = run;
		run += n;
	}
	if (threadIdx.x == blockDim.x - 1)
		lengths[blockIdx.x] = (unsigned long long) header_len + ((totals[blockIdx.x] + 7) >> 3) + s_part[threadIdx.x] + 2;
}

/* stuffing, pass 3: header, stuffed scan, EOI into the caller's stream (a stream that does not fit is cut: the host
 * compares lengths[frame] with the stride and reports it)
 */
__global__ void __launch_bounds__(128)
jpeg_stuff_kernel(const unsigned long long *__restrict__ totals, const unsigned char *__restrict__ raw, size_t raw_bytes, int max_chunks,
	const unsigned *__restrict__ counts, const unsigned char *__restrict__ header, unsigned header_len, unsigned char *__restrict__ out,
	size_t out_stride, const unsigned long long *__restrict__ lengths)
{
	const int c = blockIdx.x * blockDim.x + threadIdx.x;
	unsigned char *o = out + (size_t) blockIdx.y * out_stride;
	const unsigned long long len = lengths[blockIdx.y];
	if (len > out_stride)
		return;
	if (c < (int) ((header_len + kStuffChunk - 1) / kStuffChunk)) {
		/* the first spans' threads also copy the header */
		for (unsigned i = (unsigned) c * kStuffChunk; i < min(header_len, (unsigned) (c + 1) * kStuffChunk); i++)
			o[i] = header[i];
	}
	if (c >= max_chunks)
		return;
	const unsigned long long nbytes = (totals[blockIdx.y] + 7) >> 3;
	const unsigned char *p = raw + (size_t) blockIdx.y * raw_bytes;
	const unsigned long long a = (unsigned long long) c * kStuffChunk, e = min(nbytes, a + kStuffChunk);
	unsigned char *d = o + header_len + a + counts[(size_t) blockIdx.y * max_chunks + c];
	for (unsigned long long i = a; i < e; i++) {
		const unsigned char v = p[i];
		*d++ = v;
		if (v == 0xFF)
			*d++ = 0;
	}
	if (c == 0) {
		o[len - 2] = 0xFF;
		o[len - 1] = 0xD9;
	}
}

} // namespace

/* n equally sized 8-bit frames (1 or 3 bands) on the device -> n JPEG streams at out + i * out_stride (device), their
 * lengths to lengths_host[n].  Stream-ordered on s; returns after the lengths are known.
 */
int
dev_jpeg_encode_batch(const char *domain, const void *frames, size_t bpl, size_t frame_stride, int n, int w, int h, int bands, int quality,
	int subsample_mode, void *out, size_t out_stride, size_t *lengths_host, cudaStream_t s)
{
	EncodeGeom G;
	if (make_geom(domain, w, h, bands, quality, subsample_mode, &G))
		return -1;
	if ((size_t) G.blocks * kMaxBlockBytes >= (size_t) 1 << 29) {
		error(domain, "frame too large for the device encoder");
		return -1;
	}
	EncodeTables T;
	make_tables(quality, &T);
	std::vector<unsigned char> header;
	write_headers(G, T, header);
	const size_t raw_bytes = (((size_t) G.blocks * kMaxBlockBytes + 3) & ~(size_t) 3) + 4;
	const int max_chunks = (int) ((raw_bytes + kStuffChunk - 1) / kStuffChunk);
	/* one block of device scratch: tables | header | coefficients | bit counts / offsets | totals | lengths | raw | span counts */
	size_t off = 0;
	auto take = [&](size_t bytes) {
		const size_t o = off;
		off += (bytes + 255) & ~(size_t) 255;
		return o;
	};
	const size_t o_tab = take(sizeof(T)), o_hdr = take(header.size()), o_coef = take((size_t) n * G.blocks * 64 * sizeof(short)),
				 o_bits = take((size_t) n * G.blocks * sizeof(unsigned)), o_tot = take((size_t) n * sizeof(unsigned long long)),
				 o_len = take((size_t) n * sizeof(unsigned long long)), o_raw = take((size_t) n * raw_bytes),
				 o_cnt = take((size_t) n * max_chunks * sizeof(unsigned));
	char *scratch = nullptr;
	if (dev_alloc(domain, (void **) &scratch, off, s))
		return -1;
	int rc = -1;
	do {
		/* tables and header from pageable memory: small, staged by the driver before the call returns */
		if (cudaMemcpyAsync(scratch + o_tab, &T, sizeof(T), cudaMemcpyHostToDevice, s) != cudaSuccess ||
			cudaMemcpyAsync(scratch + o_hdr, header.data(), header.size(), cudaMemcpyHostToDevice, s) != cudaSuccess ||
			cudaMemsetAsync(scratch + o_raw, 0, (size_t) n * raw_bytes, s) != cudaSuccess) {
			cuda_fail(domain, cudaGetLastError(), "jpeg encode setup");
			break;
		}
		const EncodeTables *dT = (const EncodeTables *) (scratch + o_tab);
		short *coef = (short *) (scratch + o_coef);
		unsigned *bits = (unsigned *) (scratch + o_bits);
		unsigned long long *totals = (unsigned long long *) (scratch + o_tot), *lengths = (unsigned long long *) (scratch + o_len);
		unsigned *counts = (unsigned *) (scratch + o_cnt);
		const int mcus = G.mcus_x * G.mcus_y;
		/* the frame is gridDim.y (or x) of every kernel: chunks of at most kMaxBatchFrames, each on its slice of the scratch */
		cudaError_t e = cudaSuccess;
		for (int c0 = 0; c0 < n && e == cudaSuccess; c0 += kMaxBatchFrames) {
			const int cn = std::min(kMaxBatchFrames, n - c0);
			short *ccoef = coef + (size_t) c0 * G.blocks * 64;
			unsigned *cbits = bits + (size_t) c0 * G.blocks;
			unsigned long long *ctotals = totals + c0, *clengths = lengths + c0;
			unsigned char *craw = (unsigned char *) (scratch + o_raw) + (size_t) c0 * raw_bytes;
			unsigned *ccounts = counts + (size_t) c0 * max_chunks;
			jpeg_fdct_kernel<<<dim3((mcus + 127) / 128, cn), 128, 0, s>>>(G, dT, (const unsigned char *) frames + (size_t) c0 * frame_stride, bpl,
				frame_stride, ccoef);
			jpeg_count_kernel<<<dim3((G.blocks + 127) / 128, cn), 128, 0, s>>>(G, dT, ccoef, cbits);
			jpeg_bitscan_kernel<<<cn, 1024, 0, s>>>(G.blocks, cbits, ctotals);
			jpeg_emit_kernel<<<dim3((G.blocks + 127) / 128, cn), 128, 0, s>>>(G, dT, ccoef, cbits, ctotals, (unsigned *) craw, raw_bytes / 4);
			jpeg_ffcount_kernel<<<dim3((max_chunks + 127) / 128, cn), 128, 0, s>>>(ctotals, craw, raw_bytes, max_chunks, ccounts);
			jpeg_ffscan_kernel<<<cn, 1024, 0, s>>>(ctotals, max_chunks, ccounts, (unsigned) header.size(), clengths);
			jpeg_stuff_kernel<<<dim3((max_chunks + 127) / 128, cn), 128, 0, s>>>(ctotals, craw, raw_bytes, max_chunks, ccounts,
				(const unsigned char *) (scratch + o_hdr), (unsigned) header.size(), (unsigned char *) out + (size_t) c0 * out_stride, out_stride,
				clengths);
			e = cudaGetLastError();
			if (e == cudaSuccess)
				for (int k = 0; k < 7; k++)
					count_launch();
		}
		if (e != cudaSuccess) {
			cuda_fail(domain, e, "jpeg encode kernels launch");
			break;
		}
		std::vector<unsigned long long> len(n);
		if (cudaMemcpyAsync(len.data(), lengths, (size_t) n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
			cudaStreamSynchronize(s) != cudaSuccess) {
			cuda_fail(domain, cudaGetLastError(), "jpeg encode");
			break;
		}
		rc = 0;
		for (int i = 0; i < n; i++) {
			if (lengths_host)
				lengths_host[i] = (size_t) len[i];
			if (len[i] > out_stride) {
				error(domain, "frame %d: the stream takes %llu bytes, the output stride is %zu", i, len[i], out_stride);
				rc = -1;
			}
		}
	} while (0);
	dev_free(scratch, s);
	return rc;
}

/* the whole encoder on the CPU through the same per-block code: test hook */
int
host_jpeg_encode(const char *domain, const unsigned char *img, size_t bpl, int w, int h, int bands, int quality, int subsample_mode,
	std::vector<unsigned char> &out)
{
	EncodeGeom G;
	if (make_geom(domain, w, h, bands, quality, subsample_mode, &G))
		return -1;
	EncodeTables T;
	make_tables(quality, &T);
	std::vector<short> coef((size_t) G.blocks * 64);
	for (int my = 0; my < G.mcus_y; my++)
		for (int mx = 0; mx < G.mcus_x; mx++)
			encode_mcu(G, T.q, img, bpl, mx, my, coef.data() + ((size_t) my * G.mcus_x + mx) * G.blocks_per_mcu * 64);
	write_headers(G, T, out);
	unsigned long long acc = 0;
	int nacc = 0;
	auto flush_byte = [&](unsigned char b) {
		out.push_back(b);
		if (b == 0xFF)
			out.push_back(0);
	};
	auto emit = [&](unsigned code, int len) {
		acc = (acc << len) | code;
		nacc += len;
		while (nacc >= 8) {
			flush_byte((unsigned char) (acc >> (nacc - 8)));
			nacc -= 8;
		}
	};
	for (unsigned b = 0; b < (unsigned) G.blocks; b++)
		code_block(T, coef.data() + (size_t) b * 64, block_comp(G, (int) (b % (unsigned) G.blocks_per_mcu)), previous_dc(G, coef.data(), b), emit);
	if (nacc > 0)
		flush_byte((unsigned char) (((acc << (8 - nacc)) | ((1u << (8 - nacc)) - 1)) & 0xFF));
	put16(out, 0xFFD9);
	return 0;
}

} // namespace vb200

using namespace vb200;

/* Test hook, host only: vips_jpegsave_buffer's stream for an 8-bit 1- or 3-band image through the encoder's per-block code
 * on the CPU.  subsample_mode: 0 auto (4:2:0 below Q 90), 1 on, 2 off (VipsForeignSubsample).  *len = bytes written;
 * -1 with the size needed in *len when cap is too small.
 */
extern "C" int
vb200_debug_jpeg_encode(const void *pixels, size_t bpl, int width, int height, int bands, int quality, int subsample_mode, void *out, size_t cap,
	size_t *len)
{
	std::vector<unsigned char> o;
	if (host_jpeg_encode("jpeg_encode (host twin)", (const unsigned char *) pixels, bpl, width, height, bands, quality, subsample_mode, o))
		return -1;
	if (len)
		*len = o.size();
	if (!out || cap < o.size()) {
		error("jpeg_encode (host twin)", "output buffer too small: %zu bytes needed", o.size());
		return -1;
	}
	memcpy(out, o.data(), o.size());
	return 0;
}

/* vips_jpegsave_buffer (foreign/vips2jpeg.c) for a batch of equally sized 8-bit frames (1 or 3 bands), on the device:
 * frames in host or device memory (frames_location), n streams to out + i * out_stride in host or device memory
 * (out_location), lengths[n] on the host.  Q and subsample_mode as the reference's arguments (0 auto, 1 on, 2 off);
 * everything else is the reference's default (baseline, standard Huffman tables, JFIF header).
 */
extern "C" int
vb200_jpegsave_batch(const void *frames, int frames_location, size_t bpl, size_t frame_stride, int n, int width, int height, int bands, int Q,
	int subsample_mode, void *out, int out_location, size_t out_stride, size_t *lengths)
{
	const char *domain = "jpegsave_batch";
	if (!frames || !out || n < 1) {
		error(domain, "null argument");
		return -1;
	}
	if (ensure_init(domain))
		return -1;
	cudaStream_t s = current_stream();
	const size_t line = (size_t) width * bands;
	if (bpl < line || (n > 1 && frame_stride < bpl * height)) {
		error(domain, "frame strides too small for %d x %d x %d", width, height, bands);
		return -1;
	}
	void *din = nullptr, *dout = nullptr;
	int rc = -1;
	do {
		const void *src = frames;
		size_t sbpl = bpl, sstride = frame_stride;
		if (frames_location != VB200_DEVICE) {
			if (dev_alloc(domain, &din, line * height * n, s))
				break;
			bool bad = false;
			for (int i = 0; i < n && !bad; i++)
				bad = cudaMemcpy2DAsync((char *) din + (size_t) i * line * height, line, (const char *) frames + (size_t) i * frame_stride, bpl, line,
						  height, cudaMemcpyHostToDevice, s) != cudaSuccess;
			if (bad) {
				cuda_fail(domain, cudaGetLastError(), "copy to device");
				break;
			}
			src = din;
			sbpl = line;
			sstride = line * height;
		}
		void *dst = out;
		if (out_location != VB200_DEVICE) {
			if (dev_alloc(domain, &dout, out_stride * n, s))
				break;
			dst = dout;
		}
		std::vector<size_t> len(n);
		if (dev_jpeg_encode_batch(domain, src, sbpl, sstride, n, width, height, bands, Q, subsample_mode, dst, out_stride, len.data(), s))
			break;
		if (lengths)
			memcpy(lengths, len.data(), n * sizeof(size_t));
		if (out_location != VB200_DEVICE) {
			bool bad = false;
			for (int i = 0; i < n && !bad; i++)
				bad = cudaMemcpyAsync((char *) out + (size_t) i * out_stride, (char *) dout + (size_t) i * out_stride, len[i], cudaMemcpyDeviceToHost,
						  s) != cudaSuccess;
			if (bad || cudaStreamSynchronize(s) != cudaSuccess) {
				cuda_fail(domain, cudaGetLastError(), "copy to host");
				break;
			}
		}
		rc = 0;
	} while (0);
	if (din)
		dev_free(din, s);
	if (dout)
		dev_free(dout, s);
	return rc;
}

