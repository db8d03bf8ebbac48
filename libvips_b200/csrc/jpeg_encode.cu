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
 * With vips_jpegsave's options (vips2jpeg.c:590-597):
 *   optimize_coding        jpeg_stats_kernel (symbol counts per frame) and jpeg_huffopt_kernel (jchuff.c
 *                          jpeg_gen_optimal_table per table, the frame's code tables and header) after the FDCT; the count,
 *                          emit and stuffing kernels then take the frame's tables and header
 *   restart_interval       jpeg_intervals_kernel after the bit prefix sum: every interval starts on a byte boundary, the
 *                          stuffing kernels put FF Dn before each interval after the first
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

/* jchuff.c jpeg_make_c_derived_tbl: canonical codes from (bits, values); bits[l - 1] codes of length l */
HD void
derive_codes(const unsigned char bits[16], const unsigned char *vals, unsigned *co, unsigned char *si)
{
	for (int i = 0; i < 256; i++) {
		co[i] = 0;
		si[i] = 0;
	}
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

/* Walk one block's symbols in jchuff.c's order (encode_one_block, and htest_one_block for the statistics): sym(table,
 * symbol) for every Huffman-coded symbol -- table 0 DC, 1 AC, 2 / 3 the same for chroma --, extra(value, n) for the n
 * magnitude bits that follow it
 */
template <typename Sym, typename Extra>
HD void
walk_block(const unsigned char *zz, const short *blk, int comp, int prev_dc, Sym sym, Extra extra)
{
	const int dt = comp ? 2 : 0, at = dt + 1;
	int diff = blk[0] - prev_dc;
	int t2 = diff;
	if (diff < 0) {
		diff = -diff;
		t2--; /* one's complement of the magnitude for negative values (F.1.2.1) */
	}
	int nb = bit_size(diff);
	sym(dt, nb);
	if (nb)
		extra((unsigned) t2 & ((1u << nb) - 1), nb);
	int run = 0;
	for (int k = 1; k < 64; k++) {
		int v = blk[zz[k]];
		if (v == 0) {
			run++;
			continue;
		}
		while (run > 15) {
			sym(at, 0xF0);
			run -= 16;
		}
		t2 = v;
		if (v < 0) {
			v = -v;
			t2--;
		}
		nb = bit_size(v);
		sym(at, (run << 4) + nb);
		extra((unsigned) t2 & ((1u << nb) - 1), nb);
		run = 0;
	}
	if (run > 0)
		sym(at, 0);
}

/* Code one block: emit(code, length) for every Huffman code and its extra bits, with the code / length tables co / si
 * (the batch's standard tables, or a frame's optimised ones); returns the bit count
 */
template <typename Emit>
HD unsigned
code_block(const unsigned (*co)[256], const unsigned char (*si)[256], const unsigned char *zz, const short *blk, int comp, int prev_dc, Emit emit)
{
	unsigned bits = 0;
	walk_block(
		zz, blk, comp, prev_dc,
		[&](int t, int s) {
			emit(co[t][s], si[t][s]);
			bits += si[t][s];
		},
		[&](unsigned v, int n) {
			emit(v, n);
			bits += n;
		});
	return bits;
}

/* The DC value the block's difference is taken against: the previous block of its component in scan order.  restart:
 * MCUs per restart interval (0: none); the first block of each component in an MCU that starts an interval predicts
 * from 0 (jchuff.c: emit_restart, and encode_mcu_gather in the statistics pass, reset last_dc_val)
 */
HD int
previous_dc(const EncodeGeom &G, const short *coef, unsigned blk, int restart)
{
	const int nb = G.blocks_per_mcu;
	const unsigned mcu = blk / (unsigned) nb;
	const int bi = (int) (blk - mcu * (unsigned) nb);
	if (G.ncomp == 3 && G.sub && bi >= 1 && bi <= 3)
		return coef[(size_t) (blk - 1) * 64]; /* luma blocks 1..3 follow luma block bi - 1 */
	if (mcu == 0 || (restart > 0 && mcu % (unsigned) restart == 0))
		return 0;
	/* the last block of the component in the previous MCU */
	const int last = (G.ncomp == 3 && G.sub && bi == 0) ? 3 : bi;
	return coef[((size_t) (mcu - 1) * nb + last) * 64];
}

/* ------------------------------------------------------------------ optimised Huffman tables (host + device) */

constexpr unsigned kFreqSentinel = 1000000000u; /* jchuff.c jpeg_gen_optimal_table: v = 1000000000L */
constexpr int kMaxCodeLen = 32;					/* MAX_CLEN: the longest code before the 16-bit limit */

/* Huffman tables of one frame when it is coded with its own: code / length per symbol, tables as in EncodeTables */
struct FrameHuff {
	unsigned ehufco[4][256];
	unsigned char ehufsi[4][256];
};

/* jchuff.c jpeg_gen_optimal_table, restated.  freq[257] holds the symbol counts and is consumed (freq[256], the reserved
 * all-ones code, is set to 1 here); codesize / others [257] are scratch; bits[17] (bits[l]: codes of length l, bits[0]
 * unused) and huffval[256] receive the table.
 * pick(exclude) returns the LARGEST index i != exclude whose freq[i] is the smallest in (0, kFreqSentinel], or -1 (libjpeg
 * scans upwards with freq[i] <= v, so a tie goes to the larger index): a serial scan on the host, a warp reduction on the
 * device.  All other work runs on the lead thread; the other lanes take part in pick only.
 * huffval is ordered by code size BEFORE the 16-bit limit, then by symbol, as libjpeg orders it: after the limit it need
 * not be ordered by final length.  Returns -1 when a code would be longer than 32 bits (JERR_HUFF_CLEN_OVERFLOW).
 */
template <typename Pick>
HD int
gen_optimal_table(unsigned *freq, int *codesize, int *others, unsigned char *bits, unsigned char *huffval, bool lead, Pick pick)
{
	if (lead) {
		for (int i = 0; i < 257; i++) {
			codesize[i] = 0;
			others[i] = -1;
		}
		freq[256] = 1;
	}
	for (;;) {
		int c1 = pick(-1);
		int c2 = pick(c1);
		if (c2 < 0)
			break;
		if (lead) {
			freq[c1] += freq[c2];
			freq[c2] = 0;
			codesize[c1]++;
			while (others[c1] >= 0) {
				c1 = others[c1];
				codesize[c1]++;
			}
			others[c1] = c2;
			codesize[c2]++;
			while (others[c2] >= 0) {
				c2 = others[c2];
				codesize[c2]++;
			}
		}
	}
	if (!lead)
		return 0;
	unsigned char b[kMaxCodeLen + 1]; /* UINT8, as libjpeg counts them */
	for (int i = 0; i <= kMaxCodeLen; i++)
		b[i] = 0;
	for (int i = 0; i <= 256; i++)
		if (codesize[i]) {
			if (codesize[i] > kMaxCodeLen)
				return -1;
			b[codesize[i]]++;
		}
	/* JPEG codes are at most 16 bits: move pairs of the longest codes up (T.81 Annex K.3 Figure K.3) */
	for (int i = kMaxCodeLen; i > 16; i--)
		while (b[i] > 0) {
			int j = i - 2;
			while (b[j] == 0)
				j--;
			b[i] -= 2;
			b[i - 1]++;
			b[j + 1] += 2;
			b[j]--;
		}
	/* drop the reserved symbol's code: one of the longest */
	int i = 16;
	while (b[i] == 0)
		i--;
	b[i]--;
	for (int l = 0; l <= 16; l++)
		bits[l] = b[l];
	/* symbols 0..255 by pre-limit code size, then by value: a counting sort of libjpeg's size-major double loop */
	int start[kMaxCodeLen + 1];
	for (int l = 0; l <= kMaxCodeLen; l++)
		start[l] = 0;
	for (int j = 0; j < 256; j++)
		if (codesize[j])
			start[codesize[j]]++;
	for (int l = 1, p = 0; l <= kMaxCodeLen; l++) {
		const int c = start[l];
		start[l] = p;
		p += c;
	}
	for (int j = 0; j < 256; j++)
		if (codesize[j])
			huffval[start[codesize[j]]++] = (unsigned char) j;
	return 0;
}

/* the symbols a table holds: the sum of bits[1..16] */
HD int
table_values(const unsigned char *bits)
{
	int n = 0;
	for (int l = 1; l <= 16; l++)
		n += bits[l];
	return n;
}

/* jcmarker.c emit_dht: table t (0 DC lum, 1 AC lum, 2 DC chr, 3 AC chr) with bits[1..16] / huffval; returns its bytes */
HD int
put_dht(unsigned char *o, int t, const unsigned char *bits, const unsigned char *huffval)
{
	const int nv = table_values(bits);
	const int len = 19 + nv;
	o[0] = 0xFF;
	o[1] = 0xC4;
	o[2] = (unsigned char) (len >> 8);
	o[3] = (unsigned char) len;
	o[4] = (unsigned char) (((t & 1) << 4) | (t >> 1));
	for (int l = 1; l <= 16; l++)
		o[4 + l] = bits[l];
	for (int k = 0; k < nv; k++)
		o[21 + k] = huffval[k];
	return 2 + len;
}

/* ------------------------------------------------------------------ stream assembly (host) */

void
put16(std::vector<unsigned char> &o, unsigned v)
{
	o.push_back((unsigned char) (v >> 8));
	o.push_back((unsigned char) v);
}

/* the markers before the Huffman tables, in libjpeg's order: SOI, JFIF APP0, DQT per table, SOF0 */
void
header_prefix(const EncodeGeom &G, const EncodeTables &T, std::vector<unsigned char> &o)
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
}

/* the markers after the Huffman tables: DRI when there are restart intervals (jcmarker.c write_scan_header: after the
 * DHTs, before SOS, also when the interval covers the whole frame), then SOS
 */
void
header_suffix(const EncodeGeom &G, int restart, std::vector<unsigned char> &o)
{
	if (restart > 0) {
		put16(o, 0xFFDD);
		put16(o, 4);
		put16(o, (unsigned) restart);
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

/* one frame's DHT segments: tables 0..3 (0 and 1 only for greyscale), bits[t][1..16] / huffval[t] */
void
put_dhts(const EncodeGeom &G, const unsigned char (*bits)[17], const unsigned char (*huffval)[256], std::vector<unsigned char> &o)
{
	for (int t = 0; t < (G.ncomp == 1 ? 2 : 4); t++) {
		unsigned char seg[4 + 17 + 256];
		const int n = put_dht(seg, t, bits[t], huffval[t]);
		o.insert(o.end(), seg, seg + n);
	}
}

/* the standard tables (T.81 Annex K.3) in put_dhts' form */
void
standard_tables(unsigned char (*bits)[17], unsigned char (*huffval)[256])
{
	const unsigned char *b[4] = {kBitsDcLum, kBitsAcLum, kBitsDcChr, kBitsAcChr};
	const unsigned char *v[4] = {kValDc, kValAcLum, kValDc, kValAcChr};
	for (int t = 0; t < 4; t++) {
		bits[t][0] = 0;
		memcpy(bits[t] + 1, b[t], 16);
		memcpy(huffval[t], v[t], (size_t) table_values(bits[t]));
	}
}

/* everything up to and including SOS with the standard Huffman tables, in libjpeg's order: SOI, JFIF APP0, DQT per
 * table, SOF0, DHT per table, DRI when restart > 0, SOS
 */
void
write_headers(const EncodeGeom &G, const EncodeTables &T, int restart, std::vector<unsigned char> &o)
{
	unsigned char bits[4][17], huffval[4][256];
	standard_tables(bits, huffval);
	header_prefix(G, T, o);
	put_dhts(G, bits, huffval, o);
	header_suffix(G, restart, o);
}

/* restart_interval as vips_jpegsave takes it (jpegsave.c:284-289): 0 for none.  The reference passes larger values
 * on to libjpeg, which writes DRI modulo 65536 but spaces the markers by the full value: a stream no reader can follow,
 * so they are refused here.
 */
int
check_restart(const char *domain, int restart)
{
	if (restart < 0 || restart > 65535) {
		error(domain, "restart_interval %d outside 0..65535", restart);
		return -1;
	}
	return 0;
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
/* a table counts at most 64 symbols per block (a DC category, or 63 AC symbols + EOB), and frames are refused from
 * 2^29 / kMaxBlockBytes blocks on: every count, and every sum of counts, stays below libjpeg's search sentinel
 */
static_assert(((1u << 29) / kMaxBlockBytes) * 64u + 1u < kFreqSentinel, "symbol counts must stay below the sentinel");
/* a frame's header with its own tables: SOI + APP0 + 2 DQT + SOF0 (177 bytes for 3 components) + 4 DHT (84 bytes + at
 * most 12 DC and 162 AC symbols per table pair) + DRI + SOS (20) = 629 bytes at most; a larger one fails the frame
 */
constexpr int kHeaderSlot = 640;

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

/* the Huffman tables a block of frame f is coded with: the batch's standard ones, or the frame's own */
template <bool kFrameHuff>
__device__ __forceinline__ void
frame_tables(const EncodeTables *T, const FrameHuff *huff, unsigned f, const unsigned (**co)[256], const unsigned char (**si)[256])
{
	if (kFrameHuff) {
		*co = huff[f].ehufco;
		*si = huff[f].ehufsi;
	}
	else {
		*co = T->ehufco;
		*si = T->ehufsi;
	}
}

/* optimise_coding, pass 1 (jchuff.c encode_mcu_gather): one thread per block walks its symbols into the CTA's
 * histograms (4 tables x 256 symbols; Cb and Cr share tables 2 / 3), then the non-zero bins are added to the frame's
 * counts[frame][4][256]
 */
__global__ void __launch_bounds__(128)
jpeg_stats_kernel(const EncodeGeom G, const EncodeTables *__restrict__ T, const short *__restrict__ coef, int restart, unsigned *__restrict__ counts)
{
	__shared__ unsigned s_hist[4 * 256];
	for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x)
		s_hist[i] = 0;
	__syncthreads();
	const unsigned b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b < (unsigned) G.blocks) {
		const short *fc = coef + (size_t) blockIdx.y * G.blocks * 64;
		walk_block(
			T->zz, fc + (size_t) b * 64, block_comp(G, (int) (b % (unsigned) G.blocks_per_mcu)), previous_dc(G, fc, b, restart),
			[&](int t, int s) { atomicAdd(&s_hist[t * 256 + s], 1u); }, [](unsigned, int) {});
	}
	__syncthreads();
	unsigned *dst = counts + (size_t) blockIdx.y * 4 * 256;
	for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x)
		if (s_hist[i])
			atomicAdd(dst + i, s_hist[i]);
}

/* optimise_coding, pass 2: one CTA per frame, one warp per table (tables 0, 1 for greyscale).  Each warp runs
 * gen_optimal_table on its counts with a warp-wide minimum search, writes the frame's code / length table, and the CTA
 * then writes the frame's header -- prefix (SOI .. SOF0), its own DHTs, suffix (DRI, SOS) -- into its kHeaderSlot-byte
 * slot and the header's length into header_lens[frame].  A frame whose tables cannot be built sets *bad.
 */
__global__ void __launch_bounds__(128)
jpeg_huffopt_kernel(int ntab, const unsigned *__restrict__ counts, FrameHuff *__restrict__ huff, const unsigned char *__restrict__ prefix,
	unsigned prefix_len, const unsigned char *__restrict__ suffix, unsigned suffix_len, unsigned char *__restrict__ headers,
	unsigned *__restrict__ header_lens, int *__restrict__ bad)
{
	__shared__ unsigned s_freq[4][257];
	__shared__ int s_size[4][257], s_others[4][257];
	__shared__ unsigned char s_bits[4][17], s_val[4][256];
	__shared__ int s_fail;
	const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const unsigned *cnt = counts + (size_t) blockIdx.x * 4 * 256;
	if (threadIdx.x == 0)
		s_fail = 0;
	for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x)
		s_freq[i >> 8][i & 255] = cnt[i];
	__syncthreads();
	FrameHuff *fh = huff + blockIdx.x;
	if (w < ntab) {
		unsigned *freq = s_freq[w];
		auto pick = [&](int exclude) {
			__syncwarp();
			/* key: frequency, then the larger index first */
			unsigned long long best = ~0ull;
			for (int i = lane; i <= 256; i += 32) {
				const unsigned f = freq[i];
				if (f && f <= kFreqSentinel && i != exclude) {
					const unsigned long long key = ((unsigned long long) f << 9) | (unsigned) (511 - i);
					best = key < best ? key : best;
				}
			}
			for (int o = 16; o; o >>= 1) {
				const unsigned long long v = __shfl_xor_sync(0xffffffffu, best, o);
				best = v < best ? v : best;
			}
			return best == ~0ull ? -1 : 511 - (int) (best & 511u);
		};
		if (gen_optimal_table(freq, s_size[w], s_others[w], s_bits[w], s_val[w], lane == 0, pick))
			s_fail = 1;
		__syncwarp();
		if (lane == 0)
			derive_codes(s_bits[w] + 1, s_val[w], fh->ehufco[w], fh->ehufsi[w]);
	}
	__syncthreads();
	unsigned len = prefix_len + suffix_len;
	for (int t = 0; t < ntab; t++)
		len += 21 + table_values(s_bits[t]);
	if (s_fail || len > kHeaderSlot) {
		if (threadIdx.x == 0) {
			header_lens[blockIdx.x] = 0;
			atomicExch(bad, 1);
		}
		return;
	}
	unsigned char *o = headers + (size_t) blockIdx.x * kHeaderSlot;
	for (unsigned i = threadIdx.x; i < prefix_len; i += blockDim.x)
		o[i] = prefix[i];
	for (unsigned i = threadIdx.x; i < suffix_len; i += blockDim.x)
		o[len - suffix_len + i] = suffix[i];
	if (w < ntab && lane == 0) {
		unsigned at = prefix_len;
		for (int t = 0; t < w; t++)
			at += 21 + table_values(s_bits[t]);
		put_dht(o + at, w, s_bits[w], s_val[w]);
	}
	if (threadIdx.x == 0)
		header_lens[blockIdx.x] = len;
}

/* one thread per block: how many bits its code takes */
template <bool kFrameHuff, bool kRestart>
__global__ void __launch_bounds__(128)
jpeg_count_kernel(const EncodeGeom G, const EncodeTables *__restrict__ T, const FrameHuff *__restrict__ huff, int restart,
	const short *__restrict__ coef, unsigned *__restrict__ bits)
{
	const unsigned b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= (unsigned) G.blocks)
		return;
	const short *fc = coef + (size_t) blockIdx.y * G.blocks * 64;
	const unsigned (*co)[256];
	const unsigned char (*si)[256];
	frame_tables<kFrameHuff>(T, huff, blockIdx.y, &co, &si);
	bits[(size_t) blockIdx.y * G.blocks + b] = code_block(co, si, T->zz, fc + (size_t) b * 64, block_comp(G, (int) (b % (unsigned) G.blocks_per_mcu)),
		previous_dc(G, fc, b, kRestart ? restart : 0), [](unsigned, int) {});
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

/* restart intervals, one CTA per frame: each interval takes its blocks' bits rounded up to a whole byte (the 1-padding
 * before each RSTn), istart[frame][k] = the byte where interval k starts in the raw scan (an exclusive prefix sum over
 * intervals), and totals[frame] becomes the padded scan's length in bits (whole bytes)
 */
__global__ void __launch_bounds__(1024)
jpeg_intervals_kernel(int blocks, int blocks_per_interval, int nint, const unsigned *__restrict__ offs, unsigned long long *__restrict__ totals,
	unsigned *__restrict__ istart)
{
	__shared__ unsigned long long s_part[1024];
	const unsigned *o = offs + (size_t) blockIdx.x * blocks;
	unsigned *st = istart + (size_t) blockIdx.x * nint;
	const unsigned long long total = totals[blockIdx.x];
	auto ibytes = [&](unsigned k) {
		const unsigned long long b0 = o[(size_t) k * blocks_per_interval];
		const unsigned long long b1 = k + 1 < (unsigned) nint ? o[(size_t) (k + 1) * blocks_per_interval] : total;
		return (b1 - b0 + 7) >> 3;
	};
	const unsigned per = ((unsigned) nint + blockDim.x - 1) / blockDim.x;
	const unsigned a = min((unsigned) nint, threadIdx.x * per), e = min((unsigned) nint, a + per);
	unsigned long long sum = 0;
	for (unsigned k = a; k < e; k++)
		sum += ibytes(k);
	s_part[threadIdx.x] = sum;
	__syncthreads();
	for (unsigned d = 1; d < blockDim.x; d <<= 1) {
		const unsigned long long v = threadIdx.x >= d ? s_part[threadIdx.x - d] : 0;
		__syncthreads();
		s_part[threadIdx.x] += v;
		__syncthreads();
	}
	unsigned long long run = s_part[threadIdx.x] - sum;
	for (unsigned k = a; k < e; k++) {
		st[k] = (unsigned) run;
		run += ibytes(k);
	}
	if (threadIdx.x == blockDim.x - 1)
		totals[blockIdx.x] = s_part[threadIdx.x] * 8;
}

/* the number of the n ascending values p[] below v */
__device__ __forceinline__ int
count_below(const unsigned *p, int n, unsigned long long v)
{
	int lo = 0, hi = n;
	while (lo < hi) {
		const int mid = (lo + hi) >> 1;
		if (p[mid] < v)
			lo = mid + 1;
		else
			hi = mid;
	}
	return lo;
}

/* one thread per block: its bits into the frame's (zeroed) raw bit buffer, whole bytes OR-ed in (neighbouring blocks share
 * their boundary bytes); the thread that ends the frame -- with restart intervals, each interval -- also pads the last
 * byte with 1-bits.  With restart intervals a block's bit offset is relative to its interval, which starts at byte
 * istart[frame][k].
 */
template <bool kFrameHuff, bool kRestart>
__global__ void __launch_bounds__(128)
jpeg_emit_kernel(const EncodeGeom G, const EncodeTables *__restrict__ T, const FrameHuff *__restrict__ huff, int restart, int nint,
	const unsigned *__restrict__ istart, const short *__restrict__ coef, const unsigned *__restrict__ offs, unsigned *__restrict__ raw,
	size_t raw_words)
{
	const unsigned b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= (unsigned) G.blocks)
		return;
	const short *fc = coef + (size_t) blockIdx.y * G.blocks * 64;
	unsigned *out = raw + (size_t) blockIdx.y * raw_words;
	const unsigned *fo = offs + (size_t) blockIdx.y * G.blocks;
	unsigned pos = fo[b]; /* bit index */
	bool last = b == (unsigned) G.blocks - 1;
	if (kRestart) {
		const unsigned bpm = (unsigned) G.blocks_per_mcu, mcu = b / bpm, k = mcu / (unsigned) restart;
		pos += istart[(size_t) blockIdx.y * nint + k] * 8 - fo[k * (unsigned) restart * bpm];
		last = last || (b - mcu * bpm == bpm - 1 && (mcu + 1) % (unsigned) restart == 0);
	}
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
	const unsigned (*co)[256];
	const unsigned char (*si)[256];
	frame_tables<kFrameHuff>(T, huff, blockIdx.y, &co, &si);
	code_block(co, si, T->zz, fc + (size_t) b * 64, block_comp(G, (int) (b % (unsigned) G.blocks_per_mcu)), previous_dc(G, fc, b, kRestart ? restart : 0),
		put);
	if (nacc > 0) {
		unsigned v = (unsigned) (acc << (8 - nacc)) & 0xffu;
		if (last)
			v |= (1u << (8 - nacc)) - 1; /* jchuff.c flush_bits: pad the last byte with ones */
		if (v)
			atomicOr(out + (byte >> 2), v << (8 * (byte & 3u)));
	}
}

/* stuffing, pass 1: 0xFF bytes per kStuffChunk-byte span of each frame's raw scan; with restart intervals, plus 2 bytes
 * for every RSTn marker that goes before a byte of the span (interval starts 1 .. nint - 1)
 */
template <bool kRestart>
__global__ void __launch_bounds__(128)
jpeg_ffcount_kernel(const unsigned long long *__restrict__ totals, const unsigned char *__restrict__ raw, size_t raw_bytes, int max_chunks,
	int nint, const unsigned *__restrict__ istart, unsigned *__restrict__ counts)
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
	if (kRestart && a < e) {
		const unsigned *st = istart + (size_t) blockIdx.y * nint + 1;
		n += 2 * (unsigned) (count_below(st, nint - 1, e) - count_below(st, nint - 1, a));
	}
	counts[(size_t) blockIdx.y * max_chunks + c] = n;
}

/* stuffing, pass 2: prefix sum of the spans' counts, one CTA per frame; lengths[frame] = header + scan + stuffed zeros +
 * markers + EOI.  The header is the batch's (header_len) or, with optimised tables, the frame's (header_lens[frame]).
 */
template <bool kFrameHeader>
__global__ void __launch_bounds__(1024)
jpeg_ffscan_kernel(const unsigned long long *__restrict__ totals, int max_chunks, unsigned *__restrict__ counts, unsigned header_len,
	const unsigned *__restrict__ header_lens, unsigned long long *__restrict__ lengths)
{
	if (kFrameHeader)
		header_len = header_lens[blockIdx.x];
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
 * compares lengths[frame] with the stride and reports it).  With optimised tables the header is the frame's slot of
 * kHeaderSlot bytes; with restart intervals FF D0+((k - 1) & 7) goes before the first byte of interval k >= 1 (padding
 * bytes are stuffed, markers are not).
 */
template <bool kFrameHeader, bool kRestart>
__global__ void __launch_bounds__(128)
jpeg_stuff_kernel(const unsigned long long *__restrict__ totals, const unsigned char *__restrict__ raw, size_t raw_bytes, int max_chunks,
	const unsigned *__restrict__ counts, const unsigned char *__restrict__ header, unsigned header_len, const unsigned *__restrict__ header_lens,
	int nint, const unsigned *__restrict__ istart, unsigned char *__restrict__ out, size_t out_stride, const unsigned long long *__restrict__ lengths)
{
	const int c = blockIdx.x * blockDim.x + threadIdx.x;
	unsigned char *o = out + (size_t) blockIdx.y * out_stride;
	const unsigned long long len = lengths[blockIdx.y];
	if (len > out_stride)
		return;
	if (kFrameHeader) {
		header += (size_t) blockIdx.y * kHeaderSlot;
		header_len = header_lens[blockIdx.y];
	}
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
	const unsigned *st = istart + (size_t) blockIdx.y * nint;
	int k = kRestart && a < e ? 1 + count_below(st + 1, nint - 1, a) : 0; /* the next interval starting in the span */
	for (unsigned long long i = a; i < e; i++) {
		const unsigned char v = p[i];
		if (kRestart && k < nint && st[k] == i) {
			*d++ = 0xFF;
			*d++ = (unsigned char) (0xD0 + ((k - 1) & 7));
			k++;
		}
		*d++ = v;
		if (v == 0xFF)
			*d++ = 0;
	}
	if (c == 0) {
		o[len - 2] = 0xFF;
		o[len - 1] = 0xD9;
	}
}

/* the device buffers of one chunk of frames */
struct ChunkArgs {
	EncodeGeom G;
	const EncodeTables *T;
	const unsigned char *frames;
	size_t bpl, frame_stride;
	int cn, restart, nint, max_chunks;
	short *coef;
	unsigned *bits, *counts, *istart, *freq, *header_lens;
	unsigned long long *totals, *lengths;
	unsigned char *raw;
	size_t raw_bytes;
	FrameHuff *huff;
	const unsigned char *header; /* the batch's header, or with optimised tables the prefix and suffix around the DHTs */
	unsigned header_len, prefix_len, suffix_len;
	unsigned char *headers; /* per-frame header slots */
	int *bad;
	unsigned char *out;
	size_t out_stride;
};

/* the kernels of one chunk: 7 launches with the standard tables and no restart intervals, +1 with restart intervals
 * (jpeg_intervals_kernel), +2 with optimised tables (jpeg_stats_kernel, jpeg_huffopt_kernel); returns the launch count,
 * -1 when the counts could not be cleared
 */
template <bool kOpt, bool kRestart>
int
launch_chunk(const ChunkArgs &A, cudaStream_t s)
{
	const EncodeGeom &G = A.G;
	const int mcus = G.mcus_x * G.mcus_y, cn = A.cn;
	const dim3 per_block((G.blocks + 127) / 128, cn), per_span((A.max_chunks + 127) / 128, cn);
	int launches = 7;
	jpeg_fdct_kernel<<<dim3((mcus + 127) / 128, cn), 128, 0, s>>>(G, A.T, A.frames, A.bpl, A.frame_stride, A.coef);
	if (kOpt) {
		if (cudaMemsetAsync(A.freq, 0, (size_t) cn * 4 * 256 * sizeof(unsigned), s) != cudaSuccess)
			return -1;
		jpeg_stats_kernel<<<per_block, 128, 0, s>>>(G, A.T, A.coef, A.restart, A.freq);
		jpeg_huffopt_kernel<<<cn, 128, 0, s>>>(G.ncomp == 1 ? 2 : 4, A.freq, A.huff, A.header, A.prefix_len, A.header + A.prefix_len, A.suffix_len,
			A.headers, A.header_lens, A.bad);
		launches += 2;
	}
	jpeg_count_kernel<kOpt, kRestart><<<per_block, 128, 0, s>>>(G, A.T, A.huff, A.restart, A.coef, A.bits);
	jpeg_bitscan_kernel<<<cn, 1024, 0, s>>>(G.blocks, A.bits, A.totals);
	if (kRestart) {
		jpeg_intervals_kernel<<<cn, 1024, 0, s>>>(G.blocks, A.restart * G.blocks_per_mcu, A.nint, A.bits, A.totals, A.istart);
		launches++;
	}
	jpeg_emit_kernel<kOpt, kRestart><<<per_block, 128, 0, s>>>(G, A.T, A.huff, A.restart, A.nint, A.istart, A.coef, A.bits, (unsigned *) A.raw,
		A.raw_bytes / 4);
	jpeg_ffcount_kernel<kRestart><<<per_span, 128, 0, s>>>(A.totals, A.raw, A.raw_bytes, A.max_chunks, A.nint, A.istart, A.counts);
	jpeg_ffscan_kernel<kOpt><<<cn, 1024, 0, s>>>(A.totals, A.max_chunks, A.counts, A.header_len, A.header_lens, A.lengths);
	jpeg_stuff_kernel<kOpt, kRestart><<<per_span, 128, 0, s>>>(A.totals, A.raw, A.raw_bytes, A.max_chunks, A.counts, kOpt ? A.headers : A.header,
		A.header_len, A.header_lens, A.nint, A.istart, A.out, A.out_stride, A.lengths);
	return launches;
}

} // namespace

/* n equally sized 8-bit frames (1 or 3 bands) on the device -> n JPEG streams at out + i * out_stride (device), their
 * lengths to lengths_host[n].  optimize: per-frame Huffman tables from the frame's symbol counts; restart: MCUs per
 * restart interval (0: none).  Stream-ordered on s; returns after the lengths are known.
 */
int
dev_jpeg_encode_batch(const char *domain, const void *frames, size_t bpl, size_t frame_stride, int n, int w, int h, int bands, int quality,
	int subsample_mode, int optimize, int restart, void *out, size_t out_stride, size_t *lengths_host, cudaStream_t s)
{
	EncodeGeom G;
	if (make_geom(domain, w, h, bands, quality, subsample_mode, &G) || check_restart(domain, restart))
		return -1;
	const int mcus = G.mcus_x * G.mcus_y;
	const int nint = restart ? (mcus + restart - 1) / restart : 1;
	/* every interval may end with one byte of padding */
	const size_t scan_bound = (size_t) G.blocks * kMaxBlockBytes + (restart ? (size_t) nint : 0);
	if (scan_bound >= (size_t) 1 << 29) {
		error(domain, "frame too large for the device encoder");
		return -1;
	}
	EncodeTables T;
	make_tables(quality, &T);
	/* standard tables: the whole header; optimised tables: the markers before and after the DHTs (prefix_len bytes, then
	 * the suffix), which jpeg_huffopt_kernel puts around each frame's own tables
	 */
	std::vector<unsigned char> header, suffix;
	unsigned prefix_len = 0;
	if (optimize) {
		header_prefix(G, T, header);
		prefix_len = (unsigned) header.size();
		header_suffix(G, restart, suffix);
		header.insert(header.end(), suffix.begin(), suffix.end());
	}
	else
		write_headers(G, T, restart, header);
	const size_t raw_bytes = ((scan_bound + 3) & ~(size_t) 3) + 4;
	const int max_chunks = (int) ((raw_bytes + kStuffChunk - 1) / kStuffChunk);
	/* per-frame tables and header slots (about 10 KB a frame) for one chunk of frames, reused by the next */
	const size_t nopt = optimize ? (size_t) std::min(n, kMaxBatchFrames) : 0;
	/* one block of device scratch: tables | header | coefficients | bit counts / offsets | totals | lengths | raw | span counts
	 * | interval starts | symbol counts | frame tables | header slots | header lengths | failure flag
	 */
	size_t off = 0;
	auto take = [&](size_t bytes) {
		const size_t o = off;
		off += (bytes + 255) & ~(size_t) 255;
		return o;
	};
	const size_t o_tab = take(sizeof(T)), o_hdr = take(header.size()), o_coef = take((size_t) n * G.blocks * 64 * sizeof(short)),
				 o_bits = take((size_t) n * G.blocks * sizeof(unsigned)), o_tot = take((size_t) n * sizeof(unsigned long long)),
				 o_len = take((size_t) n * sizeof(unsigned long long)), o_raw = take((size_t) n * raw_bytes),
				 o_cnt = take((size_t) n * max_chunks * sizeof(unsigned)), o_ist = take(restart ? (size_t) n * nint * sizeof(unsigned) : 0),
				 o_freq = take(nopt * 4 * 256 * sizeof(unsigned)), o_huff = take(nopt * sizeof(FrameHuff)), o_slots = take(nopt * kHeaderSlot),
				 o_hlen = take(nopt * sizeof(unsigned)), o_bad = take(sizeof(int));
	char *scratch = nullptr;
	if (dev_alloc(domain, (void **) &scratch, off, s))
		return -1;
	int rc = -1;
	do {
		/* tables and header from pageable memory: small, staged by the driver before the call returns */
		if (cudaMemcpyAsync(scratch + o_tab, &T, sizeof(T), cudaMemcpyHostToDevice, s) != cudaSuccess ||
			cudaMemcpyAsync(scratch + o_hdr, header.data(), header.size(), cudaMemcpyHostToDevice, s) != cudaSuccess ||
			cudaMemsetAsync(scratch + o_raw, 0, (size_t) n * raw_bytes, s) != cudaSuccess ||
			cudaMemsetAsync(scratch + o_bad, 0, sizeof(int), s) != cudaSuccess) {
			cuda_fail(domain, cudaGetLastError(), "jpeg encode setup");
			break;
		}
		ChunkArgs A;
		A.G = G;
		A.T = (const EncodeTables *) (scratch + o_tab);
		A.bpl = bpl;
		A.frame_stride = frame_stride;
		A.restart = restart;
		A.nint = nint;
		A.max_chunks = max_chunks;
		A.raw_bytes = raw_bytes;
		A.freq = (unsigned *) (scratch + o_freq);
		A.huff = (FrameHuff *) (scratch + o_huff);
		A.header = (const unsigned char *) (scratch + o_hdr);
		A.header_len = (unsigned) header.size();
		A.prefix_len = prefix_len;
		A.suffix_len = (unsigned) suffix.size();
		A.headers = (unsigned char *) (scratch + o_slots);
		A.header_lens = (unsigned *) (scratch + o_hlen);
		A.bad = (int *) (scratch + o_bad);
		A.out_stride = out_stride;
		unsigned long long *lengths = (unsigned long long *) (scratch + o_len);
		/* the frame is gridDim.y (or x) of every kernel: chunks of at most kMaxBatchFrames, each on its slice of the scratch */
		cudaError_t e = cudaSuccess;
		for (int c0 = 0; c0 < n && e == cudaSuccess; c0 += kMaxBatchFrames) {
			A.cn = std::min(kMaxBatchFrames, n - c0);
			A.frames = (const unsigned char *) frames + (size_t) c0 * frame_stride;
			A.coef = (short *) (scratch + o_coef) + (size_t) c0 * G.blocks * 64;
			A.bits = (unsigned *) (scratch + o_bits) + (size_t) c0 * G.blocks;
			A.totals = (unsigned long long *) (scratch + o_tot) + c0;
			A.lengths = lengths + c0;
			A.raw = (unsigned char *) (scratch + o_raw) + (size_t) c0 * raw_bytes;
			A.counts = (unsigned *) (scratch + o_cnt) + (size_t) c0 * max_chunks;
			A.istart = (unsigned *) (scratch + o_ist) + (size_t) c0 * nint;
			A.out = (unsigned char *) out + (size_t) c0 * out_stride;
			const int launches = optimize ? (restart ? launch_chunk<true, true>(A, s) : launch_chunk<true, false>(A, s))
										  : (restart ? launch_chunk<false, true>(A, s) : launch_chunk<false, false>(A, s));
			e = cudaGetLastError();
			if (e == cudaSuccess && launches < 0)
				e = cudaErrorUnknown;
			if (e == cudaSuccess)
				for (int k = 0; k < launches; k++)
					count_launch();
		}
		if (e != cudaSuccess) {
			cuda_fail(domain, e, "jpeg encode kernels launch");
			break;
		}
		std::vector<unsigned long long> len(n);
		int bad = 0;
		if (cudaMemcpyAsync(len.data(), lengths, (size_t) n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
			cudaMemcpyAsync(&bad, scratch + o_bad, sizeof(int), cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) {
			cuda_fail(domain, cudaGetLastError(), "jpeg encode");
			break;
		}
		if (bad) {
			/* libjpeg's JERR_HUFF_CLEN_OVERFLOW: a symbol distribution no image of the sizes taken here produces */
			error(domain, "optimised Huffman table: a code longer than 32 bits");
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

/* jpeg_gen_optimal_table on the host (libjpeg's own serial minimum search), for the host twin and its test hook */
int
host_optimal_table(unsigned *freq, unsigned char *bits, unsigned char *huffval)
{
	int codesize[257], others[257];
	auto pick = [&](int exclude) {
		int c = -1;
		unsigned v = kFreqSentinel;
		for (int i = 0; i <= 256; i++)
			if (freq[i] && freq[i] <= v && i != exclude) {
				v = freq[i];
				c = i;
			}
		return c;
	};
	return gen_optimal_table(freq, codesize, others, bits, huffval, true, pick);
}

/* the whole encoder on the CPU through the same per-block code, in the order libjpeg runs it: statistics and table
 * generation when optimising, then the scan with its restart markers (test hook)
 */
int
host_jpeg_encode(const char *domain, const unsigned char *img, size_t bpl, int w, int h, int bands, int quality, int subsample_mode, int optimize,
	int restart, std::vector<unsigned char> &out)
{
	EncodeGeom G;
	if (make_geom(domain, w, h, bands, quality, subsample_mode, &G) || check_restart(domain, restart))
		return -1;
	EncodeTables T;
	make_tables(quality, &T);
	std::vector<short> coef((size_t) G.blocks * 64);
	for (int my = 0; my < G.mcus_y; my++)
		for (int mx = 0; mx < G.mcus_x; mx++)
			encode_mcu(G, T.q, img, bpl, mx, my, coef.data() + ((size_t) my * G.mcus_x + mx) * G.blocks_per_mcu * 64);
	const unsigned bpm = (unsigned) G.blocks_per_mcu;
	unsigned char bits[4][17], huffval[4][256];
	FrameHuff fh;
	const unsigned (*co)[256] = T.ehufco;
	const unsigned char (*si)[256] = T.ehufsi;
	if (optimize) {
		std::vector<unsigned> freq(4 * 257, 0);
		for (unsigned b = 0; b < (unsigned) G.blocks; b++)
			walk_block(
				T.zz, coef.data() + (size_t) b * 64, block_comp(G, (int) (b % bpm)), previous_dc(G, coef.data(), b, restart),
				[&](int t, int s) { freq[t * 257 + s]++; }, [](unsigned, int) {});
		for (int t = 0; t < (G.ncomp == 1 ? 2 : 4); t++) {
			if (host_optimal_table(freq.data() + t * 257, bits[t], huffval[t])) {
				error(domain, "optimised Huffman table: a code longer than 32 bits");
				return -1;
			}
			derive_codes(bits[t] + 1, huffval[t], fh.ehufco[t], fh.ehufsi[t]);
		}
		co = fh.ehufco;
		si = fh.ehufsi;
	}
	else
		standard_tables(bits, huffval);
	header_prefix(G, T, out);
	put_dhts(G, bits, huffval, out);
	header_suffix(G, restart, out);
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
	/* jchuff.c flush_bits: the partial byte padded with 1-bits (and stuffed) */
	auto pad = [&]() {
		if (nacc > 0)
			flush_byte((unsigned char) (((acc << (8 - nacc)) | ((1u << (8 - nacc)) - 1)) & 0xFF));
		nacc = 0;
	};
	for (unsigned b = 0; b < (unsigned) G.blocks; b++) {
		const unsigned mcu = b / bpm;
		if (restart > 0 && b % bpm == 0 && mcu > 0 && mcu % (unsigned) restart == 0) {
			/* jchuff.c emit_restart: before MCU k * restart, RST((k - 1) mod 8), not stuffed */
			pad();
			out.push_back(0xFF);
			out.push_back((unsigned char) (0xD0 + ((mcu / (unsigned) restart - 1) & 7)));
		}
		code_block(co, si, T.zz, coef.data() + (size_t) b * 64, block_comp(G, (int) (b % bpm)), previous_dc(G, coef.data(), b, restart), emit);
	}
	pad();
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
	const VB200JpegSaveOptions opt = {quality, subsample_mode, 0, 0};
	return vb200_debug_jpeg_encode_opts(pixels, bpl, width, height, bands, &opt, out, cap, len);
}

/* Test hook, host only: vb200_debug_jpeg_encode with every option of VB200JpegSaveOptions */
extern "C" int
vb200_debug_jpeg_encode_opts(const void *pixels, size_t bpl, int width, int height, int bands, const VB200JpegSaveOptions *opt, void *out, size_t cap,
	size_t *len)
{
	if (!opt) {
		error("jpeg_encode (host twin)", "null options");
		return -1;
	}
	std::vector<unsigned char> o;
	if (host_jpeg_encode("jpeg_encode (host twin)", (const unsigned char *) pixels, bpl, width, height, bands, opt->Q, opt->subsample_mode,
			opt->optimize_coding, opt->restart_interval, o))
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

/* Test hook, host only: jpeg_gen_optimal_table (jchuff.c) on the symbol counts freq[256] -> bits[17] (bits[0] unused),
 * huffval[256] (sum of bits[1..16] entries used).  -1 when the counts add up to 10^9 or more (the frames the encoder takes
 * stay far below) or a code would be longer than 32 bits.
 */
extern "C" int
vb200_debug_jpeg_optimal_table(const unsigned *freq, unsigned char *bits, unsigned char *huffval)
{
	unsigned f[257];
	unsigned long long total = 0;
	for (int i = 0; i < 256; i++)
		total += f[i] = freq[i];
	if (total + 1 >= kFreqSentinel) {
		error("jpeg_optimal_table", "symbol counts add up to %llu, the table generator takes less than %u", total, kFreqSentinel - 1);
		return -1;
	}
	if (host_optimal_table(f, bits, huffval)) {
		error("jpeg_optimal_table", "a code longer than 32 bits");
		return -1;
	}
	return 0;
}

/* vips_jpegsave_buffer (foreign/vips2jpeg.c) for a batch of equally sized 8-bit frames (1 or 3 bands), on the device:
 * frames in host or device memory (frames_location), n streams to out + i * out_stride in host or device memory
 * (out_location), lengths[n] on the host.  Q and subsample_mode as the reference's arguments (0 auto, 1 on, 2 off);
 * everything else is the reference's default (baseline, standard Huffman tables, no restart markers, JFIF header).
 */
extern "C" int
vb200_jpegsave_batch(const void *frames, int frames_location, size_t bpl, size_t frame_stride, int n, int width, int height, int bands, int Q,
	int subsample_mode, void *out, int out_location, size_t out_stride, size_t *lengths)
{
	const VB200JpegSaveOptions opt = {Q, subsample_mode, 0, 0};
	return vb200_jpegsave_batch_opts(frames, frames_location, bpl, frame_stride, n, width, height, bands, &opt, out, out_location, out_stride,
		lengths);
}

/* vb200_jpegsave_batch with vips_jpegsave's entropy-coding options too: optimize_coding (per-frame Huffman tables) and
 * restart_interval (RSTn every N MCUs, 0..65535)
 */
extern "C" int
vb200_jpegsave_batch_opts(const void *frames, int frames_location, size_t bpl, size_t frame_stride, int n, int width, int height, int bands,
	const VB200JpegSaveOptions *opt, void *out, int out_location, size_t out_stride, size_t *lengths)
{
	const char *domain = "jpegsave_batch";
	if (!frames || !out || !opt || n < 1) {
		error(domain, "null argument");
		return -1;
	}
	const int Q = opt->Q, subsample_mode = opt->subsample_mode;
	if (check_restart(domain, opt->restart_interval))
		return -1;
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
		if (dev_jpeg_encode_batch(domain, src, sbpl, sstride, n, width, height, bands, Q, subsample_mode, opt->optimize_coding != 0,
				opt->restart_interval, dst, out_stride, len.data(), s))
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

