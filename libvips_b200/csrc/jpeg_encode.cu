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
 *   (stuffing)             FF -> FF00 and the markers around the scan: per 256-byte span count (jpeg_stuffcount_kernel),
 *                          prefix sum (jpeg_ffscan_kernel), copy (jpeg_stuffcopy_kernel)
 * With vips_jpegsave's options (vips2jpeg.c:590-597):
 *   optimize_coding        jpeg_stats_kernel (symbol counts per frame) and jpeg_tables_kernel (jchuff.c
 *                          jpeg_gen_optimal_table per table, the frame's code tables and header) after the FDCT; the count,
 *                          emit and stuffing kernels then take the frame's tables and header
 *   restart_interval       jpeg_segments_kernel after the bit prefix sum: every interval starts on a byte boundary, the
 *                          stuffing kernels put FF Dn before each interval after the first
 * A sequential stream is the one-scan case of the progressive script (ScanScript): the table, segment and stuffing kernels
 * serve both; only the coders differ.
 */
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/vb200.h"
#include "vb200_internal.h"
#include "jpeg_common.cuh"

namespace vb200 {

namespace {

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
	memcpy(T->zz, kZigzag, 64);
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

/* jfdctint.c jpeg_fdct_islow on d[64] (samples already centred on 0), in place */
HD void
fdct_islow(int *d)
{
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
				p[0] = descale(tmp10 + tmp11, P1);
				p[4 * step] = descale(tmp10 - tmp11, P1);
			}
			const int sh = pass == 0 ? CB - P1 : CB + P1;
			int z1 = (tmp12 + tmp13) * F_0_541196100;
			p[2 * step] = descale(z1 + tmp13 * F_0_765366865, sh);
			p[6 * step] = descale(z1 + tmp12 * (-F_1_847759065), sh);
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
			p[7 * step] = descale(t4 + z1 + z3, sh);
			p[5 * step] = descale(t5 + z2 + z4, sh);
			p[3 * step] = descale(t6 + z2 + z3, sh);
			p[1 * step] = descale(t7 + z1 + z4, sh);
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

/* the markers before the Huffman tables, in libjpeg's order: SOI, JFIF APP0, DQT per table, SOF0 (sof: SOF2 for a
 * progressive stream)
 */
void
header_prefix(const EncodeGeom &G, const EncodeTables &T, std::vector<unsigned char> &o, unsigned sof = 0xFFC0)
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
			o.push_back((unsigned char) T.q[t][kZigzag[i]]);
	}
	put16(o, sof);
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

/* ------------------------------------------------------------------ the scan script (host + device) */

constexpr int kMaxProgScans = 10;  /* jcparam.c jpeg_simple_progression: 10 scans for YCbCr, 6 for greyscale */
constexpr int kMaxProgTables = 10; /* one table per DC-first component table and per AC scan: 10 for YCbCr, 5 for greyscale */
constexpr int kMaxCorrBits = 1000; /* jcphuff.c MAX_CORR_BITS: the correction bits an EOB run may hold */

/* One scan of the script.  A unit is what a restart interval counts: an MCU of the interleaved scans (the sequential
 * scan, the progressive DC scans), one block of the component's own grid (ceil(comp_w / 8) x ceil(comp_h / 8), no dummy
 * blocks; T.81 A.2.2) in the others.
 */
struct Scan {
	int comp;			/* the scan's component, -1 for an interleaved scan */
	int ss, se, ah, al; /* spectral band and successive-approximation bits */
	int ux, units;		/* units per row, units */
	int unit_base;		/* the scan's first unit in the frame's list of units */
	int seg_base, nseg; /* its restart intervals (segments) in the frame's list of segments; 1 without restart markers */
	int tab, nt;		/* its first table in the frame's list of tables and their number (0 for DC refinement) */
};

/* A stream's scans: the progressive script, or the sequential stream's one scan (Ss 0, Se 63, Ah Al 0) */
struct ScanScript {
	int nscans, ntab, units, nseg, restart;
	Scan s[kMaxProgScans];
	int tab_class[kMaxProgTables]; /* put_dht's t: 0 DC lum, 1 AC lum, 2 DC chr, 3 AC chr */
	/* the device's header template: the frame's markers before the first scan (prefix_len bytes), then each scan's DRI / SOS
	 * at sfx_at[s] .. sfx_at[s + 1]
	 */
	int prefix_len, sfx_at[kMaxProgScans + 1];
};

/* the component's own block grid */
HD void
comp_grid(const EncodeGeom &G, int c, int *bw, int *bh)
{
	if (G.ncomp == 3 && G.sub && c == 0) {
		*bw = (G.w + 7) / 8;
		*bh = (G.h + 7) / 8;
	}
	else {
		*bw = G.mcus_x;
		*bh = G.mcus_y;
	}
}

/* block (bx, by) of component c's grid -> its index in the MCU-ordered coefficients */
HD unsigned
comp_block_index(const EncodeGeom &G, int c, int bx, int by)
{
	if (G.ncomp == 3 && G.sub) {
		if (c == 0)
			return ((unsigned) (by >> 1) * G.mcus_x + (unsigned) (bx >> 1)) * 6 + (unsigned) ((by & 1) * 2 + (bx & 1));
		return ((unsigned) by * G.mcus_x + (unsigned) bx) * 6 + 3 + (unsigned) c;
	}
	return ((unsigned) by * G.mcus_x + (unsigned) bx) * G.blocks_per_mcu + (unsigned) c;
}

/* The scans of one geometry.  Sequential: one interleaved scan, Ss 0, Se 63, with tables DC and AC per component class
 * (0 DC lum, 1 AC lum, 2 DC chr, 3 AC chr).  Progressive: jcparam.c jpeg_simple_progression (fill_dc_scans, fill_a_scan /
 * fill_scans), YCbCr
 *   DC 0-0 Al 1 (interleaved); Y 1-5 Al 2; Cr 1-63 Al 1; Cb 1-63 Al 1; Y 6-63 Al 2; Y 1-63 Ah 2 Al 1;
 *   DC Ah 1 Al 0 (interleaved); Cr 1-63 Ah 1 Al 0; Cb 1-63 Ah 1 Al 0; Y 1-63 Ah 1 Al 0
 * and greyscale the same without the chroma scans.  Tables: the DC-first scan one per dc_tbl_no (Y 0, Cb and Cr 1), every
 * AC scan its own (finish_pass_gather_phuff builds a table per scan), DC refinement none.
 */
void
scan_script(const EncodeGeom &G, int restart, bool progressive, ScanScript *P)
{
	static const int sequential[1][5] = {{-1, 0, 63, 0, 0}};
	static const int colour[10][5] = {{-1, 0, 0, 0, 1}, {0, 1, 5, 0, 2}, {2, 1, 63, 0, 1}, {1, 1, 63, 0, 1}, {0, 6, 63, 0, 2}, {0, 1, 63, 2, 1},
		{-1, 0, 0, 1, 0}, {2, 1, 63, 1, 0}, {1, 1, 63, 1, 0}, {0, 1, 63, 1, 0}};
	static const int grey[6][5] = {{-1, 0, 0, 0, 1}, {0, 1, 5, 0, 2}, {0, 6, 63, 0, 2}, {0, 1, 63, 2, 1}, {-1, 0, 0, 1, 0}, {0, 1, 63, 1, 0}};
	const int(*script)[5] = !progressive ? sequential : G.ncomp == 3 ? colour : grey;
	memset(P, 0, sizeof(*P));
	P->nscans = !progressive ? 1 : G.ncomp == 3 ? 10 : 6;
	P->restart = restart;
	for (int i = 0; i < P->nscans; i++) {
		Scan &S = P->s[i];
		S.comp = script[i][0];
		S.ss = script[i][1];
		S.se = script[i][2];
		S.ah = script[i][3];
		S.al = script[i][4];
		int bw = G.mcus_x, bh = G.mcus_y;
		if (S.comp >= 0)
			comp_grid(G, S.comp, &bw, &bh);
		S.ux = bw;
		S.units = bw * bh;
		S.unit_base = P->units;
		P->units += S.units;
		S.nseg = restart ? (S.units + restart - 1) / restart : 1;
		S.seg_base = P->nseg;
		P->nseg += S.nseg;
		/* per component class of the scan (luma, chroma): a DC table unless it refines DC, an AC table unless Se is 0 */
		S.tab = P->ntab;
		for (int k = 0; k < (S.comp < 0 && G.ncomp == 3 ? 2 : 1); k++) {
			const int chr = S.comp < 0 ? k : S.comp > 0;
			if (S.ss == 0 && S.ah == 0)
				P->tab_class[P->ntab++] = 2 * chr;
			if (S.se > 0)
				P->tab_class[P->ntab++] = 2 * chr + 1;
		}
		S.nt = P->ntab - S.tab;
	}
}

/* jcmarker.c write_scan_header after the DHTs: DRI before the first scan when there are restart intervals (emitted when
 * the interval differs from the last one written; also when it covers the whole frame), then emit_sos with 0 for the
 * table selectors a scan does not use
 */
void
scan_suffix(const EncodeGeom &G, const Scan &S, bool first, int restart, std::vector<unsigned char> &o)
{
	if (first && restart > 0) {
		put16(o, 0xFFDD);
		put16(o, 4);
		put16(o, (unsigned) restart);
	}
	const int nc = S.comp < 0 ? G.ncomp : 1;
	put16(o, 0xFFDA);
	put16(o, 6 + 2 * nc);
	o.push_back((unsigned char) nc);
	for (int i = 0; i < nc; i++) {
		const int c = S.comp < 0 ? i : S.comp;
		o.push_back((unsigned char) (c + 1));
		/* dc_tbl_no when the scan codes a DC first pass, ac_tbl_no when it codes AC coefficients */
		const int dc = S.ss == 0 && S.ah == 0 && c ? 0x10 : 0, ac = S.se > 0 && c ? 1 : 0;
		o.push_back((unsigned char) (dc | ac));
	}
	o.push_back((unsigned char) S.ss);
	o.push_back((unsigned char) S.se);
	o.push_back((unsigned char) ((S.ah << 4) | S.al));
}

/* The symbols and bits of one block in an AC scan of the script, without its EOB run (jcphuff.c encode_mcu_AC_first,
 * encode_mcu_AC_refine; sym(symbol) for every Huffman symbol, bits(value, n) for the bits that follow it: the magnitude,
 * or the sign of a newly non-zero coefficient followed by the correction bits buffered since the previous symbol (BR)).
 * Returns the block's place in the EOB run structure: kEmits when it codes a symbol -- a pending EOB run is flushed just
 * before its first one --, kTail when it ends in an EOB (it joins the run), and << 2 the correction bits it leaves to the
 * run (BE), which tail(bit) receives in order.  None of this depends on the Huffman tables.
 */
constexpr unsigned kEmits = 1, kTail = 2;

HD int
ac_abs(const short *blk, const unsigned char *zz, int k, int al)
{
	const int v = blk[zz[k]];
	return (v < 0 ? -v : v) >> al;
}

template <typename Sym, typename Bits, typename Tail>
HD unsigned
walk_ac_block(const unsigned char *zz, const short *blk, int ss, int se, int ah, int al, Sym sym, Bits bits, Tail tail)
{
	unsigned flags = 0;
	int r = 0;
	if (ah == 0) {
		for (int k = ss; k <= se; k++) {
			const int t = ac_abs(blk, zz, k, al); /* the point transform: |v| >> Al, the sign put back after */
			if (t == 0) {
				r++;
				continue;
			}
			flags |= kEmits;
			while (r > 15) {
				sym(0xF0);
				r -= 16;
			}
			const int nb = bit_size(t);
			sym((r << 4) + nb);
			bits((unsigned) (blk[zz[k]] < 0 ? ~t : t) & ((1u << nb) - 1), nb);
			r = 0;
		}
		return r > 0 ? flags | kTail : flags;
	}
	int eob = 0; /* the last newly non-zero coefficient */
	for (int k = ss; k <= se; k++)
		if (ac_abs(blk, zz, k, al) == 1)
			eob = k;
	int kbr = ss, nbr = 0; /* BR: coefficients kbr .. k - 1 with |value| > 1, nbr of them */
	auto put_br = [&](int k) {
		for (int j = kbr; j < k; j++) {
			const int t = ac_abs(blk, zz, j, al);
			if (t > 1)
				bits((unsigned) t & 1u, 1);
		}
		nbr = 0;
	};
	for (int k = ss; k <= se; k++) {
		const int t = ac_abs(blk, zz, k, al);
		if (t == 0) {
			r++;
			continue;
		}
		/* ZRLs, but not where they fold into the EOB */
		while (r > 15 && k <= eob) {
			flags |= kEmits;
			sym(0xF0);
			r -= 16;
			put_br(k);
			kbr = k;
		}
		if (t > 1) {
			nbr++; /* a coefficient already non-zero: one correction bit, buffered */
			continue;
		}
		flags |= kEmits;
		sym((r << 4) + 1);
		bits(blk[zz[k]] < 0 ? 0u : 1u, 1);
		put_br(k);
		kbr = k + 1;
		r = 0;
	}
	if (r > 0 || nbr > 0) {
		flags |= kTail | (unsigned) nbr << 2;
		for (int j = kbr; j <= se; j++) {
			const int t = ac_abs(blk, zz, j, al);
			if (t > 1)
				tail((unsigned) t & 1u);
		}
	}
	return flags;
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

/* a frame's own Huffman tables, code / length per symbol: N = 4 for a sequential frame (tables as in EncodeTables),
 * kMaxProgTables for a progressive one (one per table of the script)
 */
template <int N>
struct HuffSet {
	unsigned ehufco[N][256];
	unsigned char ehufsi[N][256];
};

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
template <bool kFrameTables>
__device__ __forceinline__ void
frame_tables(const EncodeTables *T, const HuffSet<4> *huff, unsigned f, const unsigned (**co)[256], const unsigned char (**si)[256])
{
	if (kFrameTables) {
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

/* optimise_coding, pass 2: tables and headers, one CTA per frame, one warp per table of the script (N: the tables a
 * frame can have, which sets the block size).  Each warp runs gen_optimal_table on its counts with a warp-wide minimum
 * search and writes the frame's code / length table; the CTA then writes the frame's headers into its slot_bytes-byte
 * slot -- the markers before the first scan (SOI .. SOF), and per scan its DHTs and DRI / SOS from the template.
 * hdr_end[frame][s] = where scan s's header ends: the first scan's comes with the frame's markers, so hdr_end[frame][0] is
 * the bytes before the scan data (with one scan, the whole header); the stuffing passes insert the later ones.  A frame
 * whose tables cannot be built sets *bad.
 */
template <int N>
__global__ void __launch_bounds__(32 * N)
jpeg_tables_kernel(const __grid_constant__ ScanScript P, const unsigned *__restrict__ counts, HuffSet<N> *__restrict__ huff,
	const unsigned char *__restrict__ tmpl, unsigned char *__restrict__ headers, unsigned slot_bytes, unsigned *__restrict__ hdr_end,
	int *__restrict__ bad)
{
	__shared__ unsigned s_freq[N][257];
	__shared__ int s_size[N][257], s_others[N][257];
	__shared__ unsigned char s_bits[N][17], s_val[N][256];
	__shared__ unsigned s_dht_at[N], s_sfx_dst[kMaxProgScans], s_len;
	__shared__ int s_fail;
	const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const unsigned *cnt = counts + (size_t) blockIdx.x * N * 256;
	if (threadIdx.x == 0)
		s_fail = 0;
	for (int i = threadIdx.x; i < N * 256; i += blockDim.x)
		s_freq[i >> 8][i & 255] = cnt[i];
	__syncthreads();
	HuffSet<N> *fh = huff + blockIdx.x;
	if (w < P.ntab) {
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
	unsigned *end = hdr_end + (size_t) blockIdx.x * P.nscans;
	if (threadIdx.x == 0) {
		unsigned len = (unsigned) P.prefix_len;
		for (int s = 0; s < P.nscans; s++) {
			for (int t = P.s[s].tab; t < P.s[s].tab + P.s[s].nt; t++) {
				s_dht_at[t] = len;
				len += 21 + table_values(s_bits[t]);
			}
			s_sfx_dst[s] = len;
			len += (unsigned) (P.sfx_at[s + 1] - P.sfx_at[s]);
			end[s] = len;
		}
		s_len = len;
		if (s_fail || len > slot_bytes) {
			end[0] = 0;
			atomicExch(bad, 1);
		}
	}
	__syncthreads();
	if (s_fail || s_len > slot_bytes)
		return;
	unsigned char *o = headers + (size_t) blockIdx.x * slot_bytes;
	for (int i = threadIdx.x; i < P.prefix_len; i += blockDim.x)
		o[i] = tmpl[i];
	for (int s = 0; s < P.nscans; s++)
		for (int i = P.sfx_at[s] + threadIdx.x; i < P.sfx_at[s + 1]; i += blockDim.x)
			o[s_sfx_dst[s] + (unsigned) (i - P.sfx_at[s])] = tmpl[i];
	if (w < P.ntab && lane == 0)
		put_dht(o + s_dht_at[w], P.tab_class[w], s_bits[w], s_val[w]);
}

/* one thread per block: how many bits its code takes, into the frame's list of G.blocks + 1 slots (the last is the
 * bit prefix sum's)
 */
template <bool kFrameTables, bool kRestart>
__global__ void __launch_bounds__(128)
jpeg_count_kernel(const EncodeGeom G, const EncodeTables *__restrict__ T, const HuffSet<4> *__restrict__ huff, int restart,
	const short *__restrict__ coef, unsigned *__restrict__ bits)
{
	const unsigned b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= (unsigned) G.blocks)
		return;
	const short *fc = coef + (size_t) blockIdx.y * G.blocks * 64;
	const unsigned (*co)[256];
	const unsigned char (*si)[256];
	frame_tables<kFrameTables>(T, huff, blockIdx.y, &co, &si);
	bits[(size_t) blockIdx.y * (G.blocks + 1) + b] = code_block(co, si, T->zz, fc + (size_t) b * 64, block_comp(G, (int) (b % (unsigned) G.blocks_per_mcu)),
		previous_dc(G, fc, b, kRestart ? restart : 0), [](unsigned, int) {});
}

/* exclusive prefix sum of a frame's bit counts (in place) over its nslots slots, the last of which receives the total,
 * as does totals[frame]: one CTA per frame
 */
__global__ void __launch_bounds__(1024)
jpeg_bitscan_kernel(int nslots, unsigned *__restrict__ bits, unsigned long long *__restrict__ totals)
{
	__shared__ unsigned long long s_part[1024];
	unsigned *b = bits + (size_t) blockIdx.x * nslots;
	/* a frame's scan stays far below 2^32 bits (65535 x 65535 would not, and is refused) */
	const unsigned long long total = cta_exclusive_scan(
		(unsigned) nslots - 1, s_part, [&](unsigned i) { return b[i]; }, [&](unsigned i, unsigned long long run) { b[i] = (unsigned) run; });
	if (threadIdx.x == blockDim.x - 1) {
		b[nslots - 1] = (unsigned) total;
		totals[blockIdx.x] = total;
	}
}

/* a sequential frame's segments in its bit list: restart interval g starts at slot g * per, the final slot is end */
struct IntervalSlots {
	unsigned per, nseg, end;
	__device__ __forceinline__ unsigned operator()(unsigned g) const { return g < nseg ? g * per : end; }
};

/* Segments after the bit prefix sum, one CTA per frame: segment g (a restart interval of a scan, or a whole scan without
 * them) spans slots M(g) .. M(g + 1) of the frame's nslots and takes their bits rounded up to a whole byte (the 1-padding
 * before each RSTn or scan header); istart[frame][g] = the byte where it starts in the raw scan data, totals[frame] =
 * their length in bits (whole bytes)
 */
template <typename Slots>
__global__ void __launch_bounds__(1024)
jpeg_segments_kernel(const __grid_constant__ Slots M, int nseg, int nslots, const unsigned *__restrict__ offs, unsigned long long *__restrict__ totals,
	unsigned *__restrict__ istart)
{
	__shared__ unsigned long long s_part[1024];
	const unsigned *o = offs + (size_t) blockIdx.x * nslots;
	unsigned *st = istart + (size_t) blockIdx.x * nseg;
	const unsigned long long bytes = cta_exclusive_scan(
		(unsigned) nseg, s_part, [&](unsigned g) { return ((unsigned long long) o[M(g + 1)] - o[M(g)] + 7) >> 3; },
		[&](unsigned g, unsigned long long run) { st[g] = (unsigned) run; });
	if (threadIdx.x == blockDim.x - 1)
		totals[blockIdx.x] = bytes * 8;
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
template <bool kFrameTables, bool kRestart>
__global__ void __launch_bounds__(128)
jpeg_emit_kernel(const EncodeGeom G, const EncodeTables *__restrict__ T, const HuffSet<4> *__restrict__ huff, int restart, int nint,
	const unsigned *__restrict__ istart, const short *__restrict__ coef, const unsigned *__restrict__ offs, unsigned *__restrict__ raw,
	size_t raw_words)
{
	const unsigned b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= (unsigned) G.blocks)
		return;
	const short *fc = coef + (size_t) blockIdx.y * G.blocks * 64;
	unsigned *out = raw + (size_t) blockIdx.y * raw_words;
	const unsigned *fo = offs + (size_t) blockIdx.y * G.blocks + blockIdx.y;
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
	frame_tables<kFrameTables>(T, huff, blockIdx.y, &co, &si);
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

/* ------------------------------------------------------------------ progressive save (interlace) on the device
 *
 * Every scan of the script is coded in the same launches: a frame's units (Scan) of all scans form one list, each
 * unit owns two bit slots -- [the EOB run flushed before it + its own symbols] and [the run flushed after it] -- and a
 * final empty slot makes the frame's total.  A segment is a restart interval of a scan (the whole scan without them);
 * every segment starts on a byte boundary and ends padded with 1-bits, and the stuffing stage puts the next scan's
 * header (DHTs, SOS) or FF Dn between segments.  The coders are numbered in launch order; 3 (jpeg_tables_kernel),
 * 5 (jpeg_segments_kernel) and the stuffing passes are the sequential stream's too.
 */

/* a unit's bit slots and a frame's bit slot count */
constexpr int kProgSlotsPerUnit = 2;
/* the bits one block takes over all the scans of the script, at most: DC first (a 16-bit code + 11 bits), DC refinement
 * (1), the first AC scans over 63 positions (a 16-bit code + 10 bits each, ZRLs at most a bit per zero), the refinement
 * scans over 63 positions twice (a 16-bit code + sign for a newly non-zero coefficient, else at most a correction bit or a
 * bit of ZRL), and two EOB-run flushes (EOBn code 16 bits + 14 run bits; their correction bits are the blocks' own,
 * counted above) per unit in each of the 4 AC scans of a luma block (chroma blocks take 2)
 */
constexpr int kProgBlockBits = (16 + 11) + 1 + 63 * (16 + 10) + 2 * 63 * (16 + 1) + 4 * 2 * (16 + 14);
constexpr int kProgBlockBytes = (kProgBlockBits + 7) / 8;
/* a table counts at most 65 symbols per block (63 AC symbols and two EOBn, or one DC category) */
static_assert(((1u << 29) / kProgBlockBytes) * 65u + 1u < kFreqSentinel, "symbol counts must stay below the sentinel");
/* a frame's headers: SOI + APP0 + 2 DQT + SOF2 (177 bytes for 3 components), a DHT per table (21 bytes + at most 256
 * symbols), one DRI (6), an SOS per scan (at most 14)
 */
constexpr int kProgHeaderBound = 177 + kMaxProgTables * (21 + 256) + 6 + kMaxProgScans * 14;
constexpr int kProgHeaderSlot = 3200;
static_assert(kProgHeaderBound <= kProgHeaderSlot, "a frame's progressive headers must fit their slot");
/* EOB runs: jcphuff.c flushes at 0x7FFF blocks, or when the buffered correction bits pass MAX_CORR_BITS - DCTSIZE2 + 1 */
constexpr unsigned kMaxEobRun = 0x7FFF;
static_assert(kMaxEobRun < (1u << 16) && kMaxCorrBits < (1 << 16), "a flush packs its run and its correction bits in 16 bits each");

__device__ __forceinline__ int
prog_scan_of_unit(const ScanScript &P, unsigned u)
{
	int s = 0;
	while (s + 1 < P.nscans && u >= (unsigned) P.s[s + 1].unit_base)
		s++;
	return s;
}

__device__ __forceinline__ int
scan_of_seg(const ScanScript &P, unsigned g)
{
	int s = 0;
	while (s + 1 < P.nscans && g >= (unsigned) P.s[s + 1].seg_base)
		s++;
	return s;
}

/* the first bit slot of segment g (g == nseg: the frame's final slot) */
__device__ __forceinline__ unsigned
prog_seg_slot(const ScanScript &P, unsigned g)
{
	if (g >= (unsigned) P.nseg)
		return kProgSlotsPerUnit * (unsigned) P.units;
	const Scan &S = P.s[scan_of_seg(P, g)];
	const unsigned per = P.restart ? (unsigned) P.restart : (unsigned) S.units;
	return kProgSlotsPerUnit * ((unsigned) S.unit_base + (g - (unsigned) S.seg_base) * per);
}

/* a progressive frame's segments in its bit list (jpeg_segments_kernel) */
struct ScriptSlots {
	ScanScript P;
	__device__ __forceinline__ unsigned operator()(unsigned g) const { return prog_seg_slot(P, g); }
};

/* the block of unit i of a single-component scan */
__device__ __forceinline__ unsigned
prog_block(const EncodeGeom &G, const Scan &S, unsigned i)
{
	return comp_block_index(G, S.comp, (int) (i % (unsigned) S.ux), (int) (i / (unsigned) S.ux));
}

/* one MCU of the interleaved DC-first scan (jcphuff.c encode_mcu_DC_first): the point-transformed DC (arithmetic shift by
 * Al) against the previous block of its component, reset at each restart interval; sym(table 0 / 1, category), bits
 */
template <typename Sym, typename Bits>
__device__ __forceinline__ void
walk_dc_first(const EncodeGeom &G, const short *fc, unsigned mcu, int al, int restart, Sym sym, Bits bits)
{
	for (int j = 0; j < G.blocks_per_mcu; j++) {
		const unsigned b = mcu * (unsigned) G.blocks_per_mcu + (unsigned) j;
		const int comp = block_comp(G, j);
		int diff = (fc[(size_t) b * 64] >> al) - (previous_dc(G, fc, b, restart) >> al);
		int t2 = diff;
		if (diff < 0) {
			diff = -diff;
			t2--;
		}
		const int nb = bit_size(diff);
		sym(comp ? 1 : 0, nb);
		if (nb)
			bits((unsigned) t2 & ((1u << nb) - 1), nb);
	}
}

/* the EOBn symbol of a run of r blocks (emit_eobrun): n = floor(log2 r), then n bits of r */
__device__ __forceinline__ int
eobrun_n(unsigned r)
{
	return 31 - __clz((int) r);
}

/* bits written OR-ed into a zeroed bit buffer from bit pos on (neighbours share their boundary bytes) */
struct BitSink {
	unsigned *out;
	unsigned byte;
	unsigned long long acc;
	int nacc;
	__device__ BitSink(unsigned *o, unsigned pos) : out(o), byte(pos >> 3), acc(0), nacc((int) (pos & 7u)) {}
	__device__ __forceinline__ void or_byte(unsigned at, unsigned v)
	{
		if (v)
			atomicOr(out + (at >> 2), v << (8 * (at & 3u)));
	}
	__device__ __forceinline__ void put(unsigned code, int len)
	{
		acc = (acc << len) | code;
		nacc += len;
		while (nacc >= 8) {
			or_byte(byte, (unsigned) (acc >> (nacc - 8)) & 0xffu);
			byte++;
			nacc -= 8;
		}
	}
	/* n bits left to other threads */
	__device__ __forceinline__ void skip(unsigned n)
	{
		for (; n > 16; n -= 16)
			put(0, 16);
		put(0, (int) n);
	}
	__device__ __forceinline__ void finish()
	{
		if (nacc > 0)
			or_byte(byte, (unsigned) (acc << (8 - nacc)) & 0xffu);
	}
};

/* 1. block summaries and statistics, one thread per unit (all scans): each AC unit's place in the EOB run structure
 * (walk_ac_block's flags, a byte) into summ, and the symbols of its own -- everything but the EOBn of the runs -- into the
 * CTA's histograms (a table per scan), added to the frame's counts[kMaxProgTables][256]
 */
__global__ void __launch_bounds__(128)
jpeg_prog_summary_kernel(const EncodeGeom G, const __grid_constant__ ScanScript P, const EncodeTables *__restrict__ T, const short *__restrict__ coef,
	unsigned char *__restrict__ summ, unsigned *__restrict__ counts)
{
	__shared__ unsigned s_hist[kMaxProgTables * 256];
	for (int i = threadIdx.x; i < kMaxProgTables * 256; i += blockDim.x)
		s_hist[i] = 0;
	__syncthreads();
	const unsigned u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u < (unsigned) P.units) {
		const Scan &S = P.s[prog_scan_of_unit(P, u)];
		const unsigned i = u - (unsigned) S.unit_base;
		const short *fc = coef + (size_t) blockIdx.y * G.blocks * 64;
		unsigned *h = s_hist + S.tab * 256;
		if (S.ss == 0) {
			if (S.ah == 0)
				walk_dc_first(G, fc, i, S.al, P.restart, [&](int t, int sym) { atomicAdd(&h[t * 256 + sym], 1u); }, [](unsigned, int) {});
		}
		else
			summ[(size_t) blockIdx.y * P.units + u] = (unsigned char) walk_ac_block(
				T->zz, fc + (size_t) prog_block(G, S, i) * 64, S.ss, S.se, S.ah, S.al, [&](int sym) { atomicAdd(&h[sym], 1u); }, [](unsigned, int) {},
				[](unsigned) {});
	}
	__syncthreads();
	unsigned *dst = counts + (size_t) blockIdx.y * kMaxProgTables * 256;
	for (int i = threadIdx.x; i < P.ntab * 256; i += blockDim.x)
		if (s_hist[i])
			atomicAdd(dst + i, s_hist[i]);
}

/* 2. the chain walk, one thread per segment of an AC scan: jcphuff.c's EOB run state (EOBRUN, BE) over the segment's
 * summaries.  A run is flushed before the first unit that codes a symbol, after the unit that takes it to 0x7FFF blocks
 * or past MAX_CORR_BITS - 63 correction bits, and after the segment's last unit (emit_restart / finish_pass).  Each
 * flush goes into its slot of runs[] as (run << 16) | correction bits, its EOBn into the counts; each run member with
 * correction bits gets the flush's slot (defer_slot) and the offset of its bits among the flush's (defer_off).
 */
__global__ void __launch_bounds__(128)
jpeg_prog_walk_kernel(const __grid_constant__ ScanScript P, const unsigned char *__restrict__ summ, unsigned *__restrict__ runs,
	unsigned *__restrict__ defer_slot, unsigned short *__restrict__ defer_off, unsigned *__restrict__ counts)
{
	const unsigned g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= (unsigned) P.nseg)
		return;
	const Scan &S = P.s[scan_of_seg(P, g)];
	if (S.ss == 0)
		return;
	const size_t f = blockIdx.y;
	const unsigned char *sm = summ + f * P.units;
	unsigned *rn = runs + f * kProgSlotsPerUnit * P.units, *ds = defer_slot + f * P.units;
	unsigned short *dof = defer_off + f * P.units;
	unsigned *cnt = counts + f * kMaxProgTables * 256 + (size_t) S.tab * 256;
	const unsigned u0 = prog_seg_slot(P, g) / kProgSlotsPerUnit;
	const unsigned u1 = min(u0 + (P.restart ? (unsigned) P.restart : (unsigned) S.units), (unsigned) (S.unit_base + S.units));
	unsigned run = 0, be = 0, start = 0;
	auto flush = [&](unsigned slot, unsigned last) {
		rn[slot] = run << 16 | be;
		for (unsigned v = start; v <= last; v++)
			if (sm[v] >> 2)
				ds[v] = slot;
		atomicAdd(cnt + (eobrun_n(run) << 4), 1u);
		run = be = 0;
	};
	for (unsigned u = u0; u < u1; u++) {
		const unsigned fl = sm[u];
		rn[kProgSlotsPerUnit * u] = 0;
		rn[kProgSlotsPerUnit * u + 1] = 0;
		if ((fl & kEmits) && run)
			flush(kProgSlotsPerUnit * u, u - 1);
		if (fl & kTail) {
			if (!run)
				start = u;
			dof[u] = (unsigned short) be;
			run++;
			be += fl >> 2;
			if (run == kMaxEobRun || be > (unsigned) (kMaxCorrBits - 64 + 1))
				flush(kProgSlotsPerUnit * u + 1, u);
		}
	}
	if (run)
		flush(kProgSlotsPerUnit * (u1 - 1) + 1, u1 - 1);
}

/* the bits of a flushed EOB run: EOBn code, n bits of the run, its correction bits */
__device__ __forceinline__ unsigned
flush_bits(const unsigned char *si, unsigned r)
{
	if (!r)
		return 0;
	const int n = eobrun_n(r >> 16);
	return si[n << 4] + (unsigned) n + (r & 0xffffu);
}

/* 4. one thread per unit: the bits of its two slots with the frame's tables */
__global__ void __launch_bounds__(128)
jpeg_prog_count_kernel(const EncodeGeom G, const __grid_constant__ ScanScript P, const EncodeTables *__restrict__ T, const HuffSet<kMaxProgTables> *__restrict__ huff,
	const short *__restrict__ coef, const unsigned *__restrict__ runs, unsigned *__restrict__ bits)
{
	const unsigned u = blockIdx.x * blockDim.x + threadIdx.x;
	const size_t nslots = (size_t) kProgSlotsPerUnit * P.units + 1;
	unsigned *fb = bits + blockIdx.y * nslots;
	if (u >= (unsigned) P.units)
		return;
	const Scan &S = P.s[prog_scan_of_unit(P, u)];
	const unsigned i = u - (unsigned) S.unit_base;
	const short *fc = coef + (size_t) blockIdx.y * G.blocks * 64;
	const HuffSet<kMaxProgTables> &H = huff[blockIdx.y];
	unsigned body = 0, post = 0;
	if (S.ss == 0) {
		if (S.ah == 0)
			walk_dc_first(G, fc, i, S.al, P.restart, [&](int t, int sym) { body += H.ehufsi[S.tab + t][sym]; }, [&](unsigned, int n) { body += n; });
		else
			body = (unsigned) G.blocks_per_mcu; /* encode_mcu_DC_refine: a bit per block */
	}
	else {
		const unsigned char *si = H.ehufsi[S.tab];
		const unsigned *rn = runs + blockIdx.y * (nslots - 1) + kProgSlotsPerUnit * u;
		walk_ac_block(
			T->zz, fc + (size_t) prog_block(G, S, i) * 64, S.ss, S.se, S.ah, S.al, [&](int sym) { body += si[sym]; }, [&](unsigned, int n) { body += n; },
			[](unsigned) {});
		body += flush_bits(si, rn[0]);
		post = flush_bits(si, rn[1]);
	}
	fb[kProgSlotsPerUnit * u] = body;
	fb[kProgSlotsPerUnit * u + 1] = post;
}

/* 6. one thread per unit: its symbols and the runs flushed around them OR-ed into the frame's raw bit buffer at its
 * slots, its deferred correction bits at the offset the walk gave them behind their flush's EOBn and run bits; the
 * segment's last unit pads the segment's last byte with 1-bits
 */
__global__ void __launch_bounds__(128)
jpeg_prog_emit_kernel(const EncodeGeom G, const __grid_constant__ ScanScript P, const EncodeTables *__restrict__ T, const HuffSet<kMaxProgTables> *__restrict__ huff,
	const unsigned *__restrict__ istart, const short *__restrict__ coef, const unsigned *__restrict__ offs, const unsigned char *__restrict__ summ,
	const unsigned *__restrict__ runs, const unsigned *__restrict__ defer_slot, const unsigned short *__restrict__ defer_off, unsigned *__restrict__ raw,
	size_t raw_words)
{
	const unsigned u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u >= (unsigned) P.units)
		return;
	const size_t f = blockIdx.y, nslots = (size_t) kProgSlotsPerUnit * P.units + 1;
	const Scan &S = P.s[prog_scan_of_unit(P, u)];
	const unsigned i = u - (unsigned) S.unit_base;
	const unsigned g = (unsigned) S.seg_base + (P.restart ? i / (unsigned) P.restart : 0);
	const unsigned *fo = offs + f * nslots;
	/* bit positions in the raw buffer: slot offset - the segment's first slot offset + the segment's start */
	const unsigned base = istart[f * P.nseg + g] * 8 - fo[prog_seg_slot(P, g)];
	unsigned *out = raw + f * raw_words;
	const short *fc = coef + f * G.blocks * 64;
	const HuffSet<kMaxProgTables> &H = huff[f];
	BitSink w(out, base + fo[kProgSlotsPerUnit * u]);
	if (S.ss == 0) {
		if (S.ah == 0)
			walk_dc_first(
				G, fc, i, S.al, P.restart, [&](int t, int sym) { w.put(H.ehufco[S.tab + t][sym], H.ehufsi[S.tab + t][sym]); },
				[&](unsigned v, int n) { w.put(v, n); });
		else
			for (int j = 0; j < G.blocks_per_mcu; j++)
				w.put((unsigned) (fc[((size_t) i * G.blocks_per_mcu + j) * 64] >> S.al) & 1u, 1);
	}
	else {
		const unsigned *co = H.ehufco[S.tab];
		const unsigned char *si = H.ehufsi[S.tab];
		const unsigned *rn = runs + f * (nslots - 1);
		/* a flushed run: EOBn and the run's bits, then room for its members' correction bits, which they write */
		auto put_flush = [&](BitSink &b, unsigned r) {
			if (r) {
				const unsigned run = r >> 16;
				const int n = eobrun_n(run);
				b.put(co[n << 4], si[n << 4]);
				if (n)
					b.put(run & ((1u << n) - 1), n);
				b.skip(r & 0xffffu);
			}
		};
		put_flush(w, rn[kProgSlotsPerUnit * u]);
		/* this unit's correction bits for the run it joins, if any */
		const bool deferred = summ[f * P.units + u] >> 2;
		unsigned dpos = 0;
		if (deferred) {
			const unsigned slot = defer_slot[f * P.units + u], r = rn[slot];
			const int n = eobrun_n(r >> 16);
			dpos = base + fo[slot] + si[n << 4] + (unsigned) n + defer_off[f * P.units + u];
		}
		BitSink d(out, dpos);
		walk_ac_block(
			T->zz, fc + (size_t) prog_block(G, S, i) * 64, S.ss, S.se, S.ah, S.al, [&](int sym) { w.put(co[sym], si[sym]); },
			[&](unsigned v, int n) { w.put(v, n); }, [&](unsigned bit) { d.put(bit, 1); });
		put_flush(w, rn[kProgSlotsPerUnit * u + 1]);
		if (deferred)
			d.finish();
	}
	w.finish();
	const bool last = i + 1 == (unsigned) S.units || (P.restart && (i + 1) % (unsigned) P.restart == 0);
	if (last) {
		const unsigned end = base + fo[prog_seg_slot(P, g + 1)];
		if (end & 7u)
			w.or_byte(end >> 3, (1u << (8 - (end & 7u))) - 1); /* flush_bits: pad with ones */
	}
}

/* ------------------------------------------------------------------ stuffing (sequential and progressive)
 *
 * A frame's raw data is its segments, each starting on a byte.  The stream is the frame's header, the raw data with
 * FF -> FF 00 and, before each segment after the first, the next scan's header (DHTs, SOS) where a scan starts, else
 * FF Dn; then EOI.  The header is the frame's own (slots of hdr_stride bytes, hdr_end[frame][nscans] from
 * jpeg_tables_kernel) or, with the standard tables, the batch's: hdr_stride and hend_stride 0.  What goes between
 * segments is a compile-time choice, so that a sequential stream's byte loop carries no scan-header copy:
 */
enum {
	kOneSegment,	 /* nothing: a sequential stream without restart markers */
	kRestartMarkers, /* FF Dn: the restart intervals of a sequential stream */
	kScanHeaders	 /* FF Dn, or the next scan's header where a scan starts: a progressive stream */
};

/* insertion bytes before segments 1 .. j: the header of each scan that starts there, FF Dn before the others */
template <int kInserts>
__device__ __forceinline__ unsigned
inserts_before(const ScanScript &P, const unsigned *hend, unsigned j)
{
	unsigned n = 2 * j;
	if (kInserts == kScanHeaders)
		for (int s = 1; s < P.nscans && (unsigned) P.s[s].seg_base <= j; s++)
			n += hend[s] - hend[s - 1] - 2;
	return n;
}

/* stuffing, pass 1: 0xFF bytes per kStuffChunk-byte span of each frame's raw data, plus the bytes inserted before the
 * segments that start in the span
 */
template <int kInserts>
__global__ void __launch_bounds__(128)
jpeg_stuffcount_kernel(const __grid_constant__ ScanScript P, const unsigned long long *__restrict__ totals, const unsigned char *__restrict__ raw,
	size_t raw_bytes, int max_chunks, const unsigned *__restrict__ istart, const unsigned *__restrict__ hdr_end, int hend_stride,
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
	if (kInserts != kOneSegment && a < e) {
		const unsigned *st = istart + (size_t) blockIdx.y * P.nseg + 1;
		const unsigned *hend = hdr_end + (size_t) blockIdx.y * hend_stride;
		n += inserts_before<kInserts>(P, hend, (unsigned) count_below(st, P.nseg - 1, e)) -
			 inserts_before<kInserts>(P, hend, (unsigned) count_below(st, P.nseg - 1, a));
	}
	counts[(size_t) blockIdx.y * max_chunks + c] = n;
}

/* stuffing, pass 2: prefix sum of the spans' counts, one CTA per frame; lengths[frame] = header (hdr_end[frame][0]) + raw
 * data + stuffed zeros + inserted bytes + EOI
 */
__global__ void __launch_bounds__(1024)
jpeg_ffscan_kernel(const unsigned long long *__restrict__ totals, int max_chunks, unsigned *__restrict__ counts, const unsigned *__restrict__ hdr_end,
	int hend_stride, unsigned long long *__restrict__ lengths)
{
	__shared__ unsigned s_part[1024];
	unsigned *cnt = counts + (size_t) blockIdx.x * max_chunks;
	const unsigned added = cta_exclusive_scan(
		(unsigned) max_chunks, s_part, [&](unsigned i) { return cnt[i]; }, [&](unsigned i, unsigned run) { cnt[i] = run; });
	if (threadIdx.x == blockDim.x - 1)
		lengths[blockIdx.x] = (unsigned long long) hdr_end[(size_t) blockIdx.x * hend_stride] + ((totals[blockIdx.x] + 7) >> 3) + added + 2;
}

/* stuffing, pass 3: the header, the stuffed data with the next scan's header or FF D0+((k - 1) & 7) before segment k >= 1
 * of a scan (RSTn numbering restarts with every scan; padding bytes are stuffed, markers are not), EOI, into the frame's
 * stream at out + at[frame]
 */
template <int kInserts>
__global__ void __launch_bounds__(128)
jpeg_stuffcopy_kernel(const __grid_constant__ ScanScript P, const unsigned long long *__restrict__ totals, const unsigned char *__restrict__ raw,
	size_t raw_bytes, int max_chunks, const unsigned *__restrict__ counts, const unsigned char *__restrict__ headers, size_t hdr_stride,
	const unsigned *__restrict__ hdr_end, int hend_stride, const unsigned *__restrict__ istart, const unsigned long long *__restrict__ at,
	unsigned char *__restrict__ out, const unsigned long long *__restrict__ lengths)
{
	const int c = blockIdx.x * blockDim.x + threadIdx.x;
	unsigned char *o = out + at[blockIdx.y];
	const unsigned long long len = lengths[blockIdx.y];
	const unsigned char *hdr = headers + (size_t) blockIdx.y * hdr_stride;
	const unsigned *hend = hdr_end + (size_t) blockIdx.y * hend_stride;
	const unsigned h0 = hend[0];
	if (c < (int) ((h0 + kStuffChunk - 1) / kStuffChunk)) {
		/* the first spans' threads also copy the header */
		for (unsigned i = (unsigned) c * kStuffChunk; i < min(h0, (unsigned) (c + 1) * kStuffChunk); i++)
			o[i] = hdr[i];
	}
	if (c >= max_chunks)
		return;
	const unsigned long long nbytes = (totals[blockIdx.y] + 7) >> 3;
	const unsigned char *p = raw + (size_t) blockIdx.y * raw_bytes;
	const unsigned long long a = (unsigned long long) c * kStuffChunk, e = min(nbytes, a + kStuffChunk);
	unsigned char *d = o + h0 + a + counts[(size_t) blockIdx.y * max_chunks + c];
	const unsigned *st = istart + (size_t) blockIdx.y * P.nseg;
	const unsigned nseg = (unsigned) P.nseg;
	/* the next segment starting in the span */
	unsigned k = kInserts != kOneSegment && a < e ? 1 + (unsigned) count_below(st + 1, (int) nseg - 1, a) : nseg;
	for (unsigned long long i = a; i < e; i++) {
		const unsigned char v = p[i];
		if (kInserts != kOneSegment && k < nseg && st[k] == i) {
			const int s = kInserts == kScanHeaders ? scan_of_seg(P, k) : 0;
			const unsigned base = kInserts == kScanHeaders ? (unsigned) P.s[s].seg_base : 0;
			if (kInserts == kScanHeaders && k == base)
				for (unsigned j = hend[s - 1]; j < hend[s]; j++)
					*d++ = hdr[j];
			else {
				*d++ = 0xFF;
				*d++ = (unsigned char) (0xD0 + ((k - base - 1) & 7));
			}
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

/* What one call encodes with, from its options: the geometry, the quantisation and standard tables, the scan script, the
 * header -- with the standard tables the whole of it, else the template the table kernel builds each frame's headers from
 * (the markers before the Huffman tables, then each scan's DRI / SOS) -- and the sizes of the per-frame buffers
 */
struct EncodePlan {
	EncodeGeom G;
	EncodeTables T;
	ScanScript P;
	std::vector<unsigned char> header;
	bool prog, opt;			   /* progressive; the frame's own tables (libjpeg forces them for a progressive stream) */
	size_t nslots;			   /* bit slots per frame: a block each, or two a unit of the progressive script; and the final one */
	size_t scan_bound;		   /* the raw data's bound: every segment may end with one byte of padding */
	size_t raw_bytes;		   /* a frame's raw data buffer */
	int max_chunks;			   /* its kStuffChunk-byte spans */
	int ntab;				   /* the tables a frame can have: HuffSet<ntab> */
	unsigned slot;			   /* a frame's header slot */
};

int
make_plan(const char *domain, int w, int h, int bands, const VB200JpegSaveOptions &o, EncodePlan *E)
{
	EncodeGeom &G = E->G;
	ScanScript &P = E->P;
	const int restart = o.restart_interval;
	if (make_geom(domain, w, h, bands, o.Q, o.subsample_mode, &G) || check_restart(domain, restart))
		return -1;
	E->prog = o.interlace != 0;
	E->opt = E->prog || o.optimize_coding;
	scan_script(G, restart, E->prog, &P);
	E->nslots = (E->prog ? kProgSlotsPerUnit * (size_t) P.units : (size_t) G.blocks) + 1;
	E->scan_bound = (size_t) G.blocks * (E->prog ? kProgBlockBytes : kMaxBlockBytes) + (size_t) P.nseg;
	if (E->scan_bound >= (size_t) 1 << 29) {
		error(domain, "frame too large for the device encoder");
		return -1;
	}
	make_tables(o.Q, &E->T);
	std::vector<unsigned char> &hd = E->header;
	header_prefix(G, E->T, hd, E->prog ? 0xFFC2 : 0xFFC0);
	if (!E->opt) {
		unsigned char bits[4][17], huffval[4][256];
		standard_tables(bits, huffval);
		put_dhts(G, bits, huffval, hd);
	}
	P.prefix_len = (int) hd.size();
	for (int i = 0; i < P.nscans; i++) {
		P.sfx_at[i] = (int) hd.size();
		scan_suffix(G, P.s[i], i == 0, restart, hd);
	}
	P.sfx_at[P.nscans] = (int) hd.size();
	E->raw_bytes = ((E->scan_bound + 3) & ~(size_t) 3) + 4;
	E->max_chunks = (int) ((E->raw_bytes + kStuffChunk - 1) / kStuffChunk);
	E->ntab = E->prog ? kMaxProgTables : 4;
	E->slot = E->prog ? kProgHeaderSlot : kHeaderSlot;
	return 0;
}

/* The device scratch of a chunk of n frames, one allocation: the buffers' offsets and the total.  Per frame: coefficients,
 * bit slots, totals, lengths, stream offsets, raw data, span counts, segment starts, the progressive coder's unit
 * summaries, flushed runs and deferred correction bits, and with the frame's own tables its symbol counts, code tables,
 * header slot and header ends (with the standard tables, the chunk's one header length).  Every buffer grows with n or is
 * shared, so carve(n) takes at most n times carve(1).
 */
struct Scratch {
	size_t tab, hdr, coef, bits, tot, len, at, raw, cnt, ist, summ, runs, dslot, doff, freq, huff, slots, hend, bad, bytes;
};

Scratch
carve(const EncodePlan &E, int n)
{
	const size_t nf = (size_t) n, units = E.prog ? (size_t) E.P.units : 0, nopt = E.opt ? nf : 0;
	size_t off = 0;
	auto take = [&](size_t bytes) {
		const size_t o = off;
		off += (bytes + 255) & ~(size_t) 255;
		return o;
	};
	Scratch S;
	S.tab = take(sizeof(EncodeTables));
	S.hdr = take(E.header.size());
	S.coef = take(nf * E.G.blocks * 64 * sizeof(short));
	S.bits = take(nf * E.nslots * sizeof(unsigned));
	S.tot = take(nf * sizeof(unsigned long long));
	S.len = take(nf * sizeof(unsigned long long));
	S.at = take(nf * sizeof(unsigned long long));
	S.raw = take(nf * E.raw_bytes);
	S.cnt = take(nf * E.max_chunks * sizeof(unsigned));
	S.ist = take(E.prog || E.P.restart ? nf * E.P.nseg * sizeof(unsigned) : 0);
	S.summ = take(nf * units);
	S.runs = take(nf * kProgSlotsPerUnit * units * sizeof(unsigned));
	S.dslot = take(nf * units * sizeof(unsigned));
	S.doff = take(nf * units * sizeof(unsigned short));
	S.freq = take(nopt * E.ntab * 256 * sizeof(unsigned));
	S.huff = take(nopt * (E.prog ? sizeof(HuffSet<kMaxProgTables>) : sizeof(HuffSet<4>)));
	S.slots = take(nopt * E.slot);
	S.hend = take((E.opt ? nopt * E.P.nscans : 1) * sizeof(unsigned));
	S.bad = take(sizeof(int));
	S.bytes = off;
	return S;
}

/* the device buffers of one chunk of frames */
struct ChunkArgs {
	const EncodePlan *E;
	const EncodeTables *T;
	const unsigned char *frames;
	size_t bpl, frame_stride;
	int cn;
	short *coef;
	unsigned *bits, *counts, *istart, *freq, *hdr_end;
	unsigned long long *totals, *lengths, *at;
	unsigned char *raw;
	void *huff;				   /* the frames' HuffSet<E->ntab> */
	const unsigned char *tmpl; /* the plan's header */
	unsigned char *slots;	   /* the frames' header slots */
	unsigned char *summ;	   /* progressive: unit summaries, flushed runs, deferred correction bits */
	unsigned *runs, *dslot;
	unsigned short *doff;
	int *bad;
};

/* a sequential chunk through the lengths: 6 launches with the standard tables and no restart intervals, +1 with restart
 * intervals (jpeg_segments_kernel), +2 with optimised tables (jpeg_stats_kernel, jpeg_tables_kernel); returns the launch
 * count, -1 when the counts could not be cleared
 */
template <bool kOpt, bool kRestart>
int
launch_chunk(const ChunkArgs &A, cudaStream_t s)
{
	const EncodePlan &E = *A.E;
	const EncodeGeom &G = E.G;
	const ScanScript &P = E.P;
	const int mcus = G.mcus_x * G.mcus_y, cn = A.cn, nslots = (int) E.nslots;
	const dim3 per_block((G.blocks + 127) / 128, cn), per_span((E.max_chunks + 127) / 128, cn);
	HuffSet<4> *huff = (HuffSet<4> *) A.huff;
	/* the frames' own headers, or the batch's for every frame */
	const int hend_stride = kOpt ? 1 : 0;
	int launches = 6;
	jpeg_fdct_kernel<<<dim3((mcus + 127) / 128, cn), 128, 0, s>>>(G, A.T, A.frames, A.bpl, A.frame_stride, A.coef);
	if (kOpt) {
		if (cudaMemsetAsync(A.freq, 0, (size_t) cn * 4 * 256 * sizeof(unsigned), s) != cudaSuccess)
			return -1;
		jpeg_stats_kernel<<<per_block, 128, 0, s>>>(G, A.T, A.coef, P.restart, A.freq);
		jpeg_tables_kernel<4><<<cn, 32 * 4, 0, s>>>(P, A.freq, huff, A.tmpl, A.slots, kHeaderSlot, A.hdr_end, A.bad);
		launches += 2;
	}
	jpeg_count_kernel<kOpt, kRestart><<<per_block, 128, 0, s>>>(G, A.T, huff, P.restart, A.coef, A.bits);
	jpeg_bitscan_kernel<<<cn, 1024, 0, s>>>(nslots, A.bits, A.totals);
	if (kRestart) {
		const IntervalSlots M = {(unsigned) (P.restart * G.blocks_per_mcu), (unsigned) P.nseg, (unsigned) G.blocks};
		jpeg_segments_kernel<<<cn, 1024, 0, s>>>(M, P.nseg, nslots, A.bits, A.totals, A.istart);
		launches++;
	}
	jpeg_emit_kernel<kOpt, kRestart><<<per_block, 128, 0, s>>>(G, A.T, huff, P.restart, P.nseg, A.istart, A.coef, A.bits, (unsigned *) A.raw,
		E.raw_bytes / 4);
	constexpr int kInserts = kRestart ? kRestartMarkers : kOneSegment;
	jpeg_stuffcount_kernel<kInserts><<<per_span, 128, 0, s>>>(P, A.totals, A.raw, E.raw_bytes, E.max_chunks, A.istart, A.hdr_end, hend_stride, A.counts);
	jpeg_ffscan_kernel<<<cn, 1024, 0, s>>>(A.totals, E.max_chunks, A.counts, A.hdr_end, hend_stride, A.lengths);
	return launches;
}

/* a progressive chunk through the lengths: 10 launches whatever the frame count, scan count or restart interval -- FDCT,
 * summaries, chain walk, tables and headers, bit counts, bit prefix sum, segments, emit, and the first two stuffing passes;
 * -1 when the counts could not be cleared
 */
int
launch_progressive(const ChunkArgs &A, cudaStream_t s)
{
	const EncodePlan &E = *A.E;
	const EncodeGeom &G = E.G;
	const ScanScript &P = E.P;
	const int mcus = G.mcus_x * G.mcus_y, cn = A.cn, nslots = (int) E.nslots;
	const dim3 per_unit((P.units + 127) / 128, cn), per_span((E.max_chunks + 127) / 128, cn);
	HuffSet<kMaxProgTables> *huff = (HuffSet<kMaxProgTables> *) A.huff;
	jpeg_fdct_kernel<<<dim3((mcus + 127) / 128, cn), 128, 0, s>>>(G, A.T, A.frames, A.bpl, A.frame_stride, A.coef);
	if (cudaMemsetAsync(A.freq, 0, (size_t) cn * kMaxProgTables * 256 * sizeof(unsigned), s) != cudaSuccess)
		return -1;
	jpeg_prog_summary_kernel<<<per_unit, 128, 0, s>>>(G, P, A.T, A.coef, A.summ, A.freq);
	jpeg_prog_walk_kernel<<<dim3((P.nseg + 127) / 128, cn), 128, 0, s>>>(P, A.summ, A.runs, A.dslot, A.doff, A.freq);
	jpeg_tables_kernel<kMaxProgTables><<<cn, 32 * kMaxProgTables, 0, s>>>(P, A.freq, huff, A.tmpl, A.slots, kProgHeaderSlot, A.hdr_end, A.bad);
	jpeg_prog_count_kernel<<<per_unit, 128, 0, s>>>(G, P, A.T, huff, A.coef, A.runs, A.bits);
	jpeg_bitscan_kernel<<<cn, 1024, 0, s>>>(nslots, A.bits, A.totals);
	jpeg_segments_kernel<<<cn, 1024, 0, s>>>(ScriptSlots{P}, P.nseg, nslots, A.bits, A.totals, A.istart);
	jpeg_prog_emit_kernel<<<per_unit, 128, 0, s>>>(G, P, A.T, huff, A.istart, A.coef, A.bits, A.summ, A.runs, A.dslot, A.doff, (unsigned *) A.raw,
		E.raw_bytes / 4);
	jpeg_stuffcount_kernel<kScanHeaders><<<per_span, 128, 0, s>>>(P, A.totals, A.raw, E.raw_bytes, E.max_chunks, A.istart, A.hdr_end, P.nscans, A.counts);
	jpeg_ffscan_kernel<<<cn, 1024, 0, s>>>(A.totals, E.max_chunks, A.counts, A.hdr_end, P.nscans, A.lengths);
	return 10;
}

/* stuffing, pass 3, every kind of chunk: each frame's stream at out + A.at[frame] */
void
launch_stuffcopy(const ChunkArgs &A, unsigned char *out, cudaStream_t s)
{
	const EncodePlan &E = *A.E;
	const ScanScript &P = E.P;
	const dim3 per_span((E.max_chunks + 127) / 128, A.cn);
	/* the frames' own headers, or the chunk's for every frame */
	const unsigned char *hdr = E.opt ? A.slots : A.tmpl;
	const size_t hdr_stride = E.opt ? E.slot : 0;
	const int hend_stride = E.prog ? P.nscans : E.opt ? 1 : 0;
	const auto copy = E.prog ? jpeg_stuffcopy_kernel<kScanHeaders> : P.restart ? jpeg_stuffcopy_kernel<kRestartMarkers> : jpeg_stuffcopy_kernel<kOneSegment>;
	copy<<<per_span, 128, 0, s>>>(P, A.totals, A.raw, E.raw_bytes, E.max_chunks, A.counts, hdr, hdr_stride, A.hdr_end, hend_stride, A.istart, A.at, out,
		A.lengths);
}

/* cn equally sized 8-bit frames (1 or 3 bands) at src (device memory) -> their streams, with vips_jpegsave's options:
 * sequential with the standard tables or, optimize_coding, per-frame tables from the frame's symbol counts; interlace,
 * progressive with the scan script of jpeg_simple_progression, every scan with its own optimal tables; restart_interval
 * MCUs per restart interval (0: none).  7 / 8 / 9 / 10 launches per chunk for a sequential stream, 11 for a progressive one.
 */
int
jpeg_chunk(const char *domain, const EncodePlan &E, const unsigned char *src, size_t bpl, size_t frame_stride, int cn, const EncodePlace &place,
	cudaStream_t s)
{
	const Scratch S = carve(E, cn);
	char *scratch = nullptr;
	if (dev_alloc(domain, (void **) &scratch, S.bytes, s))
		return -1;
	const unsigned header_len = (unsigned) E.header.size();
	int rc = -1;
	do {
		/* tables and header (with the standard tables, its length too) from pageable memory: small, staged by the driver
		 * before the call returns
		 */
		if (cudaMemcpyAsync(scratch + S.tab, &E.T, sizeof(E.T), cudaMemcpyHostToDevice, s) != cudaSuccess ||
			cudaMemcpyAsync(scratch + S.hdr, E.header.data(), E.header.size(), cudaMemcpyHostToDevice, s) != cudaSuccess ||
			(!E.opt && cudaMemcpyAsync(scratch + S.hend, &header_len, sizeof(header_len), cudaMemcpyHostToDevice, s) != cudaSuccess) ||
			cudaMemsetAsync(scratch + S.raw, 0, (size_t) cn * E.raw_bytes, s) != cudaSuccess ||
			cudaMemsetAsync(scratch + S.bad, 0, sizeof(int), s) != cudaSuccess) {
			cuda_fail(domain, cudaGetLastError(), "jpeg encode setup");
			break;
		}
		ChunkArgs A;
		A.E = &E;
		A.T = (const EncodeTables *) (scratch + S.tab);
		A.frames = src;
		A.bpl = bpl;
		A.frame_stride = frame_stride;
		A.cn = cn;
		A.coef = (short *) (scratch + S.coef);
		A.bits = (unsigned *) (scratch + S.bits);
		A.counts = (unsigned *) (scratch + S.cnt);
		A.istart = (unsigned *) (scratch + S.ist);
		A.freq = (unsigned *) (scratch + S.freq);
		A.hdr_end = (unsigned *) (scratch + S.hend);
		A.totals = (unsigned long long *) (scratch + S.tot);
		A.lengths = (unsigned long long *) (scratch + S.len);
		A.at = (unsigned long long *) (scratch + S.at);
		A.raw = (unsigned char *) (scratch + S.raw);
		A.huff = scratch + S.huff;
		A.tmpl = (const unsigned char *) (scratch + S.hdr);
		A.slots = (unsigned char *) (scratch + S.slots);
		A.summ = (unsigned char *) (scratch + S.summ);
		A.runs = (unsigned *) (scratch + S.runs);
		A.dslot = (unsigned *) (scratch + S.dslot);
		A.doff = (unsigned short *) (scratch + S.doff);
		A.bad = (int *) (scratch + S.bad);
		const bool restart = E.P.restart > 0;
		const int launches = E.prog ? launch_progressive(A, s)
						   : E.opt	? (restart ? launch_chunk<true, true>(A, s) : launch_chunk<true, false>(A, s))
									: (restart ? launch_chunk<false, true>(A, s) : launch_chunk<false, false>(A, s));
		cudaError_t e = cudaGetLastError();
		if (e == cudaSuccess && launches < 0)
			e = cudaErrorUnknown;
		if (e != cudaSuccess) {
			cuda_fail(domain, e, "jpeg encode kernels launch");
			break;
		}
		count_launch(launches);
		/* read back with the lengths: place synchronises */
		int bad = 0;
		unsigned char *out = nullptr;
		if (cudaMemcpyAsync(&bad, scratch + S.bad, sizeof(int), cudaMemcpyDeviceToHost, s) != cudaSuccess) {
			cuda_fail(domain, cudaGetLastError(), "jpeg encode");
			break;
		}
		if (place(A.lengths, sizeof(unsigned long long), A.at, &out))
			break;
		if (bad) {
			/* libjpeg's JERR_HUFF_CLEN_OVERFLOW: a symbol distribution no image of the sizes taken here produces */
			error(domain, "optimised Huffman table: a code longer than 32 bits");
			break;
		}
		launch_stuffcopy(A, out, s);
		count_launch(1);
		if ((e = cudaGetLastError()) != cudaSuccess) {
			cuda_fail(domain, e, "jpeg_stuffcopy_kernel");
			break;
		}
		rc = 0;
	} while (0);
	dev_free(scratch, s);
	return rc;
}

} // namespace

int
jpeg_encoder(const char *domain, int w, int h, int bands, const VB200JpegSaveOptions &o, Encoder *enc)
{
	EncodePlan E;
	if (make_plan(domain, w, h, bands, o, &E))
		return -1;
	enc->scratch_bytes = carve(E, 1).bytes;
	/* the header slot, the raw data's bound, FF Dn or a scan header (counted in the slot) before each segment, EOI */
	enc->stream_bytes = E.slot + E.scan_bound + 2 * (size_t) E.P.nseg + 2;
	enc->chunk = [domain, E](const unsigned char *src, size_t bpl, size_t frame_stride, int cn, const EncodePlace &place, cudaStream_t s) {
		return jpeg_chunk(domain, E, src, bpl, frame_stride, cn, place, s);
	};
	return 0;
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

/* a host twin's set-up: the geometry, the tables and the frame's quantised coefficients, MCU by MCU through
 * jpeg_fdct_kernel's code
 */
int
host_coefficients(const char *domain, const unsigned char *img, size_t bpl, int w, int h, int bands, int quality, int subsample_mode, int restart,
	EncodeGeom *G, EncodeTables *T, std::vector<short> &coef)
{
	if (make_geom(domain, w, h, bands, quality, subsample_mode, G) || check_restart(domain, restart))
		return -1;
	make_tables(quality, T);
	coef.assign((size_t) G->blocks * 64, 0);
	for (int my = 0; my < G->mcus_y; my++)
		for (int mx = 0; mx < G->mcus_x; mx++)
			encode_mcu(*G, T->q, img, bpl, mx, my, coef.data() + ((size_t) my * G->mcus_x + mx) * G->blocks_per_mcu * 64);
	return 0;
}

/* a host twin's optimal table from the symbol counts freq[257] (consumed): bits / huffval for its DHT, and the code /
 * length per symbol co / si
 */
int
host_table(const char *domain, unsigned *freq, unsigned char *bits, unsigned char *huffval, unsigned *co, unsigned char *si)
{
	if (host_optimal_table(freq, bits, huffval)) {
		error(domain, "optimised Huffman table: a code longer than 32 bits");
		return -1;
	}
	derive_codes(bits + 1, huffval, co, si);
	return 0;
}

/* the whole encoder on the CPU through the same per-block code, in the order libjpeg runs it: statistics and table
 * generation when optimising, then the scan with its restart markers (test hook)
 */
int
host_jpeg_encode(const char *domain, const unsigned char *img, size_t bpl, int w, int h, int bands, int quality, int subsample_mode, int optimize,
	int restart, std::vector<unsigned char> &out)
{
	EncodeGeom G;
	EncodeTables T;
	std::vector<short> coef;
	if (host_coefficients(domain, img, bpl, w, h, bands, quality, subsample_mode, restart, &G, &T, coef))
		return -1;
	const unsigned bpm = (unsigned) G.blocks_per_mcu;
	unsigned char bits[4][17], huffval[4][256];
	HuffSet<4> fh;
	const unsigned (*co)[256] = T.ehufco;
	const unsigned char (*si)[256] = T.ehufsi;
	if (optimize) {
		std::vector<unsigned> freq(4 * 257, 0);
		for (unsigned b = 0; b < (unsigned) G.blocks; b++)
			walk_block(
				T.zz, coef.data() + (size_t) b * 64, block_comp(G, (int) (b % bpm)), previous_dc(G, coef.data(), b, restart),
				[&](int t, int s) { freq[t * 257 + s]++; }, [](unsigned, int) {});
		for (int t = 0; t < (G.ncomp == 1 ? 2 : 4); t++)
			if (host_table(domain, freq.data() + t * 257, bits[t], huffval[t], fh.ehufco[t], fh.ehufsi[t]))
				return -1;
		co = fh.ehufco;
		si = fh.ehufsi;
	}
	else
		standard_tables(bits, huffval);
	ScanScript P;
	scan_script(G, restart, false, &P);
	header_prefix(G, T, out);
	put_dhts(G, bits, huffval, out);
	scan_suffix(G, P.s[0], true, restart, out);
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

/* jcphuff.c on the CPU, serially and in libjpeg's order, for one scan of the progressive script: encode_mcu_DC_first,
 * encode_mcu_DC_refine, encode_mcu_AC_first, encode_mcu_AC_refine with emit_eobrun inline and emit_restart between
 * restart intervals.  counts != null: the statistics pass (gather_statistics; finish_pass_gather_phuff's last
 * emit_eobrun), counts[table of the scan][symbol]; else the output pass with the scan's tables co / si into out (stuffed,
 * RSTn between intervals, finish_pass_phuff's flush).  Deliberately not the device's decomposition, which it checks.
 */
void
host_prog_scan(const EncodeGeom &G, const Scan &S, const short *coef, int restart, unsigned (*counts)[257], const unsigned (*co)[256],
	const unsigned char (*si)[256], std::vector<unsigned char> &out, unsigned long long *events)
{
	const bool gather = counts != nullptr;
	unsigned long long put_buffer = 0;
	int put_bits = 0;
	auto emit_bits = [&](unsigned code, int size) {
		if (gather)
			return;
		put_buffer = (put_buffer << size) | (code & ((1u << size) - 1));
		put_bits += size;
		while (put_bits >= 8) {
			const unsigned char c = (unsigned char) (put_buffer >> (put_bits - 8));
			out.push_back(c);
			if (c == 0xFF)
				out.push_back(0);
			put_bits -= 8;
		}
	};
	auto flush_bits = [&]() {
		emit_bits(0x7F, 7); /* fill any partial byte with ones */
		put_buffer = 0;
		put_bits = 0;
	};
	auto emit_symbol = [&](int tbl, int symbol) {
		if (gather)
			counts[tbl][symbol]++;
		else
			emit_bits(co[tbl][symbol], si[tbl][symbol]);
	};
	int EOBRUN = 0, BE = 0;
	char bit_buffer[kMaxCorrBits];
	int last_dc_val[3] = {0, 0, 0};
	auto emit_eobrun = [&]() {
		if (EOBRUN > 0) {
			int temp = EOBRUN, nbits = 0;
			while ((temp >>= 1))
				nbits++;
			emit_symbol(0, nbits << 4);
			if (nbits)
				emit_bits((unsigned) EOBRUN, nbits);
			EOBRUN = 0;
			for (int i = 0; i < BE; i++)
				emit_bits((unsigned) bit_buffer[i], 1);
			BE = 0;
		}
	};
	auto emit_restart = [&](int restart_num) {
		emit_eobrun();
		if (!gather) {
			flush_bits();
			out.push_back(0xFF);
			out.push_back((unsigned char) (0xD0 + restart_num));
		}
		if (S.ss == 0)
			last_dc_val[0] = last_dc_val[1] = last_dc_val[2] = 0;
		else
			EOBRUN = BE = 0;
	};
	auto nbits_of = [](int temp) {
		int nbits = 0;
		while (temp) {
			nbits++;
			temp >>= 1;
		}
		return nbits;
	};
	int restarts_to_go = restart, next_restart_num = 0;
	for (int unit = 0; unit < S.units; unit++) {
		if (restart) {
			if (restarts_to_go == 0) {
				emit_restart(next_restart_num);
				restarts_to_go = restart;
				next_restart_num = (next_restart_num + 1) & 7;
			}
			restarts_to_go--;
		}
		if (S.ss == 0) {
			/* an interleaved MCU (a single block for greyscale) */
			for (int blkn = 0; blkn < G.blocks_per_mcu; blkn++) {
				const short *block = coef + ((size_t) unit * G.blocks_per_mcu + blkn) * 64;
				const int ci = block_comp(G, blkn);
				if (S.ah == 0) {
					const int temp2 = block[0] >> S.al; /* IRIGHT_SHIFT: arithmetic */
					int temp = temp2 - last_dc_val[ci];
					last_dc_val[ci] = temp2;
					int t2 = temp;
					if (temp < 0) {
						temp = -temp;
						t2--;
					}
					const int nbits = nbits_of(temp);
					emit_symbol(ci ? 1 : 0, nbits);
					if (nbits)
						emit_bits((unsigned) t2, nbits);
				}
				else
					emit_bits((unsigned) (block[0] >> S.al), 1);
			}
			continue;
		}
		const short *block = coef + (size_t) comp_block_index(G, S.comp, unit % S.ux, unit / S.ux) * 64;
		if (S.ah == 0) {
			int r = 0;
			for (int k = S.ss; k <= S.se; k++) {
				int temp = block[kZigzag[k]], temp2;
				if (temp == 0) {
					r++;
					continue;
				}
				if (temp < 0) {
					temp = -temp;
					temp >>= S.al;
					temp2 = ~temp;
				}
				else {
					temp >>= S.al;
					temp2 = temp;
				}
				if (temp == 0) {
					r++;
					continue;
				}
				if (EOBRUN > 0)
					emit_eobrun();
				while (r > 15) {
					emit_symbol(0, 0xF0);
					r -= 16;
				}
				const int nbits = nbits_of(temp);
				emit_symbol(0, (r << 4) + nbits);
				emit_bits((unsigned) temp2, nbits);
				r = 0;
			}
			if (r > 0) {
				EOBRUN++;
				if (EOBRUN == 0x7FFF) {
					if (!gather)
						events[0]++;
					emit_eobrun();
				}
			}
			continue;
		}
		int absvalues[64];
		int EOB = 0;
		for (int k = S.ss; k <= S.se; k++) {
			int temp = block[kZigzag[k]];
			if (temp < 0)
				temp = -temp;
			temp >>= S.al;
			absvalues[k] = temp;
			if (temp == 1)
				EOB = k;
		}
		int r = 0, BR = 0;
		char *BR_buffer = bit_buffer + BE;
		for (int k = S.ss; k <= S.se; k++) {
			int temp = absvalues[k];
			if (temp == 0) {
				r++;
				continue;
			}
			while (r > 15 && k <= EOB) {
				emit_eobrun();
				if (!gather)
					events[2]++;
				emit_symbol(0, 0xF0);
				r -= 16;
				for (int i = 0; i < BR; i++)
					emit_bits((unsigned) BR_buffer[i], 1);
				BR_buffer = bit_buffer;
				BR = 0;
			}
			if (temp > 1) {
				BR_buffer[BR++] = (char) (temp & 1);
				continue;
			}
			emit_eobrun();
			emit_symbol(0, (r << 4) + 1);
			emit_bits(block[kZigzag[k]] < 0 ? 0u : 1u, 1);
			for (int i = 0; i < BR; i++)
				emit_bits((unsigned) BR_buffer[i], 1);
			BR_buffer = bit_buffer;
			BR = 0;
			r = 0;
		}
		if (r > 0 || BR > 0) {
			EOBRUN++;
			BE += BR;
			if (EOBRUN == 0x7FFF || BE > kMaxCorrBits - 64 + 1) {
				if (!gather)
					events[EOBRUN == 0x7FFF ? 0 : 1]++;
				emit_eobrun();
			}
		}
	}
	emit_eobrun();
	if (!gather)
		flush_bits();
}

/* the progressive stream on the CPU (test hook): libjpeg's multi-pass order, scan by scan a statistics pass, the scan's
 * tables (jpeg_gen_optimal_table), its header (DHTs, DRI before the first scan, SOS) and the output pass.  events[3]
 * counts what the output passes reach: EOB runs forced out at 0x7FFF blocks, EOB runs forced out by the correction-bit
 * buffer, ZRLs in refinement scans.
 */
int
host_jpeg_encode_progressive(const char *domain, const unsigned char *img, size_t bpl, int w, int h, int bands, int quality, int subsample_mode,
	int restart, std::vector<unsigned char> &out, unsigned long long *events)
{
	EncodeGeom G;
	EncodeTables T;
	std::vector<short> coef;
	if (host_coefficients(domain, img, bpl, w, h, bands, quality, subsample_mode, restart, &G, &T, coef))
		return -1;
	ScanScript P;
	scan_script(G, restart, true, &P);
	header_prefix(G, T, out, 0xFFC2);
	for (int s = 0; s < P.nscans; s++) {
		const Scan &S = P.s[s];
		HuffSet<2> fh; /* tables 0, 1 of the scan */
		if (S.nt) {
			unsigned counts[2][257];
			memset(counts, 0, sizeof(counts));
			host_prog_scan(G, S, coef.data(), restart, counts, nullptr, nullptr, out, events);
			for (int t = 0; t < S.nt; t++) {
				unsigned char bits[17], huffval[256];
				if (host_table(domain, counts[t], bits, huffval, fh.ehufco[t], fh.ehufsi[t]))
					return -1;
				unsigned char seg[4 + 17 + 256];
				const int n = put_dht(seg, P.tab_class[S.tab + t], bits, huffval);
				out.insert(out.end(), seg, seg + n);
			}
		}
		scan_suffix(G, S, s == 0, restart, out);
		host_prog_scan(G, S, coef.data(), restart, nullptr, fh.ehufco, fh.ehufsi, out, events);
	}
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
	const VB200JpegSaveOptions opt = {quality, subsample_mode, 0, 0, 0};
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
	unsigned long long events[3] = {0, 0, 0};
	if (opt->interlace ? host_jpeg_encode_progressive("jpeg_encode (host twin)", (const unsigned char *) pixels, bpl, width, height, bands, opt->Q,
							 opt->subsample_mode, opt->restart_interval, o, events)
					   : host_jpeg_encode("jpeg_encode (host twin)", (const unsigned char *) pixels, bpl, width, height, bands, opt->Q,
							 opt->subsample_mode, opt->optimize_coding, opt->restart_interval, o))
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

/* Test hook, host only: what the host twin's progressive coder reached for an image (options as
 * vb200_debug_jpeg_encode_opts, interlace implied): events[0] EOB runs forced out at 0x7FFF blocks, [1] EOB runs forced out
 * by the correction-bit buffer (BE > MAX_CORR_BITS - 63), [2] ZRLs in refinement scans
 */
extern "C" int
vb200_debug_jpeg_prog_events(const void *pixels, size_t bpl, int width, int height, int bands, const VB200JpegSaveOptions *opt,
	unsigned long long *events)
{
	if (!opt || !events) {
		error("jpeg_prog_events (host twin)", "null argument");
		return -1;
	}
	std::vector<unsigned char> o;
	events[0] = events[1] = events[2] = 0;
	return host_jpeg_encode_progressive("jpeg_prog_events (host twin)", (const unsigned char *) pixels, bpl, width, height, bands, opt->Q,
		opt->subsample_mode, opt->restart_interval, o, events);
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
	const VB200JpegSaveOptions opt = {Q, subsample_mode, 0, 0, 0};
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
	return encode_batch_abi(domain, opt, [&](Encoder *enc) { return jpeg_encoder(domain, width, height, bands, *opt, enc); }, frames, frames_location, bpl,
		frame_stride, n, width, height, bands, out, out_location, out_stride, lengths);
}

