/* webp.cu -- vips_webpload_buffer's lossy, still, opaque frames decoded on the device.
 *
 * What the reference does (foreign/webp2vips.c through webpload.c's buffer loader): the sniff is RIFF + 4 bytes + WEBP
 * (:321); read_header (:400-560) runs WebPDemux and reads the format flags; read_frame (:600-645) decodes each frame with
 * WebPDecode in MODE_RGBA and WebPInitDecoderConfig's defaults (fancy upsampling on, no dithering); without alpha the
 * fourth band is dropped (:740-790), so a lossy opaque frame loads as 3-band uchar sRGB.  The pixels are libwebp's, and
 * libwebp decodes a lossy frame as the VP8 key-frame format (RFC 6386) specifies; the code below is written from that
 * format and the WebP container's, and pinned pixel for pixel against libwebp by the test-suite.
 *
 * Scope: a RIFF / WEBP stream whose image is one "VP8 " chunk, either alone (the simple format) or after a VP8X chunk
 * whose flags have neither ANIMATION nor ALPHA (its ICCP / EXIF / XMP chunks do not change the pixels), and whose key
 * frame is up to 16383 x 16383 with every key-frame feature: segmentation, 1 to 8 token partitions, the simple and the
 * normal loop filter, skip flags, probability updates, every intra mode.  Returned -1 with the reason (the host keeps
 * webpload): VP8L (lossless), ALPH or the ALPHA flag, ANIM / ANMF, a frame that is not a key frame, a bad signature or
 * chunk sizes that run past the RIFF or the buffer, a VP8X canvas that differs from the frame.  A frame libwebp refuses
 * while decoding (a segment / filter header or a partition that ends early, a bad partition table) fails the batch.
 *
 * Device pipeline per chunk of frames (the VP8 chunk payloads are all that crosses PCIe):
 *   webp_header_kernel  one thread per frame: the bool-coded frame header of partition 0, then every macroblock's segment,
 *                       skip flag and intra modes (the 4x4 sub-mode contexts run along the row and down the columns)
 *   webp_token_kernel   one thread per frame: the residual tokens of every macroblock, row r from partition r mod P,
 *                       dequantised, the Y2 block through the inverse WHT; out: coefficients and libwebp's per-block
 *                       non-zero codes
 *   webp_recon_kernel   one CTA per frame: intra prediction from unfiltered neighbours plus the inverse DCT, one thread
 *                       per macroblock along the wavefront x + 2y = t; then the loop filter in raster order's
 *                       dependencies, the same wavefront again, in place
 *   webp_rgb_kernel     one thread per pixel, only once every frame of the chunk has decoded clean: libwebp's fancy
 *                       upsampler and its 14-bit YUV -> RGB, cropped to w x h, written at the caller's stride
 *   webp_scaled_rgb_kernel  in its place for vips_webpload_buffer's `scale` (libwebp's scaled decode, webp2vips.c:630-634):
 *                       one thread per output pixel, its Y, U and V samples from libwebp's rescaler in closed form, then
 *                       the same YUV -> RGB; the reconstruction then skips the filter pass when libwebp bypasses it
 * The per-symbol, per-block and per-pixel code is __host__ __device__: vb200_debug_webp_decode runs it on the CPU in raster
 * order, so that the CPU test-suite pins it against libwebp without a GPU.
 */
#include <algorithm>
#include <cmath>
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

/* ------------------------------------------------------------------ the format's constant tables (RFC 6386) */

/* Mode numbers are libwebp's, which are the leaves of the key-frame sub-block mode tree in order: the 16 x 16 and chroma
 * modes share DC / TM / V / H with the first four sub-block modes.
 */
enum { M_DC = 0, M_TM = 1, M_VE = 2, M_HE = 3, M_RD = 4, M_VR = 5, M_LD = 6, M_VL = 7, M_HD = 8, M_HU = 9 };
/* DC prediction with missing edges, for the 16 x 16 and chroma predictors */
enum { M_DC_NOTOP = 10, M_DC_NOLEFT = 11, M_DC_NOTOPLEFT = 12 };

struct WebpTables {
	unsigned char coeff0[4][8][3][11];		 /* default coefficient probabilities (13.5) */
	unsigned char coeff_update[4][8][3][11]; /* their update probabilities (13.4) */
	unsigned char bmodes[10][10][9];		 /* key-frame sub-block mode probabilities [above][left] (11.5) */
	unsigned char dc[128];					 /* dc quantiser steps (14.1) */
	unsigned short ac[128];					 /* ac quantiser steps */
	unsigned char zigzag[16];
	unsigned char bands[17]; /* coefficient position -> band, and a 0 past the end */
	unsigned char cat[4][12]; /* DCT_CAT3 .. DCT_CAT6 extra-bit probabilities, 0-terminated */
};

#define WEBP_TABLES_INIT                                                                                                                                   \
	{                                                                                                                                                      \
		{{{{128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128}, {128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128},                               \
			  {128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128}},                                                                                    \
			 {{253, 136, 254, 255, 228, 219, 128, 128, 128, 128, 128}, {189, 129, 242, 255, 227, 213, 255, 219, 128, 128, 128},                            \
				 {106, 126, 227, 252, 214, 209, 255, 255, 128, 128, 128}},                                                                                 \
			 {{1, 98, 248, 255, 236, 226, 255, 255, 128, 128, 128}, {181, 133, 238, 254, 221, 234, 255, 154, 128, 128, 128},                               \
				 {78, 134, 202, 247, 198, 180, 255, 219, 128, 128, 128}},                                                                                  \
			 {{1, 185, 249, 255, 243, 255, 128, 128, 128, 128, 128}, {184, 150, 247, 255, 236, 224, 128, 128, 128, 128, 128},                              \
				 {77, 110, 216, 255, 236, 230, 128, 128, 128, 128, 128}},                                                                                  \
			 {{1, 101, 251, 255, 241, 255, 128, 128, 128, 128, 128}, {170, 139, 241, 252, 236, 209, 255, 255, 128, 128, 128},                              \
				 {37, 116, 196, 243, 228, 255, 255, 255, 128, 128, 128}},                                                                                  \
			 {{1, 204, 254, 255, 245, 255, 128, 128, 128, 128, 128}, {207, 160, 250, 255, 238, 128, 128, 128, 128, 128, 128},                              \
				 {102, 103, 231, 255, 211, 171, 128, 128, 128, 128, 128}},                                                                                 \
			 {{1, 152, 252, 255, 240, 255, 128, 128, 128, 128, 128}, {177, 135, 243, 255, 234, 225, 128, 128, 128, 128, 128},                              \
				 {80, 129, 211, 255, 194, 224, 128, 128, 128, 128, 128}},                                                                                  \
			 {{1, 1, 255, 128, 128, 128, 128, 128, 128, 128, 128}, {246, 1, 255, 128, 128, 128, 128, 128, 128, 128, 128},                                  \
				 {255, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128}}},                                                                                \
			{{{198, 35, 237, 223, 193, 187, 162, 160, 145, 155, 62}, {131, 45, 198, 221, 172, 176, 220, 157, 252, 221, 1},                                 \
				 {68, 47, 146, 208, 149, 167, 221, 162, 255, 223, 128}},                                                                                   \
				{{1, 149, 241, 255, 221, 224, 255, 255, 128, 128, 128}, {184, 141, 234, 253, 222, 220, 255, 199, 128, 128, 128},                           \
					{81, 99, 181, 242, 176, 190, 249, 202, 255, 255, 128}},                                                                                \
				{{1, 129, 232, 253, 214, 197, 242, 196, 255, 255, 128}, {99, 121, 210, 250, 201, 198, 255, 202, 128, 128, 128},                            \
					{23, 91, 163, 242, 170, 187, 247, 210, 255, 255, 128}},                                                                                \
				{{1, 200, 246, 255, 234, 255, 128, 128, 128, 128, 128}, {109, 178, 241, 255, 231, 245, 255, 255, 128, 128, 128},                           \
					{44, 130, 201, 253, 205, 192, 255, 255, 128, 128, 128}},                                                                               \
				{{1, 132, 239, 251, 219, 209, 255, 165, 128, 128, 128}, {94, 136, 225, 251, 218, 190, 255, 255, 128, 128, 128},                            \
					{22, 100, 174, 245, 186, 161, 255, 199, 128, 128, 128}},                                                                               \
				{{1, 182, 249, 255, 232, 235, 128, 128, 128, 128, 128}, {124, 143, 241, 255, 227, 234, 128, 128, 128, 128, 128},                           \
					{35, 77, 181, 251, 193, 211, 255, 205, 128, 128, 128}},                                                                                \
				{{1, 157, 247, 255, 236, 231, 255, 255, 128, 128, 128}, {121, 141, 235, 255, 225, 227, 255, 255, 128, 128, 128},                           \
					{45, 99, 188, 251, 195, 217, 255, 224, 128, 128, 128}},                                                                                \
				{{1, 1, 251, 255, 213, 255, 128, 128, 128, 128, 128}, {203, 1, 248, 255, 255, 128, 128, 128, 128, 128, 128},                               \
					{137, 1, 177, 255, 224, 255, 128, 128, 128, 128, 128}}},                                                                               \
			{{{253, 9, 248, 251, 207, 208, 255, 192, 128, 128, 128}, {175, 13, 224, 243, 193, 185, 249, 198, 255, 255, 128},                               \
				 {73, 17, 171, 221, 161, 179, 236, 167, 255, 234, 128}},                                                                                   \
				{{1, 95, 247, 253, 212, 183, 255, 255, 128, 128, 128}, {239, 90, 244, 250, 211, 209, 255, 255, 128, 128, 128},                             \
					{155, 77, 195, 248, 188, 195, 255, 255, 128, 128, 128}},                                                                               \
				{{1, 24, 239, 251, 218, 219, 255, 205, 128, 128, 128}, {201, 51, 219, 255, 196, 186, 128, 128, 128, 128, 128},                             \
					{69, 46, 190, 239, 201, 218, 255, 228, 128, 128, 128}},                                                                                \
				{{1, 191, 251, 255, 255, 128, 128, 128, 128, 128, 128}, {223, 165, 249, 255, 213, 255, 128, 128, 128, 128, 128},                           \
					{141, 124, 248, 255, 255, 128, 128, 128, 128, 128, 128}},                                                                              \
				{{1, 16, 248, 255, 255, 128, 128, 128, 128, 128, 128}, {190, 36, 230, 255, 236, 255, 128, 128, 128, 128, 128},                             \
					{149, 1, 255, 128, 128, 128, 128, 128, 128, 128, 128}},                                                                                \
				{{1, 226, 255, 128, 128, 128, 128, 128, 128, 128, 128}, {247, 192, 255, 128, 128, 128, 128, 128, 128, 128, 128},                           \
					{240, 128, 255, 128, 128, 128, 128, 128, 128, 128, 128}},                                                                              \
				{{1, 134, 252, 255, 255, 128, 128, 128, 128, 128, 128}, {213, 62, 250, 255, 255, 128, 128, 128, 128, 128, 128},                            \
					{55, 93, 255, 128, 128, 128, 128, 128, 128, 128, 128}},                                                                                \
				{{128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128}, {128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128},                         \
					{128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128}}},                                                                             \
			{{{202, 24, 213, 235, 186, 191, 220, 160, 240, 175, 255}, {126, 38, 182, 232, 169, 184, 228, 174, 255, 187, 128},                              \
				 {61, 46, 138, 219, 151, 178, 240, 170, 255, 216, 128}},                                                                                   \
				{{1, 112, 230, 250, 199, 191, 247, 159, 255, 255, 128}, {166, 109, 228, 252, 211, 215, 255, 174, 128, 128, 128},                           \
					{39, 77, 162, 232, 172, 180, 245, 178, 255, 255, 128}},                                                                                \
				{{1, 52, 220, 246, 198, 199, 249, 220, 255, 255, 128}, {124, 74, 191, 243, 183, 193, 250, 221, 255, 255, 128},                             \
					{24, 71, 130, 219, 154, 170, 243, 182, 255, 255, 128}},                                                                                \
				{{1, 182, 225, 249, 219, 240, 255, 224, 128, 128, 128}, {149, 150, 226, 252, 216, 205, 255, 171, 128, 128, 128},                           \
					{28, 108, 170, 242, 183, 194, 254, 223, 255, 255, 128}},                                                                               \
				{{1, 81, 230, 252, 204, 203, 255, 192, 128, 128, 128}, {123, 102, 209, 247, 188, 196, 255, 233, 128, 128, 128},                            \
					{20, 95, 153, 243, 164, 173, 255, 203, 128, 128, 128}},                                                                                \
				{{1, 222, 248, 255, 216, 213, 128, 128, 128, 128, 128}, {168, 175, 246, 252, 235, 205, 255, 255, 128, 128, 128},                           \
					{47, 116, 215, 255, 211, 212, 255, 255, 128, 128, 128}},                                                                               \
				{{1, 121, 236, 253, 212, 214, 255, 255, 128, 128, 128}, {141, 84, 213, 252, 201, 202, 255, 219, 128, 128, 128},                            \
					{42, 80, 160, 240, 162, 185, 255, 205, 128, 128, 128}},                                                                                \
				{{1, 1, 255, 128, 128, 128, 128, 128, 128, 128, 128}, {244, 1, 255, 128, 128, 128, 128, 128, 128, 128, 128},                               \
					{238, 1, 255, 128, 128, 128, 128, 128, 128, 128, 128}}}},                                                                              \
			{{{{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},                           \
				  {255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                                \
				 {{176, 246, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {223, 241, 252, 255, 255, 255, 255, 255, 255, 255, 255},                        \
					 {249, 253, 253, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                             \
				 {{255, 244, 252, 255, 255, 255, 255, 255, 255, 255, 255}, {234, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255},                        \
					 {253, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                             \
				 {{255, 246, 254, 255, 255, 255, 255, 255, 255, 255, 255}, {239, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255},                        \
					 {254, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                             \
				 {{255, 248, 254, 255, 255, 255, 255, 255, 255, 255, 255}, {251, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255},                        \
					 {255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                             \
				 {{255, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255}, {251, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255},                        \
					 {254, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                             \
				 {{255, 254, 253, 255, 254, 255, 255, 255, 255, 255, 255}, {250, 255, 254, 255, 254, 255, 255, 255, 255, 255, 255},                        \
					 {254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                             \
				 {{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},                        \
					 {255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}}},                                                                            \
				{{{217, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {225, 252, 241, 253, 255, 255, 254, 255, 255, 255, 255},                        \
					 {234, 250, 241, 250, 253, 255, 253, 254, 255, 255, 255}},                                                                             \
					{{255, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {223, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{238, 253, 254, 254, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 248, 254, 255, 255, 255, 255, 255, 255, 255, 255}, {249, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 253, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {247, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255}, {252, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255}, {253, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 254, 253, 255, 255, 255, 255, 255, 255, 255, 255}, {250, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}}},                                                                         \
				{{{186, 251, 250, 255, 255, 255, 255, 255, 255, 255, 255}, {234, 251, 244, 254, 255, 255, 255, 255, 255, 255, 255},                        \
					 {251, 251, 243, 253, 254, 255, 254, 255, 255, 255, 255}},                                                                             \
					{{255, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255}, {236, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{251, 253, 253, 254, 254, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255}, {254, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {254, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}}},                                                                         \
				{{{248, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {250, 254, 252, 254, 255, 255, 255, 255, 255, 255, 255},                        \
					 {248, 254, 249, 253, 255, 255, 255, 255, 255, 255, 255}},                                                                             \
					{{255, 253, 253, 255, 255, 255, 255, 255, 255, 255, 255}, {246, 253, 253, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{252, 254, 251, 254, 254, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 254, 252, 255, 255, 255, 255, 255, 255, 255, 255}, {248, 254, 253, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{253, 255, 254, 254, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 251, 254, 255, 255, 255, 255, 255, 255, 255, 255}, {245, 251, 254, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{253, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 251, 253, 255, 255, 255, 255, 255, 255, 255, 255}, {252, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 252, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {249, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 255, 253, 255, 255, 255, 255, 255, 255, 255, 255}, {250, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}},                                                                          \
					{{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}, {254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},                     \
						{255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255}}}},                                                                        \
			{{{231, 120, 48, 89, 115, 113, 120, 152, 112}, {152, 179, 64, 126, 170, 118, 46, 70, 95}, {175, 69, 143, 80, 85, 82, 72, 155, 103},            \
				 {56, 58, 10, 171, 218, 189, 17, 13, 152}, {114, 26, 17, 163, 44, 195, 21, 10, 173}, {121, 24, 80, 195, 26, 62, 44, 64, 85},               \
				 {144, 71, 10, 38, 171, 213, 144, 34, 26}, {170, 46, 55, 19, 136, 160, 33, 206, 71}, {63, 20, 8, 114, 114, 208, 12, 9, 226},               \
				 {81, 40, 11, 96, 182, 84, 29, 16, 36}},                                                                                                   \
				{{134, 183, 89, 137, 98, 101, 106, 165, 148}, {72, 187, 100, 130, 157, 111, 32, 75, 80}, {66, 102, 167, 99, 74, 62, 40, 234, 128},         \
					{41, 53, 9, 178, 241, 141, 26, 8, 107}, {74, 43, 26, 146, 73, 166, 49, 23, 157}, {65, 38, 105, 160, 51, 52, 31, 115, 128},             \
					{104, 79, 12, 27, 217, 255, 87, 17, 7}, {87, 68, 71, 44, 114, 51, 15, 186, 23}, {47, 41, 14, 110, 182, 183, 21, 17, 194},              \
					{66, 45, 25, 102, 197, 189, 23, 18, 22}},                                                                                              \
				{{88, 88, 147, 150, 42, 46, 45, 196, 205}, {43, 97, 183, 117, 85, 38, 35, 179, 61}, {39, 53, 200, 87, 26, 21, 43, 232, 171},               \
					{56, 34, 51, 104, 114, 102, 29, 93, 77}, {39, 28, 85, 171, 58, 165, 90, 98, 64}, {34, 22, 116, 206, 23, 34, 43, 166, 73},              \
					{107, 54, 32, 26, 51, 1, 81, 43, 31}, {68, 25, 106, 22, 64, 171, 36, 225, 114}, {34, 19, 21, 102, 132, 188, 16, 76, 124},              \
					{62, 18, 78, 95, 85, 57, 50, 48, 51}},                                                                                                 \
				{{193, 101, 35, 159, 215, 111, 89, 46, 111}, {60, 148, 31, 172, 219, 228, 21, 18, 111}, {112, 113, 77, 85, 179, 255, 38, 120, 114},        \
					{40, 42, 1, 196, 245, 209, 10, 25, 109}, {88, 43, 29, 140, 166, 213, 37, 43, 154}, {61, 63, 30, 155, 67, 45, 68, 1, 209},              \
					{100, 80, 8, 43, 154, 1, 51, 26, 71}, {142, 78, 78, 16, 255, 128, 34, 197, 171}, {41, 40, 5, 102, 211, 183, 4, 1, 221},                \
					{51, 50, 17, 168, 209, 192, 23, 25, 82}},                                                                                              \
				{{138, 31, 36, 171, 27, 166, 38, 44, 229}, {67, 87, 58, 169, 82, 115, 26, 59, 179}, {63, 59, 90, 180, 59, 166, 93, 73, 154},               \
					{40, 40, 21, 116, 143, 209, 34, 39, 175}, {47, 15, 16, 183, 34, 223, 49, 45, 183}, {46, 17, 33, 183, 6, 98, 15, 32, 183},              \
					{57, 46, 22, 24, 128, 1, 54, 17, 37}, {65, 32, 73, 115, 28, 128, 23, 128, 205}, {40, 3, 9, 115, 51, 192, 18, 6, 223},                  \
					{87, 37, 9, 115, 59, 77, 64, 21, 47}},                                                                                                 \
				{{104, 55, 44, 218, 9, 54, 53, 130, 226}, {64, 90, 70, 205, 40, 41, 23, 26, 57}, {54, 57, 112, 184, 5, 41, 38, 166, 213},                  \
					{30, 34, 26, 133, 152, 116, 10, 32, 134}, {39, 19, 53, 221, 26, 114, 32, 73, 255}, {31, 9, 65, 234, 2, 15, 1, 118, 73},                \
					{75, 32, 12, 51, 192, 255, 160, 43, 51}, {88, 31, 35, 67, 102, 85, 55, 186, 85}, {56, 21, 23, 111, 59, 205, 45, 37, 192},              \
					{55, 38, 70, 124, 73, 102, 1, 34, 98}},                                                                                                \
				{{125, 98, 42, 88, 104, 85, 117, 175, 82}, {95, 84, 53, 89, 128, 100, 113, 101, 45}, {75, 79, 123, 47, 51, 128, 81, 171, 1},               \
					{57, 17, 5, 71, 102, 57, 53, 41, 49}, {38, 33, 13, 121, 57, 73, 26, 1, 85}, {41, 10, 67, 138, 77, 110, 90, 47, 114},                   \
					{115, 21, 2, 10, 102, 255, 166, 23, 6}, {101, 29, 16, 10, 85, 128, 101, 196, 26}, {57, 18, 10, 102, 102, 213, 34, 20, 43},             \
					{117, 20, 15, 36, 163, 128, 68, 1, 26}},                                                                                               \
				{{102, 61, 71, 37, 34, 53, 31, 243, 192}, {69, 60, 71, 38, 73, 119, 28, 222, 37}, {68, 45, 128, 34, 1, 47, 11, 245, 171},                  \
					{62, 17, 19, 70, 146, 85, 55, 62, 70}, {37, 43, 37, 154, 100, 163, 85, 160, 1}, {63, 9, 92, 136, 28, 64, 32, 201, 85},                 \
					{75, 15, 9, 9, 64, 255, 184, 119, 16}, {86, 6, 28, 5, 64, 255, 25, 248, 1}, {56, 8, 17, 132, 137, 255, 55, 116, 128},                  \
					{58, 15, 20, 82, 135, 57, 26, 121, 40}},                                                                                               \
				{{164, 50, 31, 137, 154, 133, 25, 35, 218}, {51, 103, 44, 131, 131, 123, 31, 6, 158}, {86, 40, 64, 135, 148, 224, 45, 183, 128},           \
					{22, 26, 17, 131, 240, 154, 14, 1, 209}, {45, 16, 21, 91, 64, 222, 7, 1, 197}, {56, 21, 39, 155, 60, 138, 23, 102, 213},               \
					{83, 12, 13, 54, 192, 255, 68, 47, 28}, {85, 26, 85, 85, 128, 128, 32, 146, 171}, {18, 11, 7, 63, 144, 171, 4, 4, 246},                \
					{35, 27, 10, 146, 174, 171, 12, 26, 128}},                                                                                             \
				{{190, 80, 35, 99, 180, 80, 126, 54, 45}, {85, 126, 47, 87, 176, 51, 41, 20, 32}, {101, 75, 128, 139, 118, 146, 116, 128, 85},             \
					{56, 41, 15, 176, 236, 85, 37, 9, 62}, {71, 30, 17, 119, 118, 255, 17, 18, 138}, {101, 38, 60, 138, 55, 70, 43, 26, 142},              \
					{146, 36, 19, 30, 171, 255, 97, 27, 20}, {138, 45, 61, 62, 219, 1, 81, 188, 64}, {32, 41, 20, 117, 151, 142, 20, 21, 163},             \
					{112, 19, 12, 61, 195, 128, 48, 4, 24}}},                                                                                              \
			{4, 5, 6, 7, 8, 9, 10, 10, 11, 12, 13, 14, 15, 16, 17, 17, 18, 19, 20, 20, 21, 21, 22, 22, 23, 23, 24, 25, 25, 26, 27, 28, 29, 30, 31, 32,  \
				33, 34, 35, 36, 37, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 46, 47, 48, 49, 50, 51, 52, 53, 54, 55, 56, 57, 58, 59, 60, 61, 62, 63, 64, \
				65, 66, 67, 68, 69, 70, 71, 72, 73, 74, 75, 76, 76, 77, 78, 79, 80, 81, 82, 83, 84, 85, 86, 87, 88, 89, 91, 93, 95, 96, 98, 100, 101,  \
				102, 104, 106, 108, 110, 112, 114, 116, 118, 122, 124, 126, 128, 130, 132, 134, 136, 138, 140, 143, 145, 148, 151, 154, 157},         \
			{4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35, 36, 37, 38,     \
				39, 40, 41, 42, 43, 44, 45, 46, 47, 48, 49, 50, 51, 52, 53, 54, 55, 56, 57, 58, 60, 62, 64, 66, 68, 70, 72, 74, 76, 78, 80, 82, 84,    \
				86, 88, 90, 92, 94, 96, 98, 100, 102, 104, 106, 108, 110, 112, 114, 116, 119, 122, 125, 128, 131, 134, 137, 140, 143, 146, 149, 152,   \
				155, 158, 161, 164, 167, 170, 173, 177, 181, 185, 189, 193, 197, 201, 205, 209, 213, 217, 221, 225, 229, 234, 239, 245, 249, 254, 259, \
				264, 269, 274, 279, 284},                                                                                                                  \
			{0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15}, {0, 1, 2, 3, 6, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6, 7, 0},                                   \
			{{173, 148, 140, 0}, {176, 155, 140, 135, 0}, {180, 157, 141, 134, 130, 0}, {254, 254, 243, 230, 196, 177, 153, 140, 133, 130, 129, 0}},       \
	}
/* global, not __constant__: one thread per frame reads them at data-dependent indices */
__device__ WebpTables d_webp_tables = WEBP_TABLES_INIT;
const WebpTables h_webp_tables = WEBP_TABLES_INIT;
#ifdef __CUDA_ARCH__
#define WT d_webp_tables
#else
#define WT h_webp_tables
#endif

enum { WERR_SEGMENT = 1, WERR_FILTER = 2, WERR_PARTITIONS = 3, WERR_P0_EOF = 4, WERR_TOKENS_EOF = 5 };

const char *
werr_text(int e)
{
	switch (e) {
	case WERR_SEGMENT:
		return "cannot parse segment header";
	case WERR_FILTER:
		return "cannot parse filter header";
	case WERR_PARTITIONS:
		return "cannot parse partitions";
	case WERR_P0_EOF:
		return "premature end of partition 0";
	default:
		return "premature end of a token partition";
	}
}

/* ------------------------------------------------------------------ the boolean decoder (RFC 6386 7.3) */

/* Bytes come in one at a time.  eof is libwebp's: set when a bit is wanted once every byte has been taken and the bits
 * left are spent, with one zero byte appended; libwebp fails the frame when it is set after a partition-0 row of modes or
 * a macroblock's tokens, so the point where a truncated stream fails is the same.  range holds range - 1.
 */
struct BoolDec {
	const unsigned char *buf;
	unsigned pos, end;
	unsigned value, range;
	int bits, eof;
};

VB_HD void
bd_load(BoolDec &b)
{
	if (b.pos < b.end) {
		b.bits += 8;
		b.value = (b.value << 8) | b.buf[b.pos++];
	}
	else if (!b.eof) {
		b.value <<= 8;
		b.bits += 8;
		b.eof = 1;
	}
	else
		b.bits = 0;
}

VB_HD void
bd_init(BoolDec &b, const unsigned char *buf, unsigned size)
{
	b.buf = buf;
	b.pos = 0;
	b.end = size;
	b.value = 0;
	b.range = 254;
	b.bits = -8;
	b.eof = 0;
	bd_load(b);
}

VB_HD int
floor_log2(unsigned v)
{
#ifdef __CUDA_ARCH__
	return 31 - __clz(v);
#else
	return 31 - __builtin_clz(v);
#endif
}

VB_HD int
bd_bit(BoolDec &b, int prob)
{
	if (b.bits < 0)
		bd_load(b);
	unsigned range = b.range;
	const unsigned split = (range * (unsigned) prob) >> 8;
	const unsigned value = b.value >> b.bits;
	int bit;
	if (value > split) {
		range -= split;
		b.value -= (split + 1) << b.bits;
		bit = 1;
	}
	else {
		range = split + 1;
		bit = 0;
	}
	const int shift = 7 ^ floor_log2(range);
	b.range = (range << shift) - 1;
	b.bits -= shift;
	return bit;
}

/* a coefficient's sign: probability one half, and (range - 1 <= 253 past a partition's first bit) always a 1-bit shift */
VB_HD int
bd_signed(BoolDec &b, int v)
{
	if (b.bits < 0)
		bd_load(b);
	const int pos = b.bits;
	const unsigned split = b.range >> 1;
	const unsigned value = b.value >> pos;
	const int mask = (int) (split - value) >> 31;
	b.bits -= 1;
	b.range = (b.range + (unsigned) mask) | 1;
	b.value -= ((split + 1) & (unsigned) mask) << pos;
	return (v ^ mask) - mask;
}

VB_HD int
bd_value(BoolDec &b, int nbits)
{
	int v = 0;
	while (nbits-- > 0)
		v |= bd_bit(b, 0x80) << nbits;
	return v;
}

VB_HD int
bd_signed_value(BoolDec &b, int nbits)
{
	const int v = bd_value(b, nbits);
	return bd_bit(b, 0x80) ? -v : v;
}

/* ------------------------------------------------------------------ frame header and modes (partition 0) */

/* one frame's header as the later stages read it */
struct WebpHdr {
	unsigned char proba[4][8][3][11]; /* coefficient probabilities [type][band][context][node] */
	unsigned char seg_p[3];
	unsigned char update_map, use_skip, skip_p, filter_type, num_parts;
	unsigned char f_limit[4][2], f_ilevel[4][2], f_hev[4][2]; /* [segment][is_i4x4] */
	short q[4][6];											  /* [segment]: y1 dc, ac; y2 dc, ac; uv dc, ac */
	unsigned part_off[8], part_len[8];						  /* token partitions, from the frame tag */
	int status;
};

/* one macroblock: partition 0's modes, then the token stage's non-zero codes (libwebp's non_zero_y / non_zero_uv: two
 * bits per block, 0 none, 1 dc only, 2 up to the third coefficient, 3 more) and whether the inner edges are filtered */
struct WebpMb {
	unsigned char imodes[16]; /* sub-block modes, or imodes[0] the 16 x 16 mode */
	unsigned char uvmode, segment, is_i4x4, skip, inner, pad[3];
	unsigned nz_y, nz_uv;
};

VB_HD int
clip_q(int v, int m)
{
	return v < 0 ? 0 : v > m ? m : v;
}

/* Partition 0's frame header (RFC 6386 9.3-9.11, 19.2) of the VP8 data d (len bytes, the 10-byte frame tag first, partition
 * 0 first_len bytes after it; the host has checked both).  Leaves br at the first macroblock's modes; 0 or a WERR_.
 */
VB_HD int
webp_header(const unsigned char *d, unsigned len, unsigned first_len, WebpHdr *H, BoolDec &br)
{
	bd_init(br, d + 10, first_len);
	bd_bit(br, 0x80); /* colour space */
	bd_bit(br, 0x80); /* clamping type: libwebp always clamps */
	int use_segment = bd_bit(br, 0x80), update_map = 0, abs_delta = 1;
	int quant[4] = {0, 0, 0, 0}, fstr[4] = {0, 0, 0, 0};
	H->seg_p[0] = H->seg_p[1] = H->seg_p[2] = 255;
	if (use_segment) {
		update_map = bd_bit(br, 0x80);
		if (bd_bit(br, 0x80)) {
			abs_delta = bd_bit(br, 0x80);
			for (int s = 0; s < 4; s++)
				quant[s] = bd_bit(br, 0x80) ? bd_signed_value(br, 7) : 0;
			for (int s = 0; s < 4; s++)
				fstr[s] = bd_bit(br, 0x80) ? bd_signed_value(br, 6) : 0;
		}
		if (update_map)
			for (int s = 0; s < 3; s++)
				H->seg_p[s] = (unsigned char) (bd_bit(br, 0x80) ? bd_value(br, 8) : 255);
	}
	H->update_map = (unsigned char) update_map;
	if (br.eof)
		return WERR_SEGMENT;
	const int simple = bd_bit(br, 0x80), level = bd_value(br, 6), sharp = bd_value(br, 3), use_lf = bd_bit(br, 0x80);
	int ref_d0 = 0, mode_d0 = 0;
	if (use_lf && bd_bit(br, 0x80)) {
		/* only the intra-frame deltas (ref 0, mode 0: B_PRED) apply to a key frame; the others are read past */
		for (int i = 0; i < 4; i++)
			if (bd_bit(br, 0x80)) {
				const int v = bd_signed_value(br, 6);
				if (i == 0)
					ref_d0 = v;
			}
		for (int i = 0; i < 4; i++)
			if (bd_bit(br, 0x80)) {
				const int v = bd_signed_value(br, 6);
				if (i == 0)
					mode_d0 = v;
			}
	}
	H->filter_type = (unsigned char) (level == 0 ? 0 : simple ? 1 : 2);
	if (br.eof)
		return WERR_FILTER;
	/* the partition table: P - 1 3-byte sizes after partition 0, each clamped to what is left; the last runs to the end and
	 * must not be empty */
	const int last = (1 << bd_value(br, 2)) - 1;
	H->num_parts = (unsigned char) (last + 1);
	const unsigned size = len - 10 - first_len;
	if (size < 3u * last)
		return WERR_PARTITIONS;
	const unsigned char *sz = d + 10 + first_len;
	unsigned start = 10 + first_len + 3 * last, left = size - 3 * last;
	for (int p = 0; p < last; p++) {
		unsigned psize = sz[3 * p] | (sz[3 * p + 1] << 8) | (sz[3 * p + 2] << 16);
		if (psize > left)
			psize = left;
		H->part_off[p] = start;
		H->part_len[p] = psize;
		start += psize;
		left -= psize;
	}
	H->part_off[last] = start;
	H->part_len[last] = left;
	if (left == 0)
		return WERR_PARTITIONS;
	/* quantisers (9.6, 14.1) */
	const int base_q = bd_value(br, 7);
	int dq[5];
	for (int i = 0; i < 5; i++)
		dq[i] = bd_bit(br, 0x80) ? bd_signed_value(br, 4) : 0; /* y1 dc, y2 dc, y2 ac, uv dc, uv ac */
	for (int s = 0; s < 4; s++) {
		const int q = use_segment ? quant[s] + (abs_delta ? 0 : base_q) : base_q;
		H->q[s][0] = WT.dc[clip_q(q + dq[0], 127)];
		H->q[s][1] = WT.ac[clip_q(q, 127)];
		H->q[s][2] = WT.dc[clip_q(q + dq[1], 127)] * 2;
		const int y2ac = (WT.ac[clip_q(q + dq[2], 127)] * 101581) >> 16; /* x * 155 / 100 for every x of the table */
		H->q[s][3] = y2ac < 8 ? 8 : y2ac;
		H->q[s][4] = WT.dc[clip_q(q + dq[3], 117)];
		H->q[s][5] = WT.ac[clip_q(q + dq[4], 127)];
	}
	bd_bit(br, 0x80); /* refresh_entropy_probs: one frame, no effect */
	for (int t = 0; t < 4; t++)
		for (int b = 0; b < 8; b++)
			for (int c = 0; c < 3; c++)
				for (int p = 0; p < 11; p++)
					H->proba[t][b][c][p] = (unsigned char) (bd_bit(br, WT.coeff_update[t][b][c][p]) ? bd_value(br, 8) : WT.coeff0[t][b][c][p]);
	H->use_skip = (unsigned char) bd_bit(br, 0x80);
	H->skip_p = (unsigned char) (H->use_skip ? bd_value(br, 8) : 0);
	/* loop-filter strengths per segment and per 16 x 16 / 4 x 4 macroblock (9.6, 15.1) */
	for (int s = 0; s < 4; s++) {
		const int base = use_segment ? fstr[s] + (abs_delta ? 0 : level) : level;
		for (int i4 = 0; i4 < 2; i4++) {
			int lvl = base;
			if (use_lf)
				lvl += ref_d0 + (i4 ? mode_d0 : 0);
			lvl = lvl < 0 ? 0 : lvl > 63 ? 63 : lvl;
			int limit = 0, ilevel = 0, hev = 0;
			if (lvl > 0) {
				ilevel = lvl;
				if (sharp > 0) {
					ilevel >>= sharp > 4 ? 2 : 1;
					if (ilevel > 9 - sharp)
						ilevel = 9 - sharp;
				}
				if (ilevel < 1)
					ilevel = 1;
				limit = 2 * lvl + ilevel;
				hev = lvl >= 40 ? 2 : lvl >= 15 ? 1 : 0;
			}
			H->f_limit[s][i4] = (unsigned char) (H->filter_type ? limit : 0);
			H->f_ilevel[s][i4] = (unsigned char) ilevel;
			H->f_hev[s][i4] = (unsigned char) hev;
		}
	}
	return 0;
}

/* One macroblock's segment, skip flag and modes (11.2-11.4); top: this column's 4 sub-mode contexts, left: the row's. */
VB_HD void
webp_mb_modes(BoolDec &br, const WebpHdr &H, unsigned char *top, unsigned char *left, WebpMb &m)
{
	m.segment = (unsigned char) (H.update_map ? (!bd_bit(br, H.seg_p[0]) ? bd_bit(br, H.seg_p[1]) : 2 + bd_bit(br, H.seg_p[2])) : 0);
	m.skip = (unsigned char) (H.use_skip ? bd_bit(br, H.skip_p) : 0);
	m.is_i4x4 = (unsigned char) !bd_bit(br, 145);
	if (!m.is_i4x4) {
		const int ymode = bd_bit(br, 156) ? (bd_bit(br, 128) ? M_TM : M_HE) : (bd_bit(br, 163) ? M_VE : M_DC);
		m.imodes[0] = (unsigned char) ymode;
		for (int i = 0; i < 4; i++)
			top[i] = left[i] = (unsigned char) ymode;
	}
	else {
		for (int y = 0; y < 4; y++) {
			int ym = left[y];
			for (int x = 0; x < 4; x++) {
				const unsigned char *p = WT.bmodes[top[x]][ym];
				ym = !bd_bit(br, p[0])	 ? M_DC
					 : !bd_bit(br, p[1]) ? M_TM
					 : !bd_bit(br, p[2]) ? M_VE
					 : !bd_bit(br, p[3]) ? (!bd_bit(br, p[4]) ? M_HE : !bd_bit(br, p[5]) ? M_RD : M_VR)
										 : (!bd_bit(br, p[6]) ? M_LD : !bd_bit(br, p[7]) ? M_VL : !bd_bit(br, p[8]) ? M_HD : M_HU);
				top[x] = (unsigned char) ym;
				m.imodes[4 * y + x] = (unsigned char) ym;
			}
			left[y] = (unsigned char) ym;
		}
	}
	m.uvmode = (unsigned char) (!bd_bit(br, 142) ? M_DC : !bd_bit(br, 114) ? M_VE : bd_bit(br, 183) ? M_TM : M_HE);
}

/* ------------------------------------------------------------------ tokens (13) */

/* one block's tokens from position n on, dequantised (dq[0] the dc step, dq[1] the ac step) into out (raster order);
 * returns the position after the last coefficient read, as libwebp's GetCoeffs does */
VB_HD int
webp_coeffs(BoolDec &br, const unsigned char (*bands)[3][11], int ctx, const short *dq, int n, short *out)
{
	const unsigned char *p = bands[WT.bands[n]][ctx];
	for (; n < 16; ++n) {
		if (!bd_bit(br, p[0]))
			return n;
		while (!bd_bit(br, p[1])) {
			p = bands[WT.bands[++n]][0];
			if (n == 16)
				return 16;
		}
		const unsigned char (*p_ctx)[11] = bands[WT.bands[n + 1]];
		int v;
		if (!bd_bit(br, p[2])) {
			v = 1;
			p = p_ctx[1];
		}
		else {
			if (!bd_bit(br, p[3]))
				v = !bd_bit(br, p[4]) ? 2 : 3 + bd_bit(br, p[5]);
			else if (!bd_bit(br, p[6])) {
				if (!bd_bit(br, p[7]))
					v = 5 + bd_bit(br, 159);
				else {
					v = 7 + 2 * bd_bit(br, 165);
					v += bd_bit(br, 145);
				}
			}
			else {
				const int bit1 = bd_bit(br, p[8]);
				const int bit0 = bd_bit(br, p[9 + bit1]);
				const int cat = 2 * bit1 + bit0;
				v = 0;
				for (const unsigned char *t = WT.cat[cat]; *t; ++t)
					v += v + bd_bit(br, *t);
				v += 3 + (8 << cat);
			}
			p = p_ctx[2];
		}
		out[WT.zigzag[n]] = (short) (bd_signed(br, v) * dq[n > 0]);
	}
	return 16;
}

VB_HD void
webp_wht(const short *in, short *out)
{
	int tmp[16];
	for (int i = 0; i < 4; ++i) {
		const int a0 = in[0 + i] + in[12 + i], a1 = in[4 + i] + in[8 + i];
		const int a2 = in[4 + i] - in[8 + i], a3 = in[0 + i] - in[12 + i];
		tmp[0 + i] = a0 + a1;
		tmp[8 + i] = a0 - a1;
		tmp[4 + i] = a3 + a2;
		tmp[12 + i] = a3 - a2;
	}
	for (int i = 0; i < 4; ++i) {
		const int dc = tmp[0 + i * 4] + 3;
		const int a0 = dc + tmp[3 + i * 4], a1 = tmp[1 + i * 4] + tmp[2 + i * 4];
		const int a2 = tmp[1 + i * 4] - tmp[2 + i * 4], a3 = dc - tmp[3 + i * 4];
		out[0] = (short) ((a0 + a1) >> 3);
		out[16] = (short) ((a3 + a2) >> 3);
		out[32] = (short) ((a0 - a1) >> 3);
		out[48] = (short) ((a3 - a2) >> 3);
		out += 64;
	}
}

VB_HD unsigned
nz_code(unsigned nz_coeffs, int nz, int dc_nz)
{
	return (nz_coeffs << 2) | (nz > 3 ? 3u : nz > 1 ? 2u : (unsigned) dc_nz);
}

/* One macroblock's residuals into coeffs[384] (16 Y, 4 U, 4 V blocks of 16).  tnz / tdc: this column's non-zero contexts
 * (Y bits 0-3, U 4-5, V 6-7; the Y2 block's), lnz / ldc the row's.  Sets m.nz_y / nz_uv / inner.
 */
VB_HD void
webp_mb_tokens(BoolDec &br, const WebpHdr &H, WebpMb &m, unsigned char &tnz_io, unsigned char &tdc, unsigned char &lnz_io, unsigned char &ldc,
	short *coeffs)
{
	int skip = H.use_skip ? m.skip : 0;
	if (skip) {
		tnz_io = lnz_io = 0;
		if (!m.is_i4x4)
			tdc = ldc = 0;
		m.nz_y = m.nz_uv = 0;
	}
	else {
		const short *q = H.q[m.segment];
		short *dst = coeffs;
		for (int i = 0; i < 384; i++)
			dst[i] = 0;
		int first;
		const unsigned char (*ac_proba)[3][11];
		if (!m.is_i4x4) {
			short dc[16] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
			const int nz = webp_coeffs(br, H.proba[1], tdc + ldc, q + 2, 0, dc);
			tdc = ldc = (unsigned char) (nz > 0);
			webp_wht(dc, dst);
			first = 1;
			ac_proba = H.proba[0];
		}
		else {
			first = 0;
			ac_proba = H.proba[3];
		}
		unsigned tnz = tnz_io & 0x0f, lnz = lnz_io & 0x0f, non_zero_y = 0, non_zero_uv = 0;
		for (int y = 0; y < 4; ++y) {
			int l = lnz & 1;
			unsigned nz_coeffs = 0;
			for (int x = 0; x < 4; ++x) {
				const int nz = webp_coeffs(br, ac_proba, l + (tnz & 1), q, first, dst);
				l = nz > first;
				tnz = (tnz >> 1) | (l << 7);
				nz_coeffs = nz_code(nz_coeffs, nz, dst[0] != 0);
				dst += 16;
			}
			tnz >>= 4;
			lnz = (lnz >> 1) | (l << 7);
			non_zero_y = (non_zero_y << 8) | nz_coeffs;
		}
		unsigned out_t = tnz, out_l = lnz >> 4;
		for (int ch = 0; ch < 4; ch += 2) {
			unsigned nz_coeffs = 0;
			tnz = (unsigned) tnz_io >> (4 + ch);
			lnz = (unsigned) lnz_io >> (4 + ch);
			for (int y = 0; y < 2; ++y) {
				int l = lnz & 1;
				for (int x = 0; x < 2; ++x) {
					const int nz = webp_coeffs(br, H.proba[2], l + (tnz & 1), q + 4, 0, dst);
					l = nz > 0;
					tnz = (tnz >> 1) | (l << 3);
					nz_coeffs = nz_code(nz_coeffs, nz, dst[0] != 0);
					dst += 16;
				}
				tnz >>= 2;
				lnz = (lnz >> 1) | (l << 5);
			}
			non_zero_uv |= nz_coeffs << (4 * ch);
			out_t |= (tnz << 4) << ch;
			out_l |= (lnz & 0xf0) << ch;
		}
		tnz_io = (unsigned char) out_t;
		lnz_io = (unsigned char) out_l;
		m.nz_y = non_zero_y;
		m.nz_uv = non_zero_uv;
		skip = !(non_zero_y | non_zero_uv);
	}
	m.inner = (unsigned char) (m.is_i4x4 | !skip);
}

/* ------------------------------------------------------------------ reconstruction (12, 14) */

/* libwebp's work area: BPS-wide rows, Y with its top row (and 4 top-right pixels) and left column, then U and V */
constexpr int BPS = 32, Y_OFF = BPS * 1 + 8, U_OFF = Y_OFF + BPS * 16 + BPS, V_OFF = U_OFF + 16, WB_SIZE = BPS * 17 + BPS * 9;

VB_HD unsigned char
clip8(int v)
{
	return (unsigned char) (v < 0 ? 0 : v > 255 ? 255 : v);
}

VB_HD int
avg3(int a, int b, int c)
{
	return (a + 2 * b + c + 2) >> 2;
}

VB_HD int
avg2(int a, int b)
{
	return (a + b + 1) >> 1;
}

/* the inverse DCT of one block (14.3) added to dst */
VB_HD void
idct_add(const short *in, unsigned char *dst)
{
	int C[16];
	int *tmp = C;
	for (int i = 0; i < 4; ++i) {
		const int a = in[0] + in[8], b = in[0] - in[8];
		const int c = ((in[4] * 35468) >> 16) - (((in[12] * 20091) >> 16) + in[12]);
		const int d = (((in[4] * 20091) >> 16) + in[4]) + ((in[12] * 35468) >> 16);
		tmp[0] = a + d;
		tmp[1] = b + c;
		tmp[2] = b - c;
		tmp[3] = a - d;
		tmp += 4;
		in++;
	}
	tmp = C;
	for (int i = 0; i < 4; ++i) {
		const int dc = tmp[0] + 4;
		const int a = dc + tmp[8], b = dc - tmp[8];
		const int c = ((tmp[4] * 35468) >> 16) - (((tmp[12] * 20091) >> 16) + tmp[12]);
		const int d = (((tmp[4] * 20091) >> 16) + tmp[4]) + ((tmp[12] * 35468) >> 16);
		dst[0] = clip8(dst[0] + ((a + d) >> 3));
		dst[1] = clip8(dst[1] + ((b + c) >> 3));
		dst[2] = clip8(dst[2] + ((b - c) >> 3));
		dst[3] = clip8(dst[3] + ((a - d) >> 3));
		tmp++;
		dst += BPS;
	}
}

VB_HD void
true_motion(unsigned char *dst, int size)
{
	const unsigned char *top = dst - BPS;
	const int tl = top[-1];
	for (int y = 0; y < size; ++y) {
		const int l = dst[-1];
		for (int x = 0; x < size; ++x)
			dst[x] = clip8(top[x] + l - tl);
		dst += BPS;
	}
}

/* 16 x 16 luma and 8 x 8 chroma prediction (12.2); mode may be one of the M_DC_NO* edge forms */
VB_HD void
predict_block(unsigned char *dst, int size, int mode)
{
	const int shift = size == 16 ? 5 : 4;
	int dc = 0;
	switch (mode) {
	case M_VE:
		for (int y = 0; y < size; y++)
			for (int x = 0; x < size; x++)
				dst[y * BPS + x] = dst[x - BPS];
		return;
	case M_HE:
		for (int y = 0; y < size; y++)
			for (int x = 0; x < size; x++)
				dst[y * BPS + x] = dst[y * BPS - 1];
		return;
	case M_TM:
		true_motion(dst, size);
		return;
	case M_DC:
		for (int i = 0; i < size; i++)
			dc += dst[i - BPS] + dst[i * BPS - 1];
		dc = (dc + size) >> shift;
		break;
	case M_DC_NOTOP:
		for (int i = 0; i < size; i++)
			dc += dst[i * BPS - 1];
		dc = (dc + (size >> 1)) >> (shift - 1);
		break;
	case M_DC_NOLEFT:
		for (int i = 0; i < size; i++)
			dc += dst[i - BPS];
		dc = (dc + (size >> 1)) >> (shift - 1);
		break;
	default:
		dc = 0x80;
	}
	for (int y = 0; y < size; y++)
		for (int x = 0; x < size; x++)
			dst[y * BPS + x] = (unsigned char) dc;
}

#define DST(x, y) dst[(x) + (y) * BPS]

/* the ten 4 x 4 sub-block predictors (12.3) */
VB_HD void
predict4(unsigned char *dst, int mode)
{
	const int X = dst[-1 - BPS], A = dst[0 - BPS], B = dst[1 - BPS], C = dst[2 - BPS], D = dst[3 - BPS];
	const int E = dst[4 - BPS], F = dst[5 - BPS], G = dst[6 - BPS], Hh = dst[7 - BPS];
	const int I = dst[-1], J = dst[-1 + BPS], K = dst[-1 + 2 * BPS], L = dst[-1 + 3 * BPS];
	switch (mode) {
	case M_DC: {
		int dc = 4;
		for (int i = 0; i < 4; ++i)
			dc += dst[i - BPS] + dst[-1 + i * BPS];
		dc >>= 3;
		for (int y = 0; y < 4; y++)
			for (int x = 0; x < 4; x++)
				DST(x, y) = (unsigned char) dc;
		break;
	}
	case M_TM:
		true_motion(dst, 4);
		break;
	case M_VE: {
		const int v[4] = {avg3(X, A, B), avg3(A, B, C), avg3(B, C, D), avg3(C, D, E)};
		for (int y = 0; y < 4; y++)
			for (int x = 0; x < 4; x++)
				DST(x, y) = (unsigned char) v[x];
		break;
	}
	case M_HE: {
		const int v[4] = {avg3(X, I, J), avg3(I, J, K), avg3(J, K, L), avg3(K, L, L)};
		for (int y = 0; y < 4; y++)
			for (int x = 0; x < 4; x++)
				DST(x, y) = (unsigned char) v[y];
		break;
	}
	case M_RD:
		DST(0, 3) = avg3(J, K, L);
		DST(1, 3) = DST(0, 2) = avg3(I, J, K);
		DST(2, 3) = DST(1, 2) = DST(0, 1) = avg3(X, I, J);
		DST(3, 3) = DST(2, 2) = DST(1, 1) = DST(0, 0) = avg3(A, X, I);
		DST(3, 2) = DST(2, 1) = DST(1, 0) = avg3(B, A, X);
		DST(3, 1) = DST(2, 0) = avg3(C, B, A);
		DST(3, 0) = avg3(D, C, B);
		break;
	case M_LD:
		DST(0, 0) = avg3(A, B, C);
		DST(1, 0) = DST(0, 1) = avg3(B, C, D);
		DST(2, 0) = DST(1, 1) = DST(0, 2) = avg3(C, D, E);
		DST(3, 0) = DST(2, 1) = DST(1, 2) = DST(0, 3) = avg3(D, E, F);
		DST(3, 1) = DST(2, 2) = DST(1, 3) = avg3(E, F, G);
		DST(3, 2) = DST(2, 3) = avg3(F, G, Hh);
		DST(3, 3) = avg3(G, Hh, Hh);
		break;
	case M_VR:
		DST(0, 0) = DST(1, 2) = avg2(X, A);
		DST(1, 0) = DST(2, 2) = avg2(A, B);
		DST(2, 0) = DST(3, 2) = avg2(B, C);
		DST(3, 0) = avg2(C, D);
		DST(0, 3) = avg3(K, J, I);
		DST(0, 2) = avg3(J, I, X);
		DST(0, 1) = DST(1, 3) = avg3(I, X, A);
		DST(1, 1) = DST(2, 3) = avg3(X, A, B);
		DST(2, 1) = DST(3, 3) = avg3(A, B, C);
		DST(3, 1) = avg3(B, C, D);
		break;
	case M_VL:
		DST(0, 0) = avg2(A, B);
		DST(1, 0) = DST(0, 2) = avg2(B, C);
		DST(2, 0) = DST(1, 2) = avg2(C, D);
		DST(3, 0) = DST(2, 2) = avg2(D, E);
		DST(0, 1) = avg3(A, B, C);
		DST(1, 1) = DST(0, 3) = avg3(B, C, D);
		DST(2, 1) = DST(1, 3) = avg3(C, D, E);
		DST(3, 1) = DST(2, 3) = avg3(D, E, F);
		DST(3, 2) = avg3(E, F, G);
		DST(3, 3) = avg3(F, G, Hh);
		break;
	case M_HD:
		DST(0, 0) = DST(2, 1) = avg2(I, X);
		DST(0, 1) = DST(2, 2) = avg2(J, I);
		DST(0, 2) = DST(2, 3) = avg2(K, J);
		DST(0, 3) = avg2(L, K);
		DST(3, 0) = avg3(A, B, C);
		DST(2, 0) = avg3(X, A, B);
		DST(1, 0) = DST(3, 1) = avg3(I, X, A);
		DST(1, 1) = DST(3, 2) = avg3(J, I, X);
		DST(1, 2) = DST(3, 3) = avg3(K, J, I);
		DST(1, 3) = avg3(L, K, J);
		break;
	default: /* M_HU */
		DST(0, 0) = avg2(I, J);
		DST(2, 0) = DST(0, 1) = avg2(J, K);
		DST(2, 1) = DST(0, 2) = avg2(K, L);
		DST(1, 0) = avg3(I, J, K);
		DST(3, 0) = DST(1, 1) = avg3(J, K, L);
		DST(3, 1) = DST(1, 2) = avg3(K, L, L);
		DST(3, 2) = DST(2, 2) = DST(0, 3) = DST(1, 3) = DST(2, 3) = DST(3, 3) = (unsigned char) L;
	}
}

#undef DST

VB_HD int
edge_mode(int mbx, int mby, int mode)
{
	if (mode != M_DC)
		return mode;
	return mbx == 0 ? (mby == 0 ? (int) M_DC_NOTOPLEFT : (int) M_DC_NOLEFT) : (mby == 0 ? (int) M_DC_NOTOP : (int) M_DC);
}

/* The planes a frame is reconstructed and filtered in: mb_w * 16 x mb_h * 16 luma, half that chroma. */
struct Planes {
	unsigned char *y, *u, *v;
	int ys, uvs;
};

/* Macroblock (mbx, mby) predicted from the unfiltered pixels of its left, top, top-left and top-right neighbours (127
 * above the frame, 129 left of it) plus its residuals, written into the planes.
 */
VB_HD void
webp_recon_mb(const WebpMb &m, const short *coeffs, int mbx, int mby, int mb_w, const Planes &P)
{
	unsigned char wb[WB_SIZE];
	unsigned char *yd = wb + Y_OFF, *ud = wb + U_OFF, *vd = wb + V_OFF;
	const unsigned char *py = P.y + (size_t) mby * 16 * P.ys + mbx * 16;
	const unsigned char *pu = P.u + (size_t) mby * 8 * P.uvs + mbx * 8, *pv = P.v + (size_t) mby * 8 * P.uvs + mbx * 8;
	for (int j = 0; j < 16; j++)
		yd[j * BPS - 1] = mbx > 0 ? py[(size_t) j * P.ys - 1] : 129;
	for (int j = 0; j < 8; j++) {
		ud[j * BPS - 1] = mbx > 0 ? pu[(size_t) j * P.uvs - 1] : 129;
		vd[j * BPS - 1] = mbx > 0 ? pv[(size_t) j * P.uvs - 1] : 129;
	}
	if (mby == 0) {
		for (int i = -1; i < 20; i++)
			yd[i - BPS] = 127;
		for (int i = -1; i < 8; i++)
			ud[i - BPS] = vd[i - BPS] = 127;
	}
	else {
		yd[-1 - BPS] = mbx > 0 ? py[-(ptrdiff_t) P.ys - 1] : 129;
		ud[-1 - BPS] = mbx > 0 ? pu[-(ptrdiff_t) P.uvs - 1] : 129;
		vd[-1 - BPS] = mbx > 0 ? pv[-(ptrdiff_t) P.uvs - 1] : 129;
		for (int i = 0; i < 16; i++)
			yd[i - BPS] = py[i - (ptrdiff_t) P.ys];
		for (int i = 0; i < 8; i++) {
			ud[i - BPS] = pu[i - (ptrdiff_t) P.uvs];
			vd[i - BPS] = pv[i - (ptrdiff_t) P.uvs];
		}
		/* above-right: the next macroblock's bottom row, or the last pixel repeated at the right edge */
		for (int i = 16; i < 20; i++)
			yd[i - BPS] = mbx < mb_w - 1 ? py[i - (ptrdiff_t) P.ys] : py[15 - (ptrdiff_t) P.ys];
	}
	unsigned bits = m.nz_y;
	if (m.is_i4x4) {
		/* the sub-blocks of the right column below the first take the macroblock's above-right pixels */
		for (int r = 3; r < 12; r += 4)
			for (int i = 16; i < 20; i++)
				yd[r * BPS + i] = yd[i - BPS];
		for (int n = 0; n < 16; ++n, bits <<= 2) {
			unsigned char *dst = yd + (n & 3) * 4 + (n >> 2) * 4 * BPS;
			predict4(dst, m.imodes[n]);
			if (bits >> 30)
				idct_add(coeffs + n * 16, dst);
		}
	}
	else {
		predict_block(yd, 16, edge_mode(mbx, mby, m.imodes[0]));
		for (int n = 0; n < 16; ++n, bits <<= 2)
			if (bits >> 30)
				idct_add(coeffs + n * 16, yd + (n & 3) * 4 + (n >> 2) * 4 * BPS);
	}
	const int uvm = edge_mode(mbx, mby, m.uvmode);
	predict_block(ud, 8, uvm);
	predict_block(vd, 8, uvm);
	for (int c = 0; c < 2; c++) {
		unsigned char *d = c ? vd : ud;
		if ((m.nz_uv >> (8 * c)) & 0xff)
			for (int n = 0; n < 4; n++)
				idct_add(coeffs + (16 + 4 * c + n) * 16, d + (n & 1) * 4 + (n >> 1) * 4 * BPS);
	}
	unsigned char *oy = P.y + (size_t) mby * 16 * P.ys + mbx * 16;
	for (int j = 0; j < 16; j++)
		for (int i = 0; i < 16; i++)
			oy[(size_t) j * P.ys + i] = yd[j * BPS + i];
	unsigned char *ou = P.u + (size_t) mby * 8 * P.uvs + mbx * 8, *ov = P.v + (size_t) mby * 8 * P.uvs + mbx * 8;
	for (int j = 0; j < 8; j++)
		for (int i = 0; i < 8; i++) {
			ou[(size_t) j * P.uvs + i] = ud[j * BPS + i];
			ov[(size_t) j * P.uvs + i] = vd[j * BPS + i];
		}
}

/* ------------------------------------------------------------------ loop filter (15) */

VB_HD int
sclip1(int v)
{
	return v < -128 ? -128 : v > 127 ? 127 : v;
}

VB_HD int
sclip2(int v)
{
	return v < -16 ? -16 : v > 15 ? 15 : v;
}

VB_HD int
iabs(int v)
{
	return v < 0 ? -v : v;
}

VB_HD void
do_filter2(unsigned char *p, ptrdiff_t step)
{
	const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
	const int a = 3 * (q0 - p0) + sclip1(p1 - q1);
	const int a1 = sclip2((a + 4) >> 3), a2 = sclip2((a + 3) >> 3);
	p[-step] = clip8(p0 + a2);
	p[0] = clip8(q0 - a1);
}

VB_HD void
do_filter4(unsigned char *p, ptrdiff_t step)
{
	const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
	const int a = 3 * (q0 - p0);
	const int a1 = sclip2((a + 4) >> 3), a2 = sclip2((a + 3) >> 3), a3 = (a1 + 1) >> 1;
	p[-2 * step] = clip8(p1 + a3);
	p[-step] = clip8(p0 + a2);
	p[0] = clip8(q0 - a1);
	p[step] = clip8(q1 - a3);
}

VB_HD void
do_filter6(unsigned char *p, ptrdiff_t step)
{
	const int p2 = p[-3 * step], p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step], q2 = p[2 * step];
	const int a = sclip1(3 * (q0 - p0) + sclip1(p1 - q1));
	const int a1 = (27 * a + 63) >> 7, a2 = (18 * a + 63) >> 7, a3 = (9 * a + 63) >> 7;
	p[-3 * step] = clip8(p2 + a3);
	p[-2 * step] = clip8(p1 + a2);
	p[-step] = clip8(p0 + a1);
	p[0] = clip8(q0 - a1);
	p[step] = clip8(q1 - a2);
	p[2 * step] = clip8(q2 - a3);
}

VB_HD bool
needs_filter(const unsigned char *p, ptrdiff_t step, int t)
{
	return 4 * iabs(p[-step] - p[0]) + iabs(p[-2 * step] - p[step]) <= t;
}

VB_HD bool
needs_filter2(const unsigned char *p, ptrdiff_t step, int t, int it)
{
	const int p3 = p[-4 * step], p2 = p[-3 * step], p1 = p[-2 * step], p0 = p[-step];
	const int q0 = p[0], q1 = p[step], q2 = p[2 * step], q3 = p[3 * step];
	if (4 * iabs(p0 - q0) + iabs(p1 - q1) > t)
		return false;
	return iabs(p3 - p2) <= it && iabs(p2 - p1) <= it && iabs(p1 - p0) <= it && iabs(q3 - q2) <= it && iabs(q2 - q1) <= it && iabs(q1 - q0) <= it;
}

/* size pixels along an edge: hstride across it, vstride along it; the normal filter's macroblock-edge (six-tap) or
 * inner-edge (four-tap) form */
VB_HD void
filter_loop(unsigned char *p, ptrdiff_t hstride, ptrdiff_t vstride, int size, int thresh, int ithresh, int hev_t, bool edge)
{
	const int thresh2 = 2 * thresh + 1;
	for (int i = 0; i < size; i++, p += vstride)
		if (needs_filter2(p, hstride, thresh2, ithresh)) {
			if (iabs(p[-2 * hstride] - p[-hstride]) > hev_t || iabs(p[hstride] - p[0]) > hev_t)
				do_filter2(p, hstride);
			else if (edge)
				do_filter6(p, hstride);
			else
				do_filter4(p, hstride);
		}
}

VB_HD void
simple_loop(unsigned char *p, ptrdiff_t hstride, ptrdiff_t vstride, int thresh)
{
	const int thresh2 = 2 * thresh + 1;
	for (int i = 0; i < 16; i++, p += vstride)
		if (needs_filter(p, hstride, thresh2))
			do_filter2(p, hstride);
}

/* Macroblock (mbx, mby)'s edges in libwebp's order: left edge, inner vertical edges, top edge, inner horizontal edges.  Run
 * in raster order, or any order in which (mbx - 1, mby) and (mbx + 1, mby - 1) come first.
 */
VB_HD void
webp_filter_mb(const WebpHdr &H, const WebpMb &m, int mbx, int mby, const Planes &P)
{
	const int limit = H.f_limit[m.segment][m.is_i4x4];
	if (limit == 0)
		return;
	const int ilevel = H.f_ilevel[m.segment][m.is_i4x4], hev = H.f_hev[m.segment][m.is_i4x4];
	const ptrdiff_t ys = P.ys, uvs = P.uvs;
	unsigned char *y = P.y + (size_t) mby * 16 * ys + mbx * 16;
	if (H.filter_type == 1) {
		if (mbx > 0)
			simple_loop(y, 1, ys, limit + 4);
		if (m.inner)
			for (int k = 4; k < 16; k += 4)
				simple_loop(y + k, 1, ys, limit);
		if (mby > 0)
			simple_loop(y, ys, 1, limit + 4);
		if (m.inner)
			for (int k = 4; k < 16; k += 4)
				simple_loop(y + k * ys, ys, 1, limit);
		return;
	}
	unsigned char *u = P.u + (size_t) mby * 8 * uvs + mbx * 8, *v = P.v + (size_t) mby * 8 * uvs + mbx * 8;
	if (mbx > 0) {
		filter_loop(y, 1, ys, 16, limit + 4, ilevel, hev, true);
		filter_loop(u, 1, uvs, 8, limit + 4, ilevel, hev, true);
		filter_loop(v, 1, uvs, 8, limit + 4, ilevel, hev, true);
	}
	if (m.inner) {
		for (int k = 4; k < 16; k += 4)
			filter_loop(y + k, 1, ys, 16, limit, ilevel, hev, false);
		filter_loop(u + 4, 1, uvs, 8, limit, ilevel, hev, false);
		filter_loop(v + 4, 1, uvs, 8, limit, ilevel, hev, false);
	}
	if (mby > 0) {
		filter_loop(y, ys, 1, 16, limit + 4, ilevel, hev, true);
		filter_loop(u, uvs, 1, 8, limit + 4, ilevel, hev, true);
		filter_loop(v, uvs, 1, 8, limit + 4, ilevel, hev, true);
	}
	if (m.inner) {
		for (int k = 4; k < 16; k += 4)
			filter_loop(y + k * ys, ys, 1, 16, limit, ilevel, hev, false);
		filter_loop(u + 4 * uvs, uvs, 1, 8, limit, ilevel, hev, false);
		filter_loop(v + 4 * uvs, uvs, 1, 8, limit, ilevel, hev, false);
	}
}

/* ------------------------------------------------------------------ YUV -> RGB */

VB_HD int
mult_hi(int v, int coeff)
{
	return (v * coeff) >> 8;
}

VB_HD int
yuv_clip8(int v)
{
	return (v & ~16383) == 0 ? v >> 6 : v < 0 ? 0 : 255;
}

/* libwebp's 14-bit fixed-point YUV -> RGB of one pixel (VP8YuvToRgb) */
VB_HD void
webp_yuv_rgb(int Y, int u, int v, unsigned char *dst)
{
	dst[0] = (unsigned char) yuv_clip8(mult_hi(Y, 19077) + mult_hi(v, 26149) - 14234);
	dst[1] = (unsigned char) yuv_clip8(mult_hi(Y, 19077) - mult_hi(u, 6419) - mult_hi(v, 13320) + 8708);
	dst[2] = (unsigned char) yuv_clip8(mult_hi(Y, 19077) + mult_hi(u, 33050) - 17685);
}

/* Pixel (x, y) of a w x h frame: libwebp's fancy upsampler (each output row pair between two chroma rows, the (9, 3, 3, 1)
 * taps, the first and an even height's last row on one chroma row, an even width's last column on one chroma column),
 * then its 14-bit fixed-point YUV -> RGB.
 */
VB_HD void
webp_rgb_pixel(const Planes &P, int w, int h, int x, int y, unsigned char *dst)
{
	int trow, crow;
	bool top_line;
	if (y == 0 || (y == h - 1 && !(h & 1))) {
		trow = crow = (y + 1) >> 1;
		if (y)
			trow = crow = (y - 1) >> 1;
		top_line = true;
	}
	else if (y & 1) {
		trow = (y - 1) >> 1;
		crow = (y + 1) >> 1;
		top_line = true;
	}
	else {
		trow = (y >> 1) - 1;
		crow = y >> 1;
		top_line = false;
	}
	int uv[2];
	for (int c = 0; c < 2; c++) {
		const unsigned char *T = (c ? P.v : P.u) + (size_t) trow * P.uvs, *Cr = (c ? P.v : P.u) + (size_t) crow * P.uvs;
		const int j = (x + 1) >> 1;
		if (x == 0 || j > ((w - 1) >> 1)) {
			const int k = x == 0 ? 0 : (w - 1) >> 1;
			const int tl = T[k], l = Cr[k];
			uv[c] = top_line ? (3 * tl + l + 2) >> 2 : (3 * l + tl + 2) >> 2;
		}
		else {
			const int tl = T[j - 1], t = T[j], l = Cr[j - 1], cc = Cr[j];
			const int d12 = (tl + 3 * t + 3 * l + cc + 8) >> 3, d03 = (3 * tl + t + l + 3 * cc + 8) >> 3;
			if (x & 1)
				uv[c] = top_line ? (d12 + tl) >> 1 : (d03 + l) >> 1;
			else
				uv[c] = top_line ? (d03 + t) >> 1 : (d12 + cc) >> 1;
		}
	}
	webp_yuv_rgb(P.y[(size_t) y * P.ys + x], uv[0], uv[1], dst);
}

/* ------------------------------------------------------------------ libwebp's rescaler (the scaled decode)
 *
 * With options.use_scaling (what webpload asks for at scale != 1, webp2vips.c:630-634) libwebp skips the upsampler: three
 * WebPRescalers take Y (W x H) and U and V ((W + 1) / 2 x (H + 1) / 2) each to sw x sh, and every output pixel is the 14-bit
 * YUV -> RGB of its three samples.  Each axis either shrinks (src >= dst: an area average with a fractional carry into
 * the next output) or expands (src < dst: linear interpolation), all in 32-bit fixed point.
 *
 * libwebp streams rows through the rescaler, but every output sample has a closed form over a window of source pixels:
 * the horizontal carry into column x is MULT_FIX(frac, fx_scale) of one boundary pixel, the vertical carry into row y is
 * MULT_FIX_FLOOR(frow, yscale) of one boundary row, and the sums are uint32 that wrap, so the order of additions does not
 * matter.  RescaleTap tables hold each output index's window; rescale_sample evaluates one sample from them alone.
 */

constexpr unsigned long long RESCALER_ONE = 1ull << 32, RESCALER_ROUNDER = RESCALER_ONE >> 1;

VB_HD unsigned
mult_fix(unsigned x, unsigned y)
{
	return (unsigned) (((unsigned long long) x * y + RESCALER_ROUNDER) >> 32);
}

VB_HD unsigned
mult_fix_floor(unsigned x, unsigned y)
{
	return (unsigned) (((unsigned long long) x * y) >> 32);
}

unsigned
rescaler_frac(unsigned long long x, unsigned long long y)
{
	return (unsigned) ((x << 32) / y);
}

/* one plane's WebPRescalerInit: the increments and fixed-point scales of src_w x src_h -> dst_w x dst_h */
struct RescaleParams {
	int x_expand, y_expand;
	unsigned x_add, x_sub, y_add, y_sub;
	unsigned fx_scale, fy_scale, fxy_scale;
	int src_w, src_h, dst_w, dst_h;
};

RescaleParams
rescale_params(int src_w, int src_h, int dst_w, int dst_h)
{
	RescaleParams p{};
	p.src_w = src_w;
	p.src_h = src_h;
	p.dst_w = dst_w;
	p.dst_h = dst_h;
	p.x_expand = src_w < dst_w;
	p.y_expand = src_h < dst_h;
	/* expanding, the increments are the gaps between the first and last samples: bilinear interpolation */
	p.x_add = p.x_expand ? dst_w - 1 : src_w;
	p.x_sub = p.x_expand ? src_w - 1 : dst_w;
	p.y_add = p.y_expand ? src_h - 1 : src_h;
	p.y_sub = p.y_expand ? dst_h - 1 : dst_h;
	if (!p.x_expand)
		p.fx_scale = rescaler_frac(1, p.x_sub);
	if (!p.y_expand) {
		/* dst_h / (x_add * y_add) is 1.0 only for a 1-pixel-wide source kept at its height: fxy_scale 0 marks the copy */
		const unsigned long long ratio = (unsigned long long) dst_h * RESCALER_ONE / ((unsigned long long) p.x_add * p.y_add);
		p.fxy_scale = ratio != (unsigned) ratio ? 0 : (unsigned) ratio;
		p.fy_scale = rescaler_frac(1, p.y_sub);
	}
	else
		p.fy_scale = rescaler_frac(1, p.x_add);
	return p;
}

/* One output index's window on one axis:
 *   shrink  i0 the first source index, i1 the count; w0 the carry's multiplier of source i0 - 1 (0: none), w1 the
 *           multiplier taken off the last source (horizontally -accum, vertically yscale = fy_scale * -y_accum)
 *   expand  horizontally i0 / i1 the left and right sources and w0 the accumulator; vertically i0 / i1 the previous and
 *           the current row and w0 the previous row's weight B (0: the current row alone)
 */
struct RescaleTap {
	int i0, i1;
	unsigned w0, w1;
};

/* the taps of one axis, from the accumulators' walk in ImportRowShrink / ImportRowExpand (horizontal) or WebPRescalerImport
 * and the two ExportRow forms (vertical) */
void
rescale_taps(const RescaleParams &p, bool vertical, RescaleTap *t)
{
	const int expand = vertical ? p.y_expand : p.x_expand, dst = vertical ? p.dst_h : p.dst_w, src = vertical ? p.src_h : p.src_w;
	const int add = (int) (vertical ? p.y_add : p.x_add), sub = (int) (vertical ? p.y_sub : p.x_sub);
	if (!expand) {
		int accum = vertical ? add : 0, at = 0;
		unsigned carry = 0;
		for (int o = 0; o < dst; o++) {
			RescaleTap &k = t[o];
			k.i0 = at;
			k.w0 = carry;
			if (!vertical)
				accum += add;
			int n = 0;
			while (accum > 0) {
				accum -= sub;
				at++;
				n++;
			}
			k.i1 = n;
			k.w1 = vertical ? p.fy_scale * (unsigned) -accum : (unsigned) -accum;
			carry = k.w1;
			if (vertical)
				accum += add;
		}
		return;
	}
	if (!vertical) {
		int accum = add, l = 0, r = src > 1 ? 1 : 0;
		for (int o = 0; o < dst; o++) {
			t[o] = RescaleTap{l, r, (unsigned) accum, 0};
			accum -= sub;
			if (accum < 0 && o + 1 < dst) {
				l = r++;
				accum += add;
			}
		}
		return;
	}
	int accum = sub, prev = 0, cur = -1;
	for (int o = 0; o < dst; o++) {
		while (accum > 0) {
			prev = cur < 0 ? 0 : cur;
			cur++;
			accum -= sub;
		}
		t[o] = RescaleTap{prev, cur, accum == 0 ? 0u : rescaler_frac((unsigned) -accum, (unsigned) sub), 0};
		accum += add;
	}
}

/* the horizontal pass of source row `row` at one output column: ImportRowExpand's interpolation or ImportRowShrink's sum
 * times x_sub, less the fraction of the last pixel, plus the carry from the previous column */
VB_HD unsigned
rescale_h(const unsigned char *row, const RescaleParams &p, const RescaleTap &t)
{
	if (p.x_expand) {
		const unsigned left = row[t.i0], right = row[t.i1];
		return right * p.x_add + (left - right) * t.w0;
	}
	unsigned sum = t.w0 ? mult_fix(row[t.i0 - 1] * t.w0, p.fx_scale) : 0u, base = 0;
	for (int k = 0; k < t.i1; k++) {
		base = row[t.i0 + k];
		sum += base;
	}
	return sum * p.x_sub - base * t.w1;
}

/* One rescaled sample of a plane: the vertical pass (ExportRowExpand, or ExportRowShrink with its carry) over rescale_h's
 * rows, clipped as WebPRescalerExportRow clips. */
VB_HD unsigned char
rescale_sample(const unsigned char *plane, size_t stride, const RescaleParams &p, const RescaleTap &tx, const RescaleTap &ty)
{
	int v;
	if (p.y_expand) {
		const unsigned f = rescale_h(plane + (size_t) ty.i1 * stride, p, tx);
		unsigned J = f;
		if (ty.w0) {
			const unsigned i = rescale_h(plane + (size_t) ty.i0 * stride, p, tx);
			const unsigned long long I = (unsigned long long) (unsigned) (RESCALER_ONE - ty.w0) * f + (unsigned long long) ty.w0 * i;
			J = (unsigned) ((I + RESCALER_ROUNDER) >> 32);
		}
		v = (int) mult_fix(J, p.fy_scale);
	}
	else {
		unsigned irow = ty.w0 ? mult_fix_floor(rescale_h(plane + (size_t) (ty.i0 - 1) * stride, p, tx), ty.w0) : 0u, f = 0;
		for (int k = 0; k < ty.i1; k++) {
			f = rescale_h(plane + (size_t) (ty.i0 + k) * stride, p, tx);
			irow += f;
		}
		if (!p.fxy_scale)
			return (unsigned char) irow;
		v = (int) mult_fix(ty.w1 ? irow - mult_fix_floor(f, ty.w1) : irow, p.fxy_scale);
	}
	return v > 255 ? 255 : (unsigned char) v;
}

/* A batch's scaled decode: its output size, whether the loop filter is bypassed, and the Y and U / V rescalers' constants and
 * taps (taps: Y across [sw], Y down [sh], U / V across [sw], U / V down [sh], one after another). */
struct WebpScale {
	int sw = 0, sh = 0, bypass = 0;
	RescaleParams y{}, uv{};
	std::vector<RescaleTap> taps;
};

/* webpload at scale: webp2vips.c:513-514 rounds the frame to rint(w * scale) x rint(h * scale) and refuses an axis outside
 * 1 .. 16383 (:541-552), webpload.c:189-193 limits scale to [0, 1024]; libwebp then bypasses the loop filter when both axes
 * shrink below three quarters (WebPIoInitFromOptions) */
int
webp_scale_geometry(const char *domain, int w, int h, double scale, WebpScale *S)
{
	if (!(scale >= 0 && scale <= 1024)) {
		error(domain, "scale %g is outside webpload's range 0 to 1024", scale);
		return -1;
	}
	const double fw = rint(w * scale), fh = rint(h * scale);
	if (fw <= 0 || fh <= 0 || fw > 0x3FFF || fh > 0x3FFF) {
		error(domain, "bad image dimensions: %d x %d at scale %g is %.0f x %.0f", w, h, scale, fw, fh);
		return -1;
	}
	S->sw = (int) fw;
	S->sh = (int) fh;
	S->bypass = S->sw < w * 3 / 4 && S->sh < h * 3 / 4;
	S->y = rescale_params(w, h, S->sw, S->sh);
	S->uv = rescale_params((w + 1) >> 1, (h + 1) >> 1, S->sw, S->sh);
	return 0;
}

void
webp_scale_taps(WebpScale *S)
{
	const int sw = S->sw, sh = S->sh;
	S->taps.resize(2 * ((size_t) sw + sh));
	rescale_taps(S->y, false, S->taps.data());
	rescale_taps(S->y, true, S->taps.data() + sw);
	rescale_taps(S->uv, false, S->taps.data() + sw + sh);
	rescale_taps(S->uv, true, S->taps.data() + 2 * sw + sh);
}

/* libwebp's WebPRescaler as it runs, for the host twin: rows imported one at a time into frow (and summed into irow, or
 * swapped with it when expanding), an output row exported whenever y_accum has gone to 0 or below.  Written from the
 * streaming form, independently of the closed form above, which the test-suite checks against it. */
struct RowRescaler {
	RescaleParams p;
	int y_accum, dst_y = 0;
	std::vector<unsigned> irow, frow;
	std::vector<unsigned char> out; /* the last exported row */

	explicit RowRescaler(const RescaleParams &q) : p(q), y_accum(q.y_expand ? (int) q.y_sub : (int) q.y_add), irow(q.dst_w, 0), frow(q.dst_w, 0), out(q.dst_w)
	{
	}
	bool
	pending() const
	{
		return dst_y < p.dst_h && y_accum <= 0;
	}
	int
	needed_lines(int max_lines) const
	{
		const int k = (y_accum + (int) p.y_sub - 1) / (int) p.y_sub;
		return k > max_lines ? max_lines : k;
	}
	void
	import_row(const unsigned char *src)
	{
		if (!p.x_expand) {
			unsigned sum = 0;
			int accum = 0, x_in = 0;
			for (int x = 0; x < p.dst_w; x++) {
				unsigned base = 0;
				accum += (int) p.x_add;
				while (accum > 0) {
					accum -= (int) p.x_sub;
					base = src[x_in++];
					sum += base;
				}
				const unsigned frac = base * (unsigned) -accum;
				frow[x] = sum * p.x_sub - frac;
				sum = mult_fix(frac, p.fx_scale);
			}
			return;
		}
		int accum = (int) p.x_add, x_in = 0;
		unsigned left = src[0], right = p.src_w > 1 ? src[1] : left;
		x_in++;
		for (int x = 0;;) {
			frow[x] = right * p.x_add + (left - right) * (unsigned) accum;
			if (++x >= p.dst_w)
				break;
			accum -= (int) p.x_sub;
			if (accum < 0) {
				left = right;
				right = src[++x_in];
				accum += (int) p.x_add;
			}
		}
	}
	/* WebPRescalerImport: up to n rows while no output is pending */
	int
	import(int n, const unsigned char *src, size_t stride)
	{
		int k = 0;
		for (; k < n && !pending(); k++, src += stride) {
			if (p.y_expand)
				irow.swap(frow);
			import_row(src);
			if (!p.y_expand)
				for (int x = 0; x < p.dst_w; x++)
					irow[x] += frow[x];
			y_accum -= (int) p.y_sub;
		}
		return k;
	}
	void
	export_row()
	{
		for (int x = 0; x < p.dst_w; x++) {
			int v;
			if (p.y_expand) {
				unsigned J = frow[x];
				if (y_accum != 0) {
					const unsigned B = rescaler_frac((unsigned) -y_accum, p.y_sub), A = (unsigned) (RESCALER_ONE - B);
					J = (unsigned) (((unsigned long long) A * frow[x] + (unsigned long long) B * irow[x] + RESCALER_ROUNDER) >> 32);
				}
				v = (int) mult_fix(J, p.fy_scale);
			}
			else if (!p.fxy_scale) {
				out[x] = (unsigned char) irow[x];
				irow[x] = 0;
				continue;
			}
			else {
				const unsigned yscale = p.fy_scale * (unsigned) -y_accum;
				const unsigned frac = yscale ? mult_fix_floor(frow[x], yscale) : 0u;
				v = (int) mult_fix(irow[x] - frac, p.fxy_scale);
				irow[x] = frac;
			}
			out[x] = v > 255 ? 255 : (unsigned char) v;
		}
		y_accum += (int) p.y_add;
		dst_y++;
	}
};

/* EmitRescaledRGB over a whole frame: Y rows in, U and V rows as the U rescaler needs them, and an RGB row out whenever Y
 * and U both have one pending; out is sw x sh x 3 at out_bpl.  0, or -1 if the rows run out before the last output row. */
int
rescale_frame_rows(const Planes &P, int h, const WebpScale &S, unsigned char *out, size_t out_bpl)
{
	RowRescaler ry(S.y), ru(S.uv), rv(S.uv);
	const int uv_h = (h + 1) >> 1;
	int j = 0, uv_j = 0, y_out = 0;
	while (j < h) {
		j += ry.import(h - j, P.y + (size_t) j * P.ys, P.ys);
		if (ru.needed_lines(uv_h - uv_j) > 0) {
			const int k = ru.import(uv_h - uv_j, P.u + (size_t) uv_j * P.uvs, P.uvs);
			rv.import(uv_h - uv_j, P.v + (size_t) uv_j * P.uvs, P.uvs);
			uv_j += k;
		}
		for (; ry.pending() && ru.pending(); y_out++) {
			ry.export_row();
			ru.export_row();
			rv.export_row();
			unsigned char *o = out + (size_t) y_out * out_bpl;
			for (int x = 0; x < S.sw; x++)
				webp_yuv_rgb(ry.out[x], ru.out[x], rv.out[x], o + 3 * x);
		}
	}
	return y_out == S.sh ? 0 : -1;
}

/* ------------------------------------------------------------------ the device pipeline */

/* one frame as the kernels see it; offsets are into the chunk's pools */
struct WebpFrameDev {
	unsigned long long data_off;	/* the VP8 data in the data pool */
	unsigned long long scratch_off; /* header, macroblocks, contexts, coefficients and planes in the scratch pool */
	unsigned len, first_len;
	int w, h, mb_w, mb_h;
};

VB_HD size_t
al16(size_t v)
{
	return (v + 15) & ~(size_t) 15;
}

/* a frame's scratch: header, macroblocks, the column contexts (4 sub-modes, the non-zero bits, the Y2 bit), the
 * coefficients (384 per macroblock) and the three planes */
struct ScratchLayout {
	size_t mb, ctx, coef, y, u, v, total;
};

VB_HD ScratchLayout
scratch_layout(int mb_w, int mb_h)
{
	const size_t mbs = (size_t) mb_w * mb_h;
	ScratchLayout L;
	L.mb = al16(sizeof(WebpHdr));
	L.ctx = L.mb + al16(mbs * sizeof(WebpMb));
	L.coef = L.ctx + al16((size_t) mb_w * 6);
	L.y = L.coef + mbs * 384 * sizeof(short);
	L.u = L.y + mbs * 256;
	L.v = L.u + mbs * 64;
	L.total = L.v + mbs * 64;
	return L;
}

VB_HD Planes
layout_planes(const ScratchLayout &L, unsigned char *s, int mb_w)
{
	return Planes{s + L.y, s + L.u, s + L.v, mb_w * 16, mb_w * 8};
}

__global__ void
webp_header_kernel(const WebpFrameDev *frames, int n, const unsigned char *data, unsigned char *scratch, int *status)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n)
		return;
	const WebpFrameDev F = frames[i];
	unsigned char *s = scratch + F.scratch_off;
	const ScratchLayout L = scratch_layout(F.mb_w, F.mb_h);
	WebpHdr *H = (WebpHdr *) s;
	WebpMb *mbs = (WebpMb *) (s + L.mb);
	unsigned char *top = s + L.ctx;
	BoolDec br;
	int rc = webp_header(data + F.data_off, F.len, F.first_len, H, br);
	for (int x = 0; x < 4 * F.mb_w; x++)
		top[x] = M_DC;
	for (int y = 0; y < F.mb_h && !rc; y++) {
		unsigned char left[4] = {M_DC, M_DC, M_DC, M_DC};
		for (int x = 0; x < F.mb_w; x++)
			webp_mb_modes(br, *H, top + 4 * x, left, mbs[(size_t) y * F.mb_w + x]);
		if (br.eof)
			rc = WERR_P0_EOF;
	}
	H->status = rc;
	status[i] = rc;
}

__global__ void
webp_token_kernel(const WebpFrameDev *frames, int n, const unsigned char *data, unsigned char *scratch, int *status)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n || status[i])
		return;
	const WebpFrameDev F = frames[i];
	unsigned char *s = scratch + F.scratch_off;
	const ScratchLayout L = scratch_layout(F.mb_w, F.mb_h);
	const WebpHdr *H = (const WebpHdr *) s;
	WebpMb *mbs = (WebpMb *) (s + L.mb);
	unsigned char *tnz = s + L.ctx + 4 * F.mb_w, *tdc = tnz + F.mb_w;
	short *coef = (short *) (s + L.coef);
	const unsigned char *d = data + F.data_off;
	BoolDec parts[8];
	const int np = H->num_parts;
	for (int p = 0; p < np; p++)
		bd_init(parts[p], d + H->part_off[p], H->part_len[p]);
	for (int x = 0; x < F.mb_w; x++)
		tnz[x] = tdc[x] = 0;
	for (int y = 0; y < F.mb_h; y++) {
		BoolDec &br = parts[y & (np - 1)];
		unsigned char lnz = 0, ldc = 0;
		for (int x = 0; x < F.mb_w; x++) {
			const size_t k = (size_t) y * F.mb_w + x;
			webp_mb_tokens(br, *H, mbs[k], tnz[x], tdc[x], lnz, ldc, coef + k * 384);
			if (br.eof) {
				status[i] = WERR_TOKENS_EOF;
				return;
			}
		}
	}
}

/* One CTA per frame.  Macroblock (x, y) needs (x - 1, y) and (x + 1, y - 1) done first, for prediction and for the filter
 * alike, so the CTA walks the diagonals x + 2y = t, one thread per macroblock of a diagonal: first reconstructing every
 * macroblock, then filtering them in place.  bypass: the scaled decode's filter bypass, one pass only.
 */
__global__ void __launch_bounds__(256)
webp_recon_kernel(const WebpFrameDev *frames, unsigned char *scratch, const int *status, int bypass)
{
	const int i = blockIdx.x;
	if (status[i])
		return;
	const WebpFrameDev F = frames[i];
	unsigned char *s = scratch + F.scratch_off;
	const ScratchLayout L = scratch_layout(F.mb_w, F.mb_h);
	const WebpHdr *H = (const WebpHdr *) s;
	const WebpMb *mbs = (const WebpMb *) (s + L.mb);
	const short *coef = (const short *) (s + L.coef);
	const Planes P = layout_planes(L, s, F.mb_w);
	const int steps = F.mb_w + 2 * (F.mb_h - 1);
	for (int pass = 0; pass < (H->filter_type && !bypass ? 2 : 1); pass++)
		for (int t = 0; t < steps; t++) {
			/* y from max(0, ceil((t - mb_w + 1) / 2)) to min(mb_h - 1, t / 2) */
			const int y0 = t >= F.mb_w ? (t - F.mb_w + 2) >> 1 : 0, y1 = min(F.mb_h - 1, t >> 1);
			for (int y = y0 + (int) threadIdx.x; y <= y1; y += blockDim.x) {
				const int x = t - 2 * y;
				const size_t k = (size_t) y * F.mb_w + x;
				if (pass == 0)
					webp_recon_mb(mbs[k], coef + k * 384, x, y, F.mb_w, P);
				else
					webp_filter_mb(*H, mbs[k], x, y, P);
			}
			__syncthreads();
		}
}

__global__ void
webp_rgb_kernel(const WebpFrameDev *frames, unsigned char *scratch, unsigned char *out, size_t out_bpl, size_t out_frame_stride)
{
	const WebpFrameDev F = frames[blockIdx.z];
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= F.w)
		return;
	const Planes P = layout_planes(scratch_layout(F.mb_w, F.mb_h), scratch + F.scratch_off, F.mb_w);
	unsigned char *o = out + (size_t) blockIdx.z * out_frame_stride;
	for (int y = blockIdx.y; y < F.h; y += gridDim.y)
		webp_rgb_pixel(P, F.w, F.h, x, y, o + (size_t) y * out_bpl + (size_t) x * 3);
}

/* the scaled decode's constants as the output kernel takes them: the two rescalers and their taps in device memory */
struct WebpScaleDev {
	RescaleParams y, uv;
	const RescaleTap *yx, *yy, *uvx, *uvy;
	int sw, sh;
};

/* The scaled decode's output, one thread per output pixel: its Y, U and V samples each in closed form from the planes
 * (rescale_sample), then libwebp's YUV -> RGB, written straight into out. */
__global__ void
webp_scaled_rgb_kernel(const WebpFrameDev *frames, unsigned char *scratch, WebpScaleDev S, unsigned char *out, size_t out_bpl,
	size_t out_frame_stride)
{
	const WebpFrameDev F = frames[blockIdx.z];
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= S.sw)
		return;
	const Planes P = layout_planes(scratch_layout(F.mb_w, F.mb_h), scratch + F.scratch_off, F.mb_w);
	const RescaleTap yx = S.yx[x], uvx = S.uvx[x];
	unsigned char *o = out + (size_t) blockIdx.z * out_frame_stride + (size_t) x * 3;
	for (int y = blockIdx.y; y < S.sh; y += gridDim.y) {
		const RescaleTap yy = S.yy[y], uvy = S.uvy[y];
		const int Y = rescale_sample(P.y, P.ys, S.y, yx, yy);
		const int u = rescale_sample(P.u, P.uvs, S.uv, uvx, uvy);
		const int v = rescale_sample(P.v, P.uvs, S.uv, uvx, uvy);
		webp_yuv_rgb(Y, u, v, o + (size_t) y * out_bpl);
	}
}

/* ------------------------------------------------------------------ the container, on the host */

struct WebpHeader {
	int w = 0, h = 0;
	const unsigned char *vp8 = nullptr; /* the VP8 data the decoder reads: the chunk's payload and its pad byte */
	unsigned len = 0, first_len = 0;
	const unsigned char *icc = nullptr;
	size_t icc_len = 0;
};

unsigned
le32(const unsigned char *p)
{
	return p[0] | (p[1] << 8) | (p[2] << 16) | ((unsigned) p[3] << 24);
}

/* RIFF / VP8X / chunk structure and the VP8 frame tag (RFC 6386 9.1, 19.1); 0, or -1 with the reason */
int
parse_webp(const char *domain, const unsigned char *d, size_t len, WebpHeader *H)
{
	*H = WebpHeader();
	if (!webp_signature(d, len)) {
		error(domain, "not a WebP stream (no RIFF / WEBP signature)");
		return -1;
	}
	const size_t riff = le32(d + 4);
	if (riff < 12 || riff + 8 > len) {
		error(domain, "bad RIFF size %zu for a %zu-byte buffer", riff, len);
		return -1;
	}
	const size_t end = 8 + riff;
	bool vp8x = false;
	int canvas_w = 0, canvas_h = 0;
	for (size_t at = 12; at + 8 <= end;) {
		const unsigned char *c = d + at;
		const size_t size = le32(c + 4), padded = size + (size & 1);
		if (padded > end - at - 8) {
			error(domain, "chunk %.4s of %zu bytes runs past the RIFF", (const char *) c, size);
			return -1;
		}
		const bool first = at == 12;
		if (!memcmp(c, "VP8L", 4)) {
			error(domain, "lossless WebP (VP8L) is not decoded on the device");
			return -1;
		}
		if (!memcmp(c, "ALPH", 4) || (first && !memcmp(c, "VP8X", 4) && size >= 1 && (c[8] & 0x10))) {
			error(domain, "WebP with alpha is not decoded on the device");
			return -1;
		}
		if (!memcmp(c, "ANIM", 4) || !memcmp(c, "ANMF", 4) || (first && !memcmp(c, "VP8X", 4) && size >= 1 && (c[8] & 0x02))) {
			error(domain, "animated WebP is not decoded on the device");
			return -1;
		}
		if (first && !memcmp(c, "VP8X", 4)) {
			if (size < 10) {
				error(domain, "VP8X chunk of %zu bytes", size);
				return -1;
			}
			vp8x = true;
			canvas_w = 1 + (c[12] | (c[13] << 8) | (c[14] << 16));
			canvas_h = 1 + (c[15] | (c[16] << 8) | (c[17] << 16));
		}
		else if (!memcmp(c, "VP8 ", 4)) {
			if (H->vp8) {
				error(domain, "more than one VP8 chunk");
				return -1;
			}
			H->vp8 = c + 8;
			H->len = (unsigned) padded;
			const unsigned char *v = H->vp8;
			if (size < 10) {
				error(domain, "truncated VP8 frame header");
				return -1;
			}
			const unsigned bits = v[0] | (v[1] << 8) | (v[2] << 16);
			if (bits & 1) {
				error(domain, "VP8 frame is not a key frame");
				return -1;
			}
			if (v[3] != 0x9d || v[4] != 0x01 || v[5] != 0x2a) {
				error(domain, "bad VP8 start code");
				return -1;
			}
			if (((bits >> 1) & 7) > 3 || !((bits >> 4) & 1)) {
				error(domain, "bad VP8 frame tag (profile %u, show %u)", (bits >> 1) & 7, (bits >> 4) & 1);
				return -1;
			}
			H->first_len = bits >> 5;
			H->w = (v[6] | (v[7] << 8)) & 0x3fff;
			H->h = (v[8] | (v[9] << 8)) & 0x3fff;
			if (H->w == 0 || H->h == 0) {
				error(domain, "VP8 frame of zero width or height");
				return -1;
			}
			if (H->first_len >= size || H->first_len > H->len - 10) {
				error(domain, "bad partition length %u in a VP8 chunk of %zu bytes", H->first_len, size);
				return -1;
			}
		}
		else if (first) {
			error(domain, "first chunk %.4s is none of VP8, VP8L and VP8X", (const char *) c);
			return -1;
		}
		else if (!memcmp(c, "ICCP", 4) && vp8x && !H->icc) {
			H->icc = c + 8;
			H->icc_len = size;
		}
		if (!vp8x && H->vp8)
			break; /* the simple format: what follows the image chunk is not read */
		at += 8 + padded;
	}
	if (!H->vp8) {
		error(domain, "no VP8 chunk");
		return -1;
	}
	if (vp8x && (canvas_w != H->w || canvas_h != H->h)) {
		error(domain, "VP8X canvas %d x %d differs from the %d x %d frame", canvas_w, canvas_h, H->w, H->h);
		return -1;
	}
	return 0;
}

/* VB200_WEBP_TIMING set: the last batch's device milliseconds in the header, token, reconstruction and RGB kernels, summed
 * over its chunks and read by vb200_debug_webp_times (each chunk then waits for its events) */
thread_local float t_webp_ms[4] = {-1, -1, -1, -1};

struct WebpTimer {
	bool on = false;
	cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
	WebpTimer()
	{
		const char *e = getenv("VB200_WEBP_TIMING");
		on = e && *e;
		for (int k = 0; k < 5 && on; k++)
			on = cudaEventCreate(&ev[k]) == cudaSuccess;
	}
	~WebpTimer()
	{
		for (cudaEvent_t e : ev)
			if (e)
				cudaEventDestroy(e);
	}
	void
	mark(int k, cudaStream_t s)
	{
		if (on)
			cudaEventRecord(ev[k], s);
	}
	/* after mark(0 .. 4): add the four kernels' times */
	void
	add()
	{
		if (!on || cudaEventSynchronize(ev[4]) != cudaSuccess)
			return;
		for (int k = 0; k < 4; k++) {
			float t = 0;
			if (cudaEventElapsedTime(&t, ev[k], ev[k + 1]) == cudaSuccess)
				t_webp_ms[k] += t;
		}
	}
};

/* device bytes a frame takes in a chunk: its staged VP8 data and its scratch */
size_t
frame_device_bytes(const WebpHeader &H)
{
	return align16(H.len) + align16(scratch_layout((H.w + 15) >> 4, (H.h + 15) >> 4).total);
}

} // namespace

bool
webp_signature(const void *buf, size_t len)
{
	const unsigned char *d = (const unsigned char *) buf;
	return buf && len >= 12 && !memcmp(d, "RIFF", 4) && !memcmp(d + 8, "WEBP", 4);
}

int
webp_icc_profile(const char *domain, const unsigned char *d, size_t len, std::vector<unsigned char> *profile)
{
	profile->clear();
	WebpHeader H;
	if (parse_webp(domain, d, len, &H))
		return -1;
	if (H.icc)
		profile->assign(H.icc, H.icc + H.icc_len);
	return 0;
}

/* Decode n WebP streams (host memory) of one geometry into out[n][h][w][3] on the device (out = nullptr: only report the
 * geometry).  Containers and frame tags are read on the host workers; the frames go up in chunks bounded by device
 * memory, each one pinned block (frame records and VP8 data) copied to the device and decoded on s.  Every frame of a
 * chunk must decode clean before its pixels are converted into out; the call returns when they are.
 *
 * scale != 1 is libwebp's scaled decode at webpload's rounding: the frames must share one source size, g is the scaled
 * size, the loop filter is bypassed when both axes shrink below three quarters, and webp_scaled_rgb_kernel writes the
 * rescaled pixels straight into out from the planes (so a chunk still holds only VP8 data and planes), with the taps
 * uploaded once for the batch.
 */
int
dev_webp_decode_batch(const char *domain, const void *const *bufs, const size_t *lens, int n, double scale, void *out, size_t out_bpl,
	size_t out_frame_stride, StreamGeometry *g, cudaStream_t s)
{
	std::vector<WebpHeader> hdr(n);
	if (parse_streams(
			domain, "frame", n, [&](int i) { return parse_webp(domain, (const unsigned char *) bufs[i], lens[i], &hdr[i]); },
			[&](int i) { return StreamGeometry{hdr[i].w, hdr[i].h, 3, 0}; }, g))
		return -1;
	const int W = g->w, Hh = g->h, mb_w = (W + 15) >> 4, mb_h = (Hh + 15) >> 4;
	const bool scaled = scale != 1.0;
	WebpScale S;
	if (scaled) {
		if (webp_scale_geometry(domain, W, Hh, scale, &S))
			return -1;
		g->w = S.sw;
		g->h = S.sh;
	}
	if (!out)
		return 0;
	if (check_out_strides(domain, *g, out_bpl, out_frame_stride))
		return -1;
	WebpScaleDev SD{};
	RescaleTap *taps = nullptr;
	if (scaled) {
		webp_scale_taps(&S);
		const size_t bytes = S.taps.size() * sizeof(RescaleTap);
		if (dev_alloc(domain, (void **) &taps, bytes, s))
			return -1;
		if (cudaMemcpyAsync(taps, S.taps.data(), bytes, cudaMemcpyHostToDevice, s) != cudaSuccess) {
			dev_free(taps, s);
			return cuda_fail(domain, cudaGetLastError(), "webp rescaler taps");
		}
		SD = WebpScaleDev{S.y, S.uv, taps, taps + S.sw, taps + S.sw + S.sh, taps + 2 * S.sw + S.sh, S.sw, S.sh};
	}
	const size_t scratch_bytes = align16(scratch_layout(mb_w, mb_h).total);
	WebpTimer timer;
	for (float &t : t_webp_ms)
		t = timer.on ? 0.f : -1.f;
	const int rc = decode_chunks(domain, "webp", "frame", n, [&](int i) { return frame_device_bytes(hdr[i]); }, [&](int c0, int cn) {
		/* the block: records and VP8 data staged; each frame's macroblock scratch */
		std::vector<WebpFrameDev> F(cn);
		size_t data = 0;
		for (int i = 0; i < cn; i++) {
			const WebpHeader &H = hdr[c0 + i];
			F[i] = WebpFrameDev{data, (unsigned long long) i * scratch_bytes, H.len, H.first_len, H.w, H.h, mb_w, mb_h};
			data += align16(H.len);
		}
		const size_t off_data = align16(cn * sizeof(WebpFrameDev)), total = off_data + data;
		return decode_chunk(
			domain, "webp", {total, scratch_bytes * cn, cn},
			[&](unsigned char *hst) {
				memcpy(hst, F.data(), cn * sizeof(WebpFrameDev));
				parallel_for(cn, host_workers(), [&](int i) { memcpy(hst + off_data + F[i].data_off, hdr[c0 + i].vp8, hdr[c0 + i].len); });
			},
			[&](unsigned char *dev, int *status) {
				const WebpFrameDev *dF = (const WebpFrameDev *) dev;
				unsigned char *dS = dev + align16(total);
				/* the diagonals of a frame hold at most min(mb_h, ceil(mb_w / 2)) macroblocks */
				const int diag = std::min(mb_h, (mb_w + 1) / 2), threads = std::min(256, (diag + 31) / 32 * 32);
				timer.mark(0, s);
				webp_header_kernel<<<(cn + 63) / 64, 64, 0, s>>>(dF, cn, dev + off_data, dS, status);
				timer.mark(1, s);
				webp_token_kernel<<<(cn + 63) / 64, 64, 0, s>>>(dF, cn, dev + off_data, dS, status);
				timer.mark(2, s);
				webp_recon_kernel<<<cn, threads, 0, s>>>(dF, dS, status, S.bypass);
				timer.mark(3, s);
				return 3;
			},
			[&](int i, int st) { error(domain, "frame %d: %s", c0 + i, werr_text(st)); },
			[&](unsigned char *dev) {
				unsigned char *o = (unsigned char *) out + (size_t) c0 * out_frame_stride;
				if (scaled)
					webp_scaled_rgb_kernel<<<dim3((S.sw + 127) / 128, std::min(S.sh, kMaxGridY), cn), 128, 0, s>>>((const WebpFrameDev *) dev,
						dev + align16(total), SD, o, out_bpl, out_frame_stride);
				else
					webp_rgb_kernel<<<dim3((W + 127) / 128, std::min(Hh, kMaxGridY), cn), 128, 0, s>>>((const WebpFrameDev *) dev, dev + align16(total),
						o, out_bpl, out_frame_stride);
				timer.mark(4, s);
				timer.add();
				return 1;
			},
			s);
	}, s);
	if (taps)
		dev_free(taps, s);
	return rc;
}

/* the same decode on the CPU through the same per-symbol, per-block and per-pixel code, in raster order: the test-suite's
 * host twin.  At scale != 1 the planes go through RowRescaler in libwebp's row order instead of the closed form. */
int
host_webp_decode(const char *domain, const void *buf, size_t len, double scale, unsigned char *out, size_t out_bpl, int *out_w, int *out_h,
	int *out_bands)
{
	WebpHeader W;
	if (parse_webp(domain, (const unsigned char *) buf, len, &W))
		return -1;
	WebpScale S;
	const bool scaled = scale != 1.0;
	if (scaled && webp_scale_geometry(domain, W.w, W.h, scale, &S))
		return -1;
	if (out_w)
		*out_w = scaled ? S.sw : W.w;
	if (out_h)
		*out_h = scaled ? S.sh : W.h;
	if (out_bands)
		*out_bands = 3;
	if (!out)
		return 0;
	const int mb_w = (W.w + 15) >> 4, mb_h = (W.h + 15) >> 4;
	const size_t nmb = (size_t) mb_w * mb_h;
	WebpHdr H;
	BoolDec br;
	int rc = webp_header(W.vp8, W.len, W.first_len, &H, br);
	std::vector<WebpMb> mbs(nmb);
	std::vector<unsigned char> top(4 * (size_t) mb_w, M_DC), tnz(mb_w, 0), tdc(mb_w, 0);
	for (int y = 0; y < mb_h && !rc; y++) {
		unsigned char left[4] = {M_DC, M_DC, M_DC, M_DC};
		for (int x = 0; x < mb_w; x++)
			webp_mb_modes(br, H, &top[4 * x], left, mbs[(size_t) y * mb_w + x]);
		if (br.eof)
			rc = WERR_P0_EOF;
	}
	std::vector<short> coef(nmb * 384);
	if (!rc) {
		BoolDec parts[8];
		for (int p = 0; p < H.num_parts; p++)
			bd_init(parts[p], W.vp8 + H.part_off[p], H.part_len[p]);
		for (int y = 0; y < mb_h && !rc; y++) {
			BoolDec &tb = parts[y & (H.num_parts - 1)];
			unsigned char lnz = 0, ldc = 0;
			for (int x = 0; x < mb_w && !rc; x++) {
				const size_t k = (size_t) y * mb_w + x;
				webp_mb_tokens(tb, H, mbs[k], tnz[x], tdc[x], lnz, ldc, &coef[k * 384]);
				if (tb.eof)
					rc = WERR_TOKENS_EOF;
			}
		}
	}
	if (rc) {
		error(domain, "%s", werr_text(rc));
		return -1;
	}
	std::vector<unsigned char> planes(nmb * 384);
	const Planes P{planes.data(), planes.data() + nmb * 256, planes.data() + nmb * 320, mb_w * 16, mb_w * 8};
	for (int y = 0; y < mb_h; y++)
		for (int x = 0; x < mb_w; x++)
			webp_recon_mb(mbs[(size_t) y * mb_w + x], &coef[((size_t) y * mb_w + x) * 384], x, y, mb_w, P);
	if (H.filter_type && !S.bypass)
		for (int y = 0; y < mb_h; y++)
			for (int x = 0; x < mb_w; x++)
				webp_filter_mb(H, mbs[(size_t) y * mb_w + x], x, y, P);
	if (scaled) {
		if (rescale_frame_rows(P, W.h, S, out, out_bpl)) {
			error(domain, "the rescaler ran out of rows");
			return -1;
		}
		return 0;
	}
	for (int y = 0; y < W.h; y++)
		for (int x = 0; x < W.w; x++)
			webp_rgb_pixel(P, W.w, W.h, x, y, out + (size_t) y * out_bpl + (size_t) x * 3);
	return 0;
}

} // namespace vb200

/* ------------------------------------------------------------------ C ABI */

using namespace vb200;

extern "C" int
vb200_webp_geometry(const void *buf, size_t len, int *width, int *height, int *bands)
{
	return host_webp_decode("webp_geometry", buf, len, 1.0, nullptr, 0, width, height, bands);
}

extern "C" int
vb200_webp_decode_batch(const void *const *bufs, const size_t *lens, int n, void *out, int out_location, size_t out_bpl, size_t out_frame_stride,
	int *width, int *height, int *bands)
{
	return decode_batch_abi("webp_decode_batch", {STREAM_WEBP}, bufs, lens, n, out, out_location, out_bpl, out_frame_stride, width, height, bands);
}

static DecodeRequest
webp_request(double scale)
{
	DecodeRequest req{STREAM_WEBP};
	req.scale = scale;
	return req;
}

extern "C" int
vb200_webp_decode_batch_scaled(const void *const *bufs, const size_t *lens, int n, double scale, void *out, int out_location, size_t out_bpl,
	size_t out_frame_stride, int *width, int *height, int *bands)
{
	return decode_batch_abi("webp_decode_batch", webp_request(scale), bufs, lens, n, out, out_location, out_bpl, out_frame_stride, width, height,
		bands);
}

/* reference: vips_webpload_buffer(buf, len, &out, NULL), foreign/webpload.c */
extern "C" int
vb200_webpload_buffer(const void *buf, size_t len, VB200Image *out)
{
	return load_abi("webpload_buffer", {STREAM_WEBP}, buf, len, out);
}

/* reference: vips_webpload_buffer(buf, len, &out, "scale", scale, NULL) */
extern "C" int
vb200_webpload_buffer_scaled(const void *buf, size_t len, double scale, VB200Image *out)
{
	return load_abi("webpload_buffer", webp_request(scale), buf, len, out);
}

extern "C" int
vb200_debug_webp_decode_scaled(const void *buf, size_t len, double scale, void *out, size_t out_bpl, int *width, int *height, int *bands)
{
	return host_twin_abi("webp_decode (host twin)",
		[&](const char *domain) { return host_webp_decode(domain, buf, len, scale, (unsigned char *) out, out_bpl, width, height, bands); });
}

/* One plane of src_w x src_h (stride bytes a row) rescaled to dst_w x dst_h into out (out_bpl a row): closed_form set, by
 * rescale_sample over the taps, sample by sample, as webp_scaled_rgb_kernel runs it; otherwise by RowRescaler in row order. */
extern "C" int
vb200_debug_webp_rescale(const void *plane, size_t stride, int src_w, int src_h, int dst_w, int dst_h, int closed_form, void *out, size_t out_bpl)
{
	if (!plane || !out || src_w < 1 || src_h < 1 || dst_w < 1 || dst_h < 1 || stride < (size_t) src_w || out_bpl < (size_t) dst_w) {
		error("debug_webp_rescale", "bad arguments");
		return -1;
	}
	const unsigned char *src = (const unsigned char *) plane;
	unsigned char *dst = (unsigned char *) out;
	const RescaleParams p = rescale_params(src_w, src_h, dst_w, dst_h);
	if (closed_form) {
		std::vector<RescaleTap> tx(dst_w), ty(dst_h);
		rescale_taps(p, false, tx.data());
		rescale_taps(p, true, ty.data());
		for (int y = 0; y < dst_h; y++)
			for (int x = 0; x < dst_w; x++)
				dst[(size_t) y * out_bpl + x] = rescale_sample(src, stride, p, tx[x], ty[y]);
		return 0;
	}
	RowRescaler r(p);
	int j = 0;
	while (r.dst_y < dst_h) {
		j += r.import(src_h - j, src + (size_t) j * stride, stride);
		if (!r.pending()) {
			error("debug_webp_rescale", "the rescaler ran out of rows");
			return -1;
		}
		while (r.pending()) {
			r.export_row();
			memcpy(dst + (size_t) (r.dst_y - 1) * out_bpl, r.out.data(), dst_w);
		}
	}
	return 0;
}

extern "C" int
vb200_webp_icc_profile(const void *buf, size_t len, void *out, size_t cap, size_t *profile_len)
{
	return profile_abi("webp_icc_profile", out, cap, profile_len,
		[&](const char *domain, std::vector<unsigned char> *prof) { return webp_icc_profile(domain, (const unsigned char *) buf, len, prof); });
}

extern "C" int
vb200_debug_webp_decode(const void *buf, size_t len, void *out, size_t out_bpl, int *width, int *height, int *bands)
{
	return host_twin_abi("webp_decode (host twin)",
		[&](const char *domain) { return host_webp_decode(domain, buf, len, 1.0, (unsigned char *) out, out_bpl, width, height, bands); });
}

/* ms[4]: the last batch's device milliseconds in the header, token, reconstruction and RGB kernels on this thread, with
 * VB200_WEBP_TIMING set (-1 without it) */
extern "C" void
vb200_debug_webp_times(float *ms)
{
	if (ms)
		memcpy(ms, t_webp_ms, sizeof(t_webp_ms));
}

/* the constant tables as the decoder holds them, one after another (coefficient defaults, their update probabilities, the
 * sub-block mode probabilities, dc steps, ac steps as little-endian 16-bit, zigzag, bands): *len bytes, copied when they fit */
extern "C" int
vb200_debug_webp_tables(void *out, size_t cap, size_t *len)
{
	if (!len)
		return -1;
	*len = sizeof(WebpTables);
	if (out && cap >= sizeof(WebpTables))
		memcpy(out, &h_webp_tables, sizeof(WebpTables));
	return 0;
}
