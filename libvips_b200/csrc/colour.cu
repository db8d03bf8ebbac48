/* colour.cu -- vips_colourspace() for sRGB / RGB16 / scRGB / XYZ / LAB / LABS as ONE
 * fused kernel per route: each pixel is carried in registers through every
 * step the reference would run as a separate operation with a float image in
 * between (colourspace.c:223-497 route table; vips_colour_gen colour.c:119-156).
 *
 * Step arithmetic restates the reference's process_line functions exactly --
 * same float/double mix, same evaluation order, explicit round-to-nearest
 * intrinsics so nothing is contracted into an FMA:
 *   sRGB2scRGB.c:71-107, scRGB2XYZ.c:58-79, XYZ2Lab.c:108-171, Lab2LabS.c:58-74,
 *   LabS2Lab.c:54-69, Lab2XYZ.c:83-143, XYZ2scRGB.c:72-97 (LabQ2sRGB.c:263-284),
 *   scRGB2sRGB.c:83-131 (LabQ2sRGB.c:290-361).
 * LUTs (powf / cbrtf) are built on the HOST with the host libm, like the
 * reference does (LabQ2sRGB.c:130-159, XYZ2Lab.c:91-106), and uploaded once.
 * Bands beyond the third ride along exactly as vips_colour_build re-attaches
 * them: rescale by max_alpha_after / max_alpha_before in float, then
 * vips_cast to the step's output format (colour.c:252-291).
 */
#include <cmath>
#include <cstring>
#include <mutex>
#include <vector>

#include <math_constants.h>

#include "vb200_internal.h"
#include "colour_steps.cuh"

namespace vb200 {

namespace {

std::mutex g_tables_lock;
ColourTables g_tables[16];
bool g_tables_ready[16];

/* calcul_tables, LabQ2sRGB.c:130-159 */
void
host_rgb_tables(int range, std::vector<int> &Y2v, std::vector<float> &v2Y)
{
	Y2v.resize(range + 1);
	v2Y.resize(range);
	for (int i = 0; i < range; i++) {
		float f = (float) i / (range - 1);
		float v;
		if (f <= 0.0031308)
			v = 12.92F * f;
		else
			v = (1.0F + 0.055F) * powf(f, 1.0F / 2.4F) - 0.055F;
		Y2v[i] = rintf((range - 1) * v);
	}
	Y2v[range] = Y2v[range - 1];
	for (int i = 0; i < range; i++) {
		float f = (float) i / (range - 1);
		if (f <= 0.04045)
			v2Y[i] = f / 12.92F;
		else
			v2Y[i] = powf((f + 0.055F) / (1 + 0.055F), 2.4F);
	}
}

} // namespace

int
get_tables(const char *domain, ColourTables *out)
{
	int dev = 0;
	VB200_CUDA(domain, cudaGetDevice(&dev));
	std::lock_guard<std::mutex> lock(g_tables_lock);
	if (dev < 16 && g_tables_ready[dev]) {
		*out = g_tables[dev];
		return 0;
	}
	std::vector<int> y8, y16;
	std::vector<float> v8, v16, cb(kQuant);
	host_rgb_tables(256, y8, v8);
	host_rgb_tables(65536, y16, v16);
	/* table_init, XYZ2Lab.c:91-106 */
	for (int i = 0; i < kQuant; i++) {
		float Y = (double) i / kQuant;
		if (Y < 0.008856)
			cb[i] = 7.787F * Y + (16.0F / 116.0F);
		else
			cb[i] = cbrtf(Y);
	}
	/* the same table as (t[i], t[i + 1]) pairs: one aligned 8-byte gather per lookup */
	std::vector<float> cb2(2 * (size_t) kQuant);
	for (int i = 0; i < kQuant; i++) {
		cb2[2 * i] = cb[i];
		cb2[2 * i + 1] = cb[std::min(i + 1, kQuant - 1)];
	}
	const size_t bytes = (y8.size() + v8.size() + y16.size() + v16.size() + cb.size() + cb2.size()) * 4 + 16;
	char *block = nullptr;
	VB200_CUDA(domain, cudaMalloc(&block, bytes));
	char *p = block;
	auto put = [&](const void *src, size_t n) {
		cudaMemcpy(p, src, n, cudaMemcpyHostToDevice);
		char *at = p;
		p += n;
		return at;
	};
	ColourTables t;
	t.v2Y_8 = (const float *) put(v8.data(), v8.size() * 4);
	t.Y2v_8 = (const int *) put(y8.data(), y8.size() * 4);
	t.v2Y_16 = (const float *) put(v16.data(), v16.size() * 4);
	t.Y2v_16 = (const int *) put(y16.data(), y16.size() * 4);
	t.cbrt = (const float *) put(cb.data(), cb.size() * 4);
	p = (char *) (((uintptr_t) p + 15) & ~(uintptr_t) 15);
	t.cbrt2 = (const float2 *) put(cb2.data(), cb2.size() * 4);
	VB200_CUDA(domain, cudaDeviceSynchronize());
	if (dev < 16) {
		g_tables[dev] = t;
		g_tables_ready[dev] = true;
	}
	*out = t;
	return 0;
}

namespace {

template <bool LOOP>
__global__ void __launch_bounds__(256)
colour_route_kernel(const __grid_constant__ RouteParams P, int h, const void *__restrict__ in, void *__restrict__ out)
{
	__shared__ float s_v2Y_8[256];
	__shared__ float s_Y2v_8[257]; /* integers <= 255 held as floats: scRGB2sRGB_channel_f */
	for (int i = threadIdx.x; i < 257; i += blockDim.x) {
		if (i < 256)
			s_v2Y_8[i] = P.t.v2Y_8[i];
		s_Y2v_8[i] = (float) P.t.Y2v_8[i];
	}
	__syncthreads();

	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= P.w)
		return;
	int y = blockIdx.y;
	do {
		const char *pin = (const char *) in + (size_t) y * P.in_bpl;
		char *pout = (char *) out + (size_t) y * P.out_bpl;
		const int base = x * P.bands;

		/* the pixel: integer inputs are held exactly in float until their LUT step */
		float a = (float) load_elem(pin, P.in_fmt, base);
		float b = (float) load_elem(pin, P.in_fmt, base + 1);
		float c = (float) load_elem(pin, P.in_fmt, base + 2);
		int ia = 0, ib = 0, ic = 0; /* integer outputs (sRGB / RGB16 / LabS) */

		for (int s = 0; s < P.n_steps; s++) {
			switch (P.steps[s].step) {
			case S_sRGB2scRGB:
				a = s_v2Y_8[(int) a];
				b = s_v2Y_8[(int) b];
				c = s_v2Y_8[(int) c];
				break;
			case S_RGB162scRGB:
				a = __ldg(P.t.v2Y_16 + (int) a);
				b = __ldg(P.t.v2Y_16 + (int) b);
				c = __ldg(P.t.v2Y_16 + (int) c);
				break;
			case S_scRGB2XYZ:
				step_scRGB2XYZ(a, b, c);
				break;
			case S_XYZ2Lab:
				step_XYZ2Lab(P.t.cbrt, a, b, c);
				break;
			case S_Lab2XYZ:
				step_Lab2XYZ(a, b, c);
				break;
			case S_XYZ2scRGB:
				step_XYZ2scRGB(a, b, c);
				break;
			case S_LabS2Lab:
				a = (float) DIVC((double) a, 32767.0 / 100.0);
				b = (float) DIVC((double) b, 32768.0 / 128.0);
				c = (float) DIVC((double) c, 32768.0 / 128.0);
				break;
			case S_Lab2LabS:
				ia = (int) (short) clipd(0, __dmul_rn((double) a, 32767.0 / 100.0), 32767);
				ib = (int) (short) clipd(-32768, __dmul_rn((double) b, 32768.0 / 128.0), 32767);
				ic = (int) (short) clipd(-32768, __dmul_rn((double) c, 32768.0 / 128.0), 32767);
				break;
			case S_scRGB2sRGB:
				if (isnan(a) || isnan(b) || isnan(c))
					ia = ib = ic = 0;
				else {
					ia = scRGB2sRGB_channel_f(s_Y2v_8, 255.0f, a);
					ib = scRGB2sRGB_channel_f(s_Y2v_8, 255.0f, b);
					ic = scRGB2sRGB_channel_f(s_Y2v_8, 255.0f, c);
				}
				break;
			case S_Lab2LCh:
				step_Lab2LCh(a, b, c);
				break;
			case S_LCh2Lab:
				step_LCh2Lab(a, b, c);
				break;
			case S_XYZ2Yxy:
				step_XYZ2Yxy(a, b, c);
				break;
			case S_Yxy2XYZ:
				step_Yxy2XYZ(a, b, c);
				break;
			case S_scRGB2RGB16:
				if (isnan(a) || isnan(b) || isnan(c))
					ia = ib = ic = 0;
				else {
					ia = scRGB2sRGB_channel(P.t.Y2v_16, 65535, a);
					ib = scRGB2sRGB_channel(P.t.Y2v_16, 65535, b);
					ic = scRGB2sRGB_channel(P.t.Y2v_16, 65535, c);
				}
				break;
			}
		}

		switch (P.out_fmt) {
		case VB200_FORMAT_UCHAR:
			((uint8_t *) pout)[base] = (uint8_t) ia;
			((uint8_t *) pout)[base + 1] = (uint8_t) ib;
			((uint8_t *) pout)[base + 2] = (uint8_t) ic;
			break;
		case VB200_FORMAT_USHORT:
			((uint16_t *) pout)[base] = (uint16_t) ia;
			((uint16_t *) pout)[base + 1] = (uint16_t) ib;
			((uint16_t *) pout)[base + 2] = (uint16_t) ic;
			break;
		case VB200_FORMAT_SHORT:
			((int16_t *) pout)[base] = (int16_t) ia;
			((int16_t *) pout)[base + 1] = (int16_t) ib;
			((int16_t *) pout)[base + 2] = (int16_t) ic;
			break;
		default:
			((float *) pout)[base] = a;
			((float *) pout)[base + 1] = b;
			((float *) pout)[base + 2] = c;
			break;
		}

		/* extra bands: colour.c:252-291 per step */
		for (int e = 3; e < P.bands; e++) {
			store_elem(pout, P.out_fmt, base + e, carry_extra_band(load_elem(pin, P.in_fmt, base + e), P.steps, P.n_steps));
		}
	} while (LOOP && (y += gridDim.y) < h);
}

/* The two hot routes (BASELINE config 4), 3-band packed rows, four pixels per thread: sRGB bytes come
 * in as three 32-bit words and leave as three, Lab floats as three float4; the route is
 * compiled in (no per-step switch) and the cbrt table is read as aligned (t[i], t[i + 1]) pairs.
 * Same steps, same roundings as colour_route_kernel.
 */
template <bool LOOP>
__global__ void __launch_bounds__(256)
colour_srgb2lab_x4_kernel(const __grid_constant__ RouteParams P, int h, const uint8_t *__restrict__ in, float *__restrict__ out)
{
	__shared__ float s_v2Y_8[256];
	for (int i = threadIdx.x; i < 256; i += blockDim.x)
		s_v2Y_8[i] = P.t.v2Y_8[i];
	__syncthreads();
	const int q = blockIdx.x * blockDim.x + threadIdx.x; /* group of 4 pixels */
	if (q * 4 >= P.w)
		return;
	int y = blockIdx.y;
	do {
		const uint32_t *pin = (const uint32_t *) (in + (size_t) y * P.in_bpl) + (size_t) q * 3;
		float4 *pout = (float4 *) ((char *) out + (size_t) y * P.out_bpl) + (size_t) q * 3;
		const uint32_t w0 = __ldg(pin), w1 = __ldg(pin + 1), w2 = __ldg(pin + 2);
		const uint32_t bytes[12] = {w0 & 255, (w0 >> 8) & 255, (w0 >> 16) & 255, w0 >> 24, w1 & 255, (w1 >> 8) & 255,
			(w1 >> 16) & 255, w1 >> 24, w2 & 255, (w2 >> 8) & 255, (w2 >> 16) & 255, w2 >> 24};
		float r[12];
#pragma unroll
		for (int k = 0; k < 4; k++) {
			float a = s_v2Y_8[bytes[3 * k]], b = s_v2Y_8[bytes[3 * k + 1]], c = s_v2Y_8[bytes[3 * k + 2]];
			step_scRGB2XYZ(a, b, c);
			const float nX = (float) DIVC((double) __fmul_rn(100000.0f, a), 95.0470);
			const float nY = (float) DIVC((double) __fmul_rn(100000.0f, b), 100.0);
			const float nZ = (float) DIVC((double) __fmul_rn(100000.0f, c), 108.8827);
			const float cbx = cbrt_lookup2(P.t.cbrt2, nX);
			const float cby = cbrt_lookup2(P.t.cbrt2, nY);
			const float cbz = cbrt_lookup2(P.t.cbrt2, nZ);
			r[3 * k] = __fsub_rn(__fmul_rn(116.0F, cby), 16.0F);
			r[3 * k + 1] = __fmul_rn(500.0F, __fsub_rn(cbx, cby));
			r[3 * k + 2] = __fmul_rn(200.0F, __fsub_rn(cby, cbz));
		}
		pout[0] = make_float4(r[0], r[1], r[2], r[3]);
		pout[1] = make_float4(r[4], r[5], r[6], r[7]);
		pout[2] = make_float4(r[8], r[9], r[10], r[11]);
	} while (LOOP && (y += gridDim.y) < h);
}

template <bool LOOP>
__global__ void __launch_bounds__(256)
colour_lab2srgb_x4_kernel(const __grid_constant__ RouteParams P, int h, const float *__restrict__ in, uint8_t *__restrict__ out)
{
	__shared__ float s_Y2v_8[257];
	for (int i = threadIdx.x; i < 257; i += blockDim.x)
		s_Y2v_8[i] = (float) P.t.Y2v_8[i];
	__syncthreads();
	const int q = blockIdx.x * blockDim.x + threadIdx.x;
	if (q * 4 >= P.w)
		return;
	int y = blockIdx.y;
	do {
		const float4 *pin = (const float4 *) ((const char *) in + (size_t) y * P.in_bpl) + (size_t) q * 3;
		uint32_t *pout = (uint32_t *) (out + (size_t) y * P.out_bpl) + (size_t) q * 3;
		const float4 v0 = __ldg(pin), v1 = __ldg(pin + 1), v2 = __ldg(pin + 2);
		const float f[12] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w, v2.x, v2.y, v2.z, v2.w};
		uint32_t o[12];
#pragma unroll
		for (int k = 0; k < 4; k++) {
			float a = f[3 * k], b = f[3 * k + 1], c = f[3 * k + 2];
			step_Lab2XYZ(a, b, c);
			step_XYZ2scRGB(a, b, c);
			if (isnan(a) || isnan(b) || isnan(c))
				o[3 * k] = o[3 * k + 1] = o[3 * k + 2] = 0;
			else {
				o[3 * k] = (uint32_t) scRGB2sRGB_channel_f(s_Y2v_8, 255.0f, a) & 255u;
				o[3 * k + 1] = (uint32_t) scRGB2sRGB_channel_f(s_Y2v_8, 255.0f, b) & 255u;
				o[3 * k + 2] = (uint32_t) scRGB2sRGB_channel_f(s_Y2v_8, 255.0f, c) & 255u;
			}
		}
		pout[0] = o[0] | (o[1] << 8) | (o[2] << 16) | (o[3] << 24);
		pout[1] = o[4] | (o[5] << 8) | (o[6] << 16) | (o[7] << 24);
		pout[2] = o[8] | (o[9] << 8) | (o[10] << 16) | (o[11] << 24);
	} while (LOOP && (y += gridDim.y) < h);
}

/* identity routes: a cast to the space's format (colourspace.c rows X -> X) */
__global__ void __launch_bounds__(256)
cast_kernel(const void *__restrict__ in, size_t in_bpl, int in_fmt, void *__restrict__ out, size_t out_bpl, int out_fmt,
	int ne, int h)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= ne)
		return;
	for (int y = blockIdx.y; y < h; y += gridDim.y) {
		const char *pin = (const char *) in + (size_t) y * in_bpl;
		char *pout = (char *) out + (size_t) y * out_bpl;
		store_elem(pout, out_fmt, x, cast_value(load_elem(pin, in_fmt, x), out_fmt));
	}
}

/* sRGB <-> RGB16 are not colour conversions in the reference: vips_sRGB2RGB16 / vips_RGB162sRGB (colourspace.c:85-110)
 * are vips_cast(..., "shift", TRUE) over EVERY band, extra bands included, and a re-tag.  cast.c:137-164: going down a
 * right shift by the width difference; going up a left shift with the bottom bit copied into the new bits.
 */
__global__ void __launch_bounds__(256)
shift_cast_kernel(const void *__restrict__ in, size_t in_bpl, void *__restrict__ out, size_t out_bpl, int up, int ne, int h)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= ne)
		return;
	for (int y = blockIdx.y; y < h; y += gridDim.y) {
		const char *pin = (const char *) in + (size_t) y * in_bpl;
		char *pout = (char *) out + (size_t) y * out_bpl;
		if (up) {
			const unsigned v = ((const uint8_t *) pin)[x];
			((uint16_t *) pout)[x] = (uint16_t) ((v << 8) | (((v & 1u) << 8) - (v & 1u)));
		}
		else
			((uint8_t *) pout)[x] = (uint8_t) (((const uint16_t *) pin)[x] >> 8);
	}
}

int
space_format(int space)
{
	switch (space) {
	case VB200_INTERPRETATION_sRGB: return VB200_FORMAT_UCHAR;
	case VB200_INTERPRETATION_RGB16: return VB200_FORMAT_USHORT;
	case VB200_INTERPRETATION_LABS: return VB200_FORMAT_SHORT;
	default: return VB200_FORMAT_FLOAT;
	}
}

/* The rows of the reference's route table among these spaces
 * (colourspace.c:223-497), e.g. sRGB -> LAB = sRGB2scRGB, scRGB2XYZ, XYZ2Lab.
 */
int
build_route(int from, int to, int *steps)
{
	const int XYZ = VB200_INTERPRETATION_XYZ, LAB = VB200_INTERPRETATION_LAB, LABS = VB200_INTERPRETATION_LABS;
	const int sRGB = VB200_INTERPRETATION_sRGB, RGB16 = VB200_INTERPRETATION_RGB16, scRGB = VB200_INTERPRETATION_scRGB;
	const int LCH = VB200_INTERPRETATION_LCH, YXY = VB200_INTERPRETATION_YXY;
	int n = 0;
	bool known_from = from == XYZ || from == LAB || from == LABS || from == sRGB || from == RGB16 || from == scRGB ||
		from == LCH || from == YXY;
	bool known_to = to == XYZ || to == LAB || to == LABS || to == sRGB || to == RGB16 || to == scRGB || to == LCH || to == YXY;
	if (!known_from || !known_to)
		return -1;
	if (from == to)
		return 0;
	/* colourspace.c:372, 420: these two rows are shifting casts, not steps of the route kernel (dev_colourspace) */
	if ((from == sRGB && to == RGB16) || (from == RGB16 && to == sRGB))
		return -1;
	/* LCH hangs off LAB and YXY off XYZ in every row of the table (colourspace.c:226, 236, 242, 252, 275-290):
	 * route to the hub, then one more step
	 */
	if (to == LCH || to == YXY) {
		const int hub = to == LCH ? LAB : XYZ;
		int m = 0;
		if (from != hub) {
			m = build_route(from, hub, steps);
			if (m < 0)
				return -1;
		}
		steps[m++] = to == LCH ? S_Lab2LCh : S_XYZ2Yxy;
		return m;
	}
	if (from == LCH) {
		steps[n++] = S_LCh2Lab;
		from = LAB;
	}
	else if (from == YXY) {
		steps[n++] = S_Yxy2XYZ;
		from = XYZ;
	}
	if (from == to)
		return n;
	if (from == sRGB) {
		steps[n++] = S_sRGB2scRGB;
		from = scRGB;
	}
	else if (from == RGB16) {
		steps[n++] = S_RGB162scRGB;
		from = scRGB;
	}
	else if (from == LABS) {
		steps[n++] = S_LabS2Lab;
		from = LAB;
	}
	if (from == to)
		return n;
	if (from == scRGB && (to == XYZ || to == LAB || to == LABS)) {
		steps[n++] = S_scRGB2XYZ;
		from = XYZ;
	}
	else if (from == LAB && to != LABS) {
		steps[n++] = S_Lab2XYZ;
		from = XYZ;
	}
	if (from == to)
		return n;
	if (from == XYZ && (to == LAB || to == LABS)) {
		steps[n++] = S_XYZ2Lab;
		from = LAB;
	}
	else if (from == XYZ) {
		steps[n++] = S_XYZ2scRGB;
		from = scRGB;
	}
	if (from == to)
		return n;
	if (from == LAB && to == LABS)
		steps[n++] = S_Lab2LabS;
	else if (from == scRGB && to == sRGB)
		steps[n++] = S_scRGB2sRGB;
	else if (from == scRGB && to == RGB16)
		steps[n++] = S_scRGB2RGB16;
	else
		return -1;
	return n;
}

void
step_io(int step, int *in_fmt, int *out_fmt, int *out_type)
{
	switch (step) {
	case S_sRGB2scRGB: *in_fmt = VB200_FORMAT_UCHAR; *out_fmt = VB200_FORMAT_FLOAT; *out_type = VB200_INTERPRETATION_scRGB; break;
	case S_RGB162scRGB: *in_fmt = VB200_FORMAT_USHORT; *out_fmt = VB200_FORMAT_FLOAT; *out_type = VB200_INTERPRETATION_scRGB; break;
	case S_scRGB2XYZ: *in_fmt = VB200_FORMAT_FLOAT; *out_fmt = VB200_FORMAT_FLOAT; *out_type = VB200_INTERPRETATION_XYZ; break;
	case S_XYZ2Lab: *in_fmt = VB200_FORMAT_FLOAT; *out_fmt = VB200_FORMAT_FLOAT; *out_type = VB200_INTERPRETATION_LAB; break;
	case S_Lab2LabS: *in_fmt = VB200_FORMAT_FLOAT; *out_fmt = VB200_FORMAT_SHORT; *out_type = VB200_INTERPRETATION_LABS; break;
	case S_LabS2Lab: *in_fmt = VB200_FORMAT_SHORT; *out_fmt = VB200_FORMAT_FLOAT; *out_type = VB200_INTERPRETATION_LAB; break;
	case S_Lab2XYZ: *in_fmt = VB200_FORMAT_FLOAT; *out_fmt = VB200_FORMAT_FLOAT; *out_type = VB200_INTERPRETATION_XYZ; break;
	case S_XYZ2scRGB: *in_fmt = VB200_FORMAT_FLOAT; *out_fmt = VB200_FORMAT_FLOAT; *out_type = VB200_INTERPRETATION_scRGB; break;
	case S_scRGB2sRGB: *in_fmt = VB200_FORMAT_FLOAT; *out_fmt = VB200_FORMAT_UCHAR; *out_type = VB200_INTERPRETATION_sRGB; break;
	case S_Lab2LCh: *in_fmt = VB200_FORMAT_FLOAT; *out_fmt = VB200_FORMAT_FLOAT; *out_type = VB200_INTERPRETATION_LCH; break;
	case S_LCh2Lab: *in_fmt = VB200_FORMAT_FLOAT; *out_fmt = VB200_FORMAT_FLOAT; *out_type = VB200_INTERPRETATION_LAB; break;
	case S_XYZ2Yxy: *in_fmt = VB200_FORMAT_FLOAT; *out_fmt = VB200_FORMAT_FLOAT; *out_type = VB200_INTERPRETATION_YXY; break;
	case S_Yxy2XYZ: *in_fmt = VB200_FORMAT_FLOAT; *out_fmt = VB200_FORMAT_FLOAT; *out_type = VB200_INTERPRETATION_XYZ; break;
	default: *in_fmt = VB200_FORMAT_FLOAT; *out_fmt = VB200_FORMAT_USHORT; *out_type = VB200_INTERPRETATION_RGB16; break;
	}
}

} // namespace

int
colour_route_params(const char *domain, int source_space, int space, RouteParams *P)
{
	int steps[8];
	const int n = build_route(source_space, space, steps);
	if (n < 0) {
		error(domain, "no known route from %d to %d on the device path", source_space, space);
		return -1;
	}
	memset(P, 0, sizeof(*P));
	if (get_tables(domain, &P->t))
		return -1;
	P->n_steps = n;
	int type = source_space;
	for (int i = 0; i < n; i++) {
		int ifmt, ofmt, otype;
		step_io(steps[i], &ifmt, &ofmt, &otype);
		const double before = interpretation_max_alpha(type), after = interpretation_max_alpha(otype);
		P->steps[i].step = steps[i];
		P->steps[i].out_fmt = ofmt;
		P->steps[i].rescale = before != after;
		P->steps[i].alpha_a = (float) (after / before);
		type = otype;
	}
	return 0;
}

int
dev_colourspace(const char *domain, const DevImage &in, DevImage *out, int space, int source_space, cudaStream_t s)
{
	if (colour_ext_space(space) || colour_ext_space(source_space))
		return dev_colourspace_ext(domain, in, out, space, source_space, s); /* colour_ext.cu */
	int steps[8];
	const dim3 block(256);
	const bool up = source_space == VB200_INTERPRETATION_sRGB && space == VB200_INTERPRETATION_RGB16;
	const bool down = source_space == VB200_INTERPRETATION_RGB16 && space == VB200_INTERPRETATION_sRGB;
	if (up || down) {
		const int want = up ? VB200_FORMAT_UCHAR : VB200_FORMAT_USHORT;
		if (in.fmt != want) {
			/* cast.c:476-495: a copy, or a cast through the guessed format first: not built */
			error(domain, "source space %d wants band format %d, image has %d", source_space, want, in.fmt);
			return -1;
		}
		if (dev_image_new(domain, out, in.w, in.h, in.bands, up ? VB200_FORMAT_USHORT : VB200_FORMAT_UCHAR, space, s))
			return -1;
		const int ne = in.w * in.bands;
		shift_cast_kernel<<<row_grid(ne, in.h), block, 0, s>>>(in.data, in.bpl, out->data, out->bpl, up ? 1 : 0, ne, in.h);
		cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess)
			return cuda_fail(domain, e, "shift_cast_kernel");
		count_launch();
		return 0;
	}
	const int n = build_route(source_space, space, steps);
	if (n < 0) {
		error(domain, "no known route from %d to %d on the device path", source_space, space);
		return -1;
	}
	if (!format_is_supported(in.fmt)) {
		error(domain, "band format %d not supported on the device path", in.fmt);
		return -1;
	}
	if (n == 0) {
		const int ofmt = space_format(space);
		if (dev_image_new(domain, out, in.w, in.h, in.bands, ofmt, space, s))
			return -1;
		const int ne = in.w * in.bands;
		cast_kernel<<<row_grid(ne, in.h), block, 0, s>>>(in.data, in.bpl, in.fmt, out->data, out->bpl, ofmt, ne, in.h);
		cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess)
			return cuda_fail(domain, e, "cast_kernel");
		count_launch();
		return 0;
	}
	if (in.bands < 3) {
		error(domain, "too few bands for operation");
		return -1;
	}
	int first_in, o, t;
	step_io(steps[0], &first_in, &o, &t);
	if (in.fmt != first_in) {
		/* the reference would insert a vips_cast first (colour.c:421-428, 338-342) */
		error(domain, "source space %d wants band format %d, image has %d", source_space, first_in, in.fmt);
		return -1;
	}
	RouteParams P;
	if (colour_route_params(domain, source_space, space, &P))
		return -1;
	P.w = in.w;
	P.bands = in.bands;
	P.in_fmt = in.fmt;
	P.out_fmt = P.steps[n - 1].out_fmt;
	if (dev_image_new(domain, out, in.w, in.h, in.bands, P.out_fmt, space, s))
		return -1;
	P.in_bpl = in.bpl;
	P.out_bpl = out->bpl;
	const bool x4 = in.bands == 3 && (in.w & 3) == 0 && ((uintptr_t) in.data & 15) == 0 && ((uintptr_t) out->data & 15) == 0 &&
		(in.bpl & 15) == 0 && (out->bpl & 15) == 0 && getenv("VB200_NO_COLOUR_X4") == nullptr;
	const dim3 grid4 = row_grid(in.w / 4, in.h);
	const bool loop = rows_loop(in.h);
	if (x4 && n == 3 && steps[0] == S_sRGB2scRGB && steps[1] == S_scRGB2XYZ && steps[2] == S_XYZ2Lab)
		(loop ? colour_srgb2lab_x4_kernel<true> : colour_srgb2lab_x4_kernel<false>)<<<grid4, block, 0, s>>>(P, in.h, (const uint8_t *) in.data, (float *) out->data);
	else if (x4 && n == 3 && steps[0] == S_Lab2XYZ && steps[1] == S_XYZ2scRGB && steps[2] == S_scRGB2sRGB)
		(loop ? colour_lab2srgb_x4_kernel<true> : colour_lab2srgb_x4_kernel<false>)<<<grid4, block, 0, s>>>(P, in.h, (const float *) in.data, (uint8_t *) out->data);
	else
		(loop ? colour_route_kernel<true> : colour_route_kernel<false>)<<<row_grid(in.w, in.h), block, 0, s>>>(P, in.h, in.data, out->data);
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
		return cuda_fail(domain, e, "colour_route_kernel");
	count_launch();
	return 0;
}

} // namespace vb200
