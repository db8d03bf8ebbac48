/* icc_eval.cuh -- the ICC evaluator's per-pixel code (icc.cu): profile sides, jobs and their __host__ __device__
 * evaluation.  Shared by the ICC kernels of icc.cu, the linear thumbnail kernels (thumbnail_linear.cu) and the host
 * twin vb200_debug_icc_eval, so that every target runs the same source.  Parsing and job building stay in icc.cu.
 */
#ifndef VB200_ICC_EVAL_CUH
#define VB200_ICC_EVAL_CUH

#include <cmath>
#include <cstdint>

#include "vb200_internal.h"

namespace vb200 {

enum { MODEL_MATRIX = 1, MODEL_GREY = 2, MODEL_LUT = 3, MODEL_MAB = 4 };
enum { CURVE_IDENTITY = 0, CURVE_TABLE = 1, CURVE_PARA = 2 };

struct IccCurve {
	int kind = CURVE_IDENTITY;
	int ptype = 0;	  /* parametricCurveType function 0..4 */
	double p[7] = {1, 1, 0, 0, 0, 0, 0}; /* g a b c d e f */
	int n = 0;		  /* table entries */
	int table_off = 0; /* into the float pool */
};

struct IccLut {
	int in_ch = 0, out_ch = 0, grid = 0, n_in = 0, n_out = 0;
	int in_off = 0, clut_off = 0, out_off = 0; /* float pool offsets, values 0..1 */
	int has_matrix = 0;
	int trilinear = 0; /* lcms2 reads B2A luts of Lab-PCS profiles with trilinear, everything else tetrahedral (cmsio1.c) */
	double m[9];
};

/* lutAtoBType / lutBtoAType (ICC.1:2010 10.10, 10.11): optional stages around a CLUT whose grid may
 * differ per dimension.  A2B runs A curves -> CLUT -> M curves -> matrix -> B curves, B2A runs
 * B curves -> matrix -> M curves -> CLUT -> A curves; values are the tags' 0..1 encodings.
 */
struct IccMab {
	int in_ch = 0, out_ch = 0;
	int has_a = 0, has_clut = 0, has_m = 0, has_matrix = 0;
	int trilinear = 0; /* B2A of a Lab-PCS profile: lcms2 interpolates it multilinearly (cmsio1.c) */
	int grid[4] = {0, 0, 0, 0};
	int clut_off = 0;
	IccCurve a[4], m[3], b[4];
	double mat[12]; /* 3 x 3 then the three offsets */
};

struct IccSide {
	int model = 0;
	int bands = 0;		 /* device channels */
	int pcs_lab = 0;	 /* profile PCS is Lab (else XYZ) */
	IccCurve curve[3];
	double m[9];		 /* device-linear -> XYZ D50 (import) or its inverse (export) */
	IccLut lut;
	IccMab mab;
	int to_pcs = 0; /* direction of this side (MODEL_MAB needs it) */
	const float *pool = nullptr; /* device or host pointer, set at use */
};
namespace {

/* ------------------------------------------------------------------ evaluation (host + device) */

#define HD __host__ __device__ __forceinline__

HD double
clamp01(double v)
{
	return v < 0.0 ? 0.0 : (v > 1.0 ? 1.0 : v);
}

HD double
curve_fwd(const IccCurve &c, const float *pool, double x)
{
	if (c.kind == CURVE_IDENTITY)
		return x;
	if (c.kind == CURVE_TABLE) {
		const double t = clamp01(x) * (c.n - 1);
		int i = (int) t;
		if (i > c.n - 2)
			i = c.n - 2;
		const double f = t - i;
		const double a = pool[c.table_off + i], b = pool[c.table_off + i + 1];
		return a + f * (b - a);
	}
	const double g = c.p[0], a = c.p[1], b = c.p[2], cc = c.p[3], d = c.p[4], e = c.p[5], f = c.p[6];
	switch (c.ptype) {
	case 0: return x < 0 ? 0.0 : pow(x, g);
	case 1: return x >= -b / a ? pow(a * x + b, g) : 0.0;
	case 2: return x >= -b / a ? pow(a * x + b, g) + cc : cc;
	case 3: return x >= d ? pow(a * x + b, g) : cc * x;
	default: return x >= d ? pow(a * x + b, g) + e : cc * x + f;
	}
}

HD double
curve_inv(const IccCurve &c, const float *pool, double y)
{
	if (c.kind == CURVE_IDENTITY)
		return y;
	if (c.kind == CURVE_TABLE) {
		/* monotone table: bisect, then interpolate inside the segment */
		const float *t = pool + c.table_off;
		const bool up = t[c.n - 1] >= t[0];
		int lo = 0, hi = c.n - 1;
		while (hi - lo > 1) {
			const int mid = (lo + hi) >> 1;
			if ((t[mid] <= y) == up)
				lo = mid;
			else
				hi = mid;
		}
		const double a = t[lo], b = t[hi];
		const double f = b != a ? (y - a) / (b - a) : 0.0;
		return clamp01((lo + clamp01(f)) / (c.n - 1));
	}
	const double g = c.p[0], a = c.p[1], b = c.p[2], cc = c.p[3], d = c.p[4], e = c.p[5], f = c.p[6];
	switch (c.ptype) {
	case 0: return y < 0 ? 0.0 : pow(y, 1.0 / g);
	case 1: return y <= 0 ? -b / a : (pow(y, 1.0 / g) - b) / a;
	case 2: return y <= cc ? -b / a : (pow(y - cc, 1.0 / g) - b) / a;
	case 3: {
		const double brk = pow(a * d + b, g);
		return y >= brk ? (pow(y, 1.0 / g) - b) / a : (cc != 0 ? y / cc : 0.0);
	}
	default: {
		const double brk = pow(a * d + b, g) + e;
		return y >= brk ? (pow(y - e, 1.0 / g) - b) / a : (cc != 0 ? (y - f) / cc : 0.0);
	}
	}
}

/* ICC PCS Lab <-> XYZ, D50, Y = 1 */
#define D50X 0.9642
#define D50Y 1.0
#define D50Z 0.8249

HD double
lab_f(double t)
{
	return t > 216.0 / 24389.0 ? cbrt(t) : (841.0 / 108.0) * t + 16.0 / 116.0;
}

HD double
lab_finv(double t)
{
	return t > 24.0 / 116.0 ? t * t * t : (108.0 / 841.0) * (t - 16.0 / 116.0);
}

HD void
xyz2lab(const double *xyz, double *lab)
{
	const double fx = lab_f(xyz[0] / D50X), fy = lab_f(xyz[1] / D50Y), fz = lab_f(xyz[2] / D50Z);
	lab[0] = 116.0 * fy - 16.0;
	lab[1] = 500.0 * (fx - fy);
	lab[2] = 200.0 * (fy - fz);
}

HD void
lab2xyz(const double *lab, double *xyz)
{
	const double fy = (lab[0] + 16.0) / 116.0, fx = fy + lab[1] / 500.0, fz = fy - lab[2] / 200.0;
	xyz[0] = lab_finv(fx) * D50X;
	xyz[1] = lab_finv(fy) * D50Y;
	xyz[2] = lab_finv(fz) * D50Z;
}

HD double
table_lerp(const float *t, int n, double x)
{
	const double p = clamp01(x) * (n - 1);
	int i = (int) p;
	if (i > n - 2)
		i = n - 2;
	const double f = p - i;
	return t[i] + f * ((double) t[i + 1] - t[i]);
}

/* Tetrahedral interpolation over the last three input channels of the CLUT at a fixed index of the
 * channels before them (`base_idx` already folded in): the six-tetrahedra split lcms2 uses
 * (cmsintrp.c), so that results inside a cell agree with it and not merely at the nodes.
 */
HD void
clut_tetra3(const IccLut &l, const float *pool, size_t base_idx, const int *b3, const double *f3, double *out)
{
	const size_t sx = (size_t) l.grid * l.grid, sy = (size_t) l.grid, sz = 1;
	const size_t o = (base_idx * l.grid * l.grid * l.grid) + b3[0] * sx + b3[1] * sy + b3[2] * sz;
	const double rx = f3[0], ry = f3[1], rz = f3[2];
	/* corner offsets (x, y, z) of the path c000 -> ... -> c111 through the tetrahedron that holds the point */
	size_t p1, p2, p3; /* nodes after the first, second and third step */
	double w1, w2, w3; /* weights of the three steps, in step order */
	if (rx >= ry && ry >= rz) { p1 = sx; p2 = sx + sy; w1 = rx; w2 = ry; w3 = rz; }
	else if (rx >= rz && rz >= ry) { p1 = sx; p2 = sx + sz; w1 = rx; w2 = rz; w3 = ry; }
	else if (rz >= rx && rx >= ry) { p1 = sz; p2 = sz + sx; w1 = rz; w2 = rx; w3 = ry; }
	else if (ry >= rx && rx >= rz) { p1 = sy; p2 = sy + sx; w1 = ry; w2 = rx; w3 = rz; }
	else if (ry >= rz && rz >= rx) { p1 = sy; p2 = sy + sz; w1 = ry; w2 = rz; w3 = rx; }
	else { p1 = sz; p2 = sz + sy; w1 = rz; w2 = ry; w3 = rx; }
	p3 = sx + sy + sz;
	const float *n0 = pool + l.clut_off + o * l.out_ch;
	const float *n1 = pool + l.clut_off + (o + p1) * l.out_ch;
	const float *n2 = pool + l.clut_off + (o + p2) * l.out_ch;
	const float *n3 = pool + l.clut_off + (o + p3) * l.out_ch;
	for (int c = 0; c < l.out_ch; c++)
		out[c] = n0[c] + ((double) n1[c] - n0[c]) * w1 + ((double) n2[c] - n1[c]) * w2 + ((double) n3[c] - n2[c]) * w3;
}

/* lut8 / lut16: input tables, CLUT (first channel varies slowest), output tables.  3 inputs:
 * tetrahedral; 4 inputs: linear along the first channel between two tetrahedral lookups (lcms2's
 * Eval4Inputs); 1 / 2 inputs: multilinear.
 */
HD void
lut_eval(const IccLut &l, const float *pool, const double *in, double *out)
{
	int base[4];
	double frac[4];
	for (int c = 0; c < l.in_ch; c++) {
		const double x = table_lerp(pool + l.in_off + c * l.n_in, l.n_in, in[c]);
		const double p = clamp01(x) * (l.grid - 1);
		int i = (int) p;
		if (i > l.grid - 2)
			i = l.grid - 2;
		base[c] = i;
		frac[c] = p - i;
	}
	double acc[4] = {0, 0, 0, 0};
	if (l.in_ch == 3 && !l.trilinear)
		clut_tetra3(l, pool, 0, base, frac, acc);
	else if (l.in_ch == 4 && !l.trilinear) {
		double lo[4], hi[4];
		clut_tetra3(l, pool, (size_t) base[0], base + 1, frac + 1, lo);
		clut_tetra3(l, pool, (size_t) base[0] + 1, base + 1, frac + 1, hi);
		for (int o = 0; o < l.out_ch; o++)
			acc[o] = lo[o] + (hi[o] - lo[o]) * frac[0];
	}
	else {
		const int corners = 1 << l.in_ch;
		for (int k = 0; k < corners; k++) {
			double w = 1.0;
			size_t idx = 0;
			for (int c = 0; c < l.in_ch; c++) {
				const int bit = (k >> c) & 1;
				w *= bit ? frac[c] : 1.0 - frac[c];
				idx = idx * l.grid + (size_t) (base[c] + bit);
			}
			const float *node = pool + l.clut_off + idx * l.out_ch;
			for (int o = 0; o < l.out_ch; o++)
				acc[o] += w * node[o];
		}
	}
	for (int o = 0; o < l.out_ch; o++)
		out[o] = table_lerp(pool + l.out_off + o * l.n_out, l.n_out, acc[o]);
}

/* lut16 / lut8 encode PCS Lab the ICC v2 way: L 0..100 -> 0..0xFF00, a, b -128..127+255/256 -> 0..0xFFFF
 * with 0x8000 = 0; XYZ as u1.15 (1.0 = 0x8000).  As 0..1 fractions of 0xFFFF:
 */
HD void
pcs_from_lut(const IccSide &s, const double *v, double *xyz)
{
	if (s.pcs_lab) {
		const double lab[3] = {v[0] * 65535.0 / 65280.0 * 100.0, v[1] * 65535.0 / 256.0 - 128.0, v[2] * 65535.0 / 256.0 - 128.0};
		lab2xyz(lab, xyz);
	}
	else
		for (int i = 0; i < 3; i++)
			xyz[i] = v[i] * 65535.0 / 32768.0;
}

HD void
pcs_to_lut(const IccSide &s, const double *xyz, double *v)
{
	if (s.pcs_lab) {
		double lab[3];
		xyz2lab(xyz, lab);
		v[0] = clamp01(lab[0] / 100.0 * 65280.0 / 65535.0);
		v[1] = clamp01((lab[1] + 128.0) * 256.0 / 65535.0);
		v[2] = clamp01((lab[2] + 128.0) * 256.0 / 65535.0);
	}
	else
		for (int i = 0; i < 3; i++)
			v[i] = clamp01(xyz[i] * 32768.0 / 65535.0);
}

/* n-dimensional CLUT with per-dimension grids: tetrahedral over the last three inputs, linear over a
 * fourth in front of them (as clut_tetra3 / lut_eval above), multilinear for 1 or 2 inputs
 */
HD void
mab_clut(const IccMab &m, const float *pool, const double *x, double *out)
{
	int base[4];
	double frac[4];
	for (int c = 0; c < m.in_ch; c++) {
		const double p = clamp01(x[c]) * (m.grid[c] - 1);
		int i = (int) p;
		if (i > m.grid[c] - 2)
			i = m.grid[c] - 2;
		base[c] = i;
		frac[c] = p - i;
	}
	/* strides in nodes, first input slowest */
	size_t stride[4];
	size_t acc_s = 1;
	for (int c = m.in_ch - 1; c >= 0; c--) {
		stride[c] = acc_s;
		acc_s *= (size_t) m.grid[c];
	}
	auto node = [&](size_t idx) { return pool + m.clut_off + idx * m.out_ch; };
	auto tetra = [&](size_t o, const int first, double *res) {
		const size_t sx = stride[first], sy = stride[first + 1], sz = stride[first + 2];
		const double rx = frac[first], ry = frac[first + 1], rz = frac[first + 2];
		size_t p1, p2;
		double w1, w2, w3;
		if (rx >= ry && ry >= rz) { p1 = sx; p2 = sx + sy; w1 = rx; w2 = ry; w3 = rz; }
		else if (rx >= rz && rz >= ry) { p1 = sx; p2 = sx + sz; w1 = rx; w2 = rz; w3 = ry; }
		else if (rz >= rx && rx >= ry) { p1 = sz; p2 = sz + sx; w1 = rz; w2 = rx; w3 = ry; }
		else if (ry >= rx && rx >= rz) { p1 = sy; p2 = sy + sx; w1 = ry; w2 = rx; w3 = rz; }
		else if (ry >= rz && rz >= rx) { p1 = sy; p2 = sy + sz; w1 = ry; w2 = rz; w3 = rx; }
		else { p1 = sz; p2 = sz + sy; w1 = rz; w2 = ry; w3 = rx; }
		const float *n0 = node(o), *n1 = node(o + p1), *n2 = node(o + p2), *n3 = node(o + sx + sy + sz);
		for (int c = 0; c < m.out_ch; c++)
			res[c] = n0[c] + ((double) n1[c] - n0[c]) * w1 + ((double) n2[c] - n1[c]) * w2 + ((double) n3[c] - n2[c]) * w3;
	};
	size_t o = 0;
	for (int c = 0; c < m.in_ch; c++)
		o += (size_t) base[c] * stride[c];
	if (m.in_ch == 3 && !m.trilinear)
		tetra(o, 0, out);
	else if (m.in_ch == 4 && !m.trilinear) {
		double lo[4], hi[4];
		tetra(o, 1, lo);
		tetra(o + stride[0], 1, hi);
		for (int c = 0; c < m.out_ch; c++)
			out[c] = lo[c] + (hi[c] - lo[c]) * frac[0];
	}
	else {
		for (int c = 0; c < m.out_ch; c++)
			out[c] = 0.0;
		for (int k = 0; k < (1 << m.in_ch); k++) {
			double w = 1.0;
			size_t idx = o;
			for (int c = 0; c < m.in_ch; c++) {
				const int bit = (k >> c) & 1;
				w *= bit ? frac[c] : 1.0 - frac[c];
				idx += bit ? stride[c] : 0;
			}
			const float *n = node(idx);
			for (int c = 0; c < m.out_ch; c++)
				out[c] += w * n[c];
		}
	}
}

HD void
mab_matrix(const IccMab &m, double *v)
{
	const double x = v[0], y = v[1], z = v[2];
	for (int r = 0; r < 3; r++)
		v[r] = m.mat[r * 3] * x + m.mat[r * 3 + 1] * y + m.mat[r * 3 + 2] * z + m.mat[9 + r];
}

/* v4 PCS encodings as 0..1: XYZ u1.15 of 16 bits (1.0 -> 32768 / 65535), Lab L / 100, (a, b + 128) / 255 */
HD void
mab_to_xyz(const IccSide &s, const double *dev, double *xyz)
{
	const IccMab &m = s.mab;
	double v[4] = {dev[0], dev[1], dev[2], dev[3]}, w[4];
	if (m.has_a)
		for (int c = 0; c < m.in_ch; c++)
			v[c] = curve_fwd(m.a[c], s.pool, v[c]);
	if (m.has_clut) {
		mab_clut(m, s.pool, v, w);
		for (int c = 0; c < m.out_ch; c++)
			v[c] = w[c];
	}
	if (m.has_m)
		for (int c = 0; c < 3; c++)
			v[c] = curve_fwd(m.m[c], s.pool, v[c]);
	if (m.has_matrix)
		mab_matrix(m, v);
	for (int c = 0; c < 3; c++)
		v[c] = curve_fwd(m.b[c], s.pool, v[c]);
	if (s.pcs_lab) {
		const double lab[3] = {v[0] * 100.0, v[1] * 255.0 - 128.0, v[2] * 255.0 - 128.0};
		lab2xyz(lab, xyz);
	}
	else
		for (int i = 0; i < 3; i++)
			xyz[i] = v[i] * 65535.0 / 32768.0;
}

HD void
mab_from_xyz(const IccSide &s, const double *xyz, double *dev)
{
	const IccMab &m = s.mab;
	double v[4] = {0, 0, 0, 0}, w[4];
	if (s.pcs_lab) {
		double lab[3];
		xyz2lab(xyz, lab);
		v[0] = lab[0] / 100.0;
		v[1] = (lab[1] + 128.0) / 255.0;
		v[2] = (lab[2] + 128.0) / 255.0;
	}
	else
		for (int i = 0; i < 3; i++)
			v[i] = xyz[i] * 32768.0 / 65535.0;
	for (int c = 0; c < 3; c++)
		v[c] = curve_fwd(m.b[c], s.pool, v[c]);
	if (m.has_matrix)
		mab_matrix(m, v);
	if (m.has_m)
		for (int c = 0; c < 3; c++)
			v[c] = curve_fwd(m.m[c], s.pool, v[c]);
	if (m.has_clut) {
		mab_clut(m, s.pool, v, w);
		for (int c = 0; c < m.out_ch; c++)
			v[c] = w[c];
	}
	if (m.has_a)
		for (int c = 0; c < m.out_ch; c++)
			v[c] = curve_fwd(m.a[c], s.pool, v[c]);
	for (int c = 0; c < m.out_ch; c++)
		dev[c] = clamp01(v[c]);
}

/* device values (0..1) -> PCS XYZ (D50, Y = 1) */
HD void
side_to_xyz(const IccSide &s, const double *dev, double *xyz)
{
	if (s.model == MODEL_MATRIX) {
		double lin[3];
		for (int i = 0; i < 3; i++)
			lin[i] = curve_fwd(s.curve[i], s.pool, dev[i]);
		for (int r = 0; r < 3; r++)
			xyz[r] = s.m[r * 3] * lin[0] + s.m[r * 3 + 1] * lin[1] + s.m[r * 3 + 2] * lin[2];
	}
	else if (s.model == MODEL_GREY) {
		const double y = curve_fwd(s.curve[0], s.pool, dev[0]);
		xyz[0] = y * D50X;
		xyz[1] = y * D50Y;
		xyz[2] = y * D50Z;
	}
	else if (s.model == MODEL_MAB)
		mab_to_xyz(s, dev, xyz);
	else {
		double v[4];
		lut_eval(s.lut, s.pool, dev, v);
		pcs_from_lut(s, v, xyz);
	}
}

/* PCS XYZ -> device values (0..1, clipped) */
HD void
side_from_xyz(const IccSide &s, const double *xyz, double *dev)
{
	if (s.model == MODEL_MATRIX) {
		for (int r = 0; r < 3; r++) {
			const double lin = s.m[r * 3] * xyz[0] + s.m[r * 3 + 1] * xyz[1] + s.m[r * 3 + 2] * xyz[2];
			dev[r] = clamp01(curve_inv(s.curve[r], s.pool, lin));
		}
	}
	else if (s.model == MODEL_GREY)
		dev[0] = clamp01(curve_inv(s.curve[0], s.pool, xyz[1] / D50Y));
	else if (s.model == MODEL_MAB)
		mab_from_xyz(s, xyz, dev);
	else {
		double v[3];
		pcs_to_lut(s, xyz, v);
		lut_eval(s.lut, s.pool, v, dev);
		for (int i = 0; i < s.bands; i++)
			dev[i] = clamp01(dev[i]);
	}
}

HD double
load_dev(const void *p, int fmt, size_t i)
{
	if (fmt == VB200_FORMAT_UCHAR)
		return ((const uint8_t *) p)[i] / 255.0;
	if (fmt == VB200_FORMAT_USHORT)
		return ((const uint16_t *) p)[i] / 65535.0;
	return ((const float *) p)[i];
}

HD void
store_dev(void *p, int depth, size_t i, double v)
{
	/* lcms2's _cmsQuickSaturateByte / Word: round half up after scaling */
	if (depth == 8)
		((uint8_t *) p)[i] = (uint8_t) (int) floor(v * 255.0 + 0.5);
	else
		((uint16_t *) p)[i] = (uint16_t) (int) floor(v * 65535.0 + 0.5);
}

HD double
sat16(double v)
{
	v = floor(v + 0.5);
	return v < 0.0 ? 0.0 : (v > 65535.0 ? 65535.0 : v);
}

/* float multiply / add without FMA contraction on either target (the reference's float steps round each operation) */
#ifdef __CUDA_ARCH__
#define FMUL_RN(a, b) __fmul_rn((a), (b))
#define FADD_RN(a, b) __fadd_rn((a), (b))
#else
#define FMUL_RN(a, b) ((float) (a) * (float) (b))
#define FADD_RN(a, b) ((float) (a) + (float) (b))
#endif

} // namespace

enum { MODE_IMPORT = 0, MODE_EXPORT = 1, MODE_TRANSFORM = 2, MODE_XYZ_EXPORT = 3 };

struct IccJob {
	IccSide in, out; /* whichever the mode uses */
	/* 0 import, 1 export, 2 transform, 3 vips_colourspace(sRGB or B_W -> XYZ) then export with XYZ PCS (thumbnail.c:957-970:
	 * an 8-bit image without an input profile); in mode 3, in.bands is 3 (sRGB) or 1 (B_W) and in_tab the sRGB2scRGB table
	 */
	int mode;
	int pcs_xyz;	 /* import / export: the vips PCS is XYZ (D65, Y = 100), else Lab */
	int in_fmt, depth;
	/* integer input / output through a matrix or grey profile: the TRCs tabulated once on the host
	 * (pool offsets, -1 = evaluate the curves per pixel): in_tab[c][code] = curve(code / max), and
	 * out_thr[c][k] = curve((k - 0.5) / max), so that the output code is the number of thresholds
	 * <= the linear value -- the same code floor(inverse(lin) * max + 0.5) gives, without a pow()
	 */
	int in_tab, in_tab_n, out_thr, out_thr_n;
	/* bands after the colour channels ride along (vips_colour_build, colour.c:196-291): rescaled by the ratio
	 * of the interpretations' alpha ranges in float, then cast to the output format with a clip
	 */
	int extra, out_fmt, alpha_rescale;
	float alpha_a;
};

namespace {

/* import / transform input: device codes -> PCS XYZ (D50, Y = 1).  tab: the job's tabulated TRCs when J.in_tab >= 0, wherever
 * they are staged (the pool, or a shared-memory copy in the linear thumbnail's V kernel)
 */
HD void
icc_tab_to_xyz(const IccJob &J, const float *tab, const int *code, double *xyz)
{
	double lin[3] = {0, 0, 0};
	for (int i = 0; i < 3; i++)
		if (i < J.in.bands)
			lin[i] = tab[i * J.in_tab_n + code[i]];
	if (J.in.model == MODEL_MATRIX)
		for (int r = 0; r < 3; r++)
			xyz[r] = J.in.m[r * 3] * lin[0] + J.in.m[r * 3 + 1] * lin[1] + J.in.m[r * 3 + 2] * lin[2];
	else {
		xyz[0] = lin[0] * D50X;
		xyz[1] = lin[0] * D50Y;
		xyz[2] = lin[0] * D50Z;
	}
}

HD void
icc_codes_to_xyz(const IccJob &J, const float *tab, const void *pin, double *xyz)
{
	if (J.in_tab >= 0) {
		int code[3] = {0, 0, 0};
		for (int i = 0; i < 3; i++)
			if (i < J.in.bands)
				code[i] = J.in_fmt == VB200_FORMAT_UCHAR ? ((const uint8_t *) pin)[i] : ((const uint16_t *) pin)[i];
		icc_tab_to_xyz(J, tab, code, xyz);
	}
	else {
		double dev[4] = {0, 0, 0, 0};
		for (int i = 0; i < J.in.bands; i++)
			dev[i] = load_dev(pin, J.in_fmt, i);
		side_to_xyz(J.in, dev, xyz);
	}
}

/* the import's XYZ16 (1.0 = 0x8000), then decode_xyz (icc_transform.c:879-909): float arithmetic, Bradford D50 -> D65 */
HD void
icc_decode_xyz16(const double *xyz, float *q)
{
	const float X = (float) (sat16(xyz[0] * 32768.0) / 32768.0) * 100.0f;
	const float Y = (float) (sat16(xyz[1] * 32768.0) / 32768.0) * 100.0f;
	const float Z = (float) (sat16(xyz[2] * 32768.0) / 32768.0) * 100.0f;
	q[0] = 0.955513F * X + -0.023073F * Y + 0.063309F * Z;
	q[1] = -0.028325F * X + 1.009942F * Y + 0.021055F * Z;
	q[2] = 0.012329F * X + -0.020536F * Y + 1.330714F * Z;
}

/* one pixel; pin / pout point at the pixel's first element */
HD void
icc_colour(const IccJob &J, const void *pin, void *pout)
{
	double dev[4] = {0, 0, 0, 0}, xyz[3] = {0, 0, 0};
	if (J.mode == 0 || J.mode == 2)
		icc_codes_to_xyz(J, J.in.pool + (J.in_tab >= 0 ? J.in_tab : 0), pin, xyz);
	if (J.mode == 0) {
		float *q = (float *) pout;
		if (!J.pcs_xyz) {
			/* Lab16, v4 encoding, then decode_lab (icc_transform.c:856-872) */
			double lab[3];
			xyz2lab(xyz, lab);
			q[0] = (float) (sat16(lab[0] * 655.35) / 655.35);
			q[1] = (float) (sat16((lab[1] + 128.0) * 257.0) / 257.0 - 128.0);
			q[2] = (float) (sat16((lab[2] + 128.0) * 257.0) / 257.0 - 128.0);
		}
		else
			icc_decode_xyz16(xyz, q);
		return;
	}
	float vxyz[3];
	if (J.mode == MODE_XYZ_EXPORT) {
		/* BW2sRGB (a grey pixel as three equal bands), vips_col_sRGB2scRGB_8 (sRGB2scRGB.c:71-107: the 8-bit table), then
		 * scRGB2XYZ.c:58-79 in float -- the route kernel's steps, evaluated operation by operation
		 */
		const uint8_t *q = (const uint8_t *) pin;
		float rgb[3];
		for (int c = 0; c < 3; c++)
			rgb[c] = J.in.pool[J.in_tab + q[J.in.bands == 1 ? 0 : c]];
		const float R = FMUL_RN(rgb[0], 100.0F), G = FMUL_RN(rgb[1], 100.0F), B = FMUL_RN(rgb[2], 100.0F);
		vxyz[0] = FADD_RN(FADD_RN(FMUL_RN(0.4124F, R), FMUL_RN(0.3576F, G)), FMUL_RN(0.1805F, B));
		vxyz[1] = FADD_RN(FADD_RN(FMUL_RN(0.2126F, R), FMUL_RN(0.7152F, G)), FMUL_RN(0.0722F, B));
		vxyz[2] = FADD_RN(FADD_RN(FMUL_RN(0.0193F, R), FMUL_RN(0.1192F, G)), FMUL_RN(0.9505F, B));
	}
	if (J.mode == MODE_EXPORT || J.mode == MODE_XYZ_EXPORT) {
		const float *p = J.mode == MODE_XYZ_EXPORT ? vxyz : (const float *) pin;
		if (!J.pcs_xyz) {
			const double lab[3] = {p[0], p[1], p[2]};
			lab2xyz(lab, xyz);
		}
		else {
			/* encode_xyz (icc_transform.c:1050-1076), then lcms2's XYZ float (1.0 = 1.0) */
			const float X = p[0] / 100.0f, Y = p[1] / 100.0f, Z = p[2] / 100.0f;
			xyz[0] = 1.047886F * X + 0.022919F * Y + -0.050216F * Z;
			xyz[1] = 0.029582F * X + 0.990484F * Y + -0.017079F * Z;
			xyz[2] = -0.009252F * X + 0.015073F * Y + 0.751678F * Z;
		}
	}
	if (J.out_thr >= 0) {
		for (int r = 0; r < J.out.bands; r++) {
			const float lin = (float) (J.out.model == MODEL_MATRIX
					? J.out.m[r * 3] * xyz[0] + J.out.m[r * 3 + 1] * xyz[1] + J.out.m[r * 3 + 2] * xyz[2]
					: xyz[1] / D50Y);
			/* thresholds 1 .. n - 1 ascend: count those <= lin */
			const float *thr = J.out.pool + J.out_thr + r * J.out_thr_n;
			int lo = 0, hi = J.out_thr_n - 1; /* the answer lies in [lo, hi] */
			while (lo < hi) {
				const int mid = (lo + hi + 1) >> 1;
				if (thr[mid] <= lin)
					lo = mid;
				else
					hi = mid - 1;
			}
			if (J.depth == 8)
				((uint8_t *) pout)[r] = (uint8_t) lo;
			else
				((uint16_t *) pout)[r] = (uint16_t) lo;
		}
		return;
	}
	side_from_xyz(J.out, xyz, dev);
	for (int i = 0; i < J.out.bands; i++)
		store_dev(pout, J.depth, i, dev[i]);
}

HD void
icc_pixel(const IccJob &J, const void *pin, void *pout)
{
	icc_colour(J, pin, pout);
	const int in_bands = J.mode == 1 ? 3 : J.in.bands;
	const int out_bands = J.mode == 0 ? 3 : J.out.bands;
	for (int e = 0; e < J.extra; e++) {
		double v = J.in_fmt == VB200_FORMAT_UCHAR ? (double) ((const uint8_t *) pin)[in_bands + e]
			: J.in_fmt == VB200_FORMAT_USHORT	  ? (double) ((const uint16_t *) pin)[in_bands + e]
												  : (double) ((const float *) pin)[in_bands + e];
		if (J.mode == MODE_XYZ_EXPORT) {
			/* vips_colour_build on the route's two float steps: sRGB (255) -> scRGB (1.0) -> XYZ (255) */
			v = (double) FADD_RN(FMUL_RN((float) (1.0 / 255.0), (float) v), 0.0f);
			v = (double) FADD_RN(FMUL_RN(255.0f, (float) v), 0.0f);
		}
		if (J.alpha_rescale) {
			const float scaled = J.alpha_a * (float) v + 0.0f;
			v = (double) scaled;
		}
		if (J.out_fmt == VB200_FORMAT_UCHAR) {
			const double m = 255.0 < v ? 255.0 : v; /* VIPS_CLIP with C's ?: (NaN -> 0) */
			((uint8_t *) pout)[out_bands + e] = (uint8_t) (0.0 > m ? 0.0 : m);
		}
		else if (J.out_fmt == VB200_FORMAT_USHORT) {
			const double m = 65535.0 < v ? 65535.0 : v;
			((uint16_t *) pout)[out_bands + e] = (uint16_t) (0.0 > m ? 0.0 : m);
		}
		else
			((float *) pout)[out_bands + e] = (float) v;
	}
}

} // namespace

} // namespace vb200

#endif
