/* icc.cu -- vips_icc_import / vips_icc_export / vips_icc_transform on the device (SURVEY 8a a20).
 *
 * reference: colour/icc_transform.c
 *   :294-470   vips_icc_build: pixel formats, cmsCreateTransform(in, fmt, out, fmt, intent, cmsFLAGS_NOCACHE)
 *   :813-945   import: device -> Lab16 (v4 encoding) or XYZ16 by lcms2, then decode_lab / decode_xyz to float
 *   :995-1117  export: PCS float (Lab, or XYZ through encode_xyz) -> device 8 / 16 bit by lcms2
 *   :1166-1220 transform: device -> device, one lcms2 transform
 *
 * The arithmetic of the reference lives inside lcms2 (not under /root/reference, no version pinned by
 * meson.build:444-447).  This is a from-specification ICC evaluator (ICC.1:2010 / ICC.1:2001-04):
 *   - RGB matrix/TRC profiles (rXYZ gXYZ bXYZ + curv / para TRCs), grey TRC profiles,
 *   - lut16 / lut8 (mft2 / mft1) and v4 lutAtoB / lutBtoA (mAB / mBA) A2Bn / B2An profiles, XYZ or Lab PCS,
 *   - relative colorimetric (the reference's default intent); perceptual / saturation where lcms2's
 *     black point compensation is the identity (matrix / grey profiles whose TRCs map 0 to 0);
 *   - absolute colorimetric on matrix / TRC profiles (the media-white scale of lcms2's ComputeAbsoluteIntent folds into
 *     the colorant matrix on the host, parse_side), and on any profile where that scale is the identity.
 * Absolute colorimetric of lut / grey profiles with a scale, black point compensation proper, device-link and
 * named-colour profiles return -1 ("keep the host path").
 *
 * PARITY: pinned to lcms2 2.18 (oracle/pylcms.py makes the reference's exact lcms2 calls) within a
 * tolerance, not bit for bit -- lcms2's integer transforms are table interpolations of this same
 * colorimetry.  tests/test_icc.py states the bounds (they are far inside the reference's own
 * dE < 6 / |diff| < 3).
 *
 * One source, two targets: the per-pixel evaluation below is __host__ __device__, the kernels call it
 * per thread and vb200_debug_icc_eval calls it on the CPU, so the CPU test-suite exercises the same code.
 */
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "vb200_internal.h"

namespace vb200 {

namespace {

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

/* ------------------------------------------------------------------ parsing (host) */

struct Blob {
	const unsigned char *d;
	size_t n;
	bool ok(size_t off, size_t len) const { return off <= n && len <= n - off; }
	unsigned u32(size_t o) const { return ((unsigned) d[o] << 24) | (d[o + 1] << 16) | (d[o + 2] << 8) | d[o + 3]; }
	unsigned u16(size_t o) const { return (d[o] << 8) | d[o + 1]; }
	double s15f16(size_t o) const { return (double) (int) u32(o) / 65536.0; }
};

bool
find_tag(const Blob &b, const char *sig, size_t *off, size_t *len)
{
	if (!b.ok(128, 4))
		return false;
	const unsigned nt = b.u32(128);
	for (unsigned i = 0; i < nt; i++) {
		const size_t e = 132 + 12 * (size_t) i;
		if (!b.ok(e, 12))
			return false;
		if (memcmp(b.d + e, sig, 4) == 0) {
			*off = b.u32(e + 4);
			*len = b.u32(e + 8);
			return b.ok(*off, *len) && *len >= 8;
		}
	}
	return false;
}

bool
parse_curve(const Blob &b, const char *sig, IccCurve *c, std::vector<float> &pool)
{
	size_t off, len;
	if (!find_tag(b, sig, &off, &len))
		return false;
	if (memcmp(b.d + off, "curv", 4) == 0) {
		if (len < 12)
			return false;
		const unsigned n = b.u32(off + 8);
		if (n == 0) {
			c->kind = CURVE_IDENTITY;
			return true;
		}
		if (n == 1) {
			if (!b.ok(off + 12, 2))
				return false; /* truncated 'curv' tag */
			c->kind = CURVE_PARA;
			c->ptype = 0;
			c->p[0] = b.u16(off + 12) / 256.0;
			return true;
		}
		if (!b.ok(off + 12, 2 * (size_t) n))
			return false;
		c->kind = CURVE_TABLE;
		c->n = (int) n;
		c->table_off = (int) pool.size();
		for (unsigned i = 0; i < n; i++)
			pool.push_back((float) (b.u16(off + 12 + 2 * i) / 65535.0));
		return true;
	}
	if (memcmp(b.d + off, "para", 4) == 0) {
		if (len < 12)
			return false;
		const int t = (int) b.u16(off + 8);
		static const int count[5] = {1, 3, 4, 5, 7};
		if (t < 0 || t > 4 || !b.ok(off + 12, 4 * (size_t) count[t]))
			return false;
		c->kind = CURVE_PARA;
		c->ptype = t;
		for (int i = 0; i < count[t]; i++)
			c->p[i] = b.s15f16(off + 12 + 4 * i);
		return true;
	}
	return false;
}

/* a curveType / parametricCurveType element inside another tag; *used = its length padded to 4 */
bool
parse_curve_at(const Blob &b, size_t off, IccCurve *c, std::vector<float> &pool, size_t *used)
{
	if (!b.ok(off, 12))
		return false;
	if (memcmp(b.d + off, "curv", 4) == 0) {
		const unsigned n = b.u32(off + 8);
		if (!b.ok(off + 12, 2 * (size_t) n))
			return false;
		*used = (12 + 2 * (size_t) n + 3) & ~(size_t) 3;
		if (n == 0)
			c->kind = CURVE_IDENTITY;
		else if (n == 1) {
			c->kind = CURVE_PARA;
			c->ptype = 0;
			c->p[0] = b.u16(off + 12) / 256.0;
		}
		else {
			c->kind = CURVE_TABLE;
			c->n = (int) n;
			c->table_off = (int) pool.size();
			for (unsigned i = 0; i < n; i++)
				pool.push_back((float) (b.u16(off + 12 + 2 * i) / 65535.0));
		}
		return true;
	}
	if (memcmp(b.d + off, "para", 4) == 0) {
		const int t = (int) b.u16(off + 8);
		static const int count[5] = {1, 3, 4, 5, 7};
		if (t < 0 || t > 4 || !b.ok(off + 12, 4 * (size_t) count[t]))
			return false;
		c->kind = CURVE_PARA;
		c->ptype = t;
		for (int i = 0; i < count[t]; i++)
			c->p[i] = b.s15f16(off + 12 + 4 * i);
		*used = 12 + 4 * (size_t) count[t];
		return true;
	}
	return false;
}

bool
parse_mab(const Blob &b, const char *sig, bool to_pcs, IccMab *m, std::vector<float> &pool)
{
	size_t off, len;
	if (!find_tag(b, sig, &off, &len) || len < 32)
		return false;
	if (memcmp(b.d + off, to_pcs ? "mAB " : "mBA ", 4) != 0)
		return false;
	m->in_ch = b.d[off + 8];
	m->out_ch = b.d[off + 9];
	if (m->in_ch < 1 || m->in_ch > 4 || m->out_ch < 1 || m->out_ch > 4)
		return false;
	const size_t ob = b.u32(off + 12), omat = b.u32(off + 16), om = b.u32(off + 20), oc = b.u32(off + 24), oa = b.u32(off + 28);
	/* B curves are on the PCS side, A curves on the device side */
	const int nb = to_pcs ? m->out_ch : m->in_ch, na = to_pcs ? m->in_ch : m->out_ch;
	if (!ob)
		return false;
	auto curves = [&](size_t o, int n, IccCurve *c) {
		size_t p = off + o;
		for (int i = 0; i < n; i++) {
			size_t used = 0;
			if (!parse_curve_at(b, p, &c[i], pool, &used))
				return false;
			p += used;
		}
		return true;
	};
	if (!curves(ob, nb, m->b))
		return false;
	if (omat) {
		if (nb != 3 || !b.ok(off + omat, 48))
			return false;
		for (int i = 0; i < 12; i++)
			m->mat[i] = b.s15f16(off + omat + 4 * i);
		m->has_matrix = 1;
	}
	if (om) {
		if (nb != 3 || !curves(om, 3, m->m))
			return false;
		m->has_m = 1;
	}
	if (oa) {
		if (!curves(oa, na, m->a))
			return false;
		m->has_a = 1;
	}
	if (oc) {
		if (!b.ok(off + oc, 20))
			return false;
		size_t nodes = 1;
		for (int i = 0; i < m->in_ch; i++) {
			m->grid[i] = b.d[off + oc + i];
			if (m->grid[i] < 2)
				return false;
			nodes *= (size_t) m->grid[i];
		}
		const int prec = b.d[off + oc + 16];
		if (prec != 1 && prec != 2)
			return false;
		const size_t count = nodes * m->out_ch;
		if (!b.ok(off + oc + 20, count * prec))
			return false;
		m->clut_off = (int) pool.size();
		for (size_t i = 0; i < count; i++)
			pool.push_back(prec == 2 ? (float) (b.u16(off + oc + 20 + 2 * i) / 65535.0) : (float) (b.d[off + oc + 20 + i] / 255.0));
		m->has_clut = 1;
	}
	else if (m->in_ch != m->out_ch)
		return false;
	return true;
}

bool
parse_xyz(const Blob &b, const char *sig, double *xyz)
{
	size_t off, len;
	if (!find_tag(b, sig, &off, &len) || len < 20 || memcmp(b.d + off, "XYZ ", 4) != 0)
		return false;
	for (int i = 0; i < 3; i++)
		xyz[i] = b.s15f16(off + 8 + 4 * i);
	return true;
}

bool
parse_lut(const Blob &b, const char *sig, IccLut *l, std::vector<float> &pool)
{
	size_t off, len;
	if (!find_tag(b, sig, &off, &len) || len < 48)
		return false;
	const bool is16 = memcmp(b.d + off, "mft2", 4) == 0, is8 = memcmp(b.d + off, "mft1", 4) == 0;
	if (!is16 && !is8)
		return false; /* mAB / mBA (v4): not handled */
	l->in_ch = b.d[off + 8];
	l->out_ch = b.d[off + 9];
	l->grid = b.d[off + 10];
	if (l->in_ch < 1 || l->in_ch > 4 || l->out_ch < 1 || l->out_ch > 4 || l->grid < 2)
		return false;
	l->has_matrix = 0;
	for (int i = 0; i < 9; i++) {
		l->m[i] = b.s15f16(off + 12 + 4 * i);
		if (fabs(l->m[i] - (i % 4 == 0 ? 1.0 : 0.0)) > 1e-6)
			l->has_matrix = 1;
	}
	size_t p = off + 48;
	if (is16) {
		if (!b.ok(p, 4))
			return false; /* truncated 'mft2' tag */
		l->n_in = (int) b.u16(p);
		l->n_out = (int) b.u16(p + 2);
		p += 4;
	}
	else
		l->n_in = l->n_out = 256;
	if (l->n_in < 2 || l->n_out < 2)
		return false;
	size_t clut_n = (size_t) l->out_ch;
	for (int i = 0; i < l->in_ch; i++)
		clut_n *= (size_t) l->grid;
	const size_t es = is16 ? 2 : 1;
	const size_t total = ((size_t) l->in_ch * l->n_in + clut_n + (size_t) l->out_ch * l->n_out) * es;
	if (!b.ok(p, total))
		return false;
	const double scale = is16 ? 65535.0 : 255.0;
	auto rd = [&](size_t count) {
		const int at = (int) pool.size();
		for (size_t i = 0; i < count; i++, p += es)
			pool.push_back((float) ((is16 ? b.u16(p) : b.d[p]) / scale));
		return at;
	};
	l->in_off = rd((size_t) l->in_ch * l->n_in);
	l->clut_off = rd(clut_n);
	l->out_off = rd((size_t) l->out_ch * l->n_out);
	return true;
}

bool
invert3(const double *m, double *inv)
{
	const double det = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
	if (fabs(det) < 1e-12)
		return false;
	inv[0] = (m[4] * m[8] - m[5] * m[7]) / det;
	inv[1] = (m[2] * m[7] - m[1] * m[8]) / det;
	inv[2] = (m[1] * m[5] - m[2] * m[4]) / det;
	inv[3] = (m[5] * m[6] - m[3] * m[8]) / det;
	inv[4] = (m[0] * m[8] - m[2] * m[6]) / det;
	inv[5] = (m[2] * m[3] - m[0] * m[5]) / det;
	inv[6] = (m[3] * m[7] - m[4] * m[6]) / det;
	inv[7] = (m[1] * m[6] - m[0] * m[7]) / det;
	inv[8] = (m[0] * m[4] - m[1] * m[3]) / det;
	return true;
}

int black_is_zero(const char *domain, const IccSide *s, const std::vector<float> &pool, int intent);

/* One direction of one profile: to_pcs (A2B / forward matrix) or from_pcs (B2A / inverse matrix). */
int
parse_side(const char *domain, const void *data, size_t len, int intent, bool to_pcs, bool other_is_lab4_d65, IccSide *s,
	std::vector<float> &pool)
{
	const Blob b{(const unsigned char *) data, len};
	if (!data || len < 132 || b.u32(0) > len || memcmp(b.d + 36, "acsp", 4) != 0) {
		error(domain, "not an ICC profile");
		return -1;
	}
	if (intent < 0 || intent > 3) {
		error(domain, "rendering intent %d not supported on the device path", intent);
		return -1;
	}
	/* Absolute colorimetric (lcms2 cmscnvrt.c ComputeAbsoluteIntent at its default adaptation state 1.0): the relative
	 * transform with PCS XYZ scaled by media white / D50 on the way in and D50 / media white on the way out.  The media
	 * white is the wtpt tag, D50 when it is absent or for a v2 display-class profile (cmsio1.c _cmsReadMediaWhitePoint).
	 * The profile at the other end is another device profile (vips_icc_transform: both sides scale against D50 and the
	 * D50s cancel), the XYZ PCS profile (cmsCreateXYZProfile: D50), or the Lab PCS profile the reference makes with
	 * cmsCreateLab4Profile(cmsWhitePointFromTemp(6504 K)) (icc_transform.c:355-362), whose media white in lcms2 2.18 is
	 * that D65 white -- so with the Lab PCS absolute colorimetric scales even a D50 profile.
	 * For a matrix / TRC profile the scale folds into the colorant matrix right here, on the host; where it is the
	 * identity the intent is the relative one; anything else (a lut or grey profile with another media white) would need
	 * the scale inside the evaluator and is declined.
	 */
	double white_scale[3] = {1.0, 1.0, 1.0};
	bool scaled = false;
	if (intent == 3) {
		double wp[3] = {0.9642, 1.0, 0.8249}, other[3] = {0.9642, 1.0, 0.8249}; /* cmsD50X / Y / Z */
		const bool v2_display = b.u32(8) < 0x04000000u && memcmp(b.d + 12, "mntr", 4) == 0;
		double tag[3];
		if (!v2_display && parse_xyz(b, "wtpt", tag))
			memcpy(wp, tag, sizeof(wp));
		if (other_is_lab4_d65) {
			/* cmsWhitePointFromTemp(6504), cmswtpnt.c (4000 .. 7000 K branch), then xyY -> XYZ at Y = 1 */
			const double T = 6504.0, T2 = T * T, T3 = T2 * T;
			const double x = -4.6070 * (1E9 / T3) + 2.9678 * (1E6 / T2) + 0.09911 * (1E3 / T) + 0.244063;
			const double y = -3.000 * (x * x) + 2.870 * x - 0.275;
			other[0] = x / y;
			other[1] = 1.0;
			other[2] = (1.0 - x - y) / y;
		}
		for (int i = 0; i < 3; i++) {
			if (!(wp[i] > 0.0)) {
				error(domain, "bad media white point");
				return -1;
			}
			white_scale[i] = to_pcs ? wp[i] / other[i] : other[i] / wp[i];
			scaled = scaled || white_scale[i] != 1.0;
		}
		intent = 1;
	}
	const unsigned char *cs = b.d + 16, *pcs = b.d + 20;
	s->pcs_lab = memcmp(pcs, "Lab ", 4) == 0;
	if (!s->pcs_lab && memcmp(pcs, "XYZ ", 4) != 0) {
		error(domain, "unsupported profile connection space");
		return -1;
	}
	if (memcmp(cs, "RGB ", 4) == 0)
		s->bands = 3;
	else if (memcmp(cs, "GRAY", 4) == 0)
		s->bands = 1;
	else if (memcmp(cs, "CMYK", 4) == 0)
		s->bands = 4;
	else {
		error(domain, "unimplemented device colour space %.4s on the device path", cs);
		return -1;
	}
	/* LUT tags win over matrix/TRC when present (ICC.1 9.2, lcms2 does the same) */
	static const char *a2b[3] = {"A2B0", "A2B1", "A2B2"}, *b2a[3] = {"B2A0", "B2A1", "B2A2"};
	const char *const *tags = to_pcs ? a2b : b2a;
	size_t off, tl;
	const char *want = find_tag(b, tags[intent], &off, &tl) ? tags[intent] : (find_tag(b, tags[0], &off, &tl) ? tags[0] : nullptr);
	s->to_pcs = to_pcs;
	if (want && scaled) {
		error(domain, "absolute colorimetric intent of a lut-based profile whose media white is not D50 is not supported on the device path");
		return -1;
	}
	if (want && intent != 1) {
		/* perceptual / saturation against the v4 Lab / XYZ PCS profiles make lcms2 turn black point compensation
		 * on (cmscnvrt.c); for a lut profile that needs its black point, which is not evaluated here
		 */
		error(domain, "rendering intent %d of a lut-based profile is not supported on the device path", intent);
		return -1;
	}
	if (want && memcmp(b.d + off, to_pcs ? "mAB " : "mBA ", 4) == 0) {
		if (!parse_mab(b, want, to_pcs, &s->mab, pool)) {
			error(domain, "malformed %s tag", want);
			return -1;
		}
		if ((to_pcs ? s->mab.in_ch : s->mab.out_ch) != s->bands || (to_pcs ? s->mab.out_ch : s->mab.in_ch) != 3) {
			error(domain, "lut channel counts do not match the profile header");
			return -1;
		}
		s->mab.trilinear = !to_pcs && s->pcs_lab;
		s->model = MODEL_MAB;
		return 0;
	}
	if (want) {
		if (!parse_lut(b, want, &s->lut, pool)) {
			error(domain, "%s is neither lut8 / lut16 nor lutAtoB / lutBtoA", want);
			return -1;
		}
		if ((to_pcs ? s->lut.in_ch : s->lut.out_ch) != s->bands || (to_pcs ? s->lut.out_ch : s->lut.in_ch) != 3) {
			error(domain, "lut channel counts do not match the profile header");
			return -1;
		}
		s->lut.trilinear = !to_pcs && s->pcs_lab;
		s->model = MODEL_LUT;
		return 0;
	}
	if (s->pcs_lab) {
		error(domain, "matrix/TRC profile with a Lab PCS");
		return -1;
	}
	if (s->bands == 1) {
		if (!parse_curve(b, "kTRC", &s->curve[0], pool)) {
			error(domain, "grey profile without a usable kTRC");
			return -1;
		}
		if (scaled) {
			error(domain, "absolute colorimetric intent of a grey profile whose media white is not D50 is not supported on the device path");
			return -1;
		}
		s->model = MODEL_GREY;
		return black_is_zero(domain, s, pool, intent);
	}
	if (s->bands == 3) {
		double col[3][3];
		static const char *xyz[3] = {"rXYZ", "gXYZ", "bXYZ"}, *trc[3] = {"rTRC", "gTRC", "bTRC"};
		for (int i = 0; i < 3; i++)
			if (!parse_xyz(b, xyz[i], col[i]) || !parse_curve(b, trc[i], &s->curve[i], pool)) {
				error(domain, "RGB profile without usable %s / %s", xyz[i], trc[i]);
				return -1;
			}
		double m[9];
		for (int r = 0; r < 3; r++)
			for (int c = 0; c < 3; c++)
				m[r * 3 + c] = col[c][r];
		if (to_pcs) {
			for (int r = 0; r < 3; r++) /* XYZ_abs = diag(white / D50) M lin */
				for (int c = 0; c < 3; c++)
					s->m[r * 3 + c] = white_scale[r] * m[r * 3 + c];
		}
		else {
			if (!invert3(m, s->m)) {
				error(domain, "singular colorant matrix");
				return -1;
			}
			for (int r = 0; r < 3; r++) /* lin = M^-1 diag(D50 / white) XYZ_abs */
				for (int c = 0; c < 3; c++)
					s->m[r * 3 + c] *= white_scale[c];
		}
		s->model = MODEL_MATRIX;
		return black_is_zero(domain, s, pool, intent);
	}
	error(domain, "profile has neither lut nor matrix/TRC tags usable on the device path");
	return -1;
}

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

/* Perceptual and saturation intents of a matrix / grey profile: lcms2 applies black point compensation
 * between the profile's black and the PCS profile's (zero); when the TRCs map 0 to 0 the profile's black
 * is XYZ 0 too, the compensation is the identity, and the transform equals the relative colorimetric
 * one bit for bit (checked against lcms2 in tests/test_icc.py).  Anything else is declined.
 */
int
black_is_zero(const char *domain, const IccSide *s, const std::vector<float> &pool, int intent)
{
	if (intent == 1)
		return 0;
	const int n = s->model == MODEL_GREY ? 1 : 3;
	for (int i = 0; i < n; i++)
		if (curve_fwd(s->curve[i], pool.data(), 0.0) != 0.0) {
			error(domain, "rendering intent %d with a non-zero black point is not supported on the device path", intent);
			return -1;
		}
	return 0;
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

/* one pixel; pin / pout point at the pixel's first element */
HD void
icc_colour(const IccJob &J, const void *pin, void *pout)
{
	double dev[4] = {0, 0, 0, 0}, xyz[3] = {0, 0, 0};
	if (J.mode == 0 || J.mode == 2) {
		if (J.in_tab >= 0) {
			double lin[3] = {0, 0, 0};
			for (int i = 0; i < J.in.bands; i++) {
				const int code = J.in_fmt == VB200_FORMAT_UCHAR ? ((const uint8_t *) pin)[i] : ((const uint16_t *) pin)[i];
				lin[i] = J.in.pool[J.in_tab + i * J.in_tab_n + code];
			}
			if (J.in.model == MODEL_MATRIX)
				for (int r = 0; r < 3; r++)
					xyz[r] = J.in.m[r * 3] * lin[0] + J.in.m[r * 3 + 1] * lin[1] + J.in.m[r * 3 + 2] * lin[2];
			else {
				xyz[0] = lin[0] * D50X;
				xyz[1] = lin[0] * D50Y;
				xyz[2] = lin[0] * D50Z;
			}
		}
		else {
			for (int i = 0; i < J.in.bands; i++)
				dev[i] = load_dev(pin, J.in_fmt, i);
			side_to_xyz(J.in, dev, xyz);
		}
	}
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
		else {
			/* XYZ16 (1.0 = 0x8000), then decode_xyz (:879-909): float arithmetic, Bradford D50 -> D65 */
			const float X = (float) (sat16(xyz[0] * 32768.0) / 32768.0) * 100.0f;
			const float Y = (float) (sat16(xyz[1] * 32768.0) / 32768.0) * 100.0f;
			const float Z = (float) (sat16(xyz[2] * 32768.0) / 32768.0) * 100.0f;
			q[0] = 0.955513F * X + -0.023073F * Y + 0.063309F * Z;
			q[1] = -0.028325F * X + 1.009942F * Y + 0.021055F * Z;
			q[2] = 0.012329F * X + -0.020536F * Y + 1.330714F * Z;
		}
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
			/* encode_xyz (:1050-1076), then lcms2's XYZ float (1.0 = 1.0) */
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

static_assert(sizeof(IccJob) <= 4096, "IccJob travels as a kernel parameter");

template <bool LOOP>
__global__ void __launch_bounds__(256)
icc_kernel(const __grid_constant__ IccJob J, const char *__restrict__ in, size_t in_bpl, size_t in_ps, char *__restrict__ out,
	size_t out_bpl, size_t out_ps, int w, int h)
{
	const int x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= w)
		return;
	int y = blockIdx.y;
	do
		icc_pixel(J, in + (size_t) y * in_bpl + (size_t) x * in_ps, out + (size_t) y * out_bpl + (size_t) x * out_ps);
	while (LOOP && (y += gridDim.y) < h);
}

struct JobSpec {
	int mode, intent, pcs_xyz, depth;
	const void *pa;
	size_t la;
	const void *pb;
	size_t lb;
};

int
build_job(const char *domain, const JobSpec &sp, int in_fmt, int in_bands, int in_type, IccJob *J, std::vector<float> &pool,
	int *out_bands, int *out_fmt, int *out_type)
{
	memset((void *) J, 0, sizeof(*J));
	J->mode = sp.mode;
	J->pcs_xyz = sp.pcs_xyz;
	J->in_fmt = in_fmt;
	J->depth = sp.depth;
	if (sp.depth != 8 && sp.depth != 16) {
		error(domain, "depth must be 8 or 16");
		return -1;
	}
	if (sp.mode == 0 || sp.mode == 2) {
		if (parse_side(domain, sp.pa, sp.la, sp.intent, true, sp.mode == 0 && !sp.pcs_xyz, &J->in, pool))
			return -1;
		if (in_fmt != VB200_FORMAT_UCHAR && in_fmt != VB200_FORMAT_USHORT && in_fmt != VB200_FORMAT_FLOAT) {
			error(domain, "band format %d not supported on the device path", in_fmt);
			return -1;
		}
		if (in_bands < J->in.bands) {
			error(domain, "image has %d bands, the input profile wants %d", in_bands, J->in.bands);
			return -1;
		}
		J->extra = in_bands - J->in.bands;
	}
	if (sp.mode == MODE_XYZ_EXPORT) {
		if (in_fmt != VB200_FORMAT_UCHAR || in_bands < 1) {
			error(domain, "the XYZ export of a thumbnail wants an 8-bit image");
			return -1;
		}
		J->pcs_xyz = 1;
		J->in.bands = in_bands < 3 ? 1 : 3; /* B_W or sRGB, as the thumbnail's processing space */
		J->extra = in_bands - J->in.bands;
		/* the 8-bit sRGB2scRGB table, calcul_tables (LabQ2sRGB.c:130-159) as colour.cu builds it */
		J->in_tab = (int) pool.size();
		J->in_tab_n = 256;
		for (int i = 0; i < 256; i++) {
			const float f = (float) i / 255;
			pool.push_back(f <= 0.04045 ? f / 12.92F : powf((f + 0.055F) / (1 + 0.055F), 2.4F));
		}
		in_type = VB200_INTERPRETATION_XYZ; /* the export's input; the route's own alpha steps are in icc_pixel */
	}
	if (sp.mode == 1 || sp.mode == 2 || sp.mode == MODE_XYZ_EXPORT) {
		const void *p = sp.mode == 2 ? sp.pb : sp.pa;
		const size_t l = sp.mode == 2 ? sp.lb : sp.la;
		if (parse_side(domain, p, l, sp.intent, false, sp.mode == 1 && !sp.pcs_xyz, &J->out, pool))
			return -1;
	}
	if (sp.mode == 1) {
		if (in_fmt != VB200_FORMAT_FLOAT || in_bands < 3) {
			error(domain, "export wants a float PCS image of 3 bands (+ extra bands)");
			return -1;
		}
		J->extra = in_bands - 3;
	}
	if (sp.mode == 0) {
		*out_bands = 3;
		*out_fmt = VB200_FORMAT_FLOAT;
		*out_type = sp.pcs_xyz ? VB200_INTERPRETATION_XYZ : VB200_INTERPRETATION_LAB;
	}
	else {
		*out_bands = J->out.bands;
		*out_fmt = sp.depth == 8 ? VB200_FORMAT_UCHAR : VB200_FORMAT_USHORT;
		/* icc_transform.c:374-433 */
		*out_type = J->out.bands == 1 ? (sp.depth == 8 ? VB200_INTERPRETATION_B_W : VB200_INTERPRETATION_GREY16)
			: J->out.bands == 3		  ? (sp.depth == 8 ? VB200_INTERPRETATION_sRGB : VB200_INTERPRETATION_RGB16)
									  : VB200_INTERPRETATION_CMYK;
	}
	{
		/* the extra bands: colour.c:252-291 */
		const double before = interpretation_max_alpha(in_type), after = interpretation_max_alpha(*out_type);
		J->alpha_rescale = before != after;
		J->alpha_a = (float) (after / before);
		J->out_fmt = *out_fmt;
		*out_bands += J->extra;
	}
	/* tabulate the TRCs for integer codes (the curves read `pool` themselves: evaluate against the host copy) */
	J->out_thr = -1;
	if (sp.mode != MODE_XYZ_EXPORT)
		J->in_tab = -1;
	const bool tabulate = getenv("VB200_NO_ICC_TABLES") == nullptr;
	if (tabulate && (sp.mode == 0 || sp.mode == 2) && (J->in.model == MODEL_MATRIX || J->in.model == MODEL_GREY) &&
		(in_fmt == VB200_FORMAT_UCHAR || in_fmt == VB200_FORMAT_USHORT)) {
		const int n = in_fmt == VB200_FORMAT_UCHAR ? 256 : 65536;
		std::vector<float> tab((size_t) J->in.bands * n);
		for (int c = 0; c < J->in.bands; c++)
			for (int i = 0; i < n; i++)
				tab[(size_t) c * n + i] = (float) curve_fwd(J->in.curve[c], pool.data(), (double) i / (n - 1));
		J->in_tab = (int) pool.size();
		J->in_tab_n = n;
		pool.insert(pool.end(), tab.begin(), tab.end());
	}
	if (tabulate && sp.mode != MODE_IMPORT && (J->out.model == MODEL_MATRIX || J->out.model == MODEL_GREY)) {
		const int n = sp.depth == 8 ? 256 : 65536;
		std::vector<float> thr((size_t) J->out.bands * n);
		bool monotone = true;
		for (int c = 0; c < J->out.bands; c++) {
			thr[(size_t) c * n] = -3.0e38f; /* code 0 is always reached */
			for (int k = 1; k < n; k++) {
				thr[(size_t) c * n + k] = (float) curve_fwd(J->out.curve[c], pool.data(), (k - 0.5) / (n - 1));
				if (thr[(size_t) c * n + k] < thr[(size_t) c * n + k - 1])
					monotone = false;
			}
		}
		if (monotone) {
			J->out_thr = (int) pool.size();
			J->out_thr_n = n;
			pool.insert(pool.end(), thr.begin(), thr.end());
		}
	}
	return 0;
}

int
run_icc(const char *domain, const VB200Image *in, VB200Image *out, const JobSpec &sp)
{
	if (!in || !out) {
		error(domain, "null argument");
		return -1;
	}
	if (ensure_init(domain))
		return -1;
	cudaStream_t s = current_stream();
	IccJob J;
	std::vector<float> pool;
	int ob, of, ot;
	if (build_job(domain, sp, in->BandFmt, in->Bands, in->Type, &J, pool, &ob, &of, &ot))
		return -1;
	DevImage din, dout;
	if (to_device(domain, in, &din, s))
		return -1;
	float *dpool = nullptr;
	int rc = 0;
	if (!pool.empty()) {
		rc = dev_alloc(domain, (void **) &dpool, pool.size() * sizeof(float), s);
		if (!rc && cudaMemcpyAsync(dpool, pool.data(), pool.size() * sizeof(float), cudaMemcpyHostToDevice, s) != cudaSuccess)
			rc = -1;
	}
	J.in.pool = J.out.pool = dpool;
	preset_output(&dout, in, out, (size_t) din.w * ob * format_sizeof(of), din.h); /* the exact result extent (grey -> Lab widens 1 band to 3 floats) */
	if (!rc)
		rc = dev_image_new(domain, &dout, din.w, din.h, ob, of, ot, s);
	if (!rc) {
		const dim3 grid = row_grid(din.w, din.h);
		(rows_loop(din.h) ? icc_kernel<true> : icc_kernel<false>)<<<grid, 256, 0, s>>>(J, (const char *) din.data, din.bpl, format_sizeof(din.fmt) * din.bands, (char *) dout.data,
			dout.bpl, format_sizeof(of) * ob, din.w, din.h);
		const cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess)
			rc = cuda_fail(domain, e, "icc_kernel");
		else
			count_launch();
	}
	if (!rc) {
		/* the pool is read by the kernel: free it stream-ordered, after the launch */
		rc = deliver(domain, &dout, in, out, s);
	}
	if (dpool)
		dev_free(dpool, s);
	dev_image_release(&din, s);
	return rc;
}

/* ------------------------------------------------------------------ the ICC stage of the thumbnail plan */

/* What cmsOpenProfileFromMem (lcms2 2.18, cmsio0.c _cmsReadHeader) accepts: a 128-byte header with the 'acsp' magic, a
 * version below 5.0 after _validatedVersion's clamp, a known device class (or 0), at most 100 tags whose directory can be read
 * and no tag signature twice.  Tags whose offset + size fall outside the header's size (or the blob) are dropped from the
 * directory, not refused.  *tags receives the signatures that stay.  No tag contents are read: lcms2 reads them lazily.
 */
bool
lcms_would_open(const unsigned char *d, size_t n, std::vector<unsigned> *tags)
{
	tags->clear();
	if (!d || n < 132)
		return false;
	const Blob b{d, n};
	if (memcmp(d + 36, "acsp", 4) != 0)
		return false;
	unsigned char ver[4] = {d[8], d[9], 0, 0};
	if (ver[0] > 0x09)
		ver[0] = 0x09;
	unsigned char hi = ver[1] & 0xf0, lo = ver[1] & 0x0f;
	ver[1] = (unsigned char) ((hi > 0x90 ? 0x90 : hi) | (lo > 0x09 ? 0x09 : lo));
	const unsigned version = ((unsigned) ver[0] << 24) | ((unsigned) ver[1] << 16);
	if (version > 0x5000000u)
		return false;
	/* validDeviceClass: the ICC classes, or 0 (what older lcms versions wrote) */
	static const char *classes[] = {"scnr", "mntr", "prtr", "link", "abst", "spac", "nmcl", "cenc", "mid ", "mlnk", "mvis", "\0\0\0\0"};
	bool known = false;
	for (const char *c : classes)
		known = known || memcmp(d + 12, c, 4) == 0;
	if (!known)
		return false;
	size_t header_size = b.u32(0);
	if (header_size >= n)
		header_size = n;
	const unsigned count = b.u32(128);
	if (count > 100 || !b.ok(132, 12 * (size_t) count))
		return false;
	for (unsigned i = 0; i < count; i++) {
		const size_t e = 132 + 12 * (size_t) i;
		const unsigned sig = b.u32(e), off = b.u32(e + 4), size = b.u32(e + 8);
		if (size == 0 || off == 0)
			continue;
		if ((uint64_t) off + size > header_size || off + size < off) /* lcms2 adds in 32 bits */
			continue;
		for (unsigned t : *tags)
			if (t == sig)
				return false; /* "Duplicate tag found" */
		tags->push_back(sig);
	}
	return true;
}

/* vips_icc_info (icc_transform.c:233-260): the profile colour spaces the reference handles, with their band counts */
int
icc_space_bands(const unsigned char *d)
{
	static const struct {
		const char *sig;
		int bands;
	} table[] = {{"GRAY", 1}, {"RGB ", 3}, {"Lab ", 3}, {"XYZ ", 3}, {"CMYK", 4}, {"4CLR", 4}, {"5CLR", 5}, {"6CLR", 6}, {"7CLR", 7},
		{"8CLR", 8}, {"9CLR", 9}, {"ACLR", 10}, {"BCLR", 11}, {"CCLR", 12}};
	for (const auto &e : table)
		if (memcmp(d + 16, e.sig, 4) == 0)
			return e.bands;
	return 0;
}

bool
has_tag(const std::vector<unsigned> &tags, const char *sig)
{
	const unsigned s = ((unsigned) (unsigned char) sig[0] << 24) | ((unsigned char) sig[1] << 16) | ((unsigned char) sig[2] << 8) |
		(unsigned char) sig[3];
	for (unsigned t : tags)
		if (t == s)
			return true;
	return false;
}

/* cmsIsIntentSupported (cmsio1.c): a lut tag for the intent in that direction, or a matrix / shaper profile */
bool
intent_supported(const unsigned char *d, const std::vector<unsigned> &tags, int intent, bool input)
{
	static const char *a2b[4] = {"A2B0", "A2B1", "A2B2", "A2B1"}, *b2a[4] = {"B2A0", "B2A1", "B2A2", "B2A1"};
	if (memcmp(d + 12, "link", 4) == 0) {
		if ((int) Blob{d, 128}.u32(64) == intent) /* cmsIsCLUT: a device link supports its header's intent */
			return true;
	}
	else if (intent >= 0 && intent <= 3 && has_tag(tags, (input ? a2b : b2a)[intent]))
		return true;
	if (memcmp(d + 16, "GRAY", 4) == 0)
		return has_tag(tags, "kTRC");
	if (memcmp(d + 16, "RGB ", 4) == 0)
		return has_tag(tags, "rXYZ") && has_tag(tags, "gXYZ") && has_tag(tags, "bXYZ") && has_tag(tags, "rTRC") && has_tag(tags, "gTRC") &&
			has_tag(tags, "bTRC");
	return false;
}

enum { PROFILE_USABLE = 0, PROFILE_UNUSABLE = 1, PROFILE_OTHER_INTENT = 2 };

/* vips_icc_load_profile_blob (icc_transform.c:581-652) for an input profile of an image whose interpretation wants
 * `want_bands`: PROFILE_UNUSABLE where the reference drops the profile and tries the next one; PROFILE_OTHER_INTENT where
 * it would keep the profile with the header's intent in place of the one asked for
 */
int
classify_input_profile(const void *p, size_t len, int want_bands, int intent)
{
	const unsigned char *d = (const unsigned char *) p;
	std::vector<unsigned> tags;
	if (!lcms_would_open(d, len, &tags))
		return PROFILE_UNUSABLE;
	int selected = intent;
	if (!intent_supported(d, tags, intent, true)) {
		const unsigned header_intent = Blob{d, len}.u32(64);
		if (header_intent > 3)
			return PROFILE_UNUSABLE;
		selected = (int) header_intent;
	}
	const int bands = icc_space_bands(d);
	if (bands == 0 || bands != want_bands)
		return PROFILE_UNUSABLE;
	if (!intent_supported(d, tags, selected, true))
		return PROFILE_UNUSABLE;
	return selected == intent ? PROFILE_USABLE : PROFILE_OTHER_INTENT;
}

struct IccProfileRef {
	const void *data;
	size_t len;
};

/* vips_icc_set_import (icc_transform.c:692-752) for one frame of a thumbnail: the embedded profile, then input_profile,
 * then the built-in profile for the frame's interpretation.  Returns MODE_TRANSFORM with *use = the profile, MODE_XYZ_EXPORT
 * when the frame has neither an embedded profile nor input_profile (thumbnail.c:957-970), or -1.  *source: 0 embedded,
 * 1 input_profile, 2 built-in.
 */
int
select_input_profile(const char *domain, int frame, const VB200ThumbnailIcc &icc, int bands, const void *embedded, size_t embedded_len,
	IccProfileRef *use, int *source)
{
	const bool has_embedded = embedded && embedded_len > 0;
	if (!has_embedded && !icc.input_profile)
		return MODE_XYZ_EXPORT;
	const bool grey = bands < 3;
	const IccProfileRef candidates[3] = {{has_embedded ? embedded : nullptr, embedded_len}, {icc.input_profile, icc.input_len},
		{grey ? icc.builtin_grey : icc.builtin_rgb, grey ? icc.builtin_grey_len : icc.builtin_rgb_len}};
	for (int k = 0; k < 3; k++) {
		if (!candidates[k].data) {
			if (k == 2) {
				error(domain, "frame %d: no usable embedded or input profile, and no built-in %s profile was passed", frame,
					grey ? "grey" : "RGB");
				return -1;
			}
			continue;
		}
		const int c = classify_input_profile(candidates[k].data, candidates[k].len, grey ? 1 : 3, icc.intent);
		if (c == PROFILE_UNUSABLE)
			continue;
		if (c == PROFILE_OTHER_INTENT) {
			error(domain, "frame %d: the input profile does not support rendering intent %d: its header intent is not supported on the "
				"device path", frame, icc.intent);
			return -1;
		}
		*use = candidates[k];
		*source = k;
		return MODE_TRANSFORM;
	}
	error(domain, "frame %d: unable to load or find any compatible input profile", frame);
	return -1;
}

/* One launch per chunk of frames, whatever profiles they carry: frame f runs jobs[job_of[f]].  A CTA serves one frame,
 * copies that frame's job into shared memory once and walks the frame's pixels.
 */
__global__ void __launch_bounds__(256)
icc_frames_kernel(const IccJob *__restrict__ jobs, const int *__restrict__ job_of, const uint8_t *__restrict__ in, size_t in_stride,
	int in_ps, uint8_t *__restrict__ out, size_t out_stride, int out_ps, size_t pixels)
{
	__shared__ __align__(16) unsigned char smem[sizeof(IccJob)];
	const int f = blockIdx.y;
	const unsigned *src = (const unsigned *) (jobs + job_of[f]);
	for (int i = threadIdx.x; i < (int) (sizeof(IccJob) / 4); i += blockDim.x)
		((unsigned *) smem)[i] = src[i];
	__syncthreads();
	const IccJob &J = *(const IccJob *) smem;
	const uint8_t *fin = in + (size_t) f * in_stride;
	uint8_t *fout = out + (size_t) f * out_stride;
	for (size_t p = (size_t) blockIdx.x * blockDim.x + threadIdx.x; p < pixels; p += (size_t) gridDim.x * blockDim.x)
		icc_pixel(J, fin + p * in_ps, fout + p * out_ps);
}
static_assert(sizeof(IccJob) % 4 == 0, "IccJob is copied to shared memory in words");

uint64_t
fnv1a64(const void *p, size_t n)
{
	const unsigned char *d = (const unsigned char *) p;
	uint64_t h = 1469598103934665603ull;
	for (size_t i = 0; i < n; i++)
		h = (h ^ d[i]) * 1099511628211ull;
	return h;
}

} // namespace

/* A parsed and tabulated job on the device, keyed by the input profile's bytes (none: branch X) */
struct IccCacheEntry {
	int mode = 0;
	uint64_t hash = 0;
	std::vector<unsigned char> bytes;
	IccJob job;
	float *dpool = nullptr;
	/* one event per stream that launched a kernel reading dpool, recorded after its latest such launch: the host pump runs
	 * its slices on several streams, and an eviction waits for all of them
	 */
	std::vector<std::pair<cudaStream_t, cudaEvent_t>> used;
	uint64_t tick = 0;
};

struct IccStage {
	static constexpr size_t kCacheEntries = 16;
	std::mutex lock;
	std::vector<unsigned char> input, output, builtin_rgb, builtin_grey;
	VB200ThumbnailIcc icc{}; /* pointers into the copies above */
	int bands = 0, out_bands = 0;
	std::vector<IccCacheEntry *> cache;
	uint64_t tick = 0;
};

namespace {

void
entry_free(IccCacheEntry *e)
{
	for (auto &u : e->used)
		cudaEventSynchronize(u.second);
	if (e->dpool)
		cudaFree(e->dpool);
	for (auto &u : e->used)
		cudaEventDestroy(u.second);
	delete e;
}

int
stage_job_spec(const IccStage &st, int mode, const IccProfileRef &in, JobSpec *sp)
{
	*sp = JobSpec{mode, st.icc.intent, mode == MODE_XYZ_EXPORT, 8, mode == MODE_XYZ_EXPORT ? st.icc.output_profile : in.data,
		mode == MODE_XYZ_EXPORT ? st.icc.output_len : in.len, st.icc.output_profile, st.icc.output_len};
	return 0;
}

/* the cached job for (mode, profile), built and uploaded on a miss; entries used by the current batch are never evicted */
IccCacheEntry *
stage_entry(const char *domain, IccStage &st, int frame, int mode, const IccProfileRef &in, const std::vector<IccCacheEntry *> &pinned)
{
	const uint64_t h = mode == MODE_TRANSFORM ? fnv1a64(in.data, in.len) : 0;
	for (IccCacheEntry *e : st.cache)
		if (e->mode == mode && (mode != MODE_TRANSFORM || (e->hash == h && e->bytes.size() == in.len && memcmp(e->bytes.data(), in.data, in.len) == 0))) {
			e->tick = ++st.tick;
			return e;
		}
	auto *e = new IccCacheEntry();
	e->mode = mode;
	e->hash = h;
	if (mode == MODE_TRANSFORM)
		e->bytes.assign((const unsigned char *) in.data, (const unsigned char *) in.data + in.len);
	JobSpec sp;
	stage_job_spec(st, mode, in, &sp);
	std::vector<float> pool;
	int ob, of, ot;
	const int in_type = st.bands < 3 ? VB200_INTERPRETATION_B_W : VB200_INTERPRETATION_sRGB;
	if (build_job(domain, sp, VB200_FORMAT_UCHAR, st.bands, in_type, &e->job, pool, &ob, &of, &ot)) {
		error(domain, "frame %d: its colour transform is not supported on the device path", frame);
		delete e;
		return nullptr;
	}
	if (ob != st.out_bands) {
		error(domain, "frame %d: the transform gives %d bands, the plan expects %d", frame, ob, st.out_bands);
		delete e;
		return nullptr;
	}
	if (cudaMalloc(&e->dpool, std::max<size_t>(1, pool.size()) * sizeof(float)) != cudaSuccess ||
		cudaMemcpy(e->dpool, pool.data(), pool.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
		cuda_fail(domain, cudaGetLastError(), "ICC job upload");
		entry_free(e);
		return nullptr;
	}
	e->job.in.pool = e->job.out.pool = e->dpool;
	e->tick = ++st.tick;
	/* a small LRU: evict the least recently used entry the batch in flight does not hold */
	if (st.cache.size() >= IccStage::kCacheEntries) {
		int victim = -1;
		for (int i = 0; i < (int) st.cache.size(); i++) {
			bool held = false;
			for (IccCacheEntry *p : pinned)
				held = held || p == st.cache[i];
			if (!held && (victim < 0 || st.cache[i]->tick < st.cache[victim]->tick))
				victim = i;
		}
		if (victim >= 0) {
			entry_free(st.cache[victim]);
			st.cache.erase(st.cache.begin() + victim);
		}
	}
	st.cache.push_back(e);
	return e;
}

} // namespace

struct IccTiming {
	cudaEvent_t start = nullptr, stop = nullptr;
	bool pending = false;
};
thread_local IccTiming g_icc_timing;

float
icc_stage_last_ms()
{
	float ms = -1.0f;
	if (g_icc_timing.pending && cudaEventSynchronize(g_icc_timing.stop) == cudaSuccess &&
		cudaEventElapsedTime(&ms, g_icc_timing.start, g_icc_timing.stop) != cudaSuccess)
		ms = -1.0f;
	return ms;
}

IccStage *
icc_stage_new()
{
	return new IccStage();
}

void
icc_stage_free(IccStage *st)
{
	if (!st)
		return;
	for (IccCacheEntry *e : st->cache)
		entry_free(e);
	delete st;
}

int
icc_stage_set(const char *domain, IccStage *st, const VB200ThumbnailIcc *icc, int bands, int *out_bands)
{
	std::lock_guard<std::mutex> lock(st->lock);
	for (IccCacheEntry *e : st->cache)
		entry_free(e);
	st->cache.clear();
	auto copy = [](std::vector<unsigned char> &v, const void *p, size_t n) -> const void * {
		v.assign((const unsigned char *) p, (const unsigned char *) p + (p ? n : 0));
		return p ? v.data() : nullptr;
	};
	st->icc = *icc;
	st->icc.input_profile = copy(st->input, icc->input_profile, icc->input_len);
	st->icc.output_profile = copy(st->output, icc->output_profile, icc->output_len);
	st->icc.builtin_rgb = copy(st->builtin_rgb, icc->builtin_rgb, icc->builtin_rgb_len);
	st->icc.builtin_grey = copy(st->builtin_grey, icc->builtin_grey, icc->builtin_grey_len);
	st->bands = bands;
	/* vips_icc_transform / vips_icc_export fail outright when the output profile does not load (icc_transform.c:1032-1037) */
	std::vector<unsigned> tags;
	if (!lcms_would_open((const unsigned char *) st->icc.output_profile, st->icc.output_len, &tags)) {
		error(domain, "no output profile: corrupt profile");
		return -1;
	}
	const int ob = icc_space_bands((const unsigned char *) st->icc.output_profile);
	if (ob != 1 && ob != 3 && ob != 4) {
		error(domain, "output profile colour space %.4s not supported on the device path", (const char *) st->icc.output_profile + 16);
		return -1;
	}
	if (!intent_supported((const unsigned char *) st->icc.output_profile, tags, icc->intent, false)) {
		error(domain, "the output profile does not support rendering intent %d: its header intent is not supported on the device path",
			icc->intent);
		return -1;
	}
	st->out_bands = ob + bands - (bands < 3 ? 1 : 3);
	/* parse the output side once now, so that a profile the evaluator declines fails here rather than per batch */
	JobSpec sp;
	stage_job_spec(*st, MODE_XYZ_EXPORT, IccProfileRef{nullptr, 0}, &sp);
	IccJob J;
	std::vector<float> pool;
	int b, f, t;
	if (build_job(domain, sp, VB200_FORMAT_UCHAR, bands, bands < 3 ? VB200_INTERPRETATION_B_W : VB200_INTERPRETATION_sRGB, &J, pool, &b, &f, &t))
		return -1;
	*out_bands = st->out_bands;
	return 0;
}

int
icc_stage_run(const char *domain, IccStage *st, const void *in, size_t in_stride, void *out, size_t out_stride, int n, size_t pixels,
	const void *const *embedded, const size_t *embedded_lens, cudaStream_t s)
{
	if (n <= 0)
		return 0;
	std::lock_guard<std::mutex> lock(st->lock);
	std::vector<IccCacheEntry *> used; /* distinct entries of this batch, in first-use order */
	std::vector<int> job_of(n);
	for (int f = 0; f < n; f++) {
		IccProfileRef ref{nullptr, 0};
		int source = 0;
		const int mode = select_input_profile(domain, f, st->icc, st->bands, embedded ? embedded[f] : nullptr,
			embedded && embedded_lens ? embedded_lens[f] : 0, &ref, &source);
		if (mode < 0)
			return -1;
		IccCacheEntry *e = stage_entry(domain, *st, f, mode, ref, used);
		if (!e)
			return -1;
		int k = 0;
		while (k < (int) used.size() && used[k] != e)
			k++;
		if (k == (int) used.size())
			used.push_back(e);
		job_of[f] = k;
	}
	std::vector<IccJob> jobs(used.size());
	for (size_t k = 0; k < used.size(); k++)
		jobs[k] = used[k]->job;
	const size_t jobs_bytes = jobs.size() * sizeof(IccJob);
	void *table = nullptr;
	if (dev_alloc(domain, &table, jobs_bytes + (size_t) n * sizeof(int), s))
		return -1;
	int rc = 0;
	if (cudaMemcpyAsync(table, jobs.data(), jobs_bytes, cudaMemcpyHostToDevice, s) != cudaSuccess ||
		cudaMemcpyAsync((char *) table + jobs_bytes, job_of.data(), (size_t) n * sizeof(int), cudaMemcpyHostToDevice, s) != cudaSuccess)
		rc = cuda_fail(domain, cudaGetLastError(), "ICC job table upload");
	const int in_ps = st->bands, out_ps = st->out_bands;
	/* a few CTAs per frame, each walking its share of the pixels; frames on gridDim.y, at most kMaxBatchFrames a launch */
	const unsigned per_frame = (unsigned) std::min<size_t>((pixels + 255) / 256, 64);
	/* VB200_ICC_TIMING: CUDA events around this call's launches, read back by vb200_debug_icc_stage_ms */
	const bool timing = getenv("VB200_ICC_TIMING") != nullptr;
	if (timing) {
		for (cudaEvent_t *ev : {&g_icc_timing.start, &g_icc_timing.stop})
			if (!*ev && cudaEventCreate(ev) != cudaSuccess)
				rc = cuda_fail(domain, cudaGetLastError(), "ICC timing event");
		if (!rc)
			cudaEventRecord(g_icc_timing.start, s);
		g_icc_timing.pending = !rc;
	}
	for (int f0 = 0; f0 < n && !rc; f0 += kMaxBatchFrames) {
		const int nf = std::min(n - f0, (int) kMaxBatchFrames);
		icc_frames_kernel<<<dim3(per_frame, nf), 256, 0, s>>>((const IccJob *) table, (const int *) ((char *) table + jobs_bytes) + f0,
			(const uint8_t *) in + (size_t) f0 * in_stride, in_stride, in_ps, (uint8_t *) out + (size_t) f0 * out_stride, out_stride,
			out_ps, pixels);
		const cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess)
			rc = cuda_fail(domain, e, "icc_frames_kernel");
		else
			count_launch();
	}
	if (timing && g_icc_timing.pending)
		cudaEventRecord(g_icc_timing.stop, s);
	for (IccCacheEntry *e : used) {
		size_t k = 0;
		while (k < e->used.size() && e->used[k].first != s)
			k++;
		if (k == e->used.size()) {
			cudaEvent_t ev = nullptr;
			if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) {
				rc = cuda_fail(domain, cudaGetLastError(), "ICC job event");
				continue;
			}
			e->used.emplace_back(s, ev);
		}
		cudaEventRecord(e->used[k].second, s);
	}
	dev_free(table, s);
	return rc;
}

/* test hook: the selection of one frame, as the stage makes it */
int
icc_debug_select(const VB200ThumbnailIcc *icc, int bands, const void *embedded, size_t embedded_len, int *source)
{
	IccProfileRef ref{nullptr, 0};
	*source = -1;
	const int mode = select_input_profile("icc_select", 0, *icc, bands, embedded, embedded_len, &ref, source);
	return mode < 0 ? -1 : mode == MODE_XYZ_EXPORT ? 1 : 0;
}

int
icc_debug_classify(const void *profile, size_t len, int want_bands, int intent)
{
	return classify_input_profile(profile, len, want_bands, intent);
}

} // namespace vb200

using namespace vb200;

extern "C" int
vb200_icc_import(const VB200Image *in, VB200Image *out, const void *profile, size_t len, int intent, int pcs)
{
	const JobSpec sp = {0, intent, pcs == VB200_PCS_XYZ, 8, profile, len, nullptr, 0};
	return run_icc("icc_import", in, out, sp);
}

extern "C" int
vb200_icc_export(const VB200Image *in, VB200Image *out, const void *profile, size_t len, int intent, int depth, int pcs)
{
	const JobSpec sp = {1, intent, pcs == VB200_PCS_XYZ, depth, profile, len, nullptr, 0};
	return run_icc("icc_export", in, out, sp);
}

extern "C" int
vb200_icc_transform(const VB200Image *in, VB200Image *out, const void *in_profile, size_t in_len, const void *out_profile,
	size_t out_len, int intent, int depth)
{
	const JobSpec sp = {2, intent, 0, depth, in_profile, in_len, out_profile, out_len};
	return run_icc("icc_transform", in, out, sp);
}

/* Test hook, host only: the same per-pixel code on the CPU (tests/test_icc.py compares it with lcms2). */
extern "C" int
vb200_debug_icc_eval(int mode, const void *in, int in_fmt, int in_bands, void *out, int n, const void *pa, size_t la,
	const void *pb, size_t lb, int intent, int depth, int pcs)
{
	const JobSpec sp = {mode, intent, pcs == VB200_PCS_XYZ, depth, pa, la, pb, lb};
	IccJob J;
	std::vector<float> pool;
	int ob, of, ot;
	const int in_type = mode == 1 ? (pcs == VB200_PCS_XYZ ? VB200_INTERPRETATION_XYZ : VB200_INTERPRETATION_LAB)
		: in_fmt == VB200_FORMAT_USHORT ? VB200_INTERPRETATION_RGB16 : VB200_INTERPRETATION_sRGB;
	if (build_job("icc_eval", sp, in_fmt, in_bands, in_type, &J, pool, &ob, &of, &ot))
		return -1;
	J.in.pool = J.out.pool = pool.data();
	const size_t ips = format_sizeof(in_fmt) * in_bands, ops = format_sizeof(of) * ob;
	for (int i = 0; i < n; i++)
		icc_pixel(J, (const char *) in + (size_t) i * ips, (char *) out + (size_t) i * ops);
	return ob;
}

/* Test hooks, host only: the input-profile selection of one thumbnail frame (0: transform, *source = 0 embedded / 1 input_profile /
 * 2 built-in; 1: no input profile, the XYZ export; -1: error), and the open / compatibility / intent check behind it.
 */
extern "C" int
vb200_debug_icc_select(const VB200ThumbnailIcc *icc, int bands, const void *embedded, size_t embedded_len, int *source)
{
	if (!icc || !source) {
		error("icc_select", "null argument");
		return -1;
	}
	return icc_debug_select(icc, bands, embedded, embedded_len, source);
}

extern "C" int
vb200_debug_icc_classify(const void *profile, size_t len, int want_bands, int intent)
{
	return icc_debug_classify(profile, len, want_bands, intent);
}

/* with env VB200_ICC_TIMING set: CUDA-event time of the calling thread's last ICC stage (its icc_frames_kernel launches); -1 if none */
extern "C" float
vb200_debug_icc_stage_ms(void)
{
	return icc_stage_last_ms();
}
