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

#include "icc_eval.cuh"
#include "vb200_internal.h"

namespace vb200 {

namespace {


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
	IccJob J;
	std::vector<float> pool;
	int ob, of, ot;
	return run_image(domain, in, out,
		[&](size_t *preset_line) {
			if (build_job(domain, sp, in->BandFmt, in->Bands, in->Type, &J, pool, &ob, &of, &ot))
				return -1;
			*preset_line = (size_t) in->Xsize * ob * format_sizeof(of); /* the exact result extent (grey -> Lab widens 1 band to 3 floats) */
			return 0;
		},
		[&](const DevImage &din, DevImage *dout, cudaStream_t s) {
			float *dpool = nullptr;
			int rc = 0;
			if (!pool.empty()) {
				rc = dev_alloc(domain, (void **) &dpool, pool.size() * sizeof(float), s);
				if (!rc && cudaMemcpyAsync(dpool, pool.data(), pool.size() * sizeof(float), cudaMemcpyHostToDevice, s) != cudaSuccess)
					rc = -1;
			}
			J.in.pool = J.out.pool = dpool;
			if (!rc)
				rc = dev_image_new(domain, dout, din.w, din.h, ob, of, ot, s);
			if (!rc) {
				const dim3 grid = row_grid(din.w, din.h);
				(rows_loop(din.h) ? icc_kernel<true> : icc_kernel<false>)<<<grid, 256, 0, s>>>(J, (const char *) din.data, din.bpl, format_sizeof(din.fmt) * din.bands, (char *) dout->data,
					dout->bpl, format_sizeof(of) * ob, din.w, din.h);
				const cudaError_t e = cudaGetLastError();
				if (e != cudaSuccess)
					rc = cuda_fail(domain, e, "icc_kernel");
				else
					count_launch();
			}
			/* the pool is read by the kernel: free it stream-ordered, after the launch */
			if (dpool)
				dev_free(dpool, s);
			return rc;
		});
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

/* One launch per chunk of frames, whatever profiles they carry: frame f runs jobs[frames[f].exp].  A CTA serves one frame,
 * copies that frame's job into shared memory once and walks the frame's pixels.
 */
__global__ void __launch_bounds__(256)
icc_frames_kernel(const IccJob *__restrict__ jobs, const IccFrame *__restrict__ frames, const uint8_t *__restrict__ in, size_t in_stride,
	int in_ps, uint8_t *__restrict__ out, size_t out_stride, int out_ps, size_t pixels)
{
	__shared__ __align__(16) unsigned char smem[sizeof(IccJob)];
	const int f = blockIdx.y;
	const unsigned *src = (const unsigned *) (jobs + frames[f].exp);
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
	bool linear = false; /* vb200_thumbnail_plan_set_linear_icc: import and export jobs, keyed by their profile */
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
	if (mode == MODE_IMPORT || mode == MODE_EXPORT) {
		/* the linear mode: the import to, or the export from, the XYZ PCS with `in` as the profile */
		*sp = JobSpec{mode, st.icc.intent, 1, 8, in.data, in.len, nullptr, 0};
		return 0;
	}
	*sp = JobSpec{mode, st.icc.intent, mode == MODE_XYZ_EXPORT, 8, mode == MODE_XYZ_EXPORT ? st.icc.output_profile : in.data,
		mode == MODE_XYZ_EXPORT ? st.icc.output_len : in.len, st.icc.output_profile, st.icc.output_len};
	return 0;
}

/* the cached job for (mode, profile), built and uploaded on a miss; entries used by the current batch are never evicted */
IccCacheEntry *
stage_entry(const char *domain, IccStage &st, int frame, int mode, const IccProfileRef &in, const std::vector<IccCacheEntry *> &pinned)
{
	const bool keyed = mode != MODE_XYZ_EXPORT; /* every mode but the XYZ export reads a profile of its own */
	const uint64_t h = keyed ? fnv1a64(in.data, in.len) : 0;
	for (IccCacheEntry *e : st.cache)
		if (e->mode == mode && (!keyed || (e->hash == h && e->bytes.size() == in.len && memcmp(e->bytes.data(), in.data, in.len) == 0))) {
			e->tick = ++st.tick;
			return e;
		}
	auto *e = new IccCacheEntry();
	e->mode = mode;
	e->hash = h;
	if (keyed)
		e->bytes.assign((const unsigned char *) in.data, (const unsigned char *) in.data + in.len);
	JobSpec sp;
	stage_job_spec(st, mode, in, &sp);
	std::vector<float> pool;
	int ob, of, ot;
	/* the linear export reads the float XYZ image (3 bands + the extra ones) the float resize leaves */
	const int in_type = mode == MODE_EXPORT ? VB200_INTERPRETATION_XYZ : st.bands < 3 ? VB200_INTERPRETATION_B_W : VB200_INTERPRETATION_sRGB;
	const int in_fmt = mode == MODE_EXPORT ? VB200_FORMAT_FLOAT : VB200_FORMAT_UCHAR;
	const int in_bands = mode == MODE_EXPORT ? st.bands - (st.bands < 3 ? 1 : 3) + 3 : st.bands;
	if (build_job(domain, sp, in_fmt, in_bands, in_type, &e->job, pool, &ob, &of, &ot)) {
		error(domain, "frame %d: its colour transform is not supported on the device path", frame);
		delete e;
		return nullptr;
	}
	if (mode != MODE_IMPORT && ob != st.out_bands) {
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

namespace {

/* the stage's own copies of the profiles, its cache emptied */
void
stage_copy(IccStage *st, const VB200ThumbnailIcc *icc, int bands)
{
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
}

/* vips_icc_transform / vips_icc_export fail outright when the output profile does not load (icc_transform.c:1032-1037);
 * *ob: its colour bands
 */
int
check_output_profile(const char *domain, const IccStage &st, int *ob)
{
	std::vector<unsigned> tags;
	if (!lcms_would_open((const unsigned char *) st.icc.output_profile, st.icc.output_len, &tags)) {
		error(domain, "no output profile: corrupt profile");
		return -1;
	}
	*ob = icc_space_bands((const unsigned char *) st.icc.output_profile);
	if (*ob != 1 && *ob != 3 && *ob != 4) {
		error(domain, "output profile colour space %.4s not supported on the device path", (const char *) st.icc.output_profile + 16);
		return -1;
	}
	if (!intent_supported((const unsigned char *) st.icc.output_profile, tags, st.icc.intent, false)) {
		error(domain, "the output profile does not support rendering intent %d: its header intent is not supported on the device path",
			st.icc.intent);
		return -1;
	}
	return 0;
}

/* one event per (entry, stream), recorded after the launches just queued on s that read the entries' pools */
int
stage_hold(const char *domain, const std::vector<IccCacheEntry *> &used, cudaStream_t s)
{
	int rc = 0;
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
	return rc;
}

/* What one frame of a linear colour-managed thumbnail runs (thumbnail.c:766-805, 929-987) */
struct LinChoice {
	int branch = LIN_PLAIN, source = -1, export_from = -1;
	IccProfileRef imp{nullptr, 0}, exp{nullptr, 0};
};

int
select_linear(const char *domain, int frame, const VB200ThumbnailIcc &icc, int bands, const void *embedded, size_t embedded_len,
	LinChoice *c)
{
	*c = LinChoice();
	IccProfileRef ref{nullptr, 0};
	int source = -1;
	const int mode = select_input_profile(domain, frame, icc, bands, embedded, embedded_len, &ref, &source);
	if (mode < 0)
		return -1;
	const IccProfileRef out{icc.output_profile, icc.output_len};
	if (mode == MODE_XYZ_EXPORT) {
		/* no profile to import with: with an output profile vips_colourspace(XYZ) + export (:957-970), else plain (:971-987) */
		if (icc.output_profile) {
			c->branch = LIN_XYZ;
			c->export_from = 0;
			c->exp = out;
		}
		return 0;
	}
	c->branch = LIN_IMPORT;
	c->source = source;
	c->imp = ref;
	if (icc.output_profile) {
		c->export_from = 0;
		c->exp = out;
		return 0;
	}
	/* no output profile: vips_icc_export_build exports to the image's own profile (icc_transform.c:995-1040), the embedded one the
	 * import used or the fallback it attached (:835-849); one that cannot serve as an output profile fails there
	 */
	std::vector<unsigned> tags;
	const unsigned char *d = (const unsigned char *) ref.data;
	if (!lcms_would_open(d, ref.len, &tags) || icc_space_bands(d) != 3 || !intent_supported(d, tags, icc.intent, false)) {
		error(domain, "frame %d: no output profile: the image's profile cannot be used as an output profile", frame);
		return -1;
	}
	c->export_from = 1;
	c->exp = ref;
	return 0;
}

} // namespace

int
icc_stage_set(const char *domain, IccStage *st, const VB200ThumbnailIcc *icc, int bands, bool linear, int *out_bands)
{
	std::lock_guard<std::mutex> lock(st->lock);
	if (linear && bands < 3) {
		error(domain, "linear colour-managed thumbnails on the device path need 3+ band frames (sGrey / GREY16 import is not built)");
		return -1;
	}
	stage_copy(st, icc, bands);
	st->linear = linear;
	st->out_bands = bands; /* linear without an output profile: each frame exports to its own (RGB) profile, or runs the plain path */
	if (!linear || icc->output_profile) {
		int ob = 0;
		if (check_output_profile(domain, *st, &ob))
			return -1;
		st->out_bands = ob + bands - (bands < 3 ? 1 : 3);
		/* parse the export once now, so that a profile the evaluator declines fails here rather than per batch: from the float
		 * XYZ the linear resize leaves, or from the 8-bit thumbnail
		 */
		JobSpec sp;
		stage_job_spec(*st, linear ? MODE_EXPORT : MODE_XYZ_EXPORT, IccProfileRef{st->icc.output_profile, st->icc.output_len}, &sp);
		IccJob J;
		std::vector<float> pool;
		int b, f, t;
		if (build_job(domain, sp, linear ? VB200_FORMAT_FLOAT : VB200_FORMAT_UCHAR, bands,
				linear ? VB200_INTERPRETATION_XYZ : bands < 3 ? VB200_INTERPRETATION_B_W : VB200_INTERPRETATION_sRGB, &J, pool, &b, &f, &t))
			return -1;
	}
	*out_bands = st->out_bands;
	return 0;
}

int
icc_stage_batch(const char *domain, IccStage *st, int n, const void *const *embedded, const size_t *embedded_lens, cudaStream_t s,
	int frame0, const std::function<int(const IccBatch &)> &body)
{
	if (n <= 0)
		return 0;
	std::lock_guard<std::mutex> lock(st->lock);
	std::vector<IccCacheEntry *> used; /* distinct entries of this batch, in first-use order */
	/* *k: the batch's index of the cached job for (mode, profile) */
	auto job = [&](int f, int mode, const IccProfileRef &ref, int *k) {
		IccCacheEntry *e = stage_entry(domain, *st, frame0 + f, mode, ref, used);
		if (!e)
			return -1;
		*k = 0;
		while (*k < (int) used.size() && used[*k] != e)
			++*k;
		if (*k == (int) used.size())
			used.push_back(e);
		return 0;
	};
	std::vector<IccFrame> frames(n);
	for (int f = 0; f < n; f++) {
		const void *emb = embedded ? embedded[f] : nullptr;
		const size_t emb_len = embedded && embedded_lens ? embedded_lens[f] : 0;
		if (!st->linear) {
			IccProfileRef ref{nullptr, 0};
			int source = 0;
			const int mode = select_input_profile(domain, frame0 + f, st->icc, st->bands, emb, emb_len, &ref, &source);
			frames[f] = IccFrame{LIN_PLAIN, -1, -1};
			if (mode < 0 || job(f, mode, ref, &frames[f].exp))
				return -1;
			continue;
		}
		LinChoice c;
		if (select_linear(domain, frame0 + f, st->icc, st->bands, emb, emb_len, &c))
			return -1;
		frames[f] = IccFrame{c.branch, -1, -1};
		if (c.branch == LIN_IMPORT && job(f, MODE_IMPORT, c.imp, &frames[f].imp))
			return -1;
		if (c.branch != LIN_PLAIN && job(f, MODE_EXPORT, c.exp, &frames[f].exp))
			return -1;
	}
	std::vector<IccJob> jobs(used.size());
	for (size_t k = 0; k < used.size(); k++)
		jobs[k] = used[k]->job;
	const size_t jobs_bytes = jobs.size() * sizeof(IccJob);
	void *table = nullptr;
	if (dev_alloc(domain, &table, jobs_bytes + (size_t) n * sizeof(IccFrame), s))
		return -1;
	int rc = 0;
	if (cudaMemcpyAsync(table, jobs.data(), jobs_bytes, cudaMemcpyHostToDevice, s) != cudaSuccess ||
		cudaMemcpyAsync((char *) table + jobs_bytes, frames.data(), (size_t) n * sizeof(IccFrame), cudaMemcpyHostToDevice, s) != cudaSuccess)
		rc = cuda_fail(domain, cudaGetLastError(), "ICC job table upload");
	if (!rc) {
		const IccBatch b{(const IccJob *) table, (const IccFrame *) ((char *) table + jobs_bytes), jobs.data(), frames.data()};
		rc = body(b);
	}
	if (stage_hold(domain, used, s))
		rc = -1;
	dev_free(table, s);
	/* the host copies above die here: body's leaf chain passes jobs to its launches by value */
	return rc;
}

int
icc_job_apply(const char *domain, const IccJob *jobs, int k, const DevImage &in, DevImage *out, cudaStream_t s)
{
	const IccJob *J = jobs + k;
	const int ob = (J->mode == MODE_IMPORT ? 3 : J->out.bands) + J->extra;
	const int of = J->mode == MODE_IMPORT ? VB200_FORMAT_FLOAT : J->out_fmt;
	const int colour = J->out.bands;
	const int ot = J->mode == MODE_IMPORT ? VB200_INTERPRETATION_XYZ
		: colour == 1					  ? VB200_INTERPRETATION_B_W
		: colour == 3					  ? VB200_INTERPRETATION_sRGB
										  : VB200_INTERPRETATION_CMYK;
	if (dev_image_new(domain, out, in.w, in.h, ob, of, ot, s))
		return -1;
	const dim3 grid = row_grid(in.w, in.h);
	(rows_loop(in.h) ? icc_kernel<true> : icc_kernel<false>)<<<grid, 256, 0, s>>>(*J, (const char *) in.data, in.bpl,
		format_sizeof(in.fmt) * in.bands, (char *) out->data, out->bpl, format_sizeof(of) * ob, in.w, in.h);
	const cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
		return cuda_fail(domain, e, "icc_kernel");
	count_launch();
	return 0;
}

int
icc_stage_run(const char *domain, IccStage *st, const void *in, size_t in_stride, void *out, size_t out_stride, int n, size_t pixels,
	const void *const *embedded, const size_t *embedded_lens, cudaStream_t s, int frame0)
{
	return icc_stage_batch(domain, st, n, embedded, embedded_lens, s, frame0, [&](const IccBatch &b) {
		const int in_ps = st->bands, out_ps = st->out_bands;
		int rc = 0;
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
			icc_frames_kernel<<<dim3(per_frame, nf), 256, 0, s>>>(b.d_jobs, b.d_frames + f0, (const uint8_t *) in + (size_t) f0 * in_stride,
				in_stride, in_ps, (uint8_t *) out + (size_t) f0 * out_stride, out_stride, out_ps, pixels);
			const cudaError_t e = cudaGetLastError();
			if (e != cudaSuccess)
				rc = cuda_fail(domain, e, "icc_frames_kernel");
			else
				count_launch();
		}
		if (timing && g_icc_timing.pending)
			cudaEventRecord(g_icc_timing.stop, s);
		return rc;
	});
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

/* test hook: the linear-mode choice of one frame, as the stage makes it */
int
icc_debug_select_linear(const VB200ThumbnailIcc *icc, int bands, const void *embedded, size_t embedded_len, int *branch, int *source,
	int *export_from)
{
	LinChoice c;
	const int rc = select_linear("icc_select_linear", 0, *icc, bands, embedded, embedded_len, &c);
	*branch = c.branch;
	*source = c.source;
	*export_from = c.export_from;
	return rc;
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

extern "C" int
vb200_debug_icc_select_linear(const VB200ThumbnailIcc *icc, int bands, const void *embedded, size_t embedded_len, int *branch,
	int *source, int *export_from)
{
	if (!icc || !branch || !source || !export_from) {
		error("icc_select_linear", "null argument");
		return -1;
	}
	return icc_debug_select_linear(icc, bands, embedded, embedded_len, branch, source, export_from);
}

/* with env VB200_ICC_TIMING set: CUDA-event time of the calling thread's last ICC stage (its icc_frames_kernel launches); -1 if none */
extern "C" float
vb200_debug_icc_stage_ms(void)
{
	return icc_stage_last_ms();
}
