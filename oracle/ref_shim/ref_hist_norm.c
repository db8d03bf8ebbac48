/* ref_hist_norm.c -- the reference's histogram/hist_norm.c compiled in place.  TEST INFRASTRUCTURE ONLY.
 *
 * Its build (hist_norm.c:86-132) runs as written.  vips_stats is served for what the build reads from it, each band's
 * maximum (the matrix's column 1); vips_linear with equal constants over the bands goes to ref_linear.c's vips_linear1,
 * the reference's own single-element loop, and vips_cast to ref_cast.c.  hist_equal (histogram/hist_equal.c:81-89) is
 * then ref_hist_equal_lut below: find, cum, norm and the cast to the input's format, the LUT that maplut applies.
 */
#include <stdarg.h>
#include <vips/vips.h>
#ifndef VIPS_IMAGE_N_PELS
#define VIPS_IMAGE_N_PELS(I) ((guint64) (I)->Xsize * (I)->Ysize)
#endif

VipsImage *vips__shim_materialise(VipsImage *in);
int vips_linear1(VipsImage *in, VipsImage **out, double a, double b, ...);
int vips_cast(VipsImage *in, VipsImage **out, VipsBandFormat format, ...);
void *ref_hist_find(void *in, int band);
void *ref_hist_cum(void *in);

/* stats.c's matrix: row 0 all bands, row b + 1 band b; column 1 the maximum (stats.c:50-80) */
static int
ref_hist_norm_stats(VipsImage *in, VipsImage **out, ...)
{
	VipsImage *m = vips__shim_materialise(in);
	VipsImage *st;
	int b, i;

	if (!m || m->BandFmt != VIPS_FORMAT_UINT)
		return -1;
	st = vips_image_new_matrix(10, m->Bands + 1);
	for (b = 0; b < m->Bands; b++) {
		const unsigned int *p = (const unsigned int *) m->data;
		double mx = p[b];
		for (i = 0; i < m->Xsize * m->Ysize; i++)
			mx = VIPS_MAX(mx, (double) p[(size_t) i * m->Bands + b]);
		*VIPS_MATRIX(st, 1, b + 1) = mx;
	}
	*out = st;
	return 0;
}

static int
ref_hist_norm_linear(VipsImage *in, VipsImage **out, const double *a, const double *b, int n, ...)
{
	int i;
	for (i = 1; i < n; i++)
		if (a[i] != a[0] || b[i] != b[0]) {
			vips_error("hist_norm", "unequal constants are not served");
			return -1;
		}
	return vips_linear1(in, out, a[0], b[0], NULL);
}

#define vips_stats ref_hist_norm_stats
#define vips_linear ref_hist_norm_linear
#define g_object_set(OBJ, NAME, VAL, END) (((VipsHistNorm *) (OBJ))->out = (VAL))
#define vips_hist_norm vips_hist_norm__via_call_split
#include "../histogram/hist_norm.c"
#undef vips_hist_norm
#undef g_object_set
#undef vips_linear
#undef vips_stats

void *
ref_hist_norm(void *in)
{
	VipsHistNorm *norm = (VipsHistNorm *) vips__shim_object_new(vips_hist_norm_get_type());
	norm->in = (VipsImage *) in;
	if (vips_hist_norm_build((VipsObject *) norm))
		return NULL;
	return norm->out;
}

/* hist_equal.c:81-87 up to the LUT: hist_find -> hist_cum -> hist_norm -> cast to the input's format */
void *
ref_hist_equal_lut(void *in, int band)
{
	VipsImage *t[4] = {NULL, NULL, NULL, NULL};
	if (!(t[0] = (VipsImage *) ref_hist_find(in, band)) || !(t[1] = (VipsImage *) ref_hist_cum(t[0])) ||
		!(t[2] = (VipsImage *) ref_hist_norm(t[1])) || vips_cast(t[2], &t[3], ((VipsImage *) in)->BandFmt, NULL))
		return NULL;
	return t[3];
}
