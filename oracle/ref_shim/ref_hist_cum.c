/* ref_hist_cum.c -- the reference's histogram/hist_cum.c compiled in place.  TEST INFRASTRUCTURE ONLY.
 *
 * Only its accumulate loop, vips_hist_cum_process (hist_cum.c:88-131), and its format table (:135-142) are served: a
 * histogram is one line, which is materialised and accumulated into a memory image of the table's format.  The
 * VipsHistogram / VipsHistUnary base classes (region plumbing for n inputs) are not compiled; their types are given
 * here so that the class definition links.
 */
#include <stdarg.h>
#include <vips/vips.h>
#include "../histogram/phistogram.h"
#include "../histogram/hist_unary.h"

VipsImage *vips__shim_materialise(VipsImage *in);
VipsImage *vips__shim_new_memory(int w, int h, int bands, VipsBandFormat fmt, VipsInterpretation type);

int
vips_image_get_bands(const VipsImage *image)
{
	return image->Bands; /* iofuncs/header.c */
}

GType
vips_hist_unary_get_type(void)
{
	return vips__shim_operation_get_type();
}

#define vips_hist_cum vips_hist_cum__via_call_split
#include "../histogram/hist_cum.c"
#undef vips_hist_cum

void *
ref_hist_cum(void *in)
{
	VipsImage *m = vips__shim_materialise((VipsImage *) in);
	VipsHistogram histogram;
	VipsImage *ready[2];
	VipsImage *out;
	VipsPel *p[2];

	if (!m || m->Ysize != 1)
		return NULL;
	memset(&histogram, 0, sizeof(histogram));
	ready[0] = m;
	ready[1] = NULL;
	histogram.ready = ready;
	out = vips__shim_new_memory(m->Xsize, 1, m->Bands, vips_hist_cum_format_table[m->BandFmt], m->Type);
	p[0] = m->data;
	p[1] = NULL;
	vips_hist_cum_process(&histogram, out->data, p, m->Xsize);
	return out;
}
