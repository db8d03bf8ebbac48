/* ref_hist_local.c -- the reference's histogram/hist_local.c compiled in place.  TEST INFRASTRUCTURE ONLY.
 *
 * Its build embeds the input with VIPS_EXTEND_MIRROR (hist_local.c:301-306); the shim's vips_embed serves
 * VIPS_EXTEND_COPY only, so this file's embed serves the mirror: conversion/embed.c:398-430 tiles [in | flip(in)] over
 * [flip(in) ...] with period 2 * size and cuts the embedded window out of it, which is, per coordinate s of the input's
 * frame, u = s mod 2n, u < n ? u : 2n - 1 - u.
 */
#include <stdarg.h>
#include <vips/vips.h>

int
vips_check_format(const char *domain, VipsImage *im, VipsBandFormat fmt)
{
	/* iofuncs/error.c:741-751 */
	if (im->BandFmt != fmt) {
		vips_error(domain, "image must be %s", fmt == VIPS_FORMAT_UCHAR ? "uchar" : "of another format");
		return -1;
	}
	return 0;
}

typedef struct { VipsImage *in; int x, y; } RefMirror;

static int
ref_mirror(int s, int n)
{
	int u = s % (2 * n);
	if (u < 0)
		u += 2 * n;
	return u < n ? u : 2 * n - 1 - u;
}

static int
ref_mirror_gen(VipsRegion *out_region, void *seq, void *a, void *b, gboolean *stop)
{
	VipsRegion *ir = (VipsRegion *) seq;
	RefMirror *m = (RefMirror *) b;
	VipsImage *in = m->in;
	VipsRect *r = &out_region->valid;
	const size_t ps = VIPS_IMAGE_SIZEOF_PEL(in);
	VipsRect all;
	int x, y;

	all.left = 0;
	all.top = 0;
	all.width = in->Xsize;
	all.height = in->Ysize;
	if (vips_region_prepare(ir, &all))
		return -1;
	for (y = 0; y < r->height; y++) {
		const int sy = ref_mirror(r->top + y - m->y, in->Ysize);
		VipsPel *q = VIPS_REGION_ADDR(out_region, r->left, r->top + y);
		for (x = 0; x < r->width; x++)
			memcpy(q + x * ps, VIPS_REGION_ADDR(ir, ref_mirror(r->left + x - m->x, in->Xsize), sy), ps);
	}
	return 0;
}

static int
ref_embed_mirror(VipsImage *in, VipsImage **out, int x, int y, int width, int height, ...)
{
	RefMirror *m = (RefMirror *) calloc(1, sizeof(RefMirror));
	VipsImage *o = vips_image_new();
	va_list ap;
	const char *name;

	va_start(ap, height);
	name = va_arg(ap, const char *);
	if (!name || strcmp(name, "extend") != 0 || va_arg(ap, int) != VIPS_EXTEND_MIRROR) {
		va_end(ap);
		vips_error("embed", "only VIPS_EXTEND_MIRROR is served here");
		return -1;
	}
	va_end(ap);
	m->in = in;
	m->x = x;
	m->y = y;
	vips_image_pipelinev(o, VIPS_DEMAND_STYLE_SMALLTILE, in, NULL); /* conversion/embed.c:440 */
	o->Xsize = width;
	o->Ysize = height;
	vips_image_generate(o, vips_start_one, ref_mirror_gen, vips_stop_one, in, m);
	*out = o;
	return 0;
}

#define vips_embed ref_embed_mirror
#define g_object_set(OBJ, NAME, VAL, END) (((VipsHistLocal *) (OBJ))->out = (VAL))
#define vips_hist_local vips_hist_local__via_call_split
#include "../histogram/hist_local.c"
#undef vips_hist_local
#undef g_object_set
#undef vips_embed

void *
ref_hist_local(void *in, int width, int height, int max_slope)
{
	VipsHistLocal *local = (VipsHistLocal *) vips__shim_object_new(vips_hist_local_get_type());
	local->in = (VipsImage *) in;
	local->width = width;
	local->height = height;
	local->max_slope = max_slope;
	if (vips_hist_local_build((VipsObject *) local))
		return NULL;
	return local->out;
}
