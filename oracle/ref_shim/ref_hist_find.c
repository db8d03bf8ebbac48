/* ref_hist_find.c -- the reference's arithmetic/statistic.c and arithmetic/hist_find.c compiled in place.  TEST
 * INFRASTRUCTURE ONLY.
 *
 * VipsStatistic's build runs vips_sink(start, scan, stop) over its input (statistic.c:118-123): the sink here walks the
 * image in 64 x 64 tiles, one sequence per row of tiles, as threads would, so hist_find's sub-histograms are merged by
 * its own stop function.  hist_find's output line goes through vips_image_write_line into a memory image.
 */
#include <stdarg.h>
#include <vips/vips.h>
#ifndef VIPS_IMAGE_N_PELS
#define VIPS_IMAGE_N_PELS(I) ((guint64) (I)->Xsize * (I)->Ysize)
#endif

int
vips_check_bandno(const char *domain, VipsImage *im, int bandno)
{
	/* iofuncs/error.c:1013-1023 */
	if (bandno < -1 || bandno > im->Bands - 1) {
		vips_error(domain, "bandno must be -1, or less than %d", im->Bands);
		return -1;
	}
	return 0;
}

int
vips_image_write_line(VipsImage *image, int ypos, VipsPel *linebuffer)
{
	const size_t line = VIPS_IMAGE_SIZEOF_LINE(image);
	if (!image->data)
		image->data = (VipsPel *) calloc((size_t) image->Ysize, line);
	memcpy(image->data + (size_t) ypos * line, linebuffer, line);
	return 0;
}

int
vips_sink(VipsImage *im, VipsStartFn start_fn, VipsGenerateFn generate_fn, VipsStopFn stop_fn, void *a, void *b)
{
	int x, y;
	for (y = 0; y < im->Ysize; y += 64) {
		void *seq = start_fn(im, a, b);
		VipsRegion *reg = vips_region_new(im);
		int rc = 0;
		if (!seq)
			return -1;
		for (x = 0; x < im->Xsize && !rc; x += 64) {
			VipsRect r;
			gboolean stop = FALSE;
			r.left = x;
			r.top = y;
			r.width = VIPS_MIN(64, im->Xsize - x);
			r.height = VIPS_MIN(64, im->Ysize - y);
			rc = vips_region_prepare(reg, &r) || generate_fn(reg, seq, a, b, &stop);
		}
		g_object_unref(reg);
		if (stop_fn(seq, a, b) || rc)
			return -1;
	}
	return 0;
}

#include "statistic.c"

#define g_object_set(OBJ, NAME, VAL, END) (((VipsHistFind *) (OBJ))->out = (VAL))
#define vips_hist_find vips_hist_find__via_call_split
#include "hist_find.c"
#undef vips_hist_find
#undef g_object_set

void *
ref_hist_find(void *in, int band)
{
	VipsHistFind *hist_find = (VipsHistFind *) vips__shim_object_new(vips_hist_find_get_type());
	((VipsStatistic *) hist_find)->in = (VipsImage *) in;
	hist_find->band = band;
	if (vips_hist_find_build((VipsObject *) hist_find))
		return NULL;
	return hist_find->out;
}
