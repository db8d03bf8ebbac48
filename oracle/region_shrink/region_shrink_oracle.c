/* region_shrink_oracle.c -- the reference's 2 x 2 shrinks of one row of output pixels for uchar, as
 * vips_region_shrink_alpha and vips_region_shrink_uncoded_mean run them (iofuncs/region.c): the macros themselves are
 * extracted from the reference at build time (Makefile) and expanded here with the locals those functions declare.
 *
 * p: the top-left input pixel, ls: bytes from an input row to the next, width: output pixels, nb: bands; q: the output.
 */
#include <stddef.h>

typedef unsigned char VipsPel;
typedef struct {
	int left, top, width, height;
} VipsRect;

#include "region_shrink_macros.h"

void
region_shrink_alpha_uchar(const VipsPel *in, int ls, int width, int nb, VipsPel *out)
{
	const VipsRect t = {0, 0, width, 1};
	const VipsRect *target = &t;
	VipsPel *p = (VipsPel *) in, *q = out;
	int x, z;

	SHRINK_ALPHA_TYPE(unsigned char);
}

void
region_shrink_mean_uchar(const VipsPel *in, int ls, int width, int nb, VipsPel *out)
{
	const VipsRect t = {0, 0, width, 1};
	const VipsRect *target = &t;
	int ps = nb;
	VipsPel *p = (VipsPel *) in, *q = out;
	int x, z;

	SHRINK_TYPE_MEAN_INT(unsigned char);
}
