/* nsgif_oracle.c -- TEST INFRASTRUCTURE ONLY: what vips_gifload_buffer(buf, len, &out, "page", page, "n", n, NULL) gives
 * with fail_on = none, restated over the reference's own libnsgif (compiled in place by the Makefile beside this file).
 *
 *   foreign/nsgifload.c:635-653   the bitmap callbacks, with their dimension limits
 *   foreign/nsgifload.c:364-474   header: scan (errors are warnings), nsgif_data_complete, "no frames in GIF", bands from
 *                                 any frame's transparency, n = -1 and "bad page number"
 *   foreign/nsgifload.c:477-539   generate: nsgif_frame_decode(page) per page, RGBA copied or its fourth byte dropped
 *
 * nsgif_oracle_load returns 0 (out, if given, holds n pages of height rows of width x bands bytes) or -1 with the loader's
 * message; info[] = {width, height, bands, frame_count, scan result} as far as the call got.
 */
#include <limits.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "nsgif.h"

static nsgif_bitmap_t *
bm_create(int width, int height)
{
	if (width <= 0 || width > 65535 || height <= 0 || height > 65535 || (uint64_t) width * height > INT_MAX / 4)
		return NULL;
	return calloc((size_t) width * height, 4);
}

static void
bm_destroy(nsgif_bitmap_t *bitmap)
{
	free(bitmap);
}

static uint8_t *
bm_buffer(nsgif_bitmap_t *bitmap)
{
	return bitmap;
}

static const nsgif_bitmap_cb_vt callbacks = {bm_create, bm_destroy, bm_buffer};

static int
fail(char *msg, size_t msglen, const char *text)
{
	if (msg && msglen)
		snprintf(msg, msglen, "%s", text);
	return -1;
}

int
nsgif_oracle_load(const uint8_t *buf, size_t len, int page, int n, uint8_t *out, int *info, char *msg, size_t msglen)
{
	nsgif_t *gif = NULL;
	int rc = -1;
	memset(info, 0, 5 * sizeof(int));
	if (nsgif_create(&callbacks, NSGIF_BITMAP_FMT_R8G8B8A8, &gif) != NSGIF_OK)
		return fail(msg, msglen, "nsgif_create");
	info[4] = nsgif_data_scan(gif, len, buf);
	nsgif_data_complete(gif);
	const nsgif_info_t *gi = nsgif_get_info(gif);
	do {
		if (!gi->frame_count) {
			fail(msg, msglen, "no frames in GIF");
			break;
		}
		int alpha = 0;
		for (uint32_t i = 0; i < gi->frame_count; i++) {
			const nsgif_frame_info_t *fi = nsgif_get_frame_info(gif, i);
			if (fi && fi->transparency)
				alpha = 1;
		}
		const int gif_n = n == -1 ? (int) gi->frame_count - page : n;
		info[0] = (int) gi->width;
		info[1] = (int) gi->height;
		info[2] = alpha ? 4 : 3;
		info[3] = (int) gi->frame_count;
		if (page < 0 || gif_n <= 0 || page + gif_n > (int) gi->frame_count) {
			fail(msg, msglen, "bad page number");
			break;
		}
		rc = 0;
		if (!out)
			break;
		const size_t line = (size_t) gi->width * info[2];
		for (int k = 0; k < gif_n && !rc; k++) {
			nsgif_bitmap_t *bm = NULL;
			const nsgif_error e = nsgif_frame_decode(gif, page + k, &bm);
			if (e != NSGIF_OK) {
				rc = fail(msg, msglen, nsgif_strerror(e));
				break;
			}
			const uint8_t *p = bm;
			uint8_t *q = out + (size_t) k * line * gi->height;
			for (size_t i = 0; i < (size_t) gi->width * gi->height; i++, p += 4, q += info[2]) {
				q[0] = p[0], q[1] = p[1], q[2] = p[2];
				if (alpha)
					q[3] = p[3];
			}
		}
	} while (0);
	nsgif_destroy(gif);
	return rc;
}
