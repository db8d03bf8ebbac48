/* decode.cu -- what the JPEG, PNG, GIF, TIFF and WebP decoders share around their kernels: the stream kinds and the one switch over
 * the five batch decoders, the C ABI bodies of vb200_*_decode_batch, vb200_*load_buffer, vb200_*_icc_profile and the host-twin
 * hooks, the host-worker header pass, and (for PNG, GIF, TIFF and WebP) the pinned staging block, the chunks bounded by the
 * device budget and the one body every such chunk runs.
 */
#include <cstdint>
#include <cstring>
#include <exception>
#include <mutex>
#include <string>

#include "../../include/vb200.h"
#include "vb200_internal.h"

namespace vb200 {

namespace {

size_t g_chunk_budget = 0; /* vb200_debug_png_set_budget: device bytes per chunk, 0 = an eighth of the device (at least 1 GiB) */

/* pinned staging, grow-only (vb200_shutdown releases it); one chunk at a time uses it, under g_staging_lock */
void *g_staging = nullptr;
size_t g_staging_cap = 0;
std::mutex g_staging_lock;

void
staging_free()
{
	if (g_staging)
		cudaFreeHost(g_staging);
	g_staging = nullptr;
	g_staging_cap = 0;
}

std::string
worker_error()
{
	/* the worker's thread-local "domain: reason\n", without the domain (restated with the stream's index) */
	std::string e = vb200_error_buffer();
	vb200_error_clear();
	const size_t at = e.find(": ");
	e = e.substr(at == std::string::npos ? 0 : at + 2);
	return e.substr(0, e.find('\n'));
}

} // namespace

size_t
align16(size_t v)
{
	return (v + 15) & ~(size_t) 15;
}

int
parse_streams(const char *domain, const char *noun, int n, const std::function<int(int)> &parse,
	const std::function<StreamGeometry(int)> &geometry, StreamGeometry *g)
{
	std::vector<std::string> errs(n);
	parallel_for(n, host_workers(), [&](int i) {
		if (parse(i))
			errs[i] = worker_error();
	});
	for (int i = 0; i < n; i++)
		if (!errs[i].empty()) {
			error(domain, "%s %d: %s", noun, i, errs[i].c_str());
			return -1;
		}
	const StreamGeometry g0 = geometry(0);
	for (int i = 1; i < n; i++) {
		const StreamGeometry gi = geometry(i);
		if (gi.w != g0.w || gi.h != g0.h || gi.bands != g0.bands || gi.pages != g0.pages) {
			if (g0.pages)
				error(domain, "%ss of a batch must decode to one geometry (%d x %d x %d, %d pages; %s %d: %d x %d x %d, %d pages)", noun, g0.w, g0.h,
					g0.bands, g0.pages, noun, i, gi.w, gi.h, gi.bands, gi.pages);
			else
				error(domain, "%ss of a batch must decode to one geometry (%d x %d x %d, %s %d: %d x %d x %d)", noun, g0.w, g0.h, g0.bands, noun, i,
					gi.w, gi.h, gi.bands);
			return -1;
		}
	}
	*g = g0;
	return 0;
}

int
check_out_strides(const char *domain, const StreamGeometry &g, size_t out_bpl, size_t out_frame_stride)
{
	const int rows = g.rows();
	if (out_bpl < (size_t) g.w * g.bands || out_frame_stride < out_bpl * rows) {
		error(domain, "output strides too small for %d x %d x %d", g.w, rows, g.bands);
		return -1;
	}
	return 0;
}

/* device bytes per chunk of the PNG, GIF, TIFF and WebP decoders and the JPEG and PNG encoders */
size_t
chunk_budget()
{
	/* the device's size, asked once: cudaMemGetInfo costs more than a small encoder batch's host work */
	static const size_t device_default = [] {
		size_t free_b = 0, total_b = 0;
		cudaMemGetInfo(&free_b, &total_b);
		return std::max<size_t>(total_b / 8, (size_t) 1 << 30);
	}();
	return g_chunk_budget ? g_chunk_budget : device_default;
}

int
decode_chunks(const char *domain, const char *what, const char *noun, int n, const std::function<size_t(int)> &device_bytes,
	const std::function<int(int, int)> &chunk, cudaStream_t s)
{
	const size_t budget = chunk_budget();
	std::lock_guard<std::mutex> lock(g_staging_lock);
	for (int c0 = 0; c0 < n;) {
		/* the chunk: streams while they fit the budget (at least one) */
		size_t dev_bytes = 0;
		int cn = 0;
		while (c0 + cn < n && cn < kMaxBatchFrames) {
			const size_t b = device_bytes(c0 + cn);
			if (cn > 0 && dev_bytes + b > budget)
				break;
			dev_bytes += b;
			cn++;
		}
		if (dev_bytes > budget) {
			error(domain, "%s %d needs %zu bytes of device memory, more than the %zu allowed", noun, c0, dev_bytes, budget);
			return -1;
		}
		if (chunk(c0, cn))
			return -1;
		c0 += cn;
	}
	if (cudaStreamSynchronize(s) != cudaSuccess)
		return cuda_fail(domain, cudaGetLastError(), (std::string(what) + " decode").c_str());
	return 0;
}

int
decode_chunk(const char *domain, const char *what, const DecodeBlock &b, const std::function<void(unsigned char *)> &stage,
	const std::function<int(unsigned char *, int *)> &decode, const std::function<void(int, int)> &refuse,
	const std::function<int(unsigned char *)> &place, cudaStream_t s)
{
	/* the previous chunk's copy out of the pinned block has finished: its status was read after it */
	unsigned char *hst = (unsigned char *) decode_staging(domain, b.host_bytes);
	if (!hst)
		return -1;
	stage(hst);
	const size_t off_status = align16(b.host_bytes) + align16(b.scratch_bytes);
	unsigned char *dev = nullptr;
	if (dev_alloc(domain, (void **) &dev, off_status + b.n_status * sizeof(int), s))
		return -1;
	int *status = (int *) (dev + off_status);
	std::vector<int> st(b.n_status, 0);
	const std::string label = what;
	int rc = 0;
	if (cudaMemcpyAsync(dev, hst, b.host_bytes, cudaMemcpyHostToDevice, s) != cudaSuccess ||
		cudaMemsetAsync(status, 0, b.n_status * sizeof(int), s) != cudaSuccess)
		rc = cuda_fail(domain, cudaGetLastError(), (label + " staging copy").c_str());
	else {
		const int launched = decode(dev, status);
		count_launch(std::max(launched, 0));
		/* a decode that failed has its reason set; its launches still finish before the block is freed */
		const cudaError_t e = cudaGetLastError();
		const bool failed = e != cudaSuccess || cudaMemcpyAsync(st.data(), status, b.n_status * sizeof(int), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
							cudaStreamSynchronize(s) != cudaSuccess;
		if (launched < 0)
			rc = -1;
		else if (failed)
			rc = cuda_fail(domain, e != cudaSuccess ? e : cudaGetLastError(), (label + " decode kernels").c_str());
	}
	for (int k = 0; k < b.n_status && !rc; k++)
		if (st[k]) {
			refuse(k, st[k]);
			rc = -1;
		}
	if (!rc) {
		const int launched = place(dev);
		count_launch(std::max(launched, 0));
		const cudaError_t e = cudaGetLastError();
		if (launched < 0)
			rc = -1;
		else if (e != cudaSuccess)
			rc = cuda_fail(domain, e, (label + " placement").c_str());
	}
	dev_free(dev, s);
	return rc;
}

int
profile_abi(const char *domain, void *out, size_t cap, size_t *profile_len, const std::function<int(const char *, std::vector<unsigned char> *)> &fetch)
{
	if (!profile_len) {
		error(domain, "null argument");
		return -1;
	}
	std::vector<unsigned char> prof;
	if (fetch(domain, &prof))
		return -1;
	*profile_len = prof.size();
	if (!out)
		return 0;
	if (cap < prof.size()) {
		error(domain, "the profile is %zu bytes, the buffer %zu", prof.size(), cap);
		return -1;
	}
	if (!prof.empty())
		memcpy(out, prof.data(), prof.size());
	return 0;
}

int
host_twin_abi(const char *domain, const std::function<int(const char *)> &fn)
{
	try {
		return fn(domain);
	}
	catch (const std::exception &e) {
		error(domain, "%s", e.what());
		return -1;
	}
}

void *
decode_staging(const char *domain, size_t bytes)
{
	if (g_staging_cap < bytes) {
		staging_free();
		if (cudaMallocHost(&g_staging, bytes + bytes / 4) != cudaSuccess) {
			g_staging = nullptr;
			cuda_fail(domain, cudaGetLastError(), "cudaMallocHost (decode staging)");
			return nullptr;
		}
		g_staging_cap = bytes + bytes / 4;
	}
	return g_staging;
}

void
decode_staging_release()
{
	std::lock_guard<std::mutex> lock(g_staging_lock);
	staging_free();
}

StreamKind
stream_kind(const void *buf, size_t len)
{
	return png_signature(buf, len)	   ? STREAM_PNG
		   : gif_signature(buf, len)  ? STREAM_GIF
		   : tiff_signature(buf, len) ? STREAM_TIFF
		   : webp_signature(buf, len) ? STREAM_WEBP
									  : STREAM_JPEG;
}

/* The decoder and where the embedded profile comes from are all that differ between the kinds.  PNG and GIF have no
 * load-time shrink (thumbnail.c:609-660 lists the loaders that do), and a PNG with eXIf is declined: its orientation would
 * need vips_autorot (thumbnail.c:989-996), which is not built.  The same goes for a TIFF IFD whose Orientation is not 1.
 * A GIF carries no profile.
 */
int
stream_profile(const char *domain, const DecodeRequest &req, const unsigned char *d, size_t n, std::vector<unsigned char> *profile)
{
	const StreamKind kind = req.kind;
	if (kind == STREAM_TIFF) {
		int orientation = 1;
		if (tiff_icc_profile(domain, d, n, req.page, req.n_pages, req.subifd, profile, &orientation))
			return -1;
		if (orientation != 1) {
			error(domain, "TIFF with Orientation %d: it would need vips_autorot, which is not built", orientation);
			return -1;
		}
		return 0;
	}
	if (kind == STREAM_GIF) {
		profile->clear();
		return 0;
	}
	if (kind == STREAM_WEBP)
		return webp_icc_profile(domain, d, n, profile);
	if (kind == STREAM_JPEG)
		return jpeg_icc_profile(domain, d, n, profile);
	bool exif = false;
	if (png_icc_profile(domain, d, n, profile, &exif))
		return -1;
	if (exif) {
		error(domain, "PNG with eXIf: its orientation would need vips_autorot, which is not built");
		return -1;
	}
	return 0;
}

int
dev_decode_batch(const char *domain, const DecodeRequest &req, const void *const *bufs, const size_t *lens, int n, void *out, size_t out_bpl,
	size_t out_frame_stride, int *w, int *h, int *bands, int *page_h, cudaStream_t s)
{
	/* vips_thumbnail_buffer hands its option string to the loader (thumbnail.c:1486-1490, 1585-1590): page and n are
	 * nsgifload's; jpegload and spngload have neither, so any other value fails there.  webpload's page and n select frames
	 * of an animation, which is not decoded here.
	 */
	if (req.kind == STREAM_WEBP && (req.page != 0 || req.n_pages != 1)) {
		error(domain, "webpload's page and n select animation frames, which are not decoded on the device (page %d, n %d)", req.page, req.n_pages);
		return -1;
	}
	if (req.kind != STREAM_GIF && req.kind != STREAM_TIFF && (req.page != 0 || req.n_pages != 1)) {
		error(domain, "%s has no page or n option (page %d, n %d)", req.kind == STREAM_PNG ? "pngload" : "jpegload", req.page, req.n_pages);
		return -1;
	}
	if (req.kind != STREAM_TIFF && req.subifd != -1) {
		error(domain, "only tiffload has a subifd option (subifd %d)", req.subifd);
		return -1;
	}
	if (n < 1 || !bufs || !lens) {
		error(domain, "no %s", req.kind == STREAM_GIF ? "streams" : "frames");
		return -1;
	}
	StreamGeometry g;
	int rc;
	switch (req.kind) {
	case STREAM_PNG:
		rc = dev_png_decode_batch(domain, bufs, lens, n, out, out_bpl, out_frame_stride, &g, s);
		break;
	case STREAM_GIF:
		rc = dev_gif_decode_batch(domain, bufs, lens, n, req.page, req.n_pages, out, out_bpl, out_frame_stride, &g, s);
		break;
	case STREAM_TIFF:
		rc = dev_tiff_decode_batch(domain, bufs, lens, n, req.page, req.n_pages, req.subifd, out, out_bpl, out_frame_stride, &g, s);
		break;
	case STREAM_WEBP:
		rc = dev_webp_decode_batch(domain, bufs, lens, n, req.scale, out, out_bpl, out_frame_stride, &g, s);
		break;
	default:
		rc = dev_jpeg_decode_batch(domain, bufs, lens, n, req.shrink, out, out_bpl, out_frame_stride, &g, s);
	}
	if (rc)
		return -1;
	if (w)
		*w = g.w;
	if (h)
		*h = g.rows();
	if (bands)
		*bands = g.bands;
	if (page_h)
		*page_h = g.pages > 1 ? g.h : 0;
	return 0;
}

int
decode_batch_abi(const char *domain, const DecodeRequest &req, const void *const *bufs, const size_t *lens, int n, void *out, int out_location,
	size_t out_bpl, size_t out_frame_stride, int *width, int *height, int *bands)
{
	/* one frame has no frame stride to respect */
	const size_t frame_stride = n > 1 ? out_frame_stride : SIZE_MAX;
	int w = 0, h = 0, b = 0;
	if (!out) {
		/* geometry only: the headers, no device */
		if (dev_decode_batch(domain, req, bufs, lens, n, nullptr, 0, 0, &w, &h, &b, nullptr, nullptr))
			return -1;
	}
	else {
		if (ensure_init(domain))
			return -1;
		cudaStream_t s = current_stream();
		if (out_location == VB200_DEVICE) {
			if (dev_decode_batch(domain, req, bufs, lens, n, out, out_bpl, frame_stride, &w, &h, &b, nullptr, s))
				return -1;
		}
		else {
			if (dev_decode_batch(domain, req, bufs, lens, n, nullptr, 0, 0, &w, &h, &b, nullptr, s) ||
				check_out_strides(domain, StreamGeometry{w, h, b, 0}, out_bpl, frame_stride))
				return -1;
			/* decoded whole on the device first: a batch that fails leaves the caller's memory as it was */
			const size_t line = (size_t) w * b;
			void *dev = nullptr;
			if (dev_alloc(domain, &dev, line * h * n, s))
				return -1;
			int rc = dev_decode_batch(domain, req, bufs, lens, n, dev, line, line * h, nullptr, nullptr, nullptr, nullptr, s);
			for (int i = 0; i < n && !rc; i++)
				if (cudaMemcpy2DAsync((char *) out + (size_t) i * out_frame_stride, out_bpl, (char *) dev + (size_t) i * line * h, line, line, h,
						cudaMemcpyDeviceToHost, s) != cudaSuccess)
					rc = cuda_fail(domain, cudaGetLastError(), "copy to host");
			if (!rc && cudaStreamSynchronize(s) != cudaSuccess)
				rc = cuda_fail(domain, cudaGetLastError(), "decode");
			dev_free(dev, s);
			if (rc)
				return -1;
		}
	}
	if (width)
		*width = w;
	if (height)
		*height = h;
	if (bands)
		*bands = b;
	return 0;
}

int
dev_load(const char *domain, const DecodeRequest &req, const void *buf, size_t len, DevImage *out, int *page_h, cudaStream_t s)
{
	int w, h, b;
	if (dev_decode_batch(domain, req, &buf, &len, 1, nullptr, 0, 0, &w, &h, &b, page_h, s))
		return -1;
	if (dev_image_new(domain, out, w, h, b, VB200_FORMAT_UCHAR, b <= 2 ? VB200_INTERPRETATION_B_W : VB200_INTERPRETATION_sRGB, s))
		return -1;
	if (dev_decode_batch(domain, req, &buf, &len, 1, out->data, out->bpl, out->bpl * h, nullptr, nullptr, nullptr, nullptr, s)) {
		dev_image_release(out, s);
		return -1;
	}
	return 0;
}

int
load_abi(const char *domain, const DecodeRequest &req, const void *buf, size_t len, VB200Image *out)
{
	if (!buf || !out) {
		error(domain, "null argument");
		return -1;
	}
	if (ensure_init(domain))
		return -1;
	cudaStream_t s = current_stream();
	DevImage d;
	if (dev_load(domain, req, buf, len, &d, nullptr, s))
		return -1;
	VB200Image like = *out;
	return deliver(domain, &d, &like, out, s);
}

} // namespace vb200

extern "C" void
vb200_debug_png_set_budget(size_t bytes)
{
	vb200::g_chunk_budget = bytes;
}
