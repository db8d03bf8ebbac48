#include <algorithm>
/* runtime.cu -- init, error buffer, stream and memory plumbing of libvb200.so.
 *
 * Mirrors the reference's conventions: 0 / -1 returns with a text buffer
 * (libvips/iofuncs/error.c:120-350), an on/off switch like
 * vips_vector_isenabled() (iofuncs/vector.cpp:83-110, env VB200_DISABLE like
 * VIPS_NOVECTOR), and tile-geometry globals (iofuncs/thread.c:74-77).
 */
#include <atomic>
#include <cctype>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>

#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>

#include "vb200_internal.h"

namespace vb200 {

static thread_local std::string g_error;
static thread_local cudaStream_t g_stream = nullptr;
static std::atomic<uint64_t> g_launches{0};
static std::atomic<int> g_device{-1};
static std::atomic<int> g_sm_count{132};
static std::mutex g_init_lock;
/* reference: VIPS__TILE_WIDTH/HEIGHT 128, FATSTRIP 16, THINSTRIP 1,
 * include/vips/private.h:147-153
 */
static TileGeometry g_tiles = {128, 128, 16, 1};
static std::mutex g_tiles_lock;
/* the device this thread's CUDA runtime is bound to: generate() callbacks arrive on worker threads
 * the library has never seen (iofuncs/region.c:1600-1626), and a fresh thread defaults to device 0
 */
static thread_local int t_bound_device = -1;

void
error(const char *domain, const char *fmt, ...)
{
	char buf[1024];
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(buf, sizeof(buf), fmt, ap);
	va_end(ap);
	g_error += domain;
	g_error += ": ";
	g_error += buf;
	g_error += "\n";
}

void
error_truncate(size_t len)
{
	if (g_error.size() > len)
		g_error.resize(len);
}

int
cuda_fail(const char *domain, cudaError_t e, const char *what)
{
	error(domain, "CUDA error %s (%s) in %s", cudaGetErrorName(e), cudaGetErrorString(e), what);
	return -1;
}

cudaStream_t
current_stream()
{
	return g_stream;
}

void
count_launch(int n)
{
	g_launches.fetch_add(n, std::memory_order_relaxed);
}

int
sm_count()
{
	return g_sm_count.load(std::memory_order_relaxed);
}

TileGeometry
tile_geometry()
{
	std::lock_guard<std::mutex> lock(g_tiles_lock);
	return g_tiles;
}

int
ensure_init(const char *domain)
{
	int dev = g_device.load();
	if (dev < 0) {
		if (vb200_init(0)) {
			error(domain, "libvb200 is not initialised and no CUDA device is usable");
			return -1;
		}
		dev = g_device.load();
	}
	if (t_bound_device != dev) {
		VB200_CUDA(domain, cudaSetDevice(dev));
		t_bound_device = dev;
	}
	return 0;
}

int
dev_alloc(const char *domain, void **p, size_t bytes, cudaStream_t s)
{
	*p = nullptr;
	if (bytes == 0)
		bytes = 16;
	VB200_CUDA(domain, cudaMallocAsync(p, bytes, s));
	return 0;
}

void
dev_free(void *p, cudaStream_t s)
{
	if (p)
		cudaFreeAsync(p, s);
}

size_t
format_sizeof(int fmt)
{
	switch (fmt) {
	case VB200_FORMAT_UCHAR:
	case VB200_FORMAT_CHAR:
		return 1;
	case VB200_FORMAT_USHORT:
	case VB200_FORMAT_SHORT:
		return 2;
	case VB200_FORMAT_UINT:
	case VB200_FORMAT_INT:
	case VB200_FORMAT_FLOAT:
		return 4;
	case VB200_FORMAT_COMPLEX:
	case VB200_FORMAT_DOUBLE:
		return 8;
	case VB200_FORMAT_DPCOMPLEX:
		return 16;
	}
	return 0;
}

bool
format_is_supported(int fmt)
{
	switch (fmt) {
	case VB200_FORMAT_UCHAR:
	case VB200_FORMAT_CHAR:
	case VB200_FORMAT_USHORT:
	case VB200_FORMAT_SHORT:
	case VB200_FORMAT_UINT:
	case VB200_FORMAT_INT:
	case VB200_FORMAT_FLOAT:
		return true;
	}
	return false;
}

int
interpretation_bands(int type)
{
	/* reference: vips_interpretation_bands, iofuncs/header.c:217-249 (the interpretations this ABI names) */
	switch (type) {
	case VB200_INTERPRETATION_B_W:
	case VB200_INTERPRETATION_GREY16:
		return 1;
	case VB200_INTERPRETATION_XYZ:
	case VB200_INTERPRETATION_LAB:
	case VB200_INTERPRETATION_LABS:
	case VB200_INTERPRETATION_sRGB:
	case VB200_INTERPRETATION_RGB16:
	case VB200_INTERPRETATION_scRGB:
	case 17: /* RGB */
	case 18: /* CMC */
	case 19: /* LCH */
	case 23: /* YXY */
	case 29: /* HSV */
		return 3;
	case VB200_INTERPRETATION_CMYK:
		return 4;
	default:
		return 0;
	}
}

bool
image_hasalpha(int type, int bands)
{
	/* reference: vips_image_hasalpha, iofuncs/image.c:3113-3119 */
	const int real = interpretation_bands(type);
	return real > 0 && bands > real;
}

double
interpretation_max_alpha(int type)
{
	/* reference: vips_interpretation_max_alpha, iofuncs/header.c:195-206 */
	switch (type) {
	case VB200_INTERPRETATION_GREY16:
	case VB200_INTERPRETATION_RGB16:
		return 65535.0;
	case VB200_INTERPRETATION_scRGB:
		return 1.0;
	default:
		return 255.0;
	}
}

int
dev_image_new(const char *domain, DevImage *d, int w, int h, int bands, int fmt, int type, cudaStream_t s)
{
	d->w = w;
	d->h = h;
	d->bands = bands;
	d->fmt = fmt;
	d->type = type;
	const size_t line = (size_t) w * bands * format_sizeof(fmt);
	const size_t es = format_sizeof(fmt);
	if (d->preset && d->data && (uintptr_t) d->data % es == 0 && d->bpl % es == 0) {
		/* the caller's buffer (preset_output): sized by contract for this op's result */
		d->preset = false;
		d->owned = false;
		if (d->bpl < line)
			d->bpl = line;
		return 0;
	}
	/* a caller's buffer off the element grid of this result is not written by the kernel: deliver() copies into it */
	d->preset = false;
	d->bpl = line;
	d->owned = true;
	return dev_alloc(domain, &d->data, d->bpl * h, s);
}

void
preset_output(DevImage *dout, const VB200Image *in, const VB200Image *out, size_t out_line_bytes, int out_rows)
{
	if (in->where != VB200_DEVICE || !out->data || !in->data)
		return;
	const size_t in_bytes = (in->bpl ? in->bpl : (size_t) in->Xsize * in->Bands * format_sizeof(in->BandFmt)) * in->Ysize;
	const char *a = (const char *) in->data, *o = (const char *) out->data;
	/* no aliasing: the result (out_rows lines of out_line_bytes, at the caller's stride if that is
	 * larger) must lie wholly before or after the input
	 */
	const size_t out_line = std::max((size_t) out->bpl, out_line_bytes);
	if (o >= a + in_bytes || o + out_line * (size_t) out_rows <= a) {
		dout->data = out->data;
		dout->bpl = out->bpl;
		dout->preset = true;
	}
}

void
dev_image_release(DevImage *d, cudaStream_t s)
{
	if (d->owned && d->data)
		dev_free(d->data, s);
	d->data = nullptr;
	d->owned = false;
}

int
to_device(const char *domain, const VB200Image *in, DevImage *d, cudaStream_t s)
{
	if (!in || !in->data) {
		error(domain, "no input image");
		return -1;
	}
	if (in->Xsize <= 0 || in->Ysize <= 0 || in->Bands <= 0) {
		error(domain, "bad image dimensions %d x %d x %d", in->Xsize, in->Ysize, in->Bands);
		return -1;
	}
	const size_t line = (size_t) in->Xsize * in->Bands * format_sizeof(in->BandFmt);
	if (line == 0) {
		error(domain, "unknown band format %d", in->BandFmt);
		return -1;
	}
	const size_t bpl = in->bpl ? in->bpl : line;
	/* checked before any copy or launch: a shorter stride makes rows overlap and the last row run past the buffer */
	if (bpl < line) {
		error(domain, "line stride %zu too small for %d x %d x %zu bytes", bpl, in->Xsize, in->Bands, format_sizeof(in->BandFmt));
		return -1;
	}
	/* kernels read rows as arrays of the element type: a device base or stride off that grid is a misaligned load */
	const size_t es = format_sizeof(in->BandFmt);
	if (in->where == VB200_DEVICE && (((uintptr_t) in->data % es) != 0 || bpl % es != 0)) {
		error(domain, "device image data %p / line stride %zu not a multiple of the %zu-byte element", in->data, bpl, es);
		return -1;
	}

	d->w = in->Xsize;
	d->h = in->Ysize;
	d->bands = in->Bands;
	d->fmt = in->BandFmt;
	d->type = in->Type;
	if (in->where == VB200_DEVICE) {
		d->data = in->data;
		d->bpl = bpl;
		d->owned = false;
		return 0;
	}
	d->bpl = line;
	d->owned = true;
	if (dev_alloc(domain, &d->data, line * in->Ysize, s))
		return -1;
	VB200_CUDA(domain,
		cudaMemcpy2DAsync(d->data, line, in->data, bpl, line, in->Ysize, cudaMemcpyHostToDevice, s));
	return 0;
}

void
adopt_pass_through(DevImage *in, DevImage *out)
{
	if (out->data == in->data) {
		out->owned = in->owned;
		in->owned = false;
	}
}

static void
describe(const DevImage &d, int where, VB200Image *out)
{
	out->Xsize = d.w;
	out->Ysize = d.h;
	out->Bands = d.bands;
	out->BandFmt = d.fmt;
	out->Type = d.type;
	out->where = where;
}

int
deliver_host(const char *domain, DevImage *d, const VB200Image *like, VB200Image *out, cudaStream_t s)
{
	const size_t line = (size_t) d->w * d->bands * format_sizeof(d->fmt);
	void *dst = out->data;
	const size_t dst_bpl = (out->data && out->bpl) ? out->bpl : line;
	if (!dst) {
		dst = malloc(line * d->h > 0 ? line * d->h : 1);
		if (!dst) {
			error(domain, "out of memory");
			return -1;
		}
	}
	describe(*d, like->where, out);
	out->data = dst;
	out->bpl = dst_bpl;
	VB200_CUDA(domain, cudaMemcpy2DAsync(dst, dst_bpl, d->data, d->bpl, line, d->h, cudaMemcpyDeviceToHost, s));
	dev_image_release(d, s);
	return 0;
}

int
deliver(const char *domain, DevImage *d, const VB200Image *like, VB200Image *out, cudaStream_t s)
{
	if (like->where != VB200_DEVICE) {
		if (deliver_host(domain, d, like, out, s))
			return -1;
		VB200_CUDA(domain, cudaStreamSynchronize(s));
		return 0;
	}
	const size_t line = (size_t) d->w * d->bands * format_sizeof(d->fmt);
	void *dst = out->data;
	size_t dst_bpl = (out->data && out->bpl) ? out->bpl : line;
	describe(*d, like->where, out);
	if (!dst && d->owned) {
		/* hand our buffer over */
		out->data = d->data;
		out->bpl = d->bpl;
		d->owned = false;
		return 0;
	}
	if (dst && dst == d->data) {
		/* the op wrote into the caller's buffer (preset_output) */
		out->bpl = d->bpl;
		return 0;
	}
	if (!dst) {
		if (dev_alloc(domain, &dst, line * d->h, s))
			return -1;
		out->data = dst;
	}
	out->bpl = dst_bpl;
	VB200_CUDA(domain, cudaMemcpy2DAsync(dst, dst_bpl, d->data, d->bpl, line, d->h, cudaMemcpyDeviceToDevice, s));
	dev_image_release(d, s);
	return 0;
}

} // namespace vb200

using namespace vb200;

extern "C" int
vb200_init(int device)
{
	std::lock_guard<std::mutex> lock(g_init_lock);
	int n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if (e != cudaSuccess || n <= 0) {
		error("vb200_init", "no CUDA device (%s)", cudaGetErrorString(e));
		return -1;
	}
	if (device < 0 || device >= n) {
		error("vb200_init", "device %d out of range (%d visible)", device, n);
		return -1;
	}
	VB200_CUDA("vb200_init", cudaSetDevice(device));
	cudaDeviceProp prop;
	VB200_CUDA("vb200_init", cudaGetDeviceProperties(&prop, device));
	if (prop.major != 9 || prop.minor != 0) {
		error("vb200_init", "device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major,
			prop.minor);
		return -1;
	}
	/* keep freed scratch in the pool instead of returning it to the driver */
	cudaMemPool_t pool;
	if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
		uint64_t threshold = UINT64_MAX;
		cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &threshold);
	}
	g_sm_count.store(prop.multiProcessorCount);
	g_device.store(device);
	t_bound_device = device;
	return 0;
}

extern "C" void
vb200_shutdown(void)
{
	std::lock_guard<std::mutex> lock(g_init_lock);
	if (g_device.load() >= 0) {
		cudaDeviceSynchronize();
		resample_cache_clear();
		jpeg_pump_release();
		decode_staging_release();
	}
	g_device.store(-1);
}

extern "C" const char *
vb200_error_buffer(void)
{
	return g_error.c_str();
}

extern "C" void
vb200_error_clear(void)
{
	g_error.clear();
}

extern "C" int
vb200_isenabled(void)
{
	const char *off = getenv("VB200_DISABLE");
	if (off && *off && strcmp(off, "0") != 0)
		return 0;
	int n = 0;
	return cudaGetDeviceCount(&n) == cudaSuccess && n > 0;
}

extern "C" void
vb200_set_stream(void *cuda_stream)
{
	g_stream = (cudaStream_t) cuda_stream;
}

extern "C" void *
vb200_get_stream(void)
{
	return (void *) g_stream;
}

extern "C" void
vb200_set_tile_geometry(int tile_width, int tile_height, int fatstrip_height, int thinstrip_height)
{
	std::lock_guard<std::mutex> lock(g_tiles_lock);
	if (tile_width > 0)
		g_tiles.tile_width = tile_width;
	if (tile_height > 0)
		g_tiles.tile_height = tile_height;
	if (fatstrip_height > 0)
		g_tiles.fatstrip_height = fatstrip_height;
	if (thinstrip_height > 0)
		g_tiles.thinstrip_height = thinstrip_height;
}

extern "C" uint64_t
vb200_launch_count(void)
{
	return g_launches.load();
}

extern "C" void
vb200_image_free(VB200Image *image)
{
	if (!image || !image->data)
		return;
	if (image->where == VB200_DEVICE)
		cudaFree(image->data);
	else
		free(image->data);
	image->data = nullptr;
}

extern "C" size_t
vb200_format_sizeof(int band_format)
{
	return format_sizeof(band_format);
}

/* ---------------------------------------------------------------- pinned host memory
 * The pump's host buffers: page-locked, and placed on the NUMA node the GPU hangs off (on the 8-GPU
 * boxes GPUs 4-7 sit on node 1; a plain cudaHostAlloc from a process that runs on node 0 makes every
 * H2D copy of those ranks cross the socket interconnect).  mmap + mbind(MPOL_PREFERRED) + first touch
 * + cudaHostRegister; any failure falls back to cudaHostAlloc.
 */
namespace {

std::mutex g_host_lock;
std::map<void *, size_t> g_host_registered; /* mmap'ed + registered blocks */

int
gpu_numa_node(int device)
{
	char bus[64];
	if (device < 0 || cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) {
		cudaGetLastError();
		return -1;
	}
	for (char *c = bus; *c; c++)
		*c = (char) tolower(*c);
	char path[160];
	snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
	FILE *f = fopen(path, "r");
	if (!f)
		return -1;
	int node = -1;
	if (fscanf(f, "%d", &node) != 1)
		node = -1;
	fclose(f);
	if (node < 0)
		return -1;
	/* only worth it on a machine with more than one node */
	if (access("/sys/devices/system/node/node1", F_OK) != 0)
		return -1;
	return node;
}

void *
numa_pinned_alloc(size_t bytes, int node)
{
	const size_t huge = (size_t) 2 << 20;
	const size_t len = (bytes + huge - 1) & ~(huge - 1);
	void *p = mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
	if (p == MAP_FAILED)
		return nullptr;
#ifdef SYS_mbind
	unsigned long mask[16];
	memset(mask, 0, sizeof(mask));
	mask[node / (8 * sizeof(unsigned long))] |= 1UL << (node % (8 * sizeof(unsigned long)));
	/* MPOL_PREFERRED = 1: pages come from `node` while it has memory, never an OOM kill */
	if (syscall(SYS_mbind, p, len, 1, mask, (unsigned long) (8 * sizeof(mask) + 1), 0) != 0) {
		munmap(p, len);
		return nullptr; /* no policy, no point: let cudaHostAlloc do it */
	}
#else
	munmap(p, len);
	return nullptr;
#endif
	memset(p, 0, len); /* first touch under the policy */
	if (cudaHostRegister(p, len, cudaHostRegisterDefault) != cudaSuccess) {
		cudaGetLastError();
		munmap(p, len);
		return nullptr;
	}
	std::lock_guard<std::mutex> lock(g_host_lock);
	g_host_registered[p] = len;
	return p;
}

} // namespace

extern "C" void *
vb200_host_alloc(size_t bytes)
{
	if (ensure_init("host_alloc"))
		return nullptr;
	if (bytes == 0)
		bytes = 1;
	const char *off = getenv("VB200_NO_NUMA");
	if (!(off && *off && strcmp(off, "0") != 0)) {
		const int node = gpu_numa_node(g_device.load());
		if (node >= 0) {
			void *p = numa_pinned_alloc(bytes, node);
			if (p)
				return p;
		}
	}
	void *p = nullptr;
	if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess)
		return nullptr;
	return p;
}

extern "C" void
vb200_host_free(void *p)
{
	if (!p)
		return;
	size_t len = 0;
	{
		std::lock_guard<std::mutex> lock(g_host_lock);
		auto it = g_host_registered.find(p);
		if (it != g_host_registered.end()) {
			len = it->second;
			g_host_registered.erase(it);
		}
	}
	if (len) {
		cudaHostUnregister(p);
		munmap(p, len);
	}
	else
		cudaFreeHost(p);
}

/* the NUMA node of the current device (-1: unknown or a single-node machine); the host binding
 * may want to run its feeder threads there (bench.py does)
 */
extern "C" int
vb200_device_numa_node(void)
{
	return gpu_numa_node(g_device.load());
}
