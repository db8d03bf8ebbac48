/* encode.cu -- what the JPEG and PNG encoders share around their kernels: the C ABI body of vb200_jpegsave_batch_opts and
 * vb200_pngsave_batch, and the one chunk loop that stages host frames, bounds device memory, checks every stream against
 * its slot and writes the streams to device slots or packs them for the host.
 */
#include <cstring>
#include <vector>

#include "../../include/vb200.h"
#include "vb200_internal.h"

namespace vb200 {

int
dev_encode_batch(const char *domain, const Encoder &enc, const void *frames, int frames_location, size_t bpl, size_t frame_stride, int n, size_t line,
	int h, EncodeDest &dst, size_t *lengths, cudaStream_t s)
{
	const bool host_in = frames_location != VB200_DEVICE, host_out = dst.bytes != nullptr;
	const size_t frame_in = line * h, per = enc.scratch_bytes + (host_in ? frame_in : 0) + (host_out ? enc.stream_bytes : 0);
	const size_t budget = chunk_budget();
	if (host_out)
		dst.at.resize(n);
	std::vector<unsigned char> raw;
	std::vector<unsigned long long> at;
	for (int c0 = 0; c0 < n;) {
		/* a frame larger than the budget runs alone */
		const int cn = (int) std::min<size_t>({(size_t) (n - c0), (size_t) kMaxBatchFrames, std::max<size_t>(1, budget / per)});
		const unsigned char *src = (const unsigned char *) frames + (size_t) c0 * frame_stride;
		size_t sbpl = bpl, sstride = frame_stride;
		unsigned char *din = nullptr, *packed = nullptr;
		unsigned long long packed_bytes = 0;
		int rc = 0;
		if (host_in) {
			if (dev_alloc(domain, (void **) &din, frame_in * cn, s))
				return -1;
			/* one copy when the chunk's frames are packed */
			const bool one = bpl == line && (cn == 1 || frame_stride == frame_in);
			cudaError_t e = one ? cudaMemcpyAsync(din, src, frame_in * cn, cudaMemcpyHostToDevice, s) : cudaSuccess;
			for (int i = 0; i < cn && !one && e == cudaSuccess; i++)
				e = cudaMemcpy2DAsync(din + i * frame_in, line, src + i * frame_stride, bpl, line, h, cudaMemcpyHostToDevice, s);
			if (e != cudaSuccess)
				rc = cuda_fail(domain, e, "copy to device");
			src = din;
			sbpl = line;
			sstride = frame_in;
		}
		/* the encoder's lengths back on the host: each stream checked against its slot and given its place */
		const EncodePlace place = [&](const void *lens, size_t len_stride, unsigned long long *d_at, unsigned char **out) {
			raw.resize((cn - 1) * len_stride + sizeof(unsigned long long));
			if (cudaMemcpyAsync(raw.data(), lens, raw.size(), cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess)
				return cuda_fail(domain, cudaGetLastError(), "encode kernels");
			at.resize(cn);
			for (int i = 0; i < cn; i++) {
				unsigned long long len;
				memcpy(&len, raw.data() + i * len_stride, sizeof(len));
				if (len > dst.slot) {
					error(domain, "frame %d: its %llu-byte stream does not fit the %zu-byte slot (out_stride)", c0 + i, len, dst.slot);
					return -1;
				}
				lengths[c0 + i] = len;
				at[i] = host_out ? packed_bytes : (unsigned long long) (c0 + i) * dst.slot;
				packed_bytes += len;
			}
			if (host_out && dev_alloc(domain, (void **) &packed, packed_bytes, s))
				return -1;
			if (cudaMemcpyAsync(d_at, at.data(), cn * sizeof(unsigned long long), cudaMemcpyHostToDevice, s) != cudaSuccess)
				return cuda_fail(domain, cudaGetLastError(), "stream offsets");
			*out = host_out ? packed : dst.dev;
			return 0;
		};
		if (!rc)
			rc = enc.chunk(src, sbpl, sstride, cn, place, s);
		/* the streams written: packed ones copied back in one piece */
		if (!rc) {
			cudaError_t e = cudaSuccess;
			if (host_out) {
				const size_t base = dst.bytes->size();
				dst.bytes->resize(base + packed_bytes);
				for (int i = 0; i < cn; i++)
					dst.at[c0 + i] = base + at[i];
				e = cudaMemcpyAsync(dst.bytes->data() + base, packed, packed_bytes, cudaMemcpyDeviceToHost, s);
			}
			if (e != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess)
				rc = cuda_fail(domain, e != cudaSuccess ? e : cudaGetLastError(), "encode");
		}
		if (packed)
			dev_free(packed, s);
		if (din)
			dev_free(din, s);
		if (rc)
			return -1;
		c0 += cn;
	}
	return 0;
}

int
encode_batch_abi(const char *domain, const void *options, const std::function<int(Encoder *)> &make, const void *frames, int frames_location,
	size_t bpl, size_t frame_stride, int n, int w, int h, int bands, void *out, int out_location, size_t out_stride, size_t *lengths)
{
	if (!frames || !out || !options || n < 1) {
		error(domain, "null argument");
		return -1;
	}
	if (bpl < (size_t) w * bands || (n > 1 && frame_stride < bpl * h)) {
		error(domain, "frame strides too small for %d x %d x %d", w, h, bands);
		return -1;
	}
	Encoder enc;
	if (make(&enc) || ensure_init(domain))
		return -1;
	/* host slots: the streams packed on the host first, so that a batch that fails leaves the caller's memory as it was;
	 * the thread's packing buffer is kept, so that a batch does not fault in fresh pages */
	static thread_local std::vector<unsigned char> bytes;
	bytes.clear();
	EncodeDest dst;
	dst.slot = out_stride;
	if (out_location == VB200_DEVICE)
		dst.dev = (unsigned char *) out;
	else
		dst.bytes = &bytes;
	std::vector<size_t> len(n);
	if (dev_encode_batch(domain, enc, frames, frames_location, bpl, frame_stride, n, (size_t) w * bands, h, dst, len.data(), current_stream()))
		return -1;
	if (dst.bytes)
		for (int i = 0; i < n; i++)
			memcpy((unsigned char *) out + (size_t) i * out_stride, bytes.data() + dst.at[i], len[i]);
	if (lengths)
		memcpy(lengths, len.data(), n * sizeof(size_t));
	return 0;
}

} // namespace vb200
