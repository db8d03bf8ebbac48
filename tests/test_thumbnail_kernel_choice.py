"""Which fused thumbnail kernel a plan runs.

The plan chooses the kernel once (plan_build_fused): the tensor-pipe kernel where its tables, bands and shared memory fit
and its (VS, HS) box pair is instantiated, else the TMA-fed kernel where rows are 16-byte aligned and a band fits its
stage, else the ld.global kernel.  A batch call launches that kernel, template arguments included, except for a batch
whose base pointer or frame stride is off 16 bytes, which runs the ld.global kernel.  The CPU tests pin the names
through the host-only hook vb200_debug_thumbnail_kernel; the GPU test runs two host threads on one plan."""
import ctypes as C
import re
import threading

import numpy as np
import pytest

import libvips_b200 as vb

SIZES = {"both": 0, "force": 3}


def mma(vs, np_, hs, alpha="premul"):
    return "thumbnail_fused_mma_kernel<VS=%d,NP=%d,%s,HS=%d,cols=768,cpt=2>" % (vs, np_, alpha, hs)


def kernel_name(w, h, tw, th=None, size="both", alpha=True, bands=4):
    L = C.CDLL(vb.library_path())
    L.vb200_debug_thumbnail_kernel.argtypes = [C.c_int] * 7 + [C.c_char_p, C.c_int]
    buf = C.create_string_buffer(160)
    rc = L.vb200_debug_thumbnail_kernel(w, h, bands, int(alpha), tw, th or 0, SIZES[size], buf, len(buf))
    assert rc == 0, (w, h, tw, th, size)
    return buf.value.decode()


# (W, H, target_w, target_h, size, has_alpha): the rows of test_resample_gpu.V4_CASES, then the other families
CHOICES = [
    ((2048, 2048, 256, None, "both", True), mma(4, 6, 4)),
    ((1024, 1024, 256, None, "both", True), mma(2, 6, 2)),
    ((1600, 1200, 200, None, "both", True), mma(4, 6, 4)),
    ((2048, 1024, 256, 256, "force", True), mma(2, 0, 4)),
    ((1024, 2048, 256, 256, "force", True), mma(4, 0, 2)),
    ((4096, 512, 256, 128, "force", True), mma(2, 0, 8)),
    ((1600, 1600, 200, None, "both", False), mma(4, 6, 4, "plain")),
    ((4096, 4096, 512, None, "both", True), mma(4, 6, 4)),            # the headline
    ((2000, 1000, 420, None, "both", True), mma(2, 0, 2)),
    ((3000, 2000, 640, None, "both", True), mma(2, 0, 2)),
    ((4000, 3000, 410, None, "both", True), mma(4, 0, 4)),
    ((4096, 4096, 256, None, "both", True), mma(8, 6, 8)),
    ((3840, 2160, 225, None, "both", True), mma(8, 7, 8)),
    ((1200, 900, 150, None, "both", True), mma(3, 0, 4)),
    ((3000, 2000, 428, None, "both", True), mma(3, 0, 3)),
    ((2400, 1800, 340, None, "both", False), mma(3, 0, 3, "plain")),
    ((4000, 3000, 364, None, "both", True), mma(5, 0, 5)),
    ((4096, 4096, 320, None, "both", True), mma(6, 0, 6)),
    ((4096, 4096, 280, None, "both", True), mma(7, 0, 7)),
    ((1920, 1080, 274, None, "both", True), mma(3, 0, 3)),
    ((2048, 1536, 256, 256, "force", True), mma(3, 0, 4)),
    ((4096, 2048, 500, None, "both", True), mma(4, 7, 4)),
    ((1003, 2057, 120, None, "both", True), "thumbnail_fused_kernel<VS=8,premul>"),      # rows off 16 bytes
    ((2560, 1280, 256, 183, "force", True), "thumbnail_fused_tma_kernel<VS=3,NP=0,premul>"),  # boxes 3 / 10
    ((1024, 4096, 256, 256, "force", True), "thumbnail_fused_kernel<VS=8,premul>"),      # (8, 2): no v4 instantiation
    ((1000, 1000, 400, None, "both", True), "thumbnail_fused_tma_kernel<VS=1,NP=0,premul>"),  # box 1
    ((4096, 4096, 150, None, "both", True), "thumbnail_fused_kernel<VS=0(13),premul>"),  # box 13: the run-time form
    ((2052, 2052, 128, None, "both", True), "thumbnail_fused_kernel<VS=8,premul>"),      # box 8 cut short at the right edge
]


@pytest.mark.parametrize("case,want", CHOICES, ids=lambda c: "%dx%d-%s-%s" % c[:4] if isinstance(c, tuple) else "")
def test_plan_kernel_choice(case, want):
    w, h, tw, th, size, alpha = case
    assert kernel_name(w, h, tw, th, size, alpha) == want


def test_plan_kernel_choice_other_bands():
    """3-band frames ride the RGBA kernels without premultiply; an enlarging plan and 2-band frames take the leaf kernels"""
    assert kernel_name(1200, 900, 150, alpha=False, bands=3) == mma(3, 0, 4, "plain")
    assert kernel_name(100, 100, 400) == "leaf kernels"
    assert kernel_name(100, 100, 50, bands=2) == "leaf kernels"


# the instantiations of thumbnail_fused_mma_kernel (VB200_V4_LIST in thumbnail_fused.cu)
V4_LIST = {(4, 6, 4), (4, 7, 4), (2, 6, 2), (2, 7, 2), (8, 6, 8), (8, 7, 8),
           (4, 0, 4), (2, 0, 2), (4, 0, 2), (2, 0, 4), (4, 0, 8), (2, 0, 8), (8, 0, 8), (8, 0, 4),
           (3, 0, 3), (5, 0, 5), (6, 0, 6), (7, 0, 7), (2, 0, 3), (3, 0, 2), (3, 0, 4), (4, 0, 3),
           (4, 0, 5), (5, 0, 4), (5, 0, 6), (6, 0, 5), (6, 0, 7), (7, 0, 6), (7, 0, 8), (8, 0, 7)}


def test_plan_names_only_instantiated_tensor_pipe_kernels():
    """Over a grid of frame sizes and targets, uniform and forced, a plan never names a v4 instantiation that does
    not exist"""
    seen = set()
    for w, h in [(4096, 4096), (3840, 2160), (4032, 3024), (6000, 4000), (1920, 1080), (1024, 4096), (2048, 512)]:
        for t in range(64, 1025, 24):
            for th, size in ((None, "both"), (min(t // 2 + 1, h), "force"), (min(t * 2, h), "force")):
                name = kernel_name(w, h, t, th, size)
                m = re.fullmatch(r"thumbnail_fused_mma_kernel<VS=(\d+),NP=(\d+),premul,HS=(\d+),cols=768,cpt=2>", name)
                if m:
                    key = tuple(int(g) for g in m.groups())
                    assert key in V4_LIST, (w, h, t, th, size, name)
                    seen.add(key)
                else:
                    assert re.fullmatch(r"thumbnail_fused_tma_kernel<VS=([1-48]|0\(\d+\)),NP=[067],premul>|"
                                        r"thumbnail_fused_kernel<VS=([1-68]|0\(\d+\)),premul>|leaf kernels", name), name
    assert len(seen) >= 10, seen


def test_debug_thumbnail_kernel_bad_arguments():
    L = C.CDLL(vb.library_path())
    L.vb200_debug_thumbnail_kernel.argtypes = [C.c_int] * 7 + [C.c_char_p, C.c_int]
    buf = C.create_string_buffer(8)
    assert L.vb200_debug_thumbnail_kernel(0, 4096, 4, 1, 512, 0, 0, buf, len(buf)) == -1
    assert L.vb200_debug_thumbnail_kernel(4096, 4096, 4, 1, 512, 0, 0, buf, len(buf)) == -1  # name longer than the buffer


@pytest.mark.gpu
def test_two_threads_share_a_plan_on_the_ldg_path(vb, oracle):
    """Two host threads run one plan at once, both on the ld.global kernel (base pointer 4 bytes off 16), with batches
    of 1 and 40 frames, so their rows per CTA differ: the per-launch geometry is the caller's, never the plan's"""
    import torch
    w, h, tw = 1024, 512, 128
    rng = np.random.default_rng(5)
    frames = rng.integers(0, 256, (40, h, w, 4), dtype=np.uint8)
    want = np.stack([oracle.thumbnail_image(f, tw) for f in frames])
    plan = vb.ThumbnailPlan(w, h, 4, tw)
    assert plan.fused, plan.kernel
    L = vb.lib()
    L.vb200_thumbnail_batch_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
    frame_bytes = h * w * 4
    raw = torch.from_numpy(np.concatenate([np.zeros(4, np.uint8), frames.reshape(-1)])).cuda()
    torch.cuda.synchronize()
    results, errors = {}, []

    def run(n, rounds=20):
        try:
            stream = torch.cuda.Stream()
            out = torch.zeros((n, plan.out_height, plan.out_width, 4), dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            with torch.cuda.stream(stream):
                vb.set_stream(stream.cuda_stream)
                for _ in range(rounds):
                    vb._check(L.vb200_thumbnail_batch_device(plan._p, raw.data_ptr() + 4, frame_bytes, out.data_ptr(),
                                                             plan.out_frame_bytes, n))
                stream.synchronize()
            results[n] = out.cpu().numpy()
        except Exception as e:  # noqa: BLE001 -- reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=run, args=(n,)) for n in (1, 40)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    np.testing.assert_array_equal(results[1], want[:1])
    np.testing.assert_array_equal(results[40], want)
