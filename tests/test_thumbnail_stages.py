"""How the thumbnail plan's stages compose over one device batch: the resize stage (with a linear plan's colour management
inside it), then the ICC stage of a plan that is not linear, then sharpen.

Launch counts pin what each stage adds to the plain batch on the same frames, and one case of each plan the leaf kernels
run (2 bands, upsizing, a one-axis shrink, and a linear colour-managed batch without the two-kernel path) is held to the
oracle or to the two-kernel path."""
import ctypes as C
import os

import numpy as np
import pytest

PROFILES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "profiles")


def P(name):
    with open(os.path.join(PROFILES, name), "rb") as f:
        return f.read()


SRGB, P3 = P("sRGB.icm"), P("p3.icm")
SHARPEN = (0.5, 2.0, 10.0, 20.0, 0.0, 3.0)  # ThumbnailPlan.set_sharpen's defaults


def _frames(seed, shape):
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def _run(vb, plan, din, embedded=None):
    """(output, kernel launches) of one device batch"""
    import torch
    dout = torch.empty((din.shape[0], plan.out_height, plan.out_width, plan.out_bands), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    before = vb.launch_count()
    plan.run_device(din.data_ptr(), dout.data_ptr(), din.shape[0], embedded=embedded)
    launches = vb.launch_count() - before
    torch.cuda.synchronize()
    return dout, launches


def _sharpen(vb, x):
    """vb200_sharpen_batch_device over a device batch: (output, kernel launches)"""
    import torch
    out = torch.empty_like(x)
    n, h, w, b = x.shape
    before = vb.launch_count()
    vb._check(vb.lib().vb200_sharpen_batch_device(C.c_void_p(x.data_ptr()), x[0].numel(), C.c_void_p(out.data_ptr()), out[0].numel(),
                                                  n, w, h, b, *SHARPEN))
    launches = vb.launch_count() - before
    torch.cuda.synchronize()
    return out, launches


def _with_env(env, make):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return make()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.mark.gpu
def test_gpu_sharpen_adds_its_own_launches(vb):
    import torch
    din = torch.from_numpy(_frames(1, (3, 64, 64, 3))).cuda()
    plan = vb.ThumbnailPlan(64, 64, 3, 16)
    plain, n0 = _run(vb, plan, din)
    assert _run(vb, plan, din)[1] == n0 > 0                  # the plain count is stable
    want, ns = _sharpen(vb, plain)
    plan.set_sharpen()
    got, n1 = _run(vb, plan, din)
    assert n1 == n0 + ns and torch.equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 32769])
def test_gpu_icc_stage_adds_one_launch_per_32768_frames(vb, n):
    import torch
    din = torch.from_numpy(_frames(2, (3, 16, 16, 3))[np.arange(n) % 3]).cuda()
    plan = vb.ThumbnailPlan(16, 16, 3, 4)
    _, n0 = _run(vb, plan, din)
    assert _run(vb, plan, din)[1] == n0 > 0
    plan.set_icc(SRGB, input_profile=P3)
    _, n1 = _run(vb, plan, din, embedded=[None] * n)
    assert n1 == n0 + (n + 32767) // 32768


@pytest.mark.gpu
def test_gpu_linear_icc_launches_as_plain_linear(vb):
    import torch
    din = torch.from_numpy(_frames(3, (3, 512, 512, 4))).cuda()
    plan = vb.ThumbnailPlan(512, 512, 4, 64, linear=True)
    assert plan.kernel == "linear_v_kernel + linear_h_kernel"
    _, n0 = _run(vb, plan, din)
    assert _run(vb, plan, din)[1] == n0 > 0
    plan.set_linear_icc(SRGB)
    _, n1 = _run(vb, plan, din, embedded=[P3, None, SRGB])
    assert n1 == n0
    plan.set_linear_icc(None)
    _, n2 = _run(vb, plan, din, embedded=[P3, None, SRGB])
    assert n2 == n0


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["2-band", "upsize", "one-axis"])
def test_gpu_leaf_chain_is_the_oracle(vb, oracle, case):
    import torch
    shape, args = {"2-band": ((2, 90, 120, 2), (40,)), "upsize": ((2, 50, 80, 4), (200,)),
                   "one-axis": ((2, 120, 160, 4), (40, 120, "force"))}[case]
    frames = _frames(4, shape)
    n, h, w, b = shape
    plan = vb.ThumbnailPlan(w, h, b, args[0], target_height=args[1] if len(args) > 1 else None, size=args[2] if len(args) > 2 else "both")
    assert plan.kernel == "leaf kernels"
    got, _ = _run(vb, plan, torch.from_numpy(frames).cuda())
    for i in range(n):
        want = oracle.thumbnail_image(frames[i], *args)
        assert np.array_equal(got[i].cpu().numpy(), want), (case, i)


@pytest.mark.gpu
@pytest.mark.parametrize("output", ["srgb", "none"])
def test_gpu_linear_icc_leaf_chain_then_sharpen(vb, output):
    """VB200_NO_LINEAR_FUSED: a batch of LIN_IMPORT and LIN_XYZ frames (with an output profile) or LIN_IMPORT and LIN_PLAIN
    frames (without), then sharpen, equals the two-kernel path followed by vb200_sharpen_batch_device"""
    import torch
    din = torch.from_numpy(_frames(5, (3, 512, 512, 4))).cuda()
    emb = [P3, None, SRGB]
    pout = SRGB if output == "srgb" else None

    def plan(env):
        p = _with_env(env, lambda: vb.ThumbnailPlan(512, 512, 4, 64, linear=True))
        p.set_linear_icc(pout)
        return p

    two = plan({})
    assert two.kernel == "linear_v_kernel + linear_h_kernel"
    mid, _ = _run(vb, two, din, embedded=emb)
    want, _ = _sharpen(vb, mid)
    leaf = plan({"VB200_NO_LINEAR_FUSED": "1"})
    assert leaf.kernel == "leaf kernels"
    leaf.set_sharpen()
    got, _ = _run(vb, leaf, din, embedded=emb)
    assert torch.equal(got, want)
