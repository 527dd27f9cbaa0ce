"""bfloat16 templates with their gradient accumulated in fp32 (MVP_FLAG_TPLATE_BF16 | MVP_FLAG_GRAD_TPLATE_F32) on the emulated
product kernels, against the fp32 kernels on the widened template.

The template is read as bf16 and widened exactly, and everything after the load is the fp32 kernels' arithmetic, the template
gradient's fp32 reduction included.  So images and raysat must be bit-identical to the fp32 run on `from_bf16(tb)`, and every
gradient, the template's included, equal to it within the order of the fp32 atomics (TOL of max|.|).  The template gradient
buffer is fp32 [N,K,TD,TH,TW,4]: twice the bf16 gradient's size, so a stride, clear or memset that still counts bf16 words
leaves half of it NaN or mixes up voxels, which the comparison catches.  The bf16 template goes through the emulation's
front-end as in tests/test_emul_bf16_payload.py: uint16 bit patterns in fp32-typed words.  The fp32 reference runs through
that front-end (tests/emul/kernels.py); the bf16 run with its fp32 gradient buffer through forward_backward_f32 below, which
makes the same C-ABI calls with a template gradient of [..., 4] fp32 words."""
import ctypes

import numpy as np
import pytest

from tests.helpers import CASES, DENSE_CASES, DENSE_K3, build_case, build_dense_case, relerr, scene_args_np
from tests.test_emul_bf16_payload import from_bf16, to_bf16

TOL = 1e-5
GRAD_NAMES = ("primpos", "primrot", "primscale", "template", "warp")


@pytest.fixture()
def kernels():
    from tests.emul import kernels as k
    k.use_variant(())
    k.load()
    yield k
    k.set_lane_order("forward")
    loaded, rebuilt = ctypes.c_int(), ctypes.c_int()            # reset the saved-list counters the dense scenes leave behind
    k.load().mvp_emul_saved_list_tiles(ctypes.byref(loaded), ctypes.byref(rebuilt))
    k.use_variant(())


def _flags():
    from ava256_b200 import lib
    return lib.FLAG_TPLATE_BF16 | lib.FLAG_GRAD_TPLATE_F32


def _split(s):
    """(widened fp32 scene args, bf16 scene args, kwargs) of scene s with its template rounded to bf16."""
    a, kw = scene_args_np(s)
    tb = to_bf16(a[7])
    a32, ab = list(a), list(a)
    a32[7], ab[7] = from_bf16(tb), tb.view(np.float32)
    return a32, ab, kw


def _nan16(shape):
    """NaN-filled float32 array whose data pointer is 16-byte aligned."""
    n = int(np.prod(shape))
    raw = np.empty(n + 4, np.float32)
    off = (-raw.ctypes.data // 4) % 4
    out = raw[off:off + n].reshape(shape)
    out[...] = np.nan
    return out


def forward_backward_f32(kernels, raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template, grad_rayrgba, warp=None,
                         fadescale=8.0, fadeexp=8.0, fwd_flags=0, bwd_flags=0, planes=False, clear_in_forward=False):
    """Emulated forward + backward of a bf16 template (uint16 pairs in fp32-typed words [..., 2]) with MVP_FLAG_TPLATE_BF16 |
    MVP_FLAG_GRAD_TPLATE_F32 added to both calls and an fp32 template gradient [..., 4].  The gradient buffers start NaN: the
    forward clears them (clear_in_forward, clear_grad_*), the library does (MVP_FLAG_ZERO_GRADS in bwd_flags), or, with neither,
    they are zero-filled here.  Returns (rayrgba, raysat, grads, (heavy tiles of the forward, of the backward))."""
    from ava256_b200 import lib
    L = kernels.load()
    f32 = lambda x: None if x is None else np.ascontiguousarray(x, dtype=np.float32)  # noqa: E731
    P = lambda x: None if x is None else ctypes.c_void_p(x.ctypes.data)  # noqa: E731
    raypos, raydir, tminmax, primpos, primrot, primscale, template, warp, grad_rayrgba = map(
        f32, (raypos, raydir, tminmax, primpos, primrot, primscale, template, warp, grad_rayrgba))
    N, H, W = raypos.shape[:3]
    K, (TD, TH, TW) = primpos.shape[1], template.shape[2:5]
    shape = lib.Shape(N, H, W, K, TD, TH, TW)
    wsb = L.mvp_workspace_bytes(ctypes.byref(shape))
    raw = np.zeros(wsb + 256, np.uint8)
    ws = raw[(-raw.ctypes.data) % 256:][:wsb]
    hoff = L.mvp_debug_heavy_offset(ctypes.byref(shape))
    heavy = lambda: int(ws[hoff:hoff + 4].view(np.int32)[0])  # noqa: E731
    rayrgba, raysat = np.full((N, H, W, 4), np.nan, np.float32), np.full((N, H, W, 3), np.nan, np.float32)
    rayaux = np.zeros((N, H, W, 4), np.int32)
    rgb_p, alpha_p = (np.full((N, c, H, W), np.nan, np.float32) for c in (3, 1)) if planes else (None, None)
    grads = [_nan16(x.shape) for x in (primpos, primrot, primscale)] + [_nan16(template.shape[:-1] + (4,))] + \
        ([_nan16(warp.shape)] if warp is not None else [])
    if not clear_in_forward and not (bwd_flags & lib.FLAG_ZERO_GRADS):
        for g in grads:
            g[...] = 0.0
    a = lib.ForwardArgs()
    a.shape, a.stepsize, a.fadescale, a.fadeexp = shape, float(stepsize), float(fadescale), float(fadeexp)
    a.flags = fwd_flags | _flags()
    a.raypos, a.raydir, a.tminmax = P(raypos), P(raydir), P(tminmax)
    a.primpos, a.primrot, a.primscale, a.tplate = P(primpos), P(primrot), P(primscale), P(template)
    a.rayrgba, a.raysat, a.rayaux = (None if planes else P(rayrgba)), P(raysat), P(rayaux)
    a.rayrgb_nchw, a.rayalpha_nchw = P(rgb_p), P(alpha_p)
    a.workspace, a.workspace_bytes = P(ws), wsb
    if warp is not None:
        a.algo, a.warp = 1, P(warp)
        a.WD, a.WH, a.WW = warp.shape[2:5]
    if clear_in_forward:
        a.clear_grad_primpos, a.clear_grad_primrot, a.clear_grad_primscale, a.clear_grad_tplate = (P(g) for g in grads[:4])
        a.clear_grad_warp = P(grads[4]) if warp is not None else None
    assert L.mvp_raymarch_forward(ctypes.byref(a), None) == 0
    hf = heavy()
    if clear_in_forward:
        assert not any(g.any() for g in grads), "the forward must leave the clear_grad_* buffers zero"
    if planes:
        rayrgba = np.ascontiguousarray(np.concatenate([rgb_p, alpha_p], axis=1).transpose(0, 2, 3, 1))
    b = lib.BackwardArgs()
    b.shape, b.stepsize, b.fadescale, b.fadeexp = shape, a.stepsize, a.fadescale, a.fadeexp
    b.flags = lib.FLAG_ACCEL_VALID | bwd_flags | _flags()
    b.raypos, b.raydir, b.tminmax = a.raypos, a.raydir, a.tminmax
    b.primpos, b.primrot, b.primscale, b.tplate = a.primpos, a.primrot, a.primscale, a.tplate
    if planes:
        gp = grad_rayrgba.transpose(0, 3, 1, 2)
        g_rgb, g_alpha = np.ascontiguousarray(gp[:, :3]), np.ascontiguousarray(gp[:, 3:4])
        b.grad_rayrgb_nchw, b.grad_rayalpha_nchw = P(g_rgb), P(g_alpha)
    else:
        b.grad_rayrgba = P(grad_rayrgba)
    b.raysat, b.rayaux = P(raysat), P(rayaux)
    b.grad_primpos, b.grad_primrot, b.grad_primscale, b.grad_tplate = (P(g) for g in grads[:4])
    b.workspace, b.workspace_bytes = P(ws), wsb
    if warp is not None:
        b.algo, b.warp, b.grad_warp = 1, a.warp, P(grads[4])
        b.WD, b.WH, b.WW = a.WD, a.WH, a.WW
    assert L.mvp_raymarch_backward(ctypes.byref(b), None) == 0
    return rayrgba, raysat, grads, (hf, heavy())


def check_grads(gb, g32):
    for nm, x, y in zip(GRAD_NAMES, gb, g32):
        assert x.dtype == np.float32 and x.shape == y.shape, nm
        assert np.isfinite(x).all(), nm
        assert relerr(x, y) <= TOL, (nm, relerr(x, y))
    assert np.abs(g32[3]).max() > 0, "the scene must give the template a gradient"


def run_pair(kernels, s, grad, **opts):
    """The scene with its template rounded to bf16: once through the fp32 kernels on the widened template, once through the bf16
    kernels with an fp32 gradient.  Checks the contract; returns the heavy-tile counts (forward, backward) of the gradient run."""
    a32, ab, kw = _split(s)
    out32, sat32, g32 = kernels.forward_backward(*a32, grad_rayrgba=grad, **kw, **opts)
    heavy32 = kernels.last_heavy_tiles
    outb, satb, gb, heavyb = forward_backward_f32(kernels, *ab, grad, **kw, **opts)
    assert heavyb == heavy32
    assert np.array_equal(outb, out32) and np.array_equal(satb, sat32)          # the bf16 path's forward: bit-identical
    check_grads(gb, g32)
    return heavy32


@pytest.mark.parametrize("order", ["forward", "random"])
@pytest.mark.parametrize("name", list(CASES))
def test_emulated_bf16_grad_f32_named_cases(kernels, name, order):
    """T = 8 (head_small), 16 (head_t16), runtime dims (gradcheck_*, noncubic, many_views) and algo 1 (warp_*)."""
    s, grad = build_case(name)
    kernels.set_lane_order(order)
    run_pair(kernels, s, grad.numpy())


@pytest.mark.parametrize("cap", list(DENSE_K3))
@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_emulated_bf16_grad_f32_heavy_kernels(kernels, name, cap):
    """Every tile through the 512-entry kernels, with and without the reference's 512 cap."""
    s, grad = build_dense_case(name, cap)
    kernels.set_lane_order("random" if cap == "capped" else "forward")
    heavy = run_pair(kernels, s, grad.numpy())
    N, H, W = s["raypos"].shape[:3]
    assert heavy == (N * -(-H // 4) * -(-W // 8),) * 2


@pytest.mark.parametrize("name", ["head_small", "head_t16", "gradcheck_ragged", "warp_small", "dense_t8", "dense_warp"])
def test_emulated_bf16_grad_f32_ray_grads(kernels, name):
    """The kRayGrad instantiations (mvp_raymarch_backward_rays), fast and 512-entry: rays and every gradient as the fp32 kernels'
    on the widened template."""
    from tests.test_ray_grads_cpu import emulated_ray_grads, ray_backward
    s, grad = build_dense_case(name[len("dense_"):], "uncapped") if name.startswith("dense_") else build_case(name)
    a32, ab, kw = _split(s)
    _, _, g32, r32 = emulated_ray_grads(kernels, a32, kw, grad.numpy())
    heavy32 = kernels.last_heavy_tiles
    with ray_backward(kernels, *a32[0].shape[:3]) as rb:               # mvp_raymarch_backward_rays in place of the plain backward
        _, _, gb, heavyb = forward_backward_f32(kernels, *ab, grad.numpy(), **kw)
    assert heavyb == heavy32 and (heavy32[1] > 0) == name.startswith("dense_")
    check_grads(gb, g32)
    for x, y in zip(rb, r32):
        assert np.isfinite(x).all() and relerr(x, y) <= TOL


@pytest.mark.parametrize("name", ["gradcheck_ragged", "warp_small", "head_t16"])
def test_emulated_bf16_grad_f32_gradient_buffers_cleared(kernels, name):
    """The forward's clear of clear_grad_tplate counts fp32 words: every word of the NaN-filled fp32 buffer is zero afterwards (a
    clear at the bf16 gradient's size leaves half of it NaN)."""
    s, grad = build_case(name)
    run_pair(kernels, s, grad.numpy(), clear_in_forward=True)


def test_emulated_bf16_grad_f32_zero_grads_flag(kernels):
    """MVP_FLAG_ZERO_GRADS (the op's retain_graph second backward): the library zero-fills the whole NaN-filled fp32 buffer."""
    from ava256_b200 import lib
    s, grad = build_case("head_small")
    run_pair(kernels, s, grad.numpy(), bwd_flags=lib.FLAG_ZERO_GRADS)


def test_emulated_bf16_grad_f32_image_planes(kernels):
    s, grad = build_case("gradcheck_small")
    run_pair(kernels, s, grad.numpy(), planes=True)


def test_emulated_grad_f32_flag_alone_changes_nothing(kernels):
    """Without MVP_FLAG_TPLATE_BF16 the flag is ignored: an fp32 template renders and back-propagates as without it."""
    from ava256_b200 import lib
    s, grad = build_case("head_small")
    a, kw = scene_args_np(s)
    out0, sat0, g0 = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw, clear_in_forward=True)
    f = lib.FLAG_GRAD_TPLATE_F32
    out1, sat1, g1 = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw, clear_in_forward=True, fwd_flags=f, bwd_flags=f)
    assert np.array_equal(out1, out0) and np.array_equal(sat1, sat0)
    check_grads(g1, g0)
