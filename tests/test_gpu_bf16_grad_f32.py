"""GPU tests of bfloat16 templates with their gradient accumulated in fp32 (`pytest -m gpu`): MVP_FLAG_GRAD_TPLATE_F32 at the
C-ABI, and `template_grad_dtype=torch.float32` (context manager, `mvpraymarch_camera` keyword, `Raymarcher` keyword) at the op.

Reference of every check: the same call on the fp32 widening `tb.float()` of the bf16 template `tb`.  At the C-ABI the images,
raysat and rayaux are bit-identical and every gradient, the fp32 template gradient included, within TOL of max|.| (the order of
the fp32 atomics).  Through the op autograd casts the fp32 template gradient to the input's bf16, so `template.grad` is the fp32
sum rounded once: element by element |g - g32| <= 2^-8 |g32| + TOL max|g32| (ROUND_ONCE)."""
import contextlib
import ctypes
import gc

import pytest
import torch

from tests.helpers import CASES, abi_raymarch, build_case, build_dense_case, gradcheck_like_scene, relerr
from tests.test_gpu_bf16_payload import _cuda_scene, _relerr, render
from tests.test_gpu_large_launch import _require_memory

pytestmark = pytest.mark.gpu

TOL = 1e-5
ROUND_ONCE = 2.0 ** -8          # half a bf16 ulp, relative: one round-to-nearest of the fp32 sum


def _flags():
    from ava256_b200 import lib
    return lib.FLAG_TPLATE_BF16 | lib.FLAG_GRAD_TPLATE_F32


def check_rounded_once(gb, g32, what=""):
    """gb (bf16) is g32 (fp32) rounded once, up to the order of the fp32 atomics."""
    assert gb.dtype == torch.bfloat16 and gb.shape == g32.shape, what
    g, r = gb.double(), g32.double()
    bound = ROUND_ONCE * r.abs() + TOL * float(r.abs().max())
    excess = float(((g - r).abs() - bound).max())
    assert bool(torch.isfinite(g).all()) and excess <= 0, (what, excess)
    assert float(r.abs().max()) > 0, what


def compare_op(s, grad, **kw):
    """The public op on the bf16 template under template_grad_dtype(torch.float32) against the fp32 widening.  Returns the bf16
    run's (image, gradients) and the fp32 run's gradients."""
    from ava256_b200.op import template_grad_dtype
    tb = s["template"].to(torch.bfloat16)
    out32, g32 = render(s, tb.float(), grad, **kw)
    with template_grad_dtype(torch.float32):
        outb, gb = render(s, tb.clone(), grad, **kw)
    assert torch.equal(outb, out32)
    for nm in g32:
        if nm == "template":
            check_rounded_once(gb[nm], g32[nm], nm)
        else:
            assert gb[nm].dtype == torch.float32 and _relerr(gb[nm], g32[nm]) <= TOL, nm
    return outb, gb, g32


# ---- C-ABI ---------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _ray_backward(N, H, W):
    """abi_raymarch's backward goes to mvp_raymarch_backward_rays (the kRayGrad instantiations); yields the ray gradients."""
    from ava256_b200 import lib
    out = [torch.full((N, H, W, c), float("nan"), device="cuda") for c in (3, 3, 2)]
    plain = lib.LIB.mvp_raymarch_backward
    lib.LIB.mvp_raymarch_backward = lambda b, st: lib.LIB.mvp_raymarch_backward_rays(b, *(ctypes.c_void_p(t.data_ptr()) for t in out), st)
    try:
        yield out
    finally:
        lib.LIB.mvp_raymarch_backward = plain


def abi_raymarch_f32(s, grad, clear_in_forward=False, keep=None):
    """tests.helpers.abi_raymarch for a bf16 template with its gradient accumulated in fp32: MVP_FLAG_TPLATE_BF16 |
    MVP_FLAG_GRAD_TPLATE_F32 in the forward and the backward, and an fp32 template gradient buffer.  The gradient buffers start
    as NaN; the forward clears them (clear_in_forward) or the backward does (MVP_FLAG_ZERO_GRADS).  Same return value and `keep`."""
    from ava256_b200 import lib
    P = lambda x: None if x is None else ctypes.c_void_p(x.data_ptr())  # noqa: E731
    N, H, W = s["raypos"].shape[:3]
    K, (TD, TH, TW) = s["primpos"].shape[1], s["template"].shape[2:5]
    shape = lib.Shape(N, H, W, K, TD, TH, TW)
    wsb = lib.workspace_bytes(N, H, W, K, TD, TH, TW)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    hoff = lib.LIB.mvp_debug_heavy_offset(ctypes.byref(shape))
    heavy = lambda: int(ws[hoff:hoff + 4].view(torch.int32).item())  # noqa: E731
    warp = s.get("warp")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rgba = torch.full((N, H, W, 4), float("nan"), device="cuda")
    rsat, raux = torch.empty(N, H, W, 3, device="cuda"), torch.empty(N, H, W, 4, dtype=torch.int32, device="cuda")
    if keep is not None:
        keep["workspace"], keep["rayaux"] = ws, raux
    gs = [torch.full(s[n].shape, float("nan"), device="cuda") for n in ("primpos", "primrot", "primscale", "template")] + \
        ([torch.full_like(warp, float("nan"))] if warp is not None else [])
    a = lib.ForwardArgs()
    a.shape, a.stepsize, a.fadescale, a.fadeexp = shape, s["stepsize"], s.get("fadescale", 8.0), s.get("fadeexp", 8.0)
    a.flags = _flags()
    a.raypos, a.raydir, a.tminmax = P(s["raypos"]), P(s["raydir"]), P(s["tminmax"])
    a.primpos, a.primrot, a.primscale, a.tplate = P(s["primpos"]), P(s["primrot"]), P(s["primscale"]), P(s["template"])
    a.rayrgba, a.raysat, a.rayaux = P(rgba), P(rsat), P(raux)
    a.workspace, a.workspace_bytes = P(ws), wsb
    if warp is not None:
        a.algo, a.warp = 1, P(warp)
        a.WD, a.WH, a.WW = warp.shape[2:5]
    if clear_in_forward:
        a.clear_grad_primpos, a.clear_grad_primrot, a.clear_grad_primscale, a.clear_grad_tplate = (P(g) for g in gs[:4])
        a.clear_grad_warp = P(gs[4]) if warp is not None else None
    lib.check(lib.LIB.mvp_raymarch_forward(ctypes.byref(a), st))
    hf = heavy()
    b = lib.BackwardArgs()
    b.shape, b.stepsize, b.fadescale, b.fadeexp = a.shape, a.stepsize, a.fadescale, a.fadeexp
    b.flags = lib.FLAG_ACCEL_VALID | (0 if clear_in_forward else lib.FLAG_ZERO_GRADS) | _flags()
    b.raypos, b.raydir, b.tminmax = a.raypos, a.raydir, a.tminmax
    b.primpos, b.primrot, b.primscale, b.tplate = a.primpos, a.primrot, a.primscale, a.tplate
    b.grad_rayrgba, b.raysat, b.rayaux = P(grad), P(rsat), P(raux)
    b.grad_primpos, b.grad_primrot, b.grad_primscale, b.grad_tplate = (P(g) for g in gs[:4])
    b.workspace, b.workspace_bytes = P(ws), wsb
    if warp is not None:
        b.algo, b.warp, b.grad_warp = 1, P(warp), P(gs[4])
        b.WD, b.WH, b.WW = a.WD, a.WH, a.WW
    lib.check(lib.LIB.mvp_raymarch_backward(ctypes.byref(b), st))
    hb = heavy()
    torch.cuda.synchronize()
    return rgba, rsat, gs, (hf, hb)


def _abi(s, grad, rays, f32grad=False, **kw):
    """abi_raymarch (fp32 template) or abi_raymarch_f32 (bf16 template, f32grad), optionally through the ray-gradient backward."""
    N, H, W = s["raypos"].shape[:3]
    keep = {}
    with (_ray_backward(N, H, W) if rays else contextlib.nullcontext()) as r:
        out, sat, gs, heavy = (abi_raymarch_f32 if f32grad else abi_raymarch)(s, grad, keep=keep, **kw)
    return out, sat, keep["rayaux"], gs, heavy, r


ABI_CASES = ["head_small", "head_t16", "gradcheck_small", "warp_small", "dense_t8", "dense_t16", "dense_noncubic", "dense_warp"]


@pytest.mark.parametrize("rays", [False, True])
@pytest.mark.parametrize("name", ABI_CASES)
def test_abi_bf16_grad_f32_every_instantiation(name, rays):
    """Fast (T = 8, 16, runtime dims, warp field) and 512-entry (dense_*) backward kernels, without and with kRayGrad."""
    dense = name.startswith("dense_")
    s, grad = build_dense_case(name[len("dense_"):], "uncapped") if dense else build_case(name)
    s, grad = _cuda_scene(s), grad.cuda()
    tb = s["template"].to(torch.bfloat16)
    clear = not dense                                  # the forward's clear on the named cases, MVP_FLAG_ZERO_GRADS on the dense
    o32, sat32, aux32, g32, h32, r32 = _abi(dict(s, template=tb.float()), grad, rays, clear_in_forward=clear)
    ob, satb, auxb, gb, hb, rb = _abi(dict(s, template=tb), grad, rays, f32grad=True, clear_in_forward=clear)
    assert hb == h32 and (hb[1] > 0) == dense
    assert torch.equal(ob, o32) and torch.equal(satb, sat32) and torch.equal(auxb, aux32)
    assert gb[3].dtype == torch.float32 and gb[3].shape == tb.shape
    for nm, x, y in zip(("primpos", "primrot", "primscale", "template", "warp"), gb, g32):
        assert bool(torch.isfinite(x).all()) and relerr(x.cpu().numpy(), y.cpu().numpy()) <= TOL, nm
    assert float(g32[3].abs().max()) > 0
    if rays:
        for x, y in zip(rb, r32):
            assert bool(torch.isfinite(x).all()) and relerr(x.cpu().numpy(), y.cpu().numpy()) <= TOL


def test_abi_bf16_grad_f32_rejects_misaligned_and_missing_buffers():
    """The fp32 gradient buffers need 16 bytes (8 is enough for a bf16 one); a missing grad_tplate is rejected as before.  Both
    before any device work."""
    from ava256_b200 import lib
    s, grad = build_case("head_small")
    s, grad = _cuda_scene(s), grad.cuda()
    tb = s["template"].to(torch.bfloat16)
    keep = {}
    _, raysat, _, _ = abi_raymarch_f32(dict(s, template=tb), grad, keep=keep)
    N, H, W = s["raypos"].shape[:3]
    K, (TD, TH, TW) = s["primpos"].shape[1], tb.shape[2:5]
    P = lambda x: ctypes.c_void_p(x.data_ptr())  # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ws = keep["workspace"]
    g = torch.zeros(tb.numel() + 4, device="cuda")                     # fp32 buffer with room for an 8-byte offset
    gpp, gpr, gps = (torch.zeros_like(s[k]) for k in ("primpos", "primrot", "primscale"))
    rayaux = keep["rayaux"]

    def backward(gt, flags=_flags()):
        b = lib.BackwardArgs()
        b.shape, b.stepsize, b.fadescale, b.fadeexp = lib.Shape(N, H, W, K, TD, TH, TW), s["stepsize"], 8.0, 8.0
        b.flags = lib.FLAG_ACCEL_VALID | flags
        b.raypos, b.raydir, b.tminmax = P(s["raypos"]), P(s["raydir"]), P(s["tminmax"])
        b.primpos, b.primrot, b.primscale, b.tplate = P(s["primpos"]), P(s["primrot"]), P(s["primscale"]), P(tb)
        b.grad_rayrgba, b.raysat, b.rayaux = P(grad), P(raysat), P(rayaux)
        b.grad_primpos, b.grad_primrot, b.grad_primscale, b.grad_tplate = P(gpp), P(gpr), P(gps), gt
        b.workspace, b.workspace_bytes = P(ws), ws.numel()
        return lib.LIB.mvp_raymarch_backward(ctypes.byref(b), st)

    g8 = ctypes.c_void_p(g.data_ptr() + 8)
    assert backward(g8) == -6                                              # MVP_ERR_ALIGN
    assert backward(g8, lib.FLAG_TPLATE_BF16) == 0                         # the same address holds a bf16 gradient
    assert backward(None) == -1                                            # MVP_ERR_NULL
    a = lib.ForwardArgs()
    a.shape, a.stepsize, a.fadescale, a.fadeexp = lib.Shape(N, H, W, K, TD, TH, TW), s["stepsize"], 8.0, 8.0
    a.flags = _flags()
    a.raypos, a.raydir, a.tminmax = P(s["raypos"]), P(s["raydir"]), P(s["tminmax"])
    a.primpos, a.primrot, a.primscale, a.tplate = P(s["primpos"]), P(s["primrot"]), P(s["primscale"]), P(tb)
    out, sat, aux = torch.empty(N, H, W, 4, device="cuda"), torch.empty_like(raysat), torch.empty_like(rayaux)
    a.rayrgba, a.raysat, a.rayaux = P(out), P(sat), P(aux)
    a.workspace, a.workspace_bytes = P(ws), ws.numel()
    a.clear_grad_tplate = g8
    assert lib.LIB.mvp_raymarch_forward(ctypes.byref(a), st) == -6
    torch.cuda.synchronize()
    assert "GRAD_TPLATE_F32=1" in lib.LIB.mvp_build_config().decode().split()


# ---- the op -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_op_bf16_grad_f32_named_cases(name):
    s, grad = build_case(name)
    compare_op(_cuda_scene(s), grad.cuda())


def test_op_bf16_grad_f32_heavy_kernels():
    s, grad = build_dense_case("t8", "capped")
    compare_op(_cuda_scene(s), grad.cuda())


def test_op_bf16_grad_f32_shared_primitives():
    """One [1,K,...] set for 4 views (the scene of test_bf16_template_shared_primitives, whose bf16 accumulation needs the dense
    gates 0.15 / 0.05): all views reduce into the one fp32 gradient, rounded once."""
    s = _cuda_scene(gradcheck_like_scene(N=4, H=20, W=24, k3=3, M=6, seed=41, alpha_gain=8.0))
    grad = torch.randn(4, 20, 24, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    compare_op(s, grad, shared=True)


def _head_scene():
    from ava256_b200 import scene
    n, H, W, K, T = 2, 96, 64, 256, 8
    s = scene.make_scene(n, H, W, K, T, alpha_mu=3.0, alpha_sigma=3.0, share_primitives=False, device="cuda")
    s["stepsize"], s["fadescale"], s["fadeexp"] = 1.0 / 64, 8.0, 8.0
    grad = torch.randn(n, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    cams = [c.cuda() for c in scene.make_cameras(n, H, W)]
    return s, grad, (cams[0], cams[1], cams[2], cams[3], (W, H), scene.VOLRADIUS)


def test_op_bf16_grad_f32_planes_and_camera_rays():
    s, grad, camera = _head_scene()
    compare_op(s, grad, planes=True)
    compare_op(s, grad, camera=camera)
    compare_op(s, grad, camera=camera, planes=True)


def _camera_march(s, cams, template, camera_grad, **kw):
    from ava256_b200 import scene
    from ava256_b200.op import mvpraymarch_camera
    W, H = cams[4]
    prims = [s[k].detach().clone().requires_grad_(True) for k in ("primpos", "primrot", "primscale")] + [template.clone().requires_grad_(True)]
    leaves = [c.clone().requires_grad_(camera_grad) for c in cams[:4]]
    out = mvpraymarch_camera(*leaves, (W, H), scene.VOLRADIUS, s["stepsize"], tuple(prims[:3]), prims[3], None, camera_grad=camera_grad,
                             fadescale=8.0, fadeexp=8.0, **kw)
    return out, prims, leaves


@pytest.mark.parametrize("camera_grad", [False, True])
def test_op_bf16_grad_f32_camera_keyword(camera_grad):
    """`mvpraymarch_camera(template_grad_dtype=torch.float32)`, also with camera_grad=True (MVPRaymarchCameraGrad): the camera
    gradients are those of the fp32 template within 1e-5, like the two forms of tests/test_gpu_camera_grads.py."""
    s, grad, cams = _head_scene()
    tb = s["template"].to(torch.bfloat16)
    out32, p32, c32 = _camera_march(s, cams, tb.float(), camera_grad)
    (out32 * grad).sum().backward()
    outb, pb, cb = _camera_march(s, cams, tb, camera_grad, template_grad_dtype=torch.float32)
    assert outb.grad_fn.tflags == _flags()
    (outb * grad).sum().backward()
    assert torch.equal(outb, out32)
    check_rounded_once(pb[3].grad, p32[3].grad, "template")
    for x, y in zip(pb[:3], p32[:3]):
        assert _relerr(x.grad, y.grad) <= TOL
    for x, y in zip(cb, c32):
        if camera_grad:
            assert bool(torch.isfinite(x.grad).all()) and float(y.grad.abs().max()) > 0 and _relerr(x.grad, y.grad) <= TOL
        else:
            assert x.grad is None


def test_op_bf16_grad_f32_retain_graph_second_backward():
    """The second backward through the same graph gets a fresh fp32 buffer, zero-filled by the library (MVP_FLAG_ZERO_GRADS)."""
    from ava256_b200.op import template_grad_dtype
    s, grad = build_case("head_small")
    s, grad = _cuda_scene(s), grad.cuda()
    tb = s["template"].to(torch.bfloat16)
    _, g32 = render(s, tb.float(), grad)
    keep = {}
    with template_grad_dtype(torch.float32):
        _, gb = render(s, tb, grad, retain=True, keep=keep)
    for g in (gb, dict(zip(gb, keep["second"]))):
        check_rounded_once(g["template"], g32["template"])
        for nm in ("primpos", "primrot", "primscale"):
            assert _relerr(g[nm], g32[nm]) <= TOL, nm


def test_op_bf16_grad_f32_decision_taken_by_the_forward():
    """The backward follows the forward's setting, not the context around the backward (autograd runs it on its own thread)."""
    from ava256_b200.op import mvpraymarch, template_grad_dtype
    s, grad = build_case("head_small")
    s, grad = _cuda_scene(s), grad.cuda()
    tb = s["template"].to(torch.bfloat16)
    _, g32 = render(s, tb.float(), grad)
    prim = tuple(s[k] for k in ("primpos", "primrot", "primscale"))
    args = (s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], prim)
    t1 = tb.clone().requires_grad_(True)
    with template_grad_dtype(torch.float32):
        out1 = mvpraymarch(*args, t1, None, fadescale=8.0, fadeexp=8.0)
    out1.backward(grad)
    check_rounded_once(t1.grad, g32["template"])
    t2 = tb.clone().requires_grad_(True)
    out2 = mvpraymarch(*args, t2, None, fadescale=8.0, fadeexp=8.0)
    with template_grad_dtype(torch.float32):
        out2.backward(grad)
    from ava256_b200 import lib
    assert out1.grad_fn.tflags == _flags() and out2.grad_fn.tflags == lib.FLAG_TPLATE_BF16
    assert t2.grad.dtype == torch.bfloat16 and bool(torch.isfinite(t2.grad.float()).all())


def test_op_bf16_grad_f32_raymarcher():
    from ava256_b200.raymarcher import Raymarcher
    s, grad, cams = _head_scene()
    tb = s["template"].to(torch.bfloat16)
    gp = grad.permute(0, 3, 1, 2)
    res = {}
    R, dt = cams[5], s["stepsize"] * cams[5]                  # Raymarcher's step is dt / volradius
    for key, rm, tpl in (("f32", Raymarcher(R, dt), tb.float()), ("bf16", Raymarcher(R, dt, template_grad_dtype=torch.float32), tb)):
        for form in ("rays", "camera"):
            t = tpl.clone().requires_grad_(True)
            decout = {"primpos": s["primpos"], "primrot": s["primrot"], "primscale": s["primscale"], "template": t}
            opts = {"fadescale": 8.0, "fadeexp": 8.0}
            if form == "rays":
                rgb, alpha, _, _ = rm(s["raypos"], s["raydir"], s["tminmax"], decout, renderoptions=opts)
            else:
                rgb, alpha, _, _ = rm.forward_camera(*cams[:5], decout, renderoptions=opts)
            ((rgb * gp[:, :3]).sum() + (alpha * gp[:, 3:]).sum()).backward()
            res[key, form] = (rgb.detach(), alpha.detach(), t.grad)
    for form in ("rays", "camera"):
        assert torch.equal(res["bf16", form][0], res["f32", form][0]) and torch.equal(res["bf16", form][1], res["f32", form][1])
        check_rounded_once(res["bf16", form][2], res["f32", form][2], form)


def test_op_bf16_grad_f32_overlay_context_manager():
    """An unmodified caller of the drop-in `extensions.mvpraymarch.mvpraymarch.mvpraymarch` opts in with the context manager."""
    import ava256_b200.op
    from extensions.mvpraymarch.mvpraymarch import mvpraymarch
    s, grad = build_case("warp_head")
    s, grad = _cuda_scene(s), grad.cuda()
    tb = s["template"].to(torch.bfloat16)
    res = []
    for tpl, ctx in ((tb.float(), contextlib.nullcontext()), (tb, ava256_b200.op.template_grad_dtype(torch.float32))):
        t = tpl.clone().requires_grad_(True)
        with ctx:
            out = mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], (s["primpos"], s["primrot"], s["primscale"]), t,
                              s["warp"], algo=1, fadescale=8.0, fadeexp=8.0)
        (out * grad).sum().backward()
        res.append((out.detach(), t.grad))
    assert torch.equal(res[1][0], res[0][0])
    check_rounded_once(res[1][1], res[0][1])


def test_template_grad_dtype_arguments():
    """Only None and torch.float32; with an fp32 template the setting changes nothing."""
    from ava256_b200.op import mvpraymarch, mvpraymarch_camera, template_grad_dtype
    from ava256_b200.raymarcher import Raymarcher
    for bad in (torch.bfloat16, torch.float16, torch.float64, "float32", 32):
        with pytest.raises(ValueError, match="template_grad_dtype"):
            with template_grad_dtype(bad):
                pass
        with pytest.raises(ValueError, match="template_grad_dtype"):
            Raymarcher(1.0, template_grad_dtype=bad)
        with pytest.raises(ValueError, match="template_grad_dtype"):
            mvpraymarch_camera(None, None, None, None, (4, 4), 1.0, 0.1, None, None, None, template_grad_dtype=bad)
    s, grad = build_case("head_small")
    s, grad = _cuda_scene(s), grad.cuda()
    prim = tuple(s[k] for k in ("primpos", "primrot", "primscale"))
    res = []
    for ctx in (contextlib.nullcontext(), template_grad_dtype(torch.float32), template_grad_dtype(None)):
        t = s["template"].clone().requires_grad_(True)
        with ctx:
            out = mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], prim, t, None, fadescale=8.0, fadeexp=8.0)
        assert out.grad_fn.tflags == 0
        out.backward(grad)
        res.append((out.detach(), t.grad))
    for out, g in res[1:]:
        assert torch.equal(out, res[0][0]) and g.dtype == torch.float32 and _relerr(g, res[0][1]) <= TOL


# ---- the 80-view benchmark launch ------------------------------------------------------------------------------------------
def test_op_bf16_grad_f32_80_view_launch_per_view():
    """80 views with their own bf16 payloads: the fp32 gradient is twice the template's size (its byte offsets pass 2^32 at view
    32), so a gradient stride that counted the template's words would put views on each other.  Views 0, 31, 32, 63, 64 and 79
    equal the view rendered alone: images bit for bit, transform gradients within TOL; the template gradients are both rounded
    once from fp32 sums taken in different orders, so they may differ by one bf16 ulp (2^-7 relative)."""
    from ava256_b200 import lib, scene
    from ava256_b200.op import template_grad_dtype
    N, H, W, K, T = 80, 1024, 667, 16384, 8
    vox = N * K * T ** 3
    # bf16 template, fp32 gradient, its bf16 cast (autograd's temporary) and the returned bf16 gradient; fp32 transforms + grads
    need = vox * 4 * (2 + 4 + 2 + 2) + 2 * N * K * (3 + 9 + 3) * 4 + N * H * W * (3 + 3 + 2 + 4 + 4 + 3 + 4) * 4 + \
        lib.workspace_bytes(N, H, W, K, T, T, T) + (2 << 30)
    _require_memory(need, "80-view launch, bf16 per-view payloads, fp32 template gradient")
    s = scene.make_scene(N, H, W, K, T, alpha_mu=17.0, alpha_sigma=6.0, share_primitives=False, device="cuda")
    tpl = s.pop("template")
    tb = torch.empty(tpl.shape, dtype=torch.bfloat16, device="cuda")
    del tpl
    gc.collect()
    torch.cuda.empty_cache()
    for v in range(N):
        tb[v] = scene.make_payload(K, T, seed=1112 + v, alpha_mu=17.0, alpha_sigma=6.0, device="cuda").to(torch.bfloat16)
    grad = torch.randn(N, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    with template_grad_dtype(torch.float32):
        out, gs = render(s, tb, grad)
        for v in (0, 31, 32, 63, 64, 79):
            sv = {k: (x[v:v + 1].contiguous() if torch.is_tensor(x) else x) for k, x in s.items()}
            out_v, gs_v = render(sv, tb[v:v + 1].contiguous(), grad[v:v + 1].contiguous())
            assert torch.equal(out[v:v + 1], out_v), v
            for nm in gs_v:
                if nm != "template":
                    assert _relerr(gs[nm][v:v + 1], gs_v[nm]) <= TOL, (v, nm)
            g, r = gs["template"][v:v + 1].double(), gs_v["template"].double()
            assert gs["template"].dtype == torch.bfloat16 and float(r.abs().max()) > 0, v
            excess = float(((g - r).abs() - (2 * ROUND_ONCE * r.abs() + TOL * float(r.abs().max()))).max())
            assert excess <= 0, (v, excess)
            del sv, out_v, gs_v


# ---- the one-subject bf16 step ----------------------------------------------------------------------------------------------
# The one-subject step (assemble_payload(dtype=bf16) -> expand_views -> op -> back) with fp32 accumulation, against the fp32 step.
# What remains is the bf16 template alone: the fp32 step renders other alpha values (2^-9 relative) and rays saturate at other
# samples, and each view's fp32 gradient is rounded once to bf16 before the views are summed in fp32.  Measured on an H100 80GB
# HBM3: grad_tex max 0.0036 / sum 0.0024 at 4 views, 0.0042 / 0.0026 at 80 (bf16 accumulation: 0.0097 / 0.0040 and
# 0.0084 / 0.0044, tests/test_gpu_bf16_handoff.py); grad_opacity 0.208 / 0.0109 at 4 views, 0.093 / 0.031 at 80 (bf16
# accumulation: 0.21 / 0.0122 and 0.095 / 0.032).  So accumulation accounts for about half of the grad_tex error and almost
# none of the grad_opacity error: that comes from the template's own rounding, which fp32 accumulation cannot remove, and keeps
# the opacity gate of the bf16 step.  The tex gate is about twice the measured values.
GATE_STEP_F32_TEX = (0.008, 0.005)
GATE_STEP_F32_OPACITY = (0.3, 0.05)


def _step_errors(nv):
    from tests.test_gpu_bf16_handoff import _errors, _one_subject_step, _pipeline_case
    from ava256_b200.op import template_grad_dtype
    s, tex, opa, grad = _pipeline_case(nv, True)
    out32, _, gtex32, gopa32, _ = _one_subject_step(s, tex, opa, grad, torch.float32, nv)
    del out32
    with template_grad_dtype(torch.float32):
        _, _, gtexb, gopab, peak = _one_subject_step(s, tex, opa, grad, torch.bfloat16, nv)
    assert gtexb.dtype == torch.float32 and bool(torch.isfinite(gtexb).all()) and bool(torch.isfinite(gopab).all())
    et, ot = _errors(gtexb, gtex32), _errors(gopab, gopa32)
    print("%d views, fp32 accumulation: grad_tex max %.3g l1 %.3g, grad_opacity max %.3g l1 %.3g; peak %.2f GB"
          % (nv, et[0], et[1], ot[0], ot[1], peak / 1e9))
    assert et[0] <= GATE_STEP_F32_TEX[0] and et[1] <= GATE_STEP_F32_TEX[1], et
    assert ot[0] <= GATE_STEP_F32_OPACITY[0] and ot[1] <= GATE_STEP_F32_OPACITY[1], ot


def test_op_bf16_grad_f32_one_subject_step_four_bench_views():
    _step_errors(4)


def test_op_bf16_grad_f32_one_subject_step_80_view_launch():
    from ava256_b200 import lib
    nv, H, W, K, T = 80, 1024, 667, 16384, 8
    tplb = nv * K * T ** 3 * 4 * 4                                             # fp32 expanded template / fp32 gradient
    need = 2 * tplb + nv * H * W * (3 + 3 + 2 + 4 + 4 + 3 + 4) * 4 + lib.workspace_bytes(nv, H, W, K, T, T, T) + (4 << 30)
    _require_memory(need, "one-subject step, 80 views, fp32 template gradient")
    _step_errors(nv)
