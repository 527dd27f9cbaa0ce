"""GPU tests of the reduced gradient sets of the raymarch backward (`pytest -m gpu`): MVP_FLAG_NO_TPLATE_GRAD ("no payload") and
MVP_FLAG_RAY_GRADS_ONLY ("rays only") in every new instantiation (T = 8, 16, runtime dims and algo 1 through CASES; the 512-entry
kernels through DENSE_CASES x DENSE_K3; fp32, bf16 and bf16 with the fp32-gradient request) against the full backward; the ray
gradients against the fp32 C oracle; the autograd front end choosing the set from what requires grad; a pose recovery through a
frozen avatar; and the memory a frozen template no longer costs.  The reduced sets' gradients equal the full backward's up to the
order of the fp32 atomics (1e-5 of max|.|); the buffers outside a set are passed as NULL."""
import ctypes

import numpy as np
import pytest
import torch

from tests.helpers import CASES, DENSE_CASES, DENSE_K3, build_case, build_dense_case, relerr
from tests.test_gpu_camera_grads import _cuda, _head, _rotvec, check_vs_oracle

pytestmark = pytest.mark.gpu

ATOMIC_TOL = 1e-5


def _flags(gset):
    from ava256_b200 import lib
    return {"all": 0, "no_payload": lib.FLAG_NO_TPLATE_GRAD, "rays_only": lib.FLAG_RAY_GRADS_ONLY}[gset]


def gpu_march(s, grad, gset="all", rays=True, dtype="fp32"):
    """Forward + backward of scene s (CUDA tensors) through the C-ABI with gradient set gset: the requested gradient buffers start
    NaN and are cleared by the forward's render kernel, the others are NULL.  dtype: "fp32", "bf16" (bf16 template and gradient) or
    "bf16_g32" (bf16 template, fp32 gradient).  Returns ([primpos, primrot, primscale, template, warp] gradients on the host, None
    where not requested; ray gradients on the host or None; (heavy tiles of the forward, of the backward))."""
    from ava256_b200 import lib
    P = lambda x: None if x is None else ctypes.c_void_p(x.data_ptr())  # noqa: E731
    N, H, W = s["raypos"].shape[:3]
    K = s["primpos"].shape[1]
    tpl = s["template"].to(torch.bfloat16).contiguous() if dtype != "fp32" else s["template"]
    TD, TH, TW = tpl.shape[2:5]
    warp = s.get("warp")
    tflags = {"fp32": 0, "bf16": lib.FLAG_TPLATE_BF16, "bf16_g32": lib.FLAG_TPLATE_BF16 | lib.FLAG_GRAD_TPLATE_F32}[dtype]
    fl = tflags | _flags(gset)
    shape = lib.Shape(N, H, W, K, TD, TH, TW)
    wsb = lib.workspace_bytes(N, H, W, K, TD, TH, TW)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    hoff = lib.LIB.mvp_debug_heavy_offset(ctypes.byref(shape))
    heavy = lambda: int(ws[hoff:hoff + 4].view(torch.int32).item())  # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    nan = float("nan")
    tf = gset != "rays_only"
    gs = [torch.full_like(s[n], nan) if tf else None for n in ("primpos", "primrot", "primscale")]
    if gset == "all":
        gs.append(torch.full(tpl.shape, nan, device="cuda", dtype=torch.float32 if dtype != "bf16" else torch.bfloat16))
        gs.append(torch.full_like(warp, nan) if warp is not None else None)
    else:
        gs += [None, None]
    rgba = torch.empty(N, H, W, 4, device="cuda")
    rsat = torch.empty(N, H, W, 3, device="cuda")
    raux = torch.empty(N, H, W, 4, dtype=torch.int32, device="cuda")
    a = lib.ForwardArgs()
    a.shape, a.stepsize, a.fadescale, a.fadeexp, a.flags = shape, s["stepsize"], s.get("fadescale", 8.0), s.get("fadeexp", 8.0), fl
    a.raypos, a.raydir, a.tminmax = P(s["raypos"]), P(s["raydir"]), P(s["tminmax"])
    a.primpos, a.primrot, a.primscale, a.tplate = P(s["primpos"]), P(s["primrot"]), P(s["primscale"]), P(tpl)
    a.rayrgba, a.raysat, a.rayaux = P(rgba), P(rsat), P(raux)
    a.workspace, a.workspace_bytes = P(ws), wsb
    a.clear_grad_primpos, a.clear_grad_primrot, a.clear_grad_primscale, a.clear_grad_tplate, a.clear_grad_warp = (P(g) for g in gs)
    if warp is not None:
        a.algo, a.warp = 1, P(warp)
        a.WD, a.WH, a.WW = warp.shape[2:5]
    lib.check(lib.LIB.mvp_raymarch_forward(ctypes.byref(a), st))
    hf = heavy()
    b = lib.BackwardArgs()
    b.shape, b.stepsize, b.fadescale, b.fadeexp, b.flags = shape, a.stepsize, a.fadescale, a.fadeexp, lib.FLAG_ACCEL_VALID | fl
    b.raypos, b.raydir, b.tminmax = a.raypos, a.raydir, a.tminmax
    b.primpos, b.primrot, b.primscale, b.tplate = a.primpos, a.primrot, a.primscale, a.tplate
    b.grad_rayrgba, b.raysat, b.rayaux = P(grad), P(rsat), P(raux)
    b.grad_primpos, b.grad_primrot, b.grad_primscale, b.grad_tplate = (P(g) for g in gs[:4])
    b.workspace, b.workspace_bytes = P(ws), wsb
    if warp is not None:
        b.algo, b.warp, b.grad_warp = 1, P(warp), P(gs[4])
        b.WD, b.WH, b.WW = a.WD, a.WH, a.WW
    r = None
    if rays:
        r = [torch.full((N, H, W, c), nan, device="cuda") for c in (3, 3, 2)]
        lib.check(lib.LIB.mvp_raymarch_backward_rays(ctypes.byref(b), *(P(t) for t in r), st))
    else:
        lib.check(lib.LIB.mvp_raymarch_backward(ctypes.byref(b), st))
    hb = heavy()
    torch.cuda.synchronize()
    host = lambda t: None if t is None else t.float().cpu().numpy()  # noqa: E731
    return [host(g) for g in gs], (None if r is None else [host(t) for t in r]), (hf, hb)


def check_sets(s, grad, dtype, oracle=True):
    """Every reduced set against the full backward of the same template type, with and without ray gradients; the ray gradients
    of the reduced sets against the fp32 C oracle (on the template's fp32 widening for bf16)."""
    gc = grad.cuda()
    full, _, heavy = gpu_march(s, gc, "all", rays=False, dtype=dtype)
    fullr, fr, _ = gpu_march(s, gc, "all", rays=True, dtype=dtype)
    assert np.abs(full[0]).max() > 0
    for gset, rays in (("no_payload", False), ("no_payload", True), ("rays_only", True)):
        g, r, h = gpu_march(s, gc, gset, rays=rays, dtype=dtype)
        assert h == heavy, (gset, rays)
        assert g[3] is None and g[4] is None
        if gset == "no_payload":
            for nm, x, y in zip(("primpos", "primrot", "primscale"), g[:3], (fullr if rays else full)[:3]):
                assert np.isfinite(x).all() and relerr(x, y) <= ATOMIC_TOL, (gset, rays, nm, relerr(x, y))
        else:
            assert all(x is None for x in g[:3])
        if rays:
            for x, y in zip(r, fr):
                assert np.isfinite(x).all() and relerr(x, y) <= ATOMIC_TOL, (gset, relerr(x, y))
            if oracle:
                sc = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in s.items()}
                if dtype != "fp32":
                    sc["template"] = sc["template"].to(torch.bfloat16).float()
                check_vs_oracle(r, sc, grad)
    return heavy


@pytest.mark.parametrize("dtype", ["fp32", "bf16", "bf16_g32"])
@pytest.mark.parametrize("name", list(CASES))
def test_gpu_grad_sets_named_cases(name, dtype):
    s, grad = build_case(name)
    check_sets(_cuda(s), grad, dtype)


@pytest.mark.parametrize("dtype", ["fp32", "bf16", "bf16_g32"])
@pytest.mark.parametrize("cap", list(DENSE_K3))
@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_gpu_grad_sets_heavy_kernels(name, cap, dtype):
    s, grad = build_dense_case(name, cap)
    N, H, W = s["raypos"].shape[:3]
    heavy = check_sets(_cuda(s), grad, dtype, oracle=dtype == "fp32")
    assert heavy == (N * -(-H // 4) * -(-W // 8),) * 2


def _leaves(s, frozen):
    return [s[k].detach().clone().requires_grad_(not frozen) for k in ("primpos", "primrot", "primscale", "template")]


@pytest.mark.parametrize("planes", [False, True])
def test_gpu_camera_grad_with_a_frozen_avatar(planes):
    """mvpraymarch_camera(camera_grad=True): detached primitives give the undetached call's camera gradients through the rays-only
    backward; detached template alone, the transforms' gradients through the no-payload backward."""
    from ava256_b200 import lib, scene
    from ava256_b200.op import mvpraymarch_camera
    n, H, W = 2, 96, 64
    s, cams = _head(n, H, W, 256, 8)
    s = _cuda(s)
    gout = torch.randn(n, H, W, 4, generator=torch.Generator().manual_seed(5)).cuda()

    def loss_of(out):
        if planes:
            return (out[0] * gout.permute(0, 3, 1, 2)[:, :3]).sum() + (out[1] * gout.permute(0, 3, 1, 2)[:, 3:]).sum()
        return (out * gout).sum()

    flags_seen = []
    orig = lib.LIB.mvp_raymarch_backward_rays

    def spy(b, *rest):
        flags_seen.append(b._obj.flags)
        return orig(b, *rest)

    def run(frozen_prims, frozen_template):
        leaves = [c.clone().requires_grad_(True) for c in cams]
        prims = _leaves(s, frozen_prims)
        if frozen_template:
            prims[3].requires_grad_(False)
        out = mvpraymarch_camera(*leaves, (W, H), scene.VOLRADIUS, s["stepsize"], tuple(prims[:3]), prims[3], None, planes=planes,
                                 camera_grad=True, fadescale=8.0, fadeexp=8.0)
        loss_of(out).backward()
        return out, [t.grad for t in leaves], prims

    lib.LIB.mvp_raymarch_backward_rays = spy
    try:
        out0, cam0, p0 = run(False, False)
        out1, cam1, p1 = run(True, True)
        out2, cam2, p2 = run(False, True)
    finally:
        lib.LIB.mvp_raymarch_backward_rays = orig
    assert [f & (lib.FLAG_NO_TPLATE_GRAD | lib.FLAG_RAY_GRADS_ONLY) for f in flags_seen] == \
        [0, lib.FLAG_RAY_GRADS_ONLY, lib.FLAG_NO_TPLATE_GRAD], flags_seen
    for x, y in zip(out1 if planes else (out1,), out0 if planes else (out0,)):
        assert torch.equal(x, y)                                             # images bit-identical
    for cam in (cam1, cam2):
        for x, y in zip(cam, cam0):
            assert relerr(x.cpu().numpy(), y.cpu().numpy()) <= ATOMIC_TOL
    assert all(t.grad is None for t in p1)
    assert p2[3].grad is None
    for x, y in zip(p2[:3], p0[:3]):
        assert relerr(x.grad.cpu().numpy(), y.grad.cpu().numpy()) <= ATOMIC_TOL


def test_gpu_rays_requiring_grad_with_a_frozen_avatar():
    """Rays that require grad without the ray-gradient option, and a frozen avatar: the op has no gradient to compute, yet its output
    sits in an autograd graph.  backward runs, gives the rays nothing from the image (as the full backward did) and the other terms
    of the loss their gradients; the library's backward is not called.  Both through the drop-in `mvpraymarch` with rays from an
    autograd graph, and through `mvpraymarch_camera(camera_grad=False)` with a pixelcoords tensor and a viewpos that requires grad."""
    from ava256_b200 import scene
    from ava256_b200.op import mvpraymarch, mvpraymarch_camera
    from tests.test_gpu_camera_grads import _Counter
    n, H, W = 1, 64, 48
    s, cams = _head(n, H, W, 256, 8)
    s = _cuda(s)
    prims = (s["primpos"], s["primrot"], s["primscale"])
    with torch.no_grad():
        ref = mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], prims, s["template"], None, fadescale=8.0, fadeexp=8.0)
    leaf = s["raypos"].clone().requires_grad_(True)
    with _Counter("mvp_raymarch_backward", "mvp_raymarch_backward_rays") as cnt:
        out = mvpraymarch(leaf * 1.0, s["raydir"], s["stepsize"], s["tminmax"], prims, s["template"], None, fadescale=8.0, fadeexp=8.0)
        assert out.grad_fn is not None and torch.equal(out.detach(), ref)
        (out.sum() + 2.0 * leaf.sum()).backward()
    assert cnt.n == {"mvp_raymarch_backward": 0, "mvp_raymarch_backward_rays": 0}, cnt.n
    assert torch.equal(leaf.grad, torch.full_like(leaf, 2.0))
    py, px = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    pix = torch.stack([px, py], -1)[None].contiguous().cuda()
    vp = cams[0].clone().requires_grad_(True)
    out = mvpraymarch_camera(vp, cams[1], cams[2], cams[3], pix, scene.VOLRADIUS, s["stepsize"], prims, s["template"], None,
                             camera_grad=False, fadescale=8.0, fadeexp=8.0)
    (out.sum() + vp.sum()).backward()
    assert torch.equal(vp.grad, torch.ones_like(vp))


def test_gpu_no_input_needs_grad_renders_as_inference():
    """Grad mode on, nothing requires grad: the image of torch.no_grad, no gradient buffers, no backward."""
    from ava256_b200 import scene
    from ava256_b200.op import mvpraymarch_camera
    n, H, W = 1, 64, 48
    s, cams = _head(n, H, W, 256, 8)
    s = _cuda(s)
    prims = (s["primpos"], s["primrot"], s["primscale"])
    args = (*cams, (W, H), scene.VOLRADIUS, s["stepsize"], prims, s["template"], None)
    with torch.no_grad():
        ref = mvpraymarch_camera(*args, fadescale=8.0, fadeexp=8.0)
    out = mvpraymarch_camera(*args, camera_grad=True, fadescale=8.0, fadeexp=8.0)
    assert torch.equal(out, ref) and not out.requires_grad and out.grad_fn is None


def test_gpu_retain_graph_follows_the_set():
    """A second backward through the same graph allocates the set's buffers again (MVP_FLAG_ZERO_GRADS) and gives the same result."""
    from ava256_b200 import scene
    from ava256_b200.op import mvpraymarch_camera
    n, H, W = 1, 64, 48
    s, cams = _head(n, H, W, 256, 8)
    s = _cuda(s)
    for frozen_template in (True, False):
        leaves = [c.clone().requires_grad_(True) for c in cams]
        prims = _leaves(s, False)
        prims[3].requires_grad_(not frozen_template)
        out = mvpraymarch_camera(*leaves, (W, H), scene.VOLRADIUS, s["stepsize"], tuple(prims[:3]), prims[3], None,
                                 camera_grad=True, fadescale=8.0, fadeexp=8.0)
        loss = (out * out).sum()
        loss.backward(retain_graph=True)
        first = [t.grad.clone() for t in leaves + prims[:3]]
        for t in leaves + prims[:3]:
            t.grad = None
        loss.backward()
        for x, y in zip(leaves + prims[:3], first):
            assert relerr(x.grad.cpu().numpy(), y.cpu().numpy()) <= ATOMIC_TOL
        assert (prims[3].grad is None) == frozen_template


def test_gpu_pose_recovery_frozen_avatar():
    """The pose recovery of tests/test_gpu_camera_grads.py through the rays-only backward (avatar frozen, the flag checked at the
    library call), to the same tolerances."""
    from ava256_b200 import lib, scene
    from ava256_b200.op import mvpraymarch_camera
    n, H, W = 1, 128, 84
    s, cams = _head(n, H, W, 1024, 8, alpha_mu=3.0, alpha_sigma=3.0)
    s = _cuda(s)
    prims = (s["primpos"], s["primrot"], s["primscale"])

    def render(vp, vr):
        return mvpraymarch_camera(vp, vr, cams[2], cams[3], (W, H), scene.VOLRADIUS, s["stepsize"], prims, s["template"], None,
                                  camera_grad=True, fadescale=8.0, fadeexp=8.0)

    with torch.no_grad():
        target = render(cams[0], cams[1])
    dpos = torch.tensor([[8.0, -6.0, 7.0]], device="cuda", requires_grad=True)        # mm
    rvec = torch.tensor([0.006, -0.005, 0.007], device="cuda", requires_grad=True)      # rad
    opt = torch.optim.Adam([{"params": [dpos], "lr": 0.5}, {"params": [rvec], "lr": 4e-4}])
    hist, flags = [], []
    orig = lib.LIB.mvp_raymarch_backward_rays

    def spy(b, *rest):
        flags.append(b._obj.flags)
        return orig(b, *rest)

    lib.LIB.mvp_raymarch_backward_rays = spy
    try:
        for it in range(60):
            opt.zero_grad()
            vp = (cams[0] + dpos).contiguous()
            vr = (cams[1][0] @ _rotvec(rvec))[None].contiguous()
            loss = ((render(vp, vr) - target) ** 2).mean()
            loss.backward()
            hist.append((float(loss), float(dpos.detach().norm()), float(rvec.detach().norm())))
            opt.step()
    finally:
        lib.LIB.mvp_raymarch_backward_rays = orig
    assert len(flags) == 60 and all(f & lib.FLAG_RAY_GRADS_ONLY for f in flags)
    print("pose recovery (frozen avatar): loss %.4g -> %.4g, position error %.3f -> %.3f mm, rotation error %.5f -> %.5f rad"
          % (hist[0][0], hist[-1][0], hist[0][1], hist[-1][1], hist[0][2], hist[-1][2]))
    assert hist[-1][0] < 0.02 * hist[0][0]
    assert hist[-1][1] < 0.6 * hist[0][1]
    assert hist[-1][2] < 0.55 * hist[0][2]


def test_gpu_camera_only_step_saves_the_template_buffer():
    """8 views of 512x334, K = 4096, 16^3 slabs: the peak memory of a camera-only forward + backward is below the full step's by at
    least 0.9 x the template's size (the template gradient buffer it no longer allocates)."""
    from ava256_b200 import scene
    from ava256_b200.op import mvpraymarch_camera
    n, H, W = 8, 334, 512
    s = scene.make_scene(n, H, W, 4096, 16, device="cuda", alpha_mu=1.0, alpha_sigma=2.0, share_primitives=False)
    s["stepsize"] = 1.0 / 64
    cams = [t.cuda() for t in scene.make_cameras(n, H, W)]
    tbytes = s["template"].numel() * s["template"].element_size()

    def step(frozen):
        leaves = [c.clone().requires_grad_(True) for c in cams]
        prims = _leaves(s, frozen)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = mvpraymarch_camera(*leaves, (W, H), scene.VOLRADIUS, s["stepsize"], tuple(prims[:3]), prims[3], None,
                                 camera_grad=True, fadescale=8.0, fadeexp=8.0)
        out.sum().backward()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        del out, prims, leaves
        return peak

    full, frozen = step(False), step(True)
    print("peak memory of the step: %.1f MB full, %.1f MB camera only; template %.1f MB" % (full / 1e6, frozen / 1e6, tbytes / 1e6))
    assert full - frozen >= 0.9 * tbytes
