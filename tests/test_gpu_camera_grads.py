"""GPU tests of the gradients of rays and cameras (`pytest -m gpu`): mvp_raymarch_backward_rays against the fp32 C oracle
(tests/oracle_rays.c) in every render-kernel instantiation, camera mode against ray tensors, the ray generator's adjoint
mvp_compute_raydirs_backward against torch fp64 autograd, `mvpraymarch_camera(camera_grad=True)` end to end, and a short pose
recovery through the photometric loss.  Gates: max|d|/max|ref| <= 1e-3 per tensor and |sum|x| - sum|ref|| / sum|ref| <= 1e-3
against the oracle; 1e-5 between runs that differ only in the order of the gradient atomics."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from tests.helpers import CASES, DENSE_CASES, DENSE_K3, abi_raymarch, build_case, build_dense_case, relerr, scene_args_np
from tests.oracle_rays import backward_rays, rays_torch

pytestmark = pytest.mark.gpu

TOL = 1e-3
RAY_NAMES = ("raypos", "raydir", "tminmax")


def _cuda(s):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in s.items()}


@contextlib.contextmanager
def ray_backward(N, H, W, extra_flags=0):
    """abi_raymarch's backward becomes mvp_raymarch_backward_rays (with extra_flags OR-ed into its flags); yields the NaN-filled
    ray-gradient tensors it writes."""
    from ava256_b200 import lib
    out = [torch.full((N, H, W, c), float("nan"), device="cuda") for c in (3, 3, 2)]
    plain = lib.LIB.mvp_raymarch_backward

    def call(b, st):
        b._obj.flags |= extra_flags
        return lib.LIB.mvp_raymarch_backward_rays(b, *(ctypes.c_void_p(t.data_ptr()) for t in out), st)

    lib.LIB.mvp_raymarch_backward = call
    try:
        yield out
    finally:
        lib.LIB.mvp_raymarch_backward = plain


def gpu_ray_grads(s, grad, extra_flags=0, **kw):
    camera = kw.get("camera")
    N, H, W = (camera[0].shape[0], camera[5], camera[6]) if camera is not None else s["raypos"].shape[:3]
    with ray_backward(N, H, W, extra_flags) as rays:
        out, rsat, grads, heavy = abi_raymarch(s, grad.cuda(), fwd_flags=kw.pop("fwd_flags", 0) | extra_flags, **kw)
    return out, grads, [r.cpu().numpy() for r in rays], heavy


def check_vs_oracle(rays, s, grad, tol=TOL):
    from oracle import oracle
    a, kw = scene_args_np(s)
    _, rsat = oracle.forward(*a, **kw)
    ref = backward_rays(*a, grad.numpy(), rsat, **kw)[1]
    for nm, x, r in zip(RAY_NAMES, rays, ref):
        assert np.isfinite(x).all(), nm
        assert relerr(x, r) <= tol, (nm, relerr(x, r))
        l1 = np.abs(r).sum()
        assert abs(np.abs(x).astype(np.float64).sum() - l1) <= tol * l1, nm
    assert np.abs(ref[0]).max() > 0


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("name", list(CASES))
def test_gpu_ray_grads_vs_oracle(name, bf16):
    from ava256_b200 import lib
    s, grad = build_case(name)
    if bf16:        # the oracle renders the widened bf16 template: the same numbers the bf16 kernels read
        s["template"] = s["template"].bfloat16().float()
    sg = _cuda(s)
    if bf16:
        sg["template"] = sg["template"].bfloat16()
    _, _, rays, _ = gpu_ray_grads(sg, grad, extra_flags=lib.FLAG_TPLATE_BF16 if bf16 else 0)
    check_vs_oracle(rays, s, grad)


@pytest.mark.parametrize("name", ["head_small", "warp_small", "gradcheck_ragged"])
def test_gpu_ray_grads_primitive_grads_and_options(name):
    """The primitive gradients are the plain backward's; image-plane gradient input, rebuilt lists, a Morton order and shared
    primitives give the ray gradients of the default call."""
    from ava256_b200 import lib
    from ava256_b200.op import morton_order
    s, grad = build_case(name)
    sg = _cuda(s)
    _, _, plain, _ = abi_raymarch(sg, grad.cuda())
    _, grads, base, _ = gpu_ray_grads(sg, grad)
    for x, y in zip(grads, plain):
        assert relerr(x.cpu().numpy(), y.cpu().numpy()) <= 1e-5
    for kw in (dict(planes=True), dict(fwd_flags=lib.FLAG_TEST_TINY_LISTS)):
        _, _, rays, _ = gpu_ray_grads(sg, grad, **kw)
        for x, y in zip(rays, base):
            assert relerr(x, y) <= 1e-5, kw
    order = morton_order(sg["primpos"]).to(torch.int32).contiguous()
    _, _, rays, _ = gpu_ray_grads(sg, grad, order=order)
    so = dict(s)
    oc = order.long().cpu()
    for key in ("primpos", "primrot", "primscale", "template", "warp"):
        if key in so:
            so[key] = torch.gather(so[key], 1, oc.view(oc.shape + (1,) * (so[key].dim() - 2)).expand(so[key].shape)).contiguous()
    check_vs_oracle(rays, so, grad)
    # one set of primitives for all views
    s1 = dict(s)
    for key in ("primpos", "primrot", "primscale", "template", "warp"):
        if key in s1:
            s1[key] = s1[key][:1].expand_as(s1[key]).contiguous()
    _, _, full, _ = gpu_ray_grads(_cuda(s1), grad)
    sh = {k: (v[:1].contiguous() if k in ("primpos", "primrot", "primscale", "template", "warp") else v) for k, v in _cuda(s1).items()}
    _, _, shared, _ = gpu_ray_grads(sh, grad, shared=True)
    for x, y in zip(shared, full):
        assert relerr(x, y) <= 1e-5


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("cap", list(DENSE_K3))
@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_gpu_ray_grads_heavy_kernels(name, cap, bf16):
    """Every 512-entry ray-gradient instantiation (T = 8, 16, runtime dims, algo 1; fp32 and bf16 templates)."""
    from ava256_b200 import lib
    s, grad = build_dense_case(name, cap)
    if bf16:
        s["template"] = s["template"].bfloat16().float()
    sg = _cuda(s)
    if bf16:
        sg["template"] = sg["template"].bfloat16()
    _, _, rays, heavy = gpu_ray_grads(sg, grad, extra_flags=lib.FLAG_TPLATE_BF16 if bf16 else 0)
    print("%s/%s/%s: heavy tiles forward %d, backward %d" % (name, cap, "bf16" if bf16 else "fp32", heavy[0], heavy[1]))
    assert heavy[1] > 0
    check_vs_oracle(rays, s, grad)


def _head(n, H, W, K, T, **kw):
    from ava256_b200 import scene
    s = scene.make_scene(n, H, W, K, T, alpha_mu=kw.get("alpha_mu", 1.0), alpha_sigma=kw.get("alpha_sigma", 2.0), share_primitives=False)
    s["fadescale"], s["fadeexp"] = 8.0, 8.0
    s["stepsize"] = kw.get("stepsize", 1.0 / 64)
    cams = [t.cuda() for t in scene.make_cameras(n, H, W)]
    return s, cams


def _rays_from_cameras(cams, H, W, pixelcoords=None):
    from ava256_b200 import scene
    from ava256_b200.raydirs import compute_raydirs
    return compute_raydirs(*cams, pixelcoords if pixelcoords is not None else (W, H), scene.VOLRADIUS)


def test_gpu_camera_mode_ray_grads_match_ray_tensors():
    from ava256_b200 import scene
    n, H, W = 2, 96, 64
    s, cams = _head(n, H, W, 256, 8)
    grad = torch.randn(n, H, W, 4, generator=torch.Generator().manual_seed(3))
    sg = _cuda(s)
    sg["raypos"], sg["raydir"], sg["tminmax"] = _rays_from_cameras(cams, H, W)
    _, g0, r0, _ = gpu_ray_grads(sg, grad)
    _, g1, r1, _ = gpu_ray_grads(sg, grad, camera=tuple(cams) + (scene.VOLRADIUS, H, W))
    for x, y in zip(r1, r0):
        assert relerr(x, y) <= 1e-5
    for x, y in zip(g1, g0):
        assert relerr(x.cpu().numpy(), y.cpu().numpy()) <= 1e-5


@pytest.mark.parametrize("with_pixelcoords", [False, True])
@pytest.mark.parametrize("N,H,W", [(2, 33, 47), (1, 1024, 667)])
def test_gpu_raydirs_backward_vs_torch_autograd(N, H, W, with_pixelcoords):
    from ava256_b200 import scene
    from ava256_b200.raydirs import raydirs_backward
    cams = scene.make_cameras(N, H, W)
    g = torch.Generator().manual_seed(11)
    pc = None
    if with_pixelcoords:
        py, px = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
        pc = (torch.stack([px, py], -1)[None].repeat(N, 1, 1, 1) + torch.rand(N, H, W, 2, generator=g) - 0.5).contiguous()
    grads = [torch.randn(N, H, W, c, generator=g) for c in (3, 3, 2)]
    out = raydirs_backward(*(t.cuda() for t in cams), pc.cuda() if pc is not None else None, scene.VOLRADIUS, *(t.cuda() for t in grads))
    leaves = [t.double().clone().requires_grad_(True) for t in cams]
    rays = rays_torch(*leaves, pc.double() if pc is not None else (W, H), scene.VOLRADIUS)
    torch.autograd.backward(rays, [t.double() for t in grads])
    for nm, x, r in zip(("viewpos", "viewrot", "focal", "princpt"), out, leaves):
        assert relerr(x.cpu().numpy(), r.grad.numpy()) <= TOL, (nm, relerr(x.cpu().numpy(), r.grad.numpy()))


def _march(cams, pix, s, camera_grad, planes=False):
    from ava256_b200 import scene
    from ava256_b200.op import mvpraymarch_camera
    prims = [s[k].detach().clone().requires_grad_(True) for k in ("primpos", "primrot", "primscale", "template")]
    out = mvpraymarch_camera(*cams, pix, scene.VOLRADIUS, s["stepsize"], tuple(prims[:3]), prims[3], None, planes=planes,
                             camera_grad=camera_grad, fadescale=8.0, fadeexp=8.0)
    return out, prims


class _Counter:
    """Counts the calls of the named C-ABI entry points (wrapped in place, restored on exit)."""

    def __init__(self, *names):
        from ava256_b200 import lib
        self.lib, self.names, self.n = lib, names, {n: 0 for n in names}

    def __enter__(self):
        self.orig = {n: getattr(self.lib.LIB, n) for n in self.names}
        for n in self.names:
            def f(*a, _n=n):
                self.n[_n] += 1
                return self.orig[_n](*a)
            setattr(self.lib.LIB, n, f)
        return self

    def __exit__(self, *exc):
        for n, f in self.orig.items():
            setattr(self.lib.LIB, n, f)


@pytest.mark.parametrize("planes", [False, True])
def test_gpu_mvpraymarch_camera_grad(planes):
    from ava256_b200 import scene
    from oracle import oracle
    n, H, W = 2, 96, 64
    s, cams = _head(n, H, W, 256, 8)
    s = _cuda(s)
    g = torch.Generator().manual_seed(5)
    gout = torch.randn(n, H, W, 4, generator=g).cuda()

    def loss_of(out):
        if planes:
            return (out[0] * gout.permute(0, 3, 1, 2)[:, :3]).sum() + (out[1] * gout.permute(0, 3, 1, 2)[:, 3:]).sum()
        return (out * gout).sum()

    # camera_grad=False: plain op, images and primitive gradients as reference
    out0, p0 = _march(cams, (W, H), s, False, planes)
    loss_of(out0).backward()
    results = {}
    py, px = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    pct = torch.stack([px, py], -1)[None].repeat(n, 1, 1, 1).contiguous().cuda()
    for form, pix in (("tuple", (W, H)), ("tensor", pct)):
        leaves = [c.clone().requires_grad_(True) for c in cams]
        with _Counter("mvp_raymarch_backward_rays", "mvp_compute_raydirs_backward") as cnt:
            out, prims = _march(leaves, pix, s, True, planes)
            loss_of(out).backward()
        assert cnt.n["mvp_raymarch_backward_rays"] == 1 and cnt.n["mvp_compute_raydirs_backward"] == 1, cnt.n
        for x, y in zip(out if planes else (out,), out0 if planes else (out0,)):
            assert torch.equal(x, y), form                                   # images bit-identical
        for x, y in zip(prims, p0):
            assert relerr(x.grad.cpu().numpy(), y.grad.cpu().numpy()) <= 1e-5, form
        results[form] = [t.grad.cpu().numpy() for t in leaves]
    for x, y in zip(results["tuple"], results["tensor"]):
        assert relerr(x, y) <= 1e-5
    # the oracle chain: fp32 C-oracle ray gradients on the same rays, then torch fp64 autograd of the ray formula
    rp, rd, tm = (t.cpu() for t in _rays_from_cameras(cams, H, W))
    sc = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in s.items()}
    a, kw = scene_args_np(dict(sc, raypos=rp, raydir=rd, tminmax=tm))
    _, rsat = oracle.forward(*a, **kw)
    ref_rays = backward_rays(*a, gout.cpu().numpy(), rsat, **kw)[1]
    leaves = [c.cpu().double().clone().requires_grad_(True) for c in cams]
    torch.autograd.backward(rays_torch(*leaves, (W, H), scene.VOLRADIUS), [torch.from_numpy(r) for r in ref_rays])
    for nm, x, r in zip(("viewpos", "viewrot", "focal", "princpt"), results["tuple"], leaves):
        print("camera gradient %s: max|d|/max|ref| %.2e" % (nm, relerr(x, r.grad.numpy())))
        assert relerr(x, r.grad.numpy()) <= TOL, nm
    # no camera tensor requires grad: the plain backward runs and the camera gets nothing
    leaves = [c.clone() for c in cams]
    with _Counter("mvp_raymarch_backward_rays", "mvp_compute_raydirs_backward", "mvp_raymarch_backward") as cnt:
        out, prims = _march(leaves, (W, H), s, True, planes)
        loss_of(out).backward()
    assert cnt.n == {"mvp_raymarch_backward_rays": 0, "mvp_compute_raydirs_backward": 0, "mvp_raymarch_backward": 1}, cnt.n
    assert all(t.grad is None for t in leaves)
    # only some camera tensors require grad: the others get None
    leaves = [c.clone() for c in cams]
    leaves[0].requires_grad_(True)
    out, _ = _march(leaves, (W, H), s, True, planes)
    loss_of(out).backward()
    assert leaves[0].grad is not None and all(t.grad is None for t in leaves[1:])


@pytest.mark.parametrize("form", ["tuple", "tensor"])
def test_gpu_camera_grad_sees_in_place_changes(form):
    """The adjoint recomputes the rays from the camera tensors, so they are saved for backward: changing one in place between the
    forward and the backward raises, as autograd does for any saved input."""
    n, H, W = 1, 32, 24
    s, cams = _head(n, H, W, 64, 8)
    s = _cuda(s)
    py, px = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    pix = (W, H) if form == "tuple" else torch.stack([px, py], -1)[None].contiguous().cuda()
    leaf = cams[0].clone().requires_grad_(True)
    vp = leaf * 1.0
    out, _ = _march([vp] + cams[1:], pix, s, True)
    with torch.no_grad():
        vp.add_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        out.sum().backward()


def _rotvec(w):
    th = torch.sqrt((w * w).sum() + 1e-20)
    k = w / th
    Kx = torch.zeros(3, 3, device=w.device, dtype=w.dtype)
    Kx[0, 1], Kx[0, 2], Kx[1, 0], Kx[1, 2], Kx[2, 0], Kx[2, 1] = -k[2], k[1], k[2], -k[0], -k[1], k[0]
    return torch.eye(3, device=w.device) + torch.sin(th) * Kx + (1 - torch.cos(th)) * (Kx @ Kx)


def test_gpu_pose_recovery():
    """Perturb one view's position (12 mm at 1.4 m) and orientation (0.6 degrees), then take a fixed number of Adam steps on the L2
    image loss against the unperturbed render: the loss and the pose error must both fall clearly."""
    from ava256_b200 import scene
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
    hist = []
    for it in range(60):
        opt.zero_grad()
        vp = (cams[0] + dpos).contiguous()
        vr = (cams[1][0] @ _rotvec(rvec))[None].contiguous()
        loss = ((render(vp, vr) - target) ** 2).mean()
        loss.backward()
        hist.append((float(loss), float(dpos.detach().norm()), float(rvec.detach().norm())))
        opt.step()
    print("pose recovery: loss %.4g -> %.4g, position error %.3f -> %.3f mm, rotation error %.5f -> %.5f rad"
          % (hist[0][0], hist[-1][0], hist[0][1], hist[-1][1], hist[0][2], hist[-1][2]))
    # measured on an H100 80GB HBM3 (700 W): loss 392.8 -> 1.519, position error 12.21 -> 5.93 mm, rotation error 0.01049 -> 0.00425
    assert hist[-1][0] < 0.02 * hist[0][0]
    assert hist[-1][1] < 0.6 * hist[0][1]
    assert hist[-1][2] < 0.55 * hist[0][2]
