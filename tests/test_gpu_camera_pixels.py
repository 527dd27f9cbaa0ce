"""GPU tests of the camera form at caller-given sample positions: `mvpraymarch_camera` with a pixelcoords tensor [N,H,W,2] generates
each ray inside the render kernels from the camera and its own sample position (C-ABI mvp_raymarch_forward_pixels /
mvp_raymarch_backward_pixels) and must equal the two-call form `compute_raydirs(..., pixelcoords, ...)` -> `mvpraymarch(...)`: the
same image bits, gradients within 1e-5 of max|.|.  Sample fields: the integer grid, crops at integer offsets, a stride-2 grid,
half-pixel centres (culled through the affine map) and a shuffled grid (the all-slabs fallback)."""
import contextlib
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

NAMES = ("primpos", "primrot", "primscale", "template")
TOL = 1e-5


def _trelerr(a, b):
    return float((a.float() - b.float()).abs().max()) / max(float(b.float().abs().max()), 1e-30)


def _coords(kind, n, H, W, seed=0):
    """[n,H,W,2] float32 CUDA sample positions (see tests/test_emul_camera_pixels.py)."""
    py, px = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    g = torch.Generator().manual_seed(seed)
    out = []
    for v in range(n):
        if kind == "crop":
            x, y = px + (5 + 2 * v), py + (3 - v)
        elif kind == "stride2":
            x, y = 2 * px - W // 2, 2 * py - H // 2
        elif kind == "half":
            x, y = px + 0.5, py + 0.5
        else:
            x, y = px, py
        pc = torch.stack([x, y], -1)
        if kind == "shuffled":
            pc = pc.reshape(-1, 2)[torch.randperm(H * W, generator=g)].reshape(H, W, 2)
        out.append(pc)
    return torch.stack(out).contiguous().cuda()


def _scene(n, H, W, K, T, view_offset=2, **kw):
    from ava256_b200 import scene
    cams = tuple(t.cuda() for t in scene.make_cameras(n, H, W, view_offset=view_offset))
    s = scene.make_scene(n, H, W, K, T, view_offset=view_offset, device="cuda", **kw)
    return cams, s


def _march(fused, cams, pc, step, prims, warp=None, planes=False, view_set=None, tgd=None, **kw):
    """The fused call (mvpraymarch_camera with the tensor) or the two-call form on the same inputs."""
    from ava256_b200 import op, scene
    from extensions.utils.utils import compute_raydirs
    if fused:
        return op.mvpraymarch_camera(*cams, pc, scene.VOLRADIUS, step, tuple(prims[:3]), prims[3], warp, planes=planes,
                                     template_grad_dtype=tgd, view_set=view_set, **kw)
    rp, rd, tmm = compute_raydirs(*cams, pc, scene.VOLRADIUS)
    if view_set is not None:
        return op.mvpraymarch_sets(rp, rd, step, tmm, tuple(prims[:3]), prims[3], warp, view_set, planes=planes,
                                   template_grad_dtype=tgd, **kw)
    march = op.mvpraymarch_planes if planes else op.mvpraymarch
    with op.template_grad_dtype(tgd) if tgd is not None else contextlib.nullcontext():
        return march(rp, rd, step, tmm, tuple(prims[:3]), prims[3], warp, **kw)


def _pair(cams, pc, step, base, grad, warp=None, planes=False, **kw):
    """Images and gradients of the fused call and of the two-call form."""
    res = []
    for fused in (True, False):
        leaves = [t.detach().clone().requires_grad_(True) for t in base]
        wl = warp.detach().clone().requires_grad_(True) if warp is not None else None
        out = _march(fused, cams, pc, step, leaves, warp=wl, planes=planes, **kw)
        outs = out if planes else (out,)
        if planes:
            g = grad.permute(0, 3, 1, 2)
            torch.autograd.backward(list(outs), [g[:, :3].contiguous(), g[:, 3:].contiguous()])
        else:
            out.backward(grad)
        res.append(([o.detach() for o in outs], [x.grad for x in leaves] + ([wl.grad] if wl is not None else [])))
    torch.cuda.synchronize()
    return res


def _check(res, bf16_sums=False):
    """Images bit-equal, gradients within TOL.  bf16_sums: the template gradient is accumulated in bf16 (every reduction rounds the
    running sum, so two orders of the same reductions differ by bf16 roundings): within the bf16 gates of test_emul_bf16_payload."""
    from tests.test_emul_bf16_payload import GATE_L1, GATE_MAX
    from tests.test_gpu_bf16_payload import _tgrad_errors
    (o1, g1), (o2, g2) = res
    assert float(o2[-1].max()) > 0.05
    for a, b in zip(o1, o2):
        assert torch.equal(a, b)
    for i, (a, b) in enumerate(zip(g1, g2)):
        assert a.dtype == b.dtype and bool(torch.isfinite(a.float()).all()), i
        if bf16_sums and i == 3:
            emax, el1 = _tgrad_errors(a, b)
            assert emax <= GATE_MAX and el1 <= GATE_L1, (emax, el1)
        else:
            assert _trelerr(a, b) <= TOL, (i, _trelerr(a, b))


@pytest.mark.parametrize("n,H,W,K,T,mu,sg,kind", [(3, 96, 70, 256, 8, 1.0, 2.0, k) for k in ("grid", "crop", "stride2", "half", "shuffled")] +
                         [(1, 1024, 667, 16384, 8, 17.0, 6.0, k) for k in ("half", "crop")])
def test_pixels_identical_to_two_call_form(n, H, W, K, T, mu, sg, kind):
    """A small multi-view scene with every kind of field, and one full C3 view (the benchmark's shape) with the dataset's pixel
    centres and a crop; inference mode (the kGrad = false kernels) gives the same image as well."""
    cams, s = _scene(n, H, W, K, T, alpha_mu=mu, alpha_sigma=sg)
    pc = _coords(kind, n, H, W)
    step = s["stepsize"] if H >= 512 else 1.0 / 64
    grad = torch.randn(n, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    res = _pair(cams, pc, step, [s[k] for k in NAMES], grad)
    _check(res)
    with torch.no_grad():
        out0 = _march(True, cams, pc, step, [s[k] for k in NAMES])
    assert torch.equal(out0, res[1][0][0])
    if kind == "grid":                                              # the integer grid as a tensor is the tuple form
        from ava256_b200 import op, scene
        with torch.no_grad():
            out_t = op.mvpraymarch_camera(*cams, (W, H), scene.VOLRADIUS, step, tuple(s[k] for k in NAMES[:3]), s["template"], None)
        assert torch.equal(out_t, out0)
    # a non-contiguous tensor (a strided view of a larger field) is taken as well
    if kind == "crop" and n > 1:
        big = torch.zeros(n, H, 2 * W, 2, device="cuda")
        big[:, :, ::2] = pc
        with torch.no_grad():
            assert torch.equal(_march(True, cams, big[:, :, ::2], step, [s[k] for k in NAMES]), out0)


@pytest.mark.parametrize("opt", ["view_set", "bf16", "bf16_grad_f32", "planes", "usebvh", "algo1"])
def test_pixels_options_match_two_call_form(opt):
    from tests.helpers import make_warp
    n, H, W, K, T = 4, 96, 70, 256, 8
    cams, s = _scene(n, H, W, K, T, alpha_mu=1.0, alpha_sigma=2.0)
    pc = _coords("crop", n, H, W)
    grad = torch.randn(n, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    base = [s[k] for k in NAMES]
    kw, warp = {}, None
    if opt == "view_set":
        base = [t[:2].contiguous() for t in base]
        kw["view_set"] = torch.tensor([1, 0, 1, 0], dtype=torch.int32, device="cuda")
    elif opt.startswith("bf16"):
        base[3] = base[3].to(torch.bfloat16)
        if opt == "bf16_grad_f32":
            kw["tgd"] = torch.float32
    elif opt == "planes":
        kw["planes"] = True
    elif opt == "usebvh":
        kw["usebvh"] = True
    elif opt == "algo1":
        warp, kw["algo"] = make_warp(n, K, 4, 4, 4).cuda(), 1
    _check(_pair(cams, pc, 1.0 / 64, base, grad, warp=warp, **kw), bf16_sums=opt == "bf16")


@contextlib.contextmanager
def _pixels_calls(pc, rays=None):
    """helpers.abi_raymarch through the pixels entry points (rays: the three ray-gradient outputs, or None)."""
    from ava256_b200 import lib
    P = lambda x: None if x is None else ctypes.c_void_p(x.data_ptr())  # noqa: E731
    fwd, bwd = lib.LIB.mvp_raymarch_forward, lib.LIB.mvp_raymarch_backward
    rp = [P(r) for r in rays] if rays is not None else [None] * 3
    lib.LIB.mvp_raymarch_forward = lambda a, st: lib.LIB.mvp_raymarch_forward_pixels(a, P(pc), None, 0, st)
    lib.LIB.mvp_raymarch_backward = lambda b, st: lib.LIB.mvp_raymarch_backward_pixels(b, P(pc), None, 0, *rp, st)
    try:
        yield
    finally:
        lib.LIB.mvp_raymarch_forward, lib.LIB.mvp_raymarch_backward = fwd, bwd


@contextlib.contextmanager
def _ray_backward(rays):
    from ava256_b200 import lib
    P = lambda x: ctypes.c_void_p(x.data_ptr())  # noqa: E731
    bwd = lib.LIB.mvp_raymarch_backward
    lib.LIB.mvp_raymarch_backward = lambda b, st: lib.LIB.mvp_raymarch_backward_rays(b, *(P(r) for r in rays), st)
    try:
        yield
    finally:
        lib.LIB.mvp_raymarch_backward = bwd


def _fallback_flags(ws, shape):
    from ava256_b200 import lib
    off = lib.LIB.mvp_debug_view_fallback_offset(ctypes.byref(shape))
    return ws[off:off + 4 * shape.N].view(torch.int32).tolist()


@pytest.mark.parametrize("kind", ["crop", "shuffled"])
def test_pixels_heavy_kernels_and_ray_grads_through_the_c_abi(kind):
    """16384 slabs of twice their usual size in a small image: the tiles' lists outgrow the fast kernels, so the 512-entry kernels render and
    differentiate the crop (mvp_debug_heavy_offset counts them) -- with the culled accel structure for the crop and the all-slabs
    fallback for the shuffled field (mvp_debug_view_fallback_offset).  The ray gradients of mvp_raymarch_backward_pixels equal those
    of mvp_raymarch_backward_rays on the two-call form's rays, and the camera gradients chained from them (mvp_compute_raydirs_backward
    at the same pixelcoords) agree."""
    from ava256_b200 import lib, scene
    from ava256_b200.raydirs import raydirs_backward
    from extensions.utils.utils import compute_raydirs
    from tests.helpers import abi_raymarch
    n, H, W, K, T = 2, 128, 84, 16384, 8
    cams, s = _scene(n, H, W, K, T, alpha_mu=0.3, alpha_sigma=1.0)
    s["primscale"] = (s["primscale"] * 0.5).contiguous()
    s["stepsize"] = 1.0 / 64
    pc = _coords(kind, n, H, W, seed=1)
    grad = torch.randn(n, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    rp, rd, tmm = compute_raydirs(*cams, pc, scene.VOLRADIUS)
    r_ref = [torch.empty(n, H, W, c, device="cuda") for c in (3, 3, 2)]
    with _ray_backward(r_ref):
        ref = abi_raymarch(dict(s, raypos=rp, raydir=rd, tminmax=tmm), grad, clear_in_forward=True)
    r_got = [torch.empty(n, H, W, c, device="cuda") for c in (3, 3, 2)]
    keep = {}
    with _pixels_calls(pc, r_got):
        got = abi_raymarch(s, grad, camera=cams + (scene.VOLRADIUS, H, W), keep=keep, clear_in_forward=True)
    torch.cuda.synchronize()
    print("%s: heavy tiles forward %d, backward %d" % (kind, *got[3]))
    assert got[3][0] > 0 and got[3][1] > 0 and got[3] == ref[3]
    assert _fallback_flags(keep["workspace"], lib.Shape(n, H, W, K, T, T, T)) == ([1] * n if kind == "shuffled" else [0] * n)
    assert float(ref[0][..., 3].max()) > 0.05
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    for i, (a, b) in enumerate(zip(got[2], ref[2])):
        assert _trelerr(a, b) <= TOL, i
    for i, (a, b) in enumerate(zip(r_got, r_ref)):
        assert _trelerr(a, b) <= TOL, ("ray", i)
    c_got = raydirs_backward(*cams, pc, scene.VOLRADIUS, *r_got)
    c_ref = raydirs_backward(*cams, pc, scene.VOLRADIUS, *r_ref)
    for i, (a, b) in enumerate(zip(c_got, c_ref)):
        assert _trelerr(a, b) <= TOL, ("camera", i)



@pytest.mark.parametrize("kind", ["crop", "shuffled"])
def test_pixels_camera_grad_matches_differentiable_two_call_form(kind):
    """mvpraymarch_camera(pixelcoords tensor, camera_grad=True) against the differentiable two-call chain on the same tensor: the
    rays of compute_raydirs, the ray-tensor raymarch with its ray gradients (mvp_raymarch_backward_rays) and the ray generator's
    adjoint at the same pixelcoords.  Images bit-equal, primitive and camera gradients within 1e-5 of max|.|."""
    from ava256_b200 import op, scene
    from ava256_b200.raydirs import raydirs_backward
    from extensions.utils.utils import compute_raydirs
    from tests.helpers import abi_raymarch
    n, H, W, K, T = 2, 96, 64, 256, 8
    cams, s = _scene(n, H, W, K, T, alpha_mu=1.0, alpha_sigma=2.0)
    s["stepsize"] = 1.0 / 64
    pc = _coords(kind, n, H, W, seed=2)
    grad = torch.randn(n, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    cl = [c.clone().requires_grad_(True) for c in cams]
    pl = [s[k].detach().clone().requires_grad_(True) for k in NAMES]
    out = op.mvpraymarch_camera(*cl, pc, scene.VOLRADIUS, s["stepsize"], tuple(pl[:3]), pl[3], None, camera_grad=True)
    out.backward(grad)
    rp, rd, tmm = compute_raydirs(*cams, pc, scene.VOLRADIUS)
    r_ref = [torch.empty(n, H, W, c, device="cuda") for c in (3, 3, 2)]
    with _ray_backward(r_ref):
        ref = abi_raymarch(dict(s, raypos=rp, raydir=rd, tminmax=tmm), grad, clear_in_forward=True)
    c_ref = raydirs_backward(*cams, pc, scene.VOLRADIUS, *r_ref)
    torch.cuda.synchronize()
    assert float(ref[0][..., 3].max()) > 0.05 and torch.equal(out.detach(), ref[0])
    for nm, a, b in zip(NAMES, [x.grad for x in pl], ref[2]):
        assert _trelerr(a, b) <= TOL, nm
    for nm, a, b in zip(("viewpos", "viewrot", "focal", "princpt"), [x.grad for x in cl], c_ref):
        assert float(b.abs().max()) > 0 and _trelerr(a, b) <= TOL, nm
