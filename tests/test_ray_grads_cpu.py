"""CPU tests of the gradients of rays and cameras: the fp64 C oracle's ray gradients against torch autograd of the reference's
loop with attached positions (tests/torch_ref_rays.py); the product kernels' ray-gradient backward on the CPU emulation
(tests/emul/) against the fp32 C oracle, in every instantiation and build variant the suite iterates; the ray generator's
adjoint (host build of raydirs.cu) against torch fp64 autograd; and the C-ABI of the two new entry points."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from tests.helpers import CASES, DENSE_CASES, DENSE_K3, build_case, build_dense_case, gradcheck_like_scene, relerr, scene_args_np
from tests.oracle_rays import backward_rays, rays_torch

RAY_TOL = 1e-4          # emulated kernels vs the fp32 oracle (same IEEE arithmetic; sums in another order)
RAY_NAMES = ("raypos", "raydir", "tminmax")


@pytest.fixture()
def kernels():
    from tests.emul import kernels as k
    k.use_variant(())
    k.load()
    yield k
    k.set_lane_order("forward")
    k.use_variant(())


@contextlib.contextmanager
def ray_backward(kernels, N, H, W):
    """Makes kernels.forward_backward call mvp_raymarch_backward_rays instead of mvp_raymarch_backward; yields the NaN-filled
    ray-gradient arrays it writes."""
    L = kernels.load()
    L.mvp_raymarch_backward_rays.restype = ctypes.c_int
    L.mvp_raymarch_backward_rays.argtypes = [ctypes.c_void_p] * 5
    out = [np.full((N, H, W, 3), np.nan, np.float32), np.full((N, H, W, 3), np.nan, np.float32), np.full((N, H, W, 2), np.nan, np.float32)]
    plain = L.mvp_raymarch_backward
    P = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    L.mvp_raymarch_backward = lambda b, st: L.mvp_raymarch_backward_rays(ctypes.addressof(b._obj), P(out[0]), P(out[1]), P(out[2]), st)
    try:
        yield out
    finally:
        L.mvp_raymarch_backward = plain


def emulated_ray_grads(kernels, a, kw, grad, **opts):
    N, H, W = a[0].shape[:3] if a[0] is not None else opts["camera"][0].shape[0:1] + tuple(opts["camera"][5:7])
    with ray_backward(kernels, N, H, W) as rays:
        out, raysat, grads = kernels.forward_backward(*a, grad_rayrgba=grad, **kw, **opts)
    return out, raysat, grads, rays


def check_rays(rays, ref, tol=RAY_TOL):
    for nm, x, r in zip(RAY_NAMES, rays, ref):
        assert np.isfinite(x).all(), nm
        assert relerr(x, r) <= tol, (nm, relerr(x, r))
    assert np.abs(ref[0]).max() > 0, "the scene must give the rays a gradient"


# ---- fp64 oracle == torch autograd of the attached loop ----------------------------------------------------------------
# The named cases on which the C oracle and the reference's Python loop (oracle/torch_ref.py) already agree on the primitive
# gradients; on gradcheck_small, gradcheck_ragged and many_overlaps they do not, with positions detached as well, so those
# cases pin nothing about the rays (the kernels are checked on them against the fp32 oracle below).
TORCH_CASES = ["tiny", "noncubic", "warp_small", "many_views", "head_small", "warp_head", "head_t16"]


@pytest.mark.parametrize("name", TORCH_CASES)
def test_oracle_f64_ray_grads_match_torch_autograd(name):
    from oracle import oracle
    from tests.torch_ref_rays import ray_grads_torch
    s, grad = build_case(name)
    a, kw = scene_args_np(s, np.float64)
    _, raysat = oracle.forward(*a, dtype=np.float64, **kw)
    prim, rays = backward_rays(*a, grad.numpy().astype(np.float64), raysat, dtype=np.float64, **kw)
    t = {k: (v.double() if torch.is_tensor(v) else v) for k, v in s.items()}
    ref = ray_grads_torch(t["raypos"], t["raydir"], t["stepsize"], t["tminmax"], t["primpos"], t["primrot"], t["primscale"],
                          t["template"], grad.double(), fadescale=s["fadescale"], fadeexp=s["fadeexp"], warp=t.get("warp"))
    for nm, mine, theirs in zip(RAY_NAMES, rays, ref[1:]):
        assert relerr(mine, theirs.numpy()) <= 1e-9, (nm, relerr(mine, theirs.numpy()))
    assert np.abs(rays[0]).max() > 0
    # the primitive gradients of the extended oracle are the plain oracle's
    for x, y in zip(prim, oracle.backward(*a, grad.numpy().astype(np.float64), raysat, dtype=np.float64, **kw)):
        assert relerr(x, y) <= 1e-12                  # summation order of the oracle's threads only


def test_oracle_ray_grads_f32_close_to_f64():
    from oracle import oracle
    s, grad = build_case("gradcheck_small")
    out = []
    for dt in (np.float32, np.float64):
        a, kw = scene_args_np(s, dt)
        _, raysat = oracle.forward(*a, dtype=dt, **kw)
        out.append(backward_rays(*a, grad.numpy().astype(dt), raysat, dtype=dt, **kw)[1])
    for x, y in zip(*out):
        assert relerr(x, y) < 2e-4


# ---- emulated product kernels vs the fp32 oracle ------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_emulated_ray_grads_vs_oracle(kernels, name):
    from oracle import oracle
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    _, _, plain = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    out, raysat, grads, rays = emulated_ray_grads(kernels, a, kw, grad.numpy())
    _, rsat = oracle.forward(*a, **kw)
    prim, ref = backward_rays(*a, grad.numpy(), rsat, **kw)
    check_rays(rays, ref)
    for nm, g, r, q in zip(("primpos", "primrot", "primscale", "template", "warp"), grads, prim, plain):
        assert relerr(g, r) <= 1e-4, nm
        assert relerr(g, q) <= 1e-5, nm              # the plain backward's, up to the order of the atomics


@pytest.mark.parametrize("cap", list(DENSE_K3))
@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_emulated_ray_grads_heavy_kernels(kernels, name, cap):
    """The 512-entry instantiations (every tile of these scenes is heavy), uncapped and at the reference's 512-entry cap."""
    from oracle import oracle
    s, grad = build_dense_case(name, cap)
    a, kw = scene_args_np(s)
    _, _, _, rays = emulated_ray_grads(kernels, a, kw, grad.numpy())
    assert kernels.last_heavy_tiles[1] > 0
    _, rsat = oracle.forward(*a, **kw)
    check_rays(rays, backward_rays(*a, grad.numpy(), rsat, **kw)[1])


def _bf16_pair(kernels, s, grad, **opts):
    """Ray gradients of the scene with its template rounded to bf16: once from the bf16 kernels (MVP_FLAG_TPLATE_BF16; the template
    as uint16 bit patterns in fp32-typed words, as tests/test_emul_bf16_payload.py passes it) and once from the fp32 kernels on the
    widened template.  Returns (bf16 rays, fp32 rays, widened scene arguments, kwargs)."""
    from ava256_b200 import lib
    from tests.test_emul_bf16_payload import from_bf16, to_bf16
    a, kw = scene_args_np(s)
    tb = to_bf16(a[7])
    a32, ab = list(a), list(a)
    a32[7], ab[7] = from_bf16(tb), tb.view(np.float32)
    _, _, _, r32 = emulated_ray_grads(kernels, a32, kw, grad, **opts)
    heavy32 = kernels.last_heavy_tiles
    f = lib.FLAG_TPLATE_BF16
    _, _, _, rb = emulated_ray_grads(kernels, ab, kw, grad, **dict(opts, fwd_flags=opts.get("fwd_flags", 0) | f,
                                                                  bwd_flags=opts.get("bwd_flags", 0) | f))
    assert kernels.last_heavy_tiles == heavy32
    return rb, r32, a32, kw


@pytest.mark.parametrize("name", list(CASES))
def test_emulated_ray_grads_bf16_template(kernels, name):
    """The bf16-template instantiations: their ray gradients are the fp32 kernels' on the widened template (the template is only
    read; its bf16 gradient does not enter the rays), and the fp32 oracle's."""
    from oracle import oracle
    s, grad = build_case(name)
    rb, r32, a32, kw = _bf16_pair(kernels, s, grad.numpy())
    for x, y in zip(rb, r32):
        assert relerr(x, y) <= 1e-5
    _, rsat = oracle.forward(*a32, **kw)
    check_rays(rb, backward_rays(*a32, grad.numpy(), rsat, **kw)[1])


@pytest.mark.parametrize("cap", list(DENSE_K3))
@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_emulated_ray_grads_bf16_template_heavy_kernels(kernels, name, cap):
    from oracle import oracle
    s, grad = build_dense_case(name, cap)
    rb, r32, a32, kw = _bf16_pair(kernels, s, grad.numpy())
    assert kernels.last_heavy_tiles[1] > 0
    for x, y in zip(rb, r32):
        assert relerr(x, y) <= 1e-5
    _, rsat = oracle.forward(*a32, **kw)
    check_rays(rb, backward_rays(*a32, grad.numpy(), rsat, **kw)[1])


@pytest.mark.parametrize("name", ["head_small", "warp_small", "gradcheck_ragged"])
def test_emulated_ray_grads_rebuilt_lists_planes_order_shared(kernels, name):
    """Lists rebuilt in the backward (forward keeps at most 16 entries), image-plane gradient input, a Morton marching order
    and one set of primitives shared by the views: each against the ray gradients of the default call."""
    from ava256_b200 import lib
    from ava256_b200.op import morton_codes
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    _, _, _, base = emulated_ray_grads(kernels, a, kw, grad.numpy())
    for opts in (dict(fwd_flags=lib.FLAG_TEST_TINY_LISTS), dict(planes=True)):
        _, _, _, rays = emulated_ray_grads(kernels, a, kw, grad.numpy(), **opts)
        for x, y in zip(rays, base):
            assert relerr(x, y) <= 1e-5, opts
    # Morton order: changes the result only through saturation, so compare with the oracle run in that order
    from oracle import oracle
    order = torch.sort(morton_codes(s["primpos"]), dim=-1, stable=True)[1].to(torch.int32).numpy()
    _, _, _, rays = emulated_ray_grads(kernels, a, kw, grad.numpy(), order=order)
    ao = list(a)
    for i, key in ((4, "primpos"), (5, "primrot"), (6, "primscale"), (7, "template")):
        ao[i] = np.take_along_axis(a[i], order.reshape(order.shape + (1,) * (a[i].ndim - 2)).astype(np.int64), axis=1)
    kwo = dict(kw)
    if "warp" in kw:
        kwo["warp"] = np.take_along_axis(kw["warp"], order.reshape(order.shape + (1,) * 4).astype(np.int64), axis=1)
    _, rsat = oracle.forward(*ao, **kwo)
    check_rays(rays, backward_rays(*ao, grad.numpy(), rsat, **kwo)[1])


@pytest.mark.parametrize("name", ["head_small", "warp_head"])
def test_emulated_ray_grads_shared_primitives(kernels, name):
    from ava256_b200 import lib
    s, grad = build_case(name)
    s = dict(s)
    for key in ("primpos", "primrot", "primscale", "template", "warp"):
        if key in s:
            s[key] = s[key][:1].expand_as(s[key]).contiguous()
    a, kw = scene_args_np(s)
    _, _, _, full = emulated_ray_grads(kernels, a, kw, grad.numpy())
    a1 = list(a)
    for i in (4, 5, 6, 7):
        a1[i] = np.ascontiguousarray(a[i][:1])
    kw1 = dict(kw)
    if "warp" in kw:
        kw1["warp"] = np.ascontiguousarray(kw["warp"][:1])
    _, _, _, shared = emulated_ray_grads(kernels, a1, kw1, grad.numpy(), fwd_flags=lib.FLAG_SHARED_PRIMS, bwd_flags=lib.FLAG_SHARED_PRIMS)
    for x, y in zip(shared, full):
        assert relerr(x, y) <= 1e-5


@pytest.mark.parametrize("order", ["reverse", "random"])
@pytest.mark.parametrize("name", ["head_small", "warp_small", "many_overlaps"])
def test_emulated_ray_grads_do_not_depend_on_lane_schedule(kernels, name, order):
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    _, _, _, r0 = emulated_ray_grads(kernels, a, kw, grad.numpy())
    kernels.set_lane_order(order)
    _, _, _, r1 = emulated_ray_grads(kernels, a, kw, grad.numpy())
    for x, y in zip(r0, r1):
        assert relerr(x, y) <= 1e-5


def _variants():
    from tests.test_emul_kernels import VARIANTS
    return VARIANTS


@pytest.mark.parametrize("variant", list(_variants()))
@pytest.mark.parametrize("name", ["head_small", "warp_small", "gradcheck_ragged", "noncubic"])
def test_emulated_ray_grads_in_every_build_variant(kernels, name, variant):
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    _, _, _, r0 = emulated_ray_grads(kernels, a, kw, grad.numpy())
    kernels.use_variant(_variants()[variant], opt="-O0")
    for order in ("forward", "random"):
        kernels.set_lane_order(order)
        _, _, _, r1 = emulated_ray_grads(kernels, a, kw, grad.numpy())
        for x, y in zip(r0, r1):
            assert relerr(x, y) <= 1e-5


@pytest.mark.parametrize("n,H,W,K,T", [(2, 64, 42, 64, 8), (1, 13, 19, 16, 4)])
def test_emulated_camera_mode_ray_grads_match_ray_tensors(kernels, n, H, W, K, T):
    """Camera mode generates the rays mvp_compute_raydirs writes, bit for bit: the per-ray gradients of both forms agree."""
    from ava256_b200 import scene
    from tests.emul.build import build_aux
    aux = ctypes.CDLL(build_aux())
    s = scene.make_scene(n, H, W, K, T, alpha_mu=1.0, alpha_sigma=2.0, share_primitives=False)
    s["fadescale"], s["fadeexp"] = 8.0, 8.0
    vp, vr, fo, pp = scene.make_cameras(n, H, W)
    rays = [np.empty((n, H, W, c), np.float32) for c in (3, 3, 2)]
    P = lambda t: ctypes.c_void_p(t.ctypes.data) if t is not None else None  # noqa: E731
    cam_np = [np.ascontiguousarray(t.numpy()) for t in (vp, vr, fo, pp)]
    aux.mvp_compute_raydirs.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 5 + [ctypes.c_float] + [ctypes.c_void_p] * 4
    assert aux.mvp_compute_raydirs(n, H, W, *(P(t) for t in cam_np), None, scene.VOLRADIUS, *(P(t) for t in rays), None) == 0
    s["raypos"], s["raydir"], s["tminmax"] = (torch.from_numpy(r) for r in rays)
    grad = torch.randn(n, H, W, 4, generator=torch.Generator().manual_seed(8))
    a, kw = scene_args_np(s)
    _, _, g0, r0 = emulated_ray_grads(kernels, a, kw, grad.numpy())
    ac = [None, None] + a[2:3] + [None] + a[4:]
    _, _, g1, r1 = emulated_ray_grads(kernels, ac, kw, grad.numpy(), camera=tuple(cam_np) + (scene.VOLRADIUS, H, W))
    for x, y in zip(r1, r0):
        assert relerr(x, y) <= 1e-5
    for x, y in zip(g1, g0):
        assert relerr(x, y) <= 1e-5


# ---- camera adjoint: host build of raydirs.cu vs torch fp64 autograd ---------------------------------------------------
def _camera_adjoint_case(N, H, W, with_pixelcoords, seed=3):
    from ava256_b200 import scene
    vp, vr, fo, pp = scene.make_cameras(N, H, W)
    g = torch.Generator().manual_seed(seed)
    pc = None
    if with_pixelcoords:
        py, px = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
        pc = (torch.stack([px, py], -1)[None].repeat(N, 1, 1, 1) + torch.rand(N, H, W, 2, generator=g) - 0.5).contiguous()
    grads = [torch.randn(N, H, W, c, generator=g) for c in (3, 3, 2)]
    return (vp, vr, fo, pp), pc, grads


def _torch_camera_grads(cam, pc, volradius, grads, H, W):
    leaves = [t.double().clone().requires_grad_(True) for t in cam]
    rays = rays_torch(*leaves, pc.double() if pc is not None else (W, H), volradius)
    torch.autograd.backward(rays, [g.double() for g in grads])
    return [t.grad.numpy() for t in leaves]


@pytest.mark.parametrize("with_pixelcoords", [False, True])
@pytest.mark.parametrize("N,H,W", [(2, 33, 47), (1, 64, 300)])
def test_emulated_camera_adjoint_vs_torch_autograd(with_pixelcoords, N, H, W):
    from ava256_b200 import scene
    from tests.emul.build import build_aux
    aux = ctypes.CDLL(build_aux())
    aux.mvp_compute_raydirs_backward.restype = ctypes.c_int
    aux.mvp_compute_raydirs_backward.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 5 + [ctypes.c_float] + [ctypes.c_void_p] * 8
    cam, pc, grads = _camera_adjoint_case(N, H, W, with_pixelcoords)
    cam_np = [np.ascontiguousarray(t.numpy()) for t in cam]
    g_np = [np.ascontiguousarray(t.numpy()) for t in grads]
    pc_np = np.ascontiguousarray(pc.numpy()) if pc is not None else None
    out = [np.zeros_like(t) for t in cam_np]
    P = lambda t: ctypes.c_void_p(t.ctypes.data) if t is not None else None  # noqa: E731
    rc = aux.mvp_compute_raydirs_backward(N, H, W, *(P(t) for t in cam_np), P(pc_np), scene.VOLRADIUS, *(P(t) for t in g_np),
                                          *(P(t) for t in out), None)
    assert rc == 0
    ref = _torch_camera_grads(cam, pc, scene.VOLRADIUS, grads, H, W)
    for nm, x, r in zip(("viewpos", "viewrot", "focal", "princpt"), out, ref):
        assert relerr(x, r) <= 1e-4, (nm, relerr(x, r))


def test_emulated_camera_adjoint_rays_parallel_to_a_face():
    """An axis-aligned camera off-axis in x, integer principal point: the rays of its centre column have a direction component of
    exactly +0 and an origin outside the cube's x-slab, so the forward's clip selects tmin = +inf.  Such a ray takes no sample and has
    no tmin gradient; the adjoint must not turn 0 / 0 into a NaN that the block reduction spreads over the whole view."""
    from tests.emul.build import build_aux
    aux = ctypes.CDLL(build_aux())
    aux.mvp_compute_raydirs_backward.restype = ctypes.c_int
    aux.mvp_compute_raydirs_backward.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 5 + [ctypes.c_float] + [ctypes.c_void_p] * 8
    N, H, W, vr = 1, 16, 16, 256.0
    cam = [np.array([[-3.1 * vr, 0.37 * vr, -4.3 * vr]], np.float32), np.eye(3, dtype=np.float32)[None].copy(),
           np.array([[20.0, 20.0]], np.float32), np.array([[8.0, 8.0]], np.float32)]
    g = np.random.default_rng(2)
    grads = [g.standard_normal((N, H, W, c)).astype(np.float32) for c in (3, 3, 2)]
    P = lambda t: ctypes.c_void_p(t.ctypes.data) if t is not None else None  # noqa: E731
    rays = [np.empty((N, H, W, c), np.float32) for c in (3, 3, 2)]
    aux.mvp_compute_raydirs.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 5 + [ctypes.c_float] + [ctypes.c_void_p] * 4
    assert aux.mvp_compute_raydirs(N, H, W, *(P(t) for t in cam), None, vr, *(P(t) for t in rays), None) == 0
    par = rays[1][..., 0] == 0.0
    assert par.any() and np.isinf(rays[2][..., 0][par]).all()
    grads[2][..., 0][par] = 0.0               # what the render backward gives a ray without samples: <d, 0> = 0
    out = [np.zeros_like(t) for t in cam]
    assert aux.mvp_compute_raydirs_backward(N, H, W, *(P(t) for t in cam), None, vr, *(P(t) for t in grads), *(P(t) for t in out), None) == 0
    for t in out:
        assert np.isfinite(t).all()
    # The other rays' gradients are those of the torch formula over the other pixels (as a pixelcoords list; the parallel rays'
    # upstream gradients are zeroed for this comparison).  The centre row
    # (d_y = +0 inside the y-slab) is left out as well: autograd's -1/d_y = inf times the unselected face's zero gradient is a NaN
    # there, where the kernel's adjoint only differentiates the selected face.
    row = rays[1][..., 1] == 0.0
    out = [np.zeros_like(t) for t in cam]
    for t in grads:
        t[row | par] = 0.0
    assert aux.mvp_compute_raydirs_backward(N, H, W, *(P(t) for t in cam), None, vr, *(P(t) for t in grads), *(P(t) for t in out), None) == 0
    py, px = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
    keep = ~(par[0] | row[0])
    pc = torch.from_numpy(np.stack([px[keep], py[keep]], -1)[None, :, None, :].copy())
    gk = [torch.from_numpy(t[0][keep][None, :, None, :].copy()) for t in grads]
    ref = _torch_camera_grads([torch.from_numpy(t) for t in cam], pc, vr, gk, H, W)
    for nm, x, r in zip(("viewpos", "viewrot", "focal", "princpt"), out, ref):
        assert relerr(x, r) <= 1e-4, nm


# ---- C-ABI ----------------------------------------------------------------------------------------------------------------
def test_ray_grad_entry_points_abi():
    """Argument errors come back before any device work (no device here: a launch would fail), RAY_GRADS=1 is listed, and the
    ABI version and struct layouts are those of the plain backward."""
    from ava256_b200 import lib
    L = lib.LIB
    assert "RAY_GRADS=1" in L.mvp_build_config().decode().split()
    lib.require_ray_grads()
    assert L.mvp_abi_version() == 8 == lib.ABI_VERSION
    assert ctypes.sizeof(lib.BackwardArgs) == lib.SIZEOF["BackwardArgs"] == 272
    buf = torch.zeros(64, dtype=torch.float32)
    ok = ctypes.c_void_p(buf.data_ptr())
    odd = ctypes.c_void_p(buf.data_ptr() + 4)
    b = lib.BackwardArgs()
    assert L.mvp_raymarch_backward_rays(None, ok, ok, ok, None) == -1
    assert L.mvp_raymarch_backward_rays(ctypes.byref(b), None, ok, ok, None) == -1
    assert L.mvp_raymarch_backward_rays(ctypes.byref(b), ok, ok, None, None) == -1
    b.struct_size = 8
    assert L.mvp_raymarch_backward_rays(ctypes.byref(b), ok, ok, ok, None) == -7
    # a complete argument set whose only fault is a misaligned ray-gradient buffer
    b = lib.BackwardArgs()
    b.shape = lib.Shape(1, 8, 8, 4, 2, 2, 2)
    b.stepsize, b.fadescale, b.fadeexp = 0.1, 8.0, 8.0
    for f in ("raypos", "raydir", "tminmax", "primpos", "primrot", "primscale", "tplate", "grad_rayrgba", "raysat", "rayaux",
              "grad_primpos", "grad_primrot", "grad_primscale", "grad_tplate"):
        setattr(b, f, ok.value)
    ws = np.zeros(lib.workspace_bytes(1, 8, 8, 4, 2, 2, 2) + 256, np.uint8)
    b.workspace = ws.ctypes.data + (-ws.ctypes.data) % 256
    b.workspace_bytes = ws.size - 256
    assert L.mvp_raymarch_backward_rays(ctypes.byref(b), ok, ok, odd, None) == -6
    assert L.mvp_raymarch_backward_rays(ctypes.byref(b), odd.value + 1, ok, ok, None) == -6
    # the ray generator's adjoint
    args = [1, 8, 8] + [ok] * 4 + [None, 256.0] + [ok] * 3 + [ok] * 4 + [None]
    bad = list(args); bad[9] = None                                           # grad_raypos
    assert L.mvp_compute_raydirs_backward(*bad) == -1
    bad = list(args); bad[13] = None                                          # grad_viewpos
    assert L.mvp_compute_raydirs_backward(*bad) == -1
    bad = list(args); bad[8] = 0.0                                            # volradius
    assert L.mvp_compute_raydirs_backward(*bad) == -8
    bad = list(args); bad[0] = 0
    assert L.mvp_compute_raydirs_backward(*bad) == -2
    bad = list(args); bad[11] = odd                                           # grad_tminmax 8-byte aligned
    assert L.mvp_compute_raydirs_backward(*bad) == -6
    bad = list(args); bad[7] = odd                                            # pixelcoords 8-byte aligned
    assert L.mvp_compute_raydirs_backward(*bad) == -6


def test_camera_grad_off_keeps_the_plain_signature():
    import inspect
    from ava256_b200 import op, raydirs, raymarcher
    assert inspect.signature(op.mvpraymarch_camera).parameters["camera_grad"].default is False
    assert inspect.signature(raymarcher.Raymarcher.forward_camera).parameters["camera_grad"].default is False
    p = inspect.signature(raydirs.compute_raydirs).parameters["differentiable"]
    assert p.default is False and p.kind == inspect.Parameter.KEYWORD_ONLY
