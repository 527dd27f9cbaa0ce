"""The camera form at caller-given sample positions (mvp_raymarch_forward_pixels / mvp_raymarch_backward_pixels) on the CPU emulation
of the product kernels (tests/emul/): the rays are generated in the render kernels from the camera and pixelcoords [N,H,W,2], and
must give the images of mvp_compute_raydirs(pixelcoords) followed by the ray-tensor raymarch bit for bit, and its gradients up to the
order of the fp32 atomics.  The accel build keeps the slab culling for views whose coordinates follow an axis-aligned affine map
(the integer grid, a crop, a stride, pixel centres) and falls back to "every slab is a candidate" for any other field; the per-view
flag the accel build leaves in the workspace (mvp_debug_view_fallback_offset) shows which path each view took."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from tests.helpers import build_case, relerr, scene_args_np

GRAD_TOL = 1e-5                    # fused vs two-call: the same fp32 atomics, added in another order
FWD_TOL, BWD_TOL = 1e-5, 1e-4      # vs the oracle, as in test_emul_kernels.py
PRIM_KEYS = ("primpos", "primrot", "primscale", "template")
KINDS = ("grid", "crop", "stride2", "half", "shuffled")


@pytest.fixture()
def kernels():
    from tests.emul import kernels as k
    k.use_variant(())
    L = k.load()
    L.mvp_raymarch_forward_pixels.restype = ctypes.c_int
    L.mvp_raymarch_forward_pixels.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p]
    L.mvp_raymarch_backward_pixels.restype = ctypes.c_int
    L.mvp_raymarch_backward_pixels.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32] + [ctypes.c_void_p] * 4
    L.mvp_raymarch_backward_rays.restype = ctypes.c_int
    L.mvp_raymarch_backward_rays.argtypes = [ctypes.c_void_p] * 5
    L.mvp_raymarch_forward_sets.restype = ctypes.c_int
    L.mvp_raymarch_forward_sets.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p]
    L.mvp_raymarch_backward_sets.restype = ctypes.c_int
    L.mvp_raymarch_backward_sets.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32] + [ctypes.c_void_p] * 4
    L.mvp_debug_view_fallback_offset.restype = ctypes.c_size_t
    L.mvp_debug_view_fallback_offset.argtypes = [ctypes.c_void_p]
    yield k


def _P(a):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


def pixelcoords(kind, N, H, W, seed=0):
    """[N,H,W,2] float32 sample positions: the integer grid, a crop at an integer offset (another one per view), a stride-2 grid
    around the principal point, half-pixel centres, or the integer grid shuffled within each view (no affine map)."""
    w = np.broadcast_to(np.arange(W, dtype=np.float32)[None, :], (H, W))
    h = np.broadcast_to(np.arange(H, dtype=np.float32)[:, None], (H, W))
    pcs = []
    rng = np.random.default_rng(seed)
    for n in range(N):
        if kind in ("grid", "shuffled"):
            x, y = w, h
        elif kind == "crop":
            x, y = w + (5 + 2 * n), h + (3 - n)
        elif kind == "stride2":
            x, y = 2 * w - W // 2, 2 * h - H // 2
        elif kind == "half":
            x, y = w + 0.5, h + 0.5
        pc = np.stack([x, y], -1).astype(np.float32)
        if kind == "shuffled":
            pc = pc.reshape(-1, 2)[rng.permutation(H * W)].reshape(H, W, 2)
        pcs.append(pc)
    return np.ascontiguousarray(np.stack(pcs))


def two_call_rays(cams, pc, volradius):
    """mvp_compute_raydirs of the library's generator (host build) at the positions pc (None: the integer grid)."""
    from tests.emul.build import build_aux
    aux = ctypes.CDLL(build_aux())
    aux.mvp_compute_raydirs.restype = ctypes.c_int
    aux.mvp_compute_raydirs.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 5 + [ctypes.c_float] + [ctypes.c_void_p] * 4
    N = cams[0].shape[0]
    H, W = pc.shape[1:3]
    rays = [np.empty((N, H, W, c), np.float32) for c in (3, 3, 2)]
    assert aux.mvp_compute_raydirs(N, H, W, *(_P(t) for t in cams), _P(pc), volradius, *(_P(t) for t in rays), None) == 0
    return rays


@contextlib.contextmanager
def calls(kernels, pix=None, view_set=None, nsets=0, ray_shape=None):
    """Makes kernels.forward_backward call the pixels entry points (pix: [N,H,W,2]), or the ray-gradient / sets forms of the ray-tensor
    calls (pix None).  Yields (ray gradients: NaN-filled arrays written by the backward, or [] without ray_shape; the accel build's
    per-view fallback flags, filled in by the forward)."""
    L = kernels.load()
    rays = []
    if ray_shape is not None:
        N, H, W = ray_shape
        rays = [np.full((N, H, W, c), np.nan, np.float32) for c in (3, 3, 2)]
    rp = [_P(r) for r in rays] if rays else [None] * 3
    vs = None if view_set is None else np.ascontiguousarray(view_set, dtype=np.int32)
    flags = []
    fwd, bwd = L.mvp_raymarch_forward, L.mvp_raymarch_backward

    def forward(a, st):
        args = a._obj
        if pix is not None:
            rc = L.mvp_raymarch_forward_pixels(ctypes.addressof(args), _P(pix), _P(vs), nsets, st)
        elif vs is not None:
            rc = L.mvp_raymarch_forward_sets(ctypes.addressof(args), _P(vs), nsets, st)
        else:
            rc = fwd(a, st)
        off = L.mvp_debug_view_fallback_offset(ctypes.addressof(args.shape))
        flags[:] = list((ctypes.c_int32 * args.shape.N).from_address(args.workspace + off))
        return rc

    def backward(b, st):
        if pix is not None:
            return L.mvp_raymarch_backward_pixels(ctypes.addressof(b._obj), _P(pix), _P(vs), nsets, *rp, st)
        if vs is not None:
            return L.mvp_raymarch_backward_sets(ctypes.addressof(b._obj), _P(vs), nsets, *rp, st)
        if rays:
            return L.mvp_raymarch_backward_rays(ctypes.addressof(b._obj), *rp, st)
        return bwd(b, st)

    L.mvp_raymarch_forward, L.mvp_raymarch_backward = forward, backward
    try:
        yield rays, flags
    finally:
        L.mvp_raymarch_forward, L.mvp_raymarch_backward = fwd, bwd


def scene_and_cameras(name="head_small"):
    from ava256_b200 import scene
    s, _ = build_case(name)
    N, H, W = s["raypos"].shape[:3]
    cams = [np.ascontiguousarray(t.numpy()) for t in scene.make_cameras(N, H, W)]
    return s, cams, scene.VOLRADIUS


def run_pair(kernels, s, cams, volradius, pc, grad, prims=None, warp=None, view_set=None, nsets=0, ray_grads=True, **opts):
    """(two-call result, its ray gradients, its fallback flags), (fused result, ray gradients, flags)."""
    N, H, W = pc.shape[:3]
    prims = prims or {k: s[k].numpy() for k in PRIM_KEYS}
    kw = dict(fadescale=s["fadescale"], fadeexp=s["fadeexp"], grad_rayrgba=grad, warp=warp, **opts)
    rays = two_call_rays(cams, pc, volradius)
    shape = (N, H, W) if ray_grads else None
    with calls(kernels, view_set=view_set, nsets=nsets, ray_shape=shape) as (r_ref, f_ref):
        ref = kernels.forward_backward(rays[0], rays[1], s["stepsize"], rays[2], *(prims[k] for k in PRIM_KEYS), **kw)
    with calls(kernels, pix=pc, view_set=view_set, nsets=nsets, ray_shape=shape) as (r_got, f_got):
        got = kernels.forward_backward(None, None, s["stepsize"], None, *(prims[k] for k in PRIM_KEYS),
                                       camera=tuple(cams) + (volradius, H, W), **kw)
    return (ref, r_ref, list(f_ref), rays), (got, r_got, list(f_got))


def check_pair(ref, got, r_ref, r_got, tol=GRAD_TOL):
    assert float(ref[0][..., 3].max()) > 0.05
    assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1])
    for x, y in zip(ref[2], got[2]):
        if not x.any():             # a buffer outside a reduced gradient set: left as zero-filled
            assert not y.any()
            continue
        assert relerr(y, x) <= tol
    assert len(r_ref) == len(r_got)
    if r_ref:
        assert np.abs(r_ref[1]).max() > 0
    for x, y in zip(r_ref, r_got):
        assert relerr(y, x) <= tol


@pytest.mark.parametrize("kind", KINDS)
def test_emulated_pixels_match_two_call_form(kernels, kind):
    """Bit-equal images and raysat, gradients (primitives and rays) within the atomics' order of the two-call form, the oracle's
    images and gradients on the same rays, and the path each view took: the culled one for an affine field, the fallback for the
    shuffled one (where the two-call form's camera fit fails as well)."""
    from oracle import oracle
    s, cams, volradius = scene_and_cameras()
    N, H, W = s["raypos"].shape[:3]
    pc = pixelcoords(kind, N, H, W)
    grad = torch.randn(N, H, W, 4, generator=torch.Generator().manual_seed(4)).numpy()
    (ref, r_ref, f_ref, rays), (got, r_got, f_got) = run_pair(kernels, s, cams, volradius, pc, grad)
    check_pair(ref, got, r_ref, r_got)
    expect = [1] * N if kind == "shuffled" else [0] * N
    assert [int(f != 0) for f in f_got] == expect, f_got
    assert [int(f != 0) for f in f_ref] == expect, f_ref
    a, kw = scene_args_np(s)
    a[0], a[1], a[3] = rays
    out, rsat = oracle.forward(*a, **kw)
    assert relerr(got[0], out) <= FWD_TOL
    gref = oracle.backward(*a, grad, rsat, **kw)
    for nm, g, r in zip(PRIM_KEYS, got[2], gref):
        assert relerr(g, r) <= BWD_TOL, nm
    if kind == "grid":          # the integer grid as a tensor is the tuple form
        kw = dict(fadescale=s["fadescale"], fadeexp=s["fadeexp"], grad_rayrgba=grad)
        tup = kernels.forward_backward(None, None, s["stepsize"], None, *(s[k].numpy() for k in PRIM_KEYS),
                                       camera=tuple(cams) + (volradius, H, W), **kw)
        assert np.array_equal(tup[0], got[0]) and np.array_equal(tup[1], got[1])
        for x, y in zip(tup[2], got[2]):
            assert relerr(y, x) <= GRAD_TOL


@pytest.mark.parametrize("kind", ["crop", "shuffled"])
def test_emulated_pixels_warp_sets_and_reduced_gradients(kernels, kind):
    """algo 1 with a warp field, a view -> set map and the reduced gradient sets, each against its two-call form."""
    from ava256_b200 import lib, scene
    s, _ = build_case("warp_head")
    N, H, W = 3, s["raypos"].shape[1], s["raypos"].shape[2]
    cams = [np.ascontiguousarray(t.numpy()) for t in scene.make_cameras(N, H, W)]
    pc = pixelcoords(kind, N, H, W, seed=3)
    grad = torch.randn(N, H, W, 4, generator=torch.Generator().manual_seed(5)).numpy()
    view_set, nsets = [1, 0, 1], 2
    NS = s["primpos"].shape[0]
    prims = {k: np.ascontiguousarray(s[k].numpy()[[i % NS for i in range(nsets)]]) for k in PRIM_KEYS}
    warp = np.ascontiguousarray(s["warp"].numpy()[[i % NS for i in range(nsets)]])
    (ref, r_ref, _, _), (got, r_got, f_got) = run_pair(kernels, s, cams, scene.VOLRADIUS, pc, grad, prims=prims, warp=warp,
                                                       view_set=view_set, nsets=nsets)
    check_pair(ref, got, r_ref, r_got)
    assert [int(f != 0) for f in f_got] == ([1] * N if kind == "shuffled" else [0] * N)
    for flag in (lib.FLAG_NO_TPLATE_GRAD, lib.FLAG_RAY_GRADS_ONLY):
        (ref, r_ref, _, _), (got, r_got, _) = run_pair(kernels, s, cams, scene.VOLRADIUS, pc, grad, prims=prims, warp=warp,
                                                       view_set=view_set, nsets=nsets, fwd_flags=flag, bwd_flags=flag)
        check_pair(ref, got, r_ref, r_got)


def test_emulated_pixels_rebuilt_lists_and_planes(kernels):
    """MVP_FLAG_TEST_TINY_LISTS (the backward rebuilds almost every tile's list from the sample positions) and the image planes."""
    from ava256_b200 import lib
    s, cams, volradius = scene_and_cameras()
    N, H, W = s["raypos"].shape[:3]
    pc = pixelcoords("stride2", N, H, W)
    grad = torch.randn(N, H, W, 4, generator=torch.Generator().manual_seed(6)).numpy()
    for opts in (dict(fwd_flags=lib.FLAG_TEST_TINY_LISTS), dict(planes=True)):
        (ref, r_ref, _, _), (got, r_got, _) = run_pair(kernels, s, cams, volradius, pc, grad, **opts)
        check_pair(ref, got, r_ref, r_got)


def test_pixels_argument_errors_and_build_config():
    """The pixels entry points' argument errors come back before any device work (dummy pointers are never dereferenced), and the
    library reports the feature."""
    from ava256_b200 import lib
    assert "CAMERA_PIXELS=1" in lib.LIB.mvp_build_config().decode().split()
    lib.require_camera_pixels()
    dummy = ctypes.c_void_p(256)
    a = lib.ForwardArgs()
    a.shape = lib.Shape(4, 8, 8, 4, 2, 2, 2)
    a.stepsize = 0.1
    for f in ("primpos", "primrot", "primscale", "tplate", "rayrgba", "workspace"):
        setattr(a, f, dummy)
    a.workspace_bytes = 1 << 30
    b = lib.BackwardArgs()
    b.shape = a.shape
    b.stepsize = 0.1
    for f in ("primpos", "primrot", "primscale", "tplate", "grad_rayrgba", "raysat", "rayaux", "grad_primpos", "grad_primrot",
              "grad_primscale", "grad_tplate", "workspace"):
        setattr(b, f, dummy)
    b.workspace_bytes = 1 << 30
    F, B = lib.LIB.mvp_raymarch_forward_pixels, lib.LIB.mvp_raymarch_backward_pixels
    none3 = (None, None, None)
    assert F(ctypes.byref(a), dummy, None, 0, None) == -1                   # MVP_ERR_NULL: no camera to generate rays from
    assert B(ctypes.byref(b), dummy, None, 0, *none3, None) == -1
    a.camera = b.camera = lib.Camera(dummy, dummy, dummy, dummy, 1.0, 0)
    assert F(ctypes.byref(a), None, None, 0, None) == -1                    # MVP_ERR_NULL: no pixelcoords
    assert B(ctypes.byref(b), None, None, 0, *none3, None) == -1
    assert F(ctypes.byref(a), ctypes.c_void_p(260), None, 0, None) == -6    # MVP_ERR_ALIGN: pixelcoords is read as float2
    assert B(ctypes.byref(b), ctypes.c_void_p(260), None, 0, *none3, None) == -6
    assert B(ctypes.byref(b), dummy, None, 0, dummy, None, None, None) == -1  # some ray-gradient pointers, not all three
    for nsets in (0, 5):                                                    # MVP_ERR_SHAPE: a map with nsets outside [1, N]
        assert F(ctypes.byref(a), dummy, dummy, nsets, None) == -2
        assert B(ctypes.byref(b), dummy, dummy, nsets, *none3, None) == -2
    a.struct_size -= 8
    assert F(ctypes.byref(a), dummy, None, 0, None) == -7
    assert F(None, dummy, None, 0, None) == -1 and B(None, dummy, None, 0, *none3, None) == -1
    a.struct_size = ctypes.sizeof(lib.ForwardArgs)
    a.workspace_bytes = b.workspace_bytes = 16                              # past the pixels checks: the workspace is too small
    assert F(ctypes.byref(a), dummy, None, 0, None) == -4
    assert B(ctypes.byref(b), dummy, None, 0, *none3, None) == -4


@pytest.mark.parametrize("kind", ["crop", "shuffled"])
def test_emulated_pixels_forward_then_ray_tensor_backward(kernels, kind):
    """The op's camera-gradient backward after a pixels forward: mvp_raymarch_backward_rays on the forward's workspace
    (MVP_FLAG_ACCEL_VALID) with the rays mvp_compute_raydirs makes from the same pixelcoords and no camera.  Its primitive and ray
    gradients equal those of the pixels backward within the atomics' order."""
    from ava256_b200 import lib
    s, cams, volradius = scene_and_cameras()
    N, H, W = s["raypos"].shape[:3]
    pc = pixelcoords(kind, N, H, W, seed=5)
    grad = torch.randn(N, H, W, 4, generator=torch.Generator().manual_seed(7)).numpy()
    rays = two_call_rays(cams, pc, volradius)
    kw = dict(fadescale=s["fadescale"], fadeexp=s["fadeexp"], grad_rayrgba=grad, camera=tuple(cams) + (volradius, H, W))
    prims = [s[k].numpy() for k in PRIM_KEYS]
    with calls(kernels, pix=pc, ray_shape=(N, H, W)) as (r_pix, _):
        ref = kernels.forward_backward(None, None, s["stepsize"], None, *prims, **kw)
    L = kernels.load()
    r_got = [np.full((N, H, W, c), np.nan, np.float32) for c in (3, 3, 2)]

    def backward(b, st):
        args = b._obj
        args.raypos, args.raydir, args.tminmax = (_P(r) for r in rays)
        args.camera = lib.Camera()
        assert args.flags & lib.FLAG_ACCEL_VALID
        return L.mvp_raymarch_backward_rays(ctypes.addressof(args), *(_P(r) for r in r_got), st)

    with calls(kernels, pix=pc):
        plain = L.mvp_raymarch_backward
        L.mvp_raymarch_backward = backward
        try:
            got = kernels.forward_backward(None, None, s["stepsize"], None, *prims, **kw)
        finally:
            L.mvp_raymarch_backward = plain
    check_pair(ref, got, r_pix, r_got)
