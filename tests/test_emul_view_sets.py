"""Per-view primitive sets (mvp_raymarch_forward_sets / mvp_raymarch_backward_sets) on the CPU emulation of the product kernels
(tests/emul/): S sets of primitives rendered over N views in one launch, view n from set view_set[n], against the per-view form
built by repeating each set to its views -- bit-equal images and raysat, each set's gradient the sum of its views' -- and the
argument checks of the two entry points."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from tests.helpers import build_case, build_dense_case, relerr

SET_TOL = 1e-5          # a set's gradient vs the sum of its views' (the same fp32 atomics, added in another order)
PRIM_KEYS = ("primpos", "primrot", "primscale", "template")


@pytest.fixture()
def kernels():
    from tests.emul import kernels as k
    k.use_variant(())
    k.load()
    yield k
    k.set_lane_order("forward")
    k.use_variant(())


@contextlib.contextmanager
def view_sets(kernels, view_set, nsets, ray_shape=None):
    """Makes kernels.forward_backward call the sets entry points with the map `view_set` (host int32 [N]); with ray_shape = (N, H, W)
    the backward computes ray gradients into the NaN-filled arrays it yields, else the yielded list is empty."""
    L = kernels.load()
    L.mvp_raymarch_forward_sets.restype = ctypes.c_int
    L.mvp_raymarch_forward_sets.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p]
    L.mvp_raymarch_backward_sets.restype = ctypes.c_int
    L.mvp_raymarch_backward_sets.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32] + [ctypes.c_void_p] * 4
    vs = np.ascontiguousarray(view_set, dtype=np.int32)
    P = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    rays = []
    if ray_shape is not None:
        N, H, W = ray_shape
        rays = [np.full((N, H, W, 3), np.nan, np.float32), np.full((N, H, W, 3), np.nan, np.float32),
                np.full((N, H, W, 2), np.nan, np.float32)]
    rp = [P(r) for r in rays] if rays else [None] * 3
    fwd, bwd = L.mvp_raymarch_forward, L.mvp_raymarch_backward
    L.mvp_raymarch_forward = lambda a, st: L.mvp_raymarch_forward_sets(ctypes.addressof(a._obj), P(vs), nsets, st)
    L.mvp_raymarch_backward = lambda b, st: L.mvp_raymarch_backward_sets(ctypes.addressof(b._obj), P(vs), nsets, *rp, st)
    try:
        yield rays
    finally:
        L.mvp_raymarch_forward, L.mvp_raymarch_backward = fwd, bwd


@contextlib.contextmanager
def ray_backward(kernels, N, H, W):
    """kernels.forward_backward with mvp_raymarch_backward_rays (the per-view reference of the ray gradients)."""
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


def scene_sets(s, view_set, nsets, seed=11):
    """nsets distinct primitive sets from scene s (its views' primitives, cycled, each moved a little so that no two sets are equal),
    the per-view copies the map makes of them, and the rays of len(view_set) views.  Returns (rays, sets, per_view, warp_sets,
    warp_per_view) as numpy arrays (warp entries None without a warp field)."""
    from ava256_b200 import scene
    N = len(view_set)
    H, W = s["raypos"].shape[1:3]
    rp, rd, tmm = scene.make_rays(N, H, W, view_offset=1)
    g = torch.Generator().manual_seed(seed)
    NS = s["primpos"].shape[0]
    sets = {k: s[k][[i % NS for i in range(nsets)]].clone() for k in PRIM_KEYS}
    sets["primpos"] += 0.02 * torch.randn(sets["primpos"].shape, generator=g)
    sets["template"] *= 0.75 + 0.5 * torch.rand(sets["template"].shape[:2] + (1, 1, 1, 1), generator=g)
    sets = {k: np.ascontiguousarray(v.numpy()) for k, v in sets.items()}
    idx = np.asarray(view_set)
    per_view = {k: np.ascontiguousarray(v[idx]) for k, v in sets.items()}
    wsets = wview = None
    if "warp" in s:
        wsets = np.ascontiguousarray(s["warp"][[i % NS for i in range(nsets)]].numpy())
        wview = np.ascontiguousarray(wsets[idx])
    return (rp.numpy(), rd.numpy(), tmm.numpy()), sets, per_view, wsets, wview


def morton_orders(primpos):
    from ava256_b200.op import morton_order
    return morton_order(torch.from_numpy(primpos)).to(torch.int32).numpy()


def run(kernels, rays, prims, warp, s, grad, **opts):
    kw = dict(fadescale=s["fadescale"], fadeexp=s["fadeexp"])
    return kernels.forward_backward(*rays[:2], s["stepsize"], rays[2], prims["primpos"], prims["primrot"], prims["primscale"],
                                    prims["template"], grad_rayrgba=grad, warp=warp, **kw, **opts)


def check_against_per_view(view_set, nsets, ref, got, tol=SET_TOL):
    """Images and raysat bit-equal; every set's gradient the sum of its views' gradients; an unreferenced set's exactly zero."""
    (out_v, sat_v, g_v), (out_s, sat_s, g_s) = ref, got
    assert float(out_v[..., 3].max()) > 0.05
    assert np.array_equal(out_v, out_s)
    if sat_v is not None:
        assert np.array_equal(sat_v, sat_s)
    if g_v is None:
        return
    idx = np.asarray(view_set)
    for i, (x, y) in enumerate(zip(g_v, g_s)):
        if x is None:
            assert y is None
            continue
        assert y.shape[0] == nsets, (i, y.shape)
        for j in range(nsets):
            if (idx == j).any():
                e = relerr(y[j], x[idx == j].sum(axis=0))
                assert e <= tol, (i, j, e)
            else:
                assert not y[j].any(), (i, j)


MAPS = [([2, 0, 1, 0, 2], 3), ([1, 1, 0, 1], 2), ([0, 2, 2], 3)]     # the last: no view shows set 1


@pytest.mark.parametrize("order", ["fixed", "morton"])
@pytest.mark.parametrize("view_set,nsets", MAPS)
@pytest.mark.parametrize("name", ["head_small", "warp_head"])
def test_emulated_view_sets_match_per_view_copies(kernels, name, view_set, nsets, order):
    s, _ = build_case(name)
    rays, sets, per_view, wsets, wview = scene_sets(s, view_set, nsets)
    N, H, W = rays[0].shape[:3]
    grad = torch.randn(N, H, W, 4, generator=torch.Generator().manual_seed(3)).numpy()
    ord_s = ord_v = None
    if order == "morton":
        ord_s = morton_orders(sets["primpos"])
        ord_v = np.ascontiguousarray(ord_s[np.asarray(view_set)])
    ref = run(kernels, rays, per_view, wview, s, grad, order=ord_v)
    with view_sets(kernels, view_set, nsets):
        got = run(kernels, rays, sets, wsets, s, grad, order=ord_s)
    check_against_per_view(view_set, nsets, ref, got)
    # gradient buffers cleared by the forward's render kernel (sized nsets * K), and by MVP_FLAG_ZERO_GRADS in the backward
    from ava256_b200 import lib
    with view_sets(kernels, view_set, nsets):
        got = run(kernels, rays, sets, wsets, s, grad, order=ord_s, clear_in_forward=True)
    check_against_per_view(view_set, nsets, ref, got)
    with view_sets(kernels, view_set, nsets):
        got = run(kernels, rays, sets, wsets, s, grad, order=ord_s, bwd_flags=lib.FLAG_ZERO_GRADS)
    check_against_per_view(view_set, nsets, ref, got)


@pytest.mark.parametrize("name", ["head_small", "warp_head"])
def test_emulated_one_set_equals_shared_and_identity_equals_plain(kernels, name):
    from ava256_b200 import lib
    s, _ = build_case(name)
    N = 3
    rays, sets, per_view, wsets, wview = scene_sets(s, [0] * N, 1)
    grad = torch.randn(N, *rays[0].shape[1:3], 4, generator=torch.Generator().manual_seed(5)).numpy()
    ref = run(kernels, rays, sets, wsets, s, grad, fwd_flags=lib.FLAG_SHARED_PRIMS, bwd_flags=lib.FLAG_SHARED_PRIMS)
    with view_sets(kernels, [0] * N, 1):
        got = run(kernels, rays, sets, wsets, s, grad)
    assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1])
    for x, y in zip(ref[2], got[2]):
        assert relerr(y, x) <= SET_TOL
    rays, sets, per_view, wsets, wview = scene_sets(s, list(range(N)), N)
    ref = run(kernels, rays, sets, wsets, s, grad)
    with view_sets(kernels, list(range(N)), N):
        got = run(kernels, rays, sets, wsets, s, grad)
    assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1])
    for x, y in zip(ref[2], got[2]):
        assert relerr(y, x) <= SET_TOL


@pytest.mark.parametrize("cap", ["uncapped", "capped"])
@pytest.mark.parametrize("name", ["t8", "warp"])
def test_emulated_view_sets_heavy_kernels(kernels, name, cap):
    """Dense scenes: every tile's list outgrows the fast kernels, so the 512-entry kernels render and differentiate the sets."""
    s, _ = build_dense_case(name, cap)
    view_set, nsets = [1, 0, 1], 2
    rays, sets, per_view, wsets, wview = scene_sets(s, view_set, nsets)
    # the dense scene's own rays (its tmax spread makes a part of the rays saturate)
    rays = tuple(np.ascontiguousarray(np.concatenate([s[k].numpy()] * 2)[:3]) for k in ("raypos", "raydir", "tminmax"))
    grad = torch.randn(3, *rays[0].shape[1:3], 4, generator=torch.Generator().manual_seed(6)).numpy()
    ref = run(kernels, rays, per_view, wview, s, grad)
    heavy_ref = kernels.last_heavy_tiles
    with view_sets(kernels, view_set, nsets):
        got = run(kernels, rays, sets, wsets, s, grad)
    assert kernels.last_heavy_tiles == heavy_ref and heavy_ref[0] > 0 and heavy_ref[1] > 0
    check_against_per_view(view_set, nsets, ref, got)


def test_emulated_view_sets_rebuilt_lists_planes(kernels):
    """MVP_FLAG_TEST_TINY_LISTS (almost every tile's list rebuilt by the backward) and the image-plane outputs / gradient."""
    from ava256_b200 import lib
    s, _ = build_case("head_small")
    view_set, nsets = [1, 0, 1, 1], 2
    rays, sets, per_view, wsets, wview = scene_sets(s, view_set, nsets)
    grad = torch.randn(4, *rays[0].shape[1:3], 4, generator=torch.Generator().manual_seed(7)).numpy()
    ref = run(kernels, rays, per_view, wview, s, grad)
    for opts in (dict(fwd_flags=lib.FLAG_TEST_TINY_LISTS), dict(planes=True)):
        with view_sets(kernels, view_set, nsets):
            got = run(kernels, rays, sets, wsets, s, grad, **opts)
        check_against_per_view(view_set, nsets, ref, got)


@pytest.mark.parametrize("name", ["head_small", "warp_head"])
def test_emulated_view_sets_ray_grads_and_reduced_sets(kernels, name):
    """Ray gradients of the sets backward equal those of the per-view backward_rays, in the full, NO_TPLATE_GRAD and
    RAY_GRADS_ONLY gradient sets; the reduced sets leave the buffers they do not request untouched and match the full one."""
    from ava256_b200 import lib
    s, _ = build_case(name)
    view_set, nsets = [2, 0, 1, 0, 2], 3
    rays, sets, per_view, wsets, wview = scene_sets(s, view_set, nsets)
    N, H, W = rays[0].shape[:3]
    grad = torch.randn(N, H, W, 4, generator=torch.Generator().manual_seed(8)).numpy()
    with ray_backward(kernels, N, H, W) as rays_ref:
        ref = run(kernels, rays, per_view, wview, s, grad)
    with view_sets(kernels, view_set, nsets, (N, H, W)) as rays_got:
        got = run(kernels, rays, sets, wsets, s, grad)
    check_against_per_view(view_set, nsets, ref, got)
    assert np.abs(rays_ref[0]).max() > 0
    for x, y in zip(rays_ref, rays_got):
        assert relerr(y, x) <= SET_TOL
    full = got[2]
    for flag in (lib.FLAG_NO_TPLATE_GRAD, lib.FLAG_RAY_GRADS_ONLY):
        with view_sets(kernels, view_set, nsets, (N, H, W)) as rays_sel:
            out, _, g = run(kernels, rays, sets, wsets, s, grad, fwd_flags=flag, bwd_flags=flag)
        assert np.array_equal(out, ref[0])
        for x, y in zip(rays_ref, rays_sel):
            assert relerr(y, x) <= SET_TOL
        computed = 3 if flag == lib.FLAG_NO_TPLATE_GRAD else 0
        for i, (x, y) in enumerate(zip(full, g)):
            if i < computed:
                assert relerr(y, x) <= SET_TOL, i
            else:
                assert not y.any(), i          # not requested: the zero-filled buffer is neither read nor written


def test_emulated_view_sets_camera_rays(kernels):
    """The camera form (rays generated in the kernels) with a sets map, ray gradients included, equals the ray-tensor form."""
    from ava256_b200 import scene
    s, _ = build_case("head_small")
    view_set, nsets = [1, 0, 1], 2
    rays, sets, per_view, wsets, wview = scene_sets(s, view_set, nsets)
    N, (H, W) = 3, rays[0].shape[1:3]
    cams = [np.ascontiguousarray(t.numpy()) for t in scene.make_cameras(N, H, W)]
    from tests.emul.build import build_aux
    aux = ctypes.CDLL(build_aux())
    aux.mvp_compute_raydirs.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 5 + [ctypes.c_float] + [ctypes.c_void_p] * 4
    gen = [np.empty((N, H, W, c), np.float32) for c in (3, 3, 2)]
    P = lambda t: ctypes.c_void_p(t.ctypes.data) if t is not None else None  # noqa: E731
    assert aux.mvp_compute_raydirs(N, H, W, *(P(t) for t in cams), None, scene.VOLRADIUS, *(P(t) for t in gen), None) == 0
    grad = torch.randn(N, H, W, 4, generator=torch.Generator().manual_seed(9)).numpy()
    with view_sets(kernels, view_set, nsets, (N, H, W)) as r0:
        ref = run(kernels, gen, sets, None, s, grad)
    camera = tuple(cams) + (scene.VOLRADIUS, H, W)
    kw = dict(fadescale=s["fadescale"], fadeexp=s["fadeexp"])
    with view_sets(kernels, view_set, nsets, (N, H, W)) as r1:
        got = kernels.forward_backward(None, None, s["stepsize"], None, *(sets[k] for k in PRIM_KEYS), grad_rayrgba=grad,
                                       camera=camera, **kw)
    assert float(ref[0][..., 3].max()) > 0.05
    assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1])
    for x, y in zip(ref[2], got[2]):
        assert relerr(y, x) <= SET_TOL
    for x, y in zip(r0, r1):
        assert relerr(y, x) <= SET_TOL


@pytest.mark.parametrize("bad", [-1, "nsets", 2 ** 31 - 1, -2 ** 31])
def test_emulated_out_of_range_entries_render_empty(kernels, bad):
    """A map entry outside [0, nsets) (the map is input from outside the program): its view renders empty, takes no gradient and
    gets zero ray gradients; the other views are those of the valid map, and nothing outside the buffers is touched (the emulation
    runs on host arrays: an out-of-bounds access would read other host memory, which the bit-equality below would show)."""
    s, _ = build_case("head_small")
    nsets = 2
    bad = nsets if bad == "nsets" else bad
    good_map, view_set = [1, 0, 1, 0], [1, bad, 1, 0]
    rays, sets, _, _, _ = scene_sets(s, good_map, nsets)
    N, H, W = rays[0].shape[:3]
    grad = torch.randn(N, H, W, 4, generator=torch.Generator().manual_seed(10)).numpy()
    with view_sets(kernels, good_map, nsets, (N, H, W)) as r_good:
        good = run(kernels, rays, sets, None, s, grad)
    with view_sets(kernels, view_set, nsets, (N, H, W)) as r_bad:
        out, sat, g = run(kernels, rays, sets, None, s, grad)
    assert float(good[0][1][..., 3].max()) > 0.05            # the view that goes empty did show something
    assert not out[1].any()
    assert (sat[1] == -1.0).all()
    for r in r_bad:
        assert not r[1].any()
    keep = [0, 2, 3]
    assert np.array_equal(out[keep], good[0][keep]) and np.array_equal(sat[keep], good[1][keep])
    for x, y in zip(r_good, r_bad):
        assert relerr(y[keep], x[keep]) <= SET_TOL
    # the gradients: those of the valid map without view 1's contribution (the per-view form with view 1's gradient zeroed)
    g0 = grad.copy()
    g0[1] = 0.0
    with view_sets(kernels, good_map, nsets):
        ref = run(kernels, rays, sets, None, s, g0)
    for x, y in zip(ref[2], g):
        assert relerr(y, x) <= SET_TOL


def test_view_sets_argument_errors_and_build_config():
    """The sets entry points' argument errors come back before any device work (dummy pointers are never dereferenced), and the
    library reports the feature."""
    from ava256_b200 import lib
    assert "VIEW_SETS=1" in lib.LIB.mvp_build_config().decode().split()
    lib.require_view_sets()
    dummy = ctypes.c_void_p(256)
    a = lib.ForwardArgs()
    a.shape = lib.Shape(4, 8, 8, 4, 2, 2, 2)
    a.stepsize = 0.1
    for f in ("raypos", "raydir", "tminmax", "primpos", "primrot", "primscale", "tplate", "rayrgba", "workspace"):
        setattr(a, f, dummy)
    a.workspace_bytes = 1 << 30
    b = lib.BackwardArgs()
    b.shape = a.shape
    b.stepsize = 0.1
    for f in ("raypos", "raydir", "tminmax", "primpos", "primrot", "primscale", "tplate", "grad_rayrgba", "raysat", "rayaux",
              "grad_primpos", "grad_primrot", "grad_primscale", "grad_tplate", "workspace"):
        setattr(b, f, dummy)
    b.workspace_bytes = 1 << 30
    F, B = lib.LIB.mvp_raymarch_forward_sets, lib.LIB.mvp_raymarch_backward_sets
    none3 = (None, None, None)
    assert F(ctypes.byref(a), None, 2, None) == -1                       # MVP_ERR_NULL: no map
    assert B(ctypes.byref(b), None, 2, *none3, None) == -1
    for nsets in (0, -1, 5):                                              # MVP_ERR_SHAPE: nsets outside [1, N]
        assert F(ctypes.byref(a), dummy, nsets, None) == -2
        assert B(ctypes.byref(b), dummy, nsets, *none3, None) == -2
    a.flags = b.flags = lib.FLAG_SHARED_PRIMS                             # MVP_ERR_SHAPE: a map and the one-set flag
    assert F(ctypes.byref(a), dummy, 1, None) == -2
    assert B(ctypes.byref(b), dummy, 1, *none3, None) == -2
    a.flags = b.flags = 0
    assert B(ctypes.byref(b), dummy, 2, dummy, None, None, None) == -1    # some ray-gradient pointers, not all three
    assert B(ctypes.byref(b), dummy, 2, None, dummy, dummy, None) == -1
    assert F(ctypes.byref(a), ctypes.c_void_p(258), 2, None) == -6       # MVP_ERR_ALIGN: the map is read as int32
    a.struct_size -= 8
    assert F(ctypes.byref(a), dummy, 2, None) == -7
    assert F(None, dummy, 2, None) == -1 and B(None, dummy, 2, *none3, None) == -1
    # past the map checks, the common ones: the workspace is too small
    a.struct_size = ctypes.sizeof(lib.ForwardArgs)
    a.workspace_bytes = b.workspace_bytes = 16
    assert F(ctypes.byref(a), dummy, 2, None) == -4
    assert B(ctypes.byref(b), dummy, 2, *none3, None) == -4


def test_op_view_set_host_validation():
    """mvpraymarch_sets checks a host map (and the primitive batch) before anything runs; these raise on a machine without a GPU
    as well, ahead of the op's CUDA-tensor checks."""
    from ava256_b200.op import _view_set_tensor
    dev = torch.device("cpu")
    assert _view_set_tensor([1, 0, 1], 3, 2, dev).tolist() == [1, 0, 1]
    assert _view_set_tensor(torch.tensor([0, 0], dtype=torch.int64), 2, 1, dev).dtype == torch.int32
    for vs, N, S, err in (([0, 2, 1], 3, 2, ValueError), ([-1, 0], 2, 1, ValueError), ([0, 1], 3, 2, ValueError),
                          ([0, 1, 1], 3, 4, ValueError), ([0, 0], 2, 0, ValueError), (torch.zeros(2, 1, dtype=torch.int32), 2, 1, ValueError),
                          (torch.zeros(2), 2, 1, TypeError), ([0.5, 1], 2, 2, TypeError), (7, 2, 1, TypeError), ([True, 0], 2, 2, TypeError)):
        with pytest.raises(err):
            _view_set_tensor(vs, N, S, dev)
