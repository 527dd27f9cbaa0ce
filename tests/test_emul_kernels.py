"""The PRODUCT kernels' source (ava-256_b200/csrc/mvp_kernels.cu) compiled for the host on a CPU emulation of warps,
blocks and shared memory (tests/emul/), run against the oracle and the reference's golden vectors WITHOUT a GPU.

This is test infrastructure: it checks the kernels' logic (accel build, tile lists, interval marching, sample compaction,
slab-major adjoint, the 256/512-entry variants, algo 1) in a container that has no GPU; floating point is IEEE on the
CPU (no MUFU approximations), so agreement is to rounding.  The GPU tests (`-m gpu`) remain the parity gate."""
import os

import numpy as np
import pytest

import torch

from tests.helpers import CASES, DENSE_CASES, DENSE_K3, EDGE_KINDS, build_case, build_dense_case, dense_scene, edge_scene, relerr, scene_args_np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FWD_TOL, BWD_TOL = 1e-5, 1e-4        # vs the oracle (same IEEE arithmetic; gradients differ by summation order)


@pytest.fixture()
def kernels():
    from tests.emul import kernels as k
    k.use_variant(())
    k.load()
    yield k
    k.set_lane_order("forward")
    k.use_variant(())


@pytest.mark.parametrize("name", list(CASES))
def test_emulated_kernels_vs_oracle(kernels, name):
    from oracle import oracle
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    kernels.set_lane_order("forward")
    out, raysat, grads = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    ref, rsat = oracle.forward(*a, **kw)
    assert relerr(out, ref) <= FWD_TOL
    assert np.array_equal(raysat[..., 0] > -1.0, rsat[..., 0] > -1.0)            # same rays saturate
    gref = oracle.backward(*a, grad.numpy(), rsat, **kw)
    assert len(grads) == len(gref)
    for nm, g, r in zip(("primpos", "primrot", "primscale", "template", "warp"), grads, gref):
        assert relerr(g, r) <= BWD_TOL, nm
    # inference path (no raysat / rayaux): same image
    out2, _, _ = kernels.forward_backward(*a, **kw)
    assert np.array_equal(out2, out)


@pytest.mark.parametrize("name", ["head_small", "many_overlaps", "warp_small", "gradcheck_ragged"])
def test_emulated_kernels_vs_reference_golden(kernels, name):
    """Vectors produced by the unmodified reference CUDA extension on a GPU (tests/golden/make_golden.py)."""
    gold = np.load(os.path.join(GOLDEN, name + ".npz"))
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    out, _, grads = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    assert relerr(out, gold["rayrgba"]) <= 1e-4
    for nm, g in zip(("primpos", "primrot", "primscale", "template", "warp"), grads):
        assert relerr(g, gold["grad_" + nm]) <= 1e-3, nm


@pytest.mark.parametrize("order", ["reverse", "random"])
@pytest.mark.parametrize("name", ["head_small", "many_overlaps", "warp_small", "tiny"])
def test_result_does_not_depend_on_lane_schedule(kernels, name, order):
    """Lanes of a warp have no defined order between collectives; a kernel that relies on one (missing __syncwarp
    between a shared-memory write and another lane's read) gives different images under different schedules."""
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    kernels.set_lane_order("forward")
    out0, sat0, g0 = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    kernels.set_lane_order(order)
    out1, sat1, g1 = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    kernels.set_lane_order("forward")
    assert np.array_equal(out0, out1) and np.array_equal(sat0, sat1)        # forward has no atomics: bit-identical
    for x, y in zip(g0, g1):
        assert relerr(x, y) <= 1e-5                                         # atomics: summation order only


def test_emulated_argument_validation_matches_product(kernels):
    import ctypes
    from ava256_b200 import lib
    L = kernels.load()
    a = lib.ForwardArgs()
    a.shape = lib.Shape(1, 8, 8, 4, 2, 2, 2)
    a.stepsize = 0.1
    assert L.mvp_raymarch_forward(ctypes.byref(a), None) == lib.LIB.mvp_raymarch_forward(ctypes.byref(a), None) == -1
    s = lib.Shape(2, 64, 42, 64, 8, 8, 8)
    assert L.mvp_workspace_bytes(ctypes.byref(s)) == lib.LIB.mvp_workspace_bytes(ctypes.byref(s)) > 0


@pytest.mark.parametrize("variant", [(), ("MVP_LIST_MARGIN=1", "MVP_LIST_REUSE=1"), ("MVP_LIST_MARGIN=0", "MVP_LIST_REUSE=0")])
@pytest.mark.parametrize("kind", EDGE_KINDS)
def test_emulated_edge_cases_vs_oracle(kernels, kind, variant):
    """Degenerate inputs the reference tolerates (zero scale = infinite slab, rays missing the volume, one-step and
    many-step marches), for the default build and the list variants either way round."""
    from oracle import oracle
    s = edge_scene(kind)
    grad = torch.randn(*s["raypos"].shape[:3], 4, generator=torch.Generator().manual_seed(17))
    a, kw = scene_args_np(s)
    kernels.use_variant(variant, opt="-O0" if variant else "-O1")
    out, _, grads = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    ref, raysat = oracle.forward(*a, **kw)
    assert np.isfinite(out).all() and relerr(out, ref) <= FWD_TOL
    gref = oracle.backward(*a, grad.numpy(), raysat, **kw)
    for nm, g, r in zip(("primpos", "primrot", "primscale", "template"), grads, gref):
        assert np.isfinite(g).all(), nm
        assert relerr(g, r) <= BWD_TOL, nm


# build-time variants of the kernels (former defaults, and candidates waiting for a GPU measurement): same results required
VARIANTS = {
    "list_rebuild": ("MVP_LIST_REUSE=0",),                                 # backward rebuilds the lists (the former default)
    "list_reuse": ("MVP_LIST_REUSE=1",),                                   # backward loads the lists the forward saved (default)
    "list_reuse_overflow": ("MVP_LIST_REUSE=1", "MVP_LIST_CAP_PER_TILE=1", "MVP_LIST_CAP_MIN=16"),  # most tiles do not fit: mixes both paths
    "xbuckets": ("MVP_XBUCKETS=1",),                                        # second bucketing level in x
    "xbuckets_all": ("MVP_XBUCKETS=1", "MVP_LIST_MARGIN=1"),
    "list_margin": ("MVP_LIST_MARGIN=1",),                                  # step intervals from the fp-drift bound
    "list_margin_reuse": ("MVP_LIST_MARGIN=1", "MVP_LIST_REUSE=1"),
    "no_xbuckets_no_margin": ("MVP_XBUCKETS=0", "MVP_LIST_MARGIN=0"),      # the round-1 defaults
    "fastcap_small": ("MVP_FASTCAP=8",),                                   # most tiles overflow the fast list -> handed to the 512-entry kernel
    "bwd_regrecord": ("MVP_BWD_SMEMREC=0",),
    "grid_order": ("MVP_CTA_ORDER=0",),                                    # plain grid order instead of the cost-sorted CTA order
    "queue_compaction": ("MVP_FWD_RING=0",),                                # forward sample queue compacted to the front after every flush (the former form)
    "separate_stage": ("MVP_SMEM_UNION=0",),                               # bucket staging buffer not overlaid on the sample queue (the former layout)
    "split_fastcaps": ("MVP_FWD_FASTCAP=16", "MVP_BWD_FASTCAP=8"),         # backward's fast list shorter than the forward's: saved lists that only fit the forward's
    "bwd_lanesmem": ("MVP_BWD_LANESMEM=1",),                               # per-lane between-batch state in shared memory                               # slab record in registers across the adjoint (round-1 form)
}


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name", ["head_small", "many_overlaps", "warp_small", "gradcheck_ragged", "noncubic", "tiny"])
def test_kernel_variants_match_the_default_build(kernels, name, variant):
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    out0, sat0, g0 = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    kernels.use_variant(VARIANTS[variant], opt="-O0")
    for order in ("forward", "random"):
        kernels.set_lane_order(order)
        out1, sat1, g1 = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
        assert np.array_equal(out0, out1) and np.array_equal(sat0, sat1)
        for x, y in zip(g0, g1):
            assert relerr(x, y) <= 1e-5
    if variant in ("list_reuse", "list_reuse_overflow"):
        import ctypes
        loaded, rebuilt = ctypes.c_int(), ctypes.c_int()
        kernels.load().mvp_emul_saved_list_tiles(ctypes.byref(loaded), ctypes.byref(rebuilt))
        if variant == "list_reuse":
            assert loaded.value > 0 and rebuilt.value == 0                # every tile's saved list was loaded
        else:
            assert loaded.value + rebuilt.value > 0
            if name == "head_small":
                assert loaded.value > 0 and rebuilt.value > 0             # tiny workspace: both paths in one launch


@pytest.mark.parametrize("name", ["head_small", "gradcheck_ragged", "warp_small"])
def test_emulated_image_plane_outputs(kernels, name):
    """rayrgb [N,3,H,W] / rayalpha [N,1,H,W] written by the forward's epilogue and the gradient read as planes by the backward's
    prologue (C-ABI 6) == the channels-last run, bit for bit in the forward."""
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    out0, sat0, g0 = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    out1, sat1, g1 = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), planes=True, **kw)
    assert np.array_equal(out0, out1) and np.array_equal(sat0, sat1)
    for x, y in zip(g0, g1):
        assert relerr(x, y) <= 1e-5


@pytest.mark.parametrize("seed", list(range(10)))
def test_emulated_random_small_scenes_vs_oracle(kernels, seed):
    """The seeded random shapes of tests/test_gpu_parity.py::test_random_small_scenes_vs_oracle on the CPU emulation."""
    from oracle import oracle
    from tests.helpers import gradcheck_like_scene
    rng = np.random.default_rng(1000 + seed)
    N = int(rng.integers(1, 4))
    H, W = int(rng.integers(3, 30)), int(rng.integers(3, 40))
    k3 = int(rng.integers(1, 5))
    cubic = bool(rng.integers(0, 2))
    M = int(rng.choice([2, 3, 4, 8]))
    dims = None if cubic else (int(rng.integers(1, 6)), int(rng.integers(1, 6)), int(rng.integers(1, 6)))
    s = gradcheck_like_scene(N=N, H=H, W=W, k3=k3, M=M, seed=50 + seed, alpha_gain=float(rng.choice([0.5, 8.0, 60.0])),
                             scale=float(rng.uniform(0.9, 2.5)), dims=dims, fadescale=float(rng.uniform(4.0, 9.0)),
                             fadeexp=float(rng.uniform(5.0, 9.0)))
    s["stepsize"] = float(rng.choice([1.3, 0.39, 0.11, 0.03]))
    grad = torch.randn(N, H, W, 4, generator=torch.Generator().manual_seed(seed))
    a, kw = scene_args_np(s)
    out, _, grads = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    ref, raysat = oracle.forward(*a, **kw)
    assert np.isfinite(out).all() and relerr(out, ref) <= FWD_TOL
    gref = oracle.backward(*a, grad.numpy(), raysat, **kw)
    for nm, g_, r in zip(("primpos", "primrot", "primscale", "template"), grads, gref):
        assert np.isfinite(g_).all(), nm
        if np.abs(r).max() > 0:
            assert relerr(g_, r) <= BWD_TOL, nm


@pytest.mark.parametrize("name", ["head_small", "gradcheck_ragged", "many_overlaps", "warp_small"])
def test_emulated_marching_order_indirection(kernels, name):
    """An explicit marching order (C-ABI `order`, what usebvh=True passes) == the fixed-order kernels on primitive tensors
    gathered into that order, gradients scattered back: forward bit for bit."""
    from ava256_b200.op import morton_order
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    order = morton_order(s["primpos"]).numpy().astype(np.int32)              # [N,K]
    if name == "gradcheck_ragged":                                            # a non-trivial permutation in any case
        order = order[:, ::-1].copy()
    out_i, sat_i, g_i = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), order=order, **kw)
    take = lambda x: np.take_along_axis(x, order.reshape(order.shape + (1,) * (x.ndim - 2)).astype(np.int64), axis=1)
    a2 = list(a)
    for i in (4, 5, 6, 7):
        a2[i] = take(a[i])
    kw2 = dict(kw)
    if "warp" in kw:
        kw2["warp"] = take(kw["warp"])
    out_g, sat_g, g_g = kernels.forward_backward(*a2, grad_rayrgba=grad.numpy(), **kw2)
    assert np.array_equal(out_i, out_g) and np.array_equal(sat_i, sat_g)
    for x, y in zip(g_i, g_g):
        back = np.zeros_like(y)
        np.put_along_axis(back, order.reshape(order.shape + (1,) * (y.ndim - 2)).astype(np.int64), y, axis=1)
        assert relerr(x, back) <= 1e-5
    out_f, _, _ = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    assert not np.array_equal(order, np.arange(order.shape[1])[None].repeat(order.shape[0], 0))


@pytest.mark.parametrize("name", ["head_small", "warp_head", "many_views", "odd_k"])
def test_emulated_forward_clears_gradient_buffers(kernels, name):
    """mvp_forward_args::clear_grad_*: the gradient-mode forward leaves the (NaN-filled) gradient buffers zero -- every float of
    every buffer, also when the count is not a multiple of 4 or of the warps of the launch -- and the backward that follows
    without MVP_FLAG_ZERO_GRADS returns the same gradients."""
    if name == "odd_k":                                   # K = 9: 54 / 162 floats, tails and empty slices
        from ava256_b200 import scene
        sc = scene.make_scene(2, 24, 40, 9, 8, seed=5)
        a = (sc["raypos"].numpy(), sc["raydir"].numpy(), sc["stepsize"], sc["tminmax"].numpy(), sc["primpos"].numpy(),
             sc["primrot"].numpy(), sc["primscale"].numpy(), sc["template"].numpy())
        kw = {}
        grad = torch.randn(2, 24, 40, 4, generator=torch.Generator().manual_seed(3))
    else:
        s, grad = build_case(name)
        a, kw = scene_args_np(s)
    out0, sat0, g0 = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    out1, sat1, g1 = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), clear_in_forward=True, **kw)
    assert np.array_equal(out0, out1) and np.array_equal(sat0, sat1)
    for x, y in zip(g0, g1):
        assert np.isfinite(y).all() and relerr(x, y) <= 1e-5


def test_emulated_runtime_flags(kernels):
    """C-ABI flags of the product library on the emulation: MVP_FLAG_TEST_TINY_LISTS (almost every tile takes the backward's
    rebuild path), MVP_FLAG_ZERO_GRADS (the library zero-fills NaN-initialised gradient buffers)."""
    import ctypes
    from ava256_b200 import lib
    s, grad = build_case("head_small")
    a, kw = scene_args_np(s)
    out0, sat0, g0 = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    loaded, rebuilt = ctypes.c_int(), ctypes.c_int()
    kernels.load().mvp_emul_saved_list_tiles(ctypes.byref(loaded), ctypes.byref(rebuilt))
    assert loaded.value > 0 and rebuilt.value == 0
    out1, sat1, g1 = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), fwd_flags=lib.FLAG_TEST_TINY_LISTS,
                                              bwd_flags=lib.FLAG_ZERO_GRADS, **kw)
    kernels.load().mvp_emul_saved_list_tiles(ctypes.byref(loaded), ctypes.byref(rebuilt))
    assert rebuilt.value > loaded.value > 0
    assert np.array_equal(out0, out1) and np.array_equal(sat0, sat1)
    for x, y in zip(g0, g1):
        assert np.isfinite(y).all() and relerr(x, y) <= 1e-5


@pytest.mark.parametrize("name", ["head_small", "warp_head"])
def test_emulated_shared_primitives(kernels, name):
    """MVP_FLAG_SHARED_PRIMS: one [1,K,...] set of primitives rendered by all views == materialised per-view copies, with
    the gradients of all views accumulated into the one set."""
    from ava256_b200 import lib
    s, grad = build_case(name)
    N = 3
    from ava256_b200 import scene
    H, W = s["raypos"].shape[1:3]
    rp, rd, tmm = scene.make_rays(N, H, W, view_offset=2)
    one = {k: s[k][:1].numpy() for k in ("primpos", "primrot", "primscale", "template")}
    rep = {k: np.repeat(v, N, axis=0) for k, v in one.items()}
    warp1 = s["warp"][:1].numpy() if "warp" in s else None
    g = torch.randn(N, H, W, 4, generator=torch.Generator().manual_seed(2)).numpy()
    kw = dict(fadescale=s["fadescale"], fadeexp=s["fadeexp"])
    out_m, sat_m, g_m = kernels.forward_backward(rp.numpy(), rd.numpy(), s["stepsize"], tmm.numpy(), rep["primpos"], rep["primrot"],
                                                 rep["primscale"], rep["template"], grad_rayrgba=g,
                                                 warp=None if warp1 is None else np.repeat(warp1, N, axis=0), **kw)
    out_s, sat_s, g_s = kernels.forward_backward(rp.numpy(), rd.numpy(), s["stepsize"], tmm.numpy(), one["primpos"], one["primrot"],
                                                 one["primscale"], one["template"], grad_rayrgba=g, warp=warp1,
                                                 fwd_flags=lib.FLAG_SHARED_PRIMS, bwd_flags=lib.FLAG_SHARED_PRIMS | lib.FLAG_ZERO_GRADS, **kw)
    assert float(out_m[..., 3].max()) > 0.05
    assert np.array_equal(out_m, out_s) and np.array_equal(sat_m, sat_s)
    for x, y in zip(g_m, g_s):
        assert y.shape[0] == 1
        assert relerr(y, x.sum(axis=0, keepdims=True)) <= 1e-5


@pytest.mark.parametrize("order", ["forward", "random"])
@pytest.mark.parametrize("cap", list(DENSE_K3))
@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_emulated_heavy_kernels_vs_oracle(kernels, name, cap, order):
    """The default build on scenes whose every tile's slab list outgrows the fast kernels' 256 entries: the 512-entry kernels
    render them all (counted by mvp_debug_heavy_offset), with 343-entry lists and with 729 cut at the reference's 512."""
    from oracle import oracle
    s, grad = build_dense_case(name, cap)
    a, kw = scene_args_np(s)
    kernels.set_lane_order(order)
    out, raysat, grads = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    heavy = kernels.last_heavy_tiles
    N, H, W = s["raypos"].shape[:3]
    assert heavy == (N * -(-H // 4) * -(-W // 8),) * 2, heavy
    ref, rsat, stats = oracle.forward(*a, return_stats=True, **kw)
    assert (stats["capped_warps"] > 0) == (cap == "capped")
    assert 0.1 <= float((rsat[..., 0] > -1.0).mean()) <= 0.9
    assert relerr(out, ref) <= FWD_TOL
    assert np.array_equal(raysat[..., 0] > -1.0, rsat[..., 0] > -1.0)
    gref = oracle.backward(*a, grad.numpy(), rsat, **kw)
    for nm, g, r in zip(("primpos", "primrot", "primscale", "template", "warp"), grads, gref):
        assert relerr(g, r) <= BWD_TOL, nm
    out2, _, _ = kernels.forward_backward(*a, **kw)
    assert kernels.last_heavy_tiles[0] == heavy[0] and np.array_equal(out2, out)


def test_emulated_heavy_persistent_loop(kernels):
    """Twice as many heavy tiles as the emulated persistent grid has warps (4 CTAs x 132 SMs x 4 warps): every warp renders
    more than one tile.  Few rays saturate here: a saturating ray's gradient jumps when rounding moves the sample at which it
    saturates, and among 280 000 rays some sit that close to the threshold (float32 and float64 oracles differ by 1e-2 on the
    scene of test_emulated_heavy_kernels_vs_oracle at this size)."""
    from oracle import oracle
    s = dense_scene(N=2, H=250, W=270, k3=7, M=8, seed=9, gain=(0.02, 0.4))
    grad = torch.randn(2, 250, 270, 4, generator=torch.Generator().manual_seed(7))
    a, kw = scene_args_np(s)
    out, raysat, grads = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    assert min(kernels.last_heavy_tiles) >= 2 * 4 * 132 * 4, kernels.last_heavy_tiles
    ref, rsat = oracle.forward(*a, **kw)
    assert relerr(out, ref) <= FWD_TOL
    assert np.array_equal(raysat[..., 0] > -1.0, rsat[..., 0] > -1.0) and (rsat[..., 0] > -1.0).any()
    gref = oracle.backward(*a, grad.numpy(), rsat, **kw)
    for nm, g, r in zip(("primpos", "primrot", "primscale", "template"), grads, gref):
        assert relerr(g, r) <= BWD_TOL, nm


# ------------------------------------------------------------------------------------------------------------------
# auxiliary kernels (raydirs.cu, epilogue.cu) on the same emulation: thread -> element mapping, vector paths, block reduction
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def aux():
    import ctypes
    from tests.emul.build import build_aux
    L = ctypes.CDLL(build_aux())
    P, I, F = ctypes.c_void_p, ctypes.c_int32, ctypes.c_float
    L.mvp_compute_raydirs.argtypes = [I] * 3 + [P] * 5 + [F] + [P] * 4
    L.mvp_composite_forward.argtypes = [I] * 3 + [P] * 7
    L.mvp_composite_backward.argtypes = [I] * 3 + [P] * 10
    L.mvp_assemble_payload_forward.argtypes = [I] * 4 + [P] * 2 + [F] * 2 + [P] * 2
    L.mvp_assemble_payload_backward.argtypes = [I] * 4 + [P] * 2 + [F] + [P] * 3
    return L


def _ptr(t):
    return None if t is None else t.data_ptr()


@pytest.mark.parametrize("with_pixelcoords", [False, True])
def test_emulated_raydirs_kernel(aux, with_pixelcoords):
    from ava256_b200 import scene
    n, H, W = 3, 37, 301                                   # W > 256: two blocks per image row, ragged tail
    campos, camrot = scene.look_at_cameras(n)
    campos, camrot = campos.float().contiguous(), camrot.float().contiguous()
    focal = torch.full((n, 2), scene.FOCAL_FULLRES / (scene.FULLRES_H / H))
    princpt = torch.tensor([[W / 2.0, H / 2.0]]).expand(n, 2).contiguous()
    pc = None
    if with_pixelcoords:
        py, px = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
        pc = torch.stack([px, py], dim=-1)[None].repeat(n, 1, 1, 1).contiguous()
    rp, rd, tmm = torch.full((n, H, W, 3), float("nan")), torch.full((n, H, W, 3), float("nan")), torch.full((n, H, W, 2), float("nan"))
    assert aux.mvp_compute_raydirs(n, H, W, _ptr(campos), _ptr(camrot), _ptr(focal), _ptr(princpt), _ptr(pc), scene.VOLRADIUS,
                                   _ptr(rp), _ptr(rd), _ptr(tmm), None) == 0
    hp, hd, ht = scene.compute_raydirs_host(campos, camrot, focal, princpt, H, W)
    assert relerr(rp.numpy(), hp.numpy()) < 1e-6 and relerr(rd.numpy(), hd.numpy()) < 1e-6
    # clip range: rays that cross the cube to 1e-5; a ray that misses it parallel to a face has a clip distance of 1 / (a direction
    # component that nearly cancels), which follows the kernel's fused multiply-adds (raygen.h), not torch's separate roundings
    hit = (ht[..., 0] < ht[..., 1]).numpy()
    assert hit.mean() > 0.05
    assert relerr(tmm.numpy()[hit], ht.numpy()[hit]) < 1e-5
    assert np.array_equal(tmm.numpy()[..., 0] < tmm.numpy()[..., 1], hit)
    assert relerr(tmm.numpy()[~hit], ht.numpy()[~hit]) < 1e-2


@pytest.mark.parametrize("shape", [(3, 6, 10), (2, 7, 9), (2, 33, 67), (1, 64, 48)])
@pytest.mark.parametrize("with_cc,with_bg", [(False, False), (True, True)])
def test_emulated_composite_kernels(aux, shape, with_cc, with_bg):
    from oracle.epilogue_ref import composite_ref
    N, H, W = shape
    g = torch.Generator().manual_seed(H)
    rayrgba = torch.rand(N, H, W, 4, generator=g)
    rayrgba[..., :3] *= 255.0
    ccw = (1.0 + 0.3 * torch.randn(N, 3, generator=g)) if with_cc else None
    ccb = (5.0 * torch.randn(N, 3, generator=g)) if with_cc else None
    bg = (255.0 * torch.rand(N, 3, H, W, generator=g)) if with_bg else None
    g_rgb, g_alpha = torch.randn(N, 3, H, W, generator=g), torch.randn(N, 1, H, W, generator=g)
    leaves = [None if t is None else t.clone().requires_grad_(True) for t in (rayrgba, ccw, ccb, bg)]
    ref_rgb, ref_alpha = composite_ref(*leaves)
    ((ref_rgb * g_rgb).sum() + (ref_alpha * g_alpha).sum()).backward()
    rgb, alpha = torch.full((N, 3, H, W), float("nan")), torch.full((N, 1, H, W), float("nan"))
    assert aux.mvp_composite_forward(N, H, W, _ptr(rayrgba), _ptr(ccw), _ptr(ccb), _ptr(bg), _ptr(rgb), _ptr(alpha), None) == 0
    assert torch.equal(rgb, ref_rgb.detach()) and torch.equal(alpha, ref_alpha.detach())
    grad_rayrgba = torch.full((N, H, W, 4), float("nan"))
    grad_ccw = torch.zeros(N, 3) if with_cc else None
    grad_ccb = torch.zeros(N, 3) if with_cc else None
    grad_bg = torch.full((N, 3, H, W), float("nan")) if with_bg else None
    assert aux.mvp_composite_backward(N, H, W, _ptr(rayrgba), _ptr(ccw), _ptr(bg), _ptr(g_rgb), _ptr(g_alpha), _ptr(grad_rayrgba),
                                      _ptr(grad_ccw), _ptr(grad_ccb), _ptr(grad_bg), None) == 0
    torch.testing.assert_close(grad_rayrgba, leaves[0].grad, rtol=1e-6, atol=1e-4)
    if with_cc:
        torch.testing.assert_close(grad_ccw, leaves[1].grad, rtol=1e-4, atol=1e-1)
        torch.testing.assert_close(grad_ccb, leaves[2].grad, rtol=1e-4, atol=1e-3)
    if with_bg:
        torch.testing.assert_close(grad_bg, leaves[3].grad, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("N,hb,wb,B", [(2, 2, 3, 8), (1, 3, 2, 4), (1, 4, 2, 3), (1, 1, 1, 1), (1, 2, 2, 16), (1, 9, 9, 8)])
def test_emulated_payload_kernels(aux, N, hb, wb, B):
    from oracle.epilogue_ref import assemble_payload_ref
    g = torch.Generator().manual_seed(B)
    tex = (torch.randn(N, 3 * B, hb * B, wb * B, generator=g) * 4.0 - 2.0).requires_grad_(True)
    opa = torch.randn(N, B, hb * B, wb * B, generator=g).requires_grad_(True)
    gt = torch.randn(N, hb * wb, B, B, B, 4, generator=g)
    ref = assemble_payload_ref(tex, opa, B)
    (ref * gt).sum().backward()
    tp = torch.full(tuple(ref.shape), float("nan"))
    assert aux.mvp_assemble_payload_forward(N, hb, wb, B, _ptr(tex), _ptr(opa), 25.0, 100.0, _ptr(tp), None) == 0
    assert torch.equal(tp, ref.detach())
    gtex, gopa = torch.full(tuple(tex.shape), float("nan")), torch.full(tuple(opa.shape), float("nan"))
    assert aux.mvp_assemble_payload_backward(N, hb, wb, B, _ptr(tp), _ptr(gt), 25.0, _ptr(gtex), _ptr(gopa), None) == 0
    assert torch.equal(gtex, tex.grad) and torch.equal(gopa, opa.grad)


@pytest.mark.parametrize("variant", [(), ("MVP_XBUCKETS=1",)])
def test_emulated_non_pinhole_rays_fall_back(kernels, variant):
    """Shuffled pixels: the camera fit rejects the view and every slab becomes a candidate of every tile (same as the GPU test)."""
    from oracle import oracle
    s, grad = build_case("gradcheck_ragged")
    g = torch.Generator().manual_seed(3)
    N, H, W = s["raypos"].shape[:3]
    perm = torch.randperm(H * W, generator=g)
    for k in ("raypos", "raydir", "tminmax"):
        v = s[k]
        s[k] = v.reshape(N, H * W, -1)[:, perm].reshape(v.shape).contiguous()
    a, kw = scene_args_np(s)
    kernels.use_variant(variant, opt="-O0" if variant else "-O1")
    out, _, grads = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    ref, raysat = oracle.forward(*a, **kw)
    assert relerr(out, ref) <= FWD_TOL
    gref = oracle.backward(*a, grad.numpy(), raysat, **kw)
    for nm, g_, r in zip(("primpos", "primrot", "primscale", "template"), grads, gref):
        assert relerr(g_, r) <= BWD_TOL, nm


def test_emulated_row_bucket_overflow_falls_back_to_all_slabs(kernels):
    """More slabs in one tile row than the bucket holds (K > 2048 slabs, all pulled onto the optical axis so that every one
    projects into every tile row): the row is scanned slab by slab instead, and every tile hits the reference's 512-entry
    cap.  Checked against the oracle, which implements that cap."""
    from ava256_b200 import scene
    from oracle import oracle
    K = 2304
    s = scene.make_scene(1, 16, 24, K, 2, alpha_mu=0.05, alpha_sigma=0.02)
    s["primpos"] = (s["primpos"] * 0.02).contiguous()
    s["stepsize"] = 1.0 / 16
    grad = torch.randn(1, 16, 24, 4, generator=torch.Generator().manual_seed(5))
    a, kw = scene_args_np(s)
    out, _, grads = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
    ref, raysat, stats = oracle.forward(*a, return_stats=True, **kw)
    assert stats["capped_warps"] >= 1 and float(out[..., 3].max()) > 0     # > 2048 candidates in the row, 512-entry cap hit
    assert relerr(out, ref) <= FWD_TOL
    gref = oracle.backward(*a, grad.numpy(), raysat, **kw)
    for nm, g_, r in zip(("primpos", "primrot", "primscale", "template"), grads, gref):
        assert relerr(g_, r) <= BWD_TOL, nm


# ------------------------------------------------------------------------------------------------------------------
# rays generated in the render kernels' prologue from the camera (mvp_camera; SURVEY.md section 8f row 1) must be the rays
# mvp_compute_raydirs writes, and the images / gradients those of the two-call form
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,H,W,K,T,planes", [(2, 64, 42, 64, 8, False), (1, 13, 19, 16, 4, True), (3, 30, 50, 64, 8, False)])
def test_emulated_camera_rays_match_ray_tensors(kernels, aux, n, H, W, K, T, planes):
    from ava256_b200 import scene
    viewpos, viewrot, focal, princpt = scene.make_cameras(n, H, W, view_offset=3)
    rp, rd, tmm = torch.full((n, H, W, 3), float("nan")), torch.full((n, H, W, 3), float("nan")), torch.full((n, H, W, 2), float("nan"))
    assert aux.mvp_compute_raydirs(n, H, W, _ptr(viewpos), _ptr(viewrot), _ptr(focal), _ptr(princpt), None, scene.VOLRADIUS,
                                   _ptr(rp), _ptr(rd), _ptr(tmm), None) == 0
    s = scene.make_scene(n, H, W, K, T, view_offset=3, alpha_mu=1.0, alpha_sigma=2.0, share_primitives=False)
    g = torch.randn(n, H, W, 4, generator=torch.Generator().manual_seed(5)).numpy()
    prim = (s["primpos"].numpy(), s["primrot"].numpy(), s["primscale"].numpy(), s["template"].numpy())
    step = 1.0 / 64
    out_t, sat_t, g_t = kernels.forward_backward(rp.numpy(), rd.numpy(), step, tmm.numpy(), *prim, grad_rayrgba=g, planes=planes)
    cam = (viewpos.numpy(), viewrot.numpy(), focal.numpy(), princpt.numpy(), scene.VOLRADIUS, H, W)
    out_c, sat_c, g_c = kernels.forward_backward(None, None, step, None, *prim, grad_rayrgba=g, planes=planes, camera=cam)
    assert float(out_t[..., 3].max()) > 0.05
    assert np.array_equal(out_t, out_c) and np.array_equal(sat_t, sat_c)
    for x, y in zip(g_t, g_c):
        assert relerr(y, x) <= 1e-6
    # inference mode (no raysat / rayaux) through the same prologue
    out_i, _, _ = kernels.forward_backward(None, None, step, None, *prim, camera=cam)
    assert np.array_equal(out_i, out_c)


def test_emulated_camera_argument_errors(kernels):
    import ctypes
    from ava256_b200 import lib as abi
    L = kernels.load()
    a = abi.ForwardArgs()
    a.shape = abi.Shape(1, 8, 8, 4, 2, 2, 2)
    a.stepsize = 0.1
    dummy = ctypes.c_void_p(256)
    for f in ("primpos", "primrot", "primscale", "tplate", "rayrgba", "workspace"):
        setattr(a, f, dummy)
    a.workspace_bytes = 1 << 30
    assert L.mvp_raymarch_forward(ctypes.byref(a), None) == -1                 # neither rays nor a camera
    a.camera = abi.Camera(dummy, dummy, dummy, None, 256.0, 0)
    assert L.mvp_raymarch_forward(ctypes.byref(a), None) == -1                 # three of the four camera arrays
    a.camera = abi.Camera(dummy, dummy, dummy, dummy, 0.0, 0)
    assert L.mvp_raymarch_forward(ctypes.byref(a), None) == -8                 # MVP_ERR_CAMERA
    a.camera = abi.Camera(dummy, dummy, dummy, ctypes.c_void_p(258), 256.0, 0)
    assert L.mvp_raymarch_forward(ctypes.byref(a), None) == -6                 # MVP_ERR_ALIGN


def test_emulated_degenerate_camera_falls_back(kernels):
    """focal = 0 for one view: its rays are not finite and nothing can be projected -- the view is flagged like a failed camera fit
    (every slab a candidate, no hits) and the other view renders as before."""
    from ava256_b200 import scene
    n, H, W, K, T = 2, 16, 20, 16, 4
    viewpos, viewrot, focal, princpt = scene.make_cameras(n, H, W)
    s = scene.make_scene(n, H, W, K, T, alpha_mu=2.0, alpha_sigma=2.0, share_primitives=False)
    prim = (s["primpos"].numpy(), s["primrot"].numpy(), s["primscale"].numpy(), s["template"].numpy())
    good, _, _ = kernels.forward_backward(None, None, 1.0 / 32, None, *prim,
                                          camera=(viewpos.numpy(), viewrot.numpy(), focal.numpy(), princpt.numpy(), scene.VOLRADIUS, H, W))
    bad_focal = focal.clone()
    bad_focal[1] = 0.0
    out, _, _ = kernels.forward_backward(None, None, 1.0 / 32, None, *prim,
                                         camera=(viewpos.numpy(), viewrot.numpy(), bad_focal.numpy(), princpt.numpy(), scene.VOLRADIUS, H, W))
    assert float(good[0, ..., 3].max()) > 0.0
    assert np.array_equal(out[0], good[0])
    assert not out[1].any()
