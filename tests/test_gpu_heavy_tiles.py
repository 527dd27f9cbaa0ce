"""GPU tests of the 512-entry ("heavy") render kernels (`pytest -m gpu`).  A tile whose slab list outgrows the fast kernels'
256-entry shared-memory list is handed over, possibly with a TMA copy of the next bucket chunk still in flight, to a small
persistent CAP = 512 kernel whose warps walk the list of such tiles and re-initialise their staging mbarriers for every tile.
The scenes of tests/helpers.py DENSE_CASES make every tile heavy; each test reads the number of heavy tiles of every forward and
backward call back from the workspace (`mvp_debug_heavy_offset`) and asserts that the path ran.  Gates as in the rest of the
suite: forward max|d|/max|ref| <= 1e-4 and gradients <= 1e-3 against the oracle; 1e-5 between runs that differ only in the
order of the gradient atomics."""
import pytest
import torch

from tests.helpers import DENSE_CASES, DENSE_K3, abi_raymarch, build_dense_case, dense_scene, relerr, scene_args_np

pytestmark = pytest.mark.gpu

FWD_TOL = 1e-4
BWD_TOL = 1e-3
NAMES = ("primpos", "primrot", "primscale", "template", "warp")
HEAVY_CTAS_PER_SM = 4          # kHeavyCtasPerSM in csrc/mvp_kernels.cu: the persistent grid is 4 CTAs per SM


def _cuda(s):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in s.items()}


def _report(tag, heavy):
    print("%s: heavy tiles forward %d, backward %d" % (tag, heavy[0], heavy[1]))
    assert heavy[0] > 0 and heavy[1] > 0, heavy


def _vs_oracle(s, grad, out, grads):
    from oracle import oracle
    a, kw = scene_args_np(s)
    ref, raysat, stats = oracle.forward(*a, return_stats=True, **kw)
    assert relerr(out.cpu().numpy(), ref) <= FWD_TOL
    gref = oracle.backward(*a, grad.numpy(), raysat, **kw)
    assert len(grads) == len(gref)
    for nm, g, r in zip(NAMES, grads, gref):
        assert bool(torch.isfinite(g).all()), nm
        assert relerr(g.cpu().numpy(), r) <= BWD_TOL, nm
    return stats


@pytest.mark.parametrize("cap", list(DENSE_K3))
@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_heavy_kernels_vs_oracle(name, cap):
    """Every instantiation of the 512-entry kernels (T = 8, 16, runtime dims, warp field) with lists of 343 entries and with
    lists of 729 cut at the reference's 512; the inference-mode forward (kGrad = false) gives the same image bits."""
    s, grad = build_dense_case(name, cap)
    t = _cuda(s)
    out, rsat, grads, heavy = abi_raymarch(t, grad.cuda())
    _report("%s/%s" % (name, cap), heavy)
    sat = float((out[..., 3] >= 1.0).float().mean())
    assert 0.1 <= sat <= 0.9, sat
    stats = _vs_oracle(s, grad, out, grads)
    assert (stats["capped_warps"] > 0) == (cap == "capped"), stats
    out_i, _, _, heavy_i = abi_raymarch(t)
    assert heavy_i[0] == heavy[0]
    assert torch.equal(out_i, out)


def test_heavy_persistent_loop_walks_every_tile():
    """More heavy tiles in one launch than the persistent grid has warps (twice as many, for the SM count of this device): every
    warp renders a second tile and re-initialises its staging mbarriers on a barrier it used before.  Against the oracle, against
    the views rendered one per launch (forward bit for bit), and run twice (bit-identical forward: the list of heavy tiles is
    filled in atomic order, which must not matter)."""
    from ava256_b200 import lib
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    warps = int(lib.LIB.mvp_build_config().decode().split("WARPS=")[1].split()[0])
    grid_warps = HEAVY_CTAS_PER_SM * sms * warps
    N, W = 2, 270                                            # 34 tile columns, the last one partial
    rows = -(-2 * grid_warps // (N * 34))
    H = 4 * rows - 2                                         # the last tile row partial
    s = dense_scene(N=N, H=H, W=W, k3=7, M=8, seed=9, gain=(0.02, 0.4))   # few saturated rays (see test_emul_kernels.py)
    grad = torch.randn(N, H, W, 4, generator=torch.Generator().manual_seed(7))
    t, g = _cuda(s), grad.cuda()
    out, _, grads, heavy = abi_raymarch(t, g)
    _report("persistent %dx%dx%d, %d heavy-grid warps on %d SMs" % (N, H, W, grid_warps, sms), heavy)
    assert heavy[0] >= 2 * grid_warps and heavy[1] >= 2 * grid_warps, (heavy, grid_warps)
    out2, _, grads2, heavy2 = abi_raymarch(t, g)
    assert heavy2 == heavy and torch.equal(out2, out)
    for x, y in zip(grads, grads2):
        assert relerr(x.cpu().numpy(), y.cpu().numpy()) <= 1e-5
    for v in range(N):
        sv = {k: (x[v:v + 1].contiguous() if torch.is_tensor(x) else x) for k, x in t.items()}
        out_v, _, grads_v, heavy_v = abi_raymarch(sv, g[v:v + 1].contiguous())
        assert heavy_v[0] > 0 and torch.equal(out_v, out[v:v + 1])
        for nm, x, y in zip(NAMES, grads_v, grads):
            assert relerr(x.cpu().numpy(), y[v:v + 1].cpu().numpy()) <= 1e-5, (v, nm)
    _vs_oracle(s, grad, out, grads)


@pytest.mark.parametrize("cap", list(DENSE_K3))
def test_heavy_backward_saved_lists_equal_rebuilt(cap):
    """The heavy backward loads the lists the forward saved (longer than the fast backward's 256 entries) for the tiles whose
    list fit the per-view list storage, and rebuilds the others; under MVP_FLAG_TEST_TINY_LISTS (16 entries per view) no heavy
    tile's list is saved and every one is rebuilt.  Same gradients."""
    from ava256_b200 import lib
    from tests.test_gpu_scale_parity import _saved_tiles
    s, grad = build_dense_case("t8", cap)
    t, g = _cuda(s), grad.cuda()
    N, H, W = s["raypos"].shape[:3]
    K, T = s["primpos"].shape[1], s["template"].shape[2]
    ws0, ws1 = {}, {}
    out0, _, g0, heavy0 = abi_raymarch(t, g, keep=ws0)
    _report("saved lists/%s" % cap, heavy0)
    out1, _, g1, heavy1 = abi_raymarch(t, g, fwd_flags=lib.FLAG_TEST_TINY_LISTS, keep=ws1)
    _report("rebuilt lists/%s" % cap, heavy1)
    saved0, not_saved0 = _saved_tiles(ws0["workspace"], N, H, W, K, T)
    saved1, not_saved1 = _saved_tiles(ws1["workspace"], N, H, W, K, T)
    tiles = N * -(-H // 4) * -(-W // 8)
    assert heavy0[0] == tiles and saved0 > 0, (heavy0, saved0, not_saved0)  # heavy tiles whose saved list the backward loads
    assert not_saved1 == tiles, (saved1, not_saved1)                         # every tile rebuilt
    assert torch.equal(out0, out1)
    for nm, x, y in zip(NAMES, g0, g1):
        assert relerr(y.cpu().numpy(), x.cpu().numpy()) <= 1e-5, nm


def test_heavy_shared_primitives_equal_materialised():
    """MVP_FLAG_SHARED_PRIMS through the heavy kernels: one [1,K,...] set for 3 views == 3 materialised copies."""
    s = _cuda(dense_scene(N=3, H=17, W=27, k3=7, M=8, seed=11))
    grad = torch.randn(3, 17, 27, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    one = {k: (v[:1].contiguous() if k in NAMES else v) for k, v in s.items()}
    rep = {k: (v[:1].expand_as(v).contiguous() if k in NAMES else v) for k, v in s.items()}
    out_m, _, g_m, heavy_m = abi_raymarch(rep, grad)
    out_s, _, g_s, heavy_s = abi_raymarch(one, grad, shared=True)
    _report("shared primitives", heavy_s)
    assert heavy_s == heavy_m and torch.equal(out_s, out_m)
    for nm, x, y in zip(NAMES, g_m, g_s):
        assert y.shape[0] == 1
        assert relerr(y.cpu().numpy(), x.sum(dim=0, keepdim=True).cpu().numpy()) <= 1e-5, nm


@pytest.mark.parametrize("cap", list(DENSE_K3))
def test_heavy_marching_order_equals_gathered(cap):
    """An explicit marching order (what usebvh=True passes) through the heavy kernels == the primitives gathered into that order;
    with the 512-entry cap the order also decides which slabs make the list."""
    from ava256_b200.op import morton_order
    s, grad = build_dense_case("t8", cap)
    t, g = _cuda(s), grad.cuda()
    order = morton_order(t["primpos"]).to(torch.int32).contiguous()
    assert not torch.equal(order, torch.arange(order.size(1), device="cuda", dtype=torch.int32).expand_as(order))
    out_o, _, g_o, heavy_o = abi_raymarch(t, g, order=order)
    _report("marching order/%s" % cap, heavy_o)
    idx = order.long()
    take = lambda x: torch.gather(x, 1, idx.view(idx.shape + (1,) * (x.dim() - 2)).expand(idx.shape + tuple(x.shape[2:]))).contiguous()  # noqa: E731
    tg = {k: (take(v) if k in NAMES else v) for k, v in t.items()}
    out_g, _, g_g, heavy_g = abi_raymarch(tg, g)
    assert heavy_g == heavy_o and torch.equal(out_o, out_g)
    for nm, x, y in zip(NAMES, g_o, g_g):
        back = torch.zeros_like(y).scatter_(1, idx.view(idx.shape + (1,) * (y.dim() - 2)).expand_as(y), y)
        assert relerr(x.cpu().numpy(), back.cpu().numpy()) <= 1e-5, nm


@pytest.mark.parametrize("name", ["t8", "warp"])
def test_heavy_image_planes_equal_channels_last(name):
    """rayrgb [N,3,H,W] / rayalpha [N,1,H,W] written by the heavy kernels' epilogue and the gradient read as planes by their
    prologue == the channels-last run (forward bit for bit)."""
    s, grad = build_dense_case(name, "uncapped")
    t, g = _cuda(s), grad.cuda()
    out0, _, g0, heavy0 = abi_raymarch(t, g)
    out1, _, g1, heavy1 = abi_raymarch(t, g, planes=True)
    _report("image planes/%s" % name, heavy1)
    assert heavy1 == heavy0 and torch.equal(out0, out1)
    for nm, x, y in zip(NAMES, g0, g1):
        assert relerr(y.cpu().numpy(), x.cpu().numpy()) <= 1e-5, nm


def test_heavy_camera_rays_equal_two_call_form():
    """Rays generated in the heavy kernels' prologue from the camera == the rays of mvp_compute_raydirs passed as tensors."""
    from ava256_b200 import scene
    from extensions.utils.utils import compute_raydirs
    n, H, W = 2, 37, 45
    s = _cuda(dense_scene(N=n, H=H, W=W, k3=7, M=8, seed=10))
    s["stepsize"] = 1.0 / 16
    cams = [c.cuda() for c in scene.make_cameras(n, H, W, view_offset=3)]
    rp, rd, tmm = compute_raydirs(cams[0], cams[1], cams[2], cams[3], (W, H), scene.VOLRADIUS)
    grad = torch.randn(n, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    out_t, _, g_t, heavy_t = abi_raymarch(dict(s, raypos=rp, raydir=rd, tminmax=tmm), grad)
    out_c, _, g_c, heavy_c = abi_raymarch(s, grad, camera=tuple(cams) + (scene.VOLRADIUS, H, W))
    _report("camera rays", heavy_c)
    assert heavy_c == heavy_t
    assert float(out_t[..., 3].max()) > 0.05 and torch.equal(out_t, out_c)
    for nm, x, y in zip(NAMES, g_t, g_c):
        assert relerr(y.cpu().numpy(), x.cpu().numpy()) <= 1e-5, nm
