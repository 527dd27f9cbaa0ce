"""GPU parity at BASELINE.json's sizes against the UNMODIFIED reference CUDA extension -- its outputs on the same seeded inputs,
sampled and stored in tests/golden/scale_*.npz by tests/golden/make_scale_golden.py -- plus the capacity paths that only trigger
at scale or under a forced cap.

The reference's own harness for this comparison only prints (/root/reference/extensions/mvpraymarch/mvpraymarch.py:708-745);
here the same quantities are asserts with the north star's gates (SURVEY.md section 8d): forward max|d|/max|ref| <= 1e-4,
saturated-ray mask identical up to 1e-4 of the rays, every gradient <= 1e-3 (max|d| over the stored sample, which holds each
tensor's largest entries, over max|ref| of the whole tensor; sum|x| of the whole tensor, and the sum and max|.| of every image
row and column / every slab (template) or 4 slabs, within what the element-wise gate implies).
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests.helpers import reductions_relerr, relerr, sampled_relerr, scale_case, scene_args_np

pytestmark = pytest.mark.gpu

FWD_TOL = 1e-4
BWD_TOL = 1e-3
SATMASK_TOL = 1e-4
NAMES = ("primpos", "primrot", "primscale", "template")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _trelerr(a, b):
    """max|a-b| / max|b| on device tensors (no 10 GB host copies)."""
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)


def _ours(s, grad):
    from extensions.mvpraymarch.mvpraymarch import mvpraymarch
    lv = [s[n].detach().clone().requires_grad_(True) for n in NAMES]
    out = mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], (lv[0], lv[1], lv[2]), lv[3], None)
    out.backward(grad)
    torch.cuda.synchronize()
    return out.detach(), [x.grad for x in lv]


def assert_parity_with_golden(out, grads, name):
    """This library's rayrgba `out` and gradients `grads` (primpos, primrot, primscale, template) of the inputs of
    tests/helpers.py scale_case(name) against the reference's stored outputs."""
    gold = np.load(os.path.join(GOLDEN, "scale_%s.npz" % name))
    d, l1 = sampled_relerr(gold, "rayrgba", out)
    r = reductions_relerr(gold, "rayrgba", out)
    assert d <= FWD_TOL and l1 <= FWD_TOL and r <= FWD_TOL, (d, l1, r)
    # saturated-ray mask: the reference marks a saturated ray by raysat != -1 (primaccum.h:51-56); ours by alpha == 1
    shape = tuple(int(v) for v in gold["satmask_shape"])
    ref_mask = torch.from_numpy(np.unpackbits(gold["satmask_bits"], count=int(np.prod(shape))).astype(bool).reshape(shape))
    our_mask = (out[..., 3] >= 1.0).cpu()
    mism = float((ref_mask != our_mask).float().mean())
    assert mism <= SATMASK_TOL, "saturated-ray masks differ on %.2e of the rays" % mism
    assert float(ref_mask.float().mean()) > 0.005, "scene must exercise saturation"
    for nm, g_ in zip(NAMES, grads):
        assert bool(torch.isfinite(g_).all()), nm
        d, l1 = sampled_relerr(gold, "grad_" + nm, g_)
        r = reductions_relerr(gold, "grad_" + nm, g_)
        assert d <= BWD_TOL and l1 <= BWD_TOL and r <= BWD_TOL, (nm, d, l1, r)


def assert_scale_case_parity(name):
    """This library's fwd+bwd of scale_case(name) against the reference's stored outputs."""
    out, grads = _ours(*scale_case(name))
    assert_parity_with_golden(out, grads, name)


def test_c2_full_size_vs_reference_extension():
    """BASELINE.json config 2: 1 subject, 4 views 512x334, K=4096, 16^3, fwd+bwd vs the reference mvpraymarch."""
    assert_scale_case_parity("c2")


def test_c3_bench_scene_vs_reference_extension():
    """The scene bench.py times (C3: 1024x667, K=16384, 8^3, alpha 17/6, dt=1/256), 4 of its 80 views (views 0, 1 and the
    two most oblique ones come from different view offsets), every default capacity path of the benchmarked binary live."""
    import bench
    assert (bench.H, bench.W, bench.K, bench.T, bench.ALPHA_MU, bench.ALPHA_SIGMA) == (1024, 667, 16384, 8, 17.0, 6.0)
    for name in ("c3_view0", "c3_view78"):
        assert_scale_case_parity(name)
        torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------------------------
# capacity paths
# ----------------------------------------------------------------------------------------------------------------
def _abi_fwd_bwd(s, grad, fwd_flags=0, shared=False):
    """forward + backward straight through the C-ABI (so test-hook flags can be passed)."""
    from ava256_b200 import lib
    N, H, W = s["raypos"].shape[:3]
    K = s["primpos"].shape[1]
    TD, TH, TW = s["template"].shape[2:5]
    P = lambda x: ctypes.c_void_p(x.data_ptr())  # noqa: E731
    wsb = lib.workspace_bytes(N, H, W, K, TD, TH, TW)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    rgba = torch.empty(N, H, W, 4, device="cuda")
    rsat = torch.empty(N, H, W, 3, device="cuda")
    raux = torch.empty(N, H, W, 4, dtype=torch.int32, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    sh = lib.FLAG_SHARED_PRIMS if shared else 0
    a = lib.ForwardArgs()
    a.shape = lib.Shape(N, H, W, K, TD, TH, TW)
    a.stepsize, a.fadescale, a.fadeexp, a.flags = s["stepsize"], s.get("fadescale", 8.0), s.get("fadeexp", 8.0), fwd_flags | sh
    a.raypos, a.raydir, a.tminmax = P(s["raypos"]), P(s["raydir"]), P(s["tminmax"])
    a.primpos, a.primrot, a.primscale, a.tplate = P(s["primpos"]), P(s["primrot"]), P(s["primscale"]), P(s["template"])
    a.rayrgba, a.raysat, a.rayaux, a.workspace, a.workspace_bytes = P(rgba), P(rsat), P(raux), P(ws), wsb
    lib.check(lib.LIB.mvp_raymarch_forward(ctypes.byref(a), st))
    gs = [torch.full_like(s[n], float("nan")) for n in NAMES]           # ZERO_GRADS must overwrite these
    b = lib.BackwardArgs()
    b.shape, b.stepsize, b.fadescale, b.fadeexp = a.shape, a.stepsize, a.fadescale, a.fadeexp
    b.flags = lib.FLAG_ACCEL_VALID | lib.FLAG_ZERO_GRADS | sh
    b.raypos, b.raydir, b.tminmax = a.raypos, a.raydir, a.tminmax
    b.primpos, b.primrot, b.primscale, b.tplate = a.primpos, a.primrot, a.primscale, a.tplate
    b.grad_rayrgba, b.raysat, b.rayaux = P(grad), P(rsat), P(raux)
    b.grad_primpos, b.grad_primrot, b.grad_primscale, b.grad_tplate = (P(g) for g in gs)
    b.workspace, b.workspace_bytes = P(ws), wsb
    lib.check(lib.LIB.mvp_raymarch_backward(ctypes.byref(b), st))
    torch.cuda.synchronize()
    return rgba, gs, ws


def _saved_tiles(ws, N, H, W, K, T):
    """(tiles with a saved list, tiles marked not-saved) read back from the workspace's tile headers -- layout as in
    csrc/mvp_kernels.cu make_layout(); only used to prove which path the backward took."""
    from ava256_b200 import lib
    n = lib.LIB.mvp_debug_saved_tiles
    n.restype = ctypes.c_int
    n.argtypes = [ctypes.POINTER(lib.Shape), ctypes.c_void_p, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
    sh = lib.Shape(N, H, W, K, T, T, T)
    a, b = ctypes.c_int(0), ctypes.c_int(0)
    host = ws.cpu()
    assert n(ctypes.byref(sh), ctypes.c_void_p(host.data_ptr()), ctypes.byref(a), ctypes.byref(b)) == 0
    return a.value, b.value


def test_list_reuse_overflow_fallback_on_device():
    """With the list storage capped at 16 entries per view almost every tile is marked not-saved by the forward and the
    backward rebuilds its list (the path that, at the default cap, no test scene can reach on the GPU)."""
    from ava256_b200 import lib, scene
    from oracle import oracle
    s = scene.make_scene(2, 96, 64, 256, 8, alpha_mu=6.0, alpha_sigma=4.0, share_primitives=False)
    grad = torch.randn(2, 96, 64, 4, generator=torch.Generator().manual_seed(12))
    sc = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in s.items()}
    out0, g0, ws0 = _abi_fwd_bwd(sc, grad.cuda())
    out1, g1, ws1 = _abi_fwd_bwd(sc, grad.cuda(), fwd_flags=lib.FLAG_TEST_TINY_LISTS)
    sv0, ns0 = _saved_tiles(ws0, 2, 96, 64, 256, 8)
    sv1, ns1 = _saved_tiles(ws1, 2, 96, 64, 256, 8)
    assert ns0 == 0 and sv0 > 50, (sv0, ns0)
    assert ns1 > 50 and sv1 <= 2 * 16, (sv1, ns1)              # the rebuild path really ran
    assert torch.equal(out0, out1)
    a, kw = scene_args_np(s)
    ref, raysat = oracle.forward(*a, **kw)
    assert relerr(out1.cpu().numpy(), ref) <= FWD_TOL
    gref = oracle.backward(*a, grad.numpy(), raysat, **kw)
    for nm, x0, x1, r in zip(NAMES, g0, g1, gref):
        assert relerr(x1.cpu().numpy(), r) <= BWD_TOL, nm
        assert relerr(x1.cpu().numpy(), x0.cpu().numpy()) <= 1e-5, nm


def test_row_bucket_overflow_and_512_cap_on_device():
    """K = 2304 slabs pulled onto the optical axis: every tile row sees more candidates than a row bucket holds (2048), so
    the list build scans all slabs, and every tile's list is cut at the reference's 512 entries (utils.h:779-781).  Same
    scene as the emulated test (tests/test_emul_kernels.py); the oracle implements the cap and reports that it was hit."""
    from ava256_b200 import scene
    from oracle import oracle
    from tests.test_gpu_parity import run_ours
    s = scene.make_scene(1, 16, 24, 2304, 2, alpha_mu=0.05, alpha_sigma=0.02)
    s["primpos"] = (s["primpos"] * 0.02).contiguous()
    s["stepsize"] = 1.0 / 16
    grad = torch.randn(1, 16, 24, 4, generator=torch.Generator().manual_seed(5))
    out, grads = run_ours(s, grad)
    a, kw = scene_args_np(s)
    ref, raysat, stats = oracle.forward(*a, return_stats=True, **kw)
    assert stats["capped_warps"] >= 1 and float(out[..., 3].max()) > 0
    assert relerr(out, ref) <= FWD_TOL
    gref = oracle.backward(*a, grad.numpy(), raysat, **kw)
    for nm, g_, r in zip(NAMES, grads, gref):
        assert relerr(g_, r) <= BWD_TOL, nm


# ----------------------------------------------------------------------------------------------------------------
# extensions of the boundary: shared primitives, unaligned views
# ----------------------------------------------------------------------------------------------------------------
def test_shared_primitives_equal_materialised_views():
    """Primitive tensors with a batch of 1 are shared by all views: same images as the materialised [N,K,...] copies,
    gradients = the sum over views of the per-view gradients."""
    from ava256_b200 import scene
    from extensions.mvpraymarch.mvpraymarch import mvpraymarch
    N = 3
    s = scene.make_scene(N, 128, 96, 1024, 8, alpha_mu=10.0, alpha_sigma=5.0, device="cuda")
    grad = torch.randn(N, 128, 96, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    out_m, g_m = _ours(s, grad)
    lv = [s[n][:1].detach().clone().requires_grad_(True) for n in NAMES]
    out_s = mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], (lv[0], lv[1], lv[2]), lv[3], None)
    out_s.backward(grad)
    assert torch.equal(out_s.detach(), out_m)
    for nm, x, gm in zip(NAMES, lv, g_m):
        assert x.grad.shape == x.shape, nm
        assert _trelerr(x.grad, gm.sum(dim=0, keepdim=True)) <= 1e-5, nm


def test_unaligned_contiguous_views_are_accepted():
    """A contiguous template / tminmax / incoming gradient that starts in the middle of a larger buffer (data_ptr not a
    multiple of 16) must not fault (C-ABI: MVP_ERR_ALIGN; the op re-homes such tensors)."""
    from ava256_b200 import lib, scene
    from extensions.mvpraymarch.mvpraymarch import mvpraymarch
    s = scene.make_scene(1, 64, 48, 64, 8, alpha_mu=6.0, alpha_sigma=4.0, device="cuda")
    grad = torch.randn(1, 64, 48, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    out0, g0 = _ours(s, grad)

    def shifted(t):
        buf = torch.empty(t.numel() + 1, device="cuda")
        v = buf[1:].view(t.shape)
        v.copy_(t)
        assert v.data_ptr() % 16 == 4 and v.is_contiguous()
        return v

    s2 = dict(s, template=shifted(s["template"]), tminmax=shifted(s["tminmax"]))
    lv = [s2[n].detach().clone().requires_grad_(True) if n != "template" else s2[n].detach().requires_grad_(True) for n in NAMES]
    out = mvpraymarch(s2["raypos"], s2["raydir"], s2["stepsize"], s2["tminmax"], (lv[0], lv[1], lv[2]), lv[3], None)
    out.backward(shifted(grad))
    assert torch.equal(out.detach(), out0)
    for nm, x, g_ in zip(NAMES, lv, g0):
        assert _trelerr(x.grad, g_) <= 1e-5, nm
    # and the C-ABI itself reports it instead of faulting
    a = lib.ForwardArgs()
    a.shape = lib.Shape(1, 64, 48, 64, 8, 8, 8)
    a.stepsize, a.fadescale, a.fadeexp = s["stepsize"], 8.0, 8.0
    P = lambda x: ctypes.c_void_p(x.data_ptr())  # noqa: E731
    wsb = lib.workspace_bytes(1, 64, 48, 64, 8, 8, 8)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    rgba = torch.empty(1, 64, 48, 4, device="cuda")
    a.raypos, a.raydir, a.tminmax = P(s["raypos"]), P(s["raydir"]), P(s["tminmax"])
    a.primpos, a.primrot, a.primscale, a.tplate = P(s["primpos"]), P(s["primrot"]), P(s["primscale"]), P(s2["template"])
    a.rayrgba, a.workspace, a.workspace_bytes = P(rgba), P(ws), wsb
    assert lib.LIB.mvp_raymarch_forward(ctypes.byref(a), None) == -6          # MVP_ERR_ALIGN


def test_image_plane_outputs_equal_channels_last_op():
    """`mvpraymarch_planes` / the `Raymarcher` mirror: rayrgb [N,3,H,W] and rayalpha [N,1,H,W] straight from the render kernel,
    gradients straight into the backward == the channels-last op followed by the reference's permute + contiguous copies
    (models/raymarchers/mvpraymarcher.py:50-51), forward bit-identical."""
    from ava256_b200 import scene
    from ava256_b200.op import mvpraymarch_planes
    from ava256_b200.raymarcher import Raymarcher
    s = scene.make_scene(2, 160, 104, 1024, 8, alpha_mu=10.0, alpha_sigma=5.0, device="cuda")
    g_rgb = torch.randn(2, 3, 160, 104, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    g_alpha = torch.randn(2, 1, 160, 104, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    grad_nhwc = torch.cat([g_rgb, g_alpha], dim=1).permute(0, 2, 3, 1).contiguous()
    out, grads = _ours(s, grad_nhwc)
    lv = [s[n].detach().clone().requires_grad_(True) for n in NAMES]
    rgb, alpha = mvpraymarch_planes(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], (lv[0], lv[1], lv[2]), lv[3], None)
    assert rgb.shape == (2, 3, 160, 104) and alpha.shape == (2, 1, 160, 104) and rgb.is_contiguous() and alpha.is_contiguous()
    ref = out.permute(0, 3, 1, 2)
    assert torch.equal(rgb, ref[:, :3]) and torch.equal(alpha, ref[:, 3:4])
    ((rgb * g_rgb).sum() + (alpha * g_alpha).sum()).backward()
    for nm, x, g_ in zip(NAMES, lv, grads):
        assert _trelerr(x.grad, g_) <= 1e-5, nm
    # only one of the two outputs used downstream: the other gradient is None and must count as zero
    lv2 = [s[n].detach().clone().requires_grad_(True) for n in NAMES]
    rgb2, _ = mvpraymarch_planes(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], (lv2[0], lv2[1], lv2[2]), lv2[3], None)
    (rgb2 * g_rgb).sum().backward()
    g0 = torch.cat([g_rgb, torch.zeros_like(g_alpha)], dim=1).permute(0, 2, 3, 1).contiguous()
    _, grads0 = _ours(s, g0)
    for nm, x, g_ in zip(NAMES, lv2, grads0):
        assert _trelerr(x.grad, g_) <= 1e-5, nm
    # the module mirror
    rm = Raymarcher(scene.VOLRADIUS)
    decout = dict(primpos=s["primpos"], primrot=s["primrot"], primscale=s["primscale"], template=s["template"])
    with torch.no_grad():
        r1, a1, third, fourth = rm(s["raypos"], s["raydir"], s["tminmax"], decout)
        r2, a2, full, _ = Raymarcher(scene.VOLRADIUS, with_rgba=True)(s["raypos"], s["raydir"], s["tminmax"], decout)
    assert third is None and fourth is None and torch.equal(r1, rgb) and torch.equal(a1, alpha)
    assert torch.equal(r2, rgb) and torch.equal(a2, alpha) and torch.equal(full, ref)
