"""GPU tests of deterministic primitive gradients (`pytest -m gpu`): `op.deterministic_grads()` / `deterministic=True`, the C-ABI's
mvp_raymarch_backward_deterministic.  Every primitive gradient is summed in 64-bit fixed point, so:
  * two runs give the same bits, the 80-view benchmark launch included;
  * permuting the views (shared primitives, view sets) permutes the images and leaves every gradient bit unchanged;
  * a heavy-tile scene (512-entry kernels) gives the same bits run after run;
  * every supported combination agrees with the default backward within TOL of max|.|, and the bf16 gradient is the fp32 one
    rounded once;
  * the reference goldens are met at the north-star gates."""
import gc

import pytest
import torch

from tests.test_gpu_large_launch import _require_memory
from tests.test_gpu_scale_parity import _trelerr, assert_parity_with_golden

pytestmark = pytest.mark.gpu

TOL = 1e-5
NAMES = ("primpos", "primrot", "primscale", "template")


def march(s, grad, det, grad_names=NAMES, planes=False, camera=None, pixels=None, view_set=None, **kw):
    """Forward + backward of scene s (scene.make_scene form, on the GPU) through the public op; returns (image, [gradients])."""
    from ava256_b200 import op, scene
    lv = {n: s[n].detach().requires_grad_(n in grad_names) for n in NAMES}     # no copy: the 80-view template is 10.7 GB
    prim = (lv["primpos"], lv["primrot"], lv["primscale"])
    with op.deterministic_grads(det):
        if camera is not None:
            H, W = s["raypos"].shape[1:3]
            out = op.mvpraymarch_camera(*camera, pixels if pixels is not None else (W, H), scene.VOLRADIUS, s["stepsize"], prim,
                                        lv["template"], None, planes=planes, view_set=view_set, **kw)
        elif view_set is not None:
            out = op.mvpraymarch_sets(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], prim, lv["template"], None, view_set,
                                      planes=planes, **kw)
        else:
            fn = op.mvpraymarch_planes if planes else op.mvpraymarch
            out = fn(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], prim, lv["template"], None, **kw)
    img = torch.cat([out[0], out[1]], dim=1).permute(0, 2, 3, 1) if planes else out
    img.backward(grad)
    torch.cuda.synchronize()
    return img.detach(), [lv[n].grad for n in NAMES]


def _scene(N=4, H=256, W=168, K=1024, T=8, share=False, seed=1112, **kw):
    from ava256_b200 import scene
    s = scene.make_scene(N, H, W, K, T, seed=seed, alpha_mu=3.0, alpha_sigma=3.0, device="cuda", **kw)
    if share:                       # one set [1,K,...] shared by all views (MVP_FLAG_SHARED_PRIMS)
        s = dict(s, **{n: s[n][:1].contiguous() for n in NAMES})
    g = torch.randn(N, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))
    return s, g


def _equal(a, b):
    return all((x is None and y is None) or torch.equal(x, y) for x, y in zip(a, b))


def test_bench_launch_twice_bit_identical_and_close_to_default():
    """The benchmark launch (80 views 1024x667, K = 16384, 8^3, per-view primitives) through the op, twice in one process."""
    from ava256_b200 import scene
    N, H, W, K, T = 80, 1024, 667, 16384, 8
    _require_memory(int(60e9), "80-view deterministic backward")
    s = scene.make_scene(N, H, W, K, T, alpha_mu=17.0, alpha_sigma=6.0, share_primitives=False, device="cuda")
    grad = torch.randn(N, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))
    torch.cuda.reset_peak_memory_stats()
    out1, g1 = march(s, grad, True)
    print("deterministic step peak memory: %.2f GB" % (torch.cuda.max_memory_allocated() / 1e9))
    out0, g0 = march(s, grad, False)
    assert torch.equal(out0, out1)
    for nm, x, y in zip(NAMES, g1, g0):
        assert bool(torch.isfinite(x).all()), nm
        assert _trelerr(x, y) <= TOL, (nm, _trelerr(x, y))
    del out0, g0
    gc.collect()
    torch.cuda.empty_cache()
    out2, g2 = march(s, grad, True)
    assert torch.equal(out1, out2)
    for nm, x, y in zip(NAMES, g1, g2):
        assert torch.equal(x, y), nm


def test_shared_primitives_views_permuted():
    s, grad = _scene(N=6, share=True)
    perm = torch.tensor([3, 0, 5, 1, 4, 2], device="cuda")
    sp = dict(s, raypos=s["raypos"][perm].contiguous(), raydir=s["raydir"][perm].contiguous(), tminmax=s["tminmax"][perm].contiguous())
    out, g = march(s, grad, True)
    outp, gp = march(sp, grad[perm].contiguous(), True)
    assert torch.equal(out[perm], outp)
    assert _equal(g, gp)


def test_view_sets_views_permuted_and_close_to_default():
    from tests.test_gpu_view_sets import subjects
    s, grad = _scene(N=6)
    prims = subjects(2, 1024, 8, "cuda", alpha_mu=3.0, alpha_sigma=3.0)
    s = dict(s, **prims)
    vs = torch.tensor([0, 1, 1, 0, 1, 0], device="cuda")
    perm = torch.tensor([5, 2, 0, 4, 1, 3], device="cuda")
    sp = dict(s, raypos=s["raypos"][perm].contiguous(), raydir=s["raydir"][perm].contiguous(), tminmax=s["tminmax"][perm].contiguous())
    out, g = march(s, grad, True, view_set=vs)
    outp, gp = march(sp, grad[perm].contiguous(), True, view_set=vs[perm])
    assert torch.equal(out[perm], outp)
    assert _equal(g, gp)
    out0, g0 = march(s, grad, False, view_set=vs)
    assert torch.equal(out, out0)
    assert all(_trelerr(x, y) <= TOL for x, y in zip(g, g0))


def test_heavy_tiles_bit_identical_and_close_to_default():
    """A dense scene whose lists overflow the fast kernels (the 512-entry kernels take them), as in tests/test_gpu_heavy_tiles.py."""
    from tests.helpers import build_dense_case
    s, grad = build_dense_case("t8", "capped")
    s = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in s.items()}
    grad = grad.cuda()
    out1, g1 = march(s, grad, True)
    out2, g2 = march(s, grad, True)
    out0, g0 = march(s, grad, False)
    assert torch.equal(out1, out2) and torch.equal(out1, out0)
    assert _equal(g1, g2)
    assert all(_trelerr(x, y) <= TOL for x, y in zip(g1, g0))


COMBOS = {
    "per_view": {},
    "shared": {"share": True},
    "morton": {"kw": {"usebvh": True}},
    "planes": {"planes": True},
    "camera": {"camera": True},
    "pixels": {"camera": True, "pixels": True},
    "no_payload": {"grad_names": NAMES[:3]},
    "pixels_sets": {"camera": True, "pixels": True, "sets": True},
}


@pytest.mark.parametrize("combo", list(COMBOS))
def test_supported_combination_close_to_default(combo):
    from ava256_b200 import scene
    c = COMBOS[combo]
    s, grad = _scene(N=4, share=c.get("share", False))
    opts = dict(c.get("kw", {}), planes=c.get("planes", False), grad_names=c.get("grad_names", NAMES))
    if c.get("camera"):
        N, H, W = s["raypos"].shape[:3]
        opts["camera"] = [t.cuda() for t in scene.make_cameras(N, H, W)]
        if c.get("pixels"):
            ys, xs = torch.meshgrid(torch.arange(H, device="cuda"), torch.arange(W, device="cuda"), indexing="ij")
            opts["pixels"] = torch.stack([xs, ys], -1).float().expand(N, H, W, 2).contiguous()
    if c.get("sets"):
        opts["view_set"] = torch.tensor([0, 1, 0, 1], device="cuda")
        s = dict(s, **{n: s[n][:2].contiguous() for n in NAMES})
    out1, g1 = march(s, grad, True, **opts)
    out2, g2 = march(s, grad, True, **opts)
    out0, g0 = march(s, grad, False, **opts)
    assert torch.equal(out1, out0) and torch.equal(out1, out2)
    assert _equal(g1, g2)
    for nm, x, y in zip(NAMES, g1, g0):
        if nm not in opts["grad_names"]:
            assert x is None and y is None
            continue
        assert bool(torch.isfinite(x).all()) and _trelerr(x, y) <= TOL, (combo, nm, _trelerr(x, y))


def test_bf16_template_both_gradient_dtypes():
    """bf16 template: with template_grad_dtype=float32 the transform gradients within TOL of the default path's and the template's
    within one bf16 rounding (autograd casts both to bf16); the bf16 gradient is the deterministic fp32 result rounded once (bit for
    bit what autograd's cast makes of it)."""
    from ava256_b200 import op
    s, grad = _scene(N=4)
    sb = dict(s, template=s["template"].to(torch.bfloat16))
    with op.template_grad_dtype(torch.float32):
        out32, g32 = march(sb, grad, True)
        out0, g0 = march(sb, grad, False)
    outb, gb = march(sb, grad, True)
    assert torch.equal(out32, out0) and torch.equal(out32, outb)
    assert all(_trelerr(x, y) <= TOL for x, y in zip(g32[:3], g0[:3]))
    # autograd hands both template gradients over as bf16 roundings of their fp32 sums: equal to within one bf16 step
    assert g32[3].dtype == torch.bfloat16 and _trelerr(g32[3].float(), g0[3].float()) <= 2.0 ** -7
    assert gb[3].dtype == torch.bfloat16 and torch.equal(gb[3], g32[3])
    assert _equal(gb[:3], g32[:3])


@pytest.mark.parametrize("name", ["head_256x168", "c3_view0"])
def test_reference_goldens_at_north_star_gates(name):
    from tests.helpers import scale_case
    s, grad = scale_case(name)
    out, g = march(s, grad, True)
    assert_parity_with_golden(out, g, name)
