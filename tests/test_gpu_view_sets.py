"""GPU tests of per-view primitive sets (`pytest -m gpu`): S subjects' primitives [S,K,...] rendered over N views in one launch,
view n from set view_set[n] (`op.mvpraymarch_sets`, `mvpraymarch_camera(..., view_set=)`, `Raymarcher(..., view_set=)`).

Reference of every check: the per-view form -- each set copied to its views (`x[view_set]`), the plain op, and each set's
gradient the sum of its views' gradients (`payload.sum_views`).  fp32: images bit-identical, gradients within TOL of max|.| (the
order of the fp32 atomics), a set no view shows exactly zero.  A bf16 template with fp32 accumulation: the same against the
per-view form on the fp32 widening, the template's gradient that fp32 sum rounded once (autograd casts it to bf16).  A bf16
template with bf16 accumulation: within the dense-scene gates of tests/test_emul_bf16_payload.py of the fp32-accumulated result."""
import gc

import pytest
import torch

from tests.test_emul_bf16_payload import GATE_DENSE_L1, GATE_DENSE_MAX
from tests.test_gpu_bf16_grad_f32 import check_rounded_once
from tests.test_gpu_bf16_payload import _relerr, _tgrad_errors
from tests.test_gpu_large_launch import _require_memory

pytestmark = pytest.mark.gpu

TOL = 1e-5
NAMES = ("primpos", "primrot", "primscale", "template", "warp")


def subjects(S, K, T, dev, seed=1112, alpha_mu=6.0, alpha_sigma=6.0, warp=False):
    """S distinct subjects' primitives as [S,K,...] CUDA tensors (+ a warp field [S,K,3,4,5,3] with warp=True)."""
    from ava256_b200 import scene
    prims = [scene.make_primitives(K, seed + 101 * i) for i in range(S)]
    out = {nm: torch.stack([p[j] for p in prims]).to(dev).contiguous() for j, nm in enumerate(NAMES[:3])}
    out["template"] = torch.stack([scene.make_payload(K, T, seed + 101 * i, alpha_mu, alpha_sigma, device=dev) for i in range(S)])
    if warp:
        from tests.helpers import make_warp
        out["warp"] = make_warp(S, K, 3, 4, 5, seed=seed).to(dev)
    return out


def views(N, H, W, dev):
    from ava256_b200 import scene
    rays = [t.to(dev) for t in scene.make_rays(N, H, W)]
    cams = [t.to(dev) for t in scene.make_cameras(N, H, W)]
    return rays, cams


def march(rays, prims, grad, view_set=None, cams=None, planes=False, camera_grad=False, retain=False, **kw):
    """Forward + backward through the public op: the sets form with view_set, else the plain per-view call.  Returns (image,
    {name: gradient}, {camera name: gradient})."""
    from ava256_b200 import scene
    from ava256_b200.op import mvpraymarch, mvpraymarch_camera, mvpraymarch_planes, mvpraymarch_sets
    leaves = {nm: prims[nm].detach().clone().requires_grad_(True) for nm in NAMES if nm in prims}
    cam_leaves = [c.detach().clone().requires_grad_(camera_grad) for c in cams] if cams is not None else None
    kw = dict(kw, algo=1 if "warp" in leaves else 0)
    prim = (leaves["primpos"], leaves["primrot"], leaves["primscale"])
    stepsize = 1.0 / scene.VOLRADIUS
    if cam_leaves is not None:
        H, W = rays[0].shape[1:3]
        out = mvpraymarch_camera(*cam_leaves, (W, H), scene.VOLRADIUS, stepsize, prim, leaves["template"], leaves.get("warp"),
                                 planes=planes, camera_grad=camera_grad, view_set=view_set, **kw)
    elif view_set is not None:
        out = mvpraymarch_sets(rays[0], rays[1], stepsize, rays[2], prim, leaves["template"], leaves.get("warp"), view_set,
                               planes=planes, **kw)
    else:
        out = (mvpraymarch_planes if planes else mvpraymarch)(rays[0], rays[1], stepsize, rays[2], prim, leaves["template"],
                                                              leaves.get("warp"), **kw)
    img = torch.cat([out[0], out[1]], dim=1).permute(0, 2, 3, 1) if planes else out
    img.backward(grad, retain_graph=retain)
    if retain:                      # a second backward through the same graph: the gradients double
        img.backward(grad)
    torch.cuda.synchronize()
    cg = {nm: c.grad for nm, c in zip(("viewpos", "viewrot", "focal", "princpt"), cam_leaves or []) if c.grad is not None}
    return img.detach(), {nm: x.grad for nm, x in leaves.items()}, cg


def per_view(prims, view_set):
    idx = torch.as_tensor(view_set, device=prims["primpos"].device)
    return {nm: x[idx].contiguous() for nm, x in prims.items()}


def set_sums(g_view, view_set, S):
    """Each set's gradient from the per-view ones: sum_views over its views (zero for a set no view shows)."""
    from ava256_b200.payload import sum_views
    idx = torch.as_tensor(view_set, device=g_view.device)
    return torch.stack([sum_views(g_view[idx == j].float()) if bool((idx == j).any()) else
                        torch.zeros(g_view.shape[1:], device=g_view.device) for j in range(S)])


def check_sets(view_set, S, ref, got, tol=TOL):
    (img_v, g_v, c_v), (img_s, g_s, c_s) = ref, got
    assert float(img_v[..., 3].max()) > 0.05
    assert torch.equal(img_s, img_v)
    for nm, gv in g_v.items():
        gs = g_s[nm]
        assert gs.shape[0] == S and gs.dtype == gv.dtype, nm
        want = set_sums(gv, view_set, S)
        for j in range(S):
            if j in list(view_set):
                assert _relerr(gs[j], want[j]) <= tol, (nm, j, _relerr(gs[j], want[j]))
            else:
                assert not bool(gs[j].any()), (nm, j)
    for nm in c_v:
        assert _relerr(c_s[nm], c_v[nm]) <= tol, nm


def _map(N, S, seed, unused=None):
    g = torch.Generator().manual_seed(seed)
    choices = [j for j in range(S) if j != unused]
    return [choices[int(i)] for i in torch.randint(len(choices), (N,), generator=g)]


# <= 16 views: the CTA-ordered launch and the parallel bucket kernel; > 16 views: grid order and the warp-per-row kernel
MAPS = {"5views": ([2, 0, 1, 0, 2], 3), "24views": (_map(24, 5, 1, unused=3), 5), "18views_one_set": ([0] * 18, 1)}


@pytest.mark.parametrize("usebvh", ["fixedorder", True])
@pytest.mark.parametrize("case", list(MAPS))
def test_view_sets_fp32(case, usebvh):
    view_set, S = MAPS[case]
    dev = torch.device("cuda")
    N, H, W = len(view_set), 96, 64
    rays, _ = views(N, H, W, dev)
    prims = subjects(S, 256, 8, dev)
    grad = torch.randn(N, H, W, 4, device=dev, generator=torch.Generator(device=dev).manual_seed(2))
    ref = march(rays, per_view(prims, view_set), grad, usebvh=usebvh)
    got = march(rays, prims, grad, view_set=view_set, usebvh=usebvh)
    check_sets(view_set, S, ref, got)
    # the same map as an int64 CUDA tensor and as an int32 CPU tensor
    for vs in (torch.tensor(view_set, device=dev), torch.tensor(view_set, dtype=torch.int32)):
        again = march(rays, prims, grad, view_set=vs, usebvh=usebvh)
        assert torch.equal(again[0], got[0])
        for nm in got[1]:
            assert _relerr(again[1][nm], got[1][nm]) <= TOL, nm


def test_view_sets_algo1_planes_retain_graph():
    view_set, S = [1, 0, 1, 2], 3
    dev = torch.device("cuda")
    N, H, W = len(view_set), 80, 56
    rays, _ = views(N, H, W, dev)
    prims = subjects(S, 256, 4, dev, warp=True)
    grad = torch.randn(N, H, W, 4, device=dev, generator=torch.Generator(device=dev).manual_seed(3))
    check_sets(view_set, S, march(rays, per_view(prims, view_set), grad), march(rays, prims, grad, view_set=view_set))
    check_sets(view_set, S, march(rays, per_view(prims, view_set), grad, planes=True, retain=True),
               march(rays, prims, grad, view_set=view_set, planes=True, retain=True))


def test_view_sets_camera_grad_and_frozen_template():
    """Camera form with camera gradients; then a frozen avatar (no primitive gradient: the rays-only backward) and a frozen
    template (no payload gradient)."""
    view_set, S = [0, 1, 1, 0, 1], 2
    dev = torch.device("cuda")
    N, H, W = len(view_set), 96, 64
    rays, cams = views(N, H, W, dev)
    prims = subjects(S, 256, 8, dev)
    grad = torch.randn(N, H, W, 4, device=dev, generator=torch.Generator(device=dev).manual_seed(4))
    ref = march(rays, per_view(prims, view_set), grad, cams=cams, camera_grad=True)
    got = march(rays, prims, grad, view_set=view_set, cams=cams, camera_grad=True)
    assert ref[2] and float(ref[2]["viewpos"].abs().max()) > 0
    check_sets(view_set, S, ref, got)
    from ava256_b200 import scene
    from ava256_b200.op import mvpraymarch_camera
    for frozen in (("primpos", "primrot", "primscale", "template"), ("template",)):
        out = {}
        for vs, pr in ((None, per_view(prims, view_set)), (view_set, prims)):
            cl = [c.clone().requires_grad_(True) for c in cams]
            lv = {nm: x.clone().requires_grad_(nm not in frozen) for nm, x in pr.items()}
            img = mvpraymarch_camera(*cl, (W, H), scene.VOLRADIUS, 1.0 / scene.VOLRADIUS, (lv["primpos"], lv["primrot"], lv["primscale"]),
                                     lv["template"], None, camera_grad=True, view_set=vs)
            img.backward(grad)
            out[vs is None] = (img.detach(), [c.grad for c in cl], {nm: x.grad for nm, x in lv.items()})
        assert torch.equal(out[True][0], out[False][0])
        for a, b in zip(out[True][1], out[False][1]):
            assert _relerr(b, a) <= TOL
        for nm, gv in out[True][2].items():
            gs = out[False][2][nm]
            assert (gv is None) == (nm in frozen) and (gs is None) == (nm in frozen), nm
            if gv is not None:
                assert _relerr(gs, set_sums(gv, view_set, S)) <= TOL, nm


def test_view_sets_raymarcher_module():
    from ava256_b200 import scene
    from ava256_b200.raymarcher import Raymarcher
    view_set, S = [1, 0, 1], 2
    dev = torch.device("cuda")
    N, H, W = 3, 64, 48
    rays, cams = views(N, H, W, dev)
    prims = subjects(S, 256, 8, dev)
    rm = Raymarcher(scene.VOLRADIUS)
    pv = per_view(prims, view_set)
    with torch.no_grad():
        a = rm(rays[0], rays[1], rays[2], pv)
        b = rm(rays[0], rays[1], rays[2], prims, view_set=view_set)
        ac = rm.forward_camera(*cams, (W, H), pv)
        bc = rm.forward_camera(*cams, (W, H), prims, view_set=view_set)
    assert float(a[1].max()) > 0.05 and float(ac[1].max()) > 0.05
    for x, y in zip(a[:2] + ac[:2], b[:2] + bc[:2]):
        assert torch.equal(x, y)


@pytest.mark.parametrize("case", ["5views", "24views"])
def test_view_sets_bf16_template(case):
    """bf16 template: with fp32 accumulation against the per-view form on the fp32 widening (template gradient rounded once);
    with bf16 accumulation within the dense gates of the fp32-accumulated result."""
    from ava256_b200.op import template_grad_dtype
    view_set, S = MAPS[case]
    dev = torch.device("cuda")
    N, H, W = len(view_set), 96, 64
    rays, _ = views(N, H, W, dev)
    prims = subjects(S, 256, 8, dev)
    prims["template"] = prims["template"].to(torch.bfloat16)
    p32 = dict(prims, template=prims["template"].float())
    grad = torch.randn(N, H, W, 4, device=dev, generator=torch.Generator(device=dev).manual_seed(5))
    img_v, g_v, _ = march(rays, per_view(p32, view_set), grad)
    with template_grad_dtype(torch.float32):
        img_f, g_f, _ = march(rays, prims, grad, view_set=view_set)
    assert torch.equal(img_f, img_v)
    for nm, gv in g_v.items():
        want = set_sums(gv, view_set, S)
        if nm == "template":
            for j in range(S):
                if j in view_set:
                    check_rounded_once(g_f[nm][j], want[j], nm)
        else:
            assert _relerr(g_f[nm], want) <= TOL, nm
    img_b, g_b, _ = march(rays, prims, grad, view_set=view_set)
    assert torch.equal(img_b, img_v)
    emax, el1 = _tgrad_errors(g_b["template"], g_f["template"])
    assert emax <= GATE_DENSE_MAX and el1 <= GATE_DENSE_L1, (emax, el1)
    for nm in ("primpos", "primrot", "primscale"):
        assert _relerr(g_b[nm], g_f[nm]) <= TOL, nm


def test_view_sets_host_map_errors():
    from ava256_b200.op import mvpraymarch_sets
    dev = torch.device("cuda")
    rays, _ = views(3, 32, 32, dev)
    prims = subjects(2, 256, 4, dev)
    args = (rays[0], rays[1], 1.0 / 256.0, rays[2], (prims["primpos"], prims["primrot"], prims["primscale"]), prims["template"], None)
    for vs, err in (([0, 2, 1], ValueError), ([0, -1, 1], ValueError), ([0, 1], ValueError), (torch.tensor([0, 1, 2]), ValueError),
                    (torch.tensor([0.0, 1.0, 1.0], device=dev), TypeError), (None, TypeError)):
        with pytest.raises(err):
            mvpraymarch_sets(*args, vs)
    four = subjects(4, 256, 4, dev)
    with pytest.raises(ValueError):            # S > N
        mvpraymarch_sets(rays[0], rays[1], 1.0 / 256.0, rays[2], (four["primpos"], four["primrot"], four["primscale"]),
                         four["template"], None, [0, 1, 2])


def test_view_sets_benchmark_scale():
    """4 subjects x 20 views at 1024x667, K = 16384, 8^3 (the benchmark's launch, grouped by subject) against expand_views + the
    per-view op + sum_views per subject."""
    from ava256_b200 import scene
    from ava256_b200.payload import expand_views, sum_views
    S, V, H, W, K, T = 4, 20, 1024, 667, 16384, 8
    N = S * V
    dev = torch.device("cuda")
    _require_memory(2 * 2 * N * K * T ** 3 * 16 + 8 * 2 ** 30, "4 x 20 views, per-view reference")
    rays, _ = views(N, H, W, dev)
    prims = subjects(S, K, T, dev, alpha_mu=17.0, alpha_sigma=6.0)
    view_set = [i // V for i in range(N)]
    grad = torch.randn(N, H, W, 4, device=dev, generator=torch.Generator(device=dev).manual_seed(6))
    with torch.no_grad():
        pv = {nm: torch.cat([expand_views(x[j], V) for j in range(S)]) for nm, x in prims.items()}
    img_v, g_v, _ = march(rays, pv, grad)
    del pv
    g_v = {nm: torch.stack([sum_views(g[j * V:(j + 1) * V]) for j in range(S)]) for nm, g in g_v.items()}
    gc.collect()
    torch.cuda.empty_cache()
    img_s, g_s, _ = march(rays, prims, grad, view_set=torch.tensor(view_set, dtype=torch.int32, device=dev))
    assert float(img_v[..., 3].max()) > 0.5
    assert torch.equal(img_s, img_v)
    for nm in g_v:
        assert _relerr(g_s[nm], g_v[nm]) <= TOL, (nm, _relerr(g_s[nm], g_v[nm]))
