"""Shared test-input builders (seeded, CPU-generated so CPU and GPU runs see identical bytes)."""
import math

import numpy as np
import torch


def gradcheck_like_scene(N=2, H=13, W=13, k3=2, M=4, seed=1112, fadescale=6.5, fadeexp=7.5, alpha_gain=40.0, scale=2.2, dims=None):
    """Small scene in the style of the reference's gradcheck inputs
    (/root/reference/extensions/mvpraymarch/mvpraymarch.py:464-565): pinhole rays from z=-4, a k3^3 grid of
    randomly rotated slabs around the origin, softplus payload, random tminmax."""
    g = torch.Generator().manual_seed(seed)
    K = k3 ** 3
    focal = torch.tensor([[W * 4.0, W * 4.0]] * N)
    princpt = torch.tensor([[W * 0.5, H * 0.5]] * N)
    py, px = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    pc = torch.stack([px, py], dim=-1)[None].repeat(N, 1, 1, 1)
    rd = (pc - princpt[:, None, None, :]) / focal[:, None, None, :]
    rd = torch.cat([rd, torch.ones_like(rd[..., :1])], dim=-1)
    rd = rd / rd.norm(dim=-1, keepdim=True)
    rp = torch.tensor([0.0, 0.0, -4.0])[None, None, None, :].repeat(N, H, W, 1)
    max_len = 6.0
    stepsize = max_len / 15.386928
    tminmax = max_len * torch.arange(2, dtype=torch.float32)[None, None, None, :].repeat(N, H, W, 1) \
        + torch.rand(N, H, W, 2, generator=g)
    TD, TH, TW = dims if dims is not None else (M, M, M)
    tpl = torch.nn.functional.softplus(1.5 * (torch.randn(N, K, TD, TH, TW, 4, generator=g)
                                              - torch.tensor([0, 0, 0, 3.5]))) * torch.tensor([1, 1, 1, alpha_gain])
    lin = torch.linspace(-1.0, 1.0, k3)
    gz, gy, gx = torch.meshgrid(lin, lin, lin, indexing="ij")
    grid = torch.stack([gx, gy, gz], dim=-1).reshape(1, K, 3)
    pos = 0.3 * (grid + 0.1 * torch.randn(N, K, 3, generator=g))
    rv = torch.randn(N * K, 3, generator=g)
    th = torch.sqrt(1e-5 + (rv ** 2).sum(-1, keepdim=True))
    kx = rv / th
    Kx = torch.zeros(N * K, 3, 3)
    Kx[:, 0, 1], Kx[:, 0, 2], Kx[:, 1, 0] = -kx[:, 2], kx[:, 1], kx[:, 2]
    Kx[:, 1, 2], Kx[:, 2, 0], Kx[:, 2, 1] = -kx[:, 0], -kx[:, 1], kx[:, 0]
    rot = (torch.eye(3)[None] + torch.sin(th)[..., None] * Kx + (1 - torch.cos(th))[..., None] * (Kx @ Kx)).view(N, K, 3, 3)
    scale = scale * torch.exp(0.1 * torch.randn(N, K, 3, generator=g))
    return dict(raypos=rp.contiguous(), raydir=rd.contiguous(), tminmax=tminmax.contiguous(), stepsize=stepsize,
                primpos=pos.contiguous(), primrot=rot.contiguous(), primscale=scale.contiguous(),
                template=tpl.contiguous(), fadescale=fadescale, fadeexp=fadeexp)


def make_warp(N, K, WD, WH, WW, seed=77, amp=0.05):
    """Warp field like the reference gradcheck's (mvpraymarch.py:498-510): identity grid + small noise; channels-last
    [N,K,WD,WH,WW,3] with channel order (x, y, z) = (W, H, D) axes."""
    g = torch.Generator().manual_seed(seed)
    lz, ly, lx = (torch.linspace(-1.0, 1.0, n) if n > 1 else torch.zeros(1) for n in (WD, WH, WW))
    gz, gy, gx = torch.meshgrid(lz, ly, lx, indexing="ij")
    grid = torch.stack([gx, gy, gz], dim=-1)[None, None]
    return (grid + amp * torch.randn(N, K, WD, WH, WW, 3, generator=g)).contiguous()


def dense_scene(N=1, H=17, W=27, k3=7, M=4, dims=None, seed=5, warp=False, gain=(0.05, 1.0)):
    """k3^3 large slabs that overlap on every pixel: every 8x4 tile's slab list holds all of them (k3 = 7: 343 entries, past the
    256 of the fast render kernels; k3 >= 9: more than the reference's 512-entry cap).  K stays below the 2048-entry row bucket, so
    the lists are built from the TMA-staged bucket, not from the row-overflow scan.  Every ray crosses every slab, so a uniform
    alpha gain leaves either no ray or every ray saturated; here the gain is log-uniform per slab in `gain` * 343 / K and each
    ray ends at its own depth inside the slab cloud (tmax = tmin + 2.5 ... 6.5), which saturates a part of the rays.  H and W
    that are not multiples of 4 and 8 give partial tiles."""
    s = gradcheck_like_scene(N=N, H=H, W=W, k3=k3, M=M, seed=seed, alpha_gain=1.0, scale=1.1, dims=dims)
    K = k3 ** 3
    g = torch.Generator().manual_seed(seed + 1)
    lo, hi = (x * 343.0 / K for x in gain)
    s["template"][..., 3] *= (lo * (hi / lo) ** torch.rand(N, K, generator=g)).view(N, K, 1, 1, 1)
    s["tminmax"][..., 1] = s["tminmax"][..., 0] + 2.5 + 4.0 * torch.rand(N, H, W, generator=g)
    if warp:
        s["warp"] = make_warp(N, K, 3, 4, 5, seed=seed + 2, amp=0.05)
    return s


# Dense scenes whose tiles are all "heavy" (slab list > 256 entries: rendered by the 512-entry kernels), one per instantiation of
# those kernels (T = 8, 16, runtime dims; algo 1 = runtime dims with a warp field), each without and with the 512-entry cap hit.
DENSE_CASES = {
    "t8": lambda k3: dense_scene(N=2, k3=k3, M=8, seed=5),
    "t16": lambda k3: dense_scene(N=1, H=14, W=19, k3=k3, M=16, seed=6),
    "noncubic": lambda k3: dense_scene(N=2, H=13, W=21, k3=k3, dims=(3, 5, 4), seed=7),
    "warp": lambda k3: dense_scene(N=2, H=18, W=22, k3=k3, M=4, seed=8, warp=True),
}
DENSE_K3 = {"uncapped": 7, "capped": 9}


def build_dense_case(name, cap):
    s = DENSE_CASES[name](DENSE_K3[cap])
    g = torch.Generator().manual_seed(4243)
    return s, torch.randn(*s["raypos"].shape[:3], 4, generator=g)


ABI_GRAD_NAMES = ("primpos", "primrot", "primscale", "template", "warp")


def abi_raymarch(s, grad=None, fwd_flags=0, order=None, planes=False, camera=None, shared=False, keep=None, clear_in_forward=False):
    """Forward (+ backward when `grad` is given) of scene `s` (CUDA tensors) straight through the C-ABI.  camera =
    (viewpos, viewrot, focal, princpt, volradius, H, W): rays generated in the kernels, s's ray tensors are not passed.
    The gradient buffers start as NaN; the backward zero-fills them (MVP_FLAG_ZERO_GRADS), or, with clear_in_forward, the
    forward's render kernel does (clear_grad_*) and the backward runs without the flag, as the op does.
    Returns (rayrgba, raysat, grads or None, (heavy tiles of the forward, of the backward)); when `keep` is a dict it receives
    the workspace ("workspace") and rayaux ("rayaux")."""
    import ctypes
    from ava256_b200 import lib
    P = lambda x: None if x is None else ctypes.c_void_p(x.data_ptr())  # noqa: E731
    K = s["primpos"].shape[1]
    if camera is not None:
        N, H, W = camera[0].shape[0], camera[5], camera[6]
        cam = lib.Camera(P(camera[0]), P(camera[1]), P(camera[2]), P(camera[3]), float(camera[4]), 0)
        rays = (None, None, None)
    else:
        N, H, W = s["raypos"].shape[:3]
        cam = lib.Camera()
        rays = (s["raypos"], s["raydir"], s["tminmax"])
    TD, TH, TW = s["template"].shape[2:5]
    shape = lib.Shape(N, H, W, K, TD, TH, TW)
    wsb = lib.workspace_bytes(N, H, W, K, TD, TH, TW)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    hoff = lib.LIB.mvp_debug_heavy_offset(ctypes.byref(shape))
    heavy = lambda: int(ws[hoff:hoff + 4].view(torch.int32).item())  # noqa: E731
    warp = s.get("warp")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    sh = lib.FLAG_SHARED_PRIMS if shared else 0
    rgba = torch.full((N, H, W, 4), float("nan"), device="cuda")
    rgb_p = torch.full((N, 3, H, W), float("nan"), device="cuda") if planes else None
    alpha_p = torch.full((N, 1, H, W), float("nan"), device="cuda") if planes else None
    rsat = torch.empty(N, H, W, 3, device="cuda") if grad is not None else None
    raux = torch.empty(N, H, W, 4, dtype=torch.int32, device="cuda") if grad is not None else None
    if keep is not None:
        keep["workspace"], keep["rayaux"] = ws, raux
    gs = None
    if grad is not None:
        gs = [torch.full_like(s[n], float("nan")) for n in ABI_GRAD_NAMES[:4]] + \
             ([torch.full_like(warp, float("nan"))] if warp is not None else [])
    a = lib.ForwardArgs()
    a.shape, a.stepsize, a.fadescale, a.fadeexp = shape, s["stepsize"], s.get("fadescale", 8.0), s.get("fadeexp", 8.0)
    a.flags = fwd_flags | sh
    a.raypos, a.raydir, a.tminmax = (P(x) for x in rays)
    a.camera = cam
    a.primpos, a.primrot, a.primscale, a.tplate = P(s["primpos"]), P(s["primrot"]), P(s["primscale"]), P(s["template"])
    a.rayrgba, a.raysat, a.rayaux = (None if planes else P(rgba)), P(rsat), P(raux)
    a.rayrgb_nchw, a.rayalpha_nchw = P(rgb_p), P(alpha_p)
    a.order = P(order)
    a.workspace, a.workspace_bytes = P(ws), wsb
    if warp is not None:
        a.algo, a.warp = 1, P(warp)
        a.WD, a.WH, a.WW = warp.shape[2:5]
    if clear_in_forward:
        assert gs is not None, "the forward clears the gradient buffers of a backward"
        a.clear_grad_primpos, a.clear_grad_primrot, a.clear_grad_primscale, a.clear_grad_tplate = (P(g) for g in gs[:4])
        a.clear_grad_warp = P(gs[4]) if warp is not None else None
    lib.check(lib.LIB.mvp_raymarch_forward(ctypes.byref(a), st))
    hf = heavy()
    if planes:
        rgba = torch.cat([rgb_p, alpha_p], dim=1).permute(0, 2, 3, 1).contiguous()
    if grad is None:
        torch.cuda.synchronize()
        return rgba, None, None, (hf, 0)
    b = lib.BackwardArgs()
    b.shape, b.stepsize, b.fadescale, b.fadeexp = a.shape, a.stepsize, a.fadescale, a.fadeexp
    b.flags = lib.FLAG_ACCEL_VALID | (0 if clear_in_forward else lib.FLAG_ZERO_GRADS) | sh
    b.raypos, b.raydir, b.tminmax = a.raypos, a.raydir, a.tminmax
    b.camera = cam
    b.primpos, b.primrot, b.primscale, b.tplate = a.primpos, a.primrot, a.primscale, a.tplate
    if planes:
        gp = grad.permute(0, 3, 1, 2)
        g_rgb, g_alpha = gp[:, :3].contiguous(), gp[:, 3:4].contiguous()
        b.grad_rayrgb_nchw, b.grad_rayalpha_nchw = P(g_rgb), P(g_alpha)
    else:
        b.grad_rayrgba = P(grad)
    b.raysat, b.rayaux = P(rsat), P(raux)
    b.grad_primpos, b.grad_primrot, b.grad_primscale, b.grad_tplate = (P(g) for g in gs[:4])
    b.order = a.order
    b.workspace, b.workspace_bytes = P(ws), wsb
    if warp is not None:
        b.algo, b.warp, b.grad_warp = 1, P(warp), P(gs[4])
        b.WD, b.WH, b.WW = a.WD, a.WH, a.WW
    lib.check(lib.LIB.mvp_raymarch_backward(ctypes.byref(b), st))
    hb = heavy()
    torch.cuda.synchronize()
    return rgba, rsat, gs, (hf, hb)


def scene_args_np(s, dtype=np.float32):
    """(positional args for oracle.forward, kwargs)."""
    a = [s["raypos"].numpy().astype(dtype), s["raydir"].numpy().astype(dtype), float(s["stepsize"]),
         s["tminmax"].numpy().astype(dtype), s["primpos"].numpy().astype(dtype), s["primrot"].numpy().astype(dtype),
         s["primscale"].numpy().astype(dtype), s["template"].numpy().astype(dtype)]
    kw = dict(fadescale=float(s.get("fadescale", 8.0)), fadeexp=float(s.get("fadeexp", 8.0)))
    if s.get("warp") is not None:
        kw["warp"] = s["warp"].numpy().astype(dtype)
    return a, kw


def relerr(a, b):
    """max|a-b| / max|b| -- the parity measure of SURVEY.md section 8d (the reference's own report format)."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


# ----------------------------------------------------------------------------------------------------------
# Named, seeded parity cases (inputs are regenerated from seeds; tests/golden/*.npz hold reference OUTPUTS)
# ----------------------------------------------------------------------------------------------------------
def _head_case(n_views, H, W, K, T, seed=1112, view_offset=0, alpha_mu=6.0, alpha_sigma=6.0, stepsize=None):
    import sys, os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    from ava256_b200 import scene
    s = scene.make_scene(n_views, H, W, K, T, seed=seed, view_offset=view_offset, alpha_mu=alpha_mu,
                         alpha_sigma=alpha_sigma, share_primitives=False)
    if stepsize is not None:
        s["stepsize"] = stepsize
    s["fadescale"], s["fadeexp"] = 8.0, 8.0
    return s


CASES = {
    # gradcheck-style (mvpraymarch.py:434-440 shapes scaled down), fade 6.5/7.5 like the reference's __main__ (:748-774)
    "gradcheck_small": lambda: gradcheck_like_scene(N=2, H=24, W=20, k3=3, M=6, seed=1112, alpha_gain=8.0),
    # odd image size (partial tiles in x and y), K not a power of two (rotated DFS order)
    "gradcheck_ragged": lambda: gradcheck_like_scene(N=1, H=13, W=19, k3=3, M=4, seed=7, alpha_gain=8.0),
    # head scene, C1-like but small: pinhole dome cameras, UV-grid slabs on an ellipsoid
    "head_small": lambda: _head_case(2, 64, 42, 64, 8, stepsize=1.0 / 64, alpha_mu=1.0, alpha_sigma=2.0),
    # 125 large overlapping slabs: every tile sees > 96 candidates; the lists stay below the fast kernels' 256 entries (the
    # 512-entry kernels: DENSE_CASES, tests/test_gpu_heavy_tiles.py)
    "many_overlaps": lambda: gradcheck_like_scene(N=1, H=12, W=20, k3=5, M=4, seed=3, alpha_gain=0.4, scale=1.1),
    # non-cubic payload (runtime-stride sampler path) incl. a 1-voxel axis
    "noncubic": lambda: gradcheck_like_scene(N=1, H=14, W=17, k3=2, seed=21, alpha_gain=30.0, dims=(3, 1, 5)),
    # image smaller than one 8x4 tile, a single slab
    "tiny": lambda: gradcheck_like_scene(N=2, H=3, W=5, k3=1, M=2, seed=5, alpha_gain=15.0, scale=1.0),
    # algo 1: warp field (PrimSamplerTW<true>); large noise so warped positions leave the slab (zero padding)
    "warp_small": lambda: dict(gradcheck_like_scene(N=2, H=20, W=18, k3=2, M=6, seed=31, alpha_gain=60.0),
                               warp=make_warp(2, 8, 3, 4, 5, seed=5, amp=0.12)),
    "warp_head": lambda: dict(_head_case(1, 48, 32, 64, 8, stepsize=1.0 / 32, alpha_mu=2.0, alpha_sigma=2.0),
                              warp=make_warp(1, 64, 4, 4, 4, seed=9, amp=0.05)),
    # 18 views in one launch: above MVP_CTA_ORDER_MAXVIEWS (16), i.e. the large-launch forms of the accel build (warp-per-row
    # bucket kernel, plain grid order); every other case runs the small-launch forms
    "many_views": lambda: gradcheck_like_scene(N=18, H=9, W=11, k3=2, M=3, seed=13, alpha_gain=20.0),
    "head_t16": lambda: _head_case(1, 48, 32, 16, 16, stepsize=1.0 / 32, view_offset=11, alpha_mu=0.5, alpha_sigma=1.0),
}


def build_case(name):
    s = CASES[name]()
    g = torch.Generator().manual_seed(4242)
    grad = torch.randn(*s["raypos"].shape[:3], 4, generator=g)
    return s, grad


# ----------------------------------------------------------------------------------------------------------
# Scenes compared with the reference CUDA extension at sizes whose outputs are too large to store whole
# (tests/golden/scale_*.npz hold a sample of the reference's outputs: tests/golden/make_scale_golden.py)
# ----------------------------------------------------------------------------------------------------------
def scale_case(name, device="cuda"):
    """(scene dict on `device`, grad_rayrgba on `device`) of a named large case; same bytes on every run."""
    from ava256_b200 import scene
    if name == "head_256x168":            # mid-size head scene, generated on the host
        s = scene.make_scene(2, 256, 168, 1024, 8, alpha_mu=3.0, alpha_sigma=3.0, share_primitives=False)
        grad = torch.randn(2, 256, 168, 4, generator=torch.Generator().manual_seed(99))
        return {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in s.items()}, grad.to(device)
    if name == "c2":                      # BASELINE.json config 2: 4 views 512x334, K=4096, 16^3
        s = scene.make_scene(4, 512, 334, 4096, 16, alpha_mu=17.0, alpha_sigma=6.0, device=device)
        return s, torch.randn(4, 512, 334, 4, device=device, generator=torch.Generator(device=device).manual_seed(5))
    if name in ("c3_view0", "c3_view78"):  # two views of the bench scene (1024x667, K=16384, 8^3, alpha 17/6)
        off = int(name[len("c3_view"):])
        s = scene.make_scene(2, 1024, 667, 16384, 8, view_offset=off, alpha_mu=17.0, alpha_sigma=6.0, device=device)
        return s, torch.randn(2, 1024, 667, 4, device=device, generator=torch.Generator(device=device).manual_seed(6 + off))
    raise KeyError(name)


SCALE_CASES = ("head_256x168", "c2", "c3_view0", "c3_view78")
GOLDEN_TOP, GOLDEN_UNIFORM = 256, 1024


def sample_for_golden(name, x, seed):
    """A fixed sample of tensor `x` for a golden file: its GOLDEN_TOP largest-magnitude entries plus GOLDEN_UNIFORM seeded
    uniform ones (flat indices and values), and the whole tensor's max|x| and sum|x|, the denominators of the checks."""
    f = x.detach().reshape(-1).float()
    top = torch.topk(f.abs(), min(GOLDEN_TOP, f.numel())).indices.cpu()
    uni = torch.randint(f.numel(), (GOLDEN_UNIFORM,), generator=torch.Generator().manual_seed(seed))
    idx = torch.unique(torch.cat([top, uni])).to(torch.int64)
    return {name + "__idx": idx.numpy().astype(np.int32), name + "__val": f[idx.to(f.device)].cpu().numpy(),
            name + "__numel": np.int64(f.numel()), name + "__maxabs": np.float64(f.abs().max()),
            name + "__l1": np.float64(f.double().abs().sum())}


def sampled_relerr(gold, name, x):
    """(max|x - ref| over the sampled entries / max|ref| over the whole reference tensor,
        |sum|x| - sum|ref|| / sum|ref| over all entries) of tensor `x` against the sample `name` in `gold`."""
    f = x.detach().reshape(-1).float()
    assert f.numel() == int(gold[name + "__numel"]), name
    idx = torch.from_numpy(gold[name + "__idx"].astype(np.int64)).to(f.device)
    ref = torch.from_numpy(gold[name + "__val"]).to(f.device)
    d = float((f[idx] - ref).abs().max()) / max(float(gold[name + "__maxabs"]), 1e-30)
    l1 = float(gold[name + "__l1"])
    return d, abs(float(f.double().abs().sum()) - l1) / max(l1, 1e-30)


def _reductions(x, group):
    """Whole-tensor reductions of a golden tensor that together touch every entry: for an image [N,H,W,C] (group None) the sum
    and the max|.| of every (row, channel) and (column, channel); for a per-slab tensor [N,K,...] the sum and max|.| over every
    group of `group` consecutive slabs of a view.  (name suffix -> (sums, maxabs, entries per reduction))"""
    x = x.detach().float()
    if group is None:
        return {"rows": (x.double().sum(2), x.abs().amax(2), x.shape[2]),
                "cols": (x.double().sum(1), x.abs().amax(1), x.shape[1])}
    n, k = x.shape[:2]
    f = x.reshape(n, k, -1)
    pad = (-k) % group
    if pad:
        f = torch.cat([f, f.new_zeros(n, pad, f.shape[2])], dim=1)
    g = f.reshape(n, -1, group * f.shape[2])
    return {"groups": (g.double().sum(2), g.abs().amax(2), g.shape[2])}


def reductions_for_golden(name, x, group=None):
    """The reductions of `x` (see _reductions) for a golden file; `group` slabs per reduction, None for an image."""
    rec = {name + "__group": np.int64(0 if group is None else group)}
    for tag, (sums, maxabs, _) in _reductions(x, group).items():
        rec["%s__%s_sum" % (name, tag)] = sums.float().cpu().numpy()
        rec["%s__%s_max" % (name, tag)] = maxabs.cpu().numpy()
    return rec


def reductions_relerr(gold, name, x):
    """Largest deviation of the reductions of `x` from the stored ones, in units that an element-wise gate of
    max|x - ref| <= tol * max|ref| bounds by tol: |d max| / max|ref| and |d sum| / (entries * max|ref|)."""
    ref_max = max(float(gold[name + "__maxabs"]), 1e-30)
    worst = 0.0
    group = int(gold[name + "__group"]) or None
    for tag, (sums, maxabs, m) in _reductions(x, group).items():
        rs = torch.from_numpy(gold["%s__%s_sum" % (name, tag)]).to(sums.device).double()
        rm = torch.from_numpy(gold["%s__%s_max" % (name, tag)]).to(maxabs.device)
        assert rs.shape == sums.shape and rm.shape == maxabs.shape, (name, tag)
        worst = max(worst, float((maxabs - rm).abs().max()) / ref_max, float((sums - rs).abs().max()) / (m * ref_max))
    return worst


EDGE_KINDS = ("zero_scale", "rays_miss_volume", "large_step", "tiny_step")


def edge_scene(kind):
    s = gradcheck_like_scene(N=1, H=12, W=16, k3=2, M=4, seed=11, alpha_gain=30.0)
    if kind == "zero_scale":
        # SURVEY.md "input-distribution caveat": a decoder that skipped its warm-up feeds primscale = 0 (infinite slabs)
        s["primscale"][0, 1] = 0.0
        s["primscale"][0, 5, 2] = 0.0
    elif kind == "rays_miss_volume":
        # tmin > tmax for half of the rays (compute_raydirs gives that for rays missing the unit cube)
        s["tminmax"][0, :, :8, 0] = 9.0
        s["tminmax"][0, :, :8, 1] = 8.0
    elif kind == "large_step":
        s["stepsize"] = 1.7
    elif kind == "tiny_step":
        s["stepsize"] = 6.0 / 400.0
        s["template"][..., 3] *= 0.05
    return s
