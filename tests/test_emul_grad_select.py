"""Reduced gradient sets of the raymarch backward (MVP_FLAG_NO_TPLATE_GRAD, MVP_FLAG_RAY_GRADS_ONLY) on the emulated product kernels.

The "no payload" set drops the payload-gradient scatter and the "rays only" set also the transform-gradient sums; everything
they still compute is the full backward's arithmetic.  The blocks run one after the other here (MVP_EMUL_THREADS=1) with a fixed
lane order, and the full backward is then deterministic: two runs agree bit for bit.  What a reduced set changes is where the
emulation switches between the lanes and warps of a block, which it does at every warp collective:
  * algo 1 without a payload gradient drops no collective (its lanes already left short batches early and its warp-field
    gradient is plain atomics), so its transform and ray gradients are bit-identical to the full backward's (checked);
  * algo 0 without a payload gradient drops the merge's match/shuffle collectives, and "rays only" also the transform butterfly.
    Both sums then land in another order: the transform gradients (global atomics from the warps of a block) and the ray gradients
    (shared-memory atomics of the lanes that share an owner).  On gradcheck_small about 3 % of the ray values differ, in the last
    bits; head_small about 21 %.  These are checked within TOL of max|.|, and the images bit for bit.
Buffers outside a set may be NULL; when they are not, they are neither read nor written by the forward's clear or by the
backward, which sentinel-filled buffers show.

A bf16 template goes through as in tests/test_emul_bf16_payload.py: uint16 bit patterns in fp32-typed words [..., 2]."""
import ctypes

import numpy as np
import pytest
import torch

from tests.helpers import CASES, DENSE_CASES, DENSE_K3, build_case, build_dense_case, relerr, scene_args_np

SENTINEL = 1234.5
TOL = 1e-6
TRANSFORMS = slice(0, 3)


@pytest.fixture()
def kernels(monkeypatch):
    from tests.emul import kernels as k
    monkeypatch.setenv("MVP_EMUL_THREADS", "1")        # blocks in launch order: the atomics' order is fixed
    k.use_variant(())
    L = k.load()
    L.mvp_raymarch_backward_rays.restype = ctypes.c_int
    L.mvp_raymarch_backward_rays.argtypes = [ctypes.c_void_p] * 5
    k.set_lane_order("forward")
    yield k
    k.set_lane_order("forward")
    loaded, rebuilt = ctypes.c_int(), ctypes.c_int()            # reset the saved-list counters the dense scenes leave behind
    L.mvp_emul_saved_list_tiles(ctypes.byref(loaded), ctypes.byref(rebuilt))


def _flags(gset):
    from ava256_b200 import lib
    return {"all": 0, "no_payload": lib.FLAG_NO_TPLATE_GRAD, "rays_only": lib.FLAG_RAY_GRADS_ONLY}[gset]


def _arr16(shape, value):
    """float32 array filled with value whose data pointer is 16-byte aligned."""
    n = int(np.prod(shape))
    raw = np.empty(n + 4, np.float32)
    off = (-raw.ctypes.data // 4) % 4
    out = raw[off:off + n].reshape(shape)
    out[...] = value
    return out


def march(kernels, a, kw, grad, gset="all", rays=False, tflags=0, flags=0, unused="null", init="clear", order=None):
    """Emulated forward + backward of the scene (scene_args_np form; a[7] may be a bf16 template as fp32-typed words) computing the
    gradient set gset, with mvp_raymarch_backward_rays when rays.  The requested gradient buffers start NaN and are zeroed by the
    forward's clear (init="clear") or by MVP_FLAG_ZERO_GRADS (init="zero").  The others are NULL (unused="null") or
    sentinel-filled and handed to both calls (unused="sentinel").  tflags go to both calls (template type), flags too (e.g.
    MVP_FLAG_SHARED_PRIMS).  Returns (rayrgba, [primpos, primrot, primscale, template, warp] gradients (None: not requested),
    ray gradients or None, the sentinel buffers); the heavy-tile counts of forward and backward are left in march.last_heavy."""
    from ava256_b200 import lib
    L = kernels.load()
    P = lambda x: None if x is None else ctypes.c_void_p(x.ctypes.data)  # noqa: E731
    raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template = a
    warp = kw.get("warp")
    N, H, W = raypos.shape[:3]
    K, (TD, TH, TW) = primpos.shape[1], template.shape[2:5]
    gwords = 4 if (tflags & lib.FLAG_GRAD_TPLATE_F32) else template.shape[-1]
    shapes = [primpos.shape, primrot.shape, primscale.shape, template.shape[:-1] + (gwords,)] + ([warp.shape] if warp is not None else [])
    want = [gset != "rays_only"] * 3 + [gset == "all"] * (len(shapes) - 3)
    bufs, sentinels = [], []
    for sh, w in zip(shapes, want):
        if w:
            bufs.append(_arr16(sh, np.nan))
        elif unused == "sentinel":
            bufs.append(_arr16(sh, SENTINEL))
            sentinels.append(bufs[-1])
        else:
            bufs.append(None)
    shape = lib.Shape(N, H, W, K, TD, TH, TW)
    wsb = L.mvp_workspace_bytes(ctypes.byref(shape))
    raw = np.zeros(wsb + 256, np.uint8)
    ws = raw[(-raw.ctypes.data) % 256:][:wsb]
    rayrgba, raysat = np.full((N, H, W, 4), np.nan, np.float32), np.full((N, H, W, 3), np.nan, np.float32)
    rayaux = np.zeros((N, H, W, 4), np.int32)
    fl = flags | tflags | _flags(gset)
    fa = lib.ForwardArgs()
    fa.shape, fa.stepsize, fa.fadescale, fa.fadeexp, fa.flags = shape, float(stepsize), kw["fadescale"], kw["fadeexp"], fl
    fa.raypos, fa.raydir, fa.tminmax = P(raypos), P(raydir), P(tminmax)
    fa.primpos, fa.primrot, fa.primscale, fa.tplate = P(primpos), P(primrot), P(primscale), P(template)
    fa.rayrgba, fa.raysat, fa.rayaux = P(rayrgba), P(raysat), P(rayaux)
    fa.workspace, fa.workspace_bytes = P(ws), wsb
    if order is not None:
        fa.order = P(order)
    if warp is not None:
        fa.algo, fa.warp = 1, P(warp)
        fa.WD, fa.WH, fa.WW = warp.shape[2:5]
    if init == "clear" or unused == "sentinel":
        clr = [b if (w and init == "clear") or not w else None for b, w in zip(bufs, want)]
        fa.clear_grad_primpos, fa.clear_grad_primrot, fa.clear_grad_primscale, fa.clear_grad_tplate = (P(b) for b in clr[:4])
        fa.clear_grad_warp = P(clr[4]) if warp is not None else None
    assert L.mvp_raymarch_forward(ctypes.byref(fa), None) == 0
    hoff = L.mvp_debug_heavy_offset(ctypes.byref(shape))
    heavy = lambda: int(ws[hoff:hoff + 4].view(np.int32)[0])  # noqa: E731
    hf = heavy()
    ba = lib.BackwardArgs()
    ba.shape, ba.stepsize, ba.fadescale, ba.fadeexp = shape, fa.stepsize, fa.fadescale, fa.fadeexp
    ba.flags = lib.FLAG_ACCEL_VALID | fl | (lib.FLAG_ZERO_GRADS if init == "zero" else 0)
    ba.raypos, ba.raydir, ba.tminmax = fa.raypos, fa.raydir, fa.tminmax
    ba.primpos, ba.primrot, ba.primscale, ba.tplate = fa.primpos, fa.primrot, fa.primscale, fa.tplate
    g = np.ascontiguousarray(grad, np.float32)
    ba.grad_rayrgba, ba.raysat, ba.rayaux = P(g), P(raysat), P(rayaux)
    ba.grad_primpos, ba.grad_primrot, ba.grad_primscale, ba.grad_tplate = (P(b) for b in bufs[:4])
    ba.workspace, ba.workspace_bytes, ba.order = fa.workspace, wsb, fa.order
    if warp is not None:
        ba.algo, ba.warp, ba.grad_warp = 1, fa.warp, P(bufs[4])
        ba.WD, ba.WH, ba.WW = fa.WD, fa.WH, fa.WW
    rg = None
    if rays:
        rg = [np.full((N, H, W, c), np.nan, np.float32) for c in (3, 3, 2)]
        assert L.mvp_raymarch_backward_rays(ctypes.addressof(ba), *(P(x) for x in rg), None) == 0
    else:
        assert L.mvp_raymarch_backward(ctypes.byref(ba), None) == 0
    march.last_heavy = (hf, heavy())
    grads = [b if w else None for b, w in zip(bufs, want)] + ([None] if warp is None else [])
    return rayrgba, grads, rg, sentinels


def same(x, y, exact):
    return np.array_equal(x, y) if exact else relerr(x, y) <= TOL


def check_sets(kernels, a, kw, grad, **opts):
    """Every reduced set against the full backward, with and without ray gradients: the same image, the transform and ray gradients
    bit for bit where the set drops no warp collective (algo 1 without a payload gradient), else within the atomics' order; the
    sentinel buffers stay untouched."""
    out, full, _, _ = march(kernels, a, kw, grad, "all", rays=False, **opts)
    outr, fullr, fr, _ = march(kernels, a, kw, grad, "all", rays=True, **opts)
    assert all(np.isfinite(x).all() for x in full if x is not None)
    assert np.abs(full[0]).max() > 0 and np.abs(fr[0]).max() > 0, "the scene must give the transforms and the rays a gradient"
    for gset, rays in (("no_payload", False), ("no_payload", True), ("rays_only", True)):
        exact = gset == "no_payload" and kw.get("warp") is not None
        o, g, r, sent = march(kernels, a, kw, grad, gset, rays=rays, unused="sentinel", **opts)
        assert np.array_equal(o, out), (gset, rays)
        assert all(np.all(s == SENTINEL) for s in sent), ("a buffer outside the set was written", gset, rays)
        assert all(x is None for x in g[3:]), gset
        if gset == "no_payload":
            for nm, x, y in zip(("primpos", "primrot", "primscale"), g[TRANSFORMS], (fullr if rays else full)[TRANSFORMS]):
                assert same(x, y, exact), (gset, rays, nm, relerr(x, y))
        else:
            assert all(x is None for x in g[TRANSFORMS])
        if rays:
            for nm, x, y in zip(("raypos", "raydir", "tminmax"), r, fr):
                assert same(x, y, exact), (gset, nm, relerr(x, y))


@pytest.mark.parametrize("name", ["head_small", "warp_small"])
def test_emulated_full_backward_is_deterministic_here(kernels, name):
    """The premise of the comparisons above: with one block at a time and a fixed lane order, two full backwards agree bit for bit."""
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    _, f1, r1, _ = march(kernels, a, kw, grad.numpy(), "all", rays=True)
    _, f2, r2, _ = march(kernels, a, kw, grad.numpy(), "all", rays=True)
    assert all(np.array_equal(x, y) for x, y in zip(f1[:4] + r1, f2[:4] + r2))


def _bf16(a):
    from tests.test_emul_bf16_payload import to_bf16
    ab = list(a)
    ab[7] = to_bf16(a[7]).view(np.float32)
    return ab


def _tflags(dtype):
    from ava256_b200 import lib
    return {"fp32": 0, "bf16": lib.FLAG_TPLATE_BF16, "bf16_g32": lib.FLAG_TPLATE_BF16 | lib.FLAG_GRAD_TPLATE_F32}[dtype]


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("name", list(CASES))
def test_emulated_grad_sets_named_cases(kernels, name, dtype):
    """T = 8 (head_small), 16 (head_t16), runtime dims (gradcheck_*, noncubic, tiny, many_*) and algo 1 (warp_*)."""
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    check_sets(kernels, _bf16(a) if dtype == "bf16" else a, kw, grad.numpy(), tflags=_tflags(dtype))


@pytest.mark.parametrize("cap", list(DENSE_K3))
@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_emulated_grad_sets_heavy_kernels(kernels, name, cap):
    """Every tile through the 512-entry kernels."""
    s, grad = build_dense_case(name, cap)
    a, kw = scene_args_np(s)
    check_sets(kernels, a, kw, grad.numpy())
    N, H, W = s["raypos"].shape[:3]
    assert march.last_heavy == (N * -(-H // 4) * -(-W // 8),) * 2


@pytest.mark.parametrize("name", ["head_small", "warp_small", "gradcheck_ragged"])
def test_emulated_grad_sets_bf16_grad_f32_request(kernels, name):
    """MVP_FLAG_GRAD_TPLATE_F32 with a reduced set runs the Bf16x4 kernels: the same transform and ray gradients as the full bf16
    backward."""
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    ab = _bf16(a)
    _, full, fr, _ = march(kernels, ab, kw, grad.numpy(), "all", rays=True, tflags=_tflags("bf16"))
    for gset in ("no_payload", "rays_only"):
        _, g, r, sent = march(kernels, ab, kw, grad.numpy(), gset, rays=True, tflags=_tflags("bf16_g32"), unused="sentinel")
        assert all(np.all(x == SENTINEL) for x in sent)
        if gset == "no_payload":
            assert all(relerr(x, y) <= TOL for x, y in zip(g[TRANSFORMS], full[TRANSFORMS]))
        assert all(relerr(x, y) <= TOL for x, y in zip(r, fr))


@pytest.mark.parametrize("name", ["head_small", "warp_head"])
def test_emulated_grad_sets_shared_primitives(kernels, name):
    from ava256_b200 import lib
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    a1 = list(a)
    for i in (4, 5, 6, 7):
        a1[i] = np.ascontiguousarray(a[i][:1])
    kw1 = dict(kw)
    if "warp" in kw:
        kw1["warp"] = np.ascontiguousarray(kw["warp"][:1])
    check_sets(kernels, a1, kw1, grad.numpy(), flags=lib.FLAG_SHARED_PRIMS)


@pytest.mark.parametrize("name", ["head_small", "warp_small"])
def test_emulated_grad_sets_morton_order(kernels, name):
    from ava256_b200.op import morton_codes
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    order = np.ascontiguousarray(torch.sort(morton_codes(s["primpos"]), dim=-1, stable=True)[1].to(torch.int32).numpy())
    check_sets(kernels, a, kw, grad.numpy(), order=order)


@pytest.mark.parametrize("name", ["head_small", "warp_small"])
def test_emulated_grad_sets_zero_grads_flag(kernels, name):
    """MVP_FLAG_ZERO_GRADS zero-fills the requested buffers (NaN before) and leaves the others alone."""
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    _, full, fr, _ = march(kernels, a, kw, grad.numpy(), "all", rays=True)
    for gset in ("no_payload", "rays_only"):
        _, g, r, sent = march(kernels, a, kw, grad.numpy(), gset, rays=True, unused="sentinel", init="zero")
        assert sent and all(np.all(x == SENTINEL) for x in sent), gset
        for x, y in zip(g, full):
            assert x is None or relerr(x, y) <= TOL, gset
        assert all(relerr(x, y) <= TOL for x, y in zip(r, fr))


def test_emulated_grad_sets_accept_null_only_with_a_flag(kernels):
    """With the flags the unrequested buffers may be NULL (a full run); without them a NULL gradient pointer is MVP_ERR_NULL, and
    MVP_FLAG_RAY_GRADS_ONLY without the ray outputs is MVP_ERR_NULL too."""
    from ava256_b200 import lib
    s, grad = build_case("warp_small")
    a, kw = scene_args_np(s)
    _, full, fr, _ = march(kernels, a, kw, grad.numpy(), "all", rays=True)
    _, g, r, _ = march(kernels, a, kw, grad.numpy(), "no_payload", rays=True, unused="null")
    assert all(relerr(x, y) <= TOL for x, y in zip(g[TRANSFORMS], full[TRANSFORMS]))
    _, g, r, _ = march(kernels, a, kw, grad.numpy(), "rays_only", rays=True, unused="null")
    assert all(relerr(x, y) <= TOL for x, y in zip(r, fr))
    _abi_rejections(kernels.load(), lib)


def _backward_args(lib, flags, nulls):
    """A complete argument set (host buffers, never launched) with the given gradient pointers set to NULL."""
    keep = []

    def buf(n):
        keep.append(np.zeros(n + 4, np.float32))
        x = keep[-1]
        return x.ctypes.data + (-x.ctypes.data) % 16

    b = lib.BackwardArgs()
    b.shape = lib.Shape(1, 8, 8, 4, 2, 2, 2)
    b.stepsize, b.fadescale, b.fadeexp, b.flags = 0.1, 8.0, 8.0, flags
    for f in ("raypos", "raydir", "tminmax", "primpos", "primrot", "primscale", "tplate", "grad_rayrgba", "raysat", "rayaux",
              "grad_primpos", "grad_primrot", "grad_primscale", "grad_tplate", "warp", "grad_warp"):
        setattr(b, f, buf(1024))
    b.algo, b.WD, b.WH, b.WW = 1, 2, 2, 2
    b.workspace, b.workspace_bytes = buf(1024), 4096          # the NULL checks come first: never used
    for f in nulls:
        setattr(b, f, None)
    return b, keep


def _abi_rejections(L, lib):
    L.mvp_raymarch_backward_rays.restype = ctypes.c_int
    L.mvp_raymarch_backward_rays.argtypes = [ctypes.c_void_p] * 5
    rays = [np.zeros(64 * 3 + 4, np.float32) for _ in range(3)]
    rp = [r.ctypes.data + (-r.ctypes.data) % 16 for r in rays]
    NO, RO = lib.FLAG_NO_TPLATE_GRAD, lib.FLAG_RAY_GRADS_ONLY
    for nulls in (("grad_tplate",), ("grad_warp",), ("grad_primpos",), ("grad_primrot",), ("grad_primscale",)):
        b, keep = _backward_args(lib, 0, nulls)
        assert L.mvp_raymarch_backward(ctypes.byref(b), None) == -1, nulls
        assert L.mvp_raymarch_backward_rays(ctypes.addressof(b), *rp, None) == -1, nulls
    for nulls in (("grad_primpos",), ("grad_primrot",), ("grad_primscale",)):      # the transforms stay required with NO_TPLATE_GRAD
        b, keep = _backward_args(lib, NO, nulls + ("grad_tplate", "grad_warp"))
        assert L.mvp_raymarch_backward(ctypes.byref(b), None) == -1, nulls
    b, keep = _backward_args(lib, RO, ())
    assert L.mvp_raymarch_backward(ctypes.byref(b), None) == -1                      # no output requested


def test_product_library_grad_select_abi():
    """The product library lists GRAD_SELECT=1, keeps the ABI version and struct sizes, and rejects before any device work."""
    from ava256_b200 import lib
    assert "GRAD_SELECT=1" in lib.LIB.mvp_build_config().decode().split()
    lib.require_grad_select()
    assert lib.LIB.mvp_abi_version() == 8 == lib.ABI_VERSION
    assert ctypes.sizeof(lib.ForwardArgs) == ctypes.sizeof(lib.BackwardArgs) == 272
    assert (lib.FLAG_NO_TPLATE_GRAD, lib.FLAG_RAY_GRADS_ONLY) == (32, 64)
    _abi_rejections(lib.LIB, lib)


def test_header_documents_the_flags():
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "mvpraymarch_b200.h")) as f:
        hdr = f.read()
    assert "#define MVP_FLAG_NO_TPLATE_GRAD 32u" in hdr and "#define MVP_FLAG_RAY_GRADS_ONLY 64u" in hdr
