"""Deterministic primitive gradients (mvp_raymarch_backward_deterministic, MVP_FLAG_DETERMINISTIC) on the emulated product kernels.

The backward sums grad_primpos / primrot / primscale / tplate in 64-bit fixed point: a measure pass finds each tensor's largest
reduction, an accumulate pass adds llrint(x / q) with integer reductions, and a conversion writes (float)sum * q.  Checked here:
  * every named case with algo 0, fp32 and bf16 templates: the same image as the default path, and every gradient within TOL of
    max|.| of the default path's (a bf16 template against its fp32-accumulated gradient; its bf16 gradient is that fp32 result
    rounded once, bit for bit);
  * the schedule: with MVP_EMUL_THREADS=1 the blocks run one after the other and the emulation's lane order (forward, reverse,
    random: the order in which the lanes and warps of a block issue their reductions) fixes the order of every atomic.  Another
    lane order, or the views of a shared-primitive launch in another order (their blocks then run in another order), changes the
    default path's gradient bits (fp32 atomics in another order) and leaves the fixed-point sums' bits alone;
  * the quantum rule on the host, NaN propagation, and the argument errors of the entry point and of the unsupported modes (algo 1,
    ray gradients) at the C-ABI and, for the op, NotImplementedError."""
import ctypes

import numpy as np
import pytest
import torch

from tests.helpers import CASES, build_case, relerr, scene_args_np

TOL = 1e-5
ALGO0 = [n for n in CASES if not n.startswith("warp")]
NAMES = ("primpos", "primrot", "primscale", "template")


@pytest.fixture()
def kernels(monkeypatch):
    from tests.emul import kernels as k
    monkeypatch.setenv("MVP_EMUL_THREADS", "1")        # blocks one after the other: the order of the atomics is fixed
    k.use_variant(())
    L = k.load()
    L.mvp_raymarch_backward_deterministic.restype = ctypes.c_int
    L.mvp_raymarch_backward_deterministic.argtypes = [ctypes.c_void_p] * 8 + [ctypes.c_int32, ctypes.c_void_p]
    L.mvp_emul_det_quantum_exp.restype = ctypes.c_int
    L.mvp_emul_det_quantum_exp.argtypes = [ctypes.c_uint32]
    k.set_lane_order("forward")
    yield k
    k.set_lane_order("forward")


def _arr(shape, dtype, fill):
    """Array of dtype filled with fill whose data pointer is 16-byte aligned."""
    n = int(np.prod(shape))
    it = np.dtype(dtype).itemsize
    raw = np.empty(n + 16 // it, dtype)
    off = (-raw.ctypes.data // it) % (16 // it)
    out = raw[off:off + n].reshape(shape)
    out[...] = fill
    return out


def march(kernels, a, kw, grad, det, tflags=0, flags=0, gset="all", zero=False, warp=None):
    """Emulated forward + backward of the scene (scene_args_np form; a[7] may be a bf16 template as fp32-typed words).  det: the
    deterministic backward, its int64 sums cleared by the forward (or by MVP_FLAG_ZERO_GRADS with zero=True).  Returns (rayrgba,
    [primpos, primrot, primscale, template] gradients (template None for gset="no_payload"), backward return code)."""
    from ava256_b200 import lib
    L = kernels.load()
    P = lambda x: None if x is None else ctypes.c_void_p(x.ctypes.data)  # noqa: E731
    raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template = a
    N, H, W = raypos.shape[:3]
    K, (TD, TH, TW) = primpos.shape[1], template.shape[2:5]
    gwords = 4 if (tflags & lib.FLAG_GRAD_TPLATE_F32) else template.shape[-1]
    want_t = gset == "all"
    bufs = [_arr(primpos.shape, np.float32, np.nan), _arr(primrot.shape, np.float32, np.nan), _arr(primscale.shape, np.float32, np.nan),
            _arr(template.shape[:-1] + (gwords,), np.float32, np.nan) if want_t else None]
    sums = [_arr(primpos.shape, np.int64, -1), _arr(primrot.shape, np.int64, -1), _arr(primscale.shape, np.int64, -1),
            _arr(template.shape[:-1] + (4,), np.int64, -1) if want_t else None] if det else None
    shape = lib.Shape(N, H, W, K, TD, TH, TW)
    wsb = L.mvp_workspace_bytes(ctypes.byref(shape))
    raw = np.zeros(wsb + 256, np.uint8)
    ws = raw[(-raw.ctypes.data) % 256:][:wsb]
    rayrgba, raysat = np.full((N, H, W, 4), np.nan, np.float32), np.full((N, H, W, 3), np.nan, np.float32)
    rayaux = np.zeros((N, H, W, 4), np.int32)
    fl = flags | tflags | (lib.FLAG_NO_TPLATE_GRAD if gset == "no_payload" else 0)
    fa = lib.ForwardArgs()
    fa.shape, fa.stepsize, fa.fadescale, fa.fadeexp = shape, float(stepsize), kw["fadescale"], kw["fadeexp"]
    fa.flags = fl | (lib.FLAG_DETERMINISTIC if det else 0)
    fa.raypos, fa.raydir, fa.tminmax = P(raypos), P(raydir), P(tminmax)
    fa.primpos, fa.primrot, fa.primscale, fa.tplate = P(primpos), P(primrot), P(primscale), P(template)
    fa.rayrgba, fa.raysat, fa.rayaux = P(rayrgba), P(raysat), P(rayaux)
    fa.workspace, fa.workspace_bytes = P(ws), wsb
    if warp is not None:
        fa.algo, fa.warp = 1, P(warp)
        fa.WD, fa.WH, fa.WW = warp.shape[2:5]
    clr = sums if det else bufs
    if not zero:
        fa.clear_grad_primpos, fa.clear_grad_primrot, fa.clear_grad_primscale, fa.clear_grad_tplate = (P(b) for b in clr)
    assert L.mvp_raymarch_forward(ctypes.byref(fa), None) == 0
    if not zero:
        assert all(b is None or not b.any() for b in clr), "the forward must clear the gradient buffers"
    ba = lib.BackwardArgs()
    ba.shape, ba.stepsize, ba.fadescale, ba.fadeexp = shape, fa.stepsize, fa.fadescale, fa.fadeexp
    ba.flags = lib.FLAG_ACCEL_VALID | fl | (lib.FLAG_ZERO_GRADS if zero else 0)
    ba.raypos, ba.raydir, ba.tminmax = fa.raypos, fa.raydir, fa.tminmax
    ba.primpos, ba.primrot, ba.primscale, ba.tplate = fa.primpos, fa.primrot, fa.primscale, fa.tplate
    g = np.ascontiguousarray(grad, np.float32)
    ba.grad_rayrgba, ba.raysat, ba.rayaux = P(g), P(raysat), P(rayaux)
    ba.grad_primpos, ba.grad_primrot, ba.grad_primscale, ba.grad_tplate = (P(b) for b in bufs)
    ba.workspace, ba.workspace_bytes = fa.workspace, wsb
    if warp is not None:
        ba.algo, ba.warp, ba.grad_warp = 1, fa.warp, P(_arr(warp.shape, np.float32, 0.0))
        ba.WD, ba.WH, ba.WW = fa.WD, fa.WH, fa.WW
    if det:
        dmax = _arr((4,), np.uint32, 0)
        rc = L.mvp_raymarch_backward_deterministic(ctypes.addressof(ba), *(P(x) for x in sums), P(dmax), None, None, 0, None)
    else:
        rc = L.mvp_raymarch_backward(ctypes.byref(ba), None)
    return rayrgba, bufs, rc


def _bf16(a):
    from tests.test_emul_bf16_payload import to_bf16
    ab = list(a)
    ab[7] = to_bf16(a[7]).view(np.float32)
    return ab


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("name", ALGO0)
def test_deterministic_agrees_with_default(kernels, name, dtype):
    from ava256_b200 import lib
    from tests.test_emul_bf16_payload import to_bf16
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    tf = 0
    if dtype == "bf16":
        a, tf = _bf16(a), lib.FLAG_TPLATE_BF16 | lib.FLAG_GRAD_TPLATE_F32
    out0, g0, rc0 = march(kernels, a, kw, grad.numpy(), False, tflags=tf)
    out1, g1, rc1 = march(kernels, a, kw, grad.numpy(), True, tflags=tf)
    assert rc0 == 0 and rc1 == 0
    assert np.array_equal(out0, out1, equal_nan=True)
    for nm, x, y in zip(NAMES, g1, g0):
        assert np.isfinite(x).all() and np.abs(y).max() > 0, nm
        assert relerr(x, y) <= TOL, (nm, relerr(x, y))
    if dtype == "bf16":
        # the bf16 gradient is the fixed-point result rounded once more
        _, gb, rc = march(kernels, a, kw, grad.numpy(), True, tflags=lib.FLAG_TPLATE_BF16)
        assert rc == 0
        assert np.array_equal(gb[3].view(np.uint16), to_bf16(g1[3]).reshape(gb[3].view(np.uint16).shape))
        assert all(np.array_equal(x, y) for x, y in zip(gb[:3], g1[:3]))


@pytest.mark.parametrize("name", ["head_small", "gradcheck_small", "many_overlaps"])
def test_lane_order_changes_default_bits_not_deterministic(kernels, name):
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    runs = {}
    for order in ("forward", "reverse", "random"):
        kernels.set_lane_order(order)
        runs[order] = [march(kernels, a, kw, grad.numpy(), det) for det in (False, True)]
    (o0, d0, _), (o1, e1, _) = runs["forward"]
    assert np.array_equal(o0, o1, equal_nan=True)
    changed = False
    for order in ("reverse", "random"):
        (p0, r0, _), (p1, f1, _) = runs[order]
        assert np.array_equal(o0, p0, equal_nan=True) and np.array_equal(o1, p1, equal_nan=True), order
        changed |= any(not np.array_equal(x, y) for x, y in zip(d0, r0))
        assert all(np.array_equal(x, y) for x, y in zip(e1, f1)), ("the fixed-point sums must not depend on the schedule", order)
    assert changed, "another lane order should change the float atomics' sums"


@pytest.mark.parametrize("name", ["head_small", "gradcheck_small"])
def test_view_order_changes_default_bits_not_deterministic(kernels, name):
    """Shared primitives [1,K,...] (MVP_FLAG_SHARED_PRIMS): every view adds into the same gradients, so reversing the views reverses
    the order of the blocks' reductions into them."""
    from ava256_b200 import lib
    s, grad = build_case(name)
    a, kw = scene_args_np(s)
    a = list(a)
    for i in range(4, 8):
        a[i] = np.ascontiguousarray(a[i][:1])
    rev = list(a)
    for i in (0, 1, 3):
        rev[i] = np.ascontiguousarray(a[i][::-1])
    g = grad.numpy()
    o0, d0, _ = march(kernels, a, kw, g, False, flags=lib.FLAG_SHARED_PRIMS)
    p0, r0, _ = march(kernels, rev, kw, np.ascontiguousarray(g[::-1]), False, flags=lib.FLAG_SHARED_PRIMS)
    o1, e1, _ = march(kernels, a, kw, g, True, flags=lib.FLAG_SHARED_PRIMS)
    p1, f1, _ = march(kernels, rev, kw, np.ascontiguousarray(g[::-1]), True, flags=lib.FLAG_SHARED_PRIMS)
    assert np.array_equal(o0, p0[::-1], equal_nan=True) and np.array_equal(o1, p1[::-1], equal_nan=True)
    assert np.array_equal(o0, o1, equal_nan=True)
    assert any(not np.array_equal(x, y) for x, y in zip(d0, r0)), "the view order should change the float atomics' sums"
    assert all(np.array_equal(x, y) for x, y in zip(e1, f1)), "the fixed-point sums must not depend on the view order"


def test_deterministic_repeat_zero_grads_and_no_payload(kernels):
    """Two runs are bit-identical; MVP_FLAG_ZERO_GRADS in place of the forward's clear gives the same bits; the "no payload" set
    gives the same transform gradients as the full set (their reductions are the same values)."""
    s, grad = build_case("head_small")
    a, kw = scene_args_np(s)
    _, g1, _ = march(kernels, a, kw, grad.numpy(), True)
    _, g2, _ = march(kernels, a, kw, grad.numpy(), True, zero=True)
    _, g3, rc = march(kernels, a, kw, grad.numpy(), True, gset="no_payload")
    assert rc == 0 and g3[3] is None
    assert all(np.array_equal(x, y) for x, y in zip(g1, g2))
    assert all(np.array_equal(x, y) for x, y in zip(g1[:3], g3[:3]))


def test_quantum_and_headroom_rule(kernels):
    """q = 2^(e - 38) with 2^e the smallest power of two >= M; every |x| <= M is then at most 2^38 quanta, so fewer than 2^24
    reductions into an entry stay below 2^62; q >= 2^-126."""
    L = kernels.load()
    rng = np.random.default_rng(3)
    ms = np.concatenate([np.float32([1.0, 2.0, 0.75, 1.5, 3.0e38, 1e-30, 2.0 ** -100, 2.0 ** -88, 1e-45]),
                         (10.0 ** rng.uniform(-20, 20, 200)).astype(np.float32)])
    for m in ms:
        bits = int(np.float32(m).view(np.uint32))
        qe = L.mvp_emul_det_quantum_exp(bits)
        e = int(np.ceil(np.log2(np.float64(m))))
        assert qe == max(e - 38, -126), (m, qe, e)
        assert float(m) <= 2.0 ** (qe + 38)                                  # |x| / q <= 2^38
        assert qe == -126 or float(m) > 2.0 ** (qe + 37)                      # and no coarser than needed
    assert L.mvp_emul_det_quantum_exp(0) == -126
    assert (2 ** 24 - 1) * 2 ** 38 < 2 ** 62


def test_nan_poisons_the_same_entries(kernels):
    """A NaN in the incoming gradient: the entries it reaches come out NaN, exactly those the default path makes non-finite."""
    s, grad = build_case("head_small")
    a, kw = scene_args_np(s)
    g = grad.numpy().copy()
    out, _, _ = march(kernels, a, kw, g, False)
    seen = np.argwhere(out[..., 3] > 0.5)                                   # pixels that see the head
    n, h, w = seen[len(seen) // 2]
    g[n, h, w, 1] = np.nan
    _, gd, _ = march(kernels, a, kw, g, False)
    _, gx, _ = march(kernels, a, kw, g, True)
    for nm, x, y in zip(NAMES, gx, gd):
        bad = ~np.isfinite(y)
        assert bad.any(), nm
        assert np.array_equal(np.isnan(x), bad), nm
        assert np.isfinite(x[~bad]).all()


def test_unsupported_modes_are_argument_errors(kernels):
    from ava256_b200 import lib
    s, grad = build_case("warp_small")
    a, kw = scene_args_np(s)
    _, _, rc = march(kernels, a, kw, grad.numpy(), True, zero=True, warp=np.ascontiguousarray(kw["warp"], np.float32))
    assert rc == -5                                                           # MVP_ERR_ALGO
    s, grad = build_case("gradcheck_small")
    a, kw = scene_args_np(s)
    _, _, rc = march(kernels, a, kw, grad.numpy(), True, zero=True, flags=lib.FLAG_RAY_GRADS_ONLY)
    assert rc == -1                                                           # MVP_ERR_NULL: no ray gradients here


def test_entry_point_argument_errors():
    """mvp_raymarch_backward_deterministic of the product library returns its argument errors before any device work (the pointers
    below are never dereferenced): a NULL or stale struct, missing or misaligned sums and maxima, algo 1, a bad view-set map."""
    from ava256_b200 import lib
    f = lib.LIB.mvp_raymarch_backward_deterministic
    P = ctypes.c_void_p
    assert "DETERMINISTIC=1" in lib.LIB.mvp_build_config().decode().split()
    assert f(None, *([None] * 6), None, 0, None) == -1                       # MVP_ERR_NULL
    b = lib.BackwardArgs()
    b.struct_size = 0
    assert f(ctypes.byref(b), *([None] * 6), None, 0, None) == -7             # MVP_ERR_STRUCT
    b = lib.BackwardArgs()
    b.shape = lib.Shape(1, 8, 8, 4, 2, 2, 2)
    b.stepsize = 0.1
    d = P(256)
    b.raypos = b.raydir = b.tminmax = b.primpos = b.primrot = b.primscale = b.tplate = d
    b.grad_rayrgba = b.raysat = b.rayaux = b.grad_primpos = b.grad_primrot = b.grad_primscale = b.grad_tplate = d
    b.workspace, b.workspace_bytes = d, 1 << 30
    sums = [d, d, d, d]
    assert f(ctypes.byref(b), *([None] * 4), d, None, None, 0, None) == -1    # the sums are required
    assert f(ctypes.byref(b), *sums, None, None, None, 0, None) == -1         # and so are the maxima
    assert f(ctypes.byref(b), P(260), d, d, d, d, None, None, 0, None) == -6  # MVP_ERR_ALIGN: sums need 8 bytes
    b.algo = 1
    b.warp = b.grad_warp = d
    b.WD = b.WH = b.WW = 2
    assert f(ctypes.byref(b), *sums, d, None, None, 0, None) == -5            # MVP_ERR_ALGO
    b.algo = 0
    assert f(ctypes.byref(b), *sums, d, None, d, 0, None) == -2               # MVP_ERR_SHAPE: nsets outside [1, N]
    b.flags = lib.FLAG_RAY_GRADS_ONLY
    assert f(ctypes.byref(b), *sums, d, None, None, 0, None) == -1            # no ray gradients from this entry point


def _leaf(shape):
    return torch.rand(shape).requires_grad_(True)


def test_op_raises_not_implemented():
    """The op refuses algo 1 and ray / camera gradients in the mode, before it looks at devices."""
    from ava256_b200 import op
    N, H, W, K = 1, 8, 8, 2
    prims = (_leaf((N, K, 3)), _leaf((N, K, 3, 3)), _leaf((N, K, 3)))
    tpl, warp = _leaf((N, K, 2, 2, 2, 4)), torch.rand(N, K, 2, 2, 2, 3)
    rays = (torch.rand(N, H, W, 3), torch.rand(N, H, W, 3), torch.rand(N, H, W, 2))
    with op.deterministic_grads(), pytest.raises(NotImplementedError):
        op.mvpraymarch(rays[0], rays[1], 0.1, rays[2], prims, tpl, warp, algo=1)
    cam = (_leaf((N, 3)), torch.eye(3).expand(N, 3, 3).contiguous(), torch.ones(N, 2), torch.ones(N, 2))
    with pytest.raises(NotImplementedError):
        op.mvpraymarch_camera(*cam, (W, H), 1.0, 0.1, prims, tpl, None, camera_grad=True, deterministic=True)
