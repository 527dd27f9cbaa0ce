"""CPU tests of the bfloat16 payload hand-off (`mvp_assemble_payload_*_bf16`) and the bf16 view sum (`mvp_sum_views_bf16`).

The payload bodies run on the host build of csrc/epilogue_body.h (tests/emul/epilogue_bf16_emul.cpp) and through the entry points of
epilogue.cu on the CPU emulation (tests/emul/aux_emul.cpp).  Contracts:
  - forward: bit-identical to assemble_payload_ref(tex, opacity, B).to(torch.bfloat16);
  - backward: bit-identical to eager autograd through that expression for the same bf16 incoming gradient, except where the
    fp32 relu output lies in (0, 2^-134]: it rounds to bf16 zero, so the mask taken from the bf16 template drops the gradient;
  - view sum: the fp32 dst equals the emulated mvp_sum_views of the widened source bit for bit, the bf16 dst is that rounded once."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle.epilogue_ref import assemble_payload_ref
from tests.test_epilogue import PAYLOAD_SHAPES, _payload_case

F32P = ctypes.POINTER(ctypes.c_float)
VP = ctypes.c_void_p
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _p(a):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    """tests/emul/epilogue_bf16_emul.cpp compiled with g++ into a temporary directory (flags of tests/emul/build.py)."""
    out = str(tmp_path_factory.mktemp("bf16_emul") / "libepilogue_bf16_emul.so")
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-shared", "-fPIC", "-I" + cuda_inc,
                           "-I" + os.path.join(ROOT, "ava-256_b200", "csrc"),
                           os.path.join(ROOT, "tests", "emul", "epilogue_bf16_emul.cpp"), "-o", out])
    lib = ctypes.CDLL(out)
    lib.emul_payload_forward_bf16.argtypes = [ctypes.c_int] * 6 + [VP] * 2 + [ctypes.c_float] * 2 + [VP]
    lib.emul_payload_backward_bf16.argtypes = [ctypes.c_int] * 6 + [VP] * 2 + [ctypes.c_float] + [VP] * 2
    return lib


@pytest.fixture(scope="module")
def aux():
    from tests.emul.build import build_aux
    lib = ctypes.CDLL(build_aux())
    lib.mvp_assemble_payload_forward_bf16.argtypes = [ctypes.c_int32] * 4 + [VP] * 2 + [ctypes.c_float] * 2 + [VP] * 2
    lib.mvp_assemble_payload_backward_bf16.argtypes = [ctypes.c_int32] * 4 + [VP] * 2 + [ctypes.c_float] + [VP] * 3
    lib.mvp_sum_views.argtypes = [VP, VP, ctypes.c_size_t, ctypes.c_int32, VP]
    lib.mvp_sum_views_bf16.argtypes = [VP, VP, ctypes.c_size_t, ctypes.c_int32, ctypes.c_int32, VP]
    return lib


def _bits(t):
    """A bf16 CPU tensor as its uint16 bit patterns."""
    return t.contiguous().view(torch.int16).numpy().view(np.uint16)


def _widen(u16):
    return torch.from_numpy(u16.astype(np.uint16).view(np.int16).copy()).view(torch.bfloat16).float().numpy()


def _eager_bf16(tex, opacity, gb, B):
    """Forward bits and gradients of assemble_payload_ref(...).to(torch.bfloat16) for the bf16 incoming gradient gb."""
    t, o = tex.detach().clone().requires_grad_(True), opacity.detach().clone().requires_grad_(True)
    tp = assemble_payload_ref(t, o, B).to(torch.bfloat16)
    tp.backward(gb)
    return tp.detach(), t.grad, o.grad


def _emul_bf16(emul, tex, opacity, gb, B, V, BT, N, hb, wb):
    tpl = np.full((N, hb * wb, B, B, B, 4), 0x7fff, np.uint16)            # NaN-filled: every texel must be written
    assert emul.emul_payload_forward_bf16(N, hb, wb, B, V, BT, _p(tex.numpy()), _p(opacity.numpy()), 25.0, 100.0, _p(tpl)) == 0
    gtex = np.full(tuple(tex.shape), np.nan, np.float32)
    gop = np.full(tuple(opacity.shape), np.nan, np.float32)
    assert emul.emul_payload_backward_bf16(N, hb, wb, B, V, BT, _p(tpl), _p(_bits(gb)), 25.0, _p(gtex), _p(gop)) == 0
    return tpl, gtex, gop


@pytest.mark.parametrize("N,hb,wb,B,V,BT", PAYLOAD_SHAPES)
def test_emul_bf16_payload_matches_eager_torch(emul, N, hb, wb, B, V, BT):
    tex, opacity, gt = _payload_case(N, hb, wb, B, seed=B + 100)
    gb = gt.to(torch.bfloat16)
    ref, gtex_ref, gop_ref = _eager_bf16(tex, opacity, gb, B)
    tpl, gtex, gop = _emul_bf16(emul, tex, opacity, gb, B, V, BT, N, hb, wb)
    assert np.array_equal(tpl, _bits(ref))
    assert np.array_equal(gtex, gtex_ref.numpy()) and np.array_equal(gop, gop_ref.numpy())
    # both sides of every relu and both halves of every pair are exercised (the one-texel case aside)
    w = _widen(tpl)
    assert B == 1 or (w[..., :3] == 0).any() and (w[..., :3] > 0).any() and (w[..., 3] == 0).any() and (w[..., 3] > 0).any()


def test_emul_bf16_payload_rounds_to_nearest_even_and_keeps_nan(emul):
    """Values half-way between two bf16 neighbours (ties to even), just above half-way (rounds up: truncation would not), and
    NaN, which stays NaN."""
    N, hb, wb, B = 1, 1, 1, 4
    opacity = torch.zeros(N, B, B, B)
    one = 1.0
    vals = [one + 2 ** -8, one + 3 * 2 ** -8, one + 2 ** -8 + 2 ** -20, 3.0 + 3 * 2 ** -7, float("nan"), 2 ** -133, 1.5 * 2 ** -134]
    opacity.view(-1)[:len(vals)] = torch.tensor(vals)
    tex = torch.zeros(N, 3 * B, B, B)
    tex.view(-1)[:3] = torch.tensor([float("nan"), 0.1234567, -4.0])
    gb = torch.ones(N, hb * wb, B, B, B, 4, dtype=torch.bfloat16)
    ref, _, _ = _eager_bf16(tex, opacity, gb, B)
    for V in (1, 4):
        tpl, _, _ = _emul_bf16(emul, tex, opacity, gb, B, V, 0, N, hb, wb)
        rb = _bits(ref)
        nan = np.isnan(_widen(rb))
        assert np.array_equal(np.isnan(_widen(tpl)), nan) and nan.sum() == 2
        assert np.array_equal(tpl[~nan], rb[~nan])
        a = _widen(tpl)[0, 0, 0, 0, :, 3]
        assert list(a[:4]) == [1.0, one + 4 * 2 ** -8, one + 2 * 2 ** -8, 3.0 + 2 ** -5]


def test_emul_bf16_payload_mask_below_the_smallest_subnormal(emul):
    """The one documented departure: an fp32 relu output in (0, 2^-134] is bf16 zero, so its gradient is masked where eager
    autograd (mask taken on the fp32 relu output) passes it.  Everywhere else the gradients are bit-identical."""
    N, hb, wb, B = 1, 2, 2, 4
    tex, opacity, gt = _payload_case(N, hb, wb, B, seed=7)
    tiny = torch.tensor([2.0 ** -134, 2.0 ** -140, 2.0 ** -149, 2.0 ** -135 * 1.5])    # all round to bf16 +0
    kept = torch.tensor([2.0 ** -133, 2.0 ** -134 * 1.25, 2.0 ** -126])                  # round to a non-zero bf16
    flat = opacity.view(-1)
    flat[:4], flat[10:13] = tiny, kept
    gb = gt.to(torch.bfloat16)
    ref, gtex_ref, gop_ref = _eager_bf16(tex, opacity, gb, B)
    for V, BT in ((1, 0), (4, 0)):
        tpl, gtex, gop = _emul_bf16(emul, tex, opacity, gb, B, V, BT, N, hb, wb)
        assert np.array_equal(tpl, _bits(ref))
        assert np.array_equal(gtex, gtex_ref.numpy())
        assert (gop_ref.view(-1)[:4] != 0).all() and (gop_ref.view(-1)[10:13] != 0).all()   # eager passes all seven
        diff = np.flatnonzero((gop != gop_ref.numpy()).reshape(-1))
        assert list(diff) == [0, 1, 2, 3] and (gop.reshape(-1)[:4] == 0).all()


@pytest.mark.parametrize("N,hb,wb,B", [(2, 2, 3, 8), (1, 3, 2, 4), (1, 4, 2, 3), (1, 2, 2, 16)])
def test_emulated_bf16_payload_entry_points(aux, emul, N, hb, wb, B):
    """mvp_assemble_payload_{forward,backward}_bf16 on the CPU emulation (thread -> element mapping, variant choice) against
    the host bodies; then the scalar variant forced by an 8-byte-aligned (not 16) template and gradient."""
    tex, opacity, gt = _payload_case(N, hb, wb, B, seed=B + 3)
    gb = gt.to(torch.bfloat16)
    tpl_ref, gtex_ref, gop_ref = _emul_bf16(emul, tex, opacity, gb, B, 1, 0, N, hb, wb)
    n = tpl_ref.size
    for off in (0, 4):                                                   # bf16 elements: 0 and 8 bytes past a 16-byte boundary
        raw = np.full(n + 16, 0x7fff, np.uint16)
        base = (-raw.ctypes.data // 2) % 8
        tpl = raw[base + off:base + off + n]
        assert aux.mvp_assemble_payload_forward_bf16(N, hb, wb, B, _p(tex.numpy()), _p(opacity.numpy()), 25.0, 100.0, _p(tpl), None) == 0
        assert np.array_equal(tpl, tpl_ref.reshape(-1))
        graw = np.zeros(n + 16, np.uint16)
        g = graw[base + off:base + off + n]
        g[:] = _bits(gb).reshape(-1)
        gtex = np.full(tuple(tex.shape), np.nan, np.float32)
        gop = np.full(tuple(opacity.shape), np.nan, np.float32)
        assert aux.mvp_assemble_payload_backward_bf16(N, hb, wb, B, _p(tpl), _p(g), 25.0, _p(gtex), _p(gop), None) == 0
        assert np.array_equal(gtex, gtex_ref) and np.array_equal(gop, gop_ref)


@pytest.mark.parametrize("count,n,off", [(8 * 300, 1, 0), (8 * 300, 7, 0), (8 * 300, 8, 0), (8 * 300, 9, 0), (8 * 300, 80, 0),
                                         (8 * 300 + 3, 9, 0), (8 * 300, 19, 1), (4 * 77, 80, 3)])
@pytest.mark.parametrize("dst_bf16", [0, 1])
def test_emul_sum_views_bf16(aux, count, n, off, dst_bf16):
    """The bf16 view sum on the emulation: 16-byte path (count % 8 == 0, 16-byte aligned: 8 views per round + tail) and scalar
    path (count % 8 != 0, or a source `off` elements past a 16-byte boundary), into fp32 or bf16; guard words stay untouched."""
    rng = np.random.default_rng(count + 31 * n + off)
    vals = torch.from_numpy(rng.standard_normal(n * count).astype(np.float32) * 8.0).to(torch.bfloat16)
    raw = np.zeros(n * count + 16, np.uint16)
    base = (-raw.ctypes.data // 2) % 8
    src = raw[base + off:base + off + n * count]
    src[:] = _bits(vals)
    wide = _widen(src)                                                   # exact widening, 16-byte aligned fresh array
    ref = np.full(count, np.nan, np.float32)
    assert aux.mvp_sum_views(_p(wide), _p(ref), count, n, None) == 0
    if dst_bf16:
        draw = np.full(count + 16, 0x1234, np.uint16)
        dbase = (-draw.ctypes.data // 2) % 8 + 8
        dst = draw[dbase:dbase + count]
        assert aux.mvp_sum_views_bf16(_p(src), _p(dst), count, n, 1, None) == 0
        assert np.array_equal(dst, _bits(torch.from_numpy(ref).to(torch.bfloat16)))
        assert (draw[:dbase] == 0x1234).all() and (draw[dbase + count:] == 0x1234).all()
    else:
        draw = np.full(count + 8, 7.0, np.float32)
        dbase = (-draw.ctypes.data // 4) % 4 + 4
        dst = draw[dbase:dbase + count]
        assert aux.mvp_sum_views_bf16(_p(src), _p(dst), count, n, 0, None) == 0
        assert np.array_equal(dst, ref)
        assert (draw[:dbase] == 7.0).all() and (draw[dbase + count:] == 7.0).all()


def test_emul_sum_views_bf16_argument_errors(aux):
    src = np.zeros(64 + 8, np.uint16)
    dst32 = np.zeros(64 + 4, np.float32)
    dst16 = np.zeros(64 + 8, np.uint16)
    s0 = (-src.ctypes.data // 2) % 8
    assert aux.mvp_sum_views_bf16(None, _p(dst32), 64, 2, 0, None) == -1                         # MVP_ERR_NULL
    assert aux.mvp_sum_views_bf16(_p(src), None, 64, 2, 1, None) == -1
    assert aux.mvp_sum_views_bf16(_p(src), _p(dst32), 64, 0, 0, None) == -2                      # MVP_ERR_SHAPE
    odd = ctypes.c_void_p(src.ctypes.data + 1)
    assert aux.mvp_sum_views_bf16(odd, _p(dst32), 32, 1, 0, None) == -6                          # MVP_ERR_ALIGN: src
    half = ctypes.c_void_p(dst32.ctypes.data + 2)
    assert aux.mvp_sum_views_bf16(_p(src[s0:]), half, 32, 1, 0, None) == -6                      # fp32 dst needs 4 bytes
    assert aux.mvp_sum_views_bf16(_p(src[s0:]), ctypes.c_void_p(dst16.ctypes.data + 1), 32, 1, 1, None) == -6
    assert aux.mvp_sum_views_bf16(_p(src[s0:]), half, 32, 1, 1, None) == 0                       # a bf16 dst needs 2
    assert aux.mvp_sum_views_bf16(_p(src), _p(dst32), 0, 1, 0, None) == 0                        # nothing to do


def test_bf16_handoff_argument_errors_do_not_need_a_device():
    from ava256_b200 import lib
    L = lib.LIB
    assert "EPILOGUE_BF16=1" in L.mvp_build_config().decode().split()
    lib.require_epilogue_bf16()
    p, p8, p4 = ctypes.c_void_p(4096), ctypes.c_void_p(4104), ctypes.c_void_p(4100)
    assert L.mvp_assemble_payload_forward_bf16(1, 2, 2, 8, None, p, 25.0, 100.0, p, None) == -1
    assert L.mvp_assemble_payload_forward_bf16(1, 2, 2, 8, p, p, 25.0, 100.0, None, None) == -1
    assert L.mvp_assemble_payload_forward_bf16(1, 2, 2, 0, p, p, 25.0, 100.0, p, None) == -2
    assert L.mvp_assemble_payload_forward_bf16(1, 2, 2, 65, p, p, 25.0, 100.0, p, None) == -2
    assert L.mvp_assemble_payload_forward_bf16(1, 2, 2, 8, p, p, 25.0, 100.0, p4, None) == -6
    assert L.mvp_assemble_payload_backward_bf16(1, 2, 2, 8, p, p, 25.0, p, None, None) == -1
    assert L.mvp_assemble_payload_backward_bf16(1, 0, 2, 8, p, p, 25.0, p, p, None) == -2
    assert L.mvp_assemble_payload_backward_bf16(1, 2, 2, 8, p4, p, 25.0, p, p, None) == -6
    assert L.mvp_assemble_payload_backward_bf16(1, 2, 2, 8, p, p4, 25.0, p, p, None) == -6
    assert L.mvp_assemble_payload_backward_bf16(0, 2, 2, 8, p8, p8, 25.0, p, p, None) == -2     # 8-byte aligned passes the check
    assert L.mvp_sum_views_bf16(None, p, 16, 2, 0, None) == -1
    assert L.mvp_sum_views_bf16(p, p, 16, 0, 0, None) == -2
    assert L.mvp_sum_views_bf16(ctypes.c_void_p(4097), p, 16, 1, 0, None) == -6
    assert L.mvp_sum_views_bf16(p, ctypes.c_void_p(4098), 16, 1, 0, None) == -6
    assert L.mvp_sum_views_bf16(p, ctypes.c_void_p(4098), 0, 1, 1, None) == 0


def test_bf16_handoff_dtype_checks_do_not_need_a_device():
    from ava256_b200.payload import assemble_payload, expand_views, sum_views
    x = torch.zeros(1, 24, 8, 8)
    with pytest.raises(RuntimeError, match="float32 or bfloat16"):
        assemble_payload(x, torch.zeros(1, 8, 8, 8), dtype=torch.float16)
    with pytest.raises(RuntimeError, match="CUDA"):
        expand_views(torch.zeros(6, dtype=torch.bfloat16), 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        sum_views(torch.zeros(2, 6, dtype=torch.bfloat16))


def test_host_reduce_primitive_grads_widens_a_bf16_template_gradient():
    """The host (gloo) path of the per-subject reduction: a bf16 template gradient is summed into an fp32 flat buffer, equal to
    the reduction of its fp32 widening."""
    from ava256_b200.parallel import reduce_primitive_grads
    g = torch.Generator().manual_seed(5)
    nv, K, T = 5, 6, 4
    gt = torch.randn(nv, K, T, T, T, 4, generator=g).to(torch.bfloat16)
    rest = [torch.randn(nv, K, 3, generator=g), torch.randn(nv, K, 3, 3, generator=g), torch.randn(nv, K, 3, generator=g)]
    flat_b, views_b = reduce_primitive_grads(gt, *rest)
    flat_f, _ = reduce_primitive_grads(gt.float(), *rest)
    assert flat_b.dtype == torch.float32 and torch.equal(flat_b, flat_f)
    assert views_b[0].shape == (K, T, T, T, 4) and views_b[0].dtype == torch.float32
