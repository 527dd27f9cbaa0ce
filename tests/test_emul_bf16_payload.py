"""bfloat16 templates (MVP_FLAG_TPLATE_BF16) on the emulated product kernels, against the fp32 kernels on the widened template.

A bf16 template is rendered exactly as its fp32 widening, so the forward must be bit-identical to the fp32 run on
`from_bf16(tb)` and the transform gradients equal to it within the order of the fp32 atomics.  The template gradient is
accumulated in bf16, one rounding per reduction; it is checked against the fp32 run's gradient g32 with the gates below,
per tensor.  The run order of the blocks (several OS threads) and, with lane_order="random", of the lanes changes the order
of the reductions, so the template gradient is not deterministic either way.

numpy has no bfloat16: a bf16 tensor is held as uint16 bit patterns here (to_bf16 / from_bf16), and goes through the emulation's
front-end (tests/emul/kernels.py, which takes fp32 arrays) as a float32 array of the same bytes, one word per channel pair
[..., 2].  Its gradient buffers, allocated by the front-end like the template, have the bf16 gradient's size and come back the
same way."""
import ctypes

import numpy as np
import pytest

from tests.helpers import CASES, DENSE_CASES, DENSE_K3, build_case, build_dense_case, relerr, scene_args_np

GATE_MAX, GATE_L1 = 2e-2, 8e-3     # max|dg| <= GATE_MAX * max|g32|,  sum|dg| <= GATE_L1 * sum|g32|
# Every reduction rounds the voxel's running sum to bf16, so the error grows with the reductions a voxel receives and with the
# cancellation among them.  The named cases take 11-14 per voxel per view (the benchmark view about 4).  In the dense heavy-tile
# scenes every ray crosses every slab: the warp-field case, whose path does not merge a batch's samples per cell, takes 107 per
# voxel, and the others see more cancellation.  Measured on the emulation: max 0.05-0.10 and sum 0.019-0.021 for the warp
# field, at most 0.021 and 0.007 for the others.
GATE_DENSE_MAX, GATE_DENSE_L1 = 0.15, 0.05
TRANSFORM_TOL = 1e-5


def to_bf16(x):
    """float32 array -> its bfloat16 rounding (nearest even) as uint16 bit patterns."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def from_bf16(h):
    """uint16 bfloat16 bit patterns -> float32 (exact)."""
    return (np.asarray(h, np.uint16).astype(np.uint32) << 16).view(np.float32)


@pytest.fixture()
def kernels():
    from tests.emul import kernels as k
    k.use_variant(())
    k.load()
    yield k
    k.set_lane_order("forward")
    # the dense scenes leave tiles whose lists were rebuilt in the library's saved-list counters: read them, which resets them,
    # so that a later test of the same process starts from zero
    loaded, rebuilt = ctypes.c_int(), ctypes.c_int()
    k.load().mvp_emul_saved_list_tiles(ctypes.byref(loaded), ctypes.byref(rebuilt))
    k.use_variant(())


def template_grad_errors(gb, g32):
    """(max|dg| / max|g32|, sum|dg| / sum|g32|) of a bf16 template gradient (uint16 bit patterns) against the fp32 one."""
    d = np.abs(from_bf16(gb).astype(np.float64) - g32.astype(np.float64))
    return float(d.max() / max(np.abs(g32).max(), 1e-30)), float(d.sum() / max(np.abs(g32).astype(np.float64).sum(), 1e-30))


def run_pair(kernels, s, grad, gates=(GATE_MAX, GATE_L1), **opts):
    """The scene with its template rounded to bf16, once as bf16 and once widened to fp32.  Checks the contract and returns
    the template-gradient errors and the heavy-tile counts (forward, backward) of the gradient run."""
    from ava256_b200 import lib
    a, kw = scene_args_np(s)
    tb = to_bf16(a[7])
    a32, ab = list(a), list(a)
    a32[7], ab[7] = from_bf16(tb), tb.view(np.float32)                           # bf16 channel pairs in fp32-typed words
    out32, sat32, g32 = kernels.forward_backward(*a32, grad_rayrgba=grad, **kw, **opts)
    heavy32 = kernels.last_heavy_tiles
    flag = lib.FLAG_TPLATE_BF16
    optb = dict(opts, fwd_flags=opts.get("fwd_flags", 0) | flag, bwd_flags=opts.get("bwd_flags", 0) | flag)
    outb, satb, gb = kernels.forward_backward(*ab, grad_rayrgba=grad, **kw, **optb)
    gb[3] = gb[3].view(np.uint16)
    assert kernels.last_heavy_tiles == heavy32
    assert np.array_equal(outb, out32) and np.array_equal(satb, sat32)            # forward: bit-identical
    assert gb[3].shape == tb.shape
    for nm, x, y in zip(("primpos", "primrot", "primscale", "template", "warp"), gb, g32):
        if nm != "template":
            assert np.isfinite(x).all() and relerr(x, y) <= TRANSFORM_TOL, nm
    assert np.isfinite(from_bf16(gb[3])).all()
    emax, el1 = template_grad_errors(gb[3], g32[3])
    assert emax <= gates[0] and el1 <= gates[1], (emax, el1)
    outi, _, _ = kernels.forward_backward(*ab, fwd_flags=flag, **kw, **{k: v for k, v in opts.items() if k == "planes"})
    assert np.array_equal(outi, out32)                                            # inference forward
    return emax, el1, heavy32


@pytest.mark.parametrize("order", ["forward", "random"])
@pytest.mark.parametrize("name", list(CASES))
def test_emulated_bf16_template_named_cases(kernels, name, order):
    """T = 8 (head_small), 16 (head_t16), runtime dims (gradcheck_*, noncubic, many_views) and algo 1 (warp_*)."""
    s, grad = build_case(name)
    kernels.set_lane_order(order)
    errs = run_pair(kernels, s, grad.numpy())[:2]
    print("bf16 grad_template %s/%s: max %.3g  l1 %.3g" % (name, order, *errs))


@pytest.mark.parametrize("cap", list(DENSE_K3))
@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_emulated_bf16_template_heavy_kernels(kernels, name, cap):
    """Every tile through the 512-entry kernels, with and without the reference's 512 cap."""
    s, grad = build_dense_case(name, cap)
    kernels.set_lane_order("random" if cap == "capped" else "forward")
    emax, el1, heavy = run_pair(kernels, s, grad.numpy(), gates=(GATE_DENSE_MAX, GATE_DENSE_L1))
    N, H, W = s["raypos"].shape[:3]
    assert heavy == (N * -(-H // 4) * -(-W // 8),) * 2
    print("bf16 grad_template dense %s/%s: max %.3g  l1 %.3g" % (name, cap, emax, el1))


@pytest.mark.parametrize("name", ["gradcheck_ragged", "warp_small"])
def test_emulated_bf16_template_gradient_buffers_cleared(kernels, name):
    """The forward's clear of clear_grad_tplate counts bf16 words: every word of the NaN-filled buffer is zero afterwards (a
    clear at fp32 size writes twice the buffer's bytes)."""
    s, grad = build_case(name)
    run_pair(kernels, s, grad.numpy(), clear_in_forward=True)


def test_emulated_bf16_template_zero_grads_flag(kernels):
    """MVP_FLAG_ZERO_GRADS (the op's retain_graph second backward): the library zero-fills the NaN-filled bf16 buffer."""
    from ava256_b200 import lib
    s, grad = build_case("head_small")
    run_pair(kernels, s, grad.numpy(), bwd_flags=lib.FLAG_ZERO_GRADS)


def test_emulated_bf16_template_image_planes(kernels):
    s, grad = build_case("gradcheck_small")
    run_pair(kernels, s, grad.numpy(), planes=True)


def test_bf16_helpers_round_to_nearest_even():
    """to_bf16 / from_bf16, the test side's bf16: ties to even, subnormals kept."""
    x = np.array([1.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -2.5, 2.0 ** -130, 3.4e38], np.float32)
    assert np.array_equal(from_bf16(to_bf16(x)), np.array([1.0, 1.0, 1.0 + 2.0 ** -6, -2.5, 2.0 ** -130, np.inf], np.float32))
