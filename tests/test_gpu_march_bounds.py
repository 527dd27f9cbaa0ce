"""GPU tests (`pytest -m gpu`) of the step intervals of the render kernels where the marched positions leave the unit cube: the
scenes of tests/test_emul_march_bounds.py (a thin slab's face between the exact and the drifted position of one step) through
the C-ABI and through the drop-in mvpraymarch, and the small head scene moved off the cube, each against the fp32 oracle."""
import numpy as np
import pytest
import torch

from tests.helpers import abi_raymarch, build_case, relerr, scene_args_np
from tests.test_emul_march_bounds import BINADES, DIRS, OWARP, drift_scene, grad_of, pad_slabs
from tests.test_gpu_parity import BWD_TOL, FWD_TOL, run_ours

pytestmark = pytest.mark.gpu

NAMES = ("primpos", "primrot", "primscale", "template")
KEYS = ("raypos", "raydir", "stepsize", "tminmax") + NAMES


def as_scene(a, kw):
    s = {k: (torch.from_numpy(np.ascontiguousarray(v)) if isinstance(v, np.ndarray) else v) for k, v in zip(KEYS, a)}
    s.update(kw)
    return s


def check_both(a, kw, blocksize=OWARP):
    """abi_raymarch and mvpraymarch on scene (a, kw) against the oracle: images and raysat at the suite's forward gate, the
    gradients at its gradient gate."""
    from oracle import oracle
    grad = torch.from_numpy(grad_of(a))
    ref, rsat = oracle.forward(*a, **kw, blocksize=blocksize)
    gref = oracle.backward(*a, grad.numpy(), rsat, **kw, blocksize=blocksize)
    s = as_scene(a, kw)
    out, sat, grads, _ = abi_raymarch({k: (v.cuda() if torch.is_tensor(v) else v) for k, v in s.items()}, grad.cuda())
    assert relerr(out.cpu().numpy(), ref) <= FWD_TOL and relerr(sat.cpu().numpy(), rsat) <= FWD_TOL
    for nm, g, r in zip(NAMES, grads, gref):
        assert torch.isfinite(g).all() and relerr(g.cpu().numpy(), r) <= BWD_TOL, ("abi", nm)
    out, grads = run_ours(s, grad)
    assert relerr(out, ref) <= FWD_TOL
    for nm, g, r in zip(NAMES, grads, gref):
        assert relerr(g, r) <= BWD_TOL, ("mvpraymarch", nm)


@pytest.mark.parametrize("drift", ["lead", "lag"])
@pytest.mark.parametrize("direction", list(DIRS))
@pytest.mark.parametrize("binade", list(BINADES))
def test_drift_vs_oracle(binade, direction, drift):
    a, kw, _ = drift_scene(BINADES[binade], direction, drift)
    check_both(a, kw)


@pytest.mark.parametrize("drift", ["lead", "lag"])
def test_drift_heavy_kernels_and_long_march(drift):
    """The 512-entry kernels (list padded past 256 entries) and a march of 33000 steps (saturated int16 step intervals)."""
    a, kw, _ = drift_scene(8.0, "diag", drift)
    check_both(pad_slabs(a, 300), kw)
    a, kw, _ = drift_scene(8.0, "diag", drift, steps=33000, dt_target=2e-4)
    check_both(a, kw)


@pytest.mark.parametrize("dist", [100.0, 1000.0])
def test_far_origin(dist):
    for shift in range(8):
        a, kw, _ = drift_scene(0.5, "diag", "lead", steps=200, tmin=dist - 0.3, origin=-dist * DIRS["diag"], shift=shift * 1e-3 / 8)
        check_both(a, kw)


def test_head_scene_off_the_cube():
    """The small head scene with its slabs and ray origins moved by (8, 8, 8)."""
    s, grad = build_case("head_small")
    for k in ("raypos", "primpos"):
        s[k] = s[k] + 8.0
    a, kw = scene_args_np(s)
    from oracle import oracle
    ref, rsat = oracle.forward(*a, **kw)
    gref = oracle.backward(*a, grad.numpy(), rsat, **kw)
    out, sat, grads, _ = abi_raymarch({k: (v.cuda() if torch.is_tensor(v) else v) for k, v in s.items()}, grad.cuda())
    assert relerr(out.cpu().numpy(), ref) <= FWD_TOL and relerr(sat.cpu().numpy(), rsat) <= FWD_TOL
    for nm, g, r in zip(NAMES, grads, gref):
        assert relerr(g.cpu().numpy(), r) <= BWD_TOL, nm
    out, grads = run_ours(s, grad)
    assert relerr(out, ref) <= FWD_TOL
    for nm, g, r in zip(NAMES, grads, gref):
        assert relerr(g, r) <= BWD_TOL, nm
