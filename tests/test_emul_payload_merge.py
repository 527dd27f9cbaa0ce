"""The backward merges the payload-gradient updates of the samples of a batch that fall in the same voxel cell, and only the
lowest lane of each such group issues the group's 8 reductions.  These scenes make whole batches land in one cell: the
merge then runs all of its stages (groups of up to 32 lanes), and short batches leave idle lanes next to the group.
Checked against the oracle on the emulated kernels (tests/emul), with the emulation's counters showing that the merge ran."""
import ctypes

import numpy as np
import pytest

from tests.helpers import gradcheck_like_scene, relerr, scene_args_np

BWD_TOL = 1e-4


def one_cell_scene(M, shared_path):
    """One slab of M^3 voxels in front of 8x16 pinhole rays.  M = 2: a single voxel cell, every sample of a batch is in it.
    shared_path: all rays start at the same point on the same t lattice and differ in direction by 1e-5, so the 32 samples a
    tile takes at one lattice step share a cell for any M."""
    s = gradcheck_like_scene(N=1, H=8, W=16, k3=1, M=M, seed=21, alpha_gain=4.0)
    if shared_path:
        H, W = s["raypos"].shape[1:3]
        py, px = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
        d = np.stack([1e-5 * (px - W / 2), 1e-5 * (py - H / 2), np.ones_like(px)], -1)
        d /= np.linalg.norm(d, axis=-1, keepdims=True)
        s["raydir"][0] = s["raydir"].new_tensor(d)
        s["tminmax"][..., 0], s["tminmax"][..., 1] = 2.0, 6.5
    return s


CASES = {"single_cell_generic": (2, False), "shared_path_t8": (8, True), "shared_path_generic": (4, True)}


@pytest.mark.parametrize("order", ["forward", "random"])
@pytest.mark.parametrize("name", list(CASES))
def test_merged_payload_scatter_vs_oracle(name, order):
    import torch
    from oracle import oracle
    from tests.emul import kernels

    s = one_cell_scene(*CASES[name])
    grad = torch.randn(*s["raypos"].shape[:3], 4, generator=torch.Generator().manual_seed(7))
    a, kw = scene_args_np(s)
    kernels.use_variant(("MVP_EMUL_STATS",))
    try:
        L = kernels.load()
        kernels.set_lane_order(order)
        stats, groups = (ctypes.c_longlong * 8)(), (ctypes.c_longlong * 33)()
        L.mvp_emul_bwd_stats(stats)
        L.mvp_emul_bwd_groups(groups)           # reset both
        out, _, grads = kernels.forward_backward(*a, grad_rayrgba=grad.numpy(), **kw)
        L.mvp_emul_bwd_stats(stats)
        L.mvp_emul_bwd_groups(groups)
    finally:
        kernels.set_lane_order("forward")
        kernels.use_variant(())
    ref, rsat = oracle.forward(*a, **kw)
    assert relerr(out, ref) <= 1e-5
    gref = oracle.backward(*a, grad.numpy(), rsat, **kw)
    for nm, g, r in zip(("primpos", "primrot", "primscale", "template"), grads, gref):
        assert np.isfinite(g).all() and relerr(g, r) <= BWD_TOL, nm
    samples, reds = stats[4], stats[7]
    sizes = np.arange(1, 33)
    assert int((np.array(groups[:32]) * sizes).sum()) == samples      # every sample in exactly one group
    assert reds == 8 * sum(groups[:32])                                 # one set of 8 reductions per group
    assert groups[31] > 0 and 4 * reds < 8 * samples                    # full 32-lane groups, > 4x fewer reductions
