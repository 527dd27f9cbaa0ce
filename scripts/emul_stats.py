"""Design study on the CPU emulation (tests/emul): work counters of the emulated forward kernel for one view of the bench
scene, for the default build and for build-time variants.  No GPU needed; counts are exact, times are not GPU times.

  python scripts/emul_stats.py [H W K T [DEFINE ...]]   (default: the C3 view 1024 667 16384 8; extra -D defines = variants)
"""
import ctypes
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ava256_b200 import scene  # noqa: E402
from tests.emul import kernels  # noqa: E402

H, W, K, T = (int(x) for x in sys.argv[1:5]) if len(sys.argv) >= 5 else (1024, 667, 16384, 8)
s = scene.make_scene(1, H, W, K, T, seed=1112, alpha_mu=17.0, alpha_sigma=6.0)
args = [s[k].numpy() if hasattr(s[k], "numpy") else s[k] for k in ("raypos", "raydir", "stepsize", "tminmax", "primpos", "primrot", "primscale", "template")]
NAMES = ("ballots", "events", "events_any_valid", "samples", "flushes", "tiles_with_list", "events_any_inside", "lanes_inside")
ref = None
VARIANTS = [("default", ("MVP_EMUL_STATS",))] + [(d, ("MVP_EMUL_STATS", d)) for d in sys.argv[5:]]
for tag, defs in VARIANTS:
    kernels.use_variant(defs)
    L = kernels.load()
    t0 = time.time()
    grad = np.random.default_rng(1).standard_normal(args[0].shape[:3] + (4,)).astype(np.float32)
    out, _, _ = kernels.forward_backward(*args, grad_rayrgba=grad)
    dt = time.time() - t0
    st = (ctypes.c_longlong * 8)()
    L.mvp_emul_fwd_stats(st)
    L.mvp_emul_list_chunks.restype = ctypes.c_longlong
    chunks = L.mvp_emul_list_chunks()
    print("%-9s %6.1fs  " % (tag, dt) + "  ".join("%s=%d" % (n, v) for n, v in zip(NAMES, st)) + "  list_chunks=%d" % chunks)
    s2 = (ctypes.c_longlong * 8)()
    L.mvp_emul_fwd_stats2(s2)
    print("          forward loop: " + "  ".join("%s=%d" % (n, v) for n, v in zip(("sweep_steps", "skipped_steps", "events_same_slab_as_previous", "words_with_2plus_slabs", "events_in_such_words", "tiles_list_gt128", "tiles_list_gt160", "tiles_list_gt192"), s2)))
    bs = (ctypes.c_longlong * 8)()
    L.mvp_emul_bwd_stats(bs)
    print("          backward: " + "  ".join("%s=%d" % (n, v) for n, v in zip(("slab_visits", "visits_with_work", "warp_steps", "lane_steps", "samples", "batches", "carry_steps", "payload_reds"), bs)))
    # payload-gradient reductions: one per corner of every sample without the per-cell merge, one per corner of every cell
    # group of a batch with it, and one per distinct voxel of a batch if corners shared between neighbouring cells were merged too
    gr = (ctypes.c_longlong * 33)()
    L.mvp_emul_bwd_groups(gr)
    print("          payload reductions: unmerged=%d  per cell=%d (x%.2f fewer)  per voxel=%d (x%.2f fewer)" % (
        8 * bs[4], bs[7], 8 * bs[4] / max(bs[7], 1), gr[32], 8 * bs[4] / max(gr[32], 1)))
    print("          cell group sizes (groups / samples): " + "  ".join(
        "%d:%d/%d" % (g + 1, gr[g], (g + 1) * gr[g]) for g in range(32) if gr[g]))
    if ref is None:
        ref = out
    else:
        print("          same image as default:", bool(np.array_equal(ref, out)))
