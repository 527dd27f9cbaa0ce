"""fp32 against bf16 template payloads at the benchmark launch: 80 views of 1024x667, K = 16384 slabs of 8^3, the benchmark's
scene (seed 1112, alpha 17 / 6).  The two payload types are timed in alternation in one process: forward and backward kernel
time per view (CUDA events around the op's forward and backward), and the peak device memory of each step with its template.
Also printed: the algorithmic bytes per view from the shapes, the GPU's name and power limit (read as bench.py reads them).

  python scripts/time_bf16_payload.py [--views 80] [--reps 3] [--out FILE.json]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import device_record  # noqa: E402
from ava256_b200 import scene  # noqa: E402
from ava256_b200.op import mvpraymarch  # noqa: E402

H, W, K, T = 1024, 667, 16384, 8
ALPHA_MU, ALPHA_SIGMA = 17.0, 6.0


def algorithmic_bytes(voxel_bytes):
    """Bytes per view the kernels must move at least: forward reads the template, primitives and rays and writes the image and
    the saturation records; backward reads the template, primitives, rays, records and the image gradient and writes the template
    and primitive gradients."""
    tpl = K * T ** 3 * voxel_bytes
    prims = K * (3 + 9 + 3) * 4
    rays = H * W * (3 + 3 + 2) * 4
    records = H * W * (3 + 4) * 4
    image = H * W * 4 * 4
    return {"forward": tpl + prims + rays + image + records, "backward": 2 * tpl + 2 * prims + rays + records + image}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=80)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_bf16_payload.py measures on a GPU; none is available")
    dev = torch.device("cuda")
    N = a.views
    s = scene.make_scene(N, H, W, K, T, seed=1112, device=dev, alpha_mu=ALPHA_MU, alpha_sigma=ALPHA_SIGMA)
    tpl32 = s.pop("template")
    grad = torch.randn(N, H, W, 4, device=dev, generator=torch.Generator(device=dev).manual_seed(1112))
    prims = [s[n].requires_grad_(True) for n in ("primpos", "primrot", "primscale")]
    res = {"fp32": {"fwd_us": [], "bwd_us": [], "peak_bytes": []}, "bf16": {"fwd_us": [], "bwd_us": [], "peak_bytes": []}}

    def step(tag, timed):
        t = (tpl32 if tag == "fp32" else tpl32.to(torch.bfloat16)).detach().requires_grad_(True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated() - t.numel() * t.element_size()   # the peak below counts the template
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        out = mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], tuple(prims), t, None, fadescale=8.0, fadeexp=8.0)
        e[1].record()
        gs = torch.autograd.grad(out, prims + [t], grad)
        e[2].record()
        torch.cuda.synchronize()
        if timed:
            r = res[tag]
            r["fwd_us"].append(e[0].elapsed_time(e[1]) * 1e3 / N)
            r["bwd_us"].append(e[1].elapsed_time(e[2]) * 1e3 / N)
            r["peak_bytes"].append(torch.cuda.max_memory_allocated() - base)
        del out, gs, t

    for tag in ("fp32", "bf16"):
        step(tag, False)                                           # warm-up of both
    for _ in range(a.reps):
        for tag in ("fp32", "bf16"):
            step(tag, True)
    rec = {"device": device_record(torch.cuda.current_device()), "views": N, "H": H, "W": W, "K": K, "T": T,
           "algorithmic_bytes_per_view": {"fp32": algorithmic_bytes(16), "bf16": algorithmic_bytes(8)}, "runs": res,
           "median": {tag: {k: sorted(v)[len(v) // 2] for k, v in r.items()} for tag, r in res.items()}}
    print(json.dumps(rec))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
