"""Price of deterministic primitive gradients (`op.deterministic_grads`) at the benchmark launch: 80 views 1024x667, K = 16384, 8^3,
fp32 and bf16 templates, per-view and shared primitives.  For each configuration:
  * the backward's time (CUDA events around `loss.backward()`, median of --reps) in the default path and in the deterministic one;
  * the deterministic backward split into its measure pass, accumulate pass and conversion (kernel times from torch.profiler in a
    run of its own; kernels named by their template arguments), against the default backward's render kernels;
  * the step's peak memory (torch.cuda.max_memory_allocated over forward + backward) of both.
Prints the card's name and power limit first.  Needs an H100 with about 60 GB free.

    python scripts/time_deterministic.py [--reps 5] [--out time_deterministic.json]"""
import argparse
import json
import os
import re
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def step(s, grad, det, timed=True):
    from ava256_b200 import op
    lv = [s[n].detach().requires_grad_(True) for n in ("primpos", "primrot", "primscale", "template")]
    with op.deterministic_grads(det):
        out = op.mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], (lv[0], lv[1], lv[2]), lv[3], None)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out.backward(grad)
    e1.record()
    torch.cuda.synchronize()
    del out, lv
    return e0.elapsed_time(e1)


def kind(name):
    if "det_convert_kernel" in name:
        return "convert"
    m = re.search(r"render_backward_kernel<(.*)>", name)
    if not m:
        return None
    last = m.group(1).split(",")[-1].strip()
    return {"1": "measure", "2": "accumulate"}.get(last, "default_render")


def profile(s, grad, det):
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        step(s, grad, det)
    agg = {}
    for ev in p.events():
        k = kind(ev.name)
        if k and ev.device_type == torch.autograd.DeviceType.CUDA:
            agg[k] = agg.get(k, 0.0) + ev.device_time / 1e3
    return agg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--views", type=int, default=80)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from ava256_b200 import scene
    res = {"card": card(), "rows": []}
    print("card:", res["card"], flush=True)
    N, H, W, K, T = a.views, 1024, 667, 16384, 8
    grad = torch.randn(N, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))
    for shared in (False, True):
        base = scene.make_scene(N, H, W, K, T, alpha_mu=17.0, alpha_sigma=6.0, device="cuda")
        if shared:                                                   # one subject's primitives [1,K,...] shared by all views
            base = dict(base, **{n: base[n][:1].contiguous() for n in ("primpos", "primrot", "primscale", "template")})
        for dtype in (torch.float32, torch.bfloat16):
            s = dict(base, template=base["template"].to(dtype))
            row = {"prims": "shared" if shared else "per_view", "template": str(dtype).split(".")[-1]}
            for det in (False, True):
                step(s, grad, det)                                   # warm-up
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats()
                ts = sorted(step(s, grad, det) for _ in range(a.reps))
                tag = "det" if det else "default"
                row[tag + "_backward_ms"] = ts[len(ts) // 2]
                row[tag + "_peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
                row[tag + "_kernels_ms"] = profile(s, grad, det)
            print(json.dumps(row), flush=True)
            res["rows"].append(row)
            del s
        del base
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
