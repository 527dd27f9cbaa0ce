"""fp32 against bf16 payload hand-off, timed in alternation in one process (one warm-up of both, then --reps rounds each, CUDA
events, device synchronised before each reading):

  (a) assemble_payload forward and backward at one subject of the benchmark: tex [1,24,1024,1024], opacity [1,8,1024,1024],
      K = 16384 slabs of 8^3; GB/s from the algorithmic bytes (fp32: 16 + 16 B per texel forward, 32 + 16 backward; bf16:
      16 + 8 forward, 16 + 16 backward) and their share of the H100 SXM data-sheet 3.35 TB/s;
  (b) expand_views of the template to 80 views, sum_views of 80 template-sized gradients (bf16: into bf16, and into fp32 as
      GradReducer.reduce does) and GradReducer.reduce itself;
  (c) the one-subject step on the benchmark scene (80 x 1024x667, seed 1112, alpha 17 / 6): assemble -> expand -> op forward +
      backward -> expand adjoint -> assemble backward, per stage, with torch.cuda.max_memory_allocated.

The GPU's name and power limit are read in the same process (as bench.py reads them).

  python scripts/time_bf16_handoff.py [--views 80] [--reps 3] [--out FILE.json]
"""
import argparse
import gc
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import device_record  # noqa: E402
from ava256_b200 import scene  # noqa: E402
from ava256_b200.op import mvpraymarch  # noqa: E402
from ava256_b200.parallel import GradReducer  # noqa: E402
from ava256_b200.payload import assemble_payload, expand_views, sum_views  # noqa: E402

H, W, K, T = 1024, 667, 16384, 8
HB = WB = 128
TEXELS = K * T ** 3
PEAK_BW = 3.35e12
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}
PAYLOAD_BYTES = {"fp32": {"fwd": 32, "bwd": 48}, "bf16": {"fwd": 24, "bwd": 32}}   # per texel


def _images(tpl):
    t = tpl.view(HB, WB, T, T, T, 4)
    tex = ((t[..., :3] - 100.0) / 25.0).permute(2, 5, 0, 3, 1, 4).reshape(1, 3 * T, HB * T, WB * T).contiguous()
    opa = t[..., 3].permute(2, 0, 3, 1, 4).reshape(1, T, HB * T, WB * T).contiguous()
    return tex, opa


class Timer:
    def __init__(self):
        self.ev = []

    def mark(self, name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.ev.append((name, e))

    def ms(self):
        torch.cuda.synchronize()
        return {n: a.elapsed_time(b) for (_, a), (n, b) in zip(self.ev[:-1], self.ev[1:])}


def time_payload(tag, tex, opa, reps=10):
    """(a): forward and backward of the hand-off alone, mean of `reps` back-to-back calls."""
    dt = DTYPES[tag]
    t, o = tex.detach().requires_grad_(True), opa.detach().requires_grad_(True)
    g = torch.randn(1, K, T, T, T, 4, device="cuda").to(dt)
    tm = Timer()
    tm.mark("start")
    for _ in range(reps):
        tp = assemble_payload(t, o, boxsize=T, dtype=dt)
    tm.mark("fwd")
    for _ in range(reps):
        gt, go = torch.autograd.grad(tp, (t, o), g, retain_graph=True)
    tm.mark("bwd")
    ms = tm.ms()
    r = {}
    for k in ("fwd", "bwd"):
        us = ms[k] * 1e3 / reps
        gbs = PAYLOAD_BYTES[tag][k] * TEXELS / (us * 1e-6) / 1e9
        r[k + "_us"], r[k + "_GBps"], r[k + "_share_of_3.35TBps"] = us, gbs, gbs * 1e9 / PEAK_BW
    return r


def time_views(tag, tp, nv, reps=3):
    """(b): expand to nv views; sum of nv template-sized gradients (bf16 into bf16 and into fp32); GradReducer.reduce."""
    dt = DTYPES[tag]
    g = torch.randn(nv, K, T, T, T, 4, device="cuda").to(dt)
    rest = [torch.randn(nv, K, 3, device="cuda"), torch.randn(nv, K, 3, 3, device="cuda"), torch.randn(nv, K, 3, device="cuda")]
    red = GradReducer(K, T, T, T, "cuda")
    f32 = torch.empty(TEXELS * 4, device="cuda")
    tm = Timer()
    tm.mark("start")
    for _ in range(reps):
        y = expand_views(tp, nv)
    tm.mark("expand")
    del y
    for _ in range(reps):
        sum_views(g)
    tm.mark("sum")
    for _ in range(reps):
        sum_views(g, f32)
    tm.mark("sum_to_fp32")
    for _ in range(reps):
        red.reduce(g, *rest)
    tm.mark("reducer")
    ms = tm.ms()
    red.finish()
    b = g.element_size() * TEXELS * 4
    r = {k + "_ms": v / reps for k, v in ms.items()}
    r["expand_GBps"] = (b + nv * b) / (r["expand_ms"] * 1e-3) / 1e9
    r["sum_GBps"] = (nv * b + b) / (r["sum_ms"] * 1e-3) / 1e9
    return r


def time_step(tag, s, tex, opa, grad, nv):
    """(c): the one-subject step, per stage, and its peak memory above what was allocated before it."""
    dt = DTYPES[tag]
    t, o = tex.detach().requires_grad_(True), opa.detach().requires_grad_(True)
    gc.collect()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    tm = Timer()
    tm.mark("start")
    tp = assemble_payload(t, o, boxsize=T, dtype=dt)
    tm.mark("assemble")
    tpv = expand_views(tp[0], nv)
    tm.mark("expand")
    out = mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], (s["primpos"], s["primrot"], s["primscale"]), tpv,
                      None, fadescale=8.0, fadeexp=8.0)
    tm.mark("op_forward")
    gtpv, = torch.autograd.grad(out, tpv, grad)
    tm.mark("op_backward")
    gtp = sum_views(gtpv)
    tm.mark("expand_adjoint")
    gt, go = torch.autograd.grad(tp[0], (t, o), gtp)
    tm.mark("assemble_backward")
    r = {k + "_ms": v for k, v in tm.ms().items()}
    r["step_ms"] = sum(r.values())
    r["peak_bytes"] = torch.cuda.max_memory_allocated() - base
    del out, gtpv, gtp, gt, go, tpv, tp
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=80)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_bf16_handoff.py measures on a GPU; none is available")
    nv = a.views
    s = scene.make_scene(nv, H, W, K, T, seed=1112, device="cuda", alpha_mu=17.0, alpha_sigma=6.0)
    tpl = s.pop("template")[0].clone()
    gc.collect()
    torch.cuda.empty_cache()
    tex, opa = _images(tpl)
    del tpl
    grad = torch.randn(nv, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1112))
    res = {tag: {"payload": [], "views": [], "step": []} for tag in DTYPES}

    def round_(timed):
        for tag in DTYPES:
            p = time_payload(tag, tex, opa)
            with torch.no_grad():
                tp = assemble_payload(tex, opa, boxsize=T, dtype=DTYPES[tag])[0]
            v = time_views(tag, tp, nv)
            del tp
            gc.collect()
            torch.cuda.empty_cache()
            st = time_step(tag, s, tex, opa, grad, nv)
            gc.collect()
            torch.cuda.empty_cache()
            if timed:
                res[tag]["payload"].append(p)
                res[tag]["views"].append(v)
                res[tag]["step"].append(st)

    round_(False)                                                     # warm-up of both
    for _ in range(a.reps):
        round_(True)
    med = {}
    for tag, r in res.items():
        med[tag] = {}
        for part, runs in r.items():
            med[tag][part] = {k: sorted(x[k] for x in runs)[len(runs) // 2] for k in runs[0]}
    rec = {"device": device_record(torch.cuda.current_device()), "views": nv, "H": H, "W": W, "K": K, "T": T,
           "payload_bytes_per_texel": PAYLOAD_BYTES, "median": med, "runs": res}
    print(json.dumps(rec))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
