"""Several subjects' views in one raymarch launch (per-view primitive sets, `op.mvpraymarch_sets`) against the two ways a caller had
before: S subjects x V views at 1024x667, K = 16384, 8^3, the benchmark's scene (one subject per seed), fp32 and bf16 templates.
Three forms on the same seeded inputs, their outputs checked equal first (images bit-identical, gradients within 1e-5 of max|.|):
  sets      one mvpraymarch_sets launch over the S*V views, primitives [S,K,...]
  shared    S launches of the shared form, subject s's V views with its primitives [1,K,...]
  expand    payload.expand_views of every subject to its V views, one mvpraymarch launch over [S*V,K,...], payload.sum_views back
            (the adjoint of expand_views) -- what bench.py's end-to-end leg does for one subject
Through the public op (autograd), forward alone (no_grad) and forward + backward, alternated over rounds after a warm-up of each,
CUDA events, medians; then the peak memory of one forward + backward of each form (torch.cuda.max_memory_allocated above what the
inputs hold).  Prints one JSON line per configuration, with the card's name and power limit read in the same process.

    python scripts/time_view_sets.py [--configs 4x20,8x10] [--iters 3] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FORMS = ("sets", "shared", "expand")
NAMES = ("primpos", "primrot", "primscale", "template")


def subjects(S, K, T, dev, dtype):
    from ava256_b200 import scene
    prims = [scene.make_primitives(K, 1112 + 101 * i) for i in range(S)]
    out = {nm: torch.stack([p[j] for p in prims]).to(dev).contiguous() for j, nm in enumerate(NAMES[:3])}
    out["template"] = torch.stack([scene.make_payload(K, T, 1112 + 101 * i, 17.0, 6.0, device=dev) for i in range(S)]).to(dtype)
    return out


def relerr(a, b):
    return float((a.double() - b.double()).abs().max() / max(float(b.double().abs().max()), 1e-30))


def measure(S, V, dtype, args, card):
    from ava256_b200 import scene
    from ava256_b200.op import mvpraymarch, mvpraymarch_sets
    from ava256_b200.payload import expand_views
    N, H, W, K, T = S * V, 1024, 667, 16384, 8
    dev = torch.device("cuda")
    rp, rd, tmm = (t.to(dev) for t in scene.make_rays(N, H, W))
    prims = subjects(S, K, T, dev, dtype)
    view_set = torch.arange(S, device=dev, dtype=torch.int32).repeat_interleave(V)
    gout = torch.randn(N, H, W, 4, device=dev, generator=torch.Generator(device=dev).manual_seed(7))
    step = 1.0 / scene.VOLRADIUS

    def run(name, lv):
        """The form's images, one tensor per launch."""
        tf = (lv["primpos"], lv["primrot"], lv["primscale"])
        if name == "sets":
            return [mvpraymarch_sets(rp, rd, step, tmm, tf, lv["template"], None, view_set)]
        if name == "shared":
            return [mvpraymarch(rp[s * V:(s + 1) * V], rd[s * V:(s + 1) * V], step, tmm[s * V:(s + 1) * V], tuple(x[s:s + 1] for x in tf),
                                lv["template"][s:s + 1], None) for s in range(S)]
        e = [torch.cat([expand_views(lv[nm][s], V) for s in range(S)]) for nm in NAMES]
        return [mvpraymarch(rp, rd, step, tmm, (e[0], e[1], e[2]), e[3], None)]

    def leaves(grad):
        return {nm: prims[nm].detach().requires_grad_(grad) for nm in NAMES}

    def fwd_bwd(name):
        lv = leaves(True)
        outs = run(name, lv)
        torch.autograd.backward(outs, list(gout.split(N // len(outs))))
        return torch.cat([o.detach() for o in outs]), {nm: x.grad for nm, x in lv.items()}

    def fwd(name):
        with torch.no_grad():
            return run(name, leaves(False))

    # outputs first: the three forms compute the same image and gradients (a bf16 template's gradient is accumulated in bf16, in
    # another order per form: its difference is recorded, not gated)
    ref_img, ref_g = fwd_bwd("sets")
    check = {}
    gated = NAMES if dtype == torch.float32 else NAMES[:3]
    for name in FORMS[1:]:
        img, g = fwd_bwd(name)
        check[name] = {"image_equal": bool(torch.equal(img, ref_img)), **{nm: relerr(g[nm], ref_g[nm]) for nm in NAMES}}
        assert check[name]["image_equal"] and all(check[name][nm] <= 1e-5 for nm in gated), (name, check[name])
        del img, g
    sat = float((ref_img[..., 3] >= 0.999).float().mean())
    del ref_img, ref_g
    torch.cuda.synchronize()

    def timed(fn, name):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            fn(name)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.iters

    for name in FORMS:                      # warm-up of every shape
        fwd(name)
        fwd_bwd(name)
    torch.cuda.synchronize()
    res = {k: {"fwd": [], "fwd_bwd": []} for k in FORMS}
    for _ in range(args.rounds):
        for name in FORMS:
            res[name]["fwd"].append(timed(fwd, name))
            res[name]["fwd_bwd"].append(timed(fwd_bwd, name))
    peak = {}
    for name in FORMS:
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        r = fwd_bwd(name)
        torch.cuda.synchronize()
        peak[name] = (torch.cuda.max_memory_allocated() - base) / 1e9
        del r
    tb = prims["template"]
    return {
        "what": "%d subjects x %d views %dx%d K=%d %d^3, %s template: one sets launch vs %d shared-form launches vs expand_views + op + "
                "sum_views" % (S, V, H, W, K, T, "bf16" if dtype == torch.bfloat16 else "fp32", S),
        "gpu": card, "saturated_ray_fraction": sat,
        "fwd_ms": {k: statistics.median(v["fwd"]) for k, v in res.items()},
        "fwd_bwd_ms": {k: statistics.median(v["fwd_bwd"]) for k, v in res.items()},
        "step_peak_GB": peak, "template_GB_per_subject": tb[0].numel() * tb.element_size() / 1e9,
        "check_vs_sets": check, "rounds_ms": res,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="4x20,8x10", help="comma-separated SxV")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from ava256_b200 import lib
    lib.require_view_sets()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    card = q.splitlines()[0] if q else torch.cuda.get_device_name()
    for cfg in args.configs.split(","):
        S, V = (int(x) for x in cfg.split("x"))
        for dtype in (torch.float32, torch.bfloat16):
            print(json.dumps(measure(S, V, dtype, args, card)), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
