"""The camera form with a pixelcoords tensor (rays generated in the render kernels at the caller's sample positions) against the
two-call form it replaces and the tuple form, through the public op with autograd:
  two_call      compute_raydirs(viewpos, viewrot, focal, princpt, pixelcoords, volradius) -> mvpraymarch(...)
  fused_tensor  mvpraymarch_camera(viewpos, viewrot, focal, princpt, pixelcoords, ...)   (mvp_raymarch_forward_pixels)
  fused_tuple   mvpraymarch_camera(viewpos, viewrot, focal, princpt, (W, H), ...)        (the integer grid, no coordinate reads)
pixelcoords is the integer pixel grid as the ava-256 dataset builds it, a [N,H,W,2] float32 meshgrid, so all three render the same
image.  Shapes: c3 = 80 views of 1024x667, K = 16384, 8^3, the benchmark's scene; ava = 4 views of 512x334 (ava-256's per-GPU
training shape) with per-view primitives.  The outputs are checked first (images bit-identical, gradients within 1e-5 of max|.|);
then one forward + backward step of each form, alternated over rounds after a warm-up, CUDA events, medians; then the peak memory
of one step above what the inputs hold.  Prints one JSON line per shape, with the card's name and power limit.

    python scripts/time_camera_pixels.py [--shapes c3,ava] [--iters 5] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FORMS = ("two_call", "fused_tensor", "fused_tuple")
NAMES = ("primpos", "primrot", "primscale", "template")
SHAPES = {"c3": (80, 1024, 667, 16384, 8), "ava": (4, 512, 334, 16384, 8)}


def relerr(a, b):
    """max|a - b| / max|b|, one view at a time (the per-view gradients of the c3 shape are 10.7 GB)."""
    d = max(float((x - y).abs().max()) for x, y in zip(a, b))
    return d / max(float(b.abs().max()), 1e-30)


def measure(shape, args, card):
    from ava256_b200 import scene
    from ava256_b200.op import mvpraymarch, mvpraymarch_camera
    from extensions.utils.utils import compute_raydirs
    N, H, W, K, T = SHAPES[shape]
    dev = torch.device("cuda")
    cams = tuple(t.to(dev) for t in scene.make_cameras(N, H, W))
    s = scene.make_scene(N, H, W, K, T, device=dev)
    prims = {nm: s[nm].contiguous() for nm in NAMES}
    del s
    py, px = torch.meshgrid(torch.arange(H, dtype=torch.float32, device=dev), torch.arange(W, dtype=torch.float32, device=dev),
                            indexing="ij")
    pixelcoords = torch.stack([px, py], -1)[None].repeat(N, 1, 1, 1).contiguous()
    gout = torch.randn(N, H, W, 4, device=dev, generator=torch.Generator(device=dev).manual_seed(7))
    step = 1.0 / scene.VOLRADIUS

    def run(name, lv):
        tf = (lv["primpos"], lv["primrot"], lv["primscale"])
        if name == "two_call":
            rp, rd, tmm = compute_raydirs(*cams, pixelcoords, scene.VOLRADIUS)
            return mvpraymarch(rp, rd, step, tmm, tf, lv["template"], None)
        pc = pixelcoords if name == "fused_tensor" else (W, H)
        return mvpraymarch_camera(*cams, pc, scene.VOLRADIUS, step, tf, lv["template"], None)

    def fwd_bwd(name):
        lv = {nm: prims[nm].detach().requires_grad_(True) for nm in NAMES}
        out = run(name, lv)
        out.backward(gout)
        return out.detach(), {nm: x.grad for nm, x in lv.items()}

    ref_img, ref_g = fwd_bwd("two_call")
    check = {}
    for name in FORMS[1:]:
        img, g = fwd_bwd(name)
        check[name] = {"image_equal": bool(torch.equal(img, ref_img)), **{nm: relerr(g[nm], ref_g[nm]) for nm in NAMES}}
        assert check[name]["image_equal"] and all(check[name][nm] <= 1e-5 for nm in NAMES), (name, check[name])
        del img, g
    alpha = float(ref_img[..., 3].max())
    del ref_img, ref_g
    torch.cuda.synchronize()

    def timed(name):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            fwd_bwd(name)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.iters

    for name in FORMS:
        fwd_bwd(name)
    torch.cuda.synchronize()
    res = {k: [] for k in FORMS}
    for _ in range(args.rounds):
        for name in FORMS:
            res[name].append(timed(name))
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
    return {
        "what": "%s: %d views %dx%d K=%d %d^3 per-view primitives, fp32 template, forward + backward through the op" % (shape, N, H, W, K, T),
        "gpu": card, "max_alpha": alpha,
        "step_ms": {k: statistics.median(v) for k, v in res.items()},
        "step_peak_GB": peak, "check_vs_two_call": check, "rounds_ms": res,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c3,ava")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    from ava256_b200 import lib
    lib.require_camera_pixels()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    card = q.splitlines()[0] if q else torch.cuda.get_device_name()
    for shape in args.shapes.split(","):
        print(json.dumps(measure(shape, args, card)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
