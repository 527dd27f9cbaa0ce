"""Cost of the camera gradient at the benchmark launch (80 views, 1024x667, K = 16384, 8^3, bench scene, rays generated in the
kernels from the cameras): the plain backward (mvp_raymarch_backward) against the ray-gradient backward
(mvp_raymarch_backward_rays) plus the ray generator's adjoint (mvp_compute_raydirs_backward), alternated in one process after a
warm-up of both, three rounds, CUDA events, medians.  The adjoint's achieved bandwidth is over its algorithmic bytes: 32 B per ray
read (+ 8 B with a pixelcoords tensor, not used here).  Prints one JSON line with the card's name and power limit.

    python scripts/time_camera_grads.py [--views 80] [--iters 5]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=80)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    from ava256_b200 import lib, scene
    N, H, W, K, T = args.views, 1024, 667, 16384, 8
    dev = torch.device("cuda")
    s = scene.make_scene(N, H, W, K, T, seed=1112, device=dev, alpha_mu=17.0, alpha_sigma=6.0)
    cams = [c.to(dev) for c in scene.make_cameras(N, H, W)]
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    cam = lib.Camera(P(cams[0]), P(cams[1]), P(cams[2]), P(cams[3]), scene.VOLRADIUS, 0)
    shape = lib.Shape(N, H, W, K, T, T, T)
    wsb = lib.workspace_bytes(N, H, W, K, T, T, T)
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rgba = torch.empty(N, H, W, 4, device=dev)
    rsat = torch.empty(N, H, W, 3, device=dev)
    raux = torch.empty(N, H, W, 4, dtype=torch.int32, device=dev)
    grads = [torch.empty_like(s[k]) for k in ("primpos", "primrot", "primscale", "template")]
    fa = lib.ForwardArgs()
    fa.shape, fa.stepsize, fa.fadescale, fa.fadeexp = shape, s["stepsize"], 8.0, 8.0
    fa.camera = cam
    fa.primpos, fa.primrot, fa.primscale, fa.tplate = (P(s[k]) for k in ("primpos", "primrot", "primscale", "template"))
    fa.rayrgba, fa.raysat, fa.rayaux = P(rgba), P(rsat), P(raux)
    fa.workspace, fa.workspace_bytes = P(ws), wsb
    lib.check(lib.LIB.mvp_raymarch_forward(ctypes.byref(fa), st))
    gout = torch.randn(N, H, W, 4, device=dev, generator=torch.Generator(device=dev).manual_seed(7))
    ba = lib.BackwardArgs()
    ba.shape, ba.stepsize, ba.fadescale, ba.fadeexp = shape, fa.stepsize, 8.0, 8.0
    ba.flags = lib.FLAG_ACCEL_VALID | lib.FLAG_ZERO_GRADS
    ba.camera = cam
    ba.primpos, ba.primrot, ba.primscale, ba.tplate = fa.primpos, fa.primrot, fa.primscale, fa.tplate
    ba.grad_rayrgba, ba.raysat, ba.rayaux = P(gout), P(rsat), P(raux)
    ba.grad_primpos, ba.grad_primrot, ba.grad_primscale, ba.grad_tplate = (P(g) for g in grads)
    ba.workspace, ba.workspace_bytes = P(ws), wsb
    rays = [torch.empty(N, H, W, c, device=dev) for c in (3, 3, 2)]
    gcam = [torch.zeros_like(c) for c in cams]

    def plain():
        lib.check(lib.LIB.mvp_raymarch_backward(ctypes.byref(ba), st))

    def with_rays():
        lib.check(lib.LIB.mvp_raymarch_backward_rays(ctypes.byref(ba), *(P(r) for r in rays), st))

    def adjoint():
        lib.check(lib.LIB.mvp_compute_raydirs_backward(N, H, W, *(P(c) for c in cams), None, scene.VOLRADIUS, *(P(r) for r in rays),
                                                       *(P(g) for g in gcam), st))

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.iters

    for fn in (plain, with_rays, adjoint):       # warm-up
        fn()
    torch.cuda.synchronize()
    res = {"plain": [], "rays": [], "adjoint": []}
    for _ in range(3):
        res["plain"].append(timed(plain))
        res["rays"].append(timed(with_rays))
        res["adjoint"].append(timed(adjoint))
    med = {k: statistics.median(v) for k, v in res.items()}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    bytes_adj = 32.0 * N * H * W
    line = {
        "what": "camera gradient cost at %d views %dx%d K=%d %d^3, rays from the cameras" % (N, H, W, K, T),
        "gpu": q.splitlines()[0] if q else torch.cuda.get_device_name(),
        "backward_plain_ms": med["plain"], "backward_rays_ms": med["rays"], "raydirs_backward_ms": med["adjoint"],
        "backward_plain_us_per_view": 1e3 * med["plain"] / N, "backward_rays_us_per_view": 1e3 * med["rays"] / N,
        "raydirs_backward_us_per_view": 1e3 * med["adjoint"] / N,
        "overhead_pct": 100.0 * (med["rays"] + med["adjoint"] - med["plain"]) / med["plain"],
        "raydirs_backward_GBps": bytes_adj / (med["adjoint"] * 1e-3) / 1e9,
        "rounds_ms": res,
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
