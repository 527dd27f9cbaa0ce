"""Cost of the backward's gradient sets at the benchmark launch (80 views, 1024x667, K = 16384, 8^3, bench scene, rays generated in
the kernels from the cameras), fp32 and bf16 templates.  Four backwards through the C-ABI, alternated in one process after a warm-up
of each, three rounds, CUDA events, medians:
  plain        mvp_raymarch_backward, every primitive gradient (the training step's backward)
  rays_all     mvp_raymarch_backward_rays, every primitive gradient and the rays (camera refinement while training)
  rays_nopay   mvp_raymarch_backward_rays with MVP_FLAG_NO_TPLATE_GRAD: transforms and rays, no template gradient
  rays_only    mvp_raymarch_backward_rays with MVP_FLAG_RAY_GRADS_ONLY: a frozen avatar, the rays alone
Each backward zero-fills the buffers of its set (MVP_FLAG_ZERO_GRADS), like scripts/time_camera_grads.py.  Then the peak memory
(torch.cuda.max_memory_allocated above what the scene holds) of one autograd step, mvpraymarch_camera forward + backward, with the
inputs of each set requiring grad.  Prints one JSON line per template type, with the card's name and power limit.

    python scripts/time_grad_select.py [--views 80] [--iters 5]
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

SETS = ("plain", "rays_all", "rays_nopay", "rays_only")


def measure(args, s, cams, tpl, card):
    from ava256_b200 import lib, scene
    from ava256_b200.op import mvpraymarch_camera
    N, H, W, K, T = args.views, 1024, 667, 16384, 8
    dev = tpl.device
    bf16 = tpl.dtype == torch.bfloat16
    tflags = lib.tplate_flags(bf16)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    cam = lib.Camera(P(cams[0]), P(cams[1]), P(cams[2]), P(cams[3]), scene.VOLRADIUS, 0)
    shape = lib.Shape(N, H, W, K, T, T, T)
    wsb = lib.workspace_bytes(N, H, W, K, T, T, T)
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rgba = torch.empty(N, H, W, 4, device=dev)
    rsat = torch.empty(N, H, W, 3, device=dev)
    raux = torch.empty(N, H, W, 4, dtype=torch.int32, device=dev)
    grads = [torch.empty_like(s[k]) for k in ("primpos", "primrot", "primscale")] + [torch.empty_like(tpl)]
    fa = lib.ForwardArgs()
    fa.shape, fa.stepsize, fa.fadescale, fa.fadeexp, fa.flags = shape, s["stepsize"], 8.0, 8.0, tflags
    fa.camera = cam
    fa.primpos, fa.primrot, fa.primscale, fa.tplate = P(s["primpos"]), P(s["primrot"]), P(s["primscale"]), P(tpl)
    fa.rayrgba, fa.raysat, fa.rayaux = P(rgba), P(rsat), P(raux)
    fa.workspace, fa.workspace_bytes = P(ws), wsb
    lib.check(lib.LIB.mvp_raymarch_forward(ctypes.byref(fa), st))
    gout = torch.randn(N, H, W, 4, device=dev, generator=torch.Generator(device=dev).manual_seed(7))
    rays = [torch.empty(N, H, W, c, device=dev) for c in (3, 3, 2)]

    def args_for(extra, with_tf, with_tpl):
        ba = lib.BackwardArgs()
        ba.shape, ba.stepsize, ba.fadescale, ba.fadeexp = shape, fa.stepsize, 8.0, 8.0
        ba.flags = lib.FLAG_ACCEL_VALID | lib.FLAG_ZERO_GRADS | tflags | extra
        ba.camera = cam
        ba.primpos, ba.primrot, ba.primscale, ba.tplate = fa.primpos, fa.primrot, fa.primscale, fa.tplate
        ba.grad_rayrgba, ba.raysat, ba.rayaux = P(gout), P(rsat), P(raux)
        if with_tf:
            ba.grad_primpos, ba.grad_primrot, ba.grad_primscale = (P(g) for g in grads[:3])
        if with_tpl:
            ba.grad_tplate = P(grads[3])
        ba.workspace, ba.workspace_bytes = P(ws), wsb
        return ba

    calls = {
        "plain": (args_for(0, True, True), False),
        "rays_all": (args_for(0, True, True), True),
        "rays_nopay": (args_for(lib.FLAG_NO_TPLATE_GRAD, True, False), True),
        "rays_only": (args_for(lib.FLAG_RAY_GRADS_ONLY, False, False), True),
    }

    def run(name):
        ba, with_rays = calls[name]
        if with_rays:
            lib.check(lib.LIB.mvp_raymarch_backward_rays(ctypes.byref(ba), *(P(r) for r in rays), st))
        else:
            lib.check(lib.LIB.mvp_raymarch_backward(ctypes.byref(ba), st))

    def timed(name):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            run(name)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.iters

    for name in SETS:                       # warm-up
        run(name)
    torch.cuda.synchronize()
    res = {k: [] for k in SETS}
    for _ in range(3):
        for name in SETS:
            res[name].append(timed(name))
    med = {k: statistics.median(v) for k, v in res.items()}
    del ws, rgba, rsat, raux, grads, rays, calls
    torch.cuda.empty_cache()

    # peak memory of one autograd step per set: which inputs require grad picks the set
    wants = {"plain": (False, True, True), "rays_all": (True, True, True), "rays_nopay": (True, True, False),
             "rays_only": (True, False, False)}
    peak = {}
    for name in SETS:
        cam_grad, tf_grad, tpl_grad = wants[name]
        leaves = [c.clone().requires_grad_(cam_grad) for c in cams]
        prims = [s[k].detach().requires_grad_(tf_grad) for k in ("primpos", "primrot", "primscale")]
        t = tpl.detach().requires_grad_(tpl_grad)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = mvpraymarch_camera(*leaves, (W, H), scene.VOLRADIUS, s["stepsize"], tuple(prims), t, None, camera_grad=cam_grad,
                                 fadescale=8.0, fadeexp=8.0)
        out.backward(gout)
        torch.cuda.synchronize()
        peak[name] = (torch.cuda.max_memory_allocated() - base) / 1e9
        del out, leaves, prims, t
    return {
        "what": "backward gradient sets at %d views %dx%d K=%d %d^3, rays from the cameras, %s template" % (N, H, W, K, T,
                                                                                                     "bf16" if bf16 else "fp32"),
        "gpu": card,
        "backward_ms": med, "backward_us_per_view": {k: 1e3 * v / N for k, v in med.items()},
        "step_peak_GB": peak, "template_GB": tpl.numel() * tpl.element_size() / 1e9, "rounds_ms": res,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=80)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    from ava256_b200 import lib, scene
    lib.require_grad_select()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    card = q.splitlines()[0] if q else torch.cuda.get_device_name()
    N, H, W, K, T = args.views, 1024, 667, 16384, 8
    dev = torch.device("cuda")
    s = scene.make_scene(N, H, W, K, T, seed=1112, device=dev, alpha_mu=17.0, alpha_sigma=6.0)
    cams = [c.to(dev) for c in scene.make_cameras(N, H, W)]
    for dtype in (torch.float32, torch.bfloat16):
        tpl = s["template"] if dtype == torch.float32 else s["template"].to(torch.bfloat16)
        print(json.dumps(measure(args, s, cams, tpl, card)), flush=True)
        del tpl
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
