"""bf16 templates with fp32 gradient accumulation (`template_grad_dtype=torch.float32`) at the benchmark launch: 80 views of
1024x667, K = 16384 slabs of 8^3, the benchmark's scene (seed 1112, alpha 17 / 6).  Three configurations are timed in alternation
in one process, one warm-up and --reps rounds:

  fp32        fp32 template, fp32 gradient
  bf16        bf16 template, bf16 gradient (accumulated in bf16, one rounding per reduction)
  bf16_f32    bf16 template, fp32 gradient (MVP_FLAG_GRAD_TPLATE_F32), cast to bf16 by autograd

each in two forms: the per-view template [N,K,...] and the shared-primitive template [1,K,...] into which all views reduce.
Per configuration: the forward and backward KERNEL time per view (CUDA events around the library's mvp_raymarch_forward /
mvp_raymarch_backward calls, which launch nothing else), the backward step per view (events around autograd.grad, which includes
autograd's cast of the fp32 gradient), and the step's peak device memory with its template, the cast's temporary included.
Also printed: the GPU's name and power limit (read as bench.py reads them).

  python scripts/time_bf16_grad_f32.py [--views 80] [--reps 3] [--out FILE.json]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import device_record  # noqa: E402
from ava256_b200 import lib, scene  # noqa: E402
from ava256_b200.op import mvpraymarch, template_grad_dtype  # noqa: E402

H, W, K, T = 1024, 667, 16384, 8
ALPHA_MU, ALPHA_SIGMA = 17.0, 6.0
CONFIGS = ("fp32", "bf16", "bf16_f32")


class KernelTimer:
    """Events around every call of the named C-ABI entry points (wrapped in place, restored on exit)."""

    def __init__(self, *names):
        self.names, self.events = names, {n: [] for n in names}

    def __enter__(self):
        self.orig = {n: getattr(lib.LIB, n) for n in self.names}
        for n in self.names:
            def f(*a, _n=n):
                e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                e[0].record()
                rc = self.orig[_n](*a)
                e[1].record()
                self.events[_n].append(e)
                return rc
            setattr(lib.LIB, n, f)
        return self

    def __exit__(self, *exc):
        for n, f in self.orig.items():
            setattr(lib.LIB, n, f)

    def ms(self, name):
        (e,) = self.events[name]
        return e[0].elapsed_time(e[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=80)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_bf16_grad_f32.py measures on a GPU; none is available")
    dev = torch.device("cuda")
    N = a.views
    s = scene.make_scene(N, H, W, K, T, seed=1112, device=dev, alpha_mu=ALPHA_MU, alpha_sigma=ALPHA_SIGMA)
    tpl32 = s.pop("template")
    grad = torch.randn(N, H, W, 4, device=dev, generator=torch.Generator(device=dev).manual_seed(1112))
    forms = {"per_view": {k: s[k] for k in ("primpos", "primrot", "primscale")},
             "shared": {k: s[k][:1].contiguous() for k in ("primpos", "primrot", "primscale")}}
    res = {f: {c: {"fwd_kernel_us": [], "bwd_kernel_us": [], "bwd_step_us": [], "peak_bytes": []} for c in CONFIGS} for f in forms}

    def step(form, cfg, timed):
        src = tpl32 if form == "per_view" else tpl32[:1]
        t = (src if cfg == "fp32" else src.to(torch.bfloat16)).detach().requires_grad_(True)
        prims = [x.detach().requires_grad_(True) for x in forms[form].values()]
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated() - t.numel() * t.element_size()   # the peak below counts the template
        with KernelTimer("mvp_raymarch_forward", "mvp_raymarch_backward") as kt, \
                template_grad_dtype(torch.float32 if cfg == "bf16_f32" else None):
            out = mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], tuple(prims), t, None, fadescale=8.0, fadeexp=8.0)
            e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            e[0].record()
            gs = torch.autograd.grad(out, prims + [t], grad)
            e[1].record()
            torch.cuda.synchronize()
        assert gs[3].dtype == t.dtype
        if timed:
            r = res[form][cfg]
            r["fwd_kernel_us"].append(kt.ms("mvp_raymarch_forward") * 1e3 / N)
            r["bwd_kernel_us"].append(kt.ms("mvp_raymarch_backward") * 1e3 / N)
            r["bwd_step_us"].append(e[0].elapsed_time(e[1]) * 1e3 / N)
            r["peak_bytes"].append(torch.cuda.max_memory_allocated() - base)
        del out, gs, t, prims

    for form in forms:
        for cfg in CONFIGS:
            step(form, cfg, False)                                 # warm-up of every configuration
    for _ in range(a.reps):
        for form in forms:
            for cfg in CONFIGS:
                step(form, cfg, True)
    rec = {"device": device_record(torch.cuda.current_device()), "views": N, "H": H, "W": W, "K": K, "T": T,
           "kernel_build": lib.LIB.mvp_build_config().decode(), "runs": res,
           "median": {f: {c: {k: sorted(v)[len(v) // 2] for k, v in r.items()} for c, r in rf.items()} for f, rf in res.items()}}
    print(json.dumps(rec))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
