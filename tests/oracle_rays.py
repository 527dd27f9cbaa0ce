"""TEST INFRASTRUCTURE -- ctypes front-end of tests/oracle_rays.c: the C oracle's backward with the rays' gradients
(float and double builds in one shared object next to the source), and the torch fp64 restatement of the ray generator
that the camera adjoint is checked against."""
import ctypes
import os
import subprocess

import numpy as np
import torch

from oracle import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "oracle_rays.c")
DEP = [SRC, os.path.join(os.path.dirname(HERE), "oracle", "mvp_oracle.c")]
LIB = os.path.join(HERE, "liboracle_rays.so")
_lib = None


def _load():
    global _lib
    if _lib is None:
        if not (os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(f) for f in DEP)):
            objs = []
            for real, suf in (("float", "f32"), ("double", "f64")):
                obj = LIB[:-3] + "_%s.o" % suf
                subprocess.check_call(["gcc", "-O2", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-std=c11",
                                       "-DREAL=%s" % real, "-DSUFFIX=%s" % suf, "-c", SRC, "-o", obj])
                objs.append(obj)
            subprocess.check_call(["gcc", "-shared", "-fopenmp", "-o", LIB] + objs + ["-lm"])
            for o in objs:
                os.remove(o)
        _lib = ctypes.CDLL(LIB)
    return _lib


def backward_rays(raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template, grad_rayrgba, raysat,
                  fadescale=8.0, fadeexp=8.0, blocksize=(8, 16), maxhitboxes=512, dtype=np.float32, warp=None):
    """oracle.backward plus the rays' gradients.  Returns float64 ((grad_primpos, grad_primrot, grad_primscale, grad_template
    [, grad_warp]), (grad_raypos, grad_raydir, grad_tminmax))."""
    lib = _load()
    suf = "f32" if dtype == np.float32 else "f64"
    raypos, raydir, tminmax, primpos, primrot, primscale, template, grad_rayrgba, raysat = oracle._prep(
        dtype, raypos, raydir, tminmax, primpos, primrot, primscale, template, grad_rayrgba, raysat)
    if warp is not None:
        warp = np.ascontiguousarray(warp, dtype=dtype)
    cfg = oracle._cfg(raypos, primpos, template, stepsize, fadescale, fadeexp, blocksize, maxhitboxes, warp)
    g = [np.zeros(a.shape, np.float64) for a in (primpos, primrot, primscale, template)]
    gw = np.zeros(warp.shape, np.float64) if warp is not None else None
    rays = [np.zeros(raypos.shape, np.float64), np.zeros(raydir.shape, np.float64), np.zeros(tminmax.shape, np.float64)]
    fn = getattr(lib, "mvp_oracle_backward_rays_" + suf)
    fn.restype = ctypes.c_int
    P = oracle._p
    rc = fn(ctypes.byref(cfg), P(raypos), P(raydir), P(tminmax), P(primpos), P(primrot), P(primscale), P(template), P(warp),
            P(grad_rayrgba), P(raysat), P(g[0]), P(g[1]), P(g[2]), P(g[3]), P(gw), P(rays[0]), P(rays[1]), P(rays[2]))
    assert rc == 0
    return tuple(g) + ((gw,) if warp is not None else ()), tuple(rays)


def rays_torch(viewpos, viewrot, focal, princpt, pixelcoords, volradius):
    """The ray formula of compute_raydirs (extensions/utils/utils_kernel.cu:32-46, `scene.compute_raydirs_host`'s arithmetic) in
    differentiable torch, in the dtype of the inputs.  pixelcoords [N,H,W,2] tensor or (W, H)."""
    N = viewpos.shape[0]
    if isinstance(pixelcoords, tuple):
        W, H = pixelcoords
        py, px = torch.meshgrid(torch.arange(H, dtype=viewpos.dtype), torch.arange(W, dtype=viewpos.dtype), indexing="ij")
        pixelcoords = torch.stack([px, py], dim=-1)[None].expand(N, H, W, 2)
    raypos = (viewpos / volradius)[:, None, None, :].expand(pixelcoords.shape[:3] + (3,))
    uv = (pixelcoords - princpt[:, None, None, :]) / focal[:, None, None, :]
    e = torch.cat([uv, torch.ones_like(uv[..., :1])], dim=-1)
    e = torch.einsum("nij,nhwi->nhwj", viewrot, e)                 # viewrot^T (u, v, 1)
    d = e / e.norm(dim=-1, keepdim=True)
    t1 = (-1.0 - raypos) / d
    t2 = (1.0 - raypos) / d
    tmin = torch.clamp(torch.minimum(t1, t2).amax(dim=-1), min=0.0)
    tmax = torch.maximum(t1, t2).amin(dim=-1).detach()             # the march's end is a held decision: no gradient
    return raypos, d, torch.stack([tmin, tmax], dim=-1)
