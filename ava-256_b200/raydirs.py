"""compute_raydirs: host-side mirror of /root/reference/extensions/utils/utils.py:21-51 on top of the C-ABI
(`mvp_compute_raydirs`).  Same call signature and, by default, the same (non-)gradient behaviour: the reference's backward
returns None for every input (utils.py:45-46).  With `differentiable=True` the camera tensors get the gradients of the rays
(`mvp_compute_raydirs_backward`)."""
import ctypes

import torch
from torch.autograd import Function

from . import lib as _lib


def _P(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class ComputeRaydirs(Function):
    @staticmethod
    def forward(ctx, viewpos, viewrot, focal, princpt, pixelcoords, volradius):
        for name, t in (("viewpos", viewpos), ("viewrot", viewrot), ("focal", focal), ("princpt", princpt)):
            if not t.is_cuda:
                raise RuntimeError("%s must be a CUDA tensor" % name)            # utils.cpp CHECK_CUDA
            assert t.is_contiguous() and t.dtype == torch.float32                 # utils.py:24-25
        N = viewpos.size(0)
        if isinstance(pixelcoords, tuple):                                        # utils.py:28-30
            W, H = pixelcoords
            pixelcoords = None
        else:
            assert pixelcoords.is_cuda and pixelcoords.is_contiguous() and pixelcoords.dtype == torch.float32
            H, W = pixelcoords.size(1), pixelcoords.size(2)
        dev = viewpos.device
        with torch.cuda.device(dev):
            raypos = torch.empty((N, H, W, 3), device=dev)
            raydirs = torch.empty((N, H, W, 3), device=dev)
            tminmax = torch.empty((N, H, W, 2), device=dev)
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(_lib.LIB.mvp_compute_raydirs(N, H, W, _P(viewpos), _P(viewrot), _P(focal), _P(princpt), _P(pixelcoords),
                                                    float(volradius), _P(raypos), _P(raydirs), _P(tminmax), stream))
        return raypos, raydirs, tminmax

    @staticmethod
    def backward(ctx, grad_raypos, grad_raydirs, grad_tminmax):
        return None, None, None, None, None, None


class ComputeRaydirsGrad(ComputeRaydirs):
    """ComputeRaydirs whose backward carries the rays' gradients to viewpos, viewrot, focal and princpt.  The adjoint recomputes
    the rays from the camera tensors, so they are saved for backward (an in-place change before the backward raises)."""

    @staticmethod
    def forward(ctx, viewpos, viewrot, focal, princpt, pixelcoords, volradius):
        out = ComputeRaydirs.forward(ctx, viewpos, viewrot, focal, princpt, pixelcoords, volradius)
        ctx.save_for_backward(viewpos, viewrot, focal, princpt, None if isinstance(pixelcoords, tuple) else pixelcoords)
        ctx.volradius = float(volradius)
        return out

    @staticmethod
    def backward(ctx, grad_raypos, grad_raydirs, grad_tminmax):
        viewpos, viewrot, focal, princpt, pixelcoords = ctx.saved_tensors
        volradius = ctx.volradius
        N, H, W = grad_raypos.shape[:3] if grad_raypos is not None else grad_raydirs.shape[:3]
        gr = [g if g is not None else torch.zeros((N, H, W, c), device=viewpos.device)
              for g, c in ((grad_raypos, 3), (grad_raydirs, 3), (grad_tminmax, 2))]
        cam = raydirs_backward(viewpos, viewrot, focal, princpt, pixelcoords, volradius, *gr)
        return tuple(g if need else None for g, need in zip(cam, ctx.needs_input_grad[:4])) + (None, None)


def raydirs_backward(viewpos, viewrot, focal, princpt, pixelcoords, volradius, grad_raypos, grad_raydir, grad_tminmax):
    """(grad_viewpos, grad_viewrot, grad_focal, grad_princpt) of the rays mvp_compute_raydirs makes (pixelcoords None = the integer
    grid, as the render kernels generate them), given the rays' gradients [N,H,W,3 | 3 | 2]."""
    _lib.require_ray_grads()
    N, H, W = grad_raypos.shape[:3]
    dev = viewpos.device
    grad_raypos, grad_raydir = grad_raypos.float().contiguous(), grad_raydir.float().contiguous()
    grad_tminmax = grad_tminmax.float().contiguous()
    if grad_tminmax.data_ptr() % 8:
        grad_tminmax = grad_tminmax.clone()
    out = [torch.zeros_like(t) for t in (viewpos, viewrot, focal, princpt)]       # accumulated into by the library
    with torch.cuda.device(dev):
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _lib.check(_lib.LIB.mvp_compute_raydirs_backward(N, H, W, _P(viewpos), _P(viewrot), _P(focal), _P(princpt), _P(pixelcoords),
                                                         float(volradius), _P(grad_raypos), _P(grad_raydir), _P(grad_tminmax),
                                                         *(_P(t) for t in out), stream))
    return tuple(out)


def compute_raydirs(viewpos, viewrot, focal, princpt, pixelcoords, volradius, *, differentiable=False):
    """Rays (raypos, raydirs, tminmax) of the reference's compute_raydirs.  differentiable=True: viewpos, viewrot, focal and princpt
    get the gradients of the rays (off by default, like the reference, whose backward returns None for every input)."""
    fn = ComputeRaydirsGrad if differentiable else ComputeRaydirs
    raypos, raydirs, tminmax = fn.apply(viewpos, viewrot, focal, princpt, pixelcoords, volradius)
    return raypos, raydirs, tminmax
