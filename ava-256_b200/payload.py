"""Payload hand-off from the decoders to the raymarcher (SURVEY.md section 8f row 4) on top of the C-ABI
(`mvp_assemble_payload_*`).

The reference turns the colour decoder's image [N, B*3, h*B, w*B] and the geometry decoder's opacity image
[N, B, h*B, w*B] into the raymarcher's channels-last slabs with a chain of eager ops,

    rgb.view(N, B, 3, h, B, w, B).permute(0, 3, 5, 1, 4, 6, 2).reshape(N, h*w, B, B, B, 3)   models/decoders/rgb.py:128-143
    opacity.view(N, B, 1, h, B, w, B).permute(0, 3, 5, 1, 4, 6, 2).reshape(N, h*w, B, B, B, 1)  models/decoders/geometry.py:180-185
    template = cat([relu(primrgb * 25.0 + 100.0), relu(primalpha)], dim=-1)                     models/decoders/assembler.py:261

i.e. five passes over 134 MB per view at K = 16384, B = 8.  `assemble_payload` does it in one pass (16 B read + 16 B
written per texel) and its adjoint in one more; values are bit-identical to the eager chain.  With dtype=torch.bfloat16 it
writes the template as bf16 (8 B per texel), bit-identical to the eager chain followed by .to(torch.bfloat16)."""
import ctypes

import torch
from torch.autograd import Function

from . import lib as _lib
from .composite import _check_f32_cuda, _ptr


class AssemblePayload(Function):
    @staticmethod
    def forward(ctx, tex, opacity, boxsize, rgb_scale, rgb_bias, dtype):
        _check_f32_cuda("tex", tex)
        _check_f32_cuda("opacity", opacity)
        B = int(boxsize)
        assert tex.dim() == 4 and opacity.dim() == 4
        N, C, Himg, Wimg = tex.shape
        assert C == 3 * B and Himg % B == 0 and Wimg % B == 0, "tex must be [N, B*3, h*B, w*B]"
        assert tuple(opacity.shape) == (N, B, Himg, Wimg), "opacity must be [N, B, h*B, w*B]"
        hb, wb = Himg // B, Wimg // B
        tex, opacity = tex.contiguous(), opacity.contiguous()
        dev = tex.device
        bf16 = dtype == torch.bfloat16
        fwd = _lib.LIB.mvp_assemble_payload_forward_bf16 if bf16 else _lib.LIB.mvp_assemble_payload_forward
        with torch.cuda.device(dev):
            tplate = torch.empty((N, hb * wb, B, B, B, 4), dtype=dtype, device=dev)
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(fwd(N, hb, wb, B, _ptr(tex), _ptr(opacity), float(rgb_scale), float(rgb_bias), _ptr(tplate), stream))
        ctx.save_for_backward(tplate)
        ctx.dims = (N, hb, wb, B, float(rgb_scale))
        return tplate

    @staticmethod
    def backward(ctx, grad_tplate):
        (tplate,) = ctx.saved_tensors
        N, hb, wb, B, rgb_scale = ctx.dims
        grad_tplate = grad_tplate.to(tplate.dtype).contiguous()     # autograd hands the output's dtype; a no-op then
        bwd = _lib.LIB.mvp_assemble_payload_backward_bf16 if tplate.dtype == torch.bfloat16 else _lib.LIB.mvp_assemble_payload_backward
        dev = tplate.device
        with torch.cuda.device(dev):
            grad_tex = torch.empty((N, 3 * B, hb * B, wb * B), device=dev)
            grad_opacity = torch.empty((N, B, hb * B, wb * B), device=dev)
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(bwd(N, hb, wb, B, _ptr(tplate), _ptr(grad_tplate), rgb_scale, _ptr(grad_tex), _ptr(grad_opacity), stream))
        return grad_tex, grad_opacity, None, None, None, None


def _check_dtype(name, dtype):
    """float32, or bfloat16 when the library has the bf16 kernels (EPILOGUE_BF16=1); anything else raises."""
    if dtype == torch.bfloat16:
        _lib.require_epilogue_bf16()
    elif dtype != torch.float32:
        raise RuntimeError("%s must be float32 or bfloat16, got %s" % (name, dtype))


def assemble_payload(tex, opacity, boxsize=8, rgb_scale=25.0, rgb_bias=100.0, dtype=torch.float32):
    """template [N, h*w, B, B, B, 4] from the decoders' fp32 images; defaults are the reference's hard-coded
    de-normalisation (assembler.py:261).  dtype=torch.bfloat16 writes a bf16 template (each value of the fp32 template rounded
    once, to nearest even): half the bytes written here, and what the raymarcher reads with a bf16 template; its backward
    takes the bf16 template gradient the raymarcher returns and gives fp32 image gradients."""
    _check_dtype("dtype", dtype)
    return AssemblePayload.apply(tex, opacity, boxsize, rgb_scale, rgb_bias, dtype)


class ExpandViews(Function):
    @staticmethod
    def forward(ctx, x, n_views):
        _check_cuda("x", x)
        x = x.contiguous()
        if x.data_ptr() % 4:                       # a bf16 view that starts mid-word: the word copy needs 4-byte alignment
            x = x.clone()
        dev = x.device
        with torch.cuda.device(dev):
            out = torch.empty((int(n_views),) + tuple(x.shape), dtype=x.dtype, device=dev)
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            # a copy moves bits: a bf16 tensor goes through the fp32 kernel as 4-byte words, two values each
            count = x.numel() if x.dtype == torch.float32 else x.numel() // 2
            _lib.check(_lib.LIB.mvp_expand_views(_ptr(x), _ptr(out), count, int(n_views), stream))
        return out

    @staticmethod
    def backward(ctx, grad):
        return sum_views(grad), None


def _check_cuda(name, x):
    if not x.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor" % name)
    _check_dtype(name, x.dtype)
    if x.dtype == torch.bfloat16 and x.numel() % 2:
        raise RuntimeError("%s: a bfloat16 tensor needs an even number of elements (got %d)" % (name, x.numel()))


def sum_views(x, out=None):
    """x [n_views, ...] -> sum over the views [...] in one pass (view order, deterministic).  `out`: optional contiguous
    destination with x[0].numel() elements (e.g. a slice of a flat all-reduce buffer).

    fp32 x (`mvp_sum_views`): out is fp32.  bf16 x (`mvp_sum_views_bf16`): the values are widened exactly and added in fp32, so
    an fp32 `out` holds exactly sum_views(x.float()); a bf16 `out` (the default) holds that sum rounded once."""
    if not x.is_cuda:
        raise RuntimeError("x must be a CUDA tensor")
    _check_dtype("x", x.dtype)
    x = x.contiguous()
    n, count = x.shape[0], x[0].numel()
    dev = x.device
    with torch.cuda.device(dev):
        if out is None:
            out = torch.empty(tuple(x.shape[1:]), dtype=x.dtype, device=dev)
        assert out.is_cuda and out.is_contiguous() and out.numel() == count
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        if x.dtype == torch.bfloat16:
            assert out.dtype in (torch.float32, torch.bfloat16), out.dtype
            _lib.check(_lib.LIB.mvp_sum_views_bf16(_ptr(x), _ptr(out), count, int(n), int(out.dtype == torch.bfloat16), stream))
        else:
            assert out.dtype == torch.float32
            _lib.check(_lib.LIB.mvp_sum_views(_ptr(x), _ptr(out), count, int(n), stream))
    return out


def expand_views(x, n_views):
    """[n_views, *x.shape] copies of one subject's tensor (`x[None].expand(n_views, ...).contiguous()` in one pass of
    streaming stores, `mvp_expand_views`); the adjoint is the sum over the views.  fp32 or bf16 (an even element count; the
    adjoint is then the fp32 sum rounded once to bf16)."""
    return ExpandViews.apply(x, n_views)
