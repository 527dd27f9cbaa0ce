"""`Raymarcher`: host-side mirror of /root/reference/models/raymarchers/mvpraymarcher.py:17-54 (same constructor arguments,
same forward signature and return tuple).  The image planes `rayrgb` / `rayalpha` come straight out of the render kernel's
epilogue and their gradients go straight into the backward's prologue (`op.mvpraymarch_planes`); the reference makes them
with a permute + two `.contiguous()` copies (:50-51)."""
import contextlib

import torch.nn as nn

from .composite import split_rgba
from .op import (_check_template_grad_dtype, _det_context, _view_set_block, mvpraymarch, mvpraymarch_camera, mvpraymarch_planes,
                 template_grad_dtype)


class Raymarcher(nn.Module):
    def __init__(self, volradius, dt: float = 1.0, with_rgba: bool = False, template_grad_dtype=None, deterministic=None):
        """with_rgba: also return the [N,4,H,W] view of the channels-last `rayrgba` as the third item, like the reference
        (:50).  No caller in ava-256 reads it (models/autoencoder.py:246 drops it), so by default the channels-last image
        is never written and the third item is None.
        template_grad_dtype: torch.float32 accumulates a bfloat16 template's gradient in fp32 in `forward` and `forward_camera`
        (see `op.template_grad_dtype`); None (default) leaves it to the template's dtype or an enclosing `op.template_grad_dtype`.
        deterministic: True returns reproducible primitive gradients from `forward` and `forward_camera` (see
        `op.deterministic_grads`), False the default backward; None (default) leaves it to an enclosing `op.deterministic_grads`."""
        super().__init__()
        self.volume_radius = volradius
        self.dt = dt / self.volume_radius                       # mvpraymarcher.py:24
        self.with_rgba = with_rgba
        self.template_grad_dtype = _check_template_grad_dtype(template_grad_dtype)
        self.deterministic = deterministic

    def _grad_dtype(self):
        return contextlib.nullcontext() if self.template_grad_dtype is None else template_grad_dtype(self.template_grad_dtype)

    def forward(self, raypos, raydir, tminmax, decout, renderoptions={}, rayterm=None, with_pos_img=None, view_set=None):
        """view_set: the decoder output holds S subjects' (or frames') primitives [S,K,...] and view n renders set view_set[n]
        (see `op.mvpraymarch_sets`); None: one set per view, or one shared by all views."""
        with self._grad_dtype(), _view_set_block(view_set), _det_context(self.deterministic):
            return self._forward(raypos, raydir, tminmax, decout, renderoptions, rayterm)

    def _forward(self, raypos, raydir, tminmax, decout, renderoptions, rayterm):
        args = (raypos, raydir, self.dt, tminmax, (decout["primpos"], decout["primrot"], decout["primscale"]))
        kwargs = dict(template=decout["template"], warp=decout["warp"] if "warp" in decout else None, rayterm=rayterm,
                      **{k: v for k, v in renderoptions.items() if k in mvpraymarch.__code__.co_varnames})   # :45
        if self.with_rgba:
            rayrgba = mvpraymarch(*args, **kwargs)
            rayrgb, rayalpha = split_rgba(rayrgba)              # one kernel instead of the permute + two copies
            return rayrgb, rayalpha, rayrgba.permute(0, 3, 1, 2), None
        rayrgb, rayalpha = mvpraymarch_planes(*args, **kwargs)
        return rayrgb, rayalpha, None, None

    def forward_camera(self, viewpos, viewrot, focal, princpt, pixelcoords, decout, renderoptions={}, rayterm=None, camera_grad=False,
                       view_set=None, deterministic=None):
        """`compute_raydirs(viewpos, viewrot, focal, princpt, pixelcoords, volradius)` followed by `forward(raypos, raydir, tminmax,
        ...)` -- models/autoencoder.py:240-252 -- as one call.  With `pixelcoords` as the `(W, H)` tuple or as an [N,H,W,2] tensor
        of sample positions the rays are generated inside the render kernels and never stored (`op.mvpraymarch_camera`); same
        return tuple as `forward`.  camera_grad=True: the camera tensors
        that require grad get gradients (pose / calibration fitting through the image loss, see `op.mvpraymarch_camera`).  view_set:
        as in `forward`.  deterministic: True / False for this call; None (default) takes the module's setting."""
        kwargs = dict(rayterm=rayterm, **{k: v for k, v in renderoptions.items() if k in mvpraymarch.__code__.co_varnames})
        out = mvpraymarch_camera(viewpos, viewrot, focal, princpt, pixelcoords, self.volume_radius, self.dt,
                                 (decout["primpos"], decout["primrot"], decout["primscale"]), decout["template"],
                                 decout["warp"] if "warp" in decout else None, planes=not self.with_rgba, camera_grad=camera_grad,
                                 template_grad_dtype=self.template_grad_dtype, view_set=view_set,
                                 deterministic=self.deterministic if deterministic is None else deterministic, **kwargs)
        if self.with_rgba:
            rayrgb, rayalpha = split_rgba(out)
            return rayrgb, rayalpha, out.permute(0, 3, 1, 2), None
        return out[0], out[1], None, None
