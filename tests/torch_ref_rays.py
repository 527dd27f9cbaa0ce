"""TEST INFRASTRUCTURE -- oracle/torch_ref.py's restatement of the reference's PyTorch raymarch loop
(/root/reference/extensions/mvpraymarch/mvpraymarch.py:567-633) with the sample positions left ATTACHED to the rays: the
reference detaches them at :573-574 (`t0`, `raypos0`), here raypos_j = raypos + raydir * (tmin + j * stepsize), so autograd gives
the gradient of the image with respect to raypos, raydir and tminmax with every discrete decision (validity, saturation) held
fixed.  Everything else is torch_ref.raymarch_torch line for line; that function itself is unchanged."""
import torch
import torch.nn.functional as F


def raymarch_torch_attached(raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template, fadescale=8.0, fadeexp=8.0,
                            warp=None):
    N, H, W = raypos.shape[:3]
    K = primpos.shape[1]
    tplate = template.permute(0, 1, 5, 2, 3, 4)
    wfield = warp.permute(0, 1, 5, 2, 3, 4) if warp is not None else None
    rayrgba = torch.zeros((N, H, W, 4), dtype=raypos.dtype, device=raypos.device)
    tmin = tminmax[:, :, :, 0]
    t = tmin.detach().clone()
    t0 = t.clone()
    step = 0
    while (t < tminmax[:, :, :, 1]).any():
        raypos_t = raypos + raydir * (tmin + stepsize * step)[..., None]      # attached (the reference: raypos0 + raydir*dt*step)
        for k in range(K):
            y0 = torch.bmm((raypos_t - primpos[:, k, None, None, :]).view(N, -1, 3), primrot[:, k, :, :]).view_as(raypos_t) \
                * primscale[:, k, None, None, :]
            fade = torch.exp(-fadescale * torch.sum(torch.abs(y0) ** fadeexp, dim=-1, keepdim=True))
            if wfield is not None:
                y1 = F.grid_sample(wfield[:, k], y0[:, None, :, :, :], align_corners=True)[:, :, 0, :, :].permute(0, 2, 3, 1)
            else:
                y1 = y0
            sample = F.grid_sample(tplate[:, k], y1[:, None, :, :, :], align_corners=True)[:, :, 0, :, :].permute(0, 2, 3, 1)
            valid1 = torch.prod(y0 >= -1.0, dim=-1, keepdim=True) * torch.prod(y0 <= 1.0, dim=-1, keepdim=True)
            valid = ((t >= tminmax[:, :, :, 0]) & (t < tminmax[:, :, :, 1])).to(raypos.dtype)[:, :, :, None]
            alpha0 = sample[:, :, :, 3:4]
            rgb = sample[:, :, :, 0:3] * valid * valid1
            alpha = alpha0 * fade * stepsize * valid * valid1
            newalpha = rayrgba[:, :, :, 3:4] + alpha
            contrib = (newalpha.clamp(max=1.0) - rayrgba[:, :, :, 3:4]) * valid * valid1
            rayrgba = rayrgba + contrib * torch.cat([rgb, torch.ones_like(alpha)], dim=-1)
        step += 1
        t = t0 + stepsize * step
    return rayrgba


def ray_grads_torch(raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template, grad_rayrgba, fadescale=8.0,
                    fadeexp=8.0, warp=None):
    """(rayrgba, grad_raypos, grad_raydir, grad_tminmax) by autograd of the attached loop."""
    rays = [x.detach().clone().requires_grad_(True) for x in (raypos, raydir, tminmax)]
    out = raymarch_torch_attached(rays[0], rays[1], stepsize, rays[2], primpos, primrot, primscale, template, fadescale=fadescale,
                                  fadeexp=fadeexp, warp=warp)
    out.backward(grad_rayrgba)
    return (out.detach(),) + tuple(x.grad for x in rays)
