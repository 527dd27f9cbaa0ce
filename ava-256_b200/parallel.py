"""Multi-GPU plumbing of the path (SURVEY.md section 8e): views shard over ranks with no data-path collective in
forward; when the views of a step share one subject's primitives, the per-view primitive gradients are summed locally
and all-reduced once per step (one flat fp32 buffer: template, primpos, primrot, primscale).  A bf16 template gradient is
summed over the views straight into the fp32 buffer (exact widening, fp32 accumulation); the all-reduce stays fp32."""
import torch
import torch.distributed as dist


def shard_views(n_views, rank, world):
    """Contiguous block of views of `rank`: [start, stop)."""
    if n_views % world:
        raise ValueError("n_views (%d) must be divisible by world size (%d)" % (n_views, world))
    per = n_views // world
    return rank * per, (rank + 1) * per


def rank_views(n_views, rank, world, interleave=True):
    """View indices of `rank`.  Interleaved (rank, rank + world, ...) by default: neighbouring dome cameras see the subject
    under similar coverage, so contiguous blocks give the ranks unequal work and the step time is the slowest rank's;
    striding spreads every part of the dome over all ranks.  interleave=False gives the contiguous block of shard_views."""
    if n_views % world:
        raise ValueError("n_views (%d) must be divisible by world size (%d)" % (n_views, world))
    if interleave:
        return list(range(rank, n_views, world))
    lo, hi = shard_views(n_views, rank, world)
    return list(range(lo, hi))


def _sum_views(p, out):
    """out[...] = sum over the local views of p [nv, ...]: the library's one-pass kernel on the GPU (`mvp_sum_views`, or
    `mvp_sum_views_bf16` for a bf16 p and an fp32 out), torch.sum for host tensors (the world-size-2 gloo tests of this module's
    logic run on the CPU), which widens a bf16 p to out's dtype first."""
    if p.is_cuda:
        from .payload import sum_views
        sum_views(p, out)
    else:
        torch.sum(p.reshape(p.shape[0], -1).to(out.dtype), dim=0, out=out)


def flat_grad_numel(K, TD, TH, TW):
    return K * TD * TH * TW * 4 + K * 15


def reduce_primitive_grads(grad_template, grad_primpos, grad_primrot, grad_primscale, flat=None, group=None):
    """Sum per-view gradients [nv, ...] over the local views into `flat` and all-reduce it (if a process group is up).

    Returns (flat, views) where views = (g_template [K,TD,TH,TW,4], g_primpos [K,3], g_primrot [K,3,3], g_primscale [K,3])
    are views into flat.  A bf16 grad_template is summed into an fp32 flat buffer."""
    parts = (grad_template, grad_primpos, grad_primrot, grad_primscale)
    nv = grad_template.shape[0]
    total = sum(p[0].numel() for p in parts)
    if flat is None:
        dtype = torch.float32 if grad_template.dtype == torch.bfloat16 else grad_template.dtype
        flat = torch.empty(total, dtype=dtype, device=grad_template.device)
    assert flat.numel() == total
    o = 0
    views = []
    for p in parts:
        n = p[0].numel()
        _sum_views(p, flat[o:o + n])
        views.append(flat[o:o + n].view(p.shape[1:]))
        o += n
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(flat, group=group)
    return flat, tuple(views)


class GradReducer:
    """Per-step reduction of the primitive gradients of a view-sharded subject, with the collective taken off the critical
    path: the rank's per-view gradients are summed into one of two flat buffers on the compute stream and the NCCL
    all-reduce of that buffer is launched asynchronously (NCCL's own stream), so it overlaps whatever the caller enqueues
    next -- normally the next step's forward.  A buffer is waited for only when it is about to be reused, when the caller
    asks for its contents (`wait`), or at `finish()`.  A bf16 template gradient is summed into the fp32 buffer with fp32
    accumulation.

        red = GradReducer(K, TD, TH, TW, device)
        for step ...:
            out = mvpraymarch(...); out.backward(g)
            flat = red.reduce(template.grad, primpos.grad, primrot.grad, primscale.grad)   # returns at once
            ...                                                                             # next forward overlaps the all-reduce
            red.wait(flat)                                                                  # before reading `flat`
        red.finish()
    """

    def __init__(self, K, TD, TH, TW, device, group=None, dtype=torch.float32):
        n = flat_grad_numel(K, TD, TH, TW)
        self.bufs = [torch.zeros(n, dtype=dtype, device=device) for _ in range(2)]
        self.work = [None, None]
        self.group = group
        self.i = 0

    def reduce(self, grad_template, grad_primpos, grad_primrot, grad_primscale):
        i, self.i = self.i, self.i ^ 1
        if self.work[i] is not None:            # the buffer's previous all-reduce must be over before it is overwritten
            self.work[i].wait()
            self.work[i] = None
        flat = self.bufs[i]
        parts = (grad_template, grad_primpos, grad_primrot, grad_primscale)
        nv = grad_template.shape[0]
        o = 0
        for p in parts:
            n = p[0].numel()
            _sum_views(p, flat[o:o + n])
            o += n
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(self.group) > 1:
            self.work[i] = dist.all_reduce(flat, group=self.group, async_op=True)
        return flat

    def wait(self, flat):
        for i, b in enumerate(self.bufs):
            if b is flat and self.work[i] is not None:
                self.work[i].wait()
                self.work[i] = None

    def finish(self):
        for i in range(2):
            if self.work[i] is not None:
                self.work[i].wait()
                self.work[i] = None

    def views(self, flat, K, TD, TH, TW):
        """(g_template [K,TD,TH,TW,4], g_primpos [K,3], g_primrot [K,3,3], g_primscale [K,3]) as views into `flat`."""
        o, out = 0, []
        for shape in ((K, TD, TH, TW, 4), (K, 3), (K, 3, 3), (K, 3)):
            n = 1
            for d in shape:
                n *= d
            out.append(flat[o:o + n].view(shape))
            o += n
        return tuple(out)
