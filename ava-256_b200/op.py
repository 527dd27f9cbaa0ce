"""torch.autograd front-end of the H100 raymarcher: the host-side mirror of the reference's op
(/root/reference/extensions/mvpraymarch/mvpraymarch.py:87-390) on top of the C-ABI in include/mvpraymarch_b200.h.

Same contract as the reference: fp32 CUDA tensors, contiguous, caller-visible output rayrgba [N,H,W,4] that
participates in autograd with gradients for primpos, primrot, primscale, template and (algo 1) warp, None for
everything else (mvpraymarch.py:279-292).  Differences that are deliberate:
  * kernels run on torch's current stream (the reference launches on legacy stream 0, mvpraymarch.cpp:277);
  * no allocation or sync inside the native call (the reference cudaMalloc/cudaFree's per forward, bvh.cu:261-293);
  * the acceleration structure is a screen-space bucket list, not the BVH tensors of build_accel (:21-84);
    it is kept for backward instead of being rebuilt;
  * 64-bit indexing (the reference overflows int32 at N*K*T^3*4 >= 2^31, primsampler.h:31-36);
  * the template may be bfloat16 (what the decoders produce under torch.autocast): it is rendered exactly as its fp32
    widening and its gradient is bfloat16, accumulated in bf16 by the backward kernel -- or, on request (`template_grad_dtype`
    below), accumulated in fp32.  `mvpraymarch` widens bfloat16 primpos / primrot / primscale / warp to fp32 before the op
    (exact; autograd casts their gradients back).  The reference reads a half-precision template as fp32 without checking its
    dtype (mvpraymarch.cpp:250-272).
"""
import contextlib
import ctypes
import numbers

import torch
from torch.autograd import Function

from . import lib as _lib


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _aligned(t, nbytes):
    """The kernels read channels-last buffers with 128-bit accesses (C-ABI: MVP_ERR_ALIGN).  A contiguous view into a
    larger buffer can start anywhere; such a tensor is copied once to a fresh (256-byte aligned) allocation."""
    if t is not None and t.data_ptr() % nbytes:
        return t.clone()
    return t


def _check_f32_cuda(name, t, allow_bf16=False):
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor" % name)          # mvpraymarch.cpp:102
    if not t.is_contiguous():
        raise RuntimeError("%s must be contiguous" % name)             # mvpraymarch.cpp:103
    if allow_bf16:
        if t.dtype not in (torch.float32, torch.bfloat16):
            raise RuntimeError("%s must be float32 or bfloat16, got %s" % (name, t.dtype))
    elif t.dtype != torch.float32:
        raise RuntimeError("%s must be float32" % name)


_TEMPLATE_GRAD = {}   # "dtype": the setting of the innermost active `template_grad_dtype` context


def _check_template_grad_dtype(dtype):
    if dtype is not None and dtype is not torch.float32:
        raise ValueError("template_grad_dtype must be None (the template's own dtype) or torch.float32, got %r" % (dtype,))
    return dtype


@contextlib.contextmanager
def template_grad_dtype(dtype):
    """Within the block, raymarch calls with a bfloat16 template accumulate its gradient in fp32 (dtype=torch.float32) or in the
    template's own dtype (None, the default).  With fp32 the template is still read as bf16 (same images as without), the backward
    adds to an fp32 [N,K,TD,TH,TW,4] buffer that the op allocates (twice the bf16 gradient's size, cleared by the forward's render
    kernel) and every gradient equals that of the fp32 template `template.float()` up to the order of the fp32 atomics.  The op
    returns that fp32 gradient and autograd casts it to the input's dtype, so `template.grad` stays bfloat16 and holds the fp32
    sum rounded once; the cast allocates a bf16 temporary of the gradient's size besides the fp32 buffer.  An fp32 template
    ignores the setting.  The decision is taken by the forward call and kept for its backward, so the backward may run outside the
    block (autograd runs it on its own thread).  The only way an unmodified caller of `mvpraymarch` opts in:

        with ava256_b200.op.template_grad_dtype(torch.float32):
            rayrgba = mvpraymarch(raypos, raydir, stepsize, tminmax, primtransf, template_bf16, warp)
        loss(rayrgba).backward()
    """
    _check_template_grad_dtype(dtype)
    prev = _TEMPLATE_GRAD.get("dtype")
    _TEMPLATE_GRAD["dtype"] = dtype
    try:
        yield
    finally:
        _TEMPLATE_GRAD["dtype"] = prev


_template_grad_block = template_grad_dtype     # for the functions whose keyword of the same name hides it

_DETERMINISTIC = {}   # "on": the setting of the innermost active `deterministic_grads` context


@contextlib.contextmanager
def deterministic_grads(enabled=True):
    """Within the block (enabled=True), raymarch calls return reproducible primitive gradients: the backward sums grad_primpos,
    grad_primrot, grad_primscale and the template's gradient in 64-bit fixed point (C-ABI mvp_raymarch_backward_deterministic), so
    two backwards of the same inputs give the same bits, whatever the order in which the GPU runs the warps, and the same sums
    whatever the order of the views.  They agree with the default backward to within about 1e-6 of each tensor's largest entry;
    images are unchanged.  The backward runs the render kernels twice (a pass that measures each tensor's range, then the
    accumulating pass), and its int64 scratch is twice the size of the fp32 gradients (allocated by the forward for the gradients
    autograd asks for, cleared by its render kernel).  Supported: algo 0, fp32 and bf16 templates (either `template_grad_dtype`),
    per-view, shared and set primitives, usebvh=True, ray tensors, camera rays and pixelcoords, image planes.  Raises
    NotImplementedError for algo 1 and for ray / camera gradients.  The decision is taken by the forward call and kept for its
    backward.  The only way an unmodified caller of `mvpraymarch` opts in:

        with ava256_b200.op.deterministic_grads():
            rayrgba = mvpraymarch(raypos, raydir, stepsize, tminmax, primtransf, template, warp)
        loss(rayrgba).backward()

    `torch.use_deterministic_algorithms(True)` does not switch this on."""
    prev = _DETERMINISTIC.get("on")
    _DETERMINISTIC["on"] = bool(enabled)
    try:
        yield
    finally:
        _DETERMINISTIC["on"] = prev


_deterministic_block = deterministic_grads     # for the functions whose keyword `deterministic` hides it


def _det_context(deterministic):
    """The `deterministic=` keyword of the entry points: None leaves the enclosing `deterministic_grads` setting."""
    return contextlib.nullcontext() if deterministic is None else _deterministic_block(bool(deterministic))


def _widen_bf16(t):
    """A bfloat16 tensor as fp32 (exact); anything else unchanged, so that other dtypes still meet the op's dtype check."""
    return t.float() if t is not None and t.dtype == torch.bfloat16 else t


def _empty_template_grad(template, tflags):
    """The template's gradient buffer: fp32 with MVP_FLAG_GRAD_TPLATE_F32, else of the template's dtype."""
    if tflags & _lib.FLAG_GRAD_TPLATE_F32:
        return torch.empty(template.shape, dtype=torch.float32, device=template.device)
    return torch.empty_like(template)


# Gradient sets of the backward, chosen by the forward from what autograd asks for (ctx.needs_input_grad):
#   GRADS_ALL         transforms, template (+ warp), optionally rays: the template or the warp needs a gradient
#   GRADS_NO_PAYLOAD  transforms, optionally rays (MVP_FLAG_NO_TPLATE_GRAD): no payload-gradient scatter, no template-sized buffer
#   GRADS_RAYS_ONLY   rays only (MVP_FLAG_RAY_GRADS_ONLY): a frozen avatar seen through a differentiable camera
GRADS_ALL, GRADS_NO_PAYLOAD, GRADS_RAYS_ONLY = "all", "no_payload", "rays_only"
_GRAD_SET_FLAGS = {GRADS_ALL: 0, GRADS_NO_PAYLOAD: _lib.FLAG_NO_TPLATE_GRAD, GRADS_RAYS_ONLY: _lib.FLAG_RAY_GRADS_ONLY}


def _grad_set(needs, first_prim, want_rays):
    """The gradient set for ctx.needs_input_grad `needs` whose primitive inputs (primpos, primrot, primscale, template, warp) start
    at index first_prim; None when nothing needs a gradient."""
    if needs[first_prim + 3] or needs[first_prim + 4]:
        return GRADS_ALL
    if any(needs[first_prim:first_prim + 3]):
        return GRADS_NO_PAYLOAD
    return GRADS_RAYS_ONLY if want_rays else None


def _empty_det_sums(gset, primpos, primrot, primscale, template):
    """The deterministic backward's int64 sums of the set, one entry per gradient entry: [primpos, primrot, primscale, template, None]."""
    e = lambda t: torch.empty(t.shape, dtype=torch.int64, device=t.device)  # noqa: E731
    return [e(primpos), e(primrot), e(primscale), e(template) if gset == GRADS_ALL else None, None]


def _empty_grads(gset, primpos, primrot, primscale, template, warp, usewarp, tflags):
    """The backward's gradient buffers of the set: [primpos, primrot, primscale, template, warp], None where not computed."""
    tf = [torch.empty_like(primpos), torch.empty_like(primrot), torch.empty_like(primscale)] if gset != GRADS_RAYS_ONLY else [None] * 3
    if gset != GRADS_ALL:
        return tf + [None, None]
    return tf + [_empty_template_grad(template, tflags), torch.empty_like(warp) if usewarp else None]


class MVPRaymarch(Function):
    """Custom Function for raymarching Mixture of Volumetric Primitives (reference: mvpraymarch.py:87-292)."""

    @staticmethod
    def forward(ctx, raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template, warp, rayterm,
                gradmode, options):
        return MVPRaymarch._forward(ctx, raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template, warp, rayterm,
                                    gradmode, options)

    @staticmethod
    def _forward(ctx, raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template, warp, rayterm,
                 gradmode, options, saved_extra=(), first_prim=4, ray_inputs=(0, 1, 3)):
        """The forward; saved_extra: more tensors for ctx.save_for_backward, after the eleven the backward reads.  first_prim: index
        of primpos among the Function's inputs (primrot, primscale, template and warp follow); ray_inputs: the inputs through which
        the rays get gradients (with the `_ray_grads` option).  They pick the backward's gradient set from ctx.needs_input_grad."""
        algo = options["algo"]
        if algo not in (0, 1):
            raise NotImplementedError("mvpraymarch_b200: algo must be 0 or 1 (the reference launches nothing for other "
                                      "values, mvpraymarch_kernel.cu:104-105)")
        if algo == 1 and warp is None:
            raise RuntimeError("mvpraymarch_b200: algo=1 samples a warp field (PrimSamplerTW<true>); pass `warp`")
        if options["usebvh"] is False:
            raise NotImplementedError("mvpraymarch_b200: usebvh=False passes a null BVH to the reference kernels "
                                      "(mvpraymarch.py:132-134) and is not a usable mode there either")
        if options.get("_deterministic") and gradmode and any(ctx.needs_input_grad):
            if algo == 1:
                raise NotImplementedError("mvpraymarch_b200: deterministic gradients need algo 0 (the warp field's gradient is "
                                          "summed with float atomics)")
            if options.get("_ray_grads") and any(ctx.needs_input_grad[i] for i in ray_inputs):
                raise NotImplementedError("mvpraymarch_b200: deterministic gradients of rays and cameras are not supported (their "
                                          "per-ray sums use shared-memory float atomics)")
        camera = options.get("_camera")        # (viewpos, viewrot, focal, princpt, volradius, H, W): rays generated in the kernels
        pixels = options.get("_pixels")        # with a camera: [N,H,W,2] sample positions of its rays, or None (the integer grid)
        if camera is not None:
            assert raypos is None and raydir is None and tminmax is None
            viewpos, viewrot, focal, princpt, volradius, camH, camW = camera
            cam_tensors = (("viewpos", viewpos, (3,)), ("viewrot", viewrot, (3, 3)), ("focal", focal, (2,)), ("princpt", princpt, (2,)))
            if pixels is not None:
                _lib.require_camera_pixels()
                cam_tensors += (("pixelcoords", pixels, (int(camH), int(camW), 2)),)
            for name, t, tail in cam_tensors:
                _check_f32_cuda(name, t)                                  # utils.py:24-25 / utils.cpp CHECK_CUDA
                assert t.shape == (viewpos.size(0),) + tail, "%s must be [N,%s]" % (name, ",".join(map(str, tail)))
                assert t.device == primpos.device, "%s must be on the primitives' device" % name
            assert int(camH) >= 1 and int(camW) >= 1 and float(volradius) > 0.0
        else:
            # same shape contract as mvpraymarch.py:112-127
            assert raypos.is_contiguous() and raypos.size(3) == 3
            assert raydir.is_contiguous() and raydir.size(3) == 3
            assert tminmax.is_contiguous() and tminmax.size(3) == 2
        assert primpos.is_contiguous() and primpos.size(2) == 3
        assert primrot.is_contiguous() and primrot.size(2) == 3
        assert primscale.is_contiguous() and primscale.size(2) == 3
        assert template.is_contiguous() and template.dim() == 6 and template.size(-1) == 4, \
            "channels-last template [N,K,TD,TH,TW,4] required (the reference sampler is always channels-last, primsampler.h:16)"
        for name, t in (("raypos", raypos), ("raydir", raydir), ("tminmax", tminmax), ("primpos", primpos),
                        ("primrot", primrot), ("primscale", primscale)):
            if t is not None:
                _check_f32_cuda(name, t)
        _check_f32_cuda("template", template, allow_bf16=True)
        bf16 = template.dtype == torch.bfloat16                        # MVP_FLAG_TPLATE_BF16: rendered as template.float()
        gset = None
        if gradmode:
            # Only the gradients autograd asks for.  With none that this op computes, the image is rendered as in inference.  The
            # output may still get a backward (rays that require grad without the `_ray_grads` option: they get None, as before),
            # which then returns None for every input: ctx.gset = None.
            needs = ctx.needs_input_grad
            gset = _grad_set(needs, first_prim, bool(options.get("_ray_grads")) and any(needs[i] for i in ray_inputs))
            gradmode = gset is not None
            ctx.gset = gset
            if gset not in (None, GRADS_ALL):
                _lib.require_grad_select()
        grad_f32 = bf16 and _check_template_grad_dtype(options.get("_template_grad_dtype")) is torch.float32 and gset == GRADS_ALL
        tflags = _lib.tplate_flags(bf16, grad_f32)                     # + MVP_FLAG_GRAD_TPLATE_F32: fp32 template gradient
        det = bool(options.get("_deterministic")) and gradmode         # fixed-point primitive gradients (deterministic_grads)
        if det:
            _lib.require_deterministic()
        if warp is not None:                                           # mvpraymarch.py:124
            assert warp.is_contiguous() and warp.dim() == 6 and warp.size(-1) == 3, \
                "channels-last warp field [N,K,WD,WH,WW,3] required"
            _check_f32_cuda("warp", warp)
        usewarp = algo == 1                                            # algo 0 ignores a warp field, like the reference

        if camera is not None:
            N, H, W = viewpos.size(0), int(camH), int(camW)
        else:
            N, H, W = raypos.shape[:3]
        K = primpos.size(1)
        TD, TH, TW = template.shape[2:5]
        dev = primpos.device
        # The reference never checks that the leading dimensions agree (a mismatch reads out of bounds there).  Here:
        # rays and tminmax must agree; the primitive tensors must agree with each other and have a batch of N, or of 1
        # = one set of primitives shared by all N views (extension, SURVEY.md section 8e "optional fast path":
        # nothing is replicated in HBM and the gradients of all views accumulate into the one set).
        if camera is None:
            assert raydir.shape[:3] == (N, H, W) and tminmax.shape[:3] == (N, H, W), "raypos / raydir / tminmax disagree on [N,H,W]"
        NP = primpos.size(0)
        view_set = options.get("_view_set")     # per-view primitive sets (mvpraymarch_sets): NP sets, chosen per view by the map
        if view_set is not None:
            _lib.require_view_sets()
            view_set = _view_set_tensor(view_set, N, NP, dev)
        else:
            assert NP in (N, 1), "primitive batch (%d) must equal the number of views (%d) or be 1 (shared)" % (NP, N)
        assert primrot.shape[:2] == (NP, K) and primscale.shape[:2] == (NP, K) and template.shape[:2] == (NP, K), \
            "primpos / primrot / primscale / template disagree on [N,K]"
        if warp is not None:
            assert warp.shape[:2] == (NP, K), "warp disagrees with the primitives on [N,K]"
        shared = view_set is None and NP == 1 and N > 1
        template, tminmax = _aligned(template, 8 if bf16 else 16), _aligned(tminmax, 8)
        with torch.cuda.device(dev):
            wsbytes = _lib.workspace_bytes(N, H, W, K, TD, TH, TW)
            workspace = torch.empty(wsbytes, dtype=torch.uint8, device=dev)
            planes = bool(options.get("_planes", False))   # image-plane outputs (MVPRaymarchPlanes below)
            if planes:
                rayrgba = None
                rayrgb = torch.empty((N, 3, H, W), dtype=torch.float32, device=dev)
                rayalpha = torch.empty((N, 1, H, W), dtype=torch.float32, device=dev)
            else:
                rayrgba = torch.empty((N, H, W, 4), dtype=torch.float32, device=dev)
            if gradmode:
                raysat = torch.empty((N, H, W, 3), dtype=torch.float32, device=dev)
                rayaux = torch.empty((N, H, W, 4), dtype=torch.int32, device=dev)
            else:
                raysat = rayaux = None
            a = _lib.ForwardArgs()
            a.shape = _lib.Shape(N, H, W, K, TD, TH, TW)
            a.stepsize, a.fadescale, a.fadeexp = float(stepsize), float(options["fadescale"]), float(options["fadeexp"])
            a.flags = (_lib.FLAG_SHARED_PRIMS if shared else 0) | tflags | _GRAD_SET_FLAGS.get(gset, 0) | \
                (_lib.FLAG_DETERMINISTIC if det else 0)
            a.raypos, a.raydir, a.tminmax = _ptr(raypos), _ptr(raydir), _ptr(tminmax)
            if camera is not None:
                a.camera = _lib.Camera(_ptr(viewpos), _ptr(viewrot), _ptr(focal), _ptr(princpt), float(volradius), 0)
            a.primpos, a.primrot, a.primscale = _ptr(primpos), _ptr(primrot), _ptr(primscale)
            a.tplate = _ptr(template)
            a.rayrgba, a.raysat, a.rayaux = _ptr(rayrgba), _ptr(raysat), _ptr(rayaux)
            if planes:
                a.rayrgb_nchw, a.rayalpha_nchw = _ptr(rayrgb), _ptr(rayalpha)
            order = options.get("_order")                              # [NP,K] int32 marching order (usebvh=True) or None
            if order is not None:
                assert order.dtype == torch.int32 and order.is_contiguous() and tuple(order.shape) == (NP, K)
                a.order = _ptr(order)
            a.workspace, a.workspace_bytes = _ptr(workspace), wsbytes
            a.algo = 1 if usewarp else 0
            if usewarp:
                a.warp = _ptr(warp)
                a.WD, a.WH, a.WW = warp.shape[2:5]
            grads = None
            if gradmode:
                # The gradient buffers of the backward (mvpraymarch.py:240-246 zeros_like's them there) are made now and zero-filled
                # by the forward's render kernel on the side (mvp_forward_args::clear_grad_*): no memset pass in the step.  Only
                # those of the gradient set: a frozen template costs no template-sized buffer.
                # Deterministic: the int64 sums of the set take their place, and the gradients are allocated by the backward,
                # which writes them.
                grads = _empty_det_sums(gset, primpos, primrot, primscale, template) if det else \
                    _empty_grads(gset, primpos, primrot, primscale, template, warp, usewarp, tflags)
                a.clear_grad_primpos, a.clear_grad_primrot, a.clear_grad_primscale = _ptr(grads[0]), _ptr(grads[1]), _ptr(grads[2])
                a.clear_grad_tplate, a.clear_grad_warp = _ptr(grads[3]), _ptr(grads[4])
            stream = torch.cuda.current_stream(dev).cuda_stream
            if pixels is not None:
                _lib.check(_lib.LIB.mvp_raymarch_forward_pixels(ctypes.byref(a), _ptr(pixels), _ptr(view_set), NP,
                                                                ctypes.c_void_p(stream)))
            elif view_set is not None:
                _lib.check(_lib.LIB.mvp_raymarch_forward_sets(ctypes.byref(a), _ptr(view_set), NP, ctypes.c_void_p(stream)))
            else:
                _lib.check(_lib.LIB.mvp_raymarch_forward(ctypes.byref(a), ctypes.c_void_p(stream)))

        if gradmode:
            ctx.grads = grads
            ctx.save_for_backward(raypos, raydir, tminmax, primpos, primrot, primscale, template, raysat, rayaux, workspace, warp,
                                  *saved_extra)
            ctx.camera = camera                # camera tensors: no gradients (utils.py:45-46), except through MVPRaymarchCameraGrad
            ctx.nhw = (N, H, W)
            ctx.order = order
            ctx.options = options
            ctx.stepsize = float(stepsize)
            ctx.shared = shared
            ctx.view_set = view_set
            ctx.tflags = tflags
            ctx.det = det
        if planes:
            return rayrgb, rayalpha
        return rayrgba

    @staticmethod
    def backward(ctx, grad_rayrgba, grad_rayalpha=None):
        """grad_rayrgba [N,H,W,4]; or, for MVPRaymarchPlanes, (grad_rayrgb [N,3,H,W], grad_rayalpha [N,1,H,W]).  With the
        `_ray_grads` option (a differentiable `compute_raydirs` feeds the rays, see `mvpraymarch_camera`) the rays get gradients too."""
        if ctx.gset is None:                   # no input of this op gets a gradient (see _forward): nothing to compute
            return (None,) * 12
        want_rays = bool(ctx.options.get("_ray_grads")) and any(ctx.needs_input_grad[i] for i in (0, 1, 3))
        prim, rays = _march_backward(ctx, grad_rayrgba, grad_rayalpha, want_rays)
        grad_raypos, grad_raydir, grad_tminmax = rays if rays is not None else (None, None, None)
        return (grad_raypos, grad_raydir, None, grad_tminmax) + prim + (None, None, None)


def _march_backward(ctx, grad_rayrgba, grad_rayalpha, want_rays):
    """The native backward of an MVPRaymarch forward: ((grad_primpos, grad_primrot, grad_primscale, grad_template, grad_warp),
    (grad_raypos, grad_raydir, grad_tminmax) with want_rays (mvp_raymarch_backward_rays), else None).  The primitive gradients
    outside the forward's gradient set (ctx.gset) are None."""
    raypos, raydir, tminmax, primpos, primrot, primscale, template, raysat, rayaux, workspace, warp = ctx.saved_tensors[:11]
    options = ctx.options
    N, H, W = ctx.nhw
    K = primpos.size(1)
    TD, TH, TW = template.shape[2:5]
    dev = primpos.device
    with torch.cuda.device(dev):
        planes = bool(options.get("_planes", False))
        if planes:
            grad_rgb = grad_rayrgba.contiguous() if grad_rayrgba is not None else torch.zeros((N, 3, H, W), device=dev)
            grad_alpha = grad_rayalpha.contiguous() if grad_rayalpha is not None else torch.zeros((N, 1, H, W), device=dev)
            grad_rayrgba = None
        else:
            grad_rayrgba = _aligned(grad_rayrgba.contiguous(), 16)     # mvpraymarch.py:264
        usewarp = options["algo"] == 1
        gset = ctx.gset
        if gset == GRADS_RAYS_ONLY:
            assert want_rays, "a rays-only backward without ray gradients"
        grads, ctx.grads = ctx.grads, None
        # the forward's render kernel zero-filled them; a second backward through the same graph (retain_graph) gets new ones,
        # zero-filled by the library.  Deterministic: those buffers are the int64 sums, and the gradients are written by the library.
        fresh = grads is not None
        det = ctx.det
        sums = None
        if det:
            sums = grads if fresh else _empty_det_sums(gset, primpos, primrot, primscale, template)
            grads = _empty_grads(gset, primpos, primrot, primscale, template, warp, usewarp, ctx.tflags)
        elif not fresh:
            grads = _empty_grads(gset, primpos, primrot, primscale, template, warp, usewarp, ctx.tflags)
        grad_primpos, grad_primrot, grad_primscale, grad_template, grad_warp = grads
        if warp is not None and not usewarp and gset == GRADS_ALL:  # mvpraymarch.py:246 (zero when algo 0 ignores it)
            grad_warp = torch.zeros_like(warp)
        a = _lib.BackwardArgs()
        a.shape = _lib.Shape(N, H, W, K, TD, TH, TW)
        a.stepsize, a.fadescale, a.fadeexp = ctx.stepsize, float(options["fadescale"]), float(options["fadeexp"])
        a.flags = _lib.FLAG_ACCEL_VALID | (0 if fresh else _lib.FLAG_ZERO_GRADS) | (_lib.FLAG_SHARED_PRIMS if ctx.shared else 0) | \
            ctx.tflags | _GRAD_SET_FLAGS[gset]
        a.raypos, a.raydir, a.tminmax = _ptr(raypos), _ptr(raydir), _ptr(tminmax)
        if ctx.camera is not None:
            viewpos, viewrot, focal, princpt, volradius = ctx.camera[:5]
            a.camera = _lib.Camera(_ptr(viewpos), _ptr(viewrot), _ptr(focal), _ptr(princpt), float(volradius), 0)
        a.primpos, a.primrot, a.primscale = _ptr(primpos), _ptr(primrot), _ptr(primscale)
        a.tplate = _ptr(template)
        a.grad_rayrgba, a.raysat, a.rayaux = _ptr(grad_rayrgba), _ptr(raysat), _ptr(rayaux)
        if planes:
            a.grad_rayrgb_nchw, a.grad_rayalpha_nchw = _ptr(grad_rgb), _ptr(grad_alpha)
        if ctx.order is not None:
            a.order = _ptr(ctx.order)
        a.grad_primpos, a.grad_primrot, a.grad_primscale = _ptr(grad_primpos), _ptr(grad_primrot), _ptr(grad_primscale)
        a.grad_tplate = _ptr(grad_template)
        a.workspace, a.workspace_bytes = _ptr(workspace), workspace.numel()
        a.algo = 1 if usewarp else 0
        if usewarp:
            a.warp, a.grad_warp = _ptr(warp), _ptr(grad_warp)
            a.WD, a.WH, a.WW = warp.shape[2:5]
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        rays = None
        if want_rays:
            _lib.require_ray_grads()
            # written for every ray by the library: no zero-fill
            rays = (torch.empty((N, H, W, 3), device=dev), torch.empty((N, H, W, 3), device=dev), torch.empty((N, H, W, 2), device=dev))
        pixels = options.get("_pixels")
        if det:
            det_max = torch.empty(4, dtype=torch.int32, device=dev)
            _lib.check(_lib.LIB.mvp_raymarch_backward_deterministic(ctypes.byref(a), *(_ptr(t) for t in sums[:4]), _ptr(det_max),
                                                                    _ptr(pixels), _ptr(ctx.view_set), primpos.size(0), stream))
            return (grad_primpos, grad_primrot, grad_primscale, grad_template, grad_warp), None
        if pixels is not None and want_rays:
            # The ray-gradient backward of a pixels forward marches the rays mvp_compute_raydirs makes from the same pixelcoords:
            # bit for bit the rays the forward generated, so its acceleration structure and saved tile lists hold for them.  The
            # camera's adjoint (MVPRaymarchCameraGrad) then runs mvp_compute_raydirs_backward at the same pixelcoords.
            from .raydirs import compute_raydirs
            viewpos, viewrot, focal, princpt, volradius = ctx.camera[:5]
            raypos, raydir, tminmax = compute_raydirs(viewpos, viewrot, focal, princpt, pixels, volradius)
            a.raypos, a.raydir, a.tminmax = _ptr(raypos), _ptr(raydir), _ptr(tminmax)
            a.camera = _lib.Camera()
            pixels = None
        if pixels is not None:
            _lib.check(_lib.LIB.mvp_raymarch_backward_pixels(ctypes.byref(a), _ptr(pixels), _ptr(ctx.view_set), primpos.size(0),
                                                             *(_ptr(t) for t in (rays or (None,) * 3)), stream))
        elif ctx.view_set is not None:
            _lib.check(_lib.LIB.mvp_raymarch_backward_sets(ctypes.byref(a), _ptr(ctx.view_set), primpos.size(0),
                                                           *(_ptr(t) for t in (rays or (None,) * 3)), stream))
        elif want_rays:
            _lib.check(_lib.LIB.mvp_raymarch_backward_rays(ctypes.byref(a), *(_ptr(t) for t in rays), stream))
        else:
            _lib.check(_lib.LIB.mvp_raymarch_backward(ctypes.byref(a), stream))
    return (grad_primpos, grad_primrot, grad_primscale, grad_template, grad_warp), rays


class MVPRaymarchPlanes(MVPRaymarch):
    """Same op with the outputs as the caller uses them: (rayrgb [N,3,H,W], rayalpha [N,1,H,W]), written by the render
    kernel's epilogue, and the gradient taken as those two planes by the backward's prologue -- the permute + two
    `.contiguous()` copies of models/raymarchers/mvpraymarcher.py:50-51 and the `.contiguous()` of the incoming gradient
    (mvpraymarch.py:264) never run (SURVEY.md section 8f row 2)."""

    @staticmethod
    def forward(ctx, raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template, warp, rayterm, gradmode, options):
        options = dict(options, _planes=True)
        return MVPRaymarch.forward(ctx, raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template, warp, rayterm,
                                   gradmode, options)

    @staticmethod
    def backward(ctx, grad_rayrgb, grad_rayalpha):
        return MVPRaymarch.backward(ctx, grad_rayrgb, grad_rayalpha)


class MVPRaymarchCameraGrad(Function):
    """The camera form of the op (`options["_camera"]`: rays generated in the kernels) with the four camera tensors as autograd
    inputs: the backward writes each ray's gradient into a temporary 32 B/ray buffer (mvp_raymarch_backward_rays) and the ray
    generator's adjoint (mvp_compute_raydirs_backward) reduces them per view.  Outputs as MVPRaymarch (or its planes form)."""

    @staticmethod
    def forward(ctx, viewpos, viewrot, focal, princpt, stepsize, primpos, primrot, primscale, template, warp, gradmode, options):
        # the camera tensors are saved for backward: the adjoint recomputes the rays from them
        return MVPRaymarch._forward(ctx, None, None, stepsize, None, primpos, primrot, primscale, template, warp, None, gradmode, options,
                                    saved_extra=(viewpos, viewrot, focal, princpt), first_prim=5, ray_inputs=(0, 1, 2, 3))

    @staticmethod
    def backward(ctx, grad_out, grad_rayalpha=None):
        if ctx.gset is None:
            return (None,) * 12
        prim, rays = _march_backward(ctx, grad_out, grad_rayalpha, True)
        viewpos, viewrot, focal, princpt = ctx.saved_tensors[11:15]
        volradius = ctx.camera[4]
        from .raydirs import raydirs_backward
        cam = raydirs_backward(viewpos, viewrot, focal, princpt, ctx.options.get("_pixels"), volradius, *rays)
        cam = tuple(g if need else None for g, need in zip(cam, ctx.needs_input_grad[:4]))
        return cam + (None,) + prim + (None, None)


def morton_codes(primpos):
    """30-bit Morton codes of the primitive centres, normalised per view to their bounding box: the reference's
    build_accel (mvpraymarch.py:46-53) + morton3D / expand_bits (bvh.cu:20-41).  [N,K] int64."""
    cmax = primpos.max(dim=1, keepdim=True)[0]
    cmin = primpos.min(dim=1, keepdim=True)[0]
    c = (primpos - cmin) / (cmax - cmin).clamp(min=1e-8)                       # mvpraymarch.py:50
    q = (c * 1024.0).clamp(0.0, 1023.0).to(torch.int64)                        # bvh.cu:33-35, (unsigned int) truncates

    def expand_bits(v):                                                        # bvh.cu:22-28 (uint32 arithmetic)
        v = (v * 0x00010001) & 0xFF0000FF
        v = (v * 0x00000101) & 0x0F00F00F
        v = (v * 0x00000011) & 0xC30C30C3
        v = (v * 0x00000005) & 0x49249249
        return v

    return expand_bits(q[..., 0]) * 4 + expand_bits(q[..., 1]) * 2 + expand_bits(q[..., 2])   # bvh.cu:39


def morton_codes_native(primpos):
    """The same codes from the library's kernel (`mvp_compute_morton`, the reference's compute_morton): the normalisation to the
    bounding box stays in torch like in the reference (mvpraymarch.py:46-50).  [N,K] int32."""
    p = primpos.detach()
    cmax = p.max(dim=1, keepdim=True)[0]
    cmin = p.min(dim=1, keepdim=True)[0]
    c = ((p - cmin) / (cmax - cmin).clamp(min=1e-8)).contiguous()
    code = torch.empty(p.shape[:2], dtype=torch.int32, device=p.device)
    with torch.cuda.device(p.device):
        _lib.check(_lib.LIB.mvp_compute_morton(p.shape[0], p.shape[1], _ptr(c), _ptr(code),
                                               ctypes.c_void_p(torch.cuda.current_stream(p.device).cuda_stream)))
    return code


def morton_order(primpos):
    """sortedobjid [N,K] (int64): primitive indices in ascending Morton code (mvpraymarch.py:54-55).  Ties keep index
    order (stable), where the reference's torch.sort leaves them unspecified."""
    codes = morton_codes_native(primpos) if primpos.is_cuda else morton_codes(primpos.detach())
    return torch.sort(codes, dim=-1, stable=True)[1]


def _take(t, order):
    """t[n, order[n, k], ...] (differentiable)."""
    if t is None:
        return None
    idx = order.view(order.shape + (1,) * (t.dim() - 2)).expand(order.shape + tuple(t.shape[2:]))
    return torch.gather(t, 1, idx)


def mvpraymarch(
    raypos,
    raydir,
    stepsize,
    tminmax,
    primtransf,
    template,
    warp,
    rayterm=None,
    algo=0,
    usebvh="fixedorder",
    sortprims=False,
    randomorder=False,
    maxhitboxes=512,
    synchitboxes=True,
    chlast=True,
    fadescale=8.0,
    fadeexp=8.0,
    accum=0,
    termthresh=0.0,
    griddim=3,
    blocksize=(8, 16),
    bwdblocksize=(8, 16),
):
    """Drop-in for extensions.mvpraymarch.mvpraymarch.mvpraymarch (reference mvpraymarch.py:295-390).

    Same parameters, same defaults.  `sortprims`, `randomorder`, `maxhitboxes`, `synchitboxes`, `chlast`, `accum`,
    `termthresh`, `griddim`, `blocksize`, `bwdblocksize` and `rayterm` are accepted and, exactly like in the
    reference kernels (SURVEY.md section 8a, "accepted but ignored"), have no effect on the result.

    `usebvh="fixedorder"` (default) marches the primitives of a tile in index order.  `usebvh=True` marches them in
    Morton order of their centres -- the order the reference's LBVH branch computes (`sortedobjid`, mvpraymarch.py:46-55)
    but its kernels never apply (they hard-code the implicit heap, utils.h:740-742; SURVEY.md section 2.3 K5): codes from the
    library's `mvp_compute_morton`, one `torch.sort`, and the order goes to the kernels as an indirection (no tensor is
    gathered or copied).  The order only matters for rays that saturate.
    Returns rayrgba [N,H,W,4]."""
    if usebvh is False:
        raise NotImplementedError("mvpraymarch_b200: usebvh=False hands the reference kernels a null BVH "
                                  "(mvpraymarch.py:132-134); use 'fixedorder' or True")
    if isinstance(primtransf, tuple):
        primpos, primrot, primscale = primtransf
    else:                                                              # packed [N,K,5,3]  (mvpraymarch.py:353-360)
        primpos = primtransf[:, :, 0, :].contiguous()
        primrot = primtransf[:, :, 1:4, :].contiguous()
        primscale = primtransf[:, :, 4, :].contiguous()
    # under torch.autocast the decoders hand over bfloat16 transforms: widened here, outside the autograd Function, so that
    # torch casts their gradients back (the template itself goes to the kernels as bfloat16)
    primpos, primrot, primscale, warp = (_widen_bf16(t) for t in (primpos, primrot, primscale, warp))
    order = None
    if usebvh != "fixedorder":
        # Morton order of the centres as an indirection inside the kernels (C-ABI `order`): nothing is gathered or copied
        order = morton_order(primpos).to(torch.int32).contiguous()
    options = {
        "algo": algo, "usebvh": usebvh, "sortprims": sortprims, "randomorder": randomorder,
        "maxhitboxes": maxhitboxes, "synchitboxes": synchitboxes, "chlast": chlast, "fadescale": fadescale,
        "fadeexp": fadeexp, "accum": accum, "termthresh": termthresh, "griddim": griddim, "blocksize": blocksize,
        "bwdblocksize": bwdblocksize, "_order": order, "_template_grad_dtype": _TEMPLATE_GRAD.get("dtype"),
        "_deterministic": bool(_DETERMINISTIC.get("on")),
    }
    if _VIEW_SET.get("map") is not None:
        options["_view_set"] = _VIEW_SET["map"]
    if _CAMERA.get("cam") is not None:
        options["_camera"] = _CAMERA["cam"]
        options["_pixels"] = _CAMERA.get("pix")
    if _CAMERA.get("grad"):
        options["_ray_grads"] = True
        if options.get("_camera") is not None:
            if _PLANES.get("on"):
                options["_planes"] = True
            viewpos, viewrot, focal, princpt = options["_camera"][:4]
            return MVPRaymarchCameraGrad.apply(viewpos, viewrot, focal, princpt, stepsize, primpos, primrot, primscale, template, warp,
                                               torch.is_grad_enabled(), options)
    fn = MVPRaymarchPlanes if _PLANES.get("on") else MVPRaymarch
    return fn.apply(raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template, warp, rayterm,
                    torch.is_grad_enabled(), options)


_PLANES = {}
_CAMERA = {}     # "cam": the camera of a mvpraymarch_camera call (rays generated in the kernels); "pix": its pixelcoords tensor or None;
                # "grad": camera_grad=True
_VIEW_SET = {}   # "map": the view -> primitive set map of a mvpraymarch_sets call (or of view_set= elsewhere), or None


@contextlib.contextmanager
def _view_set_block(view_set):
    """Raymarch calls within the block render view n from primitive set view_set[n] (see `mvpraymarch_sets`); None: as usual."""
    prev = _VIEW_SET.get("map")
    _VIEW_SET["map"] = view_set
    try:
        yield
    finally:
        _VIEW_SET["map"] = prev


def _view_set_tensor(view_set, N, S, dev):
    """The view -> set map as a private int32 [N] tensor on `dev`, for S primitive sets.  A map given on the host (a sequence of ints
    or a CPU tensor) is range-checked here and raises ValueError; a CUDA map is not read back (no synchronisation): its entries
    outside [0, S) make their views render empty, as the library defines it (int64 entries are clamped to [-1, S] first, so that
    none wraps into range in the int32 conversion)."""
    if not torch.is_tensor(view_set):
        vals = list(view_set) if isinstance(view_set, (list, tuple, range)) else None
        if vals is None or not all(isinstance(v, numbers.Integral) and not isinstance(v, bool) for v in vals):
            raise TypeError("view_set must be an integer tensor or a sequence of ints, got %r" % (view_set,))
        view_set = torch.tensor([int(v) for v in vals], dtype=torch.int64)
    if view_set.dtype not in (torch.int32, torch.int64):
        raise TypeError("view_set must be int32 or int64, got %s" % view_set.dtype)
    if tuple(view_set.shape) != (N,):
        raise ValueError("view_set must have shape [N] = [%d], got %s" % (N, list(view_set.shape)))
    if not 1 <= S <= N:
        raise ValueError("with view_set, the primitive batch (%d sets) must lie in [1, N] = [1, %d]" % (S, N))
    if view_set.is_cuda:
        if view_set.device != dev:
            raise ValueError("view_set is on %s, the primitives on %s" % (view_set.device, dev))
        return view_set.clamp(-1, S).to(torch.int32).contiguous()
    if view_set.device.type != "cpu":
        raise ValueError("view_set must be on the CPU or on the primitives' device, got %s" % view_set.device)
    lo, hi = int(view_set.min()), int(view_set.max())
    if lo < 0 or hi >= S:
        raise ValueError("view_set entries must lie in [0, %d) (the primitive sets), got [%d, %d]" % (S, lo, hi))
    return view_set.to(dtype=torch.int32).to(dev)


def mvpraymarch_sets(raypos, raydir, stepsize, tminmax, primtransf, template, warp, view_set, planes=False, template_grad_dtype=None,
                     deterministic=None, **kwargs):
    """`mvpraymarch` over S primitive sets -- S subjects, or S frames -- rendered in one launch, view n from set view_set[n]: the
    primitives (primtransf, template, warp) are [S,K,...] with 1 <= S <= N, and so are their gradients (the template's in its dtype,
    or fp32 per `template_grad_dtype`).  Each set's gradient sums those of its views; a set no view shows gets zero gradients.
    view_set is an integer tensor [N] (int32 or int64, on the CPU or on the primitives' device) or a sequence of ints, and gets no
    gradient.  A host map is range-checked (ValueError); a CUDA map is not read back, and a view whose entry is outside [0, S)
    renders empty (zero colour and alpha) and contributes no gradient.  Replaces `payload.expand_views` + `mvpraymarch` +
    `sum_views` for views that share a subject: no per-view copy of the primitives and no per-view gradient.  With usebvh=True each
    set is marched in its own Morton order.  The other keyword arguments are those of `mvpraymarch`; ray gradients (camera fitting)
    come through `mvpraymarch_camera(..., view_set=...)`.  deterministic=True: reproducible primitive gradients (see
    `deterministic_grads`); None leaves the setting of an enclosing `deterministic_grads` block.
    Returns rayrgba [N,H,W,4], or (rayrgb [N,3,H,W], rayalpha [N,1,H,W]) with planes=True."""
    if view_set is None:
        raise TypeError("mvpraymarch_sets: view_set is required (use mvpraymarch for per-view or shared primitives)")
    march = mvpraymarch_planes if planes else mvpraymarch
    grad_block = _template_grad_block(template_grad_dtype) if _check_template_grad_dtype(template_grad_dtype) is not None \
        else contextlib.nullcontext()
    with grad_block, _view_set_block(view_set), _det_context(deterministic):
        return march(raypos, raydir, stepsize, tminmax, primtransf, template, warp, **kwargs)


def mvpraymarch_planes(*args, **kwargs):
    """`mvpraymarch` with image-plane outputs: same parameters, returns (rayrgb [N,3,H,W], rayalpha [N,1,H,W]) instead of
    rayrgba [N,H,W,4] (see MVPRaymarchPlanes; used by `ava256_b200.raymarcher.Raymarcher`)."""
    _PLANES["on"] = True
    try:
        return mvpraymarch(*args, **kwargs)
    finally:
        _PLANES["on"] = False


def mvpraymarch_camera(viewpos, viewrot, focal, princpt, pixelcoords, volradius, stepsize, primtransf, template, warp, planes=False,
                       camera_grad=False, template_grad_dtype=None, view_set=None, deterministic=None, **kwargs):
    """`compute_raydirs` + `mvpraymarch` of models/autoencoder.py:240-252 as ONE call: the first six parameters are those of the
    reference's compute_raydirs (extensions/utils/utils.py:48-51), the rest those of `mvpraymarch` after its ray arguments.

    The rays never exist in memory: the render kernels generate each tile's rays in their prologue from the camera (C-ABI
    `mvp_camera`), bit-identical to what `compute_raydirs` would have written -- 32 bytes per ray that are neither written by a
    generation pass nor read by forward and backward.  `pixelcoords` is the `(W, H)` tuple (the integer pixel grid, utils.py:28-30),
    or a float32 CUDA tensor [N,H,W,2] of sample positions on the primitives' device (e.g. the dataset's meshgrid, a crop or a
    strided sub-grid; a tensor that is not contiguous or not 8-byte aligned is copied once), from which each lane reads its own
    position (C-ABI `mvp_raymarch_forward_pixels`).  The accel build takes the camera as it is instead of fitting one to a ray field;
    a tensor whose views follow an axis-aligned map px = ox + sx w, py = oy + sy h keeps the slab culling, any other field renders
    the same image with every slab a candidate (slower).  pixelcoords gets no gradient.
    By default no gradients flow to the camera, like the reference (its compute_raydirs backward returns None for every input,
    utils.py:45-46).  With camera_grad=True, viewpos, viewrot, focal and princpt are autograd inputs and those that require grad get
    the gradient of the image with every discrete decision of the march held fixed (C-ABI mvp_raymarch_backward_rays, then the ray
    generator's adjoint mvp_compute_raydirs_backward at the same pixelcoords); pixelcoords and volradius get none.  With a
    pixelcoords tensor the forward generates the rays in the kernels as always, and the ray-gradient backward marches the rays
    `compute_raydirs` makes from the same tensor (bit-identical; they exist during the backward only).  When no camera tensor
    requires grad, the plain backward runs.  The backward computes only what requires grad: with the template and transforms
    detached (a frozen avatar) it computes the ray gradients alone, with no template-sized gradient buffer and no payload-gradient
    scatter.
    template_grad_dtype=torch.float32 accumulates a bfloat16 template's gradient in fp32 (see the `template_grad_dtype` context
    manager); None leaves the setting of an enclosing `template_grad_dtype` block, by default the template's own dtype.
    view_set: the views render S primitive sets [S,K,...], view n set view_set[n] (see `mvpraymarch_sets`).
    deterministic=True: reproducible primitive gradients (see `deterministic_grads`; not with camera_grad); None leaves the setting
    of an enclosing `deterministic_grads` block.
    Returns rayrgba [N,H,W,4], or (rayrgb [N,3,H,W], rayalpha [N,1,H,W]) with planes=True."""
    if deterministic is not None:
        with _deterministic_block(bool(deterministic)):
            return mvpraymarch_camera(viewpos, viewrot, focal, princpt, pixelcoords, volradius, stepsize, primtransf, template, warp,
                                      planes=planes, camera_grad=camera_grad, template_grad_dtype=template_grad_dtype,
                                      view_set=view_set, **kwargs)
    if view_set is not None:
        with _view_set_block(view_set):
            return mvpraymarch_camera(viewpos, viewrot, focal, princpt, pixelcoords, volradius, stepsize, primtransf, template, warp,
                                      planes=planes, camera_grad=camera_grad, template_grad_dtype=template_grad_dtype, **kwargs)
    if _check_template_grad_dtype(template_grad_dtype) is not None:
        with _template_grad_block(template_grad_dtype):
            return mvpraymarch_camera(viewpos, viewrot, focal, princpt, pixelcoords, volradius, stepsize, primtransf, template, warp,
                                      planes=planes, camera_grad=camera_grad, **kwargs)
    march = mvpraymarch_planes if planes else mvpraymarch
    grad = bool(camera_grad) and torch.is_grad_enabled() and any(t.requires_grad for t in (viewpos, viewrot, focal, princpt))
    if grad:
        _lib.require_ray_grads()
    if isinstance(pixelcoords, tuple):
        W, H = pixelcoords
        pix = None
    else:
        if not torch.is_tensor(pixelcoords) or pixelcoords.dim() != 4:
            raise TypeError("pixelcoords must be the (W, H) tuple or a tensor [N,H,W,2]")
        H, W = pixelcoords.size(1), pixelcoords.size(2)
        pix = _aligned(pixelcoords.detach().contiguous(), 8)
    _CAMERA["cam"] = (viewpos, viewrot, focal, princpt, float(volradius), int(H), int(W))
    _CAMERA["pix"] = pix
    _CAMERA["grad"] = grad
    try:
        return march(None, None, stepsize, None, primtransf, template, warp, **kwargs)
    finally:
        _CAMERA["cam"] = None
        _CAMERA["pix"] = None
        _CAMERA["grad"] = False
