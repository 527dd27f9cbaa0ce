"""TEST INFRASTRUCTURE: numpy front-end of tests/emul/libmvp_emul.so -- the PRODUCT kernels' source
(ava-256_b200/csrc/mvp_kernels.cu) compiled for the host on the CPU emulation of warps / blocks / shared memory in
cuda_emul.h.  Same C-ABI as the product library (struct layouts are taken from ava256_b200.lib), host pointers in
place of device pointers."""
import ctypes

import numpy as np

from ava256_b200 import lib as _abi
from tests.emul.build import build_kernels

_LIBS = {}
_variant = ()
_opt = "-O1"
last_heavy_tiles = (0, 0)   # (forward, backward) heavy-tile counts of the last forward_backward call (mvp_debug_heavy_offset)


def use_variant(defines=(), opt="-O1"):
    """Select the build-time variant of the kernels (a tuple of -D defines) used by subsequent calls; opt="-O0" builds
    three times faster and is plenty for the small test scenes."""
    global _variant, _opt
    _variant, _opt = tuple(defines), opt


def load():
    key = (_variant, _opt)
    if key not in _LIBS:
        L = ctypes.CDLL(build_kernels(_variant, _opt))
        L.mvp_workspace_bytes.restype = ctypes.c_size_t
        L.mvp_workspace_bytes.argtypes = [ctypes.POINTER(_abi.Shape)]
        L.mvp_raymarch_forward.restype = ctypes.c_int
        L.mvp_raymarch_forward.argtypes = [ctypes.POINTER(_abi.ForwardArgs), ctypes.c_void_p]
        L.mvp_raymarch_backward.restype = ctypes.c_int
        L.mvp_raymarch_backward.argtypes = [ctypes.POINTER(_abi.BackwardArgs), ctypes.c_void_p]
        L.mvp_abi_version.restype = ctypes.c_int
        L.mvp_debug_heavy_offset.restype = ctypes.c_size_t
        L.mvp_debug_heavy_offset.argtypes = [ctypes.POINTER(_abi.Shape)]
        assert L.mvp_abi_version() == _abi.ABI_VERSION
        _LIBS[key] = L
    return _LIBS[key]


def set_lane_order(mode):
    """'forward' | 'reverse' | 'random': order in which the lanes of a block run between collectives."""
    load().emul_set_lane_order({"forward": 0, "reverse": 1, "random": 2}[mode])


def _p(a):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


def _aligned(nbytes, align=256):
    raw = np.zeros(nbytes + align, np.uint8)
    off = (-raw.ctypes.data) % align
    return raw[off:off + nbytes]


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _nan_like16(x):
    """NaN-filled array of x's shape whose data pointer is 16-byte aligned."""
    raw = np.empty(x.size + 4, np.float32)
    off = (-raw.ctypes.data // 4) % 4
    out = raw[off:off + x.size].reshape(x.shape)
    out[...] = np.nan
    return out


def forward_backward(raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template, grad_rayrgba=None, warp=None,
                     fadescale=8.0, fadeexp=8.0, fwd_flags=0, bwd_flags=0, planes=False, order=None, clear_in_forward=False, camera=None):
    """Runs the emulated forward (and, when grad_rayrgba is given, backward) kernels.
    Returns (rayrgba, raysat, grads) with grads = [primpos, primrot, primscale, template(, warp)] or None.
    clear_in_forward: the gradient buffers are handed to the forward NaN-filled (mvp_forward_args::clear_grad_*), which must leave
    them zero; the backward then runs without MVP_FLAG_ZERO_GRADS.
    camera = (viewpos, viewrot, focal, princpt, volradius, H, W): the kernels generate the rays (mvp_camera); raypos / raydir / tminmax
    must then be None and are passed as NULL.
    The numbers of heavy tiles (rendered by the 512-entry kernels) of the forward and the backward are left in last_heavy_tiles."""
    global last_heavy_tiles
    L = load()
    primpos, primrot, primscale, template = map(_f32, (primpos, primrot, primscale, template))
    warp = None if warp is None else _f32(warp)
    cam = None
    if camera is not None:
        assert raypos is None and raydir is None and tminmax is None
        camarrs = [_f32(x) for x in camera[:4]]
        cam = _abi.Camera(_p(camarrs[0]), _p(camarrs[1]), _p(camarrs[2]), _p(camarrs[3]), float(camera[4]), 0)
        N, H, W = camarrs[0].shape[0], int(camera[5]), int(camera[6])
    else:
        raypos, raydir, tminmax = map(_f32, (raypos, raydir, tminmax))
        N, H, W = raypos.shape[:3]
    K = primpos.shape[1]
    TD, TH, TW = template.shape[2:5]
    shape = _abi.Shape(N, H, W, K, TD, TH, TW)
    wsb = L.mvp_workspace_bytes(ctypes.byref(shape))
    assert wsb > 0
    ws = _aligned(wsb)
    hoff = L.mvp_debug_heavy_offset(ctypes.byref(shape))
    heavy = lambda: int(ws[hoff:hoff + 4].view(np.int32)[0])  # noqa: E731
    rayrgba = np.full((N, H, W, 4), np.nan, np.float32)
    want_grad = grad_rayrgba is not None
    raysat = np.full((N, H, W, 3), np.nan, np.float32) if want_grad else None
    rayaux = np.zeros((N, H, W, 4), np.int32) if want_grad else None
    a = _abi.ForwardArgs()
    a.shape = shape
    a.stepsize, a.fadescale, a.fadeexp, a.flags = float(stepsize), float(fadescale), float(fadeexp), fwd_flags
    a.raypos, a.raydir, a.tminmax = _p(raypos), _p(raydir), _p(tminmax)
    if cam is not None:
        a.camera = cam
    a.primpos, a.primrot, a.primscale, a.tplate = _p(primpos), _p(primrot), _p(primscale), _p(template)
    rgb_p = np.full((N, 3, H, W), np.nan, np.float32) if planes else None
    alpha_p = np.full((N, 1, H, W), np.nan, np.float32) if planes else None
    a.rayrgba, a.raysat, a.rayaux = (None if planes else _p(rayrgba)), _p(raysat), _p(rayaux)
    if planes:
        a.rayrgb_nchw, a.rayalpha_nchw = _p(rgb_p), _p(alpha_p)
    if order is not None:
        order = np.ascontiguousarray(order, dtype=np.int32)
        a.order = _p(order)
    a.workspace, a.workspace_bytes = _p(ws), wsb
    a.algo = 1 if warp is not None else 0
    if warp is not None:
        a.warp = _p(warp)
        a.WD, a.WH, a.WW = warp.shape[2:5]
    pre = None
    if clear_in_forward:
        assert want_grad and not (bwd_flags & _abi.FLAG_ZERO_GRADS)
        pre = [_nan_like16(x) for x in (primpos, primrot, primscale, template)] + [_nan_like16(warp) if warp is not None else None]
        a.clear_grad_primpos, a.clear_grad_primrot, a.clear_grad_primscale, a.clear_grad_tplate = (_p(g) for g in pre[:4])
        a.clear_grad_warp = _p(pre[4])
    rc = L.mvp_raymarch_forward(ctypes.byref(a), None)
    assert rc == 0, rc
    last_heavy_tiles = (heavy(), 0)
    if pre is not None:
        assert all(g is None or not g.any() for g in pre), "the forward must leave the clear_grad_* buffers zero"
    if planes:                      # hand back the same layout as the channels-last run, assembled from the planes
        rayrgba = np.ascontiguousarray(np.concatenate([rgb_p, alpha_p], axis=1).transpose(0, 2, 3, 1))
    if not want_grad:
        return rayrgba, None, None
    grad_rayrgba = _f32(grad_rayrgba)
    fill = np.nan if (bwd_flags & _abi.FLAG_ZERO_GRADS) else 0.0           # ZERO_GRADS: the library must overwrite the NaNs
    grads = pre[:4] if pre is not None else [np.full_like(x, fill) for x in (primpos, primrot, primscale, template)]
    gwarp = pre[4] if pre is not None else (np.full_like(warp, fill) if warp is not None else None)
    b = _abi.BackwardArgs()
    b.shape = shape
    b.stepsize, b.fadescale, b.fadeexp, b.flags = float(stepsize), float(fadescale), float(fadeexp), _abi.FLAG_ACCEL_VALID | bwd_flags
    b.raypos, b.raydir, b.tminmax = _p(raypos), _p(raydir), _p(tminmax)
    if cam is not None:
        b.camera = cam
    b.primpos, b.primrot, b.primscale, b.tplate = _p(primpos), _p(primrot), _p(primscale), _p(template)
    if planes:
        g_rgb = np.ascontiguousarray(grad_rayrgba.transpose(0, 3, 1, 2)[:, :3])
        g_alpha = np.ascontiguousarray(grad_rayrgba.transpose(0, 3, 1, 2)[:, 3:4])
        b.grad_rayrgb_nchw, b.grad_rayalpha_nchw = _p(g_rgb), _p(g_alpha)
    b.grad_rayrgba, b.raysat, b.rayaux = (None if planes else _p(grad_rayrgba)), _p(raysat), _p(rayaux)
    b.grad_primpos, b.grad_primrot, b.grad_primscale, b.grad_tplate = (_p(g) for g in grads)
    if order is not None:
        b.order = _p(order)
    b.workspace, b.workspace_bytes = _p(ws), wsb
    b.algo = a.algo
    if warp is not None:
        b.warp, b.grad_warp = _p(warp), _p(gwarp)
        b.WD, b.WH, b.WW = warp.shape[2:5]
    rc = L.mvp_raymarch_backward(ctypes.byref(b), None)
    assert rc == 0, rc
    last_heavy_tiles = (last_heavy_tiles[0], heavy())
    if gwarp is not None:
        grads.append(gwarp)
    return rayrgba, raysat, grads
