"""GPU tests of bfloat16 templates (`pytest -m gpu`): every case runs the public op twice, on a bf16 template `tb` and on its
fp32 widening `tb.float()`.  The contract: images (channels-last or planes) bit-identical; primpos / primrot / primscale (and
warp) gradients within 1e-5 of max|.| (the order of the fp32 atomics); the bf16 template gradient within the gates of
tests/test_emul_bf16_payload.py, which also explains them."""
import ctypes
import gc

import pytest
import torch

from tests.helpers import CASES, DENSE_CASES, DENSE_K3, build_case, build_dense_case, gradcheck_like_scene
from tests.test_emul_bf16_payload import GATE_DENSE_L1, GATE_DENSE_MAX, GATE_L1, GATE_MAX

pytestmark = pytest.mark.gpu

NAMES = ("primpos", "primrot", "primscale", "template", "warp")


def _relerr(a, b):
    return float((a.double() - b.double()).abs().max() / max(float(b.double().abs().max()), 1e-30))


def _tgrad_errors(gb, g32):
    d = (gb.double() - g32.double()).abs()
    return float(d.max() / max(float(g32.double().abs().max()), 1e-30)), float(d.sum() / max(float(g32.double().abs().sum()), 1e-30))


def _cuda_scene(s):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in s.items()}


def render(s, template, grad, planes=False, camera=None, shared=False, retain=False, keep=None):
    """Forward (+ backward when grad is given) through the public op.  Returns (image, {name: gradient})."""
    from ava256_b200.op import mvpraymarch, mvpraymarch_camera, mvpraymarch_planes
    sl = (lambda x: x[:1].contiguous()) if shared else (lambda x: x)
    leaves = {"primpos": sl(s["primpos"]), "primrot": sl(s["primrot"]), "primscale": sl(s["primscale"]), "template": sl(template)}
    if s.get("warp") is not None:
        leaves["warp"] = s["warp"]
    with torch.set_grad_enabled(grad is not None):
        for x in leaves.values():
            x.requires_grad_(grad is not None)
        kw = dict(fadescale=s.get("fadescale", 8.0), fadeexp=s.get("fadeexp", 8.0), algo=1 if "warp" in leaves else 0)
        prim = (leaves["primpos"], leaves["primrot"], leaves["primscale"])
        if camera is not None:
            out = mvpraymarch_camera(*camera, s["stepsize"], prim, leaves["template"], leaves.get("warp"), planes=planes, **kw)
        else:
            f = mvpraymarch_planes if planes else mvpraymarch
            out = f(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], prim, leaves["template"], leaves.get("warp"), **kw)
        img = torch.cat([out[0], out[1]], dim=1).permute(0, 2, 3, 1) if planes else out
        if grad is None:
            torch.cuda.synchronize()
            return img.detach(), None
        if keep is not None:
            keep["workspace"] = img.grad_fn.saved_tensors[9] if not planes else out[0].grad_fn.saved_tensors[9]
        gs = torch.autograd.grad(img, list(leaves.values()), grad, retain_graph=retain)
        if keep is not None and retain:
            keep["second"] = torch.autograd.grad(img, list(leaves.values()), grad)
    torch.cuda.synchronize()
    return img.detach(), dict(zip(leaves, gs))


def compare(s, grad, gates=(GATE_MAX, GATE_L1), **kw):
    """bf16 template against its fp32 widening: the contract of this module.  Returns the bf16 run's (image, gradients)."""
    tb = s["template"].to(torch.bfloat16)
    out32, g32 = render(s, tb.float(), grad, **kw)
    outb, gb = render(s, tb.clone(), grad, **kw)
    assert torch.equal(outb, out32)
    assert gb["template"].dtype == torch.bfloat16 and gb["template"].shape == g32["template"].shape
    for nm in g32:
        assert bool(torch.isfinite(gb[nm].float()).all()), nm
        if nm != "template":
            assert gb[nm].dtype == torch.float32 and _relerr(gb[nm], g32[nm]) <= 1e-5, nm
    emax, el1 = _tgrad_errors(gb["template"], g32["template"])
    print("bf16 grad_template: max %.3g  l1 %.3g" % (emax, el1))
    assert emax <= gates[0] and el1 <= gates[1], (emax, el1)
    return outb, gb, g32


@pytest.mark.parametrize("name", list(CASES))
def test_bf16_template_named_cases(name):
    s, grad = build_case(name)
    s, grad = _cuda_scene(s), grad.cuda()
    out, _, _ = compare(s, grad)
    tb = s["template"].to(torch.bfloat16)
    with torch.no_grad():                                                        # inference forward: bit-identical
        assert torch.equal(render(s, tb, None)[0], out)


@pytest.mark.parametrize("cap", list(DENSE_K3))
@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_bf16_template_heavy_kernels(name, cap):
    """Every tile through the 512-entry kernels (the forward's heavy-tile count read back from the op's workspace)."""
    from ava256_b200 import lib
    s, grad = build_dense_case(name, cap)
    s, grad = _cuda_scene(s), grad.cuda()
    compare(s, grad, gates=(GATE_DENSE_MAX, GATE_DENSE_L1))
    keep = {}
    render(s, s["template"].to(torch.bfloat16), grad, keep=keep)
    N, H, W = s["raypos"].shape[:3]
    K, (TD, TH, TW) = s["primpos"].shape[1], s["template"].shape[2:5]
    off = lib.LIB.mvp_debug_heavy_offset(ctypes.byref(lib.Shape(N, H, W, K, TD, TH, TW)))
    assert int(keep["workspace"][off:off + 4].view(torch.int32).item()) == N * -(-H // 4) * -(-W // 8)   # the backward's count


def test_bf16_template_shared_primitives():
    """One [1,K,...] set for 4 views: the gradients of all views accumulate into one bf16 template gradient, so a voxel takes
    the roundings of 4 views (measured 0.030 / 0.0083): the gates of the scenes with many roundings per voxel."""
    s = _cuda_scene(gradcheck_like_scene(N=4, H=20, W=24, k3=3, M=6, seed=41, alpha_gain=8.0))
    grad = torch.randn(4, 20, 24, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    compare(s, grad, gates=(GATE_DENSE_MAX, GATE_DENSE_L1), shared=True)


def test_bf16_template_planes_and_camera_rays():
    from ava256_b200 import scene
    n, H, W, K, T = 2, 96, 64, 256, 8
    s = scene.make_scene(n, H, W, K, T, alpha_mu=3.0, alpha_sigma=3.0, share_primitives=False, device="cuda")
    s["stepsize"], s["fadescale"], s["fadeexp"] = 1.0 / 64, 8.0, 8.0
    grad = torch.randn(n, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    out, _, _ = compare(s, grad, planes=True)
    cams = [c.cuda() for c in scene.make_cameras(n, H, W)]
    camera = (cams[0], cams[1], cams[2], cams[3], (W, H), scene.VOLRADIUS)
    outc, _, _ = compare(s, grad, camera=camera)
    outcp, _, _ = compare(s, grad, camera=camera, planes=True)
    assert torch.equal(outc, outcp)


def test_bf16_template_retain_graph_second_backward():
    """The second backward through the same graph gets fresh buffers zero-filled by the library (MVP_FLAG_ZERO_GRADS)."""
    s, grad = build_case("head_small")
    s, grad = _cuda_scene(s), grad.cuda()
    tb = s["template"].to(torch.bfloat16)
    _, g32 = render(s, tb.float(), grad)
    keep = {}
    _, gb = render(s, tb, grad, retain=True, keep=keep)
    second = dict(zip(gb, keep["second"]))
    for g in (gb, second):
        for nm in g:
            if nm != "template":
                assert _relerr(g[nm], g32[nm]) <= 1e-5, nm
        assert g["template"].dtype == torch.bfloat16
        emax, el1 = _tgrad_errors(g["template"], g32["template"])
        assert emax <= GATE_MAX and el1 <= GATE_L1, (emax, el1)


def test_bf16_template_four_bench_views():
    """Four views of the benchmark scene: 1024x667, K = 16384 slabs of 8^3."""
    from ava256_b200 import scene
    s = scene.make_scene(4, 1024, 667, 16384, 8, alpha_mu=17.0, alpha_sigma=6.0, device="cuda")
    grad = torch.randn(4, 1024, 667, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    compare(s, grad)


def test_bf16_template_peak_memory():
    """Peak device memory of a forward + backward, template included: bf16 saves at least half the template and its gradient."""
    from ava256_b200 import scene
    s = scene.make_scene(4, 512, 334, 16384, 8, alpha_mu=17.0, alpha_sigma=6.0, device="cuda")
    tpl = s.pop("template")
    grad = torch.randn(4, 512, 334, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))
    peaks = {}
    for dt in (torch.float32, torch.bfloat16, torch.float32, torch.bfloat16):
        gc.collect()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t = tpl.to(dt, copy=True)
        out, gs = render(s, t, grad)
        peaks[dt] = torch.cuda.max_memory_allocated() - base
        del t, out, gs
    saved = 2 * tpl.numel() * 2                                                  # template + gradient, 2 bytes per entry each
    print("peak: fp32 %.1f MB, bf16 %.1f MB, template + gradient saving %.1f MB" % (peaks[torch.float32] / 1e6, peaks[torch.bfloat16] / 1e6, saved / 1e6))
    assert peaks[torch.float32] - peaks[torch.bfloat16] >= saved


def test_bf16_template_80_view_launch_per_view():
    """80 views with their own bf16 payloads: bf16 byte offsets pass 2^31 at view 32 and 2^32 at view 64, scalar indices 2^31
    at view 64.  Views 0, 31, 32, 63, 64 and 79 equal the view rendered alone: images bit for bit, transform gradients within
    1e-5, the template gradient within the gates."""
    from ava256_b200 import lib, scene
    from tests.test_gpu_large_launch import _require_memory
    N, H, W, K, T = 80, 1024, 667, 16384, 8
    slabs = N * K * (T ** 3 * 4 * 2 + (3 + 9 + 3) * 4)                           # bf16 template + fp32 transforms
    need = 2 * slabs + N * H * W * (3 + 3 + 2 + 4 + 4 + 3 + 4) * 4 + lib.workspace_bytes(N, H, W, K, T, T, T) + (2 << 30)
    _require_memory(need, "80-view launch, bf16 per-view payloads")
    s = scene.make_scene(N, H, W, K, T, alpha_mu=17.0, alpha_sigma=6.0, share_primitives=False, device="cuda")
    tpl = s.pop("template")
    tb = torch.empty(tpl.shape, dtype=torch.bfloat16, device="cuda")
    del tpl
    gc.collect()
    torch.cuda.empty_cache()
    for v in range(N):
        tb[v] = scene.make_payload(K, T, seed=1112 + v, alpha_mu=17.0, alpha_sigma=6.0, device="cuda").to(torch.bfloat16)
    assert tb.numel() > 2 ** 31 and tb[32].data_ptr() - tb.data_ptr() >= 2 ** 31 and tb[64].data_ptr() - tb.data_ptr() >= 2 ** 32
    assert not torch.equal(tb[64], tb[0])
    grad = torch.randn(N, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    out, gs = render(s, tb, grad)
    for v in (0, 31, 32, 63, 64, 79):
        sv = {k: (x[v:v + 1].contiguous() if torch.is_tensor(x) else x) for k, x in s.items()}
        out_v, gs_v = render(sv, tb[v:v + 1].contiguous(), grad[v:v + 1].contiguous())
        assert torch.equal(out[v:v + 1], out_v), v
        for nm in gs_v:
            assert bool(torch.isfinite(gs[nm][v].float()).all()), (v, nm)
            if nm != "template":
                assert _relerr(gs[nm][v:v + 1], gs_v[nm]) <= 1e-5, (v, nm)
        emax, el1 = _tgrad_errors(gs["template"][v:v + 1], gs_v["template"])
        assert float(gs_v["template"].float().abs().max()) > 0 and emax <= GATE_MAX and el1 <= GATE_L1, (v, emax, el1)
        if v >= 64:
            a = out[v, ..., 3]
            assert 0.02 < float((a >= 1.0 - 1e-6).float().mean()) < 0.6, v
        del sv, out_v, gs_v


def test_bf16_autocast_round_trip_through_the_overlay():
    """A bf16 conv under torch.autocast produces the template through assembler.py:261's expression; forward and backward run
    through the drop-in `extensions.mvpraymarch.mvpraymarch.mvpraymarch`, and the conv weight gets a finite gradient."""
    from extensions.mvpraymarch.mvpraymarch import mvpraymarch
    s, grad = build_case("head_small")
    s, grad = _cuda_scene(s), grad.cuda()
    N, K, T = s["template"].shape[0], s["template"].shape[1], s["template"].shape[2]
    conv = torch.nn.Conv2d(8, 4 * T, 3, padding=1).cuda()
    x = torch.randn(N * K, 8, T * T, 1, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = conv(x)                                                               # [N*K, 4T, T*T, 1] bf16
        assert y.dtype == torch.bfloat16
        y = y.view(N, K, 4, T, T, T).permute(0, 1, 3, 4, 5, 2)                     # [N,K,TD,TH,TW,4]
        rgb, alpha = y[..., :3], y[..., 3:]
        template = torch.cat([torch.relu(rgb * 25 + 100), torch.relu(alpha)], dim=-1).contiguous()   # assembler.py:261
        assert template.dtype == torch.bfloat16
        primpos = s["primpos"].to(torch.bfloat16).requires_grad_(True)           # transforms arrive as bf16 too
        out = mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], (primpos, s["primrot"], s["primscale"]),
                          template, None, fadescale=8.0, fadeexp=8.0)
    assert out.dtype == torch.float32 and bool(torch.isfinite(out).all())
    (out * grad).sum().backward()
    assert conv.weight.grad is not None and bool(torch.isfinite(conv.weight.grad).all()) and float(conv.weight.grad.abs().max()) > 0
    assert primpos.grad.dtype == torch.bfloat16 and bool(torch.isfinite(primpos.grad.float()).all())


def test_fp16_template_raises():
    from ava256_b200.op import mvpraymarch
    s, _ = build_case("tiny")
    s = _cuda_scene(s)
    with pytest.raises(RuntimeError, match="float32 or bfloat16"):
        mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], (s["primpos"], s["primrot"], s["primscale"]),
                    s["template"].half(), None)
