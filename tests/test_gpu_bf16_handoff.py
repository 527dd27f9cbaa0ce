"""GPU tests of the bfloat16 payload hand-off (`pytest -m gpu`): `assemble_payload(..., dtype=torch.bfloat16)`, bf16
`expand_views` / `sum_views`, bf16 template gradients in `parallel.reduce_primitive_grads` / `GradReducer`, and the one-subject
step that runs in bf16 from the decoder images to their gradients.  The exactness contracts are those of
tests/test_emul_bf16_handoff.py, on the device; the gradient gates are those of the bf16 template gradients
(tests/test_emul_bf16_payload.py)."""
import gc

import pytest
import torch

from oracle.epilogue_ref import assemble_payload_ref
from tests.test_emul_bf16_payload import GATE_L1, GATE_MAX
from tests.test_epilogue import _payload_case
from tests.test_gpu_large_launch import _require_memory

pytestmark = pytest.mark.gpu

# The one-subject step against the same step with the fp32 hand-off.  grad_tex stays within the bf16 template-gradient gates
# (measured on an H100 80GB HBM3: max 0.0097 / sum 0.0040 at 4 views, 0.0084 / 0.0044 at 80).  grad_opacity does not
# (0.21 / 0.0122 at 4 views, 0.095-0.096 / 0.032 at 80; the max varies with the order of the atomics): two roundings stack on it.  The template itself is bf16, so the fp32 step
# renders different alpha values (2^-9 relative) and rays saturate at other samples, and each view's alpha gradient is
# accumulated in bf16 by the render backward (tens of reductions per voxel per view, mixed signs) before the 80 views are
# summed in fp32.  The images themselves are bit-identical to the fp32 op on the widened bf16 template.  These gates record
# the measured values with headroom; they are not the bf16 template-gradient gates.
GATE_STEP_OPACITY = (0.3, 0.05)
# The autocast round trip's conv weight gradients sum the image gradients through every texel (measured max 0.0061 / sum 0.0065
# for the tex conv, 0.0146 / 0.0149 for the opacity conv, whose gradient carries the alpha gradient above).
GATE_AUTOCAST_CONV = (0.02, 0.03)

H, W, K, T = 1024, 667, 16384, 8
HB = WB = 128                                                 # K = 128 x 128 slabs: tex [1, 24, 1024, 1024]


def _bits(t):
    return t.contiguous().view(torch.int16)


def _errors(g, ref):
    d = (g.double() - ref.double()).abs()
    return float(d.max() / ref.double().abs().max()), float(d.sum() / ref.double().abs().sum())


def _eager_bf16(tex, opacity, gb, B):
    t, o = tex.detach().clone().requires_grad_(True), opacity.detach().clone().requires_grad_(True)
    tp = assemble_payload_ref(t, o, B).to(torch.bfloat16)
    tp.backward(gb)
    return tp.detach(), t.grad, o.grad


@pytest.mark.parametrize("N,hb,wb,B", [(2, 2, 3, 8), (1, 3, 2, 4), (1, 4, 2, 3), (1, 1, 1, 1), (1, 2, 2, 16), (2, 16, 16, 8),
                                       (1, HB, WB, 8)])
def test_gpu_bf16_payload_matches_eager_torch(N, hb, wb, B):
    """Every variant (V = 4 with B = 8 / generic B, scalar), the last at the subject size of the benchmark (K = 16384)."""
    from ava256_b200.payload import assemble_payload
    tex, opacity, gt = _payload_case(N, hb, wb, B, seed=B + 11, device="cuda")
    gb = gt.to(torch.bfloat16)
    ref, gtex, gop = _eager_bf16(tex, opacity, gb, B)
    t, o = tex.clone().requires_grad_(True), opacity.clone().requires_grad_(True)
    tp = assemble_payload(t, o, boxsize=B, dtype=torch.bfloat16)
    assert tp.dtype == torch.bfloat16 and tp.shape == (N, hb * wb, B, B, B, 4) and tp.is_contiguous()
    assert torch.equal(_bits(tp), _bits(ref))
    tp.backward(gb)
    assert t.grad.dtype == torch.float32 and torch.equal(t.grad, gtex) and torch.equal(o.grad, gop)


def test_gpu_bf16_payload_unaligned_views():
    """Images and gradient that start off a 16-byte boundary: the scalar variant, same bits."""
    from ava256_b200.payload import assemble_payload
    N, hb, wb, B = 1, 3, 5, 8
    tex, opacity, gt = _payload_case(N, hb, wb, B, seed=5, device="cuda")
    gb = gt.to(torch.bfloat16)
    ref, gtex, gop = _eager_bf16(tex, opacity, gb, B)
    tbuf = torch.empty(tex.numel() + 1, device="cuda")
    obuf = torch.empty(opacity.numel() + 1, device="cuda")
    tu, ou = tbuf[1:].view(tex.shape), obuf[1:].view(opacity.shape)
    tu.copy_(tex)
    ou.copy_(opacity)
    assert tu.data_ptr() % 16 and ou.data_ptr() % 16
    tu.requires_grad_(True)
    ou.requires_grad_(True)
    tp = assemble_payload(tu, ou, boxsize=B, dtype=torch.bfloat16)
    assert torch.equal(_bits(tp), _bits(ref))
    gbuf = torch.empty(gb.numel() + 4, dtype=torch.bfloat16, device="cuda")
    gu = gbuf[4:].view(gb.shape)                                               # 8 bytes past a 16-byte boundary
    gu.copy_(gb)
    assert gu.data_ptr() % 16 == 8
    tp.backward(gu)
    assert torch.equal(tu.grad, gtex) and torch.equal(ou.grad, gop)


@pytest.mark.parametrize("shape,n", [((5, 4), 4), ((16, 8, 8, 8, 4), 6), ((1, 1, 2), 1), ((7, 6), 3)])
def test_gpu_expand_views_bf16(shape, n):
    """A bf16 tensor through the word copy: bit-identical to expand().contiguous(); its adjoint is the fp32 view sum rounded
    once to bf16.  A view that starts mid-word is copied first; an odd element count raises."""
    from ava256_b200.payload import expand_views, sum_views
    x = torch.randn(*shape, device="cuda").to(torch.bfloat16).requires_grad_(True)
    y = expand_views(x, n)
    assert y.dtype == torch.bfloat16 and torch.equal(_bits(y), _bits(x.detach()[None].expand(n, *shape)))
    g = torch.randn(n, *shape, device="cuda").to(torch.bfloat16)
    y.backward(g)
    assert x.grad.dtype == torch.bfloat16 and torch.equal(_bits(x.grad), _bits(sum_views(g.float()).to(torch.bfloat16)))
    buf = torch.randn(2 * 33 + 1, device="cuda").to(torch.bfloat16)
    flat = buf[1:]                                                             # 2-byte aligned only
    assert torch.equal(_bits(expand_views(flat, 3)), _bits(flat[None].expand(3, -1)))
    with pytest.raises(RuntimeError, match="even"):
        expand_views(buf[:7], 2)


@pytest.mark.parametrize("shape,n", [((5, 8), 4), ((64, 8, 8, 8, 4), 19), ((1024, 9), 10), ((7,), 1), ((300, 8), 80), ((3, 5), 9)])
def test_gpu_sum_views_bf16(shape, n):
    """bf16 views summed in fp32 in view order: into fp32 bit-identical to sum_views(x.float()), into bf16 that rounded once;
    also into a slice of a flat fp32 buffer (4-byte aligned: the scalar path) and from a source off a 16-byte boundary."""
    from ava256_b200.payload import sum_views
    x = (torch.randn(n, *shape, device="cuda") * 4.0).to(torch.bfloat16)
    ref = sum_views(x.float())
    assert torch.equal(sum_views(x, torch.empty(shape, device="cuda")), ref)
    out = sum_views(x)
    assert out.dtype == torch.bfloat16 and torch.equal(_bits(out), _bits(ref.to(torch.bfloat16)))
    cnt = ref.numel()
    flat = torch.full((cnt + 9,), 7.0, device="cuda")
    sum_views(x, flat[5:5 + cnt])
    assert torch.equal(flat[5:5 + cnt].view(shape), ref) and bool((flat[:5] == 7.0).all()) and bool((flat[5 + cnt:] == 7.0).all())
    xb = torch.empty(x.numel() + 1, dtype=torch.bfloat16, device="cuda")[1:].view(x.shape)
    xb.copy_(x)
    assert torch.equal(sum_views(xb, torch.empty(shape, device="cuda")), ref)


def test_gpu_sum_views_bf16_80_template_sized_views():
    """80 template-sized bf16 gradients (2.68e9 values, 5.4 GB): byte offsets past 2^32.  The reference is sum_views of the
    widened source, taken in column blocks (the sum is per element, so blocks give the same bits)."""
    from ava256_b200.payload import sum_views
    N, count = 80, K * T ** 3 * 4
    block = count // 16
    need = N * count * 2 + count * (4 + 2 + 4) + N * block * 6 + (1 << 30)
    _require_memory(need, "bf16 view sum of 80 template-sized views")
    x = torch.empty(N, count, dtype=torch.bfloat16, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(80)
    for v in range(N):
        x[v] = torch.randn(count, device="cuda", generator=gen).to(torch.bfloat16)
    assert x.numel() > 2 ** 31 and x[64].data_ptr() - x.data_ptr() >= 2 ** 32
    out32 = sum_views(x, torch.empty(count, device="cuda"))
    out16 = sum_views(x)
    for b in range(0, count, block):
        r = sum_views(x[:, b:b + block].float())
        assert torch.equal(out32[b:b + block], r), b
        assert torch.equal(_bits(out16[b:b + block]), _bits(r.to(torch.bfloat16))), b
        del r


def test_gpu_grad_reducer_bf16_template_gradient():
    """reduce_primitive_grads and GradReducer (world size 1) on a bf16 template gradient: the flat buffer is fp32 and equals the
    reduction of the fp32 widening bit for bit."""
    from ava256_b200.parallel import GradReducer, reduce_primitive_grads
    nv, k = 80, 2048
    gen = torch.Generator(device="cuda").manual_seed(9)
    gt = torch.randn(nv, k, T, T, T, 4, device="cuda", generator=gen).to(torch.bfloat16)
    rest = [torch.randn(nv, k, 3, device="cuda", generator=gen), torch.randn(nv, k, 3, 3, device="cuda", generator=gen),
            torch.randn(nv, k, 3, device="cuda", generator=gen)]
    flat_b, views_b = reduce_primitive_grads(gt, *rest)
    flat_f, _ = reduce_primitive_grads(gt.float(), *rest)
    assert flat_b.dtype == torch.float32 and views_b[0].dtype == torch.float32 and torch.equal(flat_b, flat_f)
    red = GradReducer(k, T, T, T, "cuda")
    a = red.reduce(gt, *rest).clone()
    b = red.reduce(gt.float(), *rest)
    red.finish()
    assert torch.equal(a, b) and torch.equal(a, flat_f)


def _images_from_template(tpl, hb, wb, rgb_scale=25.0, rgb_bias=100.0):
    """Decoder images whose payload is (up to rounding) `tpl` [K,B,B,B,4]: the inverse of the hand-off's layout and scale."""
    B = tpl.shape[1]
    t = tpl.view(hb, wb, B, B, B, 4)                                            # i, j, d, y, x, c
    tex = ((t[..., :3] - rgb_bias) / rgb_scale).permute(2, 5, 0, 3, 1, 4).reshape(1, 3 * B, hb * B, wb * B)
    opa = t[..., 3].permute(2, 0, 3, 1, 4).reshape(1, B, hb * B, wb * B)
    return tex.contiguous(), opa.contiguous()


def _one_subject_step(s, tex, opa, grad, dtype, nv):
    """assemble -> expand to nv views -> op forward + backward -> expand adjoint -> assemble backward."""
    from ava256_b200.op import mvpraymarch
    from ava256_b200.payload import assemble_payload, expand_views
    t, o = tex.clone().requires_grad_(True), opa.clone().requires_grad_(True)
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    tp = assemble_payload(t, o, boxsize=T, dtype=dtype)
    tpv = expand_views(tp[0], nv)
    out = mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], (s["primpos"], s["primrot"], s["primscale"]), tpv,
                      None, fadescale=8.0, fadeexp=8.0)
    out.backward(grad)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    return out.detach(), tp.detach(), t.grad, o.grad, peak


def _pipeline_case(nv, share):
    from ava256_b200 import scene
    s = scene.make_scene(nv, H, W, K, T, seed=1112, alpha_mu=17.0, alpha_sigma=6.0, device="cuda", share_primitives=share)
    tpl = s.pop("template")[0].clone()
    gc.collect()
    torch.cuda.empty_cache()
    tex, opa = _images_from_template(tpl, HB, WB)
    del tpl
    grad = torch.randn(nv, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1112))
    return s, tex, opa, grad


def _check_pipeline(nv):
    from ava256_b200.op import mvpraymarch
    from ava256_b200.payload import expand_views
    s, tex, opa, grad = _pipeline_case(nv, True)
    out32, tp32, gtex32, gopa32, peak32 = _one_subject_step(s, tex, opa, grad, torch.float32, nv)
    del out32
    outb, tpb, gtexb, gopab, peakb = _one_subject_step(s, tex, opa, grad, torch.bfloat16, nv)
    assert torch.equal(_bits(tpb), _bits(tp32.to(torch.bfloat16)))
    del tp32
    with torch.no_grad():                                                     # the fp32 op on the widened bf16 template
        ref = mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], (s["primpos"], s["primrot"], s["primscale"]),
                          expand_views(tpb[0].float(), nv), None, fadescale=8.0, fadeexp=8.0)
    assert torch.equal(outb, ref)
    del ref
    assert gtexb.dtype == torch.float32 and bool(torch.isfinite(gtexb).all()) and bool(torch.isfinite(gopab).all())
    et, ot = _errors(gtexb, gtex32), _errors(gopab, gopa32)
    # at the peak (the backward) the expanded template and its per-view gradient are both live: 2 bytes less per value each
    saved = nv * K * T ** 3 * 4 * 2 * 2
    print("%d views: grad_tex max %.3g l1 %.3g, grad_opacity max %.3g l1 %.3g; peak fp32 %.2f GB bf16 %.2f GB (>= %.2f GB saved)"
          % (nv, et[0], et[1], ot[0], ot[1], peak32 / 1e9, peakb / 1e9, saved / 1e9))
    assert et[0] <= GATE_MAX and et[1] <= GATE_L1, et
    assert ot[0] <= GATE_STEP_OPACITY[0] and ot[1] <= GATE_STEP_OPACITY[1], ot
    assert peak32 - peakb >= saved


def test_gpu_bf16_one_subject_step_four_bench_views():
    _check_pipeline(4)


def test_gpu_bf16_one_subject_step_80_view_launch():
    from ava256_b200 import lib
    nv = 80
    tplb = nv * K * T ** 3 * 4 * 4                                             # fp32 expanded template
    need = 2 * tplb + nv * H * W * (3 + 3 + 2 + 4 + 4 + 3 + 4) * 4 + lib.workspace_bytes(nv, H, W, K, T, T, T) + (4 << 30)
    _require_memory(need, "one-subject step, 80 views")
    _check_pipeline(nv)


def test_gpu_bf16_autocast_decoder_tail_round_trip():
    """A decoder tail built like the reference's (conv, then `+ self.bias[None]` with an fp32 parameter) gives fp32 images under
    autocast, so the template is fp32 unless the hand-off writes bf16.  With dtype=bfloat16 the step runs through `Raymarcher`
    and back; the conv weight gradients are finite and agree with the fp32 hand-off (gates above)."""
    from ava256_b200.payload import assemble_payload
    from ava256_b200.raymarcher import Raymarcher
    from tests.helpers import build_case
    s, grad = build_case("head_small")
    s = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in s.items()}
    grad = grad.cuda()
    N, Kc, B = s["template"].shape[0], s["template"].shape[1], s["template"].shape[2]
    hb = wb = int(round(Kc ** 0.5))
    assert hb * wb == Kc
    torch.manual_seed(4)
    conv_t = torch.nn.Conv2d(8, 3 * B, 3, padding=1).cuda()
    conv_o = torch.nn.Conv2d(8, B, 3, padding=1).cuda()
    bias_t = torch.nn.Parameter(torch.zeros(3 * B, hb * B, wb * B, device="cuda"))
    bias_o = torch.nn.Parameter(torch.full((B, hb * B, wb * B), 0.3, device="cuda"))
    x = torch.randn(N, 8, hb * B, wb * B, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    rm = Raymarcher(1.0, dt=s["stepsize"])
    g_img = grad.permute(0, 3, 1, 2)
    res = {}
    for dt in (torch.float32, torch.bfloat16):
        for p in (conv_t.weight, conv_o.weight):
            p.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = conv_t(x)
            assert y.dtype == torch.bfloat16
            tex = y + bias_t[None]                                                 # models/decoders/rgb.py:125
            opa = torch.exp((conv_o(x) + bias_o[None]) * 0.1)                      # models/decoders/geometry.py:165
            assert tex.dtype == torch.float32 and opa.dtype == torch.float32
            tp = assemble_payload(tex, opa, boxsize=B, dtype=dt)
            assert tp.dtype == dt
            decout = dict(template=tp, primpos=s["primpos"], primrot=s["primrot"], primscale=s["primscale"])
            rgb, alpha, _, _ = rm(s["raypos"], s["raydir"], s["tminmax"], decout, dict(fadescale=8.0, fadeexp=8.0))
        loss = (rgb * g_img[:, :3]).sum() + (alpha * g_img[:, 3:]).sum()
        loss.backward()
        res[dt] = (conv_t.weight.grad.clone(), conv_o.weight.grad.clone())
    for a, b in zip(res[torch.bfloat16], res[torch.float32]):
        assert bool(torch.isfinite(a).all()) and float(a.abs().max()) > 0
        e = _errors(a, b)
        print("autocast conv weight grad: max %.3g l1 %.3g" % e)
        assert e[0] <= GATE_AUTOCAST_CONV[0] and e[1] <= GATE_AUTOCAST_CONV[1], e
