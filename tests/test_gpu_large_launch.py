"""GPU tests of the launch bench.py times (`pytest -m gpu`): forward and backward of 80 views of 1024x667 with K = 16384 slabs
of 8^3 voxels in ONE launch, followed by the sum of the 80 per-view gradients (mvp_sum_views, parallel.GradReducer).

At this size the per-slab tensors outgrow 32-bit offsets: one view's template holds 16384 * 8^3 * 4 = 2^25 floats, so view v
starts at float 2^25 * v.  Byte offsets pass 2^31 at view 16 and 2^32 at view 32; a signed int element index would pass 2^31
at view 64.  The template, its gradient and the source of the view sum hold 2.68e9 floats (10 GiB) each.  Each test below
asserts that its tensors cross 2^31 elements, so that the case cannot shrink below the crossings without the test saying so.

An offset that wrapped would make views 64-79 read or write the slots of views 0-15.  The benchmark scene cannot show that:
it materialises one subject's payload for every view.  So the first test gives every view its own payload and primitives and
compares every view of the 80-view launch with the same view rendered alone (a 1-view launch, offsets near zero); the second
ties the unmodified benchmark launch to the reference extension's stored outputs for views 0, 1, 78 and 79.

Each test computes the device memory it needs from its shapes (peak about 30 GB for the render tests) and skips, with both
numbers, when the device does not have that much free."""
import gc

import pytest
import torch

from tests.helpers import abi_raymarch, scale_case
from tests.test_gpu_scale_parity import _trelerr, assert_parity_with_golden

pytestmark = pytest.mark.gpu

N, H, W, K, T = 80, 1024, 667, 16384, 8            # bench.py VIEWS, H, W, K, T
ALPHA_MU, ALPHA_SIGMA = 17.0, 6.0
NAMES = ("primpos", "primrot", "primscale", "template")
GOLDEN_VIEWS = (("c3_view0", 0), ("c3_view78", 78))  # tests/golden/scale_<name>.npz: 2 views starting at that view
SLACK = 2 << 30                                      # per-view temporaries, the camera-ray launch's images


def _require_memory(need, what):
    """Skips the test when the device has less than `need` bytes free (after returning the allocator's cached blocks)."""
    gc.collect()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    print("%s: %s, %.1f GB free of %.1f GB, %.1f GB needed" % (what, torch.cuda.get_device_name(), free / 1e9, total / 1e9, need / 1e9))
    if need > free:
        pytest.skip("%s needs %.1f GB of device memory; %.1f GB are free" % (what, need / 1e9, free / 1e9))


def _render_bytes():
    """Device memory of an 80-view forward + backward: inputs and gradients of the slabs, rays, image-sized buffers, workspace."""
    from ava256_b200 import lib
    slabs = N * K * (T ** 3 * 4 + 3 + 9 + 3) * 4        # template + primpos, primrot, primscale
    rays = N * H * W * (3 + 3 + 2) * 4
    images = N * H * W * (4 + 4 + 3 + 4) * 4            # grad_rayrgba, rayrgba, raysat, rayaux
    return 2 * slabs + rays + images + lib.workspace_bytes(N, H, W, K, T, T, T) + SLACK


def _sequential_sum(x):
    """x[0] + x[1] + ... in view order, one view at a time."""
    acc = torch.zeros_like(x[0])
    for v in range(x.shape[0]):
        acc += x[v]
    return acc


def test_every_view_of_80_view_launch_equals_the_view_alone():
    """80 views with their own payload (seed 1112 + v) and primitives (jittered per view), rays from mvp_compute_raydirs.  The
    forward clears the NaN-filled gradient buffers (all 10 GiB of the template's) and the backward runs without
    MVP_FLAG_ZERO_GRADS, as the op does.  Every view v: images, saturation records and per-ray records bit-identical to a 1-view
    launch of view v, its four gradients within 1e-5 (fp32 atomic order) and finite.  Then the same 80 views with the rays
    generated in the kernels (op.mvpraymarch_camera): the same image bits."""
    from ava256_b200 import scene
    from ava256_b200.op import mvpraymarch_camera
    from extensions.utils.utils import compute_raydirs
    _require_memory(_render_bytes(), "80-view launch, per-view payloads")
    s = scene.make_scene(N, H, W, K, T, alpha_mu=ALPHA_MU, alpha_sigma=ALPHA_SIGMA, share_primitives=False, device="cuda")
    for k in ("raypos", "raydir", "tminmax"):
        del s[k]
    cams = [c.cuda() for c in scene.make_cameras(N, H, W)]
    s["raypos"], s["raydir"], s["tminmax"] = compute_raydirs(cams[0], cams[1], cams[2], cams[3], (W, H), scene.VOLRADIUS)
    for v in range(N):
        s["template"][v] = scene.make_payload(K, T, seed=1112 + v, alpha_mu=ALPHA_MU, alpha_sigma=ALPHA_SIGMA, device="cuda")
    assert s["template"].numel() > 2 ** 31
    assert not torch.equal(s["template"][64], s["template"][0]) and not torch.equal(s["primpos"][64], s["primpos"][0])
    grad = torch.randn(N, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))

    keep = {}
    out, rsat, grads, _ = abi_raymarch(s, grad, keep=keep, clear_in_forward=True)
    raux = keep.pop("rayaux")
    keep.clear()
    for v in range(N):
        sv = {k: (x[v:v + 1].contiguous() if torch.is_tensor(x) else x) for k, x in s.items()}
        kv = {}
        out_v, rsat_v, grads_v, _ = abi_raymarch(sv, grad[v:v + 1].contiguous(), keep=kv, clear_in_forward=True)
        assert torch.equal(out[v:v + 1], out_v), v
        assert torch.equal(rsat[v:v + 1], rsat_v), v
        assert torch.equal(raux[v:v + 1], kv["rayaux"]), v
        for nm, g, g_v in zip(NAMES, grads, grads_v):
            assert bool(torch.isfinite(g[v]).all()), (v, nm)
            assert float(g_v.abs().max()) > 0, (v, nm)
            assert _trelerr(g[v:v + 1], g_v) <= 1e-5, (v, nm)
        if v >= 64:                   # the views whose slabs start past float 2^31 render the subject
            a = out[v, ..., 3]
            satur = float((a >= 1.0 - 1e-6).float().mean())
            assert 0.02 < satur < 0.6 and satur < float((a > 0).float().mean()), (v, satur)
        del sv, kv, out_v, rsat_v, grads_v

    del grads, rsat, raux, grad, s["raypos"], s["raydir"], s["tminmax"]
    gc.collect()
    torch.cuda.empty_cache()
    lv = [s[n].detach().requires_grad_(True) for n in NAMES]
    out_c = mvpraymarch_camera(cams[0], cams[1], cams[2], cams[3], (W, H), scene.VOLRADIUS, s["stepsize"], (lv[0], lv[1], lv[2]),
                               lv[3], None)
    torch.cuda.synchronize()
    assert torch.equal(out_c.detach(), out)


def test_bench_launch_vs_reference_extension():
    """bench.py's tensors (one subject's payload materialised for all 80 views), forward + backward through the public op in one
    launch.  Views 0, 1 and 78, 79 of this scene are byte-identical to the scale cases c3_view0 / c3_view78 (the dome lattice has
    80 points either way, primitives and payload come from the same seeds), and so is their image gradient: their images and
    per-view gradients are checked against the reference extension's stored outputs for those cases."""
    import bench
    from ava256_b200 import scene
    from ava256_b200.op import mvpraymarch
    assert (bench.VIEWS, bench.H, bench.W, bench.K, bench.T, bench.ALPHA_MU, bench.ALPHA_SIGMA) == (N, H, W, K, T, ALPHA_MU, ALPHA_SIGMA)
    _require_memory(_render_bytes(), "80-view benchmark launch")
    s = scene.make_scene(N, H, W, K, T, view_ids=range(N), alpha_mu=ALPHA_MU, alpha_sigma=ALPHA_SIGMA, device="cuda")
    assert s["template"].numel() > 2 ** 31
    grad = torch.randn(N, H, W, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1112))
    for name, off in GOLDEN_VIEWS:
        sc, g = scale_case(name)
        for k, x in sc.items():
            assert (torch.equal(s[k][off:off + 2], x) if torch.is_tensor(x) else s[k] == x), (name, k)
        grad[off:off + 2] = g
        del sc, g

    leaves = [s[n].requires_grad_(True) for n in NAMES]
    out = mvpraymarch(s["raypos"], s["raydir"], s["stepsize"], s["tminmax"], (leaves[0], leaves[1], leaves[2]), leaves[3], None)
    out.backward(grad)
    torch.cuda.synchronize()
    for name, off in GOLDEN_VIEWS:
        assert_parity_with_golden(out.detach()[off:off + 2], [x.grad[off:off + 2] for x in leaves], name)


def test_sum_views_and_grad_reducer_past_2_31_elements():
    """mvp_sum_views over 80 distinct views of a template gradient (2.68e9 floats): the sum added in view order, bit for bit.
    parallel.GradReducer, as bench.py calls it (world size 1, no process group): each of the four parts of its flat buffer is
    the sequential sum of that gradient."""
    from ava256_b200 import parallel
    from ava256_b200.payload import sum_views
    count = K * T ** 3 * 4
    prims = N * K * 15
    _require_memory((N * count + prims + 4 * (count + K * 15)) * 4 + (64 << 20), "80-view gradient sum")
    gen = torch.Generator(device="cuda").manual_seed(31)
    g_tpl = torch.empty(N, K, T, T, T, 4, device="cuda")
    for v in range(N):
        g_tpl[v].normal_(generator=gen)
    assert g_tpl.numel() > 2 ** 31
    g_prims = [torch.randn(N, K, *tail, device="cuda", generator=gen) for tail in ((3,), (3, 3), (3,))]
    parts = [g_tpl] + g_prims
    refs = [_sequential_sum(p) for p in parts]
    assert torch.equal(sum_views(g_tpl), refs[0])
    red = parallel.GradReducer(K, T, T, T, "cuda")
    flat = red.reduce(*parts)
    red.finish()
    assert flat.numel() == sum(r.numel() for r in refs)
    for nm, got, ref in zip(("template", "primpos", "primrot", "primscale"), red.views(flat, K, T, T, T), refs):
        assert torch.equal(got, ref), nm


@pytest.mark.parametrize("count", [K * T ** 3 * 4, K * T ** 3 * 4 - 1], ids=["float4", "scalar"])
def test_expand_views_past_2_31_elements(count):
    """mvp_expand_views of one view's template-sized tensor to 80 views (2.68e9 floats): every view slice equals the source.
    A count that is a multiple of 4 takes the 16-byte path; 2^25 - 1 takes the scalar path, whose element index passes 2^31."""
    from ava256_b200.payload import expand_views
    _require_memory((N + 1) * count * 4 + (64 << 20), "80-view expand")
    x = torch.randn(count, device="cuda", generator=torch.Generator(device="cuda").manual_seed(count))
    y = expand_views(x, N)
    assert y.shape == (N, count) and y.numel() > 2 ** 31
    for v in range(N):
        assert torch.equal(y[v], x), v
