"""The render kernels decide before they march which lattice steps of a ray can sample a slab: each step interval is the exact
slab interval grown by a bound on how far the marched position (x = fma(d, dt, x), the reference's order) can drift from
o + t d.  Within one binade every step of the march can round the same way, so the drift grows linearly and reaches that bound.
These scenes make it do so where the positions leave the unit cube: dt is chosen so that d_i dt leaves just over (leading drift)
or just under (lagging drift) half an ulp of the binade, every step rounds the same way, and a thin slab's face is placed
between the exact and the marched position of one step.  A step interval that is too narrow then drops a sample the reference
evaluates, which the sample counts show exactly.  Emulated product kernels (tests/emul) against the fp32 oracle."""
import ctypes

import numpy as np
import pytest

from tests.helpers import relerr

F32 = np.float32
FWD_TOL, BWD_TOL = 1e-5, 1e-4          # the suite's forward and gradient gates (emulated kernels vs the fp32 oracle)
HALF_B = 0.02                           # half-thickness of the sampled slab B: 40 samples at dt ~ 1e-3
H, W = 4, 8                             # one 8x4 tile, every ray the same
OWARP = (8, 4)                          # the oracle's block: one warp on the tile (a larger one also marches clamped copies)


def fma32(a, b, c):
    """fp32 fma: the product of two fp32 values is exact in fp64; the sum is rounded once more, which can only differ from one
    rounding at an fp32 tie, and no value of these marches is near one (every step lies ~0.005 ulp off a tie)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def pick_dt(dcomp, ulp, frac, target=1e-3):
    """fp32 step near `target` whose exact product with the direction component `dcomp` is (n + frac) ulps of the binade whose
    ulp is `ulp`: with frac just above 0.5 every step of a march in that binade rounds up, just below it rounds down."""
    n = np.floor(float(dcomp) * target / ulp)
    dt = F32((n + frac) * ulp / float(dcomp))
    got = (float(dcomp) * float(dt) / ulp) % 1.0
    assert abs(got - frac) < 2e-3, (got, frac)
    return float(dt)


def old_bound(nsteps):
    """The drift bound the kernels used when they assumed |x| < 2 (world units)."""
    return float(F32(1.7320508) * F32(nsteps) * F32(1.1920929e-7) + F32(1.9073486e-6))


def march_positions(o, d, dt, tmin, steps):
    """The reference's march from tmin (oracle/mvp_oracle.c march_init with the march starting at tmin, then one
    x = fma(d, dt, x) per step) in fp32: positions of steps 0 .. steps."""
    x = fma32(d, F32(tmin), o)
    out = [x]
    for _ in range(steps):
        x = fma32(d, F32(dt), x)
        out.append(x)
    return np.array(out)


def rot_to(d):
    """Symmetric rotation (180 degrees about the bisector of e_z and d) that maps e_z to d: the slab's local z axis is the ray."""
    u = np.array([0.0, 0.0, 1.0]) + d / np.linalg.norm(d)
    u /= np.linalg.norm(u)
    return (2.0 * np.outer(u, u) - np.eye(3)).astype(F32)


DIRS = {"axis": np.array([1.0, 0.0, 0.0]), "diag": np.ones(3) / np.sqrt(3.0)}


def drift_scene(lo, direction, drift, steps=None, tmin=0.0, origin=None, dt_target=1e-3, shift=0.0):
    """One tile of identical rays marching through the binade [lo, 2 lo) of every moving coordinate:
      A  empty slab around the ray's start, so that the march starts at tmin (step 0);
      B  thin slab (half-thickness HALF_B, rgb 0.2 .. 1, alpha 4 .. 10, no fade) whose entry face (leading drift) or exit face (lagging
         drift) lies between the exact and the marched position of step `steps`, beyond the old bound when the drift
         exceeds it (then moved by `shift` along the ray);
      C  empty slab behind B, so that the reference's end of march (t < rt1 + 1e-5) lies past B's exit.
    `steps` defaults to the least count at which the drift passes the old bound; `origin` replaces the ray origin 1.05 lo.
    Returns (oracle args, kwargs, info)."""
    d64 = DIRS[direction]
    d = d64.astype(F32)
    ulp = lo * 2.0 ** -23
    dt = pick_dt(d[0], ulp, 0.505 if drift == "lead" else 0.495, dt_target)
    o = np.full(3, 1.05 * lo, F32) if origin is None else np.asarray(origin, F32)
    dn = d.astype(np.float64) / np.linalg.norm(d.astype(np.float64))
    if steps is None:
        # the least step count (of 200 * 2^i) at which the drift passes the old bound by 64 ulps of the binade, as long as the
        # whole scene (0.15 past the step) stays in the binade; 200 when it never does
        steps = 200
        while (2 * steps * dt + 0.15) * float(d[0]) < 0.9 * lo:
            x = march_positions(o, d, dt, tmin, steps)[-1]
            exact = o.astype(np.float64) + (tmin + steps * dt) * d.astype(np.float64)
            if abs(float((x - exact) @ dn)) > old_bound((steps * dt + 0.2) / dt + 8.0) + 64 * ulp:
                break
            steps *= 2
    x = march_positions(o, d, dt, tmin, steps)[-1].astype(np.float64)
    exact = o.astype(np.float64) + (tmin + steps * dt) * d.astype(np.float64)
    tE = float((exact - o) @ dn)        # along-ray parameter of the exact and of the marched position
    tM = float((x - o) @ dn)
    tmax = tE + 0.2
    ob = old_bound((tmax - tmin) / dt + 8.0)
    gap = abs(tM - tE)
    # the face: past the old bound when the drift leaves room, else half way; always inside the drift
    off = ob + 0.5 * (gap - ob) if gap > ob else 0.5 * gap
    tF = tE + np.sign(tM - tE) * off + shift
    tB = tF + HALF_B if drift == "lead" else tF - HALF_B
    centres = [tmin, tB, tB + 0.06 if drift == "lead" else tF + 0.04]
    halves = [0.01, HALF_B, 0.01]
    R = rot_to(d64)
    primpos = np.stack([(o + t * dn).astype(F32) for t in centres])[None]
    primrot = np.stack([R] * 3)[None]
    primscale = np.array([[[4.0, 4.0, 1.0 / h] for h in halves]], F32)
    tpl = np.zeros((1, 3, 2, 2, 2, 4), F32)
    rng = np.random.default_rng(3)      # B's payload varies over its voxels, so that moving B changes the image
    tpl[0, 1, ..., :3], tpl[0, 1, ..., 3] = rng.uniform(0.2, 1.0, (2, 2, 2, 3)), rng.uniform(4.0, 10.0, (2, 2, 2))
    tpl = (tpl.view(np.uint32) & 0xFFFF0000).view(F32)           # values exact in bf16
    raypos = np.broadcast_to(o, (1, H, W, 3)).copy()
    raydir = np.broadcast_to(d, (1, H, W, 3)).copy()
    tminmax = np.broadcast_to(np.array([tmin, tmax], F32), (1, H, W, 2)).copy()
    info = dict(steps=steps, drift=tM - tE, old_bound=ob, beyond=gap > ob, face_offset=off)
    return [raypos, raydir, dt, tminmax, primpos, primrot, primscale, tpl], dict(fadescale=0.0, fadeexp=8.0), info


def pad_slabs(a, n):
    """Appends n empty copies of slab A (the one around the march's start): every tile's list then holds n + 3 entries."""
    a = list(a)
    for i in (4, 5, 6, 7):
        a[i] = np.concatenate([a[i], np.repeat(a[i][:, :1], n, axis=1)], axis=1)
    return a


@pytest.fixture()
def kernels():
    from tests.emul import kernels as k
    k.use_variant(("MVP_EMUL_STATS",))
    L = k.load()
    stats = (ctypes.c_longlong * 8)()
    L.mvp_emul_fwd_stats(stats)
    L.mvp_emul_bwd_stats(stats)        # reset both
    yield k
    k.set_lane_order("forward")
    k.use_variant(())


def counters(k):
    """(samples the forward queued, valid lane steps of the backward) since the last call."""
    L = k.load()
    f, b = (ctypes.c_longlong * 8)(), (ctypes.c_longlong * 8)()
    L.mvp_emul_fwd_stats(f)
    L.mvp_emul_bwd_stats(b)
    return f[3], b[4]


def grad_of(a):
    return np.random.default_rng(5).standard_normal(a[0].shape[:3] + (4,)).astype(F32)


def check(k, a, kw, ref_args=None, names=("primpos", "primrot", "primscale", "template"), **opts):
    """Emulated forward + backward of scene (a, kw) against the fp32 oracle on ref_args (default a): images and raysat at the
    forward gate, the gradients `names` at the gradient gate, and the number of samples the forward and the backward evaluate
    equal to the oracle's.  Returns the oracle's gradients and raysat."""
    from oracle import oracle
    ra = a if ref_args is None else ref_args
    grad = grad_of(a)
    out, raysat, grads = k.forward_backward(*a, grad_rayrgba=grad, **kw, **opts)
    nf, nb = counters(k)
    ref, rsat, st = oracle.forward(*ra, **kw, blocksize=OWARP, return_stats=True)
    assert st["capped_warps"] == 0 and (ref[..., 3] < 0.999).all(), "the scene must stay unsaturated"
    assert (nf, nb) == (st["samples"], st["samples"]), ("samples: forward, backward, oracle", nf, nb, st["samples"])
    assert relerr(out, ref) <= FWD_TOL and relerr(raysat, rsat) <= FWD_TOL
    gref = oracle.backward(*ra, grad, rsat, **kw, blocksize=OWARP)
    for nm, g, r in zip(("primpos", "primrot", "primscale", "template"), grads, gref):
        if nm in names:
            assert np.isfinite(g).all() and relerr(g, r) <= BWD_TOL, nm
    return gref, rsat


# lower end of the binade the march runs in; "cube" is the in-cube control of each scene: the same construction in [0.5, 1)
BINADES = {"cube": 0.5, "2": 2.0, "4": 4.0, "8": 8.0, "64": 64.0}


@pytest.mark.parametrize("drift", ["lead", "lag"])
@pytest.mark.parametrize("direction", list(DIRS))
@pytest.mark.parametrize("binade", list(BINADES))
def test_drift_vs_oracle(kernels, binade, direction, drift):
    """Leading drift caught at B's entry face, lagging drift at its exit face.  From [4, 8) on the drift passes the bound the
    kernels had when they assumed |x| < 2; in [2, 4) half an ulp is still within it."""
    a, kw, info = drift_scene(BINADES[binade], direction, drift)
    if BINADES[binade] >= 4:
        assert info["beyond"], info               # B's face lies past the old bound
    check(kernels, a, kw)


@pytest.mark.parametrize("drift", ["lead", "lag"])
def test_drift_heavy_kernels(kernels, drift):
    """The 512-entry kernels: 300 empty copies of A put the tile's list past the fast kernels' 256 entries."""
    a, kw, _ = drift_scene(8.0, "diag", drift)
    check(kernels, pad_slabs(a, 300), kw)
    assert kernels.last_heavy_tiles[0] > 0 and kernels.last_heavy_tiles[1] > 0


@pytest.mark.parametrize("pad", [20, 300])
@pytest.mark.parametrize("drift", ["lead", "lag"])
def test_drift_rebuilt_lists(kernels, drift, pad):
    """The backward on lists it rebuilds itself (the forward keeps at most 16 entries per view), fast and 512-entry kernels."""
    from ava256_b200 import lib
    a, kw, _ = drift_scene(8.0, "diag", drift)
    check(kernels, pad_slabs(a, pad), kw, fwd_flags=lib.FLAG_TEST_TINY_LISTS)


@pytest.mark.parametrize("drift", ["lead", "lag"])
def test_drift_ray_grads(kernels, drift):
    """mvp_raymarch_backward_rays: the gradients of the rays and of the primitives against the oracle's."""
    from oracle import oracle
    from tests.oracle_rays import backward_rays
    from tests.test_ray_grads_cpu import check_rays, ray_backward
    a, kw, _ = drift_scene(64.0, "diag", drift)
    with ray_backward(kernels, 1, H, W) as rays:
        gref, rsat = check(kernels, a, kw)
    prim, ref = backward_rays(*a, grad_of(a), rsat, **kw, blocksize=OWARP)
    check_rays(rays, ref)
    for g, r in zip(prim, gref):
        assert relerr(g, r) <= 1e-12


@pytest.mark.parametrize("drift", ["lead", "lag"])
def test_drift_bf16_template(kernels, drift):
    """A bf16 template (the scenes' payloads are exact in bf16): the same samples and images as the oracle's, and the
    transform gradients; the template gradient is rounded to bf16 per reduction and is left to the bf16 tests."""
    from ava256_b200 import lib
    from tests.test_emul_bf16_payload import to_bf16
    a, kw, _ = drift_scene(8.0, "diag", drift)
    ab = list(a)
    ab[7] = to_bf16(a[7]).view(np.float32)
    f = lib.FLAG_TPLATE_BF16
    check(kernels, ab, kw, ref_args=a, names=("primpos", "primrot", "primscale"), fwd_flags=f, bwd_flags=f)


@pytest.mark.parametrize("drift", ["lead", "lag"])
def test_long_march(kernels, drift):
    """B lies 33000 steps into the march: its step interval does not fit the lists' int16 fields and saturates, which only
    widens it; the drift of so long a march is 20 times the old bound."""
    a, kw, info = drift_scene(8.0, "diag", drift, steps=33000, dt_target=2e-4)
    assert info["beyond"]
    check(kernels, a, kw)


@pytest.mark.parametrize("shift", range(8))
@pytest.mark.parametrize("dist", [100.0, 1000.0])
def test_far_origin(kernels, dist, shift):
    """Rays from |o| = 100 and 1000 that march near the origin, their lattice origin tmin / dt about 1e5 and 1e6 steps, where
    the float resolution of a step index passes 1/512 of a step: B's faces at eight sub-step offsets."""
    tmin = dist - 0.3
    dn = DIRS["diag"]
    a, kw, _ = drift_scene(0.5, "diag", "lead", steps=200, tmin=tmin, origin=-dist * dn, shift=shift * 1e-3 / 8)
    assert a[3][0, 0, 0, 0] / a[2] > 2 ** 16
    check(kernels, a, kw)
