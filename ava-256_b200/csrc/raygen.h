// raygen.h -- one ray of a pinhole camera and its clip against the unit cube: compute_raydirs_forward_kernel of the reference
// (/root/reference/extensions/utils/utils_kernel.cu:32-46), as ONE device function that two translation units share:
//
//   * raydirs.cu       (no -use_fast_math, like the reference's utils extension): the stand-alone generator, writes the rays to HBM;
//   * mvp_kernels.cu   (-use_fast_math, like the reference's mvpraymarch extension): the render kernels' prologue generates the
//                      rays of its tile from the camera record instead of reading them (SURVEY.md section 8f row 1).
//
// Both must produce the SAME bits -- a ray that differs in the last place moves samples across voxel cells -- so every operation
// below is an explicitly rounded intrinsic (no contraction, no dependence on the math flags of the translation unit): IEEE
// division, fused multiply-adds where written, a correctly rounded reciprocal square root.  The reference normalises with
// rnorm3df (<= 1 ulp); the result here is within 2 ulp of the reference's ray direction (tests: <= 2e-7 of max|raydir|).
#ifndef MVP_RAYGEN_H_
#define MVP_RAYGEN_H_

// per-view record the accel build derives from (viewpos, viewrot, focal, princpt, volradius): 64 bytes, read as 4 x float4
//   q0 = (o.x, o.y, o.z, R[0])   q1 = (R[1], R[2], R[3], R[4])   q2 = (R[5], R[6], R[7], R[8])   q3 = (princpt.x, princpt.y, focal.x, focal.y)
// with o = viewpos / volradius (utils_kernel.cu:32) and R = viewrot row-major.
struct MvpRayCam {
    float ox, oy, oz;
    float R[9];
    float pcx, pcy, fx, fy;
};

#ifdef MVP_CPU_EMUL
static inline float mvp_rsqrt_rn(float s) { return (float)(1.0 / std::sqrt((double)s)); }
#else
__device__ __forceinline__ float mvp_rsqrt_rn(float s) { return __frsqrt_rn(s); }
#endif

// pixel (px, py) -> unit direction d and the ray's parameter range inside [-1, 1]^3 (tmin clamped at 0, utils_kernel.cu:46)
__device__ __forceinline__ void mvp_gen_ray(const MvpRayCam &c, float px, float py, float &dx, float &dy, float &dz, float &tmin, float &tmax) {
    const float u = __fdiv_rn(__fsub_rn(px, c.pcx), c.fx);                                     // :36-37
    const float v = __fdiv_rn(__fsub_rn(py, c.pcy), c.fy);
    // raydir = viewrot0 * u + viewrot1 * v + viewrot2 * 1                                     :38-39
    // operation order as nvcc contracts the reference's expression (SASS: FMUL, FFMA, FADD): the rounding of
    // a direction component that nearly cancels decides the far-away clip distances of rays that run parallel to a cube face
    const float ex = __fadd_rn(__fmaf_rn(c.R[0], u, __fmul_rn(c.R[3], v)), c.R[6]);
    const float ey = __fadd_rn(__fmaf_rn(c.R[1], u, __fmul_rn(c.R[4], v)), c.R[7]);
    const float ez = __fadd_rn(__fmaf_rn(c.R[2], u, __fmul_rn(c.R[5], v)), c.R[8]);
    const float inv = mvp_rsqrt_rn(__fmaf_rn(ez, ez, __fmaf_rn(ey, ey, __fmul_rn(ex, ex))));    // :40 normalize
    dx = __fmul_rn(ex, inv); dy = __fmul_rn(ey, inv); dz = __fmul_rn(ez, inv);
    // unit-cube slab test                                                                     :42-46
    const float t1x = __fdiv_rn(__fsub_rn(-1.f, c.ox), dx), t1y = __fdiv_rn(__fsub_rn(-1.f, c.oy), dy), t1z = __fdiv_rn(__fsub_rn(-1.f, c.oz), dz);
    const float t2x = __fdiv_rn(__fsub_rn(1.f, c.ox), dx), t2y = __fdiv_rn(__fsub_rn(1.f, c.oy), dy), t2z = __fdiv_rn(__fsub_rn(1.f, c.oz), dz);
    tmin = fmaxf(fmaxf(fminf(t1x, t2x), fmaxf(fminf(t1y, t2y), fminf(t1z, t2z))), 0.f);
    tmax = fminf(fmaxf(t1x, t2x), fminf(fmaxf(t1y, t2y), fmaxf(t1z, t2z)));
}

// Adjoint of mvp_gen_ray: dL/d(ray origin o, direction d, tmin) of pixel (px, py) -> dL/d of the record's inputs: go (the origin
// o = viewpos / volradius), gR (R row-major), gf (focal), gpc (princpt).  tmin = (+-1 - o_a) / d_a on the face a that the forward's
// fmaxf / fminf chain selects, so dtmin/do_a = -1 / d_a and dtmin/dd_a = -tmin / d_a; zero where the chain selects the clamp at 0.
// tmax has no gradient.  The forward values are recomputed with mvp_gen_ray's operations; the adjoint itself is plain fp32.
__device__ __forceinline__ void mvp_gen_ray_adjoint(const MvpRayCam &c, float px, float py, float gox, float goy, float goz, float gdx,
                                                    float gdy, float gdz, float gtmin, float go[3], float gR[9], float gf[2], float gpc[2]) {
    const float u = __fdiv_rn(__fsub_rn(px, c.pcx), c.fx);
    const float v = __fdiv_rn(__fsub_rn(py, c.pcy), c.fy);
    const float ex = __fadd_rn(__fmaf_rn(c.R[0], u, __fmul_rn(c.R[3], v)), c.R[6]);
    const float ey = __fadd_rn(__fmaf_rn(c.R[1], u, __fmul_rn(c.R[4], v)), c.R[7]);
    const float ez = __fadd_rn(__fmaf_rn(c.R[2], u, __fmul_rn(c.R[5], v)), c.R[8]);
    const float inv = mvp_rsqrt_rn(__fmaf_rn(ez, ez, __fmaf_rn(ey, ey, __fmul_rn(ex, ex))));
    const float dx = __fmul_rn(ex, inv), dy = __fmul_rn(ey, inv), dz = __fmul_rn(ez, inv);
    const float t1x = __fdiv_rn(__fsub_rn(-1.f, c.ox), dx), t1y = __fdiv_rn(__fsub_rn(-1.f, c.oy), dy), t1z = __fdiv_rn(__fsub_rn(-1.f, c.oz), dz);
    const float t2x = __fdiv_rn(__fsub_rn(1.f, c.ox), dx), t2y = __fdiv_rn(__fsub_rn(1.f, c.oy), dy), t2z = __fdiv_rn(__fsub_rn(1.f, c.oz), dz);
    const float ax = fminf(t1x, t2x), ay = fminf(t1y, t2y), az = fminf(t1z, t2z);
    const float tm = fmaxf(ax, fmaxf(ay, az));
    go[0] = gox; go[1] = goy; go[2] = goz;
    // Not clamped (a NaN chain gives 0 from the clamp as well) and finite: tm = +inf is a ray parallel to a face whose slab it
    // lies outside (d_a = +-0), which takes no sample and has no tmin gradient; gtmin = 0 skips the term, where 0 / d_a could be NaN.
    if (tm > 0.f && tm <= 3.40282347e38f && gtmin != 0.f) {
        const int a = (tm == ax) ? 0 : (tm == ay) ? 1 : 2;
        const float q = gtmin / (a == 0 ? dx : a == 1 ? dy : dz);
        go[a] -= q;
        if (a == 0) gdx -= q * tm; else if (a == 1) gdy -= q * tm; else gdz -= q * tm;
    }
    // d = e / |e|
    const float dg = dx * gdx + dy * gdy + dz * gdz;
    const float gex = (gdx - dx * dg) * inv, gey = (gdy - dy * dg) * inv, gez = (gdz - dz * dg) * inv;
    // e = R^T (u, v, 1)
    gR[0] = u * gex; gR[1] = u * gey; gR[2] = u * gez;
    gR[3] = v * gex; gR[4] = v * gey; gR[5] = v * gez;
    gR[6] = gex; gR[7] = gey; gR[8] = gez;
    const float gu = c.R[0] * gex + c.R[1] * gey + c.R[2] * gez;
    const float gv = c.R[3] * gex + c.R[4] * gey + c.R[5] * gez;
    // u = (px - princpt.x) / focal.x, v = (py - princpt.y) / focal.y
    gpc[0] = -gu / c.fx; gpc[1] = -gv / c.fy;
    gf[0] = -gu * u / c.fx; gf[1] = -gv * v / c.fy;
}

#endif  // MVP_RAYGEN_H_
