/*
 * TEST INFRASTRUCTURE -- the C oracle's backward (oracle/mvp_oracle.c, included unchanged below) with the gradients of the rays
 * as an extra output: mvp_oracle_backward_rays_{f32,f64} is mvp_oracle_backward plus, for every ray,
 *   g_raypos = sum_j dL/dx_j,  g_raydir = sum_j (tmin + j dt) dL/dx_j,  g_tminmax = (<raydir, g_raypos>, 0)
 * over the samples x_j the backward replays (up to and including the saturating one), dL/dx_j = R (s * dL/dy_j) -- minus the
 * sample's contribution to grad_primpos.  Every discrete decision of the march (hit list, lattice start, strict validity,
 * saturation, the 512-entry cap) is held fixed.  Outputs are double and zero-initialised by the caller; each in-image ray is
 * written once.  Only tests/ build, load or call this file.
 */
#include "../oracle/mvp_oracle.c"

/* lattice step of the march's first position (march_init: t = tmin + incs dt) */
static inline int64_t lattice_start(const warp_t *w, int l, real dt) {
    real r0 = RMAX(w->rt0[l], w->tmin[l]);
    real fl = RFLOOR((r0 - w->tmin[l]) * ((real)1 / dt));
    if (!(fl < (real)2147483647.0)) fl = (real)2147483647.0;
    if (!(fl > (real)-2147483648.0)) fl = (real)-2147483648.0;
    return (int64_t)fl;
}

int FN(mvp_oracle_backward_rays)(const FN(mvp_oracle_cfg) *c, const real *raypos, const real *raydir, const real *tminmax,
                                 const real *primpos, const real *primrot, const real *primscale, const real *tplate,
                                 const real *warp, const real *grad_rayrgba, const real *raysat,
                                 double *g_primpos, double *g_primrot, double *g_primscale, double *g_tplate, double *g_warp,
                                 double *g_raypos, double *g_raydir, double *g_tminmax) {
    const size_t wslab = (size_t)c->WD * c->WH * c->WW * 3;
    const int K = c->K;
    const size_t slab = (size_t)c->TD * c->TH * c->TW * 4;
    const real dt = (real)c->stepsize, fs = (real)c->fadescale, fe = (real)c->fadeexp;
    const int gbx = (c->W + c->bsx - 1) / c->bsx, gby = (c->H + c->bsy - 1) / c->bsy;
    const int nwarps = (c->bsx * c->bsy + 31) / 32;
    for (int n = 0; n < c->N; ++n) {
        real *nodeaabb = (real *)malloc(sizeof(real) * 6 * (size_t)(2 * K - 1));
        const real *pp = primpos + (size_t)n * K * 3, *pr = primrot + (size_t)n * K * 9, *ps = primscale + (size_t)n * K * 3;
        const real *tp = tplate + (size_t)n * K * slab;
        double *gpp = g_primpos + (size_t)n * K * 3, *gpr = g_primrot + (size_t)n * K * 9, *gps = g_primscale + (size_t)n * K * 3;
        double *gtp = g_tplate + (size_t)n * K * slab;
        const real *wp = warp ? warp + (size_t)n * K * wslab : NULL;
        double *gwp = warp ? g_warp + (size_t)n * K * wslab : NULL;
        FN(mvp_oracle_aabb)(K, pp, pr, ps, nodeaabb);
#pragma omp parallel for collapse(2) schedule(dynamic, 4)
        for (int by = 0; by < gby; ++by)
            for (int bx = 0; bx < gbx; ++bx) {
                warp_t w;
                w.hit = (int *)malloc(sizeof(int) * (size_t)c->maxhitboxes);
                for (int wi = 0; wi < nwarps; ++wi) {
                    load_warp(&w, c, n, bx, by, wi, raypos, raydir, tminmax);
                    if (w.nl == 0) continue;
                    traverse(&w, K, c->maxhitboxes, nodeaabb, pp, pr, ps);
                    for (int l = 0; l < w.nl; ++l) {
                        if (!w.validthread[l]) continue; /* clamped duplicates contribute zeros (:200, :204) */
                        size_t r = ((size_t)n * c->H + w.py[l]) * c->W + w.px[l];
                        real dL[4] = { grad_rayrgba[r * 4 + 0], grad_rayrgba[r * 4 + 1], grad_rayrgba[r * 4 + 2], grad_rayrgba[r * 4 + 3] };
                        real rs[3] = { raysat[r * 3 + 0], raysat[r * 3 + 1], raysat[r * 3 + 2] };
                        march_t m; march_init(&w, l, dt, &m);
                        real acc[4] = {0, 0, 0, 0};
                        int sat = 0;
                        int64_t j = lattice_start(&w, l, dt);   /* lattice step of m.x: m.t = tmin + j dt */
                        double P[3] = {0, 0, 0}, D[3] = {0, 0, 0};   /* sum dL/dx_j, sum (tmin + j dt) dL/dx_j */
                        while (m.t < m.r1e && !sat) {
                            for (int ks = 0; ks < w.nhit; ++ks) {
                                int k = w.hit[ks];
                                const real *pt_ = pp + 3 * k, *pr_ = pr + 9 * k, *ps_ = ps + 3 * k;
                                xf_t xf; prim_forward(pt_, pr_, ps_, m.x, &xf);
                                if (!(prim_valid(xf.y) && !sat && m.t < m.r1e)) continue;
                                real fade, s[4], wgt[8]; cell_t cl;
                                real y1[3], ww[8]; cell_t wc;
                                if (wp) {
                                    fade = REXP(-fs * ((RPOW(RABS(xf.y[0]), fe) + RPOW(RABS(xf.y[1]), fe)) + RPOW(RABS(xf.y[2]), fe)));
                                    sample_generic(wp + (size_t)k * wslab, 3, xf.y, c->WD, c->WH, c->WW, y1, &wc, ww);
                                    sample_generic(tp + (size_t)k * slab, 4, y1, c->TD, c->TH, c->TW, s, &cl, wgt);
                                    s[3] *= fade;
                                } else
                                sample_forward(tp + (size_t)k * slab, xf.y, c->TD, c->TH, c->TW, fs, fe, &fade, s, &cl, wgt);
                                /* primaccum.h:81-98 */
                                real a = s[3] * dt;
                                int thissat = (acc[3] + a) >= (real)1;
                                sat = sat || thissat;
                                real weight = sat ? ((real)1 - acc[3]) : a;
                                real dLs[4];
                                dLs[0] = weight * dL[0]; dLs[1] = weight * dL[1]; dLs[2] = weight * dL[2];
                                real satrgb1[4] = {0, 0, 0, 0};
                                if (rs[0] > (real)-1) { satrgb1[0] = rs[0]; satrgb1[1] = rs[1]; satrgb1[2] = rs[2]; satrgb1[3] = 1; }
                                real dLa = sat ? (real)0
                                               : dt * ((s[0] - satrgb1[0]) * dL[0] + (s[1] - satrgb1[1]) * dL[1] +
                                                       (s[2] - satrgb1[2]) * dL[2] + ((real)1 - satrgb1[3]) * dL[3]);
                                acc[0] += s[0] * weight; acc[1] += s[1] * weight; acc[2] += s[2] * weight; acc[3] += weight;
                                /* primsampler.h:68-91 (sample.w here is alpha0*fade) */
                                real dLy[3];
                                for (int i = 0; i < 3; ++i) {
                                    real sg = xf.y[i] > 0 ? (real)1 : (real)-1;
                                    real dfade = -(fs * fe) * (RPOW(RABS(xf.y[i]), fe - (real)1) * sg);
                                    dLy[i] = dfade * s[3] * dLa;
                                }
                                dLs[3] = dLa * fade;
                                /* utils.h:504-643 */
                                real dLy1[3];
                                sample_generic_backward(tp + (size_t)k * slab, gtp + (size_t)k * slab, 4, &cl, wgt, dLs, c->TD, c->TH, c->TW, dLy1);
                                if (wp) { /* primsampler.h:82-88: through the warp field back to y0 */
                                    real dLy0w[3];
                                    sample_generic_backward(wp + (size_t)k * wslab, gwp + (size_t)k * wslab, 3, &wc, ww, dLy1, c->WD, c->WH, c->WW, dLy0w);
                                    dLy[0] += dLy0w[0]; dLy[1] += dLy0w[1]; dLy[2] += dLy0w[2];
                                } else {
                                    dLy[0] += dLy1[0]; dLy[1] += dLy1[1]; dLy[2] += dLy1[2];
                                }
                                /* primtransf.h:155-179 */
                                for (int i = 0; i < 3; ++i) atomic_add_d(gps + 3 * k + i, (double)(xf.rxmt[i] * dLy[i]));
                                real g[3] = { dLy[0] * ps_[0], dLy[1] * ps_[1], dLy[2] * ps_[2] };
                                for (int i = 0; i < 3; ++i)
                                    for (int j = 0; j < 3; ++j) atomic_add_d(gpr + 9 * k + 3 * i + j, (double)(xf.xmt[i] * g[j]));
                                for (int i = 0; i < 3; ++i)
                                    atomic_add_d(gpp + 3 * k + i, -(double)(pr_[3 * i + 0] * g[0] + pr_[3 * i + 1] * g[1] + pr_[3 * i + 2] * g[2]));
                                /* dL/dx of the sample = -(its grad_primpos contribution) */
                                const real tj = w.tmin[l] + (real)j * dt;
                                for (int i = 0; i < 3; ++i) {
                                    const real dx = pr_[3 * i + 0] * g[0] + pr_[3 * i + 1] * g[1] + pr_[3 * i + 2] * g[2];
                                    P[i] += (double)dx; D[i] += (double)(tj * dx);
                                }
                            }
                            m.t = m.t + dt;
                            m.x.x = FMA(w.d[l].x, dt, m.x.x); m.x.y = FMA(w.d[l].y, dt, m.x.y); m.x.z = FMA(w.d[l].z, dt, m.x.z);
                            ++j;
                        }
                        for (int i = 0; i < 3; ++i) { g_raypos[r * 3 + i] = P[i]; g_raydir[r * 3 + i] = D[i]; }
                        g_tminmax[r * 2 + 0] = (double)w.d[l].x * P[0] + (double)w.d[l].y * P[1] + (double)w.d[l].z * P[2];
                        g_tminmax[r * 2 + 1] = 0;
                    }
                }
                free(w.hit);
            }
        free(nodeaabb);
    }
    return 0;
}
