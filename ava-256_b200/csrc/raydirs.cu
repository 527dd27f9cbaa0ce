// raydirs.cu -- pinhole ray generation + unit-cube clip, the step right before the raymarcher
// (SURVEY.md section 8f row 1).  Replaces /root/reference/extensions/utils/utils_kernel.cu:12-52
// (compute_raydirs_forward_kernel).  The reference's backward kernel is an empty stub and its Python backward returns
// None for every input (extensions/utils/utils.py:45-46); here the adjoint (compute_raydirs_backward_kernel) carries the
// rays' gradients on to the camera, for pose and calibration fitting through the photometric loss.
//
// Compiled WITHOUT -use_fast_math, like the reference's utils extension (extensions/utils/setup.py has no such flag).
// The per-ray arithmetic is raygen.h's mvp_gen_ray -- explicitly rounded operations only, because the render kernels' prologue
// (mvp_kernels.cu, compiled WITH -use_fast_math) generates the same rays from the same function and must get the same bits.
// Pure streaming kernel: 32 B written per ray, no reads to speak of
// -> HBM-write bound; one thread per ray, x fastest for coalesced 12/12/8-byte stores.
#ifdef MVP_CPU_EMUL   // test-only host build on the CPU emulation (tests/emul/), see mvp_kernels.cu
#include "cuda_emul.h"
#else
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "mvpraymarch_b200.h"
#include "raygen.h"

namespace {

__global__ void __launch_bounds__(256) compute_raydirs_kernel(int N, int H, int W, const float *__restrict__ viewpos,
                                                              const float *__restrict__ viewrot, const float *__restrict__ focal,
                                                              const float *__restrict__ princpt, const float2 *__restrict__ pixelcoords,
                                                              float volradius, float *__restrict__ raypos, float *__restrict__ raydir,
                                                              float2 *__restrict__ tminmax) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    const int h = blockIdx.y;
    const int n = blockIdx.z;
    if (w >= W) return;
    MvpRayCam c;
    // raypos = viewpos / volradius                                           utils_kernel.cu:32
    c.ox = __fdiv_rn(viewpos[n * 3 + 0], volradius); c.oy = __fdiv_rn(viewpos[n * 3 + 1], volradius); c.oz = __fdiv_rn(viewpos[n * 3 + 2], volradius);
#pragma unroll
    for (int i = 0; i < 9; ++i) c.R[i] = viewrot[n * 9 + i];
    c.pcx = princpt[n * 2 + 0]; c.pcy = princpt[n * 2 + 1]; c.fx = focal[n * 2 + 0]; c.fy = focal[n * 2 + 1];
    const size_t r = ((size_t)n * H + h) * W + w;
    const float2 pc = pixelcoords ? __ldg(pixelcoords + r) : make_float2((float)w, (float)h);
    float dx, dy, dz, tmin, tmax;
    mvp_gen_ray(c, pc.x, pc.y, dx, dy, dz, tmin, tmax);                       // :36-46, shared with the render kernels' prologue
    const float rx = c.ox, ry = c.oy, rz = c.oz;
    raypos[r * 3 + 0] = rx; raypos[r * 3 + 1] = ry; raypos[r * 3 + 2] = rz;
    raydir[r * 3 + 0] = dx; raydir[r * 3 + 1] = dy; raydir[r * 3 + 2] = dz;
    tminmax[r] = make_float2(tmin, tmax);
}

// Adjoint (mvp_compute_raydirs_backward): same thread -> ray mapping; each thread recomputes its ray and chains its gradients into
// the 16 scalars of its view (viewpos 3, viewrot 9, focal 2, princpt 2).  A block is one row segment of one view, so the 16 sums
// are reduced per block -- a 16-value butterfly over the warp, then across the warps in shared memory -- and added to global memory
// with one atomic per block and value.  Streaming: 32 B read per ray (+ 8 B of pixelcoords).
constexpr int kRdWarps = 256 / 32;
__global__ void __launch_bounds__(256) compute_raydirs_backward_kernel(int N, int H, int W, const float *__restrict__ viewpos,
                                                                       const float *__restrict__ viewrot, const float *__restrict__ focal,
                                                                       const float *__restrict__ princpt, const float2 *__restrict__ pixelcoords,
                                                                       float volradius, const float *__restrict__ grad_raypos,
                                                                       const float *__restrict__ grad_raydir, const float2 *__restrict__ grad_tminmax,
                                                                       float *__restrict__ grad_viewpos, float *__restrict__ grad_viewrot,
                                                                       float *__restrict__ grad_focal, float *__restrict__ grad_princpt) {
    __shared__ float red[kRdWarps][16];
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    const int h = blockIdx.y;
    const int n = blockIdx.z;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float g[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) g[i] = 0.f;
    if (w < W) {
        MvpRayCam c;
        c.ox = __fdiv_rn(viewpos[n * 3 + 0], volradius); c.oy = __fdiv_rn(viewpos[n * 3 + 1], volradius); c.oz = __fdiv_rn(viewpos[n * 3 + 2], volradius);
#pragma unroll
        for (int i = 0; i < 9; ++i) c.R[i] = viewrot[n * 9 + i];
        c.pcx = princpt[n * 2 + 0]; c.pcy = princpt[n * 2 + 1]; c.fx = focal[n * 2 + 0]; c.fy = focal[n * 2 + 1];
        const size_t r = ((size_t)n * H + h) * W + w;
        const float2 pc = pixelcoords ? __ldg(pixelcoords + r) : make_float2((float)w, (float)h);
        const float2 gt = __ldg(grad_tminmax + r);
        float go[3], gR[9], gf[2], gpc[2];
        mvp_gen_ray_adjoint(c, pc.x, pc.y, __ldg(grad_raypos + r * 3 + 0), __ldg(grad_raypos + r * 3 + 1), __ldg(grad_raypos + r * 3 + 2),
                            __ldg(grad_raydir + r * 3 + 0), __ldg(grad_raydir + r * 3 + 1), __ldg(grad_raydir + r * 3 + 2), gt.x, go, gR, gf, gpc);
        // o = viewpos / volradius
        g[0] = go[0] / volradius; g[1] = go[1] / volradius; g[2] = go[2] / volradius;
#pragma unroll
        for (int i = 0; i < 9; ++i) g[3 + i] = gR[i];
        g[12] = gf[0]; g[13] = gf[1]; g[14] = gpc[0]; g[15] = gpc[1];
    }
    // 16-value butterfly: after the 5 stages lanes 2i and 2i+1 hold the warp's sum of g[i]
#pragma unroll
    for (int s = 16, m = 8; s >= 2; s >>= 1, m >>= 1) {
#pragma unroll
        for (int i = 0; i < m; ++i) {
            const bool up = lane & s;
            const float send = up ? g[i] : g[i + m];
            const float keep = up ? g[i + m] : g[i];
            g[i] = keep + __shfl_xor_sync(0xffffffffu, send, s);
        }
    }
    g[0] += __shfl_xor_sync(0xffffffffu, g[0], 1);
    if (!(lane & 1)) red[warp][lane >> 1] = g[0];
    __syncthreads();
    if (threadIdx.x < 16) {
        const int vi = threadIdx.x;
        float s = 0.f;
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) s += red[k][vi];
        float *dst = vi < 3 ? grad_viewpos + n * 3 + vi
                            : vi < 12 ? grad_viewrot + n * 9 + (vi - 3) : vi < 14 ? grad_focal + n * 2 + (vi - 12) : grad_princpt + n * 2 + (vi - 14);
        atomicAdd(dst, s);
    }
}

// ---- Morton codes of (normalised) slab centres: compute_morton of the reference (mvpraymarch.cpp:106-121; bvh.cu:20-57) ----
// quantise each coordinate of a point of the unit cube to 10 bits and interleave them x | y | z from the top bit down
__device__ __forceinline__ unsigned spread10(unsigned v) {
    // 10 bits -> every third bit of 30: four shift-or-mask rounds (16, 8, 4, 2 positions), written as multiplies
    v = (v | (v << 16)) & 0xFF0000FFu;
    v = (v | (v << 8)) & 0x0F00F00Fu;
    v = (v | (v << 4)) & 0xC30C30C3u;
    v = (v | (v << 2)) & 0x49249249u;
    return v;
}
__global__ void __launch_bounds__(256) compute_morton_kernel(size_t NK, const float *__restrict__ centre, int *__restrict__ code) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= NK) return;
    const float qx = fminf(fmaxf(centre[i * 3 + 0] * 1024.f, 0.f), 1023.f);
    const float qy = fminf(fmaxf(centre[i * 3 + 1] * 1024.f, 0.f), 1023.f);
    const float qz = fminf(fmaxf(centre[i * 3 + 2] * 1024.f, 0.f), 1023.f);
    code[i] = (int)((spread10((unsigned)qx) << 2) | (spread10((unsigned)qy) << 1) | spread10((unsigned)qz));
}

}  // namespace

extern "C" int mvp_compute_morton(int32_t N, int32_t K, const float *centre, int32_t *code, void *stream) {
    if (!centre || !code) return MVP_ERR_NULL;
    if (N < 1 || K < 1) return MVP_ERR_SHAPE;
    const size_t NK = (size_t)N * K;
#ifdef MVP_CPU_EMUL
    MVP_LAUNCH(compute_morton_kernel, (unsigned)((NK + 255) / 256), 256, 0, stream, NK, centre, code);
#else
    compute_morton_kernel<<<(unsigned)((NK + 255) / 256), 256, 0, (cudaStream_t)stream>>>(NK, centre, code);
#endif
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? MVP_OK : (int)e;
}

extern "C" int mvp_compute_raydirs(int32_t N, int32_t H, int32_t W, const float *viewpos, const float *viewrot, const float *focal,
                                   const float *princpt, const float *pixelcoords, float volradius, float *raypos, float *raydir,
                                   float *tminmax, void *stream) {
    if (!viewpos || !viewrot || !focal || !princpt || !raypos || !raydir || !tminmax) return MVP_ERR_NULL;
    if (N < 1 || H < 1 || W < 1 || H > 65535 || N > 65535) return MVP_ERR_SHAPE;
    dim3 grid((W + 255) / 256, H, N);
#ifdef MVP_CPU_EMUL
    MVP_LAUNCH(compute_raydirs_kernel, grid, 256, 0, stream, N, H, W, viewpos, viewrot, focal, princpt,
               reinterpret_cast<const float2 *>(pixelcoords), volradius, raypos, raydir, reinterpret_cast<float2 *>(tminmax));
#else
    compute_raydirs_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(N, H, W, viewpos, viewrot, focal, princpt,
                                                                  reinterpret_cast<const float2 *>(pixelcoords), volradius, raypos,
                                                                  raydir, reinterpret_cast<float2 *>(tminmax));
#endif
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? MVP_OK : (int)e;
}

extern "C" int mvp_compute_raydirs_backward(int32_t N, int32_t H, int32_t W, const float *viewpos, const float *viewrot, const float *focal,
                                            const float *princpt, const float *pixelcoords, float volradius, const float *grad_raypos,
                                            const float *grad_raydir, const float *grad_tminmax, float *grad_viewpos, float *grad_viewrot,
                                            float *grad_focal, float *grad_princpt, void *stream) {
    if (!viewpos || !viewrot || !focal || !princpt || !grad_raypos || !grad_raydir || !grad_tminmax || !grad_viewpos || !grad_viewrot ||
        !grad_focal || !grad_princpt)
        return MVP_ERR_NULL;
    if (N < 1 || H < 1 || W < 1 || H > 65535 || N > 65535) return MVP_ERR_SHAPE;
    if (!(volradius > 0.f) || !(volradius < 3.0e38f)) return MVP_ERR_CAMERA;
    if (((uintptr_t)pixelcoords | (uintptr_t)grad_tminmax) & 7) return MVP_ERR_ALIGN;
    if (((uintptr_t)viewpos | (uintptr_t)viewrot | (uintptr_t)focal | (uintptr_t)princpt | (uintptr_t)grad_raypos | (uintptr_t)grad_raydir |
         (uintptr_t)grad_viewpos | (uintptr_t)grad_viewrot | (uintptr_t)grad_focal | (uintptr_t)grad_princpt) & 3)
        return MVP_ERR_ALIGN;
    dim3 grid((W + 255) / 256, H, N);
#ifdef MVP_CPU_EMUL
    MVP_LAUNCH(compute_raydirs_backward_kernel, grid, 256, 0, stream, N, H, W, viewpos, viewrot, focal, princpt,
               reinterpret_cast<const float2 *>(pixelcoords), volradius, grad_raypos, grad_raydir,
               reinterpret_cast<const float2 *>(grad_tminmax), grad_viewpos, grad_viewrot, grad_focal, grad_princpt);
#else
    compute_raydirs_backward_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(N, H, W, viewpos, viewrot, focal, princpt,
                                                                           reinterpret_cast<const float2 *>(pixelcoords), volradius,
                                                                           grad_raypos, grad_raydir, reinterpret_cast<const float2 *>(grad_tminmax),
                                                                           grad_viewpos, grad_viewrot, grad_focal, grad_princpt);
#endif
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? MVP_OK : (int)e;
}
