// epilogue.cu -- the two streaming kernels either side of the raymarcher (SURVEY.md section 8f rows 2 and 4):
//
//   mvp_composite_{forward,backward}        rayrgba [N,H,W,4] -> NCHW rgb (+ colour calibration + background matting)
//                                           and alpha, replacing the permute / 2x contiguous / mul / add / mul / add
//                                           chain of models/raymarchers/mvpraymarcher.py:50-51,
//                                           models/colorcals/colorcal.py:26-29, models/autoencoder.py:262-270
//   mvp_assemble_payload_{forward,backward} decoder images -> channels-last slabs with the relu(x*25+100) / relu
//                                           de-normalisation fused in, replacing the view / permute / reshape / cat /
//                                           relu chain of models/decoders/rgb.py:128-143, geometry.py:180-185,
//                                           assembler.py:261
//
// Both are pure layout + elementwise work: HBM-bound, every byte touched once.  Bytes per unit (what the roofline
// counts): composite fwd 16 B in + 16 B out per ray (+12 B with a background); bwd 16 B in (+16 B rayrgba, +12 B bg)
// + 16 B out; payload 16 B in + 16 B out per texel forward, 32 B in + 16 B out backward (bf16 template: 16 + 8 forward,
// 16 + 16 backward; mvp_assemble_payload_*_bf16, with mvp_sum_views_bf16 for the bf16 view sum).  Threads walk 4 consecutive
// pixels / columns so every global access is a 16-byte vector and a warp's request covers whole 128-byte lines on the
// planar side and 64 B per lane on the channels-last side; a scalar variant covers shapes that are not multiples of 4.
//
// Compiled WITHOUT -use_fast_math: the bodies use explicit single-rounding intrinsics so the forward results are
// bit-identical to the eager PyTorch expressions they replace.
#ifdef MVP_CPU_EMUL   // test-only host build on the CPU emulation (tests/emul/), see mvp_kernels.cu
#include "cuda_emul.h"
#define MVP_EPI_LAUNCH(grid, st, ...)              \
    do {                                           \
        auto kern_ = MVP_EPI_KERNEL;               \
        MVP_LAUNCH(kern_, grid, kThreads, 0, st, __VA_ARGS__); \
    } while (0)
#else
#include <cuda_runtime.h>
#define MVP_EPI_LAUNCH(grid, st, ...) MVP_EPI_KERNEL<<<grid, kThreads, 0, st>>>(__VA_ARGS__)
#endif
#include <stdint.h>

#include "epilogue_body.h"
#include "mvpraymarch_b200.h"

namespace {

using namespace mvp_epi;
constexpr int kThreads = 256;

template <int V>
__global__ void __launch_bounds__(kThreads) composite_forward_kernel(CompositeFwd a) {
    const size_t px = ((size_t)blockIdx.x * kThreads + threadIdx.x) * V;
    if (px < a.HW) composite_fwd<V>(a, (int)blockIdx.y, px);
}

template <int V>
__global__ void __launch_bounds__(kThreads) composite_backward_kernel(CompositeBwd a, float *__restrict__ grad_ccw,
                                                                     float *__restrict__ grad_ccb) {
    const int n = (int)blockIdx.y;
    const size_t px = ((size_t)blockIdx.x * kThreads + threadIdx.x) * V;
    float part[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (px < a.HW) composite_bwd<V>(a, n, px, part);
    if (a.want_cc) {   // uniform across the grid: every thread takes part in the reduction
        __shared__ float s_part[kThreads / 32][6];
#pragma unroll
        for (int i = 0; i < 6; ++i) {
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) part[i] += __shfl_xor_sync(0xffffffffu, part[i], off);
        }
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        if (lane == 0) {
#pragma unroll
            for (int i = 0; i < 6; ++i) s_part[warp][i] = part[i];
        }
        __syncthreads();
        if (threadIdx.x < 6) {
            float t = 0.f;
#pragma unroll
            for (int w = 0; w < kThreads / 32; ++w) t += s_part[w][threadIdx.x];
            float *dst = threadIdx.x < 3 ? grad_ccw + n * 3 + threadIdx.x : grad_ccb + n * 3 + (threadIdx.x - 3);
            atomicAdd(dst, t);
        }
    }
}

template <int V, int BT>
__global__ void __launch_bounds__(kThreads) payload_forward_kernel(PayloadArgs a, size_t total) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (e < total) payload_fwd<V, BT>(a, e);
}

template <int V, int BT>
__global__ void __launch_bounds__(kThreads) payload_backward_kernel(PayloadArgs a, size_t total) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (e < total) payload_bwd<V, BT>(a, e);
}

template <int V, int BT>
__global__ void __launch_bounds__(kThreads) payload_forward_bf16_kernel(PayloadArgs a, size_t total) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (e < total) payload_fwd_bf16<V, BT>(a, e);
}

template <int V, int BT>
__global__ void __launch_bounds__(kThreads) payload_backward_bf16_kernel(PayloadArgs a, size_t total) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (e < total) payload_bwd_bf16<V, BT>(a, e);
}

// One subject's tensor written once per view: dst[v][i] = src[i].  Streaming stores; the source stays in L2.
__global__ void __launch_bounds__(kThreads) expand_views_kernel(const float4 *__restrict__ src, float4 *__restrict__ dst, size_t count4,
                                                                int n) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (e >= count4) return;
    const float4 v = __ldg(src + e);
    for (int i = 0; i < n; ++i) __stcs(dst + (size_t)i * count4 + e, v);
}
__global__ void __launch_bounds__(kThreads) expand_views_scalar_kernel(const float *__restrict__ src, float *__restrict__ dst, size_t count,
                                                                       int n) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (e >= count) return;
    const float v = __ldg(src + e);
    for (int i = 0; i < n; ++i) dst[(size_t)i * count + e] = v;
}

// The adjoint: dst[i] = sum over the views of src[v][i], added up in view order (deterministic).  Every source byte is read once
// (streaming loads, eight views in flight per thread), the sum is written once.
__global__ void __launch_bounds__(kThreads) sum_views_kernel(const float4 *__restrict__ src, float4 *__restrict__ dst, size_t count4, int n) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (e >= count4) return;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int i = 0;
    for (; i + 8 <= n; i += 8) {
        float4 v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = __ldcs(src + (size_t)(i + j) * count4 + e);
#pragma unroll
        for (int j = 0; j < 8; ++j) { acc.x += v[j].x; acc.y += v[j].y; acc.z += v[j].z; acc.w += v[j].w; }
    }
    for (; i < n; ++i) {
        const float4 v = __ldcs(src + (size_t)i * count4 + e);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    dst[e] = acc;
}
__global__ void __launch_bounds__(kThreads) sum_views_scalar_kernel(const float *__restrict__ src, float *__restrict__ dst, size_t count, int n) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (e >= count) return;
    float acc = 0.f;
    for (int i = 0; i < n; ++i) acc += src[(size_t)i * count + e];
    dst[e] = acc;
}

// The same sum over bf16 views: each value widened exactly and added in fp32 in view order (the order of sum_views_kernel,
// so the fp32 result equals mvp_sum_views of the widened source bit for bit); a bf16 dst gets that sum rounded once.
// 16-byte path: one uint4 (8 bf16) per view and thread, eight views in flight; the fp32 dst takes two float4 stores.
template <bool kDstBf16>
__global__ void __launch_bounds__(kThreads) sum_views_bf16_kernel(const uint4 *__restrict__ src, void *__restrict__ dst, size_t count8,
                                                                  int n) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (e >= count8) return;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const auto add = [&acc](const uint4 v) {
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) { acc[2 * k] += bf16_lo(w[k]); acc[2 * k + 1] += bf16_hi(w[k]); }
    };
    int i = 0;
    for (; i + 8 <= n; i += 8) {
        uint4 v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = __ldcs(src + (size_t)(i + j) * count8 + e);
#pragma unroll
        for (int j = 0; j < 8; ++j) add(v[j]);
    }
    for (; i < n; ++i) add(__ldcs(src + (size_t)i * count8 + e));
    if (kDstBf16) {
        reinterpret_cast<uint4 *>(dst)[e] = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]),
                                                       pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
    } else {
        float4 *d = reinterpret_cast<float4 *>(dst) + 2 * e;
        d[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
        d[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
}
template <bool kDstBf16>
__global__ void __launch_bounds__(kThreads) sum_views_bf16_scalar_kernel(const uint16_t *__restrict__ src, void *__restrict__ dst,
                                                                         size_t count, int n) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (e >= count) return;
    float acc = 0.f;
    for (int i = 0; i < n; ++i) acc += bf16_lo(src[(size_t)i * count + e]);
    if (kDstBf16) reinterpret_cast<uint16_t *>(dst)[e] = (uint16_t)pack_bf16x2(acc, 0.f);
    else reinterpret_cast<float *>(dst)[e] = acc;
}

inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

inline int finish() {
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? MVP_OK : (int)e;
}

}  // namespace

extern "C" int mvp_composite_forward(int32_t N, int32_t H, int32_t W, const float *rayrgba, const float *ccw, const float *ccb,
                                     const float *bg, float *irgbrec, float *rayalpha, void *stream) {
    if (!rayrgba || !irgbrec) return MVP_ERR_NULL;
    if ((ccw == nullptr) != (ccb == nullptr)) return MVP_ERR_NULL;
    if (N < 1 || H < 1 || W < 1 || N > 65535 || H >= 32768 || W >= 32768) return MVP_ERR_SHAPE;
    if (!aligned16(rayrgba)) return MVP_ERR_ALIGN;
    CompositeFwd a;
    a.HW = (size_t)H * W;
    a.rayrgba = rayrgba; a.ccw = ccw; a.ccb = ccb; a.bg = bg; a.irgbrec = irgbrec; a.rayalpha = rayalpha;
    const bool vec = a.HW % 4 == 0 && aligned16(irgbrec) && (!bg || aligned16(bg)) && (!rayalpha || aligned16(rayalpha));
    cudaStream_t st = (cudaStream_t)stream;
    if (vec) {
        dim3 grid((unsigned)((a.HW / 4 + kThreads - 1) / kThreads), N);
        {
#define MVP_EPI_KERNEL composite_forward_kernel<4>
        MVP_EPI_LAUNCH(grid, st, a);
#undef MVP_EPI_KERNEL
        }
    } else {
        dim3 grid((unsigned)((a.HW + kThreads - 1) / kThreads), N);
        {
#define MVP_EPI_KERNEL composite_forward_kernel<1>
        MVP_EPI_LAUNCH(grid, st, a);
#undef MVP_EPI_KERNEL
        }
    }
    return finish();
}

extern "C" int mvp_composite_backward(int32_t N, int32_t H, int32_t W, const float *rayrgba, const float *ccw, const float *bg,
                                      const float *grad_irgbrec, const float *grad_rayalpha, float *grad_rayrgba,
                                      float *grad_ccw, float *grad_ccb, float *grad_bg, void *stream) {
    if (!grad_irgbrec || !grad_rayrgba) return MVP_ERR_NULL;
    if ((grad_ccw == nullptr) != (grad_ccb == nullptr)) return MVP_ERR_NULL;
    if (grad_bg && !bg) return MVP_ERR_NULL;
    if ((grad_ccw || grad_bg) && !rayrgba) return MVP_ERR_NULL;
    if (N < 1 || H < 1 || W < 1 || N > 65535 || H >= 32768 || W >= 32768) return MVP_ERR_SHAPE;
    if (!aligned16(grad_rayrgba) || (rayrgba && !aligned16(rayrgba))) return MVP_ERR_ALIGN;
    CompositeBwd a;
    a.HW = (size_t)H * W;
    a.rayrgba = rayrgba; a.ccw = ccw; a.bg = bg; a.grad_irgbrec = grad_irgbrec; a.grad_rayalpha = grad_rayalpha;
    a.grad_rayrgba = grad_rayrgba; a.grad_bg = grad_bg; a.want_cc = grad_ccw != nullptr;
    const bool vec = a.HW % 4 == 0 && aligned16(grad_irgbrec) && (!bg || aligned16(bg)) &&
                     (!grad_rayalpha || aligned16(grad_rayalpha)) && (!grad_bg || aligned16(grad_bg));
    cudaStream_t st = (cudaStream_t)stream;
    if (vec) {
        dim3 grid((unsigned)((a.HW / 4 + kThreads - 1) / kThreads), N);
        {
#define MVP_EPI_KERNEL composite_backward_kernel<4>
        MVP_EPI_LAUNCH(grid, st, a, grad_ccw, grad_ccb);
#undef MVP_EPI_KERNEL
        }
    } else {
        dim3 grid((unsigned)((a.HW + kThreads - 1) / kThreads), N);
        {
#define MVP_EPI_KERNEL composite_backward_kernel<1>
        MVP_EPI_LAUNCH(grid, st, a, grad_ccw, grad_ccb);
#undef MVP_EPI_KERNEL
        }
    }
    return finish();
}

namespace {

// Elements (threads) of a payload launch, or 0 when the shape is unsupported.
inline size_t payload_elements(int32_t N, int32_t hb, int32_t wb, int32_t B, int V) {
    if (N < 1 || hb < 1 || wb < 1 || B < 1 || B > 64) return 0;
    const size_t total = (size_t)N * hb * B * B * ((size_t)wb * B);
    const size_t e = total / V;
    if ((e + kThreads - 1) / kThreads > 0x7fffffffull) return 0;
    return e;
}

// One payload launch: direction (kBwd), template type (kBf16) and the V / BT variant.
template <bool kBwd, bool kBf16, int V, int BT>
void launch_payload_variant(unsigned grid, cudaStream_t st, const PayloadArgs &a, size_t total) {
    if constexpr (kBwd && kBf16) {
#define MVP_EPI_KERNEL payload_backward_bf16_kernel<V, BT>
        MVP_EPI_LAUNCH(grid, st, a, total);
#undef MVP_EPI_KERNEL
    } else if constexpr (kBwd) {
#define MVP_EPI_KERNEL payload_backward_kernel<V, BT>
        MVP_EPI_LAUNCH(grid, st, a, total);
#undef MVP_EPI_KERNEL
    } else if constexpr (kBf16) {
#define MVP_EPI_KERNEL payload_forward_bf16_kernel<V, BT>
        MVP_EPI_LAUNCH(grid, st, a, total);
#undef MVP_EPI_KERNEL
    } else {
#define MVP_EPI_KERNEL payload_forward_kernel<V, BT>
        MVP_EPI_LAUNCH(grid, st, a, total);
#undef MVP_EPI_KERNEL
    }
}

template <bool kBwd, bool kBf16 = false>
int launch_payload(int32_t N, int32_t hb, int32_t wb, int32_t B, const PayloadArgs &a, bool vec, cudaStream_t st) {
    const int V = vec ? 4 : 1;
    const size_t total = payload_elements(N, hb, wb, B, V);
    if (total == 0) return MVP_ERR_SHAPE;
    const unsigned grid = (unsigned)((total + kThreads - 1) / kThreads);
    if (vec && B == 8) launch_payload_variant<kBwd, kBf16, 4, 8>(grid, st, a, total);
    else if (vec) launch_payload_variant<kBwd, kBf16, 4, 0>(grid, st, a, total);
    else launch_payload_variant<kBwd, kBf16, 1, 0>(grid, st, a, total);
    return finish();
}

inline bool aligned(const void *p, uintptr_t n) { return (reinterpret_cast<uintptr_t>(p) & (n - 1)) == 0; }

}  // namespace

extern "C" int mvp_assemble_payload_forward(int32_t N, int32_t hb, int32_t wb, int32_t B, const float *tex, const float *opacity,
                                            float rgb_scale, float rgb_bias, float *tplate, void *stream) {
    if (!tex || !opacity || !tplate) return MVP_ERR_NULL;
    if (!aligned16(tplate)) return MVP_ERR_ALIGN;
    PayloadArgs a = {};
    a.hb = hb; a.wb = wb; a.B = B; a.rgb_scale = rgb_scale; a.rgb_bias = rgb_bias;
    a.tex = tex; a.opacity = opacity; a.tplate = tplate;
    const bool vec = B > 0 && B % 4 == 0 && aligned16(tex) && aligned16(opacity);
    return launch_payload<false>(N, hb, wb, B, a, vec, (cudaStream_t)stream);
}

extern "C" int mvp_assemble_payload_backward(int32_t N, int32_t hb, int32_t wb, int32_t B, const float *tplate,
                                             const float *grad_tplate, float rgb_scale, float *grad_tex, float *grad_opacity,
                                             void *stream) {
    if (!tplate || !grad_tplate || !grad_tex || !grad_opacity) return MVP_ERR_NULL;
    if (!aligned16(tplate) || !aligned16(grad_tplate)) return MVP_ERR_ALIGN;
    PayloadArgs a = {};
    a.hb = hb; a.wb = wb; a.B = B; a.rgb_scale = rgb_scale;
    a.tplate_in = tplate; a.grad_tplate = grad_tplate; a.grad_tex = grad_tex; a.grad_opacity = grad_opacity;
    const bool vec = B > 0 && B % 4 == 0 && aligned16(grad_tex) && aligned16(grad_opacity);
    return launch_payload<true>(N, hb, wb, B, a, vec, (cudaStream_t)stream);
}

// bf16 templates: 8 bytes per texel.  The vector variant (V = 4) moves 32 contiguous template bytes per thread in two 16-byte
// accesses, so it also needs a 16-byte aligned template (and gradient); the scalar variant needs 8.
extern "C" int mvp_assemble_payload_forward_bf16(int32_t N, int32_t hb, int32_t wb, int32_t B, const float *tex, const float *opacity,
                                                 float rgb_scale, float rgb_bias, void *tplate, void *stream) {
    if (!tex || !opacity || !tplate) return MVP_ERR_NULL;
    if (!aligned(tplate, 8)) return MVP_ERR_ALIGN;
    PayloadArgs a = {};
    a.hb = hb; a.wb = wb; a.B = B; a.rgb_scale = rgb_scale; a.rgb_bias = rgb_bias;
    a.tex = tex; a.opacity = opacity; a.tplate = static_cast<float *>(tplate);
    const bool vec = B > 0 && B % 4 == 0 && aligned16(tex) && aligned16(opacity) && aligned16(tplate);
    return launch_payload<false, true>(N, hb, wb, B, a, vec, (cudaStream_t)stream);
}

extern "C" int mvp_assemble_payload_backward_bf16(int32_t N, int32_t hb, int32_t wb, int32_t B, const void *tplate,
                                                  const void *grad_tplate, float rgb_scale, float *grad_tex, float *grad_opacity,
                                                  void *stream) {
    if (!tplate || !grad_tplate || !grad_tex || !grad_opacity) return MVP_ERR_NULL;
    if (!aligned(tplate, 8) || !aligned(grad_tplate, 8)) return MVP_ERR_ALIGN;
    PayloadArgs a = {};
    a.hb = hb; a.wb = wb; a.B = B; a.rgb_scale = rgb_scale;
    a.tplate_in = static_cast<const float *>(tplate); a.grad_tplate = static_cast<const float *>(grad_tplate);
    a.grad_tex = grad_tex; a.grad_opacity = grad_opacity;
    const bool vec = B > 0 && B % 4 == 0 && aligned16(grad_tex) && aligned16(grad_opacity) && aligned16(tplate) && aligned16(grad_tplate);
    return launch_payload<true, true>(N, hb, wb, B, a, vec, (cudaStream_t)stream);
}

extern "C" int mvp_expand_views(const float *src, float *dst, size_t count, int32_t n_views, void *stream) {
    if (!src || !dst) return MVP_ERR_NULL;
    if (n_views < 0) return MVP_ERR_SHAPE;
    if (count == 0 || n_views == 0) return MVP_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (count % 4 == 0 && aligned16(src) && aligned16(dst)) {
        const size_t c4 = count / 4;
        const dim3 grid((unsigned)((c4 + kThreads - 1) / kThreads));
#define MVP_EPI_KERNEL expand_views_kernel
        MVP_EPI_LAUNCH(grid, st, reinterpret_cast<const float4 *>(src), reinterpret_cast<float4 *>(dst), c4, (int)n_views);
#undef MVP_EPI_KERNEL
    } else {
        const dim3 grid((unsigned)((count + kThreads - 1) / kThreads));
#define MVP_EPI_KERNEL expand_views_scalar_kernel
        MVP_EPI_LAUNCH(grid, st, src, dst, count, (int)n_views);
#undef MVP_EPI_KERNEL
    }
    return finish();
}

extern "C" int mvp_sum_views(const float *src, float *dst, size_t count, int32_t n_views, void *stream) {
    if (!src || !dst) return MVP_ERR_NULL;
    if (n_views < 1) return MVP_ERR_SHAPE;
    if (count == 0) return MVP_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (count % 4 == 0 && aligned16(src) && aligned16(dst)) {
        const size_t c4 = count / 4;
        const dim3 grid((unsigned)((c4 + kThreads - 1) / kThreads));
#define MVP_EPI_KERNEL sum_views_kernel
        MVP_EPI_LAUNCH(grid, st, reinterpret_cast<const float4 *>(src), reinterpret_cast<float4 *>(dst), c4, (int)n_views);
#undef MVP_EPI_KERNEL
    } else {
        const dim3 grid((unsigned)((count + kThreads - 1) / kThreads));
#define MVP_EPI_KERNEL sum_views_scalar_kernel
        MVP_EPI_LAUNCH(grid, st, src, dst, count, (int)n_views);
#undef MVP_EPI_KERNEL
    }
    return finish();
}

extern "C" int mvp_sum_views_bf16(const void *src, void *dst, size_t count, int32_t n_views, int32_t dst_bf16, void *stream) {
    if (!src || !dst) return MVP_ERR_NULL;
    if (n_views < 1) return MVP_ERR_SHAPE;
    if (!aligned(src, 2) || !aligned(dst, dst_bf16 ? 2 : 4)) return MVP_ERR_ALIGN;
    if (count == 0) return MVP_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (count % 8 == 0 && aligned16(src) && aligned16(dst)) {
        const size_t c8 = count / 8;
        const dim3 grid((unsigned)((c8 + kThreads - 1) / kThreads));
        const uint4 *s = static_cast<const uint4 *>(src);
        if (dst_bf16) {
#define MVP_EPI_KERNEL sum_views_bf16_kernel<true>
            MVP_EPI_LAUNCH(grid, st, s, dst, c8, (int)n_views);
#undef MVP_EPI_KERNEL
        } else {
#define MVP_EPI_KERNEL sum_views_bf16_kernel<false>
            MVP_EPI_LAUNCH(grid, st, s, dst, c8, (int)n_views);
#undef MVP_EPI_KERNEL
        }
    } else {
        const dim3 grid((unsigned)((count + kThreads - 1) / kThreads));
        const uint16_t *s = static_cast<const uint16_t *>(src);
        if (dst_bf16) {
#define MVP_EPI_KERNEL sum_views_bf16_scalar_kernel<true>
            MVP_EPI_LAUNCH(grid, st, s, dst, count, (int)n_views);
#undef MVP_EPI_KERNEL
        } else {
#define MVP_EPI_KERNEL sum_views_bf16_scalar_kernel<false>
            MVP_EPI_LAUNCH(grid, st, s, dst, count, (int)n_views);
#undef MVP_EPI_KERNEL
        }
    }
    return finish();
}
