// epilogue_body.h -- per-element bodies of the two streaming kernels either side of the raymarcher
// (SURVEY.md section 8f rows 2 and 4).  Everything except the thread->element mapping and the block reduction lives
// here as host+device inline functions, so tests/emul/ can compile the very same bodies with g++ and check index
// arithmetic and rounding order against the PyTorch expressions of the reference on the CPU (the kernels themselves
// never run on the CPU: the emulation is test infrastructure).
//
// Arithmetic is written with explicit single roundings (no FMA contraction) because the reference evaluates these
// expressions as separate eager PyTorch kernels (one rounding per op); the forward results are therefore bit-exact.
#ifndef MVP_EPILOGUE_BODY_H_
#define MVP_EPILOGUE_BODY_H_

#include <cuda_runtime.h>  // float4 / make_float4 on host and device
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define MVP_HD __host__ __device__ __forceinline__
#else
#define MVP_HD inline
#endif

#ifdef __CUDA_ARCH__
#define MVP_MUL(a, b) __fmul_rn((a), (b))
#define MVP_ADD(a, b) __fadd_rn((a), (b))
#define MVP_SUB(a, b) __fsub_rn((a), (b))
#define MVP_LDG(p) __ldg(p)
#else  // host build (tests/emul): compiled with -ffp-contract=off
#define MVP_MUL(a, b) ((a) * (b))
#define MVP_ADD(a, b) ((a) + (b))
#define MVP_SUB(a, b) ((a) - (b))
#define MVP_LDG(p) (*(p))
#endif

namespace mvp_epi {

// V consecutive floats of one NCHW plane (V = 1 or 4; the V = 4 form needs 16-byte alignment).
template <int V>
MVP_HD void load(const float *p, float (&v)[V]) {
    if constexpr (V == 4) {
        const float4 t = MVP_LDG(reinterpret_cast<const float4 *>(p));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
#pragma unroll
        for (int i = 0; i < V; ++i) v[i] = MVP_LDG(p + i);
    }
}
template <int V>
MVP_HD void store(float *p, const float (&v)[V]) {
    if constexpr (V == 4) {
        *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
        for (int i = 0; i < V; ++i) p[i] = v[i];
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Row 2: image epilogue.  rayrgba [N,H,W,4] -> irgbrec [N,3,H,W], rayalpha [N,1,H,W]
//   rayrgb = rayrgba[..., :3] as NCHW                                   models/raymarchers/mvpraymarcher.py:50-51
//   rayrgb = w * rayrgb + b   (w, b per view and channel)               models/colorcals/colorcal.py:26-29
//   irgbrec = rayrgb + (1 - rayalpha) * bg                              models/autoencoder.py:262-270
// ------------------------------------------------------------------------------------------------------------------
struct CompositeFwd {
    size_t HW;
    const float *rayrgba;   // [N,H,W,4]
    const float *ccw, *ccb; // [N,3] each, or both NULL (no colour calibration)
    const float *bg;        // [N,3,H,W] or NULL (black background)
    float *irgbrec;         // [N,3,H,W]
    float *rayalpha;        // [N,1,H,W] or NULL
};

template <int V>
MVP_HD void composite_fwd(const CompositeFwd &a, int n, size_t px) {
    float c[3][V], al[V];
    const float4 *in = reinterpret_cast<const float4 *>(a.rayrgba) + (size_t)n * a.HW + px;
#pragma unroll
    for (int v = 0; v < V; ++v) {
        const float4 t = MVP_LDG(in + v);
        c[0][v] = t.x; c[1][v] = t.y; c[2][v] = t.z; al[v] = t.w;
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const size_t plane = ((size_t)n * 3 + ch) * a.HW + px;
        if (a.ccw) {
            const float w = MVP_LDG(a.ccw + n * 3 + ch), b = MVP_LDG(a.ccb + n * 3 + ch);
#pragma unroll
            for (int v = 0; v < V; ++v) c[ch][v] = MVP_ADD(MVP_MUL(w, c[ch][v]), b);
        }
        if (a.bg) {
            float bgv[V];
            load<V>(a.bg + plane, bgv);
#pragma unroll
            for (int v = 0; v < V; ++v) c[ch][v] = MVP_ADD(c[ch][v], MVP_MUL(MVP_SUB(1.f, al[v]), bgv[v]));
        }
        store<V>(a.irgbrec + plane, c[ch]);
    }
    if (a.rayalpha) store<V>(a.rayalpha + (size_t)n * a.HW + px, al);
}

struct CompositeBwd {
    size_t HW;
    const float *rayrgba;       // [N,H,W,4]; read only when grad_bg or the colour-calibration gradients are wanted
    const float *ccw;           // [N,3] or NULL (w = 1)
    const float *bg;            // [N,3,H,W] or NULL
    const float *grad_irgbrec;  // [N,3,H,W]
    const float *grad_rayalpha; // [N,1,H,W] or NULL
    float *grad_rayrgba;        // [N,H,W,4] out (contiguous channels-last: what the raymarch backward wants)
    float *grad_bg;             // [N,3,H,W] out or NULL
    int want_cc;                // accumulate sum(rgb*g), sum(g) into part[0..2], part[3..5]
};

template <int V>
MVP_HD void composite_bwd(const CompositeBwd &a, int n, size_t px, float (&part)[6]) {
    float g[3][V], ga[V], rgb[3][V], al[V];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) load<V>(a.grad_irgbrec + ((size_t)n * 3 + ch) * a.HW + px, g[ch]);
    if (a.grad_rayalpha) {
        load<V>(a.grad_rayalpha + (size_t)n * a.HW + px, ga);
    } else {
#pragma unroll
        for (int v = 0; v < V; ++v) ga[v] = 0.f;
    }
    const bool need_in = a.want_cc || (a.bg && a.grad_bg);
    if (need_in) {
        const float4 *in = reinterpret_cast<const float4 *>(a.rayrgba) + (size_t)n * a.HW + px;
#pragma unroll
        for (int v = 0; v < V; ++v) {
            const float4 t = MVP_LDG(in + v);
            rgb[0][v] = t.x; rgb[1][v] = t.y; rgb[2][v] = t.z; al[v] = t.w;
        }
    } else {
#pragma unroll
        for (int v = 0; v < V; ++v) { rgb[0][v] = rgb[1][v] = rgb[2][v] = 0.f; al[v] = 0.f; }
    }
    if (a.bg) {
        float s[V];
#pragma unroll
        for (int v = 0; v < V; ++v) s[v] = 0.f;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const size_t plane = ((size_t)n * 3 + ch) * a.HW + px;
            float bgv[V];
            load<V>(a.bg + plane, bgv);
#pragma unroll
            for (int v = 0; v < V; ++v) s[v] = MVP_ADD(s[v], MVP_MUL(g[ch][v], bgv[v]));     // d/d(1-alpha), summed over channels
            if (a.grad_bg) {
                float gb[V];
#pragma unroll
                for (int v = 0; v < V; ++v) gb[v] = MVP_MUL(g[ch][v], MVP_SUB(1.f, al[v]));
                store<V>(a.grad_bg + plane, gb);
            }
        }
#pragma unroll
        for (int v = 0; v < V; ++v) ga[v] = MVP_SUB(ga[v], s[v]);
    }
    if (a.want_cc) {
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                part[ch] += rgb[ch][v] * g[ch][v];
                part[3 + ch] += g[ch][v];
            }
        }
    }
    float4 *out = reinterpret_cast<float4 *>(a.grad_rayrgba) + (size_t)n * a.HW + px;
    const float w0 = a.ccw ? MVP_LDG(a.ccw + n * 3 + 0) : 1.f, w1 = a.ccw ? MVP_LDG(a.ccw + n * 3 + 1) : 1.f,
                w2 = a.ccw ? MVP_LDG(a.ccw + n * 3 + 2) : 1.f;
#pragma unroll
    for (int v = 0; v < V; ++v) out[v] = make_float4(MVP_MUL(w0, g[0][v]), MVP_MUL(w1, g[1][v]), MVP_MUL(w2, g[2][v]), ga[v]);
}

// ------------------------------------------------------------------------------------------------------------------
// Row 4: payload hand-off.  The decoders emit two NCHW images per view,
//   tex     [N, B*3, hb*B, wb*B]   (channel = d*3 + c; row = i*B + y; col = j*B + x)   models/decoders/rgb.py:128-143
//   opacity [N, B,   hb*B, wb*B]   (channel = d)                                        models/decoders/geometry.py:180-185
// and the raymarcher wants channels-last slabs tplate [N, hb*wb, B, B, B, 4] with
//   tplate[n, i*wb+j, d, y, x, :3] = relu(tex * rgb_scale + rgb_bias),  [..., 3] = relu(opacity)
//                                                                                       models/decoders/assembler.py:261
// One element = V consecutive columns of one image row, enumerated in INPUT order (n, i, d, y, col) so the four plane
// reads of a warp are full contiguous lines; the matching writes are runs of B float4 (128 B at B = 8).
// ------------------------------------------------------------------------------------------------------------------
struct PayloadArgs {
    int32_t hb, wb, B;
    float rgb_scale, rgb_bias;
    const float *tex, *opacity; // forward in
    float *tplate;              // forward out (bf16 texels in the _bf16 bodies below, as are the next two)
    const float *tplate_in;     // backward in (relu mask)
    const float *grad_tplate;   // backward in
    float *grad_tex, *grad_opacity; // backward out
};

struct PayloadIndex {
    size_t tex_off;   // offset of channel c = 0 in tex (channel c adds c * plane)
    size_t opa_off;   // offset in opacity
    size_t slab_off;  // float4 index into tplate
    size_t plane;     // Himg * Wimg
};

template <int V, int BT>
MVP_HD PayloadIndex payload_index(const PayloadArgs &a, size_t e) {
    const size_t B = BT ? (size_t)BT : (size_t)a.B;
    const size_t Wimg = (size_t)a.wb * B, Himg = (size_t)a.hb * B;
    const size_t t = e * V;
    const size_t col = t % Wimg;
    size_t r = t / Wimg;
    const size_t y = r % B; r /= B;
    const size_t d = r % B; r /= B;
    const size_t i = r % (size_t)a.hb;
    const size_t n = r / (size_t)a.hb;
    const size_t row = i * B + y;
    const size_t j = col / B, x = col % B;
    PayloadIndex o;
    o.plane = Himg * Wimg;
    o.tex_off = ((n * 3 * B + d * 3) * Himg + row) * Wimg + col;
    o.opa_off = ((n * B + d) * Himg + row) * Wimg + col;
    o.slab_off = ((n * (size_t)a.hb + i) * (size_t)a.wb + j) * (B * B * B) + (d * B + y) * B + x;
    return o;
}

MVP_HD float relu_keep_nan(float x) { return x < 0.f ? 0.f : x; }

template <int V, int BT>
MVP_HD void payload_fwd(const PayloadArgs &a, size_t e) {
    const PayloadIndex ix = payload_index<V, BT>(a, e);
    float c0[V], c1[V], c2[V], o[V];
    load<V>(a.tex + ix.tex_off, c0);
    load<V>(a.tex + ix.tex_off + ix.plane, c1);
    load<V>(a.tex + ix.tex_off + 2 * ix.plane, c2);
    load<V>(a.opacity + ix.opa_off, o);
    float4 *out = reinterpret_cast<float4 *>(a.tplate) + ix.slab_off;
#pragma unroll
    for (int v = 0; v < V; ++v)
        out[v] = make_float4(relu_keep_nan(MVP_ADD(MVP_MUL(c0[v], a.rgb_scale), a.rgb_bias)),
                             relu_keep_nan(MVP_ADD(MVP_MUL(c1[v], a.rgb_scale), a.rgb_bias)),
                             relu_keep_nan(MVP_ADD(MVP_MUL(c2[v], a.rgb_scale), a.rgb_bias)), relu_keep_nan(o[v]));
}

template <int V, int BT>
MVP_HD void payload_bwd(const PayloadArgs &a, size_t e) {
    const PayloadIndex ix = payload_index<V, BT>(a, e);
    const float4 *tp = reinterpret_cast<const float4 *>(a.tplate_in) + ix.slab_off;
    const float4 *gp = reinterpret_cast<const float4 *>(a.grad_tplate) + ix.slab_off;
    float g0[V], g1[V], g2[V], go[V];
#pragma unroll
    for (int v = 0; v < V; ++v) {
        const float4 t = MVP_LDG(tp + v), g = MVP_LDG(gp + v);
        g0[v] = t.x > 0.f ? MVP_MUL(g.x, a.rgb_scale) : 0.f;   // relu' (threshold_backward), then d(tex*s+b)/dtex = s
        g1[v] = t.y > 0.f ? MVP_MUL(g.y, a.rgb_scale) : 0.f;
        g2[v] = t.z > 0.f ? MVP_MUL(g.z, a.rgb_scale) : 0.f;
        go[v] = t.w > 0.f ? g.w : 0.f;
    }
    store<V>(a.grad_tex + ix.tex_off, g0);
    store<V>(a.grad_tex + ix.tex_off + ix.plane, g1);
    store<V>(a.grad_tex + ix.tex_off + 2 * ix.plane, g2);
    store<V>(a.grad_opacity + ix.opa_off, go);
}

// ------------------------------------------------------------------------------------------------------------------
// bfloat16 forms (mvp_assemble_payload_*_bf16, mvp_sum_views_bf16).  A bf16 texel is 8 bytes, two 32-bit words holding
// channel pairs: word 0 = ch0 | ch1 << 16, word 1 = ch2 | ch3 << 16 (little endian: channel 0 first), the layout the
// render kernels read with MVP_FLAG_TPLATE_BF16.  The PayloadArgs pointers tplate / tplate_in / grad_tplate then point to
// bf16 data.
//   forward:  the fp32 arithmetic above unchanged, then each channel rounded once to bf16 (nearest even, subnormals kept,
//             NaN stays NaN): bit-identical to assemble_payload_ref(tex, opacity, B).to(torch.bfloat16).  16 B in + 8 B out
//             per texel.
//   backward: the bf16 gradient widened exactly, masked where the bf16 template is > 0, times rgb_scale (one fp32 rounding):
//             bit-identical to eager autograd through assemble_payload_ref(...).to(torch.bfloat16) for the same bf16 gradient,
//             with one exception.  An fp32 relu output in (0, 2^-134] rounds to bf16 +0 (half the smallest bf16 subnormal,
//             2^-133, ties to even), so the mask read from the bf16 template is 0 there while eager's, taken on the fp32 relu
//             output, is 1.  16 B in + 16 B out per texel.
// ------------------------------------------------------------------------------------------------------------------
MVP_HD float bits_to_float(uint32_t u) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}

// Two fp32 values as one bf16 pair, `lo` in the low half; each rounded to nearest even (cvt.rn.bf16x2.f32 on the device).
MVP_HD uint32_t pack_bf16x2(float lo, float hi) {
#ifdef __CUDA_ARCH__
    uint32_t d;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));   // first source -> upper half
    return d;
#else
    const auto rn = [](float x) -> uint32_t {
        uint32_t u;
        memcpy(&u, &x, 4);
        if ((u & 0x7fffffffu) > 0x7f800000u) return (u >> 16) | 0x40u;    // NaN: quiet, sign and top payload kept
        return (u + 0x7fffu + ((u >> 16) & 1u)) >> 16;
    };
    return rn(lo) | (rn(hi) << 16);
#endif
}
// Exact widening of the low / high bf16 of a pair.
MVP_HD float bf16_lo(uint32_t w) { return bits_to_float(w << 16); }
MVP_HD float bf16_hi(uint32_t w) { return bits_to_float(w & 0xffff0000u); }

// The 2V words of V consecutive bf16 texels (V = 4: two 16-byte accesses, 16-byte alignment; V = 1: one 8-byte access).
template <int V>
MVP_HD void load_words(const uint32_t *p, uint32_t (&w)[2 * V]) {
    if constexpr (V == 4) {
        const uint4 a = MVP_LDG(reinterpret_cast<const uint4 *>(p)), b = MVP_LDG(reinterpret_cast<const uint4 *>(p) + 1);
        w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
    } else {
        const uint2 a = MVP_LDG(reinterpret_cast<const uint2 *>(p));
        w[0] = a.x; w[1] = a.y;
    }
}
template <int V>
MVP_HD void store_words(uint32_t *p, const uint32_t (&w)[2 * V]) {
    if constexpr (V == 4) {
        reinterpret_cast<uint4 *>(p)[0] = make_uint4(w[0], w[1], w[2], w[3]);
        reinterpret_cast<uint4 *>(p)[1] = make_uint4(w[4], w[5], w[6], w[7]);
    } else {
        *reinterpret_cast<uint2 *>(p) = make_uint2(w[0], w[1]);
    }
}

template <int V, int BT>
MVP_HD void payload_fwd_bf16(const PayloadArgs &a, size_t e) {
    const PayloadIndex ix = payload_index<V, BT>(a, e);
    float c0[V], c1[V], c2[V], o[V];
    load<V>(a.tex + ix.tex_off, c0);
    load<V>(a.tex + ix.tex_off + ix.plane, c1);
    load<V>(a.tex + ix.tex_off + 2 * ix.plane, c2);
    load<V>(a.opacity + ix.opa_off, o);
    uint32_t w[2 * V];
#pragma unroll
    for (int v = 0; v < V; ++v) {
        w[2 * v] = pack_bf16x2(relu_keep_nan(MVP_ADD(MVP_MUL(c0[v], a.rgb_scale), a.rgb_bias)),
                               relu_keep_nan(MVP_ADD(MVP_MUL(c1[v], a.rgb_scale), a.rgb_bias)));
        w[2 * v + 1] = pack_bf16x2(relu_keep_nan(MVP_ADD(MVP_MUL(c2[v], a.rgb_scale), a.rgb_bias)), relu_keep_nan(o[v]));
    }
    store_words<V>(reinterpret_cast<uint32_t *>(a.tplate) + 2 * ix.slab_off, w);
}

template <int V, int BT>
MVP_HD void payload_bwd_bf16(const PayloadArgs &a, size_t e) {
    const PayloadIndex ix = payload_index<V, BT>(a, e);
    uint32_t t[2 * V], g[2 * V];
    load_words<V>(reinterpret_cast<const uint32_t *>(a.tplate_in) + 2 * ix.slab_off, t);
    load_words<V>(reinterpret_cast<const uint32_t *>(a.grad_tplate) + 2 * ix.slab_off, g);
    float g0[V], g1[V], g2[V], go[V];
#pragma unroll
    for (int v = 0; v < V; ++v) {
        const uint32_t t01 = t[2 * v], t23 = t[2 * v + 1], g01 = g[2 * v], g23 = g[2 * v + 1];
        g0[v] = bf16_lo(t01) > 0.f ? MVP_MUL(bf16_lo(g01), a.rgb_scale) : 0.f;
        g1[v] = bf16_hi(t01) > 0.f ? MVP_MUL(bf16_hi(g01), a.rgb_scale) : 0.f;
        g2[v] = bf16_lo(t23) > 0.f ? MVP_MUL(bf16_lo(g23), a.rgb_scale) : 0.f;
        go[v] = bf16_hi(t23) > 0.f ? bf16_hi(g23) : 0.f;
    }
    store<V>(a.grad_tex + ix.tex_off, g0);
    store<V>(a.grad_tex + ix.tex_off + ix.plane, g1);
    store<V>(a.grad_tex + ix.tex_off + 2 * ix.plane, g2);
    store<V>(a.grad_opacity + ix.opa_off, go);
}

}  // namespace mvp_epi
#endif  // MVP_EPILOGUE_BODY_H_
