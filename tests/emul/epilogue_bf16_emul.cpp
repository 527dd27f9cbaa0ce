// TEST INFRASTRUCTURE.  Host build of the bfloat16 payload bodies in ava-256_b200/csrc/epilogue_body.h (payload_fwd_bf16,
// payload_bwd_bf16): the same inline functions the CUDA kernels call, driven by plain loops in place of the grid, so the
// rounding, the pair layout and the relu mask can be checked against PyTorch on a machine without a GPU.  Never loaded by
// the product.  tplate / grad_tplate hold bf16 texels (4 x uint16 each).
// Build: g++ -std=c++17 -O1 -ffp-contract=off -shared -fPIC -I/usr/local/cuda/include -I<repo>/ava-256_b200/csrc
// (tests/test_emul_bf16_handoff.py compiles it into a temporary directory)
#include "epilogue_body.h"

using namespace mvp_epi;

extern "C" {

static size_t payload_total(int N, int hb, int wb, int B, int V) { return (size_t)N * hb * B * B * ((size_t)wb * B) / V; }

int emul_payload_forward_bf16(int N, int hb, int wb, int B, int V, int BT, const float *tex, const float *opacity, float rgb_scale,
                              float rgb_bias, void *tplate) {
    PayloadArgs a = {};
    a.hb = hb; a.wb = wb; a.B = B; a.rgb_scale = rgb_scale; a.rgb_bias = rgb_bias; a.tex = tex; a.opacity = opacity;
    a.tplate = static_cast<float *>(tplate);
    if ((V == 4 && B % 4) || (BT && BT != B)) return -1;
    const size_t total = payload_total(N, hb, wb, B, V);
    for (size_t e = 0; e < total; ++e) {
        if (V == 4 && BT == 8) payload_fwd_bf16<4, 8>(a, e);
        else if (V == 4) payload_fwd_bf16<4, 0>(a, e);
        else payload_fwd_bf16<1, 0>(a, e);
    }
    return 0;
}

int emul_payload_backward_bf16(int N, int hb, int wb, int B, int V, int BT, const void *tplate, const void *grad_tplate,
                               float rgb_scale, float *grad_tex, float *grad_opacity) {
    PayloadArgs a = {};
    a.hb = hb; a.wb = wb; a.B = B; a.rgb_scale = rgb_scale; a.tplate_in = static_cast<const float *>(tplate);
    a.grad_tplate = static_cast<const float *>(grad_tplate); a.grad_tex = grad_tex; a.grad_opacity = grad_opacity;
    if ((V == 4 && B % 4) || (BT && BT != B)) return -1;
    const size_t total = payload_total(N, hb, wb, B, V);
    for (size_t e = 0; e < total; ++e) {
        if (V == 4 && BT == 8) payload_bwd_bf16<4, 8>(a, e);
        else if (V == 4) payload_bwd_bf16<4, 0>(a, e);
        else payload_bwd_bf16<1, 0>(a, e);
    }
    return 0;
}

}  // extern "C"
