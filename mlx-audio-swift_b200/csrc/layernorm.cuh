// (optional depthwise conv k over time) -> LayerNorm(eps) over channels, channels-last fp32 in, fp32 and / or bf16 hi/lo
// GEMM-operand rows out.  Used by Vocos (ConvNeXt blocks, MAXV = 4) and by SNAC's LocalMHA (MAXV = 8).
#pragma once
#include "common.cuh"
#include "conv_gemm.cuh"

namespace b2a {

// One CTA per token, one thread per channel slot: C <= DL_THREADS * MAXV.
// out_f32 (nullable): normalised row as fp32 (residual stream) ; out_hl (nullable): hi/lo tiles (GEMM input).
constexpr int DL_THREADS = 256;
template <int MAXV>
__global__ void __launch_bounds__(DL_THREADS)
dw_layernorm_kernel(const float* __restrict__ x, const float* __restrict__ dw_w /*[C,k] or null*/, const float* __restrict__ dw_b,
                    const float* __restrict__ ln_w, const float* __restrict__ ln_b, float* __restrict__ out_f32,
                    __nv_bfloat16* __restrict__ out_hl, int L, int C, int k, float eps, int ln_batch_stride = 0) {
    __shared__ float red[DL_THREADS / 32];
    const long long tok = blockIdx.x;
    const int b = (int)(tok / L), t = (int)(tok - (long long)b * L);
    ln_w += (long long)b * ln_batch_stride;     // AdaLayerNorm: the gain / shift rows of this utterance's conditioning (0 = shared LayerNorm)
    ln_b += (long long)b * ln_batch_stride;
    float v[MAXV];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
        const int c = threadIdx.x + j * DL_THREADS;
        float val = 0.f;
        if (c < C) {
            if (dw_w) {
                val = dw_b ? dw_b[c] : 0.f;
                for (int kk = 0; kk < k; ++kk) {
                    const int ti = t + kk - k / 2;
                    if (ti >= 0 && ti < L) val = fmaf(dw_w[c * k + kk], x[((long long)b * L + ti) * C + c], val);
                }
            } else {
                val = x[tok * C + c];
            }
        }
        v[j] = val;
        s += val;
    }
    const float mean = block_sum<DL_THREADS>(s, red) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
        const int c = threadIdx.x + j * DL_THREADS;
        if (c < C) { const float d = v[j] - mean; q += d * d; }
    }
    const float r = rsqrtf(block_sum<DL_THREADS>(q, red) / (float)C + eps);
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
        const int c = threadIdx.x + j * DL_THREADS;
        if (c < C) {
            const float o = (v[j] - mean) * r * ln_w[c] + ln_b[c];
            if (out_f32) out_f32[tok * C + c] = o;
            if (out_hl) tc::store_hilo(out_hl, C, tok, c, o, cg::HALF);
        }
    }
}

}  // namespace b2a
