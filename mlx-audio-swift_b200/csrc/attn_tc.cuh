// Non-causal multi-head attention on wgmma for sm_90a (head_dim 64): the Whisper encoder's 1500 x 1500 maps
// (Sources/MLXAudioSTT/Models/Whisper/WhisperLayers.swift:11-73, MLXFast.scaledDotProductAttention there).
//
// Operands: plain fp16, ONE tensor-core product per GEMM (a CPU study of the oracle with this arithmetic emulated,
// tools/whisper_attention_precision_study.py, keeps the encoder output within 5e-5: scores and probabilities do not need the
// hi/lo pairs the weight GEMMs use); softmax in fp32.
//   Qh [B*nh][Tp][64] fp16, pre-scaled by head_dim^-1/2 (a power of two here: exact)      -> A operand of  S = Q K^T
//   Kh [B*nh][Tp][64] fp16                                                                 -> B operand (K-major: d contiguous)
//   Vt [B*nh][64][Tp] fp16 (transposed so that keys are contiguous)                        -> B operand of  O = P V
//   rows / keys >= T are zero padding up to Tp (a multiple of 128)
// One CTA per (128-query tile, head, clip); 288 threads: warps 0-7 = two consumer warpgroups (64 query rows each: S = Q K^T into
// registers, softmax on the fragments, O += P V with P as the register A operand), warp 8 = TMA producer (2-stage K / V ring).
// Two passes over the keys instead of an online softmax: pass 1 only takes the row maxima of S, pass 2 recomputes S, forms
// P = exp(S - max) in fp16 and accumulates O += P V with no rescaling of O.
#pragma once
#include "tc_gemm.cuh"

#include <cuda_fp16.h>

namespace b2a {
namespace fa {

constexpr int BQ = 128, BKV = 128, HDIM = 64;
constexpr int FA_THREADS = 288;                   // two consumer warpgroups + one producer warp
constexpr int Q_BYTES = BQ * HDIM * 2, K_BYTES = BKV * HDIM * 2, V_BYTES = HDIM * BKV * 2;
constexpr int STAGE_BYTES = K_BYTES + V_BYTES, FA_STAGES = 2;
constexpr int SMEM_DATA = Q_BYTES + FA_STAGES * STAGE_BYTES;                // 80 KB
constexpr size_t FA_SMEM_BYTES = SMEM_DATA + 256 + 1024;                   // + barriers + alignment slack

struct Args {
    __nv_bfloat16* out;      // [2 * Tp_tokens, d_model] hi/lo tiles of `half` tokens (the out-projection GEMM's B operand)
    int T, Tp, nh, d_model, half;
};

__global__ void __launch_bounds__(FA_THREADS, 1)
mha_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV, Args a) {
    extern __shared__ __align__(1024) uint8_t fa_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(fa_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* sQ = smem;
    uint8_t* sKV = sQ + Q_BYTES;                                   // [stage][K 16 KB | V^T 16 KB]
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SMEM_DATA);
    uint64_t *qfull = bars, *full = bars + 1, *empty = bars + 3;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z, bh = b * a.nh + h;
    const int n_kv = a.Tp / BKV, n_it = 2 * n_kv;
    if (threadIdx.x == 0) {
        tc::tma_prefetch_desc(&tmQ); tc::tma_prefetch_desc(&tmK); tc::tma_prefetch_desc(&tmV);
        tc::mbar_init(qfull, 1);
        for (int i = 0; i < FA_STAGES; ++i) { tc::mbar_init(&full[i], 1); tc::mbar_init(&empty[i], 8); }
        tc::fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            tc::mbar_arrive_expect_tx(qfull, Q_BYTES);
            tc::tma_load_3d(sQ, &tmQ, qfull, 0, qt * BQ, bh);
            for (int i = 0; i < n_it; ++i) {
                const int j = i % n_kv, pass = i / n_kv, st = i % FA_STAGES;
                const uint32_t ph = (uint32_t)((i / FA_STAGES) & 1);
                tc::mbar_wait(&empty[st], ph ^ 1);
                uint8_t* sk = sKV + (size_t)st * STAGE_BYTES;
                tc::mbar_arrive_expect_tx(&full[st], pass ? STAGE_BYTES : K_BYTES);
                tc::tma_load_3d(sk, &tmK, &full[st], 0, j * BKV, bh);
                if (pass) {
                    tc::tma_load_3d(sk + K_BYTES, &tmV, &full[st], j * BKV, 0, bh);                 // keys [0, 64) of the tile: [64 d][64 keys]
                    tc::tma_load_3d(sk + K_BYTES + V_BYTES / 2, &tmV, &full[st], j * BKV + 64, 0, bh);
                }
            }
        }
        return;
    }
    // consumer warpgroup wg: query rows 64 wg .. 64 wg + 63.  Fragment of an m64nN accumulator: this thread holds rows
    // r0 = 16 (warp % 4) + lane / 4 and r0 + 8, columns 8 i + 2 (lane % 4) (+1) in registers 4 i (+1) and 4 i + 2 (+1).
    const int wg = warp >> 2;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c_lane = 2 * (lane & 3);
    tc::mbar_wait(qfull, 0);
    const uint64_t dq = tc::make_smem_desc(tc::smem_u32(sQ) + (uint32_t)(wg * 64 * 128));
    float mx[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float o[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) o[e] = 0.f;
    for (int i = 0; i < n_it; ++i) {
        const int j = i % n_kv, pass = i / n_kv, st = i % FA_STAGES;
        tc::mbar_wait(&full[st], (uint32_t)((i / FA_STAGES) & 1));
        const uint32_t sk = tc::smem_u32(sKV + (size_t)st * STAGE_BYTES);
        const uint64_t dk = tc::make_smem_desc(sk);
        float s[64];
#pragma unroll
        for (int e = 0; e < 64; ++e) s[e] = 0.f;
        tc::wg_fence();
#pragma unroll
        for (int k = 0; k < HDIM / 16; ++k) tc::wgmma_f16_n128(s, dq + (uint64_t)(2 * k), dk + (uint64_t)(2 * k), k ? 1u : 0u);
        tc::wg_commit();
        tc::wg_wait0();
        tc::wg_fence_operand(s);
        if (!pass) {
#pragma unroll
            for (int g = 0; g < 16; ++g)
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    if (j * BKV + 8 * g + c_lane + (e & 1) < a.T) mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * g + e]);
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(&empty[st]);
            if (i == n_kv - 1) {                                  // pass 1 done: the four lanes of a quad share a row
#pragma unroll
                for (int rh = 0; rh < 2; ++rh) {
                    mx[rh] = fmaxf(mx[rh], __shfl_xor_sync(0xffffffffu, mx[rh], 1));
                    mx[rh] = fmaxf(mx[rh], __shfl_xor_sync(0xffffffffu, mx[rh], 2));
                }
            }
            continue;
        }
        // P = exp(S - max) as fp16 A fragments: k-step kk (keys 16 kk .. + 15) = column groups 2 kk, 2 kk + 1;
        // register order {row r0 / keys 0-7, row r0 + 8 / keys 0-7, row r0 / keys 8-15, row r0 + 8 / keys 8-15}
        uint32_t pa[8][4];
#pragma unroll
        for (int g = 0; g < 16; ++g) {
#pragma unroll
            for (int rh = 0; rh < 2; ++rh) {
                const int key = j * BKV + 8 * g + c_lane;
                const float p0 = key < a.T ? __expf(s[4 * g + 2 * rh] - mx[rh]) : 0.f;
                const float p1 = key + 1 < a.T ? __expf(s[4 * g + 2 * rh + 1] - mx[rh]) : 0.f;
                const __half2 hp = __floats2half2_rn(p0, p1);
                l[rh] += __low2float(hp) + __high2float(hp);       // the sum of what the tensor core will actually multiply
                pa[g >> 1][(g & 1) * 2 + rh] = *reinterpret_cast<const uint32_t*>(&hp);
            }
        }
        tc::wg_fence();
#pragma unroll
        for (int kk = 0; kk < BKV / 16; ++kk) {
            const uint64_t dv = tc::make_smem_desc(sk + K_BYTES + (uint32_t)((kk >> 2) * (V_BYTES / 2))) + (uint64_t)(2 * (kk & 3));
            tc::wgmma_f16_rs_n64(o, pa[kk], dv, 1u);
        }
        tc::wg_commit();
        tc::wg_wait0();
        tc::wg_fence_operand(o);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&empty[st]);
    }
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
        l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 1);
        l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 2);
    }
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
        const int qrow = qt * BQ + r0 + 8 * rh;
        if (qrow >= a.T) continue;
        const float inv = 1.0f / l[rh];
        const long long tok = (long long)b * a.T + qrow;
        const long long r = (tok / a.half) * 2 * a.half + (tok % a.half);
        __nv_bfloat16* ph = a.out + r * a.d_model + h * HDIM + c_lane;
        __nv_bfloat16* pl = ph + (long long)a.half * a.d_model;
#pragma unroll
        for (int g = 0; g < 8; ++g) {
            const float o0 = o[4 * g + 2 * rh] * inv, o1 = o[4 * g + 2 * rh + 1] * inv;
            const __nv_bfloat16 h0 = __float2bfloat16_rn(o0), h1 = __float2bfloat16_rn(o1);
            *reinterpret_cast<__nv_bfloat162*>(ph + 8 * g) = __halves2bfloat162(h0, h1);
            *reinterpret_cast<__nv_bfloat162*>(pl + 8 * g) =
                __halves2bfloat162(__float2bfloat16_rn(o0 - __bfloat162float(h0)), __float2bfloat16_rn(o1 - __bfloat162float(h1)));
        }
    }
}

// qkv fp32 [B*T, 3 * d_model] (q | k | v) -> Qh (scaled), Kh, Vt.  One CTA per (64-token tile, clip, head); V goes through shared memory
// so that the transposed rows are written 128 bytes at a time.
__global__ void __launch_bounds__(256)
pack_qkv_f16_kernel(const float* __restrict__ qkv, __half* __restrict__ Qh, __half* __restrict__ Kh, __half* __restrict__ Vt, int T, int Tp,
                    int nh, float scale) {
    __shared__ __half sv[64][HDIM + 2];
    const int b = blockIdx.y, h = blockIdx.z, t0 = blockIdx.x * 64, dm = nh * HDIM;
    for (int i = threadIdx.x; i < 64 * HDIM; i += 256) {
        const int r = i >> 6, c = i & 63, t = t0 + r;
        float q = 0.f, k = 0.f, v = 0.f;
        if (t < T) {
            const float* src = qkv + ((long long)b * T + t) * 3 * dm + h * HDIM + c;
            q = src[0] * scale; k = src[dm]; v = src[2 * dm];
        }
        const long long o = (((long long)b * nh + h) * Tp + t) * HDIM + c;
        Qh[o] = __float2half_rn(q);
        Kh[o] = __float2half_rn(k);
        sv[r][c] = __float2half_rn(v);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 64 * HDIM; i += 256) {
        const int c = i >> 6, r = i & 63;                       // d = c, token = t0 + r: consecutive threads -> consecutive tokens
        Vt[(((long long)b * nh + h) * HDIM + c) * Tp + t0 + r] = sv[r][c];
    }
}

}  // namespace fa
}  // namespace b2a
