// Persistent wgmma + TMA IMPLICIT-GEMM causal convolution (SURVEY.md row N1: Qwen3-TTS speech-tokenizer decoder).
//     D[m, (b, t)] = sum_j sum_c (Wh + Wl)[m, j, c] * (Xh + Xl)[b, t + shift0 + j * dil, c]
// Same machine as conv_gemm.cuh (fp32 weights and activations as bf16 hi/lo pairs, three tensor-core products, the
// 2^-18 Wl*Xl term dropped; four wgmma warpgroups that also run the epilogue, one TMA producer warp), with two
// differences that remove the im2col matrix the dense k7 / dilated convolutions would otherwise write and re-read
// (7x the activation bytes):
//   * activations live as PLANES  hl[2 (hi | lo)][B][Ttot][C]  (channels-last, bf16).  A 4-D tensor map with box
//     {64 channels, 64 frames, 1 row, 2 planes} lands in shared memory as the same 128-row x 128-byte SWIZZLE_128B
//     tile the MMA reads in conv_gemm.cuh (rows 0..63 = hi of 64 frames, rows 64..127 = lo), but its frame
//     coordinate is free: tap j of the convolution is the SAME tile shifted by j * dil frames, so the k-loop is
//     (tap, channel block) and the B operand is read straight from the activation planes.  Out-of-range frames /
//     channels are zero-filled by TMA (C = 96 uses two 64-channel blocks, the second half zeros on both operands).
//   * every consumer's input buffer starts with H = (k - 1) * dil HISTORY frames (zeros after a reset, the previous
//     chunk's last frames while streaming), so causal left padding and streaming state are the same thing and no
//     coordinate is ever negative.  The producing epilogue writes at frame offset Hout of its output buffer.
// Transposed convolutions with kernel = n * stride are the same kernel: rows m = rho * Cout + co hold phase rho of the
// kernel, the taps run over input frames q - (n - 1) .. q, and the epilogue writes output frame q * stride + rho
// ("pixel shuffle"); the reference's trim of (k - stride) frames on the right falls out of the causal form.
#pragma once
#include "common.cuh"
#include "tc_gemm.cuh"

#include <cuda_fp16.h>

namespace b2a {
namespace ic {

using namespace b2a::tc;

constexpr int BN = 128, HALF = 64;
constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE = 2 * A_BYTES + B_BYTES;   // 48 KB
constexpr int STAGES = 3;
constexpr int EPI_WARPS = 16;
constexpr int IC_THREADS = 32 * EPI_WARPS + 32;
constexpr int ACC_LD = BN + 4;                                     // row stride (floats) of the staged accumulator
// + an all-zero 64-row weight block: the warpgroups of the lo columns multiply it in place of Wl, so that every warpgroup issues
// the same wgmma sequence (a per-warpgroup branch around the second product serialises all wgmma issue)
constexpr int ZERO_BYTES = 64 * BK * 2;
constexpr size_t SMEM_BYTES = 1024 + (size_t)STAGES * STAGE + (size_t)BM * ACC_LD * 4 + ZERO_BYTES + 256;

struct Args {
    int M, m_tiles;               // weight rows (= up * Cout)
    int taps, cblocks, dil;       // k-blocks = taps * cblocks; weight column = (tap * cblocks + cb) * 64 + c
    int shift0;                   // frame coordinate of tap 0 for output frame 0 (0 when the input carries exactly H history frames)
    int B, T, t_tiles;            // GEMM tokens: B rows x T frames, 64 frames per tile
    int Cout, up;                 // m = rho * Cout + co ; output frame = t * up + rho ; To = T * up
    const float* bias;            // [Cout] or null
    const float* gamma;           // [Cout] or null: scale applied to (acc + bias) (ConvNeXt gamma, transformer layer scale)
    int gelu;                     // exact-erf GELU on (acc + bias)
    int add;                      // xo += value (residual) instead of xo = value
    int bias_twice_t0;            // reference streaming behaviour: frames produced by input frame 0 of a non-first chunk get the bias twice
    float* xo;                    // fp32 [B, To, Cout] or null
    __nv_bfloat16* hl;            // planar hi/lo output [2][B][Hout + To][Cout] or null
    int Hout;
    int f16;                      // operands (weights and planes) are fp16 hi/lo pairs instead of bf16 ones: same three products and cost, 22
                                  // instead of 16 mantissa bits per operand (shipped decoder geometry, 6 frames: 2.7e-4 of the peak instead of
                                  // 7.0e-4); values saturate at 65504
    const float* wscale;          // [M] or null: the accumulator of row m is multiplied by wscale[m] (fp16 operands: weight rows are stored
                                  // times a power of two so that their lo halves are NORMAL fp16 numbers, not subnormals)
    int seg_kb;                   // k-blocks accumulated per tensor-core accumulation before the epilogue adds it into its fp32
                                  // running sum (0 = all).  A tensor core that truncates its fp32 accumulation biases a long
                                  // contraction systematically (tools/probe_n1_dec0.py measures it); segments added in registers with
                                  // round-to-nearest bound that bias.
    const float* sa;              // SnakeBeta on the hi/lo copy: v + sb * sin^2(sa * v), sa = exp(alpha), sb = 1 / (exp(beta) + 1e-9)
    const float* sb;
};

__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
// v -> hi + lo in the operand format, stored as raw 16-bit words at idx and plane + idx
__device__ __forceinline__ void put_hilo16(uint16_t* base, long long plane, long long idx, float v, int f16) {
    if (f16) {
        v = fminf(fmaxf(v, -65504.f), 65504.f);      // saturate instead of producing inf (fp16 range)
        const __half hi = __float2half_rn(v);
        base[idx] = __half_as_ushort(hi);
        base[plane + idx] = __half_as_ushort(__float2half_rn(v - __half2float(hi)));
    } else {
        const __nv_bfloat16 hi = __float2bfloat16_rn(v);
        base[idx] = __bfloat16_as_ushort(hi);
        base[plane + idx] = __bfloat16_as_ushort(__float2bfloat16_rn(v - __bfloat162float(hi)));
    }
}
__device__ __forceinline__ float snake_beta(float v, float a, float ib) {
    const float s = fast_sin(a * v);      // (a precise sinf changes nothing measurable: the error budget is elsewhere, DESIGN.md 3.8)
    return fmaf(ib * s, s, v);
}

template <int F16>   // == Args::f16 (a template parameter so that the wgmma issue has no branch)
static __global__ void __launch_bounds__(IC_THREADS, 1)
implicit_conv_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                     const __grid_constant__ CUtensorMap tmB, Args a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    float* sacc = reinterpret_cast<float*>(smem + (size_t)STAGES * STAGE);                     // [128][ACC_LD]
    uint8_t* zero_w = reinterpret_cast<uint8_t*>(sacc + (size_t)BM * ACC_LD);                  // [64][64] bf16 zeros (1024-aligned)
    uint64_t* full = reinterpret_cast<uint64_t*>(zero_w + ZERO_BYTES);
    uint64_t* empty = full + STAGES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmA2); tma_prefetch_desc(&tmB);
        for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], EPI_WARPS); }
        fence_barrier_init();
    }
    for (int i = threadIdx.x; i < ZERO_BYTES / 16; i += blockDim.x) reinterpret_cast<uint4*>(zero_w)[i] = make_uint4(0, 0, 0, 0);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy stores -> visible to the tensor core
    __syncthreads();
    const int k_blocks = a.taps * a.cblocks;
    const long long tiles = (long long)a.B * a.t_tiles * a.m_tiles;   // tile id = n_tile * m_tiles + m_tile, n_tile = b * t_tiles + tt

    if (warp == EPI_WARPS) {
        if (lane == 0) {
            int stage = 0; uint32_t phase = 0;
            for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
                const int nt = (int)(t / a.m_tiles), mt = (int)(t - (long long)nt * a.m_tiles);
                const int b = nt / a.t_tiles, tt = nt - b * a.t_tiles;
                int kb = 0;
                for (int j = 0; j < a.taps; ++j) {
                    const int frame = tt * HALF + a.shift0 + j * a.dil;
                    for (int cb = 0; cb < a.cblocks; ++cb, ++kb) {
                        mbar_wait(&empty[stage], phase ^ 1);
                        uint8_t* s0 = smem + (size_t)stage * STAGE;
                        mbar_arrive_expect_tx(&full[stage], STAGE);
                        tma_load_2d(s0, &tmA, &full[stage], kb * BK, mt * BM);
                        tma_load_2d(s0 + A_BYTES, &tmA2, &full[stage], kb * BK, mt * BM);
                        tma_load_4d(s0 + 2 * A_BYTES, &tmB, &full[stage], cb * BK, frame, b, 0);
                        if (++stage == STAGES) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
    } else {
        const int q = warp & 3, c0 = (warp >> 2) * 16;
        const int wg = warp >> 2, row_blk = wg & 1, col_blk = wg >> 1;   // this warpgroup's 64 x 64 block of the accumulator
        auto wgmma16 = [&](float (&d)[32], uint64_t da, uint64_t db, uint32_t sc) {
            if constexpr (F16) wgmma_f16_n64(d, da, db, sc); else wgmma_bf16_n64(d, da, db, sc);
        };
        const float* arow = sacc + (size_t)(q * 32 + lane) * ACC_LD;
        const uint64_t zero_desc = make_smem_desc(smem_u32(zero_w));
        int stage = 0; uint32_t phase = 0;
        float acc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = 0.f;
        // acc = Wh * X  over this block (+ Wl * Xh for the hi columns), k-blocks [kb0, kb1); then staged in sacc
        auto mma_block = [&](int kb0, int kb1) {
            for (int kb = kb0; kb < kb1; ++kb) {
                mbar_wait(&full[stage], phase);
                const uint32_t s0 = smem_u32(smem + (size_t)stage * STAGE);
                const uint64_t ad = make_smem_desc(s0 + (uint32_t)(row_blk * 64 * 128)), a2d = col_blk == 0 ? make_smem_desc(s0 + A_BYTES + (uint32_t)(row_blk * 64 * 128)) : zero_desc;
                const uint64_t bd = make_smem_desc(s0 + 2 * A_BYTES + (uint32_t)(col_blk * 64 * 128));
                wg_fence();
#pragma unroll
                for (int k = 0; k < BK / UMMA_K; ++k) {
                    const uint64_t off = (uint64_t)(2 * k);
                    wgmma16(acc, ad + off, bd + off, (kb == kb0 && k == 0) ? 0u : 1u);     // Wh * [Xh; Xl]
                    wgmma16(acc, a2d + (col_blk == 0 ? off : 0), bd + off, 1u);          // Wl * Xh -> columns [0, 64) (else + 0)
                }
                wg_commit();
                wg_wait0();
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[stage]);
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            wg_fence_operand(acc);
            named_sync(1, 32 * EPI_WARPS);                        // the previous epilogue has read sacc
            store_frag<64>(sacc, ACC_LD, acc, row_blk * 64, col_blk * 64);
            named_sync(1, 32 * EPI_WARPS);
        };
        const long long To = (long long)a.T * a.up;
        const long long plane = (long long)a.B * (a.Hout + To) * a.Cout;
        for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
            const int nt = (int)(t / a.m_tiles), mt = (int)(t - (long long)nt * a.m_tiles);
            const int b = nt / a.t_tiles, tt = nt - b * a.t_tiles;
            const int m = mt * BM + q * 32 + lane;
            const bool m_ok = m < a.M;
            int rho = 0, co = m;
            if (a.up > 1) { rho = m / a.Cout; co = m - rho * a.Cout; }
            float bias = 0.f, gm = 1.f, sa = 0.f, sb = 0.f, ws = 1.f;
            if (m_ok) {
                if (a.wscale) ws = a.wscale[m];
                if (a.bias) bias = a.bias[co];
                if (a.gamma) gm = a.gamma[co];
                if (a.sa) { sa = a.sa[co]; sb = a.sb[co]; }
            }
            const int t_first = tt * HALF + c0;
            // the residual operand does not depend on the accumulator: 16 independent loads issued before the MMA wait
            float xv[16];
            if (a.add) {
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int tf = t_first + j;
                    xv[j] = (m_ok && tf < a.T) ? a.xo[((long long)b * To + (long long)tf * a.up + rho) * a.Cout + co] : 0.f;
                }
            }
            float sum[16];
            const int seg = a.seg_kb > 0 ? a.seg_kb : k_blocks;
            for (int kb0 = 0; kb0 < k_blocks; kb0 += seg) {              // drain every segment's accumulator, add in registers (RN)
                mma_block(kb0, min(k_blocks, kb0 + seg));
                float v[16], w[16];
                ld_acc16(arow + c0, v);
                ld_acc16(arow + c0 + HALF, w);
                if (kb0 == 0) {
#pragma unroll
                    for (int j = 0; j < 16; ++j) sum[j] = v[j] + w[j];
                } else {
#pragma unroll
                    for (int j = 0; j < 16; ++j) sum[j] += v[j] + w[j];
                }
            }
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int tf = t_first + j;
                if (tf >= a.T || !m_ok) continue;
                float val = sum[j] * ws + bias;
                if (a.bias_twice_t0 && tf == 0) val += bias;
                if (a.gelu) val = 0.5f * val * (1.0f + erff(val * 0.70710678118654752f));
                val *= gm;
                if (a.add) val += xv[j];
                const long long fo = (long long)tf * a.up + rho;
                if (a.xo) a.xo[((long long)b * To + fo) * a.Cout + co] = val;
                if (a.hl) {
                    const float hv = a.sa ? snake_beta(val, sa, sb) : val;
                    const long long idx = ((long long)b * (a.Hout + To) + a.Hout + fo) * a.Cout + co;
                    put_hilo16(reinterpret_cast<uint16_t*>(a.hl), plane, idx, hv, a.f16);
                }
            }
        }
    }
}

}  // namespace ic
}  // namespace b2a
