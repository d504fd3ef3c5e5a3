// Persistent wgmma + TMA GEMM for the codec path (SNAC in channels-last layout):
//     D[M, N] = (Wh + Wl)[M, K] * (Xh + Xl)[N, K]^T      fp32 weights and activations as bf16 hi/lo pairs
// A  = weights, TWO K-major operands (hi and lo halves of the fp32 weight, 16 mantissa bits together)
// B  = activations [tokens, channels] (NLC), 128-row tiles = 64 tokens as hi rows | lo rows (same layout as tc_gemm)
// per k-block:  D[:, 0:128] += Wh * [Xh; Xl]   and   D[:, 0:64] += Wl * Xh        (Wl*Xl, 2^-18 relative, is dropped)
// so the result equals the fp32 convolution to ~1e-5.  One CTA per SM loops over (token tile, m tile) work items;
// the TMA ring never drains between tiles.  The epilogue warps fuse what the reference runs as separate MLX ops:
// bias, Snake, residual add, NoiseBlock, the transposed-conv phase scatter, and the hi/lo re-split that feeds the
// next GEMM (optionally written twice, shifted by one token, which is the im2col the 2-tap transposed conv needs).
#pragma once
#include "tc_gemm.cuh"

namespace b2a {
namespace cg {

using namespace b2a::tc;

constexpr int BN = 128, HALF = 64;
constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE = 2 * A_BYTES + B_BYTES;   // 48 KB
constexpr int STAGES = 3;
// warps 0..15: four wgmma warpgroups + epilogue, warp 16: TMA producer.  Warpgroup g accumulates rows 64 (g % 2) .. + 63 and
// columns 64 (g / 2) .. + 63 of the 128 x 128 tile; the tile is staged in shared memory and warp w's epilogue takes rows
// 32 (w % 4) .. + 31 and the 16-token column group w / 4.  Sixteen epilogue warps = four per scheduler: the epilogue math
// (Snake, GELU, hi/lo split) is dependent-issue latency bound with one warp per scheduler.
constexpr int EPI_WARPS = 16;
constexpr int CG_THREADS = 32 * EPI_WARPS + 32;
constexpr int ACC_LD = BN + 4;                                     // row stride (floats) of the staged accumulator
// + an all-zero 64-row weight block: the warpgroups of the lo columns multiply it in place of Wl, so that every warpgroup issues
// the same wgmma sequence (a per-warpgroup branch around the second product serialises all wgmma issue)
constexpr int ZERO_BYTES = 64 * BK * 2;
constexpr size_t SMEM_BYTES = 1024 + (size_t)STAGES * STAGE + (size_t)BM * ACC_LD * 4 + ZERO_BYTES + 256;

enum : int { E_STORE_HILO = 0, E_CONVT = 1, E_NOISE = 2, E_ADD = 3, E_ADD_HILO = 4, E_STORE_F32 = 5 };

struct Args {
    int M, K, N;              // N = tokens (rows of X)
    int m_tiles, k_blocks, n_tiles;
    int epi;
    const float* bias;        // [channels] (E_CONVT: per output channel co) or null
    const float* alpha;       // Snake alpha applied to values written as hi/lo (null = identity)
    const float* gamma;       // nullable per-channel scale applied to (acc + bias) before any add (ConvNeXt layer scale)
    int gelu;                 // exact-erf GELU on (acc + bias) (Vocos pwconv1)
    float* x;                 // fp32 [tokens, ldx] read-modify-write target (E_NOISE / E_ADD / E_ADD_HILO) or E_CONVT output
    int ldx;
    __nv_bfloat16* hl;        // hi/lo output matrix (64-token tiles), leading dimension ldh
    int ldh;
    int dual;                 // hi/lo output is the 2-tap im2col of the next transposed conv:
                              //   token (b, t) -> row b*(T+1)+t cols [m], and row b*(T+1)+t+1 cols [M + m]
    int T;                    // tokens per utterance on the OUTPUT side of this GEMM (for dual / noise / convT / frames)
    int fs, fpad;             // fs > 0: the hi/lo output is the 2-frame im2col of a strided conv (kernel 2 fs, stride fs, left
                              //   pad fpad) over utterances of T tokens, laid out by put_frames (replaces dual)
    // E_CONVT: rows m = r*Cout + co; input token n = b*(Tin+1) + q  ->  t_out = q*stride + r - pad
    int Cout, stride, pad, Tin;
    // E_NOISE: x = x + noise[b, t] * acc      (NoiseBlock, Layers.swift:271-278)
    const float* noise;       // [B, T] or null => counter-based N(0,1) from seed
    unsigned long long seed;
};

// sin with an explicit two-term 2*pi range reduction + MUFU.SIN: |error| < 5e-7 for |x| < 1e4 (the libdevice sinf slow
// path costs ~40 dependent instructions per call and made every Snake epilogue issue bound)
__device__ __forceinline__ float fast_sin(float x) {
    const float k = rintf(x * 0.15915494309189535f);
    float r = fmaf(k, -6.28318548202514648f, x);
    r = fmaf(k, 1.7484555e-7f, r);
    return __sinf(r);
}
__device__ __forceinline__ float snake(float v, float al) {
    const float s = fast_sin(al * v);
    return v + (1.0f / (al + 1e-9f)) * s * s;
}
// same with the per-channel 1 / (alpha + 1e-9) computed once by the caller
__device__ __forceinline__ float snake_inv(float v, float al, float inv) {
    const float s = fast_sin(al * v);
    return fmaf(inv * s, s, v);
}
__device__ __forceinline__ float gauss(unsigned long long seed, unsigned long long idx) {
    unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (idx + 1);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    const float u1 = ((unsigned)(z >> 40) + 1.0f) * (1.0f / 16777217.0f);
    const float u2 = (unsigned)((z >> 8) & 0xFFFFFF) * (1.0f / 16777216.0f);
    return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}
__device__ __forceinline__ void put_hilo(__nv_bfloat16* base, long long ld, long long tok, long long col, float v) {
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    const long long r = (tok / HALF) * BN + (tok % HALF);
    base[r * ld + col] = hi;
    base[(r + HALF) * ld + col] = __float2bfloat16_rn(v - __bfloat162float(hi));
}
// Input of a strided conv (kernel 2 fs, stride fs, left pad fpad < fs) over utterances of T tokens (T % fs == 0) as a 2-tap GEMM
// operand: the zero-padded sequence is cut into frames of fs tokens x C channels; output token q reads frames q and q + 1, so row
// b (T / fs + 1) + q holds frame q in columns [0, fs C) and frame q + 1 in [fs C, 2 fs C) (row q = T / fs is computed and dropped).
// Token (b, t) is padded position p = t + fpad of frame f = p / fs: it lands in row f (first half) and in row f - 1 (second half).
__device__ __forceinline__ void put_frames(__nv_bfloat16* hl, int fs, int fpad, int C, int T, long long b, int t, int c, float v) {
    const int p = t + fpad, f = p / fs, col = (p - f * fs) * C + c;
    const long long ld = 2ll * fs * C, row = b * (T / fs + 1) + f;
    put_hilo(hl, ld, row, col, v);
    if (f > 0) put_hilo(hl, ld, row - 1, (long long)fs * C + col, v);
}

static __global__ void __launch_bounds__(CG_THREADS, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
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
    const long long tiles = (long long)a.n_tiles * a.m_tiles;   // tile id = n_tile * m_tiles + m_tile, dealt round-robin

    if (warp == EPI_WARPS) {
        if (lane == 0) {
            int stage = 0; uint32_t phase = 0;
            for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
                const int nt = (int)(t / a.m_tiles), mt = (int)(t - (long long)nt * a.m_tiles);
                for (int kb = 0; kb < a.k_blocks; ++kb) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    uint8_t* s0 = smem + (size_t)stage * STAGE;
                    mbar_arrive_expect_tx(&full[stage], STAGE);
                    tma_load_2d(s0, &tmA, &full[stage], kb * BK, mt * BM);
                    tma_load_2d(s0 + A_BYTES, &tmA2, &full[stage], kb * BK, mt * BM);
                    tma_load_2d(s0 + 2 * A_BYTES, &tmB, &full[stage], kb * BK, nt * BN);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        const int q = warp & 3, c0 = (warp >> 2) * 16;
        const int wg = warp >> 2, row_blk = wg & 1, col_blk = wg >> 1;   // this warpgroup's 64 x 64 block of the accumulator
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
                    wgmma_bf16_n64(acc, ad + off, bd + off, (kb == kb0 && k == 0) ? 0u : 1u);     // Wh * [Xh; Xl]
                    wgmma_bf16_n64(acc, a2d + (col_blk == 0 ? off : 0), bd + off, 1u);        // Wl * Xh -> columns [0, 64) (else + 0)
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
        const bool rmw = a.epi == E_NOISE || a.epi == E_ADD || a.epi == E_ADD_HILO;
        for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
            const int nt = (int)(t / a.m_tiles), mt = (int)(t - (long long)nt * a.m_tiles);
            const int m = mt * BM + q * 32 + lane;
            const bool m_ok = m < a.M;
            float bias = 0.f, al = 0.f, gm = 1.f;
            int co = m, r = 0;
            if (a.epi == E_CONVT) { r = m / a.Cout; co = m - r * a.Cout; }
            if (m_ok) {
                if (a.bias) bias = a.bias[co];
                if (a.alpha) al = a.alpha[m];
                if (a.gamma) gm = a.gamma[m];
            }
            const float inv_al = 1.0f / (al + 1e-9f);
            const long long n_first = (long long)nt * HALF + c0;
            // everything that does not depend on the accumulator is fetched BEFORE waiting for the MMA: the residual /
            // read-modify-write operand (16 independent loads) and the NoiseBlock noise (one value per token: lane j computes
            // or loads token j, broadcast by shuffle below)
            float xv[16];
            if (rmw) {
#pragma unroll
                for (int j = 0; j < 16; ++j) xv[j] = (m_ok && n_first + j < a.N) ? a.x[(n_first + j) * a.ldx + m] : 0.f;
            }
            float nz_lane = 0.f;
            if (a.epi == E_NOISE) {
                const long long n = n_first + (lane & 15);
                if (n < a.N) nz_lane = a.noise ? a.noise[n] : gauss(a.seed, (unsigned long long)n);
            }
            mma_block(0, a.k_blocks);
            float v[16], w[16];
            ld_acc16(arow + c0, v);
            ld_acc16(arow + c0 + HALF, w);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const long long n = n_first + j;      // token (row of X)
                const float nz = a.epi == E_NOISE ? __shfl_sync(0xffffffffu, nz_lane, j) : 0.f;
                if (n >= a.N || !m_ok) continue;
                float val = v[j] + w[j] + bias;
                if (a.gelu) val = 0.5f * val * (1.0f + erff(val * 0.70710678118654752f));
                val *= gm;
                if (a.epi == E_STORE_F32) { a.x[n * a.ldx + m] = val; continue; }
                if (a.epi == E_CONVT) {
                    const int b = (int)(n / (a.Tin + 1)), qq = (int)(n - (long long)b * (a.Tin + 1));
                    const int to = qq * a.stride + r - a.pad;
                    if (to < 0 || to >= a.T) continue;
                    const long long tok = (long long)b * a.T + to;
                    a.x[tok * a.ldx + co] = val;
                    if (a.hl) put_hilo(a.hl, a.ldh, tok, co, val);
                    continue;
                }
                if (a.epi == E_NOISE) {
                    a.x[n * a.ldx + m] = xv[j] + nz * val;
                    continue;
                }
                if (rmw) {
                    val += xv[j];
                    a.x[n * a.ldx + m] = val;
                    if (a.epi == E_ADD) continue;
                }
                if (a.alpha) val = snake_inv(val, al, inv_al);
                if (a.fs) {
                    const long long b = n / a.T;
                    put_frames(a.hl, a.fs, a.fpad, a.M, a.T, b, (int)(n - b * a.T), m, val);
                } else if (a.dual) {
                    const long long b = n / a.T, tt = n - b * a.T;
                    const long long row = b * (a.T + 1) + tt;
                    put_hilo(a.hl, a.ldh, row, m, val);
                    put_hilo(a.hl, a.ldh, row + 1, a.M + m, val);
                } else {
                    put_hilo(a.hl, a.ldh, n, m, val);
                }
            }
        }
    }
}

}  // namespace cg
}  // namespace b2a
