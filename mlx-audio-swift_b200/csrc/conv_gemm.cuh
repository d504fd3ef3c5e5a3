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
#include "common.cuh"
#include "tc_gemm.cuh"

#include <vector>

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

// Snake (Layers.swift:44-50): v + 1/(alpha + 1e-9) * sin(alpha v)^2
__device__ __forceinline__ float snake(float v, float al) {
    const float s = fast_sin(al * v);
    return v + (1.0f / (al + 1e-9f)) * s * s;
}
// same with the per-channel 1 / (alpha + 1e-9) computed once by the caller; the fma rounds differently from snake()
__device__ __forceinline__ float snake_inv(float v, float al, float inv) {
    const float s = fast_sin(al * v);
    return fmaf(inv * s, s, v);
}
// counter-based N(0,1) for the NoiseBlock: splitmix64 -> two uniforms -> Box-Muller (MLXRandom.normal stand-in)
__device__ __forceinline__ float gauss(unsigned long long seed, unsigned long long idx) {
    unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (idx + 1);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    const float u1 = ((unsigned)(z >> 40) + 1.0f) * (1.0f / 16777217.0f);
    const float u2 = (unsigned)((z >> 8) & 0xFFFFFF) * (1.0f / 16777216.0f);
    return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}
// Input of a strided conv (kernel 2 fs, stride fs, left pad fpad < fs) over utterances of T tokens (T % fs == 0) as a 2-tap GEMM
// operand: the zero-padded sequence is cut into frames of fs tokens x C channels; output token q reads frames q and q + 1, so row
// b (T / fs + 1) + q holds frame q in columns [0, fs C) and frame q + 1 in [fs C, 2 fs C) (row q = T / fs is computed and dropped).
// Token (b, t) is padded position p = t + fpad of frame f = p / fs: it lands in row f (first half) and in row f - 1 (second half).
__device__ __forceinline__ void put_frames(__nv_bfloat16* hl, int fs, int fpad, int C, int T, long long b, int t, int c, float v) {
    const int p = t + fpad, f = p / fs, col = (p - f * fs) * C + c;
    const long long ld = 2ll * fs * C, row = b * (T / fs + 1) + f;
    store_hilo(hl, ld, row, col, v, HALF);
    if (f > 0) store_hilo(hl, ld, row - 1, (long long)fs * C + col, v, HALF);
}

// ----------------------------------------------------------------------------------------------- host (conv_gemm.cu)
// fp32 weight matrix [M, K] as two bf16 K-major operands (hi + lo) with their TMA maps
struct TcW {
    DBuf<__nv_bfloat16> hi, lo;
    CUtensorMap th{}, tl{};
    int M = 0, K = 0;
    void build(const std::vector<float>& W, int M_, int K_);
};

// D = W * X^T with the epilogue `a` (a.M, a.K and the tile counts are set here): X is the hi/lo activation matrix of x_rows rows
// and W.K columns; min(max_ctas, work items) persistent CTAs
void launch(const TcW& W, const __nv_bfloat16* X, long long x_rows, Args a, long long max_ctas, cudaStream_t s);

}  // namespace cg
}  // namespace b2a
