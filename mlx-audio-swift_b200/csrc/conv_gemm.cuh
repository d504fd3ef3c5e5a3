// Persistent wgmma + TMA GEMM for the codec path, with two entry points on one machine (conv_gemm.cu):
//     D[M, N] = (Wh + Wl)[M, K] * (Xh + Xl)[N, K]^T      fp32 weights and activations as bf16 hi/lo pairs
// A  = weights, TWO K-major operands (hi and lo halves of the fp32 weight, 16 mantissa bits together)
// B  = activations, 128-row tiles = 64 tokens as hi rows | lo rows (same layout as tc_gemm)
// per k-block:  D[:, 0:128] += Wh * [Xh; Xl]   and   D[:, 0:64] += Wl * Xh        (Wl*Xl, 2^-18 relative, is dropped)
// so the result equals the fp32 convolution to ~1e-5.  One CTA per SM loops over (token tile, m tile) work items;
// the TMA ring never drains between tiles.
//
// cg::conv_gemm_kernel (SNAC in channels-last layout, Vocos) reads B as 2-D tiles of a token matrix [tokens, channels].
// Its epilogue warps fuse what the reference runs as separate MLX ops: bias, Snake, residual add, NoiseBlock, the
// transposed-conv phase scatter, and the hi/lo re-split that feeds the next GEMM (optionally written twice, shifted by one
// token, which is the im2col the 2-tap transposed conv needs).
//
// ic::implicit_conv_kernel (Qwen3-TTS speech tokenizer, SURVEY.md row N1) is an IMPLICIT-GEMM causal convolution
//     D[m, (b, t)] = sum_j sum_c (Wh + Wl)[m, j, c] * (Xh + Xl)[b, t + shift0 + j * dil, c]
// that removes the im2col matrix the dense k7 / dilated convolutions would otherwise write and re-read (7x the activation
// bytes):
//   * activations live as PLANES  hl[2 (hi | lo)][B][Ttot][C]  (channels-last, bf16 or fp16).  A 4-D tensor map with box
//     {64 channels, 64 frames, 1 row, 2 planes} lands in shared memory as the same 128-row x 128-byte SWIZZLE_128B tile
//     the dense GEMM reads, but its frame coordinate is free: tap j of the convolution is the SAME tile shifted by
//     j * dil frames, so the k-loop is (tap, channel block) and the B operand is read straight from the activation planes.
//     Out-of-range frames / channels are zero-filled by TMA (C = 96 uses two 64-channel blocks, the second half zeros on
//     both operands).
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
// same with the per-channel 1 / (alpha + 1e-9) computed once by the caller; the fma rounds differently from snake().  Also
// SnakeBeta (v + 1/(exp(beta) + 1e-9) * sin(exp(alpha) v)^2) with al = exp(alpha), inv = 1 / (exp(beta) + 1e-9).  (A precise
// sinf changes nothing measurable: the error budget is elsewhere, DESIGN.md 3.8.)
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
// v -> hi + lo in the operand format (f16 != 0: fp16, else bf16), stored as raw 16-bit words at idx and plane + idx
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

// ----------------------------------------------------------------------------------------------- host (conv_gemm.cu)
// host-side hi / lo split in the operand format, as raw 16-bit words, and its inverse
inline void split16(float v, int f16, uint16_t& hi, uint16_t& lo) {
    if (f16) {
        const __half h = __float2half_rn(v);
        hi = __half_as_ushort(h);
        lo = __half_as_ushort(__float2half_rn(v - __half2float(h)));
    } else {
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        hi = __bfloat16_as_ushort(h);
        lo = __bfloat16_as_ushort(__float2bfloat16_rn(v - __bfloat162float(h)));
    }
}
inline float join16(uint16_t hi, uint16_t lo, int f16) {
    return f16 ? __half2float(__ushort_as_half(hi)) + __half2float(__ushort_as_half(lo))
               : __bfloat162float(__ushort_as_bfloat16(hi)) + __bfloat162float(__ushort_as_bfloat16(lo));
}

// Weight operand of both kernels: fp32 [M][taps][Cin] as K-major hi / lo matrices [M][taps * cblocks * 64] with their TMA maps,
// every tap's channel run zero-padded to whole 64-channel k-blocks.  The dense GEMM takes one tap of K = Cin (a multiple of 64).
struct TcW {
    DBuf<__nv_bfloat16> hi, lo;   // raw 16-bit words: fp16 when f16 != 0
    DBuf<float> bias, rscale;     // rscale[m] (fp16 operands only): 1 / the power of two row m is stored times
    CUtensorMap th{}, tl{};
    int M = 0, taps = 1, cblocks = 0, Cin = 0, f16 = 0;
    bool has_bias = false;
    // [M][taps][Cin] -> [M][taps][cblocks * 64]
    static std::vector<float> pad_k(const std::vector<float>& W, int M, int taps, int Cin);
    void build(const std::vector<float>& W, int M_, int taps_, int Cin_, int f16_ = 0);
    void set_bias(const std::vector<float>& b);
};

// D = W * X^T with the epilogue `a` (a.M, a.K and the tile counts are set here): X is the hi/lo activation matrix of x_rows rows
// and W.Cin columns; min(max_ctas, work items) persistent CTAs
void launch(const TcW& W, const __nv_bfloat16* X, long long x_rows, Args a, long long max_ctas, cudaStream_t s);

}  // namespace cg

namespace ic {

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
    int elu;                      // ELU(alpha 1) on the hi/lo copy instead (Mimi's SEANet decoder: the next conv's input activation)
};

// One implicit convolution of weight W over planes `in` [2][B][in_frames][W.Cin] in W's operand format.  Set here: the weight
// geometry, Cout = W.M / up, the bias (W's), the row scales, seg_kb and the tile counts; dil = 0 and up = 0 mean 1.
void launch(const cg::TcW& W, const __nv_bfloat16* in, long long in_frames, Args a, long long max_ctas, cudaStream_t s);

}  // namespace ic
}  // namespace b2a
