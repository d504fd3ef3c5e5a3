// SNAC codec decode, encode + RVQ code search for sm_90a.  Replaces (reference paths):
//   Sources/MLXAudioCodecs/SNAC/VQ.swift:14-20,47-120,150-191    (RVQ lookup / code search)
//   Sources/MLXAudioCodecs/SNAC/Layers.swift:44-50,54-183,202-232,263-315,364-421 (decoder)
//   Sources/MLXAudioCodecs/SNAC/SNACDecoder.swift:127-131          (SNAC.decode)
//   Sources/MLXAudioCodecs/SNAC/Layers.swift:236-259,319-360, SNACDecoder.swift:86-105,120-125 (encoder, SNAC.encode; DESIGN.md §3.2b)
//
// HBM layout: activations float32 [B, C, T] (time contiguous -> every load/store is coalesced
// along T); two ping-pong buffers sized for the widest stage.  Weight-norm (g*v/||v||) is folded
// once at load time instead of on every call (Layers.swift:102-103,166).  1x1 convolutions and the
// transposed convolutions are GEMMs C[M,N] = A[M,K] * B[K,N] with N = time:
//   1x1 conv : A = W[co,ci]                         B[k,n] = x[ci=k, t=n]
//   convT    : A[(co*s+r),(tap*Cin+ci)] = W[ci, r+tap*s, co]   B[k,n] = x[ci, q=n-tap]
//              (kernel 2s, stride s: exactly two taps per output phase r), scattered to
//              t_out = q*s + r - pad.
// Snake activations are fused into the epilogue of the producing kernel (or the prologue of the
// depthwise conv), the residual add / noise injection into the GEMM epilogue.
#include "common.cuh"
#include "conv_gemm.cuh"
#include "snac_fused.cuh"
#include "layernorm.cuh"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <numeric>

namespace b2a {

// ------------------------------------------------------------------------------------------------
// RVQ lookup: z[b,c,t] (+)= bias_i[c] + sum_d Wout_i[c,d] * codebook_i[codes_i[b, t/s_i], d]
// (VectorQuantize.decodeCode + outProj + repeat-interleave, VQ.swift:88-94,165-191)
// ------------------------------------------------------------------------------------------------
struct RvqLevel {
    const int* codes;      // [B, T/stride]
    const float* codebook; // [N, D]
    const float* wout;     // [C, D]
    const float* bias;     // [C]
    int stride;
};
struct RvqArgs { RvqLevel lv[4]; int n_levels; int D; int C; int T; int codebook_size; };

// sign: +1 accumulate into out (beta = 1) or write (beta = 0); used with sign=-1 for the residual
__global__ void rvq_lookup_kernel(RvqArgs a, float* __restrict__ out, float beta, float sign) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int c = blockIdx.y, b = blockIdx.z;
    if (t >= a.T) return;
    float acc = 0.f;
    for (int i = 0; i < a.n_levels; ++i) {
        const RvqLevel& L = a.lv[i];
        const int Ti = a.T / L.stride;
        int code = L.codes[(long long)b * Ti + t / L.stride];
        code = min(max(code, 0), a.codebook_size - 1);
        const float* e = L.codebook + (long long)code * a.D;
        const float* w = L.wout + (long long)c * a.D;
        float v = L.bias[c];
        for (int d = 0; d < a.D; ++d) v = fmaf(w[d], e[d], v);
        acc += v;
    }
    float* o = out + ((long long)b * a.C + c) * a.T + t;
    *o = (beta != 0.f ? beta * (*o) : 0.f) + sign * acc;
}

// ------------------------------------------------------------------------------------------------
// Depthwise conv k7 (dilation d, "same" padding) with optional Snake before and after.
// One CTA = one (b, c) row segment; the activated input tile (+halo) is staged in shared memory
// so sin() is evaluated once per element.
// ------------------------------------------------------------------------------------------------
constexpr int DW_TT = 1024, DW_THREADS = 256, DW_MAXHALO = 27;

__global__ void __launch_bounds__(DW_THREADS)
dwconv7_kernel(const float* __restrict__ in, float* __restrict__ out, const float* __restrict__ w /*[C,7]*/,
               const float* __restrict__ bias, const float* __restrict__ alpha_in,
               const float* __restrict__ alpha_out, int C, int T, int dil) {
    __shared__ float s[DW_TT + 2 * DW_MAXHALO];
    const int c = blockIdx.y, b = blockIdx.z;
    const int t0 = blockIdx.x * DW_TT;
    const int halo = 3 * dil;
    const float* x = in + ((long long)b * C + c) * T;
    const float ai = alpha_in ? alpha_in[c] : 0.f;
    for (int i = threadIdx.x; i < DW_TT + 2 * halo; i += DW_THREADS) {
        const int t = t0 + i - halo;
        float v = 0.f;
        if (t >= 0 && t < T) { v = x[t]; if (alpha_in) v = cg::snake(v, ai); }
        s[i] = v;
    }
    __syncthreads();
    float wk[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) wk[k] = w[c * 7 + k];
    const float bv = bias ? bias[c] : 0.f;
    const float ao = alpha_out ? alpha_out[c] : 0.f;
    float* y = out + ((long long)b * C + c) * T;
    for (int i = threadIdx.x; i < DW_TT; i += DW_THREADS) {
        const int t = t0 + i;
        if (t >= T) break;
        float acc = bv;
#pragma unroll
        for (int k = 0; k < 7; ++k) acc = fmaf(wk[k], s[i + k * dil], acc);
        y[t] = alpha_out ? cg::snake(acc, ao) : acc;
    }
}

// ------------------------------------------------------------------------------------------------
// fp32 GEMM core: C[M,N] = A[M,K] * B[K,N], 64x128 CTA tile, 8x8 per thread, BK = 16.
// ------------------------------------------------------------------------------------------------
constexpr int GM = 64, GN = 128, GK = 16, G_THREADS = 128;

enum : int { EPI_PLAIN = 0, EPI_RESIDUAL = 1, EPI_NOISE = 2, EPI_CONVT = 3 };

struct GemmArgs {
    const float* A;      // [M, K] row-major (folded weights)
    const float* X;      // input activations [B, Cin, Tin]
    float* Y;            // output [B, Cout, Tout]
    const float* bias;   // [Cout] or null
    const float* res;    // EPI_RESIDUAL / EPI_NOISE: [B, Cout, Tout] added to the result
    const float* noise;  // EPI_NOISE: [B, Tout] (null => generated from seed)
    const float* alpha_out;  // optional Snake on the result, [Cout]
    int M, N, K;
    int Cin, Tin, Cout, Tout;
    int stride, pad;     // EPI_CONVT
    unsigned long long seed;
    int noise_layer;
};

template <int EPI>
__global__ void __launch_bounds__(G_THREADS)
gemm_f32_kernel(GemmArgs g) {
    __shared__ __align__(16) float As[GK][GM];
    __shared__ __align__(16) float Bs[GK][GN];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.y * GM, n0 = blockIdx.x * GN, b = blockIdx.z;
    const int ty = tid / 16, tx = tid % 16;
    const float* Xb = g.X + (long long)b * g.Cin * g.Tin;

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < g.K; k0 += GK) {
        // A tile: 64 rows x 16 k ; thread loads 8 consecutive k of one row
        {
            const int r = tid >> 1, kk = (tid & 1) * 8;
            const int m = m0 + r;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int k = k0 + kk + j;
                As[kk + j][r] = (m < g.M && k < g.K) ? g.A[(long long)m * g.K + k] : 0.f;
            }
        }
        // B tile: 16 k x 128 n ; thread loads column n = tid of every row (coalesced per warp)
        {
            const int n = n0 + tid;
#pragma unroll
            for (int kk = 0; kk < GK; ++kk) {
                const int k = k0 + kk;
                float v = 0.f;
                if (k < g.K && n < g.N) {
                    if (EPI == EPI_CONVT) {
                        const int tap = k / g.Cin, ci = k - tap * g.Cin, q = n - tap;
                        if (q >= 0 && q < g.Tin) v = Xb[(long long)ci * g.Tin + q];
                    } else {
                        v = Xb[(long long)k * g.Tin + n];
                    }
                }
                Bs[kk][tid] = v;
            }
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < GK; ++kk) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[kk][32 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[kk][64 + tx * 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + (i < 4 ? ty * 4 + i : 32 + ty * 4 + (i - 4));
        if (m >= g.M) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
            if (n >= g.N) continue;
            float v = acc[i][j];
            if (EPI == EPI_CONVT) {
                const int co = m / g.stride, r = m - co * g.stride;
                const int t = n * g.stride + r - g.pad;
                if (t < 0 || t >= g.Tout) continue;
                if (g.bias) v += g.bias[co];
                if (g.alpha_out) v = cg::snake(v, g.alpha_out[co]);
                g.Y[((long long)b * g.Cout + co) * g.Tout + t] = v;
            } else {
                const long long o = ((long long)b * g.Cout + m) * g.Tout + n;
                if (g.bias) v += g.bias[m];
                if (EPI == EPI_RESIDUAL) v += g.res[o];
                if (EPI == EPI_NOISE) {
                    // NoiseBlock (Layers.swift:271-278): x + noise[b,0,t] * (W x)
                    const float nz = g.noise ? g.noise[(long long)b * g.Tout + n]
                                             : cg::gauss(g.seed + 0x1000193ull * (g.noise_layer + 1),
                                                         (unsigned long long)b * g.Tout + n);
                    v = g.res[o] + nz * v;
                }
                if (g.alpha_out) v = cg::snake(v, g.alpha_out[m]);
                g.Y[o] = v;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Final conv k7 (C -> 1) + tanh on an already Snake-activated input (Layers.swift:411-415)
// ------------------------------------------------------------------------------------------------
constexpr int FC_TT = 512, FC_THREADS = 128, FC_CH = 16;

__global__ void __launch_bounds__(FC_THREADS)
final_conv7_tanh_kernel(const float* __restrict__ in, float* __restrict__ out, const float* __restrict__ w /*[C,7]*/,
                        float bias, int C, int T) {
    __shared__ float s[FC_CH][FC_TT + 8];
    __shared__ float sw[FC_CH * 7];
    const int b = blockIdx.y, t0 = blockIdx.x * FC_TT;
    float acc[4] = {bias, bias, bias, bias};
    for (int c0 = 0; c0 < C; c0 += FC_CH) {
        const int nc = min(FC_CH, C - c0);
        for (int i = threadIdx.x; i < nc * (FC_TT + 6); i += FC_THREADS) {
            const int cc = i / (FC_TT + 6), tt = i - cc * (FC_TT + 6);
            const int t = t0 + tt - 3;
            s[cc][tt] = (t >= 0 && t < T) ? in[((long long)b * C + c0 + cc) * T + t] : 0.f;
        }
        for (int i = threadIdx.x; i < nc * 7; i += FC_THREADS) sw[i] = w[c0 * 7 + i];
        __syncthreads();
        for (int cc = 0; cc < nc; ++cc)
#pragma unroll
            for (int k = 0; k < 7; ++k) {
                const float wv = sw[cc * 7 + k];
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[j] = fmaf(wv, s[cc][threadIdx.x + j * FC_THREADS + k], acc[j]);
            }
        __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int t = t0 + threadIdx.x + j * FC_THREADS;
        if (t < T) out[(long long)b * T + t] = tanhf(acc[j]);
    }
}

// ------------------------------------------------------------------------------------------------
// RVQ encode side (VQ.swift:47-120): avg-pool + in_proj, then nearest-code search in explicitly
// ordered float32 (no FMA contraction) so indices are reproducible bit for bit.
// ------------------------------------------------------------------------------------------------
// ze[n = b*Ts + t', d] = bias[d] + sum_c Win[d,c] * mean_j res[b, c, t'*s + j]
__global__ void vq_inproj_kernel(const float* __restrict__ res, const float* __restrict__ win /*[D,C]*/,
                                 const float* __restrict__ bias, float* __restrict__ ze, int C, int T, int stride,
                                 int D) {
    const int Ts = T / stride;
    const int tp = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (tp >= Ts) return;
    float acc[16];
    for (int d = 0; d < D; ++d) acc[d] = bias[d];
    const float inv = 1.0f / (float)stride;
    for (int c = 0; c < C; ++c) {
        const float* x = res + ((long long)b * C + c) * T + (long long)tp * stride;
        float m = 0.f;
        for (int j = 0; j < stride; ++j) m += x[j];
        m *= inv;
        for (int d = 0; d < D; ++d) acc[d] = fmaf(win[d * C + c], m, acc[d]);
    }
    for (int d = 0; d < D; ++d) ze[((long long)b * Ts + tp) * D + d] = acc[d];
}

// rows of x [N, D] -> L2-normalised rows + squared norm of the normalised row (VQ.swift:14-20)
__global__ void l2_normalize_rows_kernel(const float* __restrict__ x, float* __restrict__ xn, float* __restrict__ sq,
                                         int N, int D) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    float acc = 0.f;
    for (int d = 0; d < D; ++d) acc = __fadd_rn(acc, __fmul_rn(x[(long long)n * D + d], x[(long long)n * D + d]));
    const float nrm = fmaxf(__fsqrt_rn(acc), 1e-12f);
    float s2 = 0.f;
    for (int d = 0; d < D; ++d) {
        const float v = __fdiv_rn(x[(long long)n * D + d], nrm);
        xn[(long long)n * D + d] = v;
        s2 = __fadd_rn(s2, __fmul_rn(v, v));
    }
    sq[n] = s2;
}

constexpr int NC_TILE = 1024, NC_THREADS = 128, NC_MAXD = 16;
// idx[n] = first argmin_j ((|e_n|^2 - 2 e_n.c_j) + |c_j|^2)   (== argMax(-dist), VQ.swift:111-115)
__global__ void __launch_bounds__(NC_THREADS)
nearest_code_kernel(const float* __restrict__ en, const float* __restrict__ e2, const float* __restrict__ cn,
                    const float* __restrict__ c2, int* __restrict__ idx, int N, int n_codes, int D) {
    extern __shared__ float sh[];  // [NC_TILE * D] codes + [NC_TILE] norms
    float* sc = sh;
    float* sc2 = sh + NC_TILE * D;
    const int n = blockIdx.x * NC_THREADS + threadIdx.x;
    float e[NC_MAXD];
    float my_e2 = 0.f;
    if (n < N) {
        for (int d = 0; d < D; ++d) e[d] = en[(long long)n * D + d];
        my_e2 = e2[n];
    }
    float best = INFINITY;
    int best_i = 0;
    for (int j0 = 0; j0 < n_codes; j0 += NC_TILE) {
        const int nj = min(NC_TILE, n_codes - j0);
        __syncthreads();
        for (int i = threadIdx.x; i < nj * D; i += NC_THREADS) sc[i] = cn[(long long)j0 * D + i];
        for (int i = threadIdx.x; i < nj; i += NC_THREADS) sc2[i] = c2[j0 + i];
        __syncthreads();
        if (n < N)
            for (int j = 0; j < nj; ++j) {
                float dot = 0.f;
                for (int d = 0; d < D; ++d) dot = __fadd_rn(dot, __fmul_rn(e[d], sc[j * D + d]));
                const float dist = __fadd_rn(__fsub_rn(my_e2, __fmul_rn(2.0f, dot)), sc2[j]);
                if (dist < best) { best = dist; best_i = j0 + j; }
            }
    }
    if (n < N) idx[n] = best_i;
}

// ------------------------------------------------------------------------------------------------
// Channels-last (NLC) tensor-core path: activations fp32 [B*T, C] plus bf16 hi/lo copies in 64-token tiles that
// the conv GEMM (conv_gemm.cuh) reads through TMA.  The kernels below are the non-GEMM pieces.
// ------------------------------------------------------------------------------------------------
// z[b*T + t, c] = sum_i (bias_i[c] + Wout_i[c,:] . codebook_i[codes_i[b, t/s_i], :])      (VQ.swift:165-191)
__global__ void rvq_lookup_nlc_kernel(RvqArgs a, float* __restrict__ out) {
    const long long tok = blockIdx.x;                  // b*T + t
    const int b = (int)(tok / a.T), t = (int)(tok - (long long)b * a.T);
    __shared__ float se[4][16];
    if (threadIdx.x < a.n_levels * a.D) {
        const int i = threadIdx.x / a.D, d = threadIdx.x - i * a.D;
        const RvqLevel& L = a.lv[i];
        int code = L.codes[(long long)b * (a.T / L.stride) + t / L.stride];
        code = min(max(code, 0), a.codebook_size - 1);
        se[i][d] = L.codebook[(long long)code * a.D + d];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < a.C; c += blockDim.x) {
        float acc = 0.f;
        for (int i = 0; i < a.n_levels; ++i) {
            const float* w = a.lv[i].wout + (long long)c * a.D;
            float v = a.lv[i].bias[c];
            for (int d = 0; d < a.D; ++d) v = fmaf(w[d], se[i][d], v);
            acc += v;
        }
        out[tok * a.C + c] = acc;
    }
}

// Depthwise conv k7 (dilation d) along time in NLC, optional Snake before / after, output as bf16 hi/lo tiles.
// CTA = 128 tokens (+ halo) x CT <= 64 channels; the Snake'd input tile lives in shared memory (sin once per element,
// halo overhead 1.42x at dilation 9); float4 global loads, one channel PAIR per thread so hi and lo leave as bf16x2.
// C must be even (every SNAC width is a multiple of 64); C % 4 == 0 takes the vector load path.
constexpr int DWN_TT = 128, DWN_THREADS = 256;
__global__ void __launch_bounds__(DWN_THREADS)
dw7_nlc_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out, const float* __restrict__ w /*[C,7]*/,
               const float* __restrict__ bias, const float* __restrict__ alpha_in, const float* __restrict__ alpha_out,
               int T, int C, int CT, int dil) {
    extern __shared__ __align__(16) float dsm[];     // [(128 + 6*dil)][CT]
    const int t0 = blockIdx.x * DWN_TT, c0 = blockIdx.y * CT, b = blockIdx.z;
    const int halo = 3 * dil, rows = DWN_TT + 2 * halo;
    const float* xb = x + (long long)b * T * C;
    if ((C & 3) == 0 && (CT & 3) == 0) {
        const int cq = CT >> 2;
        for (int i = threadIdx.x; i < rows * cq; i += DWN_THREADS) {
            const int r = i / cq, c = (i - r * cq) * 4;
            const int t = t0 + r - halo;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (t >= 0 && t < T && c0 + c < C) {
                v = *reinterpret_cast<const float4*>(xb + (long long)t * C + c0 + c);
                if (alpha_in) {
                    const float4 al = *reinterpret_cast<const float4*>(alpha_in + c0 + c);
                    v.x = cg::snake_inv(v.x, al.x, 1.0f / (al.x + 1e-9f)); v.y = cg::snake_inv(v.y, al.y, 1.0f / (al.y + 1e-9f));
                    v.z = cg::snake_inv(v.z, al.z, 1.0f / (al.z + 1e-9f)); v.w = cg::snake_inv(v.w, al.w, 1.0f / (al.w + 1e-9f));
                }
            }
            *reinterpret_cast<float4*>(dsm + (size_t)r * CT + c) = v;
        }
    } else {
        for (int i = threadIdx.x; i < rows * CT; i += DWN_THREADS) {
            const int r = i / CT, c = i - r * CT;
            const int t = t0 + r - halo;
            float v = 0.f;
            if (t >= 0 && t < T && c0 + c < C) {
                v = xb[(long long)t * C + c0 + c];
                if (alpha_in) v = cg::snake(v, alpha_in[c0 + c]);
            }
            dsm[i] = v;
        }
    }
    __syncthreads();
    const int hp = CT >> 1;                                    // channel pairs per row
    const int c = (threadIdx.x % hp) * 2, grp = threadIdx.x / hp, ngrp = DWN_THREADS / hp;
    if (c0 + c >= C) return;
    float wa[7], wb[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) { wa[k] = w[(c0 + c) * 7 + k]; wb[k] = w[(c0 + c + 1) * 7 + k]; }
    const float ba = bias ? bias[c0 + c] : 0.f, bb = bias ? bias[c0 + c + 1] : 0.f;
    const float aoa = alpha_out ? alpha_out[c0 + c] : 0.f, aob = alpha_out ? alpha_out[c0 + c + 1] : 0.f;
    const float ioa = 1.0f / (aoa + 1e-9f), iob = 1.0f / (aob + 1e-9f);
    for (int tt = grp; tt < DWN_TT; tt += ngrp) {
        const int t = t0 + tt;
        if (t >= T) break;
        float va = ba, vb = bb;
#pragma unroll
        for (int k = 0; k < 7; ++k) {
            const float2 xv = *reinterpret_cast<const float2*>(dsm + (size_t)(tt + k * dil) * CT + c);
            va = fmaf(wa[k], xv.x, va); vb = fmaf(wb[k], xv.y, vb);
        }
        if (alpha_out) { va = cg::snake_inv(va, aoa, ioa); vb = cg::snake_inv(vb, aob, iob); }
        const long long tok = (long long)b * T + t;
        const long long r = (tok / 64) * 128 + (tok % 64);
        const __nv_bfloat162 hi = __floats2bfloat162_rn(va, vb);
        const __nv_bfloat162 lo = __floats2bfloat162_rn(va - __low2float(hi), vb - __high2float(hi));
        *reinterpret_cast<__nv_bfloat162*>(out + r * C + c0 + c) = hi;
        *reinterpret_cast<__nv_bfloat162*>(out + (r + 64) * C + c0 + c) = lo;
    }
}

// zero the two half-rows per utterance of the 2-tap im2col matrix that no producer writes:
// row b*(T+1) cols [C, 2C) (tap 1 of q = 0) and row b*(T+1)+T cols [0, C) (tap 0 of q = T)
__global__ void x2_zero_edges_kernel(__nv_bfloat16* __restrict__ x2, int T, int C) {
    const int b = blockIdx.x;
    const long long r0 = (long long)b * (T + 1), r1 = r0 + T;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const long long h0 = (r0 / 64) * 128 + (r0 % 64), h1 = (r1 / 64) * 128 + (r1 % 64);
        const __nv_bfloat16 z = __float2bfloat16_rn(0.f);
        x2[h0 * 2 * C + C + c] = z; x2[(h0 + 64) * 2 * C + C + c] = z;
        x2[h1 * 2 * C + c] = z; x2[(h1 + 64) * 2 * C + c] = z;
    }
}

// ---- encoder (Layers.swift:236-259, 319-360) -------------------------------------------------------------------------------
// stem WNConv1d(1 -> C, k7, pad 3) on the raw waveform, zero right-padded from n to T samples: y[b*T + t, c], C % 4 == 0 (channels
// past the model width have zero weights and bias, so they stay 0).  One thread = one token x 4 channels (float4 store).
__global__ void enc_stem_kernel(const float* __restrict__ wave, float* __restrict__ y, const float* __restrict__ w /*[C,7]*/,
                                const float* __restrict__ bias, int B, long long n, int T, int C) {
    const int cq = C >> 2;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * T * cq) return;
    const long long tok = i / cq;
    const int c = (int)(i - tok * cq) * 4;
    const int b = (int)(tok / T), t = (int)(tok - (long long)b * T);
    const float* x = wave + (long long)b * n;
    float xv[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) { const long long s = (long long)t + k - 3; xv[k] = (s >= 0 && s < n) ? x[s] : 0.f; }
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float acc = bias[c + j];
#pragma unroll
        for (int k = 0; k < 7; ++k) acc = fmaf(w[(c + j) * 7 + k], xv[k], acc);
        o[j] = acc;
    }
    *reinterpret_cast<float4*>(y + tok * C + c) = make_float4(o[0], o[1], o[2], o[3]);
}

// zero the padding positions of the strided conv's 2-frame im2col (conv_gemm.cuh put_frames), which no producer writes: frame 0
// positions [0, pad), frame T/s positions [pad, s) (rows T/s and T/s - 1), and the second half of the dropped row T/s
__global__ void frames_zero_edges_kernel(__nv_bfloat16* __restrict__ hl, int T, int s, int pad, int C) {
    const long long tout = T / s, r0 = (long long)blockIdx.x * (tout + 1), rl = r0 + tout;
    const long long ld = 2ll * s * C, sc = (long long)s * C;
    const __nv_bfloat16 z = __float2bfloat16_rn(0.f);
    auto zero = [&](long long row, long long c0, long long c1) {
        const long long h = (row / 64) * 128 + (row % 64);
        for (long long c = c0 + threadIdx.x; c < c1; c += blockDim.x) { hl[h * ld + c] = z; hl[(h + 64) * ld + c] = z; }
    };
    zero(r0, 0, (long long)pad * C);
    zero(rl, (long long)pad * C, ld);
    zero(rl - 1, sc + (long long)pad * C, ld);
}

// final depthwise WNConv1d(C -> C, k7, pad 3, groups C) from NLC x [B*T, ld] (ld >= C: the last strided conv's padded width) to the
// quantizer's fp32 z [B, C, T]: 32 tokens x 32 channels per CTA, staged (with the 3-token halo) in shared memory so that both the
// load and the store are coalesced
__global__ void __launch_bounds__(256)
enc_final_dw_kernel(const float* __restrict__ x, float* __restrict__ z, const float* __restrict__ w /*[C,7]*/,
                    const float* __restrict__ bias, int T, int C, int ld) {
    __shared__ float s[38][33];
    const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32, b = blockIdx.z;
    for (int i = threadIdx.y * 32 + threadIdx.x; i < 38 * 32; i += 256) {
        const int r = i >> 5, c = i & 31, t = t0 + r - 3;
        s[r][c] = (t >= 0 && t < T && c0 + c < C) ? x[((long long)b * T + t) * ld + c0 + c] : 0.f;
    }
    __syncthreads();
    const int t = t0 + threadIdx.x;
    if (t >= T) return;
    for (int c = threadIdx.y; c < 32 && c0 + c < C; c += 8) {
        float acc = bias[c0 + c];
#pragma unroll
        for (int k = 0; k < 7; ++k) acc = fmaf(w[(c0 + c) * 7 + k], s[threadIdx.x + k][c], acc);
        z[((long long)b * C + c0 + c) * T + t] = acc;
    }
}

// final Snake -> conv k7 (C -> 1) -> tanh in NLC (Layers.swift:411-415), C == FC (64, or 128 for the zero-padded 96 of the 32 / 44 kHz
// models).  256 tokens per CTA; the Snake'd tile (+3 halo rows each side) is staged in shared memory.  Thread (tg, cg) owns 8 consecutive
// tokens x 8 channels of each 64-channel half (two float4 column groups {4cg..4cg+3} and {32+4cg..}, so a quarter-warp's LDS.128 covers
// 128 contiguous bytes): 14 row reads feed 8 x 7 x 8 FMAs against weights held in registers; the 8 channel groups are then reduced by
// shuffles.
constexpr int FN_TT = 256, FN_THREADS = 256;
template <int FC>
__global__ void __launch_bounds__(FN_THREADS)
final_nlc_kernel(const float* __restrict__ x, float* __restrict__ wave, const float* __restrict__ w /*[C,7]*/,
                 const float* __restrict__ alpha, float bias, int T, int C) {
    extern __shared__ __align__(16) float fsm[];     // [(256 + 6)][FC]
    constexpr int CQ = FC / 4;                       // float4 column groups per row; FN_THREADS % CQ == 0
    const int t0 = blockIdx.x * FN_TT, b = blockIdx.y;
    const float* xb = x + (long long)b * T * FC;
    {   // a thread always stages the same 4 channels
        const int c = (threadIdx.x % CQ) * 4;
        const float4 al = *reinterpret_cast<const float4*>(alpha + c);
        const float4 iv = make_float4(1.0f / (al.x + 1e-9f), 1.0f / (al.y + 1e-9f), 1.0f / (al.z + 1e-9f), 1.0f / (al.w + 1e-9f));
        for (int i = threadIdx.x; i < (FN_TT + 6) * CQ; i += FN_THREADS) {
            const int r = i / CQ;
            const int t = t0 + r - 3;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (t >= 0 && t < T) {
                v = *reinterpret_cast<const float4*>(xb + (long long)t * FC + c);
                v.x = cg::snake_inv(v.x, al.x, iv.x); v.y = cg::snake_inv(v.y, al.y, iv.y); v.z = cg::snake_inv(v.z, al.z, iv.z); v.w = cg::snake_inv(v.w, al.w, iv.w);
            }
            *reinterpret_cast<float4*>(fsm + r * FC + c) = v;
        }
    }
    const int cgp = threadIdx.x & 7, tg = threadIdx.x >> 3;     // 8 channel groups x 32 token groups
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int h = 0; h < FC / 64; ++h) {
        float wk[8][7];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int c = h * 64 + (i < 4 ? 0 : 28) + cgp * 4 + i;   // i >= 4 -> 32 + 4*cgp + (i - 4)
#pragma unroll
            for (int k = 0; k < 7; ++k) wk[i][k] = w[c * 7 + k];
        }
        if (h == 0) __syncthreads();
        const float* base = fsm + (tg * 8) * FC + h * 64 + cgp * 4;
#pragma unroll
        for (int r = 0; r < 14; ++r) {
            const float4 lo = *reinterpret_cast<const float4*>(base + r * FC);
            const float4 hi = *reinterpret_cast<const float4*>(base + r * FC + 32);
            const float xv[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int k = r - j;
                if (k >= 0 && k < 7) {
#pragma unroll
                    for (int i = 0; i < 8; ++i) acc[j] = fmaf(wk[i][k], xv[i], acc[j]);
                }
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        float v = acc[j];
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        acc[j] = v;
    }
    const int t = t0 + tg * 8 + cgp;                            // lane cgp of the group writes token cgp
    float out = acc[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) out = cgp == j ? acc[j] : out;
    if (t < T) wave[(long long)b * T + t] = tanhf(out + bias);
}

// ------------------------------------------------------------------------------------------------
// LocalMHA (Attention.swift:14-95) core: windowed non-causal attention of one head over qkv fp32 [B*T, 3*dim] (q | k | v, head h at
// columns h*64 .. +63 of each), rotary (rotate-half, [freqs, freqs]) applied to q and k as they are loaded, softmax(q k^T / 8) v in fp32.
// CTA = (window, head, clip), 8 warps; K and V of the window live in shared memory, warp w takes query rows w, w + 8, ...: lane j
// scores keys j and j + 32, lane d accumulates output channels d and d + 32.  The output goes straight into the hi/lo operand rows
// [tokens, dim] of to_out.  rope: cos [W][64] then sin [W][64] (angle n * inv_freq[d % 32], position n within the window).
constexpr int LA_THREADS = 256, LA_MAXW = 64, LA_D = 64;
__global__ void __launch_bounds__(LA_THREADS)
local_attn_kernel(const float* __restrict__ qkv, const float* __restrict__ rope, __nv_bfloat16* __restrict__ out, int T, int dim, int W) {
    __shared__ float Ks[LA_MAXW][LA_D + 1], Vs[LA_MAXW][LA_D];
    const int win = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long tok0 = (long long)b * T + (long long)win * W;
    const long long ld = 3ll * dim;
    const float* cs = rope;
    const float* sn = rope + W * LA_D;
    for (int n = warp; n < W; n += LA_THREADS / 32) {
        const float* row = qkv + (tok0 + n) * ld + h * LA_D;
        const float k0 = row[dim + lane], k1 = row[dim + lane + 32];
        Ks[n][lane] = k0 * cs[n * LA_D + lane] - k1 * sn[n * LA_D + lane];
        Ks[n][lane + 32] = k1 * cs[n * LA_D + lane + 32] + k0 * sn[n * LA_D + lane + 32];
        Vs[n][lane] = row[2 * dim + lane];
        Vs[n][lane + 32] = row[2 * dim + lane + 32];
    }
    __syncthreads();
    for (int n = warp; n < W; n += LA_THREADS / 32) {
        const float* row = qkv + (tok0 + n) * ld + h * LA_D;
        const float x0 = row[lane], x1 = row[lane + 32];
        const float q0 = 0.125f * (x0 * cs[n * LA_D + lane] - x1 * sn[n * LA_D + lane]);          // 1 / sqrt(64) folded into q
        const float q1 = 0.125f * (x1 * cs[n * LA_D + lane + 32] + x0 * sn[n * LA_D + lane + 32]);
        float s0 = 0.f, s1 = 0.f;
        const int j1 = min(lane + 32, LA_MAXW - 1);
#pragma unroll 8
        for (int d = 0; d < 32; ++d) {
            const float qa = __shfl_sync(0xffffffffu, q0, d), qb = __shfl_sync(0xffffffffu, q1, d);
            s0 = fmaf(qa, Ks[lane][d], s0); s0 = fmaf(qb, Ks[lane][d + 32], s0);
            s1 = fmaf(qa, Ks[j1][d], s1); s1 = fmaf(qb, Ks[j1][d + 32], s1);
        }
        if (lane >= W) s0 = -INFINITY;
        if (lane + 32 >= W) s1 = -INFINITY;
        float mx = fmaxf(s0, s1);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        const float p0 = lane < W ? expf(s0 - mx) : 0.f, p1 = lane + 32 < W ? expf(s1 - mx) : 0.f;
        float sum = p0 + p1;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        float o0 = 0.f, o1 = 0.f;
        for (int j = 0; j < W; ++j) {
            const float p = __shfl_sync(0xffffffffu, j < 32 ? p0 : p1, j & 31);
            o0 = fmaf(p, Vs[j][lane], o0); o1 = fmaf(p, Vs[j][lane + 32], o1);
        }
        const float inv = 1.0f / sum;
        tc::store_hilo(out, dim, tok0 + n, h * LA_D + lane, o0 * inv, cg::HALF);
        tc::store_hilo(out, dim, tok0 + n, h * LA_D + lane + 32, o1 * inv, cg::HALF);
    }
}

// ------------------------------------------------------------------------------------------------
// Host-side model
// ------------------------------------------------------------------------------------------------
struct ConvW {       // folded weights on the device
    DBuf<float> w, bias;
    bool has_bias = false;
};

using cg::TcW;

struct ResUnit { DBuf<float> a0, a2; ConvW dw, pw; TcW pw_tc, pw_bd; int dil; };   // pw_bd: [W 0; 0 W] for the fused C = 64 kernel
struct DecBlock {
    int cin, cout, stride, pad;
    DBuf<float> alpha;   // Snake before the transposed conv
    ConvW ct;            // A[(co*s+r), (tap*Cin+ci)]
    ConvW noise;         // [cout, cout], no bias
    TcW ct_tc, noise_tc, noise_bd; // tensor-core operands: ct_tc rows are m = r*cout + co (phase-major); *_bd block-diagonal (C = 64)
    bool has_noise;
    ResUnit ru[3];
};

// encoder block (Layers.swift:236-259) at its padded width cp: three ResidualUnits, Snake, strided conv cp -> cp_out
struct EncBlock {
    int c, cp, cout, cp_out, stride, pad;
    ResUnit ru[3];
    DBuf<float> alpha;   // Snake before the strided conv
    TcW down;            // [cp_out, 2 * stride * cp]: A[co, j * cp + ci] = w[co, j, ci]  (kernel position j < 2 stride)
    ConvW down_b;        // bias only
};
// channel width the encoder runs a C-channel stage at: the fused unit's 64 / 128 up to 128, else the conv GEMM's multiple of 64.
// The extra channels carry exact zeros (weights and biases 0, Snake alpha 1).
static int enc_padded(int c) { return c <= 64 ? 64 : c <= 128 ? 128 : (c + 63) / 64 * 64; }
// [rows, cols] -> [prow, pcol] with zeros (and `fill` for 1-D vectors) outside
static std::vector<float> pad2(const std::vector<float>& v, int rows, int cols, int prow, int pcol, float fill = 0.f) {
    std::vector<float> o((size_t)prow * pcol, fill);
    for (int r = 0; r < rows; ++r)
        for (int c = 0; c < cols; ++c) o[(size_t)r * pcol + c] = v[(size_t)r * cols + c];
    return o;
}

static std::vector<float> fold_wn(const TensorTable& tt, const std::string& prefix, int d0, int d1, int d2, bool eps) {
    // weight = g * v / (||v||_{dims 1,2} (+ 1e-12))   Layers.swift:102-103 (eps) / :166 (no eps)
    std::vector<float> v = tt.f32(prefix + ".weight_v", (int64_t)d0 * d1 * d2);
    std::vector<float> g = tt.f32(prefix + ".weight_g", d0);
    for (int i = 0; i < d0; ++i) {
        double s = 0;
        for (int j = 0; j < d1 * d2; ++j) s += (double)v[(size_t)i * d1 * d2 + j] * v[(size_t)i * d1 * d2 + j];
        const double nrm = std::sqrt(s) + (eps ? 1e-12 : 0.0);
        for (int j = 0; j < d1 * d2; ++j)
            v[(size_t)i * d1 * d2 + j] = (float)((double)g[i] * v[(size_t)i * d1 * d2 + j] / nrm);
    }
    return v;
}

// transposed-conv weight wt [cin, 2s, cout] (kernel 2s, stride s) -> GEMM rows A[(co*s + r), (tap*cin + ci)] = wt[ci, r + tap*s, co]
static std::vector<float> convt_gemm_rows(const std::vector<float>& wt, int cin, int cout, int s) {
    const int k = 2 * s;
    std::vector<float> A((size_t)cout * s * 2 * cin);
    for (int co = 0; co < cout; ++co)
        for (int r = 0; r < s; ++r)
            for (int tap = 0; tap < 2; ++tap)
                for (int ci = 0; ci < cin; ++ci)
                    A[((size_t)(co * s + r)) * (2 * cin) + tap * cin + ci] = wt[((size_t)ci * k + (r + tap * s)) * cout + co];
    return A;
}
// the same rows phase-major (m = r*cout + co) for the tensor-core operand, so a warp's 32 lanes write 32 consecutive channels
static std::vector<float> convt_phase_major(const std::vector<float>& A, int cin, int cout, int s) {
    std::vector<float> At((size_t)cout * s * 2 * cin);
    for (int co = 0; co < cout; ++co)
        for (int r = 0; r < s; ++r)
            memcpy(&At[((size_t)r * cout + co) * 2 * cin], &A[((size_t)co * s + r) * 2 * cin], (size_t)2 * cin * sizeof(float));
    return At;
}
// [64, 64] -> [128, 128] = [W 0; 0 W]: the weight operand of the fused C = 64 kernel (two 64-token sub-tiles per MMA)
static std::vector<float> block_diag2(const std::vector<float>& w) {
    std::vector<float> d((size_t)128 * 128, 0.f);
    for (int r = 0; r < 64; ++r)
        for (int c2 = 0; c2 < 64; ++c2) { d[(size_t)r * 128 + c2] = w[(size_t)r * 64 + c2]; d[(size_t)(r + 64) * 128 + 64 + c2] = w[(size_t)r * 64 + c2]; }
    return d;
}

static void load_bias(const TensorTable& tt, const std::string& prefix, int n, ConvW& c, int np = 0) {
    if (tt.find(prefix + ".bias")) {
        std::vector<float> b = pad2(tt.f32(prefix + ".bias", n), 1, n, 1, std::max(n, np));
        c.bias.upload(b.data(), b.size());
        c.has_bias = true;
    }
}

// the 32 / 44 kHz models' LocalMHA (Attention.swift:14-95) at `dim` channels: LayerNorm(eps 1e-5) -> to_qkv -> windowed attention
// (local_attn_kernel) -> to_out + residual.  Keys <prefix>.norm.weight|bias, .to_qkv.weight [3 dim, dim], .to_out.weight [dim, dim]
// (both without bias) and .rel_pos.inv_freq [32].
constexpr int SN_LN_MAXV = 8;      // LayerNorm channel slots: dim <= 2048
struct LocalAttn {
    int dim = 0, window = 0;
    DBuf<float> ln_w, ln_b, rope;   // rope: cos [window][64] | sin [window][64]
    TcW qkv, out;
};
// local_attn_kernel's rotary table: cos [window][64] | sin [window][64] of n * inv_freq[d % 32] (SinusoidalEmbeddings, xpos off)
static std::vector<float> rope_table(const float* inv, int window) {
    std::vector<float> r((size_t)2 * window * LA_D);
    for (int n = 0; n < window; ++n)
        for (int d = 0; d < LA_D; ++d) {
            const double ang = n * (double)inv[d % (LA_D / 2)];
            r[(size_t)n * LA_D + d] = (float)std::cos(ang);
            r[((size_t)window + n) * LA_D + d] = (float)std::sin(ang);
        }
    return r;
}
static void load_attn(const TensorTable& tt, const std::string& p, int dim, int window, LocalAttn& A) {
    std::vector<float> g = tt.f32(p + ".norm.weight", dim), be = tt.f32(p + ".norm.bias", dim);
    std::vector<float> wqkv = tt.f32(p + ".to_qkv.weight", 3ll * dim * dim), wo = tt.f32(p + ".to_out.weight", (int64_t)dim * dim);
    std::vector<float> inv = tt.f32(p + ".rel_pos.inv_freq", LA_D / 2);
    A.ln_w.upload(g.data(), g.size()); A.ln_b.upload(be.data(), be.size());
    A.qkv.build(wqkv, 3 * dim, 1, dim);
    A.out.build(wo, dim, 1, dim);
    std::vector<float> r = rope_table(inv.data(), window);
    A.rope.upload(r.data(), r.size());
    A.dim = dim; A.window = window;
}
// frames out of a decoder stage of stride s over t frames: the reference drops DecoderBlock's outputPadding (stride % 2), so a
// transposed conv with k = 2 s, pad = ceil(s / 2) yields s t - (s mod 2) frames (DESIGN.md, SURVEY.md section 8(c) trap 7)
static long long stage_len(long long t, int s) { return t * s - s % 2; }

}  // namespace b2a

using namespace b2a;

struct b2a_snac {
    int device;
    b2a_snac_config cfg;
    int latent, hop;
    cudaStream_t stream = nullptr;
    // quantizer
    struct Level { DBuf<float> codebook, wout, bout, win, bin, cb_n, cb_n2; int stride; };
    std::vector<Level> levels;
    // decoder
    ConvW dw0, pw0, conv0;   // depthwise: dw0 + pw0 ; otherwise conv0 (k7 dense, unsupported on device)
    TcW pw0_tc;
    bool use_tc = true;      // wgmma / NLC path (B2A_SNAC=simt selects the fp32 CUDA-core path)
    LocalAttn dec_attn, enc_attn;        // LocalMHA of the 32 / 44 kHz models (dim 0: none)
    DBuf<float> d_qkv;                   // LocalMHA q | k | v, fp32 [tokens, 3 dim]
    int num_sms = 132;
    DBuf<float> xs, xs2;                 // NLC fp32 activations of the current stage (ping-pong for the fused units)
    DBuf<__nv_bfloat16> hA, x2;          // hi/lo tiles: GEMM input of the stage / 2-tap im2col of the next transposed conv
    std::vector<DecBlock> blocks;
    DBuf<float> alpha_final;
    ConvW final_conv;
    int final_c = 0;
    float final_bias = 0.f;
    // encoder (only when the checkpoint has encoder.* keys)
    bool has_enc = false;
    std::string enc_error = "SNAC encode: the checkpoint has no encoder weights";
    int enc_hop = 1;
    ConvW enc_stem, enc_final;           // [cp0, 7] / [latent, 7] + bias
    std::vector<EncBlock> eblocks;
    // workspaces
    DBuf<float> bufX, bufY, d_wave, d_noise[8], d_ze, d_en, d_e2, d_zq, d_zenc, d_ewave;
    DBuf<int> d_codes[8], d_idx;

    ~b2a_snac() { if (stream) cudaStreamDestroy(stream); }

    b2a_snac(int dev, const b2a_snac_config& c, const TensorTable& tt) : device(dev), cfg(c) {
        B2A_CHECK(c.depthwise != 0, B2A_ERR_INVALID_INPUT, "SNAC: only depthwise=true decoders are implemented");
        B2A_CHECK(c.n_vq_strides >= 1 && c.n_vq_strides <= 4 && c.n_decoder_rates >= 1 && c.n_decoder_rates <= 8,
                  B2A_ERR_INVALID_INPUT, "SNAC: unsupported number of codebooks / decoder stages");
        B2A_CHECK(c.codebook_dim >= 1 && c.codebook_dim <= NC_MAXD, B2A_ERR_INVALID_INPUT, "SNAC: codebook_dim > 16");
        require_device(dev);
        B2A_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        latent = c.latent_dim > 0 ? c.latent_dim : c.encoder_dim << c.n_encoder_rates;
        const int win = c.attn_window_size;
        B2A_CHECK(win == 0 || (win >= 1 && win <= LA_MAXW && latent % LA_D == 0 && c.decoder_dim % LA_D == 0 &&
                               latent <= DL_THREADS * SN_LN_MAXV && c.decoder_dim <= DL_THREADS * SN_LN_MAXV),
                  B2A_ERR_INVALID_INPUT, "SNAC: LocalMHA (attn_window_size > 0) needs a window of 1 .. 64 frames and latent_dim / decoder_dim "
                  "multiples of 64 (whole heads of 64) up to 2048");
        hop = 1;
        for (int i = 0; i < c.n_decoder_rates; ++i) hop *= c.decoder_rates[i];
        const int D = c.codebook_dim, N = c.codebook_size;
        levels.resize(c.n_vq_strides);
        for (int i = 0; i < c.n_vq_strides; ++i) {
            const std::string q = "quantizer.quantizers." + std::to_string(i);
            Level& L = levels[i];
            L.stride = c.vq_strides[i];
            std::vector<float> cb = tt.f32(q + ".codebook.weight", (int64_t)N * D);
            L.codebook.upload(cb.data(), cb.size());
            std::vector<float> wo = fold_wn(tt, q + ".out_proj", latent, 1, D, true);
            L.wout.upload(wo.data(), wo.size());
            std::vector<float> bo = tt.f32(q + ".out_proj.bias", latent);
            L.bout.upload(bo.data(), bo.size());
            if (tt.find(q + ".in_proj.weight_v")) {
                std::vector<float> wi = fold_wn(tt, q + ".in_proj", D, 1, latent, true);
                L.win.upload(wi.data(), wi.size());
                std::vector<float> bi = tt.f32(q + ".in_proj.bias", D);
                L.bin.upload(bi.data(), bi.size());
            }
            L.cb_n.alloc((size_t)N * D);
            L.cb_n2.alloc(N);
            l2_normalize_rows_kernel<<<cdiv(N, 128), 128, 0, stream>>>(L.codebook.p, L.cb_n.p, L.cb_n2.p, N, D);
            count_launch();
        }
        const std::string p = "decoder.model.layers.";
        const int C = c.decoder_dim;
        {
            std::vector<float> w = fold_wn(tt, p + "0", latent, 7, 1, true);
            dw0.w.upload(w.data(), w.size());
            load_bias(tt, p + "0", latent, dw0);
            std::vector<float> w1 = fold_wn(tt, p + "1", C, 1, latent, true);
            pw0.w.upload(w1.data(), w1.size());
            host_pw0 = w1;
            load_bias(tt, p + "1", C, pw0);
        }
        int li = 2;
        if (win > 0) load_attn(tt, p + "2", C, win, dec_attn);      // decoder.model.layers.2 (Layers.swift:395-397)
        if (win > 0) li = 3;
        // stages whose width is not a multiple of 64 (the 96 and 48 of the 32 / 44 kHz models' last stages) run at the encoder's padded
        // widths: the extra channels carry exact zeros (weights and biases 0, Snake alpha 1)
        blocks.resize(c.n_decoder_rates);
        for (int i = 0; i < c.n_decoder_rates; ++i, ++li) {
            DecBlock& B = blocks[i];
            const int ci_ = C >> i, co_ = C >> (i + 1);
            B.cin = enc_padded(ci_); B.cout = enc_padded(co_); B.stride = c.decoder_rates[i];
            B.pad = (B.stride + 1) / 2;  // Int(ceil(stride/2)), Layers.swift:295
            B2A_CHECK(B.stride >= 1, B2A_ERR_INVALID_INPUT, "SNAC: decoder stride");
            const std::string b = p + std::to_string(li) + ".block.layers.";
            std::vector<float> a = pad2(tt.f32(b + "0.alpha", ci_), 1, ci_, 1, B.cin, 1.f);
            B.alpha.upload(a.data(), a.size());
            const int s = B.stride, k = 2 * s;
            std::vector<float> wt0 = fold_wn(tt, b + "1", ci_, k, co_, false);  // [ci, k, co]
            std::vector<float> wt = pad2(wt0, ci_ * k, co_, ci_ * k, B.cout);
            wt.resize((size_t)B.cin * k * B.cout, 0.f);
            std::vector<float> A = convt_gemm_rows(wt, B.cin, B.cout, s);
            B.ct.w.upload(A.data(), A.size());
            host_ct.push_back(convt_phase_major(A, B.cin, B.cout, s));
            load_bias(tt, b + "1", co_, B.ct, B.cout);
            int j = 2;
            B.has_noise = c.noise != 0;
            if (B.has_noise) {
                std::vector<float> wn_ = pad2(fold_wn(tt, b + "2.linear", co_, 1, co_, true), co_, co_, B.cout, B.cout);
                B.noise.w.upload(wn_.data(), wn_.size());
                host_noise.push_back(wn_);
                j = 3;
            }
            const int dils[3] = {1, 3, 9};
            for (int u = 0; u < 3; ++u, ++j) {
                ResUnit& R = B.ru[u];
                R.dil = dils[u];
                const std::string r = b + std::to_string(j) + ".block.layers.";
                std::vector<float> a0 = pad2(tt.f32(r + "0.alpha", co_), 1, co_, 1, B.cout, 1.f), a2 = pad2(tt.f32(r + "2.alpha", co_), 1, co_, 1, B.cout, 1.f);
                R.a0.upload(a0.data(), a0.size());
                R.a2.upload(a2.data(), a2.size());
                std::vector<float> wd = pad2(fold_wn(tt, r + "1", co_, 7, 1, true), co_, 7, B.cout, 7);
                R.dw.w.upload(wd.data(), wd.size());
                load_bias(tt, r + "1", co_, R.dw, B.cout);
                std::vector<float> wp = pad2(fold_wn(tt, r + "3", co_, 1, co_, true), co_, co_, B.cout, B.cout);
                R.pw.w.upload(wp.data(), wp.size());
                host_pw.push_back(wp);
                load_bias(tt, r + "3", co_, R.pw, B.cout);
            }
        }
        {
            const int fc = C >> c.n_decoder_rates;
            final_c = enc_padded(fc);
            std::vector<float> a = pad2(tt.f32(p + std::to_string(li) + ".alpha", fc), 1, fc, 1, final_c, 1.f);
            alpha_final.upload(a.data(), a.size());
            std::vector<float> w = fold_wn(tt, p + std::to_string(li + 1), 1, 7, fc, true);  // [1,7,C]
            std::vector<float> wt((size_t)final_c * 7, 0.f);
            for (int k = 0; k < 7; ++k)
                for (int ci = 0; ci < fc; ++ci) wt[(size_t)ci * 7 + k] = w[(size_t)k * fc + ci];
            final_conv.w.upload(wt.data(), wt.size());
            if (tt.find(p + std::to_string(li + 1) + ".bias")) final_bias = tt.f32(p + std::to_string(li + 1) + ".bias", 1)[0];
        }
        B2A_CUDA(cudaStreamSynchronize(stream));
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
        const char* env = getenv("B2A_SNAC");
        bool shapes_ok = latent % 64 == 0 && C % 64 == 0 && (final_c == 64 || final_c == 128) && c.noise != 0;
        for (auto& B : blocks) shapes_ok = shapes_ok && B.cin % 64 == 0 && B.cout % 64 == 0;
        const bool simt = env && std::string(env) == "simt";
        // the fp32 NCT decoder is the 24 kHz model's cross-check: it has no LocalMHA
        B2A_CHECK(win == 0 || (shapes_ok && !simt), B2A_ERR_INVALID_INPUT,
                  "SNAC: a LocalMHA model runs on the tensor-core path only (B2A_SNAC=simt, or a geometry it does not run)");
        use_tc = shapes_ok && !simt;
        if (use_tc) {
            B2A_CUDA(cudaFuncSetAttribute(dw7_nlc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
            fused_attrs<64>(); fused_attrs<128>();
            B2A_CUDA(cudaFuncSetAttribute(rf::convt_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rf::convt_smem_bytes()));
            B2A_CUDA(cudaFuncSetAttribute(final_nlc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (FN_TT + 6) * 64 * (int)sizeof(float)));
            B2A_CUDA(cudaFuncSetAttribute(final_nlc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (FN_TT + 6) * 128 * (int)sizeof(float)));
            pw0_tc.build(host_pw0, C, 1, latent);
            size_t ip = 0;
            for (size_t i = 0; i < blocks.size(); ++i) {
                DecBlock& B = blocks[i];
                B.ct_tc.build(host_ct[i], B.cout * B.stride, 1, 2 * B.cin);
                B.noise_tc.build(host_noise[i], B.cout, 1, B.cout);
                if (B.cout == 64) B.noise_bd.build(block_diag2(host_noise[i]), 128, 1, 128);
                for (int u = 0; u < 3; ++u) {
                    if (B.cout == 64) B.ru[u].pw_bd.build(block_diag2(host_pw[ip]), 128, 1, 128);
                    B.ru[u].pw_tc.build(host_pw[ip++], B.cout, 1, B.cout);
                }
            }
        }
        host_pw0.clear(); host_ct.clear(); host_noise.clear(); host_pw.clear();
        if (tt.find("encoder.block.layers.0.weight_v")) {
            // a malformed encoder leaves a working decoder: encode then reports why (B2A_ERR_MODEL_NOT_INITIALIZED)
            try { load_encoder(tt); has_enc = true; }
            catch (const Error& e) { eblocks.clear(); enc_error = std::string("SNAC encode: encoder weights unusable: ") + e.what(); }
            B2A_CUDA(cudaGetLastError());
        }
    }

    // encoder weights at padded widths (Layers.swift:236-259, 319-360; keys encoder.block.layers.*)
    void load_encoder(const TensorTable& tt) {
        const std::string p = "encoder.block.layers.";
        const int n = cfg.n_encoder_rates;
        B2A_CHECK(n >= 1 && n <= 8 && cfg.encoder_dim >= 1, B2A_ERR_INVALID_INPUT, "encoder_dim / encoder_rates");
        int c = cfg.encoder_dim;
        {
            const int cp = enc_padded(c);
            std::vector<float> w = pad2(fold_wn(tt, p + "0", c, 7, 1, true), c, 7, cp, 7);
            std::vector<float> b = pad2(tt.f32(p + "0.bias", c), 1, c, 1, cp);
            enc_stem.w.upload(w.data(), w.size());
            enc_stem.bias.upload(b.data(), b.size());
        }
        B2A_CUDA(cudaFuncSetAttribute(dw7_nlc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        fused_attrs<64>(); fused_attrs<128>();
        eblocks.resize(n);
        enc_hop = 1;
        for (int i = 0; i < n; ++i, c *= 2) {
            EncBlock& E = eblocks[i];
            E.c = c; E.cp = enc_padded(c); E.cout = 2 * c; E.cp_out = enc_padded(2 * c);
            E.stride = cfg.encoder_rates[i]; E.pad = (E.stride + 1) / 2;      // Int(ceil(stride / 2)), Layers.swift:251
            B2A_CHECK(E.stride >= 1, B2A_ERR_INVALID_INPUT, "encoder stride");
            enc_hop *= E.stride;
            const std::string b = p + std::to_string(i + 1) + ".block.layers.";
            const int dils[3] = {1, 3, 9};
            for (int u = 0; u < 3; ++u) {
                ResUnit& R = E.ru[u];
                R.dil = dils[u];
                const std::string r = b + std::to_string(u) + ".block.layers.";
                std::vector<float> a0 = pad2(tt.f32(r + "0.alpha", c), 1, c, 1, E.cp, 1.f), a2 = pad2(tt.f32(r + "2.alpha", c), 1, c, 1, E.cp, 1.f);
                R.a0.upload(a0.data(), a0.size());
                R.a2.upload(a2.data(), a2.size());
                std::vector<float> wd = pad2(fold_wn(tt, r + "1", c, 7, 1, true), c, 7, E.cp, 7);
                R.dw.w.upload(wd.data(), wd.size());
                std::vector<float> bd = pad2(tt.f32(r + "1.bias", c), 1, c, 1, E.cp);
                R.dw.bias.upload(bd.data(), bd.size()); R.dw.has_bias = true;
                std::vector<float> wp = pad2(fold_wn(tt, r + "3", c, 1, c, true), c, c, E.cp, E.cp);
                R.pw_tc.build(wp, E.cp, 1, E.cp);
                if (E.cp == 64) R.pw_bd.build(block_diag2(wp), 128, 1, 128);
                std::vector<float> bp = pad2(tt.f32(r + "3.bias", c), 1, c, 1, E.cp);
                R.pw.bias.upload(bp.data(), bp.size()); R.pw.has_bias = true;
            }
            std::vector<float> a = pad2(tt.f32(b + "3.alpha", c), 1, c, 1, E.cp, 1.f);
            E.alpha.upload(a.data(), a.size());
            const int k = 2 * E.stride;
            std::vector<float> wt = fold_wn(tt, b + "4", E.cout, k, c, true);        // [co, j, ci]
            std::vector<float> A((size_t)E.cp_out * k * E.cp, 0.f);
            for (int co = 0; co < E.cout; ++co)
                for (int j = 0; j < k; ++j)
                    for (int ci = 0; ci < c; ++ci) A[(size_t)co * k * E.cp + (size_t)j * E.cp + ci] = wt[((size_t)co * k + j) * c + ci];
            E.down.build(A, E.cp_out, 1, k * E.cp);
            std::vector<float> bb = pad2(tt.f32(b + "4.bias", E.cout), 1, E.cout, 1, E.cp_out);
            E.down_b.bias.upload(bb.data(), bb.size()); E.down_b.has_bias = true;
        }
        if (cfg.attn_window_size > 0) load_attn(tt, p + std::to_string(n + 1), c, cfg.attn_window_size, enc_attn);   // Layers.swift:339-341
        const std::string f = p + std::to_string(n + (cfg.attn_window_size > 0 ? 2 : 1));
        std::vector<float> w = fold_wn(tt, f, c, 7, 1, true);                            // depthwise [C, 7, 1]
        enc_final.w.upload(w.data(), w.size());
        std::vector<float> b = tt.f32(f + ".bias", c);
        enc_final.bias.upload(b.data(), b.size()); enc_final.has_bias = true;
        B2A_CUDA(cudaStreamSynchronize(stream));
    }
    std::vector<float> host_pw0;
    std::vector<std::vector<float>> host_ct, host_noise, host_pw;

    // ---- tensor-core / NLC decode --------------------------------------------------------------------------
    void dw_nlc(const ConvW& W, const float* xin, __nv_bfloat16* out, const float* a_in, const float* a_out, int batch, int T, int C,
                int dil, cudaStream_t s) {
        const int CT = std::min(C, 64);
        B2A_CHECK(C % 2 == 0 && (C <= 64 || C % 64 == 0), B2A_ERR_INVALID_INPUT, "snac: channel widths must be even (multiples of 64 above 64)");
        const size_t sm = (size_t)(DWN_TT + 6 * dil) * CT * sizeof(float);
        dw7_nlc_kernel<<<dim3(cdiv(T, DWN_TT), cdiv(C, CT), batch), DWN_THREADS, sm, s>>>(xin, out, W.w.p, W.has_bias ? W.bias.p : nullptr,
                                                                                       a_in, a_out, T, C, CT, dil);
        count_launch();
    }
    static long long pad64(long long n) { return (n + 63) / 64 * 64; }
    template <int CC>
    static void fused_attrs() {
        B2A_CUDA(cudaFuncSetAttribute(rf::ru_fused_kernel<rf::MODE_RU, 1, CC>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        B2A_CUDA(cudaFuncSetAttribute(rf::ru_fused_kernel<rf::MODE_RU, 3, CC>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        B2A_CUDA(cudaFuncSetAttribute(rf::ru_fused_kernel<rf::MODE_RU, 9, CC>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        B2A_CUDA(cudaFuncSetAttribute(rf::ru_fused_kernel<rf::MODE_NOISE, 0, CC>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    }
    // fused ResidualUnit / NoiseBlock kernels (snac_fused.cuh) for 64 or 128 channels; other widths run the unfused NLC kernels
    bool block_fused(const DecBlock& B) const {
        bool ok = B.cout == 64 || B.cout == 128;
        for (int u = 0; u < 3; ++u) ok = ok && (B.ru[u].dil == 1 || B.ru[u].dil == 3 || B.ru[u].dil == 9);
        return ok;
    }
    // Snake + transposed conv fused (snac_fused.cuh convt_fused_kernel): 128 input channels -> stride * C_out = 128 phase rows,
    // fed by a fused block (its fp32 output is the only copy)
    bool convt_fused_ok(size_t i) const {
        if (i == 0 || i >= blocks.size()) return false;
        const DecBlock& B = blocks[i];
        bool even = true;                     // lengths s * t: no odd stride up to here (stage_len)
        for (size_t j = 0; j <= i; ++j) even = even && blocks[j].stride % 2 == 0;
        return even && B.cin == 128 && B.stride * B.cout == 128 && block_fused(blocks[i - 1]) && block_fused(B);
    }
    template <int CC>
    static void fused_c(const TcW& W, const rf::Args& a, dim3 g, size_t sm, cudaStream_t s) {
        const dim3 bl(rf::THREADS);
        if (a.mode == rf::MODE_NOISE) launch_pdl(rf::ru_fused_kernel<rf::MODE_NOISE, 0, CC>, g, bl, sm, s, W.th, W.tl, a);
        else if (a.dil == 1) launch_pdl(rf::ru_fused_kernel<rf::MODE_RU, 1, CC>, g, bl, sm, s, W.th, W.tl, a);
        else if (a.dil == 3) launch_pdl(rf::ru_fused_kernel<rf::MODE_RU, 3, CC>, g, bl, sm, s, W.th, W.tl, a);
        else launch_pdl(rf::ru_fused_kernel<rf::MODE_RU, 9, CC>, g, bl, sm, s, W.th, W.tl, a);
    }
    // W: the [128, 128] operand (the layer's own weights for C = 128, the block-diagonal copy for C = 64)
    void fused(const TcW& W, rf::Args a, int batch, long long T, cudaStream_t s) { launch_fused(W, a, batch, T, num_sms, s); }
    static void launch_fused(const TcW& W, rf::Args a, int batch, long long T, long long max_ctas, cudaStream_t s) {
        a.B = batch; a.T = (int)T;
        const int tile_tokens = a.C == 64 ? 2 * rf::TOK : rf::TOK;
        a.tiles_per_utt = cdiv(T, tile_tokens); a.n_tiles = (long long)batch * a.tiles_per_utt;
        const long long ctas = std::min<long long>(max_ctas, (a.n_tiles + rf::TEAMS - 1) / rf::TEAMS);
        const size_t sm = rf::smem_bytes(a.dil, a.mode);
        if (a.C == 64) fused_c<64>(W, a, dim3((unsigned)ctas), sm, s);
        else fused_c<128>(W, a, dim3((unsigned)ctas), sm, s);
    }
    // Snake + transposed conv of the last block (convt_fused_ok); a.x .. a.pad set by the caller
    static void launch_convt(const TcW& W, rf::ConvtArgs a, long long max_ctas, cudaStream_t s) {
        a.tiles_per_utt = cdiv(a.Tin + 1, rf::TOK); a.n_tiles = (long long)a.B * a.tiles_per_utt;
        const long long ctas = std::min<long long>(max_ctas, (a.n_tiles + rf::TEAMS - 1) / rf::TEAMS);
        launch_pdl(rf::convt_fused_kernel, dim3((unsigned)ctas), dim3(rf::THREADS), rf::convt_smem_bytes(), s, W.th, W.tl, a);
    }

    // LocalMHA on the fp32 residual stream x [batch * T, dim]: LayerNorm -> hi/lo hA -> to_qkv (fp32 d_qkv) -> windowed attention ->
    // hi/lo hA -> to_out, whose epilogue `o` (E_ADD, or E_ADD_HILO into the next transposed conv's operand) adds it into x
    void local_mha(const LocalAttn& A, float* x, int batch, long long T, cg::Args o, cudaStream_t s) {
        const long long ntok = (long long)batch * T;
        d_qkv.alloc((size_t)ntok * 3 * A.dim);
        dw_layernorm_kernel<SN_LN_MAXV><<<(unsigned)ntok, DL_THREADS, 0, s>>>(x, nullptr, nullptr, A.ln_w.p, A.ln_b.p, nullptr, hA.p, (int)T,
                                                                             A.dim, 1, 1e-5f);
        count_launch();
        cg::Args a{};
        a.N = (int)ntok; a.epi = cg::E_STORE_F32; a.x = d_qkv.p; a.ldx = 3 * A.dim;
        cg::launch(A.qkv, hA.p, 2 * pad64(ntok), a, num_sms, s);
        local_attn_kernel<<<dim3((unsigned)(T / A.window), A.dim / LA_D, batch), LA_THREADS, 0, s>>>(d_qkv.p, A.rope.p, hA.p, (int)T, A.dim,
                                                                                                  A.window);
        count_launch();
        o.N = (int)ntok; o.x = x; o.ldx = A.dim;
        cg::launch(A.out, hA.p, 2 * pad64(ntok), o, num_sms, s);
    }

    // largest workspace of a tensor-core decode of `batch` clips of T latent frames (elements); sets the buffer sizes when asked
    size_t dec_workspace(int batch, long long T, size_t* mx = nullptr, size_t* mh = nullptr, size_t* mx2 = nullptr) const {
        const int C = cfg.decoder_dim;
        size_t max_x = (size_t)batch * T * std::max(latent, C), max_h = (size_t)(2 * pad64((long long)batch * T)) * (size_t)std::max(latent, C), max_x2 = 0;
        long long t = T;
        for (auto& B : blocks) {
            max_x2 = std::max<size_t>(max_x2, (size_t)(2 * pad64((long long)batch * (t + 1))) * 2 * B.cin);
            t = stage_len(t, B.stride);
            max_x = std::max<size_t>(max_x, (size_t)batch * t * B.cout);
            max_h = std::max<size_t>(max_h, (size_t)(2 * pad64((long long)batch * t)) * B.cout);
        }
        if (mx) { *mx = max_x; *mh = max_h; *mx2 = max_x2; }
        return std::max(max_x, std::max(max_h, max_x2));
    }
    // clips per call so that every workspace stays below 2^31 elements (32-bit element indices and tensor-map extents): a batch is
    // decoded / encoded in slices of whole clips, which gives exactly the batched result
    template <class F>
    static int clips_per_slice(int batch, F workspace) {
        int nb = batch;
        while (nb > 1 && workspace(nb) >= (size_t)1 << 31) nb = (nb + 1) / 2;
        return nb;
    }

    // clip0: index of this call's first clip in the caller's batch (the seeded noise is drawn per (clip, frame) of the whole batch)
    void decode_dev_tc(const int* const* d_codes_in, int batch, long long T, const float* const* d_noise_in, int noise_mode,
                       unsigned long long seed, float* d_wave_out, cudaStream_t s, long long clip0 = 0) {
        const int C = cfg.decoder_dim;
        size_t max_x, max_h, max_x2;
        dec_workspace(batch, T, &max_x, &max_h, &max_x2);
        xs.alloc(max_x); xs2.alloc(max_x); hA.alloc(max_h); x2.alloc(max_x2);
        // RVQ lookup -> z (NLC) ; depthwise k7 -> hi/lo ; 1x1 (768 -> 1024) + Snake(block 0) -> 2-tap im2col of block 0
        RvqArgs ra{};
        ra.n_levels = (int)levels.size(); ra.D = cfg.codebook_dim; ra.C = latent; ra.T = (int)T; ra.codebook_size = cfg.codebook_size;
        for (size_t i = 0; i < levels.size(); ++i)
            ra.lv[i] = RvqLevel{d_codes_in[i], levels[i].codebook.p, levels[i].wout.p, levels[i].bout.p, levels[i].stride};
        rvq_lookup_nlc_kernel<<<(unsigned)(batch * T), 256, 0, s>>>(ra, xs.p);
        count_launch();
        dw_nlc(dw0, xs.p, hA.p, nullptr, nullptr, batch, (int)T, latent, 1, s);
        {
            x2_zero_edges_kernel<<<batch, 256, 0, s>>>(x2.p, (int)T, C);
            count_launch();
            cg::Args a{};
            a.N = (int)(batch * T); a.bias = pw0.has_bias ? pw0.bias.p : nullptr;
            cg::Args o{};        // the epilogue that writes Snake(block 0) into block 0's 2-tap im2col
            o.epi = cg::E_STORE_HILO; o.alpha = blocks[0].alpha.p; o.hl = x2.p; o.ldh = 2 * C; o.dual = 1; o.T = (int)T;
            if (dec_attn.dim) { a.epi = cg::E_STORE_F32; a.x = xs.p; a.ldx = C; }
            else { a.epi = o.epi; a.alpha = o.alpha; a.hl = o.hl; a.ldh = o.ldh; a.dual = o.dual; a.T = o.T; }
            cg::launch(pw0_tc, hA.p, 2 * pad64((long long)batch * T), a, num_sms, s);
            if (dec_attn.dim) {      // LocalMHA (Layers.swift:395-397), its residual add carrying block 0's Snake into the im2col
                o.epi = cg::E_ADD_HILO;
                local_mha(dec_attn, xs.p, batch, T, o, s);
            }
        }
        long long t = T;
        for (size_t i = 0; i < blocks.size(); ++i) {
            DecBlock& B = blocks[i];
            const long long tout = stage_len(t, B.stride), ntok = (long long)batch * tout;
            // NoiseBlock seed of this stage, shifted so that a slice of clips draws what the whole batch would (cg::gauss(seed, idx))
            const unsigned long long nseed = seed + 0x1000193ull * (i + 1) + 0x9E3779B97F4A7C15ull * (unsigned long long)(clip0 * tout);
            if (convt_fused_ok(i)) {
                // last block: Snake + transposed conv straight from the previous block's fp32 output (no 2-tap im2col round trip)
                rf::ConvtArgs a{};
                a.x = xs.p; a.y = xs2.p; a.alpha = B.alpha.p; a.bias = B.ct.has_bias ? B.ct.bias.p : nullptr;
                a.Tin = (int)t; a.T = (int)tout; a.B = batch; a.stride = B.stride; a.cout = B.cout; a.pad = B.pad;
                launch_convt(B.ct_tc, a, num_sms, s);
                std::swap(xs.p, xs2.p); std::swap(xs.n, xs2.n);
            } else {   // transposed conv: tokens (b, q), q = 0..t ; rows m = r*cout + co ; scatter to t_out = q*s + r - pad
                cg::Args a{};
                a.N = (int)(batch * (t + 1)); a.epi = cg::E_CONVT; a.bias = B.ct.has_bias ? B.ct.bias.p : nullptr;
                a.x = xs.p; a.ldx = B.cout; a.hl = block_fused(B) ? nullptr : hA.p;     // the fused units read fp32 only
                a.ldh = B.cout; a.T = (int)tout; a.Cout = B.cout; a.stride = B.stride;
                a.pad = B.pad; a.Tin = (int)t;
                cg::launch(B.ct_tc, x2.p, 2 * pad64((long long)batch * (t + 1)), a, num_sms, s);
            }
            const float* nz = d_noise_in ? d_noise_in[i] : nullptr;
            const bool fz = block_fused(B);
            if (fz) {
                // narrow stages: one fused kernel per NoiseBlock / ResidualUnit, fp32 in -> fp32 out (ping-pong xs <-> xs2)
                float* cur = xs.p; float* oth = xs2.p;
                if (B.has_noise && (nz || noise_mode == 0)) {
                    rf::Args a{};
                    a.x = cur; a.y = oth; a.C = B.cout; a.mode = rf::MODE_NOISE; a.dil = 0; a.noise = nz;
                    a.seed = nseed;
                    fused(B.cout == 64 ? B.noise_bd : B.noise_tc, a, batch, tout, s);
                    std::swap(cur, oth);
                }
                for (int u = 0; u < 3; ++u) {
                    ResUnit& R = B.ru[u];
                    rf::Args a{};
                    a.x = cur; a.y = oth; a.C = B.cout; a.mode = rf::MODE_RU; a.dil = R.dil;
                    a.dw_w = R.dw.w.p; a.dw_b = R.dw.has_bias ? R.dw.bias.p : nullptr; a.a_in = R.a0.p; a.a_mid = R.a2.p;
                    a.pw_bias = R.pw.has_bias ? R.pw.bias.p : nullptr;
                    const bool to_x2 = u == 2 && i + 1 < blocks.size() && !convt_fused_ok(i + 1);
                    if (to_x2) { a.hl = x2.p; a.a_next = blocks[i + 1].alpha.p; }
                    fused(B.cout == 64 ? R.pw_bd : R.pw_tc, a, batch, tout, s);
                    if (to_x2) {
                        // after the unit (it writes other positions of x2): a plain launch between the last fused unit and the next
                        // transposed conv's GEMM, whose TMA producer reads x2 without waiting on the programmatic dependency
                        x2_zero_edges_kernel<<<batch, 256, 0, s>>>(x2.p, (int)tout, B.cout);
                        count_launch();
                    }
                    std::swap(cur, oth);
                }
                if (cur != xs.p) { std::swap(xs.p, xs2.p); std::swap(xs.n, xs2.n); }       // the live activation is always xs
                t = tout;
                continue;
            }
            if (B.has_noise && (nz || noise_mode == 0)) {
                cg::Args a{};
                a.N = (int)ntok; a.epi = cg::E_NOISE; a.x = xs.p; a.ldx = B.cout; a.noise = nz;
                a.seed = nseed; a.T = (int)tout;
                cg::launch(B.noise_tc, hA.p, 2 * pad64(ntok), a, num_sms, s);
            }
            for (int u = 0; u < 3; ++u) {
                ResUnit& R = B.ru[u];
                dw_nlc(R.dw, xs.p, hA.p, R.a0.p, R.a2.p, batch, (int)tout, B.cout, R.dil, s);
                cg::Args a{};
                a.N = (int)ntok; a.bias = R.pw.has_bias ? R.pw.bias.p : nullptr; a.x = xs.p; a.ldx = B.cout; a.T = (int)tout;
                if (u == 2 && i + 1 < blocks.size()) {
                    x2_zero_edges_kernel<<<batch, 256, 0, s>>>(x2.p, (int)tout, B.cout);
                    count_launch();
                    a.epi = cg::E_ADD_HILO; a.alpha = blocks[i + 1].alpha.p; a.hl = x2.p; a.ldh = 2 * B.cout; a.dual = 1;
                } else {
                    a.epi = cg::E_ADD;
                }
                cg::launch(R.pw_tc, hA.p, 2 * pad64(ntok), a, num_sms, s);
            }
            t = tout;
        }
        if (final_c == 64)
            final_nlc_kernel<64><<<dim3(cdiv(t, FN_TT), batch), FN_THREADS, (FN_TT + 6) * 64 * sizeof(float), s>>>(xs.p, d_wave_out, final_conv.w.p, alpha_final.p,
                                                                                                              final_bias, (int)t, final_c);
        else
            final_nlc_kernel<128><<<dim3(cdiv(t, FN_TT), batch), FN_THREADS, (FN_TT + 6) * 128 * sizeof(float), s>>>(xs.p, d_wave_out, final_conv.w.p, alpha_final.p,
                                                                                                                final_bias, (int)t, final_c);
        count_launch();
        B2A_CUDA(cudaGetLastError());
    }

    size_t max_act(int batch, long long T) const {
        size_t m = (size_t)batch * std::max(latent, cfg.decoder_dim) * T;
        long long t = T;
        for (auto& B : blocks) { t *= B.stride; m = std::max<size_t>(m, (size_t)batch * B.cout * t); }
        return m;
    }

    void gemm(int epi, const ConvW& W, const float* X, float* Y, const float* res, const float* noise,
              const float* alpha_out, int batch, int M, int N, int K, int Cin, int Tin, int Cout, int Tout, int stride,
              int pad, unsigned long long seed, int layer, cudaStream_t s) {
        GemmArgs g{W.w.p, X, Y, W.has_bias ? W.bias.p : nullptr, res, noise, alpha_out, M, N, K, Cin, Tin, Cout, Tout,
                   stride, pad, seed, layer};
        dim3 grid(cdiv(N, GN), cdiv(M, GM), batch);
        switch (epi) {
            case EPI_PLAIN: gemm_f32_kernel<EPI_PLAIN><<<grid, G_THREADS, 0, s>>>(g); break;
            case EPI_RESIDUAL: gemm_f32_kernel<EPI_RESIDUAL><<<grid, G_THREADS, 0, s>>>(g); break;
            case EPI_NOISE: gemm_f32_kernel<EPI_NOISE><<<grid, G_THREADS, 0, s>>>(g); break;
            default: gemm_f32_kernel<EPI_CONVT><<<grid, G_THREADS, 0, s>>>(g); break;
        }
        count_launch();
    }

    void dwconv(const ConvW& W, const float* in, float* out, const float* a_in, const float* a_out, int batch, int C,
                int T, int dil, cudaStream_t s) {
        dim3 grid(cdiv(T, DW_TT), C, batch);
        dwconv7_kernel<<<grid, DW_THREADS, 0, s>>>(in, out, W.w.p, W.has_bias ? W.bias.p : nullptr, a_in, a_out, C, T,
                                                   dil);
        count_launch();
    }

    // codes/noise/wave are DEVICE pointers
    void decode_dev(const int* const* d_codes_in, int batch, long long T, const float* const* d_noise_in, int noise_mode,
                    unsigned long long seed, float* d_wave_out, cudaStream_t s) {
        B2A_CHECK(batch > 0 && T > 0, B2A_ERR_INVALID_INPUT, "snac decode: empty input");
        for (auto& L : levels)
            B2A_CHECK(T % L.stride == 0, B2A_ERR_INVALID_INPUT, "snac decode: t_latent must be a multiple of every vq stride");
        B2A_CHECK(T * hop < (1ll << 31) / 2, B2A_ERR_INVALID_INPUT, "snac decode: sequence too long");
        B2A_CHECK(dec_attn.window == 0 || T % dec_attn.window == 0, B2A_ERR_INVALID_INPUT,
                  "snac decode: t_latent must be a multiple of attn_window_size (LocalMHA windows)");
        B2A_CUDA(cudaSetDevice(device));
        const bool tc_fits = (long long)batch * T * hop < (1ll << 31) - 64;
        B2A_CHECK(dec_attn.dim == 0 || tc_fits, B2A_ERR_INVALID_INPUT, "snac decode: batch * t_latent * hop must be < 2^31");
        if (use_tc && tc_fits) {
            const int nb = clips_per_slice(batch, [&](int n) { return dec_workspace(n, T); });
            const long long tw = decoded_length(T);
            for (int b0 = 0; b0 < batch; b0 += nb) {
                const int n = std::min(nb, batch - b0);
                const int* dc[8];
                const float* dn[8];
                for (size_t i = 0; i < levels.size(); ++i) dc[i] = d_codes_in[i] + (long long)b0 * (T / levels[i].stride);
                long long t = T;
                for (size_t i = 0; i < blocks.size(); ++i) {
                    t = stage_len(t, blocks[i].stride);
                    dn[i] = d_noise_in && d_noise_in[i] ? d_noise_in[i] + (long long)b0 * t : nullptr;
                }
                decode_dev_tc(dc, n, T, d_noise_in ? dn : nullptr, noise_mode, seed, d_wave_out + (long long)b0 * tw, s, b0);
            }
            return;
        }
        const size_t need = max_act(batch, T);
        bufX.alloc(need);
        bufY.alloc(need);
        float *X = bufX.p, *Y = bufY.p;
        // RVQ lookup -> X [B, latent, T]
        RvqArgs ra{};
        ra.n_levels = (int)levels.size(); ra.D = cfg.codebook_dim; ra.C = latent; ra.T = (int)T;
        ra.codebook_size = cfg.codebook_size;
        for (size_t i = 0; i < levels.size(); ++i)
            ra.lv[i] = RvqLevel{d_codes_in[i], levels[i].codebook.p, levels[i].wout.p, levels[i].bout.p, levels[i].stride};
        rvq_lookup_kernel<<<dim3(cdiv(T, 256), latent, batch), 256, 0, s>>>(ra, X, 0.f, 1.f);
        count_launch();
        // depthwise k7 + 1x1 (Layers.swift:378-389); Snake of block 0 fused into the 1x1 epilogue
        dwconv(dw0, X, Y, nullptr, nullptr, batch, latent, (int)T, 1, s);
        const int C = cfg.decoder_dim;
        gemm(EPI_PLAIN, pw0, Y, X, nullptr, nullptr, blocks[0].alpha.p, batch, C, (int)T, latent, latent, (int)T, C, (int)T,
             1, 0, 0, 0, s);
        long long t = T;
        for (size_t i = 0; i < blocks.size(); ++i) {
            DecBlock& B = blocks[i];
            const long long tout = stage_len(t, B.stride);
            // transposed conv: X [cin, t] (already Snake-activated) -> Y [cout, tout]
            gemm(EPI_CONVT, B.ct, X, Y, nullptr, nullptr, nullptr, batch, B.cout * B.stride, (int)t + 1, 2 * B.cin, B.cin,
                 (int)t, B.cout, (int)tout, B.stride, B.pad, 0, 0, s);
            float* cur = Y;
            float* other = X;
            const float* nz = d_noise_in ? d_noise_in[i] : nullptr;
            if (B.has_noise && (nz || noise_mode == 0)) {
                gemm(EPI_NOISE, B.noise, cur, other, cur, nz, nullptr, batch, B.cout, (int)tout, B.cout, B.cout, (int)tout,
                     B.cout, (int)tout, 1, 0, seed, (int)i, s);
                std::swap(cur, other);
            }
            for (int u = 0; u < 3; ++u) {
                ResUnit& R = B.ru[u];
                dwconv(R.dw, cur, other, R.a0.p, R.a2.p, batch, B.cout, (int)tout, R.dil, s);
                const float* a_next = nullptr;
                if (u == 2) a_next = (i + 1 < blocks.size()) ? blocks[i + 1].alpha.p : alpha_final.p;
                gemm(EPI_RESIDUAL, R.pw, other, cur, cur, nullptr, a_next, batch, B.cout, (int)tout, B.cout, B.cout, (int)tout,
                     B.cout, (int)tout, 1, 0, 0, 0, s);
            }
            if (cur != X) std::swap(X, Y);   // keep "X" = current activations
            t = tout;
        }
        final_conv7_tanh_kernel<<<dim3(cdiv(t, FC_TT), batch), FC_THREADS, 0, s>>>(X, d_wave_out, final_conv.w.p, final_bias,
                                                                                   final_c, (int)t);
        count_launch();
        B2A_CUDA(cudaGetLastError());
    }

    // samples out of t_latent frames: every stage's length is stage_len's
    long long decoded_length(long long T) const {
        for (auto& B : blocks) T = stage_len(T, B.stride);
        return T;
    }

    // ---- encode (SNACDecoder.swift:86-105,120-125) ----------------------------------------------------------------------------
    // padded length: a multiple of hop * lcm(vq_strides, attn_window_size) (SNACDecoder.swift:86-100)
    long long enc_pad_multiple() const {
        long long l = 1;
        for (auto& L : levels) l = std::lcm(l, (long long)L.stride);
        if (cfg.attn_window_size > 0) l = std::lcm(l, (long long)cfg.attn_window_size);
        return (long long)enc_hop * l;
    }
    long long encoded_length(long long n) const {
        const long long m = enc_pad_multiple();
        return (n + m - 1) / m * m / enc_hop;
    }
    // throws unless the handle can encode `batch` clips of n samples
    void enc_check(int batch, long long n) const {
        B2A_CHECK(batch > 0 && n > 0, B2A_ERR_AUDIO_ENCODING_FAILED, "snac encode: empty audio");
        B2A_CHECK(has_enc, B2A_ERR_MODEL_NOT_INITIALIZED, enc_error);
        for (auto& L : levels) B2A_CHECK(L.win.p, B2A_ERR_MODEL_NOT_INITIALIZED, "snac encode: quantizer in_proj weights were not provided");
        B2A_CHECK(cfg.encoder_dim << cfg.n_encoder_rates == latent, B2A_ERR_INVALID_INPUT,
                  "snac encode: latent_dim must be encoder_dim * 2^len(encoder_rates)");
        for (auto& E : eblocks) B2A_CHECK(E.stride >= 2, B2A_ERR_INVALID_INPUT, "snac encode: encoder strides must be >= 2");
        const long long np = encoded_length(n) * enc_hop;
        B2A_CHECK((long long)batch * np < (1ll << 31) - 64, B2A_ERR_INVALID_INPUT, "snac encode: batch * padded samples must be < 2^31");
    }
    // stages at the fused unit's widths; the others run dw7_nlc_kernel + the conv GEMM through the hi/lo operand hA
    static bool enc_fused(const EncBlock& E) { return E.cp == 64 || E.cp == 128; }
    // largest workspace of encoding `batch` clips of T0 padded samples (elements); sets the buffer sizes when asked
    size_t enc_workspace(int batch, long long T0, size_t* mx = nullptr, size_t* mh = nullptr, size_t* mx2 = nullptr) const {
        size_t max_x = 0, max_h = 0, max_x2 = 0;
        long long t = T0;
        for (auto& E : eblocks) {
            max_x = std::max<size_t>(max_x, (size_t)batch * t * E.cp);
            if (!enc_fused(E)) max_h = std::max<size_t>(max_h, (size_t)(2 * pad64((long long)batch * t)) * E.cp);   // dw7 -> GEMM operand
            t /= E.stride;
            max_x2 = std::max<size_t>(max_x2, (size_t)(2 * pad64((long long)batch * (t + 1))) * 2 * E.stride * E.cp);
            max_x = std::max<size_t>(max_x, (size_t)batch * t * E.cp_out);
        }
        if (enc_attn.dim) max_h = std::max<size_t>(max_h, (size_t)(2 * pad64((long long)batch * t)) * latent);   // LocalMHA operands
        if (mx) { *mx = max_x; *mh = max_h; *mx2 = max_x2; }
        return std::max(max_x, std::max(max_h, max_x2));
    }
    // d_wave [B, n] -> z [B, latent, T_lat] fp32 NCT in d_zenc (returned), in slices of whole clips (clips_per_slice)
    float* encode_latent_dev(const float* d_wave_in, int batch, long long n, cudaStream_t s) {
        const long long tl = encoded_length(n), T0 = tl * enc_hop;
        d_zenc.alloc((size_t)batch * latent * tl);
        const int nb = clips_per_slice(batch, [&](int c) { return enc_workspace(c, T0); });
        for (int b0 = 0; b0 < batch; b0 += nb)
            encode_latent_slice(d_wave_in + (long long)b0 * n, std::min(nb, batch - b0), n, d_zenc.p + (long long)b0 * latent * tl, s);
        return d_zenc.p;
    }
    // channels-last fp32 stream + bf16 hi/lo GEMM operands
    void encode_latent_slice(const float* d_wave_in, int batch, long long n, float* d_z, cudaStream_t s) {
        const long long tl = encoded_length(n), T0 = tl * enc_hop;
        size_t max_x, max_h, max_x2;
        enc_workspace(batch, T0, &max_x, &max_h, &max_x2);
        max_x = std::max<size_t>(max_x, (size_t)batch * tl * latent);
        xs.alloc(max_x); xs2.alloc(max_x); hA.alloc(max_h); x2.alloc(max_x2);
        {
            const int cp0 = eblocks[0].cp;
            const long long nthr = (long long)batch * T0 * (cp0 / 4);
            enc_stem_kernel<<<(unsigned)((nthr + 255) / 256), 256, 0, s>>>(d_wave_in, xs.p, enc_stem.w.p, enc_stem.bias.p, batch, n, (int)T0, cp0);
            count_launch();
        }
        long long t = T0;
        for (size_t i = 0; i < eblocks.size(); ++i) {
            EncBlock& E = eblocks[i];
            const long long tout = t / E.stride, ntok = (long long)batch * t;
            if (enc_fused(E)) {
                // fused ResidualUnits, fp32 in -> fp32 out (ping-pong xs <-> xs2); the last one also writes Snake(alpha) of its
                // output into the strided conv's 2-frame im2col
                for (int u = 0; u < 3; ++u) {
                    ResUnit& R = E.ru[u];
                    rf::Args a{};
                    a.x = xs.p; a.y = xs2.p; a.C = E.cp; a.mode = rf::MODE_RU; a.dil = R.dil;
                    a.dw_w = R.dw.w.p; a.dw_b = R.dw.bias.p; a.a_in = R.a0.p; a.a_mid = R.a2.p; a.pw_bias = R.pw.bias.p;
                    if (u == 2) { a.hl = x2.p; a.a_next = E.alpha.p; a.fs = E.stride; a.fpad = E.pad; }
                    fused(E.cp == 64 ? R.pw_bd : R.pw_tc, a, batch, t, s);
                    std::swap(xs.p, xs2.p); std::swap(xs.n, xs2.n);
                }
            } else {
                for (int u = 0; u < 3; ++u) {
                    ResUnit& R = E.ru[u];
                    dw_nlc(R.dw, xs.p, hA.p, R.a0.p, R.a2.p, batch, (int)t, E.cp, R.dil, s);
                    cg::Args a{};
                    a.N = (int)ntok; a.bias = R.pw.bias.p; a.x = xs.p; a.ldx = E.cp; a.T = (int)t;
                    if (u == 2) { a.epi = cg::E_ADD_HILO; a.alpha = E.alpha.p; a.hl = x2.p; a.fs = E.stride; a.fpad = E.pad; }
                    else a.epi = cg::E_ADD;
                    cg::launch(R.pw_tc, hA.p, 2 * pad64(ntok), a, num_sms, s);
                }
            }
            // after the units (it writes other positions of x2): a plain launch between the last fused unit and the strided conv's
            // GEMM, whose TMA producer reads x2 without waiting on the programmatic dependency
            frames_zero_edges_kernel<<<batch, 256, 0, s>>>(x2.p, (int)t, E.stride, E.pad, E.cp);
            count_launch();
            {   // strided conv = 2-tap GEMM over the frames: token (b, q), q = 0..tout (q = tout dropped) -> fp32 [B*tout, cp_out] + bias
                cg::Args a{};
                a.N = (int)(batch * (tout + 1)); a.epi = cg::E_CONVT; a.bias = E.down_b.bias.p;
                a.x = xs.p; a.ldx = E.cp_out; a.T = (int)tout; a.Cout = E.cp_out; a.stride = 1; a.pad = 0; a.Tin = (int)tout;
                cg::launch(E.down, x2.p, 2 * pad64((long long)batch * (tout + 1)), a, num_sms, s);
            }
            t = tout;
        }
        if (enc_attn.dim) {          // LocalMHA (Layers.swift:339-341) adds into the last block's output, ld = cp_out = latent
            cg::Args o{};
            o.epi = cg::E_ADD;
            local_mha(enc_attn, xs.p, batch, t, o, s);
        }
        enc_final_dw_kernel<<<dim3(cdiv(t, 32), cdiv(latent, 32), batch), dim3(32, 8), 0, s>>>(xs.p, d_z, enc_final.w.p, enc_final.bias.p,
                                                                                             (int)t, latent, eblocks.back().cp_out);
        count_launch();
        B2A_CUDA(cudaGetLastError());
    }
    // residual VQ (VQ.swift:47-120,150-163) of d_res = z [B, latent, T] fp32 on the device (left holding the final residual):
    // codes of level i -> d_codes_out[i] [B, T / stride_i]; z_q accumulated into d_zq_out when non-null
    void quantize_dev(float* d_res, int batch, long long T, int* const* d_codes_out, float* d_zq_out, cudaStream_t s) {
        const int C = latent, D = cfg.codebook_dim;
        if (d_zq_out) B2A_CUDA(cudaMemsetAsync(d_zq_out, 0, (size_t)batch * C * T * sizeof(float), s));
        for (size_t i = 0; i < levels.size(); ++i) {
            auto& L = levels[i];
            const int Ts = (int)(T / L.stride), N = batch * Ts;
            d_ze.alloc((size_t)N * D);
            vq_inproj_kernel<<<dim3(cdiv(Ts, 64), batch), 64, 0, s>>>(d_res, L.win.p, L.bin.p, d_ze.p, C, (int)T, L.stride, D);
            count_launch();
            nearest(d_ze.p, N, d_codes_out[i], L, s);
            RvqArgs ra{};
            ra.n_levels = 1; ra.D = D; ra.C = C; ra.T = (int)T; ra.codebook_size = cfg.codebook_size;
            ra.lv[0] = RvqLevel{d_codes_out[i], L.codebook.p, L.wout.p, L.bout.p, L.stride};
            if (d_zq_out) {
                rvq_lookup_kernel<<<dim3(cdiv(T, 256), C, batch), 256, 0, s>>>(ra, d_zq_out, 1.f, 1.f);    // zQ += zQ_i
                count_launch();
            }
            rvq_lookup_kernel<<<dim3(cdiv(T, 256), C, batch), 256, 0, s>>>(ra, d_res, 1.f, -1.f);         // residual -= zQ_i
            count_launch();
        }
        B2A_CUDA(cudaGetLastError());
    }

    void nearest(const float* d_enc, int N, int* d_out_idx, const Level& L, cudaStream_t s) {
        const int D = cfg.codebook_dim;
        d_en.alloc((size_t)N * D);
        d_e2.alloc(N);
        l2_normalize_rows_kernel<<<cdiv(N, 128), 128, 0, s>>>(d_enc, d_en.p, d_e2.p, N, D);
        const size_t sm = (size_t)NC_TILE * (D + 1) * sizeof(float);
        B2A_CUDA(cudaFuncSetAttribute(nearest_code_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        nearest_code_kernel<<<cdiv(N, NC_THREADS), NC_THREADS, sm, s>>>(d_en.p, d_e2.p, L.cb_n.p, L.cb_n2.p, d_out_idx, N,
                                                                        cfg.codebook_size, D);
        count_launch(2);
    }
};

extern "C" {

int32_t b2a_snac_create(int32_t device, const b2a_snac_config* cfg, const b2a_tensor* tensors, int32_t n,
                        b2a_snac** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_snac_create: null out");
        *out = nullptr;
        B2A_CHECK(cfg && tensors && n > 0, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_snac_create: missing config or weights");
        TensorTable tt(tensors, n);
        *out = new b2a_snac(device, *cfg, tt);
    });
}

int64_t b2a_snac_hop_length(const b2a_snac* h) { return h ? h->hop : 0; }
int64_t b2a_snac_decoded_length(const b2a_snac* h, int64_t t_latent) { return h && t_latent > 0 ? h->decoded_length(t_latent) : 0; }
void* b2a_snac_stream(b2a_snac* h) { return h ? (void*)h->stream : nullptr; }

int32_t b2a_snac_decode_dev(b2a_snac* h, const int32_t* const* d_codes, int32_t batch, int64_t T,
                            const float* const* d_noise, int32_t noise_mode, uint64_t seed, float* d_wave, void* stream) {
    return guarded([&] {
        B2A_CHECK(h && d_codes && d_wave, B2A_ERR_INVALID_INPUT, "b2a_snac_decode_dev: null argument");
        h->decode_dev(d_codes, batch, T, d_noise, noise_mode, seed, d_wave, (cudaStream_t)stream);
    });
}

int32_t b2a_snac_decode(b2a_snac* h, const int32_t* const* codes, int32_t batch, int64_t T, const float* const* noise,
                        int32_t noise_mode, uint64_t seed, float* wave) {
    return guarded([&] {
        B2A_CHECK(h && codes && wave, B2A_ERR_INVALID_INPUT, "b2a_snac_decode: null argument");
        B2A_CHECK(batch > 0 && T > 0, B2A_ERR_INVALID_INPUT, "b2a_snac_decode: empty input");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        const int nl = (int)h->levels.size();
        const int* dc[8];
        for (int i = 0; i < nl; ++i) {
            B2A_CHECK(codes[i], B2A_ERR_INVALID_INPUT, "b2a_snac_decode: null code layer");
            const size_t n = (size_t)batch * (T / h->levels[i].stride);
            h->d_codes[i].alloc(n);
            B2A_CUDA(cudaMemcpyAsync(h->d_codes[i].p, codes[i], n * sizeof(int), cudaMemcpyHostToDevice, s));
            dc[i] = h->d_codes[i].p;
        }
        const float* dn[8] = {nullptr};
        bool any_noise = false;
        long long t = T;
        for (size_t i = 0; i < h->blocks.size(); ++i) {
            t = stage_len(t, h->blocks[i].stride);
            if (noise && noise[i]) {
                h->d_noise[i].alloc((size_t)batch * t);
                B2A_CUDA(cudaMemcpyAsync(h->d_noise[i].p, noise[i], (size_t)batch * t * sizeof(float), cudaMemcpyHostToDevice, s));
                dn[i] = h->d_noise[i].p;
                any_noise = true;
            }
        }
        h->d_wave.alloc((size_t)batch * t);
        h->decode_dev(dc, batch, T, any_noise ? dn : nullptr, noise_mode, seed, h->d_wave.p, s);
        B2A_CUDA(cudaMemcpyAsync(wave, h->d_wave.p, (size_t)batch * t * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

int32_t b2a_snac_quantize(b2a_snac* h, const float* z, int32_t batch, int64_t T, int32_t* const* codes, float* z_q) {
    return guarded([&] {
        B2A_CHECK(h && z && codes, B2A_ERR_INVALID_INPUT, "b2a_snac_quantize: null argument");
        B2A_CHECK(batch > 0 && T > 0, B2A_ERR_AUDIO_ENCODING_FAILED, "b2a_snac_quantize: empty input");
        for (auto& L : h->levels) {
            B2A_CHECK(T % L.stride == 0, B2A_ERR_AUDIO_ENCODING_FAILED, "b2a_snac_quantize: T must be a multiple of every vq stride");
            B2A_CHECK(L.win.p, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_snac_quantize: in_proj weights were not provided");
        }
        for (size_t i = 0; i < h->levels.size(); ++i) B2A_CHECK(codes[i], B2A_ERR_INVALID_INPUT, "b2a_snac_quantize: null code output");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        const size_t n = (size_t)batch * h->latent * T;
        h->bufX.alloc(n);   // residual
        B2A_CUDA(cudaMemcpyAsync(h->bufX.p, z, n * sizeof(float), cudaMemcpyHostToDevice, s));
        if (z_q) h->d_zq.alloc(n);
        int* dc[8];
        for (size_t i = 0; i < h->levels.size(); ++i) {
            h->d_codes[i].alloc((size_t)batch * (T / h->levels[i].stride));
            dc[i] = h->d_codes[i].p;
        }
        h->quantize_dev(h->bufX.p, batch, T, dc, z_q ? h->d_zq.p : nullptr, s);
        for (size_t i = 0; i < h->levels.size(); ++i)
            B2A_CUDA(cudaMemcpyAsync(codes[i], dc[i], (size_t)batch * (T / h->levels[i].stride) * sizeof(int), cudaMemcpyDeviceToHost, s));
        if (z_q) B2A_CUDA(cudaMemcpyAsync(z_q, h->d_zq.p, n * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
        B2A_CUDA(cudaGetLastError());
    });
}

int64_t b2a_snac_encoded_length(const b2a_snac* h, int64_t n_samples) {
    return h && h->has_enc && n_samples > 0 ? h->encoded_length(n_samples) : 0;
}

int32_t b2a_snac_encode_dev(b2a_snac* h, const float* d_wave, int32_t batch, int64_t n_samples, int32_t* const* d_codes, void* stream) {
    return guarded([&] {
        B2A_CHECK(h && d_wave && d_codes, B2A_ERR_INVALID_INPUT, "b2a_snac_encode_dev: null argument");
        h->enc_check(batch, n_samples);
        for (size_t i = 0; i < h->levels.size(); ++i) B2A_CHECK(d_codes[i], B2A_ERR_INVALID_INPUT, "b2a_snac_encode_dev: null code output");
        B2A_CUDA(cudaSetDevice(h->device));
        const cudaStream_t s = (cudaStream_t)stream;
        float* z = h->encode_latent_dev(d_wave, batch, n_samples, s);
        h->quantize_dev(z, batch, h->encoded_length(n_samples), d_codes, nullptr, s);
    });
}

int32_t b2a_snac_encode(b2a_snac* h, const float* wave, int32_t batch, int64_t n_samples, int32_t* const* codes) {
    return guarded([&] {
        B2A_CHECK(h && wave && codes, B2A_ERR_INVALID_INPUT, "b2a_snac_encode: null argument");
        h->enc_check(batch, n_samples);
        for (size_t i = 0; i < h->levels.size(); ++i) B2A_CHECK(codes[i], B2A_ERR_INVALID_INPUT, "b2a_snac_encode: null code output");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        const long long tl = h->encoded_length(n_samples);
        h->d_ewave.alloc((size_t)batch * n_samples);
        B2A_CUDA(cudaMemcpyAsync(h->d_ewave.p, wave, (size_t)batch * n_samples * sizeof(float), cudaMemcpyHostToDevice, s));
        int* dc[8];
        for (size_t i = 0; i < h->levels.size(); ++i) {
            h->d_codes[i].alloc((size_t)batch * (tl / h->levels[i].stride));
            dc[i] = h->d_codes[i].p;
        }
        float* z = h->encode_latent_dev(h->d_ewave.p, batch, n_samples, s);
        h->quantize_dev(z, batch, tl, dc, nullptr, s);
        for (size_t i = 0; i < h->levels.size(); ++i)
            B2A_CUDA(cudaMemcpyAsync(codes[i], dc[i], (size_t)batch * (tl / h->levels[i].stride) * sizeof(int), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
        B2A_CUDA(cudaGetLastError());
    });
}

void b2a_snac_destroy(b2a_snac* h) { delete h; }

}  // extern "C"

// Single-kernel entries (include/b200audio_internal.h): one launch of the conv GEMM, of a fused ResidualUnit / NoiseBlock or of the
// fused Snake + transposed conv, through the engine's launch code.  Activations are DEVICE pointers; the weights are host fp32 and
// take the constructor's path (the same layout helpers, then TcW::build's hi/lo split).  ctas = 0: the engine's CTA count.
static long long hook_ctas(int32_t ctas) {
    if (ctas > 0) return ctas;
    int n = 0;
    B2A_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, 0));
    return n;
}

extern "C" int32_t b2a_conv_gemm_test(const float* w, int32_t M, int32_t K, const void* X, int32_t N, int32_t epi, const float* bias,
                                      const float* alpha, const float* gamma, int32_t gelu, float* x, int32_t ldx, void* hl, int32_t ldh,
                                      int32_t dual, int32_t T, int32_t Cout, int32_t stride, int32_t pad, int32_t Tin, const float* noise,
                                      uint64_t seed, int32_t ctas, void* stream) {
    return guarded([&] {
        B2A_CHECK(w && X && M > 0 && K > 0 && K % tc::BK == 0 && N > 0 && ctas >= 0 && (gelu == 0 || gelu == 1) && (dual == 0 || dual == 1),
                  B2A_ERR_INVALID_INPUT, "b2a_conv_gemm_test: bad argument");
        B2A_CHECK(epi >= cg::E_STORE_HILO && epi <= cg::E_STORE_F32, B2A_ERR_INVALID_INPUT, "b2a_conv_gemm_test: unknown epilogue");
        const bool hilo_out = epi == cg::E_STORE_HILO || epi == cg::E_ADD_HILO;
        B2A_CHECK(epi == cg::E_STORE_HILO ? !x : (x && ldx >= (epi == cg::E_CONVT ? Cout : M)), B2A_ERR_INVALID_INPUT,
                  "b2a_conv_gemm_test: every epilogue but cg::E_STORE_HILO writes the fp32 x (ldx >= its columns)");
        B2A_CHECK(hilo_out ? hl != nullptr : (!hl || epi == cg::E_CONVT), B2A_ERR_INVALID_INPUT,
                  "b2a_conv_gemm_test: hl is the output of cg::E_STORE_HILO / cg::E_ADD_HILO and the optional copy of cg::E_CONVT");
        B2A_CHECK(!hl || ldh >= (dual ? 2 * M : epi == cg::E_CONVT ? Cout : M), B2A_ERR_INVALID_INPUT, "b2a_conv_gemm_test: ldh too small");
        B2A_CHECK(!alpha || hilo_out, B2A_ERR_INVALID_INPUT, "b2a_conv_gemm_test: Snake applies to the hi/lo outputs only");
        B2A_CHECK(!dual || (hilo_out && T >= 1 && N % T == 0), B2A_ERR_INVALID_INPUT,
                  "b2a_conv_gemm_test: the 2-tap im2col (dual) is a hi/lo output of whole utterances of T tokens");
        B2A_CHECK(epi != cg::E_ADD_HILO || dual, B2A_ERR_INVALID_INPUT, "b2a_conv_gemm_test: cg::E_ADD_HILO feeds the next transposed conv (dual)");
        B2A_CHECK(!gelu || epi == cg::E_STORE_HILO, B2A_ERR_INVALID_INPUT, "b2a_conv_gemm_test: GELU is the Vocos pwconv1 epilogue (cg::E_STORE_HILO)");
        B2A_CHECK(!gamma || epi == cg::E_ADD, B2A_ERR_INVALID_INPUT, "b2a_conv_gemm_test: gamma is the ConvNeXt residual add (cg::E_ADD)");
        B2A_CHECK(epi == cg::E_NOISE ? !bias : (!noise && seed == 0), B2A_ERR_INVALID_INPUT,
                  "b2a_conv_gemm_test: noise / seed belong to cg::E_NOISE, whose linear has no bias");
        B2A_CHECK(epi != cg::E_CONVT || (Cout > 0 && stride >= 1 && M == stride * Cout && pad >= 0 && Tin >= 1 && N % (Tin + 1) == 0 &&
                                     T == Tin * stride),
                  B2A_ERR_INVALID_INPUT, "b2a_conv_gemm_test: cg::E_CONVT needs M = stride * Cout, N = B * (Tin + 1) and T = Tin * stride");
        require_device(0);
        TcW W;
        W.build(std::vector<float>(w, w + (size_t)M * K), M, 1, K);
        cg::Args a{};
        a.N = N; a.epi = epi; a.bias = bias; a.alpha = alpha; a.gamma = gamma; a.gelu = gelu; a.x = x; a.ldx = ldx;
        a.hl = (__nv_bfloat16*)hl; a.ldh = ldh; a.dual = dual; a.T = T; a.Cout = Cout; a.stride = stride; a.pad = pad; a.Tin = Tin;
        a.noise = noise; a.seed = seed;
        const cudaStream_t s = (cudaStream_t)stream;
        cg::launch(W, (const __nv_bfloat16*)X, 2 * b2a_snac::pad64(N), a, hook_ctas(ctas), s);
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

extern "C" int32_t b2a_snac_unit_test(int32_t mode, int32_t C, int32_t dil, const float* x, float* y, int32_t B, int32_t T,
                                      const float* dw_w, const float* dw_b, const float* a_in, const float* a_mid, const float* pw_w,
                                      const float* pw_bias, const float* noise, uint64_t seed, void* hl, const float* a_next, int32_t ctas,
                                      void* stream) {
    return guarded([&] {
        B2A_CHECK(x && y && x != y && pw_w && (C == 64 || C == 128) && B >= 1 && T >= 1 && (long long)B * T < (1ll << 31) - 64 && ctas >= 0,
                  B2A_ERR_INVALID_INPUT, "b2a_snac_unit_test: bad argument");
        if (mode == rf::MODE_RU)
            B2A_CHECK((dil == 1 || dil == 3 || dil == 9) && dw_w && a_in && a_mid && !noise && seed == 0, B2A_ERR_INVALID_INPUT,
                      "b2a_snac_unit_test: a ResidualUnit takes dil 1, 3 or 9, the depthwise weight and both Snake alphas, and no noise");
        else
            B2A_CHECK(mode == rf::MODE_NOISE && dil == 0 && !dw_w && !dw_b && !a_in && !a_mid && !pw_bias && !hl, B2A_ERR_INVALID_INPUT,
                      "b2a_snac_unit_test: a NoiseBlock is x + noise * (W x): no depthwise conv, bias or hi/lo copy");
        B2A_CHECK(!hl == !a_next, B2A_ERR_INVALID_INPUT, "b2a_snac_unit_test: the hi/lo copy is Snake(a_next) of y");
        require_device(0);
        b2a_snac::fused_attrs<64>();
        b2a_snac::fused_attrs<128>();
        std::vector<float> pw(pw_w, pw_w + (size_t)C * C);
        TcW W;                                              // the [128, 128] operand: W itself (C = 128) or [W 0; 0 W] (C = 64)
        W.build(C == 64 ? block_diag2(pw) : pw, 128, 1, 128);
        rf::Args a{};
        a.x = x; a.y = y; a.C = C; a.mode = mode; a.dil = dil; a.dw_w = dw_w; a.dw_b = dw_b; a.a_in = a_in; a.a_mid = a_mid;
        a.pw_bias = pw_bias; a.noise = noise; a.seed = seed; a.hl = (__nv_bfloat16*)hl; a.a_next = a_next;
        const cudaStream_t s = (cudaStream_t)stream;
        b2a_snac::launch_fused(W, a, B, T, hook_ctas(ctas), s);
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

extern "C" int32_t b2a_snac_convt_test(const float* x, float* y, const float* alpha, const float* bias, const float* w, int32_t B,
                                       int32_t Tin, int32_t stride, int32_t cout, int32_t ctas, void* stream) {
    return guarded([&] {
        constexpr int CIN = 128;
        B2A_CHECK(x && y && alpha && w && B >= 1 && Tin >= 1 && ctas >= 0 && (long long)B * Tin * stride < (1ll << 31) - 64,
                  B2A_ERR_INVALID_INPUT, "b2a_snac_convt_test: bad argument");
        B2A_CHECK((stride == 2 && cout == 64) || (stride == 1 && cout == 128), B2A_ERR_INVALID_INPUT,
                  "b2a_snac_convt_test: the fused transposed conv maps 128 channels to stride * cout = 128 phase rows");
        require_device(0);
        B2A_CUDA(cudaFuncSetAttribute(rf::convt_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rf::convt_smem_bytes()));
        const int k = 2 * stride;
        std::vector<float> wt((size_t)CIN * k * cout);      // torch [ci, co, k] -> the checkpoint's [ci, k, co]
        for (int ci = 0; ci < CIN; ++ci)
            for (int co = 0; co < cout; ++co)
                for (int j = 0; j < k; ++j) wt[((size_t)ci * k + j) * cout + co] = w[((size_t)ci * cout + co) * k + j];
        TcW W;
        W.build(convt_phase_major(convt_gemm_rows(wt, CIN, cout, stride), CIN, cout, stride), stride * cout, 1, 2 * CIN);
        rf::ConvtArgs a{};
        a.x = x; a.y = y; a.alpha = alpha; a.bias = bias;
        a.Tin = Tin; a.T = Tin * stride; a.B = B; a.stride = stride; a.cout = cout; a.pad = (stride + 1) / 2;    // DecBlock::pad
        const cudaStream_t s = (cudaStream_t)stream;
        b2a_snac::launch_convt(W, a, hook_ctas(ctas), s);
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

// One launch of LocalMHA's window core (local_attn_kernel) on HOST data: qkv fp32 [B * T, 3 dim] (q | k | v, rotary not yet applied),
// inv_freq [32] -> out fp32 [B * T, dim] (the hi + lo pair the kernel writes for to_out), T a multiple of the window.
extern "C" int32_t b2a_snac_local_attn_test(const float* qkv, const float* inv_freq, int32_t B, int32_t T, int32_t dim, int32_t window,
                                            float* out) {
    return guarded([&] {
        B2A_CHECK(qkv && inv_freq && out && B >= 1 && T >= 1 && dim >= LA_D && dim % LA_D == 0 && window >= 1 && window <= LA_MAXW &&
                      T % window == 0 && (long long)B * T * 3 * dim < (1ll << 31),
                  B2A_ERR_INVALID_INPUT, "b2a_snac_local_attn_test: bad argument");
        require_device(0);
        const long long ntok = (long long)B * T, rows = 2 * b2a_snac::pad64(ntok);
        DBuf<float> dq, dr;
        DBuf<__nv_bfloat16> dh;
        dq.upload(qkv, (size_t)ntok * 3 * dim);
        dh.alloc((size_t)rows * dim);
        const std::vector<float> r = rope_table(inv_freq, window);
        dr.upload(r.data(), r.size());
        local_attn_kernel<<<dim3(T / window, dim / LA_D, B), LA_THREADS>>>(dq.p, dr.p, dh.p, T, dim, window);
        B2A_CUDA(cudaGetLastError());
        std::vector<uint16_t> hl((size_t)rows * dim);
        B2A_CUDA(cudaMemcpy(hl.data(), dh.p, hl.size() * sizeof(uint16_t), cudaMemcpyDeviceToHost));
        for (long long t = 0; t < ntok; ++t) {
            const long long rr = (t / 64) * 128 + t % 64;
            for (int c = 0; c < dim; ++c) out[t * dim + c] = cg::join16(hl[rr * dim + c], hl[(rr + 64) * dim + c], 0);
        }
    });
}

// The device encoder's latent (before the code search) on HOST data: wave [B, n] -> z [B, latent, b2a_snac_encoded_length(n)].
extern "C" int32_t b2a_snac_encode_latent_test(b2a_snac* h, const float* wave, int32_t batch, int64_t n_samples, float* z) {
    return guarded([&] {
        B2A_CHECK(h && wave && z, B2A_ERR_INVALID_INPUT, "b2a_snac_encode_latent_test: null argument");
        h->enc_check(batch, n_samples);
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        h->d_ewave.alloc((size_t)batch * n_samples);
        B2A_CUDA(cudaMemcpyAsync(h->d_ewave.p, wave, (size_t)batch * n_samples * sizeof(float), cudaMemcpyHostToDevice, s));
        const float* dz = h->encode_latent_dev(h->d_ewave.p, batch, n_samples, s);
        B2A_CUDA(cudaMemcpyAsync(z, dz, (size_t)batch * h->latent * h->encoded_length(n_samples) * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
        B2A_CUDA(cudaGetLastError());
    });
}
