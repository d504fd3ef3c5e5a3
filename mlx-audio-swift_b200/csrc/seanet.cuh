// SEANet encoder building blocks shared by the Encodec (encodec.cu) and Qwen3-TTS speech-tokenizer (speech_tokenizer.cu)
// encoders: the fp32 implicit-GEMM conv with the ELU of its input fused, the stem from 1-2 audio channels, and the residual code
// search in ordered fp32 (DESIGN.md §3.6b).  Both encoders pad their convs causally by kernel - stride at dilation 1:
// Encodec's paddingTotal = kernelSize - stride (EncodecLayers.swift:118, extra right padding :137-139) equals Mimi's
// kEff - stride (Mimi/Conv.swift:207-211), and one residual layer per stage keeps every encoder conv at dilation 1.
// The Qwen3-TTS speaker encoder (speaker_encoder.cu) runs its convs on the same conv kernel, with the dilation, channel-slice
// strides, input addend and ReLU / tanh epilogue that only it sets (DESIGN.md §3.8c).
#pragma once
#include "common.cuh"

#include <utility>

namespace b2a {
namespace ec {

__device__ __forceinline__ float elu1(float v) { return v > 0.f ? v : expm1f(v); }

// ------------------------------------------------------------------ implicit-GEMM conv / transposed conv
struct ConvArgs {
    // source A: taps over xa [N, La, Ca]
    const float* xa; int La, Ca, taps, padL, reflect, elu_a, backward;   // forward: src = q*stride + tap - padL; backward: src = q - tap
    int edge = 0;            // forward only: out-of-range rows replicate the nearest edge row (Mimi's ConvDownsample1d pads with .edge)
    int stride = 1;          // forward only: an encoder downsampling conv (k = 2s) gathers its 2s contiguous rows per output
    int dil = 1;             // forward only: tap spacing (src = q*stride + tap*dil - padL)
    int lda = 0;             // row stride of xa in floats (0: Ca), so a conv can read a channel slice of a wider tensor
    const float* xa_add = nullptr;   // optional second addend of xa, same addressing: the conv reads xa + xa_add
    // source B (optional): one tap at src = q over xb [N, Lq, Cb]
    const float* xb; int Cb, elu_b;
    int ldb = 0;             // row stride of xb in floats (0: Cb)
    const float* A;          // [M, K] row-major, K = taps*Ca + Cb
    const float* bias;       // [M] or null
    const float* res;        // optional residual, same addressing as out
    float* out;              // [N, Tout, Cout]; element (q, m) lives at q*M + m - shift, valid inside [0, Tout*Cout)
    int M, K, Lq, N;
    long long out_per_n;     // Tout * Cout
    long long shift;         // pl * Cout (left trim of a transposed conv)
    int ldo = 0;             // output row stride in floats (0: M), so a conv can write a channel slice of a wider tensor
    int act = 0;             // epilogue after bias and residual: 1 ReLU, 2 tanh(ReLU)
    long long bias_n = 0;    // bias stride per batch row n (0: one bias for all rows)
};

constexpr int BK = 16;

__device__ __forceinline__ int src_index(int q, int tap, const ConvArgs& a) {
    if (a.backward) {
        const int s = q - tap;
        return (s >= 0 && s < a.La) ? s : -1;
    }
    int s = q * a.stride + tap * a.dil - a.padL;
    if (s < 0) return a.edge ? 0 : a.reflect ? min(-s, a.La - 1) : -1;
    if (s >= a.La) return a.edge ? a.La - 1 : a.reflect ? max(a.La - 2 - (s - a.La), 0) : -1;
    return s;
}

// BM outputs x BT tokens per CTA, 256 threads, thread (tx = tid % 16 -> m, ty = tid / 16 -> token).
template <int BM, int BT>
__global__ void __launch_bounds__(256) ec_conv_kernel(ConvArgs a) {
    constexpr int RM = BM / 16, RT = BT / 16;
    __shared__ __align__(16) float As[BK][BM + 4];
    __shared__ __align__(16) float Xs[BK][BT + 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int n = blockIdx.z;
    const int q0 = blockIdx.x * BT, m0 = blockIdx.y * BM;
    const int Ka = a.taps * a.Ca;
    float acc[RM][RT];
#pragma unroll
    for (int i = 0; i < RM; ++i)
#pragma unroll
        for (int j = 0; j < RT; ++j) acc[i][j] = 0.f;

    // register double buffering: the global loads of k-tile i+1 are in flight while tile i is multiplied out of shared memory
    constexpr int NA = (BM * 4 + 255) / 256, NX = (BT * 4 + 255) / 256;
    float4 ra[NA], rx[NX];
    auto load_tiles = [&](int k0) {
#pragma unroll
        for (int i = 0; i < NA; ++i) {
            const int e = tid + i * 256;
            const int m = e >> 2, k4 = (e & 3) * 4;
            ra[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (e < BM * 4 && m0 + m < a.M && k0 + k4 < a.K) ra[i] = *reinterpret_cast<const float4*>(a.A + (long long)(m0 + m) * a.K + k0 + k4);
        }
#pragma unroll
        for (int i = 0; i < NX; ++i) {
            const int e = tid + i * 256;
            const int t = e >> 2, k4 = (e & 3) * 4;
            const int q = q0 + t, kk = k0 + k4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (e < BT * 4 && q < a.Lq && kk < a.K) {
                if (kk < Ka) {
                    const int tap = kk / a.Ca, ci = kk - tap * a.Ca;
                    const int s = src_index(q, tap, a);
                    if (s >= 0) {
                        const long long off = ((long long)n * a.La + s) * (a.lda ? a.lda : a.Ca) + ci;
                        v = *reinterpret_cast<const float4*>(a.xa + off);
                        if (a.xa_add) {
                            const float4 u = *reinterpret_cast<const float4*>(a.xa_add + off);
                            v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w;
                        }
                        if (a.elu_a) { v.x = elu1(v.x); v.y = elu1(v.y); v.z = elu1(v.z); v.w = elu1(v.w); }
                    }
                } else {
                    v = *reinterpret_cast<const float4*>(a.xb + ((long long)n * a.Lq + q) * (a.ldb ? a.ldb : a.Cb) + (kk - Ka));
                    if (a.elu_b) { v.x = elu1(v.x); v.y = elu1(v.y); v.z = elu1(v.z); v.w = elu1(v.w); }
                }
            }
            rx[i] = v;
        }
    };
    auto store_tiles = [&]() {
#pragma unroll
        for (int i = 0; i < NA; ++i) {
            const int e = tid + i * 256;
            if (e < BM * 4) {
                const int m = e >> 2, k4 = (e & 3) * 4;
                As[k4 + 0][m] = ra[i].x; As[k4 + 1][m] = ra[i].y; As[k4 + 2][m] = ra[i].z; As[k4 + 3][m] = ra[i].w;
            }
        }
#pragma unroll
        for (int i = 0; i < NX; ++i) {
            const int e = tid + i * 256;
            if (e < BT * 4) {
                const int t = e >> 2, k4 = (e & 3) * 4;
                Xs[k4 + 0][t] = rx[i].x; Xs[k4 + 1][t] = rx[i].y; Xs[k4 + 2][t] = rx[i].z; Xs[k4 + 3][t] = rx[i].w;
            }
        }
    };
    load_tiles(0);
    store_tiles();
    __syncthreads();
    for (int k0 = 0; k0 < a.K; k0 += BK) {
        const bool more = k0 + BK < a.K;
        if (more) load_tiles(k0 + BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float av[RM], xv[RT];
#pragma unroll
            for (int i = 0; i < RM; ++i) av[i] = As[k][tx + 16 * i];
#pragma unroll
            for (int j = 0; j < RT; ++j) xv[j] = Xs[k][ty + 16 * j];
#pragma unroll
            for (int i = 0; i < RM; ++i)
#pragma unroll
                for (int j = 0; j < RT; ++j) acc[i][j] = fmaf(av[i], xv[j], acc[i][j]);
        }
        __syncthreads();
        if (more) {
            store_tiles();
            __syncthreads();
        }
    }
    float* outn = a.out + (long long)n * a.out_per_n;
    const float* resn = a.res ? a.res + (long long)n * a.out_per_n : nullptr;
    const float* biasn = a.bias ? a.bias + (long long)n * a.bias_n : nullptr;
    const int ldo = a.ldo ? a.ldo : a.M;
#pragma unroll
    for (int j = 0; j < RT; ++j) {
        const int q = q0 + ty + 16 * j;
        if (q >= a.Lq) continue;
#pragma unroll
        for (int i = 0; i < RM; ++i) {
            const int m = m0 + tx + 16 * i;
            if (m >= a.M) continue;
            const long long o = (long long)q * ldo + m - a.shift;
            if (o < 0 || o >= a.out_per_n) continue;
            float v = acc[i][j] + (biasn ? biasn[m] : 0.f);
            if (resn) v += resn[o];
            if (a.act) { v = fmaxf(v, 0.f); if (a.act == 2) v = tanhf(v); }
            outn[o] = v;
        }
    }
}


// a dense conv as ec_conv_kernel reads it: A [M, K] with K = taps * Cin (+ Cb for a second source), bias [M]
struct Conv {
    DBuf<float> A, bias;
    int M = 0, K = 0;
};

// one ec_conv_kernel launch, the tile shape picked by the output width
inline void launch_conv(const ConvArgs& a, cudaStream_t s) {
    const int M = a.M;
    if (M >= 64) {
        dim3 g(cdiv(a.Lq, 64), cdiv(M, 64), a.N);
        ec_conv_kernel<64, 64><<<g, 256, 0, s>>>(a);
    } else if (M >= 32) {
        dim3 g(cdiv(a.Lq, 128), cdiv(M, 32), a.N);
        ec_conv_kernel<32, 128><<<g, 256, 0, s>>>(a);
    } else {
        dim3 g(cdiv(a.Lq, 256), cdiv(M, 16), a.N);
        ec_conv_kernel<16, 256><<<g, 256, 0, s>>>(a);
    }
    count_launch();
}

// SEANet resnet block (EncodecResnetBlock, EncodecLayers.swift:278-337; Mimi's SeanetResnetBlock, Mimi/Seanet.swift) on x [N, L, dim]
// as two launches: r1 = k-tap conv dim -> hid over ELU(x) into z [N, L, hid], then r2 = [shortcut | k1 conv] over [x | ELU(z)] or,
// with the identity skip, the k1 conv over ELU(z) plus x.  The result lands in y and x / y swap.
inline void resnet_block(const Conv& r1, const Conv& r2, bool conv_shortcut, int k, int padL, int reflect, float*& x, float*& y, float* z,
                         int N, long long L, int dim, cudaStream_t s) {
    const int hid = r1.M;
    ConvArgs a{};
    a.xa = x; a.La = (int)L; a.Ca = dim; a.taps = k; a.padL = padL; a.reflect = reflect; a.elu_a = 1;
    a.A = r1.A.p; a.bias = r1.bias.p; a.M = hid; a.K = r1.K; a.Lq = (int)L; a.N = N; a.out = z; a.out_per_n = L * hid;
    launch_conv(a, s);
    ConvArgs b{};
    b.N = N; b.Lq = (int)L; b.M = dim; b.K = r2.K; b.A = r2.A.p; b.bias = r2.bias.p; b.out = y; b.out_per_n = L * dim;
    if (conv_shortcut) {
        b.xa = x; b.La = (int)L; b.Ca = dim; b.taps = 1; b.xb = z; b.Cb = hid; b.elu_b = 1;
    } else {
        b.xa = z; b.La = (int)L; b.Ca = hid; b.taps = 1; b.elu_a = 1; b.res = x;
    }
    launch_conv(b, s);
    std::swap(x, y);
}

// Encoder stem (Encodec.swift:24-29): k-tap conv from audio_channels (1 or 2, too few for ec_conv_kernel's float4 K axis) to
// F filters, with the config's padding, on chunk n of the waveform divided by scale[n] (when normalize).  STEM_T outputs per CTA;
// the padded input tile and the weights [F, k, C] sit in shared memory.
constexpr int STEM_T = 128;
static __global__ void __launch_bounds__(256) stem_conv_kernel(const float* __restrict__ wave, const float* __restrict__ w,
                                                               const float* __restrict__ bias, const float* __restrict__ scale,
                                                               float* __restrict__ out, int B, long long samples, int C, int Lc,
                                                               int stride_c, int F, int k, int padL, int reflect) {
    extern __shared__ float sm[];
    float* ws = sm;                        // [F][k][C]
    float* xs = sm + F * k * C;            // [STEM_T + k - 1][C]
    const int n = blockIdx.y, c = n / B, b = n - c * B, t0 = blockIdx.x * STEM_T;
    const float* src = wave + ((long long)b * samples + (long long)c * stride_c) * C;
    const float sc = scale ? scale[n] : 1.f;
    for (int e = threadIdx.x; e < F * k * C; e += 256) ws[e] = w[e];
    for (int e = threadIdx.x; e < (STEM_T + k - 1) * C; e += 256) {
        const int r = e / C, ch = e - r * C;
        int s = t0 + r - padL;
        if (s < 0) s = reflect ? min(-s, Lc - 1) : -1;
        else if (s >= Lc) s = reflect ? max(Lc - 2 - (s - Lc), 0) : -1;
        const float v = s >= 0 ? src[(long long)s * C + ch] : 0.f;
        xs[e] = scale ? __fdiv_rn(v, sc) : v;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < STEM_T * F; e += 256) {
        const int t = e / F, f = e - t * F;
        if (t0 + t >= Lc) break;
        float acc = 0.f;
        for (int kk = 0; kk < k; ++kk)
            for (int ch = 0; ch < C; ++ch) acc = fmaf(ws[(f * k + kk) * C + ch], xs[(t + kk) * C + ch], acc);
        out[((long long)n * Lc + t0 + t) * F + f] = acc + bias[f];
    }
}

// |e|^2 * mul of every codebook row, summed over d in order without contraction (the code search's `ee`; mul is a power of two,
// so the product is exact).
static __global__ void sqnorm_rows_kernel(const float* __restrict__ e, float* __restrict__ out, long long rows, int D, float mul) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    float acc = 0.f;
    for (int d = 0; d < D; ++d) acc = __fadd_rn(acc, __fmul_rn(e[r * D + d], e[r * D + d]));
    out[r] = acc * mul;
}

// Residual VQ encode: z rows [rows = N*T] of D floats at stride zld -> codes [N, nq_total, T] levels q_off .. q_off + nq - 1, levels
// in sequence with residual -= embed[idx].  Ordered fp32: for each (frame, code) dot, |x|^2 and |e|^2 are summed over d = 0..D-1
// as acc = fl(acc + fl(a*b)), and the lowest index wins ties (argMax(-dist) / argMin(dist) in the references).  The distance:
//   HALF_C2 = false, Encodec (EncodecQuantization.swift:22-38, 100-115): ee = |e|^2,   dist = fl(fl(xx - 2 dot) + ee);
//   HALF_C2 = true,  Mimi (Mimi/Quantization.swift:41-46):                ee = |e|^2/2, dist = fl(ee - dot).
// A CTA keeps VQ_FT frames' residuals in shared memory for all levels and streams VQ_KT-code tiles of each codebook through;
// thread (tx = tid % 16, ty = tid / 16) scores frames ty, ty + 16 against codes tx + 16 j, j < 4, of a tile.
constexpr int VQ_FT = 32, VQ_KT = 64;
inline size_t rvq_encode_smem(int D) { return ((size_t)(VQ_FT + VQ_KT) * (D + 1) + VQ_KT + 2 * VQ_FT) * sizeof(float); }
template <bool HALF_C2>
__global__ void __launch_bounds__(256) rvq_encode_kernel(const float* __restrict__ z, int zld, const float* __restrict__ books,
                                                         const float* __restrict__ ee, int* __restrict__ codes, int rows, int T,
                                                         int nq, int q_off, int nq_total, int K, int D) {
    extern __shared__ float sm[];
    const int ld = D + 1;
    float* rs = sm;                        // [VQ_FT][ld] residuals
    float* es = rs + VQ_FT * ld;           // [VQ_KT][ld] codebook tile
    float* ees = es + VQ_KT * ld;          // [VQ_KT]
    float* xxs = ees + VQ_KT;              // [VQ_FT]
    int* bidx = reinterpret_cast<int*>(xxs + VQ_FT);   // [VQ_FT]
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int f0 = blockIdx.x * VQ_FT;
    for (int e = tid; e < VQ_FT * D; e += 256) {
        const int f = e / D, d = e - f * D;
        rs[f * ld + d] = f0 + f < rows ? z[(long long)(f0 + f) * zld + d] : 0.f;
    }
    __syncthreads();
    for (int q = 0; q < nq; ++q) {
        const float* book = books + (long long)q * K * D;
        if (!HALF_C2 && tid < VQ_FT) {
            float xx = 0.f;
            for (int d = 0; d < D; ++d) xx = __fadd_rn(xx, __fmul_rn(rs[tid * ld + d], rs[tid * ld + d]));
            xxs[tid] = xx;
        }
        float best[2] = {INFINITY, INFINITY};
        int bi[2] = {0, 0};
        for (int k0 = 0; k0 < K; k0 += VQ_KT) {
            __syncthreads();
            for (int e = tid; e < VQ_KT * D; e += 256) {
                const int c = e / D, d = e - c * D;
                es[c * ld + d] = k0 + c < K ? book[(long long)(k0 + c) * D + d] : 0.f;
            }
            if (tid < VQ_KT) ees[tid] = k0 + tid < K ? ee[(long long)q * K + k0 + tid] : 0.f;
            __syncthreads();
            float dot[2][4];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) dot[i][j] = 0.f;
            const float* r0 = rs + ty * ld;
            const float* r1 = rs + (ty + 16) * ld;
            const float* e0 = es + tx * ld;
#pragma unroll 4
            for (int d = 0; d < D; ++d) {
                const float a0 = r0[d], a1 = r1[d];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float ev = e0[16 * j * ld + d];
                    dot[0][j] = __fadd_rn(dot[0][j], __fmul_rn(a0, ev));
                    dot[1][j] = __fadd_rn(dot[1][j], __fmul_rn(a1, ev));
                }
            }
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int c = tx + 16 * j;
                    if (k0 + c >= K) continue;
                    const float dist = HALF_C2 ? __fsub_rn(ees[c], dot[i][j])
                                               : __fadd_rn(__fsub_rn(xxs[ty + 16 * i], __fmul_rn(2.0f, dot[i][j])), ees[c]);
                    if (dist < best[i]) { best[i] = dist; bi[i] = k0 + c; }
                }
        }
        // lowest index among the 16 lanes' minima (each lane's is already its lowest)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
#pragma unroll
            for (int o = 8; o; o >>= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best[i], o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi[i], o);
                if (ob < best[i] || (ob == best[i] && oi < bi[i])) { best[i] = ob; bi[i] = oi; }
            }
            const int f = ty + 16 * i;
            if (tx == 0) {
                bidx[f] = bi[i];
                if (f0 + f < rows) {
                    const int n = (f0 + f) / T, t = (f0 + f) - n * T;
                    codes[((long long)n * nq_total + q_off + q) * T + t] = bi[i];
                }
            }
        }
        __syncthreads();
        if (q + 1 < nq)
            for (int e = tid; e < VQ_FT * D; e += 256) {
                const int f = e / D, d = e - f * D;
                rs[f * ld + d] = __fsub_rn(rs[f * ld + d], book[(long long)bidx[f] * D + d]);
            }
        __syncthreads();
    }
}

}  // namespace ec
}  // namespace b2a
