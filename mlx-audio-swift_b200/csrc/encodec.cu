// Encodec decode and encode for sm_90a (SURVEY.md rows a18, a18b).  Replaces (reference paths):
//   Sources/MLXAudioCodecs/Encodec/EncodecQuantization.swift:117-133  EncodecResidualVectorQuantizer.decode
//   Sources/MLXAudioCodecs/Encodec/Encodec.swift:94-167               EncodecDecoder
//   Sources/MLXAudioCodecs/Encodec/EncodecLayers.swift:15-88          EncodecLSTM / EncodecLSTMBlock (T sequential tiny matmuls)
//   Sources/MLXAudioCodecs/Encodec/EncodecLayers.swift:92-211         EncodecConv1d (causal / asymmetric, clamped reflect padding)
//   Sources/MLXAudioCodecs/Encodec/EncodecLayers.swift:216-273,371-450 transposed conv (a 5-deep scalar host loop in the reference)
//   Sources/MLXAudioCodecs/Encodec/EncodecLayers.swift:278-337        EncodecResnetBlock
//   Sources/MLXAudioCodecs/Encodec/Encodec.swift:294-402              decodeFrame / linearOverlapAdd / decode
//   Sources/MLXAudioCodecs/Encodec/Encodec.swift:17-88                EncodecEncoder
//   Sources/MLXAudioCodecs/Encodec/Encodec.swift:212-291              encodeFrame (normalize) / encode (chunk loop)
//   Sources/MLXAudioCodecs/Encodec/EncodecQuantization.swift:22-38,90-115  codebook quantize / residual encode
// fp32, channels-last [N, T, C] (the reference's own layout), N = chunks x batch.
//   * every dense conv is ONE kernel, ec_conv_kernel: an implicit-GEMM over (token tile x output tile) whose K axis gathers
//     the taps straight from the activation (no im2col buffer), with the ELU of the *input*, the bias and the residual /
//     shortcut fused.  A transposed conv (k = J*s) is the same kernel: output phases are stacked on the M axis
//     (row = r*C_out + co), taps run backwards in time, and because ((q*s + r)*C_out + co) == q*s*C_out + m the phase
//     scatter is a plain contiguous store.  A resnet block is two launches: k3 conv, then [shortcut | k1 conv] as one GEMM
//     over two sources (x raw, hidden through ELU).
//   * the LSTM stack is ONE persistent cooperative kernel: each CTA owns 4 hidden units of every layer, keeps its slices of
//     Wh (and Wx of the upper layers) in shared memory for the whole sequence, layers run as a wavefront (layer l works on
//     time s - l in step s), so the whole block costs T + L - 1 grid barriers instead of L*T dependent launches.
//   * the encoder reuses all of it: its downsampling convs (k = 2s, stride s) are ec_conv_kernel launches whose K axis gathers
//     the 2s contiguous input rows of an output (src = q*s + tap - padL), the right padding through the same edge rule.  New
//     kernels sit only at the edges: the stem from 1-2 audio channels (reading each chunk of the waveform in place), the
//     per-chunk RMS scale, and the residual code search in ordered fp32 (DESIGN.md §3.6b).
//   * norm_type time_group_norm (the 48 kHz stereo model; EncodecLayers.swift:128-132, 244-248) puts a GroupNorm(1, C_out) after
//     every conv.  Each such conv is its usual launch followed by gn_stats_kernel (per-row mean / rstd over all T x C_out
//     elements, so every chunk of every clip has its own) and gn_apply_kernel.  The transposed conv writes its untrimmed output
//     and the apply trims (the reference norms before the trim); the resnet's shortcut and block.3 run as two GEMMs whose normed
//     outputs one apply sums; the decoder's last apply carries the chunk scale.  The norm affines are required: a checkpoint with
//     norm layers that lacks one is modelNotInitialized, where the reference's loader would keep gamma = 1, beta = 0.
#include "common.cuh"
#include "seanet.cuh"

#include <algorithm>
#include <cmath>

namespace b2a {
namespace ec {

// ------------------------------------------------------------------ RVQ decode: sum of codebook gathers
// codes [N, n_q, T] int32, books [n_q][size, dim] contiguous -> out [N, T, dim]
__global__ void rvq_sum_kernel(const int* __restrict__ codes, const float* __restrict__ books, float* __restrict__ out,
                               int n_q, int T, int size, int dim) {
    const long long tok = blockIdx.x;
    const int n = (int)(tok / T), t = (int)(tok - (long long)n * T);
    for (int c = threadIdx.x; c < dim; c += blockDim.x) {
        float acc = 0.f;
        for (int q = 0; q < n_q; ++q) {
            int idx = codes[((long long)n * n_q + q) * T + t];
            idx = min(max(idx, 0), size - 1);
            acc += books[((long long)q * size + idx) * dim + c];
        }
        out[tok * dim + c] = acc;
    }
}

__global__ void scale_kernel(float* __restrict__ x, long long n, float f) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] *= f;
}

// ------------------------------------------------------------------ last conv: ELU -> k-tap conv C -> audio channels (1 or 2)
// x [N, L, C] -> per-chunk wave [N, L, CH] scaled by scale[n] (decodeFrame, Encodec.swift:294-301).  256 samples per CTA; the
// tile (+ left halo) goes through ELU once into shared memory; weights [CH, k, C] in shared memory.
__global__ void __launch_bounds__(256) final_conv_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                         const float* __restrict__ scale, float* __restrict__ out, int L, int C, int k,
                                                         int CH, int padL, int reflect) {
    extern __shared__ float sm[];
    float* xs = sm;                          // [(256 + k - 1)][C + 1]
    float* ws = sm + (size_t)(256 + k - 1) * (C + 1);   // [CH][k][C]
    const int n = blockIdx.y, t0 = blockIdx.x * 256;
    const int rows = 256 + k - 1;
    for (int e = threadIdx.x; e < CH * k * C; e += 256) ws[e] = w[e];
    for (int e = threadIdx.x; e < rows * C; e += 256) {
        const int r = e / C, c = e - r * C;
        int s = t0 + r - padL;
        if (s < 0) s = reflect ? min(-s, L - 1) : -1;
        else if (s >= L) s = reflect ? max(L - 2 - (s - L), 0) : -1;
        xs[r * (C + 1) + c] = s >= 0 ? elu1(x[((long long)n * L + s) * C + c]) : 0.f;
    }
    __syncthreads();
    const int t = t0 + threadIdx.x;
    if (t >= L) return;
    const float sc = scale ? scale[n] : 1.f;
    for (int ch = 0; ch < CH; ++ch) {
        float acc = 0.f;
        for (int kk = 0; kk < k; ++kk) {
            const float* xr = xs + (threadIdx.x + kk) * (C + 1);
            const float* wr = ws + (ch * k + kk) * C;
            for (int c = 0; c < C; ++c) acc = fmaf(wr[c], xr[c], acc);
        }
        out[((long long)n * L + t) * CH + ch] = (acc + bias[ch]) * sc;
    }
}

// ------------------------------------------------------------------ linearOverlapAdd (Encodec.swift:304-356) as a gather
// frames [n_chunks, B, L, CH] -> out [B, total, CH]; weight w[t] = 0.5 - |(t+1)/(L+1) - 0.5|, normalised by the weight sum.
__global__ void overlap_add_kernel(const float* __restrict__ frames, float* __restrict__ out, int n_chunks, int B, int L, int CH,
                                   int hop, long long total) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (t >= total) return;
    int c_hi = (int)min((long long)n_chunks - 1, t / hop);
    int c_lo = (int)max(0ll, (t - L + hop) / hop);        // smallest c with c*hop + L > t
    for (int ch = 0; ch < CH; ++ch) {
        float acc = 0.f, sw = 0.f;
        for (int c = c_lo; c <= c_hi; ++c) {
            const int tt = (int)(t - (long long)c * hop);
            if (tt < 0 || tt >= L) continue;
            const float wv = 0.5f - fabsf((float)(tt + 1) / (float)(L + 1) - 0.5f);
            acc += wv * frames[(((long long)c * B + b) * L + tt) * CH + ch];
            sw += wv;
        }
        out[((long long)b * total + t) * CH + ch] = sw != 0.f ? acc / sw : acc;
    }
}

// ------------------------------------------------------------------ LSTM stack, persistent wavefront kernel
constexpr int LSTM_MAX_LAYERS = 4;
constexpr int LSTM_BC = 8;          // batch rows per launch
constexpr int LSTM_UNITS = 4;       // hidden units per CTA -> 16 gate rows per layer

struct LstmArgs {
    const float* xproj;                     // [N, T, 4H]: layer-0 input projection + bias
    const float* Wh[LSTM_MAX_LAYERS];       // [4H, H]
    const float* Wx[LSTM_MAX_LAYERS];       // [4H, H] for l >= 1
    const float* bias[LSTM_MAX_LAYERS];     // [4H] for l >= 1
    float* hseq[LSTM_MAX_LAYERS];           // [N, T, H] hidden sequence of every layer (exchange buffer between CTAs)
    const float* skip;                      // [N, T, H] block input
    float* out;                             // [N, T, H] = h_last + skip
    unsigned* bar;                          // grid barrier counter (zeroed by the host)
    int n0, nb, T, H, NL;                   // this launch handles rows n0 .. n0+nb-1 (nb <= LSTM_BC)
};

__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + __expf(-v)); }

__device__ __forceinline__ void grid_barrier(unsigned* ctr, unsigned target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(ctr, 1u);
        unsigned v;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
        } while (v < target);
    }
    __syncthreads();
}

// smem: per layer Wh slice [16][H]; per layer l>=1 Wx slice [16][H]; hs [NL][BC][H]; gates [NL][16][BC]; cst [NL][4][BC]
__global__ void __launch_bounds__(256) lstm_kernel(LstmArgs a) {
    extern __shared__ __align__(16) float sm[];
    const int H = a.H, NL = a.NL, T = a.T;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int u0 = blockIdx.x * LSTM_UNITS;
    float* whs = sm;                                        // [NL][16][H]
    float* wxs = whs + (size_t)NL * 16 * H;                 // [NL-1][16][H]
    float* hs = wxs + (size_t)(NL - 1) * 16 * H;            // [NL][BC][H]
    float* gates = hs + (size_t)NL * LSTM_BC * H;           // [NL][16][BC]
    float* cst = gates + NL * 16 * LSTM_BC;                 // [NL][UNITS][BC]
    // row r of a slice = gate (r / UNITS), unit u0 + r % UNITS  ->  global row gate*H + u0 + r%UNITS
    for (int l = 0; l < NL; ++l)
        for (int e = tid; e < 16 * H; e += 256) {
            const int r = e / H, k = e - r * H;
            const long long grow = (long long)(r / LSTM_UNITS) * H + u0 + (r % LSTM_UNITS);
            whs[((size_t)l * 16 + r) * H + k] = a.Wh[l][grow * H + k];
            if (l >= 1) wxs[((size_t)(l - 1) * 16 + r) * H + k] = a.Wx[l][grow * H + k];
        }
    for (int e = tid; e < NL * LSTM_UNITS * LSTM_BC; e += 256) cst[e] = 0.f;
    __syncthreads();

    const int r0 = warp * 2;            // this warp's two rows of every slice
    for (int s = 0; s < T + NL - 1; ++s) {
        // stage hs[l] = h_l[s - l - 1] (zeros before the sequence starts).  All loads of a thread are issued before the first
        // store: a plain load/store loop with a run-time trip count is not software-pipelined by the compiler and paid one L2
        // round trip per iteration (32 dependent round trips per step).
        {
            const int hq = H >> 2, per_layer = LSTM_BC * hq;          // float4 items per layer (H % 4 == 0)
            for (int base = 0; base < NL * per_layer; base += 256 * 8) {
                float4 v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int e = base + u * 256 + tid;
                    v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (e < NL * per_layer) {
                        const int l = e / per_layer, r = e - l * per_layer, b = r / hq, k4 = r - b * hq;
                        const int tp = s - l - 1;
                        if (tp >= 0 && tp < T && b < a.nb)
                            v[u] = __ldcg(reinterpret_cast<const float4*>(a.hseq[l] + ((long long)(a.n0 + b) * T + tp) * H) + k4);
                    }
                }
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int e = base + u * 256 + tid;
                    if (e < NL * per_layer) reinterpret_cast<float4*>(hs)[e] = v[u];
                }
            }
        }
        __syncthreads();
        for (int l = 0; l < NL; ++l) {
            const int t = s - l;
            if (t < 0 || t >= T) continue;
            float acc[2][LSTM_BC];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int b = 0; b < LSTM_BC; ++b) acc[i][b] = 0.f;
            const float* w0 = whs + ((size_t)l * 16 + r0) * H;
            const float* hl = hs + (size_t)l * LSTM_BC * H;
            for (int k = lane; k < H; k += 32) {
                const float wa = w0[k], wb = w0[H + k];
#pragma unroll
                for (int b = 0; b < LSTM_BC; ++b) {
                    const float hv = hl[b * H + k];
                    acc[0][b] = fmaf(wa, hv, acc[0][b]);
                    acc[1][b] = fmaf(wb, hv, acc[1][b]);
                }
            }
            if (l >= 1) {
                const float* x0 = wxs + ((size_t)(l - 1) * 16 + r0) * H;
                const float* hp = hs + (size_t)(l - 1) * LSTM_BC * H;
                for (int k = lane; k < H; k += 32) {
                    const float wa = x0[k], wb = x0[H + k];
#pragma unroll
                    for (int b = 0; b < LSTM_BC; ++b) {
                        const float hv = hp[b * H + k];
                        acc[0][b] = fmaf(wa, hv, acc[0][b]);
                        acc[1][b] = fmaf(wb, hv, acc[1][b]);
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int b = 0; b < LSTM_BC; ++b) {
                    float v = acc[i][b];
#pragma unroll
                    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                    if (lane == 0) gates[(l * 16 + r0 + i) * LSTM_BC + b] = v;
                }
        }
        __syncthreads();
        // pointwise: thread -> (layer, unit, batch row)
        if (tid < NL * LSTM_UNITS * LSTM_BC) {
            const int l = tid / (LSTM_UNITS * LSTM_BC), u = (tid / LSTM_BC) % LSTM_UNITS, b = tid % LSTM_BC;
            const int t = s - l;
            if (t >= 0 && t < T && b < a.nb) {
                const long long row = (long long)(a.n0 + b) * T + t;
                float g[4];
#pragma unroll
                for (int gi = 0; gi < 4; ++gi) {
                    float v = gates[(l * 16 + gi * LSTM_UNITS + u) * LSTM_BC + b];
                    const long long col = (long long)gi * H + u0 + u;
                    v += (l == 0) ? a.xproj[row * 4 * H + col] : a.bias[l][col];
                    g[gi] = v;
                }
                const float ig = sigmoidf_(g[0]), fg = sigmoidf_(g[1]), gg = tanhf(g[2]), og = sigmoidf_(g[3]);
                const float c = fg * cst[tid] + ig * gg;
                cst[tid] = c;
                const float h = og * tanhf(c);
                a.hseq[l][row * H + u0 + u] = h;
                if (l == NL - 1) a.out[row * H + u0 + u] = h + a.skip[row * H + u0 + u];
            }
        }
        grid_barrier(a.bar, (unsigned)(s + 1) * gridDim.x);
    }
}

// ================================================================== encode side
// Chunk c of batch row b is the frame n = c*B + b: samples [c*stride, c*stride + Lc) of wave [B, samples, C], read in place.

// encodeFrame's normalisation (Encodec.swift:224-231): scale[n] = sqrt(mean_t(mono^2)) + 1e-8, mono = sum_ch x / C.  One CTA per
// frame; each thread sums a fixed strided subset in double, then a fixed tree: the result does not depend on scheduling.
__global__ void __launch_bounds__(256) chunk_scale_kernel(const float* __restrict__ wave, float* __restrict__ scale, int B,
                                                          long long samples, int C, int Lc, int stride_c) {
    __shared__ double red[256];
    const int n = blockIdx.x, c = n / B, b = n - c * B;
    const float* src = wave + ((long long)b * samples + (long long)c * stride_c) * C;
    double acc = 0.0;
    for (int t = threadIdx.x; t < Lc; t += 256) {
        float m = 0.f;
        for (int ch = 0; ch < C; ++ch) m += src[(long long)t * C + ch];
        m = m / (float)C;
        acc += (double)m * (double)m;
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 128; o; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) scale[n] = (float)sqrt(red[0] / (double)Lc) + 1e-8f;
}

// ================================================================== time_group_norm (GroupNorm(1, C) after every conv)
// Statistics of batch row n over all E = rows * C contiguous elements of x [N, rows, C]: GN_PARTS(E) CTAs per row each sum a
// fixed slice in double (thread t takes elements t, t + 256, ...; a fixed tree across the CTA), and the row's last CTA to finish
// combines the partials in index order into stats[n] = (mean, rstd).  The slices depend on E only, so a row's statistics do not
// depend on how many rows share the launch: batched == serial bit for bit.  cnt[n] is zero before a launch and after it.
constexpr int GN_SLICE = 16384, GN_MAX_PARTS = 2048;
inline int gn_parts(long long E) { return (int)std::min<long long>(std::max<long long>((E + GN_SLICE - 1) / GN_SLICE, 1), GN_MAX_PARTS); }

__global__ void __launch_bounds__(256) gn_stats_kernel(const float* __restrict__ x, long long E, double2* __restrict__ part,
                                                       unsigned* __restrict__ cnt, float2* __restrict__ stats, float eps) {
    __shared__ double rs[256], rq[256];
    __shared__ bool last;
    const int n = blockIdx.y, p = blockIdx.x, P = gridDim.x, tid = threadIdx.x;
    const long long slice = (E + P - 1) / P, e0 = (long long)p * slice, e1 = min(E, e0 + slice);
    const float* xn = x + (long long)n * E;
    double s = 0.0, q = 0.0;
    long long e = e0 + tid;
    for (; e + 3 * 256 < e1; e += 4 * 256) {      // four loads in flight per thread; the same per-thread order as one at a time
        const float v0 = xn[e], v1 = xn[e + 256], v2 = xn[e + 512], v3 = xn[e + 768];
        s += (double)v0; q += (double)v0 * v0;
        s += (double)v1; q += (double)v1 * v1;
        s += (double)v2; q += (double)v2 * v2;
        s += (double)v3; q += (double)v3 * v3;
    }
    for (; e < e1; e += 256) { const double v = xn[e]; s += v; q += v * v; }
    rs[tid] = s; rq[tid] = q;
    __syncthreads();
    for (int o = 128; o; o >>= 1) {
        if (tid < o) { rs[tid] += rs[tid + o]; rq[tid] += rq[tid + o]; }
        __syncthreads();
    }
    if (tid == 0) {
        part[(long long)n * P + p] = make_double2(rs[0], rq[0]);
        __threadfence();
        last = atomicAdd(cnt + n, 1u) == (unsigned)(P - 1);
    }
    __syncthreads();
    if (!last || tid >= 32) return;
    __threadfence();
    // warp 0 of the last CTA: lane l sums partials l, l + 32, ... in order, then a fixed xor tree
    double S = 0.0, Q = 0.0;
    for (int i = tid; i < P; i += 32) {
        const double2 v = __ldcg(part + (long long)n * P + i);
        S += v.x; Q += v.y;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { S += __shfl_xor_sync(0xffffffffu, S, o); Q += __shfl_xor_sync(0xffffffffu, Q, o); }
    if (tid == 0) {
        const double mean = S / (double)E, var = fmax(Q / (double)E - mean * mean, 0.0);
        stats[n] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
        cnt[n] = 0u;
    }
}

// y = GN_a(xa) [+ GN_b(xb) | + xb] [* scale[n]] over out [N, L, C].  xa has rows_a rows per batch row and is read from row off_a
// on (the transposed conv's left trim); xb is [N, L, C].  GN(x)[c] = (x - mean) * rstd * gamma[c] + beta[c].  VEC: float4 along
// channels (C % 4 == 0); the scalar path serves the final wave's 1 or 2 channels.  out may be xa (one source, off_a = 0) or xb:
// every element is read before it is written by the same thread.
struct GnApplyArgs {
    const float* xa; const float2* sa; const float* ga; const float* ba; long long rows_a, off_a;
    const float* xb; const float2* sb; const float* gb; const float* bb;    // sb null: plain addend (identity shortcut)
    const float* scale;                                                      // [N] or null
    float* out; long long L; int C;
};

template <bool VEC>
__global__ void __launch_bounds__(256) gn_apply_kernel(GnApplyArgs a) {
    const int n = blockIdx.y;
    const long long per = a.L * a.C;
    const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * (VEC ? 4 : 1);
    if (i >= per) return;
    const int c = (int)(i % a.C);
    const float2 sa = a.sa[n];
    const float sc = a.scale ? a.scale[n] : 1.f;
    const float* xa = a.xa + (long long)n * a.rows_a * a.C + a.off_a * a.C + i;
    const long long o = (long long)n * per + i;
    if constexpr (VEC) {
        const float4 v = *reinterpret_cast<const float4*>(xa);
        const float4 g = *reinterpret_cast<const float4*>(a.ga + c), b = *reinterpret_cast<const float4*>(a.ba + c);
        float r[4] = {(v.x - sa.x) * sa.y * g.x + b.x, (v.y - sa.x) * sa.y * g.y + b.y,
                      (v.z - sa.x) * sa.y * g.z + b.z, (v.w - sa.x) * sa.y * g.w + b.w};
        if (a.xb) {
            const float4 u = *reinterpret_cast<const float4*>(a.xb + o);
            float w[4] = {u.x, u.y, u.z, u.w};
            if (a.sb) {
                const float2 sb = a.sb[n];
                const float4 gb = *reinterpret_cast<const float4*>(a.gb + c), bb = *reinterpret_cast<const float4*>(a.bb + c);
                w[0] = (w[0] - sb.x) * sb.y * gb.x + bb.x; w[1] = (w[1] - sb.x) * sb.y * gb.y + bb.y;
                w[2] = (w[2] - sb.x) * sb.y * gb.z + bb.z; w[3] = (w[3] - sb.x) * sb.y * gb.w + bb.w;
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) r[k] += w[k];
        }
        *reinterpret_cast<float4*>(a.out + o) = make_float4(r[0] * sc, r[1] * sc, r[2] * sc, r[3] * sc);
    } else {
        float r = (*xa - sa.x) * sa.y * a.ga[c] + a.ba[c];
        if (a.xb) {
            float w = a.xb[o];
            if (a.sb) { const float2 sb = a.sb[n]; w = (w - sb.x) * sb.y * a.gb[c] + a.bb[c]; }
            r += w;
        }
        a.out[o] = r * sc;
    }
}

}  // namespace ec
}  // namespace b2a

using namespace b2a;

// an EncodecLSTMBlock's stack: layer 0's input projection runs as one GEMM (xproj), the rest inside lstm_kernel
struct EcLstm {
    ec::Conv xproj;
    DBuf<float> Wh[ec::LSTM_MAX_LAYERS], Wx[ec::LSTM_MAX_LAYERS], b[ec::LSTM_MAX_LAYERS];
};

// a GroupNorm(1, C)'s affine (time_group_norm only)
struct EcNorm {
    DBuf<float> g, b;
};

// an EncodecResnetBlock: r1 = k-tap conv dim -> hid (ELU of its input), r2 = [shortcut | block.3] over K = dim + hid, or
// block.3 plus the identity residual without a conv shortcut.  Under time_group_norm the two addends have statistics of their
// own, so r2 is block.3 alone, sc the shortcut alone, and n1 / n3 / ns the norms after block.1 / block.3 / the shortcut.
struct EcRes {
    ec::Conv r1, r2, sc;
    EcNorm n1, n3, ns;
};

struct b2a_encodec {
    int device = 0, num_sms = 132;
    b2a_encodec_config cfg{};
    cudaStream_t stream = nullptr;
    int n_q = 0;
    DBuf<float> books;                       // [n_q][size][dim]
    bool gn = false;                         // norm_type time_group_norm: a GroupNorm(1, C_out) after every conv
    ec::Conv conv0;
    EcNorm norm0;
    EcLstm lstm;
    struct Stage { int ratio, cin, cout, taps; ec::Conv up; EcNorm nup; EcRes res; };
    std::vector<Stage> stages;
    DBuf<float> wlast, blast;
    EcNorm nlast;
    // encoder (only when the checkpoint has encoder.* tensors)
    bool has_enc = false;
    std::string enc_error = "encodec encode: the checkpoint has no encoder weights";
    DBuf<float> wstem, bstem;                // [num_filters, kernel_size, audio_channels]
    EcNorm nstem;
    struct EStage { int ratio, cin, cout; EcRes res; ec::Conv down; EcNorm ndown; };
    std::vector<EStage> estages;
    EcLstm elstm;
    ec::Conv elast;
    EcNorm nelast;
    DBuf<float> book_sq;                     // [n_q][size] |e|^2 in search order
    // workspaces
    DBuf<float> bufA, bufB, bufC, xp, hseq[ec::LSTM_MAX_LAYERS], chunks, scales, wave, zbuf, audio;
    DBuf<int> codes;
    DBuf<unsigned> bar;
    // time_group_norm workspaces: the shortcut's output, per-CTA partial sums, per-row arrival counters, two rows of statistics
    DBuf<float> bufD;
    DBuf<double2> gn_part;
    DBuf<unsigned> gn_cnt;
    DBuf<float2> gn_sa, gn_sb;
    int dim0 = 0;

    static void up(DBuf<float>& d, const std::vector<float>& v) { d.upload(v.data(), v.size()); }
    static void chan_ok(int ch) { B2A_CHECK(ch >= 4 && ch % 4 == 0, B2A_ERR_INVALID_INPUT, "encodec: channel counts must be multiples of 4"); }

    // ---- weight loading shared by the decoder and the encoder (prefix p ends in '.')
    static void plain(const TensorTable& tt, ec::Conv& cv, const std::string& p, int cout, int k, int cin) {
        chan_ok(cin);
        cv.M = cout; cv.K = k * cin;
        up(cv.A, tt.f32(p + "conv.weight", (int64_t)cout * k * cin));      // [out, k, in] == [M, tap*Cin + ci]
        up(cv.bias, tt.f32(p + "conv.bias", cout));
    }
    // GroupNorm affine [C] of the conv at prefix p (time_group_norm only)
    void load_norm(const TensorTable& tt, EcNorm& nm, const std::string& p, int C) const {
        if (!gn) return;
        up(nm.g, tt.f32(p + "norm.weight", C));
        up(nm.b, tt.f32(p + "norm.bias", C));
    }
    void load_resnet(const TensorTable& tt, EcRes& r, const std::string& p, int dim) const {
        const int hid = dim / cfg.compress;
        chan_ok(hid);
        plain(tt, r.r1, p + "block.1.", hid, cfg.residual_kernel_size, dim);
        if (gn) {
            plain(tt, r.r2, p + "block.3.", dim, 1, hid);
            load_norm(tt, r.n1, p + "block.1.", hid);
            load_norm(tt, r.n3, p + "block.3.", dim);
            if (cfg.use_conv_shortcut) { plain(tt, r.sc, p + "shortcut.", dim, 1, dim); load_norm(tt, r.ns, p + "shortcut.", dim); }
            return;
        }
        // second launch: [shortcut | block.3] over K = dim + hid (x raw, hidden through ELU)
        std::vector<float> w1 = tt.f32(p + "block.3.conv.weight", (int64_t)dim * hid), b1 = tt.f32(p + "block.3.conv.bias", dim);
        if (cfg.use_conv_shortcut) {
            std::vector<float> ws = tt.f32(p + "shortcut.conv.weight", (int64_t)dim * dim), bs = tt.f32(p + "shortcut.conv.bias", dim);
            std::vector<float> A((size_t)dim * (dim + hid));
            for (int m = 0; m < dim; ++m) {
                memcpy(&A[(size_t)m * (dim + hid)], &ws[(size_t)m * dim], dim * sizeof(float));
                memcpy(&A[(size_t)m * (dim + hid) + dim], &w1[(size_t)m * hid], hid * sizeof(float));
                b1[m] += bs[m];
            }
            r.r2.M = dim; r.r2.K = dim + hid; up(r.r2.A, A);
        } else {
            r.r2.M = dim; r.r2.K = hid; up(r.r2.A, w1);
        }
        up(r.r2.bias, b1);
    }
    void load_lstm(const TensorTable& tt, EcLstm& m, const std::string& p, int H) const {
        if (cfg.num_lstm_layers == 0) return;
        B2A_CHECK(H % ec::LSTM_UNITS == 0, B2A_ERR_INVALID_INPUT, "encodec: LSTM width must be a multiple of 4");
        for (int l = 0; l < cfg.num_lstm_layers; ++l) {
            const std::string q = p + "lstm." + std::to_string(l) + ".";
            std::vector<float> wx = tt.f32(q + "Wx", (int64_t)4 * H * H), wh = tt.f32(q + "Wh", (int64_t)4 * H * H);
            std::vector<float> b = tt.find(q + "bias") ? tt.f32(q + "bias", 4 * H) : std::vector<float>(4 * H, 0.f);
            up(m.Wh[l], wh);
            if (l == 0) { m.xproj.M = 4 * H; m.xproj.K = H; up(m.xproj.A, wx); up(m.xproj.bias, b); }
            else { up(m.Wx[l], wx); up(m.b[l], b); }
        }
    }

    b2a_encodec(int dev, const b2a_encodec_config& c, const TensorTable& tt) : device(dev), cfg(c) {
        require_device(dev);
        B2A_CUDA(cudaSetDevice(dev));
        cudaDeviceProp prop{};
        B2A_CUDA(cudaGetDeviceProperties(&prop, dev));
        num_sms = prop.multiProcessorCount;
        B2A_CHECK(c.norm_type == 0 || c.norm_type == 1, B2A_ERR_INVALID_INPUT, "encodec: norm_type must be 0 (weight_norm) or 1 (time_group_norm)");
        gn = c.norm_type == 1;
        // config.json does not describe the norm layers: a time_group_norm config over a checkpoint without them is a config error
        B2A_CHECK(!gn || tt.find("decoder.layers.0.norm.weight"), B2A_ERR_INVALID_INPUT,
                  "encodec: norm_type time_group_norm but the checkpoint has no norm layers (decoder.layers.0.norm.weight)");
        B2A_CHECK(c.n_upsampling_ratios >= 1 && c.n_upsampling_ratios <= 8, B2A_ERR_INVALID_INPUT, "encodec: bad upsampling_ratios");
        B2A_CHECK(c.num_residual_layers == 1 || c.dilation_growth_rate == 1, B2A_ERR_INVALID_INPUT,
                  "encodec: dilated residual layers change the frame count in the reference (EncodecLayers.swift:117); not implemented");
        B2A_CHECK(c.num_lstm_layers >= 0 && c.num_lstm_layers <= ec::LSTM_MAX_LAYERS, B2A_ERR_INVALID_INPUT, "encodec: too many LSTM layers");
        B2A_CHECK(c.audio_channels >= 1 && c.audio_channels <= 2, B2A_ERR_INVALID_INPUT, "encodec: audio_channels must be 1 or 2");
        B2A_CHECK(c.compress >= 1 && c.kernel_size >= 1 && c.last_kernel_size >= 1 && c.residual_kernel_size >= 1, B2A_ERR_INVALID_INPUT, "encodec: bad config");
        B2A_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        // codebooks (as many as the checkpoint holds)
        while (tt.find("quantizer.layers." + std::to_string(n_q) + ".codebook.embed")) ++n_q;
        B2A_CHECK(n_q >= 1, B2A_ERR_MODEL_NOT_INITIALIZED, "missing tensor: quantizer.layers.0.codebook.embed");
        {
            std::vector<float> all((size_t)n_q * c.codebook_size * c.codebook_dim);
            for (int q = 0; q < n_q; ++q) {
                std::vector<float> e = tt.f32("quantizer.layers." + std::to_string(q) + ".codebook.embed", (int64_t)c.codebook_size * c.codebook_dim);
                memcpy(&all[(size_t)q * e.size()], e.data(), e.size() * sizeof(float));
            }
            up(books, all);
        }
        B2A_CHECK(c.codebook_dim == c.hidden_size, B2A_ERR_INVALID_INPUT, "encodec: codebook_dim must equal hidden_size");
        int scaling = 1 << c.n_upsampling_ratios;
        int idx = 0;
        auto key = [&](int i, const char* rest) { return "decoder.layers." + std::to_string(i) + "." + rest; };
        dim0 = scaling * c.num_filters;
        plain(tt, conv0, key(idx, ""), dim0, c.kernel_size, c.hidden_size);
        load_norm(tt, norm0, key(idx, ""), dim0); ++idx;
        load_lstm(tt, lstm, key(idx, ""), dim0);
        ++idx;   // the LSTM block occupies a slot even when it has no layers
        for (int i = 0; i < c.n_upsampling_ratios; ++i) {
            Stage st{};
            st.ratio = c.upsampling_ratios[i];
            B2A_CHECK(st.ratio >= 1, B2A_ERR_INVALID_INPUT, "encodec: bad upsampling ratio");
            st.cin = scaling * c.num_filters; st.cout = st.cin / 2;
            chan_ok(st.cin); chan_ok(st.cout);
            ++idx;                                    // ELU slot
            {   // transposed conv k = 2*ratio: phase-major rows m = r*Cout + co, K = taps*Cin, tap j <-> kernel index r + j*s
                const int k = 2 * st.ratio, s = st.ratio;
                st.taps = (k + s - 1) / s;
                std::vector<float> w = tt.f32(key(idx, "conv.weight"), (int64_t)st.cout * k * st.cin), bsrc = tt.f32(key(idx, "conv.bias"), st.cout);
                std::vector<float> A((size_t)s * st.cout * st.taps * st.cin, 0.f), bb((size_t)s * st.cout);
                for (int r = 0; r < s; ++r)
                    for (int co = 0; co < st.cout; ++co) {
                        bb[(size_t)r * st.cout + co] = bsrc[co];
                        for (int j = 0; j < st.taps; ++j) {
                            const int kk = r + j * s;
                            if (kk >= k) continue;
                            memcpy(&A[(((size_t)r * st.cout + co) * st.taps + j) * st.cin], &w[((size_t)co * k + kk) * st.cin], st.cin * sizeof(float));
                        }
                    }
                st.up.M = s * st.cout; st.up.K = st.taps * st.cin;
                up(st.up.A, A); up(st.up.bias, bb);
                load_norm(tt, st.nup, key(idx, ""), st.cout);
                ++idx;
            }
            for (int j = 0; j < c.num_residual_layers; ++j) {
                B2A_CHECK(j == 0, B2A_ERR_INVALID_INPUT, "encodec: one residual layer per stage is implemented");
                load_resnet(tt, st.res, key(idx, ""), st.cout);
                ++idx;
            }
            stages.push_back(std::move(st));
            scaling /= 2;
        }
        ++idx;   // ELU slot
        chan_ok(c.num_filters);
        up(wlast, tt.f32(key(idx, "conv.weight"), (int64_t)c.audio_channels * c.last_kernel_size * c.num_filters));
        up(blast, tt.f32(key(idx, "conv.bias"), c.audio_channels));
        load_norm(tt, nlast, key(idx, ""), c.audio_channels);
        bar.alloc(1);
        if (tt.find("encoder.layers.0.conv.weight")) {
            // a malformed encoder leaves a working decoder: encode then reports why (B2A_ERR_MODEL_NOT_INITIALIZED)
            try { load_encoder(tt); has_enc = true; }
            catch (const Error& e) { estages.clear(); enc_error = std::string("encodec encode: encoder weights unusable: ") + e.what(); }
        }
        B2A_CUDA(cudaDeviceSynchronize());
    }

    // EncodecEncoder (Encodec.swift:17-71): 0 stem, then per reversed ratio resnet(s), ELU, conv k = 2r stride r, then the LSTM
    // block, ELU, last conv -> hidden_size.  Keys encoder.layers.{i}.* in the decoder's layouts, ELU modules counted.
    void load_encoder(const TensorTable& tt) {
        const int F = cfg.num_filters, CH = cfg.audio_channels, k = cfg.kernel_size;
        auto key = [&](int i) { return "encoder.layers." + std::to_string(i) + "."; };
        chan_ok(F);
        int idx = 0;
        up(wstem, tt.f32(key(idx) + "conv.weight", (int64_t)F * k * CH));
        up(bstem, tt.f32(key(idx) + "conv.bias", F));
        load_norm(tt, nstem, key(idx), F);
        ++idx;
        int scaling = 1;
        for (int i = cfg.n_upsampling_ratios - 1; i >= 0; --i) {
            EStage st{};
            st.ratio = cfg.upsampling_ratios[i];
            st.cin = scaling * F; st.cout = 2 * st.cin;
            for (int j = 0; j < cfg.num_residual_layers; ++j) { load_resnet(tt, st.res, key(idx), st.cin); ++idx; }
            ++idx;                                    // ELU slot
            plain(tt, st.down, key(idx), st.cout, 2 * st.ratio, st.cin);
            load_norm(tt, st.ndown, key(idx), st.cout); ++idx;
            estages.push_back(std::move(st));
            scaling *= 2;
        }
        load_lstm(tt, elstm, key(idx), scaling * F); ++idx;
        ++idx;                                        // ELU slot
        plain(tt, elast, key(idx), cfg.hidden_size, cfg.last_kernel_size, scaling * F);
        load_norm(tt, nelast, key(idx), cfg.hidden_size);
        // |e|^2 of every codebook row, in the search's summation order
        const long long rows = (long long)n_q * cfg.codebook_size;
        book_sq.alloc((size_t)rows);
        ec::sqnorm_rows_kernel<<<cdiv(rows, 256), 256>>>(books.p, book_sq.p, rows, cfg.codebook_dim, 1.0f);
        B2A_CUDA(cudaGetLastError());
    }
    ~b2a_encodec() {
        if (stream) cudaStreamDestroy(stream);
    }

    int hop() const {
        int h = 1;
        for (int i = 0; i < cfg.n_upsampling_ratios; ++i) h *= cfg.upsampling_ratios[i];
        return h;
    }
    int chunk_length() const { return cfg.chunk_length_s > 0.f ? (int)(cfg.chunk_length_s * (float)cfg.sampling_rate) : 0; }
    int chunk_stride() const {
        if (cfg.chunk_length_s <= 0.f || cfg.overlap < 0.f) return 0;
        return std::max(1, (int)((1.0f - cfg.overlap) * (float)chunk_length()));
    }
    long long out_len(int n_chunks, int T) const {
        const long long per = (long long)T * hop();
        if (chunk_length() == 0) return per;
        const int st = chunk_stride() > 0 ? chunk_stride() : 1;
        return (long long)st * (n_chunks - 1) + per;
    }

    void pads(int k, int& padL) const {
        const int total = k - 1;
        padL = cfg.use_causal_conv ? total : total - total / 2;
    }

    // EncodecResnetBlock (EncodecLayers.swift:278-337) on x [N, L, dim] as two launches (z: the hidden [N, L, hid]); result in x
    void run_resnet(const EcRes& r, float*& x, float*& y, float* z, int N, long long L, int dim, cudaStream_t s) {
        int padL; pads(cfg.residual_kernel_size, padL);
        ec::resnet_block(r.r1, r.r2, cfg.use_conv_shortcut != 0, cfg.residual_kernel_size, padL, cfg.pad_mode_reflect, x, y, z, N, L, dim, s);
    }

    // ---- time_group_norm: GroupNorm(1, C) with eps 1e-5 (EncodecLayers.swift:128-132, 244-248) as statistics then apply
    // per-row (mean, rstd) of x [N, rows, C] into st
    void gn_stats(const float* x, int N, long long rows, int C, float2* st, cudaStream_t s) {
        const long long E = rows * C;
        const int P = ec::gn_parts(E);
        gn_part.alloc((size_t)N * P);
        if (gn_cnt.n < (size_t)N) {
            gn_cnt.alloc((size_t)N);
            B2A_CUDA(cudaMemsetAsync(gn_cnt.p, 0, (size_t)N * sizeof(unsigned), s));
        }
        ec::gn_stats_kernel<<<dim3(P, N), 256, 0, s>>>(x, E, gn_part.p, gn_cnt.p, st, 1e-5f);
        count_launch();
    }
    void gn_apply(const ec::GnApplyArgs& a, int N, cudaStream_t s) {
        const long long per = a.L * a.C;
        if (a.C % 4 == 0) ec::gn_apply_kernel<true><<<dim3((unsigned)cdiv(per / 4, 256), N), 256, 0, s>>>(a);
        else ec::gn_apply_kernel<false><<<dim3((unsigned)cdiv(per, 256), N), 256, 0, s>>>(a);
        count_launch();
    }
    // x [N, L, C] = GN(x) [* scale[n]], in place
    void gn_inplace(float* x, const EcNorm& nm, int N, long long L, int C, const float* scale, cudaStream_t s) {
        gn_stats(x, N, L, C, gn_sa.p, s);
        ec::GnApplyArgs a{};
        a.xa = x; a.sa = gn_sa.p; a.ga = nm.g.p; a.ba = nm.b.p; a.rows_a = L; a.scale = scale; a.out = x; a.L = L; a.C = C;
        gn_apply(a, N, s);
    }
    void gn_alloc(int N) {
        gn_sa.alloc((size_t)N); gn_sb.alloc((size_t)N);
    }

    // EncodecResnetBlock under time_group_norm (EncodecLayers.swift:319-336): GN_s(shortcut(x)) + GN_3(block.3(ELU(GN_1(block.1(ELU(x)))))),
    // or x + GN_3(...) without a conv shortcut.  z [N, L, hid] and w [N, L, dim] are scratch; the result lands in y and x / y swap.
    void run_resnet_gn(const EcRes& r, float*& x, float*& y, float* z, float* w, int N, long long L, int dim, cudaStream_t s) {
        const int hid = r.r1.M;
        ec::ConvArgs a{};
        a.xa = x; a.La = (int)L; a.Ca = dim; a.taps = cfg.residual_kernel_size; pads(cfg.residual_kernel_size, a.padL);
        a.reflect = cfg.pad_mode_reflect; a.elu_a = 1;
        a.A = r.r1.A.p; a.bias = r.r1.bias.p; a.M = hid; a.K = r.r1.K; a.Lq = (int)L; a.N = N; a.out = z; a.out_per_n = L * hid;
        ec::launch_conv(a, s);
        gn_inplace(z, r.n1, N, L, hid, nullptr, s);
        ec::ConvArgs b{};
        b.xa = z; b.La = (int)L; b.Ca = hid; b.taps = 1; b.elu_a = 1;
        b.A = r.r2.A.p; b.bias = r.r2.bias.p; b.M = dim; b.K = r.r2.K; b.Lq = (int)L; b.N = N; b.out = y; b.out_per_n = L * dim;
        ec::launch_conv(b, s);
        gn_stats(y, N, L, dim, gn_sa.p, s);
        ec::GnApplyArgs g{};
        g.xa = y; g.sa = gn_sa.p; g.ga = r.n3.g.p; g.ba = r.n3.b.p; g.rows_a = L; g.xb = x; g.out = y; g.L = L; g.C = dim;
        if (cfg.use_conv_shortcut) {
            ec::ConvArgs c{};
            c.xa = x; c.La = (int)L; c.Ca = dim; c.taps = 1;
            c.A = r.sc.A.p; c.bias = r.sc.bias.p; c.M = dim; c.K = r.sc.K; c.Lq = (int)L; c.N = N; c.out = w; c.out_per_n = L * dim;
            ec::launch_conv(c, s);
            gn_stats(w, N, L, dim, gn_sb.p, s);
            g.xb = w; g.sb = gn_sb.p; g.gb = r.ns.g.p; g.bb = r.ns.b.p;
        }
        gn_apply(g, N, s);
        std::swap(x, y);
    }

    // EncodecLSTMBlock (EncodecLayers.swift:72-88) on x [N, T, H]: the stack plus its skip; result in x
    void run_lstm_block(const EcLstm& m, float*& x, float*& y, int N, int T, int H, cudaStream_t s) {
        const int NL = cfg.num_lstm_layers;
        if (NL == 0) {
            // an EncodecLSTMBlock without layers still adds its skip: h + hiddenStates = 2x (EncodecLayers.swift:82-88)
            const long long cnt = (long long)N * T * H;
            ec::scale_kernel<<<cdiv(cnt, 256), 256, 0, s>>>(x, cnt, 2.f);
            count_launch();
            return;
        }
        xp.alloc((size_t)N * T * 4 * H);
        for (int l = 0; l < NL; ++l) hseq[l].alloc((size_t)N * T * H);
        {
            ec::ConvArgs a{};
            a.xa = x; a.La = T; a.Ca = H; a.taps = 1; a.A = m.xproj.A.p; a.bias = m.xproj.bias.p; a.M = 4 * H; a.K = H; a.Lq = T; a.N = N;
            a.out = xp.p; a.out_per_n = (long long)T * 4 * H;
            ec::launch_conv(a, s);
        }
        const size_t smem = ((size_t)(2 * NL - 1) * 16 * H + (size_t)NL * ec::LSTM_BC * H + NL * 16 * ec::LSTM_BC + NL * ec::LSTM_UNITS * ec::LSTM_BC) * sizeof(float);
        B2A_CHECK(smem <= 220 * 1024, B2A_ERR_INVALID_INPUT, "encodec: LSTM slice does not fit shared memory");
        B2A_CUDA(cudaFuncSetAttribute(ec::lstm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const int grid = H / ec::LSTM_UNITS;
        int per_sm = 0;
        B2A_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ec::lstm_kernel, 256, smem));
        B2A_CHECK((long long)per_sm * num_sms >= grid, B2A_ERR_INVALID_INPUT, "encodec: LSTM too wide for a co-resident grid");
        for (int n0 = 0; n0 < N; n0 += ec::LSTM_BC) {
            ec::LstmArgs la{};
            la.xproj = xp.p; la.skip = x; la.out = y; la.bar = bar.p; la.n0 = n0; la.nb = std::min(ec::LSTM_BC, N - n0); la.T = T; la.H = H; la.NL = NL;
            for (int l = 0; l < NL; ++l) { la.Wh[l] = m.Wh[l].p; la.Wx[l] = m.Wx[l].p; la.bias[l] = m.b[l].p; la.hseq[l] = hseq[l].p; }
            B2A_CUDA(cudaMemsetAsync(bar.p, 0, sizeof(unsigned), s));
            void* params[] = {&la};
            B2A_CUDA(cudaLaunchCooperativeKernel((void*)ec::lstm_kernel, dim3(grid), dim3(256), params, smem, s));
            count_launch();
        }
        std::swap(x, y);
    }

    // d_codes [n_chunks, B, n_q_used, T] int32 (device), d_scales [n_chunks, B] or null -> d_wave [B, out_len, channels]
    void decode_dev(const int* d_codes, int n_chunks, int B, int nq, int T, const float* d_scales, float* d_wave, cudaStream_t s) {
        B2A_CHECK(n_chunks >= 1 && B >= 1 && T >= 1, B2A_ERR_INVALID_INPUT, "encodec decode: empty input");
        B2A_CHECK(nq >= 1 && nq <= n_q, B2A_ERR_INVALID_INPUT, "encodec decode: more codebooks than the checkpoint holds");
        B2A_CHECK(chunk_length() != 0 || n_chunks == 1, B2A_ERR_AUDIO_DECODING_FAILED, "Expected one frame");   // Encodec.swift:375-377
        B2A_CUDA(cudaSetDevice(device));
        const int N = n_chunks * B, CH = cfg.audio_channels;
        const long long Lfin = (long long)T * hop();
        B2A_CHECK((long long)N * Lfin * 64 < (1ll << 40) && Lfin < (1ll << 30), B2A_ERR_INVALID_INPUT, "encodec decode: too long");
        // the widest activation: max over stages of N * L * C
        size_t big = (size_t)N * T * std::max(dim0, 4 * dim0);
        {
            long long L = T;
            for (auto& st : stages) {
                // under time_group_norm the transposed conv writes its untrimmed (L + taps - 1) * s rows
                if (gn) big = std::max(big, (size_t)((long long)N * (L + st.taps - 1) * st.ratio * st.cout));
                L *= st.ratio; big = std::max(big, (size_t)((long long)N * L * st.cout));
            }
        }
        bufA.alloc(big); bufB.alloc(big); bufC.alloc(big);
        if (gn) { bufD.alloc(big); gn_alloc(N); }
        float* x = bufA.p; float* y = bufB.p; float* z = bufC.p;
        // 1. RVQ decode
        ec::rvq_sum_kernel<<<(unsigned)((long long)N * T), 128, 0, s>>>(d_codes, books.p, x, nq, T, cfg.codebook_size, cfg.codebook_dim);
        count_launch();
        // 2. first conv
        {
            ec::ConvArgs a{};
            a.xa = x; a.La = T; a.Ca = cfg.hidden_size; a.taps = cfg.kernel_size; pads(cfg.kernel_size, a.padL); a.reflect = cfg.pad_mode_reflect;
            a.A = conv0.A.p; a.bias = conv0.bias.p; a.M = conv0.M; a.K = conv0.K; a.Lq = T; a.N = N; a.out = y; a.out_per_n = (long long)T * dim0;
            ec::launch_conv(a, s);
            if (gn) gn_inplace(y, norm0, N, T, dim0, nullptr, s);
            std::swap(x, y);
        }
        // 3. LSTM block
        run_lstm_block(lstm, x, y, N, T, dim0, s);
        // 4. upsampling stages
        long long L = T;
        for (auto& st : stages) {
            const int s_ = st.ratio, k = 2 * s_;
            const long long Lo = L * s_;                      // after the trim: (L-1)*s + k - (k - s)
            {
                const int padding_total = k - s_;
                const int pr = cfg.use_causal_conv ? (int)std::ceil((float)padding_total * cfg.trim_right_ratio) : padding_total / 2;
                const int pl = padding_total - pr;
                ec::ConvArgs a{};
                a.xa = x; a.La = (int)L; a.Ca = st.cin; a.taps = st.taps; a.backward = 1; a.elu_a = 1;
                a.A = st.up.A.p; a.bias = st.up.bias.p; a.M = st.up.M; a.K = st.up.K; a.Lq = (int)L + st.taps - 1; a.N = N;
                if (gn) {
                    // conv, then norm over all (L + taps - 1) * s rows, then trim (EncodecLayers.swift:251-272): the conv writes
                    // untrimmed into y and the apply reads from row pl into x
                    const long long Lfull = (L + st.taps - 1) * s_;
                    a.out = y; a.out_per_n = Lfull * st.cout; a.shift = 0;
                    ec::launch_conv(a, s);
                    gn_stats(y, N, Lfull, st.cout, gn_sa.p, s);
                    ec::GnApplyArgs g{};
                    g.xa = y; g.sa = gn_sa.p; g.ga = st.nup.g.p; g.ba = st.nup.b.p; g.rows_a = Lfull; g.off_a = pl;
                    g.out = x; g.L = Lo; g.C = st.cout;
                    gn_apply(g, N, s);
                } else {
                    a.out = y; a.out_per_n = Lo * st.cout; a.shift = (long long)pl * st.cout;
                    ec::launch_conv(a, s);
                    std::swap(x, y);
                }
            }
            L = Lo;
            if (gn) run_resnet_gn(st.res, x, y, z, bufD.p, N, L, st.cout, s);
            else run_resnet(st.res, x, y, z, N, L, st.cout, s);
        }
        // 5. ELU -> last conv (+ per-chunk scale), 6. overlap-add when chunked
        const bool chunked = chunk_length() != 0;
        float* dst = d_wave;
        if (chunked) { chunks.alloc((size_t)N * L * CH); dst = chunks.p; }
        {
            int padL; pads(cfg.last_kernel_size, padL);
            const int C = cfg.num_filters, k = cfg.last_kernel_size;
            const size_t smem = ((size_t)(256 + k - 1) * (C + 1) + (size_t)CH * k * C) * sizeof(float);
            B2A_CHECK(smem <= 200 * 1024, B2A_ERR_INVALID_INPUT, "encodec: last conv too wide");
            B2A_CUDA(cudaFuncSetAttribute(ec::final_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            // under time_group_norm the chunk scale follows the last conv's norm (decodeFrame, Encodec.swift:294-301)
            ec::final_conv_kernel<<<dim3(cdiv(L, 256), N), 256, smem, s>>>(x, wlast.p, blast.p, gn ? nullptr : d_scales, dst, (int)L, C, k, CH,
                                                                          padL, cfg.pad_mode_reflect);
            count_launch();
            if (gn) gn_inplace(dst, nlast, N, L, CH, d_scales, s);
        }
        if (chunked) {
            const long long total = out_len(n_chunks, T);
            const int hopc = chunk_stride() > 0 ? chunk_stride() : 1;
            ec::overlap_add_kernel<<<dim3(cdiv(total, 256), B), 256, 0, s>>>(chunks.p, d_wave, n_chunks, B, (int)L, CH, hopc, total);
            count_launch();
        }
        B2A_CUDA(cudaGetLastError());
    }

    // ---- encode (Encodec.swift:212-291)
    // EncodecConv1d's output length (EncodecLayers.swift:139-145, 191-205): padding_total = k - stride plus the extra right
    // padding that completes the last window, in the reference's Float arithmetic
    static long long conv_out_len(long long L, int k, int stride) {
        const int pt = k - stride;
        const float n_frames = (float)(L - k + pt) / (float)stride + 1.f;
        const long long ideal = ((long long)std::ceil(n_frames) - 1) * stride + k - pt;
        const long long extra = std::max(0ll, ideal - L);
        return (L + pt + extra - k) / stride + 1;
    }
    struct EncShape { int n_chunks, chunk_len, chunk_stride, frames; };
    // encode's chunk loop (:267-287): offsets 0, stride, ... below samples - (chunk_len - stride), every chunk the same length
    // (what MLX.stacked needs); frames = the encoder's output length for one chunk
    EncShape encoded_shape(long long samples) const {
        B2A_CHECK(has_enc, B2A_ERR_MODEL_NOT_INITIALIZED, enc_error);
        B2A_CHECK(samples >= 1, B2A_ERR_INVALID_INPUT, "encodec encode: empty input");
        B2A_CHECK(samples < (1ll << 30), B2A_ERR_INVALID_INPUT, "encodec encode: too long");
        const long long clen = chunk_length() > 0 ? chunk_length() : samples;
        const long long stride = chunk_stride() > 0 ? chunk_stride() : samples;
        const long long step = clen - stride;
        B2A_CHECK(samples - step > 0, B2A_ERR_INVALID_INPUT, "encodec encode: input shorter than one chunk step");
        const long long n = (samples - step + stride - 1) / stride;
        const long long first = std::min(clen, samples), last = std::min(clen, samples - (n - 1) * stride);
        B2A_CHECK(first == last && last >= 1, B2A_ERR_INVALID_INPUT,
                  "encodec encode: the last chunk would be shorter than the others (chunks of unequal length cannot be stacked)");
        long long L = first;
        for (auto& st : estages) L = conv_out_len(L, 2 * st.ratio, st.ratio);
        return EncShape{(int)n, (int)first, (int)(n > 1 ? stride : 0), (int)L};
    }

    // d_audio [B, samples, audio_channels] -> d_codes [n_chunks, B, nq, frames] (+ d_scales [n_chunks, B] when normalize, if
    // given); the latent z stays in zbuf [n_chunks*B, frames, hidden]
    void encode_dev(const float* d_audio, int B, long long samples, int nq, int* d_codes, float* d_scales, cudaStream_t s) {
        B2A_CHECK(B >= 1, B2A_ERR_INVALID_INPUT, "encodec encode: empty input");
        const EncShape sh = encoded_shape(samples);
        B2A_CHECK(nq >= 1 && nq <= n_q, B2A_ERR_INVALID_INPUT, "encodec encode: n_q must be in [1, the codebooks the checkpoint holds]");
        B2A_CUDA(cudaSetDevice(device));
        const int N = sh.n_chunks * B, CH = cfg.audio_channels, F = cfg.num_filters, D = cfg.codebook_dim;
        long long L = sh.chunk_len;
        B2A_CHECK((long long)N * L * 64 < (1ll << 40) && (long long)B * samples * CH < (1ll << 40), B2A_ERR_INVALID_INPUT, "encodec encode: too long");
        // the widest activation: max over stages of N * L * C (the LSTM and z have buffers of their own)
        size_t big = (size_t)N * L * F;
        {
            long long l = L;
            for (auto& st : estages) { l = conv_out_len(l, 2 * st.ratio, st.ratio); big = std::max(big, (size_t)((long long)N * l * st.cout)); }
        }
        bufA.alloc(big); bufB.alloc(big); bufC.alloc(big);
        if (gn) { bufD.alloc(big); gn_alloc(N); }
        float* x = bufA.p; float* y = bufB.p; float* z = bufC.p;
        // 1. per-chunk scale (normalize), 2. stem on the waveform in place
        const float* sc = nullptr;
        if (cfg.normalize) {
            float* dst = d_scales;
            if (!dst) { scales.alloc((size_t)N); dst = scales.p; }
            ec::chunk_scale_kernel<<<N, 256, 0, s>>>(d_audio, dst, B, samples, CH, sh.chunk_len, sh.chunk_stride);
            count_launch();
            sc = dst;
        }
        {
            int padL; pads(cfg.kernel_size, padL);
            const int k = cfg.kernel_size;
            const size_t smem = ((size_t)F * k * CH + (size_t)(ec::STEM_T + k - 1) * CH) * sizeof(float);
            B2A_CHECK(smem <= 200 * 1024, B2A_ERR_INVALID_INPUT, "encodec: stem too wide");
            B2A_CUDA(cudaFuncSetAttribute(ec::stem_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ec::stem_conv_kernel<<<dim3(cdiv(L, ec::STEM_T), N), 256, smem, s>>>(d_audio, wstem.p, bstem.p, sc, x, B, samples, CH, sh.chunk_len,
                                                                                sh.chunk_stride, F, k, padL, cfg.pad_mode_reflect);
            count_launch();
            if (gn) gn_inplace(x, nstem, N, L, F, nullptr, s);
        }
        // 3. downsampling stages: resnet, ELU + conv k = 2r stride r (one implicit-GEMM launch; ELU fused on its input)
        for (auto& st : estages) {
            if (cfg.num_residual_layers > 0) {
                if (gn) run_resnet_gn(st.res, x, y, z, bufD.p, N, L, st.cin, s);
                else run_resnet(st.res, x, y, z, N, L, st.cin, s);
            }
            const int r = st.ratio, k = 2 * r;
            const long long Lo = conv_out_len(L, k, r);
            ec::ConvArgs a{};
            a.xa = x; a.La = (int)L; a.Ca = st.cin; a.taps = k; a.stride = r; a.elu_a = 1; a.reflect = cfg.pad_mode_reflect;
            a.padL = cfg.use_causal_conv ? k - r : (k - r) - (k - r) / 2;     // the right pad and the extra pad: src_index's edge rule
            a.A = st.down.A.p; a.bias = st.down.bias.p; a.M = st.down.M; a.K = st.down.K; a.Lq = (int)Lo; a.N = N;
            a.out = y; a.out_per_n = Lo * st.cout;
            ec::launch_conv(a, s);
            if (gn) gn_inplace(y, st.ndown, N, Lo, st.cout, nullptr, s);
            std::swap(x, y);
            L = Lo;
        }
        const int T = (int)L, H = F << estages.size();
        // 4. LSTM block, 5. ELU -> last conv -> z
        run_lstm_block(elstm, x, y, N, T, H, s);
        zbuf.alloc((size_t)N * T * D);
        {
            ec::ConvArgs a{};
            a.xa = x; a.La = T; a.Ca = H; a.taps = cfg.last_kernel_size; pads(cfg.last_kernel_size, a.padL); a.reflect = cfg.pad_mode_reflect; a.elu_a = 1;
            a.A = elast.A.p; a.bias = elast.bias.p; a.M = elast.M; a.K = elast.K; a.Lq = T; a.N = N; a.out = zbuf.p; a.out_per_n = (long long)T * D;
            ec::launch_conv(a, s);
            if (gn) gn_inplace(zbuf.p, nelast, N, T, D, nullptr, s);
        }
        // 6. residual VQ encode
        {
            const size_t smem = ec::rvq_encode_smem(D);
            B2A_CHECK(smem <= 220 * 1024, B2A_ERR_INVALID_INPUT, "encodec: codebook_dim too large for the code search");
            B2A_CUDA(cudaFuncSetAttribute(ec::rvq_encode_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            const int rows = N * T;
            ec::rvq_encode_kernel<false><<<cdiv(rows, ec::VQ_FT), 256, smem, s>>>(zbuf.p, D, books.p, book_sq.p, d_codes, rows, T, nq, 0, nq,
                                                                                  cfg.codebook_size, D);
            count_launch();
        }
        B2A_CUDA(cudaGetLastError());
    }
};

extern "C" {

int32_t b2a_encodec_create(int32_t device, const b2a_encodec_config* cfg, const b2a_tensor* tensors, int32_t n, b2a_encodec** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_encodec_create: null out");
        *out = nullptr;
        B2A_CHECK(cfg && tensors && n > 0, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_encodec_create: missing config or weights");
        TensorTable tt(tensors, n);
        *out = new b2a_encodec(device, *cfg, tt);
    });
}

int64_t b2a_encodec_output_length(const b2a_encodec* h, int32_t n_chunks, int32_t frames) {
    return h && n_chunks >= 1 && frames >= 1 ? h->out_len(n_chunks, frames) : 0;
}
int32_t b2a_encodec_num_codebooks(const b2a_encodec* h) { return h ? h->n_q : 0; }
void* b2a_encodec_stream(b2a_encodec* h) { return h ? (void*)h->stream : nullptr; }

int32_t b2a_encodec_decode_dev(b2a_encodec* h, const int32_t* d_codes, int32_t n_chunks, int32_t B, int32_t nq, int32_t T,
                               const float* d_scales, float* d_wave, void* stream) {
    return guarded([&] {
        B2A_CHECK(h && d_codes && d_wave, B2A_ERR_INVALID_INPUT, "b2a_encodec_decode_dev: null argument");
        h->decode_dev(d_codes, n_chunks, B, nq, T, d_scales, d_wave, stream ? (cudaStream_t)stream : h->stream);
    });
}

int32_t b2a_encodec_decode(b2a_encodec* h, const int32_t* codes, int32_t n_chunks, int32_t B, int32_t nq, int32_t T,
                           const float* scales, float* wave) {
    return guarded([&] {
        B2A_CHECK(h && codes && wave, B2A_ERR_INVALID_INPUT, "b2a_encodec_decode: null argument");
        B2A_CHECK(n_chunks >= 1 && B >= 1 && T >= 1 && nq >= 1, B2A_ERR_AUDIO_DECODING_FAILED, "b2a_encodec_decode: empty codes");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        const size_t nin = (size_t)n_chunks * B * nq * T, nout = (size_t)B * h->out_len(n_chunks, T) * h->cfg.audio_channels;
        h->codes.alloc(nin); h->wave.alloc(nout);
        B2A_CUDA(cudaMemcpyAsync(h->codes.p, codes, nin * sizeof(int), cudaMemcpyHostToDevice, s));
        const float* dsc = nullptr;
        if (scales) {
            h->scales.alloc((size_t)n_chunks * B);
            B2A_CUDA(cudaMemcpyAsync(h->scales.p, scales, (size_t)n_chunks * B * sizeof(float), cudaMemcpyHostToDevice, s));
            dsc = h->scales.p;
        }
        h->decode_dev(h->codes.p, n_chunks, B, nq, T, dsc, h->wave.p, s);
        B2A_CUDA(cudaMemcpyAsync(wave, h->wave.p, nout * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

int32_t b2a_encodec_encoded_shape(const b2a_encodec* h, int64_t samples, int32_t* n_chunks, int32_t* frames) {
    return guarded([&] {
        B2A_CHECK(h && n_chunks && frames, B2A_ERR_INVALID_INPUT, "b2a_encodec_encoded_shape: null argument");
        const auto sh = h->encoded_shape(samples);
        *n_chunks = sh.n_chunks;
        *frames = sh.frames;
    });
}

int32_t b2a_encodec_encode_dev(b2a_encodec* h, const float* d_audio, int32_t batch, int64_t samples, int32_t n_q, int32_t* d_codes,
                               float* d_scales, void* stream) {
    return guarded([&] {
        B2A_CHECK(h && d_audio && d_codes, B2A_ERR_INVALID_INPUT, "b2a_encodec_encode_dev: null argument");
        h->encode_dev(d_audio, batch, samples, n_q, d_codes, d_scales, stream ? (cudaStream_t)stream : h->stream);
    });
}

// host entry: stage the waveform, encode on the handle's stream, copy codes (and scales) back; z_out (test hook) gets the latent
static void encodec_encode_host(b2a_encodec* h, const float* audio, int32_t batch, int64_t samples, int32_t n_q, int32_t* codes,
                                float* scales, float* z_out) {
    B2A_CHECK(h && audio && (codes || z_out), B2A_ERR_INVALID_INPUT, "b2a_encodec_encode: null argument");
    B2A_CHECK(batch >= 1, B2A_ERR_INVALID_INPUT, "encodec encode: empty input");
    const auto sh = h->encoded_shape(samples);
    B2A_CHECK(n_q >= 1 && n_q <= h->n_q, B2A_ERR_INVALID_INPUT, "encodec encode: n_q must be in [1, the codebooks the checkpoint holds]");
    B2A_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    const size_t nin = (size_t)batch * samples * h->cfg.audio_channels, N = (size_t)sh.n_chunks * batch;
    const size_t ncodes = N * n_q * sh.frames;
    h->audio.alloc(nin); h->codes.alloc(ncodes);
    const bool want_scales = h->cfg.normalize && scales;
    if (want_scales) h->scales.alloc(N);
    B2A_CUDA(cudaMemcpyAsync(h->audio.p, audio, nin * sizeof(float), cudaMemcpyHostToDevice, s));
    h->encode_dev(h->audio.p, batch, samples, n_q, h->codes.p, want_scales ? h->scales.p : nullptr, s);
    if (codes) B2A_CUDA(cudaMemcpyAsync(codes, h->codes.p, ncodes * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (want_scales) B2A_CUDA(cudaMemcpyAsync(scales, h->scales.p, N * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (z_out) B2A_CUDA(cudaMemcpyAsync(z_out, h->zbuf.p, N * sh.frames * h->cfg.codebook_dim * sizeof(float), cudaMemcpyDeviceToHost, s));
    B2A_CUDA(cudaStreamSynchronize(s));
}

int32_t b2a_encodec_encode(b2a_encodec* h, const float* audio, int32_t batch, int64_t samples, int32_t n_q, int32_t* codes,
                           float* scales) {
    return guarded([&] {
        B2A_CHECK(codes, B2A_ERR_INVALID_INPUT, "b2a_encodec_encode: null argument");
        encodec_encode_host(h, audio, batch, samples, n_q, codes, scales, nullptr);
    });
}

int32_t b2a_encodec_encode_latent_test(b2a_encodec* h, const float* audio, int32_t batch, int64_t samples, float* z) {
    return guarded([&] {
        B2A_CHECK(z, B2A_ERR_INVALID_INPUT, "b2a_encodec_encode_latent_test: null argument");
        encodec_encode_host(h, audio, batch, samples, 1, nullptr, nullptr, z);
    });
}

void b2a_encodec_destroy(b2a_encodec* h) { delete h; }

}  // extern "C"
