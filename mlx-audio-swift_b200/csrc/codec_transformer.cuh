// Kernels shared by the Qwen3-TTS speech-tokenizer codec (speech_tokenizer.cu) and the Mimi codec (mimi.cu): the split-RVQ
// codebook gather, LayerNorm into hi/lo planes, RoPE into a KV cache, causal attention over that cache, and the streaming
// history carries of the fp32 and planar activations (DESIGN.md §3.8, §3.8b, §3.11).
#pragma once
#include "common.cuh"
#include "conv_gemm.cuh"

#include <cstring>
#include <vector>

namespace b2a {
namespace st {

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ void put_planes(bf16* base, long long plane, long long idx, float v, int f16) {
    cg::put_hilo16(reinterpret_cast<uint16_t*>(base), plane, idx, v, f16);
}

// codes [B, nq, T] -> planes [2][B*T][2*D2]: channels [0, D2) = sum of the semantic codebooks, [D2, 2*D2) = sum of the rest
static __global__ void rvq_gather_kernel(const int* __restrict__ codes, const float* __restrict__ emb /*[nq][bins][D2]*/, bf16* __restrict__ out,
                                  int B, int T, int nq, int nq_model, int nsem, int bins, int D2, int f16) {
    const long long n = blockIdx.x;
    const int b = (int)(n / T), t = (int)(n - (long long)b * T);
    const long long plane = (long long)B * T * 2 * D2;
    for (int c = threadIdx.x; c < D2; c += blockDim.x) {
        float s0 = 0.f, s1 = 0.f;
        for (int qi = 0; qi < nq && qi < nq_model; ++qi) {
            int code = codes[((long long)b * nq + qi) * T + t];
            code = code < 0 ? 0 : (code >= bins ? bins - 1 : code);
            const float v = emb[((long long)qi * bins + code) * D2 + c];
            if (qi < nsem) s0 += v; else s1 += v;
        }
        put_planes(out, plane, n * 2 * D2 + c, s0, f16);
        put_planes(out, plane, n * 2 * D2 + D2 + c, s1, f16);
    }
}

constexpr int RN_THREADS = 128;

// RoPE on q (in place) and k (into the cache), v copied into the cache.  qkv [N, (nh + 2 nkv) * hd] fp32.  Frequency i rotates the
// pair (i, i + hd/2) (rotate-half: the decoder, DecoderTransformer) or (2i, 2i + 1) (INTERLEAVED: the encoder, MLX RoPE traditional:
// true, Mimi/Transformer.swift:130).
template <bool INTERLEAVED>
__global__ void rope_cache_kernel(float* __restrict__ qkv, float* __restrict__ Kc, float* __restrict__ Vc, const float* __restrict__ inv_freq,
                                  int T, int pos0, int nh, int nkv, int hd, int cap) {
    const long long n = blockIdx.x;
    const int b = (int)(n / T), t = (int)(n - (long long)b * T);
    const int pos = pos0 + t, half = hd / 2, ld = (nh + 2 * nkv) * hd;
    float* row = qkv + n * ld;
    for (int idx = threadIdx.x; idx < (nh + nkv) * half; idx += blockDim.x) {
        const int head = idx / half, i = idx - head * half;
        float sn, cs;
        sincosf((float)pos * inv_freq[i], &sn, &cs);
        const int i1 = INTERLEAVED ? 2 * i : i, i2 = INTERLEAVED ? 2 * i + 1 : i + half;
        const float x1 = row[head * hd + i1], x2 = row[head * hd + i2];
        const float o1 = x1 * cs - x2 * sn, o2 = x2 * cs + x1 * sn;
        if (head < nh) {
            row[head * hd + i1] = o1;
            row[head * hd + i2] = o2;
        } else {
            float* dst = Kc + (((long long)b * nkv + (head - nh)) * cap + pos) * hd;
            dst[i1] = o1;
            dst[i2] = o2;
        }
    }
    for (int idx = threadIdx.x; idx < nkv * hd; idx += blockDim.x) {
        const int kvh = idx / hd, d = idx - kvh * hd;
        Vc[(((long long)b * nkv + kvh) * cap + pos) * hd + d] = row[(nh + nkv) * hd + idx];
    }
}

// causal attention of the chunk's T queries over cache positions [key_lo, pos0 + t]: one warp per (query, head), each lane
// owns hd / 32 consecutive dims, online softmax, four keys in flight.  Output -> planes [2][N][nh * hd].  key_lo is one left edge
// for the whole call (Mimi's context window, Transformer.swift:156-164); 0 attends the whole cache.
constexpr int AT_WARPS = 4;
template <int DPL>
__global__ void __launch_bounds__(AT_WARPS * 32)
attn_kernel(const float* __restrict__ qkv, const float* __restrict__ Kc, const float* __restrict__ Vc, bf16* __restrict__ out,
            int B, int T, int pos0, int nh, int nkv, int cap, float scale, int f16, int key_lo) {
    constexpr int HD = DPL * 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t = blockIdx.x * AT_WARPS + warp, h = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    const long long n = (long long)b * T + t;
    const int ld = (nh + 2 * nkv) * HD, kvh = h / (nh / nkv);
    float q[DPL], acc[DPL];
#pragma unroll
    for (int d = 0; d < DPL; ++d) { q[d] = qkv[n * ld + h * HD + lane * DPL + d] * scale; acc[d] = 0.f; }
    const float* Kb = Kc + ((long long)b * nkv + kvh) * cap * HD + lane * DPL;
    const float* Vb = Vc + ((long long)b * nkv + kvh) * cap * HD + lane * DPL;
    float m = -INFINITY, l = 0.f;
    const int nkeys = pos0 + t + 1;
    for (int p0 = key_lo; p0 < nkeys; p0 += 4) {
        float s[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            float d0 = 0.f;
            if (p0 + u < nkeys) {
#pragma unroll
                for (int d = 0; d < DPL; ++d) d0 = fmaf(q[d], Kb[(long long)(p0 + u) * HD + d], d0);
            }
            s[u] = d0;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) s[u] = warp_sum(s[u]);
        float mx = m;
#pragma unroll
        for (int u = 0; u < 4; ++u) if (p0 + u < nkeys) mx = fmaxf(mx, s[u]);
        const float corr = __expf(m - mx);      // m = -inf on the first pass: exp(-inf) = 0
        l *= corr;
#pragma unroll
        for (int d = 0; d < DPL; ++d) acc[d] *= corr;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (p0 + u < nkeys) {
                const float e = __expf(s[u] - mx);
                l += e;
#pragma unroll
                for (int d = 0; d < DPL; ++d) acc[d] = fmaf(e, Vb[(long long)(p0 + u) * HD + d], acc[d]);
            }
        }
        m = mx;
    }
    const float inv = 1.0f / l;
    const long long N = (long long)B * T;
#pragma unroll
    for (int d = 0; d < DPL; ++d) put_planes(out, N * nh * HD, n * nh * HD + h * HD + lane * DPL + d, acc[d] * inv, f16);
}

// LayerNorm with bias over channels -> planes [2][N][C]   (MLXNN LayerNorm: (x - mean) * rsqrt(var + eps) * w + b)
static __global__ void __launch_bounds__(RN_THREADS)
layernorm_planes_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias, bf16* __restrict__ out,
                        long long N, int C, float eps, int f16) {
    __shared__ float red[RN_THREADS / 32];
    const long long n = blockIdx.x;
    float s = 0.f;
    for (int c = threadIdx.x; c < C; c += RN_THREADS) s += x[n * C + c];
    const float mean = block_sum<RN_THREADS>(s, red) / (float)C;
    float q = 0.f;
    for (int c = threadIdx.x; c < C; c += RN_THREADS) { const float d = x[n * C + c] - mean; q += d * d; }
    const float r = rsqrtf(block_sum<RN_THREADS>(q, red) / (float)C + eps);
    for (int c = threadIdx.x; c < C; c += RN_THREADS) put_planes(out, N * C, n * C + c, (x[n * C + c] - mean) * r * w[c] + bias[c], f16);
}

// fp32 history: new[b][f] = last H frames of [old | x]
static __global__ void state_update_f32_kernel(const float* __restrict__ x, const float* __restrict__ old, float* __restrict__ nw, int B, int T, int H, int C) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * H * C) return;
    const int c = (int)(i % C);
    const long long bf = i / C;
    const int f = (int)(bf % H), b = (int)(bf / H);
    const int src = T + f;        // frame index in [old (H) | x (T)]
    nw[i] = src < H ? old[((long long)b * H + src) * C + c] : x[((long long)b * T + (src - H)) * C + c];
}

// bf16 planes with a history prefix: X = [2][B][H + T][C].  Copies the old state into frames [0, H) and saves the last H
// frames of [old | new] as the new state (old and new are different buffers).  8 channels (16 bytes) per thread.
static __global__ void carry_planes_kernel(bf16* __restrict__ X, const bf16* __restrict__ old, bf16* __restrict__ nw, int B, int T, int H, int C8) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long per_plane = (long long)B * H * C8;
    if (i >= 2 * per_plane) return;
    const int c = (int)(i % C8);
    long long r = i / C8;
    const int f = (int)(r % H); r /= H;
    const int b = (int)(r % B), p = (int)(r / B);
    const uint4* o4 = reinterpret_cast<const uint4*>(old);
    uint4* n4 = reinterpret_cast<uint4*>(nw);
    uint4* x4 = reinterpret_cast<uint4*>(X);
    const long long xrow = ((long long)p * B + b) * (H + T);
    const uint4 ov = o4[i];
    x4[(xrow + f) * C8 + c] = ov;
    const int src = T + f;
    n4[i] = src < H ? o4[(((long long)p * B + b) * H + src) * C8 + c] : x4[(xrow + src) * C8 + c];
}

struct PlaneState { DBuf<bf16> s[2]; int H = 0, C = 0; };      // [2][B][H][C]
struct F32State { DBuf<float> s[2]; int H = 0, C = 0; };       // [B][H][C]

// transposed conv, MLX [out, k, in], k = n * r: rows m = rho * out + co, tap j <-> input frame q - (n - 1 - j) <-> kernel index rho + (n - 1 - j) * r
inline std::vector<float> convt_weight(const std::vector<float>& w, int out, int k, int in, int r) {
    const int n = k / r;
    std::vector<float> g((size_t)r * out * n * in);
    for (int rho = 0; rho < r; ++rho)
        for (int co = 0; co < out; ++co)
            for (int j = 0; j < n; ++j)
                memcpy(&g[(((size_t)rho * out + co) * n + j) * in], &w[((size_t)co * k + rho + (size_t)(n - 1 - j) * r) * in], (size_t)in * sizeof(float));
    return g;
}

}  // namespace st
}  // namespace b2a
