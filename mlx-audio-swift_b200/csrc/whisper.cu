// Whisper encoder-decoder STT for sm_90a.  Replaces (reference paths):
//   Sources/MLXAudioSTT/Models/Whisper/WhisperLayers.swift:11-73    WhisperAttention (k_proj has no bias)
//   Sources/MLXAudioSTT/Models/Whisper/WhisperLayers.swift:77-156   encoder (conv stem k3/k3s2 + exact GELU, pre-LN layers)
//   Sources/MLXAudioSTT/Models/Whisper/WhisperLayers.swift:169-328  decoder (self KV cache, cross K/V computed once, tied logits)
//   Sources/MLXAudioSTT/Models/Whisper/WhisperModel.swift:186-309   transcribeChunk greedy loop + suppress masks
//   Sources/MLXAudioSTT/Models/Whisper/WhisperAudio.swift:38-87     log-mel (csrc/mel.cu, kind 1)
//
// Every Linear / Conv is the wgmma "weights-as-A" GEMM (csrc/tc_gemm.cuh) on bf16 weights with bf16 hi/lo
// activation pairs (fp32-activation accuracy): the conv stem through an im2col that writes the hi/lo tiles directly,
// encoder layers with 64-token tiles, decoder steps with up to 16 rows in one 32-column tile.  Residual adds,
// biases and GELU are GEMM epilogues.  Attention: the wgmma flash-attention kernel (csrc/attn_tc.cuh, fp16 operands) for the
// 1500x1500 encoder maps and a flash-decoding kernel (bulk async K/V loads, split over keys) for the decoder's self and cross attention.
#include "common.cuh"
#include "tc_gemm.cuh"
#include "attn_tc.cuh"

#include <algorithm>
#include <chrono>
#include <memory>
#include <type_traits>
#include <cmath>
#include <cstdlib>

namespace b2a {
namespace wh {

typedef __nv_bfloat16 bf16;
constexpr int HD = 64;               // every Whisper size uses 64-dim heads
constexpr int ENC_HALF = 64;         // tokens per 128-row tile (encoder / prompt side)
constexpr int DEC_HALF = 16;         // decoder step: up to 16 rows as hi/lo in a 32-row tile

// ------------------------------------------------------------------------------------------------
// LayerNorm (eps 1e-5, biased variance) -> bf16 hi/lo.  Optionally first adds a table row
// (encoder positional embedding, WhisperLayers.swift:150) into the residual stream.
// ------------------------------------------------------------------------------------------------
constexpr int LN_THREADS = 256, LN_MAXV = 8;
__global__ void __launch_bounds__(LN_THREADS)
layernorm_hilo_kernel(float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                      bf16* __restrict__ out, int d, int half, const float* __restrict__ addend, int add_mod) {
    __shared__ float red[LN_THREADS / 32];
    pdl_trigger();
    pdl_wait();
    const long long row = blockIdx.x;
    const int tid = threadIdx.x;
    float* xr = x + row * d;
    float v[LN_MAXV];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < LN_MAXV; ++j) {
        const int i = tid + j * LN_THREADS;
        float val = 0.f;
        if (i < d) {
            val = xr[i];
            if (addend) { val += addend[(row % add_mod) * d + i]; xr[i] = val; }
        }
        v[j] = val;
        s += val;
    }
    s = warp_sum(s);
    if ((tid & 31) == 0) red[tid >> 5] = s;
    __syncthreads();
    float mean = 0.f;
#pragma unroll
    for (int i = 0; i < LN_THREADS / 32; ++i) mean += red[i];
    mean /= (float)d;
    __syncthreads();
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < LN_MAXV; ++j) {
        const int i = tid + j * LN_THREADS;
        if (i < d) { const float c = v[j] - mean; q += c * c; }
    }
    q = warp_sum(q);
    if ((tid & 31) == 0) red[tid >> 5] = q;
    __syncthreads();
    float var = 0.f;
#pragma unroll
    for (int i = 0; i < LN_THREADS / 32; ++i) var += red[i];
    const float r = rsqrtf(var / (float)d + 1e-5f);
#pragma unroll
    for (int j = 0; j < LN_MAXV; ++j) {
        const int i = tid + j * LN_THREADS;
        if (i < d) tc::store_hilo(out, d, row, i, (v[j] - mean) * r * w[i] + b[i], half);
    }
}

// Same LayerNorm for many rows (the encoder: 24000 rows of 512): one WARP per row, 8 rows per CTA, float4 loads and 8-byte hi / lo
// stores, no shared memory.  The one-CTA-per-row kernel above moved 98 MB in 75 us (1.3 TB/s); d <= 1024 and d % 128 == 0.
constexpr int LNW_ROWS = 8, LNW_MAXV = 8;            // float4 per lane
__global__ void __launch_bounds__(LNW_ROWS * 32)
layernorm_hilo_rows_kernel(float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b, bf16* __restrict__ out,
                           long long rows, int d, int half, const float* __restrict__ addend, int add_mod) {
    pdl_trigger();
    pdl_wait();
    const long long row = (long long)blockIdx.x * LNW_ROWS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31, nv = d / 128;           // float4 per lane: element index (lane + 32 j) * 4
    if (row >= rows) return;
    float4* xr = reinterpret_cast<float4*>(x + row * d);
    float4 v[LNW_MAXV];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < LNW_MAXV; ++j) {
        if (j < nv) {
            float4 t = xr[lane + 32 * j];
            if (addend) {
                const float4 ad = reinterpret_cast<const float4*>(addend + (row % add_mod) * d)[lane + 32 * j];
                t.x += ad.x; t.y += ad.y; t.z += ad.z; t.w += ad.w;
                xr[lane + 32 * j] = t;
            }
            v[j] = t;
            s += (t.x + t.y) + (t.z + t.w);
        }
    }
    s = warp_sum(s);
    const float mean = s / (float)d;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < LNW_MAXV; ++j) {
        if (j < nv) {
            const float c0 = v[j].x - mean, c1 = v[j].y - mean, c2 = v[j].z - mean, c3 = v[j].w - mean;
            q += (c0 * c0 + c1 * c1) + (c2 * c2 + c3 * c3);
        }
    }
    q = warp_sum(q);
    const float r = rsqrtf(q / (float)d + 1e-5f);
    const long long orow = (row / half) * 2 * half + (row % half);
    uint2* oh = reinterpret_cast<uint2*>(out + orow * d);
    uint2* ol = reinterpret_cast<uint2*>(out + (orow + half) * d);
#pragma unroll
    for (int j = 0; j < LNW_MAXV; ++j) {
        if (j < nv) {
            const float4 g = reinterpret_cast<const float4*>(w)[lane + 32 * j], bb = reinterpret_cast<const float4*>(b)[lane + 32 * j];
            const float y[4] = {(v[j].x - mean) * r * g.x + bb.x, (v[j].y - mean) * r * g.y + bb.y, (v[j].z - mean) * r * g.z + bb.z,
                                (v[j].w - mean) * r * g.w + bb.w};
            unsigned short hs[4], ls[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const bf16 hi = __float2bfloat16_rn(y[e]);
                hs[e] = __bfloat16_as_ushort(hi);
                ls[e] = __bfloat16_as_ushort(__float2bfloat16_rn(y[e] - __bfloat162float(hi)));
            }
            oh[lane + 32 * j] = make_uint2((unsigned)hs[0] | ((unsigned)hs[1] << 16), (unsigned)hs[2] | ((unsigned)hs[3] << 16));
            ol[lane + 32 * j] = make_uint2((unsigned)ls[0] | ((unsigned)ls[1] << 16), (unsigned)ls[2] | ((unsigned)ls[3] << 16));
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Conv stem as GEMMs: im2col writes [x[t*stride-1] | x[t*stride] | x[t*stride+1]] (zero padded) as hi/lo rows.
// in: [B, Tin, C] fp32 (NLC).  out: [2 * Tp, Kp] bf16, Kp >= 3C (extra columns zero).
// ------------------------------------------------------------------------------------------------
__global__ void im2col3_kernel(const float* __restrict__ in, bf16* __restrict__ out, int Tin, int Tout, int C, int Kp,
                               int stride) {
    const long long tok = blockIdx.x;             // b * Tout + t
    const int b = (int)(tok / Tout), t = (int)(tok - (long long)b * Tout);
    for (int i = threadIdx.x; i < Kp; i += blockDim.x) {
        float v = 0.f;
        if (i < 3 * C) {
            const int k = i / C, c = i - k * C;
            const int ti = t * stride + k - 1;
            if (ti >= 0 && ti < Tin) v = in[((long long)b * Tin + ti) * C + c];
        }
        tc::store_hilo(out, Kp, tok, i, v, ENC_HALF);
    }
}

// cross K/V: token-major projection [B*T, 2d] -> head-major fp16 caches [B][nh][T][64]   (WhisperLayers.swift:217-234).  The
// cross-attention of a decode step reads all of it (16 x 8 x 1500 x 64 x 2 tensors x 6 layers = 590 MB per step in fp32, the largest
// single item of the step): fp16 halves that.  Same operand precision as the encoder attention (attn_tc.cuh), fp32 accumulation.
__global__ void kv_relayout_kernel(const float* __restrict__ kv, __half* __restrict__ kc, __half* __restrict__ vc, int T, int d,
                                   int nh) {
    const long long tok = blockIdx.x;
    const int b = (int)(tok / T), t = (int)(tok - (long long)b * T);
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
        const int h = i / HD, c = i - h * HD;
        const long long dst = (((long long)b * nh + h) * T + t) * HD + c;
        kc[dst] = __float2half_rn(kv[tok * 2 * d + i]);
        vc[dst] = __float2half_rn(kv[tok * 2 * d + d + i]);
    }
}

// ------------------------------------------------------------------------------------------------
// Decoder attention, one query per (row, head): flash-decoding over key splits, K/V fetched with one
// cp.async.bulk each.  APPEND: self-attention over the fp32 cache, 64 keys per CTA -- the new key/value (from the
// fused q|k|v row) is written at position pos[b] first.  Otherwise cross-attention over n_keys fixed fp16 keys,
// 128 per CTA (the same 16 KB per tensor in flight).  Two threads per key.
// ------------------------------------------------------------------------------------------------
constexpr int DA_CAP = 64, DA_CAP_CROSS = 128;
struct DecAttnArgs {
    const float* q;        // [B, ldq] fp32, head h at column q_off + h*64
    const float* kv_new;   // APPEND: [B, ldq] fp32, key at k_off + h*64, value at v_off + h*64
    const int* pos;        // [B]
    void* kcache;          // [B][nh][max_t][64]  fp32 (APPEND) / fp16 (cross)
    void* vcache;
    bf16* out;             // [2*DEC_HALF, d] hi/lo
    float* part_o;         // [B][nh][S][64]
    float* part_ml;        // [B][nh][S][2]
    int* counters;         // [B][nh]
    int ldq, q_off, k_off, v_off, nh, max_t, n_keys, S, d;
    float scale;
};

template <bool APPEND>
__global__ void __launch_bounds__(APPEND ? 2 * DA_CAP : 2 * DA_CAP_CROSS)
mha_decode_kernel(DecAttnArgs a) {
    using CT = typename std::conditional<APPEND, float, __half>::type;
    constexpr int CAP = APPEND ? DA_CAP : DA_CAP_CROSS, THREADS = 2 * CAP, NSL = THREADS / HD;
    __shared__ __align__(16) CT sK[CAP * HD];
    __shared__ __align__(16) CT sV[CAP * HD];
    __shared__ __align__(16) float sq[HD];
    __shared__ float sc[CAP];
    __shared__ float spo[NSL][HD];
    __shared__ float red[THREADS / 32];
    __shared__ float stat[2];
    __shared__ int s_last;
    __shared__ __align__(8) uint64_t bar;
    const int h = blockIdx.x, b = blockIdx.y, s = blockIdx.z, tid = threadIdx.x;
    pdl_trigger();
    if (!APPEND) {
        // the cross keys / values and the split geometry do not depend on the previous kernel: start the copy before waiting for it
        const int t0 = s * CAP, nk = min(t0 + CAP, a.n_keys) - t0;
        if (tid == 0 && nk > 0) {
            const CT* kc = reinterpret_cast<const CT*>(a.kcache) + (((long long)b * a.nh + h) * a.max_t) * HD;
            const CT* vc = reinterpret_cast<const CT*>(a.vcache) + (((long long)b * a.nh + h) * a.max_t) * HD;
            tc::mbar_init(&bar, 1);
            tc::fence_barrier_init();
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            const uint32_t bytes = (uint32_t)nk * HD * sizeof(CT);
            tc::mbar_arrive_expect_tx(&bar, 2 * bytes);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(tc::smem_u32(sK)), "l"(kc + (long long)t0 * HD), "r"(bytes), "r"(tc::smem_u32(&bar)) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(tc::smem_u32(sV)), "l"(vc + (long long)t0 * HD), "r"(bytes), "r"(tc::smem_u32(&bar)) : "memory");
        }
    }
    pdl_wait();
    const int p = a.pos[b];
    if (p < 0) {                            // inactive row: the CTA must not retire with a bulk copy into its shared memory in flight
        if (!APPEND && tid == 0 && min(s * CAP + CAP, a.n_keys) - s * CAP > 0) tc::mbar_wait(&bar, 0);
        return;
    }
    const int n_total = APPEND ? p + 1 : a.n_keys;
    if (APPEND && p >= a.max_t) return;
    const int S_eff = (n_total + CAP - 1) / CAP;
    if (s >= S_eff) return;
    const int t0 = s * CAP, t1 = min(t0 + CAP, n_total), nk = t1 - t0;
    const bool has_new = APPEND && s == S_eff - 1;
    const int n_load = has_new ? nk - 1 : nk;
    CT* kc = reinterpret_cast<CT*>(a.kcache) + (((long long)b * a.nh + h) * a.max_t) * HD;
    CT* vc = reinterpret_cast<CT*>(a.vcache) + (((long long)b * a.nh + h) * a.max_t) * HD;
    if (APPEND && tid == 0) {
        tc::mbar_init(&bar, 1);
        tc::fence_barrier_init();
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if (n_load > 0) {
            const uint32_t bytes = (uint32_t)n_load * HD * sizeof(CT);
            tc::mbar_arrive_expect_tx(&bar, 2 * bytes);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(tc::smem_u32(sK)), "l"(kc + (long long)t0 * HD), "r"(bytes), "r"(tc::smem_u32(&bar)) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(tc::smem_u32(sV)), "l"(vc + (long long)t0 * HD), "r"(bytes), "r"(tc::smem_u32(&bar)) : "memory");
        } else {
            tc::mbar_arrive(&bar);
        }
    }
    if (tid < HD) {
        sq[tid] = a.q[(long long)b * a.ldq + a.q_off + h * HD + tid];
        if (APPEND && has_new) {
            const float k = a.kv_new[(long long)b * a.ldq + a.k_off + h * HD + tid];
            reinterpret_cast<float*>(kc)[(long long)p * HD + tid] = k;
            reinterpret_cast<float*>(sK)[(p - t0) * HD + tid] = k;
        }
    } else if (APPEND && has_new) {
        const int dd = tid - HD;
        const float v = a.kv_new[(long long)b * a.ldq + a.v_off + h * HD + dd];
        reinterpret_cast<float*>(vc)[(long long)p * HD + dd] = v;
        reinterpret_cast<float*>(sV)[(p - t0) * HD + dd] = v;
    }
    __syncthreads();
    tc::mbar_wait(&bar, 0);
    // scores: 2 threads per key (32 dims each), bank-rotated 16-byte columns
    const int key = tid >> 1, part = tid & 1;
    float acc = 0.f;
    if (key < nk) {
        if (APPEND) {
            const float4* kr = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(sK) + key * HD);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int d4 = part + 2 * ((j + key) & 7);
                const float4 kf = kr[d4];
                const float4 qf = reinterpret_cast<const float4*>(sq)[d4];
                acc = fmaf(qf.x, kf.x, acc); acc = fmaf(qf.y, kf.y, acc); acc = fmaf(qf.z, kf.z, acc); acc = fmaf(qf.w, kf.w, acc);
            }
        } else {
            const uint4* kr = reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(sK) + key * HD);   // 8 x 16 bytes per key
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int g = part + 2 * ((j + key) & 3);         // 8 dims; four consecutive keys x two parts hit the eight 16-byte groups
                const uint4 kk = kr[g];
                const __half2* k2 = reinterpret_cast<const __half2*>(&kk);
                const float4 q0 = reinterpret_cast<const float4*>(sq)[2 * g], q1 = reinterpret_cast<const float4*>(sq)[2 * g + 1];
                const float2 f0 = __half22float2(k2[0]), f1 = __half22float2(k2[1]), f2 = __half22float2(k2[2]), f3 = __half22float2(k2[3]);
                acc = fmaf(q0.x, f0.x, acc); acc = fmaf(q0.y, f0.y, acc); acc = fmaf(q0.z, f1.x, acc); acc = fmaf(q0.w, f1.y, acc);
                acc = fmaf(q1.x, f2.x, acc); acc = fmaf(q1.y, f2.y, acc); acc = fmaf(q1.z, f3.x, acc); acc = fmaf(q1.w, f3.y, acc);
            }
        }
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    float sval = key < nk ? acc * a.scale : -INFINITY;
    float m = sval;
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) red[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) {
        float mm = red[0];
        for (int i = 1; i < THREADS / 32; ++i) mm = fmaxf(mm, red[i]);
        stat[0] = mm;
    }
    __syncthreads();
    const float e = (key < nk && part == 0) ? __expf(sval - stat[0]) : 0.f;
    if (key < nk && part == 0) sc[key] = e;
    const float es = warp_sum(e);
    __syncthreads();
    if ((tid & 31) == 0) red[tid >> 5] = es;
    __syncthreads();
    if (tid == 0) {
        float sum = 0.f;
        for (int i = 0; i < THREADS / 32; ++i) sum += red[i];
        stat[1] = sum;
    }
    // PV: thread = (key residue mod NSL, dim)
    const int sl = tid >> 6, dd = tid & 63;
    float o = 0.f;
    for (int t = sl; t < nk; t += NSL) {
        const float vv = APPEND ? reinterpret_cast<const float*>(sV)[t * HD + dd] : __half2float(reinterpret_cast<const __half*>(sV)[t * HD + dd]);
        o = fmaf(sc[t], vv, o);
    }
    spo[sl][dd] = o;
    __syncthreads();
    const long long pbase = ((long long)b * a.nh + h) * a.S + s;
    if (tid < HD) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < NSL; ++i) t += spo[i][tid];
        a.part_o[pbase * HD + tid] = t;
    }
    if (tid == 0) { a.part_ml[pbase * 2] = stat[0]; a.part_ml[pbase * 2 + 1] = stat[1]; }
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(&a.counters[b * a.nh + h], 1) == S_eff - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (tid < HD) {
        const long long mb = ((long long)b * a.nh + h) * a.S;
        float M = -INFINITY;
        for (int j = 0; j < S_eff; ++j) M = fmaxf(M, a.part_ml[(mb + j) * 2]);
        float L = 0.f, O = 0.f;
        for (int j = 0; j < S_eff; ++j) {
            const float wj = __expf(a.part_ml[(mb + j) * 2] - M);
            L = fmaf(a.part_ml[(mb + j) * 2 + 1], wj, L);
            O = fmaf(a.part_o[(mb + j) * HD + tid], wj, O);
        }
        tc::store_hilo(a.out, a.d, (long long)b, h * HD + tid, O / L, DEC_HALF);
    }
    if (tid == 0) a.counters[b * a.nh + h] = 0;
}

// decoder input: x[b] = embed_tokens[token[b]] + embed_positions[pos[b]]   (WhisperLayers.swift:290-294)
__global__ void wh_embed_kernel(const int* __restrict__ tokens, const int* __restrict__ pos, const bf16* __restrict__ embed,
                                const float* __restrict__ pos_emb, float* __restrict__ x, int d, int V, int max_pos) {
    pdl_trigger();
    pdl_wait();
    const int b = blockIdx.x;
    const int tok = min(max(tokens[b], 0), V - 1), p = min(max(pos[b], 0), max_pos - 1);
    for (int i = threadIdx.x; i < d; i += blockDim.x)
        x[(long long)b * d + i] = __bfloat162float(embed[(long long)tok * d + i]) + pos_emb[(long long)p * d + i];
}

// forced prompt token for step p of the decoder prefix
__global__ void wh_set_tokens_kernel(const int* __restrict__ prompt, int p, int* tokens, int* pos, int B) {
    const int b = threadIdx.x;
    if (b < B) { tokens[b] = prompt[p]; pos[b] = p; }
}

// suppress masks + greedy pick + bookkeeping (WhisperModel.swift:228-244,284-309); one CTA per row
struct PickArgs {
    float* logits;           // [B, V] (masks are ADDED in place, -1e9 like the reference)
    int* tokens; int* pos; int* out_tokens; int* n_gen; int* done; int* n_active;
    const int* begin_suppress; int n_begin;
    const int* suppress; int n_suppress;
    int V, max_tokens, timestamp_begin, eot, mask_eot;
    float temperature;           // > 0: categorical(logits / T) (WhisperModel.swift:289-290, Gumbel-max draw), else argmax
    unsigned long long seed;
};
__device__ __forceinline__ float wh_uniform01(unsigned long long seed, unsigned long long a, unsigned long long b) {
    unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (a * 1000003ull + b + 1ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    return (float)(z >> 40) * (1.0f / 16777216.0f);
}
__global__ void __launch_bounds__(1024)
wh_pick_kernel(PickArgs a) {
    __shared__ float s_val[32];
    __shared__ int s_idx[32];
    pdl_trigger();
    pdl_wait();
    const int b = blockIdx.x, t = threadIdx.x;
    float* lg = a.logits + (long long)b * a.V;
    const bool first = a.n_gen[b] == 0;
    if (first) for (int i = t; i < a.n_begin; i += 1024) { const int id = a.begin_suppress[i]; if (id >= 0 && id < a.V) lg[id] += -1e9f; }
    __syncthreads();
    for (int i = t; i < a.n_suppress; i += 1024) { const int id = a.suppress[i]; if (id >= 0 && id < a.V) lg[id] += -1e9f; }
    __syncthreads();
    if (a.mask_eot && t == 0 && a.eot < a.V) lg[a.eot] = -INFINITY;
    __syncthreads();
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = t; i < a.V; i += 1024) {
        float v = lg[i];
        if (i >= a.timestamp_begin) v += -1e9f;          // suppressFromIndex: timestamps are never emitted
        if (v > best) { best = v; bi = i; }
    }
    for (int o = 16; o; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if ((t & 31) == 0) { s_val[t >> 5] = best; s_idx[t >> 5] = bi; }
    __syncthreads();
    __shared__ int s_pick;
    if (t == 0) {
        for (int i = 1; i < 32; ++i)
            if (s_val[i] > best || (s_val[i] == best && s_idx[i] < bi)) { best = s_val[i]; bi = s_idx[i]; }
        s_pick = bi;
    }
    __syncthreads();
    if (a.temperature > 0.f) {
        // categorical(logits / T) by the Gumbel-max trick: argmax_i (l_i / T - log(-log u_i)), u_i a hash of (seed, clip, step, i).
        // Deterministic for a given seed and robust to last-bit differences in the logits (an inverse-CDF walk over 51 865 nearly
        // flat probabilities is not: the stream-K residual GEMMs reorder fp32 sums from run to run).  The distribution is the
        // reference's, the stream of draws is not (MLX draws its own Gumbel noise).
        const float inv_t = 1.0f / a.temperature;
        const unsigned long long base = a.seed + 0x9E3779B97F4A7C15ull * ((unsigned long long)b * 1000003ull + (unsigned long long)a.n_gen[b] + 1ull);
        float gv = -INFINITY;
        int gi = 0x7fffffff;
        for (int i = t; i < a.V; i += 1024) {
            float v = lg[i];
            if (i >= a.timestamp_begin) v += -1e9f;
            unsigned long long z = base ^ ((unsigned long long)(unsigned)i * 0xD6E8FEB86659FD93ull);
            z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
            z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
            z ^= z >> 31;
            const float u = ((float)(z >> 40) + 0.5f) * (1.0f / 16777216.0f);
            const float k = v * inv_t - __logf(-__logf(u));
            if (k > gv) { gv = k; gi = i; }
        }
        for (int o = 16; o; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, gv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, gi, o);
            if (ov > gv || (ov == gv && oi < gi)) { gv = ov; gi = oi; }
        }
        __syncthreads();
        if ((t & 31) == 0) { s_val[t >> 5] = gv; s_idx[t >> 5] = gi; }
        __syncthreads();
        if (t == 0) {
            for (int i = 1; i < 32; ++i)
                if (s_val[i] > gv || (s_val[i] == gv && s_idx[i] < gi)) { gv = s_val[i]; gi = s_idx[i]; }
            if (gi >= 0 && gi < a.V) s_pick = gi;
        }
        __syncthreads();
    }
    if (t == 0) {
        bi = s_pick;
        a.tokens[b] = bi;
        a.pos[b] += 1;
        if (!a.done[b]) {
            if (bi == a.eot) { a.done[b] = 1; atomicSub(a.n_active, 1); }     // :237 break, token not appended
            else {
                const int n = a.n_gen[b];
                if (n < a.max_tokens) a.out_tokens[b * a.max_tokens + n] = bi;
                a.n_gen[b] = n + 1;
                if (n + 1 >= a.max_tokens) { a.done[b] = 1; atomicSub(a.n_active, 1); }
            }
        }
    }
}

__global__ void wh_init_rows_kernel(int B, int* n_gen, int* done, int* n_active) {
    const int b = threadIdx.x;
    if (b == 0) *n_active = B;
    if (b < B) { n_gen[b] = 0; done[b] = 0; }
}

__global__ void random_bf16_kernel(bf16* __restrict__ w, long long n, float std, unsigned long long seed) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (unsigned long long)(i + 1);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        z ^= z >> 31;
        const float u1 = ((unsigned)(z >> 40) + 1.0f) * (1.0f / 16777217.0f);
        const float u2 = (unsigned)((z >> 8) & 0xFFFFFF) * (1.0f / 16777216.0f);
        w[i] = __float2bfloat16_rn(std * sqrtf(-2.0f * __logf(u1)) * cospif(2.0f * u2));
    }
}

// one Linear: bf16 weight [M, K] + fp32 bias + its TMA map
struct Lin {
    DBuf<bf16> w;
    DBuf<float> b;
    CUtensorMap tm{};
    CUtensorMap tm_step{};    // decode-step GEMMs that own whole m-tiles: boxes of step_rows weight rows (tc::Args::tile_rows)
    int step_rows = 0;        // 0: tm / 128-row tiles
    int M = 0, K = 0;
    bool has_bias = false;
};
struct LNp { DBuf<float> w, b; };
struct EncLayer { Lin qkv, o, fc1, fc2; LNp ln1, ln2; };
struct DecLayer { Lin qkv, o, cq, ckv, co, fc1, fc2; LNp ln1, ln2, ln3; };

}  // namespace wh
}  // namespace b2a

using namespace b2a;
using namespace b2a::wh;

struct b2a_stt {
    int device;
    b2a_whisper_config cfg;
    cudaStream_t stream = nullptr;
    int num_sms = 132;
    b2a_logmel* mel = nullptr;
    // weights
    Lin conv1, conv2;
    DBuf<float> enc_pos, dec_pos;
    DBuf<bf16> embed;
    CUtensorMap tm_embed{};
    std::vector<EncLayer> enc;
    std::vector<DecLayer> dec;
    LNp enc_ln, dec_ln;
    // encoder workspace (sized per batch)
    int enc_cap_B = 0;
    DBuf<float> pcm, feats, h1, xe, qkve, kvbuf;
    DBuf<bf16> X1, X2, xne, attne, acte, enc_out;
    DBuf<__half> fa_q, fa_k, fa_vt;                  // attn_tc.cuh operands: [B*nh][Tp][64] x2, [B*nh][64][Tp]
    CUtensorMap tm_faq{}, tm_fak{}, tm_fav{};
    static constexpr int FA_TP = 1536;               // 1500 keys padded to whole 128-key tiles
    CUtensorMap tmx_X1{}, tmx_X2{}, tmx_xne{}, tmx_attne{}, tmx_acte{}, tmx_encout{};
    // caches
    DBuf<float> self_k, self_v;
    DBuf<__half> cross_k, cross_v;      // fp16 (kv_relayout_kernel)
    // decoder step state
    DBuf<float> x, qkv, cq, logits, part_o, part_ml;
    DBuf<bf16> xn, attn, act;
    CUtensorMap tmx_xn{}, tmx_attn{}, tmx_act{};
    DBuf<int> tokens, pos, out_tokens, n_gen, done, n_active, counters, prompt, d_begin, d_suppress;
    DBuf<float> sk_ws;       // stream-K partial tiles of the decoder's residual GEMMs, see tc::Args::part_ws
    DBuf<unsigned> sk_cnt;
    int sk_slots = 0;
    HBuf<int> h_flag;
    int da_splits_self = 1, da_splits_cross = 1;
    cudaGraphExec_t g_full = nullptr, g_layers = nullptr;
    PickArgs g_pick{};
    int g_B = 0;
    std::atomic<int> cancel{0};
    int bench_mask_eot = 0;      // b2a_stt_set_bench_flags (include/b200audio_internal.h): never stop on EOT (fixed work)

    ~b2a_stt() {
        if (g_full) cudaGraphExecDestroy(g_full);
        if (g_layers) cudaGraphExecDestroy(g_layers);
        if (mel) b2a_logmel_destroy(mel);
        if (stream) cudaStreamDestroy(stream);
    }

    int d() const { return cfg.d_model; }

    void make_lin(Lin& L, int M, int K) {
        L.M = M; L.K = K;
        L.w.alloc((size_t)M * K);
        L.b.alloc(M);
        B2A_CUDA(cudaMemset(L.b.p, 0, M * sizeof(float)));
        L.tm = tc::make_tmap_bf16(L.w.p, M, K, tc::BM);
    }
    // A decode-step GEMM that cannot split K (bias / GELU epilogue) runs on M / 128 CTAs -- 12, 4 and 16 for q|k|v, the cross query and
    // fc1 of Whisper-base.  Tiles of fewer weight rows (a multiple of 8) spread the same rows over up to one CTA per SM.
    void make_step_map(Lin& L) {
        if (cdiv(L.M, tc::BM) * 4 >= num_sms * 3) return;
        L.step_rows = std::max(8, std::min(tc::BM, cdiv(cdiv(L.M, num_sms), 8) * 8));
        L.tm_step = tc::make_tmap_bf16(L.w.p, L.M, L.K, L.step_rows);
    }

    void check_config() {
        const b2a_whisper_config& c = cfg;
        B2A_CHECK(c.d_model % 64 == 0 && c.d_model <= LN_THREADS * LN_MAXV, B2A_ERR_INVALID_INPUT, "whisper: d_model must be a multiple of 64 (<= 2048)");
        B2A_CHECK(c.d_model / c.encoder_attention_heads == HD && c.d_model / c.decoder_attention_heads == HD,
                  B2A_ERR_INVALID_INPUT, "whisper: attention heads must be 64-dimensional");
        B2A_CHECK(c.encoder_ffn_dim % 64 == 0 && c.decoder_ffn_dim % 64 == 0, B2A_ERR_INVALID_INPUT, "whisper: ffn dims must be multiples of 64");
        B2A_CHECK(c.num_mel_bins * 3 <= 512, B2A_ERR_INVALID_INPUT, "whisper: too many mel bins");
        B2A_CHECK(c.max_source_positions == 1500, B2A_ERR_INVALID_INPUT, "whisper: max_source_positions must be 1500 (30 s windows)");
        B2A_CHECK(c.max_batch >= 1 && c.max_batch <= DEC_HALF, B2A_ERR_INVALID_INPUT, "whisper: max_batch must be in 1..16");
        require_device(device);
        B2A_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        B2A_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
        tc::set_attributes();
    }

    int k1p() const { return cdiv(3 * cfg.num_mel_bins, 64) * 64; }

    void alloc_weights() {
        const b2a_whisper_config& c = cfg;
        const int D = d();
        make_lin(conv1, D, k1p());
        make_lin(conv2, D, 3 * D);
        enc_pos.alloc((size_t)c.max_source_positions * D);
        dec_pos.alloc((size_t)c.max_target_positions * D);
        embed.alloc((size_t)c.vocab_size * D);
        tm_embed = tc::make_tmap_bf16(embed.p, c.vocab_size, D, tc::BM);
        auto mk_ln = [&](LNp& l) { l.w.alloc(D); l.b.alloc(D); };
        enc.resize(c.encoder_layers);
        for (auto& L : enc) {
            make_lin(L.qkv, 3 * D, D); make_lin(L.o, D, D); make_lin(L.fc1, c.encoder_ffn_dim, D); make_lin(L.fc2, D, c.encoder_ffn_dim);
            mk_ln(L.ln1); mk_ln(L.ln2);
        }
        dec.resize(c.decoder_layers);
        for (auto& L : dec) {
            make_lin(L.qkv, 3 * D, D); make_lin(L.o, D, D); make_lin(L.cq, D, D); make_lin(L.ckv, 2 * D, D); make_lin(L.co, D, D);
            make_lin(L.fc1, c.decoder_ffn_dim, D); make_lin(L.fc2, D, c.decoder_ffn_dim);
            make_step_map(L.qkv); make_step_map(L.cq); make_step_map(L.fc1);
            mk_ln(L.ln1); mk_ln(L.ln2); mk_ln(L.ln3);
        }
        mk_ln(enc_ln); mk_ln(dec_ln);
    }

    void alloc_state() {
        const b2a_whisper_config& c = cfg;
        const int D = d(), nh = c.decoder_attention_heads, B = c.max_batch, R = 2 * DEC_HALF;
        const size_t sk = (size_t)c.decoder_layers * B * nh * c.max_target_positions * HD;
        const size_t ck = (size_t)c.decoder_layers * B * nh * c.max_source_positions * HD;
        self_k.alloc(sk); self_v.alloc(sk); cross_k.alloc(ck); cross_v.alloc(ck);
        B2A_CUDA(cudaMemset(self_k.p, 0, sk * sizeof(float)));
        B2A_CUDA(cudaMemset(self_v.p, 0, sk * sizeof(float)));
        x.alloc((size_t)DEC_HALF * D); qkv.alloc((size_t)DEC_HALF * 3 * D); cq.alloc((size_t)DEC_HALF * D);
        logits.alloc((size_t)DEC_HALF * c.vocab_size);
        xn.alloc((size_t)R * D); attn.alloc((size_t)R * D); act.alloc((size_t)R * c.decoder_ffn_dim);
        B2A_CUDA(cudaMemset(xn.p, 0, (size_t)R * D * sizeof(bf16)));
        B2A_CUDA(cudaMemset(attn.p, 0, (size_t)R * D * sizeof(bf16)));
        B2A_CUDA(cudaMemset(act.p, 0, (size_t)R * c.decoder_ffn_dim * sizeof(bf16)));
        B2A_CUDA(cudaMemset(x.p, 0, (size_t)DEC_HALF * D * sizeof(float)));
        tmx_xn = tc::make_tmap_bf16(xn.p, R, D, 32);
        tmx_attn = tc::make_tmap_bf16(attn.p, R, D, 32);
        tmx_act = tc::make_tmap_bf16(act.p, R, c.decoder_ffn_dim, 32);
        da_splits_self = cdiv(c.max_target_positions, DA_CAP);
        da_splits_cross = cdiv(c.max_source_positions, DA_CAP_CROSS);
        const int S = std::max(da_splits_self, da_splits_cross);
        part_o.alloc((size_t)B * nh * S * HD); part_ml.alloc((size_t)B * nh * S * 2);
        counters.alloc((size_t)B * nh);
        B2A_CUDA(cudaMemset(counters.p, 0, (size_t)B * nh * sizeof(int)));
        {   // stream-K workspace for the residual GEMMs (out-proj, cross out-proj: K = d_model; fc2: K = ffn), M = d_model, BN = 32
            const int mt = cdiv(D, tc::BM);
            for (const int K : {D, c.decoder_ffn_dim}) {
                const int kb = K / tc::BK;
                if (kb > 0) sk_slots = std::max(sk_slots, tc::stream_k_slots(mt, kb, (int)std::min<long long>(num_sms, std::max<long long>(1, (long long)mt * kb / 4))));
            }
            sk_ws.alloc((size_t)mt * std::max(1, sk_slots) * 32 * tc::BM);
            sk_cnt.alloc((size_t)mt);
            B2A_CUDA(cudaMemset(sk_cnt.p, 0, (size_t)mt * sizeof(unsigned)));
        }
        tokens.alloc(DEC_HALF); pos.alloc(DEC_HALF); n_gen.alloc(DEC_HALF); done.alloc(DEC_HALF); n_active.alloc(1);
        B2A_CUDA(cudaMemset(tokens.p, 0, DEC_HALF * sizeof(int)));
        B2A_CUDA(cudaMemset(pos.p, 0xff, DEC_HALF * sizeof(int)));   // -1: row inactive
        h_flag.alloc(16);
        const int32_t st = b2a_logmel_create(device, 1, 16000, 400, 160, c.num_mel_bins, &mel);
        B2A_CHECK(st == B2A_OK, st, std::string("whisper: log-mel front-end: ") + b2a_last_error());
        B2A_CUDA(cudaDeviceSynchronize());
    }

    // ---- weights from a tensor table (HF names / layouts) -------------------------------------------------
    static std::vector<bf16> to_bf16(const b2a_tensor& t, int64_t expect, const std::string& name) {
        B2A_CHECK(TensorTable::numel(t) == expect, B2A_ERR_MODEL_NOT_INITIALIZED, "bad shape for tensor: " + name);
        std::vector<bf16> v(expect);
        if (t.dtype == B2A_DTYPE_BF16) memcpy(v.data(), t.data, expect * sizeof(bf16));
        else if (t.dtype == B2A_DTYPE_F32) for (int64_t i = 0; i < expect; ++i) v[i] = __float2bfloat16_rn(((const float*)t.data)[i]);
        else throw Error(B2A_ERR_MODEL_NOT_INITIALIZED, "bad dtype for tensor: " + name);
        return v;
    }
    void load_lin_rows(Lin& L, const TensorTable& tt, const std::string& name, int row0, int rows, bool bias) {
        std::vector<bf16> w = to_bf16(tt.get(name + ".weight"), (int64_t)rows * L.K, name + ".weight");
        B2A_CUDA(cudaMemcpy(L.w.p + (size_t)row0 * L.K, w.data(), w.size() * sizeof(bf16), cudaMemcpyHostToDevice));
        if (bias) {
            std::vector<float> b = tt.f32(name + ".bias", rows);
            B2A_CUDA(cudaMemcpy(L.b.p + row0, b.data(), rows * sizeof(float), cudaMemcpyHostToDevice));
            L.has_bias = true;
        }
    }
    void load_ln(LNp& l, const TensorTable& tt, const std::string& name) {
        std::vector<float> w = tt.f32(name + ".weight", d()), b = tt.f32(name + ".bias", d());
        l.w.upload(w.data(), d()); l.b.upload(b.data(), d());
    }
    void load_conv(Lin& L, const TensorTable& tt, const std::string& name, int cin) {
        // HF / PyTorch layout [out, in, k] -> GEMM weight [out, k*in + i] (zero padded to L.K)   (WhisperModel.swift:335-365)
        const b2a_tensor& t = tt.get(name + ".weight");
        std::vector<bf16> src = to_bf16(t, (int64_t)L.M * cin * 3, name + ".weight");
        std::vector<bf16> w((size_t)L.M * L.K, __float2bfloat16_rn(0.f));
        for (int o = 0; o < L.M; ++o)
            for (int i = 0; i < cin; ++i)
                for (int k = 0; k < 3; ++k) w[(size_t)o * L.K + k * cin + i] = src[((size_t)o * cin + i) * 3 + k];
        B2A_CUDA(cudaMemcpy(L.w.p, w.data(), w.size() * sizeof(bf16), cudaMemcpyHostToDevice));
        std::vector<float> b = tt.f32(name + ".bias", L.M);
        B2A_CUDA(cudaMemcpy(L.b.p, b.data(), L.M * sizeof(float), cudaMemcpyHostToDevice));
        L.has_bias = true;
    }
    void load_attn(Lin& qkvL, Lin& oL, const TensorTable& tt, const std::string& p) {
        const int D = d();
        load_lin_rows(qkvL, tt, p + "q_proj", 0, D, true);
        load_lin_rows(qkvL, tt, p + "k_proj", D, D, false);          // k_proj has no bias (WhisperLayers.swift:29)
        load_lin_rows(qkvL, tt, p + "v_proj", 2 * D, D, true);
        qkvL.has_bias = true;
        load_lin_rows(oL, tt, p + "out_proj", 0, D, true);
    }

    b2a_stt(int dev, const b2a_whisper_config& c, const TensorTable& tt) : device(dev), cfg(c) {
        check_config();
        alloc_weights();
        const int D = d();
        load_conv(conv1, tt, "model.encoder.conv1", c.num_mel_bins);
        load_conv(conv2, tt, "model.encoder.conv2", D);
        std::vector<float> ep = tt.f32("model.encoder.embed_positions.weight", (int64_t)c.max_source_positions * D);
        enc_pos.upload(ep.data(), ep.size());
        std::vector<float> dp = tt.f32("model.decoder.embed_positions.weight", (int64_t)c.max_target_positions * D);
        dec_pos.upload(dp.data(), dp.size());
        std::vector<bf16> em = to_bf16(tt.get("model.decoder.embed_tokens.weight"), (int64_t)c.vocab_size * D, "embed_tokens");
        B2A_CUDA(cudaMemcpy(embed.p, em.data(), em.size() * sizeof(bf16), cudaMemcpyHostToDevice));
        for (int l = 0; l < c.encoder_layers; ++l) {
            const std::string p = "model.encoder.layers." + std::to_string(l) + ".";
            EncLayer& L = enc[l];
            load_attn(L.qkv, L.o, tt, p + "self_attn.");
            load_lin_rows(L.fc1, tt, p + "fc1", 0, c.encoder_ffn_dim, true);
            load_lin_rows(L.fc2, tt, p + "fc2", 0, D, true);
            load_ln(L.ln1, tt, p + "self_attn_layer_norm"); load_ln(L.ln2, tt, p + "final_layer_norm");
        }
        load_ln(enc_ln, tt, "model.encoder.layer_norm");
        for (int l = 0; l < c.decoder_layers; ++l) {
            const std::string p = "model.decoder.layers." + std::to_string(l) + ".";
            DecLayer& L = dec[l];
            load_attn(L.qkv, L.o, tt, p + "self_attn.");
            load_lin_rows(L.cq, tt, p + "encoder_attn.q_proj", 0, D, true);
            load_lin_rows(L.ckv, tt, p + "encoder_attn.k_proj", 0, D, false);
            load_lin_rows(L.ckv, tt, p + "encoder_attn.v_proj", D, D, true);
            L.ckv.has_bias = true;
            load_lin_rows(L.co, tt, p + "encoder_attn.out_proj", 0, D, true);
            load_lin_rows(L.fc1, tt, p + "fc1", 0, c.decoder_ffn_dim, true);
            load_lin_rows(L.fc2, tt, p + "fc2", 0, D, true);
            load_ln(L.ln1, tt, p + "self_attn_layer_norm"); load_ln(L.ln2, tt, p + "encoder_attn_layer_norm");
            load_ln(L.ln3, tt, p + "final_layer_norm");
        }
        load_ln(dec_ln, tt, "model.decoder.layer_norm");
        alloc_state();
    }

    // random init on the device (benchmarks): matrices N(0, std^2), biases 0, LayerNorm (1, 0), sinusoid-free positions 0.02 N
    b2a_stt(int dev, const b2a_whisper_config& c, float std, unsigned long long seed) : device(dev), cfg(c) {
        check_config();
        alloc_weights();
        unsigned long long sd = seed * 7919ull + 3;
        auto rnd = [&](bf16* p, size_t n, float s) { random_bf16_kernel<<<132 * 4, 256, 0, stream>>>(p, (long long)n, s, sd++); count_launch(); };
        auto fill = [&](DBuf<float>& b, int n, float v) { std::vector<float> h(n, v); b.upload(h.data(), n, stream); B2A_CUDA(cudaStreamSynchronize(stream)); };
        auto lin = [&](Lin& L) { rnd(L.w.p, (size_t)L.M * L.K, std); L.has_bias = true; };
        lin(conv1); lin(conv2);
        rnd(embed.p, (size_t)c.vocab_size * d(), std);
        {   // positions: small deterministic values
            std::vector<float> ep((size_t)c.max_source_positions * d()), dp((size_t)c.max_target_positions * d());
            for (size_t i = 0; i < ep.size(); ++i) ep[i] = 0.02f * sinf(0.37f * (float)(i % 9973));
            for (size_t i = 0; i < dp.size(); ++i) dp[i] = 0.02f * cosf(0.11f * (float)(i % 7919));
            enc_pos.upload(ep.data(), ep.size(), stream); dec_pos.upload(dp.data(), dp.size(), stream);
            B2A_CUDA(cudaStreamSynchronize(stream));
        }
        for (auto& L : enc) { lin(L.qkv); lin(L.o); lin(L.fc1); lin(L.fc2); fill(L.ln1.w, d(), 1.f); fill(L.ln1.b, d(), 0.f); fill(L.ln2.w, d(), 1.f); fill(L.ln2.b, d(), 0.f); }
        for (auto& L : dec) {
            lin(L.qkv); lin(L.o); lin(L.cq); lin(L.ckv); lin(L.co); lin(L.fc1); lin(L.fc2);
            fill(L.ln1.w, d(), 1.f); fill(L.ln1.b, d(), 0.f); fill(L.ln2.w, d(), 1.f); fill(L.ln2.b, d(), 0.f); fill(L.ln3.w, d(), 1.f); fill(L.ln3.b, d(), 0.f);
        }
        fill(enc_ln.w, d(), 1.f); fill(enc_ln.b, d(), 0.f); fill(dec_ln.w, d(), 1.f); fill(dec_ln.b, d(), 0.f);
        B2A_CUDA(cudaStreamSynchronize(stream));
        alloc_state();
    }

    // ---- GEMM wrappers ---------------------------------------------------------------------------------------
    // big side: T tokens in 64-token hi/lo tiles (BN = 128), whole tiles per CTA
    void gemm_big(const Lin& L, const CUtensorMap& tmX, int epi, int act, float* of32, bf16* obf16, long long T, cudaStream_t s) {
        tc::Args a{};
        a.out_f32 = of32; a.out_bf16 = obf16; a.M = L.M; a.N = (int)T; a.K = L.K; a.ldo = L.M;
        a.m_tiles = cdiv(L.M, tc::BM); a.k_blocks = L.K / tc::BK; a.stages = tc::Smem<128>::max_stages(); a.hilo = 1;
        a.epi_full = epi; a.epi_partial = -1; a.bias = L.has_bias ? L.b.p : nullptr; a.act = act;
        a.lo_rows = epi == tc::EPI_STORE_BF16 ? ENC_HALF : 0;
        const int n_tiles = cdiv(T, ENC_HALF);
        const int ctas = std::max(1, std::min(a.m_tiles, num_sms / std::max(1, n_tiles)));
        tc::launch<128>(L.tm, tmX, a, ctas, n_tiles, s);
    }
    // decoder step: B <= 16 rows as hi/lo in one 32-column tile, whole tiles per CTA
    void gemm_step(const CUtensorMap& tmW, int M, int K, const float* bias, const CUtensorMap& tmX, int epi, int act,
                   float* of32, bf16* obf16, int B, cudaStream_t s, int tile_rows = 0) {
        tc::Args a{};
        a.out_f32 = of32; a.out_bf16 = obf16; a.M = M; a.N = B; a.K = K; a.ldo = M;
        a.tile_rows = tile_rows;
        a.m_tiles = cdiv(M, tile_rows > 0 ? tile_rows : tc::BM); a.k_blocks = K / tc::BK; a.stages = 8; a.hilo = 1;
        a.epi_full = epi; a.epi_partial = -1; a.bias = bias; a.act = act;
        a.lo_rows = epi == tc::EPI_STORE_BF16 ? DEC_HALF : 0;
        int ctas = std::min(num_sms, a.m_tiles);
        if (epi == tc::EPI_ADD && act == tc::ACT_NONE) {
            // out-proj / cross out-proj / fc2 add into the residual stream: their (m_tile, k_block) units can be dealt to many CTAs
            // (stream-K), a tile's partials summed in slot order and added into x.  M = 512 gives only 4 whole-tile CTAs otherwise,
            // each streaming its K range alone.
            // At least 4 k-blocks per CTA keeps a tile to at most k_blocks / 4 + 1 partials for the reducing CTA to add (out-proj:
            // 8 CTAs, fc2: 32).  This bound was chosen for the reduction's cost, not measured against larger CTA counts.
            a.epi_partial = tc::EPI_PARTIAL;
            ctas = (int)std::min<long long>(num_sms, std::max<long long>(1, (long long)a.m_tiles * a.k_blocks / 4));
            a.part_ws = sk_ws.p; a.part_cnt = sk_cnt.p; a.part_slots = sk_slots;
        }
        tc::launch<32>(tmW, tmX, a, ctas, 1, s);
    }
    void gemm_step(const Lin& L, const CUtensorMap& tmX, int epi, int act, float* of32, bf16* obf16, int B, cudaStream_t s) {
        const bool whole = !(epi == tc::EPI_ADD && act == tc::ACT_NONE);
        if (whole && L.step_rows > 0) gemm_step(L.tm_step, L.M, L.K, L.has_bias ? L.b.p : nullptr, tmX, epi, act, of32, obf16, B, s, L.step_rows);
        else gemm_step(L.tm, L.M, L.K, L.has_bias ? L.b.p : nullptr, tmX, epi, act, of32, obf16, B, s);
    }
    void ln(const LNp& l, float* xrows, bf16* out, long long rows, int half, const float* addend, int add_mod, cudaStream_t s) {
        if (rows >= 1024 && d() % 128 == 0 && d() <= 128 * LNW_MAXV) {
            launch_pdl(layernorm_hilo_rows_kernel, dim3((unsigned)cdiv(rows, (long long)LNW_ROWS)), dim3(LNW_ROWS * 32), 0, s, xrows, (const float*)l.w.p,
                       (const float*)l.b.p, out, rows, d(), half, addend, add_mod);
            return;
        }
        launch_pdl(layernorm_hilo_kernel, dim3((unsigned)rows), dim3(LN_THREADS), 0, s, xrows, (const float*)l.w.p, (const float*)l.b.p, out, d(),
                   half, addend, add_mod);
    }

    // ---- encoder ---------------------------------------------------------------------------------------------
    void ensure_encoder_workspace(int B) {
        if (B <= enc_cap_B) return;
        const b2a_whisper_config& c = cfg;
        const int D = d();
        const long long T1 = (long long)B * 3000, T2 = (long long)B * 1500;
        const long long T1p = cdiv(T1, ENC_HALF) * (long long)ENC_HALF, T2p = cdiv(T2, ENC_HALF) * (long long)ENC_HALF;
        pcm.alloc((size_t)B * 480000); feats.alloc((size_t)T1 * c.num_mel_bins);
        h1.alloc((size_t)T1 * D); xe.alloc((size_t)T2 * D); qkve.alloc((size_t)T2 * 3 * D); kvbuf.alloc((size_t)T2 * 2 * D);
        X1.alloc((size_t)2 * T1p * k1p()); X2.alloc((size_t)2 * T2p * 3 * D);
        xne.alloc((size_t)2 * T2p * D); attne.alloc((size_t)2 * T2p * D); acte.alloc((size_t)2 * T2p * c.encoder_ffn_dim);
        enc_out.alloc((size_t)2 * T2p * D);
        B2A_CUDA(cudaMemset(X1.p, 0, (size_t)2 * T1p * k1p() * sizeof(bf16)));
        B2A_CUDA(cudaMemset(X2.p, 0, (size_t)2 * T2p * 3 * D * sizeof(bf16)));
        B2A_CUDA(cudaMemset(xne.p, 0, (size_t)2 * T2p * D * sizeof(bf16)));
        B2A_CUDA(cudaMemset(attne.p, 0, (size_t)2 * T2p * D * sizeof(bf16)));
        B2A_CUDA(cudaMemset(acte.p, 0, (size_t)2 * T2p * c.encoder_ffn_dim * sizeof(bf16)));
        B2A_CUDA(cudaMemset(enc_out.p, 0, (size_t)2 * T2p * D * sizeof(bf16)));
        tmx_X1 = tc::make_tmap_bf16(X1.p, 2 * T1p, k1p(), 128);
        tmx_X2 = tc::make_tmap_bf16(X2.p, 2 * T2p, 3 * D, 128);
        tmx_xne = tc::make_tmap_bf16(xne.p, 2 * T2p, D, 128);
        tmx_attne = tc::make_tmap_bf16(attne.p, 2 * T2p, D, 128);
        tmx_acte = tc::make_tmap_bf16(acte.p, 2 * T2p, c.encoder_ffn_dim, 128);
        tmx_encout = tc::make_tmap_bf16(enc_out.p, 2 * T2p, D, 128);
        {
            const int nh = c.encoder_attention_heads;
            const size_t n = (size_t)B * nh * FA_TP * HD;
            fa_q.alloc(n); fa_k.alloc(n); fa_vt.alloc(n);
            tm_faq = tc::make_tmap_f16_3d(fa_q.p, HD, FA_TP, (long long)B * nh, 64, fa::BQ);
            tm_fak = tc::make_tmap_f16_3d(fa_k.p, HD, FA_TP, (long long)B * nh, 64, fa::BKV);
            tm_fav = tc::make_tmap_f16_3d(fa_vt.p, FA_TP, HD, (long long)B * nh, 64, 64);
            B2A_CUDA(cudaFuncSetAttribute(fa::mha_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fa::FA_SMEM_BYTES));
            B2A_CUDA(cudaFuncSetAttribute(fa::mha_tc_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));   // two CTAs per SM
        }
        enc_cap_B = B;
    }

    // d_pcm [B, n] fp32 on the device -> encoder hidden states as hi/lo tiles in enc_out, cross K/V caches filled
    void encode_dev(const float* d_pcm, int B, long long n, cudaStream_t s) {
        const b2a_whisper_config& c = cfg;
        const int D = d(), nh = c.encoder_attention_heads;
        const long long T1 = (long long)B * 3000, T2 = (long long)B * 1500;
        ensure_encoder_workspace(B);
        int32_t st = b2a_logmel_compute_dev(mel, d_pcm, B, n, feats.p, (void*)s);
        B2A_CHECK(st == B2A_OK, st, std::string("whisper: log-mel: ") + b2a_last_error());
        im2col3_kernel<<<(unsigned)T1, 128, 0, s>>>(feats.p, X1.p, 3000, 3000, c.num_mel_bins, k1p(), 1);
        count_launch();
        gemm_big(conv1, tmx_X1, tc::EPI_STORE, tc::ACT_GELU, h1.p, nullptr, T1, s);
        im2col3_kernel<<<(unsigned)T2, 256, 0, s>>>(h1.p, X2.p, 3000, 1500, D, 3 * D, 2);
        count_launch();
        gemm_big(conv2, tmx_X2, tc::EPI_STORE, tc::ACT_GELU, xe.p, nullptr, T2, s);
        for (int l = 0; l < c.encoder_layers; ++l) {
            EncLayer& L = enc[l];
            ln(L.ln1, xe.p, xne.p, T2, ENC_HALF, l == 0 ? enc_pos.p : nullptr, 1500, s);     // + positions (:150)
            gemm_big(L.qkv, tmx_xne, tc::EPI_STORE, tc::ACT_NONE, qkve.p, nullptr, T2, s);
            // wgmma attention (attn_tc.cuh): pack q | k | v as fp16 operands, then one CTA per (128-query tile, head, clip)
            fa::pack_qkv_f16_kernel<<<dim3(FA_TP / 64, B, nh), 256, 0, s>>>(qkve.p, fa_q.p, fa_k.p, fa_vt.p, 1500, FA_TP, nh, 1.0f / sqrtf((float)HD));
            fa::Args fa_args{attne.p, 1500, FA_TP, nh, D, ENC_HALF};
            fa::mha_tc_kernel<<<dim3(FA_TP / fa::BQ, nh, B), fa::FA_THREADS, fa::FA_SMEM_BYTES, s>>>(tm_faq, tm_fak, tm_fav, fa_args);
            count_launch(2);
            gemm_big(L.o, tmx_attne, tc::EPI_ADD, tc::ACT_NONE, xe.p, nullptr, T2, s);
            ln(L.ln2, xe.p, xne.p, T2, ENC_HALF, nullptr, 1, s);
            gemm_big(L.fc1, tmx_xne, tc::EPI_STORE_BF16, tc::ACT_GELU, nullptr, acte.p, T2, s);
            gemm_big(L.fc2, tmx_acte, tc::EPI_ADD, tc::ACT_NONE, xe.p, nullptr, T2, s);
        }
        ln(enc_ln, xe.p, enc_out.p, T2, ENC_HALF, nullptr, 1, s);
        // cross-attention K/V of every decoder layer, once per clip (WhisperLayers.swift:217-234)
        const int dnh = c.decoder_attention_heads;
        const size_t ck_layer = (size_t)c.max_batch * dnh * c.max_source_positions * HD;
        for (int l = 0; l < c.decoder_layers; ++l) {
            gemm_big(dec[l].ckv, tmx_encout, tc::EPI_STORE, tc::ACT_NONE, kvbuf.p, nullptr, T2, s);
            kv_relayout_kernel<<<(unsigned)T2, 256, 0, s>>>(kvbuf.p, cross_k.p + l * ck_layer, cross_v.p + l * ck_layer, 1500, D, dnh);
            count_launch();
        }
        B2A_CUDA(cudaGetLastError());
    }

    // ---- decoder step ----------------------------------------------------------------------------------------
    void dec_attn(bool append, const float* q, int ldq, int q_off, const float* kvn, int k_off, int v_off, void* kc, void* vc,
                  int max_t, int n_keys, int S, int B, cudaStream_t s) {
        DecAttnArgs a{q, kvn, pos.p, kc, vc, attn.p, part_o.p, part_ml.p, counters.p, ldq, q_off, k_off, v_off,
                      cfg.decoder_attention_heads, max_t, n_keys, S, d(), 1.0f / sqrtf((float)HD)};
        const dim3 grid(cfg.decoder_attention_heads, B, S);
        if (append) launch_pdl(mha_decode_kernel<true>, grid, dim3(2 * DA_CAP), 0, s, a);
        else launch_pdl(mha_decode_kernel<false>, grid, dim3(2 * DA_CAP_CROSS), 0, s, a);
    }

    void run_layers(int B, cudaStream_t s) {
        const b2a_whisper_config& c = cfg;
        const int D = d(), nh = c.decoder_attention_heads;
        launch_pdl(wh_embed_kernel, dim3(B), dim3(256), 0, s, (const int*)tokens.p, (const int*)pos.p, (const bf16*)embed.p,
                   (const float*)dec_pos.p, x.p, D, c.vocab_size, c.max_target_positions);
        const size_t sk_layer = (size_t)c.max_batch * nh * c.max_target_positions * HD;
        const size_t ck_layer = (size_t)c.max_batch * nh * c.max_source_positions * HD;
        for (int l = 0; l < c.decoder_layers; ++l) {
            DecLayer& L = dec[l];
            ln(L.ln1, x.p, xn.p, B, DEC_HALF, nullptr, 1, s);
            gemm_step(L.qkv, tmx_xn, tc::EPI_STORE, tc::ACT_NONE, qkv.p, nullptr, B, s);
            dec_attn(true, qkv.p, 3 * D, 0, qkv.p, D, 2 * D, self_k.p + l * sk_layer, self_v.p + l * sk_layer,
                     c.max_target_positions, 0, da_splits_self, B, s);
            gemm_step(L.o, tmx_attn, tc::EPI_ADD, tc::ACT_NONE, x.p, nullptr, B, s);
            ln(L.ln2, x.p, xn.p, B, DEC_HALF, nullptr, 1, s);
            gemm_step(L.cq, tmx_xn, tc::EPI_STORE, tc::ACT_NONE, cq.p, nullptr, B, s);
            dec_attn(false, cq.p, D, 0, nullptr, 0, 0, cross_k.p + l * ck_layer, cross_v.p + l * ck_layer,
                     c.max_source_positions, c.max_source_positions, da_splits_cross, B, s);
            gemm_step(L.co, tmx_attn, tc::EPI_ADD, tc::ACT_NONE, x.p, nullptr, B, s);
            ln(L.ln3, x.p, xn.p, B, DEC_HALF, nullptr, 1, s);
            gemm_step(L.fc1, tmx_xn, tc::EPI_STORE_BF16, tc::ACT_GELU, nullptr, act.p, B, s);
            gemm_step(L.fc2, tmx_act, tc::EPI_ADD, tc::ACT_NONE, x.p, nullptr, B, s);
        }
    }
    void run_logits(int B, cudaStream_t s) {
        ln(dec_ln, x.p, xn.p, B, DEC_HALF, nullptr, 1, s);
        gemm_step(tm_embed, cfg.vocab_size, d(), nullptr, tmx_xn, tc::EPI_STORE, tc::ACT_NONE, logits.p, nullptr, B, s);   // tied (:325)
    }

    void drop_graphs() {
        if (g_full) { cudaGraphExecDestroy(g_full); g_full = nullptr; }
        if (g_layers) { cudaGraphExecDestroy(g_layers); g_layers = nullptr; }
    }
    static bool same_pick(const PickArgs& a, const PickArgs& b) {
        return a.out_tokens == b.out_tokens && a.begin_suppress == b.begin_suppress && a.n_begin == b.n_begin && a.suppress == b.suppress &&
               a.n_suppress == b.n_suppress && a.max_tokens == b.max_tokens && a.timestamp_begin == b.timestamp_begin && a.eot == b.eot &&
               a.mask_eot == b.mask_eot && a.V == b.V && a.temperature == b.temperature && a.seed == b.seed;
    }
    void capture(int B, const PickArgs& pa) {
        if (g_full && g_B == B && same_pick(pa, g_pick)) return;
        drop_graphs();
        cudaGraph_t g;
        B2A_CUDA(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
        run_layers(B, stream);
        run_logits(B, stream);
        launch_pdl(wh_pick_kernel, dim3(B), dim3(1024), 0, stream, pa);
        B2A_CUDA(cudaStreamEndCapture(stream, &g));
        B2A_CUDA(cudaGraphInstantiate(&g_full, g, 0));
        cudaGraphDestroy(g);
        B2A_CUDA(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
        run_layers(B, stream);
        B2A_CUDA(cudaStreamEndCapture(stream, &g));
        B2A_CUDA(cudaGraphInstantiate(&g_layers, g, 0));
        cudaGraphDestroy(g);
        g_B = B; g_pick = pa;
    }
    int launches_layers() const { return 1 + cfg.decoder_layers * 11; }
};

static double wh_now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

static void stt_transcribe_impl(b2a_stt* h, const float* pcm, bool on_device, int B, long long n, const b2a_stt_params* sp,
                                int32_t* tokens_out, int32_t* n_tokens_out, b2a_stt_info* info) {
    B2A_CHECK(h && pcm && sp, B2A_ERR_INVALID_INPUT, "stt transcribe: null argument");
    B2A_CHECK(B >= 1 && B <= h->cfg.max_batch, B2A_ERR_INVALID_INPUT, "stt transcribe: batch exceeds max_batch");
    B2A_CHECK(n > 200, B2A_ERR_INVALID_INPUT, "stt transcribe: clips must be longer than 200 samples");
    B2A_CHECK(sp->n_prompt >= 1 && sp->prompt_ids, B2A_ERR_INVALID_INPUT, "stt transcribe: empty decoder prompt");
    B2A_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    h->cancel.store(0);
    const int P = sp->n_prompt;
    // maxTokens = max(1, min(params.maxTokens, maxTargetPositions - prompt - 1))   (WhisperModel.swift:219-225)
    const int MT = std::max(1, std::min(sp->max_tokens, h->cfg.max_target_positions - P - 1));
    const double t0 = wh_now();
    const float* d_pcm = pcm;
    if (!on_device) {
        h->ensure_encoder_workspace(B);
        const long long nn = std::min<long long>(n, 480000);
        B2A_CUDA(cudaMemcpy2DAsync(h->pcm.p, nn * sizeof(float), pcm, n * sizeof(float), nn * sizeof(float), B, cudaMemcpyHostToDevice, s));
        d_pcm = h->pcm.p;
        n = nn;
    }
    h->encode_dev(d_pcm, B, n, s);
    h->prompt.upload(sp->prompt_ids, P, s);
    h->out_tokens.alloc((size_t)DEC_HALF * MT);
    const int nb = std::max(0, sp->n_begin_suppress), ns = std::max(0, sp->n_suppress);
    h->d_begin.alloc(std::max(1, nb)); h->d_suppress.alloc(std::max(1, ns));
    if (nb) h->d_begin.upload(sp->begin_suppress, nb, s);
    if (ns) h->d_suppress.upload(sp->suppress, ns, s);
    PickArgs pa{h->logits.p, h->tokens.p, h->pos.p, h->out_tokens.p, h->n_gen.p, h->done.p, h->n_active.p, h->d_begin.p, nb,
                h->d_suppress.p, ns, h->cfg.vocab_size, MT, sp->timestamp_begin, sp->eot, h->bench_mask_eot, sp->temperature > 0.f ? sp->temperature : 0.f, sp->seed};
    B2A_CUDA(cudaStreamSynchronize(s));
    h->capture(B, pa);
    wh_init_rows_kernel<<<1, 32, 0, s>>>(B, h->n_gen.p, h->done.p, h->n_active.p);
    count_launch();
    B2A_CUDA(cudaStreamSynchronize(s));
    const double t1 = wh_now();
    // decoder prefix: forced tokens; only the last prefix position needs logits (:204-211)
    for (int p = 0; p < P; ++p) {
        wh_set_tokens_kernel<<<1, 32, 0, s>>>(h->prompt.p, p, h->tokens.p, h->pos.p, B);
        count_launch();
        if (p < P - 1) { B2A_CUDA(cudaGraphLaunch(h->g_layers, s)); count_launch(h->launches_layers()); }
    }
    int steps = 0;
    bool cancelled = false;
    while (steps < MT) {
        const int burst = std::min(16, MT - steps);
        for (int i = 0; i < burst; ++i) { B2A_CUDA(cudaGraphLaunch(h->g_full, s)); count_launch(h->launches_layers() + 3); }
        steps += burst;
        B2A_CUDA(cudaMemcpyAsync(h->h_flag.p, h->n_active.p, sizeof(int), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
        if (h->cancel.load()) { cancelled = true; break; }
        if (h->h_flag.p[0] <= 0) break;
    }
    const double t2 = wh_now();
    B2A_CHECK(!cancelled, B2A_ERR_CANCELLED, "transcription cancelled");
    std::vector<int> ng(B), toks((size_t)B * MT);
    B2A_CUDA(cudaMemcpyAsync(ng.data(), h->n_gen.p, B * sizeof(int), cudaMemcpyDeviceToHost, s));
    B2A_CUDA(cudaMemcpyAsync(toks.data(), h->out_tokens.p, (size_t)B * MT * sizeof(int), cudaMemcpyDeviceToHost, s));
    B2A_CUDA(cudaStreamSynchronize(s));
    int total = 0;
    for (int b = 0; b < B; ++b) {
        ng[b] = std::min(ng[b], MT);
        total += ng[b];
        if (n_tokens_out) n_tokens_out[b] = ng[b];
        if (tokens_out) memcpy(tokens_out + (size_t)b * sp->max_tokens, toks.data() + (size_t)b * MT, ng[b] * sizeof(int));
    }
    if (info) {
        info->prompt_tokens = P * B; info->generation_tokens = total;
        info->encode_time = t1 - t0; info->decode_time = t2 - t1; info->total_time = t2 - t0;
        info->decode_steps = steps;
    }
}

extern "C" {

int32_t b2a_stt_create(int32_t device, const b2a_whisper_config* cfg, const b2a_tensor* tensors, int32_t n, b2a_stt** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_stt_create: null out");
        *out = nullptr;
        B2A_CHECK(cfg && tensors && n > 0, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_stt_create: missing config or weights");
        TensorTable tt(tensors, n);
        *out = new b2a_stt(device, *cfg, tt);
    });
}

int32_t b2a_stt_create_random(int32_t device, const b2a_whisper_config* cfg, float std, uint64_t seed, b2a_stt** out) {
    return guarded([&] {
        B2A_CHECK(out && cfg && std > 0.f, B2A_ERR_INVALID_INPUT, "b2a_stt_create_random: bad argument");
        *out = nullptr;
        *out = new b2a_stt(device, *cfg, std, seed);
    });
}

void* b2a_stt_stream(b2a_stt* h) { return h ? (void*)h->stream : nullptr; }

int32_t b2a_stt_encode(b2a_stt* h, const float* pcm, int32_t B, int64_t n, float* enc_out) {
    return guarded([&] {
        B2A_CHECK(h && pcm && enc_out, B2A_ERR_INVALID_INPUT, "b2a_stt_encode: null argument");
        B2A_CHECK(B >= 1 && B <= h->cfg.max_batch && n > 200, B2A_ERR_INVALID_INPUT, "b2a_stt_encode: bad batch / length");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        h->ensure_encoder_workspace(B);
        const long long nn = std::min<long long>(n, 480000);
        B2A_CUDA(cudaMemcpy2DAsync(h->pcm.p, nn * sizeof(float), pcm, n * sizeof(float), nn * sizeof(float), B, cudaMemcpyHostToDevice, s));
        h->encode_dev(h->pcm.p, B, nn, s);
        B2A_CUDA(cudaStreamSynchronize(s));
        // enc_out tiles (bf16 hi/lo) -> [B, 1500, d] fp32 on the host
        const int D = h->d();
        const long long T2 = (long long)B * 1500, T2p = cdiv(T2, ENC_HALF) * (long long)ENC_HALF;
        std::vector<bf16> tmp((size_t)2 * T2p * D);
        B2A_CUDA(cudaMemcpy(tmp.data(), h->enc_out.p, tmp.size() * sizeof(bf16), cudaMemcpyDeviceToHost));
        for (long long t = 0; t < T2; ++t) {
            const long long r = (t / ENC_HALF) * 2 * ENC_HALF + (t % ENC_HALF);
            for (int i = 0; i < D; ++i)
                enc_out[t * D + i] = __bfloat162float(tmp[(size_t)r * D + i]) + __bfloat162float(tmp[(size_t)(r + ENC_HALF) * D + i]);
        }
    });
}

int32_t b2a_stt_decoder_logits(b2a_stt* h, const int32_t* tokens, int32_t B, int32_t T, float* logits_out) {
    return guarded([&] {
        B2A_CHECK(h && tokens && logits_out, B2A_ERR_INVALID_INPUT, "b2a_stt_decoder_logits: null argument");
        B2A_CHECK(B >= 1 && B <= h->cfg.max_batch && T >= 1 && T < h->cfg.max_target_positions, B2A_ERR_INVALID_INPUT,
                  "b2a_stt_decoder_logits: bad batch / length");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        const int V = h->cfg.vocab_size;
        std::vector<int> tk(DEC_HALF, 0), ps(DEC_HALF, -1);
        for (int p = 0; p < T; ++p) {
            for (int b = 0; b < B; ++b) { tk[b] = tokens[(size_t)b * T + p]; ps[b] = p; }
            B2A_CUDA(cudaMemcpyAsync(h->tokens.p, tk.data(), DEC_HALF * sizeof(int), cudaMemcpyHostToDevice, s));
            B2A_CUDA(cudaMemcpyAsync(h->pos.p, ps.data(), DEC_HALF * sizeof(int), cudaMemcpyHostToDevice, s));
            h->run_layers(B, s);
            h->run_logits(B, s);
            for (int b = 0; b < B; ++b)
                B2A_CUDA(cudaMemcpyAsync(logits_out + ((size_t)b * T + p) * V, h->logits.p + (size_t)b * V, V * sizeof(float),
                                         cudaMemcpyDeviceToHost, s));
            B2A_CUDA(cudaStreamSynchronize(s));
        }
        B2A_CUDA(cudaGetLastError());
    });
}

int32_t b2a_stt_transcribe(b2a_stt* h, const float* pcm, int32_t B, int64_t n, const b2a_stt_params* sp, int32_t* tokens_out,
                           int32_t* n_tokens_out, b2a_stt_info* info) {
    return guarded([&] { stt_transcribe_impl(h, pcm, false, B, n, sp, tokens_out, n_tokens_out, info); });
}

int32_t b2a_stt_transcribe_dev(b2a_stt* h, const float* d_pcm, int32_t B, int64_t n, const b2a_stt_params* sp,
                               int32_t* tokens_out, int32_t* n_tokens_out, b2a_stt_info* info) {
    return guarded([&] { stt_transcribe_impl(h, d_pcm, true, B, n, sp, tokens_out, n_tokens_out, info); });
}

// generate(audio:) on audio longer than one window (WhisperModel.swift:95-182): chunkAudioFor30sWindows cuts the mono signal into
// consecutive 30 s windows (the last one shorter, zero-padded by padOrTrimToWindow inside transcribeChunk) and the reference
// transcribes them ONE AT A TIME; the windows are independent, so here they go through the encoder / decoder as a batch
// (groups of max_batch).  tokens_out [n_chunks, max_tokens], n_tokens_out [n_chunks], offsets_s [n_chunks] (chunk.offsetSeconds).
int32_t b2a_stt_transcribe_long(b2a_stt* h, const float* pcm, int64_t n, const b2a_stt_params* sp, int32_t max_chunks,
                                int32_t* tokens_out, int32_t* n_tokens_out, float* offsets_s, int32_t* n_chunks_out, b2a_stt_info* info) {
    return guarded([&] {
        B2A_CHECK(h && pcm && sp && tokens_out && n_tokens_out && n_chunks_out, B2A_ERR_INVALID_INPUT, "b2a_stt_transcribe_long: null argument");
        const long long W = 480000;                                        // WhisperAudioConfig.chunkLengthSamples
        const int chunks = n <= W ? 1 : (int)((n + W - 1) / W);
        B2A_CHECK(n > 0 && chunks <= max_chunks, B2A_ERR_INVALID_INPUT, "b2a_stt_transcribe_long: more chunks than the output buffers hold");
        *n_chunks_out = chunks;
        const int MT = sp->max_tokens;
        b2a_stt_info acc{}, part{};
        std::vector<float> buf;
        for (int c0 = 0; c0 < chunks; c0 += h->cfg.max_batch) {
            const int nb = std::min(h->cfg.max_batch, chunks - c0);
            buf.assign((size_t)nb * W, 0.f);
            for (int i = 0; i < nb; ++i) {
                const long long start = (long long)(c0 + i) * W, len = std::min<long long>(W, n - start);
                memcpy(&buf[(size_t)i * W], pcm + start, (size_t)len * sizeof(float));
                if (offsets_s) offsets_s[c0 + i] = (float)start / 16000.0f;
            }
            stt_transcribe_impl(h, buf.data(), false, nb, W, sp, tokens_out + (size_t)c0 * MT, n_tokens_out + c0, &part);
            acc.prompt_tokens += part.prompt_tokens; acc.generation_tokens += part.generation_tokens; acc.decode_steps += part.decode_steps;
            acc.encode_time += part.encode_time; acc.decode_time += part.decode_time; acc.total_time += part.total_time;
        }
        if (info) *info = acc;
    });
}

int32_t b2a_stt_set_bench_flags(b2a_stt* h, int32_t mask_eot) {
    if (!h) return B2A_ERR_INVALID_INPUT;
    h->bench_mask_eot = mask_eot != 0;
    return B2A_OK;
}

int32_t b2a_stt_cancel(b2a_stt* h) {
    if (!h) return B2A_ERR_INVALID_INPUT;
    h->cancel.store(1);
    return B2A_OK;
}

void b2a_stt_destroy(b2a_stt* h) { delete h; }

// ------------------------------------------------------------------------------------------------
// Streaming session (SURVEY.md 8f row N3): StreamingInferenceSession.swift:589-950 at the token level, host logic around the model's
// transcribe pass (or a host decoder).  See include/b200audio.h for the contract; oracle/stt_streaming.py is the checker.
// ------------------------------------------------------------------------------------------------
}  // extern "C"

struct b2a_stt_session {
    b2a_stt* model = nullptr;
    b2a_stt_decode_cb cb = nullptr;
    void* user = nullptr;
    b2a_stt_stream_config cfg{};
    b2a_stt_params sp{};
    std::vector<int32_t> prompt, begin_suppress, suppress;
    long long window = 0, overlap = 0;
    std::vector<float> pending;
    long long total = 0;
    bool has_last = false, active = true;
    double last_decode = 0.0, pass_enc = 0.0, pass_dec = 0.0;
    std::vector<std::vector<int32_t>> completed;
    std::vector<int32_t> confirmed, provisional;
    std::vector<double> first_seen;
    std::vector<int> agreement;

    void init(const b2a_stt_stream_config* c) {
        cfg = b2a_stt_stream_config{1.0, 8.0, 1.0, 480, 2, 512, 16000};
        if (c) cfg = *c;
        B2A_CHECK(cfg.sample_rate > 0 && cfg.window_s > 0 && cfg.window_overlap_s >= 0 && cfg.decode_interval_s >= 0 && cfg.delay_ms >= 0 &&
                      cfg.max_tokens_per_pass >= 1, B2A_ERR_INVALID_INPUT, "stt session: bad stream config");
        window = (long long)(cfg.sample_rate * cfg.window_s);
        B2A_CHECK(window >= 1, B2A_ERR_INVALID_INPUT, "stt session: window shorter than one sample");
        overlap = std::max<long long>(0, std::min<long long>(llround(cfg.window_overlap_s * cfg.sample_rate), std::max<long long>(0, window - 1)));   // :578-584
    }
    // continuation after `prefix` for `n` samples
    std::vector<int32_t> decode(const float* pcm, long long n, const std::vector<int32_t>& prefix) {
        pass_enc = pass_dec = 0.0;
        std::vector<int32_t> out((size_t)std::max(1, cfg.max_tokens_per_pass));
        int32_t got = 0;
        if (cb) {
            const int32_t rc = cb(user, pcm, n, prefix.data(), (int32_t)prefix.size(), out.data(), (int32_t)out.size(), &got);
            B2A_CHECK(rc == 0, B2A_ERR_GENERATION_FAILED, "stt session: the host decoder failed");
        } else {
            if (n <= 200) return {};                                              // shorter than the front end accepts: nothing to say yet
            std::vector<int32_t> pr = prompt;
            pr.insert(pr.end(), prefix.begin(), prefix.end());
            if ((int)pr.size() + 1 >= model->cfg.max_target_positions) return {};   // the prefix has filled the decoder context
            b2a_stt_params p = sp;
            p.prompt_ids = pr.data(); p.n_prompt = (int32_t)pr.size();
            p.begin_suppress = begin_suppress.data(); p.n_begin_suppress = (int32_t)begin_suppress.size();
            p.suppress = suppress.data(); p.n_suppress = (int32_t)suppress.size();
            p.max_tokens = cfg.max_tokens_per_pass;
            b2a_stt_info info{};
            stt_transcribe_impl(model, pcm, false, 1, n, &p, out.data(), &got, &info);
            pass_enc = info.encode_time; pass_dec = info.decode_time;
        }
        out.resize((size_t)std::max(0, std::min<int32_t>(got, (int32_t)out.size())));
        return out;
    }
    void finalize(const float* pcm, long long n) {                                // finalizeWindow :727-748
        completed.push_back(decode(pcm, n, {}));
        confirmed.clear(); provisional.clear(); first_seen.clear(); agreement.clear();
    }
    int promote(const std::vector<int32_t>& fresh, double now) {                  // promoteTokens :750-829
        const double delay = cfg.delay_ms / 1000.0;
        size_t match = 0;
        while (match < provisional.size() && match < fresh.size() && provisional[match] == fresh[match]) ++match;
        std::vector<double> seen(fresh.size());
        std::vector<int> agree(fresh.size());
        for (size_t i = 0; i < fresh.size(); ++i) {
            if (i < match) {
                seen[i] = i < first_seen.size() ? first_seen[i] : now;
                agree[i] = std::max(1, (i < agreement.size() ? agreement[i] : 1) + 1);
            } else {
                seen[i] = now; agree[i] = 1;
            }
        }
        const int need = std::max(1, cfg.min_agreement_passes);
        size_t n_promote = 0;
        for (size_t i = 0; i < fresh.size(); ++i) {
            if (now - seen[i] >= delay && agree[i] >= need) n_promote = i + 1;
            else break;
        }
        confirmed.insert(confirmed.end(), fresh.begin(), fresh.begin() + n_promote);
        provisional.assign(fresh.begin() + n_promote, fresh.end());
        first_seen.assign(seen.begin() + n_promote, seen.end());
        agreement.assign(agree.begin() + n_promote, agree.end());
        return (int)n_promote;
    }
    void fill(b2a_stt_stream_update* u, int kind, int promoted) const {
        if (!u) return;
        u->kind = kind; u->promoted = promoted; u->completed_windows = (int32_t)completed.size();
        u->n_confirmed = (int32_t)confirmed.size(); u->n_provisional = (int32_t)provisional.size();
        u->total_audio_s = (double)total / cfg.sample_rate;
        u->pass_encode_time = kind ? pass_enc : 0.0; u->pass_decode_time = kind ? pass_dec : 0.0;
    }
};

extern "C" {

int32_t b2a_stt_session_create(b2a_stt* model, const b2a_stt_params* params, const b2a_stt_stream_config* config, b2a_stt_session** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_stt_session_create: null out");
        *out = nullptr;
        B2A_CHECK(model && params && params->prompt_ids && params->n_prompt >= 1, B2A_ERR_INVALID_INPUT, "b2a_stt_session_create: model and decode parameters needed");
        std::unique_ptr<b2a_stt_session> s(new b2a_stt_session());
        s->init(config);
        B2A_CHECK(s->cfg.sample_rate == 16000 && s->window <= 480000, B2A_ERR_INVALID_INPUT, "b2a_stt_session_create: Whisper needs 16 kHz and windows of at most 30 s");
        s->model = model; s->sp = *params;
        s->prompt.assign(params->prompt_ids, params->prompt_ids + params->n_prompt);
        if (params->n_begin_suppress > 0) s->begin_suppress.assign(params->begin_suppress, params->begin_suppress + params->n_begin_suppress);
        if (params->n_suppress > 0) s->suppress.assign(params->suppress, params->suppress + params->n_suppress);
        *out = s.release();
    });
}

int32_t b2a_stt_session_create_with_decoder(b2a_stt_decode_cb decode, void* user, const b2a_stt_stream_config* config, b2a_stt_session** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_stt_session_create_with_decoder: null out");
        *out = nullptr;
        B2A_CHECK(decode, B2A_ERR_INVALID_INPUT, "b2a_stt_session_create_with_decoder: null decoder");
        std::unique_ptr<b2a_stt_session> s(new b2a_stt_session());
        s->init(config);
        s->cb = decode; s->user = user;
        *out = s.release();
    });
}

int32_t b2a_stt_session_feed(b2a_stt_session* s, const float* pcm, int64_t n, double now, b2a_stt_stream_update* u) {
    return guarded([&] {
        B2A_CHECK(s && (pcm || n == 0) && n >= 0, B2A_ERR_INVALID_INPUT, "b2a_stt_session_feed: bad argument");
        if (!s->active) { s->fill(u, 0, 0); return; }
        s->pending.insert(s->pending.end(), pcm, pcm + n);
        s->total += n;
        if ((long long)s->pending.size() >= s->window) {                           // a whole window: freeze it (:600-616)
            std::vector<float> win(s->pending.begin(), s->pending.begin() + s->window);
            s->pending.erase(s->pending.begin(), s->pending.begin() + std::max<long long>(0, s->window - s->overlap));
            s->has_last = true; s->last_decode = now;
            s->finalize(win.data(), (long long)win.size());
            s->fill(u, 2, 0);
            return;
        }
        if ((long long)s->pending.size() < s->cfg.sample_rate / 2) { s->fill(u, 0, 0); return; }
        if (s->has_last && now - s->last_decode < std::max(0.2, s->cfg.decode_interval_s)) { s->fill(u, 0, 0); return; }
        s->has_last = true; s->last_decode = now;
        const std::vector<int32_t> fresh = s->decode(s->pending.data(), (long long)s->pending.size(), s->confirmed);
        const int promoted = s->promote(fresh, now);
        s->fill(u, 1, promoted);
    });
}

int32_t b2a_stt_session_stop(b2a_stt_session* s, double now, b2a_stt_stream_update* u) {
    (void)now;
    return guarded([&] {
        B2A_CHECK(s, B2A_ERR_INVALID_INPUT, "b2a_stt_session_stop: null session");
        if (!s->active) { s->fill(u, 0, 0); return; }
        s->active = false;
        s->pass_enc = s->pass_dec = 0.0;
        if (!s->pending.empty()) s->finalize(s->pending.data(), (long long)s->pending.size());
        s->confirmed.insert(s->confirmed.end(), s->provisional.begin(), s->provisional.end());
        s->provisional.clear(); s->first_seen.clear(); s->agreement.clear();
        s->pending.clear();
        s->fill(u, 3, 0);
    });
}

int32_t b2a_stt_session_tokens(b2a_stt_session* s, int32_t which, int32_t window, int32_t* out, int32_t cap, int32_t* n_out) {
    return guarded([&] {
        B2A_CHECK(s && n_out && (out || cap == 0) && cap >= 0, B2A_ERR_INVALID_INPUT, "b2a_stt_session_tokens: bad argument");
        const std::vector<int32_t>* v = nullptr;
        if (which == 0) {
            B2A_CHECK(window >= 0 && window < (int32_t)s->completed.size(), B2A_ERR_INVALID_INPUT, "b2a_stt_session_tokens: no such completed window");
            v = &s->completed[(size_t)window];
        } else if (which == 1) v = &s->confirmed;
        else if (which == 2) v = &s->provisional;
        B2A_CHECK(v, B2A_ERR_INVALID_INPUT, "b2a_stt_session_tokens: which must be 0, 1 or 2");
        *n_out = (int32_t)v->size();
        const size_t m = std::min<size_t>(v->size(), (size_t)cap);
        if (m) memcpy(out, v->data(), m * sizeof(int32_t));
    });
}

void b2a_stt_session_destroy(b2a_stt_session* s) { delete s; }

}  // extern "C"

// The encoder attention on its own (include/b200audio_internal.h): pack_qkv_f16_kernel + mha_tc_kernel on a DEVICE fp32
// qkv [B * T, 3 * nh * 64] (q | k | v), written to `out` as the encoder's hi/lo bf16 tiles of 64 tokens, [2 * 64 * cdiv(B * T, 64), nh * 64].
extern "C" int32_t b2a_mha_tc_test(const float* qkv, void* out, int32_t B, int32_t T, int32_t nh, void* stream) {
    using namespace b2a;
    return guarded([&] {
        B2A_CHECK(qkv && out && B >= 1 && T >= 1 && nh >= 1, B2A_ERR_INVALID_INPUT, "b2a_mha_tc_test: bad argument");
        require_device(0);
        const cudaStream_t s = (cudaStream_t)stream;
        const int Tp = cdiv(T, fa::BQ) * fa::BQ;
        const size_t n = (size_t)B * nh * Tp * HD;
        DBuf<__half> q, k, vt;
        q.alloc(n); k.alloc(n); vt.alloc(n);
        const CUtensorMap tq = tc::make_tmap_f16_3d(q.p, HD, Tp, (long long)B * nh, 64, fa::BQ);
        const CUtensorMap tk = tc::make_tmap_f16_3d(k.p, HD, Tp, (long long)B * nh, 64, fa::BKV);
        const CUtensorMap tv = tc::make_tmap_f16_3d(vt.p, Tp, HD, (long long)B * nh, 64, 64);
        B2A_CUDA(cudaFuncSetAttribute(fa::mha_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fa::FA_SMEM_BYTES));
        fa::pack_qkv_f16_kernel<<<dim3(Tp / 64, B, nh), 256, 0, s>>>(qkv, q.p, k.p, vt.p, T, Tp, nh, 1.0f / sqrtf((float)HD));
        const fa::Args args{(__nv_bfloat16*)out, T, Tp, nh, nh * HD, ENC_HALF};
        fa::mha_tc_kernel<<<dim3(Tp / fa::BQ, nh, B), fa::FA_THREADS, fa::FA_SMEM_BYTES, s>>>(tq, tk, tv, args);
        count_launch(2);
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

// The decoder-step attention on its own (include/b200audio_internal.h): mha_decode_kernel with the grid and launch of
// b2a_stt::dec_attn, on DEVICE caches and workspace the caller owns; cross-attention runs kv_relayout_kernel first, as encode_dev does.
extern "C" int32_t b2a_wh_decode_attn_test(int32_t self_attn, const float* q, const float* kv, const int32_t* pos, void* kcache,
                                           void* vcache, void* out, float* part_o, float* part_ml, int32_t* counters, int32_t B,
                                           int32_t nh, int32_t max_t, void* stream) {
    using namespace b2a;
    return guarded([&] {
        B2A_CHECK(q && pos && kcache && vcache && out && part_o && part_ml && counters && (self_attn || kv) && B >= 1 && B <= DEC_HALF &&
                      nh >= 1 && max_t >= 1, B2A_ERR_INVALID_INPUT, "b2a_wh_decode_attn_test: bad argument");
        require_device(0);
        const cudaStream_t s = (cudaStream_t)stream;
        const int d = nh * HD;
        if (self_attn) {
            const int S = cdiv(max_t, DA_CAP);
            const DecAttnArgs a{q, q, pos, kcache, vcache, (bf16*)out, part_o, part_ml, counters, 3 * d, 0, d, 2 * d, nh, max_t, 0, S, d,
                                1.0f / sqrtf((float)HD)};
            launch_pdl(mha_decode_kernel<true>, dim3(nh, B, S), dim3(2 * DA_CAP), 0, s, a);
        } else {
            kv_relayout_kernel<<<(unsigned)((long long)B * max_t), 256, 0, s>>>(kv, (__half*)kcache, (__half*)vcache, max_t, d, nh);
            count_launch();
            const int S = cdiv(max_t, DA_CAP_CROSS);
            const DecAttnArgs a{q, nullptr, pos, kcache, vcache, (bf16*)out, part_o, part_ml, counters, d, 0, 0, 0, nh, max_t, max_t, S, d,
                                1.0f / sqrtf((float)HD)};
            launch_pdl(mha_decode_kernel<false>, dim3(nh, B, S), dim3(2 * DA_CAP_CROSS), 0, s, a);
        }
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}
