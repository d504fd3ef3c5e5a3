// Orpheus / Llama-3 autoregressive step for sm_90a.  Replaces (reference paths):
//   Sources/MLXAudioTTS/Models/Llama/LlamaTTS.swift:104-202  Llama3ScaledRoPE
//   Sources/MLXAudioTTS/Models/Llama/LlamaTTS.swift:206-346  attention / MLP / block / inner model
//   Sources/MLXAudioTTS/Models/Llama/LlamaTTS.swift:557-567  tied lm head
//   Sources/MLXAudioTTS/Models/Llama/LlamaTTS.swift:658-765  generate loop (+ :383-434 parseOutput,
//                                                            :41-98 SNAC frame (de)interleave)
//   mlx-swift-lm 3.31.4 (un-vendored): TopPSampler / RepetitionContext (call sites :691-692)
//
// HBM layout: weights bf16 [out, in] row-major (q|k|v fused into one matrix, gate/up row-
// interleaved so SwiGLU is a GEMM epilogue); KV cache fp32 [layer][B][kv_head][ctx][128];
// residual stream fp32 [B, H]; GEMM inputs bf16 hi/lo pairs [2R, K] at the step's width R (tc::decode_width).
// The whole decode step (embed -> 28 layers -> lm head -> logits processors -> sampler ->
// bookkeeping) is captured in one CUDA graph and replayed per token; nothing syncs with the
// host inside the loop except a poll of the "all rows finished" flag every few steps.
#include "common.cuh"
#include <cooperative_groups.h>
#include "tc_gemm.cuh"
#include "prompt_attn_tc.cuh"
#include "qwen3_sampler.cuh"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <cmath>
#include <memory>

namespace b2a {

typedef __nv_bfloat16 bf16;

// The special tokens of a TTS language model's vocabulary, how a generated row is parsed into SNAC codes and how the codes are decoded.
// A b2a_tts handle carries one; the prompt framing is [pad..] [SOH] text [EOT, EOH], a reference clip's block
// [SOH] transcript [EOT, EOH] [SOAI, SOS] codes + audio_offset [EOS, EOAI].
struct TokenLayout {
    int start_of_human, end_of_human, end_of_text;
    int start_of_ai, end_of_ai;                 // Orpheus: 128261 / 128262, the tokens around its reference codes (LlamaTTS.swift:27-28)
    int start_of_speech, end_of_speech;         // end_of_speech is the stop token: generation ends there and the token is not kept
    int pad, audio_offset;
    bool ai_fallback;   // parse: a row without start-of-speech starts at its first audio token after the last start-of-AI
    int decode_chunk;   // frames per independent SNAC decode of a row (0: the whole row at once)
};
constexpr TokenLayout ORPHEUS_TOKENS{128259, 128260, 128009, 128261, 128262, 128257, 128258, 128263, 128266, false, 0};
constexpr TokenLayout VYVO_TOKENS{151672, 151673, 151645, 151674, 151675, 151670, 151671, 151676, 151679, true, 50};   // Qwen3.swift:18-29, :47

__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// ------------------------------------------------------------------------------------------------
// embed + RMSNorm
// ------------------------------------------------------------------------------------------------
// x[b,:] = embed[token[b]]  (fp32 residual stream)
// also clears y[b,:] (the fp32 GEMM accumulation target) so a step never sees a previous step's leftovers
__global__ void embed_kernel(const int* __restrict__ tokens, const bf16* __restrict__ embed, float* __restrict__ x,
                             float* __restrict__ y, int H, int V) {
    const int b = blockIdx.x;
    pdl_trigger();
    pdl_wait();
    int tok = tokens[b];
    tok = min(max(tok, 0), V - 1);
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
        x[(long long)b * H + i] = __bfloat162float(embed[(long long)tok * H + i]);
        y[(long long)b * H + i] = 0.f;
    }
}

// inputs given as embeddings (row N1): x[b,:] = src[b,:], y cleared like embed_kernel does
__global__ void ext_embed_kernel(const float* __restrict__ src, float* __restrict__ x, float* __restrict__ y, int H) {
    const int b = blockIdx.x;
    pdl_trigger();
    pdl_wait();
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
        x[(long long)b * H + i] = src[(long long)b * H + i];
        y[(long long)b * H + i] = 0.f;
    }
}

// fused-norm step: the fp32 normalised hidden state  out[b, :] = x[b, :] * rstd[b] * w  from the partial sums of squares.
// ss is [parts, ss_ld] (ss_ld: the step's width).  slot == null (row N1): out is [B, H].  slot != null (Soprano's capture, out [B, slots, H]): row b writes slot k = slot[b] (its n_gen:
// the state of generated token k, or of the last prompt position for k = 0) only while n_cap[b] == k, then n_cap[b] = k + 1.  A stop
// token leaves n_gen unchanged, so the step that feeds it finds the slot taken and writes nothing; read on the device, the graph replays.
__global__ void finalize_norm_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ ss, int parts,
                                     float* __restrict__ out, int H, float eps, const int* __restrict__ slot, int* n_cap, int slots, int ss_ld) {
    const int b = blockIdx.x;
    pdl_trigger();
    pdl_wait();
    long long o = (long long)b * H;
    if (slot) {
        const int k = slot[b];
        const bool take = n_cap[b] == k && k < slots;
        __syncthreads();                       // every thread has read n_cap[b] before it moves on
        if (!take) return;
        if (threadIdx.x == 0) n_cap[b] = k + 1;
        o = ((long long)b * slots + k) * H;
    }
    float t = 0.f;
    for (int p = 0; p < parts; ++p) t += ss[p * ss_ld + b];
    const float r = rsqrtf(t / (float)H + eps);
    for (int i = threadIdx.x; i < H; i += blockDim.x) out[o + i] = x[(long long)b * H + i] * r * w[i];
}

// x += delta (optional, delta is zeroed afterwards);  xn = hi/lo split of  x * rsqrt(mean(x^2) + eps) * w
// One 1024-thread CTA per row, the row lives in registers (H <= 8192).
constexpr int RN_THREADS = 1024, RN_MAXV = 8;
__global__ void __launch_bounds__(RN_THREADS)
add_rmsnorm_kernel(float* __restrict__ x, float* __restrict__ delta, const float* __restrict__ w,
                   bf16* __restrict__ xn, int H, float eps, int half, float* __restrict__ ss_out, int ss_parts) {
    __shared__ float red[RN_THREADS / 32];
    const int b = blockIdx.x, tid = threadIdx.x;
    pdl_trigger();
    pdl_wait();
    float* xr = x + (long long)b * H;
    float v[RN_MAXV];
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < RN_MAXV; ++j) {
        const int i = tid + j * RN_THREADS;
        float val = 0.f;
        if (i < H) {
            val = xr[i];
            if (delta) { val += delta[(long long)b * H + i]; xr[i] = val; delta[(long long)b * H + i] = 0.f; }
        }
        v[j] = val;
        ss += val * val;
    }
    ss = warp_sum(ss);
    if ((tid & 31) == 0) red[tid >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < RN_THREADS / 32; ++i) tot += red[i];
    // ss_out != null ("raw" mode, fused-norm decode step, half = the step's width): xn = hi/lo of x * w UN-normalised, the row's sum
    // of squares goes to ss_out[0, b] of the [ss_parts, half] array (parts 1.. are cleared): the consumer GEMM applies rstd in its
    // epilogue (tc_gemm.cuh, Args::rstd_ss)
    const float r = ss_out ? 1.0f : rsqrtf(tot / (float)H + eps);
    if (ss_out && tid < ss_parts) ss_out[tid * half + b] = tid == 0 ? tot : 0.f;
#pragma unroll
    for (int j = 0; j < RN_MAXV; ++j) {
        const int i = tid + j * RN_THREADS;
        if (i < H) tc::store_hilo(xn, H, b, i, v[j] * r * w[i], half);
    }
}

// ------------------------------------------------------------------------------------------------
// Decode attention (LlamaTTS.swift:235-266): RoPE on q/k, append k/v to the fp32 cache, softmax(qK^T)V.
// ------------------------------------------------------------------------------------------------
constexpr int HD = 128, AT_THREADS = 256, MAXG = 8, AT_CAP = 64;   // AT_CAP * 4 == AT_THREADS
constexpr int AT_SLOTS = 3;                                         // ring slots of attn_decode_cluster_kernel, one 64 x 128 fp32 matrix each
// the q heads per kv head the attention kernels are instantiated for
constexpr bool gqa_supported(int G) { return G == 1 || G == 2 || G == 3 || G == 4 || G == 6 || G == 8; }
// Dynamic shared memory of attn_decode_cluster_kernel<G>: the ring (96 KB), q, the new k | v row, the peer's merged state, barriers.
// 102 528 bytes at G = 3 and 107 648 at G = 8 (plus 512 static): one CTA fits beside a decode GEMM CTA (121 088) or a split-K CTA
// (109 056) on an SM.  The 8 warp-partial outputs ([8][G][128] fp32) are written over ring slot 0 once the last chunk is consumed.
constexpr size_t attn_smem_bytes(int G) {
    return ((size_t)AT_SLOTS * AT_CAP * HD + (size_t)G * HD + 2 * HD + (size_t)G * HD + 2 * MAXG) * sizeof(float) + 64;
}
static_assert((AT_THREADS / 32) * MAXG * HD <= AT_CAP * HD, "the warp-partial outputs must fit in one ring slot");

struct AttnArgs {
    const float* qkv;      // [B, (nq + 2 nkv) * 128] fp32
    const int* pos;        // [B]
    const float* freqs;    // [64] llama3 rope divisors
    float* kcache;         // this layer: [B][nkv][max_ctx][128] fp32
    float* vcache;
    bf16* out;             // [2 lo, nq*128] hi/lo
    int nq, nkv, max_ctx;
    float scale;
    const float* qnorm;    // nullable [128]: per-head RMSNorm gain applied to every q head BEFORE RoPE (Qwen3TTSTalker.swift:127-186)
    const float* knorm;    // nullable [128]: same for the k head
    float qk_eps;
    int lo;                // the step's width (tc::decode_width): row b's lo half is row lo + b of out
};

// One thread-block cluster of two CTAs per (kv head, row), grid (kv heads, rows, 2).  Keys 0..pos are cut into 64-key chunks
// (AT_CAP) that are dealt alternately to the two CTAs: CTA r takes chunks r, r + 2, ...  Each CTA streams the matrices of its chunks
// in the order K_0, V_0, K_1, V_1, ... through a ring of AT_SLOTS one-matrix slots, one cp.async.bulk and one mbarrier per matrix:
// the score pass waits for the K slot only, the P*V pass for the V slot, and a slot is refilled as soon as every warp has left it.
// The first three (K_0, V_0, K_1) are issued BEFORE griddepcontrol.wait; the ring is kept to 96 KB so that this CTA can be resident,
// and those copies in flight, while the QKV GEMM's CTA on the same SM is still in its main loop.  Every warp keeps a running
// (max, sum, P*V) for its 8 keys of each chunk (online softmax) and the 8 warp states are merged once at the end.  CTA 1 hands its
// merged state to CTA 0 through distributed shared memory: one cluster barrier, nothing goes through HBM.  `a` is __grid_constant__
// for the reason given at tc_gemm_kernel.
template <int G>
__global__ void __cluster_dims__(1, 1, 2) __launch_bounds__(AT_THREADS)
attn_decode_cluster_kernel(const __grid_constant__ AttnArgs a) {
    namespace cgr = cooperative_groups;
    cgr::cluster_group cluster = cgr::this_cluster();
    const int rank = (int)cluster.block_rank();
    extern __shared__ __align__(16) uint8_t at_smem[];
    float* sKV = reinterpret_cast<float*>(at_smem);             // [AT_SLOTS][AT_CAP][128]: matrix j of this CTA in slot j % AT_SLOTS
    float* wpo = sKV;                                           // [8 warps][G][128] warp-partial outputs, over slot 0 after the loop
    float* sq = sKV + (size_t)AT_SLOTS * AT_CAP * HD;           // [G][128]
    float* snew = sq + G * HD;                                  // [2][128] the new k / v row of this step
    float* xo = snew + 2 * HD;                                  // [G][128] + [2][G]: the peer CTA's merged state (written remotely)
    float* xml = xo + G * HD;
    uint64_t* bars = reinterpret_cast<uint64_t*>(xml + 2 * MAXG);   // [AT_SLOTS]
    __shared__ float red_m[AT_THREADS / 32][MAXG], red_l[AT_THREADS / 32][MAXG];

    const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    pdl_trigger();
    // pos[b] is read BEFORE griddepcontrol.wait so that the cached K / V chunks stream in under the QKV GEMM's tail.  Programmatic
    // launches chain (a kernel triggers its dependents at its first instruction, even while it is itself still waiting), so on a
    // small model -- every kernel of several layers resident at once -- this prologue can run before a kernel launched many
    // launches earlier has finished (a 1e-1 logits error on a 256-wide model).  The contract that makes the early read
    // safe: EVERY kernel that writes pos[] never calls pdl_trigger() (sample_kernel, prefill_advance_kernel, the q3_* kernels that
    // set a position), so nothing launched after it starts before it has completed.
    const int p = a.pos[b];
    if (!(p >= 0 && p < a.max_ctx)) { pdl_wait(); return; }
    const int nch = p / AT_CAP + 1;
    const int n_my = nch > rank ? (nch - rank + 1) / 2 : 0;     // this CTA's chunks: rank, rank + 2, ...
    const bool owner = ((nch - 1) & 1) == rank;                 // the CTA whose last chunk holds the new position
    const int qkv_ld = (a.nq + 2 * a.nkv) * HD;
    const float* row = a.qkv + (long long)b * qkv_ld;
    float* kc = a.kcache + (((long long)b * a.nkv + h) * a.max_ctx) * HD;
    float* vc = a.vcache + (((long long)b * a.nkv + h) * a.max_ctx) * HD;
    // matrix j of this CTA: K (j even) or V (j odd) of its chunk j / 2; the rows already in the cache are copied (the new position p
    // is staged from this step's q|k|v instead)
    const int n_mat = 2 * n_my;
    auto issue = [&](int j) {
        const int slot = j % AT_SLOTS, c = rank + 2 * (j >> 1);
        const int n_load = (c < nch - 1) ? AT_CAP : p - c * AT_CAP;
        if (n_load > 0) {
            const uint32_t bytes = (uint32_t)n_load * HD * 4;
            tc::mbar_arrive_expect_tx(&bars[slot], bytes);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(tc::smem_u32(sKV + (size_t)slot * AT_CAP * HD)), "l"(((j & 1) ? vc : kc) + (long long)c * AT_CAP * HD), "r"(bytes),
                           "r"(tc::smem_u32(&bars[slot])) : "memory");
        } else {
            tc::mbar_arrive(&bars[slot]);
        }
    };
    if (tid == 0) {
        for (int i = 0; i < AT_SLOTS; ++i) tc::mbar_init(&bars[i], 1);
        tc::fence_barrier_init();
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        for (int j = 0; j < min(n_mat, AT_SLOTS); ++j) issue(j);
    }
    float sn = 0.f, cs = 1.f;
    if (tid < HD / 2) sincosf((float)p / a.freqs[tid], &sn, &cs);   // MLXFast.RoPE(freqs:): angle = pos / freqs[i]
    pdl_wait();
    const float* qsrc = row + (long long)h * G * HD;            // this kv head's G query heads, contiguous
    const float* ksrc = row + (a.nq + h) * HD;
    if (a.qnorm) {
        // per-head RMSNorm of q and k before RoPE: x * rsqrt(mean(x^2) + eps) * w, one warp per 128-vector, staged where RoPE will
        // leave the rotated vector (sq, snew): the thread that rotates the pair (d, d + 64) reads both before it writes either
        for (int vec = tid >> 5; vec < G + 1; vec += AT_THREADS / 32) {
            const float* src = vec < G ? qsrc + vec * HD : ksrc;
            const float* w = vec < G ? a.qnorm : a.knorm;
            const float4 x = reinterpret_cast<const float4*>(src)[tid & 31];
            const float ss = warp_sum(x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w);
            const float r = rsqrtf(ss * (1.0f / HD) + a.qk_eps);
            const float4 g4 = reinterpret_cast<const float4*>(w)[tid & 31];
            reinterpret_cast<float4*>(vec < G ? sq + vec * HD : snew)[tid & 31] =
                make_float4(x.x * r * g4.x, x.y * r * g4.y, x.z * r * g4.z, x.w * r * g4.w);
        }
        __syncthreads();
        qsrc = sq;
        ksrc = snew;
    }
    if (tid < HD / 2) {  // non-traditional RoPE: pairs (i, i+64)
        const int d = tid;
        _Pragma("unroll") for (int g = 0; g < G; ++g) {
            const float* q = qsrc + g * HD;
            const float x1 = q[d], x2 = q[d + HD / 2];
            sq[g * HD + d] = x1 * cs - x2 * sn;
            sq[g * HD + d + HD / 2] = x2 * cs + x1 * sn;
        }
        const float* k = ksrc;
        const float x1 = k[d], x2 = k[d + HD / 2];
        const float k1 = x1 * cs - x2 * sn, k2 = x2 * cs + x1 * sn;
        if (owner) { kc[(long long)p * HD + d] = k1; kc[(long long)p * HD + d + HD / 2] = k2; }
        snew[d] = k1;
        snew[d + HD / 2] = k2;
    } else if (tid >= 128) {
        const int d = tid - 128;
        const float v = row[(a.nq + a.nkv + h) * HD + d];
        if (owner) vc[(long long)p * HD + d] = v;
        snew[HD + d] = v;
    }
    __syncthreads();            // barrier init + q / new-row staging visible

    const int lane = tid & 31, warp = tid >> 5;
    const int kslot = warp * 8 + (lane >> 2), part = lane & 3;
    float m_run[G], l_run[G];
    float4 o4[G];
    _Pragma("unroll") for (int g = 0; g < G; ++g) { m_run[g] = -INFINITY; l_run[g] = 0.f; o4[g] = make_float4(0.f, 0.f, 0.f, 0.f); }

    for (int i = 0; i < n_my; ++i) {
        const int jk = 2 * i, jv = 2 * i + 1, c = rank + 2 * i;
        float* sK = sKV + (size_t)(jk % AT_SLOTS) * AT_CAP * HD;
        float* sV = sKV + (size_t)(jv % AT_SLOTS) * AT_CAP * HD;
        const int t0 = c * AT_CAP, nk = min(AT_CAP, p + 1 - t0);
        tc::mbar_wait(&bars[jk % AT_SLOTS], (uint32_t)((jk / AT_SLOTS) & 1));    // the bulk-copied K rows of this chunk have landed
        if (c == nch - 1) {                                      // splice in the new position (the bulk copy stopped before it)
            if (tid < HD) sK[(p - t0) * HD + tid] = snew[tid];
            __syncthreads();
        }
        float sacc[G];
        _Pragma("unroll") for (int g = 0; g < G; ++g) sacc[g] = 0.f;
        if (kslot < nk) {
            const float4* kr = reinterpret_cast<const float4*>(sK + kslot * HD);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int d4 = part + 4 * ((j + kslot) & 7);     // rotated columns: every quarter-warp hits 8 distinct bank groups
                const float4 kf = kr[d4];
                _Pragma("unroll") for (int g = 0; g < G; ++g) {
                    const float4 qf = reinterpret_cast<const float4*>(sq + g * HD)[d4];
                    sacc[g] = fmaf(qf.x, kf.x, sacc[g]); sacc[g] = fmaf(qf.y, kf.y, sacc[g]);
                    sacc[g] = fmaf(qf.z, kf.z, sacc[g]); sacc[g] = fmaf(qf.w, kf.w, sacc[g]);
                }
            }
        }
        if (jk + AT_SLOTS < n_mat) {
            __syncthreads();                                     // every warp has left the K slot: the next chunk's V goes there
            if (tid == 0) issue(jk + AT_SLOTS);
        }
        float pw[G];
        _Pragma("unroll") for (int g = 0; g < G; ++g) {
            float v = sacc[g];
            v += __shfl_xor_sync(0xffffffffu, v, 1);
            v += __shfl_xor_sync(0xffffffffu, v, 2);
            const float sv = kslot < nk ? v * a.scale : -INFINITY;
            float m = sv;
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16));
            const float m_new = fmaxf(m_run[g], m);
            const float rescale = (m_run[g] == -INFINITY) ? 0.f : __expf(m_run[g] - m_new);
            const float e = (sv == -INFINITY) ? 0.f : __expf(sv - m_new);     // all 4 lanes of a key hold the same value
            float l = part == 0 ? e : 0.f;
            l = warp_sum(l);
            l_run[g] = l_run[g] * rescale + l;
            m_run[g] = m_new;
            o4[g].x *= rescale; o4[g].y *= rescale; o4[g].z *= rescale; o4[g].w *= rescale;
            pw[g] = e;
        }
        tc::mbar_wait(&bars[jv % AT_SLOTS], (uint32_t)((jv / AT_SLOTS) & 1));    // ... and its V rows
        if (c == nch - 1) {
            if (tid >= HD) sV[(p - t0) * HD + tid - HD] = snew[tid];
            __syncthreads();
        }
        // warp-partial P*V: lane owns dims 4*lane .. 4*lane+3 (conflict-free float4 reads of a V row)
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
            const int t = warp * 8 + kk;
            if (t < nk) {
                const float4 v = reinterpret_cast<const float4*>(sV + t * HD)[lane];
                _Pragma("unroll") for (int g = 0; g < G; ++g) {
                    const float pk = __shfl_sync(0xffffffffu, pw[g], kk * 4);
                    o4[g].x = fmaf(pk, v.x, o4[g].x); o4[g].y = fmaf(pk, v.y, o4[g].y);
                    o4[g].z = fmaf(pk, v.z, o4[g].z); o4[g].w = fmaf(pk, v.w, o4[g].w);
                }
            }
        }
        if (jv + AT_SLOTS < n_mat) {
            __syncthreads();                                     // every warp has left the V slot: the K after next goes there
            if (tid == 0) issue(jv + AT_SLOTS);
        }
    }
    __syncthreads();            // every copy has landed and every warp has left the ring: slot 0 now holds the warp-partial outputs
    // merge the 8 warp states
    _Pragma("unroll") for (int g = 0; g < G; ++g) {
        reinterpret_cast<float4*>(wpo + (warp * G + g) * HD)[lane] = o4[g];
        if (lane == 0) { red_m[warp][g] = m_run[g]; red_l[warp][g] = l_run[g]; }
    }
    __syncthreads();
    float Ms[G], Ls[G], Os[G];
    if (tid < HD) {
        _Pragma("unroll") for (int g = 0; g < G; ++g) {
            float M = red_m[0][g];
#pragma unroll
            for (int w = 1; w < AT_THREADS / 32; ++w) M = fmaxf(M, red_m[w][g]);
            float L = 0.f, O = 0.f;
#pragma unroll
            for (int w = 0; w < AT_THREADS / 32; ++w) {
                const float sc_w = red_m[w][g] == -INFINITY ? 0.f : __expf(red_m[w][g] - M);
                L = fmaf(red_l[w][g], sc_w, L);
                O = fmaf(wpo[(w * G + g) * HD + tid], sc_w, O);
            }
            Ms[g] = M; Ls[g] = L; Os[g] = O;
        }
        if (rank == 1) {                                         // hand the state to CTA 0 (distributed shared memory)
            float* rxo = cluster.map_shared_rank(xo, 0);
            float* rxml = cluster.map_shared_rank(xml, 0);
            _Pragma("unroll") for (int g = 0; g < G; ++g) {
                rxo[g * HD + tid] = Os[g];
                if (tid == 0) { rxml[g] = Ms[g]; rxml[MAXG + g] = Ls[g]; }
            }
        }
    }
    cluster.sync();
    if (rank == 0 && tid < HD) {
        _Pragma("unroll") for (int g = 0; g < G; ++g) {
            const float M1 = xml[g], L1 = xml[MAXG + g], O1 = xo[g * HD + tid];
            const float M = fmaxf(Ms[g], M1);
            const float w0 = Ms[g] == -INFINITY ? 0.f : __expf(Ms[g] - M), w1 = M1 == -INFINITY ? 0.f : __expf(M1 - M);
            const float L = Ls[g] * w0 + L1 * w1, O = Os[g] * w0 + O1 * w1;
            tc::store_hilo(a.out, (long long)a.nq * HD, b, (h * G + g) * HD + tid, O / L, a.lo);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Batched prefill (LlamaTTS.swift:711 `self(inputIds, cache)` on the whole prompt): all B*L prompt tokens go
// through each layer at once -- GEMMs on the wgmma kernel with 128-column tiles (64 tokens as hi/lo pairs),
// causal attention over the prompt, K/V written to the fp32 cache.  Prompts whose K/V rows fit in shared memory take the SIMT
// prefill_attn_kernel (per (row, kv head, 32-query tile)), longer ones pack + pfa::prompt_attn_kernel (prompt_attn_tc.cuh).
// ------------------------------------------------------------------------------------------------
constexpr int PF_HALF = 64;      // tokens per 128-row TMA tile
constexpr int PA_QT = 32, PA_THREADS = 256, PA_MAXL = 128;

__global__ void embed_rows_kernel(const int* __restrict__ ids, const bf16* __restrict__ embed, float* __restrict__ x,
                                  int H, int V) {
    const int t = blockIdx.x;
    int tok = ids[t];
    tok = min(max(tok, 0), V - 1);
    for (int i = threadIdx.x; i < H; i += blockDim.x) x[(long long)t * H + i] = __bfloat162float(embed[(long long)tok * H + i]);
}

// cos/sin of pos / freqs[d] for pos < L (MLXFast.RoPE with custom freqs, LlamaTTS.swift:192-200)
__global__ void rope_table_kernel(const float* __restrict__ freqs, float2* __restrict__ tab, int L) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L * (HD / 2)) return;
    const int p = i / (HD / 2), d = i - p * (HD / 2);
    float s, c;
    sincosf((float)p / freqs[d], &s, &c);
    tab[i] = make_float2(c, s);
}

struct PrefillAttnArgs {
    const float* qkv;     // [T, (nq + 2 nkv) * 128]
    const float2* rope;   // [L, 64] (cos, sin)
    float* kcache;        // this layer [B][nkv][max_ctx][128]
    float* vcache;
    bf16* out;            // [2 * T_pad, nq * 128] hi/lo, 64-token tiles
    int nq, nkv, max_ctx, L;
    float scale;
    const float* qnorm;   // nullable [128]: per-head RMSNorm gains of q and k before RoPE, as in AttnArgs
    const float* knorm;
    float qk_eps;
};

template <int G>
__global__ void __launch_bounds__(PA_THREADS)
prefill_attn_kernel(PrefillAttnArgs a) {
    extern __shared__ __align__(16) uint8_t pa_smem[];
    __shared__ float s_rk[PA_MAXL], s_rq[G * PA_QT];           // q/k norm: rstd of every key / query vector of this tile
    const int h = blockIdx.x, b = blockIdx.y, q0 = blockIdx.z * PA_QT;
    const int nqt = min(PA_QT, a.L - q0), kmax = q0 + nqt;     // causal: keys 0 .. q0 + nqt - 1
    float* sK = reinterpret_cast<float*>(pa_smem);              // [kmax][128]
    float* sV = sK + (size_t)a.L * HD;                          // [kmax][128]
    float* sQ = sV + (size_t)a.L * HD;                          // [G][PA_QT][128]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int ld = (a.nq + 2 * a.nkv) * HD;
    const float* base = a.qkv + (long long)b * a.L * ld;
    float* kc = a.kcache + (((long long)b * a.nkv + h) * a.max_ctx) * HD;
    float* vc = a.vcache + (((long long)b * a.nkv + h) * a.max_ctx) * HD;

    if (a.qnorm) {
        // per-head RMSNorm x * rsqrt(mean(x^2) + eps) * w before RoPE: one warp per 128-vector (keys, then the tile's queries g * nqt + qi),
        // the same reduction as attn_decode_cluster_kernel's, so a prompt position normalises exactly as a decode step does
        for (int v = warp; v < kmax + G * nqt; v += PA_THREADS / 32) {
            const int qv = v - kmax;
            const float* src = v < kmax ? base + (long long)v * ld + (a.nq + h) * HD
                                        : base + (long long)(q0 + qv % nqt) * ld + (h * G + qv / nqt) * HD;
            const float4 x = reinterpret_cast<const float4*>(src)[lane];
            const float ss = warp_sum(x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w);
            const float r = rsqrtf(ss * (1.0f / HD) + a.qk_eps);
            if (lane == 0) { if (v < kmax) s_rk[v] = r; else s_rq[qv] = r; }
        }
        __syncthreads();
    }
    // K (RoPE) and V of keys [0, kmax) -> shared memory; this tile's own keys also go to the cache
    for (int i = tid; i < kmax * (HD / 2); i += PA_THREADS) {
        const int t = i / (HD / 2), d = i - t * (HD / 2);
        const float2 cs = a.rope[t * (HD / 2) + d];
        const float* k = base + (long long)t * ld + (a.nq + h) * HD;
        float x1 = k[d], x2 = k[d + HD / 2];
        if (a.knorm) { x1 = x1 * s_rk[t] * a.knorm[d]; x2 = x2 * s_rk[t] * a.knorm[d + HD / 2]; }
        const float k1 = x1 * cs.x - x2 * cs.y, k2 = x2 * cs.x + x1 * cs.y;
        sK[t * HD + d] = k1; sK[t * HD + d + HD / 2] = k2;
        if (t >= q0) { kc[(long long)t * HD + d] = k1; kc[(long long)t * HD + d + HD / 2] = k2; }
    }
    for (int i = tid; i < kmax * HD; i += PA_THREADS) {
        const int t = i / HD, d = i - t * HD;
        const float v = base[(long long)t * ld + (a.nq + a.nkv + h) * HD + d];
        sV[i] = v;
        if (t >= q0) vc[(long long)t * HD + d] = v;
    }
    for (int i = tid; i < G * nqt * (HD / 2); i += PA_THREADS) {
        const int g = i / (nqt * (HD / 2)), r = i - g * nqt * (HD / 2), qi = r / (HD / 2), d = r - qi * (HD / 2);
        const float2 cs = a.rope[(q0 + qi) * (HD / 2) + d];
        const float* q = base + (long long)(q0 + qi) * ld + (h * G + g) * HD;
        float x1 = q[d], x2 = q[d + HD / 2];
        if (a.qnorm) { const float r = s_rq[g * nqt + qi]; x1 = x1 * r * a.qnorm[d]; x2 = x2 * r * a.qnorm[d + HD / 2]; }
        sQ[(g * PA_QT + qi) * HD + d] = x1 * cs.x - x2 * cs.y;
        sQ[(g * PA_QT + qi) * HD + d + HD / 2] = x2 * cs.x + x1 * cs.y;
    }
    __syncthreads();

    // one (head, query) row per warp iteration; lanes over keys for the scores, over dims for P*V
    constexpr int KJ = PA_MAXL / 32;
    for (int r = warp; r < G * nqt; r += PA_THREADS / 32) {
        const int g = r / nqt, qi = r - g * nqt, qpos = q0 + qi;
        const float4* q4 = reinterpret_cast<const float4*>(sQ + (g * PA_QT + qi) * HD);
        float sc[KJ];
        float mx = -INFINITY;
#pragma unroll
        for (int j = 0; j < KJ; ++j) {
            const int t = j * 32 + lane;
            float acc = -INFINITY;
            if (t <= qpos) {
                const float4* k4 = reinterpret_cast<const float4*>(sK + t * HD);
                acc = 0.f;
#pragma unroll 8
                for (int i = 0; i < HD / 4; ++i) {
                    const int d4 = (i + lane) & (HD / 4 - 1);     // rotate: conflict-free rows 512 B apart
                    const float4 kf = k4[d4], qf = q4[d4];
                    acc = fmaf(qf.x, kf.x, acc); acc = fmaf(qf.y, kf.y, acc);
                    acc = fmaf(qf.z, kf.z, acc); acc = fmaf(qf.w, kf.w, acc);
                }
                acc *= a.scale;
            }
            sc[j] = acc;
            mx = fmaxf(mx, acc);
        }
        for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < KJ; ++j) { sc[j] = sc[j] == -INFINITY ? 0.f : __expf(sc[j] - mx); sum += sc[j]; }
        sum = warp_sum(sum);
        float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < KJ; ++j) {
            if (j * 32 > qpos) break;
            for (int l = 0; l < 32; ++l) {
                const int t = j * 32 + l;
                if (t > qpos) break;
                const float p = __shfl_sync(0xffffffffu, sc[j], l);
                const float4 v = reinterpret_cast<const float4*>(sV + t * HD)[lane];
                o.x = fmaf(p, v.x, o.x); o.y = fmaf(p, v.y, o.y); o.z = fmaf(p, v.z, o.z); o.w = fmaf(p, v.w, o.w);
            }
        }
        const float inv = 1.0f / sum;
        const int tok = b * a.L + qpos;
        const long long col = (long long)(h * G + g) * HD + lane * 4;
        const long long ldo = (long long)a.nq * HD;
        tc::store_hilo(a.out, ldo, tok, col + 0, o.x * inv, PF_HALF);
        tc::store_hilo(a.out, ldo, tok, col + 1, o.y * inv, PF_HALF);
        tc::store_hilo(a.out, ldo, tok, col + 2, o.z * inv, PF_HALF);
        tc::store_hilo(a.out, ldo, tok, col + 3, o.w * inv, PF_HALF);
    }
}

// Dynamic shared memory of prefill_attn_kernel<G> for L prompt positions: the K and V rows of the whole prompt and one tile's queries.
constexpr size_t PA_SMEM_MAX = 220 * 1024;
constexpr size_t pattn_smem(int L, int G) { return ((size_t)2 * L * HD + (size_t)G * PA_QT * HD) * sizeof(float); }
// The prompt attention for L positions at G q heads per kv head: the SIMT kernel while its K/V rows fit in shared memory (the outputs
// of short prompts stay what they were), the wgmma kernel beyond.  The largest SIMT L is 128 for G <= 4, 124 for G = 6, 92 for G = 8.
constexpr bool simt_prompt_attn(int L, int G) { return L <= PA_MAXL && pattn_smem(L, G) <= PA_SMEM_MAX; }

// pfa::prompt_attn_kernel's operands for B rows of L positions (padded to Lp = a multiple of pfa::BQ) and their tensor maps;
// grown, never shrunk.  run(): pack_prompt_kernel then prompt_attn_kernel, the attention of one layer.
struct PromptAttnOps {
    DBuf<__half> q, k, vt;
    CUtensorMap tq{}, tk{}, tv{};
    int B = 0, Lp = 0, nq = 0, nkv = 0;
    void prepare(int B_, int L, int nq_, int nkv_) {
        const int Lp_ = cdiv(L, pfa::BQ) * pfa::BQ;
        if (B_ == B && Lp_ == Lp && nq_ == nq && nkv_ == nkv) return;
        B = B_; Lp = Lp_; nq = nq_; nkv = nkv_;
        q.alloc((size_t)B * nq * Lp * pfa::OPW); k.alloc((size_t)B * nkv * Lp * pfa::OPW); vt.alloc((size_t)B * nkv * Lp * pfa::OPW);
        tq = tc::make_tmap_f16_3d(q.p, pfa::OPW, Lp, (long long)B * nq, 64, pfa::BQ);
        tk = tc::make_tmap_f16_3d(k.p, pfa::OPW, Lp, (long long)B * nkv, 64, pfa::BKV);
        tv = tc::make_tmap_f16_3d(vt.p, Lp, pfa::OPW, (long long)B * nkv, 64, pfa::HDIM);
        B2A_CUDA(cudaFuncSetAttribute(pfa::prompt_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pfa::SMEM_BYTES));
    }
    // qkv [B * L, (nq + 2 nkv) * 128] fp32; rope [>= L][64]; caches [B][nkv][max_ctx][128]; out: 64-token hi/lo tiles [.., nq * 128];
    // qnorm / knorm nullable (per-head q/k RMSNorm before RoPE)
    void run(const float* qkv, const float2* rope, float* kcache, float* vcache, bf16* out, int L, int max_ctx, cudaStream_t s,
             const float* qnorm = nullptr, const float* knorm = nullptr, float qk_eps = 0.f) {
        pfa::pack_prompt_kernel<<<dim3(Lp / 64, B, nq + nkv), 256, 0, s>>>(qkv, rope, q.p, k.p, vt.p, kcache, vcache, L, Lp, nq, nkv,
                                                                         max_ctx, qnorm, knorm, qk_eps);
        const pfa::Args a{out, L, Lp, nq, nkv, 1.0f / sqrtf((float)HD)};
        pfa::prompt_attn_kernel<<<dim3(Lp / pfa::BQ, nq, B), pfa::THREADS, pfa::SMEM_BYTES, s>>>(tq, tk, tv, a);
        count_launch(2);
    }
};

// decode buffers <- last prompt position of every row:  x[b] = xp[b*L + L-1], y[b] = yp[...], pos[b] = L - 1
__global__ void gather_last_kernel(const float* __restrict__ xp, const float* __restrict__ yp, float* __restrict__ x,
                                   float* __restrict__ y, int* __restrict__ pos, int L, int H) {
    const int b = blockIdx.x;
    const long long src = ((long long)b * L + L - 1) * H;
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
        x[(long long)b * H + i] = xp[src + i];
        y[(long long)b * H + i] = yp[src + i];
    }
    if (threadIdx.x == 0) pos[b] = L - 1;
}

// ------------------------------------------------------------------------------------------------
// Logits processors + sampler + bookkeeping: one CTA per row.
// ------------------------------------------------------------------------------------------------
constexpr int SM_THREADS = 1024, SM_WARPS = SM_THREADS / 32, SM_MAX_ATTEMPTS = 12;

struct SampleArgs {
    float* logits;        // [B, V]  (modified in place: penalty, EOS mask)
    float* probs;         // [B, V]  scratch
    int* tokens;          // [B] next input token (written)
    int* pos;             // [B] position of the NEXT input token (incremented)
    int* recent;          // [B, R] ring of the last R tokens (prompt + generated)
    int* recent_n;        // [B] total tokens pushed so far
    int* out_tokens;      // [B, max_tokens]
    int* n_gen;           // [B]
    int* done;            // [B]
    int* n_active;        // [1] rows not yet finished (decremented when a row emits EOS)
    const int* forced;    // nullable [B]: if set, ignore the sampler and emit forced[b] (prefill)
    int V, R, max_tokens;
    float temperature, top_p, rep_penalty;
    unsigned long long seed;
    int mask_eos;         // bench only: the stop token can never be sampled
    int stop_token;       // ends a row and is not recorded (TokenLayout::end_of_speech)
    int soprano;          // Soprano's own penalty and top-p (Soprano.swift:836-901, :996-1059), see sample_kernel
};

// Logits processors + sampler (deterministic for a given seed, no atomics):
//   RepetitionContext.process -> EOS mask (bench only) -> argmax | TopPSampler.
// Top-p = "sample from the smallest top set whose mass reaches top_p".  Implemented as rejection sampling: draw
// token ~ softmax(l/T) by the Gumbel-max trick (token = argmax_i l_i/T + g_i, g_i = -log(-log(u_i)), u_i a hash of (seed, row,
// step, attempt, i): one coalesced pass, no inverse-CDF walk), accept iff the mass of strictly more probable tokens is < top_p
// (exactly the nucleus membership test; ties are all kept).  The acceptance probability is >= top_p, so a handful of
// attempts suffice; after SM_MAX_ATTEMPTS the argmax (always in the nucleus) is returned.
// One thread-block CLUSTER of SM_CLUSTER CTAs per row: every CTA owns a contiguous 1/8 of the vocabulary (19 618 of Orpheus's
// 156 940 logits: 20 per thread) and the per-pass (max, index) / sums are exchanged through distributed shared memory -- every CTA
// writes its partial into every peer's slot, one cluster barrier, every CTA reduces the 8 partials in rank order.  (One CTA per row
// would run the sampling passes on 8 SMs, bound by a single SM's issue rate.)
constexpr int SM_CLUSTER = 8;
struct SampleExchange { float v[2][SM_CLUSTER]; int i[2][SM_CLUSTER]; float s[2][SM_CLUSTER]; };

__global__ void __cluster_dims__(SM_CLUSTER, 1, 1) __launch_bounds__(SM_THREADS)
sample_kernel(SampleArgs a) {
    namespace cgr = cooperative_groups;
    cgr::cluster_group cluster = cgr::this_cluster();
    const int rank = (int)cluster.block_rank();
    __shared__ float sred[SM_WARPS];
    __shared__ float s_val[SM_WARPS];
    __shared__ int s_idx[SM_WARPS];
    __shared__ SampleExchange ex;
    const int b = blockIdx.x / SM_CLUSTER, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    pdl_wait();                  // NO pdl_trigger(): this kernel writes pos[] (see attn_decode_cluster_kernel)
    float* lg = a.logits + (long long)b * a.V;
    const int chunk = (a.V + SM_CLUSTER - 1) / SM_CLUSTER, i0 = rank * chunk, i1 = min(a.V, i0 + chunk);
    const int nrec = min(a.recent_n[b], a.R);
    int parity = 0;
    int tok_final = 0;

    // (value, index) and a sum: block reduce, then all-to-all through distributed shared memory; every CTA ends with the same result
    auto exchange = [&](float& v, int& i, float& sum) {
        for (int o = 16; o; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, v, o);
            const int oi = __shfl_xor_sync(0xffffffffu, i, o);
            if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
        }
        sum = warp_sum(sum);
        __syncthreads();
        if (lane == 0) { s_val[warp] = v; s_idx[warp] = i; sred[warp] = sum; }
        __syncthreads();
        if (warp == 0) {
            float bv = s_val[lane], bs = sred[lane];
            int bi = s_idx[lane];
            for (int o = 16; o; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            bs = warp_sum(bs);
            if (lane < SM_CLUSTER) {             // lane p writes this CTA's partial into CTA p's slot [rank]
                SampleExchange* peer = cluster.map_shared_rank(&ex, lane);
                peer->v[parity][rank] = bv; peer->i[parity][rank] = bi; peer->s[parity][rank] = bs;
            }
        }
        cluster.sync();
        v = ex.v[parity][0]; i = ex.i[parity][0]; sum = ex.s[parity][0];
#pragma unroll
        for (int r = 1; r < SM_CLUSTER; ++r) {
            const float ov = ex.v[parity][r];
            const int oi = ex.i[parity][r];
            if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
            sum += ex.s[parity][r];
        }
        parity ^= 1;
    };

    if (a.forced == nullptr) {
        if (a.soprano) {
            // applyRepetitionPenalty (Soprano.swift:888-901) over the last R GENERATED tokens (the prompt never enters the ring: the
            // caller starts it empty, so nothing is penalised before the first token, Soprano.swift:843).  It runs once per
            // OCCURRENCE, in sequence: the first occurrence's thread applies l > 0 ? l / p : l * p as many times as the token occurs.
            // It runs at temperature 0 too, before the argmax.
            if (a.rep_penalty != 1.0f && t < nrec) {
                const int tok = a.recent[b * a.R + t];
                bool first = true;
                int k = 0;
                for (int j = 0; j < nrec; ++j)
                    if (a.recent[b * a.R + j] == tok) { first &= j >= t; ++k; }
                if (first && tok >= i0 && tok < i1) {
                    float l = lg[tok];
                    for (int j = 0; j < k; ++j) l = l > 0.f ? l / a.rep_penalty : l * a.rep_penalty;
                    lg[tok] = l;
                }
            }
        } else if (a.rep_penalty != 1.0f && t < nrec) {
            // RepetitionContext.process: once per unique token among the last R; every CTA handles the tokens of its own range
            const int tok = a.recent[b * a.R + t];
            bool dup = false;
            for (int j = 0; j < t; ++j) dup |= (a.recent[b * a.R + j] == tok);
            if (!dup && tok >= i0 && tok < i1) {
                const float l = lg[tok];
                lg[tok] = l < 0.f ? l * a.rep_penalty : l / a.rep_penalty;
            }
        }
        if (a.mask_eos && t == 0 && a.stop_token >= i0 && a.stop_token < i1) lg[a.stop_token] = -INFINITY;
        __syncthreads();

        // max (and argmax, lowest index wins ties)
        float best = -INFINITY, dummy = 0.f;
        int bi = 0x7fffffff;
        for (int i = i0 + t; i < i1; i += SM_THREADS) {
            const float v = lg[i];
            if (v > best) { best = v; bi = i; }
        }
        exchange(best, bi, dummy);
        const float mx = best;
        tok_final = bi;

        if (a.temperature > 0.f) {
            const float inv_t = 1.0f / a.temperature;
            const int step = a.n_gen[b];
            auto gumbel_key = [&](int i, float l, int att) {
                unsigned long long z = a.seed + 0x9E3779B97F4A7C15ull * ((unsigned long long)b * 1000003ull + (unsigned long long)step * 131ull + (unsigned long long)att + 1ull);
                z ^= (unsigned long long)(unsigned)i * 0xD6E8FEB86659FD93ull;
                z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
                z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
                z ^= z >> 31;
                const float u = ((float)(z >> 40) + 0.5f) * (1.0f / 16777216.0f);      // (0, 1)
                return l * inv_t - __logf(-__logf(u));
            };
            // Soprano's TopPSampler (Soprano.swift:1002-1059) filters on exp(l) of the penalised logits, NOT on probabilities: token i
            // is kept iff the ascending cumulative sum of exp(l_j) through i exceeds 1 - top_p, i.e. with g the max-shifted mass of
            // strictly larger logits and z the shifted total, iff g < z - (1 - top_p) e^(-max).  Its masses are taken at temperature 1;
            // the temperature divides the FILTERED logits afterwards (categorical(filtered / T)), which is the proposal below.
            const float zs = a.soprano ? 1.0f : inv_t;
            // pass A: Z = sum exp((l - max) / T) (Soprano: at T = 1) and the first draw
            float z = 0.f, gv = -INFINITY;
            int gi = 0x7fffffff;
            for (int i = i0 + t; i < i1; i += SM_THREADS) {
                const float l = lg[i];
                z += __expf((l - mx) * zs);
                const float k = l == -INFINITY ? -INFINITY : gumbel_key(i, l, 0);
                if (k > gv) { gv = k; gi = i; }
            }
            exchange(gv, gi, z);
            const float Z = z;
            const float cut = a.soprano ? Z - (1.0f - a.top_p) * expf(-mx) : a.top_p * Z;
            int cand = gi;
            bool accepted = a.top_p >= 1.0f;
            // Soprano, sum exp(l) <= 1 - top_p: no token passes and the reference would sample from an all -inf row.  The argmax is
            // returned instead (a deliberate difference).
            if (!accepted && a.soprano && !(cut > 0.f)) { cand = tok_final; accepted = true; }
            for (int att = 0; !accepted; ++att) {
                // nucleus test: the mass of strictly more probable tokens must be below top_p (Soprano: below cut)
                const float lc = lg[cand];
                float gm = 0.f, dv = -INFINITY;
                int di = 0x7fffffff;
                for (int i = i0 + t; i < i1; i += SM_THREADS) { const float l = lg[i]; if (l > lc) gm += __expf((l - mx) * zs); }
                exchange(dv, di, gm);
                if (gm < cut) { accepted = true; break; }
                if (att + 1 >= SM_MAX_ATTEMPTS) { cand = tok_final; break; }      // the argmax is always in the nucleus
                gv = -INFINITY; gi = 0x7fffffff;
                float ds = 0.f;
                for (int i = i0 + t; i < i1; i += SM_THREADS) {
                    const float l = lg[i];
                    const float k = l == -INFINITY ? -INFINITY : gumbel_key(i, l, att + 1);
                    if (k > gv) { gv = k; gi = i; }
                }
                exchange(gv, gi, ds);
                cand = gi;
            }
            if (cand >= 0 && cand < a.V) tok_final = cand;
        }
    } else {
        tok_final = a.forced[b];
    }

    if (rank == 0 && t == 0) {
        const int tok = tok_final;
        a.tokens[b] = tok;
        a.pos[b] += 1;
        const int rn = a.recent_n[b];
        if (a.R > 0) {
            // keep `recent` as "last R tokens" in arrival order: shift when full
            if (rn < a.R) a.recent[b * a.R + rn] = tok;
            else {
                for (int j = 1; j < a.R; ++j) a.recent[b * a.R + j - 1] = a.recent[b * a.R + j];
                a.recent[b * a.R + a.R - 1] = tok;
            }
            a.recent_n[b] = rn + 1;
        }
        if (a.forced == nullptr && !a.done[b]) {
            if (tok == a.stop_token) {           // LlamaTTS.swift:734-736, Qwen3.swift:675-681: stop, token not appended
                a.done[b] = 1;
                atomicSub(a.n_active, 1);
            } else {
                const int n = a.n_gen[b];
                if (n < a.max_tokens) a.out_tokens[b * a.max_tokens + n] = tok;
                a.n_gen[b] = n + 1;
                if (n + 1 >= a.max_tokens) { a.done[b] = 1; atomicSub(a.n_active, 1); }
            }
        }
    }
}

// prefill bookkeeping for positions that do not need logits: next token = ids[b, pos+1]
__global__ void prefill_advance_kernel(const int* __restrict__ ids, int L, int* tokens, int* pos, int B) {
    const int b = threadIdx.x;
    pdl_wait();                  // NO pdl_trigger(): writes pos[]
    if (b >= B) return;
    const int p = pos[b] + 1;
    pos[b] = p;
    if (p < L) tokens[b] = ids[b * L + p];
}

__global__ void init_rows_kernel(const int* __restrict__ ids, int L, int B, int R, int* tokens, int* pos, int* recent,
                                 int* recent_n, int* n_gen, int* done, int* n_active, int start_pos) {
    const int b = threadIdx.x;
    if (b == 0) *n_active = B;
    if (b >= B) return;
    tokens[b] = ids[b * L];
    pos[b] = start_pos;
    n_gen[b] = 0;
    done[b] = 0;
    // processor.prompt(promptTokens): the ring starts with the last R prompt tokens
    const int n = min(R, L);
    for (int j = 0; j < n; ++j) recent[b * R + j] = ids[b * L + L - n + j];
    recent_n[b] = n;
}

// device-side random init (benchmarks / full-size property tests): N(0, std^2) -> bf16
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
__global__ void fill_f32_kernel(float* p, int n, float v) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// ------------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------------
// Qwen3Attention's RoPE (Qwen3.swift:177-192): MLXFast.RoPE(base: theta, scale: 1 / factor), i.e. angle = pos / (theta^(2i/d) * factor)
static std::vector<float> linear_freqs(const b2a_llama_config& c, float factor) {
    std::vector<float> f(c.head_dim / 2);
    for (int i = 0; i < c.head_dim / 2; ++i) f[i] = powf(c.rope_theta, (float)(2 * i) / (float)c.head_dim) * factor;
    return f;
}

static std::vector<float> llama3_freqs(const b2a_llama_config& c) {
    // LlamaTTS.swift:121-156 in Float
    const int d = c.head_dim;
    std::vector<float> f(d / 2);
    const float low_wl = c.rope_old_context_len / c.rope_low_freq_factor;
    const float high_wl = c.rope_old_context_len / c.rope_high_freq_factor;
    for (int i = 0; i < d / 2; ++i) {
        float fr = powf(c.rope_theta, (float)(2 * i) / (float)d);
        const float wl = 2.0f * (float)M_PI * fr;
        const float base = fr;
        if (wl > low_wl) fr = fr * c.rope_factor;
        const bool med = wl > high_wl && wl < low_wl;
        if (med) {
            const float smooth = (c.rope_old_context_len / wl - c.rope_low_freq_factor) /
                                 (c.rope_high_freq_factor - c.rope_low_freq_factor);
            fr = base / ((1.0f - smooth) / c.rope_factor + smooth);
        }
        f[i] = fr;
    }
    return f;
}

struct LayerW {
    DBuf<bf16> wqkv, wo, wgu, wdown;
    DBuf<float> ln1, ln2;
    DBuf<float> qnorm, knorm;   // [128] each, only with StackSpec::qk_norm
};

// Which checkpoint keys a transformer stack is built from.  Orpheus: {"model.", embeddings + tied head}.  The Qwen3-TTS talker
// and code predictor (row N1) reuse the same engine with per-head q/k RMSNorm, inputs given as EMBEDDINGS and heads owned by the
// caller (Qwen3TTSTalker.swift:127-310, Qwen3TTSCodePredictor.swift:14-240).
struct StackSpec {
    std::string prefix = "model.";            // "<prefix>layers.N....", "<prefix>norm.weight"
    bool qk_norm = false;                      // self_attn.q_norm / k_norm
    bool has_embed = true;                     // "<prefix>embed_tokens.weight" (false: inputs are embeddings)
    std::string head;                          // "" = tied to the embedding / none; else an untied [vocab, hidden] matrix
    bool has_head = true;
    float linear_rope = 0.f;                   // > 0: Qwen3Attention's RoPE with this linear factor (linear_freqs); 0: Llama3ScaledRoPE
};

}  // namespace b2a

using namespace b2a;

struct b2a_tts {
    int device;
    b2a_llama_config cfg;
    b2a_snac* snac;
    cudaStream_t stream = nullptr;
    std::vector<LayerW> layers;
    DBuf<bf16> embed, lm_head_w;
    const bf16* lm_head = nullptr;
    DBuf<float> final_ln, freqs;
    DBuf<float> kcache, vcache;   // [layer][B][nkv][ctx][hd] fp32
    // activations: fp32 residual stream [max_batch, H]; GEMM inputs as [2R, K] bf16 hi/lo pairs, R the call's width
    DBuf<float> x, y, qkv, logits, probs;
    DBuf<bf16> xn, attn, act;
    DBuf<float> sk_ws;       // stream-K partial tiles of the q|k|v GEMM when it runs stream-K (qkv_cluster == 0), see tc::Args::part_ws
    DBuf<unsigned> sk_cnt;
    int sk_slots = 0;
    int num_sms = 132;
    std::vector<CUtensorMap> tm_qkv, tm_o, tm_gu, tm_down;
    // weight rows per m-tile for a whole-tile GEMM of M rows (tc::Args::tile_rows): 128 unless that leaves > 1/4 of the SMs idle
    static int pick_tile_rows(int M, int sms) {
        if (cdiv(M, tc::BM) * 4 >= sms * 3) return tc::BM;
        return std::max(8, std::min(tc::BM, cdiv(cdiv(M, sms), 8) * 8));
    }
    int lm_tile_rows = 128, head_rows_now = 0;   // head_rows_now: tile rows of the map passed to the current OP_LM launch (0 = lm_tile_rows)
    std::vector<CUtensorMap> tm_gu_dec;     // gate/up with gu_tile_rows-row boxes for the decode step (tc::Args::tile_rows)
    int gu_tile_rows = 0;
    CUtensorMap tm_lm{};
    CUtensorMap tmx_xn[3]{}, tmx_attn[3]{}, tmx_act[3]{};   // per width (tc::decode_width_index): [2R, K] with 2R-row boxes
    // batched prefill workspace (sized for the largest B*L seen so far)
    DBuf<float> xp, yp, qkvp;
    DBuf<bf16> xnp, attnp, actp;
    DBuf<float2> rope_tab;
    PromptAttnOps pfa_ops;
    CUtensorMap tmp_xn{}, tmp_attn{}, tmp_act{};
    int pf_tokens_cap = 0;
    bool use_batched_prefill = true;
    DBuf<int> tokens, pos, recent, recent_n, out_tokens, n_gen, done, n_active, ids, forced;
    HBuf<int> h_flag;
    cudaEvent_t ev_poll[2] = {nullptr, nullptr};   // the generate loop's pipelined "rows still active" polls
    // fused-norm decode step: o_proj / down_proj run as cluster split-K GEMMs whose leader CTA does the residual add + the next
    // norm's gain + hi/lo split + sum of squares; one add_rmsnorm launch per step, for the first norm (tc_gemm.cuh).  q|k|v runs on
    // the same kernel in store mode (qkv_gemm)
    static constexpr int fused_cluster = 5;   // 5 CTAs per 128-row tile: 120 of 132 SMs for hidden 3072, one wave
    int qkv_cluster[3] = {0, 0, 0};           // per width: CTAs per 128-row tile of the q|k|v split-K GEMM (pick_qkv_cluster); 0: stream-K
    int qkv_sk_ctas = 0;                      // the stream-K CTA count whose cut of the k-blocks that GEMM reproduces (any width)
    // ring depths of the decode step's GEMMs per width (8, 16, 32 rows).  At 8 rows tc::Smem<16>::bytes, tc::SmemSplit<8>::bytes and
    // attn_smem_bytes() are sized so that any two kernels that follow each other in the fused step fit on one SM together
    // (b2a_debug_step_smem reports the three); DESIGN.md section 3.3 gives the wider widths' choice (b2a_debug_step_smem_rows)
    static constexpr int GEMM_STAGES[3] = {6, 4, 3}, SPLITK_STAGES[3] = {5, 4, 2};
    int width = 8, wi = 0;           // the current call's width R (tc::decode_width of its rows) and its index
    int max_width = 8;               // the width of max_batch rows: activation buffers hold [2 max_width, K]
    int fused_parts = 0;             // m-tiles of H (the last one may be partly filled): partial sums of squares per row
    DBuf<float> ss_a, ss_b;          // [fused_parts <= 64, R] partial sums of squares: ss_a feeds the post-attention norm, ss_b the input norm
    StackSpec spec;                  // which keys / features this stack was built with
    TokenLayout tok = ORPHEUS_TOKENS;  // special tokens, parse rule and decode chunking of generate (VYVO_TOKENS: b2a_qwen3_lm_create)
    const float* x_ext = nullptr;    // row N1: when set, a step starts from these embeddings [max_batch, H] instead of embed(tokens)
    float* normed_out = nullptr;     // row N1: when set, run_final_norm writes the final RMSNorm's fp32 output here [max_batch, H]
    std::atomic<int> cancel{0};
    int bench_mask_eos = 0, bench_wrap_codes = 0;   // b2a_tts_set_bench_flags (include/b200audio_internal.h): fixed-work benchmark switches
    int nb_pad = 0;   // rows rounded up to 1/2/4/8 within width 8, else the width
    bool trace_on = false;       // debug: residual stream at every RMSNorm input (eager forward only, trace_x)
    DBuf<float> trace;           // [2*layers + 1][max_batch][H]
    // CUDA graphs for the two step flavours (captured per (rows, params) configuration)
    cudaGraphExec_t g_step = nullptr, g_prefill = nullptr;
    SampleArgs g_args{};
    int g_nb = 0;
    // codec workspaces
    DBuf<int> d_codes[3];
    DBuf<float> d_wave;
    // Soprano (b2a_soprano_create): the handle owns a Vocos decoder and the step captures every row's final-norm hidden state into
    // hidden [B, hidden_slots = max_tokens + 1, H] (finalize_norm_kernel); n_cap[b] counts the states row b holds
    b2a_vocos* vocos = nullptr;
    int upscale = 0, token_size = 0;
    DBuf<float> hidden;
    DBuf<int> n_cap, d_rows;
    int hidden_slots = 0, hidden_rows = 0;
    const float* g_hidden = nullptr;   // the capture buffer the step graph was captured with

    ~b2a_tts() {
        if (vocos) b2a_vocos_destroy(vocos);
        if (g_step) cudaGraphExecDestroy(g_step);
        if (g_prefill) cudaGraphExecDestroy(g_prefill);
        for (auto& e : ev_poll) if (e) cudaEventDestroy(e);
        if (stream) cudaStreamDestroy(stream);
    }

    static void upload_bf16(const TensorTable& tt, const std::string& name, int64_t expect, DBuf<bf16>& dst, size_t offset_elems,
                            size_t total_elems) {
        const b2a_tensor& t = tt.get(name);
        B2A_CHECK(t.dtype == B2A_DTYPE_BF16 || t.dtype == B2A_DTYPE_F32, B2A_ERR_MODEL_NOT_INITIALIZED, "tensor must be bf16 or f32: " + name);
        B2A_CHECK(TensorTable::numel(t) == expect, B2A_ERR_MODEL_NOT_INITIALIZED, "bad shape for tensor: " + name);
        dst.alloc(total_elems);
        if (t.dtype == B2A_DTYPE_BF16) {
            B2A_CUDA(cudaMemcpy(dst.p + offset_elems, t.data, expect * sizeof(bf16), cudaMemcpyHostToDevice));
        } else {   // an fp32 checkpoint: the engine holds bf16 matrices, round to nearest even (stated deviation, as for Whisper)
            std::vector<bf16> tmp((size_t)expect);
            const float* src = (const float*)t.data;
            for (int64_t i = 0; i < expect; ++i) tmp[i] = __float2bfloat16_rn(src[i]);
            B2A_CUDA(cudaMemcpy(dst.p + offset_elems, tmp.data(), expect * sizeof(bf16), cudaMemcpyHostToDevice));
        }
    }

    template <int G>
    static void attn_cluster_attr() {
        B2A_CUDA(cudaFuncSetAttribute(attn_decode_cluster_kernel<G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_smem_bytes(G)));
        // it shares an SM with a GEMM CTA of the step (see tc::set_attributes)
        B2A_CUDA(cudaFuncSetAttribute(attn_decode_cluster_kernel<G>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    }
    // the decode-step attention for rows 0..B-1 (the caller has checked gqa_supported(nq / nkv))
    static void attn_launch(const AttnArgs& aa, int B, cudaStream_t s) {
        const int G = aa.nq / aa.nkv;
        const size_t sm = attn_smem_bytes(G);
        const dim3 g3(aa.nkv, B, 2);
        switch (G) {
            case 1: launch_pdl(attn_decode_cluster_kernel<1>, g3, dim3(AT_THREADS), sm, s, aa); break;
            case 2: launch_pdl(attn_decode_cluster_kernel<2>, g3, dim3(AT_THREADS), sm, s, aa); break;
            case 3: launch_pdl(attn_decode_cluster_kernel<3>, g3, dim3(AT_THREADS), sm, s, aa); break;
            case 4: launch_pdl(attn_decode_cluster_kernel<4>, g3, dim3(AT_THREADS), sm, s, aa); break;
            case 6: launch_pdl(attn_decode_cluster_kernel<6>, g3, dim3(AT_THREADS), sm, s, aa); break;
            default: launch_pdl(attn_decode_cluster_kernel<8>, g3, dim3(AT_THREADS), sm, s, aa); break;
        }
    }

    void check_config() {
        const b2a_llama_config& c = cfg;
        B2A_CHECK(c.head_dim == HD, B2A_ERR_INVALID_INPUT, "llama: head_dim must be 128");
        // every GEMM's K is a whole number of 64-wide k-blocks (tc::BK); the fused step's 1024-thread first norm holds a row in
        // registers (RN_MAXV values per thread)
        B2A_CHECK(c.hidden_size > 0 && c.hidden_size % 64 == 0 && c.hidden_size <= RN_THREADS * RN_MAXV, B2A_ERR_INVALID_INPUT,
                  "llama: hidden_size must be a multiple of 64 (<= 8192)");
        B2A_CHECK(c.intermediate_size > 0 && c.intermediate_size % 64 == 0, B2A_ERR_INVALID_INPUT,
                  "llama: intermediate_size must be a multiple of 64");
        {
            const int g = c.num_key_value_heads > 0 && c.num_attention_heads % c.num_key_value_heads == 0
                              ? c.num_attention_heads / c.num_key_value_heads : 0;
            B2A_CHECK(gqa_supported(g), B2A_ERR_INVALID_INPUT,
                      "llama: unsupported GQA ratio (q heads per kv head must be 1, 2, 3, 4, 6 or 8)");
        }
        B2A_CHECK(c.max_batch >= 1 && c.max_batch <= 32, B2A_ERR_INVALID_INPUT, "llama: max_batch must be in 1..32");
        B2A_CHECK(c.max_context >= 8, B2A_ERR_INVALID_INPUT, "llama: max_context too small");
        require_device(device);
        B2A_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    }

    void alloc_state() {
        const b2a_llama_config& c = cfg;
        const int H = c.hidden_size, I = c.intermediate_size, nq = c.num_attention_heads, nkv = c.num_key_value_heads;
        const int NQ = nq * HD, NKV = nkv * HD;
        std::vector<float> fr = spec.linear_rope > 0.f ? linear_freqs(c, spec.linear_rope) : llama3_freqs(c);
        freqs.upload(fr.data(), fr.size());
        const size_t kv = (size_t)c.num_hidden_layers * c.max_batch * nkv * c.max_context * HD;
        kcache.alloc(kv);
        vcache.alloc(kv);
        B2A_CUDA(cudaMemset(kcache.p, 0, kv * sizeof(float)));
        B2A_CUDA(cudaMemset(vcache.p, 0, kv * sizeof(float)));
        max_width = tc::decode_width(c.max_batch);
        const int B = std::max(8, c.max_batch), R16 = 2 * max_width;
        x.alloc((size_t)B * H); y.alloc((size_t)B * H); qkv.alloc((size_t)B * (NQ + 2 * NKV));
        logits.alloc((size_t)B * c.vocab_size); probs.alloc((size_t)B * c.vocab_size);
        xn.alloc((size_t)R16 * H); attn.alloc((size_t)R16 * NQ); act.alloc((size_t)R16 * I);
        B2A_CUDA(cudaMemset(xn.p, 0, (size_t)R16 * H * sizeof(bf16)));
        B2A_CUDA(cudaMemset(attn.p, 0, (size_t)R16 * NQ * sizeof(bf16)));
        B2A_CUDA(cudaMemset(act.p, 0, (size_t)R16 * I * sizeof(bf16)));
        B2A_CUDA(cudaMemset(x.p, 0, (size_t)B * H * sizeof(float)));
        B2A_CUDA(cudaMemset(y.p, 0, (size_t)B * H * sizeof(float)));
        B2A_CUDA(cudaMemset(qkv.p, 0, (size_t)B * (NQ + 2 * NKV) * sizeof(float)));
        tokens.alloc(B); pos.alloc(B); recent.alloc(B * 64); recent_n.alloc(B); n_gen.alloc(B); done.alloc(B);
        n_active.alloc(1); forced.alloc(B);
        B2A_CUDA(cudaMemset(tokens.p, 0, B * sizeof(int)));
        B2A_CUDA(cudaMemset(pos.p, 0, B * sizeof(int)));
        h_flag.alloc(16);
        // process-wide kernel attributes: always the same (largest) value, several handles may coexist
        attn_cluster_attr<1>(); attn_cluster_attr<2>(); attn_cluster_attr<3>(); attn_cluster_attr<4>(); attn_cluster_attr<6>(); attn_cluster_attr<8>();
        tc::set_attributes();
        fused_parts = cdiv(H, tc::BM);          // <= 64: H <= 8192 (check_config)
        ss_a.alloc((size_t)64 * max_width); ss_b.alloc((size_t)64 * max_width);
        B2A_CUDA(cudaMemset(ss_a.p, 0, 64 * max_width * sizeof(float)));
        B2A_CUDA(cudaMemset(ss_b.p, 0, 64 * max_width * sizeof(float)));
        B2A_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
        pick_qkv_clusters();
        const char* envp = getenv("B2A_PREFILL");
        use_batched_prefill = !(envp && std::string(envp) == "step");
        for (auto& L : layers) {
            tm_qkv.push_back(tc::make_tmap_bf16(L.wqkv.p, NQ + 2 * NKV, H, tc::BM));
            tm_o.push_back(tc::make_tmap_bf16(L.wo.p, H, NQ, tc::BM));
            tm_gu.push_back(tc::make_tmap_bf16(L.wgu.p, 2 * I, H, tc::BM));
            {   // decode step: when 128-row tiles would leave more than a quarter of the SMs idle (Qwen3-TTS: 6144 rows = 48 tiles), use
                // as many m-tiles as SMs (rows per tile a multiple of 8).  Orpheus (128 tiles on 132 SMs) keeps 128.
                gu_tile_rows = pick_tile_rows(2 * I, num_sms);
                tm_gu_dec.push_back(tc::make_tmap_bf16(L.wgu.p, 2 * I, H, gu_tile_rows));
            }
            tm_down.push_back(tc::make_tmap_bf16(L.wdown.p, H, I, tc::BM));
        }
        lm_tile_rows = pick_tile_rows(c.vocab_size, num_sms);
        if (lm_head) tm_lm = tc::make_tmap_bf16(lm_head, c.vocab_size, H, lm_tile_rows);
        for (int w = 0; w < 3 && tc::DECODE_WIDTHS[w] <= max_width; ++w) {
            const int rows = 2 * tc::DECODE_WIDTHS[w];
            tmx_xn[w] = tc::make_tmap_bf16(xn.p, rows, H, rows);
            tmx_attn[w] = tc::make_tmap_bf16(attn.p, rows, NQ, rows);
            tmx_act[w] = tc::make_tmap_bf16(act.p, rows, I, rows);
        }
        B2A_CUDA(cudaDeviceSynchronize());
    }

    b2a_tts(int dev, const b2a_llama_config& c, const TensorTable& tt, b2a_snac* sn, const StackSpec& sp = StackSpec())
        : device(dev), cfg(c), snac(sn), spec(sp) {
        check_config();
        const int H = c.hidden_size, I = c.intermediate_size, nq = c.num_attention_heads, nkv = c.num_key_value_heads;
        const int NQ = nq * HD, NKV = nkv * HD;
        if (sp.has_embed) upload_bf16(tt, sp.prefix + "embed_tokens.weight", (int64_t)c.vocab_size * H, embed, 0, (size_t)c.vocab_size * H);
        if (sp.has_head) {
            if (sp.head.empty() && c.tie_word_embeddings) {
                B2A_CHECK(sp.has_embed, B2A_ERR_MODEL_NOT_INITIALIZED, "a tied head needs the embedding");
                lm_head = embed.p;   // embedTokens.asLinear (LlamaTTS.swift:563)
            } else {
                upload_bf16(tt, sp.head.empty() ? std::string("lm_head.weight") : sp.head, (int64_t)c.vocab_size * H, lm_head_w, 0, (size_t)c.vocab_size * H);
                lm_head = lm_head_w.p;
            }
        }
        layers.resize(c.num_hidden_layers);
        std::vector<bf16> tmp;
        for (int l = 0; l < c.num_hidden_layers; ++l) {
            const std::string p = sp.prefix + "layers." + std::to_string(l) + ".";
            if (sp.qk_norm) {
                std::vector<float> qn = tt.f32(p + "self_attn.q_norm.weight", HD), kn = tt.f32(p + "self_attn.k_norm.weight", HD);
                layers[l].qnorm.upload(qn.data(), HD);
                layers[l].knorm.upload(kn.data(), HD);
            }
            LayerW& L = layers[l];
            const size_t qkv_n = (size_t)(NQ + 2 * NKV) * H;
            upload_bf16(tt, p + "self_attn.q_proj.weight", (int64_t)NQ * H, L.wqkv, 0, qkv_n);
            upload_bf16(tt, p + "self_attn.k_proj.weight", (int64_t)NKV * H, L.wqkv, (size_t)NQ * H, qkv_n);
            upload_bf16(tt, p + "self_attn.v_proj.weight", (int64_t)NKV * H, L.wqkv, (size_t)(NQ + NKV) * H, qkv_n);
            upload_bf16(tt, p + "self_attn.o_proj.weight", (int64_t)H * NQ, L.wo, 0, (size_t)H * NQ);
            upload_bf16(tt, p + "mlp.down_proj.weight", (int64_t)H * I, L.wdown, 0, (size_t)H * I);
            // gate / up rows interleaved: row 2n = gate_n, row 2n+1 = up_n
            const b2a_tensor& tg = tt.get(p + "mlp.gate_proj.weight");
            const b2a_tensor& tu = tt.get(p + "mlp.up_proj.weight");
            B2A_CHECK(tg.dtype == tu.dtype && (tg.dtype == B2A_DTYPE_BF16 || tg.dtype == B2A_DTYPE_F32) &&
                          TensorTable::numel(tg) == (int64_t)I * H && TensorTable::numel(tu) == (int64_t)I * H,
                      B2A_ERR_MODEL_NOT_INITIALIZED, "bad gate/up projection: " + p);
            tmp.resize((size_t)2 * I * H);
            for (int n = 0; n < I; ++n) {
                if (tg.dtype == B2A_DTYPE_BF16) {
                    memcpy(&tmp[(size_t)(2 * n) * H], (const bf16*)tg.data + (size_t)n * H, H * sizeof(bf16));
                    memcpy(&tmp[(size_t)(2 * n + 1) * H], (const bf16*)tu.data + (size_t)n * H, H * sizeof(bf16));
                } else {
                    for (int k = 0; k < H; ++k) {
                        tmp[(size_t)(2 * n) * H + k] = __float2bfloat16_rn(((const float*)tg.data)[(size_t)n * H + k]);
                        tmp[(size_t)(2 * n + 1) * H + k] = __float2bfloat16_rn(((const float*)tu.data)[(size_t)n * H + k]);
                    }
                }
            }
            L.wgu.alloc(tmp.size());
            B2A_CUDA(cudaMemcpy(L.wgu.p, tmp.data(), tmp.size() * sizeof(bf16), cudaMemcpyHostToDevice));
            std::vector<float> g1 = tt.f32(p + "input_layernorm.weight", H), g2 = tt.f32(p + "post_attention_layernorm.weight", H);
            L.ln1.upload(g1.data(), H);
            L.ln2.upload(g2.data(), H);
        }
        std::vector<float> gf = tt.f32(sp.prefix + "norm.weight", H);
        final_ln.upload(gf.data(), H);
        alloc_state();
    }

    // random-init weights generated on the device (b2a_tts_create_random)
    b2a_tts(int dev, const b2a_llama_config& c, float std, unsigned long long seed, b2a_snac* sn, const StackSpec& sp = StackSpec())
        : device(dev), cfg(c), snac(sn), spec(sp) {
        check_config();
        const int H = c.hidden_size, I = c.intermediate_size, nq = c.num_attention_heads, nkv = c.num_key_value_heads;
        const int NQ = nq * HD, NKV = nkv * HD;
        unsigned long long sd = seed * 1000003ull + 17;
        auto rnd = [&](DBuf<bf16>& d, size_t n) {
            d.alloc(n);
            random_bf16_kernel<<<132 * 8, 256, 0, stream>>>(d.p, (long long)n, std, sd++);
            count_launch();
        };
        auto ones = [&](DBuf<float>& d, int n) {
            d.alloc(n);
            fill_f32_kernel<<<cdiv(n, 256), 256, 0, stream>>>(d.p, n, 1.0f);
            count_launch();
        };
        if (sp.has_embed) rnd(embed, (size_t)c.vocab_size * H);
        if (sp.has_head) {
            if (sp.head.empty() && c.tie_word_embeddings && sp.has_embed) lm_head = embed.p;
            else { rnd(lm_head_w, (size_t)c.vocab_size * H); lm_head = lm_head_w.p; }
        }
        layers.resize(c.num_hidden_layers);
        for (auto& L : layers) {
            if (sp.qk_norm) { ones(L.qnorm, HD); ones(L.knorm, HD); }
            rnd(L.wqkv, (size_t)(NQ + 2 * NKV) * H);
            rnd(L.wo, (size_t)H * NQ);
            rnd(L.wgu, (size_t)2 * I * H);
            rnd(L.wdown, (size_t)H * I);
            ones(L.ln1, H);
            ones(L.ln2, H);
        }
        ones(final_ln, H);
        B2A_CUDA(cudaStreamSynchronize(stream));
        B2A_CUDA(cudaGetLastError());
        alloc_state();
    }

    int rows_cap() const { return std::max(8, cfg.max_batch); }   // rows of the per-row state buffers
    // q|k|v as clusters when they fit in one wave at a width's footprint; otherwise the stream-K GEMM, with its workspace (slots of
    // [2 max_width, 128])
    void pick_qkv_clusters() {
        const int mt = cdiv((cfg.num_attention_heads + 2 * cfg.num_key_value_heads) * HD, tc::BM), kb = cfg.hidden_size / tc::BK;
        bool stream_k = false;
        for (int w = 0; w < 3 && tc::DECODE_WIDTHS[w] <= max_width; ++w) {
            qkv_cluster[w] = pick_qkv_cluster(mt, kb, num_sms, &qkv_sk_ctas, tc::DECODE_WIDTHS[w], SPLITK_STAGES[w]);
            stream_k |= qkv_cluster[w] == 0;
        }
        if (stream_k && !sk_cnt.p) {
            sk_slots = tc::stream_k_slots(mt, kb, qkv_sk_ctas);
            sk_ws.alloc((size_t)mt * sk_slots * 2 * max_width * tc::BM);
            sk_cnt.alloc(mt);
            B2A_CUDA(cudaMemset(sk_cnt.p, 0, (size_t)mt * sizeof(unsigned)));
        }
    }

    enum { OP_QKV, OP_GU, OP_LM };
    // D[tokens, M] = X[tokens, K] * W[M, K]^T on the wgmma path (hi/lo activations, BN = 2 width)
    void tc_gemm(const CUtensorMap& tmW, const CUtensorMap& tmX, int op, float* yout, bf16* actout, int B, int M, int K,
                 cudaStream_t s, const float* rstd_ss = nullptr, const float* bias = nullptr) {
        tc::Args a{};
        a.bias = bias;
        a.rstd_ss = rstd_ss; a.rstd_parts = fused_parts; a.rstd_inv_h = 1.0f / (float)cfg.hidden_size; a.rstd_eps = cfg.rms_norm_eps;
        a.out_f32 = yout; a.out_bf16 = actout; a.M = M; a.N = B; a.K = K;
        a.m_tiles = cdiv(M, tc::BM); a.k_blocks = K / tc::BK;
        a.stages = GEMM_STAGES[wi];
        a.hilo = 1;
        int ctas = num_sms;
        if (op == OP_GU) {
            a.ldo = M / 2; a.epi_full = tc::EPI_SWIGLU; a.epi_partial = -1; a.lo_rows = width;
            a.tile_rows = gu_tile_rows; a.m_tiles = cdiv(M, gu_tile_rows);      // tmW is tm_gu_dec[layer]
            ctas = std::min(num_sms, a.m_tiles);
        } else if (op == OP_LM) {
            a.ldo = M; a.epi_full = tc::EPI_STORE; a.epi_partial = -1; a.lo_rows = 0;
            a.tile_rows = head_rows_now > 0 ? head_rows_now : lm_tile_rows; a.m_tiles = cdiv(M, a.tile_rows);
            ctas = std::min(num_sms, a.m_tiles);
        } else {   // OP_QKV when its clusters do not fit (qkv_gemm): stream-K, partial tiles summed in slot order and stored
            a.ldo = M; a.epi_full = tc::EPI_STORE; a.epi_partial = tc::EPI_PARTIAL; a.lo_rows = 0;
            ctas = (int)std::min<long long>(num_sms, (long long)a.m_tiles * a.k_blocks);
            a.part_ws = sk_ws.p; a.part_cnt = sk_cnt.p; a.part_slots = sk_slots;
        }
        if (width == 8) tc::launch<16>(tmW, tmX, a, ctas, 1, s);
        else if (width == 16) tc::launch<32>(tmW, tmX, a, ctas, 1, s, true);
        else tc::launch<64>(tmW, tmX, a, ctas, 1, s);
    }

    // o_proj / down_proj as a cluster split-K GEMM with the residual add and the next norm fused into the leader's epilogue
    void splitk_gemm(const CUtensorMap& tmW, const CUtensorMap& tmX, int M, int K, const float* gain, float* ss, int B, cudaStream_t s) {
        tc::SplitArgs a{};
        a.M = M; a.N = B; a.K = K; a.k_blocks = K / tc::BK; a.stages = SPLITK_STAGES[wi];
        a.h = x.p; a.gain = gain; a.xn = xn.p; a.ss = ss;
        a.rstd_ss = nullptr; a.rstd_parts = 0; a.rstd_inv_h = 0.f; a.rstd_eps = 0.f;
        launch_splitk(tmW, tmX, a, cdiv(M, tc::BM), std::max(1, std::min(fused_cluster, a.k_blocks)), s);
    }
    void launch_splitk(const CUtensorMap& tmW, const CUtensorMap& tmX, const tc::SplitArgs& a, int m_tiles, int cluster, cudaStream_t s) {
        if (width == 8) tc::launch_splitk<8>(tmW, tmX, a, m_tiles, cluster, s);
        else if (width == 16) tc::launch_splitk<16>(tmW, tmX, a, m_tiles, cluster, s);
        else tc::launch_splitk<32>(tmW, tmX, a, m_tiles, cluster, s);
    }
    // q|k|v projection of the fused step: q|k|v[t] = rstd[t] * Wqkv xn[t] (the input norm's scale from ss_b), stored, in clusters of
    // qkv_cluster CTAs that compute exactly what the stream-K GEMM computes (tc::SplitArgs::sk_ctas); that GEMM itself when the
    // clusters do not fit in one wave
    void qkv_gemm(int layer, int B, cudaStream_t s) {
        const int H = cfg.hidden_size, M = (cfg.num_attention_heads + 2 * cfg.num_key_value_heads) * HD;
        if (qkv_cluster[wi] < 1) { tc_gemm(tm_qkv[layer], tmx_xn[wi], OP_QKV, qkv.p, nullptr, B, M, H, s, ss_b.p); return; }
        tc::SplitArgs a{};
        a.M = M; a.N = B; a.K = H; a.k_blocks = H / tc::BK; a.stages = SPLITK_STAGES[wi]; a.sk_ctas = qkv_sk_ctas;
        a.out = qkv.p;
        a.rstd_ss = ss_b.p; a.rstd_parts = fused_parts; a.rstd_inv_h = 1.0f / (float)H; a.rstd_eps = cfg.rms_norm_eps;
        launch_splitk(tm_qkv[layer], tmx_xn[wi], a, cdiv(M, tc::BM), qkv_cluster[wi], s);
    }
    // The q|k|v split-K launch cuts each tile's k-blocks where the stream-K GEMM over *sk_ctas = min(SMs, units) CTAs cuts them (so
    // its output is bit-identical), one CTA per piece: the cluster size is the most pieces of any tile (tc::stream_k_slots).  It is
    // used when that is at most 8 and all m_tiles clusters are resident at once (cudaOccupancyMaxActiveClusters at the launch's own
    // shared-memory footprint at this width and ring depth); 0 otherwise (the stream-K GEMM runs).  Needs tc::set_attributes().
    static int pick_qkv_cluster(int m_tiles, int k_blocks, int sms, int* sk_ctas, int width = 8, int stages = SPLITK_STAGES[0]) {
        *sk_ctas = (int)std::min<long long>(sms, (long long)m_tiles * k_blocks);
        const int c = tc::stream_k_slots(m_tiles, k_blocks, *sk_ctas);
        if (c > tc::SPLIT_MAX_CLUSTER) return 0;
        return m_tiles <= splitk_active_clusters(width, c, splitk_bytes(width, stages, c)) ? c : 0;
    }
    static size_t splitk_bytes(int width, int stages, int cluster) {
        return width == 8 ? tc::SmemSplit<8>::bytes(stages, cluster) : width == 16 ? tc::SmemSplit<16>::bytes(stages, cluster)
                                                                                   : tc::SmemSplit<32>::bytes(stages, cluster);
    }
    static size_t gemm_bytes(int width, int stages) {
        return width == 8 ? tc::Smem<16>::bytes(stages) : width == 16 ? tc::Smem<32>::bytes(stages) : tc::Smem<64>::bytes(stages);
    }
    static int splitk_active_clusters(int width, int cluster, size_t bytes) {
        return width == 8 ? tc::splitk_active_clusters<8>(cluster, bytes) : width == 16 ? tc::splitk_active_clusters<16>(cluster, bytes)
                                                                                        : tc::splitk_active_clusters<32>(cluster, bytes);
    }
    // The fused-norm step: embed -> raw norm -> L x [qkv gemm (rstd in the epilogue) -> attention -> o split-K (+ residual, norm 2)
    // -> gate/up gemm (rstd, SwiGLU) -> down split-K (+ residual, next layer's norm 1 / the final norm)].  Leaves the residual
    // stream in x, xn = hi/lo of x * final_norm_gain and its sums of squares in ss_b: the lm head GEMM applies rstd itself.
    void run_layers(int B, cudaStream_t s) {
        const int H = cfg.hidden_size, I = cfg.intermediate_size, nq = cfg.num_attention_heads, nkv = cfg.num_key_value_heads;
        const int NQ = nq * HD, L = cfg.num_hidden_layers;
        if (x_ext) launch_pdl(ext_embed_kernel, dim3(B), dim3(256), 0, s, x_ext, x.p, y.p, H);
        else launch_pdl(embed_kernel, dim3(B), dim3(256), 0, s, tokens.p, embed.p, x.p, y.p, H, cfg.vocab_size);
        trace_x(0, B, s);
        launch_pdl(add_rmsnorm_kernel, dim3(B), dim3(RN_THREADS), 0, s, x.p, (float*)nullptr, layers[0].ln1.p, xn.p, H, cfg.rms_norm_eps,
                   width, ss_b.p, fused_parts);
        const size_t kv_layer = (size_t)cfg.max_batch * nkv * cfg.max_context * HD;
        for (int l = 0; l < L; ++l) {
            LayerW& Lw = layers[l];
            qkv_gemm(l, B, s);
            AttnArgs aa{qkv.p, pos.p, freqs.p, kcache.p + l * kv_layer, vcache.p + l * kv_layer, attn.p, nq, nkv, cfg.max_context,
                        1.0f / sqrtf((float)HD), spec.qk_norm ? Lw.qnorm.p : nullptr, spec.qk_norm ? Lw.knorm.p : nullptr, cfg.rms_norm_eps,
                        width};
            attn_launch(aa, B, s);
            splitk_gemm(tm_o[l], tmx_attn[wi], H, NQ, Lw.ln2.p, ss_a.p, B, s);
            trace_x(2 * l + 1, B, s);
            tc_gemm(tm_gu_dec[l], tmx_xn[wi], OP_GU, nullptr, act.p, B, 2 * I, H, s, ss_a.p);
            splitk_gemm(tm_down[l], tmx_act[wi], H, I, l + 1 < L ? layers[l + 1].ln1.p : final_ln.p, ss_b.p, B, s);
            trace_x(2 * l + 2, B, s);
        }
    }
    int launches_layers() const { return 2 + cfg.num_hidden_layers * 5; }
    // b2a_tts_debug_trace: the residual stream x [B, H] into slot i of the record, i.e. the input of the i-th RMSNorm.  Tracing is
    // for eager forwards (b2a_tts_forward_logits); tts_generate_impl turns it off before it captures its graphs
    void trace_x(int i, int B, cudaStream_t s) {
        if (trace_on)
            B2A_CUDA(cudaMemcpyAsync(trace.p + (size_t)i * rows_cap() * cfg.hidden_size, x.p, (size_t)B * cfg.hidden_size * sizeof(float),
                                     cudaMemcpyDeviceToDevice, s));
    }

    // x, xn (un-normalised) and ss_b are final after run_layers: only row N1 and Soprano's capture need the fp32 normalised hidden state
    void run_final_norm(int B, cudaStream_t s, bool capture) {
        if (normed_out)
            launch_pdl(finalize_norm_kernel, dim3(B), dim3(256), 0, s, (const float*)x.p, (const float*)final_ln.p, (const float*)ss_b.p, fused_parts,
                       normed_out, cfg.hidden_size, cfg.rms_norm_eps, (const int*)nullptr, (int*)nullptr, 0, width);
        if (capture)
            launch_pdl(finalize_norm_kernel, dim3(B), dim3(256), 0, s, (const float*)x.p, (const float*)final_ln.p, (const float*)ss_b.p, fused_parts,
                       hidden.p, cfg.hidden_size, cfg.rms_norm_eps, (const int*)n_gen.p, n_cap.p, hidden_slots, width);
    }
    // capture: Soprano's generate (hidden states into `hidden`); forward_logits never captures
    void run_lm_head(int B, cudaStream_t s, bool capture = false) {
        run_final_norm(B, s, capture);
        tc_gemm(tm_lm, tmx_xn[wi], OP_LM, logits.p, nullptr, B, cfg.vocab_size, cfg.hidden_size, s, ss_b.p);
    }
    // after prefill_batched's gather_last (x, y hold the last position un-added): the stand-alone norm + plain GEMM.  Soprano runs the
    // decode step's tail instead (raw norm, then capture + GEMM with rstd), so slot 0 is computed as every later slot is.
    void run_lm_head_after_prefill(int B, cudaStream_t s) {
        if (vocos) {
            launch_pdl(add_rmsnorm_kernel, dim3(B), dim3(RN_THREADS), 0, s, x.p, y.p, final_ln.p, xn.p, cfg.hidden_size, cfg.rms_norm_eps,
                       width, ss_b.p, fused_parts);
            run_lm_head(B, s, true);
            return;
        }
        launch_pdl(add_rmsnorm_kernel, dim3(B), dim3(RN_THREADS), 0, s, x.p, y.p, final_ln.p, xn.p, cfg.hidden_size, cfg.rms_norm_eps,
                   width, (float*)nullptr, 0);
        tc_gemm(tm_lm, tmx_xn[wi], OP_LM, logits.p, nullptr, B, cfg.vocab_size, cfg.hidden_size, s);
    }
    // a head the caller owns (row N1: the code predictor's 15 lm heads, and the talker's small_to_mtp_projection with its bias):
    // logits_out[b, :M] = W[M, H] * normed hidden (+ bias), tmW a map of W
    void run_head(const CUtensorMap& tmW, int M, float* logits_out, int B, cudaStream_t s, int tile_rows = 0, const float* bias = nullptr) {
        head_rows_now = tile_rows;              // tmW's box rows (0: this stack's own lm_tile_rows)
        tc_gemm(tmW, tmx_xn[wi], OP_LM, logits_out, nullptr, B, M, cfg.hidden_size, s, ss_b.p, bias);
        head_rows_now = 0;
    }
    // logits are [max_batch, V] row-major.

    static void pattn_attr() {
        for (auto k : {prefill_attn_kernel<1>, prefill_attn_kernel<2>, prefill_attn_kernel<3>, prefill_attn_kernel<4>,
                       prefill_attn_kernel<6>, prefill_attn_kernel<8>})
            B2A_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PA_SMEM_MAX));
    }
    // the SIMT prompt attention of B rows of pa.L positions (the caller has checked simt_prompt_attn(pa.L, G))
    static void pattn_launch(const PrefillAttnArgs& pa, int B, cudaStream_t s) {
        const int G = pa.nq / pa.nkv;
        const dim3 grid(pa.nkv, B, cdiv(pa.L, PA_QT));
        const size_t sm = pattn_smem(pa.L, G);
        switch (G) {
            case 1: prefill_attn_kernel<1><<<grid, PA_THREADS, sm, s>>>(pa); break;
            case 2: prefill_attn_kernel<2><<<grid, PA_THREADS, sm, s>>>(pa); break;
            case 3: prefill_attn_kernel<3><<<grid, PA_THREADS, sm, s>>>(pa); break;
            case 4: prefill_attn_kernel<4><<<grid, PA_THREADS, sm, s>>>(pa); break;
            case 6: prefill_attn_kernel<6><<<grid, PA_THREADS, sm, s>>>(pa); break;
            default: prefill_attn_kernel<8><<<grid, PA_THREADS, sm, s>>>(pa); break;
        }
        count_launch();
    }
    // a stack whose inputs are embeddings (the Qwen3-TTS talker and code predictor) replays the decode step per prompt position
    bool can_batch_prefill(int L) const {
        return use_batched_prefill && spec.has_embed && L >= 2 && L <= cfg.max_context;
    }

    // D[T, M] = X[T, K] W^T for all prompt tokens: 128-column tiles (64 tokens as hi/lo), CTAs own whole tiles
    void pf_gemm(const CUtensorMap& tmW, const CUtensorMap& tmX, int epi, float* yout, bf16* actout, int T, int M, int K,
                 cudaStream_t s) {
        tc::Args a{};
        a.out_f32 = yout; a.out_bf16 = actout; a.M = M; a.N = T; a.K = K;
        a.m_tiles = cdiv(M, tc::BM); a.k_blocks = K / tc::BK;
        a.stages = tc::Smem<128>::max_stages(); a.hilo = 1; a.epi_full = epi; a.epi_partial = -1;
        a.ldo = epi == tc::EPI_SWIGLU ? M / 2 : M;
        a.lo_rows = epi == tc::EPI_SWIGLU ? PF_HALF : 0;
        const int n_tiles = cdiv(T, PF_HALF);
        const int ctas = std::max(1, std::min(a.m_tiles, num_sms / n_tiles));
        tc::launch<128>(tmW, tmX, a, ctas, n_tiles, s);
    }

    // Prompt pass over all B*L tokens; leaves K/V for positions 0..L-1 in the cache and the last position's
    // residual stream in the decode buffers (x, y), pos[b] = L-1: the caller then runs lm head + sampler.
    void prefill_batched(int B, int L, cudaStream_t s) {
        const int H = cfg.hidden_size, I = cfg.intermediate_size, nq = cfg.num_attention_heads, nkv = cfg.num_key_value_heads;
        const int NQ = nq * HD, QKV_N = (nq + 2 * nkv) * HD, T = B * L, G = nq / nkv;
        const int n_tiles = cdiv(T, PF_HALF), Tp = n_tiles * PF_HALF;
        if (Tp > pf_tokens_cap) {
            xp.alloc((size_t)Tp * H); yp.alloc((size_t)Tp * H); qkvp.alloc((size_t)Tp * QKV_N);
            xnp.alloc((size_t)2 * Tp * H); attnp.alloc((size_t)2 * Tp * NQ); actp.alloc((size_t)2 * Tp * I);
            pf_tokens_cap = Tp;
            tmp_xn = tc::make_tmap_bf16(xnp.p, 2 * Tp, H, 128);
            tmp_attn = tc::make_tmap_bf16(attnp.p, 2 * Tp, NQ, 128);
            tmp_act = tc::make_tmap_bf16(actp.p, 2 * Tp, I, 128);
            pattn_attr();
        }
        rope_tab.alloc((size_t)cfg.max_context * (HD / 2));
        const bool simt_attn = simt_prompt_attn(L, G);
        if (!simt_attn) pfa_ops.prepare(B, L, nq, nkv);
        // padding tokens of the last tile must read as zero (no kernel writes them): its hi rows T % 64 .. 63 and the lo rows below
        if (const int r0 = T % PF_HALF) {
            const size_t row0 = (size_t)(n_tiles - 1) * 2 * PF_HALF + r0;
            auto zero = [&](bf16* p, int cols) {
                B2A_CUDA(cudaMemset2DAsync(p + row0 * cols, (size_t)PF_HALF * cols * sizeof(bf16), 0,
                                           (size_t)(PF_HALF - r0) * cols * sizeof(bf16), 2, s));
            };
            zero(xnp.p, H); zero(attnp.p, NQ); zero(actp.p, I);
        }
        embed_rows_kernel<<<T, 256, 0, s>>>(ids.p, embed.p, xp.p, H, cfg.vocab_size);
        rope_table_kernel<<<cdiv(L * (HD / 2), 256), 256, 0, s>>>(freqs.p, rope_tab.p, L);
        count_launch(2);
        const size_t kv_layer = (size_t)cfg.max_batch * nkv * cfg.max_context * HD;
        for (int l = 0; l < cfg.num_hidden_layers; ++l) {
            LayerW& Lw = layers[l];
            const float* qn = spec.qk_norm ? Lw.qnorm.p : nullptr;
            const float* kn = spec.qk_norm ? Lw.knorm.p : nullptr;
            launch_pdl(add_rmsnorm_kernel, dim3(T), dim3(RN_THREADS), 0, s, xp.p, l == 0 ? (float*)nullptr : yp.p, Lw.ln1.p, xnp.p, H,
                       cfg.rms_norm_eps, PF_HALF, (float*)nullptr, 0);
            pf_gemm(tm_qkv[l], tmp_xn, tc::EPI_STORE, qkvp.p, nullptr, T, QKV_N, H, s);
            if (simt_attn) {
                PrefillAttnArgs pa{qkvp.p, rope_tab.p, kcache.p + l * kv_layer, vcache.p + l * kv_layer, attnp.p, nq, nkv,
                                   cfg.max_context, L, 1.0f / sqrtf((float)HD), qn, kn, cfg.rms_norm_eps};
                pattn_launch(pa, B, s);
            } else {
                pfa_ops.run(qkvp.p, rope_tab.p, kcache.p + l * kv_layer, vcache.p + l * kv_layer, attnp.p, L, cfg.max_context, s, qn, kn,
                            cfg.rms_norm_eps);
            }
            pf_gemm(tm_o[l], tmp_attn, tc::EPI_STORE, yp.p, nullptr, T, H, NQ, s);
            launch_pdl(add_rmsnorm_kernel, dim3(T), dim3(RN_THREADS), 0, s, xp.p, yp.p, Lw.ln2.p, xnp.p, H, cfg.rms_norm_eps, PF_HALF,
                       (float*)nullptr, 0);
            pf_gemm(tm_gu[l], tmp_xn, tc::EPI_SWIGLU, nullptr, actp.p, T, 2 * I, H, s);
            pf_gemm(tm_down[l], tmp_act, tc::EPI_STORE, yp.p, nullptr, T, H, I, s);
        }
        gather_last_kernel<<<B, 256, 0, s>>>(xp.p, yp.p, x.p, y.p, pos.p, L, H);
        count_launch();
        B2A_CUDA(cudaGetLastError());
    }

    // a call of B rows runs the step at width tc::decode_width(B): 8, 16 or 32 token rows per GEMM tile
    void set_batch(int B) {
        width = tc::decode_width(B);
        wi = tc::decode_width_index(width);
        nb_pad = B <= 1 ? 1 : B <= 2 ? 2 : B <= 4 ? 4 : width;
    }

    void drop_graphs() {
        if (g_step) { cudaGraphExecDestroy(g_step); g_step = nullptr; }
        if (g_prefill) { cudaGraphExecDestroy(g_prefill); g_prefill = nullptr; }
    }

    static bool same_args(const SampleArgs& a, const SampleArgs& b) {
        return a.V == b.V && a.R == b.R && a.max_tokens == b.max_tokens && a.temperature == b.temperature &&
               a.top_p == b.top_p && a.rep_penalty == b.rep_penalty && a.seed == b.seed && a.mask_eos == b.mask_eos &&
               a.stop_token == b.stop_token && a.out_tokens == b.out_tokens && a.soprano == b.soprano;
    }

    void capture(int B, const SampleArgs& sa, int L) {
        if (g_step && g_nb == B && same_args(sa, g_args) && g_L == L && g_hidden == hidden.p) return;
        drop_graphs();
        cudaGraph_t g;
        B2A_CUDA(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
        run_layers(B, stream);
        run_lm_head(B, stream, sa.soprano != 0);
        launch_pdl(sample_kernel, dim3(B * SM_CLUSTER), dim3(SM_THREADS), 0, stream, sa);
        B2A_CUDA(cudaStreamEndCapture(stream, &g));
        B2A_CUDA(cudaGraphInstantiate(&g_step, g, 0));
        cudaGraphDestroy(g);
        B2A_CUDA(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
        run_layers(B, stream);
        launch_pdl(prefill_advance_kernel, dim3(1), dim3(32), 0, stream, ids.p, L, tokens.p, pos.p, B);
        B2A_CUDA(cudaStreamEndCapture(stream, &g));
        B2A_CUDA(cudaGraphInstantiate(&g_prefill, g, 0));
        cudaGraphDestroy(g);
        g_nb = B; g_args = sa; g_L = L; g_hidden = hidden.p;
        launches_step = launches_layers() + 1 + 1 + (sa.soprano ? 1 : 0);
        launches_prefill = launches_layers() + 1;
    }
    int g_L = 0, launches_step = 0, launches_prefill = 0;
};

// ------------------------------------------------------------------------------------------------
// host-side token plumbing (ints; the reference does these on the host too)
// ------------------------------------------------------------------------------------------------
static std::vector<int> parse_row(const TokenLayout& tl, const int* row, int n, int crop_after) {
    // LlamaTTS.swift:400-431 / Qwen3.swift:346-357 for one row: crop, drop the stop token, trim to a multiple of 7, subtract the audio offset
    std::vector<int> r;
    for (int j = crop_after + 1; j < n; ++j)
        if (row[j] != tl.end_of_speech) r.push_back(row[j]);
    r.resize((r.size() / 7) * 7);
    for (auto& t : r) t -= tl.audio_offset;
    return r;
}

// where a row's codes start (parse_row's crop_after): its last start-of-speech; failing that, with ai_fallback, just before the first audio
// token after its last start-of-AI (Qwen3.swift:336-344); -1 keeps the whole row
static int codes_start(const TokenLayout& tl, const int* row, int n) {
    int last = -1, soa = -1;
    for (int j = 0; j < n; ++j) {
        if (row[j] == tl.start_of_speech) last = j;
        if (row[j] == tl.start_of_ai) soa = j;
    }
    if (last < 0 && tl.ai_fallback && soa >= 0)
        for (int j = soa + 1; j < n; ++j)
            if (row[j] >= tl.audio_offset) { last = j - 1; break; }
    return last;
}

static void deinterleave(const int* cl, int n, std::vector<int>& l1, std::vector<int>& l2, std::vector<int>& l3) {
    // llamaDecodeAudioFromCodes, LlamaTTS.swift:46-58
    const int groups = (n + 1) / 7;
    for (int i = 0; i < groups; ++i) {
        const int b = 7 * i;
        l1.push_back(cl[b]);
        l2.push_back(cl[b + 1] - 4096);
        l3.push_back(cl[b + 2] - 2 * 4096);
        l3.push_back(cl[b + 3] - 3 * 4096);
        l2.push_back(cl[b + 4] - 4 * 4096);
        l3.push_back(cl[b + 5] - 5 * 4096);
        l3.push_back(cl[b + 6] - 6 * 4096);
    }
}

static double now_s() {
    return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// Samples of a Soprano waveform of n hidden states: the decoder's output (upscale (n - 1) hop, or the untrimmed n_fft of a one-frame
// OLA for n = 1, SopranoDecoder.swift:191-196), cut to its last (n - 1) token_size samples when that is positive (Soprano.swift:664-671).
// *offset receives the first kept sample.
static int64_t soprano_wave_len(const b2a_tts* h, int n, int64_t* offset) {
    const int64_t total = b2a_vocos_upsampled_length(h->vocos, n, h->upscale);
    const int64_t cut = (int64_t)(n - 1) * h->token_size;
    const int64_t keep = cut > 0 ? std::min(cut, total) : total;
    if (offset) *offset = total - keep;
    return keep;
}

// SopranoDecoder on rows of d_states (row r at d_states + r * row_stride, n[r] states of H floats): rows with equal counts share one
// Vocos pass, so a batch decodes exactly as its rows would one by one (no row is padded: the ConvNeXt convolutions would see it).
// wave_out [B, wave_cap] receives each row's cut waveform, wave_len[B] its length.
static void soprano_decode(b2a_tts* h, const float* d_states, int64_t row_stride, const std::vector<int>& n, float* wave_out,
                           bool wave_on_device, int64_t wave_cap, int64_t* wave_len, cudaStream_t s) {
    const int B = (int)n.size();
    std::vector<bool> used(B, false);
    for (int i = 0; i < B; ++i) {
        if (used[i]) continue;
        std::vector<int> grp;
        for (int j = i; j < B; ++j)
            if (!used[j] && n[j] == n[i]) { grp.push_back(j); used[j] = true; }
        int64_t off = 0;
        const int64_t keep = soprano_wave_len(h, n[i], &off), total = off + keep;
        B2A_CHECK(keep <= wave_cap, B2A_ERR_INVALID_INPUT, "soprano: wave buffer too small");
        h->d_rows.upload(grp.data(), grp.size(), s);
        h->d_wave.alloc((size_t)grp.size() * total);
        const int32_t st = b2a_vocos_decode_upsampled_dev(h->vocos, d_states, row_stride, h->d_rows.p, (int32_t)grp.size(), n[i], h->upscale,
                                                          h->d_wave.p, s);
        B2A_CHECK(st == B2A_OK, B2A_ERR_AUDIO_DECODING_FAILED, std::string("Soprano decode failed: ") + b2a_last_error());
        for (size_t k = 0; k < grp.size(); ++k) {
            B2A_CUDA(cudaMemcpyAsync(wave_out + (size_t)grp[k] * wave_cap, h->d_wave.p + k * total + off, keep * sizeof(float),
                                     wave_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, s));
            if (wave_len) wave_len[grp[k]] = keep;
        }
        B2A_CUDA(cudaStreamSynchronize(s));   // grp (the uploaded row list) and d_wave are reused by the next group
    }
}

// shared body of b2a_tts_generate / _dev.  ids_on_device: input ids pointer is a device pointer.
// chunked audio emission during generation (row N2): every `frames_per_chunk` new 7-token frames of a row are decoded with
// `left_context` already-emitted frames in front (the codec is convolutional: the context absorbs the left edge) and handed to
// on_audio; the samples of the context frames are dropped.
struct StreamSpec {
    int frames_per_chunk = 0;     // 0: no streaming
    int left_context = 0;
    b2a_audio_cb on_audio = nullptr;
};

static void tts_generate_impl(b2a_tts* h, const int32_t* input_ids, bool ids_on_device, int32_t B, int32_t L,
                              const b2a_gen_params* gp, int32_t* tokens_out, int32_t* n_tokens_out, float* wave_out,
                              bool wave_on_device, int64_t wave_cap, int64_t* wave_len, b2a_gen_info* info,
                              b2a_token_cb on_token, void* user, const StreamSpec& ss = StreamSpec()) {
    B2A_CHECK(h && input_ids && gp, B2A_ERR_INVALID_INPUT, "tts generate: null argument");
    B2A_CHECK(B >= 1 && B <= h->cfg.max_batch, B2A_ERR_INVALID_INPUT, "tts generate: batch exceeds max_batch");
    B2A_CHECK(L >= 1, B2A_ERR_INVALID_INPUT, "tts generate: empty prompt");
    B2A_CHECK(gp->max_tokens >= 1, B2A_ERR_INVALID_INPUT, "tts generate: max_tokens must be positive");
    B2A_CHECK(L + gp->max_tokens <= h->cfg.max_context, B2A_ERR_INVALID_INPUT, "tts generate: prompt + max_tokens exceeds max_context");
    B2A_CHECK(gp->repetition_context_size >= 0 && gp->repetition_context_size <= 64, B2A_ERR_INVALID_INPUT,
              "tts generate: repetition_context_size must be in 0..64");
    B2A_CHECK(gp->temperature >= 0.f && gp->top_p > 0.f, B2A_ERR_INVALID_INPUT, "tts generate: bad sampling parameters");
    const bool soprano = h->vocos != nullptr;
    // Soprano feeds its last generated token forward once more (its hidden state is audio): one more cache position
    if (soprano) B2A_CHECK(L + gp->max_tokens + 1 <= h->cfg.max_context, B2A_ERR_INVALID_INPUT, "soprano generate: prompt + max_tokens + 1 exceeds max_context");
    if (soprano) B2A_CHECK(ss.frames_per_chunk == 0, B2A_ERR_INVALID_INPUT, "soprano generate: audio is decoded once per call, not in chunks");
    if (wave_out && !soprano) B2A_CHECK(h->snac, B2A_ERR_MODEL_NOT_INITIALIZED, "SNAC model not loaded");   // LlamaTTS.swift:672-674
    B2A_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    h->cancel.store(0);
    h->set_batch(B);
    if (h->trace_on) { h->trace_on = false; h->drop_graphs(); }
    const int MT = gp->max_tokens, R = std::max(1, gp->repetition_context_size);
    h->ids.alloc((size_t)B * L);
    h->out_tokens.alloc((size_t)B * MT);
    h->recent.alloc((size_t)h->rows_cap() * R);
    B2A_CUDA(cudaMemcpyAsync(h->ids.p, input_ids, (size_t)B * L * sizeof(int),
                             ids_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
    SampleArgs sa{};
    sa.logits = h->logits.p; sa.probs = h->probs.p; sa.tokens = h->tokens.p; sa.pos = h->pos.p; sa.recent = h->recent.p;
    sa.recent_n = h->recent_n.p; sa.out_tokens = h->out_tokens.p; sa.n_gen = h->n_gen.p; sa.done = h->done.p;
    sa.n_active = h->n_active.p; sa.forced = nullptr; sa.V = h->cfg.vocab_size; sa.R = gp->repetition_context_size > 0 ? R : 0;
    sa.max_tokens = MT; sa.temperature = gp->temperature; sa.top_p = gp->top_p;
    sa.rep_penalty = gp->repetition_context_size > 0 ? gp->repetition_penalty : 1.0f;
    sa.seed = gp->seed; sa.mask_eos = h->bench_mask_eos; sa.stop_token = h->tok.end_of_speech;
    sa.soprano = soprano ? 1 : 0;
    if (sa.R == 0) { sa.R = 1; }
    if (soprano) {
        h->hidden_slots = MT + 1; h->hidden_rows = B;
        h->hidden.alloc((size_t)B * h->hidden_slots * h->cfg.hidden_size);
        h->n_cap.alloc(h->rows_cap());
    }
    h->capture(B, sa, L);

    const double t0 = now_s();
    // Soprano's penalty sees generated tokens only (Soprano.swift:831,868): its ring starts empty
    init_rows_kernel<<<1, 32, 0, s>>>(h->ids.p, L, B, gp->repetition_context_size > 0 && !soprano ? R : 0, h->tokens.p, h->pos.p, h->recent.p,
                                      h->recent_n.p, h->n_gen.p, h->done.p, h->n_active.p, 0);
    count_launch();
    if (soprano) B2A_CUDA(cudaMemsetAsync(h->n_cap.p, 0, h->rows_cap() * sizeof(int), s));
    // prefill.  Batched: every prompt token through each layer at once (wgmma GEMMs, 64 tokens per tile), then
    // lm head + sampler on the last position.  Fallback (B2A_PREFILL=step, q/k norm): replay the decode
    // step per position -- positions 0..L-2 need no logits, position L-1 runs the full step.
    int steps = 0;
    if (h->can_batch_prefill(L)) {
        h->prefill_batched(B, L, s);
        h->run_lm_head_after_prefill(B, s);
        launch_pdl(sample_kernel, dim3(B * SM_CLUSTER), dim3(SM_THREADS), 0, s, sa);
        steps = 1;
    } else {
        for (int p = 0; p < L - 1; ++p) {
            B2A_CUDA(cudaGraphLaunch(h->g_prefill, s));
            count_launch(h->launches_prefill);
        }
    }
    B2A_CUDA(cudaStreamSynchronize(s));
    const double t1 = now_s();
    bool cancelled = false;
    int streamed = 0;
    std::vector<int> h_tok;
    // ---- streaming audio emission state
    const bool streaming = ss.frames_per_chunk > 0 && ss.on_audio;
    if (streaming) B2A_CHECK(h->snac && !ids_on_device, B2A_ERR_MODEL_NOT_INITIALIZED, "SNAC model not loaded");
    std::vector<int> emitted(B, 0), s_prompt, s_tok, s_ng(B);
    std::vector<float> s_wave;
    double codec_stream_t = 0;
    if (streaming) { s_prompt.assign(input_ids, input_ids + (size_t)B * L); s_tok.resize((size_t)B * MT); }
    auto emit_audio = [&](bool final_call) {
        const double c0 = now_s();
        B2A_CUDA(cudaMemcpy(s_ng.data(), h->n_gen.p, B * sizeof(int), cudaMemcpyDeviceToHost));
        B2A_CUDA(cudaMemcpy(s_tok.data(), h->out_tokens.p, (size_t)B * MT * sizeof(int), cudaMemcpyDeviceToHost));
        const int64_t hop = b2a_snac_hop_length(h->snac);
        for (int b = 0; b < B; ++b) {
            const int ng = std::min(s_ng[b], MT);
            std::vector<int> all(s_prompt.begin() + (size_t)b * L, s_prompt.begin() + (size_t)(b + 1) * L);
            all.insert(all.end(), s_tok.begin() + (size_t)b * MT, s_tok.begin() + (size_t)b * MT + ng);
            std::vector<int> cl = parse_row(h->tok, all.data(), (int)all.size(), codes_start(h->tok, all.data(), (int)all.size()));
            if (h->bench_wrap_codes)
                for (size_t i = 0; i < cl.size(); ++i) cl[i] = ((cl[i] % 4096) + 4096) % 4096 + 4096 * (int)(i % 7);
            const int total = (int)cl.size() / 7;
            while (total - emitted[b] >= ss.frames_per_chunk || (final_call && total > emitted[b])) {
                const int f1 = final_call ? total : emitted[b] + ss.frames_per_chunk;
                const int f0 = std::max(0, emitted[b] - ss.left_context);
                std::vector<int> l1, l2, l3;
                deinterleave(cl.data() + (size_t)f0 * 7, (f1 - f0) * 7, l1, l2, l3);
                const int F = f1 - f0;
                h->d_codes[0].upload(l1.data(), l1.size(), s);
                h->d_codes[1].upload(l2.data(), l2.size(), s);
                h->d_codes[2].upload(l3.data(), l3.size(), s);
                const int64_t T = 4ll * F, wl = T * hop;
                h->d_wave.alloc((size_t)wl);
                const int* dc[3] = {h->d_codes[0].p, h->d_codes[1].p, h->d_codes[2].p};
                B2A_CUDA(cudaStreamSynchronize(s));
                const int32_t st = b2a_snac_decode_dev(h->snac, dc, 1, T, nullptr, 0, gp->seed + (uint64_t)b, h->d_wave.p, s);
                B2A_CHECK(st == B2A_OK, B2A_ERR_AUDIO_DECODING_FAILED, std::string("SNAC decode failed: ") + b2a_last_error());
                const int64_t skip = (int64_t)(emitted[b] - f0) * 4 * hop, n_new = wl - skip;
                s_wave.resize((size_t)n_new);
                B2A_CUDA(cudaMemcpyAsync(s_wave.data(), h->d_wave.p + skip, (size_t)n_new * sizeof(float), cudaMemcpyDeviceToHost, s));
                B2A_CUDA(cudaStreamSynchronize(s));
                emitted[b] = f1;
                ss.on_audio(user, b, s_wave.data(), n_new, (final_call && f1 == total) ? 1 : 0);
            }
        }
        codec_stream_t += now_s() - c0;
    };
    auto stream_tokens = [&]() {   // .token events (LlamaTTS.swift:862), row-major per step
        h_tok.resize((size_t)B * MT);
        std::vector<int> ng(B);
        B2A_CUDA(cudaMemcpy(ng.data(), h->n_gen.p, B * sizeof(int), cudaMemcpyDeviceToHost));
        B2A_CUDA(cudaMemcpy(h_tok.data(), h->out_tokens.p, (size_t)B * MT * sizeof(int), cudaMemcpyDeviceToHost));
        for (int b = 0; b < B; ++b)
            if (ng[b] > streamed) on_token(user, b, streamed, h_tok[(size_t)b * MT + streamed]);
        ++streamed;
    };
    if (steps == 1) {
        if (on_token) stream_tokens();
        B2A_CUDA(cudaMemcpyAsync(h->h_flag.p, h->n_active.p, sizeof(int), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    }
    // Without per-token callbacks the host keeps ONE burst of graph launches queued ahead of the burst whose "rows still active"
    // flag it is waiting for, so the GPU never idles while the host polls (synchronising after every burst would cost a share of the
    // loop).  A burst launched after every row has finished only replays steps whose tokens are not recorded; steps never exceed
    // max_tokens, so the KV cache cannot overflow.
    const bool pipelined = !on_token && !streaming;
    if (pipelined && !h->ev_poll[0]) { B2A_CUDA(cudaEventCreateWithFlags(&h->ev_poll[0], cudaEventDisableTiming)); B2A_CUDA(cudaEventCreateWithFlags(&h->ev_poll[1], cudaEventDisableTiming)); }
    int slot = 0, pending = -1;
    while (steps < MT && !(steps == 1 && h->h_flag.p[0] <= 0)) {
        const int burst = on_token ? 1 : std::min(streaming ? 7 : 16, MT - steps);
        for (int i = 0; i < burst; ++i) {
            B2A_CUDA(cudaGraphLaunch(h->g_step, s));
            count_launch(h->launches_step);
        }
        steps += burst;
        if (pipelined) {
            B2A_CUDA(cudaMemcpyAsync(h->h_flag.p + 1 + slot, h->n_active.p, sizeof(int), cudaMemcpyDeviceToHost, s));
            B2A_CUDA(cudaEventRecord(h->ev_poll[slot], s));
            if (pending >= 0) {
                B2A_CUDA(cudaEventSynchronize(h->ev_poll[pending]));
                if (h->cancel.load()) { cancelled = true; break; }
                if (h->h_flag.p[1 + pending] <= 0) break;
            }
            pending = slot; slot ^= 1;
            continue;
        }
        B2A_CUDA(cudaMemcpyAsync(h->h_flag.p, h->n_active.p, sizeof(int), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
        if (on_token) stream_tokens();
        if (streaming) emit_audio(false);
        if (h->cancel.load()) { cancelled = true; break; }
        if (h->h_flag.p[0] <= 0) break;
    }
    // Soprano: a row that reached max_tokens has its last token fed forward too (the reference's loop forwards every token it keeps,
    // Soprano.swift:836-879); one more step captures that state.  Its sample is never recorded: every row is done.
    if (soprano && steps >= MT && !cancelled) {
        B2A_CUDA(cudaGraphLaunch(h->g_step, s));
        count_launch(h->launches_step);
    }
    if (pipelined) { B2A_CUDA(cudaStreamSynchronize(s)); if (h->cancel.load()) cancelled = true; }
    if (streaming && !cancelled) emit_audio(true);
    const double t2 = now_s();
    B2A_CHECK(!cancelled, B2A_ERR_CANCELLED, "generation cancelled");

    std::vector<int> ng(B), toks((size_t)B * MT), prompt((size_t)B * L);
    B2A_CUDA(cudaMemcpyAsync(ng.data(), h->n_gen.p, B * sizeof(int), cudaMemcpyDeviceToHost, s));
    B2A_CUDA(cudaMemcpyAsync(toks.data(), h->out_tokens.p, (size_t)B * MT * sizeof(int), cudaMemcpyDeviceToHost, s));
    B2A_CUDA(cudaMemcpyAsync(prompt.data(), h->ids.p, (size_t)B * L * sizeof(int), cudaMemcpyDeviceToHost, s));
    B2A_CUDA(cudaStreamSynchronize(s));
    int total_gen = 0;
    for (int b = 0; b < B; ++b) {
        ng[b] = std::min(ng[b], MT);
        total_gen += ng[b];
        if (n_tokens_out) n_tokens_out[b] = ng[b];
        if (tokens_out) memcpy(tokens_out + (size_t)b * MT, toks.data() + (size_t)b * MT, ng[b] * sizeof(int));
    }

    double codec_t = 0;
    if (wave_out && soprano) {
        const double c0 = now_s();
        std::vector<int> nc(B);
        B2A_CUDA(cudaMemcpy(nc.data(), h->n_cap.p, B * sizeof(int), cudaMemcpyDeviceToHost));
        soprano_decode(h, h->hidden.p, (int64_t)h->hidden_slots * h->cfg.hidden_size, nc, wave_out, wave_on_device, wave_cap, wave_len, s);
        codec_t = now_s() - c0;
    } else if (wave_out) {
        const double c0 = now_s();
        // per row: generatedTokens = prompt + generated (LlamaTTS.swift:705-707,738) -> parseOutput -> frames
        const TokenLayout& tl = h->tok;
        std::vector<std::vector<int>> l1(B), l2(B), l3(B);
        std::vector<int> frames(B, 0);
        bool any = false;
        for (int b = 0; b < B; ++b) {
            std::vector<int> all(prompt.begin() + (size_t)b * L, prompt.begin() + (size_t)(b + 1) * L);
            all.insert(all.end(), toks.begin() + (size_t)b * MT, toks.begin() + (size_t)b * MT + ng[b]);
            std::vector<int> cl = parse_row(tl, all.data(), (int)all.size(), codes_start(tl, all.data(), (int)all.size()));
            if (h->bench_wrap_codes)   // benchmark only: fold random-init tokens into each slot's 4096-code range
                for (size_t i = 0; i < cl.size(); ++i) cl[i] = ((cl[i] % 4096) + 4096) % 4096 + 4096 * (int)(i % 7);
            deinterleave(cl.data(), (int)cl.size(), l1[b], l2[b], l3[b]);
            frames[b] = (int)l1[b].size();
            any |= frames[b] > 0;
            if (wave_len) wave_len[b] = 0;
        }
        B2A_CHECK(any, B2A_ERR_GENERATION_FAILED, "No audio codes generated");   // LlamaTTS.swift:752-754
        const int64_t hop = b2a_snac_hop_length(h->snac), frame_samples = 4 * hop;
        // A row is decoded whole, or -- longer than the layout's decode_chunk -- as decode_chunk-frame chunks decoded independently and
        // concatenated (decodeAudioFromCodes, Qwen3.swift:47-83).  Pieces (row, first frame, frames) of equal length share one batched
        // codec call: every full chunk of every row in one, trailing pieces grouped by length.
        struct Piece { int row, f0, nf; };
        std::vector<Piece> pieces;
        for (int b = 0; b < B; ++b) {
            if (frames[b] == 0) continue;
            B2A_CHECK(frames[b] * frame_samples <= wave_cap, B2A_ERR_INVALID_INPUT, "tts generate: wave buffer too small");
            const int chunk = tl.decode_chunk > 0 ? tl.decode_chunk : frames[b];
            for (int f0 = 0; f0 < frames[b]; f0 += chunk) pieces.push_back({b, f0, std::min(chunk, frames[b] - f0)});
        }
        std::vector<bool> used(pieces.size(), false);
        for (size_t i = 0; i < pieces.size(); ++i) {
            if (used[i]) continue;
            std::vector<Piece> grp;
            for (size_t j = i; j < pieces.size(); ++j)
                if (!used[j] && pieces[j].nf == pieces[i].nf) { grp.push_back(pieces[j]); used[j] = true; }
            const int F = pieces[i].nf, nb = (int)grp.size();
            const int64_t T = 4ll * F, wl = T * hop;
            std::vector<int> c0v, c1v, c2v;
            for (const Piece& p : grp) {
                c0v.insert(c0v.end(), l1[p.row].begin() + p.f0, l1[p.row].begin() + p.f0 + F);
                c1v.insert(c1v.end(), l2[p.row].begin() + 2 * p.f0, l2[p.row].begin() + 2 * (p.f0 + F));
                c2v.insert(c2v.end(), l3[p.row].begin() + 4 * p.f0, l3[p.row].begin() + 4 * (p.f0 + F));
            }
            h->d_codes[0].upload(c0v.data(), c0v.size(), s);
            h->d_codes[1].upload(c1v.data(), c1v.size(), s);
            h->d_codes[2].upload(c2v.data(), c2v.size(), s);
            h->d_wave.alloc((size_t)nb * wl);
            const int* dc[3] = {h->d_codes[0].p, h->d_codes[1].p, h->d_codes[2].p};
            B2A_CUDA(cudaStreamSynchronize(s));   // host vectors above go out of scope after the copy
            const int32_t st = b2a_snac_decode_dev(h->snac, dc, nb, T, nullptr, 0, gp->seed, h->d_wave.p, s);
            B2A_CHECK(st == B2A_OK, B2A_ERR_AUDIO_DECODING_FAILED, std::string("SNAC decode failed: ") + b2a_last_error());
            for (int k = 0; k < nb; ++k) {
                const Piece& p = grp[k];
                B2A_CUDA(cudaMemcpyAsync(wave_out + (size_t)p.row * wave_cap + (size_t)p.f0 * frame_samples, h->d_wave.p + (size_t)k * wl,
                                         wl * sizeof(float), wave_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, s));
                if (wave_len) wave_len[p.row] = (int64_t)frames[p.row] * frame_samples;
            }
            B2A_CUDA(cudaStreamSynchronize(s));
        }
        codec_t = now_s() - c0;
    }
    if (info) {
        info->prompt_token_count = L;
        info->generation_token_count = total_gen;
        info->prefill_time = t1 - t0;
        info->generate_time = t2 - t1;
        info->tokens_per_second = total_gen / std::max(1e-9, t2 - t1);
        info->codec_time = codec_t + codec_stream_t;
        size_t fr = 0, tot = 0;
        cudaMemGetInfo(&fr, &tot);
        info->peak_memory_gb = (double)(tot - fr) / 1e9;
    }
}

// prepareInputIds on token ids (LlamaTTS.swift:499-543, Qwen3.swift:417-464): every row is [pad..] [SOH] prompt [EOT, EOH], and with a
// reference (with_ref) [pad..] [SOH] ref_text [EOT, EOH] [SOAI, SOS] ref_codes + audio_offset [EOS, EOAI] [SOH] prompt [EOT, EOH], the
// padding in front to the longest prompt.  out NULL: only *out_len.
static void prepare_ids(const TokenLayout& tl, const int32_t* const* prompt_ids, const int32_t* lens, int32_t batch, const int32_t* ref_text_ids,
                        int32_t ref_text_len, const int32_t* ref_code_list, int32_t ref_code_len, int32_t* out, int32_t* out_len,
                        bool with_ref = false) {
    B2A_CHECK(prompt_ids && lens && out_len && batch > 0, B2A_ERR_INVALID_INPUT, "prepare_input_ids: null argument");
    B2A_CHECK(ref_code_len % 7 == 0, B2A_ERR_INVALID_INPUT, "prepare_input_ids: ref_code_len must be a multiple of 7");
    for (int i = 0; i < ref_code_len; ++i)
        B2A_CHECK(ref_code_list[i] >= 0 && ref_code_list[i] < 7 * 4096, B2A_ERR_INVALID_INPUT,
                  "prepare_input_ids: reference code out of range [0, 7 * 4096)");
    int mx = 0;
    for (int b = 0; b < batch; ++b) {
        B2A_CHECK(lens[b] >= 0 && (prompt_ids[b] || lens[b] == 0), B2A_ERR_INVALID_INPUT, "prepare_input_ids: bad prompt");
        mx = std::max(mx, lens[b]);
    }
    const int ref = with_ref ? 1 + ref_text_len + 2 + 2 + ref_code_len + 2 : 0;
    *out_len = mx + ref + 3;
    if (!out) return;
    for (int b = 0; b < batch; ++b) {
        int32_t* r = out + (size_t)b * (mx + ref + 3);
        int j = 0;
        for (; j < mx - lens[b]; ++j) r[j] = tl.pad;
        if (with_ref) {
            r[j++] = tl.start_of_human;
            for (int i = 0; i < ref_text_len; ++i) r[j++] = ref_text_ids[i];
            r[j++] = tl.end_of_text;
            r[j++] = tl.end_of_human;
            r[j++] = tl.start_of_ai;
            r[j++] = tl.start_of_speech;
            for (int i = 0; i < ref_code_len; ++i) r[j++] = ref_code_list[i] + tl.audio_offset;
            r[j++] = tl.end_of_speech;
            r[j++] = tl.end_of_ai;
        }
        r[j++] = tl.start_of_human;
        for (int i = 0; i < lens[b]; ++i) r[j++] = prompt_ids[b][i];
        r[j++] = tl.end_of_text;
        r[j++] = tl.end_of_human;
    }
}

extern "C" {

int32_t b2a_tts_generate_stream(b2a_tts* h, const int32_t* input_ids, int32_t B, int32_t L, const b2a_gen_params* gp,
                                int32_t frames_per_chunk, int32_t left_context_frames, int32_t* tokens_out, int32_t* n_tokens_out,
                                b2a_gen_info* info, b2a_token_cb on_token, b2a_audio_cb on_audio, void* user) {
    return guarded([&] {
        B2A_CHECK(on_audio && frames_per_chunk >= 1 && left_context_frames >= 0, B2A_ERR_INVALID_INPUT,
                  "b2a_tts_generate_stream: needs on_audio, frames_per_chunk >= 1, left_context_frames >= 0");
        StreamSpec ss;
        ss.frames_per_chunk = frames_per_chunk; ss.left_context = left_context_frames; ss.on_audio = on_audio;
        tts_generate_impl(h, input_ids, false, B, L, gp, tokens_out, n_tokens_out, nullptr, false, 0, nullptr, info, on_token, user, ss);
    });
}

int32_t b2a_tts_create(int32_t device, const b2a_llama_config* cfg, const b2a_tensor* tensors, int32_t n, b2a_snac* snac,
                       b2a_tts** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_tts_create: null out");
        *out = nullptr;
        B2A_CHECK(cfg && tensors && n > 0, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_tts_create: missing config or weights");
        TensorTable tt(tensors, n);
        *out = new b2a_tts(device, *cfg, tt, snac);
    });
}

int32_t b2a_tts_create_random(int32_t device, const b2a_llama_config* cfg, float std, uint64_t seed, b2a_snac* snac,
                              b2a_tts** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_tts_create_random: null out");
        *out = nullptr;
        B2A_CHECK(cfg && std > 0.f, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_tts_create_random: missing config");
        *out = new b2a_tts(device, *cfg, std, seed, snac);
    });
}

void* b2a_tts_stream(b2a_tts* h) { return h ? (void*)h->stream : nullptr; }

int32_t b2a_tts_time_steps(b2a_tts* h, int32_t B, int32_t ctx, int32_t iters, float* ms_per_step) {
    return guarded([&] {
        B2A_CHECK(h && ms_per_step && iters > 0, B2A_ERR_INVALID_INPUT, "b2a_tts_time_steps: bad argument");
        B2A_CHECK(B >= 1 && B <= h->cfg.max_batch && ctx >= 0 && ctx + iters < h->cfg.max_context, B2A_ERR_INVALID_INPUT,
                  "b2a_tts_time_steps: batch / context out of range");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        h->set_batch(B);
        const int MT = iters + 8;
        h->ids.alloc((size_t)B * 1);
        h->out_tokens.alloc((size_t)B * MT);
        h->recent.alloc(h->rows_cap());
        SampleArgs sa{};
        sa.logits = h->logits.p; sa.probs = h->probs.p; sa.tokens = h->tokens.p; sa.pos = h->pos.p; sa.recent = h->recent.p;
        sa.recent_n = h->recent_n.p; sa.out_tokens = h->out_tokens.p; sa.n_gen = h->n_gen.p; sa.done = h->done.p;
        sa.n_active = h->n_active.p; sa.forced = nullptr; sa.V = h->cfg.vocab_size; sa.R = 1; sa.max_tokens = MT;
        sa.temperature = 0.f; sa.top_p = 1.f; sa.rep_penalty = 1.f; sa.seed = 0; sa.mask_eos = 1; sa.stop_token = h->tok.end_of_speech;
        h->capture(B, sa, 1);
        B2A_CUDA(cudaMemsetAsync(h->ids.p, 0, (size_t)B * sizeof(int), s));
        init_rows_kernel<<<1, 32, 0, s>>>(h->ids.p, 1, B, 0, h->tokens.p, h->pos.p, h->recent.p, h->recent_n.p, h->n_gen.p,
                                          h->done.p, h->n_active.p, ctx);
        count_launch();
        // K/V beyond what earlier calls wrote is whatever is in the cache: zero it so reads are defined
        // (timing only; values do not matter).
        cudaEvent_t e0, e1;
        B2A_CUDA(cudaEventCreate(&e0));
        B2A_CUDA(cudaEventCreate(&e1));
        B2A_CUDA(cudaGraphLaunch(h->g_step, s));   // warm-up
        B2A_CUDA(cudaEventRecord(e0, s));
        for (int i = 0; i < iters - 1; ++i) B2A_CUDA(cudaGraphLaunch(h->g_step, s));
        B2A_CUDA(cudaEventRecord(e1, s));
        B2A_CUDA(cudaStreamSynchronize(s));
        count_launch(h->launches_step * iters);
        float ms = 0.f;
        B2A_CUDA(cudaEventElapsedTime(&ms, e0, e1));
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        *ms_per_step = ms / (float)std::max(1, iters - 1);
    });
}

int32_t b2a_tts_prepare_input_ids(const int32_t* const* prompt_ids, const int32_t* lens, int32_t batch, int32_t* out,
                                  int32_t* out_len) {
    return guarded([&] { prepare_ids(ORPHEUS_TOKENS, prompt_ids, lens, batch, nullptr, 0, nullptr, 0, out, out_len); });
}

int32_t b2a_tts_prepare_input_ids_ref(const int32_t* const* prompt_ids, const int32_t* lens, int32_t batch, const int32_t* ref_text_ids,
                                      int32_t ref_text_len, const int32_t* ref_code_list, int32_t ref_code_len, int32_t* out,
                                      int32_t* out_len) {
    return guarded([&] {
        B2A_CHECK(ref_text_len >= 0 && ref_code_len >= 0 && (ref_text_ids || ref_text_len == 0) && (ref_code_list || ref_code_len == 0),
                  B2A_ERR_INVALID_INPUT, "b2a_tts_prepare_input_ids_ref: null argument");
        prepare_ids(ORPHEUS_TOKENS, prompt_ids, lens, batch, ref_text_ids, ref_text_len, ref_code_list, ref_code_len, out, out_len, true);
    });
}

int32_t b2a_debug_step_smem(int32_t gqa, int32_t* out) {
    return guarded([&] {
        B2A_CHECK(out && gqa_supported(gqa), B2A_ERR_INVALID_INPUT,
                  "b2a_debug_step_smem: q heads per kv head must be 1, 2, 3, 4, 6 or 8");
        out[0] = (int32_t)tc::Smem<16>::bytes(b2a_tts::GEMM_STAGES[0]);
        out[1] = (int32_t)tc::SmemSplit<8>::bytes(b2a_tts::SPLITK_STAGES[0], b2a_tts::fused_cluster);
        out[2] = (int32_t)attn_smem_bytes(gqa);
    });
}

int32_t b2a_debug_step_smem_rows(int32_t rows, int32_t gqa, int32_t* out) {
    return guarded([&] {
        B2A_CHECK(out && rows >= 1 && rows <= 32 && gqa_supported(gqa), B2A_ERR_INVALID_INPUT,
                  "b2a_debug_step_smem_rows: rows must be in 1..32 and q heads per kv head 1, 2, 3, 4, 6 or 8");
        const int w = tc::decode_width(rows), wi = tc::decode_width_index(w);
        out[0] = w;
        out[1] = b2a_tts::GEMM_STAGES[wi];
        out[2] = (int32_t)b2a_tts::gemm_bytes(w, b2a_tts::GEMM_STAGES[wi]);
        out[3] = b2a_tts::SPLITK_STAGES[wi];
        out[4] = (int32_t)b2a_tts::splitk_bytes(w, b2a_tts::SPLITK_STAGES[wi], b2a_tts::fused_cluster);
        out[5] = (int32_t)attn_smem_bytes(gqa);
    });
}

int32_t b2a_debug_qkv_split(int32_t m_tiles, int32_t k_blocks, int32_t* out) {
    return guarded([&] {
        B2A_CHECK(out && m_tiles >= 1 && k_blocks >= 1, B2A_ERR_INVALID_INPUT, "b2a_debug_qkv_split: bad argument");
        require_device(0);
        tc::set_attributes();
        int sms = 0, sk_ctas = 0;
        B2A_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
        out[0] = b2a_tts::pick_qkv_cluster(m_tiles, k_blocks, sms, &sk_ctas);
        out[1] = out[0] ? (int32_t)tc::SmemSplit<8>::bytes(b2a_tts::SPLITK_STAGES[0], out[0]) : 0;
        out[2] = out[0] ? tc::splitk_active_clusters<8>(out[0], (size_t)out[1]) : 0;
        out[3] = sk_ctas;
        out[4] = tc::stream_k_slots(m_tiles, k_blocks, sk_ctas);
    });
}

// The decode-step attention on its own (include/b200audio_internal.h): attn_decode_cluster_kernel<G> with the step's launch
// (b2a_tts::attn_launch), on DEVICE buffers the caller owns.
int32_t b2a_decode_attn_test(const float* qkv, const int32_t* pos, const float* freqs, const float* qnorm, const float* knorm, float qk_eps,
                             float* kcache, float* vcache, void* out, int32_t B, int32_t nq, int32_t nkv, int32_t max_ctx, void* stream) {
    return guarded([&] {
        B2A_CHECK(qkv && pos && freqs && kcache && vcache && out && B >= 1 && B <= 8 && max_ctx >= 1 && !qnorm == !knorm,
                  B2A_ERR_INVALID_INPUT, "b2a_decode_attn_test: bad argument");
        B2A_CHECK(nkv >= 1 && nq % nkv == 0 && gqa_supported(nq / nkv), B2A_ERR_INVALID_INPUT,
                  "b2a_decode_attn_test: q heads per kv head must be 1, 2, 3, 4, 6 or 8");
        require_device(0);
        b2a_tts::attn_cluster_attr<1>(); b2a_tts::attn_cluster_attr<2>(); b2a_tts::attn_cluster_attr<3>();
        b2a_tts::attn_cluster_attr<4>(); b2a_tts::attn_cluster_attr<6>(); b2a_tts::attn_cluster_attr<8>();
        const cudaStream_t s = (cudaStream_t)stream;
        const AttnArgs aa{qkv, pos, freqs, kcache, vcache, (bf16*)out, nq, nkv, max_ctx, 1.0f / sqrtf((float)HD), qnorm, knorm, qk_eps, 8};
        b2a_tts::attn_launch(aa, B, s);
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

// The prompt attention on its own (include/b200audio_internal.h): rope_table_kernel, then path 1 prefill_attn_kernel<G> or path 2
// pack_prompt_kernel + prompt_attn_kernel, as prefill_batched runs them for one layer, on DEVICE buffers the caller owns.
int32_t b2a_prompt_attn_test(const float* qkv, const float* freqs, const float* qnorm, const float* knorm, float qk_eps, float* kcache,
                             float* vcache, void* out, int32_t B, int32_t L, int32_t nq, int32_t nkv, int32_t max_ctx, int32_t path,
                             void* stream) {
    return guarded([&] {
        B2A_CHECK(qkv && freqs && kcache && vcache && out && B >= 1 && L >= 1 && L <= max_ctx && !qnorm == !knorm && (path == 1 || path == 2),
                  B2A_ERR_INVALID_INPUT, "b2a_prompt_attn_test: bad argument");
        B2A_CHECK(nkv >= 1 && nq % nkv == 0 && gqa_supported(nq / nkv), B2A_ERR_INVALID_INPUT,
                  "b2a_prompt_attn_test: q heads per kv head must be 1, 2, 3, 4, 6 or 8");
        B2A_CHECK(path == 2 || simt_prompt_attn(L, nq / nkv), B2A_ERR_INVALID_INPUT,
                  "b2a_prompt_attn_test: L too long for the SIMT prompt attention at this GQA ratio");
        require_device(0);
        const cudaStream_t s = (cudaStream_t)stream;
        DBuf<float2> rope;
        rope.alloc((size_t)L * (HD / 2));
        rope_table_kernel<<<cdiv(L * (HD / 2), 256), 256, 0, s>>>(freqs, rope.p, L);
        count_launch();
        PromptAttnOps ops;                          // its buffers outlive the launches (freed after the synchronise)
        if (path == 1) {
            b2a_tts::pattn_attr();
            const PrefillAttnArgs pa{qkv, rope.p, kcache, vcache, (bf16*)out, nq, nkv, max_ctx, L, 1.0f / sqrtf((float)HD), qnorm, knorm,
                                     qk_eps};
            b2a_tts::pattn_launch(pa, B, s);
        } else {
            ops.prepare(B, L, nq, nkv);
            ops.run(qkv, rope.p, kcache, vcache, (bf16*)out, L, max_ctx, s, qnorm, knorm, qk_eps);
        }
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

// Debug / parity hook: residual stream seen by every RMSNorm (2 per layer + final) for the LAST position of
// the last b2a_tts_forward_logits call made while tracing was enabled; out is [2*layers+1, batch, hidden].
int32_t b2a_tts_debug_trace(b2a_tts* h, int32_t enable, int32_t batch, float* out) {
    return guarded([&] {
        B2A_CHECK(h, B2A_ERR_INVALID_INPUT, "b2a_tts_debug_trace: null handle");
        B2A_CUDA(cudaSetDevice(h->device));
        const int H = h->cfg.hidden_size, n = 2 * h->cfg.num_hidden_layers + 1;
        if (out) {
            B2A_CHECK(h->trace.p && batch >= 1 && batch <= h->rows_cap(), B2A_ERR_INVALID_INPUT, "b2a_tts_debug_trace: nothing traced");
            B2A_CUDA(cudaStreamSynchronize(h->stream));
            for (int i = 0; i < n; ++i)
                B2A_CUDA(cudaMemcpy(out + (size_t)i * batch * H, h->trace.p + (size_t)i * h->rows_cap() * H, (size_t)batch * H * sizeof(float),
                                    cudaMemcpyDeviceToHost));
        }
        h->trace_on = enable != 0;
        if (h->trace_on) { h->trace.alloc((size_t)n * h->rows_cap() * H); h->drop_graphs(); }
    });
}

int32_t b2a_tts_forward_logits(b2a_tts* h, const int32_t* ids, int32_t B, int32_t L, int32_t reset_cache, float* logits_out) {
    return guarded([&] {
        B2A_CHECK(h && ids && logits_out, B2A_ERR_INVALID_INPUT, "b2a_tts_forward_logits: null argument");
        B2A_CHECK(B >= 1 && B <= h->cfg.max_batch && L >= 1, B2A_ERR_INVALID_INPUT, "b2a_tts_forward_logits: bad batch / length");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        h->set_batch(B);
        h->drop_graphs();
        const int RC = h->rows_cap();
        std::vector<int> hp(RC, 0);
        if (!reset_cache) B2A_CUDA(cudaMemcpy(hp.data(), h->pos.p, RC * sizeof(int), cudaMemcpyDeviceToHost));
        const int start = reset_cache ? 0 : hp[0];
        B2A_CHECK(start + L <= h->cfg.max_context, B2A_ERR_INVALID_INPUT, "b2a_tts_forward_logits: context overflow");
        h->ids.alloc((size_t)B * L);
        B2A_CUDA(cudaMemcpyAsync(h->ids.p, ids, (size_t)B * L * sizeof(int), cudaMemcpyHostToDevice, s));
        const int V = h->cfg.vocab_size;
        std::vector<int> tk(RC, 0), ps(RC, -1);
        for (int p = 0; p < L; ++p) {
            for (int b = 0; b < B; ++b) { tk[b] = ids[(size_t)b * L + p]; ps[b] = start + p; }
            B2A_CUDA(cudaMemcpyAsync(h->tokens.p, tk.data(), RC * sizeof(int), cudaMemcpyHostToDevice, s));
            B2A_CUDA(cudaMemcpyAsync(h->pos.p, ps.data(), RC * sizeof(int), cudaMemcpyHostToDevice, s));
            h->run_layers(B, s);
            h->run_lm_head(B, s);
            for (int b = 0; b < B; ++b)
                B2A_CUDA(cudaMemcpyAsync(logits_out + ((size_t)b * L + p) * V, h->logits.p + (size_t)b * V, V * sizeof(float),
                                         cudaMemcpyDeviceToHost, s));
            B2A_CUDA(cudaStreamSynchronize(s));
        }
        for (int b = 0; b < B; ++b) ps[b] = start + L;
        B2A_CUDA(cudaMemcpy(h->pos.p, ps.data(), RC * sizeof(int), cudaMemcpyHostToDevice));
        B2A_CUDA(cudaGetLastError());
    });
}

int32_t b2a_tts_generate(b2a_tts* h, const int32_t* input_ids, int32_t B, int32_t L, const b2a_gen_params* gp,
                         int32_t* tokens_out, int32_t* n_tokens_out, float* wave_out, int64_t wave_cap, int64_t* wave_len,
                         b2a_gen_info* info, b2a_token_cb on_token, void* user) {
    return guarded([&] {
        tts_generate_impl(h, input_ids, false, B, L, gp, tokens_out, n_tokens_out, wave_out, false, wave_cap, wave_len, info,
                          on_token, user);
    });
}

int32_t b2a_tts_generate_dev(b2a_tts* h, const int32_t* d_input_ids, int32_t B, int32_t L, const b2a_gen_params* gp,
                             float* d_wave_out, int64_t wave_cap, int64_t* wave_len, b2a_gen_info* info) {
    return guarded([&] {
        tts_generate_impl(h, d_input_ids, true, B, L, gp, nullptr, nullptr, d_wave_out, true, wave_cap, wave_len, info, nullptr,
                          nullptr);
    });
}

int32_t b2a_tts_set_bench_flags(b2a_tts* h, int32_t mask_eos, int32_t wrap_codes) {
    if (!h) return B2A_ERR_INVALID_INPUT;
    h->bench_mask_eos = mask_eos != 0;
    h->bench_wrap_codes = wrap_codes != 0;
    return B2A_OK;
}

int32_t b2a_tts_cancel(b2a_tts* h) {
    if (!h) return B2A_ERR_INVALID_INPUT;
    h->cancel.store(1);
    return B2A_OK;
}

int32_t b2a_tts_parse_output(const int32_t* tokens, int32_t batch, int32_t n, int32_t* code_lists_out, int32_t* code_lens) {
    return guarded([&] {
        B2A_CHECK(tokens && code_lists_out && code_lens && batch > 0 && n >= 0, B2A_ERR_INVALID_INPUT, "b2a_tts_parse_output: bad argument");
        int last = -1;   // LlamaTTS.swift:391-398: last match in row-major visiting order
        for (int i = 0; i < batch; ++i)
            for (int j = 0; j < n; ++j)
                if (tokens[(size_t)i * n + j] == ORPHEUS_TOKENS.start_of_speech) last = j;
        for (int i = 0; i < batch; ++i) {
            std::vector<int> r = parse_row(ORPHEUS_TOKENS, tokens + (size_t)i * n, n, last);
            code_lens[i] = (int)r.size();
            memcpy(code_lists_out + (size_t)i * n, r.data(), r.size() * sizeof(int));
        }
    });
}

int32_t b2a_tts_deinterleave(const int32_t* code_list, int32_t n, int32_t* c0, int32_t* c1, int32_t* c2, int32_t* n_frames) {
    return guarded([&] {
        B2A_CHECK(code_list && c0 && c1 && c2 && n_frames && n >= 0, B2A_ERR_INVALID_INPUT, "b2a_tts_deinterleave: bad argument");
        const int groups = (n + 1) / 7;
        B2A_CHECK(groups * 7 <= n, B2A_ERR_INVALID_INPUT, "b2a_tts_deinterleave: code list must hold whole 7-token frames");
        std::vector<int> l1, l2, l3;
        deinterleave(code_list, n, l1, l2, l3);
        memcpy(c0, l1.data(), l1.size() * sizeof(int));
        memcpy(c1, l2.data(), l2.size() * sizeof(int));
        memcpy(c2, l3.data(), l3.size() * sizeof(int));
        *n_frames = groups;
    });
}

int32_t b2a_tts_interleave(const int32_t* c0, const int32_t* c1, const int32_t* c2, int32_t n_frames, int32_t* cl) {
    return guarded([&] {   // llamaEncodeAudioToCodes, LlamaTTS.swift:85-95
        B2A_CHECK(c0 && c1 && c2 && cl && n_frames >= 0, B2A_ERR_INVALID_INPUT, "b2a_tts_interleave: bad argument");
        for (int i = 0; i < n_frames; ++i) {
            int32_t* o = cl + 7 * i;
            o[0] = c0[i];
            o[1] = c1[2 * i] + 4096;
            o[2] = c2[4 * i] + 2 * 4096;
            o[3] = c2[4 * i + 1] + 3 * 4096;
            o[4] = c1[2 * i + 1] + 4 * 4096;
            o[5] = c2[4 * i + 2] + 5 * 4096;
            o[6] = c2[4 * i + 3] + 6 * 4096;
        }
    });
}

// ------------------------------------------------------------------------------------------------ VyvoTTS (Qwen3Model, Qwen3.swift:305-931)
static b2a_llama_config qwen3_lm_stack_cfg(const b2a_qwen3_lm_config& c) {
    B2A_CHECK(c.rope_linear_factor > 0.f, B2A_ERR_INVALID_INPUT, "qwen3 lm: rope_linear_factor must be positive");
    b2a_llama_config l{};
    l.hidden_size = c.hidden_size; l.num_hidden_layers = c.num_hidden_layers; l.intermediate_size = c.intermediate_size;
    l.num_attention_heads = c.num_attention_heads; l.num_key_value_heads = c.num_key_value_heads; l.head_dim = c.head_dim;
    l.vocab_size = c.vocab_size; l.rms_norm_eps = c.rms_norm_eps; l.rope_theta = c.rope_theta;
    l.rope_factor = 1.f; l.rope_low_freq_factor = 1.f; l.rope_high_freq_factor = 4.f; l.rope_old_context_len = 8192.f;   // unused: linear_rope
    l.tie_word_embeddings = c.tie_word_embeddings; l.max_batch = c.max_batch; l.max_context = c.max_context;
    return l;
}
// "model.embed_tokens", q/k norm, "lm_head.weight" unless tied
static StackSpec qwen3_lm_spec(const b2a_qwen3_lm_config& c) {
    StackSpec s;
    s.qk_norm = true;
    s.linear_rope = c.rope_linear_factor;
    return s;
}

int32_t b2a_qwen3_lm_create(int32_t device, const b2a_qwen3_lm_config* cfg, const b2a_tensor* tensors, int32_t n, b2a_snac* snac,
                            b2a_tts** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_qwen3_lm_create: null out");
        *out = nullptr;
        B2A_CHECK(cfg && tensors && n > 0, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_qwen3_lm_create: missing config or weights");
        TensorTable tt(tensors, n);
        std::unique_ptr<b2a_tts> h(new b2a_tts(device, qwen3_lm_stack_cfg(*cfg), tt, snac, qwen3_lm_spec(*cfg)));
        h->tok = VYVO_TOKENS;
        *out = h.release();
    });
}

int32_t b2a_qwen3_lm_create_random(int32_t device, const b2a_qwen3_lm_config* cfg, float std, uint64_t seed, b2a_snac* snac, b2a_tts** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_qwen3_lm_create_random: null out");
        *out = nullptr;
        B2A_CHECK(cfg && std > 0.f, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_qwen3_lm_create_random: missing config");
        std::unique_ptr<b2a_tts> h(new b2a_tts(device, qwen3_lm_stack_cfg(*cfg), std, seed, snac, qwen3_lm_spec(*cfg)));
        h->tok = VYVO_TOKENS;
        *out = h.release();
    });
}

int32_t b2a_qwen3_lm_prepare_input_ids(const int32_t* const* prompt_ids, const int32_t* lens, int32_t batch, int32_t* out, int32_t* out_len) {
    return guarded([&] { prepare_ids(VYVO_TOKENS, prompt_ids, lens, batch, nullptr, 0, nullptr, 0, out, out_len); });
}

int32_t b2a_qwen3_lm_prepare_input_ids_ref(const int32_t* const* prompt_ids, const int32_t* lens, int32_t batch, const int32_t* ref_text_ids,
                                           int32_t ref_text_len, const int32_t* ref_code_list, int32_t ref_code_len, int32_t* out,
                                           int32_t* out_len) {
    return guarded([&] {
        B2A_CHECK(ref_text_len >= 0 && ref_code_len >= 0 && (ref_text_ids || ref_text_len == 0) && (ref_code_list || ref_code_len == 0),
                  B2A_ERR_INVALID_INPUT, "b2a_qwen3_lm_prepare_input_ids_ref: null argument");
        prepare_ids(VYVO_TOKENS, prompt_ids, lens, batch, ref_text_ids, ref_text_len, ref_code_list, ref_code_len, out, out_len, true);
    });
}

int32_t b2a_qwen3_lm_parse_output(const int32_t* tokens, int32_t batch, int32_t n, int32_t* code_lists_out, int32_t* code_lens) {
    return guarded([&] {
        B2A_CHECK(tokens && code_lists_out && code_lens && batch > 0 && n >= 0, B2A_ERR_INVALID_INPUT, "b2a_qwen3_lm_parse_output: bad argument");
        for (int i = 0; i < batch; ++i) {
            const int32_t* row = tokens + (size_t)i * n;
            std::vector<int> r = parse_row(VYVO_TOKENS, row, n, codes_start(VYVO_TOKENS, row, n));
            code_lens[i] = (int)r.size();
            memcpy(code_lists_out + (size_t)i * n, r.data(), r.size() * sizeof(int));
        }
    });
}

// ------------------------------------------------------------------------------------------------ Soprano (SopranoModel, Soprano.swift:184-977)
static b2a_llama_config soprano_stack_cfg(const b2a_soprano_config& c) {
    b2a_qwen3_lm_config q{};
    q.hidden_size = c.hidden_size; q.num_hidden_layers = c.num_hidden_layers; q.intermediate_size = c.intermediate_size;
    q.num_attention_heads = c.num_attention_heads; q.num_key_value_heads = c.num_key_value_heads; q.head_dim = c.head_dim;
    q.vocab_size = c.vocab_size; q.rms_norm_eps = c.rms_norm_eps; q.rope_theta = c.rope_theta; q.rope_linear_factor = 1.f;
    q.tie_word_embeddings = c.tie_word_embeddings; q.max_batch = c.max_batch; q.max_context = c.max_context;
    return qwen3_lm_stack_cfg(q);
}

// the Soprano stack is Qwen3's (Soprano.swift:24-180): q/k norm, rotate-half RoPE with base rope_theta, no scaling
static StackSpec soprano_spec() {
    StackSpec s;
    s.qk_norm = true;
    s.linear_rope = 1.f;
    return s;
}

// the handle's Vocos: decoder.decoder.* -> backbone.*, decoder.head.* -> head.* (the keys b2a_vocos_create reads), Vocos's
// LayerNorm backbone at the decoder geometry of the config
static void soprano_attach_decoder(b2a_tts* h, int device, const b2a_soprano_config& c, const b2a_tensor* tensors, int n) {
    B2A_CHECK(c.upscale >= 1 && c.token_size >= 0, B2A_ERR_INVALID_INPUT, "soprano: upscale must be >= 1 and token_size >= 0");
    std::vector<std::string> names;
    std::vector<b2a_tensor> dec;
    names.reserve(n);
    for (int i = 0; i < n; ++i) {
        const std::string k = tensors[i].name ? tensors[i].name : "";
        if (k.rfind("decoder.decoder.", 0) == 0) names.push_back("backbone." + k.substr(16));
        else if (k.rfind("decoder.head.", 0) == 0) names.push_back("head." + k.substr(13));
        else continue;
        dec.push_back(tensors[i]);
    }
    for (size_t i = 0; i < dec.size(); ++i) dec[i].name = names[i].c_str();
    B2A_CHECK(!dec.empty(), B2A_ERR_MODEL_NOT_INITIALIZED, "soprano: no decoder.decoder.* / decoder.head.* weights");
    b2a_vocos_config v{};
    v.input_channels = c.hidden_size; v.dim = c.decoder_dim; v.intermediate_dim = c.decoder_intermediate_dim; v.num_layers = c.decoder_num_layers;
    v.n_fft = c.n_fft; v.hop_length = c.hop_length; v.input_kernel_size = c.input_kernel; v.dw_kernel_size = c.dw_kernel;
    v.adanorm_num_embeddings = 0;
    const int32_t st = b2a_vocos_create(device, &v, dec.data(), (int32_t)dec.size(), &h->vocos);
    if (st != B2A_OK) throw Error(st, b2a_last_error());
    h->upscale = c.upscale; h->token_size = c.token_size;
    h->tok = TokenLayout{-1, -1, -1, -1, -1, -1, c.stop_token_id, -1, 0, false, 0};
}

int32_t b2a_soprano_create(int32_t device, const b2a_soprano_config* cfg, const b2a_tensor* tensors, int32_t n, b2a_tts** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_soprano_create: null out");
        *out = nullptr;
        B2A_CHECK(cfg && tensors && n > 0, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_soprano_create: missing config or weights");
        TensorTable tt(tensors, n);
        std::unique_ptr<b2a_tts> h(new b2a_tts(device, soprano_stack_cfg(*cfg), tt, nullptr, soprano_spec()));
        soprano_attach_decoder(h.get(), device, *cfg, tensors, n);
        *out = h.release();
    });
}

int32_t b2a_soprano_create_random(int32_t device, const b2a_soprano_config* cfg, float std, uint64_t seed, const b2a_tensor* decoder_tensors,
                                  int32_t n_decoder_tensors, b2a_tts** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_soprano_create_random: null out");
        *out = nullptr;
        B2A_CHECK(cfg && std > 0.f && decoder_tensors && n_decoder_tensors > 0, B2A_ERR_MODEL_NOT_INITIALIZED,
                  "b2a_soprano_create_random: missing config or decoder weights");
        std::unique_ptr<b2a_tts> h(new b2a_tts(device, soprano_stack_cfg(*cfg), std, seed, nullptr, soprano_spec()));
        soprano_attach_decoder(h.get(), device, *cfg, decoder_tensors, n_decoder_tensors);
        *out = h.release();
    });
}

int64_t b2a_soprano_wave_length(const b2a_tts* h, int32_t n) {
    return h && h->vocos && n >= 1 ? soprano_wave_len(h, n, nullptr) : 0;
}

int32_t b2a_soprano_decode_hidden(b2a_tts* h, const float* hidden, int32_t B, int32_t n, float* wave_out, int64_t wave_cap, int64_t* wave_len) {
    return guarded([&] {
        B2A_CHECK(h && hidden && wave_out, B2A_ERR_INVALID_INPUT, "b2a_soprano_decode_hidden: null argument");
        B2A_CHECK(h->vocos, B2A_ERR_INVALID_INPUT, "b2a_soprano_decode_hidden: not a Soprano handle");
        B2A_CHECK(B >= 1 && n >= 1, B2A_ERR_INVALID_INPUT, "b2a_soprano_decode_hidden: batch and state count must be positive");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        const size_t row = (size_t)n * h->cfg.hidden_size;
        DBuf<float> d;
        d.upload(hidden, (size_t)B * row, s);
        soprano_decode(h, d.p, (int64_t)row, std::vector<int>(B, n), wave_out, false, wave_cap, wave_len, s);
    });
}

int32_t b2a_soprano_hidden_states(b2a_tts* h, int32_t B, float* out, int32_t* n_states) {
    return guarded([&] {
        B2A_CHECK(h && h->vocos && n_states && B >= 1 && B <= h->cfg.max_batch, B2A_ERR_INVALID_INPUT, "b2a_soprano_hidden_states: bad argument");
        B2A_CHECK(h->hidden.p && h->n_cap.p && B <= h->hidden_rows, B2A_ERR_INVALID_INPUT,
                  "b2a_soprano_hidden_states: batch exceeds the last generate call's");
        B2A_CUDA(cudaSetDevice(h->device));
        B2A_CUDA(cudaStreamSynchronize(h->stream));
        B2A_CUDA(cudaMemcpy(n_states, h->n_cap.p, B * sizeof(int), cudaMemcpyDeviceToHost));
        if (out)
            B2A_CUDA(cudaMemcpy(out, h->hidden.p, (size_t)B * h->hidden_slots * h->cfg.hidden_size * sizeof(float), cudaMemcpyDeviceToHost));
    });
}

void b2a_tts_destroy(b2a_tts* h) { delete h; }

}  // extern "C"

// ================================================================================================
// Qwen3-TTS talker + code predictor (SURVEY.md section 8f row N1) on the same engine.
//   Qwen3TTSTalker.swift:127-366, Qwen3TTSCodePredictor.swift:14-243, Qwen3TTS.swift:380-495 (frame loop), :1003-1118 (sampleToken)
// Two b2a_tts stacks (talker: inputs are embeddings, untied codec_head; predictor: 5 layers, heads owned here) share one stream.
// One frame = ONE CUDA graph: talker step -> sampler -> [hidden, embed(c0)] + 14 more predictor steps (cache positions 0..16 are
// simply overwritten every frame = the reference's per-frame cache trim) -> summed-embedding feedback + bookkeeping.
// ================================================================================================
namespace b2a {

__device__ __forceinline__ float q3_f32(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float q3_f32(float v) { return v; }
// dst[b, :] = float(table[ids[b * id_stride + id_col], :]);  optionally pos[b] = pos_value (the predictor's cache position).
// T = bf16: an embedding table; T = float: a table already projected to the predictor's width (b2a_qwen3_talker::proj_tab)
template <typename T>
__global__ void q3_gather_kernel(const T* __restrict__ table, int rows, const int* __restrict__ ids, int id_stride, int id_col,
                                 float* __restrict__ dst, int H, int* pos, int pos_value) {
    const int b = blockIdx.x;
    if (!pos) pdl_trigger();     // a kernel that writes pos[] must not trigger early (see attn_decode_cluster_kernel)
    pdl_wait();
    int t = ids[b * id_stride + id_col];
    t = min(max(t, 0), rows - 1);
    for (int i = threadIdx.x; i < H; i += blockDim.x) dst[(long long)b * H + i] = q3_f32(table[(long long)t * H + i]);
    if (pos && threadIdx.x == 0) pos[b] = pos_value;
}
// dst[b, :] = src[b * src_stride + :]; optionally pos[b] = pos_value (pos_value < 0: pos untouched)
__global__ void q3_copy_rows_kernel(const float* __restrict__ src, long long src_stride, float* __restrict__ dst, int H, int* pos, int pos_value) {
    const int b = blockIdx.x;
    if (!(pos && pos_value >= 0)) pdl_trigger();     // writers of pos[] never trigger early
    pdl_wait();
    for (int i = threadIdx.x; i < H; i += blockDim.x) dst[(long long)b * H + i] = src[(long long)b * src_stride + i];
    if (pos && pos_value >= 0 && threadIdx.x == 0) pos[b] = pos_value;
}
// y[t, o] = act(b[o] + sum_k W[o, k] x[t, k]); bf16 W, fp32 x / y; one warp per output, grid (ceil(O / 8), T).  The prompt's
// ResizeMLP only (text_projection, Qwen3TTSTalker.swift:209-221): a few dozen rows per utterance, off the frame loop.
__global__ void q3_linear_kernel(const bf16* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ x, float* __restrict__ y,
                                 int O, int K, int silu) {
    const int o = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), t = blockIdx.y, lane = threadIdx.x & 31;
    if (o >= O) return;
    float acc = 0.f;
    for (int k = lane; k < K; k += 32) acc = fmaf(__bfloat162float(W[(long long)o * K + k]), x[(long long)t * K + k], acc);
    acc = warp_sum(acc);
    if (lane == 0) {
        acc += bias ? bias[o] : 0.f;
        y[(long long)t * O + o] = silu ? acc / (1.0f + __expf(-acc)) : acc;
    }
}

struct Q3Feedback {
    const bf16* codec_emb; int codec_rows;
    const bf16* const* cp_emb;   // device array of G-1 tables [cp_vocab, H]
    int cp_rows;
    const int* codes;            // [max_batch, G] this frame
    const float* trailing;       // [B, n_max, H]
    const int* n_trailing;       // [B]
    int n_max;
    const float* pad;            // [H]
    float* x_in;                 // [max_batch, H] next talker input
    int* talker_pos;             // [max_batch]
    int* row_frame;              // [max_batch] frames stepped so far (= index of the trailing text row to consume)
    int* out_codes;              // [B, max_tokens, G]
    int* n_frames; int* done; int* n_active;
    int G, H, max_tokens, eos, mask_eos;
};
// x_next = text + codec_embed(c0) + sum_i predictor_embed_i(c_{i+1})  (Qwen3TTS.swift:470-487) + per-row bookkeeping (:424-428)
// channel i of one code frame's embedding: codec_embedding(c0) + sum over g >= 1 of the predictor's codec_embedding[g-1](c_g), in
// that order (the talker's feedback, Qwen3TTS.swift:470-480, and codecEmbedIcl's rows, :249-265)
__device__ __forceinline__ float q3_frame_sum(const bf16* codec_emb, int codec_rows, const bf16* const* cp_emb, int cp_rows, const int* c, int G,
                                              int H, int i) {
    float e = __bfloat162float(codec_emb[(long long)min(max(c[0], 0), codec_rows - 1) * H + i]);
    for (int g = 1; g < G; ++g) e += __bfloat162float(cp_emb[g - 1][(long long)min(max(c[g], 0), cp_rows - 1) * H + i]);
    return e;
}
__global__ void q3_feedback_kernel(Q3Feedback a) {
    const int b = blockIdx.x;
    pdl_wait();                  // NO pdl_trigger(): writes the talker's pos[]
    const int f = a.row_frame[b];
    const float* text = f < a.n_trailing[b] ? a.trailing + ((long long)b * a.n_max + f) * a.H : a.pad;
    const int* c = a.codes + b * a.G;
    for (int i = threadIdx.x; i < a.H; i += blockDim.x)
        a.x_in[(long long)b * a.H + i] = text[i] + q3_frame_sum(a.codec_emb, a.codec_rows, a.cp_emb, a.cp_rows, c, a.G, a.H, i);
    __syncthreads();
    if (threadIdx.x == 0) {
        a.row_frame[b] = f + 1;
        a.talker_pos[b] += 1;
        if (!a.done[b]) {
            if (c[0] == a.eos && !a.mask_eos) { a.done[b] = 1; atomicSub(a.n_active, 1); }
            else {
                const int n = a.n_frames[b];
                if (n < a.max_tokens) for (int g = 0; g < a.G; ++g) a.out_codes[((long long)b * a.max_tokens + n) * a.G + g] = c[g];
                a.n_frames[b] = n + 1;
                if (n + 1 >= a.max_tokens) { a.done[b] = 1; atomicSub(a.n_active, 1); }
            }
        }
    }
}
// codes [n, G] -> out [n, H]: one frame's summed embedding per row (codecEmbedIcl without its leading codec_bos row)
__global__ void q3_code_frames_kernel(const bf16* codec_emb, int codec_rows, const bf16* const* cp_emb, int cp_rows, const int* codes, int G,
                                      int H, float* out) {
    const long long r = blockIdx.x;
    for (int i = threadIdx.x; i < H; i += blockDim.x) out[r * H + i] = q3_frame_sum(codec_emb, codec_rows, cp_emb, cp_rows, codes + r * G, G, H, i);
}
// rows: the handle's row capacity (every row's state is reset; rows >= B start done)
__global__ void q3_init_rows_kernel(int B, int L, int* talker_pos, int* row_frame, int* n_frames, int* done, int* n_active, unsigned* seen, int words,
                                    int rows) {
    const int b = threadIdx.x;
    if (b == 0) *n_active = B;
    if (b < rows) { talker_pos[b] = L - 1; row_frame[b] = 0; n_frames[b] = 0; done[b] = b < B ? 0 : 1; }
    for (int i = threadIdx.x; i < rows * words; i += blockDim.x) seen[i] = 0u;
}
// bench only: the talker never emits EOS -- its logit is dropped before the sampler sees the row
__global__ void q3_mask_eos_kernel(float* logits, int V, int eos) {
    if (threadIdx.x == 0 && eos >= 0 && eos < V) logits[(long long)blockIdx.x * V + eos] = -INFINITY;
}

}  // namespace b2a

struct b2a_qwen3_talker {
    int device;
    b2a_qwen3_talker_config cfg;
    b2a_tts* talker = nullptr;
    b2a_tts* pred = nullptr;
    cudaStream_t stream = nullptr;        // = talker->stream
    DBuf<bf16> codec_emb, text_emb, fc1_w, fc2_w;
    DBuf<float> fc1_b, fc2_b;
    std::vector<DBuf<bf16>> cp_emb, cp_head;
    std::vector<CUtensorMap> tm_cp_head;
    int cp_head_rows = 128;
    DBuf<const bf16*> cp_emb_ptrs;
    // code_predictor.small_to_mtp_projection [cpH, H] + bias, present iff the predictor is narrower or wider than the talker
    // (Qwen3TTSCodePredictor.swift:200-238: 1.7B, 2048 -> 1024).  proj_tab holds every embedding row the predictor can be fed,
    // already projected (fp32): codec_embedding's [vocab, cpH], then codec_embedding[k]'s [cp_vocab, cpH] for k = 0 .. G-3
    DBuf<bf16> proj_w;
    DBuf<float> proj_b, proj_tab;
    CUtensorMap tm_proj{};
    int proj_rows = 128;
    DBuf<float> x_in, hid, px, trailing, pad, embeds, tmp_a, tmp_b;
    DBuf<int> codes, out_codes, n_frames, done, n_active, row_frame, n_trailing, ids;
    DBuf<unsigned> seen;
    HBuf<int> h_flag;
    cudaGraphExec_t g_frame = nullptr;
    b2a_qwen3_gen_params g_params{};
    int g_B = 0, g_max_tokens = 0, g_nmax = 0, g_mask = -1;
    const float* g_trailing = nullptr;
    int launches_frame = 0;
    int bench_mask_eos = 0;
    std::atomic<int> cancel{0};

    ~b2a_qwen3_talker() {
        if (g_frame) cudaGraphExecDestroy(g_frame);
        delete pred;
        delete talker;
    }
    int G() const { return cfg.num_code_groups; }
    int rows() const { return talker->rows_cap(); }   // rows of the per-row state buffers
    int H() const { return cfg.hidden_size; }
    int PH() const { return cfg.cp_hidden_size; }
    bool projected() const { return cfg.cp_hidden_size != cfg.hidden_size; }
    const float* proj_table(int k) const {   // the projected table position k + 1 gathers from: 0 = codec_embedding, k = codec_embedding[k-1]
        return proj_tab.p + (k == 0 ? 0 : ((size_t)cfg.vocab_size + (size_t)(k - 1) * cfg.cp_vocab_size) * PH());
    }

    static b2a_llama_config stack_cfg(const b2a_qwen3_talker_config& c, bool predictor) {
        b2a_llama_config l{};
        l.hidden_size = predictor ? c.cp_hidden_size : c.hidden_size;
        l.num_hidden_layers = predictor ? c.cp_num_hidden_layers : c.num_hidden_layers;
        l.intermediate_size = predictor ? c.cp_intermediate_size : c.intermediate_size;
        l.num_attention_heads = predictor ? c.cp_num_attention_heads : c.num_attention_heads;
        l.num_key_value_heads = predictor ? c.cp_num_key_value_heads : c.num_key_value_heads;
        l.head_dim = predictor ? c.cp_head_dim : c.head_dim;
        l.vocab_size = predictor ? c.cp_vocab_size : c.vocab_size;
        l.rms_norm_eps = predictor ? c.cp_rms_norm_eps : c.rms_norm_eps;
        l.rope_theta = predictor ? c.cp_rope_theta : c.rope_theta;
        // plain rotate-half RoPE: factor 1 makes Llama3ScaledRoPE's three wavelength bands collapse to base^(2i/d)
        l.rope_factor = 1.0f; l.rope_low_freq_factor = 1.0f; l.rope_high_freq_factor = 4.0f; l.rope_old_context_len = 8192.0f;
        l.tie_word_embeddings = 0;
        l.max_batch = c.max_batch;
        l.max_context = predictor ? std::max(32, c.num_code_groups + 8) : c.max_context;
        return l;
    }
    static StackSpec talker_spec() { StackSpec s; s.prefix = "model."; s.qk_norm = true; s.has_embed = false; s.head = "codec_head.weight"; s.has_head = true; return s; }
    static StackSpec pred_spec() { StackSpec s; s.prefix = "code_predictor.model."; s.qk_norm = true; s.has_embed = false; s.has_head = false; return s; }

    void check() {
        const b2a_qwen3_talker_config& c = cfg;
        B2A_CHECK(c.head_dim == HD && c.cp_head_dim == HD, B2A_ERR_INVALID_INPUT, "qwen3 talker: head_dim must be 128");
        B2A_CHECK(c.vocab_size >= 1 && c.vocab_size <= q3s::SLOTS && c.cp_vocab_size >= 1 && c.cp_vocab_size <= q3s::SLOTS, B2A_ERR_INVALID_INPUT,
                  "qwen3 talker: codec vocabularies must be <= 4096");
        B2A_CHECK(c.num_code_groups >= 2 && c.num_code_groups <= 32, B2A_ERR_INVALID_INPUT, "qwen3 talker: num_code_groups must be in 2..32");
        B2A_CHECK(c.max_batch >= 1 && c.max_batch <= 32, B2A_ERR_INVALID_INPUT, "qwen3 talker: max_batch must be in 1..32");
    }
    // proj_tab: every table row through the projection, once.  The tables are bf16, so the GEMM reads them without a lo half
    // (hilo = 0); each row is the same linear map the reference applies per position (Qwen3TTS.swift:433-451), to fp32 rounding
    void build_proj_tables() {
        const int Hh = H(), P = PH(), G2 = G() - 2;
        proj_tab.alloc(((size_t)cfg.vocab_size + (size_t)G2 * cfg.cp_vocab_size) * P);
        const CUtensorMap tw = tc::make_tmap_bf16(proj_w.p, P, Hh, tc::BM);
        for (int k = 0; k <= G2; ++k) {
            const bf16* e = k == 0 ? codec_emb.p : cp_emb[k - 1].p;
            const int rows = k == 0 ? cfg.vocab_size : cfg.cp_vocab_size;
            tc::Args a{};
            a.out_f32 = const_cast<float*>(proj_table(k)); a.M = P; a.N = rows; a.K = Hh; a.ldo = P;
            a.m_tiles = cdiv(P, tc::BM); a.k_blocks = Hh / tc::BK; a.stages = tc::Smem<128>::max_stages(); a.hilo = 0;
            a.epi_full = tc::EPI_STORE; a.epi_partial = -1; a.bias = proj_b.p;
            const int n_tiles = cdiv(rows, 128);
            tc::launch<128>(tw, tc::make_tmap_bf16(e, rows, Hh, 128), a, std::max(1, std::min(a.m_tiles, talker->num_sms / n_tiles)), n_tiles,
                            stream);
        }
        B2A_CUDA(cudaStreamSynchronize(stream));
    }
    void alloc_state() {
        stream = talker->stream;
        const int Hh = H(), P = PH(), RC = rows();
        x_in.alloc((size_t)RC * Hh); hid.alloc((size_t)RC * Hh); px.alloc((size_t)RC * P); pad.alloc(Hh);
        B2A_CUDA(cudaMemset(x_in.p, 0, (size_t)RC * Hh * sizeof(float)));
        B2A_CUDA(cudaMemset(hid.p, 0, (size_t)RC * Hh * sizeof(float)));
        B2A_CUDA(cudaMemset(px.p, 0, (size_t)RC * P * sizeof(float)));
        if (projected()) {
            build_proj_tables();
            proj_rows = b2a_tts::pick_tile_rows(P, talker->num_sms);
            tm_proj = tc::make_tmap_bf16(proj_w.p, P, Hh, proj_rows);
        }
        codes.alloc((size_t)RC * G()); n_frames.alloc(RC); done.alloc(RC); n_active.alloc(1); row_frame.alloc(RC); n_trailing.alloc(RC);
        B2A_CUDA(cudaMemset(codes.p, 0, (size_t)RC * G() * sizeof(int)));
        seen.alloc((size_t)RC * cdiv(cfg.vocab_size, 32));
        h_flag.alloc(16);
        std::vector<const bf16*> ptrs;
        for (auto& e : cp_emb) ptrs.push_back(e.p);
        cp_emb_ptrs.upload(ptrs.data(), ptrs.size());
        tm_cp_head.clear();
        cp_head_rows = b2a_tts::pick_tile_rows(cfg.cp_vocab_size, pred->num_sms);
        for (auto& hd : cp_head) tm_cp_head.push_back(tc::make_tmap_bf16(hd.p, cfg.cp_vocab_size, P, cp_head_rows));
        talker->x_ext = x_in.p; talker->normed_out = hid.p;
        pred->x_ext = px.p;
        B2A_CUDA(cudaDeviceSynchronize());
    }

    b2a_qwen3_talker(int dev, const b2a_qwen3_talker_config& c, const TensorTable& tt) : device(dev), cfg(c) {
        check();
        talker = new b2a_tts(dev, stack_cfg(c, false), tt, nullptr, talker_spec());
        pred = new b2a_tts(dev, stack_cfg(c, true), tt, nullptr, pred_spec());
        const int Hh = H(), TH = c.text_hidden_size;
        b2a_tts::upload_bf16(tt, "model.codec_embedding.weight", (int64_t)c.vocab_size * Hh, codec_emb, 0, (size_t)c.vocab_size * Hh);
        b2a_tts::upload_bf16(tt, "model.text_embedding.weight", (int64_t)c.text_vocab_size * TH, text_emb, 0, (size_t)c.text_vocab_size * TH);
        b2a_tts::upload_bf16(tt, "text_projection.linear_fc1.weight", (int64_t)TH * TH, fc1_w, 0, (size_t)TH * TH);
        b2a_tts::upload_bf16(tt, "text_projection.linear_fc2.weight", (int64_t)Hh * TH, fc2_w, 0, (size_t)Hh * TH);
        std::vector<float> b1 = tt.f32("text_projection.linear_fc1.bias", TH), b2 = tt.f32("text_projection.linear_fc2.bias", Hh);
        fc1_b.upload(b1.data(), TH); fc2_b.upload(b2.data(), Hh);
        cp_emb.resize(G() - 1); cp_head.resize(G() - 1);
        const int P = PH();
        for (int i = 0; i < G() - 1; ++i) {
            b2a_tts::upload_bf16(tt, "code_predictor.model.codec_embedding." + std::to_string(i) + ".weight", (int64_t)c.cp_vocab_size * Hh, cp_emb[i], 0,
                                 (size_t)c.cp_vocab_size * Hh);
            b2a_tts::upload_bf16(tt, "code_predictor.lm_head." + std::to_string(i) + ".weight", (int64_t)c.cp_vocab_size * P, cp_head[i], 0,
                                 (size_t)c.cp_vocab_size * P);
        }
        if (projected()) {
            b2a_tts::upload_bf16(tt, "code_predictor.small_to_mtp_projection.weight", (int64_t)P * Hh, proj_w, 0, (size_t)P * Hh);
            std::vector<float> pb = tt.f32("code_predictor.small_to_mtp_projection.bias", P);
            proj_b.upload(pb.data(), P);
        }
        alloc_state();
    }
    // device-drawn weights (bench): every matrix N(0, std^2) bf16, biases 0
    b2a_qwen3_talker(int dev, const b2a_qwen3_talker_config& c, float std, unsigned long long seed) : device(dev), cfg(c) {
        check();
        talker = new b2a_tts(dev, stack_cfg(c, false), std, seed, nullptr, talker_spec());
        pred = new b2a_tts(dev, stack_cfg(c, true), std, seed + 7777, nullptr, pred_spec());
        const int Hh = H(), TH = c.text_hidden_size;
        unsigned long long sd = seed * 7919ull + 3;
        auto rnd = [&](DBuf<bf16>& d, size_t n) {
            d.alloc(n);
            random_bf16_kernel<<<132 * 8, 256, 0, talker->stream>>>(d.p, (long long)n, std, sd++);
            count_launch();
        };
        rnd(codec_emb, (size_t)c.vocab_size * Hh); rnd(text_emb, (size_t)c.text_vocab_size * TH);
        rnd(fc1_w, (size_t)TH * TH); rnd(fc2_w, (size_t)Hh * TH);
        fc1_b.alloc(TH); fc2_b.alloc(Hh);
        B2A_CUDA(cudaMemsetAsync(fc1_b.p, 0, TH * sizeof(float), talker->stream));
        B2A_CUDA(cudaMemsetAsync(fc2_b.p, 0, Hh * sizeof(float), talker->stream));
        cp_emb.resize(G() - 1); cp_head.resize(G() - 1);
        for (int i = 0; i < G() - 1; ++i) { rnd(cp_emb[i], (size_t)c.cp_vocab_size * Hh); rnd(cp_head[i], (size_t)c.cp_vocab_size * PH()); }
        if (projected()) {
            rnd(proj_w, (size_t)PH() * Hh);
            proj_b.alloc(PH());
            B2A_CUDA(cudaMemsetAsync(proj_b.p, 0, PH() * sizeof(float), talker->stream));
        }
        B2A_CUDA(cudaStreamSynchronize(talker->stream));
        alloc_state();
    }

    // ids [n] (device) -> out [n, H]: text_projection(text_embedding(ids)) = fc2(silu(fc1(e)))
    void embed_text_dev(const int* d_ids, int n, float* d_out, cudaStream_t s) {
        const int TH = cfg.text_hidden_size, Hh = H();
        tmp_a.alloc((size_t)n * TH); tmp_b.alloc((size_t)n * TH);
        q3_gather_kernel<<<n, 256, 0, s>>>(text_emb.p, cfg.text_vocab_size, d_ids, 1, 0, tmp_a.p, TH, nullptr, 0);
        q3_linear_kernel<<<dim3(cdiv(TH, 8), n), 256, 0, s>>>(fc1_w.p, fc1_b.p, tmp_a.p, tmp_b.p, TH, TH, 1);
        q3_linear_kernel<<<dim3(cdiv(Hh, 8), n), 256, 0, s>>>(fc2_w.p, fc2_b.p, tmp_b.p, d_out, Hh, TH, 0);
        count_launch(3);
        B2A_CUDA(cudaGetLastError());
    }

    q3s::Args sampler_args(const b2a_qwen3_gen_params& p, bool is_talker, int group) const {
        q3s::Args a{};
        a.logits = is_talker ? talker->logits.p : pred->logits.p;
        a.V = is_talker ? cfg.vocab_size : cfg.cp_vocab_size;
        a.temperature = p.temperature; a.top_p = p.top_p; a.top_k = p.top_k; a.min_p = p.min_p;
        a.rep_penalty = is_talker ? p.repetition_penalty : 1.0f;
        a.eos = is_talker ? cfg.codec_eos_token_id : -1;
        a.suppress_lo = is_talker ? std::max(cfg.vocab_size - 1024, 0) : 0;      // the special-token block except EOS (:383-385)
        a.suppress_hi = is_talker ? cfg.vocab_size : 0;
        a.seen = is_talker ? seen.p : nullptr;
        a.track = is_talker ? 1 : 0;
        a.seed = p.seed;
        a.step = group; a.step_ptr = row_frame.p; a.step_mul = G();
        a.tokens = nullptr; a.filtered = nullptr;
        return a;
    }
    void talker_step(int B, cudaStream_t s, bool with_head) {
        talker->run_layers(B, s);
        if (with_head) talker->run_lm_head(B, s);
    }

    void capture_frame(int B, const b2a_qwen3_gen_params& p, int max_tokens, int nmax) {
        if (g_frame && g_B == B && g_max_tokens == max_tokens && g_nmax == nmax && g_mask == bench_mask_eos && g_trailing == trailing.p &&
            memcmp(&g_params, &p, sizeof(p)) == 0) return;
        if (g_frame) { cudaGraphExecDestroy(g_frame); g_frame = nullptr; }
        cudaStream_t s = stream;
        const int n0 = (int)b2a_launch_count();
        cudaGraph_t g;
        B2A_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
        // 1. talker step on x_in -> hid (final norm), codec logits -> c0
        talker_step(B, s, true);
        if (bench_mask_eos) { q3_mask_eos_kernel<<<B, 32, 0, s>>>(talker->logits.p, cfg.vocab_size, cfg.codec_eos_token_id); count_launch(); }
        {
            q3s::Args a = sampler_args(p, true, 0);
            a.tokens = codes.p; a.tokens_stride = G();
            q3s::launch(a, B, s);
        }
        // 2. code predictor: position 0 = the talker's hidden state, position 1 = codec_embed(c0) -> head 0 -> c1, then
        //    position k + 1 = predictor_embed_{k-1}(c_k) -> head k -> c_{k+1}.  With a projection every position goes through it:
        //    position 0 is projected here from the talker's final-norm operand (rstd and bias in the GEMM's epilogue), the others
        //    are rows of the projected tables; the zero-width copy then only sets the predictor's cache position
        if (projected()) {
            talker->run_head(tm_proj, PH(), px.p, B, s, proj_rows, proj_b.p);
            launch_pdl(q3_copy_rows_kernel, dim3(B), dim3(256), 0, s, (const float*)nullptr, 0ll, px.p, 0, pred->pos.p, 0);
        } else {
            launch_pdl(q3_copy_rows_kernel, dim3(B), dim3(256), 0, s, (const float*)hid.p, (long long)H(), px.p, H(), pred->pos.p, 0);
        }
        pred->run_layers(B, s);
        for (int k = 0; k < G() - 1; ++k) {
            const int id_rows = k == 0 ? cfg.vocab_size : cfg.cp_vocab_size;
            if (projected())
                launch_pdl(q3_gather_kernel<float>, dim3(B), dim3(256), 0, s, proj_table(k), id_rows, (const int*)codes.p, G(), k, px.p, PH(), pred->pos.p, k + 1);
            else
                launch_pdl(q3_gather_kernel<bf16>, dim3(B), dim3(256), 0, s, (const bf16*)(k == 0 ? codec_emb.p : cp_emb[k - 1].p), id_rows,
                           (const int*)codes.p, G(), k, px.p, H(), pred->pos.p, k + 1);
            pred->run_layers(B, s);
            pred->run_final_norm(B, s, false);
            pred->run_head(tm_cp_head[k], cfg.cp_vocab_size, pred->logits.p, B, s, cp_head_rows);
            q3s::Args a = sampler_args(p, false, k + 1);
            a.tokens = codes.p + (k + 1); a.tokens_stride = G();
            q3s::launch(a, B, s);
        }
        // 3. feedback + bookkeeping
        Q3Feedback f{codec_emb.p, cfg.vocab_size, cp_emb_ptrs.p, cfg.cp_vocab_size, codes.p, trailing.p, n_trailing.p, nmax, pad.p, x_in.p,
                     talker->pos.p, row_frame.p, out_codes.p, n_frames.p, done.p, n_active.p, G(), H(), max_tokens, cfg.codec_eos_token_id, bench_mask_eos};
        launch_pdl(q3_feedback_kernel, dim3(B), dim3(256), 0, s, f);
        B2A_CUDA(cudaStreamEndCapture(s, &g));
        B2A_CUDA(cudaGraphInstantiate(&g_frame, g, 0));
        cudaGraphDestroy(g);
        launches_frame = (int)b2a_launch_count() - n0;
        g_B = B; g_params = p; g_max_tokens = max_tokens; g_nmax = nmax; g_mask = bench_mask_eos; g_trailing = trailing.p;
    }

    // positions 0 .. L-2 of the prompt through the talker (no logits needed); leaves x_in = embeds[:, L-1], talker pos = L-1
    void prefill(int B, int L, cudaStream_t s) {
        for (int p = 0; p < L; ++p) {
            launch_pdl(q3_copy_rows_kernel, dim3(B), dim3(256), 0, s, (const float*)(embeds.p + (size_t)p * H()), (long long)L * H(), x_in.p, H(),
                       talker->pos.p, p);
            if (p < L - 1) talker->run_layers(B, s);
        }
    }
};

extern "C" {

int32_t b2a_qwen3_talker_create(int32_t device, const b2a_qwen3_talker_config* cfg, const b2a_tensor* tensors, int32_t n, b2a_qwen3_talker** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_qwen3_talker_create: null out");
        *out = nullptr;
        B2A_CHECK(cfg && tensors && n > 0, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_qwen3_talker_create: missing config or weights");
        TensorTable tt(tensors, n);
        *out = new b2a_qwen3_talker(device, *cfg, tt);
    });
}
int32_t b2a_qwen3_talker_create_random(int32_t device, const b2a_qwen3_talker_config* cfg, float std, uint64_t seed, b2a_qwen3_talker** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_qwen3_talker_create_random: null out");
        *out = nullptr;
        B2A_CHECK(cfg && std > 0.f, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_qwen3_talker_create_random: missing config");
        *out = new b2a_qwen3_talker(device, *cfg, std, seed);
    });
}
void* b2a_qwen3_talker_stream(b2a_qwen3_talker* h) { return h ? (void*)h->stream : nullptr; }
int32_t b2a_qwen3_talker_set_bench_flags(b2a_qwen3_talker* h, int32_t mask_eos) {
    if (!h) return B2A_ERR_INVALID_INPUT;
    h->bench_mask_eos = mask_eos != 0;
    return B2A_OK;
}
int32_t b2a_qwen3_talker_cancel(b2a_qwen3_talker* h) {
    if (!h) return B2A_ERR_INVALID_INPUT;
    h->cancel.store(1);
    return B2A_OK;
}
void b2a_qwen3_talker_destroy(b2a_qwen3_talker* h) { delete h; }

int32_t b2a_qwen3_talker_embed_text(b2a_qwen3_talker* h, const int32_t* ids, int32_t n, float* out) {
    return guarded([&] {
        B2A_CHECK(h && ids && out && n >= 1, B2A_ERR_INVALID_INPUT, "b2a_qwen3_talker_embed_text: bad argument");
        B2A_CUDA(cudaSetDevice(h->device));
        for (int i = 0; i < n; ++i) B2A_CHECK(ids[i] >= 0 && ids[i] < h->cfg.text_vocab_size, B2A_ERR_INVALID_INPUT, "b2a_qwen3_talker_embed_text: id out of range");
        cudaStream_t s = h->stream;
        h->ids.upload(ids, n, s);
        h->embeds.alloc((size_t)n * h->H());
        h->embed_text_dev(h->ids.p, n, h->embeds.p, s);
        B2A_CUDA(cudaMemcpyAsync(out, h->embeds.p, (size_t)n * h->H() * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}
int32_t b2a_qwen3_talker_embed_codec(b2a_qwen3_talker* h, const int32_t* ids, int32_t n, float* out) {
    return guarded([&] {
        B2A_CHECK(h && ids && out && n >= 1, B2A_ERR_INVALID_INPUT, "b2a_qwen3_talker_embed_codec: bad argument");
        B2A_CUDA(cudaSetDevice(h->device));
        for (int i = 0; i < n; ++i) B2A_CHECK(ids[i] >= 0 && ids[i] < h->cfg.vocab_size, B2A_ERR_INVALID_INPUT, "b2a_qwen3_talker_embed_codec: id out of range");
        cudaStream_t s = h->stream;
        h->ids.upload(ids, n, s);
        h->embeds.alloc((size_t)n * h->H());
        q3_gather_kernel<<<n, 256, 0, s>>>(h->codec_emb.p, h->cfg.vocab_size, h->ids.p, 1, 0, h->embeds.p, h->H(), nullptr, 0);
        count_launch();
        B2A_CUDA(cudaMemcpyAsync(out, h->embeds.p, (size_t)n * h->H() * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

// codecEmbedIcl's frame rows (Qwen3TTS.swift:249-265): codes [n, groups] (a frame's first `groups` code groups; groups below
// num_code_groups is the reference's `break`) -> out [n, hidden]
int32_t b2a_qwen3_talker_embed_code_frames(b2a_qwen3_talker* h, const int32_t* codes, int32_t n, int32_t groups, float* out) {
    return guarded([&] {
        B2A_CHECK(h && codes && out && n >= 1 && groups >= 1 && groups <= h->G(), B2A_ERR_INVALID_INPUT, "b2a_qwen3_talker_embed_code_frames: bad argument");
        B2A_CHECK((long long)n * groups < (1ll << 31) && (long long)n * h->H() < (1ll << 40), B2A_ERR_INVALID_INPUT, "b2a_qwen3_talker_embed_code_frames: too many frames");
        for (long long i = 0; i < (long long)n * groups; ++i) {
            const int lim = i % groups == 0 ? h->cfg.vocab_size : h->cfg.cp_vocab_size;
            B2A_CHECK(codes[i] >= 0 && codes[i] < lim, B2A_ERR_INVALID_INPUT, "b2a_qwen3_talker_embed_code_frames: code out of range");
        }
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        h->ids.upload(codes, (size_t)n * groups, s);
        h->embeds.alloc((size_t)n * h->H());
        q3_code_frames_kernel<<<n, 256, 0, s>>>(h->codec_emb.p, h->cfg.vocab_size, h->cp_emb_ptrs.p, h->cfg.cp_vocab_size, h->ids.p, groups, h->H(), h->embeds.p);
        count_launch();
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaMemcpyAsync(out, h->embeds.p, (size_t)n * h->H() * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

int32_t b2a_qwen3_talker_forward(b2a_qwen3_talker* h, const float* input_embeds, int32_t B, int32_t L, float* logits_out, float* hidden_out) {
    return guarded([&] {
        B2A_CHECK(h && input_embeds && B >= 1 && B <= h->cfg.max_batch && L >= 1 && L <= h->cfg.max_context, B2A_ERR_INVALID_INPUT,
                  "b2a_qwen3_talker_forward: bad argument");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        h->talker->set_batch(B); h->talker->drop_graphs();
        h->embeds.upload(input_embeds, (size_t)B * L * h->H(), s);
        h->prefill(B, L, s);
        h->talker_step(B, s, true);
        if (logits_out)
            B2A_CUDA(cudaMemcpyAsync(logits_out, h->talker->logits.p, (size_t)B * h->cfg.vocab_size * sizeof(float), cudaMemcpyDeviceToHost, s));
        if (hidden_out) B2A_CUDA(cudaMemcpyAsync(hidden_out, h->hid.p, (size_t)B * h->H() * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
        B2A_CUDA(cudaGetLastError());
    });
}

int32_t b2a_qwen3_talker_generate(b2a_qwen3_talker* h, const float* input_embeds, int32_t B, int32_t L, const float* trailing_text_hidden,
                                  const int32_t* n_trailing, int32_t n_trailing_max, const float* tts_pad_embed, const b2a_qwen3_gen_params* gp,
                                  int32_t* codes_out, int32_t* n_frames_out, b2a_gen_info* info, b2a_frame_cb on_frame, void* user) {
    return guarded([&] {
        B2A_CHECK(h && input_embeds && tts_pad_embed && gp && codes_out && n_frames_out, B2A_ERR_INVALID_INPUT, "qwen3 generate: null argument");
        B2A_CHECK(B >= 1 && B <= h->cfg.max_batch, B2A_ERR_INVALID_INPUT, "qwen3 generate: batch exceeds max_batch");
        B2A_CHECK(L >= 1 && gp->max_tokens >= 1 && L + gp->max_tokens <= h->cfg.max_context, B2A_ERR_INVALID_INPUT,
                  "qwen3 generate: prompt + max_tokens exceeds max_context");
        B2A_CHECK(n_trailing_max >= 0 && (n_trailing_max == 0 || (trailing_text_hidden && n_trailing)), B2A_ERR_INVALID_INPUT,
                  "qwen3 generate: bad trailing text");
        B2A_CHECK(gp->top_p > 0.f && gp->repetition_penalty > 0.f, B2A_ERR_INVALID_INPUT, "qwen3 generate: bad sampling parameters");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        h->cancel.store(0);
        const int Hh = h->H(), G = h->G(), MT = gp->max_tokens, nmax = std::max(1, n_trailing_max);
        h->talker->set_batch(B); h->pred->set_batch(B);
        h->talker->drop_graphs();
        h->embeds.upload(input_embeds, (size_t)B * L * Hh, s);
        h->trailing.alloc((size_t)B * nmax * Hh);
        std::vector<int> nt(h->rows(), 0);
        if (n_trailing_max > 0) {
            B2A_CUDA(cudaMemcpyAsync(h->trailing.p, trailing_text_hidden, (size_t)B * n_trailing_max * Hh * sizeof(float), cudaMemcpyHostToDevice, s));
            for (int b = 0; b < B; ++b) {
                B2A_CHECK(n_trailing[b] >= 0 && n_trailing[b] <= n_trailing_max, B2A_ERR_INVALID_INPUT, "qwen3 generate: n_trailing out of range");
                nt[b] = n_trailing[b];
            }
        }
        h->n_trailing.upload(nt.data(), nt.size(), s);
        h->pad.upload(tts_pad_embed, Hh, s);
        h->out_codes.alloc((size_t)B * MT * G);
        B2A_CUDA(cudaStreamSynchronize(s));       // nt goes out of scope with the lambda only, but keep uploads ordered before capture
        h->capture_frame(B, *gp, MT, nmax);
        const double t0 = now_s();
        q3_init_rows_kernel<<<1, 256, 0, s>>>(B, L, h->talker->pos.p, h->row_frame.p, h->n_frames.p, h->done.p, h->n_active.p, h->seen.p,
                                              cdiv(h->cfg.vocab_size, 32), h->rows());
        count_launch();
        h->prefill(B, L, s);
        B2A_CUDA(cudaStreamSynchronize(s));
        const double t1 = now_s();
        int steps = 0, emitted = 0;
        bool cancelled = false;
        std::vector<int> hn(h->rows()), hc;
        auto emit = [&]() {          // frames emitted since the last poll -> on_frame
            B2A_CUDA(cudaMemcpy(hn.data(), h->n_frames.p, hn.size() * sizeof(int), cudaMemcpyDeviceToHost));
            hc.resize((size_t)B * MT * G);
            B2A_CUDA(cudaMemcpy(hc.data(), h->out_codes.p, hc.size() * sizeof(int), cudaMemcpyDeviceToHost));
            for (int b = 0; b < B; ++b)
                if (std::min(hn[b], MT) > emitted) on_frame(user, b, emitted, hc.data() + ((size_t)b * MT + emitted) * G);
            ++emitted;
        };
        while (steps < MT) {
            const int burst = on_frame ? 1 : std::min(4, MT - steps);
            for (int i = 0; i < burst; ++i) { B2A_CUDA(cudaGraphLaunch(h->g_frame, s)); count_launch(h->launches_frame); }
            steps += burst;
            B2A_CUDA(cudaMemcpyAsync(h->h_flag.p, h->n_active.p, sizeof(int), cudaMemcpyDeviceToHost, s));
            B2A_CUDA(cudaStreamSynchronize(s));
            if (on_frame) emit();
            if (h->cancel.load()) { cancelled = true; break; }
            if (h->h_flag.p[0] <= 0) break;
        }
        const double t2 = now_s();
        B2A_CHECK(!cancelled, B2A_ERR_CANCELLED, "generation cancelled");
        B2A_CUDA(cudaMemcpy(hn.data(), h->n_frames.p, hn.size() * sizeof(int), cudaMemcpyDeviceToHost));
        B2A_CUDA(cudaMemcpy(codes_out, h->out_codes.p, (size_t)B * MT * G * sizeof(int), cudaMemcpyDeviceToHost));
        int total = 0;
        for (int b = 0; b < B; ++b) { n_frames_out[b] = std::min(hn[b], MT); total += n_frames_out[b]; }
        if (info) {
            info->prompt_token_count = L;
            info->generation_token_count = total;
            info->prefill_time = t1 - t0;
            info->generate_time = t2 - t1;
            info->tokens_per_second = total / std::max(1e-9, t2 - t1);
            info->codec_time = 0;
            size_t fr = 0, tot = 0;
            cudaMemGetInfo(&fr, &tot);
            info->peak_memory_gb = (double)(tot - fr) / 1e9;
        }
    });
}

}  // extern "C"
