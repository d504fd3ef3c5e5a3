// Causal GQA attention over a whole prompt on wgmma for sm_90a (head_dim 128): the Orpheus batched prefill for prompts the SIMT
// prefill_attn_kernel (llama.cu) cannot hold in shared memory, any length up to max_context.
//
// Operands: fp16 hi/lo pairs (x = hi + lo, lo = fp16(x - hi)), three tensor-core products per GEMM, fp32 accumulation and softmax:
//   S = qh kh^T + qh kl^T + ql kh^T          O += ph vh + ph vl + pl vh
// A CPU study of the oracle with the candidate arithmetics emulated (tools/prompt_attention_precision_study.py) puts the next-step
// logits of a 913-token prompt at 7e-7 of the exact run this way; any single product (fp16 q/k, v or p) costs 5e-5 to 2e-3, more
// than the 4e-5 the fp32 path keeps to the per-position replay.
// Layouts written by pack_prompt_kernel, per row b and head, positions padded with zeros to Lp (a multiple of BQ):
//   Qp [B*nq][Lp][256]   q after RoPE: columns [0, 128) hi, [128, 256) lo                 -> A operand of S (K-major: d contiguous)
//   Kp [B*nkv][Lp][256]  k after RoPE, the same                                          -> B operand of S
//   Vt [B*nkv][256][Lp]  v transposed: rows [0, 128) hi, [128, 256) lo (keys contiguous)  -> B operand of O = P V
// One CTA per (128-query tile, query head, row), heaviest tiles first; 288 threads: warps 0-7 = two consumer warpgroups (64 query
// rows each: S into registers, online softmax on the fragments, O += P V with P as the register A operand), warp 8 = TMA producer
// of a 2-stage ring of 64-key K / V tiles.  Key tiles above the diagonal are never loaded; the diagonal ones are masked.
#pragma once
#include "tc_gemm.cuh"

#include <cuda_fp16.h>

namespace b2a {
namespace pfa {

constexpr int BQ = 128, BKV = 64, HDIM = 128, OPW = 2 * HDIM;   // OPW: hi | lo columns of a Qp / Kp row
constexpr int THREADS = 288;
constexpr int CHUNK_Q = BQ * 64 * 2, CHUNK_K = BKV * 64 * 2;     // one 64-column swizzle block of the Q / K tile
constexpr int Q_BYTES = 4 * CHUNK_Q;                             // qh d 0-63, qh d 64-127, ql d 0-63, ql d 64-127: 64 KB
constexpr int K_BYTES = 4 * CHUNK_K, V_HALF = HDIM * BKV * 2;    // 32 KB of K, 2 x 16 KB of V^T
constexpr int STAGE_BYTES = K_BYTES + 2 * V_HALF, STAGES = 2;
constexpr int SMEM_DATA = Q_BYTES + STAGES * STAGE_BYTES;        // 192 KB
constexpr size_t SMEM_BYTES = SMEM_DATA + 256 + 1024;            // + barriers + alignment slack

struct Args {
    __nv_bfloat16* out;   // [2 * T_pad, nq * 128] hi/lo tiles of 64 tokens (the o-projection GEMM's B operand), token b * L + i
    int L, Lp, nq, nkv;
    float scale;
};

__global__ void __launch_bounds__(THREADS, 1)
prompt_attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                   const __grid_constant__ Args a) {
    extern __shared__ __align__(1024) uint8_t pfa_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(pfa_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* sQ = smem;
    uint8_t* sKV = sQ + Q_BYTES;                                   // [stage][K 4 x 8 KB | V^T hi 16 KB | V^T lo 16 KB]
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SMEM_DATA);
    uint64_t *qfull = bars, *full = bars + 1, *empty = bars + 1 + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = gridDim.x - 1 - blockIdx.x, hq = blockIdx.y, b = blockIdx.z;   // the longest key ranges start first
    const int G = a.nq / a.nkv, bkv = b * a.nkv + hq / G;
    const int n_kv = (qt + 1) * (BQ / BKV);                        // key tiles at or below the diagonal
    if (threadIdx.x == 0) {
        tc::tma_prefetch_desc(&tmQ); tc::tma_prefetch_desc(&tmK); tc::tma_prefetch_desc(&tmV);
        tc::mbar_init(qfull, 1);
        for (int i = 0; i < STAGES; ++i) { tc::mbar_init(&full[i], 1); tc::mbar_init(&empty[i], 8); }
        tc::fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            tc::mbar_arrive_expect_tx(qfull, Q_BYTES);
            for (int c = 0; c < 4; ++c) tc::tma_load_3d(sQ + c * CHUNK_Q, &tmQ, qfull, 64 * c, qt * BQ, b * a.nq + hq);
            for (int j = 0; j < n_kv; ++j) {
                const int st = j % STAGES;
                tc::mbar_wait(&empty[st], (uint32_t)(((j / STAGES) & 1) ^ 1));
                uint8_t* sk = sKV + (size_t)st * STAGE_BYTES;
                tc::mbar_arrive_expect_tx(&full[st], STAGE_BYTES);
                for (int c = 0; c < 4; ++c) tc::tma_load_3d(sk + c * CHUNK_K, &tmK, &full[st], 64 * c, j * BKV, bkv);
                tc::tma_load_3d(sk + K_BYTES, &tmV, &full[st], j * BKV, 0, bkv);
                tc::tma_load_3d(sk + K_BYTES + V_HALF, &tmV, &full[st], j * BKV, HDIM, bkv);
            }
        }
        return;
    }
    // consumer warpgroup wg: query rows q0 .. q0 + 63.  Fragment of an m64nN accumulator: this thread holds rows r0 = 16 (warp % 4) +
    // lane / 4 and r0 + 8 of the warpgroup's 64, columns 8 i + 2 (lane % 4) (+1) in registers 4 i (+1) and 4 i + 2 (+1).
    const int wg = warp >> 2;
    const int q0 = qt * BQ + wg * 64, r0 = (warp & 3) * 16 + (lane >> 2), c_lane = 2 * (lane & 3);
    // Key tiles this warpgroup reads: n_kv for wg 1, n_kv - 1 for wg 0, whose queries all precede the last tile's keys.  wg 0 neither
    // waits for nor releases that last tile: empty[] counts arrivals from either warpgroup, so an early release of it would complete
    // the phase that wg 1 still owes for tile n_kv - 3 (the same stage) and let the producer overwrite the stage wg 1 is reading.
    // The producer loads nothing after the last tile, so nothing waits for its release.
    const int n_mine = (q0 + 63) / BKV + 1;
    tc::mbar_wait(qfull, 0);
    const uint32_t sq = tc::smem_u32(sQ) + (uint32_t)(wg * 64 * 128);
    float mx[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float o[64];
#pragma unroll
    for (int e = 0; e < 64; ++e) o[e] = 0.f;
    for (int j = 0; j < n_mine; ++j) {
        const int st = j % STAGES;
        tc::mbar_wait(&full[st], (uint32_t)((j / STAGES) & 1));
        const uint32_t sk = tc::smem_u32(sKV + (size_t)st * STAGE_BYTES);
        float s[32];
#pragma unroll
        for (int e = 0; e < 32; ++e) s[e] = 0.f;
        tc::wg_fence();
#pragma unroll
        for (int k = 0; k < HDIM / 16; ++k) {
            const uint32_t ca = (uint32_t)(k >> 2), kk = (uint32_t)(2 * (k & 3));
            const uint64_t qh = tc::make_smem_desc(sq + ca * CHUNK_Q) + kk, ql = tc::make_smem_desc(sq + (2 + ca) * CHUNK_Q) + kk;
            const uint64_t kh = tc::make_smem_desc(sk + ca * CHUNK_K) + kk, kl = tc::make_smem_desc(sk + (2 + ca) * CHUNK_K) + kk;
            tc::wgmma_f16_n64(s, qh, kh, k ? 1u : 0u);
            tc::wgmma_f16_n64(s, qh, kl, 1u);
            tc::wgmma_f16_n64(s, ql, kh, 1u);
        }
        tc::wg_commit();
        tc::wg_wait0();
        tc::wg_fence_operand(s);
        // scale, causal mask (only the tiles that reach past this warpgroup's first query), running maximum
        const bool diag = j * BKV + BKV - 1 > q0;
        float mnew[2] = {mx[0], mx[1]};
#pragma unroll
        for (int g = 0; g < 8; ++g)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float v = s[4 * g + e] * a.scale;
                if (diag && j * BKV + 8 * g + c_lane + (e & 1) > q0 + r0 + 8 * (e >> 1)) v = -INFINITY;
                s[4 * g + e] = v;
                mnew[e >> 1] = fmaxf(mnew[e >> 1], v);
            }
        float corr[2];
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {                           // the four lanes of a quad share a row
            mnew[rh] = fmaxf(mnew[rh], __shfl_xor_sync(0xffffffffu, mnew[rh], 1));
            mnew[rh] = fmaxf(mnew[rh], __shfl_xor_sync(0xffffffffu, mnew[rh], 2));
            corr[rh] = __expf(mx[rh] - mnew[rh]);                  // key 0 is in tile 0: mnew is finite, corr = 0 on the first tile
            mx[rh] = mnew[rh];
            l[rh] *= corr[rh];
        }
#pragma unroll
        for (int g = 0; g < 16; ++g)
#pragma unroll
            for (int e = 0; e < 4; ++e) o[4 * g + e] *= corr[e >> 1];
        // P = exp(S - max) as fp16 hi / lo A fragments: k-step kk (keys 16 kk .. + 15) = column groups 2 kk, 2 kk + 1
        uint32_t ph[4][4], pl[4][4];
#pragma unroll
        for (int g = 0; g < 8; ++g)
#pragma unroll
            for (int rh = 0; rh < 2; ++rh) {
                const float p0 = __expf(s[4 * g + 2 * rh] - mx[rh]), p1 = __expf(s[4 * g + 2 * rh + 1] - mx[rh]);
                const __half2 hh = __floats2half2_rn(p0, p1);
                const float2 hf = __half22float2(hh);
                const __half2 hl = __floats2half2_rn(p0 - hf.x, p1 - hf.y);
                const float2 lf = __half22float2(hl);
                l[rh] += (hf.x + lf.x) + (hf.y + lf.y);            // the sum of what the tensor core will actually multiply
                ph[g >> 1][(g & 1) * 2 + rh] = *reinterpret_cast<const uint32_t*>(&hh);
                pl[g >> 1][(g & 1) * 2 + rh] = *reinterpret_cast<const uint32_t*>(&hl);
            }
        tc::wg_fence();
#pragma unroll
        for (int kk = 0; kk < BKV / 16; ++kk) {
            const uint64_t vh = tc::make_smem_desc(sk + K_BYTES) + (uint64_t)(2 * kk);
            const uint64_t vl = tc::make_smem_desc(sk + K_BYTES + V_HALF) + (uint64_t)(2 * kk);
            tc::wgmma_f16_rs_n128(o, ph[kk], vh, 1u);
            tc::wgmma_f16_rs_n128(o, ph[kk], vl, 1u);
            tc::wgmma_f16_rs_n128(o, pl[kk], vh, 1u);
        }
        tc::wg_commit();
        tc::wg_wait0();
        tc::wg_fence_operand(o);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&empty[st]);
    }
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
        l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 1);
        l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 2);
    }
    const long long ldo = (long long)a.nq * HDIM;
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
        const int qrow = q0 + r0 + 8 * rh;
        if (qrow >= a.L) continue;
        const float inv = 1.0f / l[rh];
        const long long tok = (long long)b * a.L + qrow;
        const long long r = (tok / 64) * 128 + (tok % 64);        // tc::store_hilo's row of token tok in 64-token tiles
        __nv_bfloat16* phi = a.out + r * ldo + hq * HDIM + c_lane;
        __nv_bfloat16* plo = phi + 64 * ldo;
#pragma unroll
        for (int g = 0; g < 16; ++g) {
            const float o0 = o[4 * g + 2 * rh] * inv, o1 = o[4 * g + 2 * rh + 1] * inv;
            const __nv_bfloat16 h0 = __float2bfloat16_rn(o0), h1 = __float2bfloat16_rn(o1);
            *reinterpret_cast<__nv_bfloat162*>(phi + 8 * g) = __halves2bfloat162(h0, h1);
            *reinterpret_cast<__nv_bfloat162*>(plo + 8 * g) =
                __halves2bfloat162(__float2bfloat16_rn(o0 - __bfloat162float(h0)), __float2bfloat16_rn(o1 - __bfloat162float(h1)));
        }
    }
}

// q|k|v GEMM output qkv fp32 [B * L, (nq + 2 nkv) * 128] -> the kernel's operands, and RoPE'd K / raw V into the fp32 cache
// [B][nkv][max_ctx][128] at positions 0 .. L-1 (rows >= L are not touched).  One CTA per (64-position tile, row, head), heads
// [0, nq) = queries, [nq, nq + nkv) = keys and values.  rope [max_ctx][64] = (cos, sin) of position / freqs[d] (rope_table_kernel).
// V goes through shared memory so that the transposed rows are written 128 bytes at a time.  Positions in [L, Lp) are zeros.
// qnorm / knorm (nullable, [128] each): per-head RMSNorm x * rsqrt(mean(x^2) + eps) * w of q and k before RoPE (Qwen3 stacks); the cache
// then holds the normalised, rotated K, as the decode step writes it.
__global__ void __launch_bounds__(256)
pack_prompt_kernel(const float* __restrict__ qkv, const float2* __restrict__ rope, __half* __restrict__ Qp, __half* __restrict__ Kp,
                   __half* __restrict__ Vt, float* __restrict__ kcache, float* __restrict__ vcache, int L, int Lp, int nq, int nkv,
                   int max_ctx, const float* __restrict__ qnorm, const float* __restrict__ knorm, float qk_eps) {
    __shared__ __half sv[2][64][HDIM + 2];
    __shared__ float srs[64];                                      // q/k norm: rstd of each position's vector
    const int b = blockIdx.y, hd = blockIdx.z, t0 = blockIdx.x * 64;
    const bool is_q = hd < nq;
    const int h = is_q ? hd : hd - nq, ld = (nq + 2 * nkv) * HDIM;
    const float* base = qkv + (long long)b * L * ld;
    __half* dst = is_q ? Qp + ((long long)b * nq + h) * Lp * OPW : Kp + ((long long)b * nkv + h) * Lp * OPW;
    const int col = is_q ? h * HDIM : (nq + h) * HDIM;
    float* kc = kcache + (((long long)b * nkv + h) * max_ctx) * HDIM;
    float* vc = vcache + (((long long)b * nkv + h) * max_ctx) * HDIM;
    const float* gain = is_q ? qnorm : knorm;
    if (gain) {   // one warp per position, the decode step's reduction (attn_decode_cluster_kernel)
        const int lane = threadIdx.x & 31;
        for (int r = threadIdx.x >> 5; r < 64; r += 8) {
            const int t = t0 + r;
            if (t >= L) continue;
            const float4 x = reinterpret_cast<const float4*>(base + (long long)t * ld + col)[lane];
            const float ss = warp_sum(x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w);
            if (lane == 0) srs[r] = rsqrtf(ss * (1.0f / HDIM) + qk_eps);
        }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < 64 * (HDIM / 2); i += 256) {
        const int r = i / (HDIM / 2), d = i - r * (HDIM / 2), t = t0 + r;
        float y1 = 0.f, y2 = 0.f;
        if (t < L) {
            const float2 cs = rope[t * (HDIM / 2) + d];
            const float* x = base + (long long)t * ld + col;
            float x1 = x[d], x2 = x[d + HDIM / 2];
            if (gain) { x1 = x1 * srs[r] * gain[d]; x2 = x2 * srs[r] * gain[d + HDIM / 2]; }
            y1 = x1 * cs.x - x2 * cs.y; y2 = x2 * cs.x + x1 * cs.y;
            if (!is_q) { kc[(long long)t * HDIM + d] = y1; kc[(long long)t * HDIM + d + HDIM / 2] = y2; }
        }
        __half* row = dst + (long long)t * OPW;
        const __half h1 = __float2half_rn(y1), h2 = __float2half_rn(y2);
        row[d] = h1; row[d + HDIM / 2] = h2;
        row[HDIM + d] = __float2half_rn(y1 - __half2float(h1));
        row[HDIM + d + HDIM / 2] = __float2half_rn(y2 - __half2float(h2));
    }
    if (is_q) return;
    for (int i = threadIdx.x; i < 64 * HDIM; i += 256) {
        const int r = i / HDIM, d = i - r * HDIM, t = t0 + r;
        float v = 0.f;
        if (t < L) {
            v = base[(long long)t * ld + (nq + nkv + h) * HDIM + d];
            vc[(long long)t * HDIM + d] = v;
        }
        const __half hi = __float2half_rn(v);
        sv[0][r][d] = hi;
        sv[1][r][d] = __float2half_rn(v - __half2float(hi));
    }
    __syncthreads();
    __half* vt = Vt + ((long long)b * nkv + h) * OPW * Lp;
    for (int i = threadIdx.x; i < 2 * HDIM * 64; i += 256) {
        const int c = i >> 6, r = i & 63;                          // row c of V^T (hi rows, then lo rows), position t0 + r
        vt[(long long)c * Lp + t0 + r] = sv[c / HDIM][r][c % HDIM];
    }
}

}  // namespace pfa
}  // namespace b2a
