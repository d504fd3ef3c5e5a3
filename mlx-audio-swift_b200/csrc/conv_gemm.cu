// The codec conv GEMM (conv_gemm.cuh): the kernel, the hi/lo weight operand and the one launch path that SNAC, Vocos and the
// test entry share.
#include "conv_gemm.cuh"

#include <algorithm>

namespace b2a {
namespace cg {

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
                    if (a.hl) store_hilo(a.hl, a.ldh, tok, co, val, HALF);
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
                    store_hilo(a.hl, a.ldh, row, m, val, HALF);
                    store_hilo(a.hl, a.ldh, row + 1, a.M + m, val, HALF);
                } else {
                    store_hilo(a.hl, a.ldh, n, m, val, HALF);
                }
            }
        }
    }
}

void TcW::build(const std::vector<float>& W, int M_, int K_) {
    M = M_; K = K_;
    std::vector<__nv_bfloat16> h((size_t)M * K), l((size_t)M * K);
    for (size_t i = 0; i < h.size(); ++i) {
        h[i] = __float2bfloat16_rn(W[i]);
        l[i] = __float2bfloat16_rn(W[i] - __bfloat162float(h[i]));
    }
    hi.upload(h.data(), h.size());
    lo.upload(l.data(), l.size());
    B2A_CUDA(cudaDeviceSynchronize());
    th = make_tmap_bf16(hi.p, M, K, BM);
    tl = make_tmap_bf16(lo.p, M, K, BM);
}

void launch(const TcW& W, const __nv_bfloat16* X, long long x_rows, Args a, long long max_ctas, cudaStream_t s) {
    // the shared-memory limit is a per-device setting: set here, every engine and device gets it without a set-up call of its own
    B2A_CUDA(cudaFuncSetAttribute(conv_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
    a.M = W.M; a.K = W.K;
    a.m_tiles = cdiv(W.M, BM); a.k_blocks = W.K / BK; a.n_tiles = cdiv(a.N, HALF);
    const CUtensorMap tb = make_tmap_bf16(X, x_rows, W.K, BN);
    const long long tiles = (long long)a.n_tiles * a.m_tiles;
    launch_pdl(conv_gemm_kernel, dim3((unsigned)std::min<long long>(max_ctas, tiles)), dim3(CG_THREADS), SMEM_BYTES, s, W.th, W.tl, tb, a);
}

}  // namespace cg
}  // namespace b2a
