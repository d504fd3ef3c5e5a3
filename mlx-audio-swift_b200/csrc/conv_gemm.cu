// The codec conv GEMM and the implicit convolution (conv_gemm.cuh): the machine they share, their two epilogues, the hi/lo weight
// operand and the one launch path of each that the engines and the test entries share.
#include "conv_gemm.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace b2a {
namespace cg {

// The machine both kernels run.  Shared memory holds the ring of STAGES (Wh, Wl, X) stages, the staged accumulator, the zero
// block and the full / empty barriers.  The producer warp walks each work item's k-blocks as (tap j, channel block cb),
// kb = j * cblocks + cb, and load_b(dst, bar, nt, j, cb) issues the activation tile of token tile nt.  The four wgmma warpgroups
// call epi(nt, mt, row, c0, mma) per work item, where row is the thread's accumulator row, c0 its first token column, and
// mma(sum) runs the item's k-blocks in segments of seg (the accumulator of each is drained and added in registers, RN) and
// leaves the thread its 16 sums of hi and lo columns.  Whatever the epilogue loads before calling mma overlaps the MMAs.
template <int F16, class LoadB, class Epi>
__device__ __forceinline__ void mainloop(const CUtensorMap* tmA, const CUtensorMap* tmA2, const CUtensorMap* tmB, long long tiles,
                                         int m_tiles, int taps, int cblocks, int seg, LoadB load_b, Epi epi) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    float* sacc = reinterpret_cast<float*>(smem + (size_t)STAGES * STAGE);                     // [128][ACC_LD]
    uint8_t* zero_w = reinterpret_cast<uint8_t*>(sacc + (size_t)BM * ACC_LD);                  // [64][64] bf16 zeros (1024-aligned)
    uint64_t* full = reinterpret_cast<uint64_t*>(zero_w + ZERO_BYTES);
    uint64_t* empty = full + STAGES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(tmA); tma_prefetch_desc(tmA2); tma_prefetch_desc(tmB);
        for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], EPI_WARPS); }
        fence_barrier_init();
    }
    for (int i = threadIdx.x; i < ZERO_BYTES / 16; i += blockDim.x) reinterpret_cast<uint4*>(zero_w)[i] = make_uint4(0, 0, 0, 0);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy stores -> visible to the tensor core
    __syncthreads();
    const int k_blocks = taps * cblocks;

    if (warp == EPI_WARPS) {
        if (lane == 0) {
            int stage = 0; uint32_t phase = 0;
            for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {   // tile id = n_tile * m_tiles + m_tile, dealt round-robin
                const int nt = (int)(t / m_tiles), mt = (int)(t - (long long)nt * m_tiles);
                int kb = 0;
                for (int j = 0; j < taps; ++j) {
                    for (int cb = 0; cb < cblocks; ++cb, ++kb) {
                        mbar_wait(&empty[stage], phase ^ 1);
                        uint8_t* s0 = smem + (size_t)stage * STAGE;
                        mbar_arrive_expect_tx(&full[stage], STAGE);
                        tma_load_2d(s0, tmA, &full[stage], kb * BK, mt * BM);
                        tma_load_2d(s0 + A_BYTES, tmA2, &full[stage], kb * BK, mt * BM);
                        load_b(s0 + 2 * A_BYTES, &full[stage], nt, j, cb);
                        if (++stage == STAGES) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
    } else {
        const int q = warp & 3, c0 = (warp >> 2) * 16;
        const int wg = warp >> 2, row_blk = wg & 1, col_blk = wg >> 1;   // this warpgroup's 64 x 64 block of the accumulator
        auto wgmma16 = [&](float (&d)[32], uint64_t da, uint64_t db, uint32_t sc) {
            if constexpr (F16) wgmma_f16_n64(d, da, db, sc); else wgmma_bf16_n64(d, da, db, sc);
        };
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
                    wgmma16(acc, ad + off, bd + off, (kb == kb0 && k == 0) ? 0u : 1u);     // Wh * [Xh; Xl]
                    wgmma16(acc, a2d + (col_blk == 0 ? off : 0), bd + off, 1u);          // Wl * Xh -> columns [0, 64) (else + 0)
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
        auto mma = [&](float (&sum)[16]) {
            for (int kb0 = 0; kb0 < k_blocks; kb0 += seg) {
                mma_block(kb0, min(k_blocks, kb0 + seg));
                float v[16], w[16];
                ld_acc16(arow + c0, v);
                ld_acc16(arow + c0 + HALF, w);
                if (kb0 == 0) {
#pragma unroll
                    for (int j = 0; j < 16; ++j) sum[j] = v[j] + w[j];
                } else {
#pragma unroll
                    for (int j = 0; j < 16; ++j) sum[j] += v[j] + w[j];
                }
            }
        };
        for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
            const int nt = (int)(t / m_tiles), mt = (int)(t - (long long)nt * m_tiles);
            epi(nt, mt, q * 32 + lane, c0, mma);
        }
    }
}

static __global__ void __launch_bounds__(CG_THREADS, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                 const __grid_constant__ CUtensorMap tmB, Args a) {
    const bool rmw = a.epi == E_NOISE || a.epi == E_ADD || a.epi == E_ADD_HILO;
    auto load_b = [&](uint8_t* dst, uint64_t* bar, int nt, int, int kb) { tma_load_2d(dst, &tmB, bar, kb * BK, nt * BN); };
    auto epi = [&](int nt, int mt, int row, int c0, auto& mma) {
        const int lane = threadIdx.x & 31;
        const int m = mt * BM + row;
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
        float sum[16];
        mma(sum);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const long long n = n_first + j;      // token (row of X)
            const float nz = a.epi == E_NOISE ? __shfl_sync(0xffffffffu, nz_lane, j) : 0.f;
            if (n >= a.N || !m_ok) continue;
            float val = sum[j] + bias;
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
    };
    mainloop<0>(&tmA, &tmA2, &tmB, (long long)a.n_tiles * a.m_tiles, a.m_tiles, 1, a.k_blocks, a.k_blocks, load_b, epi);
}

}  // namespace cg

namespace ic {

using namespace b2a::cg;

template <int F16>   // == Args::f16 (a template parameter so that the wgmma issue has no branch)
static __global__ void __launch_bounds__(CG_THREADS, 1)
implicit_conv_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                     const __grid_constant__ CUtensorMap tmB, Args a) {
    const int k_blocks = a.taps * a.cblocks;
    const long long To = (long long)a.T * a.up;
    const long long plane = (long long)a.B * (a.Hout + To) * a.Cout;
    auto load_b = [&](uint8_t* dst, uint64_t* bar, int nt, int j, int cb) {     // n_tile = b * t_tiles + tt
        const int b = nt / a.t_tiles, tt = nt - b * a.t_tiles;
        tma_load_4d(dst, &tmB, bar, cb * BK, tt * HALF + a.shift0 + j * a.dil, b, 0);
    };
    auto epi = [&](int nt, int mt, int row, int c0, auto& mma) {
        const int b = nt / a.t_tiles, tt = nt - b * a.t_tiles;
        const int m = mt * BM + row;
        const bool m_ok = m < a.M;
        int rho = 0, co = m;
        if (a.up > 1) { rho = m / a.Cout; co = m - rho * a.Cout; }
        float bias = 0.f, gm = 1.f, sa = 0.f, sb = 0.f, ws = 1.f;
        if (m_ok) {
            if (a.wscale) ws = a.wscale[m];
            if (a.bias) bias = a.bias[co];
            if (a.gamma) gm = a.gamma[co];
            if (a.sa) { sa = a.sa[co]; sb = a.sb[co]; }
        }
        const int t_first = tt * HALF + c0;
        // the residual operand does not depend on the accumulator: 16 independent loads issued before the MMA wait
        float xv[16];
        if (a.add) {
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int tf = t_first + j;
                xv[j] = (m_ok && tf < a.T) ? a.xo[((long long)b * To + (long long)tf * a.up + rho) * a.Cout + co] : 0.f;
            }
        }
        float sum[16];
        mma(sum);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int tf = t_first + j;
            if (tf >= a.T || !m_ok) continue;
            float val = sum[j] * ws + bias;
            if (a.bias_twice_t0 && tf == 0) val += bias;
            if (a.gelu) val = 0.5f * val * (1.0f + erff(val * 0.70710678118654752f));
            val *= gm;
            if (a.add) val += xv[j];
            const long long fo = (long long)tf * a.up + rho;
            if (a.xo) a.xo[((long long)b * To + fo) * a.Cout + co] = val;
            if (a.hl) {
                const float hv = a.sa ? snake_inv(val, sa, sb) : a.elu ? (val > 0.f ? val : expm1f(val)) : val;
                const long long idx = ((long long)b * (a.Hout + To) + a.Hout + fo) * a.Cout + co;
                put_hilo16(reinterpret_cast<uint16_t*>(a.hl), plane, idx, hv, a.f16);
            }
        }
    };
    mainloop<F16>(&tmA, &tmA2, &tmB, (long long)a.B * a.t_tiles * a.m_tiles, a.m_tiles, a.taps, a.cblocks,
                  a.seg_kb > 0 ? a.seg_kb : k_blocks, load_b, epi);
}

}  // namespace ic

namespace cg {

std::vector<float> TcW::pad_k(const std::vector<float>& W, int M, int taps, int Cin) {
    const int cb = cdiv(Cin, BK);
    const size_t K = (size_t)taps * cb * BK;
    std::vector<float> g((size_t)M * K, 0.f);
    for (int m = 0; m < M; ++m)
        for (int j = 0; j < taps; ++j)
            memcpy(&g[(size_t)m * K + (size_t)j * cb * BK], &W[((size_t)m * taps + j) * Cin], (size_t)Cin * sizeof(float));
    return g;
}

void TcW::build(const std::vector<float>& W, int M_, int taps_, int Cin_, int f16_) {
    M = M_; taps = taps_; Cin = Cin_; cblocks = cdiv(Cin, BK); f16 = f16_;
    const size_t K = (size_t)taps * cblocks * BK;
    std::vector<float> g = pad_k(W, M, taps, Cin);
    if (f16) {
        // fp16 pairs: a weight of magnitude 0.01 has a SUBNORMAL lo half (|lo| < 2^-11 |w| < 6.1e-5), i.e. ~18 bits instead of 22.
        // Store row m times 2^e with max|w_m| * 2^e in [8192, 16384) and undo the (exact) scaling in the epilogue.
        std::vector<float> rs((size_t)M, 1.f);
        for (int m = 0; m < M; ++m) {
            float mx = 0.f;
            for (size_t k = 0; k < K; ++k) mx = std::max(mx, fabsf(g[(size_t)m * K + k]));
            if (mx > 0.f && std::isfinite(mx)) {
                int e = 0;
                frexpf(mx, &e);                              // mx = f * 2^e, f in [0.5, 1)
                const float sc = ldexpf(1.0f, 14 - e);       // mx * sc in [8192, 16384)
                for (size_t k = 0; k < K; ++k) g[(size_t)m * K + k] *= sc;
                rs[m] = 1.0f / sc;
            }
        }
        rscale.upload(rs.data(), rs.size());
    }
    std::vector<uint16_t> h(g.size()), l(g.size());
    for (size_t i = 0; i < g.size(); ++i) split16(g[i], f16, h[i], l[i]);
    hi.upload(reinterpret_cast<const __nv_bfloat16*>(h.data()), h.size());
    lo.upload(reinterpret_cast<const __nv_bfloat16*>(l.data()), l.size());
    B2A_CUDA(cudaDeviceSynchronize());
    th = make_tmap_bf16(hi.p, M, (long long)K, BM, f16);
    tl = make_tmap_bf16(lo.p, M, (long long)K, BM, f16);
}

void TcW::set_bias(const std::vector<float>& b) { bias.upload(b.data(), b.size()); has_bias = true; B2A_CUDA(cudaDeviceSynchronize()); }

// The shared-memory limit is a per-device setting: set at every launch, every engine and device gets it without a set-up call
// of its own.
template <class A>
static void launch_ring(void (*kernel)(CUtensorMap, CUtensorMap, CUtensorMap, A), const TcW& W, const CUtensorMap& tb, const A& a,
                        long long tiles, long long max_ctas, cudaStream_t s) {
    B2A_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
    launch_pdl(kernel, dim3((unsigned)std::min<long long>(max_ctas, tiles)), dim3(CG_THREADS), SMEM_BYTES, s, W.th, W.tl, tb, a);
}

void launch(const TcW& W, const __nv_bfloat16* X, long long x_rows, Args a, long long max_ctas, cudaStream_t s) {
    a.M = W.M; a.k_blocks = W.taps * W.cblocks; a.K = a.k_blocks * BK;
    a.m_tiles = cdiv(W.M, BM); a.n_tiles = cdiv(a.N, HALF);
    const CUtensorMap tb = make_tmap_bf16(X, x_rows, a.K, BN);
    launch_ring(conv_gemm_kernel, W, tb, a, (long long)a.n_tiles * a.m_tiles, max_ctas, s);
}

}  // namespace cg

namespace ic {

// k-blocks per accumulation segment (Args::seg_kb)
constexpr int SEG_KB = 4;

void launch(const cg::TcW& W, const __nv_bfloat16* in, long long in_frames, Args a, long long max_ctas, cudaStream_t s) {
    a.M = W.M; a.m_tiles = cdiv(W.M, BM);
    a.taps = W.taps; a.cblocks = W.cblocks;
    if (a.dil == 0) a.dil = 1;
    if (a.up == 0) a.up = 1;
    a.Cout = W.M / a.up;
    a.t_tiles = cdiv(a.T, HALF);
    a.bias = W.has_bias ? W.bias.p : nullptr;
    a.f16 = W.f16;
    a.seg_kb = SEG_KB;
    a.wscale = W.f16 ? W.rscale.p : nullptr;
    const CUtensorMap tb = make_tmap_planes(in, W.Cin, in_frames, a.B, HALF, W.f16);
    launch_ring(a.f16 ? implicit_conv_kernel<1> : implicit_conv_kernel<0>, W, tb, a, (long long)a.B * a.t_tiles * a.m_tiles, max_ctas, s);
}

}  // namespace ic
}  // namespace b2a
