// Fused SNAC ResidualUnit / NoiseBlock for the narrow, memory-bound decoder stages (C = 64 or 128 channels):
//     RU    (Layers.swift:202-232):  y = x + W * snake_b(dw7_dil(snake_a(x)) + b_dw) + b_pw
//     NOISE (Layers.swift:263-279):  y = x + n[t] * (W x)
// ONE kernel per unit: fp32 activation in, fp32 activation out (8 B per element instead of the 20 B the unfused
// dw7 -> hi/lo -> GEMM -> read-modify-write sequence moves).  The depthwise conv, both Snakes and the fp32 -> bf16 hi/lo split
// run on CUDA cores straight into the wgmma B-operand tile in shared memory (K-major, 128-byte swizzle -- the layout TMA would
// have produced); the 1x1 conv is a wgmma against weights that stay resident in shared memory for the whole kernel (both
// bf16 halves, loaded once by TMA); the accumulator, in the registers of the team's two warpgroups, picks up bias + residual
// and leaves as fp32 (plus, for the last unit of a block, the Snake'd hi/lo 2-tap im2col the next transposed conv reads).
// A CTA is two independent TEAMS of 8 warps (two warpgroups) working on alternating tiles, each with its own staging buffers
// and operand tile: while one team waits on memory or the tensor core the other one computes, which is the overlap a
// producer/consumer warp specialisation would give, with none of its plumbing.
// The MMA always has M = 128 rows (warpgroup t of a team takes rows 64 t .. 64 t + 63) and K = 128.  C = 128: rows = output
// channels, the two k-blocks are the two channel halves of one 64-token tile.  C = 64: the weight operand is the block-diagonal
// [W 0; 0 W] and the two k-blocks hold two consecutive 64-token sub-tiles, so rows 0..63 / 64..127 of the accumulator are the
// 64 output channels of sub-tile 0 / 1 and both warpgroups do useful work.  C is a template parameter so that every activation address in the inner
// loops is base + immediate (the first version spent ~100 instructions per element, mostly on 64-bit address arithmetic).
#pragma once
#include "conv_gemm.cuh"

namespace b2a {
namespace rf {

using namespace b2a::tc;

constexpr int TOK = 64;                       // tokens per tile (x hi/lo = 128 B-operand rows)
constexpr int TEAM_WARPS = 8, TEAM_THREADS = TEAM_WARPS * 32, TEAMS = 2, THREADS = TEAMS * TEAM_THREADS;
constexpr int OP_KB_BYTES = 128 * BK * 2;     // one k-block of the operand tile: 128 rows x 64 bf16 = 16 KB
constexpr int W_KB_BYTES = BM * BK * 2;       // one k-block of one weight half: 128 rows x 64 bf16 = 16 KB
enum : int { MODE_RU = 0, MODE_NOISE = 1 };

struct Args {
    const float* x;            // [B*T, C] fp32
    float* y;                  // [B*T, C] fp32 (must not alias x: neighbouring tiles read x's halo)
    int C, T, B, mode, dil;
    const float* dw_w;         // [C, 7]
    const float* dw_b;         // [C] or null
    const float* a_in;         // Snake alpha before the depthwise conv
    const float* a_mid;        // Snake alpha after it
    const float* pw_bias;      // [C] or null
    const float* noise;        // [B*T] or null => counter-based N(0,1) from seed
    unsigned long long seed;
    __nv_bfloat16* hl;         // optional: Snake(a_next) of y as the next block's 2-tap im2col (conv_gemm.cuh "dual"), ld = 2*C
    const float* a_next;
    int fs, fpad;              // fs > 0: hl is instead the 2-frame im2col of the encoder's strided conv (conv_gemm.cuh put_frames)
    int tiles_per_utt;
    long long n_tiles;
};

static inline size_t team_bytes(int dil, int mode) {
    const size_t s_rows = mode == MODE_RU ? (size_t)(TOK + 6 * dil) : 0;
    return (((size_t)2 * OP_KB_BYTES + s_rows * BK * sizeof(float)) + 1023) / 1024 * 1024;   // operand tiles need 1024-B alignment
}
static inline size_t smem_bytes(int dil, int mode) {
    return 1024 + (size_t)4 * W_KB_BYTES + (size_t)TEAMS * team_bytes(dil, mode) + 256;
}

__device__ __forceinline__ void team_sync(int team) {
    asm volatile("bar.sync %0, %1;" ::"r"(team + 1), "n"(TEAM_THREADS) : "memory");
}
// byte offset of element (row, col) of a [rows][64] bf16 K-major SWIZZLE_128B tile
__device__ __forceinline__ uint32_t sw128(int row, int col) {
    return (uint32_t)(row * 128 + ((((col >> 3) ^ (row & 7)) << 4) | ((col & 7) << 1)));
}

// MODE_RU: DIL in {1, 3, 9}; MODE_NOISE: DIL = 0.  The input rows of the NEXT (tile, k-block) unit are prefetched into
// registers (P float4 per thread) before the current unit's depthwise conv / MMA / epilogue, so their latency is hidden.
template <int MODE, int DIL, int C>
static __global__ void __launch_bounds__(THREADS, 1)
ru_fused_kernel(const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, Args a) {
    static_assert(C == 64 || C == 128, "C must be 64 or 128");
    constexpr int ROWS = MODE == MODE_RU ? TOK + 6 * DIL : TOK;
    constexpr int HALO = 3 * DIL;
    constexpr int P = (ROWS * 16 + TEAM_THREADS - 1) / TEAM_THREADS;
    constexpr int TT = C == 64 ? 2 * TOK : TOK;                 // tokens per tile
    constexpr int KBS = 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* wh = smem;                                         // [2][128][64] bf16
    uint8_t* wl = wh + (size_t)KBS * W_KB_BYTES;
    uint8_t* team_base = wl + (size_t)KBS * W_KB_BYTES;
    constexpr size_t tbytes = (((size_t)KBS * OP_KB_BYTES + (size_t)(MODE == MODE_RU ? ROWS : 0) * BK * sizeof(float)) + 1023) / 1024 * 1024;
    uint64_t* wbar = reinterpret_cast<uint64_t*>(team_base + TEAMS * tbytes);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int team = warp / TEAM_WARPS, tt_id = tid % TEAM_THREADS;
    uint8_t* op = team_base + team * tbytes;                    // [2][128][64] bf16 (rows 0..63 hi, 64..127 lo)
    float* S = reinterpret_cast<float*>(op + (size_t)KBS * OP_KB_BYTES);   // [ROWS][64] fp32

    if (tid == 0) {
        tma_prefetch_desc(&tmWh); tma_prefetch_desc(&tmWl);
        mbar_init(wbar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (tid == 0) {   // weights: both halves, both k-blocks, once per CTA
        mbar_arrive_expect_tx(wbar, (uint32_t)(2 * KBS * W_KB_BYTES));
        for (int kb = 0; kb < KBS; ++kb) {
            tma_load_2d(wh + (size_t)kb * W_KB_BYTES, &tmWh, wbar, kb * BK, 0);
            tma_load_2d(wl + (size_t)kb * W_KB_BYTES, &tmWl, wbar, kb * BK, 0);
        }
    }
    pdl_wait();      // everything above is independent of the previous kernel's output

    bool w_ready = false;
    const int wrow = (tt_id >> 7) * 64;                         // this warpgroup's accumulator rows wrow .. wrow + 63
    const long long tstep = (long long)gridDim.x * TEAMS;
    long long tile = (long long)blockIdx.x * TEAMS + team;
    int kb = 0;
    float4 R[P];
    // unit (tile, kb): 64 tokens starting at t0 + (C == 64 ? 64*kb : 0), channels (C == 64 ? 0 : 64*kb) .. +64;
    // rows [tb - HALO, tb - HALO + ROWS) are fetched, zero outside [0, T)
    const int ld_r = tt_id >> 4, ld_c = (tt_id & 15) * 4;       // this thread's (row, channel) in each 16-row slab
    auto issue_loads = [&](long long tl, int kbl) {
        const int b = (int)(tl / a.tiles_per_utt), t0 = (int)(tl - (long long)b * a.tiles_per_utt) * TT;
        const int tb = t0 + (C == 64 ? kbl * TOK : 0) - HALO + ld_r;
        const float* xp = a.x + ((long long)b * a.T + tb) * C + (C == 64 ? 0 : kbl * BK) + ld_c;
#pragma unroll
        for (int p = 0; p < P; ++p) {
            const int t = tb + p * 16;
            R[p] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ld_r + p * 16 < ROWS && t >= 0 && t < a.T) R[p] = *reinterpret_cast<const float4*>(xp + p * 16 * C);
        }
    };
    if (tile < a.n_tiles) issue_loads(tile, 0);
    while (tile < a.n_tiles) {
        const int b = (int)(tile / a.tiles_per_utt), t0 = (int)(tile - (long long)b * a.tiles_per_utt) * TT;
        const int tb = t0 + (C == 64 ? kb * TOK : 0);            // first token of this unit
        const int cb = C == 64 ? 0 : kb * BK;                    // first channel of this unit
        uint8_t* opk = op + (size_t)kb * OP_KB_BYTES;
        // ---------------- registers -> Snake'd staging tile (RU) or straight to the hi/lo operand tile (NOISE)
        if (MODE == MODE_RU) {
            const float4 al = *reinterpret_cast<const float4*>(a.a_in + cb + ld_c);
            const float4 iv = make_float4(1.0f / (al.x + 1e-9f), 1.0f / (al.y + 1e-9f), 1.0f / (al.z + 1e-9f), 1.0f / (al.w + 1e-9f));
#pragma unroll
            for (int p = 0; p < P; ++p) {
                if (ld_r + p * 16 < ROWS) {
                    float4 v = R[p];
                    v.x = cg::snake_inv(v.x, al.x, iv.x); v.y = cg::snake_inv(v.y, al.y, iv.y);
                    v.z = cg::snake_inv(v.z, al.z, iv.z); v.w = cg::snake_inv(v.w, al.w, iv.w);
                    *reinterpret_cast<float4*>(S + (ld_r + p * 16) * BK + ld_c) = v;
                }
            }
        } else {
#pragma unroll
            for (int p = 0; p < P; ++p) {
                const int r = ld_r + p * 16;
                const float4 v = R[p];
                const __nv_bfloat162 h0 = __floats2bfloat162_rn(v.x, v.y), h1 = __floats2bfloat162_rn(v.z, v.w);
                const __nv_bfloat162 l0 = __floats2bfloat162_rn(v.x - __low2float(h0), v.y - __high2float(h0));
                const __nv_bfloat162 l1 = __floats2bfloat162_rn(v.z - __low2float(h1), v.w - __high2float(h1));
                uint2 hv, lv;
                hv.x = *reinterpret_cast<const uint32_t*>(&h0); hv.y = *reinterpret_cast<const uint32_t*>(&h1);
                lv.x = *reinterpret_cast<const uint32_t*>(&l0); lv.y = *reinterpret_cast<const uint32_t*>(&l1);
                *reinterpret_cast<uint2*>(opk + sw128(r, ld_c)) = hv;
                *reinterpret_cast<uint2*>(opk + sw128(r + TOK, ld_c)) = lv;
            }
        }
        if (MODE == MODE_RU) team_sync(team);
        // ---------------- prefetch the next unit's rows (in flight during everything below)
        long long ntile = tile;
        int nkb = kb + 1;
        if (nkb == KBS) { nkb = 0; ntile = tile + tstep; }
        if (ntile < a.n_tiles) issue_loads(ntile, nkb);
        const bool last_kb = kb == KBS - 1;
        if (MODE == MODE_RU) {
            // thread -> channel pair (2 * (tt_id % 32)), 8 token groups of 8 tokens
            const int c = (tt_id & 31) * 2, g = tt_id >> 5, ch = cb + c;
            float wa[7], wb[7];
#pragma unroll
            for (int k = 0; k < 7; ++k) { wa[k] = a.dw_w[ch * 7 + k]; wb[k] = a.dw_w[(ch + 1) * 7 + k]; }
            const float ba = a.dw_b ? a.dw_b[ch] : 0.f, bb = a.dw_b ? a.dw_b[ch + 1] : 0.f;
            const float ama = a.a_mid[ch], amb = a.a_mid[ch + 1];
            const float ima = 1.0f / (ama + 1e-9f), imb = 1.0f / (amb + 1e-9f);
            const float* Sp = S + (g * 8) * BK + c;
            uint8_t* oph = opk + (g * 8) * 128;                  // rows g*8 .. g*8+7: (row & 7) == j, so the swizzle is per j
            const int nv = a.T - tb - g * 8;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float va = ba, vb = bb;
#pragma unroll
                for (int k = 0; k < 7; ++k) {
                    const float2 xv = *reinterpret_cast<const float2*>(Sp + (j + k * DIL) * BK);
                    va = fmaf(wa[k], xv.x, va); vb = fmaf(wb[k], xv.y, vb);
                }
                va = cg::snake_inv(va, ama, ima); vb = cg::snake_inv(vb, amb, imb);
                if (j >= nv) { va = 0.f; vb = 0.f; }
                const __nv_bfloat162 hi = __floats2bfloat162_rn(va, vb);
                const __nv_bfloat162 lo = __floats2bfloat162_rn(va - __low2float(hi), vb - __high2float(hi));
                const uint32_t off = (uint32_t)(j * 128 + ((((c >> 3) ^ j) << 4) | ((c & 7) << 1)));
                *reinterpret_cast<__nv_bfloat162*>(oph + off) = hi;
                *reinterpret_cast<__nv_bfloat162*>(oph + TOK * 128 + off) = lo;
            }
        }
        if (!last_kb) {
            if (MODE == MODE_RU) team_sync(team);          // S is rewritten by the next k-block
            kb = nkb;
            continue;
        }
        // generic-proxy writes of the operand tile -> visible to the tensor core (async proxy)
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        team_sync(team);
        // ---------------- MMA: D[128, 0:128] = Wh * [Xh; Xl],  D[:, 0:64] += Wl * Xh   (K = 128 over the two k-blocks)
        if (!w_ready) { mbar_wait(wbar, 0); w_ready = true; }
        float acc[64];
        float (&acc_lo)[32] = *reinterpret_cast<float(*)[32]>(acc);
        float (&acc_hi)[32] = *reinterpret_cast<float(*)[32]>(acc + 32);
        wg_fence();
#pragma unroll
        for (int k2 = 0; k2 < KBS; ++k2) {
            const uint64_t ad = make_smem_desc(smem_u32(wh + (size_t)k2 * W_KB_BYTES + wrow * 128));
            const uint64_t a2d = make_smem_desc(smem_u32(wl + (size_t)k2 * W_KB_BYTES + wrow * 128));
            const uint64_t bd = make_smem_desc(smem_u32(op + (size_t)k2 * OP_KB_BYTES));
#pragma unroll
            for (int k = 0; k < BK / UMMA_K; ++k) {
                const uint64_t off = (uint64_t)(k * UMMA_K * 2 / 16);
                // three m64n64 products (one shape, so their accumulator updates are ordered): registers [0, 32) hold columns
                // [0, 64) = Wh * Xh + Wl * Xh, registers [32, 64) columns [64, 128) = Wh * Xl -- the register layout of one n128
                const uint32_t sc = (k2 == 0 && k == 0) ? 0u : 1u;
                wgmma_bf16_n64(acc_lo, ad + off, bd + off, sc);
                wgmma_bf16_n64(acc_hi, ad + off, bd + off + (uint64_t)(TOK * 128 / 16), sc);
                wgmma_bf16_n64(acc_lo, a2d + off, bd + off, 1u);
            }
        }
        wg_commit();
        wg_wait0();
        wg_fence_operand(acc);
        // ---------------- epilogue straight from the fragment: rows m, m + 8; token columns 8 i + 2 (lane % 4) (+1), i < 8;
        // the lo-activation product of token column c sits at column c + 64 of the same thread (register 4 (i + 8) + e)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = wrow + ((tt_id & 127) >> 5) * 16 + (lane >> 2) + 8 * h;
            const int ech = C == 64 ? (m & 63) : m;                               // output channel
            const int etok0 = t0 + (C == 64 ? (m >> 6) * TOK : 0);
            const float bias = a.pw_bias ? a.pw_bias[ech] : 0.f;
            const float an = a.hl ? a.a_next[ech] : 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int etok = etok0 + 8 * i + 2 * (lane & 3) + e;
                    if (etok >= a.T) continue;
                    const long long erow = (long long)b * a.T + etok;
                    const float s = acc[4 * i + 2 * h + e] + acc[4 * (i + 8) + 2 * h + e];
                    const float xr = a.x[erow * C + ech];
                    float val;
                    if (MODE == MODE_NOISE) {
                        const float nz = a.noise ? a.noise[erow] : cg::gauss(a.seed, (unsigned long long)erow);
                        val = fmaf(nz, s, xr);
                    } else {
                        val = xr + (s + bias);
                    }
                    a.y[erow * C + ech] = val;
                    if (a.hl) {
                        const float sv = cg::snake(val, an);
                        if (a.fs) {
                            cg::put_frames(a.hl, a.fs, a.fpad, C, a.T, b, etok, ech, sv);
                        } else {
                            const long long row = (long long)b * (a.T + 1) + etok;
                            store_hilo(a.hl, 2 * C, row, ech, sv, cg::HALF);
                            store_hilo(a.hl, 2 * C, row + 1, C + ech, sv, cg::HALF);
                        }
                    }
                }
            }
        }
        team_sync(team);     // the operand tile is free again
        tile = ntile; kb = nkb;
    }
    pdl_trigger();
}

// ------------------------------------------------------------------------------------------------------------------
// Fused Snake + transposed conv (k = 2s) for the LAST decoder block (C_in = 128 -> s * C_out = 128 phase-major rows, e.g. stride 2,
// 64 channels):  y[t_out] = bias + sum_tap W[:, tap] . snake(x[q - tap]),  t_out = q*s + r - pad,  row m = r*C_out + co.
// Same team structure as ru_fused_kernel.  K = 2 * 128 = four 64-channel k-blocks (tap 0: channels 0-63, 64-127; tap 1 likewise);
// all of W (both bf16 halves, 128 KB) stays resident; the operand tile holds ONE tap (2 k-blocks) at a time, so a tile is
// stage tap 0 -> MMA -> stage tap 1 -> MMA (accumulate) -> epilogue.  Replaces: the 2.1 GB hi/lo 2-tap im2col that the previous
// block's last ResidualUnit had to write and the generic conv GEMM had to read back (the im2col duplicates every activation).
struct ConvtArgs {
    const float* x;            // [B*Tin, 128] fp32 (previous block's output)
    float* y;                  // [B*T, C_out] fp32, T = Tin * stride
    const float* alpha;        // [128] Snake before the transposed conv
    const float* bias;         // [C_out] or null
    int Tin, T, B, stride, cout, pad;
    int tiles_per_utt;         // ceil((Tin + 1) / 64): q runs over 0 .. Tin
    long long n_tiles;
};
static inline size_t convt_smem_bytes() { return 1024 + (size_t)8 * W_KB_BYTES + (size_t)TEAMS * 2 * OP_KB_BYTES + 256; }

static __global__ void __launch_bounds__(THREADS, 1)
convt_fused_kernel(const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, ConvtArgs a) {
    constexpr int CIN = 128, P = 4;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* wh = smem;                                         // [4][128][64] bf16
    uint8_t* wl = wh + (size_t)4 * W_KB_BYTES;
    uint8_t* team_base = wl + (size_t)4 * W_KB_BYTES;
    constexpr size_t tbytes = (size_t)2 * OP_KB_BYTES;
    uint64_t* wbar = reinterpret_cast<uint64_t*>(team_base + TEAMS * tbytes);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int team = warp / TEAM_WARPS, tt_id = tid % TEAM_THREADS;
    uint8_t* op = team_base + team * tbytes;                    // [2][128][64] bf16: the two channel halves of one tap

    if (tid == 0) {
        tma_prefetch_desc(&tmWh); tma_prefetch_desc(&tmWl);
        mbar_init(wbar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (tid == 0) {
        mbar_arrive_expect_tx(wbar, (uint32_t)(8 * W_KB_BYTES));
        for (int kb = 0; kb < 4; ++kb) {
            tma_load_2d(wh + (size_t)kb * W_KB_BYTES, &tmWh, wbar, kb * BK, 0);
            tma_load_2d(wl + (size_t)kb * W_KB_BYTES, &tmWl, wbar, kb * BK, 0);
        }
    }
    pdl_wait();

    bool w_ready = false;
    const int wrow = (tt_id >> 7) * 64;                         // this warpgroup's accumulator rows wrow .. wrow + 63
    float acc[64];                                              // accumulates over the two taps of a tile
    float (&acc_lo)[32] = *reinterpret_cast<float(*)[32]>(acc);
    float (&acc_hi)[32] = *reinterpret_cast<float(*)[32]>(acc + 32);
    const long long tstep = (long long)gridDim.x * TEAMS;
    long long tile = (long long)blockIdx.x * TEAMS + team;
    int unit = 0;                                               // 0..3 = (tap, channel half)
    float4 R[P];
    const int ld_r = tt_id >> 4, ld_c = (tt_id & 15) * 4;
    auto issue_loads = [&](long long tl, int un) {
        const int b = (int)(tl / a.tiles_per_utt), q0 = (int)(tl - (long long)b * a.tiles_per_utt) * TOK;
        const int tap = un >> 1, half = un & 1;
        const int tb = q0 - tap + ld_r;
        const float* xp = a.x + ((long long)b * a.Tin + tb) * CIN + half * BK + ld_c;
#pragma unroll
        for (int p = 0; p < P; ++p) {
            const int t = tb + p * 16;
            R[p] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (t >= 0 && t < a.Tin) R[p] = *reinterpret_cast<const float4*>(xp + p * 16 * CIN);
        }
    };
    if (tile < a.n_tiles) issue_loads(tile, 0);
    while (tile < a.n_tiles) {
        const int b = (int)(tile / a.tiles_per_utt), q0 = (int)(tile - (long long)b * a.tiles_per_utt) * TOK;
        const int tap = unit >> 1, half = unit & 1;
        uint8_t* opk = op + (size_t)half * OP_KB_BYTES;
        {   // registers -> Snake -> hi/lo operand tile
            const float4 al = *reinterpret_cast<const float4*>(a.alpha + half * BK + ld_c);
            const float4 iv = make_float4(1.0f / (al.x + 1e-9f), 1.0f / (al.y + 1e-9f), 1.0f / (al.z + 1e-9f), 1.0f / (al.w + 1e-9f));
#pragma unroll
            for (int p = 0; p < P; ++p) {
                const int r = ld_r + p * 16;
                float4 v = R[p];
                v.x = cg::snake_inv(v.x, al.x, iv.x); v.y = cg::snake_inv(v.y, al.y, iv.y);
                v.z = cg::snake_inv(v.z, al.z, iv.z); v.w = cg::snake_inv(v.w, al.w, iv.w);
                const __nv_bfloat162 h0 = __floats2bfloat162_rn(v.x, v.y), h1 = __floats2bfloat162_rn(v.z, v.w);
                const __nv_bfloat162 l0 = __floats2bfloat162_rn(v.x - __low2float(h0), v.y - __high2float(h0));
                const __nv_bfloat162 l1 = __floats2bfloat162_rn(v.z - __low2float(h1), v.w - __high2float(h1));
                uint2 hv, lv;
                hv.x = *reinterpret_cast<const uint32_t*>(&h0); hv.y = *reinterpret_cast<const uint32_t*>(&h1);
                lv.x = *reinterpret_cast<const uint32_t*>(&l0); lv.y = *reinterpret_cast<const uint32_t*>(&l1);
                *reinterpret_cast<uint2*>(opk + sw128(r, ld_c)) = hv;
                *reinterpret_cast<uint2*>(opk + sw128(r + TOK, ld_c)) = lv;
            }
        }
        long long ntile = tile;
        int nunit = unit + 1;
        if (nunit == 4) { nunit = 0; ntile = tile + tstep; }
        if (ntile < a.n_tiles) issue_loads(ntile, nunit);
        if (half == 0) { unit = nunit; continue; }
        // both channel halves of this tap are staged: MMA over W k-blocks 2*tap, 2*tap + 1
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        team_sync(team);
        if (!w_ready) { mbar_wait(wbar, 0); w_ready = true; }
        wg_fence();
#pragma unroll
        for (int k2 = 0; k2 < 2; ++k2) {
            const int wk = 2 * tap + k2;
            const uint64_t ad = make_smem_desc(smem_u32(wh + (size_t)wk * W_KB_BYTES + wrow * 128));
            const uint64_t a2d = make_smem_desc(smem_u32(wl + (size_t)wk * W_KB_BYTES + wrow * 128));
            const uint64_t bd = make_smem_desc(smem_u32(op + (size_t)k2 * OP_KB_BYTES));
#pragma unroll
            for (int k = 0; k < BK / UMMA_K; ++k) {
                const uint64_t off = (uint64_t)(k * UMMA_K * 2 / 16);
                const uint32_t sc = (tap == 0 && k2 == 0 && k == 0) ? 0u : 1u;    // three m64n64 products, as in ru_fused_kernel
                wgmma_bf16_n64(acc_lo, ad + off, bd + off, sc);
                wgmma_bf16_n64(acc_hi, ad + off, bd + off + (uint64_t)(TOK * 128 / 16), sc);
                wgmma_bf16_n64(acc_lo, a2d + off, bd + off, 1u);
            }
        }
        wg_commit();
        wg_wait0();                           // the operand tile is reused by the next tap / tile: the MMAs must have read it
        wg_fence_operand(acc);
        if (tap == 0) { team_sync(team); unit = nunit; continue; }
        // ---------------- epilogue straight from the fragment: row m = r*C_out + co, q columns 8 i + 2 (lane % 4) (+1), i < 8
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = wrow + ((tt_id & 127) >> 5) * 16 + (lane >> 2) + 8 * h;
            const int co = m % a.cout, rr = m / a.cout;
            const float bias = a.bias ? a.bias[co] : 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int qq = q0 + 8 * i + 2 * (lane & 3) + e;
                    const int to = qq * a.stride + rr - a.pad;
                    if (qq <= a.Tin && to >= 0 && to < a.T)
                        a.y[((long long)b * a.T + to) * a.cout + co] = acc[4 * i + 2 * h + e] + acc[4 * (i + 8) + 2 * h + e] + bias;
                }
            }
        }
        team_sync(team);
        tile = ntile; unit = nunit;
    }
    pdl_trigger();
}

}  // namespace rf
}  // namespace b2a
