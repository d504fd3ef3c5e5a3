// wgmma + TMA "weights-as-A" GEMM for sm_90a:  D[M, N] = W[M, K] * X[N, K]^T   (bf16 in, fp32 accumulate)
//   W : weights, [M, K] row-major (K-major)  -> A operand, 128 x 64 tiles by TMA (SWIZZLE_128B)
//   X : activations, [N, K] row-major        -> B operand, BN x 64 tiles by TMA
//   D : accumulated in the registers of the consumer warpgroups, staged through shared memory and written
//       TRANSPOSED as out[n, m] so it is the next layer's [tokens, features] activation matrix.
// Swap-AB keeps the tensor-core M dimension (128 = two m64 wgmma blocks) full with output features even when there
// are only 8 tokens (autoregressive decode), where the kernel is purely a weight-streaming engine: one elected thread
// of the producer warp issues TMA into a deep shared-memory ring (~100-200 KB in flight per SM), the consumer
// warpgroups issue wgmma and run the epilogue.  Work is split stream-K style: the (m_tile, k_block) units are dealt
// evenly and contiguously to the CTAs; a CTA that owns only part of a tile's K range writes its partial tile to a
// workspace slot, and the last of the tile's CTAs to finish adds the slots in slot order and stores the sum into the fp32
// output (EPI_STORE) or adds it there (EPI_ADD), so the result is the same on every run.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2a {
namespace tc {

constexpr int BM = 128, BK = 64, UMMA_K = 16;
constexpr int THREADS = 160;  // warps 0-3: wgmma + epilogue (one warpgroup), warp 4: TMA producer
enum : int { EPI_STORE = 0, EPI_PARTIAL = 1, EPI_SWIGLU = 2, EPI_STORE_BF16 = 3, EPI_ADD = 4 };
enum : int { ACT_NONE = 0, ACT_GELU = 1 };

struct Args {
    float* out_f32;          // [N, ldo] fp32 (EPI_STORE / EPI_ADD / EPI_PARTIAL)
    __nv_bfloat16* out_bf16; // [N, ldo] bf16 (EPI_SWIGLU: ldo = M/2 ; EPI_STORE_BF16)
    int M, N, K;             // N = valid tokens (rows of X)
    int ldo;                 // leading dimension of the output (elements)
    int m_tiles, k_blocks;   // ceil(M/128), K/64
    int stages;              // smem ring depth
    int epi_full;            // epilogue when a CTA owns a tile's whole K range
    int epi_partial;         // epilogue for partial K ranges (EPI_PARTIAL: the tile's partials are summed and stored into
                             // out_f32, or added there when epi_full is EPI_ADD); < 0 => CTAs own whole tiles only
    int hilo;                // X rows [0, BN/2) = hi(x), rows [BN/2, BN) = lo(x) = bf16(x - hi): columns j and
                             // j + BN/2 of the accumulator are summed, giving fp32-activation accuracy for free
    const float* bias;       // nullable [M]: added to every output column before the activation
    int act;                 // ACT_NONE | ACT_GELU (exact erf GELU, WhisperLayers.swift:101)
    int tile_rows;           // whole-tile mode (epi_partial < 0) only: weight rows per m-tile when != 0 (a multiple of 8, <= 128; tmA's box must
                             // have this many rows).  fewer rows per tile spread a GEMM whose 128-row tiles
                             // would leave SMs idle over all of them.  The MMA still multiplies 128
                             // shared-memory rows; rows past tile_rows are stale and their accumulator rows are never stored.
    const float* rstd_ss;    // nullable [rstd_parts, BN / 2]: the X rows are UN-normalised (h * gain); every accumulator column t is
    int rstd_parts;          // multiplied by rsqrt(sum_p rstd_ss[p, t] * rstd_inv_h + rstd_eps) first (fused RMSNorm, hi/lo, BN = 16, 32, 64)
    float rstd_inv_h, rstd_eps;
    int lo_rows;             // != 0: bf16 outputs are written as hi/lo pairs in the same tile-interleaved row layout the
                             // kernel reads X in: token t -> hi row (t / (BN/2)) * BN + t % (BN/2), lo row = hi row + BN/2
    float* part_ws;          // EPI_PARTIAL: [n_tiles][m_tiles][part_slots][BN][128] fp32 partial tiles (stream_k_slots() sizes part_slots)
    unsigned* part_cnt;      // EPI_PARTIAL: [n_tiles][m_tiles] k-blocks arrived, zero between launches (the reducing CTA resets its tile's)
    int part_slots;
};

// Stream-K deals units [units * c / ctas, units * (c + 1) / ctas) to CTA c; the CTA that owns unit u:
__host__ __device__ __forceinline__ int stream_k_owner(long long u, long long units, int ctas) {
    return (int)(((u + 1) * ctas + units - 1) / units) - 1;
}
// the most CTAs that share one m-tile's K range: the slots per m-tile EPI_PARTIAL needs
inline int stream_k_slots(int m_tiles, int k_blocks, int ctas) {
    const long long units = (long long)m_tiles * k_blocks;
    int n = 1;
    for (int mt = 0; mt < m_tiles; ++mt)
        n = n > stream_k_owner((long long)(mt + 1) * k_blocks - 1, units, ctas) - stream_k_owner((long long)mt * k_blocks, units, ctas) + 1
                ? n : stream_k_owner((long long)(mt + 1) * k_blocks - 1, units, ctas) - stream_k_owner((long long)mt * k_blocks, units, ctas) + 1;
    return n;
}

// ----------------------------------------------------------------------------------------------- PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    // bounded spin: a protocol bug traps (cudaErrorLaunchFailure) instead of hanging the GPU
    for (uint32_t spins = 0; !mbar_try_wait(bar, parity); ++spins)
        if (spins > (1u << 28)) __trap();
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// ---- wgmma (warpgroup-wide: issued by all 128 threads of a warpgroup; the accumulator lives in their registers)
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
template <int R>
__device__ __forceinline__ void wg_fence_operand(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D(64 x N, registers) (+)= A[smem, 64 x 16] * B[smem, N x 16]^T, both K-major; scale_d == 0 overwrites D
__device__ __forceinline__ void wgmma_bf16_n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_bf16_n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_bf16_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_bf16_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_f16_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_f16_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

// D(64 x 128) (+)= A[registers, 64 x 16] * B[smem, 128 x 16]^T: A as fp16 fragments {row r0 / k 0-7, row r0 + 8 / k 0-7, row r0 / k 8-15,
// row r0 + 8 / k 8-15} (r0 and the k pair as in an accumulator fragment)
__device__ __forceinline__ void wgmma_f16_rs_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
    if constexpr (N == 16) wgmma_bf16_n16(d, da, db, scale_d);
    else if constexpr (N == 32) wgmma_bf16_n32(d, da, db, scale_d);
    else if constexpr (N == 64) wgmma_bf16_n64(d, da, db, scale_d);
    else wgmma_bf16_n128(d, da, db, scale_d);
}

// K-major SWIZZLE_128B shared-memory matrix descriptor (sm_90 GMMA layout):
// start>>4 [0,14) | LBO>>4 [16,30) = 1 (unused for swizzled K-major) | SBO>>4 [32,46) = 1024/16 | layout [62,64) = 1 (128B)
// The tile base must be 1024-byte aligned; +2 in the start field steps 16 bf16 along K, +512 steps 64 rows.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

// Accumulator fragment of an m64nN wgmma -> fp32 tile in shared memory (row-major, leading dimension ld floats):
// thread t of the warpgroup holds rows 16 (t / 32) + (t % 32) / 4 (+8) and columns 8 i + 2 (t % 4) (+1).
template <int N>
__device__ __forceinline__ void store_frag(float* s, int ld, const float (&d)[N / 2], int r0, int c0) {
    const int t = threadIdx.x & 127, r = r0 + (t >> 5) * 16 + ((t & 31) >> 2), c = c0 + 2 * (t & 3);
#pragma unroll
    for (int i = 0; i < N / 8; ++i) {
        *reinterpret_cast<float2*>(s + (size_t)r * ld + c + 8 * i) = make_float2(d[4 * i], d[4 * i + 1]);
        *reinterpret_cast<float2*>(s + (size_t)(r + 8) * ld + c + 8 * i) = make_float2(d[4 * i + 2], d[4 * i + 3]);
    }
}
// 16 consecutive fp32 of a staged accumulator row (16-byte aligned)
__device__ __forceinline__ void ld_acc16(const float* p, float* v) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float4 f = reinterpret_cast<const float4*>(p)[i];
        v[4 * i] = f.x; v[4 * i + 1] = f.y; v[4 * i + 2] = f.z; v[4 * i + 3] = f.w;
    }
}
__device__ __forceinline__ void named_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// Activation v of token t, column col, as the hi/lo pair the B operand is read in: hi = bf16(v) in row (t / half) * 2 half + t % half,
// lo = bf16(v - hi) in the row `half` below (half = tokens per tile: 8 / 16 for the decode steps, 64 for 128-row tiles).  I is the
// caller's token index type (int or long long): the division is done in it.
template <class I>
__device__ __forceinline__ void store_hilo(__nv_bfloat16* base, long long ld, I t, long long col, float v, int half) {
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    const long long r = (long long)(t / half) * 2 * half + (t % half);
    base[r * ld + col] = hi;
    base[(r + half) * ld + col] = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// Consumer warps per CTA (wgmma + epilogue), followed by one TMA producer warp.  The 128-column tile (prefill / Whisper encoder: 64
// tokens as hi/lo pairs) is split over four warpgroups (two 64-row blocks x two 64-column halves) so that the epilogue, which adds,
// activates and stores 128 x 128 values per tile, is spread over 16 warps; the narrow decode tiles need one warpgroup.
template <int BN>
struct Cfg {
    static constexpr int EPI_WARPS = BN >= 128 ? 16 : 4;
    static constexpr int WG = EPI_WARPS / 4;                   // consumer warpgroups
    static constexpr int RB = WG == 1 ? 2 : 1;                 // 64-row blocks per warpgroup
    static constexpr int WN = WG == 1 ? BN : BN * 2 / WG;      // accumulator columns per warpgroup
    static constexpr int LD = BN + 4;                          // row stride (floats) of the staged accumulator
    static constexpr int NTHREADS = 32 * EPI_WARPS + 32;
};

// The decode step runs R = 8, 16 or 32 token rows as hi/lo pairs: X is [2R, K] with hi(x_t) in row t and lo(x_t) in row R + t, and the
// GEMM tiles are BN = 2R columns wide.  One rule, here, turns a row count into that width; every kernel that writes or reads the
// layout takes its lo-row offset R from it.
constexpr int DECODE_WIDTHS[3] = {8, 16, 32};
__host__ __device__ constexpr int decode_width(int rows) { return rows <= 8 ? 8 : rows <= 16 ? 16 : 32; }
__host__ __device__ constexpr int decode_width_index(int width) { return width == 8 ? 0 : width == 16 ? 1 : 2; }
template <int BN>
struct DecodeWidth {
    static constexpr bool OK = BN == 16 || BN == 32 || BN == 64;   // tc_gemm_kernel<BN> is a decode-step GEMM
    static constexpr int TOKENS = OK ? BN / 2 : 8;
};

// rstd[t] = rsqrt(sum_p ss[p, t] * inv_h + eps) for the T tokens of a [parts, T] sum-of-squares array, by the whole warp: rs[g] holds
// rstd[8 g + (lane & 7)].  Each group of 8 tokens is reduced as the 8-token step always was: lane = part * 8 + token loads one partial
// per step, then xor 8 and xor 16, so a token's rstd does not depend on how many tokens the step runs.
template <int T>
__device__ __forceinline__ void rstd_lanes(float (&rs)[T / 8], const float* ss, int parts, float inv_h, float eps, int lane) {
#pragma unroll
    for (int g = 0; g < T / 8; ++g) {
        float t = 0.f;
        for (int p0 = 0; p0 < parts; p0 += 4) {
            const int p = p0 + (lane >> 3);
            if (p < parts) t += ss[p * T + 8 * g + (lane & 7)];
        }
        t += __shfl_xor_sync(0xffffffffu, t, 8);
        t += __shfl_xor_sync(0xffffffffu, t, 16);
        rs[g] = rsqrtf(t * inv_h + eps);
    }
}

// Dynamic shared memory of tc_gemm_kernel<BN>: the ring, the staged accumulator, 256 bytes of barriers.  The decode step runs BN = 16
// with 6 stages: 6 x 18 432 + 10 240 + 256 = 121 088 bytes, which leaves room on the SM (233 472 bytes, 1 KB of it reserved per
// resident CTA) for one CTA of either neighbour in the step, the split-K GEMM or the attention kernel, so that the neighbour's
// prefetch-before-griddepcontrol.wait runs under this kernel's main loop and vice versa.
template <int BN>
struct Smem {
    static constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE = A_BYTES + B_BYTES;
    static constexpr int ACC_BYTES = BM * Cfg<BN>::LD * 4;
    static int max_stages() { return (226 * 1024 - 256 - ACC_BYTES) / STAGE; }   // 1 KB under the 227 KB a CTA may have
    static size_t bytes(int stages) { return (size_t)stages * STAGE + ACC_BYTES + 256; }
};
// The tile bases must be 1024-byte aligned (make_smem_desc): the dynamic array is declared so, and the kernels check it once.
__device__ __forceinline__ void check_smem_base(const void* base) {
    if (threadIdx.x == 0 && (smem_u32(base) & 1023u)) __trap();
}

// `a` is __grid_constant__: the kernel reads its fields from kernel-parameter memory where they are used.  Without it nvcc 12.9 may
// copy the whole struct into registers at entry (decode GEMM, BN = 16: 106 registers instead of 92 and ~15% more instructions).
template <int BN>
__global__ void __launch_bounds__(Cfg<BN>::NTHREADS, Cfg<BN>::EPI_WARPS > 4 ? 1 : 2)
tc_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ Args a) {
    using S = Smem<BN>;
    using C = Cfg<BN>;
    extern __shared__ __align__(1024) uint8_t smem[];
    float* sacc = reinterpret_cast<float*>(smem + (size_t)a.stages * S::STAGE);            // [128][LD] staged accumulator
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)a.stages * S::STAGE + S::ACC_BYTES);
    uint64_t* empty = full + a.stages;
    int* s_reduce = reinterpret_cast<int*>(empty + a.stages);                               // this CTA sums the tile's partials

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n0 = blockIdx.y * BN;
    const int TR = a.tile_rows > 0 ? a.tile_rows : BM;                  // weight rows per m-tile
    const uint32_t stage_tx = (uint32_t)(TR * BK * 2 + S::B_BYTES);     // bytes the two TMA loads of a stage deliver
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // PDL: let the next kernel's prologue start

    check_smem_base(smem);
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < a.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], C::EPI_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    // stream-K partition of the (m_tile, k_block) units, k fastest
    const long long units = (long long)a.m_tiles * a.k_blocks;
    long long u0, u1;
    if (a.epi_partial >= 0) {
        u0 = units * blockIdx.x / gridDim.x;
        u1 = units * (blockIdx.x + 1) / gridDim.x;
    } else {   // whole tiles per CTA (epilogues that cannot be split along K, e.g. SwiGLU)
        u0 = ((long long)a.m_tiles * blockIdx.x / gridDim.x) * a.k_blocks;
        u1 = ((long long)a.m_tiles * (blockIdx.x + 1) / gridDim.x) * a.k_blocks;
    }

    if (warp == C::EPI_WARPS) {
        if (lane == 0) {
            // Weights never depend on the previous kernel: fill the whole ring with A tiles right away, then wait
            // for the previous kernel (PDL) before loading the activation (B) tiles that complete those stages.
            const int npre = (int)min((long long)a.stages, u1 - u0);
            for (int i = 0; i < npre; ++i) {
                const long long u = u0 + i;
                const int mt = (int)(u / a.k_blocks), kb = (int)(u - (long long)mt * a.k_blocks);
                mbar_arrive_expect_tx(&full[i], stage_tx);
                tma_load_2d(smem + (size_t)i * S::STAGE, &tmA, &full[i], kb * BK, mt * TR);
            }
            asm volatile("griddepcontrol.wait;" ::: "memory");
            for (int i = 0; i < npre; ++i) {
                const long long u = u0 + i;
                const int mt = (int)(u / a.k_blocks), kb = (int)(u - (long long)mt * a.k_blocks);
                tma_load_2d(smem + (size_t)i * S::STAGE + S::A_BYTES, &tmB, &full[i], kb * BK, n0);
            }
            int stage = npre == a.stages ? 0 : npre;
            uint32_t phase = npre == a.stages ? 1 : 0;
            for (long long u = u0 + npre; u < u1; ++u) {
                const int mt = (int)(u / a.k_blocks), kb = (int)(u - (long long)mt * a.k_blocks);
                mbar_wait(&empty[stage], phase ^ 1);
                uint8_t* sa = smem + (size_t)stage * S::STAGE;
                mbar_arrive_expect_tx(&full[stage], stage_tx);
                tma_load_2d(sa, &tmA, &full[stage], kb * BK, mt * TR);
                tma_load_2d(sa + S::A_BYTES, &tmB, &full[stage], kb * BK, n0);
                if (++stage == a.stages) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        const int q = warp & 3;                           // the epilogue of warp w reads accumulator rows 32 (w % 4) .. + 31
        constexpr int NCG = C::EPI_WARPS / 4;             // column groups: warps 4 g .. 4 g + 3 take every NCG-th column chunk
        const int cg = warp >> 2, wg = warp >> 2;
        const int row_blk = C::WG == 1 ? 0 : (wg & 1), col_blk = C::WG == 1 ? 0 : (wg >> 1);
        int stage = 0; uint32_t phase = 0;
        float acc[C::RB][C::WN / 2];
#pragma unroll
        for (int rb = 0; rb < C::RB; ++rb)
#pragma unroll
            for (int i = 0; i < C::WN / 2; ++i) acc[rb][i] = 0.f;
        long long u = u0;
        constexpr int NR = DecodeWidth<BN>::TOKENS;   // tokens per tile of a decode-step width (8 for the prefill tile: unused)
        float rstd[8];                                // BN = 16: every token's rstd; wider: rsg[g] = rstd[8 g + (lane & 7)]
        float rsg[NR / 8];
        bool have_rstd = false;
        if (DecodeWidth<BN>::OK && a.rstd_ss) {
            // fused RMSNorm: the producer of X left h * gain un-normalised plus per-m-tile sums of squares (SplitArgs::ss, [parts, NR]);
            // the accumulator column of token t is scaled by rstd[t].  Computed while the main loop streams weights: these warps are
            // idle until the first accumulator is ready, so they wait for the previous kernel themselves and reduce the partial
            // sums with one independent load per lane and step (lane = part * 8 + token), one group of 8 tokens at a time.
            asm volatile("griddepcontrol.wait;" ::: "memory");
            if constexpr (BN == 16) {
                float t = 0.f;
                for (int p0 = 0; p0 < a.rstd_parts; p0 += 4) {
                    const int p = p0 + (lane >> 3);
                    if (p < a.rstd_parts) t += a.rstd_ss[p * 8 + (lane & 7)];
                }
                t += __shfl_xor_sync(0xffffffffu, t, 8);
                t += __shfl_xor_sync(0xffffffffu, t, 16);
                const float rs = rsqrtf(t * a.rstd_inv_h + a.rstd_eps);
#pragma unroll
                for (int j = 0; j < 8; ++j) rstd[j] = __shfl_sync(0xffffffffu, rs, j);
            } else {
                rstd_lanes<NR>(rsg, a.rstd_ss, a.rstd_parts, a.rstd_inv_h, a.rstd_eps, lane);
            }
            have_rstd = true;
        }
        while (u < u1) {
            const int mt = (int)(u / a.k_blocks);
            const long long seg_begin = u;
            const long long seg_end = min(u1, (long long)(mt + 1) * a.k_blocks);
            u = seg_end;
            const bool whole = (seg_begin == (long long)mt * a.k_blocks) && (seg_end == (long long)(mt + 1) * a.k_blocks);
            const int epi = whole ? a.epi_full : a.epi_partial;
            for (long long uu = seg_begin; uu < seg_end; ++uu) {
                mbar_wait(&full[stage], phase);
                const uint32_t sa = smem_u32(smem + (size_t)stage * S::STAGE);
                wg_fence();
#pragma unroll
                for (int k = 0; k < BK / UMMA_K; ++k) {
#pragma unroll
                    for (int rb = 0; rb < C::RB; ++rb) {
                        const uint64_t ad = make_smem_desc(sa + (uint32_t)((row_blk + rb) * 64 * 128)) + (uint64_t)(2 * k);
                        const uint64_t bd = make_smem_desc(sa + S::A_BYTES + (uint32_t)(col_blk * C::WN * 128)) + (uint64_t)(2 * k);
                        wgmma_bf16<C::WN>(acc[rb], ad, bd, (uu == seg_begin && k == 0) ? 0u : 1u);
                    }
                }
                wg_commit();
                wg_wait0();
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[stage]);        // this warp's share of the stage has been read
                if (++stage == a.stages) { stage = 0; phase ^= 1; }
            }
#pragma unroll
            for (int rb = 0; rb < C::RB; ++rb) wg_fence_operand(acc[rb]);
            named_sync(1, 32 * C::EPI_WARPS);                     // the previous segment's epilogue has read sacc
#pragma unroll
            for (int rb = 0; rb < C::RB; ++rb) store_frag<C::WN>(sacc, C::LD, acc[rb], (row_blk + rb) * 64, col_blk * C::WN);
            named_sync(1, 32 * C::EPI_WARPS);
            const int m = mt * TR + q * 32 + lane;
            const float* arow = sacc + (size_t)(q * 32 + lane) * C::LD;
            const long long units = (long long)a.m_tiles * a.k_blocks;
            const int first_owner = stream_k_owner((long long)mt * a.k_blocks, units, gridDim.x);
            const size_t tile_id = (size_t)blockIdx.y * a.m_tiles + mt;
            float* ws_tile = whole ? nullptr : a.part_ws + (tile_id * a.part_slots + (blockIdx.x - first_owner)) * BN * BM;
            constexpr int HALF = BN / 2;
            constexpr int CH = (BN == 16) ? 8 : 16;            // token columns handled per iteration
            const int n_cols = a.hilo ? HALF : BN;              // hilo: column j of the hi half pairs with j + HALF
            const int ntok0 = a.hilo ? (int)blockIdx.y * HALF : n0;
            const bool m_ok = m < a.M && q * 32 + lane < TR;
            const int cstep = (BN == 16 && !a.hilo) ? 16 : CH;
            for (int c0 = cg * cstep; c0 < n_cols; c0 += cstep * NCG) {
                float v[16];
                if (BN == 16) {
                    ld_acc16(arow, v);                           // all 16 columns: [0,8) hi, [8,16) lo
                    if (a.hilo) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) v[j] += v[j + 8];
                    }
                    if (have_rstd) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) v[j] *= rstd[j];
                    }
                } else {
                    ld_acc16(arow + c0, v);
                    if (a.hilo) {
                        float w[16];
                        ld_acc16(arow + c0 + HALF, w);
#pragma unroll
                        for (int j = 0; j < 16; ++j) v[j] += w[j];
                    }
                    if constexpr (DecodeWidth<BN>::OK) {
                        if (have_rstd) {   // hi/lo only: c0 is a multiple of 16 below NR (a constant index into rsg per branch)
#pragma unroll
                            for (int cc = 0; cc < NR; cc += 16)
                                if (cc == c0) {
#pragma unroll
                                    for (int j = 0; j < 16; ++j) v[j] *= __shfl_sync(0xffffffffu, rsg[(cc + j) / 8], j % 8);
                                }
                        }
                    }
                }
                const int jn = (BN == 16 && !a.hilo) ? 16 : CH;
                if (a.bias || a.act) {
                    // a partial K range (stream-K) carries the bias only in the segment that starts the tile
                    const float bv = (a.bias && m_ok && (whole || seg_begin == (long long)mt * a.k_blocks)) ? a.bias[m] : 0.f;
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        float t = v[j] + bv;
                        if (a.act == ACT_GELU) t = 0.5f * t * (1.0f + erff(t * 0.70710678118654752f));
                        v[j] = t;
                    }
                }
                const int nt = ntok0 + c0;                       // first token of this chunk
                const int nvalid = min(jn, a.N - nt);            // tokens of the chunk that exist
                if (epi == EPI_SWIGLU) {
                    // rows are (gate, up) pairs: even lane = gate, odd lane = up   (LlamaTTS.swift:282-284)
                    // the chunk lies inside one HALF block, so hi rows are consecutive
                    const long long hrow = a.lo_rows ? (long long)(nt / HALF) * BN + (nt % HALF) : nt;
                    __nv_bfloat16* ph = a.out_bf16 + hrow * a.ldo + (m >> 1);
                    const long long lo_off = (long long)HALF * a.ldo;
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        if (j >= jn) break;
                        const float other = __shfl_xor_sync(0xffffffffu, v[j], 1);
                        if (j < nvalid && m_ok && (lane & 1) == 0) {
                            const float r = v[j] / (1.0f + __expf(-v[j])) * other;
                            const __nv_bfloat16 hi = __float2bfloat16_rn(r);
                            ph[0] = hi;
                            if (a.lo_rows) ph[lo_off] = __float2bfloat16_rn(r - __bfloat162float(hi));
                        }
                        ph += a.ldo;
                    }
                } else if (epi == EPI_STORE_BF16) {
                    const long long hrow = a.lo_rows ? (long long)(nt / HALF) * BN + (nt % HALF) : nt;
                    __nv_bfloat16* ph = a.out_bf16 + hrow * a.ldo + m;
                    const long long lo_off = (long long)HALF * a.ldo;
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        if (j >= jn) break;
                        if (j < nvalid && m_ok) {
                            const __nv_bfloat16 hi = __float2bfloat16_rn(v[j]);
                            ph[0] = hi;
                            if (a.lo_rows) ph[lo_off] = __float2bfloat16_rn(v[j] - __bfloat162float(hi));
                        }
                        ph += a.ldo;
                    }
                } else if (epi == EPI_PARTIAL) {
                    float* pw = ws_tile + (size_t)(nt - ntok0) * BM + q * 32 + lane;   // every row and column of the slot is written
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (j < jn) pw[(size_t)j * BM] = v[j];
                } else {
                    float* pf = a.out_f32 + (long long)nt * a.ldo + m;
                    if (epi == EPI_ADD) {     // residual accumulate (whole-tile CTAs only): all loads before any store
#pragma unroll
                        for (int j = 0; j < 16; ++j)
                            if (j < jn && j < nvalid && m_ok) v[j] += pf[(long long)j * a.ldo];
                    }
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        if (j >= jn) break;
                        if (j < nvalid && m_ok) {
                            pf[0] = v[j];
                        }
                        pf += a.ldo;
                    }
                }
            }
            if (!whole) {
                // the CTA whose k-blocks complete the tile's count adds the partials in slot order (no CTA waits for another);
                // slot p belongs to CTA first_owner + p, which owns no unit at all when there are more CTAs than units
                const int n_parts = stream_k_owner((long long)(mt + 1) * a.k_blocks - 1, units, gridDim.x) - first_owner + 1;
                const unsigned my_kb = (unsigned)(seg_end - seg_begin);
                __threadfence();
                named_sync(1, 32 * C::EPI_WARPS);
                if (threadIdx.x == 0) *s_reduce = atomicAdd(&a.part_cnt[tile_id], my_kb) + my_kb == (unsigned)a.k_blocks;
                named_sync(1, 32 * C::EPI_WARPS);
                if (*s_reduce) {
                    __threadfence();
                    const float* base = a.part_ws + tile_id * a.part_slots * BN * BM;   // slot p: [BN][128], i = column * 128 + row
                    constexpr int NT = 32 * C::EPI_WARPS, PER = 16;                      // elements per thread and pass
                    const int n_el = n_cols * BM;
                    for (int i0 = 0; i0 < n_el; i0 += NT * PER) {
                        float sum[PER];
#pragma unroll
                        for (int e = 0; e < PER; ++e) sum[e] = 0.f;
                        for (int p = 0; p < n_parts; ++p) {
                            const long long c = first_owner + p;
                            if (units * (c + 1) / gridDim.x == units * c / gridDim.x) continue;   // empty range: no partial
                            const float* slot = base + (size_t)p * BN * BM;
#pragma unroll
                            for (int e = 0; e < PER; ++e) {
                                const int i = i0 + threadIdx.x + e * NT;
                                if (i < n_el) sum[e] += __ldcg(slot + i);
                            }
                        }
#pragma unroll
                        for (int e = 0; e < PER; ++e) {
                            const int i = i0 + threadIdx.x + e * NT;
                            const int tcol = i / BM, r = i - tcol * BM, mm = mt * BM + r, tok = ntok0 + tcol;
                            if (i < n_el && tok < a.N && mm < a.M) {
                                float* o = a.out_f32 + (long long)tok * a.ldo + mm;
                                *o = a.epi_full == EPI_ADD ? *o + sum[e] : sum[e];
                            }
                        }
                    }
                    if (threadIdx.x == 0) a.part_cnt[tile_id] = 0;
                }
            }
        }
    }
}

// ----------------------------------------------------------------------------------------------- cluster split-K
// D[M, T tokens] = W[M, K] X^T (T = 8, 16 or 32: the decode width) for the two GEMMs of a decoder layer whose output feeds the residual
// stream (o_proj, down_proj), with the residual add, the NEXT RMSNorm's gain, its hi/lo split and its sum of squares fused into the
// epilogue, so the step has no stand-alone norm kernel.  One thread-block CLUSTER per 128-row m-tile: CTA r of the cluster streams
// k-blocks [kb * r / C, kb * (r + 1) / C) of the tile (same TMA ring / wgmma warpgroup as tc_gemm_kernel<2T>), then every
// non-leader writes its 128 x T fp32 partial into the leader's shared memory (distributed shared memory, st.shared::cluster),
// one cluster barrier, and the leader adds the partials IN RANK ORDER (bit-reproducible) and runs
//     h[t, m] += acc          (fp32 residual stream, updated in place)
//     xn[t, m] = hi / lo of  h[t, m] * gain[m]        (UN-normalised: the consumer GEMM scales its accumulator by rstd[t])
//     ss[mt, t] = sum over the tile's rows of h[t, m]^2   (the consumer reduces the m-tiles: rstd = rsqrt(sum / H + eps))
// RMSNorm is linear in its per-token scale, so moving rstd behind the consumer GEMM is exact up to fp32 rounding.
// Store mode (h == nullptr, the q|k|v projection): the leader instead stores out[t, m] = 0 + rstd[t] * P_0 + rstd[t] * P_1 + ...,
// P_r the partial of CTA r and rstd of the norm the input went through (rstd_ss; 1 without).  With sk_ctas > 0 CTA r streams the
// r-th piece of the tile as tc_gemm_kernel's stream-K over sk_ctas CTAs cuts it (split_range), so out is bit-identical to that
// launch: the same wgmma accumulation per piece, each piece scaled before the pieces are summed in slot order from 0.
// Every per-token operation is the same at every T, so a token's output does not depend on the width it ran at.
struct SplitArgs {
    int M, N, K;                 // N = tokens (<= T)
    int k_blocks, stages;
    int sk_ctas;                 // > 0: k-blocks cut as stream-K over this many CTAs (cluster >= stream_k_slots); 0: evenly
    float* h;                    // [T, M] residual stream (read-modify-write by the leader); nullptr: store mode
    const float* gain;           // [M] the next norm's weight
    __nv_bfloat16* xn;           // [2T, M] hi rows 0..T-1 / lo rows T..2T-1
    float* ss;                   // [m_tiles, T] partial sums of squares
    float* out;                  // store mode: [T, M] fp32, rows t < N written
    const float* rstd_ss;        // nullable: partial sums [rstd_parts, T] of the norm this GEMM's INPUT went through
    int rstd_parts;
    float rstd_inv_h, rstd_eps;
};

__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_nctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t map_to_rank(uint32_t saddr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
    return r;
}
__device__ __forceinline__ void st_cluster_f4(uint32_t addr, float a, float b, float c, float d) {
    asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// k-blocks [kb0, kb1) of m-tile mt that CTA r of its cluster of C streams (empty when kb0 == kb1)
__host__ __device__ __forceinline__ void split_range(const SplitArgs& a, int mt, int m_tiles, int r, int C, int& kb0, int& kb1) {
    if (a.sk_ctas > 0) {   // the piece of stream-K CTA first_owner + r (stream_k_owner) that lies in this tile
        const long long units = (long long)m_tiles * a.k_blocks, t0 = (long long)mt * a.k_blocks, t1 = t0 + a.k_blocks;
        const long long c = stream_k_owner(t0, units, a.sk_ctas) + r;
        const long long u0 = units * c / a.sk_ctas, u1 = units * (c + 1) / a.sk_ctas;
        kb0 = (int)(u0 > t0 ? u0 - t0 : 0);
        kb1 = (int)(u1 < t1 ? u1 - t0 : a.k_blocks);
        if (kb1 < kb0) kb1 = kb0;
    } else {
        kb0 = (int)((long long)a.k_blocks * r / C);
        kb1 = (int)((long long)a.k_blocks * (r + 1) / C);
    }
}

constexpr int SPLIT_MAX_CLUSTER = 8;
// Dynamic shared memory of tc_gemm_splitk_kernel<T>: the ring, the peers' partials (written remotely while the leader may still be
// streaming, so they have a buffer of their own), then barriers and the s_red reduction scratch.  A CTA streams ONE tile, so its ring
// is idle once the main loop ends and the 128 x 2T accumulator is staged over its first ACC_STAGES stages.  The 8-token step runs 5
// stages in clusters of 5: 5 x 18 432 + 4 x 4096 + 512 = 109 056 bytes; with tc_gemm_kernel<16>'s 121 088 and 1 KB reserved per CTA
// that is 232 192 of an SM's 233 472 bytes.  DESIGN.md section 3.3 gives the wider widths' footprints.
template <int T>
struct SmemSplit {
    static constexpr int BN = 2 * T;
    static constexpr int STAGE = Smem<BN>::STAGE;
    static constexpr int PART_BYTES = BM * T * 4;                      // one CTA's 128 x T fp32 partial
    static constexpr int SCRATCH = 16 * T + 128 > 512 ? 16 * T + 128 : 512;   // up to 8 stages of barriers + s_red [4][T]
    static constexpr int MAX_STAGES = (SCRATCH - 16 * T) / 16;
    static constexpr int ACC_STAGES = (Smem<BN>::ACC_BYTES + STAGE - 1) / STAGE;   // ring stages the staged accumulator covers
    static size_t bytes(int stages, int cluster) { return (size_t)stages * STAGE + (size_t)(cluster - 1) * PART_BYTES + SCRATCH; }
};

#ifdef B2A_TC_GEMM_IMPL   // the kernel body lives in tc_gemm.cu only
template <int T>
__global__ void __launch_bounds__(THREADS, 2)
tc_gemm_splitk_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, SplitArgs a) {
    constexpr int BN = 2 * T;
    using S = Smem<BN>;
    constexpr int LD = Cfg<BN>::LD;
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t C = cluster_nctarank(), rank = cluster_ctarank();
    float* part = reinterpret_cast<float*>(smem + (size_t)a.stages * S::STAGE);                 // [C - 1][128][T]
    float* sacc = reinterpret_cast<float*>(smem);                                                // [128][LD], over the ring
    uint64_t* full = reinterpret_cast<uint64_t*>(part + (size_t)(C - 1) * BM * T);
    uint64_t* empty = full + a.stages;
    float* s_red = reinterpret_cast<float*>(empty + a.stages);                                   // [4][T]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mt = blockIdx.x / C, m_tiles = gridDim.x / C;
    int kb0, kb1;
    split_range(a, mt, m_tiles, rank, C, kb0, kb1);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    check_smem_base(smem);
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < a.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 4); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 4) {
        if (lane == 0) {
            // weights first (they never depend on the previous kernel), then wait for it, then the activation tiles
            const int n = kb1 - kb0, npre = min(a.stages, n);
            for (int i = 0; i < npre; ++i) {
                mbar_arrive_expect_tx(&full[i], S::STAGE);
                tma_load_2d(smem + (size_t)i * S::STAGE, &tmA, &full[i], (kb0 + i) * BK, mt * BM);
            }
            asm volatile("griddepcontrol.wait;" ::: "memory");
            for (int i = 0; i < npre; ++i) tma_load_2d(smem + (size_t)i * S::STAGE + S::A_BYTES, &tmB, &full[i], (kb0 + i) * BK, 0);
            int stage = npre == a.stages ? 0 : npre;
            uint32_t phase = npre == a.stages ? 1 : 0;
            for (int i = npre; i < n; ++i) {
                mbar_wait(&empty[stage], phase ^ 1);
                uint8_t* sa = smem + (size_t)stage * S::STAGE;
                mbar_arrive_expect_tx(&full[stage], S::STAGE);
                tma_load_2d(sa, &tmA, &full[stage], (kb0 + i) * BK, mt * BM);
                tma_load_2d(sa + S::A_BYTES, &tmB, &full[stage], (kb0 + i) * BK, 0);
                if (++stage == a.stages) { stage = 0; phase ^= 1; }
            }
        }
    }
    // ---- epilogue part 1 (warps 0..3): this CTA's partial = hi + lo columns; non-leaders hand it to the leader
    float acc[T], hold[T], rstd[T];
    float g = 0.f;
    const int q = warp & 3, row = q * 32 + lane;
    const int m = mt * BM + row;
    const bool m_ok = m < a.M;
    if (warp < 4) {
        if (rank == 0) {
            // the residual rows, the gain and the input norm's sums of squares do not depend on this GEMM: fetch them while the
            // weights stream
            asm volatile("griddepcontrol.wait;" ::: "memory");
            if (a.h) {
                g = m_ok ? a.gain[m] : 0.f;
#pragma unroll
                for (int j = 0; j < T; ++j) hold[j] = (j < a.N && m_ok) ? a.h[(long long)j * a.M + m] : 0.f;
            }
            if (a.rstd_ss) {
                // rstd of the norm this GEMM's input went through (its producer wrote un-normalised hi/lo rows), reduced as
                // tc_gemm_kernel does: one independent load per lane and step (lane = part * 8 + token), per group of 8 tokens
#pragma unroll
                for (int g0 = 0; g0 < T; g0 += 8) {
                    float t = 0.f;
                    for (int p0 = 0; p0 < a.rstd_parts; p0 += 4) {
                        const int p = p0 + (lane >> 3);
                        if (p < a.rstd_parts) t += a.rstd_ss[p * T + g0 + (lane & 7)];
                    }
                    t += __shfl_xor_sync(0xffffffffu, t, 8);
                    t += __shfl_xor_sync(0xffffffffu, t, 16);
                    const float rs = rsqrtf(t * a.rstd_inv_h + a.rstd_eps);
#pragma unroll
                    for (int j = 0; j < 8; ++j) rstd[g0 + j] = __shfl_sync(0xffffffffu, rs, j);
                }
            }
        }
        float d[2][T];
#pragma unroll
        for (int rb = 0; rb < 2; ++rb)
#pragma unroll
            for (int i = 0; i < T; ++i) d[rb][i] = 0.f;
        int stage = 0; uint32_t phase = 0;
        for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait(&full[stage], phase);
            const uint32_t sa = smem_u32(smem + (size_t)stage * S::STAGE);
            wg_fence();
#pragma unroll
            for (int k = 0; k < BK / UMMA_K; ++k) {
#pragma unroll
                for (int rb = 0; rb < 2; ++rb)
                    wgmma_bf16<BN>(d[rb], make_smem_desc(sa + (uint32_t)(rb * 64 * 128)) + (uint64_t)(2 * k),
                                   make_smem_desc(sa + S::A_BYTES) + (uint64_t)(2 * k), (kb == kb0 && k == 0) ? 0u : 1u);
            }
            wg_commit();
            wg_wait0();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[stage]);
            if (++stage == a.stages) { stage = 0; phase ^= 1; }
        }
        named_sync(3, 128);                                      // every warp's last wgmma has read the ring: it is free
#pragma unroll
        for (int rb = 0; rb < 2; ++rb) {
            wg_fence_operand(d[rb]);
            store_frag<BN>(sacc, LD, d[rb], rb * 64, 0);
        }
        named_sync(3, 128);
        if constexpr (T == 8) {
            float v[16];
            ld_acc16(sacc + (size_t)row * LD, v);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = v[j] + v[j + 8];
        } else {
#pragma unroll
        for (int j0 = 0; j0 < T; j0 += 8) {                      // hi column j0 + j pairs with lo column T + j0 + j
            float hi[8], lo[8];
            const float4* ph = reinterpret_cast<const float4*>(sacc + (size_t)row * LD + j0);
            const float4* pl = reinterpret_cast<const float4*>(sacc + (size_t)row * LD + T + j0);
            const float4 h0 = ph[0], h1 = ph[1], l0 = pl[0], l1 = pl[1];
            hi[0] = h0.x; hi[1] = h0.y; hi[2] = h0.z; hi[3] = h0.w; hi[4] = h1.x; hi[5] = h1.y; hi[6] = h1.z; hi[7] = h1.w;
            lo[0] = l0.x; lo[1] = l0.y; lo[2] = l0.z; lo[3] = l0.w; lo[4] = l1.x; lo[5] = l1.y; lo[6] = l1.z; lo[7] = l1.w;
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j0 + j] = hi[j] + lo[j];
        }
        }
        if (rank != 0) {
            const uint32_t dst = map_to_rank(smem_u32(part + ((size_t)(rank - 1) * BM + row) * T), 0);
#pragma unroll
            for (int j = 0; j < T; j += 4) st_cluster_f4(dst + 4 * j, acc[j], acc[j + 1], acc[j + 2], acc[j + 3]);
        }
    }
    __syncwarp();
    cluster_sync_all();                                          // partials are in the leader's shared memory
    if (rank == 0 && warp < 4) {
        if (!a.h) {
            // store mode: each CTA's piece scaled by rstd, the pieces added to 0 in rank order, with no fused multiply-add -- the
            // arithmetic of tc_gemm_kernel's stream-K epilogue and slot reduction (a CTA with an empty piece has no slot there)
            float sum[T];
#pragma unroll
            for (int j = 0; j < T; ++j) sum[j] = __fadd_rn(0.f, a.rstd_ss ? __fmul_rn(acc[j], rstd[j]) : acc[j]);
            for (uint32_t r = 1; r < C; ++r) {
                int r0, r1;
                split_range(a, mt, m_tiles, (int)r, (int)C, r0, r1);
                if (r0 == r1) continue;
                const float* p = part + ((size_t)(r - 1) * BM + row) * T;
#pragma unroll
                for (int j = 0; j < T; ++j) sum[j] = __fadd_rn(sum[j], a.rstd_ss ? __fmul_rn(p[j], rstd[j]) : p[j]);
            }
#pragma unroll
            for (int j = 0; j < T; ++j)
                if (j < a.N && m_ok) a.out[(long long)j * a.M + m] = sum[j];
            return;
        }
        for (uint32_t r = 1; r < C; ++r) {                       // fixed order: deterministic sums
            const float4* p = reinterpret_cast<const float4*>(part + ((size_t)(r - 1) * BM + row) * T);
#pragma unroll
            for (int j = 0; j < T; j += 4) {
                const float4 pv = p[j / 4];
                acc[j] += pv.x; acc[j + 1] += pv.y; acc[j + 2] += pv.z; acc[j + 3] += pv.w;
            }
        }
        if (a.rstd_ss) {
#pragma unroll
            for (int j = 0; j < T; ++j) acc[j] *= rstd[j];
        }
        const int w4 = warp;                                     // 0..3 (s_red rows)
        float sq[T];
#pragma unroll
        for (int j = 0; j < T; ++j) {
            float hv = 0.f;
            if (j < a.N && m_ok) {
                hv = hold[j] + acc[j];
                a.h[(long long)j * a.M + m] = hv;
                const float t = hv * g;
                const __nv_bfloat16 hi = __float2bfloat16_rn(t);
                a.xn[(long long)j * a.M + m] = hi;
                a.xn[(long long)(T + j) * a.M + m] = __float2bfloat16_rn(t - __bfloat162float(hi));
            }
            sq[j] = hv * hv;
        }
#pragma unroll
        for (int j = 0; j < T; ++j) {
#pragma unroll
            for (int o = 16; o; o >>= 1) sq[j] += __shfl_xor_sync(0xffffffffu, sq[j], o);
        }
        if (lane == 0) {
#pragma unroll
            for (int j = 0; j < T; ++j) s_red[w4 * T + j] = sq[j];
        }
        asm volatile("bar.sync 2, 128;" ::: "memory");
        if (w4 == 0 && lane < T) a.ss[mt * T + lane] = s_red[lane] + s_red[T + lane] + s_red[2 * T + lane] + s_red[3 * T + lane];
    }
}
#endif  // B2A_TC_GEMM_IMPL

// ----------------------------------------------------------------------------------------------- host
// 2-D bf16 (f16 != 0: fp16) row-major [rows, cols] tensor map with a {64, box_rows} box and 128-byte swizzle
CUtensorMap make_tmap_bf16(const void* base, long long rows, long long cols, int box_rows, int f16 = 0);
CUtensorMap make_tmap_f16_3d(const void* base, long long d0, long long d1, long long d2, int b0, int b1);
// planar hi/lo activations [2][B][Ttot][C], bf16 (f16 != 0: fp16) -> rank-4 map {C, Ttot, B, 2}, box {64, box_frames, 1, 2}, 128-byte swizzle
CUtensorMap make_tmap_planes(const void* base, int C, long long Ttot, int B, int box_frames, int f16);

// share_sm: ask for the largest shared-memory carve-out at this launch (a decode-step GEMM whose neighbours share its SM)
template <int BN>
void launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const Args& a, int ctas, int n_tiles, cudaStream_t s, bool share_sm = false);

// tc_gemm_splitk_kernel<T>: T = the decode width (8, 16 or 32), X a [2T, K] hi/lo map with 2T-row boxes
template <int T>
void launch_splitk(const CUtensorMap& tmA, const CUtensorMap& tmB, const SplitArgs& a, int m_tiles, int cluster, cudaStream_t s);
// clusters of `cluster` tc_gemm_splitk_kernel<T> CTAs of smem_bytes dynamic shared memory the current device can hold at once
// (cudaOccupancyMaxActiveClusters: the clusters' GPC placement is part of the answer).  Needs set_attributes().
template <int T>
int splitk_active_clusters(int cluster, size_t smem_bytes);

void set_attributes();   // cudaFuncSetAttribute for every instantiation (call once, outside graph capture)

}  // namespace tc
}  // namespace b2a
