// Host side of the wgmma/TMA GEMM: tensor-map creation (driver entry point fetched at run time so the
// library has no link-time dependency on libcuda) and launch wrappers.
#define B2A_TC_GEMM_IMPL
#include "common.cuh"
#include "tc_gemm.cuh"

namespace b2a {
namespace tc {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        B2A_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
        B2A_CHECK(p && q == cudaDriverEntryPointSuccess, B2A_ERR_CUDA, "cuTensorMapEncodeTiled is not available in this driver");
        fn = (EncodeTiledFn)p;
    }
    return fn;
}

static CUtensorMapDataType type16(int f16) { return f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16; }

CUtensorMap make_tmap_bf16(const void* base, long long rows, long long cols, int box_rows, int f16) {
    B2A_CHECK(cols % 8 == 0 && ((uintptr_t)base & 15) == 0, B2A_ERR_INVALID_INPUT, "TMA: tensor must be 16-byte aligned with cols % 8 == 0");
    CUtensorMap m;
    const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
    const cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = encode_fn()(&m, type16(f16), 2, const_cast<void*>(base), dims, strides, box, estr,
                                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B2A_CHECK(r == CUDA_SUCCESS, B2A_ERR_CUDA, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
    return m;
}

// 3-D fp16 tensor [d2][d1][d0] (d0 contiguous), box {b0, b1, 1}, 128-byte swizzle (b0 * 2 bytes must be 128): attn_tc.cuh's operands
CUtensorMap make_tmap_f16_3d(const void* base, long long d0, long long d1, long long d2, int b0, int b1) {
    B2A_CHECK(b0 * 2 == 128 && d0 % 8 == 0 && ((uintptr_t)base & 15) == 0, B2A_ERR_INVALID_INPUT, "TMA: bad 3-D fp16 tensor");
    CUtensorMap m;
    const cuuint64_t dims[3] = {(cuuint64_t)d0, (cuuint64_t)d1, (cuuint64_t)d2};
    const cuuint64_t strides[2] = {(cuuint64_t)d0 * 2, (cuuint64_t)d0 * (cuuint64_t)d1 * 2};
    const cuuint32_t box[3] = {(cuuint32_t)b0, (cuuint32_t)b1, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B2A_CHECK(r == CUDA_SUCCESS, B2A_ERR_CUDA, "cuTensorMapEncodeTiled (3-D fp16) failed (" + std::to_string((int)r) + ")");
    return m;
}

// the operand of the implicit convolution (conv_gemm.cuh): one box is 64 channels of box_frames frames, hi plane then lo plane
CUtensorMap make_tmap_planes(const void* base, int C, long long Ttot, int B, int box_frames, int f16) {
    B2A_CHECK(C % 8 == 0 && ((uintptr_t)base & 15) == 0 && Ttot >= 1 && B >= 1, B2A_ERR_INVALID_INPUT,
              "TMA: activation planes must be 16-byte aligned with channels % 8 == 0");
    CUtensorMap m;
    const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)Ttot, (cuuint64_t)B, 2};
    const cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)Ttot * C * 2, (cuuint64_t)B * Ttot * C * 2};
    const cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)box_frames, 1, 2};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    const CUresult r = encode_fn()(&m, type16(f16), 4, const_cast<void*>(base), dims, strides, box, estr,
                                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B2A_CHECK(r == CUDA_SUCCESS, B2A_ERR_CUDA, "cuTensorMapEncodeTiled (rank 4) failed (" + std::to_string((int)r) + ")");
    return m;
}

template <int BN>
void launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const Args& a, int ctas, int n_tiles, cudaStream_t s, bool share_sm) {
    B2A_CHECK(a.stages >= 1 && a.stages <= Smem<BN>::max_stages(), B2A_ERR_INVALID_INPUT, "tc_gemm: ring depth does not fit in shared memory");
    B2A_CHECK(a.epi_partial < 0 || (a.part_ws && a.part_cnt && a.part_slots >= stream_k_slots(a.m_tiles, a.k_blocks, ctas)),
              B2A_ERR_INVALID_INPUT, "tc_gemm: stream-K workspace missing or too small");
    if (!share_sm) {
        launch_pdl(tc_gemm_kernel<BN>, dim3(ctas, n_tiles), dim3(Cfg<BN>::NTHREADS), Smem<BN>::bytes(a.stages), s, tmA, tmB, a);
        return;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(ctas, n_tiles); cfg.blockDim = dim3(Cfg<BN>::NTHREADS); cfg.dynamicSmemBytes = Smem<BN>::bytes(a.stages); cfg.stream = s;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    at[1].id = cudaLaunchAttributePreferredSharedMemoryCarveout;
    at[1].val.sharedMemCarveout = cudaSharedmemCarveoutMaxShared;
    cfg.attrs = at; cfg.numAttrs = 2;
    B2A_CUDA(cudaLaunchKernelEx(&cfg, tc_gemm_kernel<BN>, tmA, tmB, a));
    count_launch();
}
template void launch<16>(const CUtensorMap&, const CUtensorMap&, const Args&, int, int, cudaStream_t, bool);
template void launch<32>(const CUtensorMap&, const CUtensorMap&, const Args&, int, int, cudaStream_t, bool);
template void launch<64>(const CUtensorMap&, const CUtensorMap&, const Args&, int, int, cudaStream_t, bool);
template void launch<128>(const CUtensorMap&, const CUtensorMap&, const Args&, int, int, cudaStream_t, bool);

template <int T>
void launch_splitk(const CUtensorMap& tmA, const CUtensorMap& tmB, const SplitArgs& a, int m_tiles, int cluster, cudaStream_t s) {
    using SS = SmemSplit<T>;
    B2A_CHECK(SS::bytes(a.stages, cluster) <= 227 * 1024, B2A_ERR_INVALID_INPUT, "tc_gemm: split-K ring does not fit in shared memory");
    B2A_CHECK(a.stages >= SS::ACC_STAGES && a.stages <= SS::MAX_STAGES, B2A_ERR_INVALID_INPUT,
              "tc_gemm: split-K ring too shallow for the staged accumulator or too deep for the barrier scratch");
    B2A_CHECK(a.N >= 1 && a.N <= T, B2A_ERR_INVALID_INPUT, "tc_gemm: split-K token count exceeds the width");
    B2A_CHECK(a.sk_ctas <= 0 || (!a.h && cluster >= stream_k_slots(m_tiles, a.k_blocks, a.sk_ctas)), B2A_ERR_INVALID_INPUT,
              "tc_gemm: the stream-K cut is a store-mode option and needs a CTA per piece of a tile");
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)(m_tiles * cluster)); cfg.blockDim = dim3(THREADS);
    cfg.dynamicSmemBytes = SS::bytes(a.stages, cluster); cfg.stream = s;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    at[1].id = cudaLaunchAttributeClusterDimension;
    at[1].val.clusterDim.x = (unsigned)cluster; at[1].val.clusterDim.y = 1; at[1].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 2;
    B2A_CUDA(cudaLaunchKernelEx(&cfg, tc_gemm_splitk_kernel<T>, tmA, tmB, a));
    count_launch();
}
template void launch_splitk<8>(const CUtensorMap&, const CUtensorMap&, const SplitArgs&, int, int, cudaStream_t);
template void launch_splitk<16>(const CUtensorMap&, const CUtensorMap&, const SplitArgs&, int, int, cudaStream_t);
template void launch_splitk<32>(const CUtensorMap&, const CUtensorMap&, const SplitArgs&, int, int, cudaStream_t);

template <int T>
int splitk_active_clusters(int cluster, size_t smem_bytes) {
    B2A_CHECK(cluster >= 1 && cluster <= SPLIT_MAX_CLUSTER, B2A_ERR_INVALID_INPUT, "tc_gemm: split-K cluster size must be in [1, 8]");
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)cluster); cfg.blockDim = dim3(THREADS);
    cfg.dynamicSmemBytes = smem_bytes;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)cluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    int n = 0;
    B2A_CUDA(cudaOccupancyMaxActiveClusters(&n, tc_gemm_splitk_kernel<T>, &cfg));
    return n;
}
template int splitk_active_clusters<8>(int, size_t);
template int splitk_active_clusters<16>(int, size_t);
template int splitk_active_clusters<32>(int, size_t);

void set_attributes() {
    // the decode-step kernels are sized to share an SM with their neighbours in the step (Smem / SmemSplit): ask for the largest
    // shared-memory carve-out, or an SM configured for one kernel's footprint alone cannot take the next kernel's CTA beside it
    for (auto k : {tc_gemm_splitk_kernel<8>, tc_gemm_splitk_kernel<16>, tc_gemm_splitk_kernel<32>}) {
        B2A_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        B2A_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    }
    for (auto k : {tc_gemm_kernel<16>, tc_gemm_kernel<64>}) {
        B2A_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        B2A_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    }
    // tc_gemm_kernel<32> also serves Whisper's decoder, which keeps the default carve-out: the 16-row decode step asks for the largest
    // one per launch (launch(..., share_sm))
    B2A_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    B2A_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
}

}  // namespace tc
}  // namespace b2a

// Standalone entries (include/b200audio_internal.h): one launch of tc_gemm_kernel / tc_gemm_splitk_kernel on DEVICE pointers,
// with the epilogue options the engines' call sites use.

// out[N, M] = X[N, K] * W[M, K]^T through tc_gemm_kernel<bn>.  hilo: X holds cdiv(N, bn / 2) tiles of bn rows (hi rows, then lo rows).
// split != 0 lets CTAs own partial K ranges (stream-K): epi must then be a store into or an add into the caller's fp32 out.
extern "C" int32_t b2a_tc_gemm_epilogue_test(const void* W, const void* X, void* out, int32_t M, int32_t N, int32_t K, int32_t bn,
                                             int32_t epi, int32_t split, int32_t hilo, int32_t ctas, const float* bias, int32_t act,
                                             int32_t tile_rows, int32_t lo_rows, const float* rstd_ss, int32_t rstd_parts,
                                             float rstd_eps, int32_t stages, void* stream) {
    using namespace b2a;
    using namespace b2a::tc;
    return guarded([&] {
        B2A_CHECK(W && X && out && (bn == 16 || bn == 32 || bn == 128) && K % BK == 0 && M > 0 && N > 0 && ctas > 0, B2A_ERR_INVALID_INPUT,
                  "b2a_tc_gemm_epilogue_test: bad argument");
        B2A_CHECK(epi == EPI_STORE || epi == EPI_SWIGLU || epi == EPI_STORE_BF16 || epi == EPI_ADD, B2A_ERR_INVALID_INPUT,
                  "b2a_tc_gemm_epilogue_test: unknown epilogue");
        B2A_CHECK(act == ACT_NONE || act == ACT_GELU, B2A_ERR_INVALID_INPUT, "b2a_tc_gemm_epilogue_test: unknown activation");
        B2A_CHECK(!split || epi == EPI_STORE || epi == EPI_ADD, B2A_ERR_INVALID_INPUT,
                  "b2a_tc_gemm_epilogue_test: stream-K partial tiles are summed into fp32 outputs only");
        B2A_CHECK(!split || act == ACT_NONE, B2A_ERR_INVALID_INPUT, "b2a_tc_gemm_epilogue_test: GELU of a partial K range is not the GELU of the sum");
        B2A_CHECK(!split || tile_rows == 0, B2A_ERR_INVALID_INPUT, "b2a_tc_gemm_epilogue_test: tile_rows is a whole-tile option");
        B2A_CHECK(tile_rows == 0 || (tile_rows % 8 == 0 && tile_rows >= 8 && tile_rows <= BM), B2A_ERR_INVALID_INPUT,
                  "b2a_tc_gemm_epilogue_test: tile_rows must be a multiple of 8 in [8, 128]");
        B2A_CHECK(!lo_rows || (hilo && (epi == EPI_SWIGLU || epi == EPI_STORE_BF16)), B2A_ERR_INVALID_INPUT,
                  "b2a_tc_gemm_epilogue_test: hi/lo outputs need hi/lo inputs and a bf16 epilogue");
        B2A_CHECK(epi != EPI_SWIGLU || M % 2 == 0, B2A_ERR_INVALID_INPUT, "b2a_tc_gemm_epilogue_test: SwiGLU needs (gate, up) row pairs");
        B2A_CHECK(!rstd_ss || (bn == 16 && hilo && N <= 8 && rstd_parts >= 1), B2A_ERR_INVALID_INPUT,
                  "b2a_tc_gemm_epilogue_test: the fused RMSNorm scale is a BN = 16 hi/lo option");
        require_device(0);
        set_attributes();
        const int n_tiles = hilo ? cdiv(N, bn / 2) : cdiv(N, bn);
        B2A_CHECK(n_tiles <= 65535, B2A_ERR_INVALID_INPUT, "b2a_tc_gemm_epilogue_test: too many tokens");
        const int x_rows = hilo ? n_tiles * bn : N;
        const int TR = tile_rows > 0 ? tile_rows : BM;
        CUtensorMap ta = make_tmap_bf16(W, M, K, TR), tb = make_tmap_bf16(X, x_rows, K, bn);
        Args a{};
        a.out_f32 = (float*)out; a.out_bf16 = (__nv_bfloat16*)out; a.M = M; a.N = N; a.K = K;
        a.ldo = epi == EPI_SWIGLU ? M / 2 : M;
        a.tile_rows = tile_rows; a.m_tiles = cdiv(M, TR); a.k_blocks = K / BK;
        const int max_st = bn == 16 ? Smem<16>::max_stages() : bn == 32 ? Smem<32>::max_stages() : Smem<128>::max_stages();
        a.stages = stages > 0 ? stages : max_st;
        a.epi_full = epi; a.epi_partial = split ? EPI_PARTIAL : -1; a.hilo = hilo;
        a.bias = bias; a.act = act;
        a.lo_rows = lo_rows ? bn / 2 : 0;
        a.rstd_ss = rstd_ss; a.rstd_parts = rstd_parts; a.rstd_inv_h = 1.0f / (float)K; a.rstd_eps = rstd_eps;
        DBuf<float> ws;
        DBuf<unsigned> cnt;
        if (split) {
            a.part_slots = stream_k_slots(a.m_tiles, a.k_blocks, ctas);
            ws.alloc((size_t)n_tiles * a.m_tiles * a.part_slots * bn * BM);
            cnt.alloc((size_t)n_tiles * a.m_tiles);
            B2A_CUDA(cudaMemset(cnt.p, 0, (size_t)n_tiles * a.m_tiles * sizeof(unsigned)));
            a.part_ws = ws.p; a.part_cnt = cnt.p;
        }
        if (bn == 16) launch<16>(ta, tb, a, ctas, n_tiles, (cudaStream_t)stream);
        else if (bn == 32) launch<32>(ta, tb, a, ctas, n_tiles, (cudaStream_t)stream);
        else launch<128>(ta, tb, a, ctas, n_tiles, (cudaStream_t)stream);
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    });
}

// The plain GEMM with no bias, activation, tile_rows or norm scale and the deepest ring; bf16 epilogues of hi/lo inputs write hi/lo rows.
extern "C" int32_t b2a_tc_gemm_test(const void* W, const void* X, void* out, int32_t M, int32_t N, int32_t K, int32_t bn,
                                    int32_t epi, int32_t split, int32_t hilo, int32_t ctas, void* stream) {
    const int32_t lo_rows = hilo && (epi == b2a::tc::EPI_SWIGLU || epi == b2a::tc::EPI_STORE_BF16);
    return b2a_tc_gemm_epilogue_test(W, X, out, M, N, K, bn, epi, split, hilo, ctas, nullptr, b2a::tc::ACT_NONE, 0, lo_rows, nullptr, 0,
                                     0.f, 0, stream);
}

// The decode step's o_proj / down_proj GEMM: h[t] += W * (x_hi[t] + x_lo[t]) for t < N, then xn = hi / lo of h * gain and
// ss[m_tile, t] = sum over the tile's rows of h^2, one cluster of `cluster` CTAs per 128-row tile.
extern "C" int32_t b2a_tc_gemm_splitk_test(const void* W, const void* X, float* h, const float* gain, void* xn, float* ss, int32_t M,
                                           int32_t N, int32_t K, int32_t cluster, int32_t stages, void* stream) {
    using namespace b2a;
    using namespace b2a::tc;
    return guarded([&] {
        B2A_CHECK(W && X && h && gain && xn && ss && M > 0 && M % 8 == 0 && K > 0 && K % BK == 0 && N >= 1 && N <= 8 && stages >= 1,
                  B2A_ERR_INVALID_INPUT, "b2a_tc_gemm_splitk_test: bad argument");
        B2A_CHECK(cluster >= 1 && cluster <= SPLIT_MAX_CLUSTER && cluster <= K / BK, B2A_ERR_INVALID_INPUT,
                  "b2a_tc_gemm_splitk_test: cluster must be in [1, min(8, K / 64)]");
        require_device(0);
        set_attributes();
        CUtensorMap ta = make_tmap_bf16(W, M, K, BM), tb = make_tmap_bf16(X, 16, K, 16);
        SplitArgs a{};
        a.M = M; a.N = N; a.K = K; a.k_blocks = K / BK; a.stages = stages;
        a.h = h; a.gain = gain; a.xn = (__nv_bfloat16*)xn; a.ss = ss;
        launch_splitk<8>(ta, tb, a, cdiv(M, BM), cluster, (cudaStream_t)stream);
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    });
}

// The decode step's q|k|v GEMM: the same cluster split-K launch in store mode, out[t] = rstd[t] * W (x_hi[t] + x_lo[t]) for t < N,
// rstd[t] = rsqrt(sum_p rstd_ss[p, t] / K + rstd_eps) (rstd_ss nullable: rstd = 1); sk_ctas > 0: k-blocks cut as stream-K over sk_ctas CTAs.
extern "C" int32_t b2a_tc_gemm_splitk_store_test(const void* W, const void* X, float* out, const float* rstd_ss, int32_t rstd_parts,
                                                 float rstd_eps, int32_t M, int32_t N, int32_t K, int32_t cluster, int32_t sk_ctas,
                                                 int32_t stages, void* stream) {
    using namespace b2a;
    using namespace b2a::tc;
    return guarded([&] {
        B2A_CHECK(W && X && out && M > 0 && M % 8 == 0 && K > 0 && K % BK == 0 && N >= 1 && N <= 8 && stages >= 1 &&
                      (!rstd_ss || rstd_parts >= 1),
                  B2A_ERR_INVALID_INPUT, "b2a_tc_gemm_splitk_store_test: bad argument");
        B2A_CHECK(cluster >= 1 && cluster <= SPLIT_MAX_CLUSTER && cluster <= K / BK, B2A_ERR_INVALID_INPUT,
                  "b2a_tc_gemm_splitk_store_test: cluster must be in [1, min(8, K / 64)]");
        require_device(0);
        set_attributes();
        CUtensorMap ta = make_tmap_bf16(W, M, K, BM), tb = make_tmap_bf16(X, 16, K, 16);
        SplitArgs a{};
        a.M = M; a.N = N; a.K = K; a.k_blocks = K / BK; a.stages = stages; a.sk_ctas = sk_ctas;
        a.out = out;
        a.rstd_ss = rstd_ss; a.rstd_parts = rstd_parts; a.rstd_inv_h = 1.0f / (float)K; a.rstd_eps = rstd_eps;
        launch_splitk<8>(ta, tb, a, cdiv(M, BM), cluster, (cudaStream_t)stream);
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    });
}
