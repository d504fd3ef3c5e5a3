// Qwen3-TTS speech-tokenizer DECODER for sm_90a (SURVEY.md section 8f row N1: 12.5 Hz codes -> 24 kHz waveform).
// The ENCODER (24 kHz audio -> 12.5 Hz codes, voice cloning) is b2a_speech_tokenizer_encoder below, on the same kernels.
// Replaces (reference paths, file = Sources/MLXAudioTTS/Models/Qwen3TTS/Qwen3TTSSpeechTokenizer.swift):
//   :9-121      split residual vector quantizer decode (usage-normalised Euclidean codebooks, k1 output projections)
//   :135-232    CausalConv1d (+ streaming step), :257-297 ConvNeXtBlock, :301-491 DecoderTransformer (KV cache)
//   :495-638    DecoderResidualUnit / DecoderBlockUpsample / DecoderBlock, :641-731 initial / output convs, SnakeBeta
//   :888-1025   Qwen3TTSSpeechTokenizerDecoder: callAsFunction, streamingStep, chunkedDecode
//   :1070-1092  Qwen3TTSSpeechTokenizer.streamingDecode
// EXPERIMENTAL -- written against oracle/qwen3_tts_codec.py but NOT yet run on a GPU (no GPU time was left in the
// round that added it); its parity tests are gated behind B2A_EXPERIMENTAL_N1=1.  Nothing else in the library calls it.
//
// Design.  Every chunk of code frames is decoded by the streaming step with carried state; the one-shot call is the
// same step after a reset (zero state == the reference's causal zero padding).  All dense layers -- RVQ projections,
// k3 / k7 / dilated causal convolutions, transposed convolutions (as phase-major causal convolutions), transformer
// and ConvNeXt linears -- run on the implicit-GEMM wgmma kernel of conv_gemm.cuh over planar bf16 hi/lo
// activations; its epilogue fuses bias, layer scale / gamma, exact GELU, the residual add, the next layer's SnakeBeta
// and the hi/lo split, and writes behind the H history frames the consumer's taps reach back over.  Small SIMT
// kernels cover the gathers, norms, RoPE + attention over the cache, the depthwise conv + LayerNorm and the 1-channel
// output conv.  The reference's double-counted transposed-conv bias at chunk boundaries (see the oracle's header) is
// reproduced (Args::bias_twice_t0).
#include "common.cuh"
#include "conv_gemm.cuh"
#include "seanet.cuh"
#include "codec_transformer.cuh"

#include <algorithm>
#include <cmath>
#include <cstdlib>

namespace b2a {
namespace st {

// ----------------------------------------------------------------------------------------------- SIMT kernels
// (the gathers, LayerNorm, RoPE, attention and history carries shared with Mimi are in codec_transformer.cuh)
// RMSNorm over channels -> planes [2][N][C]   (DecoderRMSNorm :301-314: w * (x * rsqrt(mean(x^2) + eps)))
__global__ void __launch_bounds__(RN_THREADS)
rmsnorm_planes_kernel(const float* __restrict__ x, const float* __restrict__ w, bf16* __restrict__ out, long long N, int C, float eps, int f16) {
    __shared__ float red[RN_THREADS / 32];
    const long long n = blockIdx.x;
    float ss = 0.f;
    for (int c = threadIdx.x; c < C; c += RN_THREADS) { const float v = x[n * C + c]; ss += v * v; }
    const float r = rsqrtf(block_sum<RN_THREADS>(ss, red) / (float)C + eps);
    for (int c = threadIdx.x; c < C; c += RN_THREADS) put_planes(out, N * C, n * C + c, w[c] * (x[n * C + c] * r), f16);
}

// The split quantizer's k1 input projections in ordered fp32, so that the code search is a function of z alone:
// out[r][o] = sum over d = 0..K-1 of fl(wt[d][o] * x[r][d]), accumulated in order without contraction.  x [rows, K], wt [K, M]
// (transposed: a warp reads 32 consecutive outputs' weights), out [rows, M].  PJ_R rows per CTA share their x tile in shared memory.
constexpr int PJ_R = 8, PJ_THREADS = 256;
__global__ void __launch_bounds__(PJ_THREADS)
ordered_proj_kernel(const float* __restrict__ x, const float* __restrict__ wt, float* __restrict__ out, int rows, int K, int M) {
    extern __shared__ float xs[];          // [PJ_R][K]
    const int r0 = blockIdx.x * PJ_R, o = blockIdx.y * PJ_THREADS + threadIdx.x;
    for (int e = threadIdx.x; e < PJ_R * K; e += PJ_THREADS) {
        const int r = e / K;
        xs[e] = r0 + r < rows ? x[(long long)(r0 + r) * K + (e - r * K)] : 0.f;
    }
    __syncthreads();
    if (o >= M) return;
    float acc[PJ_R];
#pragma unroll
    for (int r = 0; r < PJ_R; ++r) acc[r] = 0.f;
    for (int d = 0; d < K; ++d) {
        const float wv = wt[(long long)d * M + o];
#pragma unroll
        for (int r = 0; r < PJ_R; ++r) acc[r] = __fadd_rn(acc[r], __fmul_rn(wv, xs[r * K + d]));
    }
#pragma unroll
    for (int r = 0; r < PJ_R; ++r)
        if (r0 + r < rows) out[(long long)(r0 + r) * M + o] = acc[r];
}

// gu [N, 2I] (gate | up) -> silu(gate) * up as planes [2][N][I]     (DecoderMLP :412-414)
__global__ void swiglu_planes_kernel(const float* __restrict__ gu, bf16* __restrict__ out, long long N, int I, int f16) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * I) return;
    const long long n = i / I;
    const int c = (int)(i - n * I);
    const float g = gu[n * 2 * I + c], u = gu[n * 2 * I + I + c];
    put_planes(out, N * I, i, g / (1.0f + __expf(-g)) * u, f16);
}

// causal depthwise conv (k taps, history from `st` [B, k-1, C]) -> LayerNorm(eps) -> planes [2][B*T][C]
constexpr int DL_THREADS = 256, DL_MAXV = 4;    // channels <= 1024
__global__ void __launch_bounds__(DL_THREADS)
dw_ln_kernel(const float* __restrict__ x, const float* __restrict__ st, const float* __restrict__ dw_w /*[C, k]*/, const float* __restrict__ dw_b,
             const float* __restrict__ ln_w, const float* __restrict__ ln_b, bf16* __restrict__ out, int B, int T, int C, int k, float eps, int f16) {
    __shared__ float red[DL_THREADS / 32];
    const long long n = blockIdx.x;
    const int b = (int)(n / T), t = (int)(n - (long long)b * T), H = k - 1;
    float v[DL_MAXV];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < DL_MAXV; ++j) {
        const int c = threadIdx.x + j * DL_THREADS;
        float val = 0.f;
        if (c < C) {
            val = dw_b[c];
            for (int kk = 0; kk < k; ++kk) {
                const int ti = t - H + kk;
                const float xin = ti >= 0 ? x[((long long)b * T + ti) * C + c] : st[((long long)b * H + (H + ti)) * C + c];
                val = fmaf(dw_w[c * k + kk], xin, val);
            }
        }
        v[j] = val;
        s += val;
    }
    const float mean = block_sum<DL_THREADS>(s, red) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < DL_MAXV; ++j) {
        const int c = threadIdx.x + j * DL_THREADS;
        if (c < C) { const float d = v[j] - mean; q += d * d; }
    }
    const float r = rsqrtf(block_sum<DL_THREADS>(q, red) / (float)C + eps);
    const long long N = (long long)B * T;
#pragma unroll
    for (int j = 0; j < DL_MAXV; ++j) {
        const int c = threadIdx.x + j * DL_THREADS;
        if (c < C) put_planes(out, N * C, n * C + c, (v[j] - mean) * r * ln_w[c] + ln_b[c], f16);
    }
}

// SnakeBeta -> causal k-tap conv to ONE channel -> clip(-1, 1)          (DecoderOutputSnake + DecoderOutputConv :693-731, :946)
// x [B, T, C] fp32 (raw, pre-activation), st [B, k-1, C] raw history.  64 outputs per CTA; the activated tile lives in smem.
constexpr int FC_TILE = 64, FC_THREADS = 128, FC_MAXK = 8;
__global__ void __launch_bounds__(FC_THREADS)
final_conv_kernel(const float* __restrict__ x, const float* __restrict__ st, const float* __restrict__ sa, const float* __restrict__ sb,
                  const float* __restrict__ w /*[k, C]*/, float bias, float* __restrict__ wave, int T, int C, int k) {
    extern __shared__ float fsm[];
    const int H = k - 1, rows = FC_TILE + H, ldc = C + 1;
    float* tile = fsm;                    // [rows][C + 1]
    float* wk = fsm + rows * ldc;         // [k][C]
    float* red = wk + k * C;              // [FC_THREADS]
    const int b = blockIdx.y, t0 = blockIdx.x * FC_TILE;
    for (int i = threadIdx.x; i < k * C; i += FC_THREADS) wk[i] = w[i];
    for (int i = threadIdx.x; i < rows * C; i += FC_THREADS) {
        const int rr = i / C, c = i - rr * C;
        const int ti = t0 - H + rr;
        float v = 0.f;
        if (ti >= 0) { if (ti < T) v = x[((long long)b * T + ti) * C + c]; }
        else v = st[((long long)b * H + (H + ti)) * C + c];
        tile[rr * ldc + c] = cg::snake_inv(v, sa[c], sb[c]);
    }
    __syncthreads();
    const int o = threadIdx.x & (FC_TILE - 1), part = threadIdx.x / FC_TILE;      // two threads per output, channels split in halves
    const int cbeg = part * ((C + 1) / 2), cend = min(C, cbeg + (C + 1) / 2);
    float acc = 0.f;
    for (int kk = 0; kk < k; ++kk)
        for (int c = cbeg; c < cend; ++c) acc = fmaf(wk[kk * C + c], tile[(o + kk) * ldc + c], acc);
    red[threadIdx.x] = acc;
    __syncthreads();
    if (part == 0 && t0 + o < T) {
        const float y = red[o] + red[o + FC_TILE] + bias;
        wave[(long long)b * T + t0 + o] = fminf(1.0f, fmaxf(-1.0f, y));
    }
}

// ----------------------------------------------------------------------------------------------- weights
using cg::TcW;

struct Snake { DBuf<float> a, ib; };                 // a = exp(alpha), ib = 1 / (exp(beta) + 1e-9)

struct TLayer { TcW qkv, o, gu, down; DBuf<float> ln1, ln2, sc_attn, sc_mlp; DBuf<float> K, V; };
struct UpLayer { TcW ct, pw1, pw2; DBuf<float> dw_w, dw_b, ln_w, ln_b, gamma; F32State st; int factor = 1; };
struct ResUnit { Snake a1, a2; TcW c1, c2; PlaneState st; int dil = 1; };
struct DecBlock { Snake sn; TcW ct; PlaneState st; ResUnit ru[3]; int rate = 1, cin = 0, cout = 0; };

}  // namespace st
}  // namespace b2a

using namespace b2a;
using namespace b2a::st;

struct b2a_speech_tokenizer {
    int device;
    b2a_speech_tokenizer_config cfg;
    cudaStream_t stream = nullptr;
    int num_sms = 132;
    int total_up = 1, D2 = 0, Mqkv = 0;
    int use_f16 = 1;              // fp16 hi/lo operand pairs (22 mantissa bits, saturating at 65504); B2A_ST_FP16=0: bf16 pairs (16 bits, fp32 range)
    // weights
    DBuf<float> emb;              // [nq][bins][D2] usage-normalised codebooks
    TcW rvq_proj, pre_conv, in_proj, out_proj, dec0;
    PlaneState st_pre, st_dec0;
    DBuf<float> final_norm, inv_freq;
    std::vector<TLayer> layers;
    std::vector<UpLayer> ups;
    std::vector<DecBlock> blocks;
    Snake out_snake;
    DBuf<float> out_w;            // [k][C]
    float out_b = 0.f;
    int out_k = 7;
    F32State st_out;
    // streaming state
    int parity = 0, chunk_idx = 0, cache_len = 0, stream_B = 0;
    // workspace
    DBuf<int> d_codes;
    DBuf<bf16> P0, P1;
    DBuf<float> Xh, Xc, Q, wave;
    // diagnostics (b2a_speech_tokenizer_debug_stage): a copy of the fp32 activation tensor after stage `dbg_stage`
    int dbg_stage = -1;
    long long dbg_n = 0;
    DBuf<float> dbg;
    void dbg_tap(int stage, const float* src, long long n, cudaStream_t s) {
        if (stage != dbg_stage) return;
        dbg.alloc((size_t)n);
        B2A_CUDA(cudaMemcpyAsync(dbg.p, src, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, s));
        dbg_n = n;
    }

    ~b2a_speech_tokenizer() { if (stream) cudaStreamDestroy(stream); }

    static std::vector<float> conv_w(const TensorTable& tt, const std::string& name, int out, int k, int in) {
        return tt.f32(name, (int64_t)out * k * in);       // MLX [out, k, in] == [M][taps][Cin] with tap j <-> kernel index j
    }
    static void up(DBuf<float>& d, const std::vector<float>& v) { d.upload(v.data(), v.size()); }
    static void load_snake(Snake& s, const TensorTable& tt, const std::string& p, int C) {
        std::vector<float> al = tt.f32(p + ".alpha", C), be = tt.f32(p + ".beta", C), a(C), ib(C);
        for (int c = 0; c < C; ++c) { a[c] = expf(al[c]); ib[c] = 1.0f / (expf(be[c]) + 1e-9f); }
        up(s.a, a); up(s.ib, ib);
    }
    void load_conv(TcW& w, const TensorTable& tt, const std::string& p, int out, int k, int in, bool bias = true) {
        w.build(conv_w(tt, p + ".weight", out, k, in), out, k, in, use_f16);
        if (bias) w.set_bias(tt.f32(p + ".bias", out));
    }
    void load_linear(TcW& w, const TensorTable& tt, const std::string& p, int out, int in, bool bias) {
        w.build(tt.f32(p + ".weight", (int64_t)out * in), out, 1, in, use_f16);
        if (bias) w.set_bias(tt.f32(p + ".bias", out));
    }

    b2a_speech_tokenizer(int dev, const b2a_speech_tokenizer_config& c, const TensorTable& tt) : device(dev), cfg(c) {
        B2A_CHECK(c.codebook_dim % 16 == 0 && c.latent_dim % 8 == 0 && c.hidden_size % 8 == 0 && c.intermediate_size % 8 == 0,
                  B2A_ERR_INVALID_INPUT, "speech tokenizer: channel counts must be multiples of 8 (codebook_dim of 16)");
        B2A_CHECK(c.head_dim == 32 || c.head_dim == 64 || c.head_dim == 128, B2A_ERR_INVALID_INPUT, "speech tokenizer: head_dim must be 32, 64 or 128");
        B2A_CHECK(c.num_attention_heads >= 1 && c.num_key_value_heads >= 1 && c.num_attention_heads % c.num_key_value_heads == 0,
                  B2A_ERR_INVALID_INPUT, "speech tokenizer: bad head counts");
        B2A_CHECK(c.num_upsample_rates >= 1 && c.num_upsample_rates <= 8 && c.num_upsampling_ratios >= 1 && c.num_upsampling_ratios <= 8,
                  B2A_ERR_INVALID_INPUT, "speech tokenizer: bad upsample lists");
        B2A_CHECK(c.num_quantizers >= 1 && c.num_semantic_quantizers >= 1 && c.num_semantic_quantizers <= c.num_quantizers && c.codebook_size >= 1,
                  B2A_ERR_INVALID_INPUT, "speech tokenizer: bad quantizer counts");
        B2A_CHECK(c.latent_dim <= DL_THREADS * DL_MAXV, B2A_ERR_INVALID_INPUT, "speech tokenizer: latent_dim must be <= 1024");
        B2A_CHECK((c.decoder_dim >> c.num_upsample_rates) >= 8 && (c.decoder_dim >> c.num_upsample_rates) % 8 == 0 &&
                      (c.decoder_dim >> c.num_upsample_rates) <= 128,
                  B2A_ERR_INVALID_INPUT, "speech tokenizer: decoder_dim / 2^blocks must be a multiple of 8 and <= 128");
        B2A_CHECK(c.max_batch >= 1 && c.max_cache_frames >= 1, B2A_ERR_INVALID_INPUT, "speech tokenizer: max_batch / max_cache_frames must be positive");
        require_device(dev);
        { const char* e = getenv("B2A_ST_FP16"); use_f16 = (e && e[0] == '0') ? 0 : 1; }
        B2A_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        B2A_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
        const int nq = c.num_quantizers, ns = c.num_semantic_quantizers, bins = c.codebook_size, cbd = c.codebook_dim, L = c.latent_dim,
                  Hd = c.hidden_size, I = c.intermediate_size, nh = c.num_attention_heads, nkv = c.num_key_value_heads, hd = c.head_dim;
        D2 = cbd / 2;
        Mqkv = (nh + 2 * nkv) * hd;
        // codebooks: embedding = embedding_sum / max(cluster_usage, 1e-5)      (Quantization.swift:29-33)
        {
            std::vector<float> e((size_t)nq * bins * D2);
            for (int qi = 0; qi < nq; ++qi) {
                const std::string p = qi < ns ? "quantizer.rvq_first.vq.layers." + std::to_string(qi) : "quantizer.rvq_rest.vq.layers." + std::to_string(qi - ns);
                std::vector<float> sum = tt.f32(p + ".codebook.embedding_sum", (int64_t)bins * D2), use = tt.f32(p + ".codebook.cluster_usage", bins);
                for (int r = 0; r < bins; ++r) {
                    const float u = std::max(use[r], 1e-5f);
                    for (int d = 0; d < D2; ++d) e[((size_t)qi * bins + r) * D2 + d] = sum[(size_t)r * D2 + d] / u;
                }
            }
            up(emb, e);
            // both k1 output projections as one [cbd, 2 * D2] matrix over the concatenated (semantic | rest) sums
            std::vector<float> w1 = tt.f32("quantizer.rvq_first.output_proj.weight", (int64_t)cbd * D2), w((size_t)cbd * 2 * D2, 0.f);
            std::vector<float> w2 = nq > ns ? tt.f32("quantizer.rvq_rest.output_proj.weight", (int64_t)cbd * D2) : std::vector<float>((size_t)cbd * D2, 0.f);
            for (int o = 0; o < cbd; ++o) {
                memcpy(&w[(size_t)o * 2 * D2], &w1[(size_t)o * D2], (size_t)D2 * sizeof(float));
                memcpy(&w[(size_t)o * 2 * D2 + D2], &w2[(size_t)o * D2], (size_t)D2 * sizeof(float));
            }
            rvq_proj.build(w, cbd, 1, 2 * D2, use_f16);
        }
        load_conv(pre_conv, tt, "pre_conv.conv", L, 3, cbd);
        st_pre.H = 2; st_pre.C = cbd;
        load_linear(in_proj, tt, "pre_transformer.input_proj", Hd, L, true);
        load_linear(out_proj, tt, "pre_transformer.output_proj", L, Hd, true);
        up(final_norm, tt.f32("pre_transformer.norm.weight", Hd));
        {
            std::vector<float> f(hd / 2);
            for (int i = 0; i < hd / 2; ++i) f[i] = 1.0f / powf(c.rope_theta, (float)(2 * i) / (float)hd);    // :330-332
            up(inv_freq, f);
        }
        layers.resize(c.num_hidden_layers);
        for (int l = 0; l < c.num_hidden_layers; ++l) {
            const std::string p = "pre_transformer.layers." + std::to_string(l) + ".";
            TLayer& T = layers[l];
            const bool ab = c.attention_bias != 0;
            {
                std::vector<float> w((size_t)Mqkv * Hd), q = tt.f32(p + "self_attn.q_proj.weight", (int64_t)nh * hd * Hd),
                                   k = tt.f32(p + "self_attn.k_proj.weight", (int64_t)nkv * hd * Hd), v = tt.f32(p + "self_attn.v_proj.weight", (int64_t)nkv * hd * Hd);
                memcpy(w.data(), q.data(), q.size() * sizeof(float));
                memcpy(w.data() + q.size(), k.data(), k.size() * sizeof(float));
                memcpy(w.data() + q.size() + k.size(), v.data(), v.size() * sizeof(float));
                T.qkv.build(w, Mqkv, 1, Hd, use_f16);
                if (ab) {
                    std::vector<float> bq = tt.f32(p + "self_attn.q_proj.bias", nh * hd), bk = tt.f32(p + "self_attn.k_proj.bias", nkv * hd),
                                       bv = tt.f32(p + "self_attn.v_proj.bias", nkv * hd);
                    bq.insert(bq.end(), bk.begin(), bk.end());
                    bq.insert(bq.end(), bv.begin(), bv.end());
                    T.qkv.set_bias(bq);
                }
            }
            load_linear(T.o, tt, p + "self_attn.o_proj", Hd, nh * hd, ab);
            {
                std::vector<float> g = tt.f32(p + "mlp.gate_proj.weight", (int64_t)I * Hd), u = tt.f32(p + "mlp.up_proj.weight", (int64_t)I * Hd);
                g.insert(g.end(), u.begin(), u.end());
                T.gu.build(g, 2 * I, 1, Hd, use_f16);
            }
            load_linear(T.down, tt, p + "mlp.down_proj", Hd, I, false);
            up(T.ln1, tt.f32(p + "input_layernorm.weight", Hd));
            up(T.ln2, tt.f32(p + "post_attention_layernorm.weight", Hd));
            up(T.sc_attn, tt.f32(p + "self_attn_layer_scale.scale", Hd));
            up(T.sc_mlp, tt.f32(p + "mlp_layer_scale.scale", Hd));
        }
        total_up = 1;
        ups.resize(c.num_upsampling_ratios);
        for (int i = 0; i < c.num_upsampling_ratios; ++i) {
            const std::string p = "upsample." + std::to_string(i) + ".layers.";
            UpLayer& U = ups[i];
            U.factor = c.upsampling_ratios[i];
            B2A_CHECK(U.factor >= 1 && U.factor <= 16, B2A_ERR_INVALID_INPUT, "speech tokenizer: bad upsampling ratio");
            total_up *= U.factor;
            U.ct.build(convt_weight(conv_w(tt, p + "0.conv.weight", L, U.factor, L), L, U.factor, L, U.factor), U.factor * L, 1, L, use_f16);
            U.ct.set_bias(tt.f32(p + "0.conv.bias", L));
            up(U.dw_w, tt.f32(p + "1.dwconv.conv.weight", (int64_t)L * 7));
            up(U.dw_b, tt.f32(p + "1.dwconv.conv.bias", L));
            up(U.ln_w, tt.f32(p + "1.norm.weight", L));
            up(U.ln_b, tt.f32(p + "1.norm.bias", L));
            load_linear(U.pw1, tt, p + "1.pwconv1", 4 * L, L, true);
            load_linear(U.pw2, tt, p + "1.pwconv2", L, 4 * L, true);
            up(U.gamma, tt.f32(p + "1.gamma", L));
            U.st.H = 6; U.st.C = L;
        }
        const int dd = c.decoder_dim, nb = c.num_upsample_rates;
        load_conv(dec0, tt, "decoder.0.conv", dd, 7, L);
        st_dec0.H = 6; st_dec0.C = L;
        blocks.resize(nb);
        for (int b = 0; b < nb; ++b) {
            const std::string p = "decoder." + std::to_string(1 + b) + ".block.";
            DecBlock& Bk = blocks[b];
            Bk.rate = c.upsample_rates[b];
            B2A_CHECK(Bk.rate >= 1 && Bk.rate <= 16, B2A_ERR_INVALID_INPUT, "speech tokenizer: bad upsample rate");
            total_up *= Bk.rate;
            Bk.cin = dd >> b; Bk.cout = dd >> (b + 1);
            B2A_CHECK(Bk.cin % 8 == 0 && Bk.cout % 8 == 0, B2A_ERR_INVALID_INPUT, "speech tokenizer: decoder channels must be multiples of 8");
            load_snake(Bk.sn, tt, p + "0", Bk.cin);
            Bk.ct.build(convt_weight(conv_w(tt, p + "1.conv.weight", Bk.cout, 2 * Bk.rate, Bk.cin), Bk.cout, 2 * Bk.rate, Bk.cin, Bk.rate), Bk.rate * Bk.cout, 2, Bk.cin, use_f16);
            Bk.ct.set_bias(tt.f32(p + "1.conv.bias", Bk.cout));
            Bk.st.H = 1; Bk.st.C = Bk.cin;
            const int dil[3] = {1, 3, 9};
            for (int j = 0; j < 3; ++j) {
                const std::string q = p + std::to_string(2 + j) + ".";
                ResUnit& R = Bk.ru[j];
                R.dil = dil[j];
                load_snake(R.a1, tt, q + "act1", Bk.cout);
                load_snake(R.a2, tt, q + "act2", Bk.cout);
                load_conv(R.c1, tt, q + "conv1.conv", Bk.cout, 7, Bk.cout);
                load_conv(R.c2, tt, q + "conv2.conv", Bk.cout, 1, Bk.cout);
                R.st.H = 6 * R.dil; R.st.C = Bk.cout;
            }
        }
        const int Cf = dd >> nb;
        load_snake(out_snake, tt, "decoder." + std::to_string(nb + 1), Cf);
        {
            const b2a_tensor& t = tt.get("decoder." + std::to_string(nb + 2) + ".conv.weight");
            B2A_CHECK(t.ndim == 3 && t.shape[0] == 1 && t.shape[2] == Cf && t.shape[1] >= 1 && t.shape[1] <= FC_MAXK, B2A_ERR_MODEL_NOT_INITIALIZED,
                      "bad shape for tensor: decoder output conv weight");
            out_k = (int)t.shape[1];
            up(out_w, tt.f32("decoder." + std::to_string(nb + 2) + ".conv.weight", (int64_t)out_k * Cf));
            out_b = tt.f32("decoder." + std::to_string(nb + 2) + ".conv.bias", 1)[0];
            st_out.H = out_k - 1; st_out.C = Cf;
        }
        B2A_CUDA(cudaDeviceSynchronize());
        alloc_state();
        reset();
    }

    // ------------------------------------------------------------------------------------------- state
    void alloc_state() {
        const int B = cfg.max_batch;
        auto ps = [&](PlaneState& s) { for (int i = 0; i < 2; ++i) s.s[i].alloc((size_t)2 * B * std::max(s.H, 1) * s.C); };
        auto fs = [&](F32State& s) { for (int i = 0; i < 2; ++i) s.s[i].alloc((size_t)B * std::max(s.H, 1) * s.C); };
        ps(st_pre); ps(st_dec0); fs(st_out);
        for (auto& U : ups) fs(U.st);
        for (auto& Bk : blocks) { ps(Bk.st); for (auto& R : Bk.ru) ps(R.st); }
        const size_t kv = (size_t)B * cfg.num_key_value_heads * cfg.max_cache_frames * cfg.head_dim;
        for (auto& T : layers) { T.K.alloc(kv); T.V.alloc(kv); }
    }

    void reset() {                // resetStreamingState (:949-970): zero history == the reference's causal zero padding
        B2A_CUDA(cudaSetDevice(device));
        auto zp = [&](PlaneState& s) { for (int i = 0; i < 2; ++i) B2A_CUDA(cudaMemsetAsync(s.s[i].p, 0, s.s[i].n * sizeof(bf16), stream)); };
        auto zf = [&](F32State& s) { for (int i = 0; i < 2; ++i) B2A_CUDA(cudaMemsetAsync(s.s[i].p, 0, s.s[i].n * sizeof(float), stream)); };
        zp(st_pre); zp(st_dec0); zf(st_out);
        for (auto& U : ups) zf(U.st);
        for (auto& Bk : blocks) { zp(Bk.st); for (auto& R : Bk.ru) zp(R.st); }
        B2A_CUDA(cudaStreamSynchronize(stream));     // a following step may run on a caller's stream
        parity = 0; chunk_idx = 0; cache_len = 0; stream_B = 0;
    }

    // ------------------------------------------------------------------------------------------- launches
    bf16* planes(DBuf<bf16>& buf, int B, long long frames, int C) {
        const size_t need = (size_t)2 * B * frames * C;
        B2A_CHECK(need <= buf.n, B2A_ERR_GENERATION_FAILED, "speech tokenizer: internal workspace too small");
        return buf.p;
    }
    void conv(const TcW& W, const bf16* in, long long in_frames, ic::Args a, cudaStream_t s) { ic::launch(W, in, in_frames, a, num_sms, s); }
    void carry(bf16* X, PlaneState& st, int B, long long T, cudaStream_t s) {
        if (st.H == 0) return;
        const long long n = (long long)2 * B * st.H * (st.C / 8);
        carry_planes_kernel<<<(unsigned)cdiv(n, 256), 256, 0, s>>>(X, st.s[parity].p, st.s[parity ^ 1].p, B, (int)T, st.H, st.C / 8);
        count_launch();
    }
    void update_f32(const float* x, F32State& st, int B, long long T, cudaStream_t s) {
        if (st.H == 0) return;
        const long long n = (long long)B * st.H * st.C;
        state_update_f32_kernel<<<(unsigned)cdiv(n, 256), 256, 0, s>>>(x, st.s[parity].p, st.s[parity ^ 1].p, B, (int)T, st.H, st.C);
        count_launch();
    }
    void attention(TLayer& L, int B, int T, bf16* out, cudaStream_t s) {
        const dim3 grid(cdiv(T, AT_WARPS), cfg.num_attention_heads, B), block(AT_WARPS * 32);
        const float scale = 1.0f / sqrtf((float)cfg.head_dim);
        const int nh = cfg.num_attention_heads, nkv = cfg.num_key_value_heads, cap = cfg.max_cache_frames;
        if (cfg.head_dim == 32) attn_kernel<1><<<grid, block, 0, s>>>(Q.p, L.K.p, L.V.p, out, B, T, cache_len, nh, nkv, cap, scale, use_f16, 0);
        else if (cfg.head_dim == 64) attn_kernel<2><<<grid, block, 0, s>>>(Q.p, L.K.p, L.V.p, out, B, T, cache_len, nh, nkv, cap, scale, use_f16, 0);
        else attn_kernel<4><<<grid, block, 0, s>>>(Q.p, L.K.p, L.V.p, out, B, T, cache_len, nh, nkv, cap, scale, use_f16, 0);
        count_launch();
    }

    long long out_len(int T) const { return (long long)T * total_up; }

    // streamingStep (:973-1008): d_codes [B, nq, T] int32 (device) -> d_wave [B, T * total_up]
    void step_dev(const int* dcodes, int B, int nq, int T, float* d_wave, cudaStream_t s) {
        const auto& c = cfg;
        B2A_CHECK(B >= 1 && B <= c.max_batch, B2A_ERR_INVALID_INPUT, "speech tokenizer: batch must be in [1, max_batch]");
        B2A_CHECK(T >= 1 && nq >= 1 && nq <= c.num_quantizers, B2A_ERR_INVALID_INPUT, "speech tokenizer: need >= 1 frame and 1..num_quantizers code groups");
        B2A_CHECK(chunk_idx == 0 || B == stream_B, B2A_ERR_INVALID_INPUT, "speech tokenizer: batch size changed inside a stream (reset first)");
        B2A_CHECK(cache_len + T <= c.max_cache_frames, B2A_ERR_INVALID_INPUT, "speech tokenizer: stream longer than max_cache_frames");
        B2A_CHECK((long long)T * total_up + 64 < (1ll << 31) && (long long)B * T * total_up / 64 < (1ll << 31), B2A_ERR_INVALID_INPUT,
                  "speech tokenizer: chunk too large");      // per-row frame indices and grid sizes are 32-bit
        B2A_CUDA(cudaSetDevice(device));
        stream_B = B;
        const int cbd = c.codebook_dim, L = c.latent_dim, Hd = c.hidden_size, I = c.intermediate_size, nh = c.num_attention_heads, hd = c.head_dim;
        const long long N = (long long)B * T;
        // workspace: the largest planar activation and fp32 tensors of the chunk
        {
            size_t pmax = 0, xc = 0;
            auto pl = [&](long long frames, int C) { pmax = std::max(pmax, (size_t)(2ll * B * frames * C)); };
            pl(T + 2, cbd); pl(T, L); pl(T, std::max(std::max(Hd, I), nh * hd));
            long long Tc = T;
            for (auto& U : ups) { Tc *= U.factor; pl(Tc + 6, L); pl(Tc, 4 * L); xc = std::max(xc, (size_t)((long long)B * Tc * L)); }
            pl(Tc + 1, c.decoder_dim);
            for (auto& Bk : blocks) { Tc *= Bk.rate; pl(Tc + 54, Bk.cout); xc = std::max(xc, (size_t)((long long)B * Tc * Bk.cout)); }
            P0.alloc(pmax); P1.alloc(pmax);
            Xh.alloc((size_t)N * Hd); Xc.alloc(xc);
            Q.alloc((size_t)N * std::max(Mqkv, 2 * I));
        }
        // 1. codebook gathers + both output projections                                    (:112-119)
        rvq_gather_kernel<<<(unsigned)N, 128, 0, s>>>(dcodes, emb.p, planes(P0, B, T, 2 * D2), B, T, nq, c.num_quantizers, c.num_semantic_quantizers,
                                                     c.codebook_size, D2, use_f16);
        count_launch();
        { ic::Args a{}; a.B = B; a.T = T; a.hl = planes(P1, B, T + 2, cbd); a.Hout = 2; conv(rvq_proj, P0.p, T, a, s); }
        // 2. pre_conv (k3 causal) -> input_proj                                             (:929-931, :454)
        carry(P1.p, st_pre, B, T, s);
        { ic::Args a{}; a.B = B; a.T = T; a.hl = planes(P0, B, T, L); conv(pre_conv, P1.p, T + 2, a, s); }
        { ic::Args a{}; a.B = B; a.T = T; a.xo = Xh.p; conv(in_proj, P0.p, T, a, s); }
        // 3. transformer layers over the KV cache                                           (:419-428, :473-476)
        for (auto& Ly : layers) {
            rmsnorm_planes_kernel<<<(unsigned)N, RN_THREADS, 0, s>>>(Xh.p, Ly.ln1.p, planes(P0, B, T, Hd), N, Hd, c.rms_norm_eps, use_f16);
            count_launch();
            { ic::Args a{}; a.B = B; a.T = T; a.xo = Q.p; conv(Ly.qkv, P0.p, T, a, s); }
            rope_cache_kernel<false><<<(unsigned)N, 256, 0, s>>>(Q.p, Ly.K.p, Ly.V.p, inv_freq.p, T, cache_len, nh, c.num_key_value_heads, hd, c.max_cache_frames);
            count_launch();
            attention(Ly, B, T, planes(P1, B, T, nh * hd), s);
            { ic::Args a{}; a.B = B; a.T = T; a.xo = Xh.p; a.add = 1; a.gamma = Ly.sc_attn.p; conv(Ly.o, P1.p, T, a, s); }
            rmsnorm_planes_kernel<<<(unsigned)N, RN_THREADS, 0, s>>>(Xh.p, Ly.ln2.p, planes(P0, B, T, Hd), N, Hd, c.rms_norm_eps, use_f16);
            count_launch();
            { ic::Args a{}; a.B = B; a.T = T; a.xo = Q.p; conv(Ly.gu, P0.p, T, a, s); }
            swiglu_planes_kernel<<<(unsigned)cdiv(N * I, 256), 256, 0, s>>>(Q.p, planes(P1, B, T, I), N, I, use_f16);
            count_launch();
            { ic::Args a{}; a.B = B; a.T = T; a.xo = Xh.p; a.add = 1; a.gamma = Ly.sc_mlp.p; conv(Ly.down, P1.p, T, a, s); }
        }
        dbg_tap(0, Xh.p, N * Hd, s);
        rmsnorm_planes_kernel<<<(unsigned)N, RN_THREADS, 0, s>>>(Xh.p, final_norm.p, planes(P0, B, T, Hd), N, Hd, c.rms_norm_eps, use_f16);
        count_launch();
        { ic::Args a{}; a.B = B; a.T = T; a.hl = planes(P1, B, T, L); conv(out_proj, P0.p, T, a, s); }
        // 4. upsample layers: transposed conv (k = stride) + ConvNeXt                       (:758-775)
        bf16* cur = P1.p;          // planes [2][B][Hcur + Tc][L]
        bf16* other = P0.p;
        long long Tc = T;
        int Hcur = 0;
        for (size_t i = 0; i < ups.size(); ++i) {
            UpLayer& U = ups[i];
            { ic::Args a{}; a.B = B; a.T = (int)Tc; a.up = U.factor; a.xo = Xc.p; conv(U.ct, cur, Hcur + Tc, a, s); }
            Tc *= U.factor;
            dw_ln_kernel<<<(unsigned)(B * Tc), DL_THREADS, 0, s>>>(Xc.p, U.st.s[parity].p, U.dw_w.p, U.dw_b.p, U.ln_w.p, U.ln_b.p, cur, B, (int)Tc, L, 7, 1e-6f, use_f16);
            count_launch();
            update_f32(Xc.p, U.st, B, Tc, s);
            { ic::Args a{}; a.B = B; a.T = (int)Tc; a.gelu = 1; a.hl = other; conv(U.pw1, cur, Tc, a, s); }
            Hcur = i + 1 < ups.size() ? 0 : st_dec0.H;
            { ic::Args a{}; a.B = B; a.T = (int)Tc; a.xo = Xc.p; a.add = 1; a.gamma = U.gamma.p; a.hl = cur; a.Hout = Hcur; conv(U.pw2, other, Tc, a, s); }
            dbg_tap(1 + (int)i, Xc.p, (long long)B * Tc * L, s);
        }
        // 5. decoder.0 (k7 causal) with block 0's SnakeBeta fused                            (:641-656)
        carry(cur, st_dec0, B, Tc, s);
        { ic::Args a{}; a.B = B; a.T = (int)Tc; a.hl = other; a.Hout = 1; a.sa = blocks[0].sn.a.p; a.sb = blocks[0].sn.ib.p; conv(dec0, cur, Hcur + Tc, a, s); }
        std::swap(cur, other);     // cur = planes [2][B][1 + Tc][decoder_dim], already activated
        // 6. decoder blocks                                                                   (:584-601)
        for (size_t b = 0; b < blocks.size(); ++b) {
            DecBlock& Bk = blocks[b];
            carry(cur, Bk.st, B, Tc, s);
            {
                ic::Args a{}; a.B = B; a.T = (int)Tc; a.up = Bk.rate; a.xo = Xc.p; a.hl = other; a.Hout = Bk.ru[0].st.H;
                a.sa = Bk.ru[0].a1.a.p; a.sb = Bk.ru[0].a1.ib.p; a.bias_twice_t0 = chunk_idx > 0 ? 1 : 0;
                conv(Bk.ct, cur, 1 + Tc, a, s);
            }
            Tc *= Bk.rate;
            dbg_tap(10 + 4 * (int)b, Xc.p, (long long)B * Tc * Bk.cout, s);
            std::swap(cur, other);
            for (int j = 0; j < 3; ++j) {
                ResUnit& R = Bk.ru[j];
                carry(cur, R.st, B, Tc, s);
                { ic::Args a{}; a.B = B; a.T = (int)Tc; a.dil = R.dil; a.hl = other; a.sa = R.a2.a.p; a.sb = R.a2.ib.p; conv(R.c1, cur, R.st.H + Tc, a, s); }
                ic::Args a{}; a.B = B; a.T = (int)Tc; a.xo = Xc.p; a.add = 1;
                if (j < 2) { a.hl = cur; a.Hout = Bk.ru[j + 1].st.H; a.sa = Bk.ru[j + 1].a1.a.p; a.sb = Bk.ru[j + 1].a1.ib.p; }
                else if (b + 1 < blocks.size()) { a.hl = cur; a.Hout = 1; a.sa = blocks[b + 1].sn.a.p; a.sb = blocks[b + 1].sn.ib.p; }
                conv(R.c2, other, Tc, a, s);
                dbg_tap(11 + 4 * (int)b + j, Xc.p, (long long)B * Tc * Bk.cout, s);
            }
        }
        // 7. output SnakeBeta + k7 conv to one channel + clip                                 (:693-731, :946)
        {
            const int Cf = st_out.C;
            const size_t smem = ((size_t)(FC_TILE + out_k - 1) * (Cf + 1) + (size_t)out_k * Cf + FC_THREADS) * sizeof(float);
            final_conv_kernel<<<dim3(cdiv(Tc, FC_TILE), B), FC_THREADS, smem, s>>>(Xc.p, st_out.s[parity].p, out_snake.a.p, out_snake.ib.p, out_w.p, out_b,
                                                                                  d_wave, (int)Tc, Cf, out_k);
            count_launch();
            update_f32(Xc.p, st_out, B, Tc, s);
        }
        B2A_CUDA(cudaGetLastError());
        parity ^= 1;
        chunk_idx += 1;
        cache_len += T;
    }

    // host codes [B, nq, T] -> host wave [B, T * total_up]
    void step_host(const int32_t* codes, int B, int nq, int T, float* out, long long out_stride, long long drop) {
        cudaStream_t s = stream;
        const size_t nin = (size_t)B * nq * T;
        const long long nout = out_len(T);
        d_codes.alloc(nin); wave.alloc((size_t)B * nout);
        B2A_CUDA(cudaMemcpyAsync(d_codes.p, codes, nin * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        step_dev(d_codes.p, B, nq, T, wave.p, s);
        B2A_CUDA(cudaMemcpy2DAsync(out, (size_t)out_stride * sizeof(float), wave.p + drop, (size_t)nout * sizeof(float), (size_t)(nout - drop) * sizeof(float),
                                   (size_t)B, cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    }
};

// ================================================================================================ encoder
// Qwen3TTSSpeechTokenizerEncoder.encode (Qwen3TTSSpeechTokenizer.swift:790-884): audio [B, 1, n] -> codes [B, G, T].
//   1. SEANet encoder (Mimi/Seanet.swift:157-257) in fp32 channels-last on the shared SEANet kernels (seanet.cuh): the stem from the
//      waveform, per reversed ratio a resnet block (identity skip) and ELU + conv k = 2r stride r, then ELU + the last conv.  Causal
//      zero padding kEff - stride on the left plus getExtraPaddingForConv1d on the right (Mimi/Conv.swift:150-156, 205-221).
//   2. The transformer (Mimi/Transformer.swift:110-369) on the decoder's machinery: LayerNorm into hi/lo planes, implicit-GEMM
//      linears with the layer scale + residual (and exact GELU) fused, interleaved RoPE, causal attention over the whole clip (the
//      encode trims its caches to empty and passes the clip at once, so the 250-frame context never drops a key).
//   3. ConvDownsample1d (Conv.swift:333-347): k = 2 s, stride s, no bias, EDGE padding -> z [B, T, hidden].
//   4. SplitResidualVectorQuantizer.encode (Mimi/Quantization.swift:7-211): both k1 input projections as one ordered-fp32 product
//      z -> [first | rest], then the code search (dist = |e|^2/2 - x.e, ordered fp32) -- rvq_first's one level, rvq_rest's first
//      G - 1 levels, the only ones the cut to valid_num_quantizers keeps.
struct b2a_speech_tokenizer_encoder {
    int device = 0, num_sms = 132;
    b2a_speech_tokenizer_encoder_config cfg{};
    cudaStream_t stream = nullptr;
    int G = 0, ds = 1;                 // code groups returned, downsample stride
    struct Stage { int ratio, cin; ec::Conv r1, r2, down; };
    DBuf<float> wstem, bstem;          // [F, k, 1]
    std::vector<Stage> stages;
    ec::Conv last, down;
    struct Layer { TcW qkv, o, fc1, fc2; DBuf<float> ln1w, ln1b, ln2w, ln2b, ls1, ls2; };
    std::vector<Layer> layers;
    DBuf<float> inv_freq, proj_t, books, c2;     // proj_t [hidden, 2 D] (first | rest, transposed); books [G][size][D]; c2 [G][size]
    // workspaces
    DBuf<float> bufA, bufB, bufC, Q, Kc, Vc, zbuf, xproj, audio;
    DBuf<bf16> P0, P1;
    DBuf<int> codes;

    static void up(DBuf<float>& d, const std::vector<float>& v) { d.upload(v.data(), v.size()); }
    static void load(const TensorTable& tt, ec::Conv& cv, const std::string& p, int cout, int k, int cin, bool bias) {
        cv.M = cout; cv.K = k * cin;
        up(cv.A, tt.f32(p + ".weight", (int64_t)cout * k * cin));       // MLX [out, k, in] == [M, tap * Cin + ci]
        if (bias) up(cv.bias, tt.f32(p + ".bias", cout));
    }
    void load_linear(TcW& w, const TensorTable& tt, const std::string& p, int out, int in) {
        w.build(tt.f32(p + ".weight", (int64_t)out * in), out, 1, in, 1);
    }

    b2a_speech_tokenizer_encoder(int dev, const b2a_speech_tokenizer_encoder_config& c, const TensorTable& tt) : device(dev), cfg(c) {
        B2A_CHECK(c.audio_channels == 1, B2A_ERR_INVALID_INPUT, "speech tokenizer encoder: audio_channels must be 1");
        B2A_CHECK(c.num_residual_layers == 1, B2A_ERR_INVALID_INPUT,
                  "speech tokenizer encoder: num_residual_layers must be 1 (dilated residual layers are not implemented)");
        B2A_CHECK(c.use_causal_conv && !c.use_conv_shortcut, B2A_ERR_INVALID_INPUT,
                  "speech tokenizer encoder: only the causal, identity-skip SEANet (use_causal_conv, !use_conv_shortcut) is implemented");
        B2A_CHECK(c.num_upsampling_ratios >= 1 && c.num_upsampling_ratios <= 8 && c.kernel_size >= 1 && c.kernel_size <= 16 &&
                      c.residual_kernel_size >= 1 && c.last_kernel_size >= 1 && c.compress >= 1 && c.num_filters >= 4 && c.num_filters % 4 == 0,
                  B2A_ERR_INVALID_INPUT, "speech tokenizer encoder: bad SEANet config");
        B2A_CHECK(c.head_dim == 32 || c.head_dim == 64 || c.head_dim == 128, B2A_ERR_INVALID_INPUT, "speech tokenizer encoder: head_dim must be 32, 64 or 128");
        B2A_CHECK(c.num_attention_heads >= 1 && c.num_key_value_heads == c.num_attention_heads && c.num_attention_heads * c.head_dim == c.hidden_size,
                  B2A_ERR_INVALID_INPUT, "speech tokenizer encoder: heads * head_dim must equal hidden_size, without grouped keys (Transformer.swift:121)");
        B2A_CHECK(c.hidden_size % 64 == 0 && c.intermediate_size % 8 == 0 && c.num_hidden_layers >= 0, B2A_ERR_INVALID_INPUT,
                  "speech tokenizer encoder: hidden_size must be a multiple of 64, intermediate_size of 8");
        B2A_CHECK(c.codebook_size >= 1 && c.codebook_dim >= 1 && ec::rvq_encode_smem(c.codebook_dim) <= 220 * 1024, B2A_ERR_INVALID_INPUT,
                  "speech tokenizer encoder: bad codebook geometry");
        B2A_CHECK(c.num_quantizers >= 1 && c.valid_num_quantizers >= 1, B2A_ERR_INVALID_INPUT, "speech tokenizer encoder: bad quantizer counts");
        B2A_CHECK(tt.find("encoder.init_conv1d.conv.conv.weight"), B2A_ERR_MODEL_NOT_INITIALIZED,
                  "speech tokenizer encoder: the checkpoint has no encoder weights");
        B2A_CHECK((size_t)PJ_R * c.hidden_size * sizeof(float) <= 200 * 1024, B2A_ERR_INVALID_INPUT,
                  "speech tokenizer encoder: hidden_size too large for the input projection's shared-memory tile");
        require_device(dev);
        B2A_CUDA(cudaSetDevice(dev));
        B2A_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
        B2A_CUDA(cudaFuncSetAttribute(ordered_proj_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(PJ_R * c.hidden_size * sizeof(float))));
        G = std::min(c.valid_num_quantizers, c.num_quantizers);
        {   // Qwen3TTSSpeechTokenizerEncoder.init (:810-812): stride = max(1, Int(sampling_rate / prod(ratios) / frame_rate))
            long long hop = 1;
            for (int i = 0; i < c.num_upsampling_ratios; ++i) {
                B2A_CHECK(c.upsampling_ratios[i] >= 1 && c.upsampling_ratios[i] <= 64, B2A_ERR_INVALID_INPUT, "speech tokenizer encoder: bad ratio");
                hop *= c.upsampling_ratios[i];
            }
            ds = std::max(1, (int)((double)c.sampling_rate / (double)hop / (double)c.frame_rate));
        }
        const int F = c.num_filters, H = c.hidden_size, D = c.codebook_dim;
        up(wstem, tt.f32("encoder.init_conv1d.conv.conv.weight", (int64_t)F * c.kernel_size));
        up(bstem, tt.f32("encoder.init_conv1d.conv.conv.bias", F));
        int ch = F;
        for (int i = 0; i < c.num_upsampling_ratios; ++i) {
            Stage st{};
            st.ratio = c.upsampling_ratios[c.num_upsampling_ratios - 1 - i];
            st.cin = ch;
            const int hid = ch / c.compress;
            B2A_CHECK(hid >= 4 && hid % 4 == 0, B2A_ERR_INVALID_INPUT, "speech tokenizer encoder: channel counts must be multiples of 4");
            const std::string p = "encoder.layers." + std::to_string(i) + ".";
            load(tt, st.r1, p + "residuals.0.block.0.conv.conv", hid, c.residual_kernel_size, ch, true);
            load(tt, st.r2, p + "residuals.0.block.1.conv.conv", ch, 1, hid, true);
            load(tt, st.down, p + "downsample.conv.conv", 2 * ch, 2 * st.ratio, ch, true);
            stages.push_back(std::move(st));
            ch *= 2;
        }
        load(tt, last, "encoder.final_conv1d.conv.conv", H, c.last_kernel_size, ch, true);
        layers.resize(c.num_hidden_layers);
        for (int l = 0; l < c.num_hidden_layers; ++l) {
            const std::string p = "encoder_transformer.transformer.layers." + std::to_string(l) + ".";
            Layer& L = layers[l];
            load_linear(L.qkv, tt, p + "self_attn.in_proj", 3 * H, H);
            load_linear(L.o, tt, p + "self_attn.out_proj", H, H);
            load_linear(L.fc1, tt, p + "gating.linear1", c.intermediate_size, H);
            load_linear(L.fc2, tt, p + "gating.linear2", H, c.intermediate_size);
            up(L.ln1w, tt.f32(p + "norm1.weight", H)); up(L.ln1b, tt.f32(p + "norm1.bias", H));
            up(L.ln2w, tt.f32(p + "norm2.weight", H)); up(L.ln2b, tt.f32(p + "norm2.bias", H));
            up(L.ls1, tt.f32(p + "layer_scale_1.scale", H)); up(L.ls2, tt.f32(p + "layer_scale_2.scale", H));
        }
        {   // RoPE(dimensions: head_dim, traditional: true, base: Float(maxPeriod)), maxPeriod = Int(ropeTheta) (:844)
            const float base = (float)(int)c.rope_theta;
            std::vector<float> f(c.head_dim / 2);
            for (int i = 0; i < c.head_dim / 2; ++i) f[i] = 1.0f / powf(base, (float)(2 * i) / (float)c.head_dim);
            up(inv_freq, f);
        }
        load(tt, down, "downsample.conv.conv.conv", H, 2 * ds, H, false);
        {   // input projections [D, 1, H] each -> proj_t [H][2 D]; codebooks: embedding = embedding_sum / max(cluster_usage, 1e-5)
            std::vector<float> w1 = tt.f32("quantizer.rvq_first.input_proj.weight", (int64_t)D * H), w2((size_t)D * H, 0.f);
            if (G > 1) w2 = tt.f32("quantizer.rvq_rest.input_proj.weight", (int64_t)D * H);
            std::vector<float> pt((size_t)H * 2 * D);
            for (int o = 0; o < D; ++o)
                for (int h = 0; h < H; ++h) { pt[(size_t)h * 2 * D + o] = w1[(size_t)o * H + h]; pt[(size_t)h * 2 * D + D + o] = w2[(size_t)o * H + h]; }
            up(proj_t, pt);
            const int bins = c.codebook_size;
            std::vector<float> e((size_t)G * bins * D);
            for (int q = 0; q < G; ++q) {
                const std::string p = q == 0 ? std::string("quantizer.rvq_first.vq.layers.0") : "quantizer.rvq_rest.vq.layers." + std::to_string(q - 1);
                const std::vector<float> sum = tt.f32(p + ".codebook.embedding_sum", (int64_t)bins * D), use = tt.f32(p + ".codebook.cluster_usage", bins);
                for (int r = 0; r < bins; ++r) {
                    const float u = std::max(use[r], 1e-5f);
                    for (int d = 0; d < D; ++d) e[((size_t)q * bins + r) * D + d] = sum[(size_t)r * D + d] / u;
                }
            }
            up(books, e);
            c2.alloc((size_t)G * bins);
            ec::sqnorm_rows_kernel<<<cdiv((long long)G * bins, 256), 256>>>(books.p, c2.p, (long long)G * bins, D, 0.5f);
            B2A_CUDA(cudaGetLastError());
        }
        B2A_CUDA(cudaDeviceSynchronize());
        // last: a check that throws above leaves no stream behind (the destructor does not run for a half-built object)
        B2A_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    }
    ~b2a_speech_tokenizer_encoder() { if (stream) cudaStreamDestroy(stream); }

    // StreamableConv1d's output length (Mimi/Conv.swift:150-156, 205-221): (L + kEff - stride + extra - kEff) / stride + 1
    static long long conv_len(long long L, int k, int stride) {
        const long long pt = k - stride, nframes = std::max(L + pt - k, 0ll);
        const double nf = (double)nframes / (double)stride + 1.0;
        const long long ideal = ((long long)std::ceil(nf) - 1) * stride + k - pt;
        return (L + pt + std::max(0ll, ideal - L) - k) / stride + 1;
    }
    long long seanet_len(long long n) const {
        long long L = n;
        for (auto& st : stages) L = conv_len(L, 2 * st.ratio, st.ratio);
        return L;
    }
    long long encoded_length(long long n) const { return n >= 1 ? conv_len(seanet_len(n), 2 * ds, ds) : 0; }

    // d_audio [B, n] -> d_codes [B, G, T]; z stays in zbuf [B, T, hidden]
    void encode_dev(const float* d_audio, int B, long long n, int* d_codes, cudaStream_t s) {
        B2A_CHECK(n >= 1, B2A_ERR_AUDIO_ENCODING_FAILED, "speech tokenizer encoder: empty audio");
        B2A_CHECK(B >= 1, B2A_ERR_INVALID_INPUT, "speech tokenizer encoder: batch must be >= 1");
        const int F = cfg.num_filters, H = cfg.hidden_size, D = cfg.codebook_dim, I = cfg.intermediate_size, nh = cfg.num_attention_heads, hd = cfg.head_dim;
        // 32-bit frame indices and grid sizes, 64-bit element offsets below 2^40
        B2A_CHECK(n < (1ll << 30) && (long long)B * n * std::max(F, 64) < (1ll << 40) && (long long)B * n < (1ll << 31), B2A_ERR_INVALID_INPUT,
                  "speech tokenizer encoder: input too long");
        B2A_CUDA(cudaSetDevice(device));
        const long long T25 = seanet_len(n), T = encoded_length(n), N25 = (long long)B * T25, N = (long long)B * T;
        size_t big = (size_t)B * n * F;
        {
            long long L = n;
            for (auto& st : stages) { L = conv_len(L, 2 * st.ratio, st.ratio); big = std::max(big, (size_t)((long long)B * L * 2 * st.cin)); }
            big = std::max(big, (size_t)(N25 * H));
        }
        bufA.alloc(big); bufB.alloc(big); bufC.alloc(big);
        float* x = bufA.p; float* y = bufB.p; float* z = bufC.p;
        // 1. SEANet
        {
            const int k = cfg.kernel_size;
            const size_t smem = ((size_t)F * k + (size_t)(ec::STEM_T + k - 1)) * sizeof(float);
            B2A_CHECK(smem <= 200 * 1024, B2A_ERR_INVALID_INPUT, "speech tokenizer encoder: stem too wide");
            B2A_CUDA(cudaFuncSetAttribute(ec::stem_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ec::stem_conv_kernel<<<dim3(cdiv(n, ec::STEM_T), B), 256, smem, s>>>(d_audio, wstem.p, bstem.p, nullptr, x, B, n, 1, (int)n, 0, F, k, k - 1, 0);
            count_launch();
        }
        long long L = n;
        for (auto& st : stages) {
            ec::resnet_block(st.r1, st.r2, false, cfg.residual_kernel_size, cfg.residual_kernel_size - 1, 0, x, y, z, B, L, st.cin, s);
            const int r = st.ratio, k = 2 * r;
            const long long Lo = conv_len(L, k, r);
            ec::ConvArgs a{};
            a.xa = x; a.La = (int)L; a.Ca = st.cin; a.taps = k; a.stride = r; a.padL = k - r; a.elu_a = 1;       // right pad: zero rows
            a.A = st.down.A.p; a.bias = st.down.bias.p; a.M = st.down.M; a.K = st.down.K; a.Lq = (int)Lo; a.N = B; a.out = y; a.out_per_n = Lo * st.down.M;
            ec::launch_conv(a, s);
            std::swap(x, y);
            L = Lo;
        }
        {
            ec::ConvArgs a{};
            a.xa = x; a.La = (int)L; a.Ca = last.K / cfg.last_kernel_size; a.taps = cfg.last_kernel_size; a.padL = cfg.last_kernel_size - 1; a.elu_a = 1;
            a.A = last.A.p; a.bias = last.bias.p; a.M = H; a.K = last.K; a.Lq = (int)L; a.N = B; a.out = y; a.out_per_n = L * H;
            ec::launch_conv(a, s);
            std::swap(x, y);
        }
        // 2. transformer on x [B, T25, H] (fp32 residual stream), one-shot: cache capacity = T25, positions from 0
        P0.alloc((size_t)2 * N25 * H); P1.alloc((size_t)2 * N25 * std::max(H, I));
        Q.alloc((size_t)N25 * 3 * H); Kc.alloc((size_t)N25 * H); Vc.alloc((size_t)N25 * H);
        const int cap = (int)T25;
        const float scale = 1.0f / sqrtf((float)hd);
        for (auto& Ly : layers) {
            layernorm_planes_kernel<<<(unsigned)N25, RN_THREADS, 0, s>>>(x, Ly.ln1w.p, Ly.ln1b.p, P0.p, N25, H, 1e-5f, 1);
            count_launch();
            { ic::Args a{}; a.B = B; a.T = cap; a.xo = Q.p; ic::launch(Ly.qkv, P0.p, cap, a, num_sms, s); }
            rope_cache_kernel<true><<<(unsigned)N25, 256, 0, s>>>(Q.p, Kc.p, Vc.p, inv_freq.p, cap, 0, nh, nh, hd, cap);
            count_launch();
            {
                const dim3 grid(cdiv(cap, AT_WARPS), nh, B), block(AT_WARPS * 32);
                if (hd == 32) attn_kernel<1><<<grid, block, 0, s>>>(Q.p, Kc.p, Vc.p, P1.p, B, cap, 0, nh, nh, cap, scale, 1, 0);
                else if (hd == 64) attn_kernel<2><<<grid, block, 0, s>>>(Q.p, Kc.p, Vc.p, P1.p, B, cap, 0, nh, nh, cap, scale, 1, 0);
                else attn_kernel<4><<<grid, block, 0, s>>>(Q.p, Kc.p, Vc.p, P1.p, B, cap, 0, nh, nh, cap, scale, 1, 0);
                count_launch();
            }
            { ic::Args a{}; a.B = B; a.T = cap; a.xo = x; a.add = 1; a.gamma = Ly.ls1.p; ic::launch(Ly.o, P1.p, cap, a, num_sms, s); }
            layernorm_planes_kernel<<<(unsigned)N25, RN_THREADS, 0, s>>>(x, Ly.ln2w.p, Ly.ln2b.p, P0.p, N25, H, 1e-5f, 1);
            count_launch();
            { ic::Args a{}; a.B = B; a.T = cap; a.gelu = 1; a.hl = P1.p; ic::launch(Ly.fc1, P0.p, cap, a, num_sms, s); }
            { ic::Args a{}; a.B = B; a.T = cap; a.xo = x; a.add = 1; a.gamma = Ly.ls2.p; ic::launch(Ly.fc2, P1.p, cap, a, num_sms, s); }
        }
        // 3. downsample: k = 2 ds, stride ds, edge padding on both sides, no bias -> z
        zbuf.alloc((size_t)N * H);
        {
            ec::ConvArgs a{};
            a.xa = x; a.La = cap; a.Ca = H; a.taps = 2 * ds; a.stride = ds; a.padL = ds; a.edge = 1;
            a.A = down.A.p; a.M = H; a.K = down.K; a.Lq = (int)T; a.N = B; a.out = zbuf.p; a.out_per_n = T * H;
            ec::launch_conv(a, s);
        }
        // 4. input projections, then the code search: level 0 on the first block, levels 1 .. G-1 on the rest block
        xproj.alloc((size_t)N * 2 * D);
        ordered_proj_kernel<<<dim3(cdiv(N, PJ_R), cdiv(2 * D, PJ_THREADS)), PJ_THREADS, (size_t)PJ_R * H * sizeof(float), s>>>(zbuf.p, proj_t.p, xproj.p, (int)N, H, 2 * D);
        count_launch();
        {
            const size_t smem = ec::rvq_encode_smem(D);
            B2A_CUDA(cudaFuncSetAttribute(ec::rvq_encode_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            const int bins = cfg.codebook_size;
            ec::rvq_encode_kernel<true><<<cdiv(N, ec::VQ_FT), 256, smem, s>>>(xproj.p, 2 * D, books.p, c2.p, d_codes, (int)N, (int)T, 1, 0, G, bins, D);
            count_launch();
            if (G > 1) {
                ec::rvq_encode_kernel<true><<<cdiv(N, ec::VQ_FT), 256, smem, s>>>(xproj.p + D, 2 * D, books.p + (size_t)bins * D, c2.p + bins, d_codes,
                                                                                 (int)N, (int)T, G - 1, 1, G, bins, D);
                count_launch();
            }
        }
        B2A_CUDA(cudaGetLastError());
    }

    // host audio [B, n] -> host codes [B, G, T] (and z [B, T, hidden] when asked)
    void encode_host(const float* a, int B, long long n, int* out_codes, float* z_out) {
        B2A_CHECK(n >= 1, B2A_ERR_AUDIO_ENCODING_FAILED, "speech tokenizer encoder: empty audio");
        B2A_CHECK(B >= 1 && (long long)B * n < (1ll << 31), B2A_ERR_INVALID_INPUT, "speech tokenizer encoder: bad batch or input too long");
        B2A_CUDA(cudaSetDevice(device));
        cudaStream_t s = stream;
        const long long T = encoded_length(n);
        audio.alloc((size_t)B * n); codes.alloc((size_t)B * G * T);
        B2A_CUDA(cudaMemcpyAsync(audio.p, a, (size_t)B * n * sizeof(float), cudaMemcpyHostToDevice, s));
        encode_dev(audio.p, B, n, codes.p, s);
        if (out_codes) B2A_CUDA(cudaMemcpyAsync(out_codes, codes.p, (size_t)B * G * T * sizeof(int), cudaMemcpyDeviceToHost, s));
        if (z_out) B2A_CUDA(cudaMemcpyAsync(z_out, zbuf.p, (size_t)B * T * cfg.hidden_size * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    }
};

extern "C" {

int32_t b2a_speech_tokenizer_create(int32_t device, const b2a_speech_tokenizer_config* cfg, const b2a_tensor* tensors, int32_t n,
                                    b2a_speech_tokenizer** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_create: null out");
        *out = nullptr;
        B2A_CHECK(cfg && tensors && n > 0, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_speech_tokenizer_create: missing config or weights");
        TensorTable tt(tensors, n);
        *out = new b2a_speech_tokenizer(device, *cfg, tt);
    });
}

int32_t b2a_speech_tokenizer_total_upsample(const b2a_speech_tokenizer* h) { return h ? h->total_up : 0; }
void* b2a_speech_tokenizer_stream(b2a_speech_tokenizer* h) { return h ? (void*)h->stream : nullptr; }

int32_t b2a_speech_tokenizer_reset(b2a_speech_tokenizer* h) {
    return guarded([&] {
        B2A_CHECK(h, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_reset: null handle");
        h->reset();
    });
}

int32_t b2a_speech_tokenizer_streaming_step_dev(b2a_speech_tokenizer* h, const int32_t* d_codes, int32_t B, int32_t nq, int32_t T, float* d_wave,
                                                void* stream) {
    return guarded([&] {
        B2A_CHECK(h && d_codes && d_wave, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_streaming_step_dev: null argument");
        h->step_dev(d_codes, B, nq, T, d_wave, stream ? (cudaStream_t)stream : h->stream);
    });
}

int32_t b2a_speech_tokenizer_streaming_step(b2a_speech_tokenizer* h, const int32_t* codes, int32_t B, int32_t nq, int32_t T, float* wave) {
    return guarded([&] {
        B2A_CHECK(h && codes && wave, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_streaming_step: null argument");
        B2A_CHECK(B >= 1 && T >= 1 && nq >= 1, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_streaming_step: empty input");
        h->step_host(codes, B, nq, T, wave, h->out_len(T), 0);
    });
}

// streamingDecode (:1070-1092): reset, step over chunk_tokens-sized pieces, reset.  codes [B, nq, T] -> wave [B, T * total_up]
int32_t b2a_speech_tokenizer_streaming_decode(b2a_speech_tokenizer* h, const int32_t* codes, int32_t B, int32_t nq, int32_t T, int32_t chunk_tokens,
                                              float* wave) {
    return guarded([&] {
        B2A_CHECK(h && codes && wave, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_streaming_decode: null argument");
        B2A_CHECK(B >= 1 && T >= 1 && nq >= 1 && chunk_tokens >= 1, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_streaming_decode: empty input");
        h->reset();
        std::vector<int32_t> piece;
        for (int start = 0; start < T; start += chunk_tokens) {
            const int n = std::min(chunk_tokens, T - start);
            piece.resize((size_t)B * nq * n);
            for (int r = 0; r < B * nq; ++r) memcpy(&piece[(size_t)r * n], &codes[(size_t)r * T + start], (size_t)n * sizeof(int32_t));
            h->step_host(piece.data(), B, nq, n, wave + h->out_len(start), h->out_len(T), 0);
        }
        h->reset();
    });
}

// chunkedDecode (:1010-1024): every chunk is decoded from a clean state with up to left_context frames of context, whose
// audio is dropped.  codes [B, nq, T] -> wave [B, T * total_up]
int32_t b2a_speech_tokenizer_chunked_decode(b2a_speech_tokenizer* h, const int32_t* codes, int32_t B, int32_t nq, int32_t T, int32_t chunk_size,
                                            int32_t left_context, float* wave) {
    return guarded([&] {
        B2A_CHECK(h && codes && wave, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_chunked_decode: null argument");
        B2A_CHECK(B >= 1 && T >= 1 && nq >= 1 && chunk_size >= 1 && left_context >= 0, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_chunked_decode: empty input");
        std::vector<int32_t> piece;
        for (int start = 0; start < T; start += chunk_size) {
            const int end = std::min(start + chunk_size, T);
            const int ctx = start - left_context > 0 ? left_context : start;
            const int n = end - (start - ctx);
            piece.resize((size_t)B * nq * n);
            for (int r = 0; r < B * nq; ++r) memcpy(&piece[(size_t)r * n], &codes[(size_t)r * T + start - ctx], (size_t)n * sizeof(int32_t));
            h->reset();
            h->step_host(piece.data(), B, nq, n, wave + h->out_len(start), h->out_len(T), h->out_len(ctx));
        }
        h->reset();
    });
}

void b2a_speech_tokenizer_destroy(b2a_speech_tokenizer* h) { delete h; }

// Diagnostics: stage >= 0 makes later decodes keep a copy of the fp32 activation tensor after that stage (0 = transformer output
// before the final norm, 1 + i = upsample layer i, 10 + 4 b = decoder block b after its transposed conv, 11 + 4 b + j = after residual
// unit j); out != null copies the last kept tensor to the host (capacity in floats) and returns its length in *n.
int32_t b2a_speech_tokenizer_debug_stage(b2a_speech_tokenizer* h, int32_t stage, float* out, int64_t capacity, int64_t* n) {
    return guarded([&] {
        B2A_CHECK(h, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_debug_stage: null handle");
        B2A_CUDA(cudaSetDevice(h->device));
        if (out) {
            B2A_CHECK(n && h->dbg_n <= capacity, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_debug_stage: output buffer too small");
            B2A_CUDA(cudaStreamSynchronize(h->stream));
            B2A_CUDA(cudaMemcpy(out, h->dbg.p, (size_t)h->dbg_n * sizeof(float), cudaMemcpyDeviceToHost));
            *n = h->dbg_n;
        }
        h->dbg_stage = stage;
    });
}

// Host-only: the GEMM weight matrix the implicit convolution reads, from an MLX-layout [out, k, in] weight.
// stride == 0: plain causal conv (rows = out, taps = k); stride > 0: transposed conv with k = n * stride (rows = stride * out
// phase-major, taps = n).  layout_out receives [rows][taps][ceil(in / 64) * 64] fp32 (capacity in floats).
int32_t b2a_speech_tokenizer_debug_layout(const float* w, int32_t out, int32_t k, int32_t in, int32_t stride, float* layout_out, int64_t capacity,
                                          int32_t* rows, int32_t* taps, int32_t* kpad) {
    return guarded([&] {
        B2A_CHECK(w && layout_out && rows && taps && kpad && out >= 1 && k >= 1 && in >= 1 && stride >= 0, B2A_ERR_INVALID_INPUT,
                  "b2a_speech_tokenizer_debug_layout: bad argument");
        B2A_CHECK(stride == 0 || k % stride == 0, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_debug_layout: kernel must be a multiple of the stride");
        std::vector<float> src(w, w + (size_t)out * k * in);
        const int M = stride ? stride * out : out, T = stride ? k / stride : k;
        const std::vector<float> g = TcW::pad_k(stride ? convt_weight(src, out, k, in, stride) : src, M, T, in);
        B2A_CHECK((int64_t)g.size() <= capacity, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_debug_layout: output buffer too small");
        memcpy(layout_out, g.data(), g.size() * sizeof(float));
        *rows = M; *taps = T; *kpad = cdiv(in, tc::BK) * tc::BK;
    });
}

// Standalone entry for tests/test_gpu_implicit_conv.py: one implicit convolution on host data, through the engines' weight
// operand and launch (ic::launch).
//   w [M][taps][Cin], x [B][Ttot][Cin] (split into hi/lo planes here), bias / gamma / sa / sb [M / up] or null,
//   xo [B][T*up][M/up] in/out or null, hl_out [B][Hout + T*up][M/up] (hi + lo recombined; frames below Hout come back 0) or null.
int32_t b2a_implicit_conv_test(const float* w, int32_t M, int32_t taps, int32_t Cin, const float* x, int32_t B, int32_t Ttot, int32_t T,
                               int32_t dil, int32_t shift0, int32_t up, const float* bias, const float* gamma, int32_t gelu, int32_t add,
                               int32_t bias_twice_t0, const float* sa, const float* sb, int32_t Hout, int32_t fp16, float* xo, float* hl_out) {
    return guarded([&] {
        B2A_CHECK(w && x && M >= 1 && taps >= 1 && Cin >= 8 && Cin % 8 == 0 && B >= 1 && Ttot >= 1 && T >= 1 && dil >= 1 && shift0 >= 0 && up >= 1 &&
                      M % up == 0 && (M / up) % 8 == 0 && Hout >= 0 && (xo || hl_out) && (!add || xo) && ((sa == nullptr) == (sb == nullptr)),
                  B2A_ERR_INVALID_INPUT, "b2a_implicit_conv_test: bad argument");
        require_device(0);
        B2A_CUDA(cudaSetDevice(0));
        int num_sms = 132;
        B2A_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, 0));
        const int Cout = M / up;
        const long long To = (long long)T * up;
        TcW W;
        W.build(std::vector<float>(w, w + (size_t)M * taps * Cin), M, taps, Cin, fp16);
        if (bias) W.set_bias(std::vector<float>(bias, bias + Cout));
        const size_t nx = (size_t)B * Ttot * Cin, no = (size_t)B * To * Cout, nh = (size_t)B * (Hout + To) * Cout;
        std::vector<uint16_t> xp(2 * nx);
        for (size_t i = 0; i < nx; ++i) cg::split16(x[i], fp16, xp[i], xp[nx + i]);
        DBuf<bf16> dx, dh;
        DBuf<float> dxo, dgamma, dsa, dsb;
        dx.upload(reinterpret_cast<const bf16*>(xp.data()), xp.size());
        ic::Args a{};
        a.dil = dil; a.shift0 = shift0; a.B = B; a.T = T; a.up = up; a.gelu = gelu; a.add = add; a.bias_twice_t0 = bias_twice_t0; a.Hout = Hout;
        if (gamma) { dgamma.upload(gamma, Cout); a.gamma = dgamma.p; }
        if (sa) { dsa.upload(sa, Cout); dsb.upload(sb, Cout); a.sa = dsa.p; a.sb = dsb.p; }
        if (xo) { dxo.upload(xo, no); a.xo = dxo.p; }
        if (hl_out) { dh.alloc(2 * nh); B2A_CUDA(cudaMemset(dh.p, 0, 2 * nh * sizeof(bf16))); a.hl = dh.p; }
        B2A_CUDA(cudaDeviceSynchronize());
        ic::launch(W, dx.p, Ttot, a, num_sms, (cudaStream_t)0);
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaDeviceSynchronize());
        if (xo) B2A_CUDA(cudaMemcpy(xo, dxo.p, no * sizeof(float), cudaMemcpyDeviceToHost));
        if (hl_out) {
            std::vector<uint16_t> hp(2 * nh);
            B2A_CUDA(cudaMemcpy(hp.data(), dh.p, 2 * nh * sizeof(uint16_t), cudaMemcpyDeviceToHost));
            for (size_t i = 0; i < nh; ++i) hl_out[i] = cg::join16(hp[i], hp[nh + i], fp16);
        }
    });
}

int32_t b2a_speech_tokenizer_encoder_create(int32_t device, const b2a_speech_tokenizer_encoder_config* cfg, const b2a_tensor* tensors, int32_t n,
                                            b2a_speech_tokenizer_encoder** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_encoder_create: null out");
        *out = nullptr;
        B2A_CHECK(cfg && tensors && n > 0, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_speech_tokenizer_encoder_create: missing config or weights");
        TensorTable tt(tensors, n);
        *out = new b2a_speech_tokenizer_encoder(device, *cfg, tt);
    });
}

int64_t b2a_speech_tokenizer_encoder_encoded_length(const b2a_speech_tokenizer_encoder* h, int64_t n_samples) {
    return h ? h->encoded_length(n_samples) : 0;
}
int32_t b2a_speech_tokenizer_encoder_num_code_groups(const b2a_speech_tokenizer_encoder* h) { return h ? h->G : 0; }
void* b2a_speech_tokenizer_encoder_stream(b2a_speech_tokenizer_encoder* h) { return h ? (void*)h->stream : nullptr; }

int32_t b2a_speech_tokenizer_encoder_encode(b2a_speech_tokenizer_encoder* h, const float* audio, int32_t batch, int64_t n_samples, int32_t* codes) {
    return guarded([&] {
        B2A_CHECK(h && audio && codes, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_encoder_encode: null argument");
        h->encode_host(audio, batch, n_samples, codes, nullptr);
    });
}

int32_t b2a_speech_tokenizer_encoder_encode_dev(b2a_speech_tokenizer_encoder* h, const float* d_audio, int32_t batch, int64_t n_samples,
                                                int32_t* d_codes, void* stream) {
    return guarded([&] {
        B2A_CHECK(h && d_audio && d_codes, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_encoder_encode_dev: null argument");
        h->encode_dev(d_audio, batch, n_samples, d_codes, stream ? (cudaStream_t)stream : h->stream);
    });
}

int32_t b2a_speech_tokenizer_encoder_latent_test(b2a_speech_tokenizer_encoder* h, const float* audio, int32_t batch, int64_t n_samples,
                                                 float* z, int32_t* codes) {
    return guarded([&] {
        B2A_CHECK(h && audio && z, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_encoder_latent_test: null argument");
        h->encode_host(audio, batch, n_samples, codes, z);
    });
}

void b2a_speech_tokenizer_encoder_destroy(b2a_speech_tokenizer_encoder* h) { delete h; }

}  // extern "C"
