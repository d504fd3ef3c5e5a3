// Mimi codec for sm_90a (DESIGN.md §3.11): 24 kHz audio <-> 12.5 Hz codes, with the streaming decoder Marvis and PocketTTS use.
// Replaces (reference paths, directory = Sources/MLXAudioCodecs/Mimi/):
//   Mimi.swift:168-202        Mimi.encode / decode / decodeStep;  :207-233 MimiStreamingDecoder (reset, decodeFrames)
//   Quantization.swift        SplitResidualVectorQuantizer.decode (:203-210), ResidualVectorQuantization.decode (:113-120)
//   Conv.swift:265-362        StreamableConvTranspose1d.step (carried tail, bias subtracted), ConvTrUpsample1d
//   Transformer.swift         ProjectedTransformer / TransformerLayer / Attention with its per-call context window
//   Seanet.swift:259-353      SeanetDecoder (ELU, transposed convs, one residual block per layer with an identity skip)
// Encode is b2a_speech_tokenizer_encoder (the Qwen3-TTS speech-tokenizer encoder is Mimi's encoder, built from the same
// classes), created from this handle's config with every quantizer level kept.
//
// Decoder design: the Qwen3-TTS speech-tokenizer decoder's (§3.8).  Every call is the streaming step with carried state; a one-shot
// decode is the step after a reset (zero history == the reference's causal zero padding).  Dense layers -- the two quantizer output
// projections, the transformer linears, the init / residual convs and the transposed convs (as phase-major 2-tap causal convs) --
// are implicit-GEMM launches (ic::launch) over hi/lo activation planes that carry each consumer's history frames in front; the
// epilogue fuses bias, layer scale, GELU, the residual add and the ELU of the next conv's input.  The transposed convs add their
// bias once: the reference subtracts it from the carried tail before the overlap-add (Conv.swift:316), which is exactly a causal
// conv over the previous chunk's last input frame.
#include "common.cuh"
#include "conv_gemm.cuh"
#include "codec_transformer.cuh"

#include <algorithm>
#include <cmath>
#include <memory>
#include <string>
#include <vector>

namespace b2a {
namespace mimi {

using namespace b2a::st;
using cg::TcW;

// ConvTrUpsample1d.step (Conv.swift:305-328, 349-362): depthwise transposed conv, kernel 2 s, stride s, no bias, written as a causal
// conv over input frames q - 1 and q:  y[q s + rho][c] = w[c][rho] x[q][c] + w[c][rho + s] x[q - 1][c].  x[-1] is the previous
// call's last input frame st [B][1][C] (zeros after a reset): the reference's carried tail is w[c][rho + s] x[T - 1][c].
static __global__ void upsample_dw_kernel(const float* __restrict__ x, const float* __restrict__ st, const float* __restrict__ w,
                                          float* __restrict__ y, int B, int T, int C, int s) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long To = (long long)T * s;
    if (i >= (long long)B * To * C) return;
    const int c = (int)(i % C);
    const long long r = i / C;
    const int f = (int)(r % To), b = (int)(r / To);
    const int q = f / s, rho = f - q * s;
    const float x0 = x[((long long)b * T + q) * C + c];
    const float xm = q > 0 ? x[((long long)b * T + q - 1) * C + c] : st[(long long)b * C + c];
    y[i] = fmaf(w[c * 2 * s + rho], x0, w[c * 2 * s + rho + s] * xm);
}

// ELU -> causal k-tap conv to ONE channel, no clip          (SeanetDecoder :341-346: elu, final_conv1d)
// x [B, T, C] fp32 (the last residual block's output), st [B, k-1, C] its raw history.  64 outputs per CTA; the activated tile
// lives in shared memory with a padded row stride.
constexpr int OC_TILE = 64, OC_THREADS = 128, OC_MAXK = 8;
static __global__ void __launch_bounds__(OC_THREADS)
elu_out_conv_kernel(const float* __restrict__ x, const float* __restrict__ st, const float* __restrict__ w /*[k, C]*/, float bias,
                    float* __restrict__ wave, int T, int C, int k) {
    extern __shared__ float osm[];
    const int H = k - 1, rows = OC_TILE + H, ldc = C + 1;
    float* tile = osm;                    // [rows][C + 1]
    float* wk = osm + rows * ldc;         // [k][C]
    float* red = wk + k * C;              // [OC_THREADS]
    const int b = blockIdx.y, t0 = blockIdx.x * OC_TILE;
    for (int i = threadIdx.x; i < k * C; i += OC_THREADS) wk[i] = w[i];
    for (int i = threadIdx.x; i < rows * C; i += OC_THREADS) {
        const int rr = i / C, c = i - rr * C;
        const int ti = t0 - H + rr;
        float v = 0.f;
        if (ti >= 0) { if (ti < T) v = x[((long long)b * T + ti) * C + c]; }
        else v = st[((long long)b * H + (H + ti)) * C + c];
        tile[rr * ldc + c] = v > 0.f ? v : expm1f(v);
    }
    __syncthreads();
    const int o = threadIdx.x & (OC_TILE - 1), part = threadIdx.x / OC_TILE;      // two threads per output, channels split in halves
    const int cbeg = part * ((C + 1) / 2), cend = min(C, cbeg + (C + 1) / 2);
    float acc = 0.f;
    for (int kk = 0; kk < k; ++kk)
        for (int c = cbeg; c < cend; ++c) acc = fmaf(wk[kk * C + c], tile[(o + kk) * ldc + c], acc);
    red[threadIdx.x] = acc;
    __syncthreads();
    if (part == 0 && t0 + o < T) wave[(long long)b * T + t0 + o] = red[o] + red[o + OC_TILE] + bias;
}

struct TLayer { TcW qkv, o, fc1, fc2; DBuf<float> ln1w, ln1b, ln2w, ln2b, ls1, ls2, K, V; };
struct DLayer { TcW ct, c1, c2; PlaneState st_ct, st_c1; int r = 1, cin = 0, cout = 0, hid = 0; };

}  // namespace mimi
}  // namespace b2a

using namespace b2a;
using namespace b2a::mimi;

struct b2a_mimi {
    int device = 0, num_sms = 132;
    b2a_mimi_config cfg{};
    cudaStream_t stream = nullptr;
    b2a_speech_tokenizer_encoder* enc = nullptr;
    int D = 0, hd = 0, ds = 1, hop = 1, spf = 1, cap = 0;     // latent width, head dim, upsample stride, SEANet hop, samples per code frame, KV capacity
    // weights
    DBuf<float> emb;               // [nq][bins][qd] usage-normalised codebooks
    TcW rvq_proj;                  // [D][first | rest] output projections over the two gathered sums
    DBuf<float> up_w;              // [D][2 ds]
    F32State st_up;
    std::vector<TLayer> layers;
    DBuf<float> inv_freq;
    TcW init_conv;
    PlaneState st_init;
    std::vector<DLayer> dl;
    DBuf<float> out_w;             // [k][n_filters]
    float out_b = 0.f;
    F32State st_out;
    // streaming state
    int parity = 0, steps = 0, cache_len = 0, stream_B = 0;
    // workspace
    DBuf<int> d_codes;
    DBuf<bf16> P0, P1;
    DBuf<float> Xh, Xc, Q, wave, wave_all;

    static constexpr int F16 = 1;  // fp16 hi/lo operand pairs (22 mantissa bits), as the speech-tokenizer decoder

    static void up(DBuf<float>& d, const std::vector<float>& v) { d.upload(v.data(), v.size()); }
    void load_linear(TcW& w, const TensorTable& tt, const std::string& p, int out, int in) {
        w.build(tt.f32(p + ".weight", (int64_t)out * in), out, 1, in, F16);
    }
    void load_conv(TcW& w, const TensorTable& tt, const std::string& p, int out, int k, int in) {
        w.build(tt.f32(p + ".weight", (int64_t)out * k * in), out, k, in, F16);      // MLX [out, k, in] == [M][taps][Cin]
        w.set_bias(tt.f32(p + ".bias", out));
    }

    static void validate(const b2a_mimi_config& c) {
        B2A_CHECK(c.channels == 1, B2A_ERR_INVALID_INPUT, "mimi: channels must be 1");
        B2A_CHECK(c.causal == 1 && c.true_skip == 1 && c.n_residual_layers == 1, B2A_ERR_INVALID_INPUT,
                  "mimi: only the causal SEANet with one identity-skip residual layer per stage is implemented");
        B2A_CHECK(c.gating == 0 && c.norm_rms == 0 && c.kv_repeat == 1, B2A_ERR_INVALID_INPUT,
                  "mimi: only the LayerNorm, GELU-MLP transformer without key repetition is implemented");
        B2A_CHECK(c.num_heads >= 1 && c.dimension % c.num_heads == 0, B2A_ERR_INVALID_INPUT, "mimi: dimension must be a multiple of num_heads");
        const int hd = c.dimension / c.num_heads;
        B2A_CHECK(hd == 32 || hd == 64 || hd == 128, B2A_ERR_INVALID_INPUT, "mimi: head_dim must be 32, 64 or 128");
        B2A_CHECK(c.dimension % 64 == 0 && c.dim_feedforward >= 8 && c.dim_feedforward % 8 == 0 && c.num_layers >= 1 && c.context >= 0 &&
                      c.max_period >= 1, B2A_ERR_INVALID_INPUT, "mimi: bad transformer geometry");
        B2A_CHECK(c.num_ratios >= 1 && c.num_ratios <= 8 && c.n_filters >= 8 && c.compress >= 1, B2A_ERR_INVALID_INPUT, "mimi: bad SEANet geometry");
        long long hop = 1;
        for (int i = 0; i < c.num_ratios; ++i) {
            B2A_CHECK(c.ratios[i] >= 1 && c.ratios[i] <= 16, B2A_ERR_INVALID_INPUT, "mimi: ratios must be in 1..16");
            hop *= c.ratios[i];
        }
        for (int i = 0; i <= c.num_ratios; ++i) {        // every decoder conv's channel counts are whole 8-channel groups
            const long long ch = (long long)c.n_filters << (c.num_ratios - i);
            B2A_CHECK(ch % 8 == 0 && (i == 0 || (ch / c.compress) % 8 == 0) && ch <= 8192, B2A_ERR_INVALID_INPUT,
                      "mimi: decoder channel counts (and their residual hidden widths) must be multiples of 8");
        }
        B2A_CHECK(c.kernel_size >= 1 && c.kernel_size <= 16 && c.residual_kernel_size >= 1 && c.residual_kernel_size <= 16 &&
                      c.last_kernel_size >= 1 && c.last_kernel_size <= OC_MAXK, B2A_ERR_INVALID_INPUT, "mimi: bad kernel sizes");
        B2A_CHECK(c.sample_rate >= 1 && c.frame_rate > 0.f && (int)((double)c.sample_rate / (double)hop / (double)c.frame_rate) >= 1,
                  B2A_ERR_INVALID_INPUT, "mimi: sample_rate / prod(ratios) / frame_rate must be >= 1");
        B2A_CHECK(c.num_codebooks >= 1 && c.codebook_size >= 1 && c.codebook_dim >= 8 && c.codebook_dim % 8 == 0, B2A_ERR_INVALID_INPUT,
                  "mimi: bad quantizer geometry");
        B2A_CHECK(c.max_batch >= 1 && c.max_cache_frames >= 1, B2A_ERR_INVALID_INPUT, "mimi: max_batch / max_cache_frames must be positive");
    }

    b2a_mimi(int dev, const b2a_mimi_config& c, const TensorTable& tt, const b2a_tensor* tensors, int n_tensors) : device(dev), cfg(c) {
        validate(c);
        require_device(dev);
        B2A_CUDA(cudaSetDevice(dev));
        B2A_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
        D = c.dimension; hd = D / c.num_heads;
        hop = 1;
        for (int i = 0; i < c.num_ratios; ++i) hop *= c.ratios[i];
        ds = (int)((double)c.sample_rate / (double)hop / (double)c.frame_rate);        // Mimi.init (:122-123)
        spf = hop * ds;
        B2A_CHECK((long long)c.max_cache_frames * ds < (1ll << 30), B2A_ERR_INVALID_INPUT, "mimi: max_cache_frames too large");
        cap = c.max_cache_frames * ds;
        const int nq = c.num_codebooks, bins = c.codebook_size, qd = c.codebook_dim, F = c.dim_feedforward;
        // ---- quantizer decode: codebooks = embedding_sum / max(cluster_usage, 1e-5) (Quantization.swift:29-33)
        {
            std::vector<float> e((size_t)nq * bins * qd);
            for (int q = 0; q < nq; ++q) {
                const std::string p = q == 0 ? std::string("quantizer.rvq_first.vq.layers.0") : "quantizer.rvq_rest.vq.layers." + std::to_string(q - 1);
                const std::vector<float> sum = tt.f32(p + ".codebook.embedding_sum", (int64_t)bins * qd), use = tt.f32(p + ".codebook.cluster_usage", bins);
                for (int r = 0; r < bins; ++r) {
                    const float u = std::max(use[r], 1e-5f);
                    for (int d = 0; d < qd; ++d) e[((size_t)q * bins + r) * qd + d] = sum[(size_t)r * qd + d] / u;
                }
            }
            up(emb, e);
            // rvq_first.output_proj on level 0's row, rvq_rest.output_proj on the sum of the others, added: one [D, 2 qd] matrix
            std::vector<float> w1 = tt.f32("quantizer.rvq_first.output_proj.weight", (int64_t)D * qd), w((size_t)D * 2 * qd, 0.f);
            std::vector<float> w2 = nq > 1 ? tt.f32("quantizer.rvq_rest.output_proj.weight", (int64_t)D * qd) : std::vector<float>((size_t)D * qd, 0.f);
            for (int o = 0; o < D; ++o) {
                memcpy(&w[(size_t)o * 2 * qd], &w1[(size_t)o * qd], (size_t)qd * sizeof(float));
                memcpy(&w[(size_t)o * 2 * qd + qd], &w2[(size_t)o * qd], (size_t)qd * sizeof(float));
            }
            rvq_proj.build(w, D, 1, 2 * qd, F16);
        }
        up(up_w, tt.f32("upsample.convtr.convtr.convtr.weight", (int64_t)D * 2 * ds));      // MLX depthwise [C, k, 1]
        st_up.H = 1; st_up.C = D;
        // ---- decoder transformer
        layers.resize(c.num_layers);
        for (int l = 0; l < c.num_layers; ++l) {
            const std::string p = "decoder_transformer.transformer.layers." + std::to_string(l) + ".";
            TLayer& L = layers[l];
            load_linear(L.qkv, tt, p + "self_attn.in_proj", 3 * D, D);
            load_linear(L.o, tt, p + "self_attn.out_proj", D, D);
            load_linear(L.fc1, tt, p + "gating.linear1", F, D);
            load_linear(L.fc2, tt, p + "gating.linear2", D, F);
            up(L.ln1w, tt.f32(p + "norm1.weight", D)); up(L.ln1b, tt.f32(p + "norm1.bias", D));
            up(L.ln2w, tt.f32(p + "norm2.weight", D)); up(L.ln2b, tt.f32(p + "norm2.bias", D));
            up(L.ls1, tt.f32(p + "layer_scale_1.scale", D)); up(L.ls2, tt.f32(p + "layer_scale_2.scale", D));
        }
        {   // RoPE(dimensions: head_dim, traditional: true, base: Float(maxPeriod))   (Transformer.swift:130)
            std::vector<float> f(hd / 2);
            for (int i = 0; i < hd / 2; ++i) f[i] = 1.0f / powf((float)c.max_period, (float)(2 * i) / (float)hd);
            up(inv_freq, f);
        }
        // ---- SEANet decoder
        const int L = c.num_ratios;
        const int C0 = c.n_filters << L;
        load_conv(init_conv, tt, "decoder.init_conv1d.conv.conv", C0, c.kernel_size, D);
        st_init.H = c.kernel_size - 1; st_init.C = D;
        dl.resize(L);
        for (int i = 0; i < L; ++i) {
            DLayer& Y = dl[i];
            const std::string p = "decoder.layers." + std::to_string(i) + ".";
            Y.r = c.ratios[i]; Y.cin = C0 >> i; Y.cout = Y.cin / 2; Y.hid = Y.cout / c.compress;
            const int k = 2 * Y.r;
            Y.ct.build(convt_weight(tt.f32(p + "upsample.convtr.convtr.weight", (int64_t)Y.cout * k * Y.cin), Y.cout, k, Y.cin, Y.r), Y.r * Y.cout, 2, Y.cin, F16);
            Y.ct.set_bias(tt.f32(p + "upsample.convtr.convtr.bias", Y.cout));
            Y.st_ct.H = 1; Y.st_ct.C = Y.cin;
            load_conv(Y.c1, tt, p + "residuals.0.block.0.conv.conv", Y.hid, c.residual_kernel_size, Y.cout);
            load_conv(Y.c2, tt, p + "residuals.0.block.1.conv.conv", Y.cout, 1, Y.hid);
            Y.st_c1.H = c.residual_kernel_size - 1; Y.st_c1.C = Y.cout;
        }
        up(out_w, tt.f32("decoder.final_conv1d.conv.conv.weight", (int64_t)c.last_kernel_size * c.n_filters));
        out_b = tt.f32("decoder.final_conv1d.conv.conv.bias", 1)[0];
        st_out.H = c.last_kernel_size - 1; st_out.C = c.n_filters;
        B2A_CUDA(cudaDeviceSynchronize());
        alloc_state();
        // ---- encoder: the speech-tokenizer encoder's implementation, every level kept
        {
            b2a_speech_tokenizer_encoder_config e{};
            e.sampling_rate = c.sample_rate; e.frame_rate = c.frame_rate; e.audio_channels = c.channels; e.num_filters = c.n_filters;
            e.num_residual_layers = c.n_residual_layers; e.num_upsampling_ratios = c.num_ratios;
            for (int i = 0; i < c.num_ratios; ++i) e.upsampling_ratios[i] = c.ratios[i];
            e.kernel_size = c.kernel_size; e.residual_kernel_size = c.residual_kernel_size; e.last_kernel_size = c.last_kernel_size;
            e.compress = c.compress; e.use_causal_conv = c.causal; e.use_conv_shortcut = !c.true_skip;
            e.hidden_size = D; e.intermediate_size = F; e.num_hidden_layers = c.num_layers; e.num_attention_heads = c.num_heads;
            e.num_key_value_heads = c.num_heads; e.head_dim = hd; e.rope_theta = (float)c.max_period;
            e.codebook_size = bins; e.codebook_dim = qd; e.num_quantizers = nq; e.valid_num_quantizers = nq;
            const int32_t st = b2a_speech_tokenizer_encoder_create(dev, &e, tensors, n_tensors, &enc);
            if (st != B2A_OK) throw Error(st, b2a_last_error());
        }
        // last: a check that throws above leaves no stream behind (the destructor does not run for a half-built object)
        B2A_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        reset();
    }
    ~b2a_mimi() {
        if (enc) b2a_speech_tokenizer_encoder_destroy(enc);
        if (stream) cudaStreamDestroy(stream);
    }

    void alloc_state() {
        const int B = cfg.max_batch;
        auto ps = [&](PlaneState& s) { for (int i = 0; i < 2; ++i) s.s[i].alloc((size_t)2 * B * std::max(s.H, 1) * s.C); };
        auto fs = [&](F32State& s) { for (int i = 0; i < 2; ++i) s.s[i].alloc((size_t)B * std::max(s.H, 1) * s.C); };
        fs(st_up); ps(st_init); fs(st_out);
        for (auto& Y : dl) { ps(Y.st_ct); ps(Y.st_c1); }
        const size_t kv = (size_t)B * D * cap;
        for (auto& L : layers) { L.K.alloc(kv); L.V.alloc(kv); }
    }

    // MimiStreamingDecoder.reset (:215-219): decoder conv histories, the upsample tail and the KV cache
    void reset() {
        B2A_CUDA(cudaSetDevice(device));
        auto zp = [&](PlaneState& s) { for (int i = 0; i < 2; ++i) B2A_CUDA(cudaMemsetAsync(s.s[i].p, 0, s.s[i].n * sizeof(bf16), stream)); };
        auto zf = [&](F32State& s) { for (int i = 0; i < 2; ++i) B2A_CUDA(cudaMemsetAsync(s.s[i].p, 0, s.s[i].n * sizeof(float), stream)); };
        zf(st_up); zp(st_init); zf(st_out);
        for (auto& Y : dl) { zp(Y.st_ct); zp(Y.st_c1); }
        B2A_CUDA(cudaStreamSynchronize(stream));     // a following step may run on a caller's stream
        parity = 0; steps = 0; cache_len = 0; stream_B = 0;
    }

    // ------------------------------------------------------------------------------------------- launches
    bf16* planes(DBuf<bf16>& buf, int B, long long frames, int C) {
        B2A_CHECK((size_t)2 * B * frames * C <= buf.n, B2A_ERR_GENERATION_FAILED, "mimi: internal workspace too small");
        return buf.p;
    }
    bf16* planes(bf16* p, int B, long long frames, int C) { return planes(p == P0.p ? P0 : P1, B, frames, C); }
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

    void check_step(int B, int K, int T) const {
        B2A_CHECK(B >= 1 && B <= cfg.max_batch, B2A_ERR_INVALID_INPUT, "mimi: batch must be in [1, max_batch]");
        B2A_CHECK(K >= 1 && K <= cfg.num_codebooks, B2A_ERR_INVALID_INPUT, "mimi: the number of codebooks must be in [1, num_codebooks]");
        B2A_CHECK(T >= 1, B2A_ERR_INVALID_INPUT, "mimi: need at least one code frame");
        B2A_CHECK(steps == 0 || B == stream_B, B2A_ERR_INVALID_INPUT, "mimi: batch size changed inside a stream (reset first)");
        B2A_CHECK((long long)cache_len + (long long)T * ds <= cap, B2A_ERR_INVALID_INPUT, "mimi: stream longer than max_cache_frames");
        B2A_CHECK((long long)T * spf < (1ll << 31) && (long long)B * T * spf / 64 < (1ll << 31), B2A_ERR_INVALID_INPUT, "mimi: chunk too large");
    }

    // Mimi.decodeStep (:196-202): d_codes [B, K, T] int32 (device) -> d_wave [B, T * spf]
    void step_dev(const int* dcodes, int B, int K, int T, float* d_wave, cudaStream_t s) {
        const auto& c = cfg;
        check_step(B, K, T);
        B2A_CUDA(cudaSetDevice(device));
        stream_B = B;
        const int qd = c.codebook_dim, F = c.dim_feedforward, nh = c.num_heads, Lr = (int)dl.size();
        const int Tl = T * ds;
        const long long N = (long long)B * Tl;
        {   // workspace: the largest planar activation and fp32 tensors of the chunk
            size_t pmax = 0, xc = (size_t)B * T * D;
            auto pl = [&](long long frames, int C) { pmax = std::max(pmax, (size_t)(2ll * B * frames * C)); };
            pl(T, 2 * qd); pl(Tl, std::max(D, F)); pl(st_init.H + Tl, D); pl(1 + Tl, dl[0].cin);
            long long Tc = Tl;
            for (auto& Y : dl) {
                Tc *= Y.r;
                pl(Y.st_c1.H + Tc, Y.cout); pl(Tc, Y.hid); pl(1 + Tc, Y.cout);
                xc = std::max(xc, (size_t)((long long)B * Tc * Y.cout));
            }
            P0.alloc(pmax); P1.alloc(pmax);
            Xh.alloc((size_t)N * D); Xc.alloc(xc); Q.alloc((size_t)N * 3 * D);
        }
        // 1. split-RVQ decode: gather-sum level 0 | levels 1..K-1, both output projections as one GEMM   (Quantization.swift:203-210)
        rvq_gather_kernel<<<(unsigned)((long long)B * T), 128, 0, s>>>(dcodes, emb.p, planes(P0, B, T, 2 * qd), B, T, K, c.num_codebooks, 1,
                                                                      c.codebook_size, qd, F16);
        count_launch();
        { ic::Args a{}; a.B = B; a.T = T; a.xo = Xc.p; conv(rvq_proj, P0.p, T, a, s); }
        // 2. ConvTrUpsample1d.step: x ds into the transformer's residual stream                          (Conv.swift:305-328)
        upsample_dw_kernel<<<(unsigned)cdiv(N * D, 256), 256, 0, s>>>(Xc.p, st_up.s[parity].p, up_w.p, Xh.p, B, T, D, ds);
        count_launch();
        update_f32(Xc.p, st_up, B, T, s);
        // 3. decoder transformer over the KV cache; the last layer also writes the init conv's input planes      (Transformer.swift)
        const float scale = 1.0f / sqrtf((float)hd);
        const int key_lo = std::max(0, cache_len - c.context);
        for (size_t l = 0; l < layers.size(); ++l) {
            TLayer& Ly = layers[l];
            layernorm_planes_kernel<<<(unsigned)N, RN_THREADS, 0, s>>>(Xh.p, Ly.ln1w.p, Ly.ln1b.p, planes(P0, B, Tl, D), N, D, 1e-5f, F16);
            count_launch();
            { ic::Args a{}; a.B = B; a.T = Tl; a.xo = Q.p; conv(Ly.qkv, P0.p, Tl, a, s); }
            rope_cache_kernel<true><<<(unsigned)N, 256, 0, s>>>(Q.p, Ly.K.p, Ly.V.p, inv_freq.p, Tl, cache_len, nh, nh, hd, cap);
            count_launch();
            {
                const dim3 grid(cdiv(Tl, AT_WARPS), nh, B), block(AT_WARPS * 32);
                bf16* out = planes(P1, B, Tl, D);
                if (hd == 32) attn_kernel<1><<<grid, block, 0, s>>>(Q.p, Ly.K.p, Ly.V.p, out, B, Tl, cache_len, nh, nh, cap, scale, F16, key_lo);
                else if (hd == 64) attn_kernel<2><<<grid, block, 0, s>>>(Q.p, Ly.K.p, Ly.V.p, out, B, Tl, cache_len, nh, nh, cap, scale, F16, key_lo);
                else attn_kernel<4><<<grid, block, 0, s>>>(Q.p, Ly.K.p, Ly.V.p, out, B, Tl, cache_len, nh, nh, cap, scale, F16, key_lo);
                count_launch();
            }
            { ic::Args a{}; a.B = B; a.T = Tl; a.xo = Xh.p; a.add = 1; a.gamma = Ly.ls1.p; conv(Ly.o, P1.p, Tl, a, s); }
            layernorm_planes_kernel<<<(unsigned)N, RN_THREADS, 0, s>>>(Xh.p, Ly.ln2w.p, Ly.ln2b.p, planes(P0, B, Tl, D), N, D, 1e-5f, F16);
            count_launch();
            { ic::Args a{}; a.B = B; a.T = Tl; a.gelu = 1; a.hl = planes(P1, B, Tl, F); conv(Ly.fc1, P0.p, Tl, a, s); }
            ic::Args a{}; a.B = B; a.T = Tl; a.xo = Xh.p; a.add = 1; a.gamma = Ly.ls2.p;
            if (l + 1 == layers.size()) { a.hl = planes(P0, B, st_init.H + Tl, D); a.Hout = st_init.H; }
            conv(Ly.fc2, P1.p, Tl, a, s);
        }
        // 4. SEANet decoder (Seanet.swift:341-353).  cur / other: planes [2][B][H + frames][C], the consumer's history in front
        bf16* cur = P0.p;
        bf16* other = P1.p;
        carry(cur, st_init, B, Tl, s);
        { ic::Args a{}; a.B = B; a.T = Tl; a.hl = planes(P1, B, 1 + Tl, dl[0].cin); a.Hout = 1; a.elu = 1; conv(init_conv, cur, st_init.H + Tl, a, s); }
        std::swap(cur, other);
        long long Tc = Tl;
        for (int i = 0; i < Lr; ++i) {
            DLayer& Y = dl[i];
            // ELU -> transposed conv (k = 2 r, stride r, bias once) -> x (fp32) and ELU(x) planes for the residual block   (:298-302)
            carry(cur, Y.st_ct, B, Tc, s);
            {
                ic::Args a{}; a.B = B; a.T = (int)Tc; a.up = Y.r; a.xo = Xc.p; a.hl = planes(other, B, Y.st_c1.H + Tc * Y.r, Y.cout); a.Hout = Y.st_c1.H; a.elu = 1;
                conv(Y.ct, cur, 1 + Tc, a, s);
            }
            Tc *= Y.r;
            std::swap(cur, other);
            // SeanetResnetBlock.step (:142-152): x + conv_k1(ELU(conv_k3(ELU(x)))); the sum also feeds the next layer's ELU planes
            carry(cur, Y.st_c1, B, Tc, s);
            { ic::Args a{}; a.B = B; a.T = (int)Tc; a.hl = planes(other, B, Tc, Y.hid); a.elu = 1; conv(Y.c1, cur, Y.st_c1.H + Tc, a, s); }
            ic::Args a{}; a.B = B; a.T = (int)Tc; a.xo = Xc.p; a.add = 1;
            if (i + 1 < Lr) { a.hl = planes(cur, B, 1 + Tc, Y.cout); a.Hout = 1; a.elu = 1; }
            conv(Y.c2, other, Tc, a, s);
        }
        // 5. ELU + final conv to one channel                                                                  (:344-345)
        {
            const int Cf = st_out.C, k = cfg.last_kernel_size;
            const size_t smem = ((size_t)(OC_TILE + k - 1) * (Cf + 1) + (size_t)k * Cf + OC_THREADS) * sizeof(float);
            B2A_CUDA(cudaFuncSetAttribute(elu_out_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            elu_out_conv_kernel<<<dim3(cdiv(Tc, OC_TILE), B), OC_THREADS, smem, s>>>(Xc.p, st_out.s[parity].p, out_w.p, out_b, d_wave, (int)Tc, Cf, k);
            count_launch();
            update_f32(Xc.p, st_out, B, Tc, s);
        }
        B2A_CUDA(cudaGetLastError());
        parity ^= 1;
        steps += 1;
        cache_len += Tl;
    }

    void check_codes(const int32_t* codes, size_t n) const {
        for (size_t i = 0; i < n; ++i)
            B2A_CHECK(codes[i] >= 0 && codes[i] < cfg.codebook_size, B2A_ERR_INVALID_INPUT, "mimi: code outside [0, codebook_size)");
    }

    // host codes [B, K, T] -> host wave [B, T * spf]
    void step_host(const int32_t* codes, int B, int K, int T, float* out) {
        check_step(B, K, T);
        check_codes(codes, (size_t)B * K * T);
        cudaStream_t s = stream;
        const size_t nin = (size_t)B * K * T, nout = (size_t)B * T * spf;
        d_codes.alloc(nin); wave.alloc(nout);
        B2A_CUDA(cudaMemcpyAsync(d_codes.p, codes, nin * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        step_dev(d_codes.p, B, K, T, wave.p, s);
        B2A_CUDA(cudaMemcpyAsync(out, wave.p, nout * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    }

    // MimiStreamingDecoder.decodeFrames (:221-232): T single-frame steps, codes uploaded once, one copy back
    void frames_host(const int32_t* codes, int B, int K, int T, float* out) {
        B2A_CHECK(B >= 1 && K >= 1 && T >= 1, B2A_ERR_INVALID_INPUT, "mimi: empty input");
        check_step(B, K, 1);
        B2A_CHECK((long long)cache_len + (long long)T * ds <= cap, B2A_ERR_INVALID_INPUT, "mimi: stream longer than max_cache_frames");
        check_codes(codes, (size_t)B * K * T);
        cudaStream_t s = stream;
        std::vector<int32_t> fr((size_t)T * B * K);          // [T][B][K]: one frame's codes contiguous
        for (int b = 0; b < B; ++b)
            for (int k = 0; k < K; ++k)
                for (int t = 0; t < T; ++t) fr[((size_t)t * B + b) * K + k] = codes[((size_t)b * K + k) * T + t];
        d_codes.alloc(fr.size()); wave.alloc((size_t)B * spf); wave_all.alloc((size_t)B * T * spf);
        B2A_CUDA(cudaMemcpyAsync(d_codes.p, fr.data(), fr.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        for (int t = 0; t < T; ++t) {
            step_dev(d_codes.p + (size_t)t * B * K, B, K, 1, wave.p, s);
            B2A_CUDA(cudaMemcpy2DAsync(wave_all.p + (size_t)t * spf, (size_t)T * spf * sizeof(float), wave.p, (size_t)spf * sizeof(float),
                                       (size_t)spf * sizeof(float), (size_t)B, cudaMemcpyDeviceToDevice, s));
        }
        B2A_CUDA(cudaMemcpyAsync(out, wave_all.p, (size_t)B * T * spf * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    }
};

extern "C" {

int32_t b2a_mimi_config_default(int32_t num_codebooks, int32_t max_batch, int32_t max_cache_frames, b2a_mimi_config* out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_mimi_config_default: null out");
        B2A_CHECK(num_codebooks >= 1 && max_batch >= 1 && max_cache_frames >= 1, B2A_ERR_INVALID_INPUT,
                  "b2a_mimi_config_default: num_codebooks, max_batch and max_cache_frames must be positive");
        b2a_mimi_config c{};
        c.sample_rate = 24000; c.frame_rate = 12.5f; c.channels = 1;
        c.dimension = 512; c.n_filters = 64; c.n_residual_layers = 1;
        c.num_ratios = 4; c.ratios[0] = 8; c.ratios[1] = 6; c.ratios[2] = 5; c.ratios[3] = 4;
        c.kernel_size = 7; c.residual_kernel_size = 3; c.last_kernel_size = 3; c.dilation_base = 2; c.compress = 2;
        c.causal = 1; c.true_skip = 1;
        c.num_heads = 8; c.num_layers = 8; c.dim_feedforward = 2048; c.context = 250; c.max_period = 10000;
        c.gating = 0; c.norm_rms = 0; c.kv_repeat = 1;
        c.num_codebooks = num_codebooks; c.codebook_size = 2048; c.codebook_dim = 256;
        c.max_batch = max_batch; c.max_cache_frames = max_cache_frames;
        *out = c;
    });
}

int32_t b2a_mimi_create(int32_t device, const b2a_mimi_config* cfg, const b2a_tensor* tensors, int32_t n, b2a_mimi** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_mimi_create: null out");
        *out = nullptr;
        B2A_CHECK(cfg, B2A_ERR_INVALID_INPUT, "b2a_mimi_create: null config");
        b2a_mimi::validate(*cfg);
        B2A_CHECK(tensors && n > 0, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_mimi_create: no weights");
        TensorTable tt(tensors, n);
        *out = new b2a_mimi(device, *cfg, tt, tensors, n);
    });
}

int32_t b2a_mimi_num_codebooks(const b2a_mimi* h) { return h ? h->cfg.num_codebooks : 0; }
int32_t b2a_mimi_samples_per_frame(const b2a_mimi* h) { return h ? h->spf : 0; }
int64_t b2a_mimi_encoded_length(const b2a_mimi* h, int64_t n_samples) { return h ? b2a_speech_tokenizer_encoder_encoded_length(h->enc, n_samples) : 0; }
void* b2a_mimi_stream(b2a_mimi* h) { return h ? (void*)h->stream : nullptr; }

int32_t b2a_mimi_encode(b2a_mimi* h, const float* audio, int32_t batch, int64_t n_samples, int32_t* codes) {
    return guarded([&] {
        B2A_CHECK(h && audio && codes, B2A_ERR_INVALID_INPUT, "b2a_mimi_encode: null argument");
        const int32_t st = b2a_speech_tokenizer_encoder_encode(h->enc, audio, batch, n_samples, codes);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
    });
}

int32_t b2a_mimi_encode_dev(b2a_mimi* h, const float* d_audio, int32_t batch, int64_t n_samples, int32_t* d_codes, void* stream) {
    return guarded([&] {
        B2A_CHECK(h && d_audio && d_codes, B2A_ERR_INVALID_INPUT, "b2a_mimi_encode_dev: null argument");
        const int32_t st = b2a_speech_tokenizer_encoder_encode_dev(h->enc, d_audio, batch, n_samples, d_codes, stream ? stream : (void*)h->stream);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
    });
}

int32_t b2a_mimi_reset(b2a_mimi* h) {
    return guarded([&] {
        B2A_CHECK(h, B2A_ERR_INVALID_INPUT, "b2a_mimi_reset: null handle");
        h->reset();
    });
}

int32_t b2a_mimi_decode_step(b2a_mimi* h, const int32_t* codes, int32_t B, int32_t K, int32_t T, float* wave) {
    return guarded([&] {
        B2A_CHECK(h && codes && wave, B2A_ERR_INVALID_INPUT, "b2a_mimi_decode_step: null argument");
        h->step_host(codes, B, K, T, wave);
    });
}

int32_t b2a_mimi_decode_step_dev(b2a_mimi* h, const int32_t* d_codes, int32_t B, int32_t K, int32_t T, float* d_wave, void* stream) {
    return guarded([&] {
        B2A_CHECK(h && d_codes && d_wave, B2A_ERR_INVALID_INPUT, "b2a_mimi_decode_step_dev: null argument");
        h->step_dev(d_codes, B, K, T, d_wave, stream ? (cudaStream_t)stream : h->stream);
    });
}

int32_t b2a_mimi_decode(b2a_mimi* h, const int32_t* codes, int32_t B, int32_t K, int32_t T, float* wave) {
    return guarded([&] {
        B2A_CHECK(h && codes && wave, B2A_ERR_INVALID_INPUT, "b2a_mimi_decode: null argument");
        h->reset();
        h->step_host(codes, B, K, T, wave);
    });
}

int32_t b2a_mimi_decode_dev(b2a_mimi* h, const int32_t* d_codes, int32_t B, int32_t K, int32_t T, float* d_wave, void* stream) {
    return guarded([&] {
        B2A_CHECK(h && d_codes && d_wave, B2A_ERR_INVALID_INPUT, "b2a_mimi_decode_dev: null argument");
        h->reset();
        h->step_dev(d_codes, B, K, T, d_wave, stream ? (cudaStream_t)stream : h->stream);
    });
}

int32_t b2a_mimi_decode_frames(b2a_mimi* h, const int32_t* codes, int32_t B, int32_t K, int32_t T, float* wave) {
    return guarded([&] {
        B2A_CHECK(h && codes && wave, B2A_ERR_INVALID_INPUT, "b2a_mimi_decode_frames: null argument");
        h->frames_host(codes, B, K, T, wave);
    });
}

void b2a_mimi_destroy(b2a_mimi* h) { delete h; }

}  // extern "C"
