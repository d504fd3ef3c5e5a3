// Vocos vocoder decode for sm_90a (SURVEY.md row a17).  Replaces (reference paths):
//   Sources/MLXAudioCodecs/Vocos/VocosBackbone.swift:18-100,109-204   ConvNeXt backbone
//   Sources/MLXAudioCodecs/Vocos/Vocos.swift:54-179                    ISTFTHead (IRFFT on device + overlap-add in
//                                                                      scalar host loops with per-frame D2H copies)
//   Sources/MLXAudioCodecs/Vocos/Vocos.swift:284-322                   Vocos.decode / decodeAudio
// Channels-last throughout (the reference's own layout).  Every Linear / dense conv -- embed conv (im2col), pwconv1/2,
// the head projection AND the inverse real FFT (a [n_fft, n_fft+2] windowed-IDFT matrix) -- is the persistent
// dual-operand wgmma GEMM of conv_gemm.cuh (fp32 weights and activations as bf16 hi/lo pairs).  Depthwise conv +
// LayerNorm are one kernel; overlap-add is a gather (every output sample sums its <= n_fft/hop frames), so nothing
// leaves the device and the result is deterministic.
#include "common.cuh"
#include "conv_gemm.cuh"
#include "layernorm.cuh"

#include <algorithm>
#include <cmath>

namespace b2a {
namespace vc {

typedef __nv_bfloat16 bf16;

// k-tap im2col along time (zero padded, "same"): out row (b, t) = [x[t-k/2] | ... | x[t+k/2]] as hi/lo, Kp >= k*C
__global__ void im2colk_kernel(const float* __restrict__ in, bf16* __restrict__ out, int L, int C, int k, int Kp) {
    const long long tok = blockIdx.x;
    const int b = (int)(tok / L), t = (int)(tok - (long long)b * L);
    for (int i = threadIdx.x; i < Kp; i += blockDim.x) {
        float v = 0.f;
        if (i < k * C) {
            const int kk = i / C, c = i - kk * C;
            const int ti = t + kk - k / 2;
            if (ti >= 0 && ti < L) v = in[((long long)b * L + ti) * C + c];
        }
        tc::store_hilo(out, Kp, tok, i, v, cg::HALF);
    }
}

// SopranoDecoder's interpolate1d(align_corners) x upscale (SopranoDecoder.swift:22-80, :263-275) fused into the embed conv's im2col:
// u[t] = y[lo] (1 - f) + y[hi] f, x_t = t * ((n-1)/(T-1)) in fp32 in that order, lo = floor(x_t), hi = min(lo + 1, n - 1), f = x_t - lo
// (u = y when T == n), over the n states of row rows[b] of src (row stride row_stride floats, C channels each); out row (b, t) =
// [u[t-k/2] | ... | u[t+k/2]] as hi/lo, zero padded.  The T upsampled frames never exist in memory.  Explicit _rn operations: no
// contraction into fma, the reference rounds every product.
__global__ void upsample_im2colk_kernel(const float* __restrict__ src, long long row_stride, const int* __restrict__ rows, int n, int T,
                                        bf16* __restrict__ out, int C, int k, int Kp) {
    const long long tok = blockIdx.x;
    const int b = (int)(tok / T), t = (int)(tok - (long long)b * T);
    const float* y = src + (long long)(rows ? rows[b] : b) * row_stride;
    const float scale = T > 1 ? (float)(n - 1) / (float)(T - 1) : 0.f;
    for (int i = threadIdx.x; i < Kp; i += blockDim.x) {
        float v = 0.f;
        if (i < k * C) {
            const int kk = i / C, c = i - kk * C;
            const int ti = t + kk - k / 2;
            if (ti >= 0 && ti < T) {
                if (T == n) {
                    v = y[(long long)ti * C + c];
                } else {
                    const float x = __fmul_rn((float)ti, scale);
                    const int lo = (int)floorf(x), hi = min(lo + 1, n - 1);
                    const float f = __fsub_rn(x, (float)lo);
                    v = __fadd_rn(__fmul_rn(y[(long long)lo * C + c], __fsub_rn(1.0f, f)), __fmul_rn(y[(long long)hi * C + c], f));
                }
            }
        }
        tc::store_hilo(out, Kp, tok, i, v, cg::HALF);
    }
}

constexpr int DL_MAXV = 4;    // channels <= 1024 (dw_layernorm_kernel, layernorm.cuh)

// AdaLayerNorm's conditioning (Vocos.swift:31-33): for every norm n and utterance b,  gain[n, b, :] = Ws_n cond_b + bs_n  and
// shift[n, b, :] = Wh_n cond_b + bh_n.  W [norms][dim][E] (scale then shift stacked: [2][norms][dim][E]), cond [B][E].
__global__ void adanorm_affine_kernel(const float* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ cond,
                                      float* __restrict__ out, int norms, int B, int D, int E) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // over [2][norms][B][D]
    if (i >= (long long)2 * norms * B * D) return;
    const int d = (int)(i % D), b = (int)((i / D) % B), n = (int)((i / ((long long)D * B)) % norms), which = (int)(i / ((long long)D * B * norms));
    const float* w = W + (((long long)which * norms + n) * D + d) * E;
    float acc = bias[((long long)which * norms + n) * D + d];
    for (int e = 0; e < E; ++e) acc = fmaf(w[e], cond[(long long)b * E + e], acc);
    out[i] = acc;
}

// head projection output h [tokens, n_fft+2] -> [mag*cos | mag*sin] as hi/lo (Vocos.swift:75-90): mag = min(exp(.), 100)
__global__ void spec_kernel(const float* __restrict__ h, bf16* __restrict__ out, int half, int Kp) {
    const long long tok = blockIdx.x;
    for (int i = threadIdx.x; i < Kp; i += blockDim.x) {
        float v = 0.f;
        if (i < 2 * half) {
            const int kq = i < half ? i : i - half;
            const float mag = fminf(expf(h[tok * 2 * half + kq]), 100.0f);
            float sn, cs;
            sincosf(h[tok * 2 * half + half + kq], &sn, &cs);
            v = mag * (i < half ? cs : sn);
        }
        tc::store_hilo(out, Kp, tok, i, v, cg::HALF);
    }
}

// overlap-add as a gather + window-sum normalisation + centre trim (Vocos.swift:123-160): output sample tp is OLA sample tp + trim
// (trim n_fft / 2; 0 for Soprano's untrimmed one-frame case)
__global__ void ola_kernel(const float* __restrict__ frames /*[B*L, n_fft] already windowed*/, const float* __restrict__ win,
                           float* __restrict__ wave, int L, int n_fft, int hop, int out_len, int trim) {
    const int b = blockIdx.y;
    const int tp = blockIdx.x * blockDim.x + threadIdx.x;     // trimmed index
    if (tp >= out_len) return;
    const int t = tp + trim;
    int i1 = t / hop;
    if (i1 > L - 1) i1 = L - 1;
    float acc = 0.f, ws = 0.f;
    for (int i = i1; i >= 0 && t - i * hop < n_fft; --i) {
        const int j = t - i * hop;
        acc += frames[((long long)b * L + i) * n_fft + j];
        ws += win[j];
    }
    wave[(long long)b * out_len + tp] = ws != 0.f ? acc / ws : acc;
}

using cg::TcW;

struct Block { DBuf<float> dw_w, dw_b, ln_w, ln_b, gamma, pw1_b, pw2_b; TcW pw1, pw2; };

}  // namespace vc
}  // namespace b2a

using namespace b2a;
using namespace b2a::vc;

struct b2a_vocos {
    int device;
    b2a_vocos_config cfg;
    cudaStream_t stream = nullptr;
    int num_sms = 132, kp_embed = 0, kp_spec = 0;
    TcW embed, head, idft;
    DBuf<float> embed_b, head_b;
    DBuf<float> n0_w, n0_b, nf_w, nf_b, win;
    DBuf<float> ada_w, ada_b, ada_out, cond;     // AdaLayerNorm: [2][1 + layers][dim][E] / [2][1 + layers][dim]; per-call [2][1 + layers][B][dim]
    std::vector<Block> blocks;
    // workspace
    DBuf<float> feats, h, spec, frames, wave;
    DBuf<bf16> xa, xb;

    ~b2a_vocos() { if (stream) cudaStreamDestroy(stream); }
    static long long pad64(long long n) { return (n + 63) / 64 * 64; }

    b2a_vocos(int dev, const b2a_vocos_config& c, const TensorTable& tt) : device(dev), cfg(c) {
        B2A_CHECK(c.dim % 64 == 0 && c.dim <= DL_THREADS * DL_MAXV && c.intermediate_dim % 64 == 0, B2A_ERR_INVALID_INPUT,
                  "vocos: dim / intermediate_dim must be multiples of 64 (dim <= 1024)");
        B2A_CHECK(c.n_fft % 2 == 0 && c.n_fft >= 16 && c.hop_length >= 1 && c.hop_length <= c.n_fft, B2A_ERR_INVALID_INPUT, "vocos: bad n_fft / hop_length");
        B2A_CHECK(c.input_kernel_size % 2 == 1 && c.dw_kernel_size % 2 == 1 && c.dw_kernel_size <= 15, B2A_ERR_INVALID_INPUT, "vocos: kernel sizes must be odd");
        B2A_CHECK(c.adanorm_num_embeddings >= 0 && c.adanorm_num_embeddings <= 64, B2A_ERR_INVALID_INPUT, "vocos: adanorm_num_embeddings must be in 0..64");
        require_device(dev);
        B2A_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        B2A_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
        const int D = c.dim, I = c.intermediate_dim, Cin = c.input_channels, k = c.input_kernel_size, N = c.n_fft, half = N / 2 + 1;
        auto up = [&](DBuf<float>& d, const std::string& name, int n) { std::vector<float> v = tt.f32(name, n); d.upload(v.data(), n); };
        // embed conv: MLX weight [out, k, in] is already [out, k*in + i]; pad K to a multiple of 64
        kp_embed = (int)pad64((long long)k * Cin);
        {
            std::vector<float> w = tt.f32("backbone.embed.weight", (int64_t)D * k * Cin), wp((size_t)D * kp_embed, 0.f);
            for (int o = 0; o < D; ++o) memcpy(&wp[(size_t)o * kp_embed], &w[(size_t)o * k * Cin], (size_t)k * Cin * sizeof(float));
            embed.build(wp, D, 1, kp_embed);
            up(embed_b, "backbone.embed.bias", D);
        }
        const int E = c.adanorm_num_embeddings, norms = 1 + c.num_layers;
        std::vector<float> aw, ab;
        if (E > 0) { aw.resize((size_t)2 * norms * D * E); ab.resize((size_t)2 * norms * D); }
        auto ada = [&](int n, const std::string& p) {      // AdaLayerNorm(numEmbeddings, dim): scale / shift are Linear(E -> dim) (Vocos.swift:17-47)
            const char* nm[2] = {"scale", "shift"};
            for (int w = 0; w < 2; ++w) {
                std::vector<float> W = tt.f32(p + nm[w] + ".weight", (int64_t)D * E), bv = tt.f32(p + nm[w] + ".bias", D);
                memcpy(&aw[((size_t)w * norms + n) * D * E], W.data(), W.size() * sizeof(float));
                memcpy(&ab[((size_t)w * norms + n) * D], bv.data(), bv.size() * sizeof(float));
            }
        };
        if (E > 0) ada(0, "backbone.norm.");
        else { up(n0_w, "backbone.norm.weight", D); up(n0_b, "backbone.norm.bias", D); }
        up(nf_w, "backbone.final_layer_norm.weight", D); up(nf_b, "backbone.final_layer_norm.bias", D);
        blocks.resize(c.num_layers);
        for (int l = 0; l < c.num_layers; ++l) {
            const std::string p = "backbone.convnext." + std::to_string(l) + ".";
            Block& B = blocks[l];
            up(B.dw_w, p + "dwconv.weight", D * c.dw_kernel_size);          // [dim, k, 1]
            up(B.dw_b, p + "dwconv.bias", D);
            if (E > 0) ada(1 + l, p + "norm.");
            else { up(B.ln_w, p + "norm.weight", D); up(B.ln_b, p + "norm.bias", D); }
            B.pw1.build(tt.f32(p + "pwconv1.weight", (int64_t)I * D), I, 1, D); up(B.pw1_b, p + "pwconv1.bias", I);
            B.pw2.build(tt.f32(p + "pwconv2.weight", (int64_t)D * I), D, 1, I); up(B.pw2_b, p + "pwconv2.bias", D);
            if (tt.find(p + "gamma")) up(B.gamma, p + "gamma", D);
        }
        if (E > 0) { ada_w.upload(aw.data(), aw.size()); ada_b.upload(ab.data(), ab.size()); B2A_CUDA(cudaDeviceSynchronize()); }
        head.build(tt.f32("head.out.weight", (int64_t)(N + 2) * D), N + 2, 1, D);
        up(head_b, "head.out.bias", N + 2);
        // windowed inverse real DFT as a matrix: frame[j] = w[j]/N * (Re0 + (-1)^j Re_{N/2} + 2 sum_k (Re_k cos - Im_k sin))
        kp_spec = (int)pad64(2 * half);
        {
            std::vector<float> wv(N), A((size_t)N * kp_spec, 0.f);
            for (int j = 0; j < N; ++j) wv[j] = N == 1 ? 1.f : (float)(0.5 - 0.5 * std::cos(2.0 * M_PI * j / (N - 1)));   // Vocos.swift:170-178
            for (int j = 0; j < N; ++j)
                for (int kq = 0; kq < half; ++kq) {
                    const double ang = 2.0 * M_PI * (double)((long long)j * kq % N) / N;
                    const double ck = (kq == 0 || kq == N / 2) ? 1.0 : 2.0;
                    A[(size_t)j * kp_spec + kq] = (float)(wv[j] * ck * std::cos(ang) / N);
                    A[(size_t)j * kp_spec + half + kq] = (kq == 0 || kq == N / 2) ? 0.f : (float)(-wv[j] * 2.0 * std::sin(ang) / N);
                }
            idft.build(A, N, 1, kp_spec);
            win.upload(wv.data(), N);
        }
        B2A_CUDA(cudaDeviceSynchronize());
    }

    long long out_len(int L) const { return (long long)(L - 1) * cfg.hop_length; }

    // d_feats [B, L, input_channels] fp32 (device) -> d_wave [B, (L-1)*hop]
    // d_cond [B, adanorm_num_embeddings] fp32 (device): the conditioning rows AdaLayerNorm's Linears see (one-hot bandwidth ids in the
    // reference's use); required iff the model was built with adanorm_num_embeddings > 0 (the reference fatalErrors without it)
    // up != null (Soprano): the features are up->n hidden states per row, upsampled to L = upscale (n - 1) + 1 frames inside the embed
    // conv's operand kernel (d_feats unused); L = 1 is allowed there and gives the untrimmed n_fft samples of the one-frame OLA
    struct Upsample { const float* src; long long row_stride; const int* rows; int n; };
    void decode_dev(const float* d_feats, int B, int L, float* d_wave, cudaStream_t s, const float* d_cond = nullptr, const Upsample* up = nullptr) {
        B2A_CHECK(B >= 1 && (L >= 2 || (up && L == 1)), B2A_ERR_INVALID_INPUT, "vocos decode: need at least 2 frames");
        B2A_CUDA(cudaSetDevice(device));
        const int D = cfg.dim, I = cfg.intermediate_dim, N = cfg.n_fft;
        const int E = cfg.adanorm_num_embeddings, norms = 1 + cfg.num_layers;
        B2A_CHECK((E > 0) == (d_cond != nullptr), B2A_ERR_INVALID_INPUT,
                  E > 0 ? "vocos decode: AdaLayerNorm requires bandwidthId (a conditioning row per utterance)" : "vocos decode: this model takes no conditioning");
        const float *g0 = n0_w.p, *b0 = n0_b.p;
        int bs = 0;
        if (E > 0) {
            ada_out.alloc((size_t)2 * norms * B * D);
            const long long n = (long long)2 * norms * B * D;
            adanorm_affine_kernel<<<(unsigned)cdiv(n, 256), 256, 0, s>>>(ada_w.p, ada_b.p, d_cond, ada_out.p, norms, B, D, E);
            count_launch();
            g0 = ada_out.p; b0 = ada_out.p + (size_t)norms * B * D; bs = D;
        }
        auto gain = [&](int n, const float* plain) { return E > 0 ? ada_out.p + (size_t)n * B * D : plain; };
        auto shift = [&](int n, const float* plain) { return E > 0 ? ada_out.p + ((size_t)norms + n) * B * D : plain; };
        const long long T = (long long)B * L, Tp = pad64(T);
        B2A_CHECK(T < (1ll << 30), B2A_ERR_INVALID_INPUT, "vocos decode: too many frames");
        const size_t kmax = (size_t)std::max(std::max(kp_embed, I), std::max(D, kp_spec));
        xa.alloc((size_t)2 * Tp * kmax); xb.alloc((size_t)2 * Tp * kmax);
        h.alloc((size_t)T * D); spec.alloc((size_t)T * (N + 2)); frames.alloc((size_t)T * N);
        // embed conv (im2col GEMM) -> LayerNorm -> residual stream h
        if (up)
            upsample_im2colk_kernel<<<(unsigned)T, 256, 0, s>>>(up->src, up->row_stride, up->rows, up->n, L, xa.p, cfg.input_channels,
                                                                 cfg.input_kernel_size, kp_embed);
        else
            im2colk_kernel<<<(unsigned)T, 256, 0, s>>>(d_feats, xa.p, L, cfg.input_channels, cfg.input_kernel_size, kp_embed);
        count_launch();
        {
            cg::Args a{}; a.N = (int)T; a.epi = cg::E_STORE_F32; a.bias = embed_b.p; a.x = spec.p; a.ldx = D;      // spec doubles as scratch [T, D]
            cg::launch(embed, xa.p, 2 * Tp, a, num_sms, s);
        }
        dw_layernorm_kernel<DL_MAXV><<<(unsigned)T, DL_THREADS, 0, s>>>(spec.p, nullptr, nullptr, g0, b0, h.p, nullptr, L, D, 1, 1e-6f, bs);
        count_launch();
        int li = 0;
        for (auto& Bk : blocks) {
            ++li;
            dw_layernorm_kernel<DL_MAXV><<<(unsigned)T, DL_THREADS, 0, s>>>(h.p, Bk.dw_w.p, Bk.dw_b.p, gain(li, Bk.ln_w.p), shift(li, Bk.ln_b.p), nullptr, xa.p, L, D,
                                                                   cfg.dw_kernel_size, 1e-6f, bs);
            count_launch();
            cg::Args a1{}; a1.N = (int)T; a1.epi = cg::E_STORE_HILO; a1.bias = Bk.pw1_b.p; a1.gelu = 1; a1.hl = xb.p; a1.ldh = I; a1.T = L;
            cg::launch(Bk.pw1, xa.p, 2 * Tp, a1, num_sms, s);
            cg::Args a2{}; a2.N = (int)T; a2.epi = cg::E_ADD; a2.bias = Bk.pw2_b.p; a2.x = h.p; a2.ldx = D; a2.gamma = Bk.gamma.p;      // h += gamma * pw2(...)
            cg::launch(Bk.pw2, xb.p, 2 * Tp, a2, num_sms, s);
        }
        dw_layernorm_kernel<DL_MAXV><<<(unsigned)T, DL_THREADS, 0, s>>>(h.p, nullptr, nullptr, nf_w.p, nf_b.p, nullptr, xa.p, L, D, 1, 1e-6f);
        count_launch();
        {
            cg::Args a{}; a.N = (int)T; a.epi = cg::E_STORE_F32; a.bias = head_b.p; a.x = spec.p; a.ldx = N + 2;
            cg::launch(head, xa.p, 2 * Tp, a, num_sms, s);
        }
        spec_kernel<<<(unsigned)T, 256, 0, s>>>(spec.p, xb.p, N / 2 + 1, kp_spec);
        count_launch();
        {
            cg::Args a{}; a.N = (int)T; a.epi = cg::E_STORE_F32; a.x = frames.p; a.ldx = N;
            cg::launch(idft, xb.p, 2 * Tp, a, num_sms, s);
        }
        const int ol = L == 1 ? N : (int)out_len(L);
        ola_kernel<<<dim3(cdiv(ol, 256), B), 256, 0, s>>>(frames.p, win.p, d_wave, L, N, cfg.hop_length, ol, L == 1 ? 0 : N / 2);
        count_launch();
        B2A_CUDA(cudaGetLastError());
    }
};

extern "C" {

int32_t b2a_vocos_create(int32_t device, const b2a_vocos_config* cfg, const b2a_tensor* tensors, int32_t n, b2a_vocos** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_vocos_create: null out");
        *out = nullptr;
        B2A_CHECK(cfg && tensors && n > 0, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_vocos_create: missing config or weights");
        TensorTable tt(tensors, n);
        *out = new b2a_vocos(device, *cfg, tt);
    });
}

int64_t b2a_vocos_output_length(const b2a_vocos* h, int32_t frames) { return h && frames >= 2 ? h->out_len(frames) : 0; }
void* b2a_vocos_stream(b2a_vocos* h) { return h ? (void*)h->stream : nullptr; }

int32_t b2a_vocos_decode_dev(b2a_vocos* h, const float* d_feats, int32_t B, int32_t L, float* d_wave, void* stream) {
    return guarded([&] {
        B2A_CHECK(h && d_feats && d_wave, B2A_ERR_INVALID_INPUT, "b2a_vocos_decode_dev: null argument");
        h->decode_dev(d_feats, B, L, d_wave, stream ? (cudaStream_t)stream : h->stream);
    });
}

int32_t b2a_vocos_decode(b2a_vocos* h, const float* feats, int32_t B, int32_t L, float* wave) {
    return guarded([&] {
        B2A_CHECK(h && feats && wave, B2A_ERR_INVALID_INPUT, "b2a_vocos_decode: null argument");
        B2A_CHECK(B >= 1 && L >= 2, B2A_ERR_AUDIO_DECODING_FAILED, "b2a_vocos_decode: need at least 2 frames");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        const size_t nin = (size_t)B * L * h->cfg.input_channels, nout = (size_t)B * h->out_len(L);
        h->feats.alloc(nin); h->wave.alloc(nout);
        B2A_CUDA(cudaMemcpyAsync(h->feats.p, feats, nin * sizeof(float), cudaMemcpyHostToDevice, s));
        h->decode_dev(h->feats.p, B, L, h->wave.p, s);
        B2A_CUDA(cudaMemcpyAsync(wave, h->wave.p, nout * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

int32_t b2a_vocos_decode_cond(b2a_vocos* h, const float* feats, const float* cond, int32_t B, int32_t L, float* wave) {
    return guarded([&] {
        B2A_CHECK(h && feats && wave, B2A_ERR_INVALID_INPUT, "b2a_vocos_decode_cond: null argument");
        B2A_CHECK(B >= 1 && L >= 2, B2A_ERR_AUDIO_DECODING_FAILED, "b2a_vocos_decode_cond: need at least 2 frames");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        const int E = h->cfg.adanorm_num_embeddings;
        const size_t nin = (size_t)B * L * h->cfg.input_channels, nout = (size_t)B * h->out_len(L);
        h->feats.alloc(nin); h->wave.alloc(nout);
        B2A_CUDA(cudaMemcpyAsync(h->feats.p, feats, nin * sizeof(float), cudaMemcpyHostToDevice, s));
        if (cond && E > 0) { h->cond.alloc((size_t)B * E); B2A_CUDA(cudaMemcpyAsync(h->cond.p, cond, (size_t)B * E * sizeof(float), cudaMemcpyHostToDevice, s)); }
        h->decode_dev(h->feats.p, B, L, h->wave.p, s, (cond && E > 0) ? h->cond.p : (cond ? cond : nullptr));
        B2A_CUDA(cudaMemcpyAsync(wave, h->wave.p, nout * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

int64_t b2a_vocos_upsampled_length(const b2a_vocos* h, int32_t n, int32_t upscale) {
    if (!h || n < 1 || upscale < 1) return 0;
    return n == 1 ? h->cfg.n_fft : h->out_len(upscale * (n - 1) + 1);
}

int32_t b2a_vocos_decode_upsampled_dev(b2a_vocos* h, const float* d_states, int64_t row_stride, const int32_t* d_rows, int32_t B, int32_t n,
                                       int32_t upscale, float* d_wave, void* stream) {
    return guarded([&] {
        B2A_CHECK(h && d_states && d_wave, B2A_ERR_INVALID_INPUT, "b2a_vocos_decode_upsampled_dev: null argument");
        B2A_CHECK(n >= 1 && upscale >= 1 && row_stride >= (int64_t)n * h->cfg.input_channels, B2A_ERR_INVALID_INPUT,
                  "b2a_vocos_decode_upsampled_dev: bad state count, upscale or row stride");
        const b2a_vocos::Upsample up{d_states, (long long)row_stride, d_rows, n};
        h->decode_dev(nullptr, B, upscale * (n - 1) + 1, d_wave, stream ? (cudaStream_t)stream : h->stream, nullptr, &up);
    });
}

void b2a_vocos_destroy(b2a_vocos* h) { delete h; }

}  // extern "C"
