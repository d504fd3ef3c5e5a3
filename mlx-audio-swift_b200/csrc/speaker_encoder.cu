// Qwen3-TTS speaker encoder on the device (Sources/MLXAudioTTS/Models/Qwen3TTS/Qwen3TTSSpeakerEncoder.swift, the x-vector of
// extractSpeakerEmbedding, Qwen3TTS.swift:839-881): an ECAPA-TDNN over the 1024-point log-mel of the reference clip.
//
// fp32, channels-last [B, T, C] like the other encoders.  Every conv is one ec_conv_kernel launch (seanet.cuh: implicit GEMM with
// clamped reflect padding, dilation, ReLU / tanh epilogue, and row strides so a conv reads or writes a channel slice):
//   block 0      TDNN: reflect-padded k0-tap conv mel -> C0, ReLU
//   block i      SE-Res2Net: tdnn1 (1x1, ReLU) -> h1; Res2Net sub-conv j = 1 .. scale-1 over h1[:, j] (+ h2[:, j-1] for j > 1,
//                added as the conv loads) -> h2[:, j]; tdnn2 (1x1, ReLU) reads chunk 0 straight from h1 and chunks 1.. from h2;
//                SE (mean over time, 1x1 + ReLU, 1x1 + sigmoid) scales it, plus the block input, into the block's slice of the
//                MFA input, so no concatenation is copied
//   MFA          TDNN over that concatenation
//   ASP          global mean / std per channel; the TDNN over [x; mean; std] as W_x x + (W_mu mean + W_sigma std + b), the
//                time-constant part folded into a per-clip bias; tanh; 1x1 conv; softmax over time; weighted mean / std
//   fc           1x1 conv 2 C -> enc_dim
// Reductions over time (SE mean, ASP statistics, softmax pooling) run in a fixed order without atomics, and the matrix-vector
// products in a fixed lane split and shuffle tree, so a clip's embedding is the same bit for bit in any batch.
#include "common.cuh"
#include "seanet.cuh"

#include <math.h>

#include <memory>

namespace b2a {
namespace spk {

constexpr float EPS = 1e-12f;   // AttentiveStatisticsPooling.eps
constexpr int ST_C = 32, ST_G = 8;   // channels x time groups per CTA of the reductions over time

// mode 0: out = mean_t x;  mode 1: out = sqrt(mean_t (x - mu)^2 + eps).  x [B, T, ld] (channels 0..C-1), out / mu at b * ldo + c.
// Thread (c, g) sums t = g, g + ST_G, ... in order; the ST_G partials are added in order of g.
__global__ void __launch_bounds__(ST_C * ST_G) time_stats_kernel(const float* __restrict__ x, int ld, int T, int C, int mode,
                                                                 const float* __restrict__ mu, float* __restrict__ out, int ldo) {
    __shared__ float part[ST_G][ST_C];
    const int tx = threadIdx.x % ST_C, g = threadIdx.x / ST_C, b = blockIdx.y, c = blockIdx.x * ST_C + tx;
    float acc = 0.f;
    if (c < C) {
        const float* p = x + (long long)b * T * ld + c;
        const float m = mode ? mu[(long long)b * ldo + c] : 0.f;
        for (int t = g; t < T; t += ST_G) {
            const float v = p[(long long)t * ld];
            acc += mode ? (v - m) * (v - m) : v;
        }
    }
    part[g][tx] = acc;
    __syncthreads();
    if (g == 0 && c < C) {
        float s = 0.f;
        for (int i = 0; i < ST_G; ++i) s += part[i][tx];
        s /= (float)T;
        out[(long long)b * ldo + c] = mode ? sqrtf(s + EPS) : s;
    }
}

// Attentive pooling: per channel c, w_t = softmax_t(e[t, c]); out[b, c] = sum_t w_t x_t, out[b, C + c] = sqrt(max(sum_t w_t
// (x_t - mean)^2, eps)).  x, e [B, T, C].  The same fixed (c, g) split as time_stats_kernel for the max, the normaliser and both sums.
__global__ void __launch_bounds__(ST_C * ST_G) attentive_pool_kernel(const float* __restrict__ x, const float* __restrict__ e, int T, int C,
                                                                     float* __restrict__ out) {
    __shared__ float part[ST_G][ST_C][2];
    __shared__ float fin[3][ST_C];       // max, 1 / Z, mean
    const int tx = threadIdx.x % ST_C, g = threadIdx.x / ST_C, b = blockIdx.y, c = blockIdx.x * ST_C + tx;
    const bool on = c < C;
    const long long base = (long long)b * T * C + c;
    float mx = -INFINITY;
    if (on)
        for (int t = g; t < T; t += ST_G) mx = fmaxf(mx, e[base + (long long)t * C]);
    part[g][tx][0] = mx;
    __syncthreads();
    if (g == 0) {
        float m = -INFINITY;
        for (int i = 0; i < ST_G; ++i) m = fmaxf(m, part[i][tx][0]);
        fin[0][tx] = m;
    }
    __syncthreads();
    const float m = fin[0][tx];
    float z = 0.f, s1 = 0.f;
    if (on)
        for (int t = g; t < T; t += ST_G) {
            const float w = expf(e[base + (long long)t * C] - m);
            z += w;
            s1 += w * x[base + (long long)t * C];
        }
    __syncthreads();
    part[g][tx][0] = z; part[g][tx][1] = s1;
    __syncthreads();
    if (g == 0) {
        float zz = 0.f, ss = 0.f;
        for (int i = 0; i < ST_G; ++i) { zz += part[i][tx][0]; ss += part[i][tx][1]; }
        fin[1][tx] = 1.f / zz;
        fin[2][tx] = ss / zz;
    }
    __syncthreads();
    const float inv_z = fin[1][tx], mean = fin[2][tx];
    float s2 = 0.f;
    if (on)
        for (int t = g; t < T; t += ST_G) {
            const float d = x[base + (long long)t * C] - mean;
            s2 += expf(e[base + (long long)t * C] - m) * d * d;
        }
    __syncthreads();
    part[g][tx][0] = s2;
    __syncthreads();
    if (g == 0 && on) {
        float v = 0.f;
        for (int i = 0; i < ST_G; ++i) v += part[i][tx][0];
        out[(long long)b * 2 * C + c] = mean;
        out[(long long)b * 2 * C + C + c] = sqrtf(fmaxf(v * inv_z, EPS));
    }
}

// y[b, m] = act(W[m, :K] . x[b, :K] + bias[m]), W rows at stride ldw; act 0 none, 1 ReLU, 2 sigmoid.  One warp per output: lane l
// sums k = l, l + 32, ... in order, then a fixed xor-shuffle tree.
constexpr int MV_WARPS = 8;
__global__ void __launch_bounds__(MV_WARPS * 32) matvec_kernel(const float* __restrict__ W, int ldw, const float* __restrict__ x, int ldx,
                                                               const float* __restrict__ bias, float* __restrict__ y, int ldy, int M, int K, int act) {
    const int lane = threadIdx.x & 31, m = blockIdx.x * MV_WARPS + (threadIdx.x >> 5), b = blockIdx.y;
    if (m >= M) return;
    const float* w = W + (long long)m * ldw;
    const float* xb = x + (long long)b * ldx;
    float acc = 0.f;
    for (int k = lane; k < K; k += 32) acc = fmaf(w[k], xb[k], acc);
    acc = warp_sum(acc);
    if (lane == 0) {
        float v = acc + (bias ? bias[m] : 0.f);
        if (act == 1) v = fmaxf(v, 0.f);
        else if (act == 2) v = 1.f / (1.f + expf(-v));
        y[(long long)b * ldy + m] = v;
    }
}

// SE scale + residual: out[b, t, c] (row stride ldo) = s[b, t, c] * g[b, c] + res[b, t, c] (row stride ldr); s [B, T, C] dense.
__global__ void se_residual_kernel(const float* __restrict__ s, const float* __restrict__ g, const float* __restrict__ res, int ldr,
                                   float* __restrict__ out, int ldo, long long rows, int T, int C) {
    const long long n = rows * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / C;
        const int c = (int)(i - r * C), b = (int)(r / T);
        out[r * ldo + c] = s[i] * g[(long long)b * C + c] + res[r * ldr + c];
    }
}

}  // namespace spk
}  // namespace b2a

using namespace b2a;

struct b2a_qwen3_speaker_encoder {
    int device = 0;
    b2a_qwen3_speaker_encoder_config cfg{};
    cudaStream_t stream = nullptr;
    std::unique_ptr<b2a_logmel, void (*)(b2a_logmel*)> mel{nullptr, b2a_logmel_destroy};
    struct Block {
        int C, k, d;
        ec::Conv tdnn1, tdnn2;
        std::vector<ec::Conv> res;
        DBuf<float> se1w, se1b, se2w, se2b;
    };
    int nb = 0, C3 = 0, att = 0, E = 0, scale = 1, max_pad = 0;
    ec::Conv b0, mfa, asp_x, asp_conv;     // asp_x: the x columns of the ASP TDNN [att, C3]
    DBuf<float> asp_ms, asp_b, fc_w, fc_b; // asp_ms: its [mean; std] columns [att, 2 C3]
    std::vector<Block> blocks;
    // workspaces
    DBuf<float> audio, mels, x0, h1, h2, sbuf, cat, y, a, e, stats, se_mean, se_hid, se_gate, cbias, pooled, emb;

    static void up(DBuf<float>& d, const std::vector<float>& v) { d.upload(v.data(), v.size()); }
    static void load(const TensorTable& tt, ec::Conv& cv, const std::string& p, int cout, int k, int cin) {
        cv.M = cout; cv.K = k * cin;
        up(cv.A, tt.f32(p + ".weight", (int64_t)cout * k * cin));       // MLX [out, k, in] == [M, tap * Cin + ci]
        up(cv.bias, tt.f32(p + ".bias", cout));
    }

    b2a_qwen3_speaker_encoder(int dev, const b2a_qwen3_speaker_encoder_config& c, const TensorTable& tt) : device(dev), cfg(c) {
        const int n = c.num_enc_layers;
        B2A_CHECK(c.mel_dim == 128, B2A_ERR_INVALID_INPUT, "speaker encoder: mel_dim must be 128 (the reference's mel front-end has 128 bins)");
        B2A_CHECK(n >= 3 && n <= 8, B2A_ERR_INVALID_INPUT, "speaker encoder: enc_channels must have 3 to 8 entries");
        B2A_CHECK(c.enc_res2net_scale >= 1 && c.enc_attention_channels >= 4 && c.enc_attention_channels % 4 == 0 && c.enc_se_channels >= 1 &&
                      c.enc_dim >= 1 && c.sample_rate > 0,
                  B2A_ERR_INVALID_INPUT, "speaker encoder: bad scale, attention / SE channels, enc_dim or sample_rate");
        scale = c.enc_res2net_scale;
        int sum = 0;
        for (int i = 0; i < n; ++i) {
            const int C = c.enc_channels[i], k = c.enc_kernel_sizes[i], d = c.enc_dilations[i];
            B2A_CHECK(C >= 1 && C % scale == 0 && (C / scale) % 4 == 0, B2A_ERR_INVALID_INPUT,
                      "speaker encoder: every channel count must be divisible by enc_res2net_scale into chunks of a multiple of 4 channels");
            B2A_CHECK(k >= 1 && k <= 16 && d >= 1 && ((k - 1) * d) % 2 == 0, B2A_ERR_INVALID_INPUT,
                      "speaker encoder: kernel sizes must be 1..16, dilations >= 1, and (k - 1) * d even (same-length reflect padding)");
            max_pad = std::max(max_pad, (k - 1) * d / 2);
            if (i >= 1 && i < n - 1) {
                B2A_CHECK(c.enc_channels[i - 1] == C, B2A_ERR_INVALID_INPUT, "speaker encoder: an SE-Res2Net block adds its input, so its width must not change");
                sum += C;
            }
        }
        C3 = c.enc_channels[n - 1];
        B2A_CHECK(sum == C3, B2A_ERR_INVALID_INPUT, "speaker encoder: sum(enc_channels[1:-1]) must equal enc_channels[-1] (the MFA input)");
        att = c.enc_attention_channels; E = c.enc_dim; nb = n - 2;
        require_device(dev);
        B2A_CUDA(cudaSetDevice(dev));
        load(tt, b0, "blocks.0.conv", c.enc_channels[0], c.enc_kernel_sizes[0], c.mel_dim);
        blocks.resize(nb);
        for (int i = 1; i <= nb; ++i) {
            Block& B = blocks[i - 1];
            B.C = c.enc_channels[i]; B.k = c.enc_kernel_sizes[i]; B.d = c.enc_dilations[i];
            const std::string p = "blocks." + std::to_string(i) + ".";
            const int w = B.C / scale;
            load(tt, B.tdnn1, p + "tdnn1.conv", B.C, 1, B.C);
            B.res.resize(scale - 1);
            for (int j = 0; j + 1 < scale; ++j) load(tt, B.res[j], p + "res2net_block.blocks." + std::to_string(j) + ".conv", w, B.k, w);
            load(tt, B.tdnn2, p + "tdnn2.conv", B.C, 1, B.C);
            up(B.se1w, tt.f32(p + "se_block.conv1.weight", (int64_t)c.enc_se_channels * B.C)); up(B.se1b, tt.f32(p + "se_block.conv1.bias", c.enc_se_channels));
            up(B.se2w, tt.f32(p + "se_block.conv2.weight", (int64_t)B.C * c.enc_se_channels)); up(B.se2b, tt.f32(p + "se_block.conv2.bias", B.C));
        }
        load(tt, mfa, "mfa.conv", C3, c.enc_kernel_sizes[n - 1], C3);
        {   // the ASP TDNN [att, 1, 3 C3] split into its x columns and its [mean; std] columns
            const std::vector<float> w = tt.f32("asp.tdnn.conv.weight", (int64_t)att * 3 * C3);
            std::vector<float> wx((size_t)att * C3), wms((size_t)att * 2 * C3);
            for (int m = 0; m < att; ++m) {
                std::copy(w.begin() + (size_t)m * 3 * C3, w.begin() + (size_t)m * 3 * C3 + C3, wx.begin() + (size_t)m * C3);
                std::copy(w.begin() + (size_t)m * 3 * C3 + C3, w.begin() + (size_t)(m + 1) * 3 * C3, wms.begin() + (size_t)m * 2 * C3);
            }
            asp_x.M = att; asp_x.K = C3;
            up(asp_x.A, wx); up(asp_ms, wms);
            up(asp_b, tt.f32("asp.tdnn.conv.bias", att));
        }
        load(tt, asp_conv, "asp.conv", C3, 1, att);
        up(fc_w, tt.f32("fc.weight", (int64_t)E * 2 * C3)); up(fc_b, tt.f32("fc.bias", E));
        B2A_CUDA(cudaDeviceSynchronize());
        {
            b2a_logmel* m = nullptr;
            const int32_t st = b2a_logmel_create(dev, 0, c.sample_rate, 1024, 256, 128, &m);
            if (st != B2A_OK) throw Error(st, b2a_last_error());
            mel.reset(m);
        }
        // last: a check that throws above leaves no stream behind (the destructor does not run for a half-built object)
        B2A_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    }
    ~b2a_qwen3_speaker_encoder() { if (stream) cudaStreamDestroy(stream); }

    static long long frames(long long n) { return 1 + n / 256; }

    // one reflect-padded "same" conv + epilogue: xa [B, T, Cin] rows at lda -> out rows at ldo
    void conv(const ec::Conv& w, const float* xa, int lda, int Cin, int k, int d, int B, int T, float* out, int ldo, int act,
              cudaStream_t s, const float* bias = nullptr, long long bias_n = 0) const {
        ec::ConvArgs a{};
        a.xa = xa; a.La = T; a.Ca = Cin; a.lda = lda; a.taps = k; a.dil = d; a.padL = (k - 1) * d / 2; a.reflect = 1;
        a.A = w.A.p; a.bias = bias ? bias : w.bias.p; a.bias_n = bias_n; a.M = w.M; a.K = w.K; a.Lq = T; a.N = B;
        a.out = out; a.ldo = ldo; a.out_per_n = (long long)T * ldo; a.act = act;
        ec::launch_conv(a, s);
    }
    void matvec(const float* W, int ldw, const float* x, int ldx, const float* bias, float* yv, int ldy, int M, int K, int B, int act,
                cudaStream_t s) const {
        spk::matvec_kernel<<<dim3(cdiv(M, spk::MV_WARPS), B), spk::MV_WARPS * 32, 0, s>>>(W, ldw, x, ldx, bias, yv, ldy, M, K, act);
        count_launch();
    }

    // log-mel [B, T, 128] in device memory -> embeddings [B, enc_dim]
    void forward(const float* d_mel, int B, long long T_, float* d_out, cudaStream_t s) {
        B2A_CHECK(B >= 1, B2A_ERR_INVALID_INPUT, "speaker encoder: batch must be >= 1");
        B2A_CHECK(T_ > max_pad, B2A_ERR_INVALID_INPUT,
                  "speaker encoder: too few frames for the reflect padding (need T > max((k - 1) * d / 2), i.e. at least 1024 samples at the default geometry)");
        B2A_CHECK(T_ < (1ll << 30) && (long long)B * T_ * std::max(C3, 3 * c_max()) < (1ll << 40), B2A_ERR_INVALID_INPUT, "speaker encoder: input too long");
        const int T = (int)T_;
        B2A_CUDA(cudaSetDevice(device));
        const long long rows = (long long)B * T;
        const int C0 = cfg.enc_channels[0];
        x0.alloc(rows * C0); cat.alloc(rows * C3); y.alloc(rows * C3); e.alloc(rows * C3); a.alloc(rows * att);
        h1.alloc(rows * c_max()); h2.alloc(rows * c_max()); sbuf.alloc(rows * c_max());
        stats.alloc((size_t)B * 2 * C3); pooled.alloc((size_t)B * 2 * C3); cbias.alloc((size_t)B * att);
        se_mean.alloc((size_t)B * c_max()); se_hid.alloc((size_t)B * cfg.enc_se_channels); se_gate.alloc((size_t)B * c_max());
        const dim3 st_blk(spk::ST_C * spk::ST_G);
        // block 0: TDNN mel -> C0
        conv(b0, d_mel, cfg.mel_dim, cfg.mel_dim, cfg.enc_kernel_sizes[0], cfg.enc_dilations[0], B, T, x0.p, C0, 1, s);
        const float* prev = x0.p;
        int prev_ld = C0, off = 0;
        for (const Block& Bk : blocks) {
            const int C = Bk.C, w = C / scale;
            conv(Bk.tdnn1, prev, prev_ld, C, 1, 1, B, T, h1.p, C, 1, s);
            for (int j = 1; j < scale; ++j) {          // Res2Net: out_j = TDNN_j(h1[:, j] (+ out_{j-1}))
                ec::ConvArgs r{};
                r.xa = h1.p + (size_t)j * w; r.xa_add = j > 1 ? h2.p + (size_t)(j - 1) * w : nullptr; r.lda = C; r.La = T; r.Ca = w;
                r.taps = Bk.k; r.dil = Bk.d; r.padL = (Bk.k - 1) * Bk.d / 2; r.reflect = 1;
                r.A = Bk.res[j - 1].A.p; r.bias = Bk.res[j - 1].bias.p; r.M = w; r.K = Bk.res[j - 1].K; r.Lq = T; r.N = B;
                r.out = h2.p + (size_t)j * w; r.ldo = C; r.out_per_n = (long long)T * C; r.act = 1;
                ec::launch_conv(r, s);
            }
            {   // tdnn2 over [h1[:, 0] | h2[:, 1..]]: the Res2Net's chunk 0 is its input chunk 0
                ec::ConvArgs r{};
                r.xa = h1.p; r.lda = C; r.La = T; r.Ca = w; r.taps = 1; r.reflect = 1;
                if (scale > 1) { r.xb = h2.p + w; r.Cb = C - w; r.ldb = C; }
                r.A = Bk.tdnn2.A.p; r.bias = Bk.tdnn2.bias.p; r.M = C; r.K = C; r.Lq = T; r.N = B;
                r.out = sbuf.p; r.out_per_n = (long long)T * C; r.act = 1;
                ec::launch_conv(r, s);
            }
            spk::time_stats_kernel<<<dim3(cdiv(C, spk::ST_C), B), st_blk, 0, s>>>(sbuf.p, C, T, C, 0, nullptr, se_mean.p, C);
            count_launch();
            matvec(Bk.se1w.p, C, se_mean.p, C, Bk.se1b.p, se_hid.p, cfg.enc_se_channels, cfg.enc_se_channels, C, B, 1, s);
            matvec(Bk.se2w.p, cfg.enc_se_channels, se_hid.p, cfg.enc_se_channels, Bk.se2b.p, se_gate.p, C, C, cfg.enc_se_channels, B, 2, s);
            spk::se_residual_kernel<<<(unsigned)std::min<long long>(cdiv(rows * C, 256), 4096), 256, 0, s>>>(sbuf.p, se_gate.p, prev, prev_ld,
                                                                                                           cat.p + off, C3, rows, T, C);
            count_launch();
            prev = cat.p + off; prev_ld = C3; off += C;
        }
        const int n = cfg.num_enc_layers;
        conv(mfa, cat.p, C3, C3, cfg.enc_kernel_sizes[n - 1], cfg.enc_dilations[n - 1], B, T, y.p, C3, 1, s);
        // ASP
        spk::time_stats_kernel<<<dim3(cdiv(C3, spk::ST_C), B), st_blk, 0, s>>>(y.p, C3, T, C3, 0, nullptr, stats.p, 2 * C3);
        spk::time_stats_kernel<<<dim3(cdiv(C3, spk::ST_C), B), st_blk, 0, s>>>(y.p, C3, T, C3, 1, stats.p, stats.p + C3, 2 * C3);
        count_launch(2);
        matvec(asp_ms.p, 2 * C3, stats.p, 2 * C3, asp_b.p, cbias.p, att, att, 2 * C3, B, 0, s);
        conv(asp_x, y.p, C3, C3, 1, 1, B, T, a.p, att, 2, s, cbias.p, att);
        conv(asp_conv, a.p, att, att, 1, 1, B, T, e.p, C3, 0, s);
        spk::attentive_pool_kernel<<<dim3(cdiv(C3, spk::ST_C), B), st_blk, 0, s>>>(y.p, e.p, T, C3, pooled.p);
        count_launch();
        matvec(fc_w.p, 2 * C3, pooled.p, 2 * C3, fc_b.p, d_out, E, E, 2 * C3, B, 0, s);
        B2A_CUDA(cudaGetLastError());
    }
    int c_max() const {
        int m = 0;
        for (int i = 0; i + 1 < cfg.num_enc_layers; ++i) m = std::max(m, cfg.enc_channels[i]);
        return m;
    }

    // device audio [B, n] -> device embeddings [B, enc_dim]
    void embed_dev(const float* d_audio, int B, long long n, float* d_out, cudaStream_t s) {
        B2A_CHECK(n >= 1 && B >= 1, B2A_ERR_INVALID_INPUT, "speaker encoder: empty audio");
        B2A_CHECK(n > 512, B2A_ERR_INVALID_INPUT, "speaker encoder: the 1024-point mel needs more than 512 samples");
        B2A_CHECK((long long)B * n < (1ll << 31), B2A_ERR_INVALID_INPUT, "speaker encoder: input too long");
        B2A_CHECK(frames(n) > max_pad, B2A_ERR_INVALID_INPUT,
                  "speaker encoder: too few frames for the reflect padding (need T > max((k - 1) * d / 2), i.e. at least 1024 samples at the default geometry)");
        B2A_CUDA(cudaSetDevice(device));
        const long long T = frames(n);
        mels.alloc((size_t)B * T * cfg.mel_dim);
        const int32_t st = b2a_logmel_compute_dev(mel.get(), d_audio, B, n, mels.p, s);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
        forward(mels.p, B, T, d_out, s);
    }
};

extern "C" {

int32_t b2a_qwen3_speaker_encoder_create(int32_t device, const b2a_qwen3_speaker_encoder_config* cfg, const b2a_tensor* tensors, int32_t n,
                                         b2a_qwen3_speaker_encoder** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_qwen3_speaker_encoder_create: null out");
        *out = nullptr;
        B2A_CHECK(cfg && tensors && n > 0, B2A_ERR_MODEL_NOT_INITIALIZED, "b2a_qwen3_speaker_encoder_create: missing config or weights");
        TensorTable tt(tensors, n);
        *out = new b2a_qwen3_speaker_encoder(device, *cfg, tt);
    });
}

int64_t b2a_qwen3_speaker_encoder_frames(const b2a_qwen3_speaker_encoder* h, int64_t n_samples) {
    return h ? b2a_qwen3_speaker_encoder::frames(n_samples) : 0;
}
void* b2a_qwen3_speaker_encoder_stream(b2a_qwen3_speaker_encoder* h) { return h ? (void*)h->stream : nullptr; }

int32_t b2a_qwen3_speaker_encoder_embed(b2a_qwen3_speaker_encoder* h, const float* audio, int32_t batch, int64_t n_samples, float* out) {
    return guarded([&] {
        B2A_CHECK(h && audio && out, B2A_ERR_INVALID_INPUT, "b2a_qwen3_speaker_encoder_embed: null argument");
        B2A_CHECK(batch >= 1 && n_samples >= 1 && (long long)batch * n_samples < (1ll << 31), B2A_ERR_INVALID_INPUT,
                  "speaker encoder: empty audio or input too long");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        h->audio.alloc((size_t)batch * n_samples); h->emb.alloc((size_t)batch * h->E);
        B2A_CUDA(cudaMemcpyAsync(h->audio.p, audio, (size_t)batch * n_samples * sizeof(float), cudaMemcpyHostToDevice, s));
        h->embed_dev(h->audio.p, batch, n_samples, h->emb.p, s);
        B2A_CUDA(cudaMemcpyAsync(out, h->emb.p, (size_t)batch * h->E * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

int32_t b2a_qwen3_speaker_encoder_embed_dev(b2a_qwen3_speaker_encoder* h, const float* d_audio, int32_t batch, int64_t n_samples,
                                            float* d_out, void* stream) {
    return guarded([&] {
        B2A_CHECK(h && d_audio && d_out, B2A_ERR_INVALID_INPUT, "b2a_qwen3_speaker_encoder_embed_dev: null argument");
        h->embed_dev(d_audio, batch, n_samples, d_out, stream ? (cudaStream_t)stream : h->stream);
    });
}

int32_t b2a_qwen3_speaker_encoder_embed_mel(b2a_qwen3_speaker_encoder* h, const float* mel, int32_t batch, int64_t frames, float* out) {
    return guarded([&] {
        B2A_CHECK(h && mel && out, B2A_ERR_INVALID_INPUT, "b2a_qwen3_speaker_encoder_embed_mel: null argument");
        B2A_CHECK(batch >= 1 && frames >= 1 && (long long)batch * frames < (1ll << 31), B2A_ERR_INVALID_INPUT,
                  "speaker encoder: empty mel or input too long");
        B2A_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = h->stream;
        const size_t nm = (size_t)batch * frames * h->cfg.mel_dim;
        h->mels.alloc(nm); h->emb.alloc((size_t)batch * h->E);
        B2A_CUDA(cudaMemcpyAsync(h->mels.p, mel, nm * sizeof(float), cudaMemcpyHostToDevice, s));
        h->forward(h->mels.p, batch, frames, h->emb.p, s);
        B2A_CUDA(cudaMemcpyAsync(out, h->emb.p, (size_t)batch * h->E * sizeof(float), cudaMemcpyDeviceToHost, s));
        B2A_CUDA(cudaStreamSynchronize(s));
    });
}

void b2a_qwen3_speaker_encoder_destroy(b2a_qwen3_speaker_encoder* h) { delete h; }

}  // extern "C"
