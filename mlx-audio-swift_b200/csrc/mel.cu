// Log-mel front-end for sm_90a: STFT(400 or 1024) -> power -> mel filterbank -> log10 in ONE kernel,
// plus the elementwise max-8 clamp pass.  Replaces (reference paths):
//   Sources/MLXAudioCore/DSP.swift:15-22,76-168,181-273
//   Sources/MLXAudioSTT/Streaming/IncrementalMelSpectrogram.swift:18-208
//   Sources/MLXAudioSTT/Models/Whisper/WhisperAudio.swift:7-120
//
// Data layout in HBM: PCM float32 [B, n] (read once, coalesced, staged per CTA in shared memory),
// log-mel float32 [B, F, n_mels] (written once by kernel 1, clamped in place by kernel 2).
// The 400-point real DFT is done as a 20x20 Cooley-Tukey split in shared memory (two passes of
// 20-point DFTs with a twiddle in between, exploiting conjugate symmetry of the real input; every
// 20-point transform is a folded real-input DFT, real_dft20: 10 FMAs per output); the 1024-point DFT (the Qwen3-TTS speaker
// encoder's front-end) is the same kernel split 32x32 with real_dft32.  The filterbank is applied in its sparse (contiguous-support)
// form.
#include "common.cuh"

#include <math.h>

namespace b2a {

// ------------------------------------------------------------------------------------------------
// Host tables -- Float arithmetic in the same order as the Swift code.
// ------------------------------------------------------------------------------------------------
static void hanning_window_host(int size, bool periodic, float* out) {
    // DSP.swift:15-22 (symmetric, /(N-1)); WhisperAudio.swift:42-43 (periodic, /N)
    const float denom = periodic ? (float)size : (float)(size - 1);
    for (int n = 0; n < size; ++n) out[n] = 0.5f * (1.0f - cosf(2.0f * (float)M_PI * (float)n / denom));
}

static void mel_filters_host(int sr, int n_fft, int n_mels, float f_min, float f_max, bool slaney_norm,
                             int mel_scale, float* out) {
    // DSP.swift:76-168
    const float f_max_val = f_max >= 0 ? f_max : (float)sr / 2.0f;
    const int n_freqs = n_fft / 2 + 1;
    std::vector<float> all_freqs(n_freqs);
    for (int i = 0; i < n_freqs; ++i) all_freqs[i] = (float)i * (float)sr / (float)n_fft;
    const float f_sp = 200.0f / 3.0f, min_log_hz = 1000.0f;
    const float min_log_mel = (min_log_hz - f_min) / f_sp;
    const float log_step = logf(6.4f) / 27.0f;
    auto hz_to_mel = [&](float f) -> float {
        if (mel_scale == 0) return 2595.0f * log10f(1.0f + f / 700.0f);
        return f < min_log_hz ? (f - f_min) / f_sp : min_log_mel + logf(f / min_log_hz) / log_step;
    };
    auto mel_to_hz = [&](float m) -> float {
        if (mel_scale == 0) return 700.0f * (powf(10.0f, m / 2595.0f) - 1.0f);
        return m < min_log_mel ? f_min + f_sp * m : min_log_hz * expf(log_step * (m - min_log_mel));
    };
    const float m_min = hz_to_mel(f_min), m_max = hz_to_mel(f_max_val);
    std::vector<float> f_pts(n_mels + 2);
    for (int i = 0; i < n_mels + 2; ++i) f_pts[i] = mel_to_hz(m_min + (float)i * (m_max - m_min) / (float)(n_mels + 1));
    for (int i = 0; i < n_freqs; ++i)
        for (int j = 0; j < n_mels; ++j) {
            const float low = f_pts[j], center = f_pts[j + 1], high = f_pts[j + 2], fr = all_freqs[i];
            float v = 0.f;
            if (fr >= low && fr < center) v = (fr - low) / (center - low);
            else if (fr >= center && fr <= high) v = (high - fr) / (high - center);
            out[(size_t)i * n_mels + j] = v;
        }
    if (slaney_norm)
        for (int j = 0; j < n_mels; ++j) {
            const float enorm = 2.0f / (f_pts[j + 2] - f_pts[j]);
            for (int i = 0; i < n_freqs; ++i) out[(size_t)i * n_mels + j] *= enorm;
        }
}

// ------------------------------------------------------------------------------------------------
// Device side
// ------------------------------------------------------------------------------------------------
// The kernel is a template on the radix R of the R x R split: R = 20 (n_fft 400) or 32 (n_fft 1024).  FR frames per CTA; R
// threads per frame in the DFT passes.  FR = 4 at R = 32 keeps the static shared memory below 48 KB.
template <int R> struct MelGeom {
    static constexpr int NFFT = R * R, NBINS = NFFT / 2 + 1, K1N = R / 2 + 1, FR = R == 20 ? 10 : 4;
};
constexpr int MEL_THREADS = 256;

// exp(-2*pi*i*j/20) = (C20[j], S20[j]): with both DFT loops fully unrolled every twiddle index is a compile-time constant, so the
// 20-point sums are pure FMAs against immediates (the first version spent ~10 instructions per term on index arithmetic and
// shared-memory twiddle loads)
__device__ constexpr float C20[20] = {1.f, 0.95105654f, 0.809017003f, 0.587785244f, 0.309017003f, 6.12323426e-17f, -0.309017003f,
                                      -0.587785244f, -0.809017003f, -0.95105654f, -1.f, -0.95105654f, -0.809017003f, -0.587785244f,
                                      -0.309017003f, -1.83697015e-16f, 0.309017003f, 0.587785244f, 0.809017003f, 0.95105654f};
__device__ constexpr float S20[20] = {-0.f, -0.309017003f, -0.587785244f, -0.809017003f, -0.95105654f, -1.f, -0.95105654f, -0.809017003f,
                                      -0.587785244f, -0.309017003f, -1.22464685e-16f, 0.309017003f, 0.587785244f, 0.809017003f,
                                      0.95105654f, 1.f, 0.95105654f, 0.809017003f, 0.587785244f, 0.309017003f};

// Forward 20-point DFT of a REAL sequence, outputs k = 0..10, with the input folded twice (x[n] +- x[20-n], then n <-> 10-n, whose
// cosine / sine differ by the sign (-1)^k): 10 FMAs per output instead of 40.  Fully unrolled: every twiddle is an immediate.
//   re[k] = x0 + (-1)^k x10 + a5 cos(pi k / 2) + sum_{n=1..4} (a[n] + (-1)^k a[10-n]) cos(2 pi n k / 20),    a[n] = x[n] + x[20-n]
//   im[k] =                   d5 S20[5k]       + sum_{n=1..4} (d[n] - (-1)^k d[10-n]) S20[n k],              d[n] = x[n] - x[20-n]
__device__ __forceinline__ void real_dft20(const float (&x)[20], float (&re)[11], float (&im)[11]) {
    constexpr int R = 20, K1N = 11;
    float a[10], d[10];
#pragma unroll
    for (int n = 1; n < 10; ++n) { a[n] = x[n] + x[R - n]; d[n] = x[n] - x[R - n]; }
    float ee[5], eo[5], de[5], dd[5];
#pragma unroll
    for (int n = 1; n < 5; ++n) { ee[n] = a[n] + a[10 - n]; eo[n] = a[n] - a[10 - n]; de[n] = d[n] - d[10 - n]; dd[n] = d[n] + d[10 - n]; }
    const float b_even = x[0] + x[10], b_odd = x[0] - x[10];
#pragma unroll
    for (int k = 0; k < K1N; ++k) {
        const bool ev = (k & 1) == 0;
        float r = fmaf(a[5], C20[(5 * k) % R], ev ? b_even : b_odd);
        float i = d[5] * S20[(5 * k) % R];
#pragma unroll
        for (int n = 1; n < 5; ++n) {
            r = fmaf(ev ? ee[n] : eo[n], C20[(n * k) % R], r);
            i = fmaf(ev ? de[n] : dd[n], S20[(n * k) % R], i);
        }
        re[k] = r; im[k] = i;
    }
}

// exp(-2*pi*i*j/32) = (C32[j], S32[j])
__device__ constexpr float C32[32] = {1.f, 0.980785251f, 0.923879504f, 0.831469595f, 0.707106769f, 0.555570245f, 0.382683426f, 0.195090324f,
                                      6.12323426e-17f, -0.195090324f, -0.382683426f, -0.555570245f, -0.707106769f, -0.831469595f, -0.923879504f,
                                      -0.980785251f, -1.f, -0.980785251f, -0.923879504f, -0.831469595f, -0.707106769f, -0.555570245f,
                                      -0.382683426f, -0.195090324f, -1.83697015e-16f, 0.195090324f, 0.382683426f, 0.555570245f, 0.707106769f,
                                      0.831469595f, 0.923879504f, 0.980785251f};
__device__ constexpr float S32[32] = {-0.f, -0.195090324f, -0.382683426f, -0.555570245f, -0.707106769f, -0.831469595f, -0.923879504f,
                                      -0.980785251f, -1.f, -0.980785251f, -0.923879504f, -0.831469595f, -0.707106769f, -0.555570245f,
                                      -0.382683426f, -0.195090324f, -1.22464685e-16f, 0.195090324f, 0.382683426f, 0.555570245f, 0.707106769f,
                                      0.831469595f, 0.923879504f, 0.980785251f, 1.f, 0.980785251f, 0.923879504f, 0.831469595f, 0.707106769f,
                                      0.555570245f, 0.382683426f, 0.195090324f};

// Forward 32-point DFT of a REAL sequence, outputs k = 0..16, folded as real_dft20 is (x[n] +- x[32-n], then n <-> 16-n):
//   re[k] = x0 + (-1)^k x16 + a8 cos(pi k / 2) + sum_{n=1..7} (a[n] + (-1)^k a[16-n]) cos(2 pi n k / 32)
//   im[k] =                   d8 S32[8k]       + sum_{n=1..7} (d[n] - (-1)^k d[16-n]) S32[n k]
__device__ __forceinline__ void real_dft32(const float (&x)[32], float (&re)[17], float (&im)[17]) {
    constexpr int R = 32, K1N = 17;
    float a[16], d[16];
#pragma unroll
    for (int n = 1; n < 16; ++n) { a[n] = x[n] + x[R - n]; d[n] = x[n] - x[R - n]; }
    float ee[8], eo[8], de[8], dd[8];
#pragma unroll
    for (int n = 1; n < 8; ++n) { ee[n] = a[n] + a[16 - n]; eo[n] = a[n] - a[16 - n]; de[n] = d[n] - d[16 - n]; dd[n] = d[n] + d[16 - n]; }
    const float b_even = x[0] + x[16], b_odd = x[0] - x[16];
#pragma unroll
    for (int k = 0; k < K1N; ++k) {
        const bool ev = (k & 1) == 0;
        float r = fmaf(a[8], C32[(8 * k) % R], ev ? b_even : b_odd);
        float i = d[8] * S32[(8 * k) % R];
#pragma unroll
        for (int n = 1; n < 8; ++n) {
            r = fmaf(ev ? ee[n] : eo[n], C32[(n * k) % R], r);
            i = fmaf(ev ? de[n] : dd[n], S32[(n * k) % R], i);
        }
        re[k] = r; im[k] = i;
    }
}

__device__ __forceinline__ void real_dft(const float (&x)[20], float (&re)[11], float (&im)[11]) { real_dft20(x, re, im); }
__device__ __forceinline__ void real_dft(const float (&x)[32], float (&re)[17], float (&im)[17]) { real_dft32(x, re, im); }

struct MelTables {          // device pointers, owned by MelCore
    const float* window;    // [n_fft]
    const float2* tw20;     // [R]     exp(-2*pi*i*j/R)
    const float2* tw400;    // [n_fft] exp(-2*pi*i*j/n_fft)
    const int* fb_start;    // [n_mels] first bin of the filter's support
    const int* fb_count;    // [n_mels]
    const int* fb_off;      // [n_mels] offset into fb_w
    const float* fb_w;      // packed non-zero weights
    int n_mels;
};

__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
    if (v >= 0.f) atomicMax((int*)addr, __float_as_int(v));
    else atomicMin((unsigned int*)addr, __float_as_uint(v));
}

// pad_mode 0: frames index the signal directly.  pad_mode 1: centred STFT -- the signal is
// virtually reflect-padded by NFFT/2 on both sides and zero-extended from n_valid to n_total
// (WhisperAudio.padOrTrimToWindow + reflectPad; DSP.stft reflect branch).
template <int R>
__global__ void __launch_bounds__(MEL_THREADS)
mel_log_kernel(const float* __restrict__ pcm, long long pcm_stride, long long n_valid, long long n_total,
               int pad_mode, int hop, int n_frames, MelTables tb, float* __restrict__ out,
               float* __restrict__ max_buf) {
    constexpr int NFFT = MelGeom<R>::NFFT, NBINS = MelGeom<R>::NBINS, K1N = MelGeom<R>::K1N, FR = MelGeom<R>::FR;
    __shared__ float s_x[(FR - 1) * 160 + NFFT + 8 + (FR - 1) * 96];  // sized for hop <= 256
    __shared__ float s_win[NFFT];
    __shared__ float2 s_tw[K1N][R];                 // tw400[n2 * k1] as [k1][n2]: the R threads of a frame read consecutive entries
    __shared__ float2 s_y[FR][K1N][R + 1];          // + 1: the rows k1 of pass 2's readers fall into different banks
    __shared__ float s_p[FR][NBINS + 3];
    __shared__ float s_red[MEL_THREADS / 32];

    const int b = blockIdx.y;
    const int f0 = blockIdx.x * FR;
    const int nf = min(FR, n_frames - f0);
    const int tid = threadIdx.x;
    const float* sig = pcm + (long long)b * pcm_stride;

    for (int i = tid; i < NFFT; i += MEL_THREADS) s_win[i] = tb.window[i];
    for (int i = tid; i < K1N * R; i += MEL_THREADS) s_tw[i / R][i % R] = tb.tw400[(i % R) * (i / R)];
    const int span = (nf - 1) * hop + NFFT;
    const long long base = (long long)f0 * hop;
    for (int i = tid; i < span; i += MEL_THREADS) {
        long long j = base + i;
        float v = 0.f;
        if (pad_mode == 1) {
            j -= NFFT / 2;
            if (j < 0) j = -j;
            if (j >= n_total) j = 2 * (n_total - 1) - j;
            if (j >= 0 && j < n_valid) v = sig[j];
        } else if (j < n_valid) {
            v = sig[j];
        }
        s_x[i] = v;
    }
    __syncthreads();

    // pass 1: Y[k1][n2] = tw400[n2*k1] * sum_n1 xw[R*n1+n2] * tw20[(n1*k1)%R], k1 = 0..R/2.  One thread per (frame, n2): its R
    // windowed samples live in registers and feed all R/2+1 k1 sums.
    for (int o = tid; o < nf * R; o += MEL_THREADS) {
        const int f = o / R, n2 = o - f * R;
        const float* x = s_x + f * hop + n2;
        float xr[R];
#pragma unroll
        for (int n1 = 0; n1 < R; ++n1) xr[n1] = x[R * n1] * s_win[R * n1 + n2];
        float re[K1N], im[K1N];
        real_dft(xr, re, im);
#pragma unroll
        for (int k1 = 0; k1 < K1N; ++k1) {
            const float2 w = s_tw[k1][n2];
            s_y[f][k1][n2] = make_float2(re[k1] * w.x - im[k1] * w.y, re[k1] * w.y + im[k1] * w.x);
        }
    }
    __syncthreads();

    // pass 2: X[k1+R*k2] = sum_n2 Y[k1][n2] tw20[(n2*k2)%R]; for k1 > R/2, Y[k1][n2] = conj(Y[R-k1][n2]) * tw20[n2] (real input),
    // i.e. X[k1+R*k2] = T[k2+1] with T[kk] = sum_n2 conj(Y[R-k1][n2]) tw20[(n2*kk)%R].  One thread per (frame, k1): it loads its
    // row of Y once and evaluates T[0..R/2] against compile-time twiddles.
    for (int o = tid; o < nf * R; o += MEL_THREADS) {
        const int f = o / R, k1 = o - f * R;
        const bool mirror = k1 > R / 2;
        const float2* y = s_y[f][mirror ? R - k1 : k1];
        const float sgn = mirror ? -1.f : 1.f;
        float yr[R], yi[R];
#pragma unroll
        for (int n2 = 0; n2 < R; ++n2) { const float2 v = y[n2]; yr[n2] = v.x; yi[n2] = sgn * v.y; }
        // DFT(yr + i yi) = DFT(yr) + i DFT(yi): two real-input transforms
        float ra[K1N], ia[K1N], rb[K1N], ib[K1N];
        real_dft(yr, ra, ia);
        real_dft(yi, rb, ib);
#pragma unroll
        for (int kk = 0; kk < K1N; ++kk) {
            const float re = ra[kk] - ib[kk], im = ia[kk] + rb[kk];
            const int k2 = mirror ? kk - 1 : kk;
            const int k = k1 + R * k2;
            if (k2 >= 0 && k < NBINS) s_p[f][k] = re * re + im * im;
        }
    }
    __syncthreads();

    // mel filterbank (sparse, contiguous support) -> max(.,1e-10) -> log10 ; track the max
    float lmax = -INFINITY;
    const int nm = tb.n_mels;
    for (int o = tid; o < nf * nm; o += MEL_THREADS) {
        const int f = o / nm, m = o - f * nm;
        const int s = tb.fb_start[m], c = tb.fb_count[m];
        const float* w = tb.fb_w + tb.fb_off[m];
        float acc = 0.f;
        for (int j = 0; j < c; ++j) acc = fmaf(s_p[f][s + j], w[j], acc);
        const float lv = log10f(fmaxf(acc, 1e-10f));
        out[((long long)b * n_frames + f0 + f) * nm + m] = lv;
        lmax = fmaxf(lmax, lv);
    }
    for (int off = 16; off; off >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, off));
    if ((tid & 31) == 0) s_red[tid >> 5] = lmax;
    __syncthreads();
    if (tid == 0) {
        for (int i = 1; i < MEL_THREADS / 32; ++i) lmax = fmaxf(lmax, s_red[i]);
        if (lmax > -INFINITY) atomic_max_float(max_buf + b, lmax);
    }
}

// (max(x, max_b - 8) + 4) / 4  in place  (IncrementalMelSpectrogram.swift:142-143, DSP.swift:267-269)
__global__ void mel_clamp_kernel(float* __restrict__ x, long long per_clip, const float* __restrict__ max_buf) {
    const int b = blockIdx.y;
    const float floor_v = max_buf[b] - 8.0f;
    float* p = x + (long long)b * per_clip;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_clip;
         i += (long long)gridDim.x * blockDim.x)
        p[i] = (fmaxf(p[i], floor_v) + 4.0f) / 4.0f;
}

__global__ void fill_kernel(float* p, int n, float v) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// ------------------------------------------------------------------------------------------------
// MelCore: tables + launches shared by the streaming and the batched front-ends
// ------------------------------------------------------------------------------------------------
struct MelCore {
    int device, sr, n_fft, hop, n_mels;
    DBuf<float> d_window, d_fbw;
    DBuf<float2> d_tw20, d_tw400;
    DBuf<int> d_start, d_count, d_off;
    MelTables tb{};

    MelCore(int device_, int sr_, int n_fft_, int hop_, int n_mels_, bool periodic, int mel_scale)
        : device(device_), sr(sr_), n_fft(n_fft_), hop(hop_), n_mels(n_mels_) {
        B2A_CHECK(n_fft == 400 || n_fft == 1024, B2A_ERR_INVALID_INPUT, "only n_fft == 400 or 1024 is implemented on the device path");
        B2A_CHECK(hop > 0 && hop <= 256, B2A_ERR_INVALID_INPUT, "hop_length must be in 1..256");
        B2A_CHECK(n_mels > 0 && n_mels <= 512, B2A_ERR_INVALID_INPUT, "n_mels must be in 1..512");
        require_device(device);
        const int R = n_fft == 400 ? 20 : 32, NBINS = n_fft / 2 + 1;
        std::vector<float> win(n_fft), fb((size_t)NBINS * n_mels);
        hanning_window_host(n_fft, periodic, win.data());
        mel_filters_host(sr, n_fft, n_mels, 0.f, -1.f, true, mel_scale, fb.data());
        std::vector<int> start(n_mels), count(n_mels), off(n_mels);
        std::vector<float> w;
        for (int m = 0; m < n_mels; ++m) {
            int lo = -1, hi = -1;
            for (int k = 0; k < NBINS; ++k)
                if (fb[(size_t)k * n_mels + m] != 0.f) { if (lo < 0) lo = k; hi = k; }
            start[m] = lo < 0 ? 0 : lo;
            count[m] = lo < 0 ? 0 : hi - lo + 1;
            off[m] = (int)w.size();
            for (int k = 0; k < count[m]; ++k) w.push_back(fb[(size_t)(start[m] + k) * n_mels + m]);
        }
        if (w.empty()) w.push_back(0.f);
        std::vector<float2> t20(R), t400(n_fft);
        for (int j = 0; j < R; ++j) t20[j] = make_float2((float)cos(2.0 * M_PI * j / R), (float)-sin(2.0 * M_PI * j / R));
        for (int j = 0; j < n_fft; ++j) t400[j] = make_float2((float)cos(2.0 * M_PI * j / n_fft), (float)-sin(2.0 * M_PI * j / n_fft));
        d_window.upload(win.data(), n_fft);
        d_fbw.upload(w.data(), w.size());
        d_tw20.upload(t20.data(), R);
        d_tw400.upload(t400.data(), n_fft);
        d_start.upload(start.data(), n_mels);
        d_count.upload(count.data(), n_mels);
        d_off.upload(off.data(), n_mels);
        B2A_CUDA(cudaDeviceSynchronize());
        tb = MelTables{d_window.p, d_tw20.p, d_tw400.p, d_start.p, d_count.p, d_off.p, d_fbw.p, n_mels};
    }

    // log-mel of `batch` clips; max_buf[b] must already hold the running max (or -inf).
    void launch(const float* d_pcm, long long stride, long long n_valid, long long n_total, int pad_mode,
                int batch, int n_frames, float* d_out, float* d_max, cudaStream_t s) const {
        if (n_frames <= 0 || batch <= 0) return;
        if (n_fft == 400) {
            dim3 grid(cdiv(n_frames, MelGeom<20>::FR), batch);
            mel_log_kernel<20><<<grid, MEL_THREADS, 0, s>>>(d_pcm, stride, n_valid, n_total, pad_mode, hop, n_frames,
                                                            tb, d_out, d_max);
        } else {
            dim3 grid(cdiv(n_frames, MelGeom<32>::FR), batch);
            mel_log_kernel<32><<<grid, MEL_THREADS, 0, s>>>(d_pcm, stride, n_valid, n_total, pad_mode, hop, n_frames,
                                                            tb, d_out, d_max);
        }
        const long long per_clip = (long long)n_frames * n_mels;
        dim3 g2((unsigned)std::min<long long>(cdiv(per_clip, 256), 1024), batch);
        mel_clamp_kernel<<<g2, 256, 0, s>>>(d_out, per_clip, d_max);
        count_launch(2);
        B2A_CUDA(cudaGetLastError());
    }
};

}  // namespace b2a

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
using namespace b2a;

struct b2a_mel {
    MelCore core;
    cudaStream_t stream = nullptr;
    std::vector<float> overlap;  // IncrementalMelSpectrogram.swift:33
    bool is_first = true;        // :36
    long long total_frames = 0;  // :41
    DBuf<float> d_sig, d_out, d_max;  // d_max = runningLogMax (:39), lives on the device
    HBuf<float> h_sig, h_out;
    b2a_mel(int dev, int sr, int nfft, int hop, int nmels) : core(dev, sr, nfft, hop, nmels, false, 0) {
        B2A_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        d_max.alloc(1);
        reset();
    }
    ~b2a_mel() { if (stream) cudaStreamDestroy(stream); }
    void reset() {
        overlap.clear();
        is_first = true;
        total_frames = 0;
        B2A_CUDA(cudaSetDevice(core.device));
        fill_kernel<<<1, 32, 0, stream>>>(d_max.p, 1, -INFINITY);
        count_launch();
        B2A_CUDA(cudaStreamSynchronize(stream));
    }
    // runs the device pipeline over `signal`, copies [n_frames, n_mels] to `out`
    void emit(const std::vector<float>& signal, int n_frames, float* out) {
        B2A_CUDA(cudaSetDevice(core.device));
        const size_t n_out = (size_t)n_frames * core.n_mels;
        h_sig.alloc(signal.size());
        d_sig.alloc(signal.size());
        h_out.alloc(n_out);
        d_out.alloc(n_out);
        memcpy(h_sig.p, signal.data(), signal.size() * sizeof(float));
        B2A_CUDA(cudaMemcpyAsync(d_sig.p, h_sig.p, signal.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
        core.launch(d_sig.p, 0, (long long)signal.size(), (long long)signal.size(), 0, 1, n_frames, d_out.p,
                    d_max.p, stream);
        B2A_CUDA(cudaMemcpyAsync(h_out.p, d_out.p, n_out * sizeof(float), cudaMemcpyDeviceToHost, stream));
        B2A_CUDA(cudaStreamSynchronize(stream));
        memcpy(out, h_out.p, n_out * sizeof(float));
        total_frames += n_frames;
    }
};

extern "C" {

int32_t b2a_hanning_window(int32_t size, int32_t periodic, float* out) {
    return guarded([&] {
        B2A_CHECK(size > 1 && out, B2A_ERR_INVALID_INPUT, "b2a_hanning_window: size must be > 1");
        hanning_window_host(size, periodic != 0, out);
    });
}

int32_t b2a_mel_filters(int32_t sr, int32_t n_fft, int32_t n_mels, float f_min, float f_max, int32_t norm_slaney,
                        int32_t mel_scale, float* out) {
    return guarded([&] {
        B2A_CHECK(sr > 0 && n_fft > 0 && n_mels > 0 && out && (mel_scale == 0 || mel_scale == 1),
                  B2A_ERR_INVALID_INPUT, "b2a_mel_filters: bad arguments");
        mel_filters_host(sr, n_fft, n_mels, f_min, f_max, norm_slaney != 0, mel_scale, out);
    });
}

int32_t b2a_mel_create(int32_t device, int32_t sr, int32_t n_fft, int32_t hop, int32_t n_mels, b2a_mel** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_mel_create: null out");
        *out = nullptr;
        B2A_CHECK(n_fft > hop, B2A_ERR_INVALID_INPUT, "b2a_mel_create: n_fft must exceed hop_length");
        *out = new b2a_mel(device, sr, n_fft, hop, n_mels);
    });
}

int64_t b2a_mel_max_frames(const b2a_mel* h, int64_t n_samples) {
    if (!h) return 0;
    // prefix (n_fft/2) or overlap (n_fft-hop, possibly a whole short signal) plus the new samples
    return (n_samples + 2 * h->core.n_fft) / h->core.hop + 2;
}

int32_t b2a_mel_process(b2a_mel* h, const float* samples, int64_t n, float* out, int64_t cap, int64_t* n_frames) {
    return guarded([&] {
        B2A_CHECK(h && n_frames, B2A_ERR_INVALID_INPUT, "b2a_mel_process: null handle");
        *n_frames = 0;
        if (n <= 0) return;  // guard !samples.isEmpty (:69)
        B2A_CHECK(samples, B2A_ERR_INVALID_INPUT, "b2a_mel_process: null samples");
        const int nfft = h->core.n_fft, hop = h->core.hop, ov = nfft - hop;
        std::vector<float> signal;
        if (h->is_first) {  // :72-95 reflect prefix of n_fft/2 samples
            const int pad = nfft / 2;
            std::vector<float> prefix;
            if (n > 1) {
                const int64_t rl = std::min<int64_t>(pad, n - 1);
                for (int64_t i = rl; i >= 1; --i) prefix.push_back(samples[i]);
            }
            if (prefix.empty()) prefix.assign(pad, samples[0]);
            else while ((int)prefix.size() < pad) {
                const size_t needed = pad - prefix.size(), have = prefix.size();
                for (size_t i = 0; i < std::min(needed, have); ++i) prefix.push_back(prefix[i]);
            }
            signal = prefix;
            h->is_first = false;
        } else {
            signal = h->overlap;  // :98
        }
        signal.insert(signal.end(), samples, samples + n);
        const int64_t sz = (int64_t)signal.size();
        const int64_t nf = sz >= nfft ? (sz - nfft) / hop + 1 : 0;
        if (nf <= 0) { h->overlap = signal; return; }  // :103-107
        B2A_CHECK(out && cap >= nf, B2A_ERR_INVALID_INPUT, "b2a_mel_process: output buffer too small");
        const int64_t consumed = (nf - 1) * hop + nfft;  // :110-115
        if (consumed < sz) h->overlap.assign(signal.begin() + (consumed - ov), signal.end());
        else h->overlap.assign(signal.end() - std::min<int64_t>(ov, sz), signal.end());
        h->emit(signal, (int)nf, out);
        *n_frames = nf;
    });
}

int32_t b2a_mel_flush(b2a_mel* h, float* out, int64_t cap, int64_t* n_frames) {
    return guarded([&] {
        B2A_CHECK(h && n_frames, B2A_ERR_INVALID_INPUT, "b2a_mel_flush: null handle");
        *n_frames = 0;
        if (h->overlap.empty()) return;  // :152
        const int nfft = h->core.n_fft, hop = h->core.hop;
        std::vector<float> signal = h->overlap;
        if ((int)signal.size() < nfft) signal.resize(nfft, 0.f);  // :155-159
        const int64_t len = (int64_t)signal.size(), pad = nfft / 2;
        const int64_t rl = std::min<int64_t>(pad, len - 1);  // :162-166 reflect suffix
        for (int64_t i = len - 2; i >= len - 1 - rl; --i) signal.push_back(signal[i]);
        h->overlap.clear();
        const int64_t sz = (int64_t)signal.size();
        const int64_t nf = sz >= nfft ? (sz - nfft) / hop + 1 : 0;
        if (nf <= 0) return;
        B2A_CHECK(out && cap >= nf, B2A_ERR_INVALID_INPUT, "b2a_mel_flush: output buffer too small");
        h->emit(signal, (int)nf, out);
        *n_frames = nf;
    });
}

int32_t b2a_mel_reset(b2a_mel* h) {
    return guarded([&] {
        B2A_CHECK(h, B2A_ERR_INVALID_INPUT, "b2a_mel_reset: null handle");
        h->reset();
    });
}

int64_t b2a_mel_total_frames(const b2a_mel* h) { return h ? h->total_frames : 0; }
void b2a_mel_destroy(b2a_mel* h) { delete h; }

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// Batched offline front-end
// ------------------------------------------------------------------------------------------------
struct b2a_logmel {
    MelCore core;
    int kind;
    cudaStream_t stream = nullptr;
    DBuf<float> d_pcm, d_out, d_max;
    b2a_logmel(int dev, int kind_, int sr, int nfft, int hop, int nmels)
        : core(dev, sr, nfft, hop, nmels, kind_ == 1, kind_ == 1 ? 1 : 0), kind(kind_) {
        B2A_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    }
    ~b2a_logmel() { if (stream) cudaStreamDestroy(stream); }
    long long frames(long long n) const {
        if (kind == 1) return 480000 / core.hop;              // 1 + 480000/hop, last frame dropped
        return 1 + n / core.hop;                              // DSP.swift:213-214 with 2*(n_fft/2) padding
    }
    void run(const float* d_in, int batch, long long n, float* d_o, cudaStream_t s) {
        B2A_CHECK(batch > 0 && n > core.n_fft / 2, B2A_ERR_INVALID_INPUT,
                  "logmel: clips must be longer than n_fft/2 samples");
        B2A_CUDA(cudaSetDevice(core.device));
        d_max.alloc(batch);
        fill_kernel<<<cdiv(batch, 256), 256, 0, s>>>(d_max.p, batch, -INFINITY);
        count_launch();
        const long long n_total = kind == 1 ? 480000 : n;
        const long long n_valid = std::min(n, n_total);
        core.launch(d_in, n, n_valid, n_total, 1, batch, (int)frames(n), d_o, d_max.p, s);
    }
};

extern "C" {

int32_t b2a_logmel_create(int32_t device, int32_t kind, int32_t sr, int32_t n_fft, int32_t hop, int32_t n_mels,
                          b2a_logmel** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_logmel_create: null out");
        *out = nullptr;
        B2A_CHECK(kind == 0 || kind == 1, B2A_ERR_INVALID_INPUT, "b2a_logmel_create: kind must be 0 or 1");
        *out = new b2a_logmel(device, kind, sr, n_fft, hop, n_mels);
    });
}

int64_t b2a_logmel_frames(const b2a_logmel* h, int64_t n_samples) { return h ? h->frames(n_samples) : 0; }

int32_t b2a_logmel_compute(b2a_logmel* h, const float* pcm, int32_t batch, int64_t n, float* out) {
    return guarded([&] {
        B2A_CHECK(h && pcm && out, B2A_ERR_INVALID_INPUT, "b2a_logmel_compute: null argument");
        B2A_CUDA(cudaSetDevice(h->core.device));
        const size_t n_in = (size_t)batch * n, n_out = (size_t)batch * h->frames(n) * h->core.n_mels;
        h->d_pcm.alloc(n_in);
        h->d_out.alloc(n_out);
        B2A_CUDA(cudaMemcpyAsync(h->d_pcm.p, pcm, n_in * sizeof(float), cudaMemcpyHostToDevice, h->stream));
        h->run(h->d_pcm.p, batch, n, h->d_out.p, h->stream);
        B2A_CUDA(cudaMemcpyAsync(out, h->d_out.p, n_out * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
        B2A_CUDA(cudaStreamSynchronize(h->stream));
    });
}

int32_t b2a_logmel_compute_dev(b2a_logmel* h, const float* d_pcm, int32_t batch, int64_t n, float* d_out,
                               void* stream) {
    return guarded([&] {
        B2A_CHECK(h && d_pcm && d_out, B2A_ERR_INVALID_INPUT, "b2a_logmel_compute_dev: null argument");
        h->run(d_pcm, batch, n, d_out, (cudaStream_t)stream);
    });
}

void b2a_logmel_destroy(b2a_logmel* h) { delete h; }

}  // extern "C"
