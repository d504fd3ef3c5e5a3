/*
 * b200audio.h -- C ABI of libb200audio.so: the H100-native (sm_90a) hot path behind
 * MLXAudio's Swift protocols.  Plain pointers and sizes only; no torch / C++ types.
 *
 * Every entry point names the reference interface it replaces (paths relative to the
 * Blaizzy/mlx-audio-swift checkout).  INTEGRATION.md shows the Swift-side binding.
 *
 * Conventions
 *   - every function returns an int32 status (B2A_OK == 0).  Codes 1..5 map 1:1 onto the cases
 *     of AudioGenerationError (Sources/MLXAudioCore/Generation/GenerationTypes.swift:66-87);
 *     the library never aborts the process.  b2a_last_error() returns the message of the last
 *     failure on the calling thread.
 *   - handles are opaque, own their device memory and CUDA stream, and are NOT thread-safe:
 *     one in-flight call per handle (SURVEY.md section 8b, "Threading").
 *   - the caller owns every host buffer.  `_dev` variants take DEVICE pointers (already resident
 *     in HBM) plus a cudaStream_t passed as void*; all other variants take HOST pointers and do
 *     the host<->device copies themselves.
 *   - there is NO CPU fallback: with no usable CUDA device every create/compute call fails with
 *     B2A_ERR_CUDA.
 */
#ifndef B200AUDIO_H
#define B200AUDIO_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2A_OK 0
#define B2A_ERR_MODEL_NOT_INITIALIZED 1 /* AudioGenerationError.modelNotInitialized */
#define B2A_ERR_GENERATION_FAILED 2     /* .generationFailed   */
#define B2A_ERR_INVALID_INPUT 3         /* .invalidInput       */
#define B2A_ERR_AUDIO_DECODING_FAILED 4 /* .audioDecodingFailed */
#define B2A_ERR_AUDIO_ENCODING_FAILED 5 /* .audioEncodingFailed */
#define B2A_ERR_CANCELLED 6             /* Task.checkCancellation (LlamaTTS.swift:715) */
#define B2A_ERR_CUDA 7                  /* no device / CUDA runtime failure */

#define B2A_DTYPE_F32 0
#define B2A_DTYPE_BF16 1
#define B2A_DTYPE_I32 2

/* One named host tensor (row-major).  Names follow the reference's safetensors keys. */
typedef struct b2a_tensor {
    const char* name;
    int32_t dtype;
    int32_t ndim;
    int64_t shape[4];
    const void* data;
} b2a_tensor;

const char* b2a_last_error(void);
const char* b2a_version(void);
/* number of visible CUDA devices (0 when none); never fails */
int32_t b2a_device_count(void);
/* kernels launched by this library on the calling process so far (for bench.py's gpu_launches) */
int64_t b2a_launch_count(void);

/* ------------------------------------------------------------------ DSP tables (host math)
 * hanningWindow  Sources/MLXAudioCore/DSP.swift:15-22  (symmetric; periodic!=0 gives the
 *                WhisperAudio.swift:42-43 window)
 * melFilters     Sources/MLXAudioCore/DSP.swift:76-168 ; out is [n_fft/2+1, n_mels] row-major;
 *                f_max < 0 means sample_rate/2; mel_scale 0 = htk, 1 = slaney; norm_slaney 0/1. */
int32_t b2a_hanning_window(int32_t size, int32_t periodic, float* out);
int32_t b2a_mel_filters(int32_t sample_rate, int32_t n_fft, int32_t n_mels, float f_min, float f_max,
                        int32_t norm_slaney, int32_t mel_scale, float* out);
/* The other two host helpers of DSP.swift, off the mel path but with known answers in the reference's tests
 * (Tests/MLXAudioCodecsTests.swift:117-140): hammingWindow (:25-42; periodic != 0 is the default) and powerToDB (:61-73;
 * top_db < 0 means no dynamic-range clipping).                                                                    */
int32_t b2a_hamming_window(int32_t size, int32_t periodic, float* out);
int32_t b2a_power_to_db(const float* spectrogram, int64_t n, float amin, float top_db, float* out);

/* ------------------------------------------------------------------ streaming log-mel
 * Replaces class IncrementalMelSpectrogram
 *   (Sources/MLXAudioSTT/Streaming/IncrementalMelSpectrogram.swift:18-208):
 *   init(sampleRate:nFft:hopLength:nMels:) :43-62 -> b2a_mel_create
 *   process(samples:) :68-147 -> b2a_mel_process   (*n_frames == 0  <=>  reference returns nil)
 *   flush() :151-200          -> b2a_mel_flush
 *   reset() :203-208          -> b2a_mel_reset
 *   totalFrames :41           -> b2a_mel_total_frames
 * `out` receives [n_frames, n_mels] float32; out_cap_frames is its capacity in frames
 * (B2A_ERR_INVALID_INPUT if too small; b2a_mel_max_frames() gives a safe bound).           */
typedef struct b2a_mel b2a_mel;
int32_t b2a_mel_create(int32_t device, int32_t sample_rate, int32_t n_fft, int32_t hop_length,
                       int32_t n_mels, b2a_mel** out);
int64_t b2a_mel_max_frames(const b2a_mel* h, int64_t n_samples);
int32_t b2a_mel_process(b2a_mel* h, const float* samples, int64_t n_samples, float* out,
                        int64_t out_cap_frames, int64_t* n_frames);
int32_t b2a_mel_flush(b2a_mel* h, float* out, int64_t out_cap_frames, int64_t* n_frames);
int32_t b2a_mel_reset(b2a_mel* h);
int64_t b2a_mel_total_frames(const b2a_mel* h);
void b2a_mel_destroy(b2a_mel* h);

/* ------------------------------------------------------------------ offline / batched log-mel
 * kind 0: computeMelSpectrogram (Sources/MLXAudioCore/DSP.swift:230-273): symmetric Hann, HTK
 *         scale, reflect pad both sides, global max-8 clamp, out [B, 1+n/hop, n_mels].
 * kind 1: WhisperAudio.encoderFeatures (Sources/MLXAudioSTT/Models/Whisper/WhisperAudio.swift:
 *         7-13,38-87): pad/trim each clip to 480000, periodic Hann, Slaney scale, last frame
 *         dropped, per-clip max-8 clamp, out [B, 3000, n_mels].
 * pcm is [B, n_samples] (every clip the same length); b2a_logmel_frames gives frames per clip.
 * n_fft is 400 or 1024 (the Qwen3-TTS speaker encoder's front-end), here and in b2a_mel_create;
 * any other size -> B2A_ERR_INVALID_INPUT. */
typedef struct b2a_logmel b2a_logmel;
int32_t b2a_logmel_create(int32_t device, int32_t kind, int32_t sample_rate, int32_t n_fft,
                          int32_t hop_length, int32_t n_mels, b2a_logmel** out);
int64_t b2a_logmel_frames(const b2a_logmel* h, int64_t n_samples);
int32_t b2a_logmel_compute(b2a_logmel* h, const float* pcm, int32_t batch, int64_t n_samples, float* out);
int32_t b2a_logmel_compute_dev(b2a_logmel* h, const float* d_pcm, int32_t batch, int64_t n_samples,
                               float* d_out, void* stream);
void b2a_logmel_destroy(b2a_logmel* h);

/* ------------------------------------------------------------------ SNAC codec
 * Replaces class SNAC (Sources/MLXAudioCodecs/SNAC/SNACDecoder.swift:12-131) behind the
 * AudioCodecModel protocol (Sources/MLXAudioCodecs/AudioCodecModel.swift:4-27):
 *   SNAC.fromConfig/fromModelDirectory :135-189 -> b2a_snac_create (config + named tensors)
 *   decode(_ codes:) :127-131 / decodeAudio :199 -> b2a_snac_decode
 *   quantizer(z) (ResidualVectorQuantize.callAsFunction, SNAC/VQ.swift:150-163), the
 *   encode-side code search                      -> b2a_snac_quantize
 *   encode(_ audioData:) :120-125 / encodeAudio :197-199 -> b2a_snac_encode (preprocess -> Encoder -> quantizer)
 * codes[i] is [B, T_i] int32 with T_i = t_latent / vq_strides[i]; wave is [B, 1, b2a_snac_decoded_length(h, t_latent)].
 * noise[i] (nullable array of nullable pointers) is the [B, 1, T] Gaussian draw of decoder
 * block i's NoiseBlock (Layers.swift:263-279), T the length of stage i's output (the decoded length of the stages up to i);
 * NULL = draw on device from `seed` (noise_mode 0) or use zero noise (noise_mode 1).
 * Both are sized by the decoded length, not by t_latent * hop: like the reference, a stage of odd stride s yields s T - 1
 * frames (DecoderBlock's outputPadding is dropped), so the 32 / 44 kHz models (decoder_rates [8, 8, 3, 2]) decode t_latent
 * frames to 384 t_latent - 2 samples.  With attn_window_size > 0, t_latent must be a multiple of it (B2A_ERR_INVALID_INPUT). */
typedef struct b2a_snac_config {
    int32_t sampling_rate;
    int32_t encoder_dim;
    int32_t n_encoder_rates;
    int32_t encoder_rates[8];
    int32_t latent_dim; /* 0 => encoder_dim * 2^n_encoder_rates */
    int32_t decoder_dim;
    int32_t n_decoder_rates;
    int32_t decoder_rates[8];
    int32_t attn_window_size; /* 0 => none (24 kHz); > 0 => LocalMHA over windows of this many frames (32 / 44 kHz models: 32),
                                 1 .. 64, latent_dim and decoder_dim multiples of 64 (heads of 64); no B2A_SNAC=simt path */
    int32_t codebook_size;
    int32_t codebook_dim;
    int32_t n_vq_strides;
    int32_t vq_strides[8];
    int32_t noise;
    int32_t depthwise;
} b2a_snac_config;

typedef struct b2a_snac b2a_snac;
int32_t b2a_snac_create(int32_t device, const b2a_snac_config* cfg, const b2a_tensor* tensors,
                        int32_t n_tensors, b2a_snac** out);
int64_t b2a_snac_hop_length(const b2a_snac* h);
/* samples decoded from t_latent frames: t_latent * hop when every decoder rate is even, less by one per odd-stride stage
 * (scaled by the later strides) otherwise; 0 for a null handle or t_latent <= 0 */
int64_t b2a_snac_decoded_length(const b2a_snac* h, int64_t t_latent);
void* b2a_snac_stream(b2a_snac* h); /* the handle's cudaStream_t, for event timing */
int32_t b2a_snac_decode(b2a_snac* h, const int32_t* const* codes, int32_t batch, int64_t t_latent,
                        const float* const* noise, int32_t noise_mode, uint64_t seed, float* wave);
int32_t b2a_snac_decode_dev(b2a_snac* h, const int32_t* const* d_codes, int32_t batch, int64_t t_latent,
                            const float* const* d_noise, int32_t noise_mode, uint64_t seed,
                            float* d_wave, void* stream);
/* z [B, latent_dim, T] float32 -> codes[i] [B, T/stride_i] int32 (+ optional z_q [B, latent, T]) */
int32_t b2a_snac_quantize(b2a_snac* h, const float* z, int32_t batch, int64_t t_latent,
                          int32_t* const* codes, float* z_q);
/* SNAC.encode (SNACDecoder.swift:86-105,120-125): wave [B, 1, n_samples] float32 is zero right-padded to a multiple of
 * hop * lcm(vq_strides, attn_window_size) (2048 for the 24 kHz model, 12288 for the 32 / 44 kHz ones), run through the encoder (Layers.swift:236-259,319-360) and the residual
 * quantizer; codes[i] [B, t_latent / vq_strides[i]] int32 with t_latent = b2a_snac_encoded_length(h, n_samples).
 * Needs the checkpoint's encoder.* tensors (a decoder-only handle returns B2A_ERR_MODEL_NOT_INITIALIZED); empty audio is
 * B2A_ERR_AUDIO_ENCODING_FAILED; an encoder geometry the device path does not run (a stride < 2, latent_dim other than
 * encoder_dim * 2^len(encoder_rates), batch * padded samples >= 2^31) is B2A_ERR_INVALID_INPUT.  Deterministic: the same
 * input gives the same codes, and a batch gives the codes of its clips encoded one by one. */
int64_t b2a_snac_encoded_length(const b2a_snac* h, int64_t n_samples); /* 0 without encoder weights */
int32_t b2a_snac_encode(b2a_snac* h, const float* wave, int32_t batch, int64_t n_samples, int32_t* const* codes);
/* the same on DEVICE pointers, enqueued on `stream` (no host synchronisation) */
int32_t b2a_snac_encode_dev(b2a_snac* h, const float* d_wave, int32_t batch, int64_t n_samples, int32_t* const* d_codes,
                            void* stream);
void b2a_snac_destroy(b2a_snac* h);

/* ------------------------------------------------------------------ Orpheus / Llama TTS
 * Replaces class LlamaTTSModel (Sources/MLXAudioTTS/Models/Llama/LlamaTTS.swift:354-977) behind
 * SpeechGenerationModel (Sources/MLXAudioTTS/Generation.swift:8-39):
 *   fromModelDirectory :942-977 (weights + config)   -> b2a_tts_create
 *   callAsFunction(_:cache:) :557-567                -> b2a_tts_forward_logits (parity hook)
 *   generate(text:voice:...) :658-765                -> b2a_tts_generate
 *   generateStream :777-913 (.token/.info/.audio)    -> b2a_tts_generate + on_token callback
 *   Task cancellation :715,911                       -> b2a_tts_cancel
 * Tokenisation stays host-side: the ABI takes token ids already framed by prepareInputIds
 * (:446-553; b2a_tts_prepare_input_ids does the framing for raw text-token ids).
 * A batch is B independent utterances ("batched == serial"; the reference itself is batch-1). */
typedef struct b2a_llama_config {
    int32_t hidden_size;
    int32_t num_hidden_layers;
    int32_t intermediate_size;
    int32_t num_attention_heads;
    int32_t num_key_value_heads;
    int32_t head_dim;
    int32_t vocab_size;
    float rms_norm_eps;
    float rope_theta;
    float rope_factor; /* llama3 rope_scaling (LlamaTTS.swift:114-118) */
    float rope_low_freq_factor;
    float rope_high_freq_factor;
    float rope_old_context_len;
    int32_t tie_word_embeddings;
    int32_t max_batch;   /* KV-cache rows, 1..32 (other values: B2A_ERR_INVALID_INPUT) */
    int32_t max_context; /* KV-cache positions per row */
} b2a_llama_config;

/* GenerateParameters as used at LlamaTTS.swift:573-581 (defaults 1200 / 0.6 / 0.8 / 1.3 / 20) */
typedef struct b2a_gen_params {
    int32_t max_tokens;
    float temperature; /* 0 => greedy argmax, lowest index wins ties */
    float top_p;
    float repetition_penalty;
    int32_t repetition_context_size;
    uint64_t seed;
} b2a_gen_params;

/* AudioGenerationInfo (GenerationTypes.swift:14-45) */
typedef struct b2a_gen_info {
    int32_t prompt_token_count;
    int32_t generation_token_count;
    double prefill_time;
    double generate_time;
    double tokens_per_second;
    double codec_time;
    double peak_memory_gb;
} b2a_gen_info;

typedef struct b2a_tts b2a_tts;
/* on_token(user, utterance, step, token): the .token(Int) events of generateStream (:862) */
typedef void (*b2a_token_cb)(void* user, int32_t utterance, int32_t step, int32_t token);

int32_t b2a_tts_create(int32_t device, const b2a_llama_config* cfg, const b2a_tensor* tensors,
                       int32_t n_tensors, b2a_snac* snac /* borrowed, may be NULL */, b2a_tts** out);
/* [SOH] ids [EOT, EOH], left-padded with 128263 to the longest prompt; out is [B, max_len+3] */
int32_t b2a_tts_prepare_input_ids(const int32_t* const* prompt_ids, const int32_t* lens, int32_t batch,
                                  int32_t* out, int32_t* out_len);
/* prepareInputIds with refAudio / refText (voice cloning, :446-553): every row is
 *   [128263 padding] [SOH] ref_text_ids [EOT, EOH] [128261, SOS] ref_code_list + 128266 [EOS, 128262] [SOH] prompt [EOT, EOH],
 * the padding in front to the longest prompt.  ref_code_list is the 7-token interleaved reference (b2a_tts_interleave of the
 * reference clip's b2a_snac_encode codes, values in [0, 7 * 4096)); ref_text_ids is the tokenised transcript (may be empty).
 * out NULL: only *out_len.  B2A_ERR_INVALID_INPUT for null arguments, ref_code_len % 7 != 0 or a code out of range. */
int32_t b2a_tts_prepare_input_ids_ref(const int32_t* const* prompt_ids, const int32_t* lens, int32_t batch,
                                      const int32_t* ref_text_ids, int32_t ref_text_len, const int32_t* ref_code_list,
                                      int32_t ref_code_len, int32_t* out, int32_t* out_len);
/* One forward over ids [B, L] appended at the cache's current offset (reset_cache != 0 clears
 * it first); logits_out [B, L, vocab] float32 (host). */
int32_t b2a_tts_forward_logits(b2a_tts* h, const int32_t* ids, int32_t batch, int32_t len,
                               int32_t reset_cache, float* logits_out);
/* Full text-token-ids -> tokens -> (parseOutput, 7-token de-interleave, SNAC decode) -> waveform.
 * input_ids [B, L] (all rows length L, as produced by b2a_tts_prepare_input_ids or the host).
 * tokens_out [B, max_tokens] (nullable) receives generated ids, n_tokens_out[B] their counts.
 * wave_out [B, wave_cap] (nullable => skip the codec) receives each waveform, wave_len[B] its
 * sample count.  Rows that yield no audio codes report wave_len 0; if every row does the call
 * fails with B2A_ERR_GENERATION_FAILED ("No audio codes generated", LlamaTTS.swift:752-754).  */
int32_t b2a_tts_generate(b2a_tts* h, const int32_t* input_ids, int32_t batch, int32_t len,
                         const b2a_gen_params* params, int32_t* tokens_out, int32_t* n_tokens_out,
                         float* wave_out, int64_t wave_cap, int64_t* wave_len, b2a_gen_info* info,
                         b2a_token_cb on_token, void* user);
/* generateStream with audio DURING generation (SURVEY.md 8f row N2).  The reference's Orpheus emits one .audio event at the end
 * (LlamaTTS.swift:901-904); its streaming models decode their codes in chunks while generating (decodeAudioFromCodes' chunk loop,
 * Sources/MLXAudioTTS/Models/Qwen3/Qwen3.swift:47-83; the CLI's --benchmark TTFB is the latency of the first .audio event,
 * Sources/Tools/mlx-audio-swift-tts/App.swift:155-211).  Here every `frames_per_chunk` new 7-token frames of a row are decoded by
 * SNAC with `left_context_frames` already-emitted frames in front of them (their samples are dropped) and handed to on_audio as
 * 2048 * frames float32 samples; is_final marks a row's last chunk.  Concatenated chunks equal the one-shot waveform except near
 * chunk boundaries (the codec's receptive field), exactly like the reference's chunked decode.                                 */
typedef void (*b2a_audio_cb)(void* user, int32_t utterance, const float* samples, int64_t n_samples, int32_t is_final);
int32_t b2a_tts_generate_stream(b2a_tts* h, const int32_t* input_ids, int32_t batch, int32_t len, const b2a_gen_params* params,
                                int32_t frames_per_chunk, int32_t left_context_frames, int32_t* tokens_out, int32_t* n_tokens_out,
                                b2a_gen_info* info, b2a_token_cb on_token, b2a_audio_cb on_audio, void* user);
/* Device-resident variant for bench.py's `value`: ids already in HBM, waveform left in HBM. */
int32_t b2a_tts_generate_dev(b2a_tts* h, const int32_t* d_input_ids, int32_t batch, int32_t len,
                             const b2a_gen_params* params, float* d_wave_out, int64_t wave_cap,
                             int64_t* wave_len, b2a_gen_info* info);
int32_t b2a_tts_cancel(b2a_tts* h);
/* the handle's cudaStream_t (as void*), so a caller can order its own work / record events on the stream the kernels run on */
void* b2a_tts_stream(b2a_tts* h);
/* parseOutput (:383-434) and llamaDecodeAudioFromCodes' de-interleave (:41-63), host-side ints.
 * tokens [B, n]; code_lists_out [B, n] / code_lens[B]; then per row codes0/1/2 sized n/7, 2n/7, 4n/7 */
int32_t b2a_tts_parse_output(const int32_t* tokens, int32_t batch, int32_t n, int32_t* code_lists_out,
                             int32_t* code_lens);
int32_t b2a_tts_deinterleave(const int32_t* code_list, int32_t n, int32_t* codes0, int32_t* codes1,
                             int32_t* codes2, int32_t* n_frames);
int32_t b2a_tts_interleave(const int32_t* codes0, const int32_t* codes1, const int32_t* codes2,
                           int32_t n_frames, int32_t* code_list);
void b2a_tts_destroy(b2a_tts* h);

/* ------------------------------------------------------------------ VyvoTTS (Qwen3 language model + SNAC 24 kHz)
 * Replaces class Qwen3Model (Sources/MLXAudioTTS/Models/Qwen3/Qwen3.swift:305-931), model_type "qwen3" / "qwen".  The constructors return a
 * b2a_tts handle: b2a_tts_generate / _stream / _dev, b2a_tts_forward_logits, b2a_tts_cancel and b2a_tts_destroy serve it unchanged, with
 * VyvoTTS's token layout (Qwen3.swift:18-29): generation stops on 151671 (not kept), a row's codes start after its last start-of-speech
 * 151670 or, without one, at its first audio token (>= 151679) after the last start-of-AI 151674 (parseOutputRow, :333-358), and a row of
 * more than 50 frames is decoded as independent 50-frame SNAC chunks whose waveforms are concatenated (decodeAudioFromCodes, :47-83).
 * The stack is Qwen3 (:145-303): per-head q/k RMSNorm before RoPE, rotate-half RoPE with base rope_theta; head_dim must be 128. */
typedef struct b2a_qwen3_lm_config {     /* Qwen3Configuration, Config.swift:15-73 */
    int32_t hidden_size;
    int32_t num_hidden_layers;
    int32_t intermediate_size;
    int32_t num_attention_heads;
    int32_t num_key_value_heads;
    int32_t head_dim;
    int32_t vocab_size;
    float rms_norm_eps;
    float rope_theta;          /* default 1e6 */
    float rope_linear_factor;  /* rope_scaling {"type": "linear", "factor": f}: f; any other rope_scaling (or none): 1 */
    int32_t tie_word_embeddings;   /* default 0 */
    int32_t max_position_embeddings;   /* default 32768 (informational) */
    int32_t sample_rate;       /* default 24000 */
    int32_t eos_token_id;      /* default 151645 (informational: generation stops on end-of-speech 151671) */
    int32_t max_batch;         /* KV-cache rows, 1..32 */
    int32_t max_context;       /* KV-cache positions per row */
} b2a_qwen3_lm_config;

int32_t b2a_qwen3_lm_create(int32_t device, const b2a_qwen3_lm_config* cfg, const b2a_tensor* tensors, int32_t n_tensors,
                            b2a_snac* snac /* borrowed, may be NULL */, b2a_tts** out);
/* config.json -> the struct with Qwen3Configuration's defaults; quant_* (nullable) from its "quantization" block (0 = none) */
int32_t b2a_qwen3_lm_config_from_json(const char* config_path, int32_t max_batch, int32_t max_context, b2a_qwen3_lm_config* cfg,
                                      int32_t* quant_group_size, int32_t* quant_bits);
/* Qwen3Model.fromModelDirectory (:892-930) without tokenizer / SNAC download: config.json + every *.safetensors ->
 * b2a_weights_sanitize_llama_config (lm_head.weight dropped when tied, MLX 2/4/8-bit layers expanded to bf16) -> b2a_qwen3_lm_create */
int32_t b2a_qwen3_lm_create_from_directory(const char* model_dir, int32_t device, int32_t max_batch, int32_t max_context, b2a_snac* snac,
                                           b2a_tts** out);
/* prepareInputIds (:377-474) on token ids: [151676 padding] [151672] prompt [151645, 151673]; with a reference
 * [151676 padding] [151672] ref_text_ids [151645, 151673] [151674, 151670] ref_code_list + 151679 [151671, 151675] [151672] prompt [151645, 151673].
 * Arguments and errors as b2a_tts_prepare_input_ids(_ref). */
int32_t b2a_qwen3_lm_prepare_input_ids(const int32_t* const* prompt_ids, const int32_t* lens, int32_t batch, int32_t* out, int32_t* out_len);
int32_t b2a_qwen3_lm_prepare_input_ids_ref(const int32_t* const* prompt_ids, const int32_t* lens, int32_t batch, const int32_t* ref_text_ids,
                                           int32_t ref_text_len, const int32_t* ref_code_list, int32_t ref_code_len, int32_t* out,
                                           int32_t* out_len);
/* parseOutputRow (:333-358) for every row of tokens [B, n]; code_lists_out [B, n], code_lens [B] */
int32_t b2a_qwen3_lm_parse_output(const int32_t* tokens, int32_t batch, int32_t n, int32_t* code_lists_out, int32_t* code_lens);

/* ------------------------------------------------------------------ Soprano (Qwen3 language model + Vocos decoder of its hidden states)
 * Replaces class SopranoModel (Sources/MLXAudioTTS/Models/Soprano/Soprano.swift:184-977) and SopranoDecoder (SopranoDecoder.swift:222-285).
 * The constructors return a b2a_tts handle that owns a Vocos decoder: b2a_tts_generate / _dev, b2a_tts_forward_logits, b2a_tts_cancel and
 * b2a_tts_destroy serve it.  Soprano decodes the final-RMSNorm hidden state of the last prompt position and of every generated token that
 * is fed back (forwardWithHiddenStates, :254-275; streamGenerate, :801-885) -- 1 + n_tokens states per row, none for the stop token --
 * into audio; the step captures them on the device.  Sampling is Soprano's own (:836-901, :996-1059): the repetition penalty looks at the
 * last repetition_context_size GENERATED tokens and applies once per occurrence (l > 0 ? l / p : l * p), also at temperature 0; top-p
 * keeps token i iff the ascending cumulative sum of exp(l) (unnormalised) through i exceeds 1 - top_p, and the temperature divides the
 * filtered logits afterwards.  When no token passes (sum exp(l) <= 1 - top_p) the argmax is returned, where the reference would sample
 * an all -inf row.  Generation stops on stop_token_id (the tokenizer's EOS, :972), which is not kept.
 * Waveform of a row with n states: interpolate1d(align_corners) to upscale (n - 1) + 1 frames, the Vocos backbone and ISTFT head, then its
 * last (n - 1) token_size samples (:664-671); for n = 1 the untrimmed n_fft samples of a one-frame overlap-add (SopranoDecoder.swift:191-196).
 * Rows of one call decode as they would one by one.  head_dim must be 128; prompt + max_tokens + 1 must fit max_context. */
typedef struct b2a_soprano_config {     /* SopranoConfiguration, SopranoConfig.swift:65-176, with its defaults */
    int32_t hidden_size;
    int32_t num_hidden_layers;
    int32_t intermediate_size;
    int32_t num_attention_heads;
    int32_t num_key_value_heads;
    int32_t head_dim;
    int32_t vocab_size;
    float rms_norm_eps;              /* 1e-6 */
    float rope_theta;                /* 1e4 */
    int32_t tie_word_embeddings;     /* 0 */
    int32_t max_position_embeddings; /* 512 (informational) */
    int32_t bos_token_id;            /* 1 (informational) */
    int32_t eos_token_id;            /* 2 (informational: generation stops on stop_token_id) */
    int32_t pad_token_id;            /* 0 (informational) */
    int32_t stop_token_id;           /* the tokenizer's EOS; 3 when it has none */
    int32_t sample_rate;             /* 32000 */
    int32_t decoder_num_layers;      /* 8 */
    int32_t decoder_dim;             /* 768 */
    int32_t decoder_intermediate_dim;/* 2304 */
    int32_t hop_length;              /* 512 */
    int32_t n_fft;                   /* 2048 */
    int32_t upscale;                 /* 4 */
    int32_t input_kernel;            /* 1 */
    int32_t dw_kernel;               /* 3 */
    int32_t token_size;              /* 2048 */
    int32_t receptive_field;         /* 4 (informational: audio is decoded once per call) */
    int32_t max_batch;               /* KV-cache rows, 1..32 */
    int32_t max_context;             /* KV-cache positions per row */
} b2a_soprano_config;

/* tensors in SopranoModel.sanitize's layout (:314-361): model.* (the Qwen3 stack), lm_head.weight unless tied, decoder.decoder.* (the
 * Vocos backbone: embed, norm, convnext.N.*, final_layer_norm) and decoder.head.out.*; conv weights in the MLX [out, k, in] layout */
int32_t b2a_soprano_create(int32_t device, const b2a_soprano_config* cfg, const b2a_tensor* tensors, int32_t n_tensors, b2a_tts** out);
/* config.json -> the struct with SopranoConfiguration's defaults.  Unless repo_hint contains "soprano-1.1" (case-insensitive) the
 * decoder is the older one: decoder_dim 512, decoder_intermediate_dim 1536 and input_kernel 3, whatever config.json says
 * (fromModelDirectory, :934-941).  repo_hint NULL: the config file's directory name.  quant_* (nullable) from "quantization" (0 = none) */
int32_t b2a_soprano_config_from_json(const char* config_path, const char* repo_hint, int32_t max_batch, int32_t max_context,
                                     b2a_soprano_config* cfg, int32_t* quant_group_size, int32_t* quant_bits);
/* fromModelDirectory (:928-976) without the tokenizer: config.json (+ the repo rule above; repo_hint NULL = the directory name) + every
 * *.safetensors -> sanitize (a leading "model." stripped, language_model.lm_head -> lm_head, language_model.* and bare keys -> model.*,
 * lm_head.weight dropped when tied) -> MLX 2/4/8-bit layers expanded -> b2a_soprano_create.  stop_token_id is 3 unless the directory's
 * tokenizer_config.json names an eos_token that tokenizer.json's added_tokens resolve. */
int32_t b2a_soprano_create_from_directory(const char* model_dir, const char* repo_hint, int32_t device, int32_t max_batch,
                                          int32_t max_context, b2a_tts** out);
/* SopranoDecoder.callAsFunction + the cut on its own: hidden [B, n, hidden_size] float32 (host) -> wave_out [B, wave_cap], wave_len[B]
 * (all rows the same length).  n >= 1. */
int32_t b2a_soprano_decode_hidden(b2a_tts* h, const float* hidden, int32_t batch, int32_t n, float* wave_out, int64_t wave_cap,
                                  int64_t* wave_len);
/* samples of the waveform of n hidden states (0 for a handle that is not Soprano's) */
int64_t b2a_soprano_wave_length(const b2a_tts* h, int32_t n);

/* ------------------------------------------------------------------ weight / format plumbing (SURVEY.md 8f, row N4)
 * Host-only.  Replaces MLX.loadArrays on *.safetensors (llamaTTSLoadWeights, LlamaTTS.swift:982-994: every file of a directory, later
 * files win), WhisperModel.detectFormat / sanitize / remapMlxWhisperKey / whisperSinusoids (WhisperModel.swift:315-480),
 * LlamaTTSModel.sanitize (LlamaTTS.swift:583-593) and the MLX affine de-quantisation behind quantize(model:) (:955-966).
 * A b2a_weights handle keeps the files mapped; b2a_weights_get returns borrowed views valid until b2a_weights_free.
 * F16 tensors are widened to F32, I64 narrowed to I32, U32 (packed quantised words) is reported as B2A_DTYPE_I32.
 *   b2a_weights_sanitize_whisper: -> HF (`transformers`) names with the "model." prefix, conv weights in the PyTorch [out, in, k]
 *     layout (what b2a_stt_create takes), missing encoder positions synthesised; *format = 0 huggingFace, 1 mlxWhisper.
 *   b2a_weights_sanitize_llama: drops rotary inv_freq (and lm_head.weight when tied); bits > 0: every layer with a ".scales"
 *     tensor is expanded to bf16 (w = scales * q + biases, value j of a uint32 word at bits [j*bits, (j+1)*bits); bits 2 / 4 / 8).
 *   b2a_tts_config_from_json: config.json -> the b2a_llama_config struct, LlamaTTSConfig.swift:100-166, + the "quantization" block.
 *   b2a_tts_create_from_directory = LlamaTTSModel.fromModelDirectory (LlamaTTS.swift:942-977) without tokenizer / SNAC download. */
typedef struct b2a_weights b2a_weights;
int32_t b2a_weights_load(const char* file_or_directory, b2a_weights** out);
int32_t b2a_weights_count(const b2a_weights* w);
int32_t b2a_weights_get(const b2a_weights* w, int32_t index, b2a_tensor* out);
int32_t b2a_weights_sanitize_whisper(b2a_weights* w, int32_t* format);
int32_t b2a_weights_sanitize_llama(b2a_weights* w, int32_t tie_word_embeddings, int32_t group_size, int32_t bits);
/* Same, with the quantisation read from config.json the way the reference's loader does (LlamaTTS.swift:955-966 through
 * mlx-swift-lm's PerLayerQuantization): "quantization": {"group_size", "bits", "<layer path>": false | {"group_size", "bits"}} --
 * per-layer settings override the default, a layer marked false must not carry .scales.  b2a_tts_create_from_directory uses this. */
int32_t b2a_weights_sanitize_llama_config(b2a_weights* w, const char* config_path);
/* SopranoModel.sanitize (Soprano.swift:314-361) + the de-quantisation config.json asks for: the key layout b2a_soprano_create takes */
int32_t b2a_weights_sanitize_soprano_config(b2a_weights* w, const char* config_path);
/* MLX affine de-quantisation (to bf16) of every layer that carries "<path>.scales", with one group_size / bits -- what
 * WhisperModel.fromDirectory's quantize(model:groupSize:bits:) implies for a quantised checkpoint (WhisperModel.swift:499-511:
 * every Linear and decoder.embed_tokens; the tied projection then multiplies by the de-quantised embedding,
 * Tests/WhisperQuantizedTiedEmbeddingTests.swift).  Call after b2a_weights_sanitize_whisper.                              */
int32_t b2a_weights_dequantize(b2a_weights* w, int32_t group_size, int32_t bits);
void b2a_weights_free(b2a_weights* w);
int32_t b2a_tts_config_from_json(const char* config_path, int32_t max_batch, int32_t max_context, b2a_llama_config* cfg,
                                 int32_t* quant_group_size, int32_t* quant_bits);
int32_t b2a_tts_create_from_directory(const char* model_dir, int32_t device, int32_t max_batch, int32_t max_context,
                                      b2a_snac* snac, b2a_tts** out);

/* ------------------------------------------------------------------ Vocos vocoder
 * Replaces class Vocos (Sources/MLXAudioCodecs/Vocos/Vocos.swift:284-322) behind AudioDecoderModel
 * (Sources/MLXAudioCodecs/AudioCodecModel.swift:4-13):
 *   Vocos(backbone:head:) + weights (keys backbone.* / head.*, MLX layouts) -> b2a_vocos_create
 *   decode(_ features:) / decodeAudio (:302-306,318-320)                   -> b2a_vocos_decode
 * features are [B, L, input_channels] float32 (the layout VocosBackbone expects, VocosBackbone.swift:170-175);
 * the waveform is [B, (L-1)*hop_length] (ISTFTHead centre trim, Vocos.swift:150-158).  AdaLayerNorm models
 * (Vocos.swift:17-47; weights backbone.norm.{scale,shift}.{weight,bias}, backbone.convnext.N.norm.{scale,shift}.*) take their
 * `bandwidthId` conditioning through b2a_vocos_decode_cond: cond [B, adanorm_num_embeddings] float32, the rows the scale / shift
 * Linears are applied to (decode(_:bandwidthId:) :302-306); decoding such a model without it fails with invalidInput where the
 * reference fatalErrors (VocosBackbone.swift:66-68,181-183).                                        */
typedef struct b2a_vocos_config {
    int32_t input_channels;
    int32_t dim;
    int32_t intermediate_dim;
    int32_t num_layers;
    int32_t n_fft;
    int32_t hop_length;
    int32_t input_kernel_size;
    int32_t dw_kernel_size;
    int32_t adanorm_num_embeddings; /* 0: LayerNorm; > 0: AdaLayerNorm(numEmbeddings, dim) for backbone.norm and every block's norm */
} b2a_vocos_config;

typedef struct b2a_vocos b2a_vocos;
int32_t b2a_vocos_create(int32_t device, const b2a_vocos_config* cfg, const b2a_tensor* tensors, int32_t n_tensors,
                         b2a_vocos** out);
int64_t b2a_vocos_output_length(const b2a_vocos* h, int32_t frames);
void* b2a_vocos_stream(b2a_vocos* h);
int32_t b2a_vocos_decode(b2a_vocos* h, const float* features, int32_t batch, int32_t frames, float* wave);
int32_t b2a_vocos_decode_dev(b2a_vocos* h, const float* d_features, int32_t batch, int32_t frames, float* d_wave, void* stream);
int32_t b2a_vocos_decode_cond(b2a_vocos* h, const float* features, const float* cond, int32_t batch, int32_t frames, float* wave);
void b2a_vocos_destroy(b2a_vocos* h);

/* ------------------------------------------------------------------ Encodec decode and encode
 * Replaces class Encodec (Sources/MLXAudioCodecs/Encodec/Encodec.swift:170-402) behind AudioCodecModel /
 * AudioDecoderModel (Sources/MLXAudioCodecs/AudioCodecModel.swift:4-27, conformance at Encodec.swift:447-461):
 *   Encodec(config:) + fromModelDirectory weights (:405-431; keys quantizer.layers.N.codebook.embed,
 *     decoder.layers.N.{conv,lstm.L.{Wx,Wh,bias},block.{1,3}.conv,shortcut.conv}.*, MLX layouts:
 *     Conv1d / ConvTranspose1d [out, k, in], LSTM [4H, in]; encoder.layers.N.* in the same layouts, loaded
 *     only when present)                                                       -> b2a_encodec_create
 *   decode(_ audioCodes:_ audioScales:paddingMask:) / decodeAudio (:366-402,458-460) -> b2a_encodec_decode
 * audio_codes are [n_chunks, B, n_q, T] int32 (n_q <= the codebooks the checkpoint holds: the bandwidth chosen at encode
 * time), audio_scales [n_chunks, B] float32 or NULL (nil scales); the waveform is [B, samples, audio_channels] with
 * samples = b2a_encodec_output_length(n_chunks, T) (T*hop un-chunked; stride*(n_chunks-1) + T*hop with linearOverlapAdd).
 * The padding-mask truncation (:397-399) is a host-side slice of the result.  The reference's fatalError on
 * "Expected one frame" (:375-377) is B2A_ERR_AUDIO_DECODING_FAILED here.  norm_type 0 is "weight_norm" (plain folded conv
 * weights, no norm layer: EncodecLayers.swift:133-137); 1 is "time_group_norm" (the 48 kHz stereo model): plain conv weights,
 * each conv followed by GroupNorm(1, C_out) with eps 1e-5 whose affine is the checkpoint's <conv prefix>norm.weight / norm.bias
 * [C_out] (EncodecLayers.swift:128-132, 244-248); statistics are per chunk and clip, so no output is causal.  Any other value
 * is B2A_ERR_INVALID_INPUT, and so is norm_type 1 over a checkpoint with no norm layers (no decoder.layers.0.norm.weight):
 * config.json does not describe those weights.  A checkpoint with norm layers that lacks one of them is
 * B2A_ERR_MODEL_NOT_INITIALIZED naming the tensor (stricter than the reference's loader, which would keep gamma 1, beta 0). */
typedef struct b2a_encodec_config {
    int32_t audio_channels;
    int32_t num_filters;
    int32_t kernel_size;
    int32_t num_residual_layers;
    int32_t dilation_growth_rate;
    int32_t codebook_size;
    int32_t codebook_dim;
    int32_t hidden_size;
    int32_t num_lstm_layers;
    int32_t residual_kernel_size;
    int32_t use_causal_conv;
    int32_t pad_mode_reflect;       /* 1 = "reflect" (clamped indices, EncodecLayers.swift:160-186), 0 = zero padding */
    int32_t norm_type;              /* 0 = weight_norm, 1 = time_group_norm; anything else -> invalidInput */
    int32_t last_kernel_size;
    int32_t compress;
    int32_t n_upsampling_ratios;
    int32_t upsampling_ratios[8];
    int32_t sampling_rate;
    int32_t use_conv_shortcut;
    float trim_right_ratio;
    float chunk_length_s;           /* <= 0: nil (one frame) */
    float overlap;                  /* < 0: nil */
    int32_t normalize;              /* encode divides each chunk by its RMS scale (Encodec.swift:224-231); decode ignores it */
} b2a_encodec_config;

typedef struct b2a_encodec b2a_encodec;
int32_t b2a_encodec_create(int32_t device, const b2a_encodec_config* cfg, const b2a_tensor* tensors, int32_t n_tensors,
                           b2a_encodec** out);
int64_t b2a_encodec_output_length(const b2a_encodec* h, int32_t n_chunks, int32_t frames);
int32_t b2a_encodec_num_codebooks(const b2a_encodec* h);
void* b2a_encodec_stream(b2a_encodec* h);
int32_t b2a_encodec_decode(b2a_encodec* h, const int32_t* audio_codes, int32_t n_chunks, int32_t batch, int32_t n_q,
                           int32_t frames, const float* audio_scales, float* wave);
int32_t b2a_encodec_decode_dev(b2a_encodec* h, const int32_t* d_audio_codes, int32_t n_chunks, int32_t batch, int32_t n_q,
                               int32_t frames, const float* d_audio_scales, float* d_wave, void* stream);
/* Encode side (AudioCodecModel.encodeAudio, Encodec.swift:457-460):
 *   EncodecEncoder (:17-88) + the residual quantizer's encode (EncodecQuantization.swift:22-38, 90-115)
 *   encodeFrame / encode (:212-291)                                             -> b2a_encodec_encode
 * audio is [B, samples, audio_channels] float32; codes are [n_chunks, B, n_q, frames] int32 with n_chunks and frames from
 * b2a_encodec_encoded_shape.  n_q is getNumQuantizersForBandwidth(bandwidth) of the caller's bandwidth (the Python wrapper
 * maps target_bandwidths); it must be in [1, the codebooks the checkpoint holds].  Chunking follows encode's loop: chunk c
 * covers samples [c*stride, c*stride + chunk_length); every chunk must have the same length (the reference's MLX.stacked
 * cannot stack a short last chunk).  With normalize, scales [n_chunks, B] receives each chunk's sqrt(mean_t(mono^2)) + 1e-8
 * (NULL allowed); without it scales is not touched (nil scales).  The padding mask only multiplies the audio ahead of the
 * normalisation, so callers apply it on the host.  Needs the checkpoint's encoder.* tensors: a decoder-only handle returns
 * B2A_ERR_MODEL_NOT_INITIALIZED.  The reference's fatalErrors, a bad n_q, empty input, ragged chunks and sizes whose index
 * arithmetic would overflow are B2A_ERR_INVALID_INPUT.  The code search is ordered fp32 (dot, |x|^2, |e|^2 each summed over
 * d in order without FMA contraction; lowest index on ties), so the codes are reproducible bit for bit, and a batch gives
 * the codes of its clips encoded one by one. */
int32_t b2a_encodec_encoded_shape(const b2a_encodec* h, int64_t samples, int32_t* n_chunks, int32_t* frames);
int32_t b2a_encodec_encode(b2a_encodec* h, const float* audio, int32_t batch, int64_t samples, int32_t n_q, int32_t* codes,
                           float* scales);
/* the same on DEVICE pointers, enqueued on `stream` (NULL: the handle's stream), no host synchronisation */
int32_t b2a_encodec_encode_dev(b2a_encodec* h, const float* d_audio, int32_t batch, int64_t samples, int32_t n_q, int32_t* d_codes,
                               float* d_scales, void* stream);
void b2a_encodec_destroy(b2a_encodec* h);

/* ------------------------------------------------------------------ Whisper STT
 * Replaces class WhisperModel (Sources/MLXAudioSTT/Models/Whisper/WhisperModel.swift:7-309) behind
 * STTGenerationModel (Sources/MLXAudioSTT/Generation.swift:52-64):
 *   fromDirectory / sanitize (:321-382)           -> b2a_stt_create (config + HF-named tensors: conv weights in the
 *                                                    PyTorch [out,in,k] layout, matrices bf16 or fp32 (rounded to bf16))
 *   model.encoder(features) (WhisperLayers.swift:146-155) -> b2a_stt_encode          (parity hook)
 *   model.decoder(tokens:...) + projectToVocab     -> b2a_stt_decoder_logits          (parity hook, after an encode)
 *   generate(audio:) / transcribeChunk (:36,186-282) -> b2a_stt_transcribe: B independent <=30 s clips
 *     ("batched == serial"; the reference transcribes one chunk at a time), greedy decode with the reference's
 *     suppress masks; returns token ids (detokenisation stays with the host tokenizer).  The 30 s chunking of
 *     longer audio (:165-182) is the caller's loop.
 * pcm is [B, n_samples] float32 16 kHz mono, every clip padded / trimmed to 30 s like WhisperAudio.padOrTrimToWindow. */
typedef struct b2a_whisper_config {
    int32_t vocab_size;
    int32_t num_mel_bins;
    int32_t d_model;
    int32_t encoder_layers;
    int32_t encoder_attention_heads;
    int32_t encoder_ffn_dim;
    int32_t max_source_positions;
    int32_t decoder_layers;
    int32_t decoder_attention_heads;
    int32_t decoder_ffn_dim;
    int32_t max_target_positions;
    int32_t max_batch; /* <= 16 clips per call */
} b2a_whisper_config;

/* STTGenerateParameters as used by transcribeChunk + WhisperGenerationConfig's suppress lists */
typedef struct b2a_stt_params {
    int32_t max_tokens;           /* defaultGenerationParameters: max_target_positions - 16 */
    float temperature;            /* 0: greedy argmax (lowest index wins ties); > 0: categorical(logits / T), WhisperModel.swift:284-291 */
    const int32_t* prompt_ids;    /* decoder prefix from buildPromptTokens (WhisperTokenizer.swift:98-113) */
    int32_t n_prompt;
    const int32_t* begin_suppress; /* suppressed at step 0 only (default [endOfText]) */
    int32_t n_begin_suppress;
    const int32_t* suppress;      /* suppressed at every step */
    int32_t n_suppress;
    int32_t timestamp_begin;      /* ids >= this are always suppressed (WhisperModel.swift:236) */
    int32_t eot;                  /* end-of-text id: stops a clip */
    uint64_t seed;                /* temperature > 0: the draw of (clip b, step s) is a pure function of (seed, b, s) */
} b2a_stt_params;

typedef struct b2a_stt_info {
    int32_t prompt_tokens;
    int32_t generation_tokens;
    int32_t decode_steps;
    double encode_time; /* log-mel + encoder + cross K/V */
    double decode_time;
    double total_time;
} b2a_stt_info;

typedef struct b2a_stt b2a_stt;
int32_t b2a_stt_create(int32_t device, const b2a_whisper_config* cfg, const b2a_tensor* tensors,
                       int32_t n_tensors, b2a_stt** out);
void* b2a_stt_stream(b2a_stt* h);
/* enc_out [B, 1500, d_model] float32 (host) */
int32_t b2a_stt_encode(b2a_stt* h, const float* pcm, int32_t batch, int64_t n_samples, float* enc_out);
/* tokens [B, T] teacher-forced from position 0 against the last encode; logits_out [B, T, vocab] (host) */
int32_t b2a_stt_decoder_logits(b2a_stt* h, const int32_t* tokens, int32_t batch, int32_t len, float* logits_out);
/* tokens_out [B, params->max_tokens], n_tokens_out [B] (host) */
int32_t b2a_stt_transcribe(b2a_stt* h, const float* pcm, int32_t batch, int64_t n_samples, const b2a_stt_params* params,
                           int32_t* tokens_out, int32_t* n_tokens_out, b2a_stt_info* info);
int32_t b2a_stt_transcribe_dev(b2a_stt* h, const float* d_pcm, int32_t batch, int64_t n_samples,
                               const b2a_stt_params* params, int32_t* tokens_out, int32_t* n_tokens_out, b2a_stt_info* info);
/* generate(audio:) beyond one window (WhisperModel.swift:95-182, chunkAudioFor30sWindows :165-182): consecutive 30 s windows of one
 * mono 16 kHz signal, transcribed as a BATCH (the reference loops over them); tokens_out [n_chunks, params->max_tokens],
 * n_tokens_out / offsets_s [n_chunks] (offsets_s nullable), *n_chunks_out = ceil(n / 480000) <= max_chunks. */
int32_t b2a_stt_transcribe_long(b2a_stt* h, const float* pcm, int64_t n_samples, const b2a_stt_params* params, int32_t max_chunks,
                                int32_t* tokens_out, int32_t* n_tokens_out, float* offsets_s, int32_t* n_chunks_out,
                                b2a_stt_info* info);
int32_t b2a_stt_cancel(b2a_stt* h);
void b2a_stt_destroy(b2a_stt* h);

/* ---- SURVEY.md section 8f row N3: the streaming STT session around the model ------------------------------------------------------
 * Sources/MLXAudioSTT/Streaming/StreamingInferenceSession.swift:589-950 (the core that drives `any STTGenerationModel` through
 * streamingDecodeTokenIds(audio:config:confirmedTokenIds:)) and StreamingTypes.swift:36-92 (StreamingConfig, DelayPreset), at the token
 * level: the host keeps the tokenizer, the text de-duplication of the window overlap and the AsyncStream of TranscriptionEvents; it calls
 * feed() from feedAudio(samples:) and stop() from stop(), passing its own clock (Date().timeIntervalSinceReferenceDate).
 *   feed : samples join the pending buffer.  A whole window (window_s) pending -> it is frozen (the buffer keeps its last
 *          window_overlap_s), decoded once without a prefix, and its tokens become completed window n (kind 2); confirmed / provisional
 *          tokens are cleared.  Otherwise, with >= 0.5 s pending and max(0.2, decode_interval_s) since the last pass, the whole pending
 *          buffer is decoded with the confirmed tokens as a forced decoder prefix (kind 1) and promoteTokens runs: a provisional
 *          position keeps its first-seen time and gains an agreement while it repeats the previous pass; the longest prefix older than
 *          delay_ms AND agreed on by min_agreement_passes passes moves to the confirmed list.  At most one decode pass per call.
 *   stop : what is pending is decoded as a last window; left-over provisional tokens are confirmed (kind 3).
 * Decode passes run synchronously on the model's stream (the reference detaches a Task and drops feeds that arrive while one runs).  */
typedef struct b2a_stt_stream_config {
    double decode_interval_s;     /* StreamingConfig.decodeIntervalSeconds, 1.0 */
    double window_s;              /* 8.0: the reference freezes 8 s windows */
    double window_overlap_s;      /* encoderWindowOverlapSeconds, 1.0 */
    int32_t delay_ms;             /* DelayPreset.delayMs: realtime 200, agent 480 (default), subtitle 2400 */
    int32_t min_agreement_passes; /* minAgreementPasses, 2 */
    int32_t max_tokens_per_pass;  /* maxTokensPerPass, 512 (clamped to what the decoder context leaves after the prefix) */
    int32_t sample_rate;          /* 16000 */
} b2a_stt_stream_config;

typedef struct b2a_stt_stream_update {
    int32_t kind;                 /* 0 nothing ran, 1 partial pass, 2 window finalised, 3 ended */
    int32_t promoted;             /* tokens moved provisional -> confirmed by this pass */
    int32_t completed_windows;    /* finalised windows so far (their tokens: b2a_stt_session_tokens(which = 0, window)) */
    int32_t n_confirmed;          /* confirmed tokens of the current (pending) window */
    int32_t n_provisional;
    double total_audio_s;         /* StreamingStats.totalAudioSeconds */
    double pass_encode_time;      /* of the pass this call ran (0 when none) */
    double pass_decode_time;
} b2a_stt_stream_update;

/* A host-side decoder (the reference accepts `any STTGenerationModel`, :162): writes the continuation AFTER `prefix` for `pcm`. */
typedef int32_t (*b2a_stt_decode_cb)(void* user, const float* pcm, int64_t n_samples, const int32_t* prefix, int32_t n_prefix,
                                     int32_t* tokens_out, int32_t capacity, int32_t* n_tokens_out);

typedef struct b2a_stt_session b2a_stt_session;
/* params: the decode parameters of every pass (prompt / suppress lists are copied; max_tokens is replaced by max_tokens_per_pass) */
int32_t b2a_stt_session_create(b2a_stt* model, const b2a_stt_params* params, const b2a_stt_stream_config* config, b2a_stt_session** out);
int32_t b2a_stt_session_create_with_decoder(b2a_stt_decode_cb decode, void* user, const b2a_stt_stream_config* config, b2a_stt_session** out);
int32_t b2a_stt_session_feed(b2a_stt_session* s, const float* pcm, int64_t n_samples, double now_s, b2a_stt_stream_update* update);
int32_t b2a_stt_session_stop(b2a_stt_session* s, double now_s, b2a_stt_stream_update* update);
/* which: 0 = completed window `window`, 1 = confirmed, 2 = provisional; *n_out = the list's length (written even when capacity is short) */
int32_t b2a_stt_session_tokens(b2a_stt_session* s, int32_t which, int32_t window, int32_t* tokens_out, int32_t capacity, int32_t* n_out);
void b2a_stt_session_destroy(b2a_stt_session* s);

/* ------------------------------------------------------------------ Qwen3-TTS speech-tokenizer decoder (SURVEY.md section 8f row N1)
 * Replaces Qwen3TTSSpeechTokenizerDecoder and the decode entry points of Qwen3TTSSpeechTokenizer
 * (Sources/MLXAudioTTS/Models/Qwen3TTS/Qwen3TTSSpeechTokenizer.swift):
 *   init(config:) + sanitized weights (keys below the "decoder." module, MLX layouts)  -> create
 *   resetStreamingState (:949-970)                                                       -> reset
 *   streamingStep (:973-1008)                                                            -> streaming_step[_dev]
 *   streamingDecode(chunkTokens:) (:1070-1092, what decodeChunk uses, Qwen3TTS.swift:214-231) -> streaming_decode
 *   chunkedDecode(chunkSize:leftContextSize:) (:1010-1024, used by decode :1059-1068)   -> chunked_decode
 * codes are [B, num_quantizers given, T] int32 (the decoder's own layout, i.e. audioCodes transposed (0, 2, 1)); the
 * waveform is [B, T * total_upsample] float32 in [-1, 1].  Config defaults: Qwen3TTSConfig.swift:358-385.            */
typedef struct b2a_speech_tokenizer_config {
    int32_t codebook_size;
    int32_t codebook_dim;
    int32_t latent_dim;
    int32_t decoder_dim;
    int32_t hidden_size;
    int32_t intermediate_size;
    int32_t head_dim;
    int32_t num_attention_heads;
    int32_t num_key_value_heads;
    int32_t num_hidden_layers;
    int32_t num_quantizers;
    int32_t num_semantic_quantizers;
    float rms_norm_eps;
    float rope_theta;
    int32_t attention_bias;
    int32_t num_upsample_rates;
    int32_t upsample_rates[8];
    int32_t num_upsampling_ratios;
    int32_t upsampling_ratios[8];
    int32_t max_batch;        /* rows decoded together */
    int32_t max_cache_frames; /* code frames one stream may span (the reference's cache is unbounded) */
} b2a_speech_tokenizer_config;

typedef struct b2a_speech_tokenizer b2a_speech_tokenizer;
int32_t b2a_speech_tokenizer_create(int32_t device, const b2a_speech_tokenizer_config* cfg, const b2a_tensor* tensors,
                                    int32_t n_tensors, b2a_speech_tokenizer** out);
int32_t b2a_speech_tokenizer_total_upsample(const b2a_speech_tokenizer* h);
void* b2a_speech_tokenizer_stream(b2a_speech_tokenizer* h);
int32_t b2a_speech_tokenizer_reset(b2a_speech_tokenizer* h);
int32_t b2a_speech_tokenizer_streaming_step(b2a_speech_tokenizer* h, const int32_t* codes, int32_t batch, int32_t num_groups,
                                            int32_t frames, float* wave);
int32_t b2a_speech_tokenizer_streaming_step_dev(b2a_speech_tokenizer* h, const int32_t* d_codes, int32_t batch, int32_t num_groups,
                                                int32_t frames, float* d_wave, void* stream);
int32_t b2a_speech_tokenizer_streaming_decode(b2a_speech_tokenizer* h, const int32_t* codes, int32_t batch, int32_t num_groups,
                                              int32_t frames, int32_t chunk_tokens, float* wave);
int32_t b2a_speech_tokenizer_chunked_decode(b2a_speech_tokenizer* h, const int32_t* codes, int32_t batch, int32_t num_groups,
                                            int32_t frames, int32_t chunk_size, int32_t left_context, float* wave);
void b2a_speech_tokenizer_destroy(b2a_speech_tokenizer* h);
/* Loading (host-only except the final create): the decoder half of Qwen3TTSSpeechTokenizer.sanitize (:1094-1440) on an open
 * checkpoint -- prefixes stripped, PyTorch conv / transposed-conv layouts moved to MLX's with the reference's shape heuristic
 * (checkArrayShapeQwen3 :1445-1455), upsample.X.Y -> upsample.X.layers.Y, codebook statistics kept, encoder.* and speaker-encoder
 * keys dropped, the leading "decoder." removed; Qwen3TTSTokenizerConfig decoding (Qwen3TTSConfig.swift:358-385,518-527; a missing
 * config.json means defaults, Qwen3TTS.swift:1246-1255); loadSpeechTokenizer (Qwen3TTS.swift:1244-1275).                       */
int32_t b2a_weights_sanitize_speech_tokenizer(b2a_weights* w);
int32_t b2a_speech_tokenizer_config_from_json(const char* config_path, int32_t max_batch, int32_t max_cache_frames,
                                              b2a_speech_tokenizer_config* cfg, int32_t* decode_upsample_rate);
int32_t b2a_speech_tokenizer_create_from_directory(const char* dir, int32_t device, int32_t max_batch, int32_t max_cache_frames,
                                                   b2a_speech_tokenizer** out, int32_t* decode_upsample_rate);
/* ------------------------------------------------------------------ Qwen3-TTS talker + code predictor (SURVEY.md section 8f row N1)
 * Replaces the autoregressive half of class Qwen3TTSModel (Sources/MLXAudioTTS/Models/Qwen3TTS/):
 *   Qwen3TTSTalkerForConditionalGeneration (Qwen3TTSTalker.swift:127-366: per-head q/k RMSNorm before RoPE, interleaved 3-section
 *     MRoPE -- all three position rows are equal for the text-only prompts the reference builds, where it is plain rotate-half
 *     RoPE --, inputs are EMBEDDINGS, codec_head)                                               -> the 28-layer stack
 *   Qwen3TTSCodePredictor (Qwen3TTSCodePredictor.swift:14-243: 5 layers, 15 lm heads / embeddings, cache reset every frame) -> the
 *     inner 15-step loop
 *   the frame loop of generate (Qwen3TTS.swift:380-495: talker step -> sampleToken -> 15 predictor steps -> summed-embedding
 *     feedback `text + codec_embed(c0) + sum_i predictor_embed_i(c_i+1)`) and sampleToken (:1003-1118) -> b2a_qwen3_talker_generate:
 *     ONE CUDA graph per 12.5 Hz frame, nothing syncs with the host inside it
 *   text_projection(text_embedding(ids)) / codec_embedding(ids) (:898-999, prepareGenerationInputs) -> b2a_qwen3_talker_embed_text /
 *     _embed_codec: the host composes the prompt from these rows exactly as prepareGenerationInputs does (tokenisation, the chat
 *     template and the special-token ids stay with the host, SURVEY.md 8b)
 * Weights: the reference's keys after sanitize strips "talker." (model.layers.N.*, model.codec_embedding.weight,
 * model.text_embedding.weight, text_projection.linear_fc{1,2}.{weight,bias}, codec_head.weight, code_predictor.model.layers.N.*,
 * code_predictor.model.codec_embedding.I.weight, code_predictor.lm_head.I.weight), bf16 or f32 (rounded to bf16: the engine holds
 * bf16 matrices; an MLX affine-quantised (8-bit) checkpoint is expanded by b2a_weights_dequantize first).  head_dim must be 128.
 * When cp_hidden_size != hidden_size (the 1.7B checkpoints: 2048 -> 1024) the checkpoint must also hold
 * code_predictor.small_to_mtp_projection.{weight [cp_hidden, hidden], bias [cp_hidden]} (else B2A_ERR_MODEL_NOT_INITIALIZED), applied
 * to every predictor input as the reference does (Qwen3TTSCodePredictor.swift:200-238); the lm heads are [cp_vocab, cp_hidden] and
 * the predictor's codec_embedding.I stay [cp_vocab, hidden].  The projected embedding tables are precomputed at creation in fp32:
 * (vocab + (num_code_groups - 2) * cp_vocab) * cp_hidden * 4 bytes of device memory, about 130 MB at 1.7B.                    */
typedef struct b2a_qwen3_talker_config {
    int32_t vocab_size;            /* codec vocabulary (3072) */
    int32_t hidden_size;
    int32_t intermediate_size;
    int32_t num_hidden_layers;
    int32_t num_attention_heads;
    int32_t num_key_value_heads;
    int32_t head_dim;
    float rms_norm_eps;
    float rope_theta;
    int32_t num_code_groups;       /* 16: one talker code + 15 predictor codes per frame */
    int32_t text_hidden_size;
    int32_t text_vocab_size;
    int32_t codec_eos_token_id;
    int32_t cp_vocab_size;         /* code predictor (Qwen3TTSConfig.swift:45-63) */
    int32_t cp_hidden_size;
    int32_t cp_intermediate_size;
    int32_t cp_num_hidden_layers;
    int32_t cp_num_attention_heads;
    int32_t cp_num_key_value_heads;
    int32_t cp_head_dim;
    float cp_rms_norm_eps;
    float cp_rope_theta;
    int32_t max_batch;             /* 1..32 utterances per call */
    int32_t max_context;           /* prompt embeddings + frames per utterance */
} b2a_qwen3_talker_config;

/* Qwen3TTS generate's sampling parameters (Qwen3TTS.swift:360-385; sampleToken :1003-1118) */
typedef struct b2a_qwen3_gen_params {
    int32_t max_tokens;            /* frames; the caller applies min(maxTokens, max(75, 6 * text tokens)) (:380) */
    float temperature;             /* <= 0: greedy argmax (lowest index wins ties) for the talker code AND the predictor codes */
    float top_p;
    int32_t top_k;
    float min_p;
    float repetition_penalty;      /* talker code only, over the unique codes generated so far */
    uint64_t seed;
} b2a_qwen3_gen_params;

typedef struct b2a_qwen3_talker b2a_qwen3_talker;
int32_t b2a_qwen3_talker_create(int32_t device, const b2a_qwen3_talker_config* cfg, const b2a_tensor* tensors, int32_t n_tensors,
                                b2a_qwen3_talker** out);
void* b2a_qwen3_talker_stream(b2a_qwen3_talker* h);
/* out [n, hidden] float32 (host): text_projection(text_embedding(ids)) resp. codec_embedding(ids) */
int32_t b2a_qwen3_talker_embed_text(b2a_qwen3_talker* h, const int32_t* ids, int32_t n, float* out);
int32_t b2a_qwen3_talker_embed_codec(b2a_qwen3_talker* h, const int32_t* ids, int32_t n, float* out);
/* codecEmbedIcl's frame rows (Qwen3TTS.swift:249-265), the reference-code part of a voice-cloning (ICL) prompt: codes [n, groups]
 * int32 (row r = frame r's first `groups` code groups, 1 <= groups <= num_code_groups; fewer groups than num_code_groups is the
 * reference's `break`) -> out [n, hidden] = codec_embedding(c0) + sum over g = 1 .. groups-1 of code_predictor.codec_embedding[g-1](c_g),
 * the same sum the frame loop feeds back.  The leading codec_bos row is the caller's (b2a_qwen3_talker_embed_codec).          */
int32_t b2a_qwen3_talker_embed_code_frames(b2a_qwen3_talker* h, const int32_t* codes, int32_t n, int32_t groups, float* out);
/* Parity hook: the talker over input_embeds [B, L, hidden] from an empty cache -> codec logits of the LAST position
 * [B, vocab] and its final-norm hidden state [B, hidden] (Qwen3TTSTalker.swift:340-350).                                   */
int32_t b2a_qwen3_talker_forward(b2a_qwen3_talker* h, const float* input_embeds, int32_t batch, int32_t len, float* logits_out,
                                 float* hidden_out);
/* The frame loop.  input_embeds [B, L, hidden] (every row the same L), trailing_text_hidden [B, n_trailing_max, hidden] with
 * n_trailing[B] valid rows each (one is consumed per frame, then tts_pad_embed [hidden] is used), codes_out [B, max_tokens,
 * num_code_groups] int32, n_frames_out[B].  A row stops after the frame whose talker code is codec_eos_token_id (that frame is not
 * emitted, :424-428) or at max_tokens.  on_frame (nullable) is called on the calling thread for every emitted frame with the
 * frame's num_code_groups codes -- the hook a streaming caller decodes audio chunks from (generateStream, Qwen3TTS.swift:500-569). */
typedef void (*b2a_frame_cb)(void* user, int32_t utterance, int32_t frame, const int32_t* codes);
int32_t b2a_qwen3_talker_generate(b2a_qwen3_talker* h, const float* input_embeds, int32_t batch, int32_t len,
                                  const float* trailing_text_hidden, const int32_t* n_trailing, int32_t n_trailing_max,
                                  const float* tts_pad_embed, const b2a_qwen3_gen_params* params, int32_t* codes_out,
                                  int32_t* n_frames_out, b2a_gen_info* info, b2a_frame_cb on_frame, void* user);
/* Loading (Qwen3TTSModel.fromModelDirectory, Qwen3TTS.swift:1136-1175, talker half): config.json's "talker_config" (+ nested
 * "code_predictor_config", defaults of Qwen3TTSConfig.swift:45-63,268-292) -> the config struct; every *.safetensors of the directory
 * -> keep "talker.*" and strip the prefix (Qwen3TTSTalker.swift:356-365) -> MLX affine de-quantisation of every layer that carries
 * ".scales" as config.json's "quantization" block says (:1156-1171; 8-bit group-64 for the shipped 8-bit checkpoints) -> create.     */
int32_t b2a_qwen3_talker_config_from_json(const char* config_path, int32_t max_batch, int32_t max_context, b2a_qwen3_talker_config* cfg);
int32_t b2a_weights_sanitize_qwen3_talker(b2a_weights* w, const char* config_path /* nullable: no quantisation */);
int32_t b2a_qwen3_talker_create_from_directory(const char* model_dir, int32_t device, int32_t max_batch, int32_t max_context,
                                               b2a_qwen3_talker** out);
int32_t b2a_qwen3_talker_cancel(b2a_qwen3_talker* h);
void b2a_qwen3_talker_destroy(b2a_qwen3_talker* h);

/* ------------------------------------------------------------------ Qwen3-TTS speech-tokenizer ENCODER (24 kHz audio -> 12.5 Hz codes)
 * Replaces Qwen3TTSSpeechTokenizerEncoder.encode (Sources/MLXAudioTTS/Models/Qwen3TTS/Qwen3TTSSpeechTokenizer.swift:790-884), the
 * speechTokenizer.encode(refAudio) step of the in-context-learning (voice-cloning) prompt (Qwen3TTS.swift:267-302): the Mimi
 * SEANet encoder (causal, zero padding), the 8-layer transformer (interleaved RoPE, full causal attention over the clip), the
 * edge-padded stride-2 downsample and the split residual quantizer's code search, cut to valid_num_quantizers code groups.
 * audio is [B, 1, n] float32 (mono 24 kHz), codes are [B, valid_num_quantizers, encoded_length(n)] int32.
 * A separate handle from the decoder's b2a_speech_tokenizer, so b2a_speech_tokenizer_config keeps its layout.  Config defaults:
 * Qwen3TTSConfig.swift:391-494 and encoder_valid_num_quantizers (:518-527).  Errors: a checkpoint without encoder tensors ->
 * B2A_ERR_MODEL_NOT_INITIALIZED (the reference's hasEncoder == false); empty audio -> B2A_ERR_AUDIO_ENCODING_FAILED; audio_channels
 * != 1, num_residual_layers != 1, a geometry the device path does not run, sizes whose indices would overflow ->
 * B2A_ERR_INVALID_INPUT.  Deterministic: the same input gives the same codes, batched or one row at a time.                  */
typedef struct b2a_speech_tokenizer_encoder_config {
    int32_t sampling_rate;
    float frame_rate;
    int32_t audio_channels;
    int32_t num_filters;
    int32_t num_residual_layers;
    int32_t num_upsampling_ratios;
    int32_t upsampling_ratios[8]; /* the decoder order; the encoder runs them reversed */
    int32_t kernel_size;
    int32_t residual_kernel_size;
    int32_t last_kernel_size;
    int32_t compress;
    int32_t use_causal_conv;
    int32_t use_conv_shortcut;
    int32_t hidden_size;
    int32_t intermediate_size;
    int32_t num_hidden_layers;
    int32_t num_attention_heads;
    int32_t num_key_value_heads;
    int32_t head_dim;
    float rope_theta;
    int32_t codebook_size;
    int32_t codebook_dim;
    int32_t num_quantizers;
    int32_t valid_num_quantizers; /* encoder_valid_num_quantizers: the code groups encode returns */
} b2a_speech_tokenizer_encoder_config;

typedef struct b2a_speech_tokenizer_encoder b2a_speech_tokenizer_encoder;
/* tensors: b2a_weights_sanitize_speech_tokenizer_encoder's keys (encoder.*, encoder_transformer.*, downsample.*, quantizer.*) */
int32_t b2a_speech_tokenizer_encoder_create(int32_t device, const b2a_speech_tokenizer_encoder_config* cfg, const b2a_tensor* tensors,
                                            int32_t n_tensors, b2a_speech_tokenizer_encoder** out);
/* code frames for n samples: ceil(ceil(n / 960) / 2) at the shipped geometry (0 for n < 1 or a null handle) */
int64_t b2a_speech_tokenizer_encoder_encoded_length(const b2a_speech_tokenizer_encoder* h, int64_t n_samples);
int32_t b2a_speech_tokenizer_encoder_num_code_groups(const b2a_speech_tokenizer_encoder* h);
int32_t b2a_speech_tokenizer_encoder_encode(b2a_speech_tokenizer_encoder* h, const float* audio, int32_t batch, int64_t n_samples,
                                            int32_t* codes);
/* device buffers, enqueued on `stream` (NULL: the handle's stream) without a host synchronisation */
int32_t b2a_speech_tokenizer_encoder_encode_dev(b2a_speech_tokenizer_encoder* h, const float* d_audio, int32_t batch, int64_t n_samples,
                                                int32_t* d_codes, void* stream);
void* b2a_speech_tokenizer_encoder_stream(b2a_speech_tokenizer_encoder* h);
void b2a_speech_tokenizer_encoder_destroy(b2a_speech_tokenizer_encoder* h);
/* Loading: the encoder half of Qwen3TTSSpeechTokenizer.sanitize (:1093-1440) on an open checkpoint (encoder.encoder.layers.N ->
 * SEANet paths, separate or fused q|k|v -> in_proj, norms, layer scales, downsample, semantic_/acoustic_residual_vector_quantizer
 * or rvq_first/rvq_rest -> rvq_first/rvq_rest with their codebook statistics; every other key dropped); config.json's
 * "encoder_config" and "encoder_valid_num_quantizers" (a missing file or block -> B2A_ERR_MODEL_NOT_INITIALIZED); both from a
 * directory.                                                                                                                  */
int32_t b2a_weights_sanitize_speech_tokenizer_encoder(b2a_weights* w);
int32_t b2a_speech_tokenizer_encoder_config_from_json(const char* config_path, b2a_speech_tokenizer_encoder_config* cfg);
int32_t b2a_speech_tokenizer_encoder_create_from_directory(const char* dir, int32_t device, b2a_speech_tokenizer_encoder** out);

/* ---- Qwen3-TTS speaker encoder (Qwen3TTSSpeakerEncoder.swift, an ECAPA-TDNN): the x-vector a Base checkpoint's voice-cloning
 * prompt carries in its codec prefix (Qwen3TTS.swift:820-823).  audio [B, n] float32 at sample_rate -> log-mel
 * (computeMelSpectrogram with n_fft 1024, hop 256, 128 mels; b2a_logmel kind 0) [B, T = 1 + n / 256, 128] -> TDNN block ->
 * SE-Res2Net blocks -> multi-layer feature aggregation -> attentive statistics pooling -> fc -> [B, enc_dim].  fp32 throughout;
 * every reduction over time has a fixed order and no atomics, so a clip's embedding does not depend on the batch it runs in.
 * Config defaults: Qwen3TTSConfig.swift:92-103.  Errors: mel_dim != 128, lists of unequal length (config_from_json), a channel count
 * not divisible by enc_res2net_scale (or whose chunks are not a multiple of 4 channels), sum(enc_channels[1:-1]) !=
 * enc_channels[-1], an SE-Res2Net block whose input and output widths differ, (k - 1) * d odd, empty audio, n <= 512 samples,
 * T <= max((k - 1) * d / 2) frames -> B2A_ERR_INVALID_INPUT; no or partial weights -> B2A_ERR_MODEL_NOT_INITIALIZED.          */
typedef struct b2a_qwen3_speaker_encoder_config {
    int32_t mel_dim;
    int32_t enc_dim;
    int32_t num_enc_layers;        /* entries used in each of the three lists below (3..8) */
    int32_t enc_channels[8];
    int32_t enc_kernel_sizes[8];
    int32_t enc_dilations[8];
    int32_t enc_attention_channels;
    int32_t enc_res2net_scale;
    int32_t enc_se_channels;
    int32_t sample_rate;
} b2a_qwen3_speaker_encoder_config;

typedef struct b2a_qwen3_speaker_encoder b2a_qwen3_speaker_encoder;
/* tensors: b2a_weights_sanitize_qwen3_speaker_encoder's keys (blocks.*, mfa.*, asp.*, fc.*) in MLX layout ([out, k, in]) */
int32_t b2a_qwen3_speaker_encoder_create(int32_t device, const b2a_qwen3_speaker_encoder_config* cfg, const b2a_tensor* tensors,
                                         int32_t n_tensors, b2a_qwen3_speaker_encoder** out);
/* mel frames T for n samples: 1 + n / 256 (0 for a null handle) */
int64_t b2a_qwen3_speaker_encoder_frames(const b2a_qwen3_speaker_encoder* h, int64_t n_samples);
/* host audio [B, n] -> host embeddings [B, enc_dim] */
int32_t b2a_qwen3_speaker_encoder_embed(b2a_qwen3_speaker_encoder* h, const float* audio, int32_t batch, int64_t n_samples, float* out);
/* device buffers, enqueued on `stream` (NULL: the handle's stream) without a host synchronisation */
int32_t b2a_qwen3_speaker_encoder_embed_dev(b2a_qwen3_speaker_encoder* h, const float* d_audio, int32_t batch, int64_t n_samples,
                                            float* d_out, void* stream);
/* the module's own input: host log-mel [B, T, mel_dim] -> host embeddings [B, enc_dim] */
int32_t b2a_qwen3_speaker_encoder_embed_mel(b2a_qwen3_speaker_encoder* h, const float* mel, int32_t batch, int64_t frames, float* out);
void* b2a_qwen3_speaker_encoder_stream(b2a_qwen3_speaker_encoder* h);
void b2a_qwen3_speaker_encoder_destroy(b2a_qwen3_speaker_encoder* h);
/* Loading: Qwen3TTSSpeakerEncoder.sanitize (:324-354) on an open checkpoint -- the keys after the "speaker_encoder" component, 3-D
 * ".weight" tensors that fail checkArrayShapeQwen3 transposed [out, in, k] -> [out, k, in], every other key dropped; the top-level
 * config.json's "speaker_encoder_config" (defaults for missing keys); both from a model directory, where a config whose
 * tts_model_type is not "base" or a checkpoint without speaker-encoder keys -> B2A_ERR_MODEL_NOT_INITIALIZED.                 */
int32_t b2a_weights_sanitize_qwen3_speaker_encoder(b2a_weights* w);
int32_t b2a_qwen3_speaker_encoder_config_from_json(const char* config_path, b2a_qwen3_speaker_encoder_config* cfg);
int32_t b2a_qwen3_speaker_encoder_create_from_directory(const char* model_dir, int32_t device, b2a_qwen3_speaker_encoder** out);

/* ------------------------------------------------------------------ Mimi (24 kHz audio <-> 12.5 Hz codes, streaming decoder)
 * Replaces Mimi and MimiStreamingDecoder (Sources/MLXAudioCodecs/Mimi/Mimi.swift), the codec Marvis and PocketTTS decode with.
 *   encode: audio [B, 1, n] float32 -> codes [B, num_codebooks, encoded_length(n)] int32, every level of the split quantizer.
 *           The same implementation as b2a_speech_tokenizer_encoder: the Qwen3-TTS encoder is Mimi's encoder.
 *   decode: codes [B, K, T] int32, 1 <= K <= num_codebooks, each in [0, codebook_size) -> waveform [B, 1, T * 1920] float32.  Level 0
 *           through rvq_first, levels 1 .. K-1 through rvq_rest (Quantization.swift:113-120, 203-210), the depthwise ×2 upsample, the
 *           decoder transformer over a KV cache and the SEANet decoder (ELU, transposed convs ×8/6/5/4, no output clip).
 * One code path: decode_step carries the upsample tail, every conv's history and the KV cache across calls (Mimi.decodeStep,
 * Mimi.swift:196-202); b2a_mimi_reset clears all three (MimiStreamingDecoder.reset, :215-219).  b2a_mimi_decode is a reset followed
 * by one step.  Unlike the reference's decode(), it therefore also resets the upsample tail, and it leaves its own state behind, so a
 * decode_step after it continues that clip (the reference's decode() uses the non-streaming convs and leaves their state empty).
 * Attention keeps, per call, the last T + min(context, p0) keys of the cache (p0 = positions decoded before the call,
 * Transformer.swift:156-164): query t sees cache positions [max(0, p0 - context), p0 + t].  A one-shot decode is therefore full
 * causal over the clip; a stream longer than `context` latent positions (10 s) is not, and differs from it.
 * Errors: K outside 1..num_codebooks, codes outside [0, codebook_size) (host entry points; the _dev ones clamp), batch outside
 * 1..max_batch, a stream longer than max_cache_frames code frames, a batch size that changes inside a stream, a geometry the
 * device path does not run -> B2A_ERR_INVALID_INPUT; a missing tensor -> B2A_ERR_MODEL_NOT_INITIALIZED; empty audio ->
 * B2A_ERR_AUDIO_ENCODING_FAILED.  Deterministic: a batch row's output is bit for bit the row's output alone.                   */
typedef struct b2a_mimi_config {
    int32_t sample_rate;           /* 24000 */
    float frame_rate;              /* 12.5 code frames per second */
    int32_t channels;              /* audio channels: 1 */
    /* SEANet (SeanetConfig) */
    int32_t dimension;             /* 512: latent width, also the transformer's d_model */
    int32_t n_filters;             /* 64 */
    int32_t n_residual_layers;     /* 1 (the only value the device path runs) */
    int32_t num_ratios;
    int32_t ratios[8];             /* [8, 6, 5, 4]: the decoder order; the encoder runs them reversed */
    int32_t kernel_size;           /* 7 */
    int32_t residual_kernel_size;  /* 3 */
    int32_t last_kernel_size;      /* 3 */
    int32_t dilation_base;         /* 2 (unused with one residual layer) */
    int32_t compress;              /* 2 */
    int32_t causal;                /* 1 (required) */
    int32_t true_skip;             /* 1 (required: identity residual) */
    /* transformer (TransformerConfig), used by both the encoder and the decoder transformer */
    int32_t num_heads;             /* 8 */
    int32_t num_layers;            /* 8 */
    int32_t dim_feedforward;       /* 2048 */
    int32_t context;               /* 250 latent positions */
    int32_t max_period;            /* 10000: RoPE base */
    int32_t gating;                /* 0 (required): exact-GELU MLP */
    int32_t norm_rms;              /* 0 (required): layer_norm, eps 1e-5 */
    int32_t kv_repeat;             /* 1 (required) */
    /* quantizer */
    int32_t num_codebooks;         /* nq */
    int32_t codebook_size;         /* 2048 */
    int32_t codebook_dim;          /* 256 */
    /* device path */
    int32_t max_batch;             /* decode rows per call */
    int32_t max_cache_frames;      /* code frames one stream may decode before a reset (KV cache capacity / 2) */
} b2a_mimi_config;

typedef struct b2a_mimi b2a_mimi;
/* mimi_202407(num_codebooks) (Mimi.swift:47-97) with the device-path bounds; num_codebooks < 1 or bounds < 1 -> INVALID_INPUT */
int32_t b2a_mimi_config_default(int32_t num_codebooks, int32_t max_batch, int32_t max_cache_frames, b2a_mimi_config* out);
/* tensors: b2a_weights_sanitize_mimi's keys in MLX layouts (encoder.*, encoder_transformer.*, downsample.*, quantizer.*, upsample.*,
 * decoder_transformer.*, decoder.*) */
int32_t b2a_mimi_create(int32_t device, const b2a_mimi_config* cfg, const b2a_tensor* tensors, int32_t n_tensors, b2a_mimi** out);
/* Mimi.sanitize (Mimi.swift:337-413) on an open checkpoint, key for key: "_"-prefixed segments lose the "_", encoder.model. /
 * decoder.model. -> encoder. / decoder., in_proj_weight -> in_proj.weight, linear1 / linear2 -> gating.linear1 / 2, the decoder index
 * map [2, 5, 8, 11] and the encoder's [1, 4, 7, 10], 0 / 14 -> init_conv1d / final_conv1d, .block.1. / .block.3. -> .block.0. /
 * .block.1., the last two axes of every .conv / .input_proj / .output_proj weight swapped, and .convtr weights to MLX's [out, k, in]
 * (depthwise (C, 1, k) -> (C, k, 1)).  No key is dropped.                                                                      */
int32_t b2a_weights_sanitize_mimi(b2a_weights* w);
/* Mimi.fromPretrained on a local single-file checkpoint: mimi_202407(num_codebooks), load, sanitize, create.  The codebooks are
 * embedding_sum / max(cluster_usage, 1e-5), computed once at load. */
int32_t b2a_mimi_create_from_file(const char* path, int32_t num_codebooks, int32_t device, int32_t max_batch, int32_t max_cache_frames,
                                  b2a_mimi** out);
int32_t b2a_mimi_num_codebooks(const b2a_mimi* h);
/* samples per code frame: prod(ratios) * (sample_rate / prod(ratios) / frame_rate) = 1920 at the shipped geometry (0: null handle) */
int32_t b2a_mimi_samples_per_frame(const b2a_mimi* h);
/* code frames for n samples: ceil(ceil(n / 960) / 2) at the shipped geometry (0 for n < 1 or a null handle) */
int64_t b2a_mimi_encoded_length(const b2a_mimi* h, int64_t n_samples);
int32_t b2a_mimi_encode(b2a_mimi* h, const float* audio, int32_t batch, int64_t n_samples, int32_t* codes);
int32_t b2a_mimi_encode_dev(b2a_mimi* h, const float* d_audio, int32_t batch, int64_t n_samples, int32_t* d_codes, void* stream);
/* one-shot: reset, then one step.  codes [B, K, T] -> wave [B, 1, T * samples_per_frame] */
int32_t b2a_mimi_decode(b2a_mimi* h, const int32_t* codes, int32_t batch, int32_t K, int32_t T, float* wave);
int32_t b2a_mimi_decode_dev(b2a_mimi* h, const int32_t* d_codes, int32_t batch, int32_t K, int32_t T, float* d_wave, void* stream);
/* Mimi.decodeStep: T more code frames of the current stream -> their T * samples_per_frame samples */
int32_t b2a_mimi_decode_step(b2a_mimi* h, const int32_t* codes, int32_t batch, int32_t K, int32_t T, float* wave);
int32_t b2a_mimi_decode_step_dev(b2a_mimi* h, const int32_t* d_codes, int32_t batch, int32_t K, int32_t T, float* d_wave, void* stream);
/* MimiStreamingDecoder.decodeFrames: T single-frame steps of the current stream (no reset), concatenated */
int32_t b2a_mimi_decode_frames(b2a_mimi* h, const int32_t* codes, int32_t batch, int32_t K, int32_t T, float* wave);
int32_t b2a_mimi_reset(b2a_mimi* h);
void* b2a_mimi_stream(b2a_mimi* h);
void b2a_mimi_destroy(b2a_mimi* h);

#ifdef __cplusplus
}
#endif
#endif /* B200AUDIO_H */
