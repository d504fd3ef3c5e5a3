/*
 * b200audio_internal.h -- NOT part of the drop-in boundary.  Test and benchmark hooks of libb200audio.so that have no
 * counterpart in the reference: device-side random-init constructors for BASELINE.json's full-size configurations (there are no
 * checkpoints here and a 3B-parameter host copy is pointless), fixed-work switches for bench.py, parity trace hooks and the
 * single-kernel test entries.  A Swift wrapper (INTEGRATION.md) binds include/b200audio.h only; tests/, bench.py and tools/ may
 * also bind these.
 */
#ifndef B200AUDIO_INTERNAL_H
#define B200AUDIO_INTERNAL_H

#include "b200audio.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ benchmark constructors / switches
 *   b2a_tts_create_random / b2a_stt_create_random : same as b2a_tts_create / b2a_stt_create but the weights are drawn ON THE
 *       DEVICE (N(0, std^2) bf16 from a counter-based generator, norm gains 1).
 *   b2a_tts_set_bench_flags : mask_eos != 0 -> never stop on the handle's stop token (fixed work per call); wrap_codes != 0 -> audio codes are
 *       taken mod 4096 per slot so that random-init tokens index the SNAC codebooks.  Both default to 0 (reference behaviour).
 *   b2a_stt_set_bench_flags : mask_eot != 0 -> a clip never stops on end-of-text (fixed work).
 *   b2a_tts_time_steps : runs `iters` captured decode steps for `batch` rows at context `ctx` (greedy, no host sync inside)
 *       between two CUDA events on the handle's stream; *ms_per_step = average device time of one step.                      */
int32_t b2a_tts_create_random(int32_t device, const b2a_llama_config* cfg, float std, uint64_t seed,
                              b2a_snac* snac, b2a_tts** out);
int32_t b2a_stt_create_random(int32_t device, const b2a_whisper_config* cfg, float std, uint64_t seed, b2a_stt** out);
/*   b2a_qwen3_lm_create_random : the same for a VyvoTTS handle (b2a_qwen3_lm_create); q/k norm gains are 1 too.               */
int32_t b2a_qwen3_lm_create_random(int32_t device, const b2a_qwen3_lm_config* cfg, float std, uint64_t seed, b2a_snac* snac,
                                   b2a_tts** out);
int32_t b2a_tts_set_bench_flags(b2a_tts* h, int32_t mask_eos, int32_t wrap_codes);
int32_t b2a_stt_set_bench_flags(b2a_stt* h, int32_t mask_eot);
int32_t b2a_tts_time_steps(b2a_tts* h, int32_t batch, int32_t ctx, int32_t iters, float* ms_per_step);
/*   b2a_qwen3_talker_create_random : the Qwen3-TTS talker + code predictor with device-drawn weights (BASELINE config 5 bench).
 *   b2a_qwen3_talker_set_bench_flags : mask_eos != 0 -> the talker never emits codec_eos_token_id (fixed work per call).        */
int32_t b2a_qwen3_talker_create_random(int32_t device, const b2a_qwen3_talker_config* cfg, float std, uint64_t seed, b2a_qwen3_talker** out);
int32_t b2a_qwen3_talker_set_bench_flags(b2a_qwen3_talker* h, int32_t mask_eos);

/* ------------------------------------------------------------------ parity hooks
 *   b2a_tts_debug_trace : enable != 0 makes later b2a_tts_forward_logits calls record the residual stream at every RMSNorm
 *       input; out (nullable) receives the record of the last traced position as [2*layers+1, batch, hidden] float32.        */
int32_t b2a_tts_debug_trace(b2a_tts* h, int32_t enable, int32_t batch, float* out);
/* Host-only (no device needed): dynamic shared-memory bytes per CTA of the fused decode step's kernels as the engine launches
 * them -- out[0] the decode GEMM (tc_gemm_kernel<16>), out[1] the cluster split-K GEMM, out[2] the attention kernel for `gqa`
 * q heads per kv head (1, 2, 3, 4, 6 or 8; its 512 static bytes are not included).  tests/test_gpu_step_coresidency.py checks
 * that neighbouring kernels of the step fit on one SM together.                                                              */
int32_t b2a_debug_step_smem(int32_t gqa, int32_t* out);
/* Host-only: the same for a call of `rows` rows (1..32), which runs the step at width R = 8, 16 or 32 -- out[0] R, out[1] the decode
 * GEMM's ring depth, out[2] its bytes (tc_gemm_kernel<2R>), out[3] the split-K ring depth, out[4] its bytes (clusters of 5),
 * out[5] the attention kernel's.  DESIGN.md section 3.3 states these values.                                                   */
int32_t b2a_debug_step_smem_rows(int32_t rows, int32_t gqa, int32_t* out);

/* Host-only (no device needed): the GEMM weight matrix the implicit convolution reads for an MLX-layout [out, k, in] weight --
 * stride 0: causal conv, rows = out, taps = k; stride > 0: transposed conv with k = n * stride, rows = stride * out
 * (phase-major), taps = n.  layout_out: [rows][taps][kpad] float32, kpad = ceil(in / 64) * 64.                              */
int32_t b2a_speech_tokenizer_debug_layout(const float* w, int32_t out, int32_t k, int32_t in, int32_t stride, float* layout_out,
                                          int64_t capacity, int32_t* rows, int32_t* taps, int32_t* kpad);
/* tools/diag_n1_stages.py: stage >= 0 makes later decodes keep a copy of the fp32 activation tensor after that stage (0 = transformer
 * output before the final norm, 1 + i = upsample layer i, 10 + 4 b = decoder block b after its transposed conv, 11 + 4 b + j = after
 * its residual unit j); out != null first copies the last kept tensor to the host (capacity in floats, length in *n).            */
int32_t b2a_speech_tokenizer_debug_stage(b2a_speech_tokenizer* h, int32_t stage, float* out, int64_t capacity, int64_t* n);
/* tests/test_gpu_qwen3_tts_encode.py: the speech-tokenizer encoder's code-search input z [B, encoded_length, hidden_size] float32
 * (the downsample's output) for audio [B, 1, n]; codes (nullable) receives the codes of the same run.                        */
int32_t b2a_speech_tokenizer_encoder_latent_test(b2a_speech_tokenizer_encoder* h, const float* audio, int32_t batch, int64_t n_samples,
                                                 float* z, int32_t* codes);
/* tests/test_gpu_qwen3_sampler.py: the Qwen3-TTS in-graph sampler kernel (csrc/qwen3_sampler.cu = sampleToken,
 * Qwen3TTS.swift:1003-1118) on HOST logits [B, V <= 4096]; suppress [lo, hi) except eos; seen = bitmap of the tokens generated
 * so far [B, ceil(V/32)] (nullable; updated when track != 0); tokens_out [B]; filtered_out [B, V] (nullable) = the logits handed
 * to categorical, -inf where removed.                                                                                     */
int32_t b2a_qwen3_sample_test(const float* logits, int32_t batch, int32_t vocab, float temperature, float top_p, int32_t top_k,
                              float min_p, float repetition_penalty, int32_t eos, int32_t suppress_lo, int32_t suppress_hi,
                              uint32_t* seen, int32_t track, uint64_t seed, int32_t step, int32_t* tokens_out, float* filtered_out);
/* tests/test_gpu_implicit_conv.py: one launch of the implicit-GEMM causal convolution kernel (csrc/conv_gemm.cu) on HOST
 * data: w [M][taps][Cin], x [B][Ttot][Cin]; out[b, t*up + rho, co] for m = rho * (M/up) + co is
 * sum_j sum_c w[m, j, c] * x[b, t + shift0 + j*dil, c] through the fused epilogue (bias, bias twice at t = 0, GELU, gamma, add,
 * SnakeBeta on the hi/lo copy).  xo [B][T*up][M/up] in/out or null; hl_out [B][Hout + T*up][M/up] or null.  fp16 != 0: operands
 * as fp16 hi/lo pairs instead of bf16 ones.                                                                               */
int32_t b2a_implicit_conv_test(const float* w, int32_t M, int32_t taps, int32_t Cin, const float* x, int32_t B, int32_t Ttot, int32_t T,
                               int32_t dil, int32_t shift0, int32_t up, const float* bias, const float* gamma, int32_t gelu, int32_t add,
                               int32_t bias_twice_t0, const float* sa, const float* sb, int32_t Hout, int32_t fp16, float* xo, float* hl_out);
/* tests/test_gpu_tc_gemm.py: one launch of tc_gemm_kernel<bn> (csrc/tc_gemm.cuh) on DEVICE pointers: out[N, M] = X[N, K] W[M, K]^T
 * through epilogue epi (0 store fp32, 2 SwiGLU bf16 [., M/2], 3 store bf16, 4 add into the caller's fp32 out), bias (nullable [M]),
 * act (1 = exact-erf GELU), tile_rows (0 = 128 weight rows per m-tile), lo_rows != 0 (bf16 outputs as hi/lo rows in X's tile layout)
 * and rstd_ss (nullable [rstd_parts, 8]: columns scaled by rsqrt(sum / K + rstd_eps), bn = 16 only).  hilo != 0: X is
 * cdiv(N, bn/2) tiles of bn rows, hi rows then lo rows.  split != 0: stream-K over ctas CTAs (store / add only, no GELU).
 * stages = 0: the deepest ring that fits.  Unsupported combinations return B2A_ERR_INVALID_INPUT.
 *   b2a_tc_gemm_test: the same with no bias, activation, tile_rows or norm scale, the deepest ring, and hi/lo rows for the bf16
 *       epilogues of hi/lo inputs.                                                                                         */
int32_t b2a_tc_gemm_epilogue_test(const void* W, const void* X, void* out, int32_t M, int32_t N, int32_t K, int32_t bn, int32_t epi,
                                  int32_t split, int32_t hilo, int32_t ctas, const float* bias, int32_t act, int32_t tile_rows,
                                  int32_t lo_rows, const float* rstd_ss, int32_t rstd_parts, float rstd_eps, int32_t stages, void* stream);
int32_t b2a_tc_gemm_test(const void* W, const void* X, void* out, int32_t M, int32_t N, int32_t K, int32_t bn, int32_t epi,
                         int32_t split, int32_t hilo, int32_t ctas, void* stream);
/* tests/test_gpu_splitk_norm.py: one launch of the cluster split-K GEMM (tc_gemm_splitk_kernel) on DEVICE pointers: W [M, K] bf16,
 * X [16, K] bf16 (hi rows 0..7, lo rows 8..15); for t < N: h[t] += W x[t] (h [8, M] fp32, in place), xn[t] / xn[8 + t] = hi / lo of
 * h[t] * gain (xn [16, M] bf16), ss[m_tile, t] = sum of h[t]^2 over the tile's rows (ss [cdiv(M, 128), 8]; 0 for t >= N).     */
int32_t b2a_tc_gemm_splitk_test(const void* W, const void* X, float* h, const float* gain, void* xn, float* ss, int32_t M, int32_t N,
                                int32_t K, int32_t cluster, int32_t stages, void* stream);
/* tests/test_gpu_splitk_store.py: the same kernel in the store mode of the decode step's q|k|v projection: for t < N,
 * out[t] = rstd[t] * W (x_hi[t] + x_lo[t]) (out [8, M] fp32, DEVICE; rows t >= N untouched), rstd[t] = rsqrt(sum_p rstd_ss[p, t] / K
 * + rstd_eps) for a DEVICE rstd_ss [rstd_parts, 8], or 1 when rstd_ss is null.  sk_ctas > 0: the k-blocks of a tile are cut as the
 * stream-K GEMM over sk_ctas CTAs cuts them (cluster >= the most pieces of a tile), and out is bit-identical to that GEMM's;
 * sk_ctas = 0: evenly over the cluster.                                                                                      */
int32_t b2a_tc_gemm_splitk_store_test(const void* W, const void* X, float* out, const float* rstd_ss, int32_t rstd_parts, float rstd_eps,
                                      int32_t M, int32_t N, int32_t K, int32_t cluster, int32_t sk_ctas, int32_t stages, void* stream);
/* Needs a device: how the fused decode step launches its q|k|v GEMM for m_tiles 128-row tiles of k_blocks 64-wide k-blocks on
 * device 0.  out[0] = the split-K cluster size (0: the stream-K GEMM runs), out[1] = its dynamic shared-memory bytes per CTA,
 * out[2] = the clusters of that size and footprint the device holds at once, out[3] = the stream-K CTA count whose cut the split-K
 * launch reproduces, out[4] = the most pieces that cut gives one tile (0 in out[1..2] when out[0] = 0).                     */
int32_t b2a_debug_qkv_split(int32_t m_tiles, int32_t k_blocks, int32_t* out);
/* tests/test_gpu_encoder_attention.py: the Whisper encoder attention (csrc/attn_tc.cuh, pack_qkv_f16_kernel + mha_tc_kernel) on a
 * DEVICE qkv [B * T, 3 * nh * 64] fp32; out [2 * 64 * cdiv(B * T, 64), nh * 64] bf16: token t = b * T + i at hi row
 * (t / 64) * 128 + t % 64, lo row = hi row + 64.  Rows of tokens >= B * T are not written.                                  */
int32_t b2a_mha_tc_test(const float* qkv, void* out, int32_t B, int32_t T, int32_t nh, void* stream);
/* tests/test_gpu_prompt_attention.py: the prompt attention of the batched prefill for one layer, all pointers DEVICE: rope_table_kernel,
 * then path 1 the SIMT prefill_attn_kernel<G> (only the L the engine gives it: L <= 128 at G <= 4, 124 at G = 6, 92 at G = 8) or path 2
 * the wgmma pack_prompt_kernel + prompt_attn_kernel (csrc/prompt_attn_tc.cuh), with the engine's launches.  qkv [B * L, (nq + 2 nkv) * 128]
 * fp32 (q | k | v of token b * L + i), freqs [64] the RoPE frequencies (angle = position / freqs[d]); qnorm / knorm [128] (both or
 * neither, nullable): per-head RMSNorm x * rsqrt(mean(x^2) + qk_eps) * gain of every q / k head before RoPE; kcache / vcache fp32
 * [B][nkv][max_ctx][128] receive the (normalised) RoPE'd keys and the values at positions 0 .. L-1, rows >= L untouched;
 * out [2 * 64 * cdiv(B * L, 64), nq * 128] bf16: the causal attention of token t at hi row (t / 64) * 128 + t % 64, lo row = hi row + 64.
 * Rows of tokens >= B * L are not written.  q heads per kv head: 1, 2, 3, 4, 6 or 8.                                          */
int32_t b2a_prompt_attn_test(const float* qkv, const float* freqs, const float* qnorm, const float* knorm, float qk_eps, float* kcache,
                             float* vcache, void* out, int32_t B, int32_t L, int32_t nq, int32_t nkv, int32_t max_ctx, int32_t path,
                             void* stream);
/* tests/test_gpu_decode_attention.py: one decode-step attention launch of the Llama / Qwen3 stacks (attn_decode_cluster_kernel<G>,
 * csrc/llama.cu) with the step's grid (nkv, B, 2), shared memory and programmatic-dependent launch, all pointers DEVICE.  Row b < B
 * (B <= 8) with 0 <= pos[b] < max_ctx normalises (qnorm / knorm as above) and rotates its q heads and new key from qkv
 * [B, (nq + 2 nkv) * 128] fp32 at position pos[b], writes the key and the raw value to row pos[b] of kcache / vcache fp32
 * [B][nkv][max_ctx][128] and attends to the cached rows 0 .. pos[b] - 1 plus the new one.  out [16, nq * 128] bf16: hi row b, lo row
 * 8 + b.  Other rows write nothing.  q heads per kv head: 1, 2, 3, 4, 6 or 8.                                                  */
int32_t b2a_decode_attn_test(const float* qkv, const int32_t* pos, const float* freqs, const float* qnorm, const float* knorm, float qk_eps,
                             float* kcache, float* vcache, void* out, int32_t B, int32_t nq, int32_t nkv, int32_t max_ctx, void* stream);
/* tests/test_gpu_whisper_decode_attention.py: one Whisper decoder-step attention launch (mha_decode_kernel, csrc/whisper.cu) with the
 * engine's grid (nh, B, S), all pointers DEVICE.  self_attn != 0: q is the fused q|k|v row [B, 3 * nh * 64] (query, new key, new
 * value), kcache / vcache fp32 [B][nh][max_t][64]; row b with 0 <= pos[b] < max_t writes its new key / value at pos[b] and attends
 * to positions 0..pos[b] in S = cdiv(max_t, 64) splits.  self_attn == 0: kv [B * max_t, 2 * nh * 64] fp32 (k | v projection of
 * the encoder states) is first relaid into the fp16 caches kcache / vcache [B][nh][max_t][64], then q [B, nh * 64] attends to all
 * max_t keys in S = cdiv(max_t, 128) splits.  Rows with pos[b] < 0 are skipped.  out [32, nh * 64] bf16: hi row b, lo row b + 16.
 * Workspace: part_o [B * nh * S * 64], part_ml [B * nh * S * 2], counters [B * nh] int, zero on entry and left zero.             */
int32_t b2a_wh_decode_attn_test(int32_t self_attn, const float* q, const float* kv, const int32_t* pos, void* kcache, void* vcache,
                                void* out, float* part_o, float* part_ml, int32_t* counters, int32_t B, int32_t nh, int32_t max_t,
                                void* stream);
/* tests/test_gpu_conv_gemm.py: one launch of the codec conv GEMM (cg::conv_gemm_kernel, csrc/conv_gemm.cu, through the launch SNAC and Vocos use):
 * acc[n, m] = W[m, :] . X[n, :] for the host fp32 weight w [M, K] (split into bf16 hi/lo like the engines' weights) and the DEVICE
 * activations X, 2 * pad64(N) rows of 64-token hi/lo tiles (hi rows, then lo rows) by K.  Then v = gamma * GELU(acc + bias) (each
 * optional) through epilogue epi: 0 E_STORE_HILO (Snake(alpha) of v as hi/lo into hl; dual: token b*T + t to row b*(T+1) + t,
 * columns [0, M), and to row b*(T+1) + t + 1, columns [M, 2M)), 1 E_CONVT (row m = r*Cout + co of input token b*(Tin+1) + q to
 * output token b*T + q*stride + r - pad, kept when inside [0, T), into x and optionally hl), 2 E_NOISE (x += noise[n] * v; noise
 * null: the seeded N(0, 1) draw for token n), 3 E_ADD (x += v), 4 E_ADD_HILO (x += v, then as E_STORE_HILO), 5 E_STORE_F32 (x = v).
 * x [., ldx] fp32 and hl [., ldh] bf16 hi/lo tiles are DEVICE pointers.  Combinations no engine launches return B2A_ERR_INVALID_INPUT.
 * ctas = 0: min(SM count, work tiles), as the engines launch it.                                                           */
int32_t b2a_conv_gemm_test(const float* w, int32_t M, int32_t K, const void* X, int32_t N, int32_t epi, const float* bias,
                           const float* alpha, const float* gamma, int32_t gelu, float* x, int32_t ldx, void* hl, int32_t ldh,
                           int32_t dual, int32_t T, int32_t Cout, int32_t stride, int32_t pad, int32_t Tin, const float* noise,
                           uint64_t seed, int32_t ctas, void* stream);
/* tests/test_gpu_snac_fused.py: one launch of the fused SNAC unit (rf::ru_fused_kernel, csrc/snac_fused.cuh) on DEVICE fp32
 * x, y [B * T, C], C = 64 or 128.  mode 0 (ResidualUnit, dil 1, 3 or 9): y = x + W Snake(a_mid, dwconv7_dil(Snake(a_in, x)) + dw_b)
 * + pw_bias; mode 1 (NoiseBlock, dil 0): y = x + noise[b*T + t] * (W x), noise null: the seeded N(0, 1) draw for token b*T + t.
 * pw_w: host fp32 [C, C].  hl (with a_next): Snake(a_next, y) as hi/lo tiles of the next transposed conv's 2-tap im2col, ld 2C,
 * laid out as conv GEMM dual outputs.  dw_w [C, 7], dw_b, a_in, a_mid, pw_bias [C], a_next [C] are DEVICE pointers (biases nullable).
 * ctas = 0: the engine's CTA count.                                                                                        */
int32_t b2a_snac_unit_test(int32_t mode, int32_t C, int32_t dil, const float* x, float* y, int32_t B, int32_t T, const float* dw_w,
                           const float* dw_b, const float* a_in, const float* a_mid, const float* pw_w, const float* pw_bias,
                           const float* noise, uint64_t seed, void* hl, const float* a_next, int32_t ctas, void* stream);
/* tests/test_gpu_snac_fused.py: one launch of the fused Snake + transposed conv (rf::convt_fused_kernel) on DEVICE fp32
 * x [B * Tin, 128] -> y [B * Tin * stride, cout]: y = conv_transpose1d(Snake(alpha, x), w, bias, stride, padding ceil(stride / 2)),
 * w the host fp32 weight in torch layout [128, cout, 2 * stride].  Only (stride, cout) = (2, 64) and (1, 128).  ctas = 0: the
 * engine's CTA count.                                                                                                      */
int32_t b2a_snac_convt_test(const float* x, float* y, const float* alpha, const float* bias, const float* w, int32_t B, int32_t Tin,
                            int32_t stride, int32_t cout, int32_t ctas, void* stream);
/* tests/test_gpu_snac_encode.py: the SNAC encoder's latent before the code search (what b2a_snac_encode quantizes) on HOST data:
 * wave [B, n_samples] -> z [B, latent, t_latent] float32, t_latent as b2a_snac_encoded_length gives it.  Errors as b2a_snac_encode. */
int32_t b2a_snac_encode_latent_test(b2a_snac* h, const float* wave, int32_t batch, int64_t n_samples, float* z);
/* tests/test_gpu_snac_44khz.py: one launch of SNAC LocalMHA's window core (local_attn_kernel, csrc/snac.cu) on HOST data:
 * qkv float32 [B * T, 3 dim] (q | k | v before the rotary rotation), inv_freq [32] -> out float32 [B * T, dim], the hi + lo pair it
 * writes for to_out.  T % window == 0, window 1 .. 64, dim a multiple of 64. */
int32_t b2a_snac_local_attn_test(const float* qkv, const float* inv_freq, int32_t B, int32_t T, int32_t dim, int32_t window, float* out);
/* tests/test_gpu_encodec_encode.py: the Encodec encoder's latent before the code search (what b2a_encodec_encode quantizes) on HOST
 * data: audio [B, samples, audio_channels] -> z [n_chunks, B, frames, hidden_size] float32, shapes as b2a_encodec_encoded_shape
 * gives them.  Errors as b2a_encodec_encode. */
int32_t b2a_encodec_encode_latent_test(b2a_encodec* h, const float* audio, int32_t batch, int64_t samples, float* z);

/* ------------------------------------------------------------------ Soprano
 *   b2a_soprano_create_random : b2a_soprano_create with the language model drawn on the device (as b2a_qwen3_lm_create_random) and the
 *       decoder from `decoder_tensors` (decoder.decoder.* / decoder.head.* keys; n_decoder_tensors may not be 0).
 *   b2a_soprano_hidden_states : the hidden states the last b2a_tts_generate captured: out [batch, max_tokens + 1, hidden_size] float32
 *       (nullable), n_states[batch] = 1 + the row's generated tokens.
 *   b2a_vocos_decode_upsampled_dev : SopranoDecoder on DEVICE rows: row b of the batch is the n states at d_states + d_rows[b] * row_stride
 *       (d_rows NULL: b), upsampled x upscale inside the embed conv's operand kernel; d_wave [B, b2a_vocos_upsampled_length].
 *   b2a_vocos_upsampled_length : (upscale (n - 1)) hop for n >= 2, n_fft (the untrimmed one-frame overlap-add) for n = 1.            */
int32_t b2a_soprano_create_random(int32_t device, const b2a_soprano_config* cfg, float std, uint64_t seed, const b2a_tensor* decoder_tensors,
                                  int32_t n_decoder_tensors, b2a_tts** out);
int32_t b2a_soprano_hidden_states(b2a_tts* h, int32_t batch, float* out, int32_t* n_states);
int32_t b2a_vocos_decode_upsampled_dev(b2a_vocos* h, const float* d_states, int64_t row_stride, const int32_t* d_rows, int32_t batch, int32_t n,
                                       int32_t upscale, float* d_wave, void* stream);
int64_t b2a_vocos_upsampled_length(const b2a_vocos* h, int32_t n, int32_t upscale);

#ifdef __cplusplus
}
#endif
#endif /* B200AUDIO_INTERNAL_H */
