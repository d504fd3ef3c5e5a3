"""The `--benchmark` report of the reference CLI (Sources/Tools/mlx-audio-swift-tts/App.swift:128-212) for the H100 path:
Audio duration / TTFB / RTFx / Tokens/s of one Orpheus-3B generate call (random-init weights, synthetic prompt ids -- there is no
tokenizer or checkpoint here).  The reference's Orpheus emits its audio once, at the end (LlamaTTS.swift:901-904), so its TTFB is the
whole generation; with --stream (row N2, b2a_tts_generate_stream) audio chunks are decoded by SNAC while tokens are still being
generated and TTFB is the latency of the first .audio event, as the CLI measures it (App.swift:155-170, streamingInterval 0.32 s).

With --ref-seconds S every row carries a voice-cloning reference block (prepareInputIds with refAudio / refText, LlamaTTS.swift:446-553):
a synthetic S-second clip encoded by SNAC on the device and a 16-token stand-in transcript.  The encode runs before the timed call;
prompts of any length take the batched prefill (longer than 128 tokens with the wgmma prompt attention, csrc/prompt_attn_tc.cuh).

--model qwen3 runs VyvoTTS (Qwen3Model, Qwen3.swift) instead: QWEN3_06B below, Qwen3-0.6B's layer shapes with VyvoTTS's 180 352-token
vocabulary -- an assumed geometry, as the published checkpoint's config.json is not at hand -- and the same prompts framed by its
prepareInputIds, ending in its start-of-speech 151670.

--model soprano runs Soprano (SopranoModel, Soprano.swift) at SOPRANO_ASSUMED below: hidden 512 (the decoder's input channels), 8 layers,
MLP 2048, 4 query / 1 key-value heads of 128, vocabulary 8192 and the Soprano-1.1 decoder (768 / 2304, 8 ConvNeXt blocks, n_fft 2048, hop
512, upscale 4, input kernel 1) -- an ASSUMED geometry, as the published config.json is not at hand.  Its language model is drawn on the
device, its decoder from oracle/vocos.py's seeded init; prompts are random ids; sampling is Soprano's defaults (T 0.7, top-p 0.95, penalty
1.5 over 30) with the stop token masked, so every row generates --max-tokens tokens.  Audio is 32 kHz and comes once, at the end.

    python tools/tts_benchmark.py [--model orpheus|qwen3|soprano] [--batch 1] [--prompt 64] [--max-tokens 512] [--model-dir DIR] [--stream]
                                  [--interval 0.32] [--ref-seconds S]"""
import argparse
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mlx_audio_swift_b200 as m  # noqa: E402
from bench import ORPHEUS, make_prompts  # noqa: E402

QWEN3_06B = dict(hidden_size=1024, num_hidden_layers=28, intermediate_size=3072, num_attention_heads=16, num_key_value_heads=8, head_dim=128,
                 vocab_size=180352, rms_norm_eps=1e-6, rope_theta=1000000.0, tie_word_embeddings=True)

SOPRANO_ASSUMED = dict(hidden_size=512, num_hidden_layers=8, intermediate_size=2048, num_attention_heads=4, num_key_value_heads=1, head_dim=128,
                       vocab_size=8192, tie_word_embeddings=False, decoder_num_layers=8, decoder_dim=768, decoder_intermediate_dim=2304,
                       hop_length=512, n_fft=2048, upscale=4, input_kernel=1, dw_kernel=3, token_size=2048)


def report(elapsed, audio, first_token, started, info, ttfb=None):
    print(f"Finished generation in {elapsed:0.2f}s")
    print("Benchmark:")
    print(f"  Audio duration: {audio:.2f}s")
    ttfb = elapsed if ttfb is None else ttfb
    print(f"  TTFB: {ttfb:.3f}s (first token after {first_token[0] - started:.3f}s)" if first_token else "  TTFB: n/a")
    print(f"  RTFx: {audio / elapsed:.3f}" if audio > 0 else "  RTFx: n/a")
    print(f"  Tokens/s: {info.tokens_per_second:.2f}")


def soprano_benchmark(a):
    from oracle import soprano as so
    cfg = so.SopranoConfig(**SOPRANO_ASSUMED)
    dec = so.decoder_weights_only(cfg, 1234)
    tts = m.SopranoModel.random_init(cfg.to_json(), dec, max_batch=a.batch, max_context=a.prompt + a.max_tokens + 2)
    ids = np.random.default_rng(0).integers(4, cfg.vocab_size, size=(a.batch, a.prompt)).astype(np.int32)
    P = m.GenerateParameters(max_tokens=a.max_tokens, temperature=0.7, top_p=0.95, repetition_penalty=1.5, repetition_context_size=30,
                             mask_eos=True)
    tts.generate_batch(ids, P)                   # warm-up (graph capture, allocations)
    first_token = []
    started = time.perf_counter()
    toks, waves, info = tts.generate_batch(ids, P, on_token=lambda b, step, tok: first_token.append(time.perf_counter()) if not first_token else None)
    elapsed = time.perf_counter() - started
    print(f"Soprano, assumed geometry {SOPRANO_ASSUMED}, batch {a.batch}, {a.prompt}-token prompt, {a.max_tokens} tokens")
    report(elapsed, sum(len(w) for w in waves) / float(tts.sample_rate), first_token, started, info)


ap = argparse.ArgumentParser()
ap.add_argument("--model", default="orpheus", choices=["orpheus", "qwen3", "soprano"])
ap.add_argument("--batch", type=int, default=1, help="utterances per call, 1..32")
ap.add_argument("--prompt", type=int, default=64)
ap.add_argument("--max-tokens", type=int, default=512)
ap.add_argument("--model-dir", default=None, help="checkpoint directory (config.json + *.safetensors); default: random init")
ap.add_argument("--stream", action="store_true", help="chunked audio emission during generation (TTFB = first audio chunk)")
ap.add_argument("--interval", type=float, default=0.32, help="streaming interval in seconds (App.swift:137)")
ap.add_argument("--ref-seconds", type=float, default=0.0, help="voice-cloning prompt with a synthetic reference clip of S seconds")
a = ap.parse_args()
if a.model == "soprano":
    soprano_benchmark(a)
    sys.exit(0)
codec = m.SNAC(weights=m.SNAC.random_init_weights(1234, encoder=a.ref_seconds > 0))
ref_len = 0
if a.ref_seconds > 0:
    n_ref = int(a.ref_seconds * 24000)
    ref_len = 7 * codec.encoded_length(n_ref) // 4 + 16 + 9            # codes + transcript + the block's framing tokens
ctx = a.prompt + ref_len + a.max_tokens + 16
Model, geometry, sos = (m.Qwen3Model, QWEN3_06B, 151670) if a.model == "qwen3" else (m.LlamaTTSModel, ORPHEUS, 128257)
if a.model_dir:
    tts = Model.from_model_directory(a.model_dir, snac=codec, max_batch=a.batch, max_context=ctx)
else:
    tts = Model.random_init(geometry, snac=codec, max_batch=a.batch, max_context=ctx)
# the untruncated make_prompts rows are [SOH] body [EOT, EOH, SOS]: a body of prompt - 4 tokens keeps the framed prompt at --prompt
prompts = make_prompts(0, max(a.batch, 8))[:a.batch]      # up to 32 rows; the first 8 are bench.py's
body = [r[1:-3][:max(a.prompt - 4, 1)].tolist() for r in prompts]
ids = prompts[:, :a.prompt]
if a.model == "qwen3":
    ids, _ = tts.prepare_input_ids(body)
    ids = np.concatenate([ids, np.full((ids.shape[0], 1), sos, dtype=np.int32)], axis=1)
if a.ref_seconds > 0:
    t = np.arange(n_ref) / 24000.0
    clip = (0.5 * np.sin(2 * np.pi * 220.0 * t) + 0.1 * np.random.default_rng(0).standard_normal(n_ref)).astype(np.float32)
    ref_text = make_prompts(1)[0, 1:17].tolist()
    ids, _ = tts.prepare_input_ids(body, tts.encode_audio_to_code_list(clip), ref_text)
    ids = np.concatenate([ids, np.full((ids.shape[0], 1), sos, dtype=np.int32)], axis=1)
    print(f"Cloning prompt: {a.ref_seconds:g}s reference -> {ids.shape[1]} tokens per row")
P = m.GenerateParameters(max_tokens=a.max_tokens, temperature=0.6, top_p=0.8, repetition_penalty=1.3, repetition_context_size=20,
                         mask_eos=True, wrap_codes=True)
tts.generate_batch(ids, P)                       # warm-up (graph capture, allocations)
first_token, first_audio = [], []
if a.stream:
    fpc = max(1, int(round(a.interval * 24000.0 / 2048.0)))
    tts.generate_audio_chunks(ids, P, frames_per_chunk=fpc)          # warm-up of the chunked codec shapes
    started = time.perf_counter()
    toks, chunks, info = tts.generate_audio_chunks(ids, P, frames_per_chunk=fpc,
                                                    on_audio=lambda b, x, fin: first_audio.append(time.perf_counter()) if not first_audio else None,
                                                    on_token=lambda b, step, tok: first_token.append(time.perf_counter()) if not first_token else None)
    elapsed = time.perf_counter() - started
    waves = [np.concatenate(c) if c else None for c in chunks]
else:
    started = time.perf_counter()
    toks, waves, info = tts.generate_batch(ids, P, on_token=lambda b, step, tok: first_token.append(time.perf_counter()) if not first_token else None)
    elapsed = time.perf_counter() - started
audio = sum(len(w) for w in waves if w is not None) / 24000.0
report(elapsed, audio, first_token, started, info, (first_audio[0] - started) if first_audio else None)
