"""Per-stage measurements for the other BASELINE.json configs (not the driver's bench line): CUDA events on the
library's streams, inputs resident in HBM, roofline numerators from SURVEY.md section 8d.

    python tools/bench_kernels.py [mel] [snac] [whisper] [encodec] [encodec48] [speech_tokenizer]      -> one JSON line per stage
"""
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mlx_audio_swift_b200 as m  # noqa: E402

PEAKS = json.loads((Path(__file__).resolve().parents[1] / "MEASURED_PEAKS.json").read_text()) \
    if (Path(__file__).resolve().parents[1] / "MEASURED_PEAKS.json").exists() else {"hbm_gbs": 6650.0, "bf16_tflops": 1590.0}


def timed(fn, stream_ptr, iters=10, warmup=3):
    s = torch.cuda.ExternalStream(stream_ptr) if stream_ptr else torch.cuda.current_stream()
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(iters):
        fn()
    e1.record(s)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def synth(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 16000.0
    return np.clip(0.5 * np.sin(2 * np.pi * 220 * t) + 0.1 * rng.standard_normal(n), -1, 1).astype(np.float32)


def bench_mel():
    for B, n, name in ((1, 160000, "config1: 10 s clip (core log-mel)"), (16, 480000, "config3 front-end: 16 x 30 s (Whisper log-mel)"),
                       (128, 480000, "128 x 30 s (Whisper log-mel, larger than L2)")):
        kind = "core" if B == 1 else "whisper"
        lm = m.LogMel(kind, n_mels=80)
        x = torch.from_numpy(np.stack([synth(n, i % 4) for i in range(min(B, 4))])).cuda().repeat((B + 3) // 4, 1)[:B].contiguous()
        F = lm.frames(n)
        out = torch.empty((B, F, 80), device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        ms = timed(lambda: lm.compute_dev(x, out, st), 0)
        alg = 4 * B * n + 4 * B * F * 80
        print(json.dumps({"stage": "mel", "workload": name, "ms": ms, "algorithmic_bytes": alg, "achieved_GBs": alg / ms / 1e6,
                          "frac_of_hbm": alg / ms / 1e6 / PEAKS["hbm_gbs"], "audio_s_per_s": B * n / 16000 / (ms * 1e-3),
                          "note": "two kernels: fused STFT->power->mel->log10 + in-place max-8 clamp (adds 2*4*F*80 bytes/clip, not counted)"}))


def bench_snac():
    codec = m.SNAC(weights=m.SNAC.random_init_weights(1234))
    B, T = 8, 1024
    rng = np.random.default_rng(2)
    codes = [torch.from_numpy(rng.integers(0, 4096, size=(B, T // s), dtype=np.int32)).cuda() for s in (4, 2, 1)]
    wave = torch.empty((B, 1, T * 512), device="cuda")
    ms = timed(lambda: codec.decode_dev(codes, wave, seed=1, stream=codec.stream), codec.stream, iters=3, warmup=1)
    flop = 212e9 * B
    fused_bytes = 441.5e6 * B
    print(json.dumps({"stage": "snac_decode", "workload": "config2: batch 8 x 1024 latent steps -> 8 x 524288 samples (174.8 s audio)",
                      "ms": ms, "dense_flop": flop, "achieved_TFLOPs": flop / ms / 1e9, "per_block_fused_bytes": fused_bytes,
                      "achieved_GBs_vs_fused_bound": fused_bytes / ms / 1e6, "frac_of_hbm": fused_bytes / ms / 1e6 / PEAKS["hbm_gbs"],
                      "x_realtime": B * T * 512 / 24000 / (ms * 1e-3),
                      "note": "channels-last wgmma conv GEMM (fp32 as bf16 hi/lo), 16 epilogue warps"}))


def bench_whisper():
    cfg = dict(vocab_size=51865, num_mel_bins=80, d_model=512, encoder_layers=6, encoder_attention_heads=8, encoder_ffn_dim=2048,
               max_source_positions=1500, decoder_layers=6, decoder_attention_heads=8, decoder_ffn_dim=2048, max_target_positions=448)
    wm = m.WhisperModel.random_init(cfg, max_batch=16)
    B = 16
    x = torch.from_numpy(np.stack([synth(480000, i) for i in range(B)])).cuda()
    P = m.STTGenerateParameters(max_tokens=64, mask_eot=True)
    toks = np.zeros((B, 64), dtype=np.int32)
    nt = np.zeros(B, dtype=np.int32)
    outs = []
    ms = timed(lambda: outs.append(wm.generate_dev(x, P, toks, nt)), wm.stream, iters=3, warmup=1)
    o = outs[-1]
    print(json.dumps({"stage": "whisper_base", "workload": "config3: 16 x 30 s, greedy, 64 forced decode steps", "ms": ms,
                      "x_realtime": B * 30 / (ms * 1e-3), "encode_ms": o.encode_time * 1e3, "decode_ms": o.decode_time * 1e3,
                      "encoder_TFLOPs_useful": 87.4e9 * B / max(o.encode_time, 1e-9) / 1e12,
                      "note": "encode = log-mel + conv stem + 6 layers + cross K/V; decode = 4-token prefix + 64 graph-replayed steps"}))


def bench_encodec():
    cfg = m.EncodecConfig()
    codec = m.Encodec(cfg, weights=m.Encodec.random_init_weights(cfg, 1234, n_codebooks=8))
    B, T = 8, 750                                           # 8 x 10 s at 75 frames/s
    rng = np.random.default_rng(2)
    codes = torch.from_numpy(rng.integers(0, 1024, size=(1, B, 8, T), dtype=np.int32)).cuda()
    wave = torch.empty((B, T * 320, 1), device="cuda")
    ms = timed(lambda: codec.decode_dev(codes, wave, stream=codec.stream), codec.stream, iters=5, warmup=2)
    print(json.dumps({"stage": "encodec_decode", "workload": "Encodec-24kHz decode, batch 8 x 750 frames (8 codebooks) -> 8 x 10 s",
                      "ms": ms, "x_realtime": B * 10.0 / (ms * 1e-3),
                      "note": "fp32 implicit-GEMM convs + persistent wavefront LSTM (T + 1 grid barriers)"}))


def bench_encodec48():
    """The 48 kHz stereo model (time_group_norm, 1 s chunks, 1 % overlap): decode of 8 clips x 31 chunks x 150 frames at 24 kbps
    (16 codebooks) with per-chunk scales -> 8 x 1 473 600 samples (30.7 s), the clips tools/bench_encodec_encode.py --model 48khz
    encodes."""
    import subprocess
    sys.path.insert(0, str(Path(__file__).resolve().parent))
    from bench_encodec_encode import config_48khz
    cfg = config_48khz()
    codec = m.Encodec(cfg, weights=m.Encodec.random_init_weights(cfg, 1234, n_codebooks=16, encoder=True))
    B, nc, T = 8, 31, 150
    rng = np.random.default_rng(2)
    codes = torch.from_numpy(rng.integers(0, 1024, size=(nc, B, 16, T), dtype=np.int32)).cuda()
    scales = torch.from_numpy(rng.uniform(0.05, 0.5, size=(nc, B)).astype(np.float32)).cuda()
    n = codec.output_length(nc, T)
    wave = torch.empty((B, n, 2), device="cuda")
    ms = timed(lambda: codec.decode_dev(codes, wave, scales, stream=codec.stream), codec.stream, iters=5, warmup=2)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip().splitlines()[0]
    print(json.dumps({"stage": "encodec48_decode", "workload": f"Encodec-48kHz decode, {B} clips x {nc} chunks x {T} frames (16 codebooks) -> {B} x {n / 48000:.1f} s stereo",
                      "ms": ms, "x_realtime": B * n / 48000 / (ms * 1e-3), "gpu": gpu,
                      "note": "time_group_norm: every conv followed by gn_stats_kernel + gn_apply_kernel"}))


def bench_speech_tokenizer():
    """Qwen3-TTS speech-tokenizer decoder, shipped geometry, 4 rows x 16 streaming chunks of 64 code frames (bench.py's qwen3 block)."""
    import importlib
    import os
    codec = importlib.import_module("mlx_audio_swift_b200.qwen3_tts_codec")
    cfg = codec.Qwen3TTSTokenizerDecoderConfig()
    B, frames, chunk = 4, 1024, 64
    dec = codec.Qwen3TTSSpeechTokenizerDecoder(cfg, weights=codec.random_init_weights(cfg, 5), max_batch=B, max_cache_frames=frames + 8)
    codes = np.random.default_rng(1).integers(0, cfg.codebook_size, (B, cfg.num_quantizers, frames)).astype(np.int32)

    def run():
        dec.reset_streaming_state()
        for f0 in range(0, frames, chunk):
            dec.streaming_step(codes[:, :, f0:f0 + chunk])

    for _ in range(2):
        run()
    t0 = time.perf_counter()
    n = 3
    for _ in range(n):
        run()
    ms = (time.perf_counter() - t0) / n * 1e3                    # every streaming_step ends synchronised (waveform copied to the host)
    print(json.dumps({"stage": "speech_tokenizer_decode", "workload": f"{B} rows x {frames} code frames in {chunk}-frame streaming chunks -> {B} x {frames * 1920 / 24000:.1f} s",
                      "ms": ms, "x_realtime": B * frames * 1920 / 24000 / (ms * 1e-3),
                      "operands": "fp16 pairs" if os.environ.get("B2A_ST_FP16", "1") != "0" else "bf16 pairs"}))


if __name__ == "__main__":
    which = sys.argv[1:] or ["mel", "snac", "whisper", "encodec"]
    for w in which:
        {"mel": bench_mel, "snac": bench_snac, "whisper": bench_whisper, "encodec": bench_encodec, "encodec48": bench_encodec48,
         "speech_tokenizer": bench_speech_tokenizer}[w]()
