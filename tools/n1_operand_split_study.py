"""CPU study: the Qwen3-TTS speech-tokenizer decoder (float64 oracle) with the operands of every weight GEMM / dense convolution
replaced by what a tensor-core split holds, products in float64 (so only the operand representation is modelled):

    bf16x2   hi + lo bf16 (16 mantissa bits), the lo*lo product dropped          -- what the implicit convolution runs
    f16x2    hi + lo fp16 (subnormals kept: absolute floor 2^-24), lo*lo dropped
    bf16x3   hi + mid + lo bf16 (24 bits), products with weight >= 2^-16 kept (hh, hm, mh, mm, hl, lh)

    python tools/n1_operand_split_study.py [frames] [geometry: default|mid]
"""
import sys
from pathlib import Path
import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from oracle import qwen3_tts_codec as oc

MODE = None


def parts(x, mode):
    x = x.to(torch.float64)
    if mode == "bf16x2":
        h = x.to(torch.bfloat16).to(torch.float64); l = (x - h).to(torch.bfloat16).to(torch.float64)
        return [h, l]
    if mode == "f16x2":
        h = x.to(torch.float16).to(torch.float64); l = (x - h).to(torch.float16).to(torch.float64)
        return [h, l]
    if mode == "bf16x3":
        h = x.to(torch.bfloat16).to(torch.float64); m = (x - h).to(torch.bfloat16).to(torch.float64)
        l = (x - h - m).to(torch.bfloat16).to(torch.float64)
        return [h, m, l]
    raise ValueError(mode)


def split_apply(fn, x, w):
    """sum of fn(x_i, w_j) over the kept products"""
    if MODE is None:
        return fn(x, w)
    xs, ws = parts(x, MODE), parts(w, MODE)
    keep = [(0, 0), (0, 1), (1, 0)] if len(xs) == 2 else [(0, 0), (0, 1), (1, 0), (1, 1), (0, 2), (2, 0)]
    y = None
    for i, j in keep:
        t = fn(xs[i], ws[j])
        y = t if y is None else y + t
    return y


_conv1d, _einsum = F.conv1d, torch.einsum


def conv1d_mlx(x, w, b, stride=1, dilation=1):
    y = split_apply(lambda a, c: _conv1d(a, c.permute(0, 2, 1), None, stride=stride, dilation=dilation), x, w)
    return y if b is None else y + b[None, :, None]


def conv_transpose1d_mlx(x, w, b, stride):
    B, cin, T = x.shape
    cout, k, _ = w.shape
    y = torch.zeros(B, cout, (T - 1) * stride + k, dtype=x.dtype)
    for j in range(k):
        y[:, :, j: j + (T - 1) * stride + 1: stride] += split_apply(lambda a, c: _einsum("bit,oi->bot", a, c), x, w[:, j, :])
    if b is not None:
        y = y + b[None, :, None]
    return y


def _lin(self, name, x):
    y = split_apply(lambda a, c: a @ c.T, x, oc._w(self.W, name + ".weight"))
    if name + ".bias" in self.W:
        y = y + oc._w(self.W, name + ".bias")
    return y


def _tail(self, x, h):
    h = h.transpose(1, 2)
    h = F.layer_norm(h, (h.shape[-1],), self.nw, self.nb, 1e-6)
    h = oc.gelu_exact(split_apply(lambda a, c: a @ c.T, h, self.w1) + self.b1)
    h = self.gamma * (split_apply(lambda a, c: a @ c.T, h, self.w2) + self.b2)
    return x + h.transpose(1, 2)


def main():
    global MODE
    T = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    geom = sys.argv[2] if len(sys.argv) > 2 else "default"
    cfg = oc.TokenizerDecoderConfig() if geom == "default" else oc.mid_config()
    W = oc.init_weights(cfg, 1)
    codes = np.random.default_rng(0).integers(0, cfg.codebook_size, (1, cfg.num_quantizers, T))
    ref = oc.SpeechTokenizerDecoder(cfg, W)(codes).numpy()[0, 0]
    oc.conv1d_mlx, oc.conv_transpose1d_mlx = conv1d_mlx, conv_transpose1d_mlx
    oc.PreTransformer._lin = _lin
    oc.ConvNeXt._tail = _tail
    up = cfg.total_upsample
    for mode in (None, "bf16x2", "f16x2", "bf16x3"):
        MODE = mode
        y = oc.SpeechTokenizerDecoder(cfg, W)(codes).numpy()[0, 0]
        e = np.abs(y - ref) / np.abs(ref).max()
        per = ["%.1e" % e[f * up:(f + 1) * up].max() for f in range(T)]
        print(f"{geom:8s} T={T} {str(mode):8s} max {e.max():.2e} per-frame {per}", flush=True)


if __name__ == "__main__":
    main()
