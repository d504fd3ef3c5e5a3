"""float64 pieces shared by the Llama / Qwen3 attention tests (test_gpu_prompt_attention.py, test_gpu_decode_attention.py): the
per-head q/k RMSNorm and RoPE that every attention kernel of those stacks applies to its fp32 q | k | v, computed in float64 from the
same fp32 inputs."""
import torch

from oracle import llama as ol

HD = 128
FREQS = torch.from_numpy(ol.llama3_rope_freqs(ol.LlamaConfig())).float()    # [64] fp32, angle = position / freqs[d]


def rope64(x, pos):
    """[.., n, 128] -> float64 non-traditional RoPE (pairs d, d + 64) at positions pos [n], with the kernels' fp32 angles."""
    ang = (torch.as_tensor(pos).cpu().float()[:, None] / FREQS[None, :]).double().to(x.device)
    c, s = torch.cos(ang), torch.sin(ang)
    x = x.double()
    x1, x2 = x[..., :HD // 2], x[..., HD // 2:]
    return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1)


def rmsnorm64(x, gain, eps):
    """[.., 128] -> float64 x * rsqrt(mean(x^2) + eps) * gain; gain None: x unchanged (the norm is off)."""
    x = x.double()
    if gain is None:
        return x
    return x * torch.rsqrt(x.square().mean(-1, keepdim=True) + eps) * gain.double()


def qk_gains(seed, q_scale=1.0):
    """Random Qwen3-style norm gains 1 + 0.3 N(0, 1) of q (times q_scale) and k, fp32 [128] each on the device.  q_scale sets the
    score spread: after the norm a q head has an RMS of about q_scale whatever its projection was."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    qn = (1.0 + 0.3 * torch.randn(HD, device="cuda", generator=g)) * q_scale
    kn = 1.0 + 0.3 * torch.randn(HD, device="cuda", generator=g)
    return qn.contiguous(), kn.contiguous()


def decode_attn(b2a, qkv, pos, kc, vc, nq, nkv, qn=None, kn=None, eps=0.0):
    """One b2a_decode_attn_test launch (B = pos.numel() rows, max_ctx = kc.shape[2]) into a fresh NaN-filled [16, nq * 128] bf16 output;
    returns (status, output)."""
    f = b2a._ffi
    out = torch.full((16, nq * HD), float("nan"), device="cuda", dtype=torch.bfloat16)
    st = f.lib().b2a_decode_attn_test(f.ptr(qkv), f.ptr(pos), f.ptr(FREQS.cuda()), f.ptr(qn), f.ptr(kn), eps, f.ptr(kc), f.ptr(vc),
                                      f.ptr(out), pos.numel(), nq, nkv, kc.shape[2], None)
    torch.cuda.synchronize()
    return st, out
