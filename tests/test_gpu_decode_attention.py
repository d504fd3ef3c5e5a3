"""The decode-step attention of the Llama / Qwen3 stacks (csrc/llama.cu: attn_decode_cluster_kernel<G>, through b2a_decode_attn_test
with the step's own launch) against float64, at every GQA ratio the engine accepts and at the kernel's chunk edges.

The kernel runs one 2-CTA cluster per (kv head, row).  Keys 0..p of a row at position p are cut into 64-key chunks dealt alternately
to the two CTAs (CTA r takes chunks r, r + 2, ...), streamed K, V, K, V, ... through a 3-slot cp.async.bulk ring.  The new position
is not read from the cache: its key is normalised (Qwen3's per-head RMSNorm) and rotated from this step's q|k|v row and spliced into
the last chunk, and the CTA that holds that chunk (the "owner", CTA (nch - 1) % 2) appends the key and the raw value to the cache.
CTA 1 hands its softmax state to CTA 0 through distributed shared memory.  The positions below cover both owners, a CTA 1 with no
chunk at all (p < 64), a new position that opens a chunk (p % 64 == 0: nothing to bulk-load), rings that wrap many times (p = 2047,
max_ctx - 1) and a context that is not a multiple of 64 (the Qwen3-TTS code predictor's 32).

The float64 reference starts from the same fp32 inputs: RMSNorm with the gains, then RoPE with the kernel's fp32 angles, then softmax
over the cached rows 0..p-1 plus the new key, times V.  Every cache row the kernel may not read (>= p) is NaN before the launch, so a
new row read from the cache instead of q|k|v shows up as a NaN output.  After the launch: row p holds the new key and the value bit
for bit, rows < p are unchanged bit for bit, rows > p are still NaN, and no output row of an inactive or skipped row is written.

The output is the o projection's B operand: bf16 hi/lo rows b and 8 + b, whose exact value carries about 17 significant bits, so a
relative error of a few 1e-6 is the floor of the format.  Errors are the worst over a launch's rows of (relative L2, max |error| /
max |reference|) per row."""
import math

import pytest
import torch

from attention_reference import FREQS, HD, decode_attn, qk_gains, rmsnorm64, rope64
from gemm_reference import assert_lo_within_half_ulp, errors

pytestmark = pytest.mark.gpu

LO_ROW, EPS, Q_SCALE = 8, 1e-6, 3.0        # q scaled so that the scores have a standard deviation of about 3
MAX_CTX = 2113                             # max_ctx - 1 = 2112 opens chunk 33
# 8 rows per launch: chunk counts odd and even in each, so both CTAs own a new position in both launches
POS_GROUPS = ([0, 65, 127, 192, 2047, 1, 320, 129], [64, 63, 255, 128, 319, 191, MAX_CTX - 1, 256])
# the Qwen3-TTS code predictor: max_context = max(32, groups + 8) = 32 for 16 code groups
CP_CTX, CP_POS = 32, [0, 1, 15, 16, 17, 23, 30, 31]
# Measured on an H100 80GB HBM3 (700 W power limit), worst over every launch of this file (relative L2 / max over peak): output
# 3.1e-6 / 6.8e-6 (every ratio; the sharp, geometry and skipped-row launches 2.5e-6 .. 3.0e-6 / 4.8e-6 .. 6.3e-6), new key row
# 1.4e-7 / 2.2e-7 with q/k norm, 4.9e-8 / 1.1e-7 without (fp32 norm, sincosf and RoPE against float64).  Bounds 3x.
TOL = (1e-5, 2e-5)
K_TOL = (4e-7, 8e-7)


def _bits(x):
    return x.view(torch.int32)


def _problem(B, nq, nkv, max_ctx, pos, seed, q_scale=Q_SCALE):
    """q|k|v rows [B, (nq + 2 nkv) * 128] (q scaled), pos [B] int32, caches with N(0, 1) rows below each row's position and NaN from it."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn(B, (nq + 2 * nkv) * HD, device="cuda", generator=g)
    qkv[:, :nq * HD] *= q_scale
    kc = torch.full((B, nkv, max_ctx, HD), float("nan"), device="cuda")
    vc = torch.full_like(kc, float("nan"))
    for b, p in enumerate(pos):
        n = min(max(p, 0), max_ctx)
        kc[b, :, :n] = torch.randn(nkv, n, HD, device="cuda", generator=g)
        vc[b, :, :n] = torch.randn(nkv, n, HD, device="cuda", generator=g)
    return qkv, torch.tensor(pos, dtype=torch.int32, device="cuda"), kc, vc


def _heads(row, nq, nkv):
    return row[:nq * HD].view(nq, HD), row[nq * HD:(nq + nkv) * HD].view(nkv, HD), row[(nq + nkv) * HD:].view(nkv, HD)


def new_qk(row, p, nq, nkv, qn, kn, eps):
    """float64 normalised, rotated q heads [nq, 128] and new key [nkv, 128] of one q|k|v row at position p."""
    q, k, _ = _heads(row, nq, nkv)
    return rope64(rmsnorm64(q, qn, eps)[:, None], [p])[:, 0], rope64(rmsnorm64(k, kn, eps)[:, None], [p])[:, 0]


def reference(qkv, pos, kc, vc, nq, nkv, qn, kn, eps):
    """{row: (float64 output [nq * 128], new key [nkv, 128], scores [nkv, G, p + 1])} for the rows with 0 <= p < max_ctx."""
    G, ref = nq // nkv, {}
    for b, p in enumerate(pos):
        if not 0 <= p < kc.shape[2]:
            continue
        qr, kr = new_qk(qkv[b], p, nq, nkv, qn, kn, eps)
        v = _heads(qkv[b], nq, nkv)[2]
        keys = torch.cat([kc[b, :, :p].double(), kr[:, None]], 1)
        vals = torch.cat([vc[b, :, :p].double(), v.double()[:, None]], 1)
        s = qr.view(nkv, G, HD) @ keys.transpose(-1, -2) / math.sqrt(HD)
        ref[b] = ((torch.softmax(s, -1) @ vals).reshape(nq * HD), kr, s)
    return ref


def check(name, out, qkv, pos, kc0, vc0, kc, vc, nq, nkv, qn=None, kn=None, eps=EPS, tol=TOL):
    """The cache contract and the output against float64; returns (worst output errors, worst new-key errors)."""
    pos = pos.tolist()
    ref = reference(qkv, pos, kc0, vc0, nq, nkv, qn, kn, eps)
    written = torch.zeros(16, dtype=torch.bool, device="cuda")
    e_out, e_k = (0.0, 0.0), (0.0, 0.0)
    for b, p in enumerate(pos):
        if b not in ref:                                     # skipped: neither cache is touched
            assert torch.equal(_bits(kc[b]), _bits(kc0[b])) and torch.equal(_bits(vc[b]), _bits(vc0[b])), (name, b, p)
            continue
        o_ref, k_ref, _ = ref[b]
        written[b] = written[LO_ROW + b] = True
        assert torch.equal(_bits(kc[b, :, :p]), _bits(kc0[b, :, :p])) and torch.equal(_bits(vc[b, :, :p]), _bits(vc0[b, :, :p])), \
            (name, b, p, "rows below the position changed")
        assert kc[b, :, p + 1:].isnan().all() and vc[b, :, p + 1:].isnan().all(), (name, b, p, "rows above the position written")
        assert torch.equal(_bits(vc[b, :, p]), _bits(_heads(qkv[b], nq, nkv)[2])), (name, b, p, "value row")
        ek = errors(kc[b, :, p], k_ref)
        e_k = max(e_k[0], ek[0]), max(e_k[1], ek[1])
        hi, lo = out[b], out[LO_ROW + b]
        assert torch.isfinite(hi.float()).all() and torch.isfinite(lo.float()).all(), (name, b, p)
        assert_lo_within_half_ulp(hi, lo)
        e = errors(hi.double() + lo.double(), o_ref)
        e_out = max(e_out[0], e[0]), max(e_out[1], e[1])
    assert out[~written].float().isnan().all(), (name, "an output row of an inactive row was written")
    print(f"{name}: out {e_out[0]:.2e} / {e_out[1]:.2e}, new key {e_k[0]:.2e} / {e_k[1]:.2e}")
    assert e_k[0] < K_TOL[0] and e_k[1] < K_TOL[1], (name, e_k)
    assert e_out[0] < tol[0] and e_out[1] < tol[1], (name, e_out)
    return e_out, e_k


def run_and_check(b2a, name, qkv, pos, kc, vc, nq, nkv, qn=None, kn=None, eps=EPS, tol=TOL):
    kc0, vc0 = kc.clone(), vc.clone()
    st, out = decode_attn(b2a, qkv, pos, kc, vc, nq, nkv, qn, kn, eps)
    assert st == 0, b2a._ffi.lib().b2a_last_error()
    return check(name, out, qkv, pos, kc0, vc0, kc, vc, nq, nkv, qn, kn, eps, tol)


@pytest.mark.parametrize("norm", [False, True], ids=["plain", "qk_norm"])
@pytest.mark.parametrize("G,nkv", [(1, 1), (1, 8), (2, 1), (2, 8), (3, 1), (3, 8), (4, 1), (4, 8), (6, 1), (6, 4), (8, 1), (8, 4)])
def test_decode_attention_every_ratio(b2a, G, nkv, norm):
    """Every GQA ratio, 16 positions around every chunk edge in two launches of 8 rows.  With q/k norm, row 1's raw k is scaled to
    about 1e-4, where eps (1e-6) outweighs mean(k^2) in the norm.  Measured: 3.1e-6 / 6.8e-6 worst (plain and q/k norm alike);
    bounds: TOL."""
    nq = nkv * G
    qn, kn = qk_gains(10 * G + nkv, Q_SCALE) if norm else (None, None)
    for i, grp in enumerate(POS_GROUPS):
        qkv, pos, kc, vc = _problem(8, nq, nkv, MAX_CTX, grp, 100 * G + 10 * nkv + i, 1.0 if norm else Q_SCALE)
        if norm:
            qkv[1, nq * HD:(nq + nkv) * HD] *= 1e-4
        run_and_check(b2a, f"G={G} nkv={nkv} norm={norm} group {i}", qkv, pos, kc, vc, nq, nkv, qn, kn)


@pytest.mark.parametrize("geometry", ["orpheus_24_8", "qwen3_16_8", "code_predictor_16_8"])
def test_decode_attention_shipped_geometry(b2a, geometry):
    """The decode steps the stacks run: Orpheus (24 q / 8 kv heads, no q/k norm), Qwen3-0.6B / VyvoTTS / the Qwen3-TTS talker (16 / 8,
    q/k norm) and the Qwen3-TTS code predictor (16 / 8, q/k norm, max_ctx 32, every position in one chunk).  Gains 1 + 0.3 N(0, 1)
    (q gains times 3 for the score spread), eps 1e-6, one k vector scaled to about 1e-4."""
    nq, nkv = (24, 8) if geometry.startswith("orpheus") else (16, 8)
    norm = not geometry.startswith("orpheus")
    max_ctx, groups = (CP_CTX, (CP_POS,)) if geometry.startswith("code") else (MAX_CTX, POS_GROUPS)
    qn, kn = qk_gains(7, Q_SCALE) if norm else (None, None)
    for i, grp in enumerate(groups):
        qkv, pos, kc, vc = _problem(8, nq, nkv, max_ctx, grp, 50 + i, 1.0 if norm else Q_SCALE)
        if norm:
            qkv[3, nq * HD:(nq + nkv) * HD] *= 1e-4
        run_and_check(b2a, f"{geometry} group {i}", qkv, pos, kc, vc, nq, nkv, qn, kn)


def test_decode_attention_skipped_rows(b2a):
    """B = 6 of 8 rows: pos = -1 and pos = max_ctx write neither the output nor the cache (whose rows are all data there), and output
    rows 6, 7, 14, 15 stay NaN."""
    nq, nkv, max_ctx = 6, 2, 200
    qkv, pos, kc, vc = _problem(6, nq, nkv, max_ctx, [5, -1, 130, max_ctx, 0, 64], 3)
    run_and_check(b2a, "skipped rows", qkv, pos, kc, vc, nq, nkv)


def _dominant_chunk(p):
    """A chunk of the CTA that does not own position p, before the last chunk, near the middle of the row."""
    nch = p // 64 + 1
    other = 1 - (nch - 1) % 2
    c = other + 2 * ((nch - 2 - other) // 4)
    assert c % 2 == other and 0 <= c < nch - 1
    return c


SHARP = {   # regime: (positions, dominant key of a row at position p)
    "other_cta": ([64, 100, 128, 200, 300, 700, 1000, 2047], lambda p: _dominant_chunk(p) * 64 + 17),
    "new_position": ([0, 1, 64, 65, 128, 320, 2047, MAX_CTX - 1], lambda p: p),
    "first_key": ([64, 129, 256, 319, 640, 1000, 2047, MAX_CTX - 1], lambda p: 0),
    "all_equal": ([0, 1, 63, 64, 191, 320, 2047, MAX_CTX - 1], None),
}


def _unrope(k, p):
    """fp32 k such that RoPE at position p gives (about) k: the rotation by the opposite angle."""
    ang = (torch.tensor([float(p)]) / FREQS).double().to(k.device)
    c, s = torch.cos(ang), torch.sin(ang)
    k1, k2 = k[..., :HD // 2].double(), k[..., HD // 2:].double()
    return torch.cat([k1 * c + k2 * s, k2 * c - k1 * s], -1).float()


@pytest.mark.parametrize("regime", list(SHARP))
def test_decode_attention_sharp_scores(b2a, regime):
    """Scores with a standard deviation of about 3 and one key about 30 logits above the rest (a score of 40 for every q head of the kv
    head): in a chunk of the CTA that does not own the new position (the DSMEM merge must carry it), at the new position (spliced from
    q|k|v) or at position 0 of a long row.  all_equal: every key of a row is the same vector, so the output is the mean of V.
    3 q heads per kv head, 2 kv heads, no q/k norm."""
    nq, nkv, G = 6, 2, 3
    positions, target = SHARP[regime]
    qkv, pos, kc, vc = _problem(8, nq, nkv, MAX_CTX, positions, 900 + list(SHARP).index(regime))
    g = torch.Generator(device="cuda").manual_seed(5)
    for b, p in enumerate(positions):
        qr, _ = new_qk(qkv[b], p, nq, nkv, None, None, 0.0)
        if target is None:
            key = torch.randn(nkv, HD, device="cuda", generator=g)
            kc[b, :, :p] = key[:, None]
            qkv[b, nq * HD:(nq + nkv) * HD] = _unrope(key, p).reshape(-1)
            continue
        u = qr.view(nkv, G, HD).sum(1)
        u = u / u.norm(dim=-1, keepdim=True)
        amp = 40.0 * math.sqrt(HD) / (qr.view(nkv, G, HD) * u[:, None]).sum(-1).min(-1).values    # [nkv]
        key = (amp[:, None] * u).float()
        t = target(p)
        if t < p:
            kc[b, :, t] = key
        else:
            qkv[b, nq * HD:(nq + nkv) * HD] = _unrope(key, p).reshape(-1)
    for b, (_, _, s) in reference(qkv, positions, kc, vc, nq, nkv, None, None, 0.0).items():
        if target is None:
            assert (s.amax(-1) - s.amin(-1)).max() < 1e-3
        elif positions[b] > 0:
            top = s.topk(2, -1).values
            assert (top[..., 0] - top[..., 1]).min() > 20.0 and (s.argmax(-1) == target(positions[b])).all()
    run_and_check(b2a, f"sharp {regime}", qkv, pos, kc, vc, nq, nkv)


def test_decode_attention_deterministic(b2a):
    """Two launches on the same inputs give the same output and cache bits."""
    nq, nkv = 24, 8
    qn, kn = qk_gains(11, Q_SCALE)
    qkv, pos, kc, vc = _problem(8, nq, nkv, MAX_CTX, POS_GROUPS[1], 77, 1.0)
    kc2, vc2 = kc.clone(), vc.clone()
    st1, out1 = decode_attn(b2a, qkv, pos, kc, vc, nq, nkv, qn, kn, EPS)
    st2, out2 = decode_attn(b2a, qkv, pos, kc2, vc2, nq, nkv, qn, kn, EPS)
    assert st1 == 0 and st2 == 0
    assert torch.equal(out1.view(torch.int16), out2.view(torch.int16))
    assert torch.equal(_bits(kc), _bits(kc2)) and torch.equal(_bits(vc), _bits(vc2))


@pytest.mark.parametrize("B,nq,nkv,norms", [(9, 8, 8, 2), (1, 12, 8, 2), (1, 5, 1, 0), (1, 7, 1, 0), (1, 16, 1, 0), (1, 8, 8, 1)],
                         ids=["B9", "nq_not_multiple", "G5", "G7", "G16", "qnorm_without_knorm"])
def test_decode_attention_rejects(b2a, B, nq, nkv, norms):
    """Arguments the kernel has no instance or room for are refused before anything is launched: more than 8 rows, nq not a multiple of
    nkv, a GQA ratio outside {1, 2, 3, 4, 6, 8} (the launch's switch would run <8> on it, with the shared memory of the smaller ratio,
    which the kernel overruns) and one norm gain without the other (the kernel reads knorm whenever qnorm is given).  The buffers are
    sized for the largest geometry these arguments name."""
    f = b2a._ffi
    qkv = torch.zeros(16 * 32 * HD, device="cuda")
    kc, vc = torch.zeros(16 * 16 * 64 * HD, device="cuda"), torch.zeros(16 * 16 * 64 * HD, device="cuda")
    out = torch.full((16 * 32 * HD,), float("nan"), device="cuda", dtype=torch.bfloat16)
    pos = torch.zeros(16, dtype=torch.int32, device="cuda")
    gain = torch.ones(HD, device="cuda")
    qn, kn = (gain, gain) if norms == 2 else (gain, None) if norms == 1 else (None, None)
    st = f.lib().b2a_decode_attn_test(f.ptr(qkv), f.ptr(pos), f.ptr(FREQS.cuda()), f.ptr(qn), f.ptr(kn), EPS, f.ptr(kc), f.ptr(vc),
                                      f.ptr(out), B, nq, nkv, 64, None)
    torch.cuda.synchronize()
    assert st == f.ERR_INVALID_INPUT, (st, f.lib().b2a_last_error())
    assert out.float().isnan().all() and not kc.any() and not vc.any()
