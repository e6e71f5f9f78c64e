"""Parity at BASELINE.json's sizes with the kernel variants the product ships (VERDICT r1 weak #2/#3):
the default GEMM (variant 0, the persistent warp-specialised wgmma kernel), the default attention (variant 2, the
wgmma flash-attention kernel), the default Hyena scan (mode-split) -- each against the CPU oracle on the same seeded
inputs, at the 7B width and the 8k / 16k / 131k lengths; plus the fused scoring head and an end-to-end bound on the
quantity evo/scoring.py returns.

Collected before tests/test_gpu_parity.py (alphabetical order) so that a time-out late in the suite cannot skip them.
The CPU oracle runs on the GPU box's host cores: the sizes are chosen so that each test's oracle side takes seconds
(row / head subsets where the full problem would take minutes; the subset always covers the first, an interior and
the ragged last tile)."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

from oracle import stripedhyena_oracle as O          # noqa: E402
from evo_b200 import _lib                             # noqa: E402
from evo_b200.stripedhyena import StripedHyena, dotdict  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "tests", "harness"))
import gpu_bringup as G                               # noqa: E402

G._imports()
DEV = "cuda:0"
BF16_EPS = 2.0 ** -7


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()
    torch.set_num_threads(min(64, os.cpu_count() or 1))


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def maxerr(a, b):
    return (a.double().cpu() - b.double().cpu()).abs().max().item()


def meanerr(a, b):
    return (a.double().cpu() - b.double().cpu()).abs().mean().item()


def _filter_sd(D, H, seed=1, pole_mag=None):
    """Filter parameters of one Hyena layer (no MLP weights: at D = 4096 those would be 0.5 GB of unused randoms)."""
    g = torch.Generator().manual_seed(seed)
    mag = (0.5 + 0.45 * torch.rand(D, 8, 1, generator=g)) if pole_mag is None else (pole_mag[0] + (pole_mag[1] - pole_mag[0]) * torch.rand(D, 8, 1, generator=g))
    ang = (torch.rand(D, 8, 1, generator=g) * 2 - 1) * math.pi
    sd = {"blocks.0.filter.short_filter_weight": (torch.randn(3 * D, 1, 3, generator=g) * 0.3).bfloat16(),
          "blocks.0.filter.short_filter_bias": (torch.randn(3 * D, generator=g) * 0.1).bfloat16(),
          "blocks.0.filter.D": torch.randn(D, generator=g).bfloat16(),
          "blocks.0.filter.poles": torch.stack([mag * torch.cos(ang), mag * torch.sin(ang)], dim=-1),
          "blocks.0.filter.residues": torch.randn(D, 8, 1, 2, generator=g) * 0.3}
    p = "blocks.0.filter."
    f = {"w": sd[p + "short_filter_weight"].to(DEV), "b": sd[p + "short_filter_bias"].to(DEV), "D": sd[p + "D"].to(DEV),
         "p": sd[p + "poles"].to(DEV), "r": sd[p + "residues"].to(DEV)}
    return sd, f


def _oracle_hyena(sd, z, H, hd, dtype, state="fft", heads_per_chunk=4):
    """The oracle's parallel (FFT) Hyena operator on z (B, L, 3D) in `dtype` arithmetic (bf16 = the reference's rounding
    points), evaluated a few heads at a time so the (channels, 8, 2L) spectra stay at ~1 GB of host memory.
    state: "fft" = prefill_via_modal_fft as the reference computes it; "direct" = sum_tau p^(L-1-tau) x1v[tau] evaluated
    term by term in complex128 (truth for long L, where the FFT's temporaries would not fit); None = skip."""
    p = "blocks.0.filter."
    cast = (lambda t: t.to(dtype)) if dtype != torch.bfloat16 else (lambda t: t)
    B, L, _ = z.shape
    ys, sts = [], []
    for h0 in range(0, H, heads_per_chunk):
        h1 = min(H, h0 + heads_per_chunk)
        c3, c1 = slice(h0 * 3 * hd, h1 * 3 * hd), slice(h0 * hd, h1 * hd)
        poles, residues = sd[p + "poles"][c1], sd[p + "residues"][c1]
        if dtype == torch.float64:
            poles, residues = poles.double(), residues.double()
        z_pre, _ = O.fir_parallel(z[:, :, c3].to(dtype), cast(sd[p + "short_filter_weight"][c3]), cast(sd[p + "short_filter_bias"][c3]))
        h = O.hyena_filter(poles, residues, L)
        y, st = O.iir_parallel(z_pre, h, cast(sd[p + "D"][c1]), poles, h1 - h0, hd, want_state=(state == "fft"))
        if state == "direct":
            _, x1, v = O.column_split(z_pre, h1 - h0, hd)
            x1v = (x1 * v).double()                                            # (B, Dc, L)
            pc = torch.view_as_complex(poles.double())[..., 0]                 # (Dc, 8)
            k = torch.arange(L - 1, -1, -1, dtype=torch.float64)               # exponent of p applied to x1v[tau]
            st = torch.stack([(x1v * torch.exp(torch.log(pc[:, s])[:, None] * k)[None]).sum(-1) for s in range(pc.shape[1])], dim=-1)
        ys.append(y)
        sts.append(st)
    return torch.cat(ys, dim=-1), (torch.cat(sts, dim=1) if state else None)


# ------------------------------------------------------------------ Hyena scan at the 7B width and at 131 072 tokens
def test_hyena_7b_width_8193_vs_oracle():
    """D = 4096 (32 heads), batch 1 x 8193 tokens: the shipped scan vs the oracle's FFT operator, bf16-faithful and fp64."""
    D, H, B, L = 4096, 32, 1, 8193
    sd, f = _filter_sd(D, H, seed=21)
    torch.manual_seed(21)
    z = torch.randn(B, L, 3 * D).bfloat16()
    y, st, _ = G._hyena_call(z.to(DEV), f, B, L, D, H)
    yb, stb = _oracle_hyena(sd, z, H, 128, torch.bfloat16)
    yt, stt = _oracle_hyena(sd, z, H, 128, torch.float64)
    assert torch.isfinite(y.float()).all()
    assert (y.cpu() == yb).float().mean() > 0.995
    assert maxerr(y, yb) <= 2 * BF16_EPS * max(1.0, yb.abs().max().item())
    assert meanerr(y, yt) <= 1.25 * meanerr(yb, yt) + 1e-6
    stc = torch.view_as_complex(st.cpu())
    assert (stc - stb).abs().max() <= 2e-4 * max(1.0, stb.abs().max().item())
    assert (stc - stt.to(torch.complex64)).abs().max() <= 1e-2 * max(1.0, stt.abs().max().item())


@pytest.mark.parametrize("nseg", [0, 1])
def test_hyena_131072_tokens_poles_near_the_unit_circle(nseg):
    """L = 131 072 (BASELINE configs[2]) on a 256-channel slice with pole magnitudes up to 0.9999 -- filter memories of
    ~10^5 tokens, the regime where an fp32 recurrence and an fp32 FFT could part ways.  nseg = 0: the launcher's own
    segmentation (16 CTAs x segments + carry pass), 1: one sequential scan."""
    D, H, B, L = 256, 2, 1, 131072
    sd, f = _filter_sd(D, H, seed=5, pole_mag=(0.9, 0.9999))
    torch.manual_seed(5)
    z = (torch.randn(B, L, 3 * D) * 0.5).bfloat16()
    y, st, _ = G._hyena_call(z.to(DEV), f, B, L, D, H, force=nseg)
    yb, _ = _oracle_hyena(sd, z, H, 128, torch.bfloat16, state=None, heads_per_chunk=1)
    yt, stt = _oracle_hyena(sd, z, H, 128, torch.float64, state="direct", heads_per_chunk=1)
    assert torch.isfinite(y.float()).all()
    scale = max(1.0, yb.abs().max().item())
    assert maxerr(y, yb) <= 2 * BF16_EPS * scale
    assert (y.cpu() == yb).float().mean() > 0.99
    assert meanerr(y, yt) <= 1.25 * meanerr(yb, yt) + 1e-6
    # the last quarter of the sequence alone (errors of a drifting recurrence would grow with t)
    q = 3 * L // 4
    assert meanerr(y[:, q:], yt[:, q:]) <= 1.25 * meanerr(yb[:, q:], yt[:, q:]) + 1e-6
    stc = torch.view_as_complex(st.cpu())
    assert (stc - stt.to(torch.complex64)).abs().max() <= 1e-2 * max(1.0, stt.abs().max().item())


# ------------------------------------------------------------------ attention, shipped variant, full head count / long rope
@pytest.mark.parametrize("variant", [2, 3])
def test_attention_variant2_32_heads_8193_vs_oracle(variant):
    """ABI variants 2 and 3 of the attention call (both run the one wgmma flash-attention kernel) at H = 32, L = 8193: every
    head against the independent CUDA-core comparator, four heads (first, two interior, last) against the CPU oracle in
    bf16-faithful and fp64 arithmetic."""
    from tests import support as TS
    B, L, H = 1, 8193, 32
    torch.manual_seed(8)
    qkv = torch.randn(B, L, 3, H, 128).bfloat16()
    out = G._attn(qkv.to(DEV), B, L, H, variant)
    comp = G._attn(qkv.to(DEV), B, L, H, variant, simple=True)
    assert not torch.isnan(out.float()).any()
    assert maxerr(out, comp) <= 4 * BF16_EPS * max(1.0, comp.float().abs().max().item())
    assert meanerr(out, comp) < 2e-4
    heads = [0, 11, 22, 31]
    sub = qkv[:, :, :, heads]
    ref = O.causal_attention(sub[:, :, 0], sub[:, :, 1], sub[:, :, 2])                       # (B, L, 4, 128)
    truth = O.causal_attention(sub[:, :, 0].double(), sub[:, :, 1].double(), sub[:, :, 2].double())
    got = out.cpu().view(B, L, H, 128)[:, :, heads]
    assert maxerr(got, ref) <= 4 * BF16_EPS * max(1.0, ref.abs().max().item())
    assert meanerr(got, truth) <= 1.25 * meanerr(ref, truth) + 1e-5
    assert TS.lib() is not None


def test_rotary_scaled_16_plus_attention_variant2_16384_vs_oracle():
    """evo-1-131k's interpolated rotary (positions / 16) applied by evo_rotary_qk, then the default attention kernel, at
    L = 16 384 (one rank's share of the 131k context) on two heads, vs the oracle."""
    B, L, H = 1, 16384, 2
    lib = _lib.lib()
    torch.manual_seed(16)
    qkv = torch.randn(B, L, 3, H, 128).bfloat16()
    cos, sin = O.rotary_tables(L, 128, scaling_factor=16.0, dtype=torch.bfloat16)
    q = O.apply_rotary(qkv[:, :, 0], cos, sin)
    k = O.apply_rotary(qkv[:, :, 1], cos, sin)
    ref = O.causal_attention(q, k, qkv[:, :, 2]).reshape(B, L, H * 128)
    truth = O.causal_attention(O.apply_rotary(qkv[:, :, 0].double(), cos.double(), sin.double()),
                               O.apply_rotary(qkv[:, :, 1].double(), cos.double(), sin.double()), qkv[:, :, 2].double()).reshape(B, L, H * 128)
    inv = (1.0 / (10000 ** (torch.arange(0, 128, 2, dtype=torch.float32) / 128))).to(DEV)
    cd = torch.empty(L, 64, dtype=torch.bfloat16, device=DEV)
    sdv = torch.empty_like(cd)
    _lib.check(lib.evo_rope_tables(_lib.ptr(cd), _lib.ptr(sdv), _lib.ptr(inv), 0, L, 64, 16.0, stream()))
    # CUDA sincosf vs the CPU libm differ by <= 1 fp32 ulp; after rounding to bf16 a handful of entries may flip
    assert (cd.cpu() == cos).float().mean() > 0.999 and (sdv.cpu() == sin).float().mean() > 0.999
    assert maxerr(cd, cos) <= 2 ** -8 and maxerr(sdv, sin) <= 2 ** -8
    qd = qkv.to(DEV).contiguous()
    _lib.check(lib.evo_rotary_qk(_lib.ptr(qd), _lib.ptr(cd), _lib.ptr(sdv), B, L, H, 128, stream()))
    assert (qd[:, :, 0].cpu() == q).float().mean() > 0.995
    out = G._attn(qd, B, L, H, 2)
    assert maxerr(out, ref) <= 4 * BF16_EPS * max(1.0, ref.abs().max().item())
    assert meanerr(out, truth) <= 1.25 * meanerr(ref, truth) + 1e-5


# ------------------------------------------------------------------ GEMM, shipped variant, BASELINE shapes
def _row_subset(M):
    """First block, an interior 256-row pair block, and the ragged tail (65544 = 256 * 256 + 8)."""
    idx = list(range(0, 256)) + list(range(M // 2 - 128, M // 2 + 128)) + list(range(M - 264, M))
    return torch.tensor(sorted(set(i for i in idx if 0 <= i < M)))


@pytest.mark.parametrize("variant", [0, 1])
def test_gemm_projection_65544x12288x4096_vs_cublaslt_and_oracle(variant):
    from tests import support as TS
    M, N, K = 65544, 12288, 4096
    torch.manual_seed(0)
    a = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=DEV) / 64).bfloat16()
    bias = torch.randn(N, device=DEV).bfloat16()
    out = G._gemm(a, w, M, N, K, _lib.EPI_BIAS, variant, bias=bias)
    ref = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ws = torch.empty(64 << 20, dtype=torch.uint8, device=DEV)
    p = _lib.GemmParams(A=a.data_ptr(), lda=K, W=w.data_ptr(), C=ref.data_ptr(), ldc=N, bias=bias.data_ptr(), residual=None, ldr=N, M=M, N=N, K=K, epilogue=1, variant=0)
    TS.check(TS.lib().evot_gemm_cublaslt(C.byref(p), _lib.ptr(ws), ws.numel(), stream()), "cublaslt comparator")
    torch.cuda.synchronize()
    assert not torch.isnan(out.float()).any()
    assert (out.float() - ref.float()).abs().max().item() <= 2 * BF16_EPS * ref.float().abs().max().item()
    assert (out == ref).float().mean().item() > 0.98
    # CPU oracle (fp64 accumulate, then the reference's rounding: bf16(acc + bias)) on a row subset
    rows = _row_subset(M)
    truth = a[rows.to(DEV)].cpu().double() @ w.cpu().double().T + bias.cpu().double()
    got = out[rows.to(DEV)].cpu()
    assert (got == truth.bfloat16()).float().mean().item() > 0.98
    assert (got.double() - truth).abs().max().item() <= 1.01 * BF16_EPS * truth.abs().max().item()


def test_gemm_gate_epilogue_65544x22016x4096_vs_oracle():
    """The fused GELU-gate GEMM at the MLP's packed width (2 x 11008): GPU vs act(l1 x) * l2 x with the reference's bf16
    rounding points, fp64 accumulation, on a row subset; finiteness and the zero padding over the full output."""
    M, K, inner, ipad = 65544, 4096, 10928, 11008
    torch.manual_seed(1)
    a = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
    l1 = (torch.randn(inner, K, device=DEV) / 64).bfloat16()
    l2 = (torch.randn(inner, K, device=DEV) / 64).bfloat16()
    pad = lambda w: torch.nn.functional.pad(w, (0, 0, 0, ipad - inner)).view(ipad // 128, 1, 128, K)
    w12 = torch.cat([pad(l1), pad(l2)], dim=1).reshape(2 * ipad, K).contiguous()
    out = G._gemm(a, w12, M, 2 * ipad, K, _lib.EPI_GELU_GATE, 0, ldc=ipad)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    assert out[:, inner:].float().abs().max().item() == 0.0            # gelu(0) * 0 in the zero-padded columns
    rows = _row_subset(M)
    ar = a[rows.to(DEV)].cpu().double()
    h1 = (ar @ l1.cpu().double().T).bfloat16()
    h2 = (ar @ l2.cpu().double().T).bfloat16()
    want = (torch.nn.functional.gelu(h1.float()).bfloat16().float() * h2.float()).bfloat16()
    got = out[rows.to(DEV), :inner].cpu()
    assert (got == want).float().mean().item() > 0.97
    assert (got.float() - want.float()).abs().max().item() <= 3 * BF16_EPS * max(1.0, want.float().abs().max().item())


# ------------------------------------------------------------------ fused scoring head
@pytest.mark.parametrize("M", [1, 129, 8200])
def test_fused_unembed_score_vs_fp64(M):
    """evo_unembed_score: logits never written; logprob / entropy vs fp64 statistics over the bf16-rounded logits (the
    reference's logits tensor is bf16), and vs evo_logprobs on the materialised logits."""
    lib = _lib.lib()
    K, V = 4096, 512
    torch.manual_seed(M)
    x = (torch.randn(M, K, device=DEV) * 0.7).bfloat16()
    w = (torch.randn(V, K, device=DEV) * (2.5 / 64)).bfloat16()
    tg = torch.randint(0, V, (M,), device=DEV)
    if M > 3:
        tg[3] = -1
    lp = torch.empty(M, dtype=torch.float32, device=DEV)
    ent = torch.empty(M, dtype=torch.float32, device=DEV)
    n = lib.evo_unembed_score_workspace(M, V)
    ws = torch.empty(max(n, 1), dtype=torch.uint8, device=DEV)
    sp = _lib.ScoreParams(x=x.data_ptr(), W=w.data_ptr(), targets=tg.data_ptr(), logprobs=lp.data_ptr(), entropy=ent.data_ptr(), M=M, V=V, K=K,
                          workspace=ws.data_ptr(), workspace_bytes=n)
    _lib.check(lib.evo_unembed_score(C.byref(sp), stream()), "evo_unembed_score")
    logits = G._gemm(x, w, M, V, K, _lib.EPI_NONE, 0)                   # the same GEMM, materialised
    torch.cuda.synchronize()
    lsm = torch.log_softmax(logits.double().cpu(), -1)
    want = lsm.gather(1, tg.clamp(min=0).cpu()[:, None])[:, 0]
    if M > 3:
        want[3] = 0
    assert maxerr(lp, want) < 2e-5
    want_ent = -(lsm.exp() * lsm).sum(-1)
    assert maxerr(ent, want_ent) < 5e-5
    old = torch.empty(M, dtype=torch.float32, device=DEV)
    _lib.check(lib.evo_logprobs(_lib.ptr(logits), _lib.ptr(tg), _lib.ptr(old), M, V, stream()))
    assert maxerr(lp, old) < 2e-5


# ------------------------------------------------------------------ 7B-width model at 8193 tokens; end-to-end scoring bound
def test_two_layer_7b_width_8193_tokens_logits_and_score_vs_oracle():
    """1 Hyena + 1 attention block at D = 4096 / 32 heads, batch 1 x 8192 nt + BOS (the per-sequence shape of BASELINE
    configs[1]): logits vs both oracle modes, and the number evo/scoring.py returns -- the mean log-likelihood through
    evo_b200.score_sequences (fused head) -- against the bf16-faithful oracle within BASELINE.md section 4's 2e-3."""
    import evo_b200
    cfg = O.evo_config("evo-1-8k-base")
    cfg.update(num_layers=2, attn_layer_idxs=[1], hyena_layer_idxs=[0])
    sd = O.random_state_dict(cfg, seed=3)
    m = StripedHyena(dotdict(cfg))
    m.load_state_dict(sd, strict=True)
    m.to_bfloat16_except_poles_residues()
    m = m.to(DEV)
    tok = evo_b200.CharLevelTokenizer(512)
    rng = np.random.default_rng(2)
    seq = "".join(rng.choice(list("ACGT"), size=8192))
    ids = torch.tensor([[tok.eod_id] + tok.tokenize(seq)], dtype=torch.long)
    lg, _ = m(ids.to(DEV))
    lb, _ = O.OracleStripedHyena(cfg, sd, torch.bfloat16)(ids)
    lt, _ = O.OracleStripedHyena(cfg, sd, torch.float32)(ids)
    lsm = lambda t: torch.log_softmax(t.double().cpu(), -1)
    e_gpu, e_ref = (lsm(lg) - lsm(lt)).abs().mean().item(), (lsm(lb) - lsm(lt)).abs().mean().item()
    assert e_gpu <= 1.25 * e_ref + 2e-3, (e_gpu, e_ref)
    # direct, GPU vs the bf16-faithful oracle: mean |delta logprob| over all positions and vocabulary entries
    assert (lsm(lg) - lsm(lb)).abs().mean().item() <= 1.25 * e_ref + 2e-3
    agree_gpu = (lg.cpu().argmax(-1) == lt.argmax(-1)).float().mean().item()
    agree_ref = (lb.argmax(-1) == lt.argmax(-1)).float().mean().item()
    assert agree_gpu >= agree_ref - 0.02, (agree_gpu, agree_ref)
    # the score: mean over 8192 positions of log p(token | prefix)
    want_b = lsm(lb)[0, :-1].gather(1, ids[0, 1:, None])[:, 0].mean().item()
    want_t = lsm(lt)[0, :-1].gather(1, ids[0, 1:, None])[:, 0].mean().item()
    got = float(evo_b200.score_sequences([seq], m, tok, device=DEV)[0])
    assert abs(got - want_b) <= 2e-3, (got, want_b, want_t)
    assert abs(got - want_t) <= abs(want_b - want_t) + 2e-3, (got, want_b, want_t)
    ent = evo_b200.positional_entropies([seq], m, tok, device=DEV)[0]
    want_ent = -(lsm(lb).exp() * lsm(lb)).sum(-1)[0, :-1].numpy()
    assert ent.shape == (8192,)
    assert np.abs(ent - want_ent).mean() <= 1.25 * e_ref * 5 + 5e-3
