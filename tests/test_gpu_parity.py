"""Parity tests proper: every sm_90a kernel, called through the C ABI, against the CPU oracle
on the same seeded inputs; plus size-independent properties at BASELINE.json's full sizes.

Tolerances.  Integer/index work (embedding gather, KV append, FIR state) and every op whose
bf16 rounding points are reproduced one-for-one (RMSNorm, rotary tables, the decode step) must
be BIT-EXACT.  Floating-point kernels with a different summation order than the CPU oracle
(scan vs FFT, tensor-core vs CPU GEMM, online softmax) are held to
    err(GPU, fp64 truth) <= 1.25 * err(bf16 oracle, fp64 truth) + eps
i.e. the GPU result must be as close to exact arithmetic as the reference's own bf16 pipeline,
and to a direct bound against the bf16-faithful oracle stated in each test."""
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

from oracle import stripedhyena_oracle as O          # noqa: E402  (tests may use the oracle)
from evo_b200 import _lib                             # noqa: E402
from evo_b200.stripedhyena import StripedHyena, dotdict  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "tests", "harness"))
import gpu_bringup as G                               # noqa: E402  (shared launch helpers, tests/harness/)

G._imports()
DEV = "cuda:0"
BF16_EPS = 2.0 ** -7      # one bf16 ulp relative to the magnitude (8 significand bits)


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()        # raises if the extension is missing: no fallback


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def maxerr(a, b):
    return (a.double().cpu() - b.double().cpu()).abs().max().item()


def meanerr(a, b):
    return (a.double().cpu() - b.double().cpu()).abs().mean().item()


# ------------------------------------------------------------------ glue kernels: bit exact
@pytest.mark.parametrize("D,rows", [(256, 37), (4096, 129), (4096, 0), (4096, 16), (8192, 3), (512, 64), (4096, 65)])
def test_rmsnorm_bit_exact(D, rows):
    torch.manual_seed(D + rows)
    x = (torch.randn(rows, D) * 3).bfloat16()
    sc = (1 + 0.1 * torch.randn(D)).bfloat16()
    xd, sd = x.to(DEV), sc.to(DEV)
    od = torch.empty(rows, D, dtype=torch.bfloat16, device=DEV)
    _lib.check(_lib.lib().evo_rmsnorm(_lib.ptr(xd), _lib.ptr(sd), _lib.ptr(od), rows, D, 1e-6, stream()))
    if rows:
        assert torch.equal(od.cpu(), O.rms_norm(x, sc, 1e-6))


def test_rmsnorm_zero_row_is_finite():
    x = torch.zeros(3, 256, dtype=torch.bfloat16, device=DEV)
    sc = torch.ones(256, dtype=torch.bfloat16, device=DEV)
    od = torch.empty_like(x)
    _lib.check(_lib.lib().evo_rmsnorm(_lib.ptr(x), _lib.ptr(sc), _lib.ptr(od), 3, 256, 1e-6, stream()))
    assert torch.equal(od.cpu(), O.rms_norm(x.cpu(), sc.cpu(), 1e-6))     # eps outside the root keeps 0/eps = 0


@pytest.mark.parametrize("dt", [torch.int64, torch.int32])
def test_embed_gather(dt):
    tab = torch.randn(512, 256).bfloat16()
    ids = torch.randint(0, 512, (3, 11))
    tabd, idd = tab.to(DEV), ids.to(dt).to(DEV)
    od = torch.empty(33, 256, dtype=torch.bfloat16, device=DEV)
    _lib.check(_lib.lib().evo_embed(_lib.ptr(idd), int(dt == torch.int64), _lib.ptr(tabd), _lib.ptr(od), 33, 256, 512, stream()))
    assert torch.equal(od.cpu().view(3, 11, 256), tab[ids])


@pytest.mark.parametrize("scaling", [1.0, 16.0])
def test_rope_tables_and_rotary(scaling):
    L = 300
    cos_ref, sin_ref = O.rotary_tables(L, 128, scaling_factor=scaling, dtype=torch.bfloat16)
    inv = (1.0 / (10000 ** (torch.arange(0, 128, 2, dtype=torch.float32) / 128))).to(DEV)
    cd = torch.empty(L, 64, dtype=torch.bfloat16, device=DEV)
    sd = torch.empty_like(cd)
    _lib.check(_lib.lib().evo_rope_tables(_lib.ptr(cd), _lib.ptr(sd), _lib.ptr(inv), 0, L, 64, scaling, stream()))
    # CUDA sincosf vs the CPU libm differ by <= 1 fp32 ulp; after rounding to bf16 a handful of entries may flip
    assert (cd.cpu() == cos_ref).float().mean() > 0.999 and (sd.cpu() == sin_ref).float().mean() > 0.999
    assert maxerr(cd, cos_ref) <= 2 ** -8 and maxerr(sd, sin_ref) <= 2 ** -8
    torch.manual_seed(1)
    qkv = torch.randn(2, L, 3, 2, 128).bfloat16()
    qd, cdev, sdev = qkv.to(DEV).contiguous(), cos_ref.to(DEV), sin_ref.to(DEV)
    _lib.check(_lib.lib().evo_rotary_qk(_lib.ptr(qd), _lib.ptr(cdev), _lib.ptr(sdev), 2, L, 2, 128, stream()))
    out = qd.cpu()
    for which in (0, 1):
        ref = O.apply_rotary(qkv[:, :, which], cos_ref, sin_ref)
        assert (out[:, :, which] == ref).float().mean() > 0.999       # fma contraction may flip a last bit
        assert maxerr(out[:, :, which], ref) <= 2 ** -6
    assert torch.equal(out[:, :, 2], qkv[:, :, 2])


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("B,L,H,off", [(2, 300, 2, 0), (1, 129, 4, 77), (1, 8193, 32, 0)])
def test_gemm_rotary_epilogue_equals_projection_then_rotary(variant, B, L, H, off):
    """EVO_EPI_BIAS_ROPE (rotary inside the Wqkv GEMM's epilogue, where flash_attn's MHA applies it, mha.py:635-648) vs the
    two-kernel path (bias epilogue, then evo_rotary_qk): same rounding points, so bit-identical up to fma contraction; and
    vs the oracle's apply_rotary on the projection output."""
    d, K, M = H * 128, 256, B * L
    torch.manual_seed(L + H)
    a = (torch.randn(M, K, device=DEV) * 0.7).bfloat16()
    w = (torch.randn(3 * d, K, device=DEV) / 16).bfloat16()
    bias = torch.randn(3 * d, device=DEV).bfloat16()
    cos, sin = O.rotary_tables(off + L, 128, scaling_factor=16.0 if H == 4 else 1.0, dtype=torch.bfloat16)
    cd, sd_ = cos.to(DEV), sin.to(DEV)
    cp, sp = cd.data_ptr() + off * 64 * 2, sd_.data_ptr() + off * 64 * 2
    two = G._gemm(a, w, M, 3 * d, K, _lib.EPI_BIAS, variant, bias=bias)
    plain = two.clone()
    _lib.check(_lib.lib().evo_rotary_qk(_lib.ptr(two), C.c_void_p(cp), C.c_void_p(sp), B, L, H, 128, stream()))
    fused = torch.full((M, 3 * d), float("nan"), dtype=torch.bfloat16, device=DEV)
    p = _lib.GemmParams(A=a.data_ptr(), lda=K, W=w.data_ptr(), C=fused.data_ptr(), ldc=3 * d, bias=bias.data_ptr(), residual=None, ldr=3 * d,
                        M=M, N=3 * d, K=K, epilogue=_lib.EPI_BIAS_ROPE, variant=variant, rope_cos=cp, rope_sin=sp, rope_L=L, rope_cols=2 * d)
    _lib.check(_lib.lib().evo_gemm(C.byref(p), stream()), "evo_gemm(rope)")
    torch.cuda.synchronize()
    assert not torch.isnan(fused.float()).any()
    assert torch.equal(fused[:, 2 * d:], plain[:, 2 * d:])                      # v: bias only
    assert (fused == two).float().mean().item() > 0.9999 and maxerr(fused, two) <= 2 ** -6 * max(1.0, two.float().abs().max().item())
    qk = plain.cpu().view(B, L, 3, H, 128)
    for which in (0, 1):
        ref = O.apply_rotary(qk[:, :, which], cos[off:], sin[off:])
        got = fused.cpu().view(B, L, 3, H, 128)[:, :, which]
        assert (got == ref).float().mean() > 0.999 and maxerr(got, ref) <= 2 ** -6 * max(1.0, ref.abs().max().item())
    bad = _lib.GemmParams(A=a.data_ptr(), lda=K, W=w.data_ptr(), C=fused.data_ptr(), ldc=3 * d, bias=bias.data_ptr(), residual=None, ldr=3 * d,
                          M=M, N=3 * d, K=K, epilogue=_lib.EPI_BIAS_ROPE, variant=variant)                       # no tables
    assert _lib.lib().evo_gemm(C.byref(bad), stream()) != 0


def test_peer_scattered_outputs_of_gemm_and_attention_on_one_gpu():
    """The Ulysses re-shard fused into the epilogues (evo_gemm c_peers / evo_attn out_peers), exercised with the 'peers' being
    four buffers on THIS GPU: the scatter must equal the permute the NCCL path does (parallel._ulysses_attention)."""
    P, Lr, H, K = 4, 256, 8, 256
    d, Hl = H * 128, H // P
    dl = Hl * 128
    L = P * Lr
    torch.manual_seed(12)
    w = (torch.randn(3 * d, K, device=DEV) / 16).bfloat16()
    bias = torch.randn(3 * d, device=DEV).bfloat16()
    cos, sin = O.rotary_tables(L, 128, dtype=torch.bfloat16)
    cd, sd_ = cos.to(DEV), sin.to(DEV)
    full = [torch.full((L, 3, Hl, 128), float("nan"), dtype=torch.bfloat16, device=DEV) for _ in range(P)]      # one per "rank"
    arr = (C.c_void_p * P)(*[f.data_ptr() for f in full])
    want_qkv = []
    for r in range(P):                                                       # every "rank" projects its own Lr tokens
        a = (torch.randn(Lr, K, device=DEV) * 0.7).bfloat16()
        ref = G._gemm(a, w, Lr, 3 * d, K, _lib.EPI_BIAS, 0, bias=bias)
        _lib.check(_lib.lib().evo_rotary_qk(_lib.ptr(ref), C.c_void_p(cd.data_ptr() + r * Lr * 128), C.c_void_p(sd_.data_ptr() + r * Lr * 128), 1, Lr, H, 128, stream()))
        want_qkv.append(ref.view(Lr, 3, P, Hl, 128))
        p = _lib.GemmParams(A=a.data_ptr(), lda=K, W=w.data_ptr(), C=None, ldc=3 * dl, bias=bias.data_ptr(), residual=None, ldr=3 * dl, M=Lr, N=3 * d, K=K,
                            epilogue=_lib.EPI_BIAS_ROPE, variant=0, rope_cos=cd.data_ptr() + r * Lr * 128, rope_sin=sd_.data_ptr() + r * Lr * 128, rope_L=Lr, rope_cols=2 * d,
                            c_peers=C.cast(arr, C.c_void_p), n_c_peers=P, peer_period=d, peer_inner=dl, peer_row0=r * Lr)
        _lib.check(_lib.lib().evo_gemm(C.byref(p), stream()), "evo_gemm(peers)")
    torch.cuda.synchronize()
    whole = torch.cat(want_qkv, 0)                                           # (L, 3, P, Hl, 128)
    for pr in range(P):
        assert not torch.isnan(full[pr].float()).any()
        assert (full[pr] == whole[:, :, pr]).float().mean().item() > 0.9999   # fma contraction in the fused rotary may flip a last bit
    # attention of "rank" 1's heads over the whole sequence, rows scattered to the four token owners' ctx buffers
    ctxs = [torch.full((Lr, d), float("nan"), dtype=torch.bfloat16, device=DEV) for _ in range(P)]
    carr = (C.c_void_p * P)(*[c.data_ptr() for c in ctxs])
    me = 1
    f = full[me]
    plain = G._attn(f.view(1, L, 3, Hl, 128), 1, L, Hl, 2)                      # (1, L, dl)
    ap = _lib.AttnParams(out=None, B=1, Lq=L, Lk=L, H=Hl, hd=128, q_pos0=0, softmax_scale=1 / math.sqrt(128))
    ap.q, ap.q_tok_stride, ap.q_batch_stride = f.data_ptr(), 3 * dl, L * 3 * dl
    ap.k, ap.v, ap.kv_tok_stride, ap.kv_batch_stride = f.data_ptr() + dl * 2, f.data_ptr() + 2 * dl * 2, 3 * dl, L * 3 * dl
    ap.out_peers, ap.n_out_peers, ap.out_rows_per_peer, ap.out_row_stride, ap.out_col0 = C.cast(carr, C.c_void_p), P, Lr, d, me * dl
    _lib.check(_lib.lib().evo_attn_fwd_ws(C.byref(ap), 2, None, 0, stream()), "evo_attn_fwd(peers)")
    torch.cuda.synchronize()
    for r in range(P):
        assert torch.equal(ctxs[r][:, me * dl:(me + 1) * dl], plain[0, r * Lr:(r + 1) * Lr])
        assert torch.isnan(ctxs[r][:, :me * dl].float()).all() and torch.isnan(ctxs[r][:, (me + 1) * dl:].float()).all()     # other ranks' columns untouched
    assert _lib.lib().evo_attn_fwd_ws(C.byref(ap), 1, None, 0, stream()) != 0                                          # variant 1 refuses


def test_kv_append_and_logprobs():
    lib = _lib.lib()
    qkv = torch.randn(2, 5, 3, 2, 128).bfloat16()
    qd = qkv.to(DEV)
    cache = torch.zeros(3, 16, 2, 2, 128, dtype=torch.bfloat16, device=DEV)
    _lib.check(lib.evo_kv_append(_lib.ptr(qd), _lib.ptr(cache), 2, 5, 2, 128, 4, 16, stream()))
    cc = cache.cpu()
    assert torch.equal(cc[:2, 4:9, 0], qkv[:, :, 1]) and torch.equal(cc[:2, 4:9, 1], qkv[:, :, 2])
    assert cc[:, :4].abs().sum() == 0 and cc[2].abs().sum() == 0 and cc[:, 9:].abs().sum() == 0
    with pytest.raises(_lib.EvoError):
        _lib.check(lib.evo_kv_append(_lib.ptr(qd), _lib.ptr(cache), 2, 5, 2, 128, 12, 16, stream()))   # mha.py:367 assert
    lg = (torch.randn(50, 512) * 3).bfloat16()
    tg = torch.randint(0, 512, (50,)); tg[3] = -1
    lgd, tgd = lg.to(DEV), tg.to(DEV)
    od = torch.empty(50, dtype=torch.float32, device=DEV)
    _lib.check(lib.evo_logprobs(_lib.ptr(lgd), _lib.ptr(tgd), _lib.ptr(od), 50, 512, stream()))
    ref = torch.log_softmax(lg.float(), -1).gather(1, tg.clamp(min=0)[:, None])[:, 0]
    ref[3] = 0
    assert maxerr(od, ref) < 1e-5


# ------------------------------------------------------------------ fused Hyena operator
def _filter(D, H, seed=1):
    cfg = O.tiny_config(num_layers=1, attn_layer_idxs=(), hidden_size=D, num_heads=H)
    sd = O.random_state_dict(cfg, seed=seed)
    p = "blocks.0.filter."
    f = {"w": sd[p + "short_filter_weight"].to(DEV), "b": sd[p + "short_filter_bias"].to(DEV), "D": sd[p + "D"].to(DEV),
         "p": sd[p + "poles"].to(DEV), "r": sd[p + "residues"].to(DEV)}
    return cfg, sd, f


@pytest.mark.parametrize("B,L,nseg", [(1, 1, 1), (2, 2, 1), (2, 7, 1), (3, 130, 1), (3, 130, 4), (2, 1025, 1), (2, 1025, 3), (1, 4099, 5)])
def test_hyena_operator_vs_oracle(B, L, nseg):
    D, H = 256, 2
    cfg, sd, f = _filter(D, H)
    ob, ot = O.OracleStripedHyena(cfg, sd, torch.bfloat16), O.OracleStripedHyena(cfg, sd, torch.float64)
    torch.manual_seed(L)
    z = torch.randn(B, L, 3 * D).bfloat16()
    ipb, ipt = ob.initialize_inference_params()["hyena"], ot.initialize_inference_params()["hyena"]
    yb, yt = ob.hyena_operator(0, z, ipb), ot.hyena_operator(0, z.double(), ipt)
    y, st, fs = G._hyena_call(z.to(DEV), f, B, L, D, H, force=nseg)
    # FIR + gating rounding points are reproduced; only the fp32 scan vs fp32 FFT summation differs
    assert (y.cpu() == yb).float().mean() > 0.995
    assert maxerr(y, yb) <= 2 * BF16_EPS * max(1.0, yb.abs().max().item())
    assert meanerr(y, yt) <= 1.25 * meanerr(yb, yt) + 1e-6
    ref_fs = ipb.fir_state_dict[0]          # the reference keeps u[..., -2:], i.e. only L columns when L < 2; we zero-fill the history
    assert torch.equal(fs.cpu()[..., -ref_fs.shape[-1]:], ref_fs)                       # bit exact
    if L < 2:
        assert fs.cpu()[..., 0].abs().sum() == 0
    stc = torch.view_as_complex(st.cpu())
    # oracle truth state is computed from unrounded x1v; tolerance = bf16 noise of the inputs accumulated over the filter memory
    assert (stc - ipt.state_dict[0].to(torch.complex64)).abs().max() <= 1e-2 * max(1.0, ipt.state_dict[0].abs().max().item())
    stb = ipb.state_dict[0]
    assert (stc - stb).abs().max() <= 2e-4 * max(1.0, stb.abs().max().item())        # same bf16 inputs: fp32-level agreement


def test_hyena_continuation_and_sequence_sharding_are_exact():
    D, H, B, L = 256, 2, 2, 600
    _, _, f = _filter(D, H)
    torch.manual_seed(0)
    z = torch.randn(B, L, 3 * D).bfloat16().to(DEV)
    y_full, st_full, fs_full = G._hyena_call(z, f, B, L, D, H, force=1)
    a, b = z[:, :250].contiguous(), z[:, 250:].contiguous()
    ya, sta, _ = G._hyena_call(a, f, B, 250, D, H, force=1)
    halo = a[:, -2:].contiguous()
    yb, stb, fsb = G._hyena_call(b, f, B, 350, D, H, force=2, halo=halo, state_in=sta)
    assert maxerr(torch.cat([ya, yb], 1), y_full) <= 2 * BF16_EPS * y_full.abs().max().item()
    assert (torch.cat([ya, yb], 1) == y_full).float().mean() > 0.9995
    assert maxerr(stb, st_full) <= 1e-4 and torch.equal(fsb, fs_full)
    # rank-sharded form: zero-start end states -> combine -> output scan (evo_b200/parallel.py)
    lib = _lib.lib()
    h1 = z[:, 298:300].contiguous()
    z0, z1 = z[:, :300].contiguous(), z[:, 300:].contiguous()
    _, e0, _ = G._hyena_call(z0, f, B, 300, D, H, state_only=True)
    _, e1, _ = G._hyena_call(z1, f, B, 300, D, H, state_only=True, halo=h1)
    ends = torch.stack([e0, e1]).contiguous()
    sin1 = torch.empty_like(e0)
    _lib.check(lib.evo_hyena_combine_states(_lib.ptr(ends), _lib.ptr(sin1), _lib.ptr(f["p"]), 1, 2, 300, B, D, 8, stream()))
    y1, st1, _ = G._hyena_call(z1, f, B, 300, D, H, halo=h1, state_in=sin1)
    assert (y1 == y_full[:, 300:]).float().mean() > 0.9995
    assert maxerr(st1, st_full) <= 1e-4


def test_hyena_step_bit_exact():
    D, H, B = 256, 2, 3
    cfg, sd, f = _filter(D, H)
    ob = O.OracleStripedHyena(cfg, sd, torch.bfloat16)
    torch.manual_seed(3)
    z = torch.randn(B, 45, 3 * D).bfloat16()
    ip = ob.initialize_inference_params()["hyena"]
    ob.hyena_operator(0, z[:, :40], ip)
    fs = ip.fir_state_dict[0].clone().to(DEV).contiguous()
    st = torch.view_as_real(ip.state_dict[0].clone()).contiguous().to(DEV)
    for t in range(40, 45):
        yref = ob.hyena_operator(0, z[:, t:t + 1], ip)[:, 0]
        u = z[:, t].contiguous().to(DEV)
        yd = torch.empty(B, D, dtype=torch.bfloat16, device=DEV)
        _lib.check(_lib.lib().evo_hyena_step(_lib.ptr(u), _lib.ptr(yd), _lib.ptr(fs), _lib.ptr(st), _lib.ptr(f["w"]), _lib.ptr(f["b"]), _lib.ptr(f["D"]),
                                             _lib.ptr(f["p"]), _lib.ptr(f["r"]), B, D, 8, H, stream()))
        assert (yd.cpu() == yref).float().mean() > 0.998 and maxerr(yd, yref) <= 2 * BF16_EPS * max(1.0, yref.abs().max().item())
        assert torch.equal(fs.cpu(), ip.fir_state_dict[0])
        assert maxerr(st, torch.view_as_real(ip.state_dict[0])) <= 1e-4


def test_hyena_full_size_properties():
    """BASELINE configs[1] shape (B=8, L=8193, D=4096): segment-count invariance and
    state-pass == output-pass end state (size-independent properties, no oracle needed)."""
    D, H, B, L = 4096, 32, 8, 8193
    _, _, f = _filter(D, H)
    torch.manual_seed(0)
    z = torch.randn(B, L, 3 * D, device=DEV).bfloat16()
    y1, s1, _ = G._hyena_call(z, f, B, L, D, H, force=1)
    y4, s4, _ = G._hyena_call(z, f, B, L, D, H, force=4)
    assert (y1 == y4).float().mean().item() > 0.999
    assert maxerr(y1, y4) <= 2 * BF16_EPS * y1.abs().max().item()
    assert maxerr(s1, s4) <= 1e-3 * max(1.0, s1.abs().max().item())
    _, s_only, _ = G._hyena_call(z, f, B, L, D, H, state_only=True)
    assert maxerr(s_only, s1) <= 1e-3 * max(1.0, s1.abs().max().item())
    assert torch.isfinite(y1.float()).all()


# ------------------------------------------------------------------ tensor-core linear layers
@pytest.mark.parametrize("variant", [1, 0, 2])
@pytest.mark.parametrize("M,N,K", [(1, 256, 64), (16, 12288, 4096), (20, 768, 256), (40, 512, 4096), (128, 256, 64), (300, 512, 256), (1000, 768, 256), (4096, 4096, 4096), (8200, 512, 1024)])
def test_gemm_all_epilogues(variant, M, N, K):
    if variant == 2 and M > 1000:
        pytest.skip("variant 2 is the small-M weight-streaming tile")
    torch.manual_seed(M + N)
    a = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
    bias = (torch.randn(N, device=DEV) * 0.2).bfloat16()
    resid = torch.randn(M, N, device=DEV).bfloat16()
    acc = a.double() @ w.double().T                     # exact products of bf16 inputs, fp64 sum

    def close(out, ref):   # fp32 accumulation order differs: allow one bf16 ulp of the result
        assert not torch.isnan(out.float()).any()
        assert maxerr(out, ref) <= BF16_EPS * max(1.0, ref.abs().max().item())
        # fp32 vs fp64 accumulation: a long K moves more sums across a bf16 rounding boundary
        assert (out == ref.to(out.dtype)).float().mean() > (0.98 if K <= 1024 else 0.90)

    close(G._gemm(a, w, M, N, K, _lib.EPI_NONE, variant), acc.bfloat16())
    close(G._gemm(a, w, M, N, K, _lib.EPI_BIAS, variant, bias=bias), (acc + bias.double()).bfloat16())
    close(G._gemm(a, w, M, N, K, _lib.EPI_BIAS_RESID, variant, bias=bias, resid=resid),
          ((acc + bias.double()).bfloat16().double() + resid.double()).bfloat16())
    close(G._gemm(a, w, M, N, K, _lib.EPI_RESID, variant, resid=resid), (acc.bfloat16().double() + resid.double()).bfloat16())
    wv = w.view(N // 256, 2, 128, K)
    z1 = (a.double() @ wv[:, 0].reshape(-1, K).double().T).bfloat16()
    z2 = (a.double() @ wv[:, 1].reshape(-1, K).double().T).bfloat16()
    ref = (torch.nn.functional.gelu(z1.float()).bfloat16().float() * z2.float()).bfloat16()
    if variant == 2:      # no fused gate on the small-M tile: plain GEMM + evo_gelu_gate_interleaved (decode path)
        with pytest.raises(_lib.EvoError):
            G._gemm(a, w, M, N, K, _lib.EPI_GELU_GATE, variant, ldc=N // 2)
        t = G._gemm(a, w, M, N, K, _lib.EPI_NONE, variant)
        out = torch.empty(M, N // 2, dtype=torch.bfloat16, device=DEV)
        _lib.check(_lib.lib().evo_gelu_gate_interleaved(_lib.ptr(t), _lib.ptr(out), M, N // 2, stream()))
    else:
        out = G._gemm(a, w, M, N, K, _lib.EPI_GELU_GATE, variant, ldc=N // 2)
    assert maxerr(out, ref) <= 2 * BF16_EPS * max(1.0, ref.abs().max().item())
    assert (out == ref).float().mean() > (0.97 if K <= 1024 else 0.88)


def test_gemm_tile_walks_are_bit_identical(monkeypatch):
    """Tile walks of the persistent GEMM: the default (chosen per shape), grouped along M, grouped along N, and small groups.
    Only the order in which tiles are visited changes: every epilogue must give the same bits in every walk, on shapes with a
    ragged last row-block and more tiles than CTAs."""
    torch.manual_seed(5)
    for M, N, K in [(8200, 1024, 256), (16500, 512, 128), (9000, 2560, 64)]:
        a = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
        w = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
        bias = (torch.randn(N, device=DEV) * 0.2).bfloat16()
        resid = torch.randn(M, N, device=DEV).bfloat16()
        outs = {}
        for raster, group in ((None, None), ("0", None), ("1", None), ("0", "3"), ("1", "2")):
            for name, val in (("EVO_B200_GEMM_RASTER_N", raster), ("EVO_B200_GEMM_GROUP", group)):
                if val is None:
                    monkeypatch.delenv(name, raising=False)
                else:
                    monkeypatch.setenv(name, val)
            outs[(raster, group)] = [G._gemm(a, w, M, N, K, _lib.EPI_NONE, 0), G._gemm(a, w, M, N, K, _lib.EPI_BIAS_RESID, 0, bias=bias, resid=resid),
                                     G._gemm(a, w, M, N, K, _lib.EPI_GELU_GATE, 0, ldc=N // 2)]
        base = outs[(None, None)]
        assert not any(torch.isnan(x.float()).any() for x in base)
        for key, got in outs.items():
            for x, y in zip(base, got):
                assert torch.equal(x, y), key
    monkeypatch.delenv("EVO_B200_GEMM_RASTER_N", raising=False)
    monkeypatch.delenv("EVO_B200_GEMM_GROUP", raising=False)


def test_gemm_tile_major_weights_variant3():
    """variant 3 = variant 2 reading W tile-major; must give exactly the same bits as variant 2."""
    torch.manual_seed(0)
    for (M, N, K) in ((16, 12288, 4096), (5, 512, 256), (16, 4096, 11008)):
        a = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
        w = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
        bias = torch.randn(N, device=DEV).bfloat16()
        wt = StripedHyena._tile64(w)
        ref = G._gemm(a, w, M, N, K, _lib.EPI_BIAS, 2, bias=bias)
        out = G._gemm(a, wt, M, N, K, _lib.EPI_BIAS, 3, bias=bias)
        assert torch.equal(out, ref)


def _gemm_smallm(a, w, M, N, K, epi, bias=None, resid=None, ws=None):
    lib = _lib.lib()
    n_out = N // 2 if epi == _lib.EPI_GELU_GATE else N
    out = torch.full((M, n_out), float("nan"), dtype=torch.bfloat16, device=DEV)
    if ws is None:
        ws = torch.zeros(lib.evo_gemm_smallm_workspace(M, N, K, epi), dtype=torch.uint8, device=DEV)
    p = _lib.GemmSmallMParams(A=a.data_ptr(), lda=K, W=w.data_ptr(), C=out.data_ptr(), ldc=n_out,
                              bias=bias.data_ptr() if bias is not None else None, residual=resid.data_ptr() if resid is not None else None, ldr=n_out,
                              M=M, N=N, K=K, epilogue=epi, workspace=ws.data_ptr(), workspace_bytes=ws.numel())
    _lib.check(lib.evo_gemm_smallm(C.byref(p), stream()), "evo_gemm_smallm")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("M", [1, 16, 17, 40, 64])
@pytest.mark.parametrize("N,K", [(256, 64), (512, 4096), (768, 256), (4096, 4096), (12288, 4096), (22016, 4096), (4096, 11008)])
def test_gemm_smallm_streamk_all_epilogues(M, N, K):
    """Decode-step weight-streaming kernel (swap-AB tiles, stream-K + ordered fix-up): every epilogue against an fp64-accumulated
    reference, the workspace counters return to zero, and repeated launches give identical bits (deterministic reduction)."""
    if M not in (16, 17) and N * K > 4096 * 4096:
        pytest.skip("large shapes are covered at M = 16 / 17")
    torch.manual_seed(M + N + K)
    a = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
    bias = (torch.randn(N, device=DEV) * 0.2).bfloat16()
    resid = torch.randn(M, N, device=DEV).bfloat16()
    acc = a.double() @ w.double().T
    lib = _lib.lib()
    ws = torch.zeros(max(lib.evo_gemm_smallm_workspace(M, N, K, e) for e in range(5)), dtype=torch.uint8, device=DEV)

    def close(out, ref, mult=1.0, eq=None):
        assert not torch.isnan(out.float()).any()
        assert maxerr(out, ref) <= mult * BF16_EPS * max(1.0, ref.abs().max().item())
        assert (out == ref.to(out.dtype)).float().mean() > (eq or (0.98 if K <= 1024 else 0.90))

    close(_gemm_smallm(a, w, M, N, K, _lib.EPI_NONE, ws=ws), acc.bfloat16())
    o1 = _gemm_smallm(a, w, M, N, K, _lib.EPI_BIAS, bias=bias, ws=ws)
    close(o1, (acc + bias.double()).bfloat16())
    close(_gemm_smallm(a, w, M, N, K, _lib.EPI_BIAS_RESID, bias=bias, resid=resid, ws=ws), ((acc + bias.double()).bfloat16().double() + resid.double()).bfloat16())
    close(_gemm_smallm(a, w, M, N, K, _lib.EPI_RESID, resid=resid, ws=ws), (acc.bfloat16().double() + resid.double()).bfloat16())
    wv = w.view(N // 256, 2, 128, K)
    z1 = (a.double() @ wv[:, 0].reshape(-1, K).double().T).bfloat16()
    z2 = (a.double() @ wv[:, 1].reshape(-1, K).double().T).bfloat16()
    ref = (torch.nn.functional.gelu(z1.float()).bfloat16().float() * z2.float()).bfloat16()
    close(_gemm_smallm(a, w, M, N, K, _lib.EPI_GELU_GATE, ws=ws), ref, mult=2.0, eq=0.97 if K <= 1024 else 0.88)
    assert int(ws[:16384].view(torch.int32).abs().sum().item()) == 0          # tile counters reset themselves
    for _ in range(3):
        assert torch.equal(_gemm_smallm(a, w, M, N, K, _lib.EPI_BIAS, bias=bias, ws=ws), o1)
    # same rounding points as the throughput tiles: results agree to an accumulation-order ulp
    big = G._gemm(a, w, M, N, K, _lib.EPI_BIAS, 1, bias=bias)
    assert (big == o1).float().mean() > 0.97


def test_gemm_smallm_rejects_bad_arguments():
    a = torch.zeros(65, 64, dtype=torch.bfloat16, device=DEV)
    w = torch.zeros(256, 64, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(_lib.EvoError, match="must be in"):
        _gemm_smallm(a, w, 65, 256, 64, _lib.EPI_NONE)
    with pytest.raises(_lib.EvoError, match="workspace too small"):
        _gemm_smallm(a, w, 16, 256, 64, _lib.EPI_NONE, ws=torch.zeros(64, dtype=torch.uint8, device=DEV))
    with pytest.raises(_lib.EvoError, match="multiple of 256"):
        _gemm_smallm(a, torch.zeros(128, 64, dtype=torch.bfloat16, device=DEV), 16, 128, 64, _lib.EPI_NONE)


def test_gemm_rejects_bad_shapes():
    a = torch.zeros(8, 64, dtype=torch.bfloat16, device=DEV)
    w = torch.zeros(100, 64, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(_lib.EvoError, match="multiple of 256"):
        G._gemm(a, w, 8, 100, 64, _lib.EPI_NONE, 1)


def test_gemm_full_size_against_cublaslt():
    """BASELINE-size projection GEMM (65544 x 12288 x 4096): wgmma kernel vs the cuBLASLt comparator."""
    M, N, K = 65544, 12288, 4096
    torch.manual_seed(0)
    a = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=DEV) / 64).bfloat16()
    bias = torch.randn(N, device=DEV).bfloat16()
    out = G._gemm(a, w, M, N, K, _lib.EPI_BIAS, 1, bias=bias)
    ref = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ws = torch.empty(64 << 20, dtype=torch.uint8, device=DEV)
    p = _lib.GemmParams(A=a.data_ptr(), lda=K, W=w.data_ptr(), C=ref.data_ptr(), ldc=N, bias=bias.data_ptr(), residual=None, ldr=N, M=M, N=N, K=K, epilogue=1, variant=0)
    from tests import support as TS
    TS.check(TS.lib().evot_gemm_cublaslt(C.byref(p), _lib.ptr(ws), ws.numel(), stream()), "cublaslt comparator")
    torch.cuda.synchronize()
    d = (out.float() - ref.float()).abs()
    assert d.max().item() <= 2 * BF16_EPS * ref.float().abs().max().item()
    assert (out == ref).float().mean().item() > 0.98
    assert (out[-8:] == ref[-8:]).float().mean().item() > 0.98     # the ragged last row-block (65544 = 512*128 + 8)


# ------------------------------------------------------------------ attention
@pytest.mark.parametrize("variant", [1, 0, 2, 3])
@pytest.mark.parametrize("B,L", [(1, 1), (2, 37), (1, 128), (2, 129), (1, 256), (1, 300), (2, 1000), (1, 2500)])
def test_attention_vs_oracle(variant, B, L):
    H = 2
    torch.manual_seed(L)
    qkv = torch.randn(B, L, 3, H, 128).bfloat16()
    ref = O.causal_attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]).reshape(B, L, H * 128)
    truth = O.causal_attention(qkv[:, :, 0].double(), qkv[:, :, 1].double(), qkv[:, :, 2].double()).reshape(B, L, H * 128)
    out = G._attn(qkv.to(DEV), B, L, H, variant)
    assert not torch.isnan(out.float()).any()
    assert maxerr(out, ref) <= 4 * BF16_EPS * max(1.0, ref.abs().max().item())
    assert meanerr(out, truth) <= 1.25 * meanerr(ref, truth) + 1e-5
    simple = G._attn(qkv.to(DEV), B, L, H, variant, simple=True)
    assert maxerr(simple, ref) <= 4 * BF16_EPS * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("variant", [1, 0, 2, 3])
def test_attention_kv_cache_form(variant):
    B, H, Lc = 2, 2, 512
    torch.manual_seed(5)
    full = torch.randn(B, 260, 3, H, 128).bfloat16()
    cache = torch.zeros(B, Lc, 2, H, 128, dtype=torch.bfloat16)
    cache[:, :260, 0] = full[:, :, 1]
    cache[:, :260, 1] = full[:, :, 2]
    ref = O.causal_attention(full[:, :, 0], full[:, :, 1], full[:, :, 2]).reshape(B, 260, H * 128)
    cd = cache.to(DEV)
    for off, Lq in ((0, 260), (200, 1), (200, 5), (255, 5), (127, 2)):
        q = full[:, off:off + Lq].contiguous().to(DEV)
        o = G._attn(q, B, Lq, H, variant, cache=cd, off=off)
        assert maxerr(o, ref[:, off:off + Lq]) <= 4 * BF16_EPS * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("Lc", [640, 600])
def test_decode_attention_with_device_position_advanced_by_counters(Lc):
    """evo_decode_qkv_prep + evo_decode_attn (position read from device memory) vs the oracle.  Lc = 640 takes the TMA-fed
    kernel (64-key tiles), Lc = 600 the per-thread-row kernel.  Cache rows past the position hold NaN (the reference
    allocates its cache with torch.empty, mha.py:349): they must not leak into the result."""
    B, H = 3, 2
    lib = _lib.lib()
    torch.manual_seed(9)
    full = torch.randn(B, 600, 3, H, 128).bfloat16()
    cos, sin = O.rotary_tables(Lc, 128, dtype=torch.bfloat16)
    q = O.apply_rotary(full[:, :, 0], cos[:600], sin[:600])
    k = O.apply_rotary(full[:, :, 1], cos[:600], sin[:600])
    ref = O.causal_attention(q, k, full[:, :, 2]).reshape(B, 600, H * 128)
    cosd, sind = cos.to(DEV), sin.to(DEV)
    for pos in (0, 1, 63, 64, 127, 130, 599):
        cache = torch.full((B + 1, Lc, 2, H, 128), float("nan"), dtype=torch.bfloat16)
        cache[:B, :pos, 0] = k[:, :pos]
        cache[:B, :pos, 1] = full[:, :pos, 2]
        cd = cache.to(DEV)
        qkv = full[:, pos].contiguous().to(DEV)                       # (B, 3, H, 128), un-rotated
        posd = torch.tensor([pos], dtype=torch.int64, device=DEV)
        _lib.check(lib.evo_decode_qkv_prep(_lib.ptr(qkv), _lib.ptr(cd), _lib.ptr(cosd), _lib.ptr(sind), _lib.ptr(posd), B, H, 128, Lc, stream()))
        assert (cd[:B, pos, 0].cpu() == k[:, pos]).float().mean() > 0.995 and torch.equal(cd[:B, pos, 1].cpu(), full[:, pos, 2])
        for nsplit in (1, 3, 4):
            n = lib.evo_decode_attn_workspace(B, H, nsplit)
            ws = torch.empty(n, dtype=torch.uint8, device=DEV)
            out = torch.empty(B, H * 128, dtype=torch.bfloat16, device=DEV)
            _lib.check(lib.evo_decode_attn(_lib.ptr(qkv), _lib.ptr(cd), _lib.ptr(out), _lib.ptr(posd), B, H, 128, Lc, nsplit,
                                           1 / math.sqrt(128), _lib.ptr(ws), n, stream()))
            assert not torch.isnan(out.float()).any()
            assert maxerr(out, ref[:, pos]) <= 4 * BF16_EPS * max(1.0, ref.abs().max().item())
    _lib.check(lib.evo_advance_counters(_lib.ptr(posd), None, 3, stream()))
    assert posd.item() == 602


def test_attention_full_length_8193_vs_cuda_core_comparator():
    """L = 8193 (8192 nt + BOS), 32 heads: wgmma kernel vs the independent CUDA-core kernel."""
    B, L, H = 1, 8193, 32
    torch.manual_seed(0)
    qkv = torch.randn(B, L, 3, H, 128, device=DEV).bfloat16()
    a = G._attn(qkv, B, L, H, 1)
    b = G._attn(qkv, B, L, H, 1, simple=True)
    assert not torch.isnan(a.float()).any()
    assert maxerr(a, b) <= 4 * BF16_EPS * max(1.0, b.float().abs().max().item())
    assert meanerr(a, b) < 2e-4


# ------------------------------------------------------------------ whole model
def _tiny(layers=4, attn=(1, 3), seed=7, **extra):
    cfg = O.tiny_config(num_layers=layers, attn_layer_idxs=attn, hidden_size=256, num_heads=2, **extra)
    sd = O.random_state_dict(cfg, seed=seed)
    m = StripedHyena(dotdict(cfg))
    m.load_state_dict(sd, strict=True)
    m.to_bfloat16_except_poles_residues()
    return cfg, sd, m.to(DEV)


def _lsm(x):
    return torch.log_softmax(x.double().cpu(), -1)


@pytest.mark.parametrize("extra", [{}, {"use_interpolated_rotary_pos_emb": True, "rotary_emb_scaling_factor": 16}])
@pytest.mark.parametrize("ids_dtype", [torch.int64, torch.int32])
def test_model_logits_vs_oracle(extra, ids_dtype):
    cfg, sd, m = _tiny(**extra)
    ob, ot = O.OracleStripedHyena(cfg, sd, torch.bfloat16), O.OracleStripedHyena(cfg, sd, torch.float64)
    torch.manual_seed(0)
    ids = torch.randint(0, 4, (2, 333)) * 3 + 65
    ids[:, 0] = 0
    lg, st = m(ids.to(ids_dtype).to(DEV))
    assert st is None and lg.shape == (2, 333, 512) and lg.dtype == torch.bfloat16
    lb, _ = ob(ids)
    lt, _ = ot(ids)
    e_gpu, e_ref = (_lsm(lg) - _lsm(lt)).abs().mean().item(), (_lsm(lb) - _lsm(lt)).abs().mean().item()
    # stated tolerance: GPU log-probs are as close to exact arithmetic as the reference's bf16 pipeline (+25 %)
    assert e_gpu <= 1.25 * e_ref + 2e-3, (e_gpu, e_ref)
    # argmax agreement with exact arithmetic: as good as the reference's own bf16 pipeline (the bf16 oracle) within 3 points
    agree_gpu = (lg.cpu().argmax(-1) == lt.argmax(-1)).float().mean().item()
    agree_ref = (lb.argmax(-1) == lt.argmax(-1)).float().mean().item()
    assert agree_gpu >= agree_ref - 0.03 and agree_gpu > 0.93, (agree_gpu, agree_ref)
    assert maxerr(lg, lb) <= 0.05 * lb.float().abs().max().item()


def test_model_matches_committed_golden_fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "tiny_model_oracle.npz"))
    cfg, sd, m = _tiny(layers=3, attn=(1,), seed=7)
    ids = torch.from_numpy(g["ids"])
    lg, _ = m(ids.to(DEV))
    lt = torch.from_numpy(g["logits"])
    assert (_lsm(lg) - _lsm(lt)).abs().mean().item() < 6e-2
    assert (lg.cpu().argmax(-1) == lt.argmax(-1)).float().mean() > 0.93
    d = m.initialize_inference_params()
    d["mha"].max_batch_size, d["mha"].max_seqlen = 2, 128
    m(ids[:, :40].to(DEV), inference_params_dict=d)
    st = d["hyena"].state_dict[0].cpu()
    assert st.dtype == torch.complex64 and tuple(st.shape) == (2, 256, 8)
    assert (st.real - torch.from_numpy(g["state0_re"])).abs().max() < 2e-2 * max(1.0, float(np.abs(g["state0_re"]).max()))
    assert maxerr(d["hyena"].fir_state_dict[0].float(), torch.from_numpy(g["fir0"])) < 0.05


def test_stateful_prefill_then_steps_equals_stateless():
    cfg, sd, m = _tiny()
    torch.manual_seed(1)
    ids = (torch.randint(0, 4, (2, 200)) * 3 + 65).to(DEV)
    full, _ = m(ids)
    d = m.initialize_inference_params()
    d["mha"].max_batch_size, d["mha"].max_seqlen = 2, 256
    pre, d = m(ids[:, :150], inference_params_dict=d)
    assert torch.equal(pre, full[:, :150])                     # same kernels, same order: identical
    assert set(d["hyena"].fir_state_dict) == {0, 2} and set(d["mha"].key_value_memory_dict) == {1, 3}
    d["mha"].seqlen_offset = d["hyena"].seqlen_offset = 150
    scale = full.float().abs().max().item()
    for t in range(150, 200):
        s, d = m(ids[:, t:t + 1], inference_params_dict=d)
        assert maxerr(s[:, 0], full[:, t]) <= 0.03 * scale
        d["mha"].seqlen_offset += 1
        d["hyena"].seqlen_offset += 1


def test_load_state_dict_rebuilds_rotary_tables_from_the_new_inv_freq():
    """A checkpoint loaded after a forward carries its own fp32 rotary inv_freq: the rotary tables the earlier forward built
    from the old buffer are dropped, so the logits are those of a model built from that checkpoint."""
    cfg, sd, m = _tiny()
    torch.manual_seed(2)
    ids = (torch.randint(0, 4, (2, 200)) * 3 + 65).to(DEV)
    before, _ = m(ids)
    sd2 = {k: (v * 0.5 if k.endswith("rotary_emb.inv_freq") else v) for k, v in sd.items()}
    assert sum(k.endswith("rotary_emb.inv_freq") for k in sd2) == len(cfg["attn_layer_idxs"])
    m.load_state_dict(sd2, strict=True)
    fresh = StripedHyena(dotdict(cfg))
    fresh.load_state_dict(sd2, strict=True)
    fresh = fresh.to_bfloat16_except_poles_residues().to(DEV)
    got, _ = m(ids)
    want, _ = fresh(ids)
    assert not torch.equal(want, before)
    assert torch.equal(got, want)


def test_decode_streamk_pdl_paths_agree():
    """Decode step through (a) the 128x64 tiles without programmatic dependent launch, (b) the stream-K kernel without it,
    (c) stream-K + PDL (levels 1 and 2) inside the CUDA graph: same logits up to accumulation order, (c) repeatable bit for bit."""
    cfg, sd, m = _tiny()
    torch.manual_seed(2)
    ids = (torch.randint(0, 4, (3, 90)) * 3 + 65).to(DEV)

    def run(streamk, pdl, graph):
        m.decode_streamk, m.decode_pdl, m.decode_graph, m._decode = streamk, pdl, graph, None
        d = m.initialize_inference_params()
        d["mha"].max_batch_size, d["mha"].max_seqlen = 3, 128
        _, d = m(ids[:, :60], inference_params_dict=d)
        d["mha"].seqlen_offset = d["hyena"].seqlen_offset = 60
        outs = []
        for t in range(60, 90):
            s, d = m(ids[:, t:t + 1], inference_params_dict=d)
            outs.append(s[:, 0].clone())
            d["mha"].seqlen_offset += 1
            d["hyena"].seqlen_offset += 1
        return torch.stack(outs, 1)

    try:
        saved = (m.decode_streamk, m.decode_pdl, m.decode_graph)
        a = run(False, 0, False)
        b = run(True, 0, False)
        c = run(True, 1, True)
        c2 = run(True, 1, True)
        e = run(True, 2, True)
        f3 = run(True, 3, True)
        f4 = run(True, 4, True)
    finally:
        m.decode_streamk, m.decode_pdl, m.decode_graph = saved
        m._decode = None
    scale = a.float().abs().max().item()
    assert maxerr(b, a) <= 0.03 * scale and maxerr(c, a) <= 0.03 * scale
    assert torch.equal(c, c2)
    assert torch.equal(b, c) and torch.equal(b, e) and torch.equal(b, f3) and torch.equal(b, f4)        # PDL and graph replay change scheduling only


def test_public_api_scoring_and_generation():
    import evo_b200
    cfg, sd, m = _tiny(layers=3, attn=(1,))
    tok = evo_b200.CharLevelTokenizer(512)
    seqs = ["ACGTTGCAACGTACGTAGCTAGCTAGGATC", "ACGTAC", "TTTTGGGGCCCCAAAA"]
    got = evo_b200.score_sequences(seqs, m, tok, device=DEV)
    ot = O.OracleStripedHyena(cfg, sd, torch.float64)
    for s, g in zip(seqs, got):
        ids = torch.tensor([[0] + tok.tokenize(s)])
        lp = torch.log_softmax(ot(ids)[0], -1)[0, :-1].gather(1, ids[0, 1:, None])[:, 0]
        # per-position bf16 noise of this tiny random model is ~3.5e-2 nats (see test_model_logits_vs_oracle);
        # a mean over 6..30 positions stays within 8e-2
        assert abs(lp.mean().item() - float(g)) < 8e-2
    ent = evo_b200.positional_entropies(seqs, m, tok, device=DEV)
    assert [len(e) for e in ent] == [len(s) for s in seqs]
    out, scores = evo_b200.generate(["ACGTACGT", "TTGACCAA"], m, tok, n_tokens=12, top_k=1, cached_generation=True, verbose=0, device=DEV)
    out2, _ = evo_b200.generate(["ACGTACGT", "TTGACCAA"], m, tok, n_tokens=12, top_k=1, cached_generation=False, verbose=0, device=DEV)
    assert len(out) == 2 and all(len(o) == 12 for o in out) and len(scores) == 2
    agree = np.mean([a == b for x, y in zip(out, out2) for a, b in zip(x, y)])
    assert agree > 0.8       # cached (recurrent) vs uncached (full forward) greedy paths: near-ties may flip


def test_baseline_config0_two_layer_7b_width_L1024():
    """BASELINE.json configs[0]: random-init 2-layer StripedHyena (1 Hyena + 1 attn) at the 7B
    width (D=4096, 32 heads), batch 1 x 1024: GPU forward vs the CPU oracle."""
    cfg = O.evo_config("evo-1-8k-base")
    cfg.update(num_layers=2, attn_layer_idxs=[1], hyena_layer_idxs=[0])
    sd = O.random_state_dict(cfg, seed=3)
    m = StripedHyena(dotdict(cfg))
    m.load_state_dict(sd, strict=True)
    m.to_bfloat16_except_poles_residues()
    m = m.to(DEV)
    rng = np.random.default_rng(1)
    ids = torch.from_numpy(rng.choice(np.array([65, 67, 71, 84]), size=(1, 1024)))
    lg, _ = m(ids.to(DEV))
    lb, _ = O.OracleStripedHyena(cfg, sd, torch.bfloat16)(ids)
    lt, _ = O.OracleStripedHyena(cfg, sd, torch.float32)(ids)
    e_gpu, e_ref = (_lsm(lg) - _lsm(lt)).abs().mean().item(), (_lsm(lb) - _lsm(lt)).abs().mean().item()
    assert e_gpu <= 1.25 * e_ref + 2e-3, (e_gpu, e_ref)
    agree_gpu = (lg.cpu().argmax(-1) == lt.argmax(-1)).float().mean().item()
    agree_ref = (lb.argmax(-1) == lt.argmax(-1)).float().mean().item()
    assert agree_gpu >= agree_ref - 0.03 and agree_gpu > 0.93, (agree_gpu, agree_ref)


def test_full_depth_7b_logits_vs_oracle():
    """The 7B architecture at full depth (32 blocks: 29 Hyena + 3 attention, D=4096, evo-1-131k rotary scaling),
    batch 1 x 128 tokens: GPU logits vs the CPU oracle.  A random-weight 32-block net amplifies bf16 noise
    (the bf16-faithful CPU oracle itself is ~0.25 nats / 85 % argmax from its fp32 twin), hence the relative bars.  Blocks of a kind share one set of random weights
    (share_blocks) so the CPU side stays small; the arithmetic per block is the full-size one."""
    cfg = O.evo_config("evo-1-131k-base")
    sd = O.random_state_dict(cfg, seed=11, share_blocks=True)
    m = StripedHyena(dotdict(cfg))
    m.load_state_dict(sd, strict=True)
    m.to_bfloat16_except_poles_residues()
    m = m.to(DEV)
    rng = np.random.default_rng(5)
    ids = torch.from_numpy(rng.choice(np.array([65, 67, 71, 84]), size=(1, 128)))
    ids[0, 0] = 0
    lg, _ = m(ids.to(DEV))
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    lb, _ = O.OracleStripedHyena(cfg, sd, torch.bfloat16)(ids)
    lt, _ = O.OracleStripedHyena(cfg, sd, torch.float32)(ids)
    e_gpu, e_ref = (_lsm(lg) - _lsm(lt)).abs().mean().item(), (_lsm(lb) - _lsm(lt)).abs().mean().item()
    assert torch.isfinite(lg.float()).all()
    assert e_gpu <= 1.25 * e_ref + 5e-3, (e_gpu, e_ref)
    agree_gpu = (lg.cpu().argmax(-1) == lt.argmax(-1)).float().mean().item()
    agree_ref = (lb.argmax(-1) == lt.argmax(-1)).float().mean().item()
    assert agree_gpu >= agree_ref - 0.08, (agree_gpu, agree_ref)
