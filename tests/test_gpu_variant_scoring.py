"""Variant scoring: the checkpointed / resumed Hyena scan (evo_hyena_fwd_varlen_ckpt), attention behind a cached prefix
(evo_attn_fwd_varlen_prefix), the model's prefill_checkpoints / score_tokens_resumed, score_variants and its CLI.

Bars.  Unsegmented scans are held bit for bit: a checkpoint to the end state of the same scan over the first k * stride rows
alone, a resumed scan to the rows and end states of the whole-sequence scan.  Forced segmentations change the carry
arithmetic, so they are held to the fp64 and bf16-oracle bars tests/test_gpu_hyena_paths.py applies to the segmented scan.
Prefix attention with prefix_len % 128 == 0 sees exactly the key tiles of a batch-1 evo_attn_fwd_ws call with q_pos0 =
prefix_len, and with prefix_len == 0 those of evo_attn_fwd_varlen: both are held bit for bit; other prefix lengths and rows
whose softmax max moves from the prefix to their own keys are held to tests/test_gpu_attention_peaked.py's bars.
score_variants is held to score_many(packed=True) on the full variant strings within 2e-3 per mean score (DESIGN.md 3.4's
end-to-end bar): the two paths tile their GEMMs and scans differently, so their bits differ."""
import csv
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

from evo_b200 import _lib  # noqa: E402
from tests.test_gpu_hyena_paths import _assert_state, _assert_vs_oracle, _bf16_oracle, _filter_sd, _fp64_oracle  # noqa: E402
from tests.test_gpu_packed import DEV, _attn_varlen, _cu, _filter, _hyena_varlen, _ids, _same, stream, tiny, wide  # noqa: E402,F401
from tests.test_gpu_attention_peaked import check as peaked_check, reference as peaked_reference  # noqa: E402

SCORE_TOL = 2e-3


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()


# ------------------------------------------------------------------ Hyena: checkpoints and resumed starts
def _one_segment(n):
    """A forced seg_len that covers n rows in one segment: with checkpoints it must be a multiple of the 16-token stage."""
    return (n + 15) // 16 * 16


def _hyena_ckpt(z, f, H, lengths, seg_len=0, stride=0, start=None, tables=None):
    """evo_hyena_fwd_varlen_ckpt: (y, state_out, fir_state_out, checkpoint table, base)."""
    lib = _lib.lib()
    T, C3 = z.shape
    D, n = C3 // 3, len(lengths)
    cu = torch.tensor(_cu(lengths), dtype=torch.int64, device=DEV)
    y = torch.empty(T, D, dtype=torch.bfloat16, device=DEV)
    st = torch.empty(n, D, 8, 2, dtype=torch.float32, device=DEV)
    fs = torch.empty(n, C3, 2, dtype=torch.bfloat16, device=DEV)
    base = _lib.HyenaVarlenParams(z=z.data_ptr(), y=y.data_ptr(), fir_w=f["w"].data_ptr(), fir_b=f["b"].data_ptr(), Dskip=f["D"].data_ptr(),
                                  poles=f["p"].data_ptr(), residues=f["r"].data_ptr(), cu_seqlens=cu.data_ptr(), n_seq=n, T=T,
                                  max_seqlen=max(lengths), D=D, S=8, nheads=H, state_out=st.data_ptr(), fir_state_out=fs.data_ptr(), seg_len=seg_len)
    p = _lib.HyenaVarlenCkptParams(base=base)
    keep, ck, b0 = [], None, None
    if stride:
        counts = [(L - 1) // stride for L in lengths]
        b0 = [0] + np.cumsum(counts).tolist()
        ck = torch.full((max(b0[-1], 1), D, 8, 2), float("nan"), device=DEV)
        bd = torch.tensor(b0[:-1], dtype=torch.int64, device=DEV)
        keep.append(bd)
        p.ckpt_states, p.ckpt_base, p.ckpt_stride, p.n_ckpt = ck.data_ptr(), bd.data_ptr(), stride, max(b0[-1], 1)
    if start is not None:
        sd = torch.tensor(start, dtype=torch.int64, device=DEV)
        keep.append(sd)
        p.start_idx, p.state_table, p.halo_table, p.n_table = sd.data_ptr(), tables[0].data_ptr(), tables[1].data_ptr(), tables[0].shape[0]
    need = lib.evo_hyena_fwd_varlen_ckpt_workspace(C.byref(p))
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
    _lib.check(lib.evo_hyena_fwd_varlen_ckpt(C.byref(p), _lib.ptr(ws), need, stream()), "evo_hyena_fwd_varlen_ckpt")
    torch.cuda.synchronize()
    return y, st, fs, ck, b0


@pytest.mark.parametrize("D", [256, 4096])
def test_checkpoints_unsegmented_are_the_prefix_scans_end_states(D):
    H, s = D // 128, 128
    f = _filter(D)
    lengths = (1000, 129, 1, 700) if D == 256 else (1030, 300)
    g = torch.Generator().manual_seed(D + 1)
    z = torch.randn(sum(lengths), 3 * D, generator=g).bfloat16().to(DEV)
    y, st, fs, ck, b0 = _hyena_ckpt(z, f, H, lengths, seg_len=_one_segment(max(lengths)), stride=s)
    y0, st0, fs0, _ = _hyena_varlen(z, f, H, lengths, seg_len=max(lengths))
    assert _same(y, y0) and _same(st, st0) and _same(fs, fs0)                    # emission does not touch the recurrence
    cu = _cu(lengths)
    for b, L in enumerate(lengths):
        assert b0[b + 1] - b0[b] == (L - 1) // s
        for k in range(1, (L - 1) // s + 1):
            _, stk, _, _ = _hyena_varlen(z[cu[b]:cu[b] + k * s].contiguous(), f, H, [k * s], seg_len=k * s)
            assert _same(ck[b0[b] + k - 1], stk[0]), (D, L, k)


@pytest.mark.parametrize("seg_len", [64, 112, 400])
def test_checkpoints_segmented_vs_oracle(seg_len):
    D, H, s = 256, 2, 128
    sd, f = _filter_sd(D)
    lengths = (700, 260)
    g = torch.Generator().manual_seed(seg_len)
    z = torch.randn(sum(lengths), 3 * D, generator=g).bfloat16()
    _, _, _, ck, b0 = _hyena_ckpt(z.to(DEV), f, H, lengths, seg_len=seg_len, stride=s)
    cu = _cu(lengths)
    for b, L in enumerate(lengths):
        for k in range(1, (L - 1) // s + 1):
            zb = z[cu[b]:cu[b] + k * s].unsqueeze(0)
            _, stb = _bf16_oracle(sd, zb, H, want_state=True)
            stt = _fp64_oracle(sd, zb, H)[1]
            what = f"seg_len={seg_len} L={L} k={k}"
            row = b0[b] + k - 1
            _assert_state(ck[row:row + 1], stb, 2e-4, what + " vs bf16 oracle")
            _assert_state(ck[row:row + 1], stt, 1e-2, what + " vs fp64")


def _tables(z, ck, lengths, b0, s):
    """The FIR half of the checkpoints: z rows c - 2, c - 1 of every checkpoint, as the model gathers them."""
    cu = _cu(lengths)
    rows = [cu[b] + k * s + d for b, L in enumerate(lengths) for k in range(1, (L - 1) // s + 1) for d in (-2, -1)]
    return ck, z[torch.tensor(rows, device=DEV)].view(-1, 2, z.shape[1]).contiguous()


@pytest.mark.parametrize("D", [256, 4096])
def test_resumed_scan_continues_the_whole_sequence_bit_for_bit(D):
    H, s = D // 128, 128
    f = _filter(D)
    lengths = (1000, 600)
    g = torch.Generator().manual_seed(D + 2)
    z = torch.randn(sum(lengths), 3 * D, generator=g).bfloat16().to(DEV)
    y, st, fs, ck, b0 = _hyena_ckpt(z, f, H, lengths, seg_len=_one_segment(max(lengths)), stride=s)
    tables = _tables(z, ck, lengths, b0, s)
    cu = _cu(lengths)
    # sequence 0 resumed at c = 256 and c = 896, sequence 1 at c = 128, and sequence 1 from a zero start
    cases = [(0, 256), (0, 896), (1, 128), (1, 0)]
    parts, plen, start = [], [], []
    for b, c in cases:
        parts.append(z[cu[b] + c:cu[b + 1]])
        start.append(b0[b] + c // s - 1 if c else -1)
        plen.append(lengths[b] - c)
    zr = torch.cat(parts).contiguous()
    yr, str_, fsr, _, _ = _hyena_ckpt(zr, f, H, plen, seg_len=max(plen), start=start, tables=tables)
    rc = _cu(plen)
    for j, (b, c) in enumerate(cases):
        assert _same(yr[rc[j]:rc[j + 1]], y[cu[b] + c:cu[b + 1]]), (D, b, c)
        assert _same(str_[j], st[b]) and _same(fsr[j], fs[b]), (D, b, c)
    # a zero start gives evo_hyena_fwd_varlen's bits
    y0, st0, fs0, _ = _hyena_varlen(zr, f, H, plen, seg_len=max(plen))
    assert _same(yr[rc[3]:], y0[rc[3]:]) and _same(str_[3], st0[3])
    # a one-row resumed sequence takes its FIR end state from the checkpoint's history
    y1, st1, fs1, _, _ = _hyena_ckpt(z[cu[0] + 256:cu[0] + 257].contiguous(), f, H, [1], seg_len=1, start=[b0[0] + 1], tables=tables)
    assert _same(fs1[0][:, 0], tables[1][b0[0] + 1][1]) and _same(fs1[0][:, 1], z[cu[0] + 256])


@pytest.mark.parametrize("seg_len", [64, 100, 300])
def test_resumed_scan_segmented_vs_oracle(seg_len):
    D, H, s = 256, 2, 128
    sd, f = _filter_sd(D)
    L, c = 900, 384
    g = torch.Generator().manual_seed(seg_len + 7)
    z = torch.randn(L, 3 * D, generator=g).bfloat16()
    zd = z.to(DEV)
    _, _, _, ck, b0 = _hyena_ckpt(zd, f, H, [L], seg_len=_one_segment(L), stride=s)
    tables = _tables(zd, ck, [L], b0, s)
    yr, str_, _, _, _ = _hyena_ckpt(zd[c:].contiguous(), f, H, [L - c], seg_len=seg_len, start=[c // s - 1], tables=tables)
    yb, stb = _bf16_oracle(sd, z.unsqueeze(0), H, want_state=True)
    yt, stt = _fp64_oracle(sd, z.unsqueeze(0), H)
    what = f"resumed at {c}, seg_len={seg_len}"
    _assert_vs_oracle(yr.unsqueeze(0), yb[:, c:], yt[:, c:], what)
    _assert_state(str_, stb, 2e-4, what + " state vs bf16 oracle")
    _assert_state(str_, stt, 1e-2, what + " state vs fp64")


def test_checkpointed_scan_rejects_bad_arguments():
    lib = _lib.lib()
    D, H = 256, 2
    f = _filter(D)
    z = torch.randn(300, 3 * D).bfloat16().to(DEV)
    for kw in (dict(stride=100), dict(stride=128, seg_len=100)):
        lib.evo_reset_launch_count()
        with pytest.raises(_lib.EvoError, match="multiple of"):
            _hyena_ckpt(z, f, H, [300], **kw)
        assert lib.evo_launch_count() == 0


# ------------------------------------------------------------------ attention behind a cached prefix
def _prefix_attn(qkv, lengths, cache, pseq, plen):
    lib = _lib.lib()
    T = qkv.shape[0]
    H = qkv.shape[2]
    cu = torch.tensor(_cu(lengths), dtype=torch.int64, device=DEV)
    ps = torch.tensor(pseq, dtype=torch.int64, device=DEV)
    pl = torch.tensor(plen, dtype=torch.int64, device=DEV)
    out = torch.empty(T, H * 128, dtype=torch.bfloat16, device=DEV)
    ap = _lib.AttnVarlenPrefixParams(qkv=qkv.data_ptr(), out=out.data_ptr(), cu_seqlens=cu.data_ptr(), n_seq=len(lengths), T=T,
                                     max_seqlen=max(lengths), cache=cache.data_ptr(), n_cache=cache.shape[0], cache_len=cache.shape[1],
                                     prefix_seq=ps.data_ptr(), prefix_len=pl.data_ptr(), H=H, hd=128, softmax_scale=1.0 / math.sqrt(128))
    _lib.check(lib.evo_attn_fwd_varlen_prefix(C.byref(ap), stream()), "evo_attn_fwd_varlen_prefix")
    torch.cuda.synchronize()
    return out


def _ws_behind(q, kv, P, out):
    """batch-1 evo_attn_fwd_ws with q_pos0 = P: q (L, H, 128), kv (P + L, 2, H, 128) one cache."""
    lib = _lib.lib()
    L, H = q.shape[0], q.shape[1]
    d = H * 128
    ap = _lib.AttnParams(out=out.data_ptr(), B=1, Lq=L, Lk=P + L, H=H, hd=128, q_pos0=P, softmax_scale=1.0 / math.sqrt(128))
    ap.q, ap.q_tok_stride, ap.q_batch_stride = q.data_ptr(), d, L * d
    ap.k, ap.v, ap.kv_tok_stride, ap.kv_batch_stride = kv.data_ptr(), kv.data_ptr() + d * 2, 2 * d, (P + L) * 2 * d
    _lib.check(lib.evo_attn_fwd_ws(C.byref(ap), 2, None, 0, stream()), "evo_attn_fwd_ws")
    torch.cuda.synchronize()


def _attn_case(H, lengths, plen, n_cache=2, S=1200, seed=0):
    """Random packed qkv (T, 3, H, 128) and cache (n_cache, S, 2, H, 128); sequence b's prefix is cache row b % n_cache."""
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(sum(lengths), 3, H, 128, generator=g).bfloat16().to(DEV)
    cache = torch.randn(n_cache, S, 2, H, 128, generator=g).bfloat16().to(DEV)
    pseq = [b % n_cache for b in range(len(lengths))]
    return qkv, cache, pseq


@pytest.mark.parametrize("H", [2, 32])
def test_prefix_attention_aligned_is_the_batch1_call_bit_for_bit(H):
    lengths = (300, 1, 129, 128) if H == 2 else (257, 3)
    plen = (128, 256, 1024, 384) if H == 2 else (512, 128)
    qkv, cache, pseq = _attn_case(H, lengths, plen)
    out = _prefix_attn(qkv, lengths, cache, pseq, plen)
    cu = _cu(lengths)
    for b, (L, P) in enumerate(zip(lengths, plen)):
        own = qkv[cu[b]:cu[b + 1]]
        kv = torch.cat([cache[pseq[b], :P], own[:, 1:]]).contiguous()
        ref = torch.empty(L, H * 128, dtype=torch.bfloat16, device=DEV)
        _ws_behind(own[:, 0].contiguous(), kv, P, ref)
        assert _same(out[cu[b]:cu[b + 1]], ref), (H, L, P)


def test_prefix_attention_without_prefix_is_the_varlen_call():
    H, lengths = 2, (300, 1, 127, 1000)
    qkv, cache, pseq = _attn_case(H, lengths, None, seed=1)
    out = _prefix_attn(qkv, lengths, cache, pseq, [0] * len(lengths))
    assert _same(out, _attn_varlen(qkv.view(qkv.shape[0], -1), lengths, H))


@pytest.mark.parametrize("moving", [False, True])
def test_prefix_attention_unaligned_vs_fp64(moving):
    """Prefix lengths 1, 127, 129 and 1000 against fp64 softmax over [prefix | own rows]; moving=True makes every row's max
    jump from the prefix to its own first key by about 300 log2 units (well past the 2^8 lazy-rescale threshold)."""
    H, lengths, plen = 2, (200, 130, 1, 260), (1, 127, 129, 1000)
    qkv, cache, pseq = _attn_case(H, lengths, plen, seed=2)
    cu = _cu(lengths)
    if moving:
        u = torch.randn(H, 128, generator=torch.Generator().manual_seed(5))
        u = u / u.norm(dim=-1, keepdim=True)
        for b in range(len(lengths)):
            qkv[cu[b]:cu[b + 1], 0] = (48.0 * u).bfloat16().to(DEV)                      # every query along u
            qkv[cu[b], 1] = (48.0 * u).bfloat16().to(DEV)                                # own key 0: score ~ 2304 / sqrt(128)
            cache[pseq[b], :plen[b], 0] = (0.1 * torch.randn(plen[b], H, 128)).bfloat16().to(DEV)
    out = _prefix_attn(qkv, lengths, cache, pseq, plen)
    for b, (L, P) in enumerate(zip(lengths, plen)):
        own = qkv[cu[b]:cu[b + 1]].cpu()
        pre = cache[pseq[b], :P].cpu()
        k = torch.cat([pre[:, 0], own[:, 1]])
        v = torch.cat([pre[:, 1], own[:, 2]])
        ref = peaked_reference(own[:, 0], k, v, list(range(L)), pos0=P)
        if moving:
            top = ref["scores"].max(-1).values * 1.4426950408889634
            first = ref["scores"][..., :P].max(-1).values * 1.4426950408889634
            assert ((top - first) > 256).all()                                           # the case reaches the regime it claims
        peaked_check(out[cu[b]:cu[b + 1]].view(L, H, 128), ref, f"P={P} L={L} moving={moving}")


def test_prefix_attention_nothing_past_prefix_len_reaches_an_output():
    H, lengths, plen = 2, (200, 130, 1, 260), (1, 127, 129, 1000)
    qkv, cache, pseq = _attn_case(H, lengths, plen, n_cache=4, seed=3)
    out = _prefix_attn(qkv, lengths, cache, pseq, plen)
    poisoned = cache.clone()
    for b, P in enumerate(plen):
        poisoned[pseq[b], P:] = float("nan")                                      # K and V rows a query must not see
    out2 = _prefix_attn(qkv, lengths, poisoned, pseq, plen)
    assert not torch.isnan(out2.float()).any()
    assert _same(out, out2)


# ------------------------------------------------------------------ model and public surface
def _ref_and_variants(L, seed):
    rng = np.random.default_rng(seed)
    ref = "".join(rng.choice(list("ACGT"), size=L))

    def sub(i):
        return ref[:i] + ("A" if ref[i] != "A" else "C") + ref[i + 1:]
    var = [sub(i) for i in (0, 1, 126, 127, 128, 129, 255, 256, 500, L - 130, L - 1)]
    var += [ref[:300] + "G" + ref[300:], ref[:700] + ref[701:], ref, ref[:400], ref + "AC", ref[:129] + "TTT" + ref[600:]]
    return ref, var


@pytest.mark.parametrize("which", ["tiny", "wide"])
def test_score_variants_matches_full_scoring(which, tiny, wide):
    import evo_b200
    from evo_b200.frontend import score_many
    m = (tiny if which == "tiny" else wide)[2]
    tok = evo_b200.CharLevelTokenizer(512)
    ref, var = _ref_and_variants(1000, seed=3)
    stats = {}
    got, refs = evo_b200.score_variants(ref, var, m, tok, device=DEV, max_tokens=3000, stats=stats)
    want = score_many(var + [ref], m, tok, max_tokens=3000, device=DEV, packed=True)
    d = np.abs(np.array(got + refs) - np.array(want)).max()
    print(f"\n{which}: score_variants vs score_many(packed=True): worst |mean score difference| {d:.2e}; {stats}")
    assert d <= SCORE_TOL, d
    assert stats["checkpoint_stride"] == 128 and stats["variant_tokens"] < sum(len(v) + 1 for v in var)
    k_eq, k_pre = var.index(ref), var.index(ref[:400])
    assert got[k_eq] == refs[0]                                                   # an equal variant is the reference's score
    sums, rsum = evo_b200.score_variants(ref, var, m, tok, device=DEV, reduce_method="sum")
    assert np.allclose(np.array(sums) / np.array([len(v) for v in var]), got, atol=1e-6, rtol=0)
    assert abs(rsum[0] / len(ref) - refs[0]) < 1e-6 and got[k_pre] * 400 == pytest.approx(sums[k_pre], abs=1e-4)


def test_reference_rows_come_from_the_reference_pass(tiny):
    """A variant's score is the reference pass's logprobs over rows [0, c) (those bits) plus the resumed pass's rows."""
    import evo_b200
    from evo_b200.frontend import packed_ids
    from evo_b200.variants import first_difference, resume_point
    m = tiny[2]
    tok = evo_b200.CharLevelTokenizer(512)
    ref, var = _ref_and_variants(1000, seed=4)
    got, _ = evo_b200.score_variants(ref, var, m, tok, device=DEV, reduce_method="sum")
    ids = packed_ids([ref], tok, device=DEV)
    ck = m.prefill_checkpoints(ids, [0, len(ref) + 1], 128)
    lp = ck.logprobs.cpu().numpy()
    for k in (2, 8, 16):                                                          # resumed at 0, 256 + ... and 128
        f = first_difference(ref, var[k])
        c = resume_point(f, 128)
        vids = packed_ids([var[k]], tok, device=DEV)[c:]
        vlp = m.score_tokens_resumed(ck, vids, [0, vids.shape[0]], [c // 128 - 1 if c else -1], [0], [c]).cpu().numpy()
        total = np.cumsum(lp[:c], dtype=np.float64)[-1] if c else 0.0
        total += vlp[:-1].sum(dtype=np.float64)
        assert got[k] == float(total), k
        full = m.score_tokens_packed(packed_ids([var[k]], tok, device=DEV), [0, len(var[k]) + 1])[0].cpu().numpy()
        assert np.abs(full[c:-1] - vlp[:-1]).max() < 0.05, k                     # the same rows, computed from the checkpoint


def test_several_references_in_one_call_equal_separate_calls(tiny):
    import evo_b200
    m = tiny[2]
    tok = evo_b200.CharLevelTokenizer(512)
    (r0, v0), (r1, v1) = _ref_and_variants(1000, seed=5), _ref_and_variants(600, seed=6)
    mixed = [(1, v) for v in v1[:5]] + [(0, v) for v in v0] + [(1, v) for v in v1[5:]]
    got, refs = evo_b200.score_variants([r0, r1], mixed, m, tok, device=DEV, max_tokens=4000)
    a, ra = evo_b200.score_variants(r0, v0, m, tok, device=DEV, max_tokens=4000)
    b, rb = evo_b200.score_variants(r1, v1, m, tok, device=DEV, max_tokens=4000)
    want = b[:5] + a + b[5:]
    assert np.abs(np.array(got) - np.array(want)).max() <= 1e-5
    assert np.abs(np.array(refs) - np.array(ra + rb)).max() <= 1e-5


def test_cli_saturation_and_mutant_csv(tiny, tmp_path, monkeypatch):
    import evo_b200
    from scripts import score_variants as cli
    m = tiny[2]
    tok = evo_b200.CharLevelTokenizer(512)
    rng = np.random.default_rng(7)
    ref = "".join(rng.choice(list("ACGT"), size=150))
    fasta = tmp_path / "ref.fasta"
    fasta.write_text(f">wt\n{ref[:80]}\n{ref[80:]}\n")

    class TinyEvo:
        def __init__(self, *a, **kw):
            self.model, self.tokenizer = m, tok
    monkeypatch.setattr(cli, "Evo", TinyEvo)
    out = tmp_path / "sat.tsv"
    cli.main(["--reference-fasta", str(fasta), "--saturation", "--output-tsv", str(out), "--device", DEV])
    rows = [line.split("\t") for line in out.read_text().splitlines()]
    sat = evo_b200.saturation_variants(ref)
    want, wref = evo_b200.score_variants(ref, [s for _, s in sat], m, tok, device=DEV)
    assert rows[0] == ["variant", "score", "delta"] and len(rows) == 1 + 3 * len(ref)
    assert [r[0] for r in rows[1:]] == [mu for mu, _ in sat]
    assert np.allclose([float(r[1]) for r in rows[1:]], want, atol=1e-6)
    assert np.allclose([float(r[2]) for r in rows[1:]], np.array(want) - wref[0], atol=1e-6)
    def write_csv(muts):
        with open(tmp_path / "m.csv", "w", newline="") as f:
            w = csv.writer(f)
            w.writerow(["mutant", "DMS_score"])
            for mu in muts:
                w.writerow([mu, 0.5])
    write_csv([("A" if ref[0] != "A" else "C") + "1G"])                          # a wrong reference base
    with pytest.raises(ValueError, match="the reference has"):
        cli.main(["--reference-fasta", str(fasta), "--variants-csv", str(tmp_path / "m.csv"), "--output-tsv", str(out), "--device", DEV])
    muts = [sat[0][0], sat[100][0], f"{sat[7][0]}:{sat[300][0]}", ""]
    write_csv(muts)
    cli.main(["--reference-fasta", str(fasta), "--variants-csv", str(tmp_path / "m.csv"), "--output-tsv", str(out), "--device", DEV])
    rows = [line.split("\t") for line in out.read_text().splitlines()]
    seqs = [evo_b200.apply_mutations(ref, mu) for mu in muts]
    want, _ = evo_b200.score_variants(ref, seqs, m, tok, device=DEV)
    assert [r[0] for r in rows[1:]] == muts and np.allclose([float(r[1]) for r in rows[1:]], want, atol=1e-6)
    assert float(rows[-1][2]) == 0.0                                              # the wild type's delta


def test_rejected_calls_raise_before_any_launch(tiny):
    import evo_b200
    lib = _lib.lib()
    m = tiny[2]
    tok = evo_b200.CharLevelTokenizer(512)
    ids = torch.cat(_ids([300], seed=1)).to(DEV)
    ck = m.prefill_checkpoints(ids, [0, 300], 128)
    v = torch.cat(_ids([20], seed=2)).to(DEV)
    cases = [lambda: m.prefill_checkpoints(ids, [0, 300], 100),
             lambda: m.prefill_checkpoints(ids, [0, 300], 0),
             lambda: m.score_tokens_resumed(ck, v, [0, 20], [2], [0], [384]),      # past the reference's checkpoints
             lambda: m.score_tokens_resumed(ck, v, [0, 20], [0], [1], [128]),      # no reference 1
             lambda: m.score_tokens_resumed(ck, v, [0, 20], [0], [0], [300]),      # prefix_len at the reference's length
             lambda: m.score_tokens_resumed(ck, v, [0, 20], [-1], [0], [128]),
             lambda: m.score_tokens_resumed(ck, v, [0, 20], [1], [0], [128]),      # the checkpoint of another prefix length
             lambda: m.score_tokens_resumed(ck, v, [0, 10, 20], [0], [0], [128]),
             lambda: evo_b200.score_variants("ACGT" * 40, ["ACGT"], m, tok, checkpoint_stride=96, device=DEV)]
    for k, call in enumerate(cases):
        torch.cuda.synchronize()
        lib.evo_reset_launch_count()
        with pytest.raises((_lib.EvoError, ValueError)):
            call()
        assert lib.evo_launch_count() == 0, k
