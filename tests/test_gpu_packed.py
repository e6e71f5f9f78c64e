"""Packed variable-length forward: sequences laid end to end as one (T,) batch with cu_seqlens offsets.

Kernels (evo_hyena_fwd_varlen, evo_attn_fwd_varlen, evo_kv_append_varlen) are held bit for bit to the calls they replace:
each sequence alone at batch 1, or the (n, L) batch when every length is equal.  Forced segmentations of the varlen scan
are held to the oracle bars tests/test_gpu_hyena_paths.py applies to the segmented batched scan.  The model's packed paths
(forward_packed, score_tokens_packed, prefill_ragged(packed=True)) are bit-identical to the batched paths on equal lengths,
and within MIXED_TAU of each sequence's solo forward on mixed lengths (the packed GEMMs tile M = T rows differently, and
the scan's segmentation depends on the batch).  Public surface: score_many(packed=True), scripts/score.py --packed,
generate(ragged=True, packed_prefill=True), and the calls that must raise before anything is launched."""
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
from tests.test_gpu_hyena_paths import _assert_state, _assert_vs_oracle, _bf16_oracle, _filter_sd, _fp64_oracle, _hyena_call  # noqa: E402

DEV = "cuda:0"
BF16_EPS = 2.0 ** -7
MIXED_TAU = 4 * BF16_EPS            # the bar of test_mixed_lengths_match_solo_generation, relative to max(1, |logits|max)
MIXED = (1, 2, 3, 15, 16, 17, 100, 1023, 1024, 4097)     # starts at rows that are no multiple of 16


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _cu(lengths):
    return [0] + np.cumsum(lengths).tolist()


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


def _same(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _filter(D, seed=1):
    if D <= 384:
        return _filter_sd(D, seed)[1]
    g = torch.Generator().manual_seed(seed)
    mag = 0.5 + 0.45 * torch.rand(D, 8, 1, generator=g)
    ang = (torch.rand(D, 8, 1, generator=g) * 2 - 1) * math.pi
    f = {"w": (torch.randn(3 * D, 1, 3, generator=g) * 0.3).bfloat16(), "b": (torch.randn(3 * D, generator=g) * 0.1).bfloat16(),
         "D": torch.randn(D, generator=g).bfloat16(), "p": torch.stack([mag * torch.cos(ang), mag * torch.sin(ang)], dim=-1),
         "r": torch.randn(D, 8, 1, 2, generator=g) * 0.3}
    return {k: v.contiguous().to(DEV) for k, v in f.items()}


def _hyena_varlen(z, f, H, lengths, seg_len=0, want_state=True):
    lib = _lib.lib()
    T, C3 = z.shape
    D, n = C3 // 3, len(lengths)
    cu = torch.tensor(_cu(lengths), dtype=torch.int64, device=DEV)
    y = torch.empty(T, D, dtype=torch.bfloat16, device=DEV)
    st = torch.empty(n, D, 8, 2, dtype=torch.float32, device=DEV) if want_state else None
    fs = torch.empty(n, C3, 2, dtype=torch.bfloat16, device=DEV) if want_state else None
    hp = _lib.HyenaVarlenParams(z=z.data_ptr(), y=y.data_ptr(), fir_w=f["w"].data_ptr(), fir_b=f["b"].data_ptr(), Dskip=f["D"].data_ptr(),
                                poles=f["p"].data_ptr(), residues=f["r"].data_ptr(), cu_seqlens=cu.data_ptr(), n_seq=n, T=T,
                                max_seqlen=max(lengths), D=D, S=8, nheads=H, state_out=st.data_ptr() if st is not None else None,
                                fir_state_out=fs.data_ptr() if fs is not None else None, seg_len=seg_len)
    need = lib.evo_hyena_fwd_varlen_workspace(C.byref(hp))
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
    _lib.check(lib.evo_hyena_fwd_varlen(C.byref(hp), _lib.ptr(ws), need, stream()), "evo_hyena_fwd_varlen")
    torch.cuda.synchronize()
    return y, st, fs, need


# ------------------------------------------------------------------ kernels, bit for bit
@pytest.mark.parametrize("D", [256, 4096])
def test_hyena_varlen_matches_each_sequence_alone(D):
    H = D // 128
    f = _filter(D)
    g = torch.Generator().manual_seed(D)
    z = torch.randn(sum(MIXED), 3 * D, generator=g).bfloat16().to(DEV)
    y, st, fs, _ = _hyena_varlen(z, f, H, MIXED, seg_len=max(MIXED))
    cu = _cu(MIXED)
    for b, L in enumerate(MIXED):
        ys, ss, fss, _ = _hyena_call(z[cu[b]:cu[b + 1]].unsqueeze(0).contiguous(), f, H, force=1, want_state=True)
        assert _same(y[cu[b]:cu[b + 1]], ys[0]), (D, L)
        assert _same(st[b], ss[0]), (D, L)
        assert _same(fs[b], fss[0]), (D, L)


@pytest.mark.parametrize("D,n,L", [(256, 3, 1025), (256, 1, 4099), (256, 5, 17), (4096, 2, 8193), (4096, 4, 300)])
def test_hyena_varlen_equal_lengths_match_the_batched_call(D, n, L):
    """Automatic geometry on both sides; (256, 1, 4099) and (4096, 2, 8193) are segmented by the batched launcher."""
    H = D // 128
    f = _filter(D)
    g = torch.Generator().manual_seed(n * L)
    z = torch.randn(n, L, 3 * D, generator=g).bfloat16().to(DEV)
    yb, sb, fb, wsb = _hyena_call(z, f, H, force=0, want_state=True)
    y, st, fs, need = _hyena_varlen(z.view(n * L, 3 * D), f, H, [L] * n)
    assert need == wsb.numel() or (need == 0 and wsb.numel() == 1)        # same segment count
    assert _same(y, yb.view(n * L, D)) and _same(st, sb) and _same(fs, fb)


@pytest.mark.parametrize("seg_len", [64, 100, 1000])
def test_hyena_varlen_segmented_vs_oracle(seg_len):
    """Forced segmentations (100 is no multiple of the 16-token stage): every sequence within the segmented batched scan's
    bars against the bf16 FFT operator and the fp64 recurrence, for y and for state_out."""
    D, H = 256, 2
    sd, f = _filter_sd(D)
    lengths = (1, 17, 100, 130, 1023, 2500)
    g = torch.Generator().manual_seed(seg_len)
    z = torch.randn(sum(lengths), 3 * D, generator=g).bfloat16()
    y, st, fs, _ = _hyena_varlen(z.to(DEV), f, H, lengths, seg_len=seg_len)
    cu = _cu(lengths)
    for b, L in enumerate(lengths):
        zb = z[cu[b]:cu[b + 1]].unsqueeze(0)
        yb, stb = _bf16_oracle(sd, zb, H, want_state=True)
        yt, stt = _fp64_oracle(sd, zb, H)
        what = f"seg_len={seg_len} L={L}"
        _assert_vs_oracle(y[cu[b]:cu[b + 1]].unsqueeze(0), yb, yt, what)
        _assert_state(st[b:b + 1], stb, 2e-4, what + " state vs bf16 oracle")
        _assert_state(st[b:b + 1], stt, 1e-2, what + " state vs fp64")
        assert torch.equal(fs[b].cpu()[:, 2 - min(L, 2):], zb[0, -2:].T), what


def _attn_batch1(qkv, r0, L, H, out):
    lib = _lib.lib()
    d = H * 128
    base = qkv.data_ptr() + r0 * 3 * d * 2
    ap = _lib.AttnParams(out=out.data_ptr(), B=1, Lq=L, Lk=L, H=H, hd=128, q_pos0=0, softmax_scale=1.0 / math.sqrt(128))
    ap.q, ap.k, ap.v = base, base + d * 2, base + 2 * d * 2
    ap.q_tok_stride = ap.kv_tok_stride = 3 * d
    ap.q_batch_stride = ap.kv_batch_stride = L * 3 * d
    _lib.check(lib.evo_attn_fwd_ws(C.byref(ap), 2, None, 0, stream()), "evo_attn_fwd_ws")


def _attn_varlen(qkv, lengths, H):
    lib = _lib.lib()
    T, d = qkv.shape[0], H * 128
    cu = torch.tensor(_cu(lengths), dtype=torch.int64, device=DEV)
    out = torch.empty(T, d, dtype=torch.bfloat16, device=DEV)
    ap = _lib.AttnVarlenParams(q=qkv.data_ptr(), k=qkv.data_ptr() + d * 2, v=qkv.data_ptr() + 2 * d * 2, out=out.data_ptr(),
                               q_tok_stride=3 * d, kv_tok_stride=3 * d, cu_seqlens=cu.data_ptr(), n_seq=len(lengths), T=T,
                               max_seqlen=max(lengths), H=H, hd=128, softmax_scale=1.0 / math.sqrt(128))
    _lib.check(lib.evo_attn_fwd_varlen(C.byref(ap), stream()), "evo_attn_fwd_varlen")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("H", [2, 32])
def test_attention_varlen_matches_batch1_and_nothing_leaks(H):
    lengths = (300, 1, 127, 128, 129, 2, 1000, 17) if H == 2 else (1025, 3, 130)
    g = torch.Generator().manual_seed(H)
    qkv = torch.randn(sum(lengths), 3 * H * 128, generator=g).bfloat16().to(DEV)
    out = _attn_varlen(qkv, lengths, H)
    cu = _cu(lengths)
    for b, L in enumerate(lengths):
        ref = torch.empty(L, H * 128, dtype=torch.bfloat16, device=DEV)
        _attn_batch1(qkv, cu[b], L, H, ref)
        torch.cuda.synchronize()
        assert _same(out[cu[b]:cu[b + 1]], ref), (H, L)
    j = 2 if H == 2 else 1                                       # perturb one sequence's q, k and v
    qkv2 = qkv.clone()
    qkv2[cu[j]:cu[j + 1]] = torch.randn(lengths[j], 3 * H * 128, generator=g).bfloat16().to(DEV)
    out2 = _attn_varlen(qkv2, lengths, H)
    for b in range(len(lengths)):
        if b != j:
            assert _same(out2[cu[b]:cu[b + 1]], out[cu[b]:cu[b + 1]]), b
    assert not _same(out2[cu[j]:cu[j + 1]], out[cu[j]:cu[j + 1]])


def test_kv_append_varlen_matches_per_sequence_append():
    lib = _lib.lib()
    H, S = 2, 1040
    lengths = (17, 1, 1024, 300)
    g = torch.Generator().manual_seed(4)
    qkv = torch.randn(sum(lengths), 3, H, 128, generator=g).bfloat16().to(DEV)
    init = torch.randn(len(lengths), S, 2, H, 128, generator=g).bfloat16().to(DEV)
    got, want = init.clone(), init.clone()
    cu = _cu(lengths)
    cud = torch.tensor(cu, dtype=torch.int64, device=DEV)
    _lib.check(lib.evo_kv_append_varlen(_lib.ptr(qkv), _lib.ptr(got), _lib.ptr(cud), len(lengths), qkv.shape[0], max(lengths), H, 128, S, stream()))
    for b, L in enumerate(lengths):
        _lib.check(lib.evo_kv_append(C.c_void_p(qkv[cu[b]].data_ptr()), C.c_void_p(want[b].data_ptr()), 1, L, H, 128, 0, S, stream()))
    torch.cuda.synchronize()
    assert _same(got, want)


# ------------------------------------------------------------------ model
def _tiny(layers=4, attn=(1, 3), seed=7):
    cfg = O.tiny_config(num_layers=layers, attn_layer_idxs=attn, hidden_size=256, num_heads=2)
    sd = O.random_state_dict(cfg, seed=seed)
    m = StripedHyena(dotdict(cfg))
    m.load_state_dict(sd, strict=True)
    m.to_bfloat16_except_poles_residues()
    return cfg, sd, m.to(DEV)


def _two_block_7b():
    cfg = O.evo_config("evo-1-8k-base")
    cfg.update(num_layers=2, attn_layer_idxs=[1], hyena_layer_idxs=[0])
    sd = O.random_state_dict(cfg, seed=3)
    m = StripedHyena(dotdict(cfg))
    m.load_state_dict(sd, strict=True)
    m.to_bfloat16_except_poles_residues()
    return cfg, sd, m.to(DEV)


def _ids(lengths, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 4, (L,), generator=g) * 3 + 65 for L in lengths]


@pytest.fixture(scope="module")
def tiny():
    return _tiny()


@pytest.fixture(scope="module")
def wide():
    return _two_block_7b()


@pytest.mark.parametrize("which,n,L", [("tiny", 3, 200), ("tiny", 2, 1025), ("wide", 2, 1024), ("wide", 2, 8193)])
def test_equal_lengths_are_bit_identical_to_the_batched_forward(which, n, L, tiny, wide):
    m = (tiny if which == "tiny" else wide)[2]
    ids = torch.stack(_ids([L] * n, seed=L)).to(DEV)
    cu = _cu([L] * n)
    flat = ids.reshape(-1)
    if L <= 1025:                                                # the (n*L, 512) logits of 8193 tokens are checked through the scores
        logits, _ = m(ids)
        assert _same(m.forward_packed(flat, cu), logits.reshape(n * L, -1))
    lp, ent = m.score_tokens(ids, want_logprobs=True, want_entropy=True)
    plp, pent = m.score_tokens_packed(flat, cu, want_logprobs=True, want_entropy=True)
    assert _same(plp, lp.reshape(-1)) and _same(pent, ent.reshape(-1))


@pytest.mark.parametrize("which", ["tiny", "wide"])
def test_mixed_lengths_match_each_sequence_alone(which, tiny, wide):
    cfg, sd, m = tiny if which == "tiny" else wide
    lengths = (130, 1, 64, 2, 1000, 17) if which == "tiny" else (1500, 1, 300, 17)
    seqs = _ids(lengths, seed=11)
    cu = _cu(lengths)
    flat = torch.cat(seqs).to(DEV)
    logits = m.forward_packed(flat, cu).cpu()
    lp, ent = m.score_tokens_packed(flat, cu, want_logprobs=True, want_entropy=True)
    lp, ent = lp.cpu(), ent.cpu()
    worst = 0.0
    for b, s in enumerate(seqs):
        solo = m(s[None].to(DEV))[0][0].cpu()
        d = (logits[cu[b]:cu[b + 1]].double() - solo.double()).abs().max().item() / max(1.0, solo.abs().max().item())
        worst = max(worst, d)
        assert d <= MIXED_TAU, (which, lengths[b], d)
        # a logit error of at most e moves a log-softmax entry by <= 2e and the entropy by <= 2e * log(V)
        e = MIXED_TAU * max(1.0, solo.abs().max().item())
        slp, sent = m.score_tokens(s[None].to(DEV), want_logprobs=True, want_entropy=True)
        assert (lp[cu[b]:cu[b + 1]] - slp[0].cpu()).abs().max().item() <= 2 * e, lengths[b]
        assert (ent[cu[b]:cu[b + 1]] - sent[0].cpu()).abs().max().item() <= 2 * e * math.log(cfg["vocab_size"]), lengths[b]
        assert lp[cu[b + 1] - 1] == 0                            # no target past a sequence's end
    print(f"\n{which}: packed vs solo logits, worst difference {worst:.3e} of max(1, |logits|max)")
    if which == "tiny":                                          # the scores against the fp64 oracle (test_public_api_scoring_and_generation's bar)
        ot = O.OracleStripedHyena(cfg, sd, torch.float64)
        for b, s in enumerate(seqs):
            if lengths[b] < 2:
                continue
            ref = torch.log_softmax(ot(s[None])[0], -1)[0, :-1].gather(1, s[1:, None])[:, 0]
            assert abs(ref.mean().item() - lp[cu[b]:cu[b + 1] - 1].double().mean().item()) < 8e-2, lengths[b]


def _prefill_both(m, prompts, cache_len):
    grouped = m.prefill_ragged(prompts, cache_len)
    packed = m.prefill_ragged(prompts, cache_len, packed=True)
    return grouped, packed


def test_packed_prefill_equal_lengths_is_bit_identical(tiny):
    m = tiny[2]
    prompts = [p.tolist() for p in _ids([50] * 3, seed=5)]
    (hg, sg), (hp, sp) = _prefill_both(m, prompts, 128)
    assert _same(hg, hp)
    for i in sg["hyena"].state_dict:
        assert _same(torch.view_as_real(sg["hyena"].state_dict[i]), torch.view_as_real(sp["hyena"].state_dict[i]))
        assert _same(sg["hyena"].fir_state_dict[i], sp["hyena"].fir_state_dict[i])
    assert set(sg["mha"].key_value_memory_dict) == set(sp["mha"].key_value_memory_dict) == {1, 3}
    for i in sg["mha"].key_value_memory_dict:
        assert _same(sg["mha"].key_value_memory_dict[i], sp["mha"].key_value_memory_dict[i])
    assert torch.equal(sg["mha"].lengths_per_sample, sp["mha"].lengths_per_sample)


def test_packed_prefill_mixed_lengths(tiny, monkeypatch):
    import evo_b200
    from tests.test_gpu_ragged_generation import TAU, _capture_logprob_inputs
    m = tiny[2]
    lengths = [1, 7, 7, 63, 64, 65, 300]
    prompts = [p.tolist() for p in _ids(lengths, seed=9)]
    (hg, _), (hp, _) = _prefill_both(m, prompts, 384)
    hg, hp = hg.double().cpu(), hp.double().cpu()
    d = ((hg - hp).abs().max(-1).values / hg.abs().max(-1).values.clamp(min=1.0)).max().item()
    print(f"\npacked vs grouped prefill head logits: worst difference {d:.3e} of max(1, |logits|max)")
    assert d <= MIXED_TAU
    # generate(ragged=True, packed_prefill=True) against each prompt generated alone: the bar of the ragged test
    tok = evo_b200.CharLevelTokenizer(512)
    g = torch.Generator().manual_seed(3)
    lens = [65, 1, 300, 7, 2, 7]
    texts_in = ["".join("ACGT"[int(i)] for i in torch.randint(0, 4, (L,), generator=g)) for L in lens]
    n = 12
    kw = dict(n_tokens=n, top_k=1, top_p=1.0, temperature=1.0, cached_generation=True, verbose=0, device=DEV)
    seen = _capture_logprob_inputs(monkeypatch)
    texts, _ = evo_b200.generate(texts_in, m, tok, ragged=True, packed_prefill=True, **kw)
    rag_logits, rag_ids = seen[0]
    order = sorted(range(len(lens)), key=lambda i: (lens[i], i))
    for k, i in enumerate(order):
        seen.clear()
        solo, _ = evo_b200.generate([texts_in[i]], m, tok, batched=True, force_prompt_threshold=4096, **kw)
        s_logits, s_ids = seen[0]
        scale = max(1.0, s_logits[0].abs().max().item())
        for t in range(n):
            assert (rag_logits[k, t] - s_logits[0, t]).abs().max().item() / scale <= TAU, (i, t)
            if rag_ids[k, t] != s_ids[0, t]:
                top2 = s_logits[0, t].topk(2).values
                assert (top2[0] - top2[1]).item() / scale <= TAU, (i, t)
                break
        else:
            assert texts[i] == solo[0]


def test_score_many_packed_in_input_order_and_cli(tiny, tmp_path, monkeypatch):
    import evo_b200
    from evo_b200.frontend import score_many
    from scripts import score as cli
    m = tiny[2]
    tok = evo_b200.CharLevelTokenizer(512)
    rng = np.random.default_rng(1)
    seqs = ["".join(rng.choice(list("ACGT"), size=n)) for n in (40, 7, 40, 129, 1, 41, 300, 8)]
    packed = score_many(seqs, m, tok, max_tokens=200, device=DEV, packed=True)
    single = [float(evo_b200.score_sequences([s], m, tok, device=DEV)[0]) for s in seqs]
    assert len(packed) == len(seqs) and np.allclose(packed, single, atol=2e-2)
    sums = score_many(seqs, m, tok, max_tokens=200, device=DEV, packed=True, reduce_method="sum")
    assert np.allclose(np.array(sums) / np.array([len(s) for s in seqs]), packed, atol=1e-5)
    fasta = tmp_path / "in.fasta"
    fasta.write_text("".join(f">s{i}\n{s}\n" for i, s in enumerate(seqs)))

    class TinyEvo:
        def __init__(self, *a, **kw):
            self.model, self.tokenizer = m, tok
    monkeypatch.setattr(cli, "Evo", TinyEvo)
    outs = {}
    for flag in ([], ["--packed"]):
        path = tmp_path / f"out{len(flag)}.tsv"
        cli.main(["--input-fasta", str(fasta), "--output-tsv", str(path), "--device", DEV, "--max-tokens", "256"] + flag)
        outs[len(flag)] = [line.split("\t") for line in path.read_text().splitlines()]
    a, b = outs[0], outs[1]
    assert a[0] == b[0] == ["seqs", "scores"] and [r[0] for r in a] == [r[0] for r in b]
    assert np.allclose([float(r[1]) for r in a[1:]], [float(r[1]) for r in b[1:]], atol=2e-2)


def test_rejected_calls_raise_before_any_launch(tiny):
    lib = _lib.lib()
    m = tiny[2]
    ids = torch.cat(_ids([5, 3], seed=1)).to(DEV)
    cfg64 = O.tiny_config(num_layers=2, attn_layer_idxs=(1,), hidden_size=256, num_heads=4)
    m64 = StripedHyena(dotdict(cfg64))
    m64.load_state_dict(O.random_state_dict(cfg64, seed=1), strict=True)
    m64 = m64.to_bfloat16_except_poles_residues().to(DEV)
    cases = [lambda: m.forward_packed(ids, [0, 5, 5, 8]),                 # empty sequence
             lambda: m.forward_packed(ids, [0, 6, 5, 8]),                 # not increasing
             lambda: m.forward_packed(ids, [0, 5, 7]),                    # does not end at T
             lambda: m.forward_packed(ids, [1, 5, 8]),
             lambda: m.score_tokens_packed(ids.cpu(), [0, 5, 8]),         # ids on another device
             lambda: m64.forward_packed(ids, [0, 5, 8]),                  # head_dim 64
             lambda: m.score_tokens_packed(ids, [0, 8, 8]),
             lambda: m.prefill_ragged([[65] * 5, []], 64, packed=True),
             lambda: m.prefill_ragged([[65] * 5, [66] * 70], 64, packed=True),
             lambda: m64.prefill_ragged([[65] * 5, [66] * 7], 64, packed=True)]
    for k, call in enumerate(cases):
        torch.cuda.synchronize()
        lib.evo_reset_launch_count()
        with pytest.raises(_lib.EvoError):
            call()
        assert lib.evo_launch_count() == 0, k
