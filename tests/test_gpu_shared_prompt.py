"""Shared-prompt sampling: the shared-prefix decode kernels (evo_decode_attn_shared, evo_decode_qkv_prep_shared),
StripedHyena.prefill_shared + decode_loop, and generate(ragged=True, share_prompts=True) / scripts.generate --share-prompts
on top of them.

Bars: the attention matches a float64 softmax over [prefix | suffix] keys within the _rows test's tolerance
(4 * 2^-7 * max(1, |ref|)); the rotary/append kernel gives evo_decode_qkv_prep_rows' bits.  Shared decoding agrees with the
replicated packed-prefill path within TAU of test_gpu_ragged_generation.py, compared the same way (kept logits before the first
token divergence, the top-1 margin where greedy tokens differ); bit-exactness is not expected, because the prefix is summed by
a different kernel (wgmma tiles of 128 keys) than the replicated cache (64-key tiles, other split counts)."""
import csv
import ctypes as C
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

from oracle import stripedhyena_oracle as O          # noqa: E402
from evo_b200 import _lib                             # noqa: E402
from evo_b200.stripedhyena import StripedHyena, dotdict  # noqa: E402

DEV = "cuda:0"
BF16_EPS = 2.0 ** -7
TAU = 4 * BF16_EPS            # test_gpu_ragged_generation.py's bar
NAN = float("nan")


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _model(hidden=256, heads=2, layers=4, attn=(1, 3), seed=7):
    cfg = O.tiny_config(num_layers=layers, attn_layer_idxs=attn, hidden_size=hidden, num_heads=heads)
    sd = O.random_state_dict(cfg, seed=seed)
    m = StripedHyena(dotdict(cfg))
    m.load_state_dict(sd, strict=True)
    m.to_bfloat16_except_poles_residues()
    return m.to(DEV)


# ------------------------------------------------------------------ kernels
# (rows per group, prefix_len per group): group sizes 1, 7, 64 and one above 64; prefix lengths 1, 127, 128, 129, 4096, 8193
GROUPINGS = {"g1x64": ([64], [4096]), "g3_mixed": ([7, 70, 1], [129, 127, 8193]), "g3_small": ([1, 7, 64], [1, 128, 4096])}
SPOS = [0, 1, 63, 64, 300]


def _shared_attention_case(rows, plen, S, seed):
    """Random prefix / suffix caches with NaN in every row a query must not see, and q of each row; float64 reference."""
    g = torch.Generator().manual_seed(seed)
    H, G, B = 2, len(rows), sum(rows)
    P = (max(plen) + 63) // 64 * 64
    pcache = torch.full((G, P, 2, H, 128), NAN, dtype=torch.bfloat16)
    for k, n in enumerate(plen):
        pcache[k, :n] = torch.randn(n, 2, H, 128, generator=g).bfloat16()
    spos = [SPOS[b % len(SPOS)] for b in range(B)]
    scache = torch.full((B, S, 2, H, 128), NAN, dtype=torch.bfloat16)
    for b, p in enumerate(spos):
        scache[b, :p + 1] = torch.randn(p + 1, 2, H, 128, generator=g).bfloat16()
    qkv = torch.full((B, 3, H, 128), NAN, dtype=torch.bfloat16)
    qkv[:, 0] = (torch.randn(B, H, 128, generator=g) * 2).bfloat16()
    group = [k for k, n in enumerate(rows) for _ in range(n)]
    scale = 1 / math.sqrt(128)
    ref = []
    for b in range(B):
        k_ = torch.cat([pcache[group[b], :plen[group[b]], 0], scache[b, :spos[b] + 1, 0]]).double()
        v_ = torch.cat([pcache[group[b], :plen[group[b]], 1], scache[b, :spos[b] + 1, 1]]).double()
        s = torch.einsum("hd,nhd->hn", qkv[b, 0].double(), k_) * scale
        ref.append(torch.einsum("hn,nhd->hd", torch.softmax(s, -1), v_).reshape(-1))
    offs = torch.tensor([0] + rows).cumsum(0)
    pos = [plen[group[b]] + spos[b] for b in range(B)]
    return dict(H=H, G=G, B=B, P=P, S=S, pcache=pcache, scache=scache, qkv=qkv, spos=spos, pos=pos, offs=offs, plen=plen,
                ref=torch.stack(ref))


def _run_shared_attention(c, nsp_p, nsp_s, dev_tensors=None):
    lib = _lib.lib()
    d = dev_tensors or {k: c[k].to(DEV) for k in ("pcache", "scache", "qkv")}
    offs = c["offs"].to(DEV)
    plen = torch.tensor(c["plen"], dtype=torch.int64, device=DEV)
    spos = torch.tensor(c["spos"], dtype=torch.int64, device=DEV)
    n = lib.evo_decode_attn_shared_workspace(c["B"], c["H"], nsp_p, nsp_s)
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    out = torch.empty(c["B"], c["H"] * 128, dtype=torch.bfloat16, device=DEV)
    _lib.check(lib.evo_decode_attn_shared(_lib.ptr(d["qkv"]), _lib.ptr(d["pcache"]), _lib.ptr(offs), _lib.ptr(plen), c["G"], c["P"],
                                          _lib.ptr(d["scache"]), _lib.ptr(spos), c["S"], _lib.ptr(out), c["B"], c["H"], 128, nsp_p, nsp_s,
                                          1 / math.sqrt(128), _lib.ptr(ws), n, stream()), "evo_decode_attn_shared")
    return out.double().cpu()


@pytest.mark.parametrize("S", [320, 310])          # 320: the TMA-fed suffix kernel; 310: the per-thread-row one
@pytest.mark.parametrize("grouping", sorted(GROUPINGS))
def test_shared_attention_matches_fp64_reference(grouping, S):
    rows, plen = GROUPINGS[grouping]
    c = _shared_attention_case(rows, plen, S, seed=len(grouping) + S)
    d = {k: c[k].to(DEV) for k in ("pcache", "scache", "qkv")}
    bar = 4 * BF16_EPS * max(1.0, c["ref"].abs().max().item())
    for nsp_p, nsp_s in [(1, 1), (3, 2), (5, 4), (64, 7)]:
        o = _run_shared_attention(c, nsp_p, nsp_s, d)
        assert not torch.isnan(o).any(), (nsp_p, nsp_s)
        err = (o - c["ref"]).abs().max().item()
        assert err <= bar, (nsp_p, nsp_s, err, bar)


def test_qkv_prep_shared_matches_rows_bits_and_writes_one_suffix_row():
    lib = _lib.lib()
    B, H, S, Pmax = 6, 2, 128, 600
    g = torch.Generator().manual_seed(4)
    cos, sin = O.rotary_tables(Pmax + S, 128, dtype=torch.bfloat16)
    cosd, sind = cos.to(DEV), sin.to(DEV)
    qkv = torch.randn(B, 3, H, 128, generator=g).bfloat16().to(DEV)
    spos = torch.tensor([0, 1, 63, 64, 100, 127], dtype=torch.int64)
    pos = spos + torch.tensor([1, 599, 128, 5, 400, 64])
    posd, sposd = pos.to(DEV), spos.to(DEV)
    full = torch.zeros(B, Pmax + S, 2, H, 128, dtype=torch.bfloat16, device=DEV)
    x_rows = qkv.clone()
    _lib.check(lib.evo_decode_qkv_prep_rows(_lib.ptr(x_rows), _lib.ptr(full), _lib.ptr(cosd), _lib.ptr(sind), _lib.ptr(posd),
                                            B, H, 128, Pmax + S, stream()))
    suffix0 = torch.full((B, S, 2, H, 128), NAN, dtype=torch.bfloat16)
    suffix = suffix0.to(DEV)
    x_sh = qkv.clone()
    _lib.check(lib.evo_decode_qkv_prep_shared(_lib.ptr(x_sh), _lib.ptr(suffix), _lib.ptr(cosd), _lib.ptr(sind), _lib.ptr(posd),
                                              _lib.ptr(sposd), B, H, 128, S, stream()), "evo_decode_qkv_prep_shared")
    assert torch.equal(x_sh.cpu().view(torch.int16), x_rows.cpu().view(torch.int16))
    got, want = suffix.cpu(), suffix0.clone()
    for b in range(B):
        want[b, spos[b]] = full[b, pos[b]].cpu()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))       # row spos[b] written, every other row untouched


def test_rejected_kernel_arguments():
    lib = _lib.lib()
    assert lib.evo_decode_attn_shared(None, None, None, None, 2, 64, None, None, 64, None, 1, 2, 128, 1, 1, 0.1, None, 0, None) < 0
    assert b"group count" in lib.evo_last_error()
    assert lib.evo_decode_attn_shared(None, None, None, None, 1, 64, None, None, 64, None, 1, 2, 64, 1, 1, 0.1, None, 0, None) < 0
    assert b"head_dim" in lib.evo_last_error()
    assert lib.evo_decode_attn_shared(None, None, None, None, 1, 64, None, None, 64, None, 1, 2, 128, 0, 1, 0.1, None, 0, None) < 0
    assert b"nsplit" in lib.evo_last_error()


# ------------------------------------------------------------------ model
def _greedy_both_arms(m, prompts, rows, n):
    """Greedy decoding of the replicated prompts from prefill_shared and from prefill_ragged(packed=True), both fed the same
    first token (the shared arm's argmax).  Returns (head + kept logits, first + picked tokens) per arm, shared arm first."""
    V = m.config.vocab_size
    rep = [p for p, k in zip(prompts, rows) for _ in range(k)]
    starts = torch.tensor([len(p) for p in rep], dtype=torch.int64)
    cache_len = (max(len(p) for p in rep) + n + 63) // 64 * 64
    out = []
    with torch.inference_mode():
        head_r, ipd_r = m.prefill_ragged(rep, cache_len, packed=True)
        head_s, ipd_s = m.prefill_shared(prompts, rows, n)
        first = head_s.float().argmax(-1)
    assert head_s.shape == head_r.shape == (len(rep), V)
    for head, ipd in ((head_s, ipd_s), (head_r, ipd_r)):
        m._loop = None
        got, kept = m.decode_loop(first, ipd, n, starts, top_k=1)
        out.append((torch.cat([head.float().cpu()[:, None], kept.cpu()], 1), torch.cat([first.cpu()[:, None], got.cpu()], 1)))
    return out


def _compare_arms(shared, replicated, rows):
    (ls, ids_s), (lr, ids_r) = shared, replicated
    worst = 0.0
    for b in range(ls.shape[0]):
        scale = max(1.0, lr[b].abs().max().item())
        for t in range(ls.shape[1]):
            d = (ls[b, t] - lr[b, t]).abs().max().item() / scale
            worst = max(worst, d)
            assert d <= TAU, (b, t, d)
            if ids_s[b, t] != ids_r[b, t]:               # logits t picked token t (t >= 1; token 0 is fed to both arms)
                top2 = lr[b, t].topk(2).values
                assert (top2[0] - top2[1]).item() / scale <= TAU, (b, t)
                break
    r0 = 0
    for k in rows:                                        # rows of one group, fed the same tokens: the same bits
        for b in range(r0 + 1, r0 + k):
            assert torch.equal(ids_s[b], ids_s[r0])
            assert torch.equal(ls[b].view(torch.int32), ls[r0].view(torch.int32)), b
        r0 += k
    return worst


def _prompts(lengths, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randint(0, 4, (n,), generator=g) * 3 + 65).tolist() for n in lengths]


def test_prefill_shared_decode_matches_replicated_prefill_tiny():
    """Three groups (3, 1 and 70 rows: one above 64), prefix lengths 300, 9 and 1100 (the prefix kernel splits)."""
    m = _model()
    rows = [3, 1, 70]
    worst = _compare_arms(*_greedy_both_arms(m, _prompts([300, 9, 1100], 1), rows, 40), rows)
    print(f"\nshared vs replicated (tiny): worst kept-logit difference {worst:.3e} of the row's max |logit|")


def test_prefill_shared_decode_matches_replicated_prefill_7b_width():
    """The 7B's width (32 heads) with random weights; one group of 5 rows over a 1500-token prefix: 4 prefix splits."""
    m = _model(hidden=4096, heads=32, layers=3, attn=(1,))
    rows = [5]
    worst = _compare_arms(*_greedy_both_arms(m, _prompts([1500], 2), rows, 24), rows)
    print(f"\nshared vs replicated (7B width): worst kept-logit difference {worst:.3e} of the row's max |logit|")


def test_decode_loop_rejects_a_shared_state_without_room():
    m = _model(layers=2, attn=(1,))
    with torch.inference_mode():
        head, ipd = m.prefill_shared(_prompts([10, 20], 3), [2, 2], 64)
    start = torch.tensor([10, 10, 20, 20])
    with pytest.raises(_lib.EvoError, match="exceeds the KV cache"):
        m.decode_loop(head.argmax(-1), ipd, 65, start)
    with pytest.raises(ValueError, match="per-row"):
        m.decode_loop(head.argmax(-1), ipd, 4, 10)
    with pytest.raises(ValueError, match="inside"):
        m.decode_loop(head.argmax(-1), ipd, 4, start - 1)


# ------------------------------------------------------------------ generate()
def _tok():
    import evo_b200
    return evo_b200.CharLevelTokenizer(512)


def test_shared_sampling_rows_differ_and_seed_reproduces():
    import evo_b200
    m = _model(layers=3, attn=(1,))
    kw = dict(n_tokens=32, top_k=4, top_p=1.0, temperature=1.0, cached_generation=True, verbose=0, device=DEV, ragged=True, share_prompts=True)
    prompts = ["ACGTTGCAAC"] * 6 + ["GATTACA"] * 2
    torch.manual_seed(11)
    a, sa = evo_b200.generate(prompts, m, _tok(), **kw)
    torch.manual_seed(11)
    b, sb = evo_b200.generate(prompts, m, _tok(), **kw)
    torch.manual_seed(12)
    c, _ = evo_b200.generate(prompts, m, _tok(), **kw)
    assert a == b and sa == sb
    assert a != c
    assert len(set(a[:6])) > 1                           # rows of one group draw different samples
    assert all(len(x) == 32 for x in a)


def test_interleaved_prompts_come_back_in_input_order():
    import evo_b200
    m = _model()
    kw = dict(n_tokens=16, top_k=1, top_p=1.0, temperature=1.0, cached_generation=True, verbose=0, device=DEV, ragged=True)
    a, b, c = "ACGTTGCAACGTAC", "TTG", "GGGACTTACAGTCAGGCATTAGC"
    prompts = [a, b, a, c, b, a]
    texts, scores = evo_b200.generate(prompts, m, _tok(), share_prompts=True, **kw)
    ref_t, ref_s = evo_b200.generate(prompts, m, _tok(), packed_prefill=True, **kw)
    assert texts == ref_t
    assert all(abs(x - y) <= TAU * max(1.0, abs(y)) for x, y in zip(scores, ref_s))
    assert texts[0] == texts[2] == texts[5] and texts[1] == texts[4] and scores[0] == scores[2] == scores[5]
    assert len({texts[0], texts[1], texts[3]}) == 3


def test_one_prompt_over_several_batches_is_prefilled_once(monkeypatch):
    import evo_b200
    m = _model(layers=3, attn=(1,))
    calls = []
    real = m.prefill_prefixes
    monkeypatch.setattr(m, "prefill_prefixes", lambda prompts: calls.append(len(prompts)) or real(prompts))
    kw = dict(n_tokens=12, top_k=1, cached_generation=True, verbose=0, device=DEV, ragged=True, share_prompts=True)
    texts, scores = evo_b200.generate(["ACGTACGTTAGC"] * 10 + ["TTAG"], m, _tok(), batch_size=4, **kw)
    assert calls == [1, 1]                               # the first prompt before batch 1, the second before batch 3
    assert len(set(texts[:10])) == 1 and len(set(scores[:10])) == 1 and len(texts) == 11


def test_rejected_calls_raise_before_any_launch():
    import evo_b200
    lib = _lib.lib()
    m = _model(layers=2, attn=(1,))
    m.config["max_seqlen"] = 16
    kw = dict(top_k=1, verbose=0, device=DEV, cached_generation=True, share_prompts=True)
    cases = [(ValueError, lambda: evo_b200.generate(["ACGT", "ACGT"], m, _tok(), n_tokens=4, **kw)),                       # not ragged
             (ValueError, lambda: evo_b200.generate(["ACGT", ""], m, _tok(), n_tokens=4, ragged=True, **kw)),
             (_lib.EvoError, lambda: evo_b200.generate(["ACGT", "A" * 17], m, _tok(), n_tokens=4, ragged=True, **kw)),
             (ValueError, lambda: evo_b200.generate(["ACGT", "ACGT"], m, _tok(), n_tokens=0, ragged=True, **kw))]
    for exc, call in cases:
        torch.cuda.synchronize()
        lib.evo_reset_launch_count()
        with pytest.raises(exc):
            call()
        assert lib.evo_launch_count() == 0


def _cli(monkeypatch, m):
    import evo_b200
    from scripts import generate as cli

    class TinyEvo:
        def __init__(self, *a, **kw):
            self.model, self.tokenizer = m, evo_b200.CharLevelTokenizer(512)
    monkeypatch.setattr(cli, "Evo", TinyEvo)
    return cli


def test_cli_share_prompts_and_samples_per_prompt(tmp_path, monkeypatch, capsys):
    m = _model(layers=2, attn=(1,))
    cli = _cli(monkeypatch, m)
    calls = []
    real = m.prefill_prefixes
    monkeypatch.setattr(m, "prefill_prefixes", lambda prompts: calls.append(len(prompts)) or real(prompts))
    texts, scores = cli.main(["--prompt", "ACGTAC", "--n-samples", "5", "--n-tokens", "8", "--top-k", "4", "--device", DEV,
                              "--share-prompts", "--seed", "3"])
    assert len(texts) == len(scores) == 5 and all(len(t) == 8 for t in texts) and calls == [1]
    assert capsys.readouterr().out.count('Prompt: "ACGTAC"') == 5

    prompts = ["ACGTACGTACGTAAC", "T", "GGCATTAGC"]
    path = tmp_path / "prompts.csv"
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["prompt", "note"])
        for i, p in enumerate(prompts):
            w.writerow([p, f"row{i}"])
    for share in (False, True):
        calls.clear()
        args = ["--prompts-csv", str(path), "--samples-per-prompt", "3", "--n-tokens", "8", "--top-k", "1", "--device", DEV, "--batch-size", "4"]
        texts, scores = cli.main(args + (["--share-prompts"] if share else []))
        assert len(texts) == 9 and all(len(t) == 8 for t in texts)
        assert calls == ([2, 1] if share else [])
        out = capsys.readouterr().out
        expect = [p for p in prompts for _ in range(3)]                  # prompt-major
        at = [out.index(f'Prompt: "{p}",\tOutput: "{t}",\tScore: {s}') for p, t, s in zip(expect, texts, scores)]
        assert at == sorted(at) and out.count("Prompt: ") == 9
