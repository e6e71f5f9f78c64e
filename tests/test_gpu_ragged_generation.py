"""Batched generation of prompts of different lengths: the per-row-position decode kernels (evo_decode_qkv_prep_rows,
evo_decode_attn_rows, evo_advance_positions), StripedHyena.prefill_ragged + decode_loop with a (B,) start position, and
generate(ragged=True) / scripts.generate --prompts-csv on top of them.

Bars: the _rows kernels match a float64 torch reference at random per-row positions with the tolerance of the scalar
decode test (test_gpu_parity.py), and give the scalar kernels' bits when every row sits at the same position.  Ragged
generation of same-length prompts is bit-identical to today's batched path; mixed lengths agree with each prompt generated
alone within TAU (bit-exactness is not expected: the decode attention's split count and the Hyena scan's L-segmentation
depend on the batch)."""
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
# mixed-length ragged vs solo generation: bound on |kept logit difference| before the first token divergence, relative to the
# row's largest |logit|, and on the solo top-1 margin where greedy tokens may differ.  Measured on one H100 with the tiny model
# of test_mixed_lengths_match_solo_generation: 0 (every row bit-identical to its solo run); the bound leaves room for the
# summation-order differences batch-dependent split counts and scan segmentations can bring at other sizes.
TAU = 4 * BF16_EPS


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _tiny(layers=4, attn=(1, 3), seed=7):
    cfg = O.tiny_config(num_layers=layers, attn_layer_idxs=attn, hidden_size=256, num_heads=2)
    sd = O.random_state_dict(cfg, seed=seed)
    m = StripedHyena(dotdict(cfg))
    m.load_state_dict(sd, strict=True)
    m.to_bfloat16_except_poles_residues()
    return m.to(DEV)


# ------------------------------------------------------------------ kernels
def _attend(q, k, v, scale):
    """q (H, 128), k/v (n, H, 128) -> (H*128,) in float64"""
    s = torch.einsum("hd,nhd->hn", q.double(), k.double()) * scale
    return torch.einsum("hn,nhd->hd", torch.softmax(s, -1), v.double()).reshape(-1)


@pytest.mark.parametrize("S", [640, 600])
def test_rows_kernels_match_reference_at_per_row_positions(S):
    """S = 640 takes the TMA-fed attention kernel, S = 600 the per-thread-row one.  Cache rows past a row's position hold
    NaN: they must not leak into that row's result."""
    B, H = 5, 2
    lib = _lib.lib()
    g = torch.Generator().manual_seed(21)
    full = torch.randn(B, S, 3, H, 128, generator=g).bfloat16()
    cos, sin = O.rotary_tables(S, 128, dtype=torch.bfloat16)
    qr = O.apply_rotary(full[:, :, 0], cos, sin)
    kr = O.apply_rotary(full[:, :, 1], cos, sin)
    pos = [0, S - 1, 1, 64, int(torch.randint(2, S - 1, (1,), generator=g))]
    cache = torch.full((B, S, 2, H, 128), float("nan"), dtype=torch.bfloat16)
    for b, p in enumerate(pos):
        cache[b, :p, 0] = kr[b, :p]
        cache[b, :p, 1] = full[b, :p, 2]
    cd = cache.to(DEV)
    qkv = torch.stack([full[b, p] for b, p in enumerate(pos)]).contiguous().to(DEV)      # (B, 3, H, 128), un-rotated
    posd = torch.tensor(pos, dtype=torch.int64, device=DEV)
    cosd, sind = cos.to(DEV), sin.to(DEV)
    _lib.check(lib.evo_decode_qkv_prep_rows(_lib.ptr(qkv), _lib.ptr(cd), _lib.ptr(cosd), _lib.ptr(sind), _lib.ptr(posd), B, H, 128, S, stream()))
    got_cache = cd.cpu()
    for b, p in enumerate(pos):
        assert (got_cache[b, p, 0] == kr[b, p]).float().mean() > 0.995 and torch.equal(got_cache[b, p, 1], full[b, p, 2])
        assert (qkv[b, 0].cpu() == qr[b, p]).float().mean() > 0.995
    scale = 1 / math.sqrt(128)
    ref = torch.stack([_attend(qr[b, p], kr[b, :p + 1], full[b, :p + 1, 2], scale) for b, p in enumerate(pos)])
    for nsplit in (1, 3, 4, 16):
        n = lib.evo_decode_attn_workspace(B, H, nsplit)
        ws = torch.empty(n, dtype=torch.uint8, device=DEV)
        out = torch.empty(B, H * 128, dtype=torch.bfloat16, device=DEV)
        _lib.check(lib.evo_decode_attn_rows(_lib.ptr(qkv), _lib.ptr(cd), _lib.ptr(out), _lib.ptr(posd), B, H, 128, S, nsplit, scale,
                                            _lib.ptr(ws), n, stream()))
        o = out.double().cpu()
        assert not torch.isnan(o).any()
        assert (o - ref).abs().max().item() <= 4 * BF16_EPS * max(1.0, ref.abs().max().item()), nsplit


@pytest.mark.parametrize("S", [640, 600])
def test_rows_kernels_with_equal_positions_are_bit_identical_to_scalar(S):
    B, H = 5, 2
    lib = _lib.lib()
    g = torch.Generator().manual_seed(5)
    cos, sin = O.rotary_tables(S, 128, dtype=torch.bfloat16)
    cosd, sind = cos.to(DEV), sin.to(DEV)
    scale = 1 / math.sqrt(128)
    for p in (0, 63, 200, S - 1):
        cache = torch.randn(B, S, 2, H, 128, generator=g).bfloat16().to(DEV)
        qkv = torch.randn(B, 3, H, 128, generator=g).bfloat16().to(DEV)
        outs = []
        for rows in (False, True):
            c, x = cache.clone(), qkv.clone()
            posd = torch.full((B,) if rows else (1,), p, dtype=torch.int64, device=DEV)
            prep = lib.evo_decode_qkv_prep_rows if rows else lib.evo_decode_qkv_prep
            attn = lib.evo_decode_attn_rows if rows else lib.evo_decode_attn
            _lib.check(prep(_lib.ptr(x), _lib.ptr(c), _lib.ptr(cosd), _lib.ptr(sind), _lib.ptr(posd), B, H, 128, S, stream()))
            res = [c, x]
            for nsplit in (1, 4):
                n = lib.evo_decode_attn_workspace(B, H, nsplit)
                ws = torch.empty(n, dtype=torch.uint8, device=DEV)
                out = torch.empty(B, H * 128, dtype=torch.bfloat16, device=DEV)
                _lib.check(attn(_lib.ptr(x), _lib.ptr(c), _lib.ptr(out), _lib.ptr(posd), B, H, 128, S, nsplit, scale, _lib.ptr(ws), n, stream()))
                res.append(out)
            outs.append([t.cpu() for t in res])
        for a, b in zip(*outs):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), p


def test_advance_positions_is_exact():
    lib = _lib.lib()
    start = torch.tensor([0, 5, 4095, 2 ** 40, 7, 300, 1], dtype=torch.int64)
    posd = start.to(DEV)
    _lib.check(lib.evo_advance_positions(_lib.ptr(posd), 7, 3, stream()))
    _lib.check(lib.evo_advance_positions(_lib.ptr(posd), 7, -1, stream()))
    assert torch.equal(posd.cpu(), start + 2)
    assert lib.evo_advance_positions(None, 0, 1, None) < 0 and b"bad batch" in lib.evo_last_error()


# ------------------------------------------------------------------ generation
def _capture_logprob_inputs(monkeypatch):
    """(kept logits, picked ids) of every batch generate() scores, in call order."""
    import evo_b200.generation as gen
    seen = []
    real = gen.logits_to_logprobs

    def spy(logits, ids, *a, **kw):
        seen.append((logits.detach().cpu().clone(), ids.detach().cpu().clone()))
        return real(logits, ids, *a, **kw)
    monkeypatch.setattr(gen, "logits_to_logprobs", spy)
    return seen


def test_same_length_prompts_are_bit_identical_to_batched_generation(monkeypatch):
    import evo_b200
    m = _tiny()
    tok = evo_b200.CharLevelTokenizer(512)
    prompts = ["ACGTTGCAACGTAC", "TTGACCAAGGTCAT", "GGGACTTACAGTCA"]
    n = 24
    m.config["max_seqlen"] = 64                 # today's path sizes its cache from the config: the ragged cache is 14 + 24 -> 64
    seen = _capture_logprob_inputs(monkeypatch)
    kw = dict(n_tokens=n, top_k=1, top_p=1.0, temperature=1.0, cached_generation=True, force_prompt_threshold=128, verbose=0, device=DEV)
    m._decode = m._loop = None
    a_txt, a_sc = evo_b200.generate(prompts, m, tok, batched=True, **kw)
    m._decode = m._loop = None
    b_txt, b_sc = evo_b200.generate(prompts, m, tok, ragged=True, **kw)
    assert len(seen) == 2
    (la, ia), (lb, ib) = seen
    assert a_txt == b_txt and a_sc == b_sc
    assert torch.equal(ia, ib)
    assert torch.equal(la.view(torch.int32), lb.view(torch.int32))
    assert la.shape == (3, n, 512)


def test_mixed_lengths_match_solo_generation(monkeypatch):
    import evo_b200
    m = _tiny()
    tok = evo_b200.CharLevelTokenizer(512)
    g = torch.Generator().manual_seed(3)
    alphabet = "ACGT"
    lengths = [65, 1, 300, 7, 63, 2, 64, 7]           # input order is not length order; length 7 twice: one group of 2 rows
    prompts = ["".join(alphabet[int(i)] for i in torch.randint(0, 4, (L,), generator=g)) for L in lengths]
    n = 16
    kw = dict(n_tokens=n, top_k=1, top_p=1.0, temperature=1.0, cached_generation=True, verbose=0, device=DEV)
    seen = _capture_logprob_inputs(monkeypatch)
    texts, scores = evo_b200.generate(prompts, m, tok, ragged=True, batch_size=64, **kw)
    assert len(seen) == 1 and len(texts) == len(prompts) == len(scores)
    rag_logits, rag_ids = seen[0]
    order = sorted(range(len(prompts)), key=lambda i: (lengths[i], i))
    worst, diverged = 0.0, 0
    for k, i in enumerate(order):
        seen.clear()
        solo_txt, _ = evo_b200.generate([prompts[i]], m, tok, batched=True, force_prompt_threshold=4096, **kw)
        s_logits, s_ids = seen[0]
        scale = max(1.0, s_logits[0].abs().max().item())
        for t in range(n):
            d = (rag_logits[k, t] - s_logits[0, t]).abs().max().item() / scale
            worst = max(worst, d)
            assert d <= TAU, (i, lengths[i], t, d)
            if rag_ids[k, t] != s_ids[0, t]:
                top2 = s_logits[0, t].topk(2).values
                assert (top2[0] - top2[1]).item() / scale <= TAU, (i, t)
                diverged += 1
                break
        else:
            assert texts[i] == solo_txt[0]
    print(f"\nragged vs solo: worst kept-logit difference {worst:.3e} of the row's max |logit|; {diverged} rows diverged at a near-tie")


def test_ragged_sampling_reproducible_and_rows_independent():
    import evo_b200
    m = _tiny(layers=3, attn=(1,))
    tok = evo_b200.CharLevelTokenizer(512)
    prompts = ["ACGTACGTAC", "TTG", "ACGTACGTAC", "GATTACAGATTACAGATTACA"]
    kw = dict(n_tokens=32, top_k=4, top_p=1.0, temperature=1.0, cached_generation=True, verbose=0, device=DEV, ragged=True)
    torch.manual_seed(11)
    a, sa = evo_b200.generate(prompts, m, tok, **kw)
    torch.manual_seed(11)
    b, sb = evo_b200.generate(prompts, m, tok, **kw)
    torch.manual_seed(12)
    c, _ = evo_b200.generate(prompts, m, tok, **kw)
    assert a == b and sa == sb
    assert a != c
    assert a[0] != a[2]                                  # same prompt, two rows of one batch: different draws
    assert all(len(x) == 32 for x in a)


def test_rejected_calls_raise_before_any_launch():
    import evo_b200
    lib = _lib.lib()
    m = _tiny(layers=2, attn=(1,))
    tok = evo_b200.CharLevelTokenizer(512)
    kw = dict(n_tokens=4, top_k=1, verbose=0, device=DEV, ragged=True)
    cpu = StripedHyena(dotdict(O.tiny_config(num_layers=2, attn_layer_idxs=(1,), hidden_size=256, num_heads=2)))
    cpu.to_bfloat16_except_poles_residues()
    m.config["max_seqlen"] = 16
    cases = [(ValueError, lambda: evo_b200.generate(["ACGT", "AC"], m, tok, cached_generation=False, **kw)),
             (ValueError, lambda: evo_b200.generate(["ACGT", "AC"], cpu, tok, cached_generation=True, **kw)),
             (ValueError, lambda: evo_b200.generate(["ACGT", ""], m, tok, cached_generation=True, **kw)),
             (_lib.EvoError, lambda: evo_b200.generate(["ACGT", "A" * 17], m, tok, cached_generation=True, **kw))]
    for exc, call in cases:
        torch.cuda.synchronize()
        lib.evo_reset_launch_count()
        with pytest.raises(exc):
            call()
        assert lib.evo_launch_count() == 0


def test_cli_prompts_csv_writes_one_output_per_prompt_in_file_order(tmp_path, monkeypatch, capsys):
    import evo_b200
    from scripts import generate as cli
    prompts = ["ACGTACGTACGTAAC", "T", "GGCATTAGC", "ACG"]
    path = tmp_path / "prompts.csv"
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["prompt", "note"])
        for i, p in enumerate(prompts):
            w.writerow([p, f"row{i}"])
    m = _tiny(layers=2, attn=(1,))

    class TinyEvo:
        def __init__(self, *a, **kw):
            self.model, self.tokenizer = m, evo_b200.CharLevelTokenizer(512)
    monkeypatch.setattr(cli, "Evo", TinyEvo)
    texts, scores = cli.main(["--prompts-csv", str(path), "--n-tokens", "8", "--top-k", "1", "--device", DEV, "--batch-size", "2", "--seed", "1"])
    assert len(texts) == len(scores) == len(prompts) and all(len(t) == 8 for t in texts)
    out = capsys.readouterr().out
    assert out.count("Prompt: ") == len(prompts)
    at = [out.index(f'Prompt: "{p}",\tOutput: "{t}",\tScore: {s}') for p, t, s in zip(prompts, texts, scores)]
    assert at == sorted(at)                              # one line per prompt, in file order
