"""Constrained generation on the GPU: evo_sample_constrained / evo_sample_step_constrained against evo_sample / evo_sample_step
and the host automaton (evo_b200/constraints.py), then generate(ragged=True, constraints=...) and scripts.generate end to end.

Bars: with a table that allows every token the constrained kernels give the unconstrained kernels' picks bit for bit; greedy
masked picks are the first argmax among allowed tokens; sampled masked picks keep the host pipeline's kept set and its
total-variation bound on masked logits (the bound of test_gpu_generation.py); the per-row state, length and stop counter
equal the host walker's; every generated output passes the plain-string checks of tests/support/constraint_check.py."""
import csv
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

from oracle import stripedhyena_oracle as O             # noqa: E402
from evo_b200 import _lib                                # noqa: E402
from evo_b200 import constraints as K                    # noqa: E402
from evo_b200.constraints import Constraints             # noqa: E402
from evo_b200.stripedhyena import StripedHyena, dotdict  # noqa: E402
from tests.support.constraint_check import check_text   # noqa: E402

DEV = "cuda:0"
ASSEMBLY = ("GGTCTC", "CGTCTC")
STOPS = ("TAA", "TAG", "TGA")


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class _Rows:
    """Device tables + per-row arrays + the evo_constraint_params that point at them, in device memory."""

    def __init__(self, tables, states, index0=0):
        self.tables = [t.to(DEV).contiguous() for t in tables]
        self.state = torch.tensor(states, dtype=torch.int32, device=DEV)
        self.length = torch.full((len(states),), -1, dtype=torch.int64, device=DEV)
        self.n_stopped = torch.zeros(1, dtype=torch.int32, device=DEV)
        nxt, allow, stop, sym = self.tables
        p = _lib.ConstraintParams(next=nxt.data_ptr(), allow=allow.data_ptr(), stop=stop.data_ptr(), token_symbol=sym.data_ptr(),
                                  n_states=nxt.shape[0], n_tokens=sym.shape[0], state=self.state.data_ptr(), length=self.length.data_ptr(),
                                  n_stopped=self.n_stopped.data_ptr(), index0=index0)
        self.dev = torch.frombuffer(bytearray(C.string_at(C.addressof(p), C.sizeof(p))), dtype=torch.uint8).to(DEV)


def _allow_all(B):
    """One state, every token allowed (symbol t % 4), never stops."""
    tables = (torch.zeros(1, 4, dtype=torch.int32), torch.tensor([15], dtype=torch.uint8), torch.zeros(1, dtype=torch.uint8),
              (torch.arange(512) % 4).to(torch.int8))
    return _Rows(tables, [0] * B)


def _auto_rows(a, states, index0=0):
    return _Rows([torch.from_numpy(t) for t in (a.next, a.allow, a.stop, a.token_symbol)], states, index0)


def sample(lg, top_k, top_p, temperature, seed, step, rows=None):
    lg = lg.to(DEV).contiguous()
    out = torch.full((lg.shape[0],), -7, dtype=torch.long, device=DEV)
    if rows is None:
        _lib.check(_lib.lib().evo_sample(_lib.ptr(lg), _lib.ptr(out), lg.shape[0], lg.shape[1], top_k, top_p, temperature, seed, step, stream()))
    else:
        _lib.check(_lib.lib().evo_sample_constrained(_lib.ptr(lg), _lib.ptr(out), lg.shape[0], lg.shape[1], top_k, top_p, temperature, seed,
                                                     step, _lib.ptr(rows.dev), stream()))
    return out.cpu()


SETTINGS = [(1, 0.0, 1.0), (4, 1.0, 1.0), (50, 0.7, 1.0), (0, 0.5, 1.3), (8, 0.9, 0.7)]


@pytest.mark.parametrize("top_k,top_p,temperature", SETTINGS)
def test_allow_all_table_is_bit_identical_to_evo_sample(top_k, top_p, temperature):
    g = torch.Generator().manual_seed(top_k)
    lg = (torch.randn(96, 512, generator=g) * 3).bfloat16()
    lg[3] = float("nan")
    lg[4, ::3] = float("nan")
    lg[5] = float("-inf")
    for seed, step in ((1, 0), (77, 5), (2 ** 40 + 3, 123456)):
        assert torch.equal(sample(lg, top_k, top_p, temperature, seed, step), sample(lg, top_k, top_p, temperature, seed, step, _allow_all(96)))


@pytest.mark.parametrize("top_k,top_p,temperature", SETTINGS[:3])
def test_allow_all_table_step_is_bit_identical_to_evo_sample_step(top_k, top_p, temperature):
    lib = _lib.lib()
    B, V, n_forced, n_out = 40, 512, 2, 5
    g = torch.Generator().manual_seed(9)
    forced = torch.randint(0, 512, (B, n_forced), generator=g).to(DEV)
    runs = []
    for constrained in (False, True):
        picked = torch.full((B, n_out), -7, dtype=torch.long, device=DEV)
        kept = torch.full((B, n_out, V), float("nan"), device=DEV)
        x = torch.zeros(B, dtype=torch.long, device=DEV)
        lp = _lib.LoopParams(forced=forced.data_ptr(), n_forced=n_forced, forced_stride=n_forced, picked=picked.data_ptr(),
                             picked_stride=n_out, kept_logits=kept.data_ptr(), n_out=n_out, top_k=top_k, top_p=top_p,
                             temperature=temperature, seed=4242, step0=3)
        lp_dev = torch.frombuffer(bytearray(C.string_at(C.addressof(lp), C.sizeof(lp))), dtype=torch.uint8).to(DEV)
        rows = _allow_all(B)
        xs = []
        for i in range(n_forced + n_out):
            lg = (torch.randn(B, V, generator=torch.Generator().manual_seed(100 + i)) * 3).bfloat16().to(DEV)
            step = torch.tensor([i], dtype=torch.int64, device=DEV)
            if constrained:
                _lib.check(lib.evo_sample_step_constrained(_lib.ptr(lg), _lib.ptr(x), B, V, _lib.ptr(lp_dev), _lib.ptr(rows.dev), _lib.ptr(step), stream()))
            else:
                _lib.check(lib.evo_sample_step(_lib.ptr(lg), _lib.ptr(x), B, V, _lib.ptr(lp_dev), _lib.ptr(step), stream()))
            xs.append(x.cpu().clone())
        runs.append((picked.cpu(), kept.cpu(), xs))
    (p0, k0, x0), (p1, k1, x1) = runs
    assert torch.equal(p0, p1) and torch.equal(k0.view(torch.int32), k1.view(torch.int32))
    assert all(torch.equal(a, b) for a, b in zip(x0, x1))
    assert torch.equal(x0[0], forced[:, 0].cpu())


def _states(a, n, seed):
    """Row states after random prompts: every codon phase, half matches, runs."""
    rng = np.random.default_rng(seed)
    return [a.initial_state(list("".join(rng.choice(list("ACGT"), rng.integers(1, 30))).encode())) for _ in range(n)]


def test_masked_greedy_is_first_argmax_among_allowed_and_degenerate_rows_pick_allowed():
    a = K.compile(Constraints(forbid=ASSEMBLY, max_homopolymer=3, stop=STOPS, stop_in_frame=True))
    B = 128
    states = _states(a, B, 1)
    g = torch.Generator().manual_seed(2)
    lg = (torch.randn(B, 512, generator=g) * 3).bfloat16()
    lg[:, [65, 67, 71, 84]] -= 4                      # the disallowed flat tail often beats the allowed bases
    lg[7, 70:72] = lg[7, 65] = lg[7, 67] = lg[7, 84] = 30.0          # ties: the first allowed maximum wins
    lg[8] = float("nan")
    lg[9] = float("-inf")
    lg[10, [65, 67, 71, 84]] = float("nan")          # every allowed entry NaN, the rest finite
    lg[11, 84] = float("nan")
    for top_k, top_p, temperature in SETTINGS:
        got = sample(lg, top_k, top_p, temperature, 5, 0, _auto_rows(a, states))
        for r in range(B):
            ok = a.allowed_tokens(states[r])
            assert ok[got[r]], (r, int(got[r]))
            if top_k == 1:
                m = a.masked(lg[r].float(), states[r])
                allowed = m[torch.from_numpy(ok)]
                if torch.isnan(allowed).all() or torch.isinf(allowed).all():
                    assert got[r] == int(np.flatnonzero(ok)[0])              # no allowed entry carries weight: allowed rank 0
                else:
                    want = torch.where(torch.isnan(m), float("-inf"), m).argmax()
                    assert got[r] == want, (r, int(got[r]), int(want))


@pytest.mark.parametrize("top_k,top_p,temperature", [(4, 1.0, 1.0), (2, 1.0, 1.0), (0, 0.9, 1.0), (50, 0.9, 1.3)])
def test_masked_draws_match_host_pipeline_on_masked_logits(top_k, top_p, temperature):
    from tests.test_gpu_generation import host_pipeline_probs
    a = K.compile(Constraints(forbid=("GGTCTC",), both_strands=False, max_homopolymer=3))
    s = a.initial_state(b"AGGTCT")                   # C is disallowed here
    row = torch.randn(512, generator=torch.Generator().manual_seed(3)).bfloat16()
    row[[65, 67, 71, 84]] += torch.tensor([2.0, 4.0, 1.5, 2.5]).bfloat16()
    want = host_pipeline_probs(a.masked(row, s), top_k, top_p, temperature).double()
    N = 40000
    draws = sample(row[None].expand(N, -1), top_k, top_p, temperature, 777, 3, _auto_rows(a, [s] * N))
    got = torch.bincount(draws, minlength=512).double() / N
    support = want > 0
    assert got[~support].sum().item() <= 2e-3
    tv = 0.5 * (got - want).abs().sum().item()
    noise = 0.5 * 0.8 * torch.sqrt(want * (1 - want) / N).sum().item()
    assert tv <= 2.0 * noise + 0.01, (tv, noise)
    assert int(support.sum()) >= 2 and got[67] == 0


def test_step_bookkeeping_equals_the_host_walker():
    lib = _lib.lib()
    a = K.compile(Constraints(forbid=ASSEMBLY, max_homopolymer=4, stop=STOPS, stop_in_frame=True))
    B, V, n_out, index0 = 64, 512, 60, 1
    states = _states(a, B, 4)
    rows = _auto_rows(a, states, index0)
    picked = torch.full((B, n_out), -7, dtype=torch.long, device=DEV)
    kept = torch.full((B, n_out, V), float("nan"), device=DEV)
    x = torch.zeros(B, dtype=torch.long, device=DEV)
    lp = _lib.LoopParams(forced=None, n_forced=0, forced_stride=0, picked=picked.data_ptr(), picked_stride=n_out, kept_logits=kept.data_ptr(),
                         n_out=n_out, top_k=0, top_p=1.0, temperature=1.0, seed=99, step0=0)
    lp_dev = torch.frombuffer(bytearray(C.string_at(C.addressof(lp), C.sizeof(lp))), dtype=torch.uint8).to(DEV)
    xs = []
    for i in range(n_out):
        lg = torch.randn(B, V, generator=torch.Generator().manual_seed(i)).bfloat16().to(DEV)
        step = torch.tensor([i], dtype=torch.int64, device=DEV)
        _lib.check(lib.evo_sample_step_constrained(_lib.ptr(lg), _lib.ptr(x), B, V, _lib.ptr(lp_dev), _lib.ptr(rows.dev), _lib.ptr(step), stream()))
        xs.append(x.cpu().clone())
    picked, kept, length = picked.cpu(), kept.cpu(), rows.length.cpu()
    n_stop = 0
    for r in range(B):
        walked, n, ok = a.walk(states[r], picked[r].tolist())
        assert ok, r
        if n is None:
            assert length[r] == -1 and len(walked) == n_out and rows.state[r].item() == walked[-1]
        else:
            n_stop += 1
            assert length[r] == index0 + n and rows.state[r].item() == walked[-1]
            assert (picked[r, n:] == -7).all() and torch.isnan(kept[r, n:]).all()      # nothing written past the stop
            assert all(int(xs[i][r]) == int(picked[r, n - 1]) for i in range(n - 1, n_out))   # keeps feeding its last token
    assert rows.n_stopped.item() == n_stop and 0 < n_stop < B


# ------------------------------------------------------------------ end to end
def _tiny(hidden=256, heads=2, layers=4, attn=(1, 3), seed=7):
    cfg = O.tiny_config(num_layers=layers, attn_layer_idxs=attn, hidden_size=hidden, num_heads=heads)
    sd = O.random_state_dict(cfg, seed=seed)
    m = StripedHyena(dotdict(cfg))
    m.load_state_dict(sd, strict=True)
    m.to_bfloat16_except_poles_residues()
    return m.to(DEV)


def _spy(monkeypatch):
    import evo_b200.generation as gen
    seen = []
    real = gen.logits_to_logprobs

    def spy(logits, ids, *a, **kw):
        seen.append((logits.detach().cpu().clone(), ids.detach().cpu().clone()))
        return real(logits, ids, *a, **kw)
    monkeypatch.setattr(gen, "logits_to_logprobs", spy)
    return seen


PROMPTS = ["ATGAAACGTCTGGTC", "ATGCC", "GGGGACGTAGGTCT", "ATGTTTGAGACG", "CATG", "ATGACCGGTCTAAGGCA", "A"]
C_FULL = Constraints(forbid=ASSEMBLY, max_homopolymer=3, stop=STOPS, stop_in_frame=True)


def _check_outputs(prompts, texts, c, n_tokens):
    for p, t in zip(prompts, texts):
        ok, stop = check_text(p, t, c)
        assert ok, (p, t)
        assert (stop == len(t)) if stop is not None else (len(t) == n_tokens), (p, t, stop)


@pytest.mark.parametrize("share", [False, True])
def test_greedy_generation_obeys_constraints_and_picks_the_allowed_argmax(monkeypatch, share):
    import evo_b200
    from evo_b200.frontend import ragged_batches, shared_batches
    m = _tiny()
    tok = evo_b200.CharLevelTokenizer(512)
    prompts = PROMPTS + PROMPTS[:3] if share else PROMPTS
    n = 48
    seen = _spy(monkeypatch)
    texts, scores = evo_b200.generate(prompts, m, tok, n_tokens=n, top_k=1, cached_generation=True, verbose=0, device=DEV, ragged=True,
                                      share_prompts=share, batch_size=4, constraints=C_FULL)
    _check_outputs(prompts, texts, C_FULL, n)
    assert any(len(t) < n for t in texts)
    a = K.compile(C_FULL)
    ids = [tok.tokenize(p) for p in prompts]
    order = ([r for rows, _ in ragged_batches([len(t) for t in ids], n, 4) for r in rows] if not share else
             [r for parts, _, _ in shared_batches(ids, n, 4)[1] for _, rr in parts for r in rr])
    flat = [(lg[j], pk[j]) for lg, pk in seen for j in range(lg.shape[0])]
    assert len(flat) == len(prompts)
    for (lg, pk), r in zip(flat, order):                   # the batch order back to the input order
        L = len(texts[r])
        assert tok.detokenize(pk[:L].tolist()) == texts[r]
        s = a.initial_state(ids[r])
        for k in range(L):
            ok = torch.from_numpy(a.allowed_tokens(s))
            want = int(torch.where(ok, lg[k], float("-inf")).argmax())
            assert int(pk[k]) == want, (r, k)
            s = int(a.next[s, a.token_symbol[want]])
        lp = torch.log_softmax(lg[:L].float(), -1)
        mean = float(np.mean([lp[k, pk[k + 1]].item() for k in range(L - 1)])) if L > 1 else float("nan")
        assert scores[r] == pytest.approx(mean, rel=1e-5, abs=1e-6) or (L == 1 and scores[r] != scores[r])


def test_sampled_shared_prompts_at_the_7b_width_obey_constraints():
    import evo_b200
    m = _tiny(hidden=4096, heads=32, layers=3, attn=(1,))
    tok = evo_b200.CharLevelTokenizer(512)
    prompts = ["ATGGCGTCTCAGG"] * 5 + ["ATGAAAAAC"] * 3
    torch.manual_seed(0)
    texts, _ = evo_b200.generate(prompts, m, tok, n_tokens=40, top_k=4, temperature=1.0, cached_generation=True, verbose=0, device=DEV,
                                 ragged=True, share_prompts=True, prepend_bos=True, constraints=C_FULL)
    _check_outputs(prompts, texts, C_FULL, 40)
    assert len(set(texts[:5])) > 1


def test_early_exit_runs_fewer_steps():
    import evo_b200
    lib = _lib.lib()
    m = _tiny(layers=2, attn=(1,))
    tok = evo_b200.CharLevelTokenizer(512)
    prompts = ["ACGTN", "GGN", "TTTTAN"]
    every_2mer = tuple(x + y for x in "ACGT" for y in "ACGT")
    kw = dict(top_k=1, cached_generation=True, verbose=0, device=DEV, ragged=True)

    def launches(n, c):
        torch.cuda.synchronize()
        lib.evo_reset_launch_count()
        out = evo_b200.generate(prompts, m, tok, n_tokens=n, constraints=c, **kw)
        torch.cuda.synchronize()
        return lib.evo_launch_count(), out
    evo_b200.generate(prompts, m, tok, n_tokens=200, constraints=Constraints(stop=every_2mer), **kw)     # capture the step first
    short, (texts, _) = launches(200, Constraints(stop=every_2mer))                # every row stops at its second token
    assert [len(t) for t in texts] == [2, 2, 2]
    full, (texts, _) = launches(200, Constraints())
    assert [len(t) for t in texts] == [200] * 3
    assert short * 5 < full, (short, full)
    # every row stops on the first pick: no loop at all
    one, (texts, _) = launches(200, Constraints(stop=tuple("ACGT")))
    assert [len(t) for t in texts] == [1, 1, 1] and one < short


def test_rejected_calls_raise_before_any_launch():
    import evo_b200
    lib = _lib.lib()
    m = _tiny(layers=2, attn=(1,))
    tok = evo_b200.CharLevelTokenizer(512)
    cases = [lambda: evo_b200.generate(["ACGT"], m, tok, n_tokens=4, cached_generation=True, verbose=0, device=DEV, constraints=C_FULL),
             lambda: evo_b200.generate(["ACGT", "AAAA"], m, tok, n_tokens=4, cached_generation=True, verbose=0, device=DEV, ragged=True,
                                       constraints=Constraints(forbid=("AA", "AC", "AG", "AT", "CA", "CC", "CG", "GA", "GC")))]
    for call in cases:
        torch.cuda.synchronize()
        lib.evo_reset_launch_count()
        with pytest.raises(ValueError):
            call()
        assert lib.evo_launch_count() == 0


def test_cli_constraint_flags(tmp_path, monkeypatch, capsys):
    import evo_b200
    from scripts import generate as cli
    prompts = ["ATGGGTCT", "ATGCCCC", "GACGAGACC"]
    path = tmp_path / "prompts.csv"
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["prompt"])
        for p in prompts:
            w.writerow([p])
    m = _tiny(layers=2, attn=(1,))

    class TinyEvo:
        def __init__(self, *a, **kw):
            self.model, self.tokenizer = m, evo_b200.CharLevelTokenizer(512)
    monkeypatch.setattr(cli, "Evo", TinyEvo)
    texts, _ = cli.main(["--prompts-csv", str(path), "--n-tokens", "30", "--top-k", "4", "--device", DEV, "--seed", "3",
                         "--forbid", "GGTCTC,CGTCTC", "--max-homopolymer", "3", "--stop", "TAA,TAG,TGA", "--stop-in-frame"])
    _check_outputs(prompts, texts, C_FULL, 30)
    out = capsys.readouterr().out
    assert all(f'Prompt: "{p}",\tOutput: "{t}"' in out for p, t in zip(prompts, texts))
