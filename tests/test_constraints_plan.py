"""Constrained generation on the host: the compiled automaton (evo_b200/constraints.py) against a predicate written directly on
strings (tests/support/constraint_check.py) for every ACGT continuation up to length 9 of prompts that end in runs, half
matches, a BOS or an N and in each codon phase; liveness of every reachable state; the rejected inputs; and the CLI flags."""
import os
import random
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from evo_b200 import constraints as K                  # noqa: E402
from evo_b200.constraints import Constraints            # noqa: E402
from tests.support.constraint_check import check_text  # noqa: E402

ASSEMBLY = ("GGTCTC", "CGTCTC")
STOPS = ("TAA", "TAG", "TGA")
CASES = {
    "acgt_only": Constraints(),
    "forbid_hp": Constraints(forbid=ASSEMBLY, max_homopolymer=4),
    "forbid_one_strand": Constraints(forbid=("GGTCTC",), both_strands=False, max_homopolymer=3),
    "stop_any_frame": Constraints(forbid=("GGTCTC",), stop=STOPS),
    "stop_in_frame": Constraints(forbid=ASSEMBLY, max_homopolymer=4, stop=STOPS, stop_in_frame=True),
}
# prompt tails: a run into the limit, half-matched motifs on both strands, a non-ACGT byte, each codon phase
PROMPTS = ["", "AAAA", "ACGGTC", "TTGAGAC", "GGTCTCA", "ACGNGG", "ATG", "ATGC", "ATGCA", "CCCCCGTCT", "TA"]


def _ids(prompt, bos=False):
    return ([K.BOS] if bos else []) + list(prompt.encode())


def _compare_tree(a, c, prompt, bos, depth):
    """Walk every ACGT continuation of `prompt` up to `depth` through the automaton and the string predicate at once."""
    s0 = a.initial_state(_ids(prompt, bos))
    stack = [("", s0)]
    nodes = 0
    while stack:
        text, s = stack.pop()
        for ch in "ACGT":
            t = text + ch
            ok, stop = check_text(prompt + text, ch, c)         # only the new last character is judged
            allowed = bool(a.allow[s] >> K.SYMBOL[ch] & 1)
            assert allowed == ok, (prompt, bos, t)
            if not ok:
                continue
            s2 = int(a.next[s, K.SYMBOL[ch]])
            assert bool(a.stop[s2]) == (stop is not None), (prompt, bos, t)
            nodes += 1
            if stop is None and len(t) < depth:
                stack.append((t, s2))
    return nodes


@pytest.mark.parametrize("name", sorted(CASES))
def test_automaton_equals_string_predicate_on_every_continuation(name):
    c = CASES[name]
    a = K.compile(c)
    for prompt in PROMPTS:
        for bos in (False, True):
            assert _compare_tree(a, c, prompt, bos, 6) > 0
    if name == "stop_in_frame":                       # length 9 on one tail per codon phase, run-in and half-matched
        for prompt in ("CCCCCGTCT", "TTGAGAC", "ACGNGGTC"):
            assert _compare_tree(a, c, prompt, False, 9) > 0


def test_full_walks_agree_with_the_string_predicate():
    """Whole strings (not just last characters): the walker's verdict and stop index equal check_text's."""
    rng = random.Random(5)
    for name, c in CASES.items():
        a = K.compile(c)
        for _ in range(300):
            prompt = "".join(rng.choice("ACGTN") for _ in range(rng.randint(0, 12)))
            text = "".join(rng.choice("ACGT") for _ in range(rng.randint(1, 14)))
            s0 = a.initial_state(list(prompt.encode()))
            states, length, ok = a.walk(s0, text.encode())
            want_ok, want_stop = check_text(prompt, text, c)
            assert ok == want_ok and (not ok or length == want_stop), (name, prompt, text)


def test_phase_counts_from_the_first_nucleotide_after_a_bos():
    c = Constraints(stop=("TAA",), stop_in_frame=True)
    a = K.compile(c)
    for bos in (False, True):
        for pre, expect in (("ATG", 3), ("ATGA", None), ("AT", None), ("ATGCCC", 3)):
            _, length, ok = a.walk(a.initial_state(_ids(pre, bos)), b"TAAC")
            assert ok and length == expect, (pre, bos)
        s = a.initial_state(_ids("ATGCC", bos))
        assert a.walk(s, b"CTAA")[1] == 4                       # ATGCC|C TAA: TAA starts at position 6
    # an N advances the phase like any prompt byte
    assert a.walk(a.initial_state(list(b"ANG")), b"TAA")[1] == 3


def test_every_reachable_state_can_continue_and_a_long_random_walk_never_sticks():
    for c in CASES.values():
        a = K.compile(c)
        seen, todo = set(), [a.initial_state(_ids(p)) for p in PROMPTS]
        while todo:
            s = todo.pop()
            if s in seen:
                continue
            seen.add(s)
            assert a.allow[s] != 0 or a.stop[s], s
            if a.stop[s]:
                continue
            todo += [int(a.next[s, x]) for x in range(4) if a.allow[s] >> x & 1]
        rng = np.random.default_rng(0)
        s = a.initial_state(b"")
        for _ in range(100_000):
            choices = [x for x in range(4) if a.allow[s] >> x & 1]
            assert choices
            s = int(a.next[s, rng.choice(choices)])
            if a.stop[s]:
                s = a.initial_state(b"ACG"[: rng.integers(0, 4)])


def test_dead_ends_are_trimmed():
    """Every two-letter word starting with A is forbidden (on both strands), so an A, which violates nothing itself, can never
    be continued: it is not allowed."""
    a = K.compile(Constraints(forbid=("AA", "AC", "AG", "AT")))
    s = a.initial_state(b"G")
    assert not a.allow[s] & 1
    assert a.allowed_tokens(s)[ord("C")] and not a.allowed_tokens(s)[ord("A")]


def test_masked_and_allowed_tokens():
    import torch
    a = K.compile(Constraints(forbid=("GGTCTC",), both_strands=False))
    s = a.initial_state(b"AGGTCT")
    ok = a.allowed_tokens(s)
    assert ok.sum() == 3 and not ok[ord("C")] and all(ok[ord(x)] for x in "AGT")
    lg = torch.randn(512)
    m = a.masked(lg, s)
    assert torch.equal(torch.isinf(m), torch.from_numpy(~ok))
    assert torch.equal(m[torch.from_numpy(ok)], lg[torch.from_numpy(ok)])


@pytest.mark.parametrize("kw", [dict(forbid=("",)), dict(forbid=("ACGN",)), dict(stop=("TAX",)), dict(max_homopolymer=0),
                                dict(max_homopolymer=-2), dict(forbid=("TAA",), stop=("TAAG",)),
                                dict(forbid=("CTTA",), stop=("TAAG",)),           # the reverse complement of TAAG
                                dict(max_homopolymer=2, stop=("TAAAG",))])
def test_rejected_descriptions(kw):
    with pytest.raises(ValueError):
        K.compile(Constraints(**kw))


def test_rejected_prompt_and_state_cap(monkeypatch):
    a = K.compile(Constraints(forbid=("A", "C")))            # with both strands every base is forbidden
    with pytest.raises(ValueError, match="no continuation"):
        a.initial_state(b"ACGT")
    monkeypatch.setattr(K, "MAX_STATES", 50)
    with pytest.raises(ValueError, match="more than 50"):
        K.compile(Constraints(max_homopolymer=20))


def test_generate_rejects_constraints_on_the_reference_path():
    import torch
    from evo_b200 import CharLevelTokenizer, generate

    class Untouchable(torch.nn.Module):
        def eval(self):
            raise AssertionError("touched the model")
    with pytest.raises(ValueError, match="ragged=True"):
        generate(["ACGT"], Untouchable(), CharLevelTokenizer(512), constraints=Constraints(), ragged=False)


def test_cli_flags_build_constraints():
    from scripts import generate as cli
    p = cli.build_parser()
    assert cli.constraints_arg(p.parse_args([])) is None
    args = p.parse_args(["--prompts-csv", "x.csv", "--forbid", "GGTCTC,CGTCTC", "--max-homopolymer", "10", "--stop", "TAA,TAG,TGA",
                         "--stop-in-frame"])
    assert cli.constraints_arg(args) == Constraints(forbid=ASSEMBLY, max_homopolymer=10, stop=STOPS, stop_in_frame=True)
    assert cli.constraints_arg(p.parse_args(["--share-prompts", "--acgt-only"])) == Constraints()
    with pytest.raises(SystemExit):
        cli.constraints_arg(p.parse_args(["--acgt-only"]))          # the per-prompt reference path takes no constraints
