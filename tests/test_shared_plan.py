"""The shared-prompt generation planner (frontend.shared_batches), on the CPU: groups of identical prompts keep their rows
contiguous, batches hold at most batch_size rows, every distinct prompt is prefilled exactly once, and the rows map back to
input order."""
import random

import pytest

from evo_b200.frontend import shared_batches


def _check(prompts, batch_size, n_new=100):
    groups, batches = shared_batches(prompts, n_new, batch_size)
    # groups: identical prompts together, first-seen order, every input index once
    assert sorted(i for g in groups for i in g) == list(range(len(prompts)))
    for g in groups:
        assert len({prompts[i] if isinstance(prompts[i], str) else tuple(prompts[i]) for i in g}) == 1
    firsts = [g[0] for g in groups]
    assert firsts == sorted(firsts)
    assert len({prompts[g[0]] if isinstance(prompts[g[0]], str) else tuple(prompts[g[0]]) for g in groups}) == len(groups)
    prefilled, rows_seen, seen_groups = [], [], set()
    for parts, fresh, suffix_len in batches:
        assert 1 <= sum(len(r) for _, r in parts) <= batch_size
        assert suffix_len % 64 == 0 and suffix_len >= n_new
        gs = [g for g, _ in parts]
        assert len(gs) == len(set(gs))                          # a group's rows are one contiguous run in the batch
        assert gs == sorted(gs)
        assert fresh == [g for g in gs if g not in seen_groups]  # prefilled before its first batch, never again
        seen_groups.update(gs)
        prefilled += fresh
        for g, r in parts:
            rows_seen += r
    assert sorted(prefilled) == list(range(len(groups)))
    assert sorted(rows_seen) == list(range(len(prompts)))      # every input row decoded once: input order is restorable
    # within a group the rows run in input order across batches
    for g, idx in enumerate(groups):
        assert [r for r in rows_seen if r in set(idx)] == idx
    # every batch but the last is full
    assert all(sum(len(r) for _, r in parts) == batch_size for parts, _, _ in batches[:-1])
    return groups, batches


def test_interleaved_prompts_group_in_first_seen_order():
    groups, batches = _check(["a", "b", "a", "c", "b", "a"], 64)
    assert groups == [[0, 2, 5], [1, 4], [3]]
    assert batches == [([(0, [0, 2, 5]), (1, [1, 4]), (2, [3])], [0, 1, 2], 128)]


def test_large_group_spans_batches_and_is_prefilled_once():
    groups, batches = _check(["P"] * 10 + ["Q"] * 3, 4, n_new=64)
    assert [len(b[0]) for b in batches] == [1, 1, 2, 1]
    assert [b[1] for b in batches] == [[0], [], [1], []]
    assert batches[2][0] == [(0, [8, 9]), (1, [10, 11])]
    assert batches[0][2] == 64


def test_token_sequences_and_random_mixes():
    _check([[1, 2, 3], [1, 2], [1, 2, 3], [4]], 2)
    rng = random.Random(5)
    for _ in range(200):
        pool = ["".join(rng.choice("ACGT") for _ in range(rng.randint(1, 4))) for _ in range(rng.randint(1, 6))]
        prompts = [rng.choice(pool) for _ in range(rng.randint(1, 40))]
        _check(prompts, rng.randint(1, 9))


def test_bad_batch_size():
    with pytest.raises(ValueError):
        shared_batches(["a"], 4, 0)
