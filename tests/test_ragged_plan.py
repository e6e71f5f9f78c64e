"""Ragged-generation planning and argument checks that need no GPU: batch order, cuts, KV-cache lengths, the exact-length
groups being adjacent rows, and the calls generate(ragged=True) refuses before touching the device."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from evo_b200.frontend import length_buckets, ragged_batches  # noqa: E402


def test_rows_sorted_by_length_then_index_and_cut_at_batch_size():
    lengths = [5, 3, 5, 9, 1, 3, 5]
    plan = ragged_batches(lengths, n_new=10, batch_size=3)
    assert [rows for rows, _ in plan] == [[4, 1, 5], [0, 2, 6], [3]]
    assert [c for _, c in plan] == [64, 64, 64]
    assert sorted(r for rows, _ in plan for r in rows) == list(range(len(lengths)))


def test_cache_length_is_longest_prompt_plus_new_tokens_rounded_to_64():
    assert ragged_batches([64], 0)[0][1] == 64
    assert ragged_batches([64], 1)[0][1] == 128
    assert ragged_batches([4096, 256], 256)[0][1] == 4352
    assert ragged_batches([100, 7], 28, align=1)[0][1] == 128


def test_equal_lengths_are_adjacent_in_every_batch():
    import random
    rng = random.Random(4)
    lengths = [rng.choice([1, 2, 7, 63, 64, 65, 300]) for _ in range(200)]
    for rows, _ in ragged_batches(lengths, n_new=8, batch_size=64):
        assert len(rows) <= 64
        for idx in length_buckets([lengths[r] * "A" for r in rows], batch_size=len(rows), mode="exact"):
            assert idx == list(range(idx[0], idx[0] + len(idx)))


def test_bad_batch_size_and_empty_list():
    with pytest.raises(ValueError):
        ragged_batches([3], 1, batch_size=0)
    assert ragged_batches([], 5) == []


def test_generate_refuses_before_touching_a_device():
    import evo_b200
    from evo_b200.stripedhyena import StripedHyena, dotdict
    from oracle import stripedhyena_oracle as O
    m = StripedHyena(dotdict(O.tiny_config(num_layers=2, attn_layer_idxs=(1,), hidden_size=256, num_heads=2)))
    m.to_bfloat16_except_poles_residues()
    tok = evo_b200.CharLevelTokenizer(512)
    kw = dict(n_tokens=4, verbose=0, device="cpu", ragged=True)
    with pytest.raises(ValueError, match="cached_generation"):
        evo_b200.generate(["ACGT", "AC"], m, tok, cached_generation=False, **kw)
    with pytest.raises(ValueError, match="CUDA"):
        evo_b200.generate(["ACGT", "AC"], m, tok, cached_generation=True, **kw)
    with pytest.raises(ValueError, match="batch_size"):
        evo_b200.generate(["ACGT", "AC"], m, tok, cached_generation=True, batch_size=0, **kw)


def test_cli_parses_prompts_csv_and_batch_size():
    from scripts.generate import build_parser
    a = build_parser().parse_args(["--prompts-csv", "p.csv", "--batch-size", "16"])
    assert a.prompts_csv == "p.csv" and a.batch_size == 16
    a = build_parser().parse_args([])
    assert a.prompts_csv is None and a.batch_size == 64
