"""Host side of the packed variable-length forward, without a GPU: the packing planner (frontend.packs) and the host check
of cu_seqlens (stripedhyena.model.packed_lengths) that every packed call runs before anything is launched."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from evo_b200 import _lib                                     # noqa: E402
from evo_b200.frontend import packs                           # noqa: E402
from evo_b200.stripedhyena.model import packed_lengths        # noqa: E402


def test_packs_cover_every_row_once_within_the_budget():
    lengths = [40, 7, 40, 129, 1, 41, 300, 8, 99, 99]
    plan = packs(lengths, max_tokens=200)
    rows = [r for p, _ in plan for r in p]
    assert sorted(rows) == list(range(len(lengths)))
    for p, cu in plan:
        assert cu[0] == 0 and len(cu) == len(p) + 1
        assert [b - a for a, b in zip(cu, cu[1:])] == [lengths[r] + 1 for r in p]         # BOS included
        assert cu[-1] <= 200 or len(p) == 1                                              # only a lone sequence may exceed it
        assert [lengths[r] for r in p] == sorted((lengths[r] for r in p), reverse=True)  # longest first inside a pack
    assert plan[0] == ([6], [0, 301])                                                    # 301 tokens > 200: a pack of its own


def test_packs_fill_greedily_in_length_order():
    assert packs([3, 3, 3, 3], max_tokens=8) == [([0, 1], [0, 4, 8]), ([2, 3], [0, 4, 8])]
    assert packs([5, 1, 2], max_tokens=100, bos=0) == [([0, 2, 1], [0, 5, 7, 8])]
    assert packs([], max_tokens=10) == []
    with pytest.raises(ValueError):
        packs([1], max_tokens=0)


def test_packed_lengths_accepts_valid_offsets():
    assert packed_lengths([0, 5, 8], 8) == [5, 3]
    assert packed_lengths(torch.tensor([0, 1]), 1) == [1]


@pytest.mark.parametrize("cu,T", [([0, 5, 5, 8], 8),      # empty sequence
                                  ([0, 6, 5, 8], 8),      # not increasing
                                  ([0, 5, 7], 8),         # does not end at T
                                  ([1, 5, 8], 8),         # does not start at 0
                                  ([0], 0), ([], 0)])
def test_packed_lengths_rejects_malformed_offsets(cu, T):
    with pytest.raises(_lib.EvoError):
        packed_lengths(cu, T)


def test_packed_calls_on_a_cpu_model_raise_before_any_launch():
    from oracle import stripedhyena_oracle as O
    from evo_b200.stripedhyena import StripedHyena, dotdict
    cfg = O.tiny_config(num_layers=2, attn_layer_idxs=(1,), hidden_size=256, num_heads=2)
    m = StripedHyena(dotdict(cfg))
    m.to_bfloat16_except_poles_residues()
    ids = torch.full((8,), 65, dtype=torch.long)
    for call in (lambda: m.forward_packed(ids, [0, 5, 8]), lambda: m.score_tokens_packed(ids, [0, 5, 8]),
                 lambda: m.prefill_ragged([[65] * 5, [65] * 3], 16, packed=True)):
        with pytest.raises(_lib.EvoError, match="CUDA"):
            call()
    m4 = StripedHyena(dotdict(O.tiny_config(num_layers=2, attn_layer_idxs=(1,), hidden_size=256, num_heads=4)))
    with pytest.raises(_lib.EvoError, match="head_dim 128"):
        m4.forward_packed(ids, [0, 5, 8])
