"""Variant scoring on the CPU: the plan (first difference, resume point, packs, stride budget), the variant helpers, and the
model's argument checks that must raise before anything is launched."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from evo_b200 import _lib, apply_mutations, saturation_variants  # noqa: E402
from evo_b200.variants import (checkpoint_bytes, choose_stride, first_difference, plan_variants,  # noqa: E402
                               reference_prefix_sums, resume_point, score_variants)

REF = "ACGTTGCAAC"


def test_first_difference():
    assert first_difference(REF, REF) == len(REF) + 1                  # equal: no difference, f = len(ids_v)
    assert first_difference(REF, REF[:4]) == 5                          # a prefix of the reference
    assert first_difference(REF, "C" + REF[1:]) == 1                    # substitution at nucleotide 1 = ids index 1
    assert first_difference(REF, REF[:6] + "A" + REF[7:]) == 7
    assert first_difference(REF, REF[:3] + "G" + REF[3:]) == 4          # insertion
    assert first_difference(REF, REF[:3] + REF[5:]) == 4                # deletion: ids differ from index 4 on
    assert first_difference(REF, REF + "GG") == len(REF) + 1            # extension: the first new token
    assert first_difference(REF, REF[:-1] + REF[-1]) == len(REF) + 1


def test_resume_point_rule():
    for s in (128, 256):
        assert resume_point(1, s) == 0
        assert resume_point(s, s) == 0                                  # row s - 1 predicts ids[s]: needs rows from < s
        assert resume_point(s + 1, s) == s                              # row s is the first after checkpoint s
        assert resume_point(3 * s + 5, s) == 3 * s
    for f in range(1, 700):
        c = resume_point(f, 128)
        assert c % 128 == 0 and c <= f - 1 < c + 128


def test_packs_cover_every_variant_once_within_max_tokens():
    rng = np.random.default_rng(0)
    ref = "".join(rng.choice(list("ACGT"), size=700))
    var = [(0, s) for _, s in saturation_variants(ref)[::7]] + [(0, ref), (0, ref[:300]), (0, ref + "A"), (0, ref[:100] + ref[101:])]
    f, c, packs = plan_variants([ref], var, 128, 2000)
    seen = [k for idx, _ in packs for k in idx]
    differ = [k for k in range(len(var)) if f[k] < len(var[k][1]) + 1]
    assert sorted(seen) == differ and len(set(seen)) == len(seen)
    assert len(var) - 2 == len(differ)                                  # the equal and the prefix variant need no pass
    for idx, cu in packs:
        assert cu[0] == 0 and len(cu) == len(idx) + 1
        assert cu[-1] <= 2000 or len(idx) == 1
        for j, k in enumerate(idx):
            assert cu[j + 1] - cu[j] == len(var[k][1]) + 1 - c[k]     # ids_v[c_v:]
    # the token arithmetic of a saturation scan: about L/2 + s/2 tokens per variant instead of L + 1
    L = len(ref)
    f, c, _ = plan_variants([ref], [(0, s) for _, s in saturation_variants(ref)], 128, 1 << 17)
    mean = np.mean([L + 1 - cv for cv in c])
    assert abs(mean - (L / 2 + 64)) < 64


def test_prefix_sum_plus_suffix_sum_is_the_full_sum():
    rng = np.random.default_rng(1)
    lp = rng.standard_normal(1000).astype(np.float32)
    p = reference_prefix_sums(lp)
    assert p[0] == 0 and p.shape == (1001,)
    for c in (0, 1, 128, 999, 1000):
        assert abs(p[c] + lp[c:].sum(dtype=np.float64) - lp.sum(dtype=np.float64)) < 1e-9


def test_saturation_order_and_count():
    v = saturation_variants(REF)
    assert len(v) == 3 * len(REF)
    assert [m for m, _ in v[:6]] == ["A1C", "A1G", "A1T", "C2A", "C2G", "C2T"]
    for m, s in v:
        assert apply_mutations(REF, m) == s and len(s) == len(REF)
        assert sum(a != b for a, b in zip(REF, s)) == 1
    assert len(set(s for _, s in v)) == len(v)


def test_mutation_strings():
    assert apply_mutations(REF, "A1G") == "G" + REF[1:]
    assert apply_mutations(REF, "A1G:C10T") == "G" + REF[1:-1] + "T"
    assert apply_mutations(REF, "") == REF
    for bad in ("C1G", "A11G", "A0G", "AG", "A1G:X3A", "1G"):
        with pytest.raises(ValueError):
            apply_mutations(REF, bad)
    with pytest.raises(ValueError, match="has 'A' at position 1"):
        apply_mutations(REF, "T1G")


def test_stride_budget_rule():
    cfg = {"hidden_size": 4096, "state_size": 8, "num_layers": 32, "attn_layer_idxs": [8, 16, 24]}
    per = checkpoint_bytes(cfg)
    assert per == 29 * (4096 * 8 * 2 * 4 + 2 * 3 * 4096 * 2)            # ~9.0 MB at the 7B config
    assert choose_stride([131072], 128, per, budget=10 << 30) == 128   # 1024 checkpoints = 9.3 GB
    s = choose_stride([131072], 128, per, budget=4 << 30)
    assert s % 128 == 0 and (131072 // s) * per <= 4 << 30 < (131072 // (s - 128)) * per
    assert choose_stride([100], 128, per, budget=0) == 128             # no checkpoint at all fits any budget
    for bad in (0, 100, -128, 128.0, True):
        with pytest.raises(ValueError):
            choose_stride([1000], bad, per)


def test_rejected_inputs_raise_before_any_work():
    class NoModel:                                                       # any call on it would fail the test
        config = {"hidden_size": 256, "state_size": 8, "num_layers": 4, "attn_layer_idxs": [1, 3]}

        def __getattr__(self, name):
            raise AssertionError(f"model.{name} reached")
    m = NoModel()
    for call in (lambda: score_variants(REF, [REF], m, None, reduce_method="max"),
                 lambda: score_variants(REF, [REF], m, None, checkpoint_stride=100),
                 lambda: score_variants(REF, [REF], m, None, max_tokens=0),
                 lambda: score_variants([REF, REF], [REF], m, None),           # several references need (index, sequence)
                 lambda: score_variants(REF, [(1, REF)], m, None),
                 lambda: score_variants(REF, [""], m, None),
                 lambda: score_variants("", [REF], m, None),
                 lambda: score_variants(REF, ["ACGé"], m, None)):
        with pytest.raises(ValueError):
            call()


def test_model_checks_raise_before_any_launch():
    """StripedHyena.prefill_checkpoints / score_tokens_resumed reject bad strides, indices and prefix lengths on the host;
    on a GPU-less box nothing could have been launched, and the check has to come first for the error to be an EvoError."""
    from oracle import stripedhyena_oracle as O
    from evo_b200.stripedhyena import StripedHyena, dotdict
    from evo_b200.stripedhyena.model import PrefixCheckpoints
    if torch.cuda.is_available():
        pytest.skip("the GPU tests check the launch count")
    cfg = O.tiny_config(num_layers=4, attn_layer_idxs=(1, 3), hidden_size=256, num_heads=2)
    m = StripedHyena(dotdict(cfg))
    ids = torch.zeros(300, dtype=torch.long)
    for stride in (0, 100, -128, 64):
        with pytest.raises(_lib.EvoError, match="multiple of 128"):
            m.prefill_checkpoints(ids, [0, 300], stride)
    ck = PrefixCheckpoints(logprobs=None, lengths=[300, 200], cu=[0, 300, 500], stride=128, base=[0, 2, 3], state={}, halo={}, kv={})
    ids = torch.zeros(10, dtype=torch.long)
    for args, msg in ((([0], [2], [0]), "outside the 2 references"),
                      (([-1], [0], [128]), "zero start"),
                      (([0], [0], [300]), "not below"),
                      (([1], [0], [128]), "not reference 0's checkpoint"),
                      (([2], [0], [128]), "not reference 0's checkpoint"),
                      (([3], [1], [128]), "not reference 1's checkpoint"),
                      (([0, 0], [0], [128]), "one entry per sequence")):
        with pytest.raises(_lib.EvoError, match=msg):
            m.score_tokens_resumed(ck, ids, [0, 10], *args)
    cfg64 = O.tiny_config(num_layers=2, attn_layer_idxs=(1,), hidden_size=256, num_heads=4)
    with pytest.raises(_lib.EvoError, match="head_dim 128"):
        StripedHyena(dotdict(cfg64)).prefill_checkpoints(torch.zeros(300, dtype=torch.long), [0, 300], 128)
