"""Compact FP8 models without a GPU: the weights= / --fp8-compact plumbing, evo_fp8_dequant_rows's argument checks, and the
CUDA-only refusal of quantize_fp8(compact=True)."""
import ctypes as C
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from evo_b200 import _lib                                                               # noqa: E402


def test_weights_argument_accepts_compact_and_still_rejects_unknown_values():
    from evo_b200 import Evo
    from evo_b200.models import WEIGHTS, load_checkpoint
    assert WEIGHTS == ("bf16", "fp8", "fp8-compact")
    with pytest.raises(ValueError, match="weights='fp8_compact': should be one of bf16, fp8, fp8-compact"):
        load_checkpoint("evo-1-8k-base", random_init=True, weights="fp8_compact")
    with pytest.raises(ValueError, match="weights='compact'"):
        Evo("evo-1-8k-base", random_init=True, weights="compact")


def test_cli_flag():
    from scripts import generate, score
    g = generate.build_parser()
    assert generate.weights_arg(g.parse_args(["--fp8-compact", "--random-init"])) == "fp8-compact"
    assert generate.weights_arg(g.parse_args(["--fp8-compact", "--fp8-weights"])) == "fp8-compact"
    assert generate.weights_arg(g.parse_args(["--fp8-weights"])) == "fp8"
    assert generate.weights_arg(g.parse_args([])) == "bf16"
    s = score.build_parser()
    base = ["--input-fasta", "x.fa", "--output-tsv", "y.tsv"]
    assert score.weights_arg(s.parse_args(base + ["--fp8-compact"])) == "fp8-compact"
    assert score.weights_arg(s.parse_args(base + ["--fp8-weights"])) == "fp8"
    assert score.weights_arg(s.parse_args(base)) == "bf16"


def test_dequant_rejects_bad_arguments_before_any_launch():
    lib = _lib.lib()

    def rejected(rc, msg):
        return rc < 0 and msg in lib.evo_last_error()

    d = lambda q, e, N, K, epi, out: lib.evo_fp8_dequant_rows(q, e, N, K, epi, out, None)
    q, e, out = C.c_void_p(0x1000), C.c_void_p(0x2000), C.c_void_p(0x3000)
    assert rejected(d(q, e, 100, 64, _lib.EPI_NONE, out),
                    b"evo_fp8_dequant_rows: needs K a positive multiple of 64 and N a positive multiple of 128 (N 100, K 64)")
    assert rejected(d(q, e, 128, 64, _lib.EPI_GELU_GATE, out),
                    b"evo_fp8_dequant_rows: needs K a positive multiple of 64 and N a positive multiple of 256 (N 128, K 64)")
    assert rejected(d(q, e, 256, 100, _lib.EPI_NONE, out), b"(N 256, K 100)")
    assert rejected(d(q, e, 0, 64, _lib.EPI_NONE, out), b"(N 0, K 64)")
    assert rejected(d(q, e, 256, -64, _lib.EPI_NONE, out), b"(N 256, K -64)")
    assert rejected(d(q, e, 1 << 31, 64, _lib.EPI_NONE, out), b"evo_fp8_dequant_rows: N * K (2147483648 x 64) too large")
    assert rejected(d(None, e, 128, 64, _lib.EPI_NONE, out), b"evo_fp8_dequant_rows: W_q, W_exp and W_out are required")
    assert rejected(d(q, None, 128, 64, _lib.EPI_NONE, out), b"W_q, W_exp and W_out are required")
    assert rejected(d(q, e, 128, 64, _lib.EPI_NONE, None), b"W_q, W_exp and W_out are required")
    assert rejected(d(C.c_void_p(0x1008), e, 128, 64, _lib.EPI_NONE, out), b"evo_fp8_dequant_rows: W_q and W_out must be 16-byte aligned")
    assert rejected(d(q, e, 128, 64, _lib.EPI_NONE, C.c_void_p(0x3002)), b"W_q and W_out must be 16-byte aligned")


def test_quantize_fp8_compact_needs_the_gpu():
    from oracle import stripedhyena_oracle as O
    from evo_b200.stripedhyena import StripedHyena, dotdict
    m = StripedHyena(dotdict(O.tiny_config(num_layers=2, attn_layer_idxs=(1,), hidden_size=256, num_heads=2))).to_bfloat16_except_poles_residues()
    before = {k: v.clone() for k, v in m.state_dict().items()}
    with pytest.raises(_lib.EvoError, match="runs on CUDA"):
        m.quantize_fp8(compact=True)
    assert not m._fp8_mode and not m._fp8_compact
    assert not any(n.endswith(("_q", "_exp")) for n, _ in m.named_buffers())
    assert all(torch.equal(before[k], v) for k, v in m.state_dict().items())
