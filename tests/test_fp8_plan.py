"""FP8 weights without a GPU: the host reference of the rounding (fp8_round_rows), the decode layout (fp8_layout), the new
entry points' argument checks, and the weights= / --fp8-weights plumbing."""
import ctypes as C
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from evo_b200 import _lib                                                               # noqa: E402
from evo_b200.stripedhyena.model import fp8_layout, fp8_round_rows, fp8_unlayout      # noqa: E402

E4M3_MAX = 448.0


def _edge_rows(K, g):
    """Rows that test the rounding's corners, then ordinary ones."""
    rows = [torch.zeros(K),                                            # all zero: e = 0, q = 0
            torch.randn(K, generator=g) * 1e-3,                        # one huge value: the rest falls into E4M3 subnormals
            torch.full((K,), -0.0),                                    # -0
            (torch.rand(K, generator=g) * 2 - 1) * E4M3_MAX * 2.0 ** -10,
            torch.randn(K, generator=g) * 2.0 ** -120]                 # tiny: the exponent floor
    rows[1][3] = 3.0e4
    rows[3][5] = E4M3_MAX * 2.0 ** -10                                 # amax exactly 448 2^e
    rows[4][0] = 2.0 ** -118
    return torch.stack(rows + [torch.randn(K, generator=g) / K ** 0.5 for _ in range(123)]).bfloat16()


def test_rounding_is_exact_in_bf16_and_idempotent():
    g = torch.Generator().manual_seed(0)
    w = _edge_rows(256, g)
    wq, q, e = fp8_round_rows(w)
    assert wq.dtype == torch.bfloat16 and q.dtype == torch.float8_e4m3fn and e.dtype == torch.int8
    # W' = q 2^e exactly: the bf16 value times 2^-e is q, with nothing lost on either side
    assert torch.equal(torch.ldexp(wq.double(), -e[:, None].double()), q.double())
    assert q.float().abs().max() <= E4M3_MAX
    assert e[0] == 0 and not q[0].float().any() and not wq[0].float().any()
    assert e[3] == -10 and q[3, 5].float() == E4M3_MAX
    assert e[4] == -124
    assert torch.equal(wq[2].view(torch.int16), w[2].view(torch.int16))          # -0 stays -0
    # nearest: no E4M3 value of the row's scale is closer to w than q
    x = torch.ldexp(w.double(), -e[:, None].double())
    assert ((x - q.double()).abs() <= x.abs() * 2.0 ** -4 + 2.0 ** -10 + 1e-30).all()
    # idempotent: W' rounds to itself
    wq2, q2, e2 = fp8_round_rows(wq)
    assert torch.equal(wq2.view(torch.int16), wq.view(torch.int16))
    assert torch.equal(torch.ldexp(q2.double(), e2[:, None].double()), torch.ldexp(q.double(), e[:, None].double()))


def test_exponent_is_the_least_that_fits():
    """e = ceil(log2(amax / 448)): 448 2^e >= amax > 448 2^(e-1), checked on every bf16 amax of one binade and its edges."""
    a = torch.arange(0x3f80, 0x4001, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)     # [1, 2]
    w = torch.zeros(a.numel(), 64, dtype=torch.bfloat16)
    w[:, 0] = a
    _, _, e = fp8_round_rows(w)
    lim = E4M3_MAX * torch.ldexp(torch.ones(a.numel(), dtype=torch.float64), e.double())
    assert (lim >= a.double()).all() and (lim / 2 < a.double()).all()


@pytest.mark.parametrize("N,K,gate", [(256, 64, False), (384, 192, False), (512, 128, True), (768, 256, True)])
def test_layout_round_trips(N, K, gate):
    g = torch.Generator().manual_seed(N + K)
    q = torch.randint(0, 256, (N, K), generator=g, dtype=torch.int32).to(torch.uint8).view(torch.float8_e4m3fn)
    flat = fp8_layout(q, gate)
    assert flat.shape == (N * K,) and flat.dtype == torch.uint8
    assert torch.equal(fp8_unlayout(flat, N, K, gate).view(torch.uint8), q.view(torch.uint8))


def test_layout_places_each_thread_fragment_as_the_kernel_reads_it():
    """Thread t of warpgroup cw reads 16 bytes at block + cw*4096 + (t/32)*1024 + (t%32)*16 (k16 steps 0, 1) and 512 bytes on
    (steps 2, 3); byte 2*reg + j of a step is the register a[reg]'s pair element j: rows r0 = 16*(t/32) + (t%32)/4 (+8 for
    a[1], a[3]), columns 2*(t%4) + j (+8 for a[2], a[3])."""
    N, K = 256, 128
    n_idx = torch.arange(N)[:, None].expand(N, K)
    k_idx = torch.arange(K)[None, :].expand(N, K)
    code = (n_idx * K + k_idx).to(torch.int64)
    # the layout of the code matrix, through the same permutation on int64
    from evo_b200.stripedhyena.model import _FP8_ORDER, _fp8_view
    flat = code.reshape(_fp8_view(N, K, 1)).permute(_FP8_ORDER).reshape(-1)
    for tile, kb, cw, t, half, step, reg, j in [(0, 0, 0, 0, 0, 0, 0, 0), (1, 1, 1, 37, 1, 1, 3, 1), (0, 1, 0, 127, 1, 0, 2, 0),
                                                 (1, 0, 1, 64, 0, 1, 1, 1)]:
        off = (tile * (K // 64) + kb) * 8192 + cw * 4096 + (t // 32) * 1024 + half * 512 + (t % 32) * 16 + step * 8 + reg * 2 + j
        n = tile * 128 + cw * 64 + 16 * (t // 32) + (t % 32) // 4 + 8 * (reg % 2)
        k = kb * 64 + (2 * half + step) * 16 + 8 * (reg // 2) + 2 * (t % 4) + j
        assert int(flat[off]) == n * K + k, (tile, kb, cw, t, half, step, reg, j)


def test_entry_points_reject_bad_arguments_before_any_launch():
    lib = _lib.lib()

    def rejected(rc, msg):
        return rc < 0 and msg in lib.evo_last_error()

    assert lib.evo_fp8_weight_bytes(256, 4096, _lib.EPI_NONE) == 256 * 4096
    assert lib.evo_fp8_weight_bytes(128, 64, _lib.EPI_NONE) == 128 * 64
    assert lib.evo_fp8_weight_bytes(128, 64, _lib.EPI_GELU_GATE) == 0 and b"multiple of 256" in lib.evo_last_error()
    assert lib.evo_fp8_weight_bytes(256, 100, _lib.EPI_NONE) == 0 and b"multiple of 64" in lib.evo_last_error()
    q = lambda *a: lib.evo_fp8_quantize_rows(*a)
    assert rejected(q(C.c_void_p(0x1000), 100, 64, 0, C.c_void_p(0x2000), C.c_void_p(0x3000), C.c_void_p(0x4000), None),
                    b"evo_fp8_quantize_rows: needs K a positive multiple of 64 and N a positive multiple of 128 (N 100, K 64)")
    assert rejected(q(None, 128, 64, 0, C.c_void_p(0x2000), C.c_void_p(0x3000), C.c_void_p(0x4000), None),
                    b"W, W_q, W_exp and status are required")
    assert rejected(q(C.c_void_p(0x1008), 128, 64, 0, C.c_void_p(0x2000), C.c_void_p(0x3000), C.c_void_p(0x4000), None),
                    b"must be 16-byte aligned")

    def fp8(**kw):
        f = dict(A=0x1000, lda=64, W=0x2000, C=0x3000, ldc=256, M=4, N=256, K=64, epilogue=0)
        f.update(kw)
        w_exp = f.pop("W_exp", 0x4000)
        return _lib.GemmSmallMFp8Params(base=_lib.GemmSmallMParams(**f), W_exp=w_exp)

    g = lambda p: lib.evo_gemm_smallm_fp8(C.byref(p), None)
    assert rejected(g(fp8(M=65)), b"evo_gemm_smallm_fp8: M (65) must be in [0, 64]")
    assert rejected(g(fp8(K=100)), b"evo_gemm_smallm_fp8: K (100) must be a positive multiple of 64")
    assert rejected(g(fp8(N=384)), b"evo_gemm_smallm_fp8: N (384) must be a multiple of 256")
    assert rejected(g(fp8(lda=60)), b"evo_gemm_smallm_fp8: lda must be a multiple of 8")
    assert rejected(g(fp8(W=0x2008)), b"evo_gemm_smallm_fp8: A and W must be 16-byte aligned")
    assert rejected(g(fp8(epilogue=_lib.EPI_BIAS)), b"evo_gemm_smallm_fp8: bias epilogue without bias")
    assert rejected(g(fp8(epilogue=_lib.EPI_RESID)), b"evo_gemm_smallm_fp8: residual epilogue without residual")
    assert rejected(g(fp8(W_exp=None)), b"evo_gemm_smallm_fp8: W_exp is required")
    assert rejected(g(fp8(epilogue=7)), b"evo_gemm_smallm_fp8: unknown epilogue 7")
    assert g(fp8(M=0)) == 0                                                     # nothing to do, nothing launched


def test_weights_argument_is_validated_before_loading():
    from evo_b200 import Evo
    from evo_b200.models import load_checkpoint
    with pytest.raises(ValueError, match="weights='int8': should be one of bf16, fp8"):
        load_checkpoint("evo-1-8k-base", random_init=True, weights="int8")
    with pytest.raises(ValueError, match="weights='FP8'"):
        Evo("evo-1-8k-base", random_init=True, weights="FP8")


def test_quantize_fp8_needs_the_gpu():
    from oracle import stripedhyena_oracle as O
    from evo_b200.stripedhyena import StripedHyena, dotdict
    m = StripedHyena(dotdict(O.tiny_config(num_layers=2, attn_layer_idxs=(1,), hidden_size=256, num_heads=2))).to_bfloat16_except_poles_residues()
    before = {k: v.clone() for k, v in m.state_dict().items()}
    with pytest.raises(_lib.EvoError, match="runs on CUDA"):
        m.quantize_fp8()
    assert not m._fp8_mode and all(torch.equal(before[k], v) for k, v in m.state_dict().items())


def test_cli_flags():
    from scripts import generate, score
    assert generate.build_parser().parse_args(["--fp8-weights", "--random-init"]).fp8_weights
    assert not generate.build_parser().parse_args([]).fp8_weights
    a = score.build_parser().parse_args(["--input-fasta", "x.fa", "--output-tsv", "y.tsv", "--fp8-weights"])
    assert a.fp8_weights
