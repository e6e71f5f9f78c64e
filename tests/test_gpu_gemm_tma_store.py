"""The 256-column GEMM tile writes C through shared memory and TMA stores, with the residual fetched by TMA.  Every epilogue
must give the same bits as the per-thread direct stores (EVO_B200_GEMM_DIRECT_STORE=1, read per launch): ragged last
row-blocks (rows >= M clipped by the store), the residual aliasing C, row strides wider than the output, the Wqkv rotary
layout, and more tiles than SMs so each CTA reuses its staging buffers."""
import ctypes as C
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

from evo_b200 import _lib  # noqa: E402

DEV = "cuda:0"
EPIS = {"none": _lib.EPI_NONE, "bias": _lib.EPI_BIAS, "bias_resid": _lib.EPI_BIAS_RESID, "resid": _lib.EPI_RESID,
        "gelu_gate": _lib.EPI_GELU_GATE, "bias_rope": _lib.EPI_BIAS_ROPE}


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def run(a, w, bias, out, resid, M, N, K, epi, ldc, ldr, rope, direct, monkeypatch):
    if direct:
        monkeypatch.setenv("EVO_B200_GEMM_DIRECT_STORE", "1")
    else:
        monkeypatch.delenv("EVO_B200_GEMM_DIRECT_STORE", raising=False)
    p = _lib.GemmParams(A=a.data_ptr(), lda=K, W=w.data_ptr(), C=out.data_ptr(), ldc=ldc,
                        bias=bias.data_ptr() if epi in (_lib.EPI_BIAS, _lib.EPI_BIAS_RESID, _lib.EPI_BIAS_ROPE) else None,
                        residual=resid.data_ptr() if resid is not None else None, ldr=ldr, M=M, N=N, K=K, epilogue=epi, variant=0, **rope)
    _lib.check(_lib.lib().evo_gemm(C.byref(p), stream()), "evo_gemm")
    torch.cuda.synchronize()


def case(epi_name, M, N, K, pad_c, pad_r, alias, monkeypatch):
    epi = EPIS[epi_name]
    g = torch.Generator(device=DEV).manual_seed(M + N + K + epi)
    n_out = N // 2 if epi == _lib.EPI_GELU_GATE else N
    ldc, ldr = n_out + pad_c, n_out + pad_r
    a = (torch.randn(M, K, device=DEV, generator=g) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=DEV, generator=g) / K ** 0.5).bfloat16()
    bias = (torch.randn(N, device=DEV, generator=g) * 0.2).bfloat16()
    rope = {}
    if epi == _lib.EPI_BIAS_ROPE:     # [q | k | v] heads of 128; q and k rotated, tables with a period shorter than M
        L = 1000
        cos, sin = (torch.rand(L, 64, device=DEV, generator=g).bfloat16() for _ in range(2))
        rope = dict(rope_cos=cos.data_ptr(), rope_sin=sin.data_ptr(), rope_L=L, rope_cols=2 * N // 3)
        rope["_keep"] = (cos, sin)
    resid0 = torch.randn(M, ldr, device=DEV, generator=g).bfloat16() if epi in (_lib.EPI_BIAS_RESID, _lib.EPI_RESID) else None
    keep = rope.pop("_keep", None)  # noqa: F841  (the tables outlive the launches)
    outs = []
    for direct in (True, False):
        if alias:      # C is the residual stream itself (out-proj, l3): ldc == ldr
            out = resid0.clone()
            resid = out
        else:
            out = torch.full((M, ldc), float("nan"), dtype=torch.bfloat16, device=DEV)
            resid = resid0
        run(a, w, bias, out, resid, M, N, K, epi, ldc if not alias else ldr, ldr, rope, direct, monkeypatch)
        outs.append(out)
    d, t = outs
    assert torch.equal(d.view(torch.int16), t.view(torch.int16)), f"{epi_name}: TMA-store output differs from the direct stores"
    if not alias and pad_c:
        assert torch.isnan(t[:, n_out:].float()).all(), "columns beyond the output width were written"


@pytest.mark.parametrize("epi_name", list(EPIS))
@pytest.mark.parametrize("M", [8193, 65544 - 37, 300])
def test_tma_store_matches_direct(epi_name, M, monkeypatch):
    N = 768 if epi_name == "bias_rope" else 1024
    case(epi_name, M, N, 256, 0, 0, False, monkeypatch)


@pytest.mark.parametrize("epi_name", list(EPIS))
def test_tma_store_wide_rows(epi_name, monkeypatch):
    """ldc (and ldr) wider than the output: the padding columns stay untouched."""
    N = 768 if epi_name == "bias_rope" else 512
    case(epi_name, 4100, N, 192, 64, 72, False, monkeypatch)


@pytest.mark.parametrize("epi_name", ["bias_resid", "resid"])
@pytest.mark.parametrize("M", [8193, 65544 - 37])
def test_tma_store_residual_aliases_c(epi_name, M, monkeypatch):
    case(epi_name, M, 1024, 512, 0, 8, True, monkeypatch)


@pytest.mark.parametrize("K", [64, 4096])
def test_tma_store_k_extremes(K, monkeypatch):
    """one k-block (the staging wait and the residual fetch share the first k-block) and a long mainloop"""
    case("bias_resid", 2 * 128 * 132 + 5, 512, K, 0, 0, False, monkeypatch)
    case("gelu_gate", 2 * 128 * 132 + 5, 512, K, 0, 0, False, monkeypatch)
