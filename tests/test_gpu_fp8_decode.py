"""FP8 weights on the GPU: the quantizer against its host reference bit for bit, evo_gemm_smallm_fp8 against evo_gemm_smallm on
the rounded weights W' bit for bit (and against the fp64 chain in exact-integer mode), and an FP8 model's decode against the same
model decoding through the bf16 kernel on W' (tokens and kept logits, bit for bit), against the oracle, and across state changes."""
import ctypes as C
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

from oracle import stripedhyena_oracle as O                                           # noqa: E402
from evo_b200 import _lib                                                              # noqa: E402
from evo_b200.stripedhyena import StripedHyena, dotdict                                # noqa: E402
from evo_b200.stripedhyena.model import fp8_layout, fp8_round_rows                    # noqa: E402
from tests.support import gemm_oracle as GO                                            # noqa: E402
from tests.test_gpu_gemm_vs_fp64 import (EPI, LINEAR, inputs, judge, nan_buf, reference,  # noqa: E402
                                         sentinels_intact, smallm)
from tests.test_gpu_decode_vs_oracle import Errors, _oracle_pair, _positions, _tokens  # noqa: E402

DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()
    yield


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.uint8)


def quantize(w, gate):
    """evo_fp8_quantize_rows on w (in place): (q bytes in the decode layout, e, status)."""
    lib = _lib.lib()
    N, K = w.shape
    epi = _lib.EPI_GELU_GATE if gate else _lib.EPI_NONE
    q = torch.full((lib.evo_fp8_weight_bytes(N, K, epi),), 0x55, dtype=torch.uint8, device=DEV)
    e = torch.zeros(N, dtype=torch.int8, device=DEV)
    st = torch.full((1,), 7, dtype=torch.int32, device=DEV)
    _lib.check(lib.evo_fp8_quantize_rows(w.data_ptr(), N, K, epi, q.data_ptr(), e.data_ptr(), st.data_ptr(), stream()), "evo_fp8_quantize_rows")
    torch.cuda.synchronize()
    return q, e, int(st.item())


def edge_weights(N, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = torch.randn(N, K, generator=g, device=DEV) / math.sqrt(K)
    w[0] = 0                                                   # all zero
    w[1, 7] = 3.0e4                                            # one huge value: the rest of the row in E4M3 subnormals
    w[2] = torch.randn(K, generator=g, device=DEV) * 2.0 ** -14 * 448
    w[2, 0] = 448 * 2.0 ** -8                                  # amax exactly 448 2^e, e = -8; others near the subnormal range
    w[3] = -0.0                                                # -0
    w[4, ::3] = -0.0
    w[5] = torch.randn(K, generator=g, device=DEV) * 2.0 ** -121
    return w.bfloat16()


# ------------------------------------------------------------------ quantizer
@pytest.mark.parametrize("N,K,gate", [(12288, 4096, False), (4096, 4096, False), (22016, 4096, True), (4096, 11008, False)])
def test_quantizer_matches_host_reference(N, K, gate):
    w = edge_weights(N, K, N + K)
    wq_ref, q_ref, e_ref = fp8_round_rows(w)
    w_dev = w.clone()
    q, e, st = quantize(w_dev, gate)
    assert st == 0
    assert torch.equal(e.cpu(), e_ref.cpu())
    assert torch.equal(bits(w_dev), bits(wq_ref))
    assert torch.equal(q, fp8_layout(q_ref, gate))
    # again on W': W' unchanged, and the copies are the host reference of W'
    q2, e2, st2 = quantize(w_dev, gate)
    assert st2 == 0 and torch.equal(bits(w_dev), bits(wq_ref))
    _, q2_ref, e2_ref = fp8_round_rows(wq_ref)
    assert torch.equal(e2.cpu(), e2_ref.cpu()) and torch.equal(q2, fp8_layout(q2_ref, gate))


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")])
def test_quantizer_refuses_non_finite_and_leaves_w(bad):
    w = edge_weights(512, 256, 1)
    w[300, 17] = bad
    w0 = w.clone()
    q, e, st = quantize(w, gate=True)
    assert st == 1
    assert torch.equal(bits(w), bits(w0))
    assert bool((q == 0x55).all())


# ------------------------------------------------------------------ evo_gemm_smallm_fp8 == evo_gemm_smallm on W'
def smallm_fp8(a, q, e, c, ldc, epi, N, bias=None, resid=None, ldr=None, ws=None):
    M, K = a.shape
    lib = _lib.lib()
    if ws is None:
        ws = torch.zeros(max(lib.evo_gemm_smallm_workspace(M, N, K, x) for x in range(5)), dtype=torch.uint8, device=DEV)
    base = _lib.GemmSmallMParams(A=a.data_ptr(), lda=a.stride(0), W=q.data_ptr(), C=c.data_ptr(), ldc=ldc,
                                 bias=bias.data_ptr() if epi in ("bias", "bias_resid") else None,
                                 residual=resid.data_ptr() if epi in ("resid", "bias_resid") else None, ldr=ldr or ldc,
                                 M=M, N=N, K=K, epilogue=EPI[epi], workspace=ws.data_ptr(), workspace_bytes=ws.numel())
    p = _lib.GemmSmallMFp8Params(base=base, W_exp=e.data_ptr())
    _lib.check(lib.evo_gemm_smallm_fp8(C.byref(p), stream()), f"evo_gemm_smallm_fp8({epi})")
    torch.cuda.synchronize()
    return ws


def case_fp8(epis, M, N, K, modes, seed, lda_pad=0, ldc_pad=0, ldr_pad=0, repeat=False, pdl=(0,)):
    lib = _lib.lib()
    for mode in modes:
        a, w, bias, resid, gam = inputs(mode, M, N, K, seed, lda=K + lda_pad, ldr=N + ldr_pad)
        for gate in sorted({epi == "gelu_gate" for epi in epis}):
            wq = w.clone()
            q, e, st = quantize(wq, gate)
            assert st == 0
            if mode == "int":                                  # integers up to 15 (times 2^-e) lie on the E4M3 grid
                assert torch.equal(bits(wq), bits(w))
                exact, S = reference(mode, a, wq)
            ws = ws_ref = None
            for epi in epis:
                if (epi == "gelu_gate") != gate:
                    continue
                n_out = N // 2 if epi == "gelu_gate" else N
                ref = nan_buf(M + 2, n_out + ldc_pad)
                ws_ref = smallm(a, wq, ref, n_out + ldc_pad, epi, bias, resid, N + ldr_pad, ws_ref)
                for level in pdl:
                    prev = lib.evo_set_pdl(level)
                    try:
                        c = nan_buf(M + 2, n_out + ldc_pad)
                        ws = smallm_fp8(a, q, e, c, n_out + ldc_pad, epi, N, bias, resid, N + ldr_pad, ws)
                        where = f"fp8 {epi} M={M} N={N} K={K} {mode} pdl={level}"
                        assert torch.equal(bits(c), bits(ref)), where
                        sentinels_intact(c, M, n_out)
                        assert int(ws[:16384].view(torch.int32).abs().sum().item()) == 0, "tile counters not back to zero"
                        if mode == "int":
                            ex = GO.expect(epi, exact, S, gam, bias=bias, resid=resid[:, :n_out])
                            judge(where, c, ex, (64, 128), mode, "streamk_gate" if gate else "streamk")
                        if repeat:
                            c2 = nan_buf(M + 2, n_out + ldc_pad)
                            smallm_fp8(a, q, e, c2, n_out + ldc_pad, epi, N, bias, resid, N + ldr_pad, ws)
                            assert torch.equal(bits(c2), bits(c)), "two launches differ"
                    finally:
                        lib.evo_set_pdl(prev)


@pytest.mark.parametrize("M", range(1, 65))
def test_fp8_every_m(M):
    case_fp8(LINEAR + ("gelu_gate",), M, 512, 256, ("int", "real"), seed=M)


@pytest.mark.parametrize("M", [1, 16, 17, 33, 64])
@pytest.mark.parametrize("epi,N,K", [("bias", 12288, 4096), ("bias_resid", 4096, 4096), ("resid", 4096, 11008), ("gelu_gate", 22016, 4096),
                                     ("none", 12288, 4096)])
def test_fp8_model_widths(M, epi, N, K):
    case_fp8((epi,), M, N, K, ("int", "real"), seed=M + N + K, pdl=(0, 4))


@pytest.mark.parametrize("N,K", [(256, 64), (512, 512), (65536, 64), (65536, 192)])
def test_fp8_grids_and_ranges(N, K):
    """fewer CTAs than SMs; ranges on tile boundaries (K = 64) and inside tiles (K = 192)"""
    case_fp8(("none", "bias_resid", "gelu_gate"), 33, N, K, ("int", "real"), seed=N + K, repeat=True, pdl=(0, 4))


def test_fp8_strides():
    case_fp8(LINEAR + ("gelu_gate",), 40, 4096, 1024, ("int", "real"), seed=3, lda_pad=64, ldc_pad=64, ldr_pad=136, repeat=True)


# ------------------------------------------------------------------ the model
def _tiny(hidden=256, heads=2, layers=4, attn=(1, 3), seed=7):
    cfg = O.tiny_config(num_layers=layers, attn_layer_idxs=attn, hidden_size=hidden, num_heads=heads)
    sd = O.random_state_dict(cfg, seed=seed)
    m = StripedHyena(dotdict(cfg))
    m.load_state_dict(sd, strict=True)
    m.to_bfloat16_except_poles_residues()
    return cfg, m.to(DEV)


def _both(m, run):
    """run() with the FP8 decode GEMMs, then with the bf16 kernel on W' (the comparator); fresh graphs for each."""
    out = []
    for bf16 in (False, True):
        m._fp8_decode_bf16 = bf16
        m._decode = m._loop = None
        out.append(run())
    m._fp8_decode_bf16 = False
    return out


def _assert_same(a, b):
    for x, y in zip(a, b):
        assert torch.equal(bits(x) if x.is_floating_point() else x, bits(y) if y.is_floating_point() else y)


def _loop_run(m, B, P, n, per_row, **kw):
    def run():
        with torch.inference_mode():
            if per_row:
                lengths = [P - 3 * (b % 8) for b in range(B)]
                g = torch.Generator().manual_seed(5)
                prompts = [(torch.randint(0, 4, (L,), generator=g) * 3 + 65).tolist() for L in lengths]
                head, ipd = m.prefill_ragged(prompts, (P + n + 63) // 64 * 64, packed=True)
                start = torch.tensor(lengths, dtype=torch.int64)
            else:
                d = m.initialize_inference_params()
                d["mha"].max_batch_size, d["mha"].max_seqlen = B, P + n + 64
                ids = _tokens(B, P, seed=P).to(DEV)
                logits, ipd = m(ids, inference_params_dict=d)
                head, start = logits[:, -1], P
            picked, kept = m.decode_loop(head.float().argmax(-1), ipd, n, start, **kw)
            return picked.clone(), kept.clone()
    return _both(m, run)


SAMPLING = dict(top_k=4, top_p=0.9, temperature=0.7, seed=1234)


@pytest.mark.parametrize("per_row", [False, True])
@pytest.mark.parametrize("sampling", [False, True])
def test_decode_loop_fp8_equals_bf16_on_rounded_weights_tiny(per_row, sampling):
    _, m = _tiny()
    m.quantize_fp8()
    f8, bf = _loop_run(m, 12, 70, 24, per_row, **(SAMPLING if sampling else {"top_k": 1}))
    _assert_same(f8, bf)


def test_decode_loop_fp8_equals_bf16_on_rounded_weights_7b_width():
    _, m = _tiny(hidden=4096, heads=32, layers=3, attn=(1,))
    m.quantize_fp8()
    for per_row, kw in ((False, {"top_k": 1}), (True, SAMPLING)):
        f8, bf = _loop_run(m, 16, 40, 12, per_row, **kw)
        _assert_same(f8, bf)


def test_per_token_steps_fp8_equal_bf16():
    _, m = _tiny()
    m.quantize_fp8()
    B, P, T = 8, 33, 6

    def run():
        d = m.initialize_inference_params()
        d["mha"].max_batch_size, d["mha"].max_seqlen = B, 128
        with torch.inference_mode():
            _, d = m(_tokens(B, P, seed=3).to(DEV), inference_params_dict=d)
            steps = _tokens(B, T, seed=4).to(DEV)
            out = []
            for k in range(T):
                d["mha"].seqlen_offset = d["hyena"].seqlen_offset = P + k
                s, d = m(steps[:, k:k + 1], inference_params_dict=d)
                out.append(s.clone())
        return (torch.cat(out, 1),)
    f8, bf = _both(m, run)
    _assert_same(f8, bf)


@pytest.mark.parametrize("share", [False, True])
def test_generate_ragged_and_shared_fp8_equal_bf16(share):
    import evo_b200
    _, m = _tiny(layers=3, attn=(1,))
    m.quantize_fp8()
    prompts = ["ACGTTGCAAC"] * 3 + ["GATTACA", "TTGACCA"]
    kw = dict(n_tokens=20, top_k=4, top_p=1.0, temperature=1.0, cached_generation=True, verbose=0, device=DEV, ragged=True, share_prompts=share)

    def run():
        torch.manual_seed(9)
        return evo_b200.generate(prompts, m, evo_b200.CharLevelTokenizer(512), **kw)
    (ta, sa), (tb, sb) = _both(m, run)
    assert ta == tb and sa == sb


def test_fp8_model_vs_oracle():
    """A quantized model against the oracle loaded with its state_dict() (W'): stateful prefill and 24 teacher-forced steps,
    at the bars of test_gpu_decode_vs_oracle.py."""
    cfg, m = _tiny()
    m.quantize_fp8()
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    B, P, T = 16, 64, 24
    prompt, steps = _tokens(B, P, seed=P), _tokens(B, T, seed=1000 + P)
    prompt[:, 0] = 0
    ref = _oracle_pair(cfg, sd, prompt, steps)
    m._decode = m._loop = None
    d = m.initialize_inference_params()
    d["mha"].max_batch_size, d["mha"].max_seqlen = B, 256
    with torch.inference_mode():
        _, d = m(prompt.to(DEV), inference_params_dict=d)
        out = []
        for k in range(T):
            d["mha"].seqlen_offset = d["hyena"].seqlen_offset = P + k
            s, d = m(steps[:, k:k + 1].to(DEV), inference_params_dict=d)
            out.append(s[:, 0].cpu())
    errs = Errors()
    errs.check_case(torch.stack(out, 1), ref["bf16"], ref["truth"], _positions([P] * B, T), "fp8 model")
    errs.check_agreement("fp8 model")


# ------------------------------------------------------------------ state handling
def _copies(m):
    c = m._ensure_fp8()
    return {(i, n): (q.clone(), e.clone()) for i in range(len(m.blocks)) for n, (q, e) in c[i].items()}


def test_state_dict_round_trip_and_reload():
    cfg, m = _tiny()
    m.quantize_fp8()
    sd = m.state_dict()
    again = {k: v.clone() for k, v in sd.items()}
    m.quantize_fp8()                                           # idempotent
    assert all(torch.equal(bits(again[k]), bits(v)) for k, v in m.state_dict().items() if v.is_floating_point())
    fresh = StripedHyena(dotdict(cfg))
    fresh.load_state_dict({k: v.cpu() for k, v in sd.items()}, strict=True)
    fresh = fresh.to_bfloat16_except_poles_residues().to(DEV).quantize_fp8()
    a, b = _copies(m), _copies(fresh)
    assert a.keys() == b.keys() and all(torch.equal(a[k][0], b[k][0]) and torch.equal(a[k][1], b[k][1]) for k in a)
    # bf16 weights loaded into an FP8 model are rounded at once
    _, plain = _tiny(seed=8)
    raw = plain.state_dict()
    m.load_state_dict(raw, strict=True)
    for name, p in m.named_parameters():
        if name.endswith(("Wqkv.weight", "out_proj.weight", "projections.weight", "out_filter_dense.weight", "mlp.w12", "mlp.w3")):
            assert torch.equal(bits(p.data), bits(fp8_round_rows(p.data)[0])), name
    assert not torch.equal(bits(m.blocks[0].mlp.w3.data), bits(plain.blocks[0].mlp.w3.data))


def test_nan_weight_refuses_and_leaves_the_model():
    _, m = _tiny()
    with torch.no_grad():
        m.blocks[2].mlp.w3[5, 9] = float("nan")
    before = {k: v.clone() for k, v in m.state_dict().items()}
    with pytest.raises(_lib.EvoError, match="not finite"):
        m.quantize_fp8()
    assert not m._fp8_mode
    for k, v in m.state_dict().items():
        assert torch.equal(bits(v) if v.is_floating_point() else v, bits(before[k]) if v.is_floating_point() else before[k]), k


def test_device_move_rebuilds_copies_and_recaptures():
    _, m = _tiny()
    m.quantize_fp8()
    f8a, _ = _loop_run(m, 4, 40, 8, False, top_k=1)
    c0 = m._fp8
    m.to("cpu")
    assert m._fp8 is None and m._loop is None
    m.to(DEV)
    f8b, bfb = _loop_run(m, 4, 40, 8, False, top_k=1)
    assert m._fp8 is not None and m._fp8 is not c0
    _assert_same(f8a, f8b)
    _assert_same(f8b, bfb)
