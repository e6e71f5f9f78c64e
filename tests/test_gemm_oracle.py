"""The GEMM reference of tests/support/gemm_oracle.py, tested on the CPU: it accepts fp32 results of every summation order a
kernel may use and rejects planted faults, naming the tile they were planted in."""
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.support import gemm_oracle as GO  # noqa: E402

TILE = (128, 256)


# ------------------------------------------------------------------ fp32 accumulations in several orders
def _trunc32(x64):
    """fp64 -> fp32 rounded toward zero."""
    f = x64.float()
    over = f.double().abs() > x64.abs()
    return torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f)


def acc_fp32(a, w, order):
    """fp32 accumulation of a @ w.T over k in the given order (products exact in fp32)."""
    A, W = a.float(), w.float()
    K = a.shape[1]

    def seq(ks, trunc=False):
        s = torch.zeros(a.shape[0], w.shape[0], dtype=torch.float32)
        for k in ks:
            p = A[:, k, None] * W[None, :, k]
            s = _trunc32(s.double() + p.double()) if trunc else s + p
        return s
    if order == "sequential":
        return seq(range(K))
    if order == "reverse":
        return seq(range(K - 1, -1, -1))
    if order == "truncating":
        return seq(range(K), trunc=True)
    if order == "blocks64_pairwise":
        parts = [seq(range(k0, k0 + 64)) for k0 in range(0, K, 64)]
        while len(parts) > 1:
            parts = [parts[i] + parts[i + 1] if i + 1 < len(parts) else parts[i] for i in range(0, len(parts), 2)]
        return parts[0]
    if order == "streamk_ranges":     # ragged contiguous ranges summed on their own, then added in range order
        cuts = [0, 64 * 1, 64 * 3, K]
        out = None
        for c0, c1 in zip(cuts[:-1], cuts[1:]):
            part = seq(range(c0, c1))
            out = part if out is None else out + part
        return out
    raise ValueError(order)


def _rope(M, N, gen, rope_L=50):
    cos = torch.rand(rope_L, 64, generator=gen).bfloat16()
    sin = torch.rand(rope_L, 64, generator=gen).bfloat16()
    return dict(cos=cos, sin=sin, rope_L=rope_L, rope_cols=2 * N // 3 // 128 * 128)


def kernel_like(epi, acc32, bias, resid, rope):
    """The epilogue chain applied to an fp32 accumulator as a kernel applies it."""
    return GO.expect(epi, acc32.double(), None, 0.0, bias=bias, resid=resid, rope=rope).mid


M0, N0, K0 = 130, 768, 320        # a ragged second row-block, three column-blocks, five k-blocks


@pytest.fixture(scope="module")
def real():
    g = torch.Generator().manual_seed(1)
    a, w, bias, resid = GO.real_inputs(M0, N0, K0, g, "cpu")
    exact, S = GO.exact_sums(a, w, rows_per_chunk=50)
    return a, w, bias, resid, exact, S, _rope(M0, N0, g)


@pytest.mark.parametrize("order", ["sequential", "reverse", "truncating", "blocks64_pairwise", "streamk_ranges"])
def test_accepts_every_summation_order(real, order):
    a, w, bias, resid, exact, S, rope = real
    acc = acc_fp32(a, w, order)
    assert ((acc.double() - exact).abs() <= GO.gamma(K0) * S).all()
    for epi in GO.EPIS:
        out = kernel_like(epi, acc, bias, resid, rope)
        e = GO.expect(epi, exact, S, GO.gamma(K0), bias=bias, resid=resid, rope=rope)
        rep = GO.check(f"{epi}/{order}", out, e, (128, 128) if epi == "gelu_gate" else TILE)
        rep.assert_ok()
        assert rep.match_all > 0.97, str(rep)


def test_chunked_exact_sums_equal_one_product():
    g = torch.Generator().manual_seed(2)
    a, w, _, _ = GO.real_inputs(37, 256, 128, g, "cpu")
    e1, s1 = GO.exact_sums(a, w, rows_per_chunk=5)
    assert torch.equal(e1, a.double() @ w.double().T) and torch.equal(s1, a.double().abs() @ w.double().abs().T)


def test_integer_mode_is_exact_in_every_order():
    g = torch.Generator().manual_seed(3)
    a, w, bias, resid, e = GO.int_inputs(M0, N0, K0, g, "cpu")
    exact, S = GO.exact_sums(a, w)
    assert GO.int_preconditions(a, w, S, e, exact) > 0.5
    rope = _rope(M0, N0, g)
    for order in ("sequential", "reverse", "truncating", "streamk_ranges"):
        acc = acc_fp32(a, w, order)
        assert torch.equal(acc.double(), exact)
        for epi in GO.EPIS:
            ex = GO.expect(epi, exact, S, 0.0, bias=bias, resid=resid, rope=rope)
            out = kernel_like(epi, acc, bias, resid, rope)
            GO.check(epi, out, ex).assert_ok(floor=1.0)


# ------------------------------------------------------------------ planted faults
def _planted(rep, tile):
    assert rep.n_viol > 0, f"fault not detected: {rep}"
    assert tile in rep.bad_tiles, f"fault planted in tile {tile} but reported in {rep.bad_tiles}"
    assert "tile " + str(tile) in str(rep)


MODES = ["real", "int"]


@pytest.fixture(scope="module", params=MODES)
def data(request):
    g = torch.Generator().manual_seed(4)
    if request.param == "int":
        a, w, bias, resid, _ = GO.int_inputs(M0, N0, K0, g, "cpu", ldr=N0 + 64)
    else:
        a, w, bias, resid = GO.real_inputs(M0, N0, K0, g, "cpu", ldr=N0 + 64)
    exact, S = GO.exact_sums(a, w)
    gam = 0.0 if request.param == "int" else GO.gamma(K0)
    acc = acc_fp32(a, w, "sequential")
    return dict(a=a, w=w, bias=bias, resid_buf=resid, resid=resid[:, :N0], exact=exact, S=S, g=gam, acc=acc, rope=_rope(M0, N0, g))


def _exp(d, epi, **kw):
    return GO.expect(epi, d["exact"], d["S"], d["g"], bias=d["bias"], resid=d["resid"], rope=d["rope"], **kw)


def test_rejects_a_dropped_k_block_in_one_tile(data):
    d = data
    acc = d["acc"].clone()
    r0, c0 = 0, 256                       # tile (0, 1), k-block 2
    drop = d["a"][r0:r0 + 128, 128:192].float() @ d["w"][c0:c0 + 256, 128:192].float().T
    acc[r0:r0 + 128, c0:c0 + 256] -= drop
    for epi in ("none", "bias_resid"):
        rep = GO.check(epi, kernel_like(epi, acc, d["bias"], d["resid"], d["rope"]), _exp(d, epi))
        _planted(rep, (0, 1))
        assert rep.bad_tiles == [(0, 1)]


def test_rejects_the_bias_shifted_by_one_column_pair(data):
    d = data
    shifted = d["bias"].clone()
    shifted[512:768] = torch.roll(d["bias"][512:768], -2)    # column-block 2 reads bias[n + 2]
    rep = GO.check("bias", kernel_like("bias", d["acc"], shifted, None, None), _exp(d, "bias"))
    _planted(rep, (0, 2))
    assert set(rep.bad_tiles) == {(0, 2), (1, 2)}


def test_rejects_the_residual_read_with_ldc_instead_of_ldr(data):
    d = data
    buf = d["resid_buf"]                                # (M, ldr) with ldr = N + 64
    wrong = buf.reshape(-1)[:M0 * N0].view(M0, N0)     # row m read at m * ldc
    rep = GO.check("resid", kernel_like("resid", d["acc"], None, wrong, None), _exp(d, "resid"))
    _planted(rep, (1, 2))
    assert (0, 0) in rep.bad_tiles                      # row 0 agrees, row 1 onwards does not


def test_rejects_l1_and_l2_swapped_in_one_gate_group(data):
    d = data
    acc = d["acc"].clone()
    grp = 1                                              # W rows 256..511: output columns 128..255
    a1 = acc[:, grp * 256:grp * 256 + 128].clone()
    acc[:, grp * 256:grp * 256 + 128] = acc[:, grp * 256 + 128:grp * 256 + 256]
    acc[:, grp * 256 + 128:grp * 256 + 256] = a1
    rep = GO.check("gelu_gate", kernel_like("gelu_gate", acc, None, None, None), _exp(d, "gelu_gate"), (128, 128))
    _planted(rep, (0, 1))
    assert {t[1] for t in rep.bad_tiles} == {1}


def test_rejects_the_rotation_applied_to_v_or_one_column_too_many(data):
    d = data
    rope = d["rope"]
    more = dict(rope, rope_cols=rope["rope_cols"] + 128)     # the first v head rotated as well
    rep = GO.check("bias_rope", kernel_like("bias_rope", d["acc"], d["bias"], None, more), _exp(d, "bias_rope"))
    _planted(rep, (0, rope["rope_cols"] // 256))
    # one column too many: column rope_cols (with its partner rope_cols + 64) rotated
    out = kernel_like("bias_rope", d["acc"], d["bias"], None, rope).clone()
    out_more = kernel_like("bias_rope", d["acc"], d["bias"], None, more)
    c = rope["rope_cols"]
    out[:, c] = out_more[:, c]
    out[:, c + 64] = out_more[:, c + 64]
    rep = GO.check("bias_rope", out, _exp(d, "bias_rope"))
    _planted(rep, (0, c // 256))
    assert rep.n_viol >= M0 // 2


def test_rejects_the_ragged_block_shifted_by_one_row(data):
    d = data
    out = kernel_like("bias", d["acc"], d["bias"], None, None).clone()
    out[128:M0 - 1] = out[129:M0].clone()               # the last row-block (rows 128, 129) read one row down
    rep = GO.check("bias", out, _exp(d, "bias"))
    _planted(rep, (1, 0))
    assert all(t[0] == 1 for t in rep.bad_tiles)


def test_rejects_a_one_ulp_flip_in_integer_mode():
    g = torch.Generator().manual_seed(5)
    a, w, bias, resid, _ = GO.int_inputs(M0, N0, K0, g, "cpu")
    exact, S = GO.exact_sums(a, w)
    for epi, (r, c), tile in (("none", (129, 700), (1, 2)), ("bias_resid", (3, 5), (0, 0)), ("gelu_gate", (100, 300), (0, 2))):
        ex = GO.expect(epi, exact, S, 0.0, bias=bias, resid=resid)
        out = ex.mid.clone()
        out.view(torch.int16)[r, c] += 1                  # one bf16 ulp
        rep = GO.check(epi, out, ex, (128, 128) if epi == "gelu_gate" else TILE)
        _planted(rep, tile)
        assert rep.n_viol == 1 and rep.bad[tile][1][:2] == (r, c)


def test_nan_is_a_violation():
    g = torch.Generator().manual_seed(6)
    a, w, bias, resid = GO.real_inputs(5, 256, 64, g, "cpu")
    exact, S = GO.exact_sums(a, w)
    ex = GO.expect("none", exact, S, GO.gamma(64))
    out = ex.mid.clone()
    out[4, 255] = float("nan")
    rep = GO.check("none", out, ex)
    assert rep.bad_tiles == [(0, 0)] and rep.bad[(0, 0)][1][:2] == (4, 255)


def test_gelu_range_hull_equals_brute_force_enumeration():
    """The sparse-table hull of bf16(GELU) over a bf16 range equals the hull over every bf16 value in it, listed one by one:
    ranges around GELU's minimum (x* = -0.7518), across zero, one value wide, and long ones."""
    g = torch.Generator().manual_seed(8)
    v, _, _ = GO._gelu_tables("cpu")
    i0 = torch.randint(0, v.numel(), (400,), generator=g)
    width = torch.cat([torch.zeros(100, dtype=torch.long), torch.randint(1, 4, (100,), generator=g),
                       torch.randint(4, 3000, (200,), generator=g)])
    star = int(torch.searchsorted(v, torch.tensor(-0.7517915246935645)))
    zero = int(torch.searchsorted(v, torch.tensor(0.0)))
    i0[:20] = star - torch.arange(20)
    i0[20:30] = zero - 5
    i1 = (i0 + width).clamp(max=v.numel() - 1)
    lo, hi = GO.gelu_range_hull(v[i0].bfloat16(), v[i1].bfloat16())
    for k in range(400):
        r = v[i0[k]:i1[k] + 1]
        t = torch.cat([GO.bf(GO.gelu32(r)).float(), GO.bf(GO.gelu64(r)).float()])
        assert lo[k] == t.min() and hi[k] == t.max(), (k, r[0].item(), r[-1].item())
    gmin = GO.bf(GO.gelu64(torch.tensor(-0.7517915246935645))).float()
    lo, _ = GO.gelu_range_hull(torch.tensor([-0.8]).bfloat16(), torch.tensor([-0.7]).bfloat16())
    assert lo[0] <= gmin


def test_gelu_interval_brackets_the_minimum():
    """l1 intervals that straddle GELU's minimum: the lower end of the hull is GELU's least bf16 value, not an end's."""
    l1 = torch.tensor([[-0.8, -0.7, -0.75]], dtype=torch.float64)
    exact = torch.zeros(1, 256, dtype=torch.float64)
    exact[0, :3] = l1
    exact[0, 128:131] = 1.0
    S = torch.ones_like(exact)
    ex = GO.expect("gelu_gate", exact, S, 0.06)
    gmin = GO.bf(GO.gelu64(torch.tensor(-0.7517915246935645))).float().item()
    assert ex.lo[0, 0].float().item() <= gmin and ex.lo[0, 1].float().item() <= gmin


def test_score_bounds_are_no_looser_than_the_fixed_tolerances():
    g = torch.Generator().manual_seed(7)
    for V in (256, 512, 1024):
        x = torch.randn(64, V, generator=g).bfloat16()
        x[0, 7] = 20.0                                                   # one peaked row
        t = torch.randint(0, V, (64,), generator=g)
        lp, ent, aux = GO.score_reference(x, t)
        tl, te = GO.score_bounds(aux, V)
        assert tl.max() < 2e-5 and te.max() < 5e-5
        lp32 = torch.log_softmax(x.float(), 1).gather(1, t[:, None])[:, 0].double()
        assert ((lp32 - lp).abs() <= tl).all()
    assert math.isclose(GO.gamma(11008), 11008 * 2.0 ** -23, rel_tol=2e-3)
