"""Every GEMM path against the fp64 reference of tests/support/gemm_oracle.py, element by element, with failures named by tile.

Two input modes run on every case:
  * exact-integer: A in [-15, 15], W in [-15, 15] 2^-e, bias and residual on power-of-two grids.  Every fp32 partial sum is
    exact whatever the order or split, so the expected bits are chain(exact) and the test asserts equality: a dropped, doubled or
    misplaced partial sum, or a moved rounding point, fails in the tile it happens in;
  * realistic: normal inputs at the model's scales.  Every element lies in its rigorous interval (fp32 accumulation in any order
    stays within gamma S of exact), and every tile's fraction of elements equal to chain(exact) is at least the path's floor
    (FLOORS, measured on an H100 80GB HBM3 SXM at 700 W, the measured minimum beside each).

Paths: evo_gemm's 256-column tile (TMA stores and direct stores, variants 0 and 1), its 64-column tile (variants 2 and 3),
evo_gemm_smallm (stream-K), peer-scattered output, and evo_unembed_score."""
import ctypes as C
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

from evo_b200 import _lib                              # noqa: E402
from evo_b200.stripedhyena import StripedHyena         # noqa: E402
from tests.support import gemm_oracle as GO            # noqa: E402

DEV = "cuda:0"
EPI = {"none": _lib.EPI_NONE, "bias": _lib.EPI_BIAS, "bias_resid": _lib.EPI_BIAS_RESID, "resid": _lib.EPI_RESID,
       "gelu_gate": _lib.EPI_GELU_GATE, "bias_rope": _lib.EPI_BIAS_ROPE}
LINEAR = ("none", "bias", "resid", "bias_resid")
MODES = ("int", "real")
# least per-tile exact-match fraction in realistic mode, per path (measured minimum in the comment)
FLOORS = {"tile256": 0.98,         # measured 0.9902
          "tile256_gate": 0.98,    # measured 0.9886
          "tile64": 0.94,          # measured 0.9531 (64-column tiles of M = 1 rows: one flip costs 1/64)
          "streamk": 0.97,         # measured 0.9844
          "streamk_gate": 0.97}    # measured 0.9844
SEEN = {}          # path -> least per-tile match seen; "gamma_used" -> largest fraction of gamma S an output proves


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()
    yield
    print("\nper-tile exact-match minima and gamma S used:", {k: round(v, 4) for k, v in sorted(SEEN.items())})


def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def inputs(mode, M, N, K, seed, lda=None, ldr=None):
    """(a, w, bias, resid, gamma): a (M, K) viewed out of an (M, lda) tensor whose extra columns hold junk."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    lda = lda or K
    if mode == "int":
        a, w, bias, resid, _ = GO.int_inputs(M, N, lda, g, DEV, ldr=ldr)
        e = GO.int_exponent(K)
        w = (torch.randint(-15, 16, (N, K), generator=g, device=DEV).float() * 2.0 ** -e).bfloat16()
        bias = (torch.randint(-128, 129, (N,), generator=g, device=DEV).float() * 2.0 ** -e).bfloat16()
        gam = 0.0
    else:
        a, w, bias, resid = GO.real_inputs(M, N, lda, g, DEV, ldr=ldr)
        w = (torch.randn(N, K, generator=g, device=DEV) / math.sqrt(K)).bfloat16()
        gam = GO.gamma(K)
    return a[:, :K], w, bias, resid, gam


def reference(mode, a, w):
    exact, S = GO.exact_sums(a, w)
    if mode == "int":
        e = GO.int_exponent(a.shape[1])
        assert GO.int_preconditions(a, w, S, e, exact) > 0.4, "integer-mode sums are mostly bf16-representable"
    return exact, S


def judge(name, out, ex, tile, mode, path):
    rep = GO.check(name, out, ex, tile)
    if mode == "int":
        rep.assert_ok(floor=1.0)
    else:
        rep.assert_ok(floor=FLOORS[path])
        SEEN[path] = min(SEEN.get(path, 1.0), rep.match_min)
        SEEN["gamma_used"] = max(SEEN.get("gamma_used", 0.0), GO.gamma_used(out[:ex.lo.shape[0], :ex.lo.shape[1]], ex))
    return rep


def rope_setup(M, N, seed, rope_L=None, rope_cols=None):
    g = torch.Generator(device=DEV).manual_seed(seed + 99)
    L = rope_L or M
    cos = (torch.rand(L, 64, generator=g, device=DEV) * 2 - 1).bfloat16()
    sin = (torch.rand(L, 64, generator=g, device=DEV) * 2 - 1).bfloat16()
    return dict(cos=cos, sin=sin, rope_L=L, rope_cols=rope_cols if rope_cols is not None else 2 * N // 3 // 128 * 128)


class _Env:
    """evo_gemm reads its store-path and tile-walk switches per launch: set them around one launch, then restore them."""
    def __init__(self, values):
        self.values = values

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.values}
        os.environ.update(self.values)

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def tile_walk(M, N, K):
    """The 256-column tile's default walk as the host picks it (evo_gemm's rasterisation estimate in csrc/gemm_wgmma.cu):
    (raster_n, blocks per group, groups) -- raster_n = 1 groups column-blocks and sweeps row-blocks, 0 the reverse."""
    a_blk, w_blk, a_tot, w_tot, budget = 128 * K * 2.0, 256 * K * 2.0, M * K * 2.0, N * K * 2.0, 16e6
    mb, nb = -(-M // 128), N // 256

    def balanced(blocks, gmax):
        groups = (blocks + gmax - 1) // gmax
        last = blocks - (groups - 1) * gmax
        if groups == 1 or 2 * last >= gmax:
            return gmax
        fewer = (blocks + groups - 2) // (groups - 1)
        return fewer if 5 * fewer <= 6 * gmax else (blocks + groups - 1) // groups
    gm = balanced(mb, int(max(1.0, min(mb, budget / a_blk))))
    gn = balanced(nb, int(max(1.0, min(nb, budget / w_blk))))
    rn = w_tot + a_tot * math.ceil(nb / gn) < a_tot + w_tot * math.ceil(mb / gm)
    g = gn if rn else gm
    return int(rn), g, -(-(nb if rn else mb) // g)


def evo_gemm(a, w, c, ldc, epi, variant=0, bias=None, resid=None, ldr=None, rope=None, direct=False, peers=None, N=None, walk=None):
    M, K = a.shape
    kw = {}
    if rope is not None:
        kw = dict(rope_cos=rope["cos"].data_ptr(), rope_sin=rope["sin"].data_ptr(), rope_L=rope["rope_L"], rope_cols=rope["rope_cols"])
    if peers is not None:
        kw.update(peers)
    p = _lib.GemmParams(A=a.data_ptr(), lda=a.stride(0), W=w.data_ptr(), C=c.data_ptr() if c is not None else None, ldc=ldc,
                        bias=bias.data_ptr() if epi in ("bias", "bias_resid", "bias_rope") else None,
                        residual=resid.data_ptr() if epi in ("resid", "bias_resid") else None, ldr=ldr or ldc,
                        M=M, N=N or w.shape[0], K=K, epilogue=EPI[epi], variant=variant, **kw)
    with _Env(dict({"EVO_B200_GEMM_DIRECT_STORE": "1" if direct else "0"}, **(walk or {}))):
        _lib.check(_lib.lib().evo_gemm(C.byref(p), stream()), f"evo_gemm({epi}, variant {variant})")
    torch.cuda.synchronize()


def nan_buf(rows, cols):
    return torch.full((rows, cols), float("nan"), dtype=torch.bfloat16, device=DEV)


def sentinels_intact(buf, M, n_out):
    assert torch.isnan(buf[M:].float()).all(), "rows past M were written"
    assert torch.isnan(buf[:, n_out:].float()).all(), "columns past the output width were written"


# ------------------------------------------------------------------ the 256-column tile
def case256(epi, M, N, K, mode, seed, lda_pad=0, ldc_pad=0, ldr_pad=0, alias=False, rope_L=None, variants=(0,), walk=None,
            rope=None):
    n_out = N // 2 if epi == "gelu_gate" else N
    ldc, ldr = n_out + ldc_pad, n_out + (ldc_pad if alias else ldr_pad)
    a, w, bias, resid, gam = inputs(mode, M, N, K, seed, lda=K + lda_pad, ldr=ldr)
    if epi == "bias_rope" and rope is None:
        rope = rope_setup(M, N, seed, rope_L)
    exact, S = reference(mode, a, w)
    ex = GO.expect(epi, exact, S, gam, bias=bias, resid=resid[:, :n_out], rope=rope)
    tile = (128, 128) if epi == "gelu_gate" else (128, 256)
    path = "tile256_gate" if epi == "gelu_gate" else "tile256"
    outs = []
    for variant in variants:
        for direct in (False, True):
            if alias:
                c = torch.cat([resid, nan_buf(3, ldr)])        # C is the residual stream itself
                r = c
            else:
                c, r = nan_buf(M + 3, ldc), resid
            evo_gemm(a, w, c, ldc, epi, variant, bias, r, ldr, rope, direct, walk=walk)
            tag = f"{epi} M={M} N={N} K={K} {mode} variant={variant} {'direct' if direct else 'TMA'}-store walk={walk or tile_walk(M, N, K)}"
            judge(tag, c, ex, tile, mode, path)
            if alias:
                assert torch.isnan(c[M:].float()).all() and torch.equal(c[:M, n_out:], resid[:, n_out:])
            else:
                sentinels_intact(c, M, n_out)
            outs.append(c[:M, :n_out])
    for o in outs[1:]:
        assert torch.equal(o.view(torch.int16), outs[0].view(torch.int16)), f"{epi}: store paths or variants differ"


@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("M", [1, 127, 128, 129])
def test_tile256_rows(epi, M):
    for mode in MODES:
        case256(epi, M, 768, 320, mode, seed=M)


@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("extra", [-1, 0, 1, "2n+1"])
def test_tile256_tile_counts(epi, extra):
    """n_sm - 1, n_sm, n_sm + 1 and 2 n_sm + 1 tiles (one column-block): a partial wave, exactly one, one tile more, and CTAs
    that take a third tile; the last row-block is ragged."""
    t = 2 * n_sm() + 1 if extra == "2n+1" else n_sm() + extra
    for mode in MODES:
        case256(epi, 128 * t - 5, 256, 128, mode, seed=t)


@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("K", [64, 128, 192, 320, 4096, 11008])
def test_tile256_k(epi, K):
    """fewer k-blocks than the 3- or 4-stage ring, counts that are not multiples of it, and 172 k-blocks"""
    for mode in MODES:
        case256(epi, 300, 512, K, mode, seed=K, variants=(0, 1) if K == 320 else (0,))


@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("shape", ["tall", "wide", "m_groups", "n_groups"])
def test_tile256_tile_walks(epi, shape):
    """The default walks as the host picks them (tile_walk records each choice): many more row-blocks than column-blocks and the
    reverse at K = 128, where both operands fit the L2 slab and one group of row-blocks covers the matrix; at K = 4096 groups of
    10 row-blocks over 19 (column-blocks swept inside each), and groups of 7 column-blocks over 11 (row-blocks swept inside
    each), the last group short in both."""
    (M, N, K), walk = {"tall": ((5123, 512, 128), (0, 41, 1)), "wide": ((200, 10240, 128), (0, 2, 1)),
                       "m_groups": ((2411, 2304, 4096), (0, 10, 2)), "n_groups": ((2411, 2816, 4096), (1, 7, 2))}[shape]
    assert tile_walk(M, N, K) == walk
    for mode in MODES:
        case256(epi, M, N, K, mode, seed=M + N + K)


@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("raster_n", ["0", "1"])
def test_tile256_forced_tile_walks(epi, raster_n):
    """Both walks with groups of 3 blocks (a short last group on each side) forced on a tall and a wide shape."""
    for M, N in ((128 * 40 + 3, 1280), (700, 256 * 20)):
        for mode in MODES:
            case256(epi, M, N, 192, mode, seed=M + N, walk={"EVO_B200_GEMM_RASTER_N": raster_n, "EVO_B200_GEMM_GROUP": "3"})


@pytest.mark.parametrize("epi,N,rope_L,M", [("bias", 12288, None, 1029), ("bias_resid", 4096, None, 1029), ("gelu_gate", 22016, None, 1029),
                                             ("bias_rope", 12288, None, 1029), ("bias_rope", 12288, 1025, 2050),
                                             ("none", 4096, None, 1029), ("resid", 4096, None, 1029)])
def test_tile256_model_widths(epi, N, rope_L, M):
    """the 7B model's projections at K = 4096 (gate: 2 x 11008 interleaved rows); rotary with one sequence and with two
    sequences of 1025 rows"""
    for mode in MODES:
        case256(epi, M, N, 4096, mode, seed=N, rope_L=rope_L)


@pytest.mark.parametrize("M", [129, 300])
def test_tile256_rope_tables_of_the_block_only(M):
    """A block of a longer sequence (rope_L > M): row m takes table row m, and the tables hold only the M rows the block has
    (a NaN-filled allocation behind them keeps every read inside it)."""
    N = 768
    for mode in MODES:
        rope = rope_setup(M, N, M, rope_L=M)
        pad = lambda t: torch.cat([t, torch.full((64, 64), float("nan"), dtype=torch.bfloat16, device=DEV)])[:M]
        rope = dict(rope, cos=pad(rope["cos"]), sin=pad(rope["sin"]), rope_L=M + 1000)
        case256("bias_rope", M, N, 256, mode, seed=M, rope=rope)


@pytest.mark.parametrize("epi", list(EPI))
def test_tile256_strides_and_sentinels(epi):
    """A a column slice of a wider tensor (lda = K + 64), C rows wider than the output, the residual at its own stride"""
    for mode in MODES:
        case256(epi, 300, 768, 192, mode, seed=7, lda_pad=64, ldc_pad=64, ldr_pad=136)


@pytest.mark.parametrize("epi", ["resid", "bias_resid"])
@pytest.mark.parametrize("M", [300, 128 * 133 + 1])
def test_tile256_residual_aliases_c(epi, M):
    for mode in MODES:
        case256(epi, M, 512, 192, mode, seed=M, ldc_pad=8, alias=True)


# ------------------------------------------------------------------ the 64-column tile (variants 2 and 3)
@pytest.mark.parametrize("M", [1, 16, 64, 65, 200])
@pytest.mark.parametrize("N,K", [(512, 256), (12288, 4096), (4096, 11008), (22016, 4096)])
def test_tile64(M, N, K):
    """variant 2 (row-major W) and 3 (tile-major W): every linear epilogue; and the decode path's gate for B > 64, the plain GEMM
    against the interleaved w12 followed by evo_gelu_gate_interleaved"""
    for mode in MODES:
        a, w, bias, resid, gam = inputs(mode, M, N, K, seed=M + N + K, ldr=N + 64)
        wt = StripedHyena._tile64(w)
        exact, S = reference(mode, a, w)
        for epi in LINEAR:
            ex = GO.expect(epi, exact, S, gam, bias=bias, resid=resid[:, :N])
            outs = []
            for variant, wv in ((2, w), (3, wt)):
                c = nan_buf(M + 2, N + 64)
                evo_gemm(a, wv, c, N + 64, epi, variant, bias, resid, N + 64, N=N)
                judge(f"{epi} M={M} N={N} K={K} {mode} variant={variant}", c, ex, (128, 64), mode, "tile64")
                sentinels_intact(c, M, N)
                outs.append(c[:M, :N])
            assert torch.equal(outs[0], outs[1]), "variant 3 differs from variant 2"
            if epi == "none":
                t = outs[0].contiguous()
                g = nan_buf(M, N // 2)
                _lib.check(_lib.lib().evo_gelu_gate_interleaved(_lib.ptr(t), _lib.ptr(g), M, N // 2, stream()))
                torch.cuda.synchronize()
                judge(f"gelu_gate_interleaved M={M} N={N} K={K} {mode}", g, GO.expect("gelu_gate", exact, S, gam), (128, 64), mode,
                      "tile64")


# ------------------------------------------------------------------ evo_gemm_smallm (stream-K)
def smallm(a, w, c, ldc, epi, bias=None, resid=None, ldr=None, ws=None):
    M, K = a.shape
    N = w.shape[0]
    lib = _lib.lib()
    if ws is None:
        ws = torch.zeros(max(lib.evo_gemm_smallm_workspace(M, N, K, e) for e in range(5)), dtype=torch.uint8, device=DEV)
    p = _lib.GemmSmallMParams(A=a.data_ptr(), lda=a.stride(0), W=w.data_ptr(), C=c.data_ptr(), ldc=ldc,
                              bias=bias.data_ptr() if epi in ("bias", "bias_resid") else None,
                              residual=resid.data_ptr() if epi in ("resid", "bias_resid") else None, ldr=ldr or ldc,
                              M=M, N=N, K=K, epilogue=EPI[epi], workspace=ws.data_ptr(), workspace_bytes=ws.numel())
    _lib.check(lib.evo_gemm_smallm(C.byref(p), stream()), f"evo_gemm_smallm({epi})")
    torch.cuda.synchronize()
    return ws


def case_smallm(epis, M, N, K, modes, seed, lda_pad=0, ldc_pad=0, ldr_pad=0, repeat=False):
    for mode in modes:
        a, w, bias, resid, gam = inputs(mode, M, N, K, seed, lda=K + lda_pad, ldr=N + ldr_pad)
        exact, S = reference(mode, a, w)
        ws = None
        for epi in epis:
            n_out = N // 2 if epi == "gelu_gate" else N
            ex = GO.expect(epi, exact, S, gam, bias=bias, resid=resid[:, :n_out])
            c = nan_buf(M + 2, n_out + ldc_pad)
            ws = smallm(a, w, c, n_out + ldc_pad, epi, bias, resid, N + ldr_pad, ws)
            judge(f"stream-K {epi} M={M} N={N} K={K} {mode}", c, ex, (64, 128), mode, "streamk_gate" if epi == "gelu_gate" else "streamk")
            sentinels_intact(c, M, n_out)
            assert int(ws[:16384].view(torch.int32).abs().sum().item()) == 0, "tile counters not back to zero"
            if repeat:
                c2 = nan_buf(M + 2, n_out + ldc_pad)
                smallm(a, w, c2, n_out + ldc_pad, epi, bias, resid, N + ldr_pad, ws)
                assert torch.equal(c2.view(torch.int16), c.view(torch.int16)), "two launches differ"


@pytest.mark.parametrize("M", range(1, 65))
def test_streamk_every_m(M):
    case_smallm(LINEAR + ("gelu_gate",), M, 512, 256, ("int",), seed=M)


@pytest.mark.parametrize("M", [1, 15, 16, 17, 31, 33, 48, 49, 63, 64])
@pytest.mark.parametrize("epi,N,K", [("bias", 12288, 4096), ("bias_resid", 4096, 4096), ("resid", 4096, 11008), ("gelu_gate", 22016, 4096),
                                     ("none", 12288, 4096)])
def test_streamk_model_widths(M, epi, N, K):
    case_smallm((epi,), M, N, K, MODES, seed=M + N + K)


@pytest.mark.parametrize("N,K", [(256, 64), (512, 512), (65536, 64), (65536, 128), (65536, 192)])
def test_streamk_grids_and_ranges(N, K):
    """256 x 64 and 512 x 512 run on fewer CTAs than SMs; at N = 65536 every range covers several whole tiles, with range
    boundaries on tile boundaries (K = 64, 128) and inside tiles (K = 192: 1536 k-blocks over the SMs)"""
    case_smallm(("none", "bias_resid", "gelu_gate"), 33, N, K, MODES, seed=N + K, repeat=True)


def test_streamk_strides():
    """lda > K, ldc > the output width, ldr != ldc"""
    case_smallm(LINEAR + ("gelu_gate",), 40, 4096, 1024, MODES, seed=3, lda_pad=64, ldc_pad=64, ldr_pad=136, repeat=True)


# ------------------------------------------------------------------ peer-scattered output on one GPU
@pytest.mark.parametrize("P", [2, 4, 8])
@pytest.mark.parametrize("epi", ["none", "bias", "bias_rope"])
def test_peer_scatter(P, epi):
    """column n of row m goes to peer (n % period) / inner at row row0 + m, column (n / period) inner + n % inner: un-scattered
    on the host and held to the same reference; rows outside the block and the other peers' buffers' spare rows stay NaN"""
    H, M, K, row0 = 8, 300, 256, 37
    d = H * 128
    inner, period = d // P, d
    N = 3 * d
    ldc = (N // period) * inner
    for mode in MODES:
        a, w, bias, resid, gam = inputs(mode, M, N, K, seed=P)
        rope = rope_setup(M, N, P, rope_L=row0 + M, rope_cols=2 * d) if epi == "bias_rope" else None
        if rope is not None:        # the caller offsets the tables by the first position: M rows left, one sequence
            rope = dict(rope, cos=rope["cos"][row0:], sin=rope["sin"][row0:], rope_L=M)
        bufs = [nan_buf(row0 + M + 2, ldc) for _ in range(P)]
        arr = (C.c_void_p * P)(*[b.data_ptr() for b in bufs])
        evo_gemm(a, w, None, ldc, epi, 0, bias, None, None, rope,
                 peers=dict(c_peers=C.cast(arr, C.c_void_p), n_c_peers=P, peer_period=period, peer_inner=inner, peer_row0=row0))
        out = torch.empty(M, N // period, P, inner, dtype=torch.bfloat16, device=DEV)
        for p, b in enumerate(bufs):
            out[:, :, p] = b[row0:row0 + M].view(M, N // period, inner)
            assert torch.isnan(b[:row0].float()).all() and torch.isnan(b[row0 + M:].float()).all()
        exact, S = reference(mode, a, w)
        ex = GO.expect(epi, exact, S, gam, bias=bias, rope=rope)
        judge(f"peers={P} {epi} {mode}", out.view(M, N), ex, (128, 256), mode, "tile256")


# ------------------------------------------------------------------ evo_unembed_score
def score(x, w, targets):
    M, K = x.shape
    V = w.shape[0]
    ws = torch.empty(_lib.lib().evo_unembed_score_workspace(M, V), dtype=torch.uint8, device=DEV)
    lp = torch.full((M,), float("nan"), device=DEV)
    ent = torch.full((M,), float("nan"), device=DEV)
    p = _lib.ScoreParams(x=x.data_ptr(), W=w.data_ptr(), targets=targets.data_ptr(), logprobs=lp.data_ptr(), entropy=ent.data_ptr(),
                         M=M, V=V, K=K, workspace=ws.data_ptr(), workspace_bytes=ws.numel())
    _lib.check(_lib.lib().evo_unembed_score(C.byref(p), stream()), "evo_unembed_score")
    torch.cuda.synchronize()
    return lp.double(), ent.double()


def score_targets(logits, g):
    """random targets, with -1 and V (both give 0) and each row's argmax and argmin mixed in"""
    M, V = logits.shape
    t = torch.randint(0, V, (M,), generator=g, device=DEV)
    r = torch.arange(M, device=DEV)
    t = torch.where(r % 5 == 1, logits.float().argmax(1), t)
    t = torch.where(r % 5 == 2, logits.float().argmin(1), t)
    t = torch.where(r % 5 == 3, torch.full_like(t, -1), t)
    t = torch.where(r % 5 == 4, torch.full_like(t, V), t)
    return t


def case_score(M, V, K, mode, seed, peaked=False):
    a, w, _, _, gam = inputs(mode, M, V, K, seed)
    if peaked:      # row 0's logit at column 5 far above the rest
        w = w.clone()
        w[5] = (a[0] * (2.0 ** -GO.int_exponent(K) if mode == "int" else 4.0 / math.sqrt(K))).bfloat16()
    exact, S = reference(mode, a, w)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    mid = GO.bf(exact)
    t = score_targets(mid, g)
    lp, ent = score(a, w, t)
    if peaked:
        assert mid[0].float().max() > mid[0].float().topk(2).values[1] + 10
    ref_lp, ref_ent, aux = GO.score_reference(mid, t)
    tol_lp, tol_ent = GO.score_bounds(aux, V)
    assert (lp[t < 0] == 0).all() and (lp[t >= V] == 0).all(), "targets -1 and V must give 0"
    if mode == "int":             # the logits are known bit for bit
        assert tol_lp.max() < 2e-5 and tol_ent.max() < 5e-5
        bad = ((lp - ref_lp).abs() > tol_lp) | ((ent - ref_ent).abs() > tol_ent)
    else:                         # the logits lie in their intervals: log-probability between the interval ends' values
        lo, hi = GO.bf(exact - gam * S).double(), GO.bf(exact + gam * S).double()
        valid = aux["valid"]
        tc = t.clamp(0, V - 1)[:, None]
        lp_lo = torch.where(valid, lo.gather(1, tc)[:, 0] - torch.logsumexp(hi, 1), torch.zeros_like(ref_lp)) - tol_lp
        lp_hi = torch.where(valid, hi.gather(1, tc)[:, 0] - torch.logsumexp(lo, 1), torch.zeros_like(ref_lp)) + tol_lp
        # entropy: dH/dx_v = -p_v (x_v - mean); moving every logit by at most d_v <= dmax changes each p_v by a factor within
        # e^(+-2 dmax) and mean by at most dmax, so |H(x') - H(x)| <= e^(2 dmax) sum_v p_v (|x_v - mean| + 2 dmax) d_v
        x = mid.double()
        d = torch.maximum(hi - x, x - lo)
        dmax = d.max(1).values
        dev = (x - aux["mean"][:, None]).abs() + 2 * dmax[:, None]
        tol_h = torch.exp(2 * dmax) * (aux["p"] * dev * d).sum(1) + tol_ent
        bad = (lp < lp_lo) | (lp > lp_hi) | ((ent - ref_ent).abs() > tol_h)
    rows = torch.nonzero(bad).flatten()
    assert rows.numel() == 0, (f"score M={M} V={V} K={K} {mode}: {rows.numel()} rows off, first {rows[:5].tolist()} (row-blocks "
                               f"{sorted(set((rows // 128).tolist()))[:8]}): lp {lp[rows[:3]].tolist()} vs {ref_lp[rows[:3]].tolist()}, "
                               f"entropy {ent[rows[:3]].tolist()} vs {ref_ent[rows[:3]].tolist()}")


@pytest.mark.parametrize("V", [256, 512, 1024])
@pytest.mark.parametrize("K", [256, 4096])
@pytest.mark.parametrize("M", [1, 127, 129, "n_sm*128+1"])
def test_unembed_score(V, K, M):
    M = n_sm() * 128 + 1 if M == "n_sm*128+1" else M
    for mode in MODES:
        case_score(M, V, K, mode, seed=V + K + M)


@pytest.mark.parametrize("V", [256, 1024])
def test_unembed_score_peaked(V):
    for mode in MODES:
        case_score(129, V, 256, mode, seed=V, peaked=True)
