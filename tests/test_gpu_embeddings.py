"""Sequence embeddings: evo_pool_varlen, StripedHyena.embed_packed (block taps, early exit) and embed_sequences / scripts/embed.py.

Kernel bars.  max and last are widened bf16 values, so they are held bit for bit to torch.  The mean is an fp32 sum tree of
depth at most 512/8 + 8 + ceil(n / 512) + 1 (a lane's share of a 512-row chunk, the 8 row groups, the chunk partials, the
division; include/evo_b200.h describes the scheme), so |mean - exact| <= depth * 2^-24 * mean|x| per column; on integer-valued
rows every partial sum is exact in fp32 and the mean is the one correctly rounded quotient, bit for bit.
Model bars.  Against the oracle: the GPU's pooled error against fp64 is at most 1.25x the bf16 oracle's plus 2e-3 of the
pooled magnitude (test_model_logits_vs_oracle's rule).  Packed against solo: MIXED_TAU of max(1, |embedding|max), the bar the
packed logits meet."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

from oracle import stripedhyena_oracle as O          # noqa: E402
from evo_b200 import _lib                             # noqa: E402
from evo_b200.stripedhyena import StripedHyena, dotdict  # noqa: E402
from tests.test_gpu_packed import MIXED, MIXED_TAU, _cu, _ids, _same, _tiny, _two_block_7b  # noqa: E402

DEV = "cuda:0"
MODES = {"mean": _lib.POOL_MEAN, "max": _lib.POOL_MAX, "last": _lib.POOL_LAST}
LONG = MIXED + (70001,)             # one sequence of 137 chunks: the two-pass reduction


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def pool(x, lengths, mode, skip=0, out=None):
    """evo_pool_varlen over x (T, D) bf16, any row stride; returns (n, D) fp32."""
    lib = _lib.lib()
    T, D = x.shape
    n = len(lengths)
    cu = torch.tensor(_cu(lengths), dtype=torch.int64, device=DEV)
    out = torch.full((n, D), 7.0, dtype=torch.float32, device=DEV) if out is None else out
    pp = _lib.PoolVarlenParams(x=x.data_ptr(), ldx=x.stride(0), cu_seqlens=cu.data_ptr(), n_seq=n, T=T, max_seqlen=max(lengths),
                               D=D, skip_first=skip, mode=MODES[mode], out=out.data_ptr(), ldo=out.stride(0))
    need = lib.evo_pool_varlen_workspace(C.byref(pp))
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
    _lib.check(lib.evo_pool_varlen(C.byref(pp), _lib.ptr(ws), need, stream()), "evo_pool_varlen")
    torch.cuda.synchronize()
    return out


def _padded(T, D, gen, integer=False):
    """(T, D) bf16 rows at row stride D + 8 whose 8 padding columns hold NaN: nothing outside [0, D) may reach an output."""
    full = torch.full((T, D + 8), float("nan"), dtype=torch.bfloat16, device=DEV)
    v = torch.randint(-4, 5, (T, D), generator=gen, device=DEV).float() if integer else torch.randn(T, D, generator=gen, device=DEV) + 0.5
    full[:, :D] = v.bfloat16()
    return full[:, :D]


def _depth(n):
    return 512 // 8 + 8 + math.ceil(n / 512) + 1


# ------------------------------------------------------------------ kernel
@pytest.mark.parametrize("D", [256, 4096])
@pytest.mark.parametrize("skip", [0, 1])
def test_pool_values_against_fp64(D, skip):
    g = torch.Generator(device=DEV).manual_seed(D + skip)
    x = _padded(sum(LONG), D, g)
    cu = _cu(LONG)
    if skip:                              # the skipped first rows hold NaN: they must not be read
        x[torch.tensor(cu[:-1], device=DEV)] = float("nan")
    got = {m: pool(x, LONG, m, skip) for m in MODES}
    for m in MODES:
        assert not got[m][[b for b, L in enumerate(LONG) if L > skip]].isnan().any(), m
    for b, L in enumerate(LONG):
        rows = x[cu[b] + skip:cu[b + 1]]
        if rows.shape[0] == 0:            # length 1 with skip 1: no kept row
            assert all(got[m][b].isnan().all() for m in MODES)
            continue
        exact = rows.double().mean(0)
        bound = _depth(rows.shape[0]) * 2.0 ** -24 * rows.double().abs().mean(0) + 1e-30
        assert ((got["mean"][b].double() - exact).abs() <= bound).all(), (D, L)
        assert _same(got["max"][b], rows.float().max(0).values), (D, L)
        assert _same(got["last"][b], rows[-1].float()), (D, L)


@pytest.mark.parametrize("D", [256, 4096])
def test_pool_mean_of_integer_rows_is_the_rounded_quotient(D):
    g = torch.Generator(device=DEV).manual_seed(5)
    x = _padded(sum(LONG), D, g, integer=True)
    got = pool(x, LONG, "mean", 1)
    cu = _cu(LONG)
    for b, L in enumerate(LONG):
        if L > 1:                         # numpy divides elementwise (torch on CUDA multiplies by a rounded reciprocal)
            s = x[cu[b] + 1:cu[b + 1]].double().sum(0).cpu().numpy().astype(np.float32)
            assert np.array_equal(got[b].cpu().numpy(), s / np.float32(L - 1)), (D, L)


@pytest.mark.parametrize("mode", list(MODES))
def test_pool_is_placement_independent_and_deterministic(mode):
    D = 512
    g = torch.Generator(device=DEV).manual_seed(11)
    lengths = (3, 70001, 513, 1, 1024, 9)
    x = _padded(sum(lengths), D, g)
    cu = _cu(lengths)
    packed = pool(x, lengths, mode, 1)
    assert _same(packed, pool(x, lengths, mode, 1))
    for b, L in enumerate(lengths):
        alone = x[cu[b]:cu[b + 1]].contiguous()
        assert _same(packed[b], pool(alone, [L], mode, 1)[0]), (mode, L)
    # the same sequences in another order and behind an offset of a different length
    order = [5, 2, 1, 0, 4, 3]
    pre = torch.randn(77, D, generator=g, device=DEV).bfloat16()
    moved = torch.cat([pre] + [x[cu[b]:cu[b + 1]] for b in order])
    got = pool(moved, [77] + [lengths[b] for b in order], mode, 1)
    for k, b in enumerate(order):
        assert _same(got[k + 1], packed[b]), (mode, lengths[b])


def test_pool_writes_only_its_output_rows_and_columns():
    D, n = 256, 3
    x = torch.randn(30, D, device=DEV).bfloat16()
    out = torch.full((n + 1, D + 16), -5.0, device=DEV)
    pool(x, [10, 10, 10], "mean", 0, out=out[:n, :D])
    assert (out[:n, D:] == -5).all() and (out[n] == -5).all() and not (out[:n, :D] == -5).any()


# ------------------------------------------------------------------ model
@pytest.fixture(scope="module")
def tiny():
    return _tiny()


@pytest.fixture(scope="module")
def wide():
    return _two_block_7b()


def _host_pool(rows, mode):
    return {"mean": lambda r: r.mean(0), "max": lambda r: r.max(0).values, "last": lambda r: r[-1]}[mode](rows)


ORACLE_LENGTHS = (300, 2, 65, 1030)


@pytest.fixture(scope="module")
def oracle_rows(tiny):
    """Per sequence, {layer: (bf16-oracle rows, fp64-oracle rows)} of the tiny model: the block taps, and the final norm of the last."""
    cfg, sd, _ = tiny
    ob, ot = O.OracleStripedHyena(cfg, sd, torch.bfloat16), O.OracleStripedHyena(cfg, sd, torch.float64)
    last = f"block{cfg['num_layers'] - 1}"
    out = []
    for s in _ids(ORACLE_LENGTHS, seed=4):
        ob(s[None], tap=True)
        ot(s[None], tap=True)
        rows = {k: (ob.taps[f"block{k}"][0], ot.taps[f"block{k}"][0]) for k in range(cfg["num_layers"])}
        rows["final"] = (O.rms_norm(ob.taps[last], ob.sd["norm.scale"], cfg["eps"])[0], O.rms_norm(ot.taps[last], ot.sd["norm.scale"], cfg["eps"])[0])
        out.append(rows)
    return out


@pytest.mark.parametrize("mode", list(MODES))
def test_embeddings_vs_oracle(tiny, oracle_rows, mode):
    m = tiny[2]
    layers = [0, 1, 2, 3, "final"]
    got = m.embed_packed(torch.cat(_ids(ORACLE_LENGTHS, seed=4)).to(DEV), _cu(ORACLE_LENGTHS), layers=layers, pool=mode)
    for b, rows in enumerate(oracle_rows):
        for k in layers:
            fb, ft = rows[k]
            want = _host_pool(ft[1:].double(), mode)
            e_ref = (_host_pool(fb[1:].double(), mode) - want).abs().mean().item()
            e_gpu = (got[k][b].cpu().double() - want).abs().mean().item()
            assert e_gpu <= 1.25 * e_ref + 2e-3 * want.abs().mean().item(), (mode, k, ORACLE_LENGTHS[b], e_gpu, e_ref)


def test_early_exit_changes_no_bit(tiny):
    m = tiny[2]
    lengths = (130, 1, 64, 1000)
    flat, cu = torch.cat(_ids(lengths, seed=8)).to(DEV), _cu(lengths)
    for pool_ in ("mean", None):
        both = m.embed_packed(flat, cu, layers=[0, 1, 2, "final"], pool=pool_, skip_bos=False)
        for k in (0, 1, 2):
            alone = m.embed_packed(flat, cu, layers=[k], pool=pool_, skip_bos=False)[k]
            assert _same(alone, both[k]), (pool_, k)


def test_launches_stop_after_the_deepest_block(tiny):
    m = tiny[2]
    flat, cu = torch.cat(_ids((100, 50), seed=2)).to(DEV), _cu((100, 50))
    counts = {}
    for k in (0, 1, 2, 3, "final"):
        m.embed_packed(flat, cu, layers=[k])            # warm: rotary tables
        torch.cuda.synchronize()
        _lib.lib().evo_reset_launch_count()
        m.embed_packed(flat, cu, layers=[k])
        counts[k] = _lib.lib().evo_launch_count()
    assert counts[0] < counts[1] < counts[2] < counts[3] < counts["final"]
    assert counts["final"] == counts[3] + 1             # the final norm; the unembedding never runs


def test_pooled_equals_per_token(tiny):
    m = tiny[2]
    lengths = (5, 1030, 2, 517, 64)
    flat, cu = torch.cat(_ids(lengths, seed=3)).to(DEV), _cu(lengths)
    rows = m.embed_packed(flat, cu, layers=[2, "final"], pool=None)
    for k in (2, "final"):
        assert rows[k].shape == (sum(lengths), 256) and rows[k].dtype == torch.bfloat16
        got = {p: m.embed_packed(flat, cu, layers=[k], pool=p)[k] for p in MODES}
        for b, L in enumerate(lengths):
            r = rows[k][cu[b] + 1:cu[b + 1]]
            assert ((got["mean"][b].double() - r.double().mean(0)).abs() <= _depth(L - 1) * 2.0 ** -24 * r.double().abs().mean(0)).all()
            assert _same(got["max"][b], r.float().max(0).values) and _same(got["last"][b], r[-1].float()), (k, L)


def test_packed_embeddings_match_each_sequence_alone(wide):
    m = wide[2]
    lengths = (1500, 2, 300, 17, 8193)
    seqs = _ids(lengths, seed=12)
    flat, cu = torch.cat(seqs).to(DEV), _cu(lengths)
    packed = m.embed_packed(flat, cu, layers=[0, "final"], pool="mean")
    for b, s in enumerate(seqs):
        solo = m.embed_packed(s.to(DEV), [0, lengths[b]], layers=[0, "final"], pool="mean")
        for k in (0, "final"):
            a, e = packed[k][b].double(), solo[k][0].double()
            assert (a - e).abs().max().item() <= MIXED_TAU * max(1.0, e.abs().max().item()), (k, lengths[b])


@pytest.mark.parametrize("L", [1024, 8193])
def test_final_rows_are_the_unembedding_input_bit_for_bit(wide, L):
    m = wide[2]
    ids = torch.stack(_ids([L] * 2, seed=L)).to(DEV)
    with torch.cuda.device(DEV), torch.no_grad():
        u = m._backbone(ids, 2, L)
    rows = m.embed_packed(ids.reshape(-1), _cu([L] * 2), layers=["final", -1], pool=None)
    assert _same(rows["final"], u)
    assert rows[-1].shape == u.shape and not _same(rows[-1], u)       # the last block's output, before the final norm


# ------------------------------------------------------------------ public surface
def test_embed_sequences_returns_input_order_across_packs(tiny):
    import evo_b200
    m = tiny[2]
    tok = evo_b200.CharLevelTokenizer(512)
    rng = np.random.default_rng(3)
    lens = [40, 7, 300, 1, 129, 41, 8, 260, 2]
    rng.shuffle(lens)
    seqs = ["".join(rng.choice(list("ACGT"), size=n)) for n in lens]
    got = evo_b200.embed_sequences(seqs, m, tok, layers=["final", 1, -1], pool="mean", max_tokens=200, device=DEV)
    assert set(got) == {"final", 1, -1} and all(v.shape == (len(seqs), 256) and v.dtype == np.float32 for v in got.values())
    for i, s in enumerate(seqs):
        alone = evo_b200.embed_sequences([s], m, tok, layers=["final", 1, -1], pool="mean", device=DEV)
        for k in got:
            assert np.abs(got[k][i] - alone[k][0]).max() <= MIXED_TAU * max(1.0, np.abs(alone[k][0]).max()), (k, lens[i])
    # the BOS row changes every mean and no last row
    with_bos, without = ({p: evo_b200.embed_sequences(seqs, m, tok, layers=[1], pool=p, include_bos=bos, max_tokens=200, device=DEV)[1]
                          for p in ("mean", "last")} for bos in (True, False))
    assert np.array_equal(with_bos["last"], without["last"])
    assert not (with_bos["mean"] == without["mean"]).all(axis=1).any()


def test_rejected_calls_raise_before_any_launch(tiny):
    import evo_b200
    cfg, sd, m = tiny
    tok = evo_b200.CharLevelTokenizer(512)
    cpu_model = StripedHyena(dotdict(cfg))
    cpu_model.load_state_dict(sd, strict=True)
    ids = torch.cat(_ids([5, 3], seed=1)).to(DEV)
    lib = _lib.lib()
    surface = [lambda: evo_b200.embed_sequences(["ACGT", ""], m, tok, device=DEV),
               lambda: evo_b200.embed_sequences(["ACGT"], cpu_model, tok, device=DEV),
               lambda: evo_b200.embed_sequences(["ACGT"], m, tok, device="cpu"),
               lambda: evo_b200.embed_sequences(["ACGT"], m, tok, layers=[4], device=DEV),
               lambda: evo_b200.embed_sequences(["ACGT"], m, tok, layers=[-5], device=DEV),
               lambda: evo_b200.embed_sequences(["ACGT"], m, tok, layers=["last"], device=DEV),
               lambda: evo_b200.embed_sequences(["ACGT"], m, tok, pool="sum", device=DEV),
               lambda: evo_b200.embed_sequences(["ACGT"], m, tok, pool=None, device=DEV),
               lambda: evo_b200.embed_sequences(["ACGT"], m, tok, max_tokens=0, device=DEV)]
    model = [lambda: m.embed_packed(ids, [0, 5, 8], layers=[True]),
             lambda: m.embed_packed(ids, [0, 5, 8], layers=[1.0]),
             lambda: m.embed_packed(ids, [0, 5, 8], layers=[]),
             lambda: m.embed_packed(ids, [0, 5, 8], pool="median"),
             lambda: m.embed_packed(ids, [0, 1, 8]),                 # sequence 0 keeps no row after its BOS
             lambda: m.embed_packed(ids, [0, 5, 5, 8]),
             lambda: m.embed_packed(ids, [0, 5, 7]),
             lambda: m.embed_packed(ids.cpu(), [0, 5, 8])]
    for k, call in enumerate(surface + model):
        torch.cuda.synchronize()
        lib.evo_reset_launch_count()
        with pytest.raises(ValueError if k < len(surface) else _lib.EvoError):
            call()
        assert lib.evo_launch_count() == 0, k
    assert m.embed_packed(ids, [0, 1, 8], pool=None)["final"].shape == (8, 256)     # per-token output keeps every row


def test_cli_writes_names_and_one_array_per_layer(tiny, tmp_path, monkeypatch):
    import evo_b200
    from scripts import embed as cli
    m = tiny[2]
    tok = evo_b200.CharLevelTokenizer(512)
    rng = np.random.default_rng(9)
    seqs = ["".join(rng.choice(list("ACGT"), size=n)) for n in (120, 3, 77, 300, 12)]
    fasta = tmp_path / "in.fasta"
    fasta.write_text("".join(f">seq{i} some description\n{s[:50]}\n{s[50:]}\n" for i, s in enumerate(seqs)))

    class TinyEvo:
        def __init__(self, *a, **kw):
            self.model, self.tokenizer = m, tok
    monkeypatch.setattr(cli, "Evo", TinyEvo)
    out = tmp_path / "emb.npz"
    cli.main(["--input-fasta", str(fasta), "--output-npz", str(out), "--layers", "final,1,-2", "--pool", "max",
              "--max-tokens", "256", "--device", DEV])
    z = np.load(out)
    assert sorted(z.files) == ["layer_-2", "layer_1", "layer_final", "names"]
    assert z["names"].tolist() == [f"seq{i}" for i in range(len(seqs))]
    want = evo_b200.embed_sequences(seqs, m, tok, layers=["final", 1, -2], pool="max", max_tokens=256, device=DEV)
    for k, v in want.items():
        assert z[f"layer_{k}"].dtype == np.float32 and np.array_equal(z[f"layer_{k}"], v), k
