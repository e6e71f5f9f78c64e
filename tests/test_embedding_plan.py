"""Host side of sequence embeddings (no GPU): layer specs, reassembly into input order across packs, the npz layout of
scripts/embed.py, and evo_pool_varlen's argument checks, which return before anything is launched."""
import ctypes as C
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from evo_b200 import _lib                                      # noqa: E402
from evo_b200.embeddings import embed_sequences, parse_layers   # noqa: E402
from evo_b200.stripedhyena.model import resolve_layers          # noqa: E402
from evo_b200.tokenizer import CharLevelTokenizer               # noqa: E402


def test_layer_specs_and_negative_indices():
    assert parse_layers("final,16,-1") == ["final", 16, -1]
    assert parse_layers(" 0 , final ") == [0, "final"]
    for bad in ("fnal", "16,", "1.5", ""):
        with pytest.raises(ValueError):
            parse_layers(bad)
    assert resolve_layers(["final", 16, -1, -32, 0], 32) == {"final": "final", 16: 16, -1: 31, -32: 0, 0: 0}
    assert resolve_layers("final", 4) == {"final": "final"} and resolve_layers(-2, 4) == {-2: 2}
    assert resolve_layers([np.int64(3)], 4) == {3: 3}
    for bad in ([4], [-5], [True], [1.0], ["Final"], [None], []):
        with pytest.raises(_lib.EvoError):
            resolve_layers(bad, 4)


class StubModel:
    """embed_packed's contract without a GPU: per layer, each sequence's row is (layer tag, its length, its first base, pack
    index), read back from the packed ids."""

    def __init__(self, num_layers=4, d=4):
        self.config = SimpleNamespace(num_layers=num_layers, hidden_size=d)
        self.embedding_layer = SimpleNamespace(weight=SimpleNamespace(device=torch.device("cuda:0")))
        self.calls = []

    def embed_packed(self, ids, cu, layers, pool, skip_bos):
        self.calls.append((int(ids.shape[0]), list(cu), list(layers), pool, skip_bos))
        out = {}
        for k in layers:
            tag = 100.0 if k == "final" else float(k)
            rows = [[tag, cu[b + 1] - cu[b] - 1, float(ids[cu[b] + 1]), len(self.calls)] for b in range(len(cu) - 1)]
            out[k] = torch.tensor(rows, dtype=torch.float32)
        return out


def _fake_packed_ids(seqs, tokenizer, device="cuda:0"):
    return torch.from_numpy(np.concatenate([np.frombuffer(b"\0" + s.encode(), dtype=np.uint8).astype(np.int64) for s in seqs]))


def test_reassembly_in_input_order_across_packs(monkeypatch):
    from evo_b200 import frontend
    monkeypatch.setattr(frontend, "packed_ids", _fake_packed_ids)
    rng = np.random.default_rng(0)
    lens = [int(n) for n in rng.permutation([1, 5, 40, 7, 100, 33, 2, 64, 9, 17])]
    seqs = ["ACGT"[i % 4] + "".join(rng.choice(list("ACGT"), size=n - 1)) for i, n in enumerate(lens)]
    model = StubModel()
    got = embed_sequences(seqs, model, CharLevelTokenizer(512), layers=["final", 2, -1, 2], pool="max", include_bos=True,
                          max_tokens=60)
    assert list(got) == ["final", 2, -1]                      # keyed as given, duplicates once
    assert len(model.calls) > 2 and all(c[0] <= 60 or len(c[1]) == 2 for c in model.calls)
    assert all(c[2] == ["final", 2, -1] and c[3] == "max" and c[4] is False for c in model.calls)
    for k, tag in (("final", 100.0), (2, 2.0), (-1, -1.0)):
        v = got[k]
        assert v.shape == (len(seqs), 4) and v.dtype == np.float32
        assert (v[:, 0] == tag).all()
        assert v[:, 1].tolist() == lens
        assert v[:, 2].tolist() == [float(ord(s[0])) for s in seqs]
    assert sorted(set(got["final"][:, 3].tolist())) == list(range(1, len(model.calls) + 1))


def test_rejected_calls_raise_before_any_pack(monkeypatch):
    from evo_b200 import frontend
    monkeypatch.setattr(frontend, "packed_ids", _fake_packed_ids)
    model, tok = StubModel(), CharLevelTokenizer(512)
    for kw in (dict(layers=[4]), dict(layers=["x"]), dict(pool="sum"), dict(pool=None), dict(max_tokens=0), dict(device="cpu"),
               dict(device="cuda:1")):
        with pytest.raises(ValueError):
            embed_sequences(["ACGT"], model, tok, **kw)
    for seqs in (["ACGT", ""], ["ACGÜ"]):
        with pytest.raises(ValueError):
            embed_sequences(seqs, model, tok)
    assert model.calls == []


def test_cli_npz_layout(tmp_path, monkeypatch):
    from scripts import embed as cli
    fasta = tmp_path / "in.fasta"
    fasta.write_text(">a first\nACGT\nAC\n>b\nGG\n>c\nTTTTT\n")
    seen = {}

    class FakeEvo:
        def __init__(self, *a, **kw):
            self.model, self.tokenizer = SimpleNamespace(eval=lambda: None), None

    def fake_embed(seqs, model, tokenizer, layers, pool, include_bos, max_tokens, device):
        seen.update(seqs=seqs, layers=layers, pool=pool, include_bos=include_bos, max_tokens=max_tokens)
        return {k: np.full((len(seqs), 3), i, dtype=np.float32) for i, k in enumerate(layers)}
    monkeypatch.setattr(cli, "Evo", FakeEvo)
    monkeypatch.setattr(cli, "embed_sequences", fake_embed)
    out = tmp_path / "e.npz"
    cli.main(["--input-fasta", str(fasta), "--output-npz", str(out), "--layers", "final,16,-1", "--pool", "last",
              "--include-bos", "--max-tokens", "99"])
    assert seen == dict(seqs=["ACGTAC", "GG", "TTTTT"], layers=["final", 16, -1], pool="last", include_bos=True, max_tokens=99)
    z = np.load(out)
    assert sorted(z.files) == ["layer_-1", "layer_16", "layer_final", "names"]
    assert z["names"].tolist() == ["a", "b", "c"]
    assert z["layer_16"].shape == (3, 3) and z["layer_16"].dtype == np.float32 and (z["layer_16"] == 1).all()
    cli.main(["--input-fasta", str(fasta), "--output-npz", str(out)])
    assert seen["layers"] == ["final"] and seen["pool"] == "mean" and seen["include_bos"] is False
    assert sorted(np.load(out).files) == ["layer_final", "names"]


def _params(**kw):
    p = dict(x=0x1000, ldx=256, cu_seqlens=0x2000, n_seq=2, T=5000, max_seqlen=4000, D=256, skip_first=1, mode=_lib.POOL_MEAN,
             out=0x3000, ldo=256)
    p.update(kw)
    return _lib.PoolVarlenParams(**p)


def test_pool_rejects_bad_arguments_before_any_launch():
    lib = _lib.lib()
    need = lib.evo_pool_varlen_workspace(C.byref(_params()))
    assert need > 0                                           # 4000 rows span several 512-row chunks
    assert lib.evo_pool_varlen_workspace(C.byref(_params(mode=_lib.POOL_LAST))) == 0
    assert lib.evo_pool_varlen_workspace(C.byref(_params(max_seqlen=513))) == 0          # 512 kept rows: one chunk
    cases = {"D (250)": dict(D=250, ldx=256, ldo=256), "ldx (128)": dict(ldx=128), "ldx (260)": dict(ldx=260),
             "ldo (255)": dict(ldo=255), "n_seq (0)": dict(n_seq=0), "T (0)": dict(T=0, max_seqlen=0),
             "max_seqlen (6000)": dict(max_seqlen=6000), "unknown mode 3": dict(mode=3), "unknown mode -1": dict(mode=-1),
             "skip_first (-1)": dict(skip_first=-1), "x, cu_seqlens and out": dict(x=None), "16-byte aligned": dict(x=0x1008)}
    cases["x, cu_seqlens and out "] = dict(cu_seqlens=None)
    cases["x, cu_seqlens and out  "] = dict(out=None)
    lib.evo_reset_launch_count()
    for msg, kw in cases.items():
        rc = lib.evo_pool_varlen(C.byref(_params(**kw)), C.c_void_p(0x4000), 1 << 30, None)
        assert rc != 0 and msg.strip().encode() in lib.evo_last_error(), (msg, lib.evo_last_error())
    rc = lib.evo_pool_varlen(C.byref(_params()), C.c_void_p(0x4000), need - 1, None)
    assert rc != 0 and b"workspace" in lib.evo_last_error()
    rc = lib.evo_pool_varlen(C.byref(_params()), None, need, None)
    assert rc != 0 and b"workspace" in lib.evo_last_error()
    assert lib.evo_pool_varlen(None, None, 0, None) != 0 and b"NULL" in lib.evo_last_error()
    assert lib.evo_launch_count() == 0
