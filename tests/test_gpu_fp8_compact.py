"""Compact FP8 models on the GPU: evo_fp8_dequant_rows against the quantizer's in-place W' and the host reference bit for bit, a
compact model against the non-compact FP8 model built from the same state dict on every path (bits), its memory, its state
handling, and the streaming load that never holds the linear weights in bf16."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

from oracle import stripedhyena_oracle as O                                           # noqa: E402
from evo_b200 import _lib                                                              # noqa: E402
from evo_b200.stripedhyena import StripedHyena, dotdict                                # noqa: E402
from evo_b200.stripedhyena.model import fp8_unlayout                                  # noqa: E402
from tests.test_gpu_decode_vs_oracle import _tokens                                    # noqa: E402
from tests.test_gpu_fp8_decode import SAMPLING, bits, edge_weights, quantize, stream  # noqa: E402

DEV = "cuda:0"
WIDE = dict(hidden=4096, heads=32, layers=3, attn=(1,))        # the 7B's width: hidden 4096, 32 heads, one attention block


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()
    yield


def dequant(q, e, N, K, gate):
    out = torch.full((N, K), float("nan"), dtype=torch.bfloat16, device=DEV)
    _lib.check(_lib.lib().evo_fp8_dequant_rows(q.data_ptr(), e.data_ptr(), N, K, _lib.EPI_GELU_GATE if gate else _lib.EPI_NONE,
                                               out.data_ptr(), stream()), "evo_fp8_dequant_rows")
    torch.cuda.synchronize()
    return out


# ------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("N,K,gate", [(12288, 4096, False), (4096, 4096, False), (22016, 4096, True), (4096, 11008, False),
                                      (128, 64, False), (256, 64, True), (384, 192, False), (768, 320, True)])
def test_dequant_is_the_quantizers_w_prime(N, K, gate):
    w = edge_weights(N, K, seed=N + K)
    if K == 11008:
        w[:, 10928:] = 0                                       # w3: the zero-padded K columns of the 7B's inner 10928
    q, e, status = quantize(w, gate)                           # w is now W'
    assert status == 0
    assert int(e[0]) == 0 and int(e[5]) == -124 and int(e[2]) == -8
    got = dequant(q, e, N, K, gate)
    assert torch.equal(bits(got), bits(w))
    host = torch.ldexp(fp8_unlayout(q, N, K, gate).float(), e[:, None].float()).to(torch.bfloat16)
    assert torch.equal(bits(got), bits(host))


# ------------------------------------------------------------------ a compact model against the FP8 model
def _model(hidden=256, heads=2, layers=4, attn=(1, 3), seed=7):
    cfg = O.tiny_config(num_layers=layers, attn_layer_idxs=attn, hidden_size=hidden, num_heads=heads)
    m = StripedHyena(dotdict(cfg))
    m.load_state_dict(O.random_state_dict(cfg, seed=seed), strict=True)
    return cfg, m.to_bfloat16_except_poles_residues().to(DEV)


@pytest.fixture(scope="module", params=["tiny", "wide"])
def pair(request):
    kw = WIDE if request.param == "wide" else {}
    _, fp8 = _model(**kw)
    cfg, compact = _model(**kw)
    fp8.quantize_fp8()
    compact.quantize_fp8(compact=True)
    yield cfg, fp8, compact
    del fp8, compact
    torch.cuda.empty_cache()


def _same(a, b):
    if isinstance(a, (tuple, list)):
        assert type(a) is type(b) and len(a) == len(b)
        for x, y in zip(a, b):
            _same(x, y)
    elif isinstance(a, dict):
        assert a.keys() == b.keys()
        for k in a:
            _same(a[k], b[k])
    elif torch.is_tensor(a):
        assert a.dtype == b.dtype and a.shape == b.shape
        assert torch.equal(bits(a) if a.is_floating_point() else a, bits(b) if b.is_floating_point() else b)
    else:
        assert a == b


def _both(pair, run):
    _, fp8, compact = pair
    for m in (fp8, compact):
        m._decode = m._loop = None
    out = [run(m) for m in (fp8, compact)]
    _same(*out)
    return out


def test_stateless_logits_and_scoring(pair):
    ids = _tokens(3, 300, seed=1).to(DEV)
    _both(pair, lambda m: (m(ids)[0], *m.score_tokens(ids, want_entropy=True)))


def test_stateful_prefill_then_steps(pair):
    B, P, T = 8, 33, 6

    def run(m):
        d = m.initialize_inference_params()
        d["mha"].max_batch_size, d["mha"].max_seqlen = B, 128
        with torch.inference_mode():
            logits, d = m(_tokens(B, P, seed=3).to(DEV), inference_params_dict=d)
            steps, out = _tokens(B, T, seed=4).to(DEV), [logits]
            for k in range(T):
                d["mha"].seqlen_offset = d["hyena"].seqlen_offset = P + k
                s, d = m(steps[:, k:k + 1], inference_params_dict=d)
                out.append(s.clone())
        return out
    _both(pair, run)


def test_packed_forward_scoring_and_embeddings(pair):
    lengths = [130, 7, 300, 64]
    ids = torch.cat([_tokens(1, n, seed=n)[0] for n in lengths]).to(DEV)
    cu = [0] + list(np.cumsum(lengths))

    def run(m):
        return (m.forward_packed(ids, cu), *m.score_tokens_packed(ids, cu, want_entropy=True),
                m.embed_packed(ids, cu, layers=(1, "final"), pool="mean"), m.embed_packed(ids, cu, layers=(-2,), pool=None))
    _both(pair, run)


def test_score_variants(pair):
    import evo_b200
    g = np.random.default_rng(3)
    ref = "".join(g.choice(list("ACGT"), 1000))
    var = [ref[:300] + "G" + ref[301:], ref[:700] + ref[701:], ref[:129] + "TTT" + ref[600:], ref + "AC", ref[:400]]
    tok = evo_b200.CharLevelTokenizer(512)
    _both(pair, lambda m: evo_b200.score_variants(ref, var, m, tok, device=DEV, max_tokens=3000))


def _loop(m, B, P, n, per_row, **kw):
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
            logits, ipd = m(_tokens(B, P, seed=P).to(DEV), inference_params_dict=d)
            head, start = logits[:, -1], P
        picked, kept = m.decode_loop(head.float().argmax(-1), ipd, n, start, **kw)
        return head, picked.clone(), kept.clone()


@pytest.mark.parametrize("B", [16, 72])                      # 72: above the stream-K kernel's 64 rows, W' through the scratch
@pytest.mark.parametrize("per_row", [False, True])
@pytest.mark.parametrize("sampling", [False, True])
def test_decode_loop(pair, B, per_row, sampling):
    _both(pair, lambda m: _loop(m, B, 40, 10, per_row, **(SAMPLING if sampling else {"top_k": 1})))


@pytest.mark.parametrize("share", [False, True])
def test_generate_ragged_and_shared(pair, share):
    import evo_b200
    prompts = ["ACGTTGCAAC"] * 3 + ["GATTACA", "TTGACCA"]
    kw = dict(n_tokens=16, top_k=4, top_p=1.0, temperature=1.0, cached_generation=True, verbose=0, device=DEV, ragged=True, share_prompts=share)

    def run(m):
        torch.manual_seed(9)
        return evo_b200.generate(prompts, m, evo_b200.CharLevelTokenizer(512), **kw)
    _both(pair, run)


def test_bf16_comparator(pair):
    """_fp8_decode_bf16: the bf16 stream-K kernel on W' (for the compact model: the scratch) gives the FP8 kernel's bits."""
    _, fp8, compact = pair
    f8 = _loop(compact, 16, 40, 10, True, **SAMPLING)
    try:
        for m in (fp8, compact):
            m._fp8_decode_bf16 = True
        a, b = _both(pair, lambda m: _loop(m, 16, 40, 10, True, **SAMPLING))
    finally:
        for m in (fp8, compact):
            m._fp8_decode_bf16 = False
            m._decode = m._loop = None
    _same(a, f8)
    assert compact._w_scratch is not None and compact._tiled is None


# ------------------------------------------------------------------ memory
def _linear_shapes(m):
    return [(e.numel(), q.numel() // e.numel()) for _, _, mod, attr, _ in m._fp8_slots() for q, e in [m._compact_qe(mod, attr)]]


def test_memory_of_a_compact_model():
    torch.cuda.empty_cache()
    _, m = _model(**WIDE)
    shapes = [tuple(getattr(mod, attr).shape) for _, _, mod, attr, _ in m._fp8_slots()]
    before = torch.cuda.memory_allocated()
    m.quantize_fp8(compact=True)
    after = torch.cuda.memory_allocated()
    assert _linear_shapes(m) == shapes
    bf16 = sum(2 * n * k for n, k in shapes)
    kept = sum(n * k + n for n, k in shapes) + 2 * max(n * k for n, k in shapes)       # q + e, and the scratch
    assert before - after >= bf16 - kept, (before, after, bf16, kept)
    sizes = {n * k for n, k in shapes}
    for name, t in list(m.named_parameters()) + list(m.named_buffers()):
        assert not (t.dtype == torch.bfloat16 and t.numel() in sizes), name
    ids = _tokens(2, 200, seed=2).to(DEV)
    m(ids)
    assert m._w_scratch.numel() == max(n * k for n, k in shapes)
    del m
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ state
def _compact_state(m):
    return {(i, n): tuple(t.clone() for t in m._compact_qe(mod, attr)) for i, n, mod, attr, _ in m._fp8_slots()}


def _is_compact(m):
    return m._fp8_compact and all(getattr(mod, attr).numel() == 0 for _, _, mod, attr, _ in m._fp8_slots())


def test_state_dict_round_trip_reload_and_idempotence():
    cfg, fp8 = _model(seed=11)
    _, m = _model(seed=11)
    fp8.quantize_fp8()
    m.quantize_fp8(compact=True)
    sd, want = m.state_dict(), fp8.state_dict()
    _same(dict(sd), dict(want))
    assert all(v.device == torch.device(DEV) for v in sd.values())
    assert _is_compact(m)
    st = _compact_state(m)
    m.quantize_fp8(compact=True)                                # idempotent, and quantize_fp8() keeps a compact model compact
    m.quantize_fp8()
    assert _is_compact(m)
    _same(_compact_state(m), st)
    # the exported checkpoint loads into a fresh compact model with the same bits (of W': rounding W' again may pick e - 1 and
    # 2q for a row whose largest q rounded down to 224, the same W')
    _, fresh = _model(seed=12)
    fresh.quantize_fp8(compact=True)
    fresh.load_state_dict({k: v.cpu() for k, v in sd.items()}, strict=True)
    assert _is_compact(fresh)
    _same(dict(fresh.state_dict()), dict(sd))
    ids = _tokens(2, 150, seed=5).to(DEV)
    _same(fresh(ids)[0], fp8(ids)[0])
    # bf16 weights loaded into a compact model are rounded, and it stays compact
    _, plain = _model(seed=8)
    raw = plain.state_dict()
    m.load_state_dict(raw, strict=True)
    fp8.load_state_dict(raw, strict=True)
    assert _is_compact(m)
    _same(dict(m.state_dict()), dict(fp8.state_dict()))
    m._decode = m._loop = fp8._decode = fp8._loop = None
    _same(_loop(m, 4, 40, 6, False, top_k=1), _loop(fp8, 4, 40, 6, False, top_k=1))


def test_non_finite_weights_are_refused_and_leave_the_model():
    _, m = _model()
    with torch.no_grad():
        m.blocks[2].mlp.w3[5, 9] = float("nan")
    before = {k: v.clone() for k, v in m.state_dict().items()}
    with pytest.raises(_lib.EvoError, match="not finite"):
        m.quantize_fp8(compact=True)
    assert not m._fp8_mode and not m._fp8_compact
    _same(dict(m.state_dict()), before)
    # a compact model refuses a checkpoint with a non-finite linear weight before anything changes
    _, c = _model()
    c.quantize_fp8(compact=True)
    st, sd = _compact_state(c), c.state_dict()
    bad = {k: v.clone() for k, v in sd.items()}
    bad["blocks.1.mlp.l2.weight"][3, 4] = float("inf")
    bad["blocks.0.projections.bias"].add_(1)
    with pytest.raises(_lib.EvoError, match="blocks.1.mlp.l2.weight has a weight that is not finite"):
        c.load_state_dict(bad, strict=True)
    assert _is_compact(c)
    _same(_compact_state(c), st)
    _same(dict(c.state_dict()), dict(sd))


def test_device_round_trip_keeps_outputs_and_recaptures():
    _, m = _model()
    m.quantize_fp8(compact=True)
    a = _loop(m, 4, 40, 8, False, top_k=1)
    b72 = _loop(m, 72, 40, 4, False, top_k=1)
    loop0, q0 = m._loop, m.blocks[0].mlp.w12_q
    m.to("cpu")
    assert m.blocks[0].mlp.w12_q.device.type == "cpu" and m._loop is None and m._w_scratch is None
    m.to(DEV)
    assert _is_compact(m) and m.blocks[0].mlp.w12_q.device == torch.device(DEV)
    _same(_loop(m, 4, 40, 8, False, top_k=1), a)
    assert m._loop is not None and m._loop is not loop0 and m._loop["graph"] is not None
    _same(_loop(m, 72, 40, 4, False, top_k=1), b72)
    _same(m.blocks[0].mlp.w12_q, q0)


# ------------------------------------------------------------------ loading
def _write_checkpoint(cfg, sd, path, shards=2):
    from safetensors.torch import save_file
    keys = sorted(sd)
    index = {}
    for s in range(shards):
        name = f"model-{s + 1:05d}-of-{shards:05d}.safetensors"
        part = {("backbone." + k): (v if "poles" in k or "residues" in k else v.to(torch.bfloat16)).clone() for k in keys[s::shards] for v in [sd[k]]}
        save_file(part, os.path.join(path, name))
        index.update({k: name for k in part})
    with open(os.path.join(path, "model.safetensors.index.json"), "w") as f:
        json.dump({"weight_map": index}, f)
    import yaml
    with open(os.path.join(path, "config.yml"), "w") as f:
        yaml.safe_dump({k: list(v) if isinstance(v, tuple) else v for k, v in cfg.items()}, f)
    return os.path.join(path, "config.yml")


def test_streaming_load_never_holds_the_linear_weights_in_bf16(tmp_path):
    import evo_b200
    from evo_b200.models import load_checkpoint
    cfg = O.tiny_config(num_layers=WIDE["layers"], attn_layer_idxs=WIDE["attn"], hidden_size=WIDE["hidden"], num_heads=WIDE["heads"])
    conf = _write_checkpoint(cfg, O.random_state_dict(cfg, seed=21), str(tmp_path))
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m = load_checkpoint("evo-1-8k-base", config_path=conf, device=DEV, model_dir=str(tmp_path), weights="fp8-compact", streaming=True)
    peak = torch.cuda.max_memory_allocated() - base
    assert _is_compact(m) and m._fp8_mode
    footprint = sum(t.numel() * t.element_size() for t in list(m.parameters()) + list(m.buffers()))
    shapes = _linear_shapes(m)
    w12 = max(n * k for n, k in shapes) * 2
    other = max(2 * n * k for n, k in shapes if 2 * n * k != w12)
    assert peak <= footprint + 2 * w12 + other, (peak, footprint, w12, other)
    ref = load_checkpoint("evo-1-8k-base", config_path=conf, device=DEV, model_dir=str(tmp_path), weights="bf16").quantize_fp8(compact=True)
    _same(_compact_state(m), _compact_state(ref))
    _same(dict(m.state_dict()), dict(ref.state_dict()))
    ids = _tokens(2, 200, seed=6).to(DEV)
    _same(m(ids)[0], ref(ids)[0])
    del m, ref
    torch.cuda.empty_cache()
    # the front door: Evo(name, weights="fp8-compact", model_dir=...) generates and scores
    evo = evo_b200.Evo("evo-1-8k-base", device=DEV, config_path=conf, model_dir=str(tmp_path), weights="fp8-compact")
    assert _is_compact(evo.model)
    out, _ = evo_b200.generate(["ACGTACGT"], evo.model, evo.tokenizer, n_tokens=6, top_k=1, cached_generation=True, verbose=0, device=DEV)
    assert len(out) == 1 and len(out[0]) == 6
    s = evo_b200.score_sequences(["ACGTACGTTAGC", "ACGT"], evo.model, evo.tokenizer, device=DEV)
    assert len(s) == 2 and all(math.isfinite(x) for x in s)
