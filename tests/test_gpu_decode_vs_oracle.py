"""Decode steps against an independent reference: the oracle's stateful step (OracleStripedHyena with inference params:
a stateful prefill, then fir_step / iir_step and KV-cache attention at seqlen_offset with its own rotary tables), run on
the CPU in bf16 (the reference's rounding points) and in fp64 (fp32 at the 7B width) as the truth.

Every decode attention path is reached: the TMA-fed kernel (cache length % 64 == 0) and the per-thread-row kernel, the
scalar-position and per-row (_rows) forms, and the shared-prefix kernel with its two-source merge; at first keys, 64-key
tile edges, split edges, and the positions of the cached-generation workload (4096 and past, from an 8192-row cache).
Below the model: decode attention at the workload's geometry (B = 16, H = 32, 8192 rows) against fp64 softmax attention,
the rotary tables at long positions, the device loop's sampling bookkeeping, and the sampler on NaN and -inf logits.

Bars (those of test_model_logits_vs_oracle in test_gpu_parity.py), with e(x) = mean |log_softmax(x) - log_softmax(truth)|:
  * pooled over a case: e(GPU) <= 1.25 e(bf16 oracle) + eps, and the GPU's argmax agrees with the truth's at no fewer
    positions than the bf16 oracle's does, minus 3 points;
  * per step: e(GPU) <= 1.25 e(bf16 oracle) + eps at the same step, each averaged over the case's rows (8 to 16 distinct
    sequences per step, so that one step is a statistic rather than the noise of one or two rows);
  * logits finite, and the Hyena states after the last step as close to the truth's as the bf16 oracle's are: the mean
    |GPU - truth| within 1.25x the oracle's (+ 1e-4 of the mean |truth|), and the worst entry within 2x (+ 1e-4 of the
    largest |truth|).  test_decode_step_vs_oracle (test_gpu_hyena_paths.py) holds the worst entry to 1.25x for one
    operator fed identical inputs, where only that operator's rounding differs.  Here the two states also carry the
    independent bf16 noise of every block upstream, so their worst entries are extremes of two independent noise fields
    of equal mean (asserted above): two GPU paths on the same tokens (caches of 256 and 200 rows) differ by 1.4x in their
    worst entry at equal means.  The worst-entry bar guards against gross local errors; the mean carries the 1.25x."""
import ctypes as C
import math
import os
import sys
import time

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

from oracle import stripedhyena_oracle as O          # noqa: E402
from evo_b200 import _lib                             # noqa: E402
from evo_b200.stripedhyena import StripedHyena, dotdict  # noqa: E402
from tests.test_gpu_generation import dev_sample, host_pipeline_probs  # noqa: E402  (the sampler helpers of the sampler tests)

DEV = "cuda:0"
BF16_EPS = 2.0 ** -7
ROPE = {"plain": {}, "scaled16": {"use_interpolated_rotary_pos_emb": True, "rotary_emb_scaling_factor": 16}}


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()
    threads = torch.get_num_threads()
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    yield
    torch.set_num_threads(threads)


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _model(cfg, sd):
    m = StripedHyena(dotdict(cfg))
    m.load_state_dict(sd, strict=True)
    m.to_bfloat16_except_poles_residues()
    return m.to(DEV)


def _tiny(rope="plain", seed=7):
    cfg = O.tiny_config(num_layers=4, attn_layer_idxs=(1, 3), hidden_size=256, num_heads=2, **ROPE[rope])
    sd = O.random_state_dict(cfg, seed=seed)
    return cfg, sd, _model(cfg, sd)


def _tokens(B, L, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 4, (B, L), generator=g) * 3 + 65


def _lsm(x):
    return torch.log_softmax(x.double().cpu(), -1)


def _nsplit(B, H):
    """The decode attention's split count, as StripedHyena._decode_body_impl picks it."""
    n_sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    return max(1, min(16, -(-8 * n_sm // (H * B))))


# ------------------------------------------------------------------ the oracle's stateful step
def _oracle_decode(cfg, sd, dtype, prompt, steps):
    """The oracle's stateful prefill of prompt (B, P), then one token of steps (B, T) per call at seqlen_offset P + k, as
    evo/generation.py drives the reference.  Returns (step logits (B, T, V), the Hyena state holder, seconds)."""
    t0 = time.perf_counter()
    o = O.OracleStripedHyena(cfg, sd, dtype)
    ipd = o.initialize_inference_params()
    (B, P), T = prompt.shape, steps.shape[1]
    ipd["mha"].max_batch_size, ipd["mha"].max_seqlen = B, P + T
    o(prompt, ipd)
    k1 = cfg["short_filter_length"] - 1
    for i, fs in ipd["hyena"].fir_state_dict.items():
        if fs.shape[-1] < k1:
            # a prompt shorter than the FIR history: the causal conv1d sees zeros before the first token
            ipd["hyena"].fir_state_dict[i] = torch.cat([fs.new_zeros(*fs.shape[:-1], k1 - fs.shape[-1]), fs], -1)
    out = []
    for k in range(T):
        ipd["mha"].seqlen_offset = ipd["hyena"].seqlen_offset = P + k
        lg, _ = o(steps[:, k:k + 1], ipd)
        out.append(lg[:, 0])
    return torch.stack(out, 1), ipd["hyena"], time.perf_counter() - t0


def _oracle_pair(cfg, sd, prompt, steps, wide=torch.float64):
    lb, hb, tb = _oracle_decode(cfg, sd, torch.bfloat16, prompt, steps)
    lt, ht, tt = _oracle_decode(cfg, sd, wide, prompt, steps)
    return {"bf16": lb, "truth": lt, "hy_bf16": hb, "hy_truth": ht, "seconds": tb + tt}


def _gpu_per_token(m, prompt, steps, cache_len):
    """The per-token protocol on the GPU: stateful prefill, then m(ids[:, k:k+1]) with seqlen_offset advanced by the caller.
    Returns (step logits (B, T, V) bf16, the inference params dict)."""
    (B, P), T = prompt.shape, steps.shape[1]
    m._decode = m._loop = None
    d = m.initialize_inference_params()
    d["mha"].max_batch_size, d["mha"].max_seqlen = B, cache_len
    _, d = m(prompt.to(DEV), inference_params_dict=d)
    sd = steps.to(DEV)
    out = []
    for k in range(T):
        d["mha"].seqlen_offset = d["hyena"].seqlen_offset = P + k
        s, d = m(sd[:, k:k + 1], inference_params_dict=d)
        out.append(s[:, 0].cpu())
    return torch.stack(out, 1), d


class Errors:
    """Log-prob errors and argmax agreement of the GPU and of the bf16 oracle against the truth, pooled over the cases added."""

    def __init__(self, eps=2e-3):
        self.eps, self.n, self.agree_gpu, self.agree_ref = eps, 0, 0, 0

    def check_case(self, gpu, bf, truth, pos, where):
        """gpu, bf, truth: (B, T, V) logits of B rows over T steps; pos (B, T): the position each step ran at (for the report).
        The pooled bar over the case, and the per-step bar on the errors averaged over the B rows of each step."""
        assert torch.isfinite(gpu.float()).all(), where
        lt = _lsm(truth)
        e_gpu, e_ref = (_lsm(gpu) - lt).abs().mean(-1), (_lsm(bf) - lt).abs().mean(-1)      # (B, T)
        pooled_gpu, pooled_ref = e_gpu.mean().item(), e_ref.mean().item()
        step_gpu, step_ref = e_gpu.mean(0), e_ref.mean(0)
        ratio = step_gpu / step_ref
        worst = ratio.argmax().item()
        print(f"{where}: e_gpu {pooled_gpu:.4f} e_bf16 {pooled_ref:.4f}; worst step {worst} (positions {sorted(set(pos[:, worst].tolist()))[:4]}):"
              f" {step_gpu[worst]:.4f} vs {step_ref[worst]:.4f} ({ratio[worst]:.2f}x)")
        at = truth.argmax(-1)
        ok_gpu, ok_ref = gpu.float().argmax(-1) == at, bf.float().argmax(-1) == at
        top2 = lt.topk(2, -1).values
        for b, t in (~ok_gpu).nonzero().tolist():
            print(f"  argmax differs from the truth's: row {b} step {t} position {pos[b, t].item()}: truth top-2 margin "
                  f"{(top2[b, t, 0] - top2[b, t, 1]).item():.4f} nats, bf16 oracle {'agrees' if ok_ref[b, t] else 'differs too'}, "
                  f"|d log p| gpu {e_gpu[b, t]:.4f} bf16 {e_ref[b, t]:.4f}")
        self.n += at.numel()
        self.agree_gpu += int(ok_gpu.sum())
        self.agree_ref += int(ok_ref.sum())
        assert pooled_gpu <= 1.25 * pooled_ref + self.eps, (where, pooled_gpu, pooled_ref)
        bad = (step_gpu > 1.25 * step_ref + self.eps).nonzero().flatten().tolist()
        assert not bad, (where, "steps", bad, step_gpu[bad].tolist(), step_ref[bad].tolist())

    def check_agreement(self, where):
        assert self.agree_gpu >= self.agree_ref - 0.03 * self.n, (where, self.agree_gpu, self.agree_ref, self.n)


def _assert_hyena_states(gpu_hy, bf_hy, truth_hy, rows=slice(None), where=""):
    """Modal and FIR states after the last step against the truth's: the mean error within 1.25x the bf16 oracle's, the
    worst entry within 2x (see the module docstring)."""
    assert set(gpu_hy.state_dict) == set(truth_hy.state_dict)
    for i in truth_hy.state_dict:
        for name, g, b, t in (("state", gpu_hy.state_dict[i][rows], bf_hy.state_dict[i], truth_hy.state_dict[i]),
                              ("fir", gpu_hy.fir_state_dict[i][rows], bf_hy.fir_state_dict[i], truth_hy.fir_state_dict[i])):
            g, b, t = (x.cpu().to(torch.complex128) if x.is_complex() else x.cpu().double() for x in (g, b, t))
            assert g.shape == t.shape, (where, name, i, g.shape, t.shape)
            dg, db = (g - t).abs(), (b - t).abs()
            mean_t = t.abs().mean().item()
            assert math.isfinite(dg.mean().item()) and dg.mean().item() <= 1.25 * db.mean().item() + 1e-4 * mean_t, \
                (where, name, i, "mean", dg.mean().item(), db.mean().item())
            scale = max(1.0, t.abs().max().item())
            e_gpu, e_ref = dg.max().item() / scale, db.max().item() / scale
            print(f"  {where} {name}[{i}]: mean err gpu {dg.mean().item():.3g} bf16 {db.mean().item():.3g}; worst gpu {e_gpu:.3g} bf16 {e_ref:.3g}")
            assert e_gpu <= 2.0 * e_ref + 1e-4, (where, name, i, "max", e_gpu, e_ref)


def _positions(starts, T):
    return torch.as_tensor(starts, dtype=torch.int64)[:, None] + torch.arange(T)[None]


def _greedy_fed(first, picked):
    """The tokens a greedy decode_loop fed at its steps: first, then its own picks.  Teacher-forcing the oracle with them
    keeps near-ties from desynchronising the two."""
    return torch.cat([first[:, None], picked[:, :-1]], 1).cpu()


# ------------------------------------------------------------------ 1. decode steps vs the oracle
_SCALAR_ORACLE = {}


@pytest.mark.parametrize("cache_len", [256, 200])
@pytest.mark.parametrize("rope", ["plain", "scaled16"])
def test_decode_steps_vs_oracle_scalar_position(rope, cache_len):
    """Per-token protocol, B = 16, prompts of 1, 63, 64, 127, 128 and 129 tokens, 40 teacher-forced steps each: the first
    keys, the 64-key tile edges and the edges of the splits the tiny model's batch gets.  cache 256: the TMA-fed decode
    attention; cache 200 (not a multiple of 64): the per-thread-row kernel."""
    cfg, sd, m = _tiny(rope)
    B, T = 16, 40
    errs = Errors()
    for P in (1, 63, 64, 127, 128, 129):
        prompt, steps = _tokens(B, P, seed=P), _tokens(B, T, seed=1000 + P)
        prompt[:, 0] = 0
        key = (rope, P)
        if key not in _SCALAR_ORACLE:
            _SCALAR_ORACLE[key] = _oracle_pair(cfg, sd, prompt, steps)
            print(f"\noracle {rope} P={P}: {_SCALAR_ORACLE[key]['seconds']:.1f} s")
        ref = _SCALAR_ORACLE[key]
        got, d = _gpu_per_token(m, prompt, steps, cache_len)
        where = f"{rope} cache={cache_len} P={P}"
        errs.check_case(got, ref["bf16"], ref["truth"], _positions([P] * B, T), where)
        _assert_hyena_states(d["hyena"], ref["hy_bf16"], ref["hy_truth"], where=where)
    errs.check_agreement(f"{rope} cache={cache_len}")


@pytest.mark.parametrize("rope", ["plain", "scaled16"])
def test_decode_loop_vs_oracle_long_positions(rope):
    """The cached-generation workload's positions and cache shape: B = 8 prompts of 4090 tokens, then 24 greedy steps of the
    captured decode loop through positions 4096 and 4100, from an 8192-row cache (TMA kernel, 16 splits of 256+ keys)."""
    cfg, sd, m = _tiny(rope)
    B, P, T = 8, 4090, 24
    prompt = _tokens(B, P, seed=4090)
    prompt[:, 0] = 0
    m._decode = m._loop = None
    d = m.initialize_inference_params()
    d["mha"].max_batch_size, d["mha"].max_seqlen = B, 8192
    head, d = m(prompt.to(DEV), inference_params_dict=d)
    first = head[:, -1].float().argmax(-1)
    picked, kept = m.decode_loop(first, d, T, P, top_k=1)
    assert torch.equal(picked, kept.argmax(-1))
    ref = _oracle_pair(cfg, sd, prompt, _greedy_fed(first, picked))
    print(f"\noracle long {rope}: {ref['seconds']:.1f} s")
    errs = Errors()
    errs.check_case(kept.cpu(), ref["bf16"], ref["truth"], _positions([P] * B, T), f"long {rope}")
    errs.check_agreement(f"long {rope}")
    _assert_hyena_states(d["hyena"], ref["hy_bf16"], ref["hy_truth"], where=f"long {rope}")


def test_ragged_decode_loop_vs_oracle_per_row():
    """prefill_ragged + decode_loop with a (B,) start position (the _rows kernels): four prompts each of 5, 64, 300 and 1000
    tokens in one batch of 16, 32 greedy steps; every row against the oracle stepping its own prompt (batched by length:
    the oracle's rows are independent)."""
    cfg, sd, m = _tiny()
    T, k = 32, 4
    lengths = [L for L in (5, 64, 300, 1000) for _ in range(k)]
    prompts = [_tokens(1, L, seed=L + 10 * r)[0] for r, L in enumerate(lengths)]
    for p in prompts:
        p[0] = 0
    m._decode = m._loop = None
    head, ipd = m.prefill_ragged([p.tolist() for p in prompts], (max(lengths) + T + 63) // 64 * 64)
    first = head.float().argmax(-1)
    picked, kept = m.decode_loop(first, ipd, T, torch.tensor(lengths, dtype=torch.int64), top_k=1)
    fed = _greedy_fed(first, picked)
    bf, truth, secs = [], [], 0.0
    for r0 in range(0, len(lengths), k):
        ref = _oracle_pair(cfg, sd, torch.stack(prompts[r0:r0 + k]), fed[r0:r0 + k])
        secs += ref["seconds"]
        bf.append(ref["bf16"])
        truth.append(ref["truth"])
        _assert_hyena_states(ipd["hyena"], ref["hy_bf16"], ref["hy_truth"], rows=slice(r0, r0 + k), where=f"ragged rows {r0}..{r0 + k - 1}")
    print(f"\noracle ragged: {secs:.1f} s")
    errs = Errors()
    errs.check_case(kept.cpu(), torch.cat(bf), torch.cat(truth), _positions(lengths, T), "ragged")
    errs.check_agreement("ragged")


def test_shared_prompt_decode_loop_vs_oracle_per_row():
    """prefill_shared + decode_loop through evo_decode_attn_shared (prefix + suffix + merge), 24 greedy steps: eight prompts
    of 129, 700, 3, 64, 65, 128, 200 and 17 tokens with 3, 70 (a group above 64 rows), 2, 1, 1, 1, 1 and 1 rows.  Every row
    against the oracle on its own prompt + suffix.  In the 3-token group each prefix key carries a large share of the
    attention, so a prefix key lost shows."""
    cfg, sd, m = _tiny()
    T = 24
    lengths, rows = [129, 700, 3, 64, 65, 128, 200, 17], [3, 70, 2, 1, 1, 1, 1, 1]
    prompts = [_tokens(1, L, seed=L)[0] for L in lengths]
    for p in prompts:
        p[0] = 0
    m._decode = m._loop = None
    head, ipd = m.prefill_shared([p.tolist() for p in prompts], rows, T)
    starts = torch.tensor([L for L, n in zip(lengths, rows) for _ in range(n)], dtype=torch.int64)
    first = head.float().argmax(-1)
    picked, kept = m.decode_loop(first, ipd, T, starts, top_k=1)
    fed, kept = _greedy_fed(first, picked), kept.cpu()
    bf, truth, firsts, secs, r0 = [], [], [], 0.0, 0
    for g, (L, n) in enumerate(zip(lengths, rows)):
        ref = _oracle_pair(cfg, sd, prompts[g][None], fed[r0:r0 + 1])
        secs += ref["seconds"]
        for b in range(r0 + 1, r0 + n):                            # one group, greedy: every row is the group's first row, bit for bit
            assert torch.equal(fed[b], fed[r0]) and torch.equal(kept[b].view(torch.int32), kept[r0].view(torch.int32)), b
        for b in range(r0, r0 + n):
            _assert_hyena_states(ipd["hyena"], ref["hy_bf16"], ref["hy_truth"], rows=slice(b, b + 1), where=f"shared row {b}")
        bf.append(ref["bf16"])
        truth.append(ref["truth"])
        firsts.append(r0)
        r0 += n
    print(f"\noracle shared: {secs:.1f} s")
    errs = Errors()                                                 # one row per group: equal rows are one sample, not many
    errs.check_case(kept[firsts], torch.cat(bf), torch.cat(truth), _positions(lengths, T), "shared")
    errs.check_agreement("shared")


def test_decode_steps_vs_oracle_7b_width():
    """BASELINE configs[0]'s model (1 Hyena + 1 attention block at D = 4096, 32 heads), B = 8, a 256-token prompt, 24
    per-token steps from an 8192-row cache: the fused Hyena step epilogue at N = 12288, the stream-K GELU gate at N = 22016,
    and the decode attention at H = 32 (5 splits on 132 SMs).  Truth in fp32, as test_baseline_config0_two_layer_7b_width_L1024."""
    cfg = O.evo_config("evo-1-8k-base")
    cfg.update(num_layers=2, attn_layer_idxs=[1], hyena_layer_idxs=[0])
    sd = O.random_state_dict(cfg, seed=3)
    m = _model(cfg, sd)
    B, P, T = 8, 256, 24
    prompt, steps = _tokens(B, P, seed=256), _tokens(B, T, seed=257)
    got, d = _gpu_per_token(m, prompt, steps, 8192)
    ref = _oracle_pair(cfg, sd, prompt, steps, wide=torch.float32)
    print(f"\noracle 7B width: {ref['seconds']:.1f} s")
    errs = Errors()
    errs.check_case(got, ref["bf16"], ref["truth"], _positions([P] * B, T), "7B width")
    errs.check_agreement("7B width")
    _assert_hyena_states(d["hyena"], ref["hy_bf16"], ref["hy_truth"], where="7B width")


# ------------------------------------------------------------------ 2. decode attention at the workload's geometry
def _attend(q, k, v, scale):
    """q (H, 128), k/v (n, H, 128) on the device -> (H*128,) softmax attention in float64."""
    s = torch.einsum("hd,nhd->hn", q.double(), k.double()) * scale
    return torch.einsum("hn,nhd->hd", torch.softmax(s, -1), v.double()).reshape(-1)


@pytest.mark.parametrize("per_row", [False, True])
def test_decode_attention_at_gen_geometry(per_row):
    """B = 16, H = 32, an 8192-row cache (the TMA kernel): evo_decode_qkv_prep(_rows) + evo_decode_attn(_rows) at positions
    4095, 4096, 6000 and 8191 (the last row), or per-row positions spread over [4096, 8191]; nsplit 1, the model's choice
    and 16.  Cache rows past each row's position hold NaN.  Against fp64 softmax attention over the bf16 cache, with the
    rotary of O.rotary_tables; the appended K,V rows and the rotated q must be bit-exact (bf16 x bf16 products are exact
    in fp32, so the kernel's fused multiply-adds round as the oracle's separate operations do)."""
    B, H, S, hd = 16, 32, 8192, 128
    lib = _lib.lib()
    g = torch.Generator(device=DEV).manual_seed(31)
    base = torch.randn(B, S, 2, H, hd, generator=g, device=DEV).bfloat16()
    cos, sin = O.rotary_tables(S, hd, dtype=torch.bfloat16)
    cosd, sind = cos.to(DEV), sin.to(DEV)
    scale = 1 / math.sqrt(hd)
    prep = lib.evo_decode_qkv_prep_rows if per_row else lib.evo_decode_qkv_prep
    attn = lib.evo_decode_attn_rows if per_row else lib.evo_decode_attn
    if per_row:
        gp = torch.Generator().manual_seed(5)
        pos_sets = [[4096, 8191] + torch.randint(4096, 8192, (B - 2,), generator=gp).tolist()]
    else:
        pos_sets = [[p] * B for p in (4095, 4096, 6000, 8191)]
    splits = sorted({1, _nsplit(B, H), 16})
    if torch.cuda.get_device_properties(DEV).multi_processor_count == 132:
        assert _nsplit(B, H) == 3                                   # H100 SXM (132 SMs): the cached-generation workload's count
    for pos in pos_sets:
        cache = base.clone()
        for b, p in enumerate(pos):
            cache[b, p:] = float("nan")
        qkv0 = torch.randn(B, 3, H, hd, generator=g, device=DEV).bfloat16()
        qkv = qkv0.clone()
        posd = torch.tensor(pos if per_row else pos[:1], dtype=torch.int64, device=DEV)
        _lib.check(prep(_lib.ptr(qkv), _lib.ptr(cache), _lib.ptr(cosd), _lib.ptr(sind), _lib.ptr(posd), B, H, hd, S, stream()))
        q0 = qkv0.cpu()
        qr = torch.stack([O.apply_rotary(q0[b:b + 1, None, 0], cos[p:p + 1], sin[p:p + 1])[0, 0] for b, p in enumerate(pos)])
        kr = torch.stack([O.apply_rotary(q0[b:b + 1, None, 1], cos[p:p + 1], sin[p:p + 1])[0, 0] for b, p in enumerate(pos)])
        new_rows = torch.stack([cache[b, p] for b, p in enumerate(pos)]).cpu()          # (B, 2, H, hd)
        assert torch.equal(new_rows[:, 0].view(torch.int16), kr.view(torch.int16)), pos[:2]
        assert torch.equal(new_rows[:, 1].view(torch.int16), q0[:, 2].view(torch.int16)), pos[:2]
        assert torch.equal(qkv[:, 0].cpu().view(torch.int16), qr.view(torch.int16)), pos[:2]
        for b, p in enumerate(pos):                                                      # nothing else written
            assert torch.isnan(cache[b, p + 1:].float()).all() and torch.equal(cache[b, :p], base[b, :p])
        ref = torch.stack([_attend(qr[b].to(DEV), cache[b, :p + 1, 0], cache[b, :p + 1, 1], scale) for b, p in enumerate(pos)]).cpu()
        for nsplit in splits:
            n = lib.evo_decode_attn_workspace(B, H, nsplit)
            ws = torch.empty(n, dtype=torch.uint8, device=DEV)
            out = torch.empty(B, H * hd, dtype=torch.bfloat16, device=DEV)
            _lib.check(attn(_lib.ptr(qkv), _lib.ptr(cache), _lib.ptr(out), _lib.ptr(posd), B, H, hd, S, nsplit, scale, _lib.ptr(ws), n, stream()))
            o = out.double().cpu()
            assert not torch.isnan(o).any(), (pos[:2], nsplit)
            err = (o - ref).abs().max().item()
            assert err <= 4 * BF16_EPS * max(1.0, ref.abs().max().item()), (pos[:2], nsplit, err)
        del cache


# ------------------------------------------------------------------ 3. rotary tables at long positions
@pytest.mark.parametrize("scaling", [1.0, 16.0])
@pytest.mark.parametrize("pos0,L", [(4000, 300), (8192 - 300, 300), (131072 - 300, 300), (65536 - 150, 300)])
def test_rope_tables_at_long_positions(pos0, L, scaling):
    """evo_rope_tables from pos0 vs O.rotary_tables over the same window, with the bars of test_rope_tables_and_rotary: the
    angle t * inv_freq is one fp32 multiply on both sides and sincosf keeps IEEE accuracy (no --use_fast_math)."""
    cos_ref, sin_ref = (t[pos0:] for t in O.rotary_tables(pos0 + L, 128, scaling_factor=scaling, dtype=torch.bfloat16))
    inv = (1.0 / (10000 ** (torch.arange(0, 128, 2, dtype=torch.float32) / 128))).to(DEV)
    cd = torch.empty(L, 64, dtype=torch.bfloat16, device=DEV)
    sd = torch.empty_like(cd)
    _lib.check(_lib.lib().evo_rope_tables(_lib.ptr(cd), _lib.ptr(sd), _lib.ptr(inv), pos0, L, 64, scaling, stream()))
    c, s = cd.cpu(), sd.cpu()
    assert (c == cos_ref).float().mean() > 0.999 and (s == sin_ref).float().mean() > 0.999
    assert (c.double() - cos_ref.double()).abs().max().item() <= 2 ** -8
    assert (s.double() - sin_ref.double()).abs().max().item() <= 2 ** -8


# ------------------------------------------------------------------ 4. the device loop's bookkeeping and the sampler
SAMPLING = dict(top_k=4, top_p=0.9, temperature=0.7)


@pytest.mark.parametrize("per_row", [False, True])
def test_decode_loop_sampling_bookkeeping_is_exact(per_row):
    """decode_loop with top_k 4, top_p 0.9, temperature 0.7, a fixed seed and 5 forced tokens: nothing is recorded for the
    forced steps; picked[:, k] is evo_sample of kept_logits[:, k] keyed by (seed, step 5 + k, row); and
    kept_logits[:, k] are the per-token protocol's logits at step 5 + k fed the forced and picked tokens, bit for bit,
    which also shows that the forced tokens were the ones fed back.  Per-row positions: each row's per-token run is that
    row alone (B = 1)."""
    cfg, sd, m = _tiny()
    B, n_forced, n_out, seed = 3, 5, 20, 4321
    n = n_forced + n_out
    lengths = [40, 40, 40] if not per_row else [17, 40, 99]
    prompts = [_tokens(1, L, seed=L + b)[0] for b, L in enumerate(lengths)]
    forced = _tokens(B, n_forced, seed=99)
    m._decode = m._loop = None
    if per_row:
        head, ipd = m.prefill_ragged([p.tolist() for p in prompts], 192)
        start = torch.tensor(lengths, dtype=torch.int64)
    else:
        prompt = torch.stack(prompts)
        ipd = m.initialize_inference_params()
        ipd["mha"].max_batch_size, ipd["mha"].max_seqlen = B, 192
        head, ipd = m(prompt.to(DEV), inference_params_dict=ipd)
        head, start = head[:, -1], lengths[0]
    first = head.float().argmax(-1)
    picked, kept = m.decode_loop(first, ipd, n, start, forced=forced, seed=seed, **SAMPLING)
    assert picked.shape == (B, n_out) and kept.shape == (B, n_out, cfg["vocab_size"])
    picked, kept = picked.cpu(), kept.cpu()
    assert ((picked >= 0) & (picked < cfg["vocab_size"])).all()
    for k in range(n_out):
        lg = kept[:, k].bfloat16()
        assert torch.equal(lg.float(), kept[:, k])                       # the exact widening of bf16 logits
        assert torch.equal(dev_sample(lg, seed=seed, step=n_forced + k, **SAMPLING), picked[:, k]), k
    assert (picked != kept.argmax(-1)).any()                             # the loop really samples
    steps = torch.cat([first.cpu()[:, None], forced, picked[:, :-1]], 1)   # the tokens fed at steps 0 .. n-1
    if per_row:                                                          # each row alone, at its own position
        got = torch.cat([_gpu_per_token(m, prompts[b][None], steps[b:b + 1], 192)[0] for b in range(B)])
    else:
        got, _ = _gpu_per_token(m, prompt, steps, 192)
    assert torch.equal(got[:, n_forced:].float().view(torch.int32), kept.view(torch.int32))


def _row(V, seed):
    g = torch.Generator().manual_seed(seed)
    row = torch.randn(V, generator=g).bfloat16()
    head = torch.randperm(V, generator=g)[:4]
    row[head] += torch.tensor([4.0, 3.5, 3.0, 4.5]).bfloat16()
    return row, g


def _assert_draws_match(row, draws, top_k, top_p, temperature, bad):
    """draws of one row: in range, never an index in `bad`, and distributed as the host pipeline on the row with NaN -> -inf
    (the total-variation bar of test_sampler_distribution_matches_host_pipeline)."""
    V, N = row.shape[0], draws.shape[0]
    assert ((draws >= 0) & (draws < V)).all()
    assert not torch.isin(draws, bad).any(), draws[torch.isin(draws, bad)][:5]
    want = host_pipeline_probs(torch.where(torch.isnan(row), torch.tensor(float("-inf"), dtype=row.dtype), row), top_k, top_p, temperature).double()
    got = torch.bincount(draws, minlength=V).double() / N
    support = want > 0
    assert got[~support].sum().item() <= 2e-3
    tv = 0.5 * (got - want).abs().sum().item()
    noise = 0.5 * 0.8 * torch.sqrt(want * (1 - want) / N).sum().item()
    assert tv <= 2.0 * noise + 0.01, (tv, noise)


@pytest.mark.parametrize("V", [512, 40])
@pytest.mark.parametrize("n_nan", [1, 2, 37])
@pytest.mark.parametrize("top_k", [0, 4, -1])
def test_sampler_nan_logits_sort_last_and_weigh_nothing(V, n_nan, top_k):
    """NaN logits are never picked while a finite one exists, whatever top_k (-1 here: top_k = V), and the draws follow the
    host pipeline with NaN read as -inf.  One NaN sits on the row's largest logit."""
    top_k = V if top_k == -1 else top_k
    row, g = _row(V, seed=V + n_nan)
    amax, perm = row.float().argmax(), torch.randperm(V, generator=g)
    nan_at = torch.cat([amax[None], perm[perm != amax][:n_nan - 1]])
    row[nan_at] = float("nan")
    assert int(torch.isnan(row).sum()) == n_nan
    N = 40000
    for temperature, top_p in ((1.0, 1.0), (0.7, 0.9)):
        draws = dev_sample(row[None].expand(N, -1), top_k, top_p, temperature, seed=777)
        _assert_draws_match(row, draws, top_k, top_p, temperature, nan_at)
    greedy = dev_sample(row[None].expand(3, -1), 1, 0.0, 1.0)
    finite = torch.where(torch.isnan(row), torch.tensor(float("-inf"), dtype=row.dtype), row)
    assert (greedy == finite.float().argmax()).all()


def test_sampler_all_nan_row_and_inf_rows():
    """An all-NaN row gives an index in [0, V) for every top_k; -inf logits are never picked while a finite one exists, and
    the draws follow the host pipeline."""
    N = 40000
    for V in (512, 40):
        nan_row = torch.full((V,), float("nan"), dtype=torch.bfloat16)
        for top_k in (0, 1, 4, V):
            d = dev_sample(nan_row[None].expand(64, -1), top_k, 0.9, 0.7)
            assert ((d >= 0) & (d < V)).all(), (V, top_k)
        row, g = _row(V, seed=3 * V)
        ninf = torch.randperm(V, generator=g)[:V // 4]
        row[ninf] = float("-inf")
        for top_k in (0, 4, V):
            for temperature, top_p in ((1.0, 1.0), (0.7, 0.9)):
                draws = dev_sample(row[None].expand(N, -1), top_k, top_p, temperature, seed=778)
                _assert_draws_match(row, draws, top_k, top_p, temperature, ninf)
        one = torch.full((V,), float("-inf"), dtype=torch.bfloat16)
        one[V // 3] = 0.5
        for top_k in (0, 1, 4, V):
            assert (dev_sample(one[None].expand(64, -1), top_k, 0.9, 0.7) == V // 3).all(), (V, top_k)
