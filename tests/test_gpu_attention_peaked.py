"""Every online-softmax kernel where the softmax max moves: the prefill attention (batched, KV-cache and varlen forms), the
three decode attention kernels and their split merges, the shared-prefix kernel, and the fused scoring head -- on inputs whose
score pattern is known in advance, against float64.

Random unit-variance q and k (the other attention tests) give scores of standard deviation ~1: a row's max is settled by its
first key tile, no row is near one-hot, and the prefill kernel's lazy rescale (attention.cu: the reference m_ref moves only when
a tile's max exceeds it by more than 8 in log2 units) never fires.  Here q and k are built along chosen directions so that
    score(i, j) = q_i . k_j / sqrt(128)
follows a pattern: a ladder of one peak key per 128-key tile, each Delta log2 units above the last (7.5: P up to 2^7.5 with no
rescale; 8.5: one rescale per tile; 30: many; 130: alpha = ex2(-130) flushes to 0), a falling max, an attention sink, a
diagonal one-hot, two bitwise-identical keys tied at the top, |score| ~ 1e4, and q, k scaled by 4.  The float64 reference always
uses the bf16 tensors the kernels see, so rounding drift in the pattern does not matter; test_cases_reach_the_regimes_they_claim
checks, from those float64 scores, that the cases reach the regimes they are named for.

Bars (attention), each derived from the kernels' arithmetic:
  * no NaN, including with NaN in every cache row past a decode position;
  * meanerr(kernel, fp64) <= 1.25 * meanerr(bf16 oracle, fp64) + 1e-5, the oracle being O.causal_attention in bf16 (the rule
    of test_gpu_parity.py);
  * per (row, head): |out - fp64| <= 2 * 2^-7 * max|v| over the keys the row sees.  The output's bf16 rounding is <= 2^-9 of
    max|v| and P's bf16 rounding moves the weighted sum by <= 2^-9 of it; twice one bf16 ulp covers both with room;
  * one-hot rows (the top score >= 40 above every other visible one: sink, diagonal, ladder(130), huge): the output bits are
    V[argmax]'s bits.  Every other probability is < e^-40 < 2^-57.  The kept one is exactly 1 where m is that very score
    (the decode kernels, the comparator); in the prefill and prefix kernels it is ex2(fma(s, scale_log2, -m)) with
    m = fl(max(s) * scale_log2), i.e. ex2 of the product's rounding residual, at most 2^-24 |m|.  For |m| < 2^15 log2 units
    that is <= 2^-10, so p = 1 +- 2^-10.5 rounds to bf16 1 in the PV product while l keeps p, and out = v / p + O(2^-44) max|v|
    is within 2^-10 of v: it rounds back to v.  (Beyond 2^15 -- scores over ~22700 -- out may land one ulp off v; those
    rows are held to the two bars above only.)
  * tie rows (two bitwise-identical keys >= 40 above the rest, different v): the output bits are (v_a + v_b) / 2, chosen to be
    exactly a bf16 value with v_a, v_b of one sign and binade.  The two kept probabilities can differ by a rounding residual
    (and by split merge weights of 1 - O(1e-6)), which moves the result by O(1e-6) * |v_a - v_b| / 2 -- harmless next to the
    half ulp 2^-9 * |avg|, but it could flip a result that lands exactly on a rounding midpoint, which is why the average is
    made representable.
Scoring head: logprob error <= 2e-5 + 2^-21 * |lse| and entropy error <= 5e-5 + 2^-21 * max|logit| (fp32 statistics: a few
ulps of the largest magnitude in play, over the fixed 2e-5 / 5e-5 of test_gpu_fullsize.py), and evo_logprobs agrees with the
fused head within the logprob bar."""
import ctypes as C
import math
import os
import sys
from functools import lru_cache

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import stripedhyena_oracle as O          # noqa: E402
from evo_b200 import _lib                             # noqa: E402

DEV = "cuda:0"
HD = 128
TILE = 128                      # keys per tile of the prefill and prefix kernels
SCALE = 1 / math.sqrt(HD)
LOG2E = 1 / math.log(2)
BF16_EPS = 2.0 ** -7
GAP = 40.0                      # natural-log units: every other probability < e^-40
NAN = float("nan")


@pytest.fixture(scope="module")
def gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()        # raises if the extension is missing: no fallback


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------ constructed inputs
def _sum_vec(totals):
    """bf16 vectors (n, 128) with entries of about total/128 whose float64 sum is total to ~2^-9 of the last entry: with
    q = ones, q . k is then the chosen score to far better than one bf16 rounding of a single scalar would give."""
    totals = torch.as_tensor(totals, dtype=torch.float64).reshape(-1)
    out = torch.empty(totals.numel(), HD, dtype=torch.float64)
    acc = torch.zeros_like(totals)
    for d in range(HD):
        out[:, d] = ((totals - acc) / (HD - d)).bfloat16().double()
        acc += out[:, d]
    return out.bfloat16()


def _values(g, *shape):
    """V entries of magnitude 0.25 .. ~4, never 0, so a one-hot output is recognisably V[argmax] bit for bit."""
    x = torch.randn(*shape, generator=g)
    return (torch.sign(x) * (0.25 + x.abs())).bfloat16()


def _codes(g, *shape):
    return (torch.randint(0, 2, (*shape, HD), generator=g) * 2 - 1).to(torch.bfloat16)


def _tie_values(g, H):
    """(v_a, v_b) per head: same sign and binade in each dim, so (v_a + v_b) / 2 = s 2^e (1 + (a + b) / 128) is a bf16 value."""
    s = (torch.randint(0, 2, (H, HD), generator=g) * 2 - 1).double()
    e = torch.randint(-2, 2, (H, HD), generator=g).double()
    a, b = torch.randint(0, 64, (2, H, HD), generator=g).double()
    return (s * 2 ** e * (1 + 2 * a / 128)).bfloat16(), (s * 2 ** e * (1 + 2 * b / 128)).bfloat16()


def _ladder_peaks(L, delta, s0=6.0):
    """(key, natural-log score) of the ladder's peaks: one per 128-key tile, tile t at s0 + t * delta log2 units."""
    g = torch.Generator().manual_seed(int(delta * 10) + L)
    out = []
    for t in range((L + TILE - 1) // TILE):
        j = t * TILE + int(torch.randint(0, TILE, (1,), generator=g))
        if j < L:
            out.append((j, (s0 + t * delta) / LOG2E))
    return out


PREFILL_PATTERNS = ["ladder7.5", "ladder8.5", "ladder30", "ladder130", "falling", "sink", "diagonal", "tie", "huge", "random"]


def _prefill_seq(pattern, L, H, seed):
    """q, k, v (L, H, 128) bf16 of one sequence."""
    g = torch.Generator().manual_seed(seed)
    v = _values(g, L, H, HD)
    if pattern in ("diagonal", "huge", "random"):
        if pattern == "diagonal":        # q_i = 4 c_i, k_j = 2 c_j, c = random +-1 codes: self score 90.5, others ~ N(0, 8)
            c = _codes(g, L, H)
            return (4 * c.float()).bfloat16(), (2 * c.float()).bfloat16(), v
        if pattern == "huge":            # entries ~ +-200 and +-25, jittered so that scores do not tie: |score| ~ 1e4
            q = (200 * _codes(g, L, H).float() + 30 * torch.randn(L, H, HD, generator=g)).bfloat16()
            return q, (25 * _codes(g, L, H).float() + 4 * torch.randn(L, H, HD, generator=g)).bfloat16(), v
        return (4 * torch.randn(L, H, HD, generator=g)).bfloat16(), (4 * torch.randn(L, H, HD, generator=g)).bfloat16(), v
    # q = ones: score_j = sum(k_j) / sqrt(128); background keys N(0, 0.3^2) entries give scores ~ N(0, 0.3^2)
    q = torch.ones(L, H, HD, dtype=torch.bfloat16)
    k = (0.3 * torch.randn(L, H, HD, generator=g)).bfloat16()
    if pattern.startswith("ladder"):
        peaks = _ladder_peaks(L, float(pattern[6:]))
    elif pattern == "falling":           # tile 0 holds the max; every later tile's peak is 3 log2 units lower
        peaks = [(j, s - 3 / LOG2E if j >= TILE else s) for j, s in _ladder_peaks(L, 0.0, s0=17.0)]
    elif pattern == "sink":
        peaks = [(0, 50.0)]
    elif pattern == "tie":               # keys 3 and 200: one 50 above the rest, the other its bitwise copy
        peaks = [(j, 50.0) for j in (3, 200) if j < L]
    else:
        raise ValueError(pattern)
    for j, s in peaks:
        k[j] = _sum_vec([s * math.sqrt(HD)] * H).view(H, HD)
    if pattern == "tie" and L > 200:
        k[200] = k[3]
        v[3], v[200] = _tie_values(g, H)
    return q, k, v


@lru_cache(maxsize=None)
def prefill_case(pattern, L, B=2, H=2):
    qs, ks, vs = zip(*[_prefill_seq(pattern, L, H, seed=1000 * b + L + 7 * PREFILL_PATTERNS.index(pattern)) for b in range(B)])
    return torch.stack(qs), torch.stack(ks), torch.stack(vs)


# ------------------------------------------------------------------ float64 reference on row subsets
def _rows_subset(L):
    """First 130 rows, three on each side of every tile boundary, last 130 rows."""
    r = set(range(min(L, 130))) | set(range(max(0, L - 130), L))
    for t in range(TILE, L, TILE):
        r |= set(range(t - 3, min(L, t + 3)))
    return sorted(r)


def _runs(rows):
    out, start = [], rows[0]
    for a, b in zip(rows, rows[1:] + [None]):
        if b != a + 1:
            out.append((start, a + 1))
            start = b
    return out


def _scores(q, k, rows, pos0):
    """float64 scores (H, n, Lk) of query rows `rows` (positions pos0 + row) of q (Lq, H, 128) against k (Lk, H, 128)."""
    s = torch.einsum("nhd,jhd->hnj", q[rows].double(), k.double()) * SCALE
    mask = torch.arange(k.shape[0])[None, :] > (torch.tensor(rows)[:, None] + pos0)
    return s.masked_fill(mask[None], -math.inf)


def reference(q, k, v, rows, pos0=0):
    """For one sequence: fp64 truth, the bf16 oracle, the per-row max|v| bound, and the rows whose output is known bit for bit
    (one-hot: V[argmax]; tie: the average of the two tied values)."""
    H = q.shape[1]
    s = _scores(q, k, rows, pos0)
    truth = torch.einsum("hnj,jhd->nhd", torch.softmax(s, -1), v.double())
    oracle = torch.cat([O.causal_attention(q[None, a:b], k[None, :pos0 + b], v[None, :pos0 + b], q_offset=pos0 + a)[0]
                        for a, b in _runs(list(rows))])
    vmax = v.abs().amax(-1).double().cummax(0).values[torch.tensor(rows) + pos0]          # (n, H)
    nk = min(3, k.shape[0])
    top, idx = s.topk(nk, -1)                                                             # (H, n, nk)
    if nk < 3:
        top = torch.cat([top, torch.full((H, len(rows), 3 - nk), -math.inf, dtype=top.dtype)], -1)
    vv = v.double()
    hh = torch.arange(H)[:, None].expand(H, len(rows))
    moderate = top[..., 0].abs() * LOG2E < 2 ** 15             # see the module docstring: beyond, bf16(p) = 1 != l = p
    one_hot = (top[..., 0] - top[..., 1] >= GAP) & moderate
    tie = (top[..., 0] == top[..., 1]) & (top[..., 0] - top[..., 2] >= GAP) & moderate
    va = vv[idx[..., 0], hh]
    vb = vv[idx[..., min(1, nk - 1)], hh]
    avg = (va + vb) / 2
    tie &= (avg.bfloat16().double() == avg).all(-1)            # only the constructed ties: a chance tie may sit on a midpoint
    expect = torch.where(tie[..., None], avg, va).bfloat16()                              # (H, n, 128)
    return dict(truth=truth, oracle=oracle, vmax=vmax, exact=(one_hot | tie).T, expect=expect.transpose(0, 1), scores=s)


def check(out, ref, what):
    """The attention bars of the module docstring.  out (n, H, 128) bf16 on the CPU."""
    out = out.cpu()
    assert not torch.isnan(out.float()).any(), what
    e_gpu = (out.double() - ref["truth"]).abs().mean().item()
    e_ref = (ref["oracle"].double() - ref["truth"]).abs().mean().item()
    assert e_gpu <= 1.25 * e_ref + 1e-5, (what, e_gpu, e_ref)
    row_err = (out.double() - ref["truth"]).abs().amax(-1)
    bound = 2 * BF16_EPS * ref["vmax"]
    assert (row_err <= bound).all(), (what, (row_err / bound).max().item())
    ex = ref["exact"]
    if ex.any():
        got, want = out[ex].view(torch.int16), ref["expect"][ex].view(torch.int16)
        assert torch.equal(got, want), (what, int(ex.sum()), int((got != want).any(-1).sum()))


# ------------------------------------------------------------------ regime analysis (CPU)
def lazy_rescale_events(s):
    """Per row of fp64 scores s (n, Lk) in natural units, replay the prefill kernel's reference update over 128-key tiles in
    log2 units: (number of rescales, largest growth of a tile max over the reference that stayed <= 8, smallest and largest
    jump that caused a rescale)."""
    s2 = (s * LOG2E).numpy()
    n, Lk = s2.shape
    nt = (Lk + TILE - 1) // TILE
    pad = np.full((n, nt * TILE), -np.inf)
    pad[:, :Lk] = s2
    tmax = pad.reshape(n, nt, TILE).max(-1)
    events = np.zeros(n, int)
    under = np.full(n, -np.inf)
    jmin, jmax = np.full(n, np.inf), np.full(n, -np.inf)
    m_ref = tmax[:, 0].copy()
    for t in range(1, nt):
        mx = tmax[:, t]
        up = mx - m_ref
        ev = up > 8
        events += ev
        jmin = np.where(ev, np.minimum(jmin, up), jmin)
        jmax = np.where(ev, np.maximum(jmax, up), jmax)
        under = np.where(~ev & np.isfinite(mx), np.maximum(under, up), under)
        m_ref = np.where(ev, mx, m_ref)
    return events, under, jmin, jmax


def split_ranges(nk, nsplit, tile):
    """Key ranges of the decode kernels' splits: ceil(nk / nsplit) keys each, rounded up to `tile` (64 for the TMA-fed kernel,
    128 for the prefix kernel, 1 for the per-thread-row kernel)."""
    per = (nk + nsplit - 1) // nsplit
    per = (per + tile - 1) // tile * tile
    return [(a, min(nk, a + per)) for a in range(0, nk, per)]


def split_weights(s, nk, nsplit, tile):
    """fp32 merge weight exp(m_s - M) of each non-empty split, and each split's share of the float64 mass."""
    sp = split_ranges(nk, nsplit, tile)
    m = np.array([s[a:b].max() for a, b in sp], dtype=np.float32)
    w = np.exp(m - m.max())
    mass = np.array([np.exp(s[a:b].astype(np.float64) - s[:nk].max()).sum() for a, b in sp])
    return w, mass / mass.sum()


# ------------------------------------------------------------------ decode inputs
DECODE_PATTERNS = ["first", "last", "sink", "random"]
D_GAP = {"first": 45.0, "last": 45.0, "sink": 120.0}     # 120: every other split's merge weight underflows to exactly 0


def decode_case(patterns, positions, S, H=2, seed=0):
    """qkv (B, 3, H, 128) with q only (k, v slots NaN: the kernels must not read them), cache (B, S, 2, H, 128) with NaN in
    every row past the row's position.  Row b follows patterns[b]: its peak key (the first split's key 1, the newest key, or
    key 0 as a sink) stands D_GAP above a N(0, 0.3^2) background; 'random' is q, k ~ N(0, 4^2) (score std ~16)."""
    g = torch.Generator().manual_seed(seed)
    B = len(patterns)
    qkv = torch.full((B, 3, H, HD), NAN, dtype=torch.bfloat16)
    cache = torch.full((B, S, 2, H, HD), NAN, dtype=torch.bfloat16)
    for b, (pat, pos) in enumerate(zip(patterns, positions)):
        nk = pos + 1
        cache[b, :nk, 1] = _values(g, nk, H, HD)
        if pat == "random":
            qkv[b, 0] = (4 * torch.randn(H, HD, generator=g)).bfloat16()
            cache[b, :nk, 0] = (4 * torch.randn(nk, H, HD, generator=g)).bfloat16()
            continue
        qkv[b, 0] = 1.0
        cache[b, :nk, 0] = (0.3 * torch.randn(nk, H, HD, generator=g)).bfloat16()
        j = {"first": min(1, pos), "last": pos, "sink": 0}[pat]
        cache[b, j, 0] = _sum_vec([D_GAP[pat] * math.sqrt(HD)] * H).view(H, HD)
    return qkv, cache


def decode_reference(qkv, cache, positions):
    refs = [reference(qkv[b, 0][None], cache[b, :p + 1, 0], cache[b, :p + 1, 1], [0], pos0=p) for b, p in enumerate(positions)]
    return {key: torch.cat([r[key] for r in refs]) if key != "scores" else [r[key] for r in refs] for key in refs[0]}


# shared prefix: groups of rows with prefix lengths 1, 128, 129, 2049; Hadamard codes c_A (prefix peak), c_B (suffix peak),
# c_T (the tied key, bitwise the same in the prefix and the suffix) are exactly orthogonal, so a row's q = 2 c selects its peak
SH_ROWS = [2, 1, 2, 2]
SH_PLEN = [1, 128, 129, 2049]
SH_SPOS = [5, 63, 64, 300, 1, 130, 309]
SH_PATTERNS = ["prefix", "suffix", "tie"]
SH_BETA = {"prefix": 2.75, "suffix": 5.5, "tie": 2.75}     # peak score 2 * beta * 128 / sqrt(128): 62, 124, 62


def _hadamard(n):
    h = torch.ones(1, 1)
    while h.shape[0] < n:
        h = torch.cat([torch.cat([h, h], 1), torch.cat([h, -h], 1)])
    return h


def shared_case(S, H=2, seed=0):
    g = torch.Generator().manual_seed(seed)
    had = _hadamard(HD)
    code = {"prefix": had[1], "suffix": had[2], "tie": had[3]}
    G, B = len(SH_ROWS), sum(SH_ROWS)
    P = (max(SH_PLEN) + 63) // 64 * 64
    group = [k for k, n in enumerate(SH_ROWS) for _ in range(n)]
    pcache = torch.full((G, P, 2, H, HD), NAN, dtype=torch.bfloat16)
    tie_v = [_tie_values(g, H) for _ in range(B)]
    for k, n in enumerate(SH_PLEN):
        pcache[k, :n, 0] = (0.15 * torch.randn(n, H, HD, generator=g)).bfloat16()
        pcache[k, :n, 1] = _values(g, n, H, HD)
        pcache[k, n - 1, 0] = (SH_BETA["prefix"] * code["prefix"]).bfloat16()       # the prefix's last key: alone in its tile at 2049
        if n > 1:
            pcache[k, n // 2, 0] = (SH_BETA["tie"] * code["tie"]).bfloat16()
    spos = [SH_SPOS[b % len(SH_SPOS)] for b in range(B)]
    scache = torch.full((B, S, 2, H, HD), NAN, dtype=torch.bfloat16)
    qkv = torch.full((B, 3, H, HD), NAN, dtype=torch.bfloat16)
    pats = [SH_PATTERNS[b % 3] for b in range(B)]
    for b, p in enumerate(spos):
        scache[b, :p + 1, 0] = (0.15 * torch.randn(p + 1, H, HD, generator=g)).bfloat16()
        scache[b, :p + 1, 1] = _values(g, p + 1, H, HD)
        scache[b, p // 2, 0] = (SH_BETA["suffix"] * code["suffix"]).bfloat16()
        scache[b, p, 0] = (SH_BETA["tie"] * code["tie"]).bfloat16()
        qkv[b, 0] = (2 * code[pats[b]]).bfloat16()
        n = SH_PLEN[group[b]]
        if pats[b] == "tie" and n > 1:                     # this row's own tied pair: prefix key n // 2 and suffix key p
            pcache[group[b], n // 2, 1], scache[b, p, 1] = tie_v[b]
    # rows of one group share the prefix: a tie row's prefix value must not be overwritten by a later row of the group
    assert all(sum(1 for c in range(B) if group[c] == k and pats[c] == "tie") <= 1 for k in range(G))
    refs = []
    for b in range(B):
        n = SH_PLEN[group[b]]
        k_ = torch.cat([pcache[group[b], :n, 0], scache[b, :spos[b] + 1, 0]])
        v_ = torch.cat([pcache[group[b], :n, 1], scache[b, :spos[b] + 1, 1]])
        refs.append(reference(qkv[b, 0][None], k_, v_, [0], pos0=k_.shape[0] - 1))
    ref = {key: torch.cat([r[key] for r in refs]) for key in refs[0] if key != "scores"}
    ref["scores"] = [r["scores"] for r in refs]
    return dict(H=H, G=G, B=B, P=P, S=S, pcache=pcache, scache=scache, qkv=qkv, spos=spos, group=group, pats=pats,
                offs=torch.tensor([0] + SH_ROWS).cumsum(0), ref=ref)


# ------------------------------------------------------------------ scoring inputs
SCORE_KINDS = ["cross_half", "one_hot", "uniform", "offset80", "offset80_one_hot", "random"]


def score_case(M, V, seed=0):
    """x (M, V + 64), W (V, V + 64) with W = [I | 10 e_0]: the logits are x[:, :V] + 10 x[:, V] exactly (one nonzero product
    per column besides the constant one), so every summation order gives the same fp32 logit and its bf16 rounding is known.
    Row r is of kind SCORE_KINDS[r % 6]: max in the upper half with the target deep in the lower one (logprob ~ -60), a 40-nat
    one-hot, all logits equal, a +80 common offset from the constant column, both, or N(0, 1.75^2)."""
    g = torch.Generator().manual_seed(seed + M + V)
    K = V + 64
    z = 1.75 * torch.randn(M, V, generator=g)
    off = torch.zeros(M)
    tg = torch.randint(0, V, (M,), generator=g)
    for r in range(M):
        kind = SCORE_KINDS[r % len(SCORE_KINDS)]
        if kind == "cross_half":
            z[r] = torch.randn(V, generator=g)
            z[r, V // 2 + int(torch.randint(0, V // 2, (1,), generator=g))] = 30
            tg[r] = int(torch.randint(0, V // 2, (1,), generator=g))
            z[r, tg[r]] = -30
        elif kind in ("one_hot", "offset80_one_hot"):
            z[r] = torch.randn(V, generator=g)
            z[r, int(torch.randint(0, V, (1,), generator=g))] = 40
        elif kind == "uniform":
            z[r] = 1.5
        if kind.startswith("offset80"):
            off[r] = 8
    if M > 7:
        tg[7] = -1
    x = torch.zeros(M, K)
    x[:, :V] = z
    x[:, V] = off
    w = torch.zeros(V, K)
    w[:, :V] = torch.eye(V)
    w[:, V] = 10
    x, w = x.bfloat16(), w.bfloat16()
    logits = (x[:, :V].double() + 10 * x[:, V:V + 1].double()).bfloat16()      # exact in fp32, then the kernel's one rounding
    lsm = torch.log_softmax(logits.double(), -1)
    lse = torch.logsumexp(logits.double(), -1)
    lp = lsm.gather(1, tg.clamp(min=0)[:, None])[:, 0]
    lp[tg < 0] = 0
    ent = -(lsm.exp() * lsm).sum(-1)
    return dict(x=x, w=w, tg=tg, logits=logits, lp=lp, ent=ent, lse=lse, K=K)


# ------------------------------------------------------------------ the premise, on the CPU
def test_cases_reach_the_regimes_they_claim():
    L = 2500
    ev = {}
    for pat in ("ladder7.5", "ladder8.5", "ladder30", "ladder130"):
        q, k, v = prefill_case(pat, L)
        rows = _rows_subset(L)
        s = _scores(q[0], k[0], rows, 0)[0]
        ev[pat] = lazy_rescale_events(s)
    n_ev, under, jmin, jmax = (np.concatenate(x) for x in zip(*ev.values()))
    assert ((n_ev == 0) & (under > 7) & (under <= 8)).any(), "no row with P up to 2^7..2^8 and no rescale"
    assert ((n_ev >= 1) & (jmin > 8) & (jmin <= 9)).any(), "no row rescaled by a jump just over the threshold"
    assert (n_ev >= 3).any(), "no row with three or more rescales"
    assert (jmax > 126).any(), "no row whose rescale factor flushes to 0"
    assert (ev["ladder7.5"][0] == 0).any() and (ev["ladder7.5"][0] >= 1).any()
    # falling: the max stays in tile 0, later tiles 3 log2 units lower still count
    q, k, v = prefill_case("falling", L)
    s = _scores(q[0], k[0], [L - 1], 0)[0]
    n_ev, under, _, _ = lazy_rescale_events(s)
    assert n_ev[0] == 0 and abs(under[0] + 3) < 0.5
    # one-hot and tie rows exist where the docstring says
    for pat in ("sink", "diagonal", "ladder130", "huge", "tie"):
        q, k, v = prefill_case(pat, 1000)
        r = reference(q[0], k[0], v[0], _rows_subset(1000))
        assert r["exact"].float().mean() > 0.5, pat
    q, k, v = prefill_case("diagonal", 1000)
    s = _scores(q[0], k[0], list(range(1000)), 0)
    assert (s.argmax(-1) == torch.arange(1000)).all()                          # the argmax is the last visible key, every in-tile slot
    q, k, v = prefill_case("tie", 1000)
    s = _scores(q[0], k[0], [999], 0)[0, 0]
    top = s.topk(3).values
    assert top[0] == top[1] and top[0] - top[2] >= GAP
    q, k, v = prefill_case("huge", 1000)
    assert _scores(q[0], k[0], [999], 0).abs().max() > 1e4 and q.float().abs().max() >= 200
    q, k, v = prefill_case("random", 1000)
    assert 12 < _scores(q[0], k[0], [999], 0)[0, 0].std() < 20
    # decode: a split whose merge weight is exactly 0 in fp32, and a split that holds all the mass
    zero_w = all_mass = False
    for pat in ("first", "last", "sink"):
        qkv, cache = decode_case([pat], [599], 640)
        s = (torch.einsum("d,jd->j", qkv[0, 0, 0].double(), cache[0, :600, 0, 0].double()) * SCALE).numpy()
        for nsplit in (3, 4):
            w, share = split_weights(s, 600, nsplit, 64)
            zero_w |= bool((w == 0).any())
            all_mass |= bool((share.astype(np.float32) == 1).any() and len(share) > 1)
    assert zero_w and all_mass
    c = shared_case(310)
    kinds = set()
    for b in range(c["B"]):
        s = c["ref"]["scores"][b][0, 0]
        n = SH_PLEN[c["group"][b]]
        top = s.topk(2)
        if c["ref"]["exact"][b].all():
            kinds.add("prefix" if top.indices[0] < n and top.values[0] != top.values[1] else
                      "suffix" if top.values[0] != top.values[1] else "tie")
    assert kinds == {"prefix", "suffix", "tie"}, kinds
    # scoring: one-hot entropy < 1e-6, uniform entropy ln V, cross-half logprob ~ -60 with max and target in different halves
    for V in (256, 512):
        sc = score_case(129, V)
        kind = [SCORE_KINDS[r % len(SCORE_KINDS)] for r in range(129)]
        for r in range(129):
            if kind[r] in ("one_hot", "offset80_one_hot"):
                assert sc["ent"][r] < 1e-6
            if kind[r] == "uniform":
                assert abs(sc["ent"][r] - math.log(V)) < 1e-12
            if kind[r] == "cross_half" and r != 7:
                assert sc["logits"][r].argmax() >= V // 2 and sc["tg"][r] < V // 2 and -61 < sc["lp"][r] < -59
            if kind[r].startswith("offset80"):
                assert sc["logits"][r].double().mean() > 75


# ------------------------------------------------------------------ prefill
def _attn(q, k, v, q_pos0, variant, simple=False, cache_rows=None):
    """evo_attn_fwd_ws (or the CUDA-core comparator) on q (B, Lq, H, 128) and keys / values (B, Lk, H, 128); with cache_rows,
    k and v sit in a (B, cache_rows, 2, H, 128) cache whose rows past Lk are NaN."""
    B, Lq, H, _ = q.shape
    Lk = k.shape[1]
    d = H * HD
    qd = q.to(DEV).contiguous()
    out = torch.full((B, Lq, d), NAN, dtype=torch.bfloat16, device=DEV)
    ap = _lib.AttnParams(out=out.data_ptr(), B=B, Lq=Lq, Lk=Lk, H=H, hd=HD, q_pos0=q_pos0, softmax_scale=SCALE)
    ap.q, ap.q_tok_stride, ap.q_batch_stride = qd.data_ptr(), d, Lq * d
    if cache_rows is None:
        kd, vd = k.to(DEV).contiguous(), v.to(DEV).contiguous()
        ap.k, ap.v, ap.kv_tok_stride, ap.kv_batch_stride = kd.data_ptr(), vd.data_ptr(), d, Lk * d
    else:
        cache = torch.full((B, cache_rows, 2, H, HD), NAN, dtype=torch.bfloat16)
        cache[:, :Lk, 0], cache[:, :Lk, 1] = k, v
        kd = cache.to(DEV)
        ap.k, ap.v, ap.kv_tok_stride, ap.kv_batch_stride = kd.data_ptr(), kd.data_ptr() + d * 2, 2 * d, cache_rows * 2 * d
    if simple:
        from tests import support as TS
        TS.check(TS.lib().evot_attn_fwd_simple(C.byref(ap), stream()), "evot_attn_fwd_simple")
    else:
        _lib.check(_lib.lib().evo_attn_fwd_ws(C.byref(ap), variant, None, 0, stream()), "evo_attn_fwd_ws")
    torch.cuda.synchronize()
    return out.view(B, Lq, H, HD).cpu()


@lru_cache(maxsize=None)
def _prefill_refs(pattern, L, B=2, H=2):
    q, k, v = prefill_case(pattern, L, B, H)
    rows = _rows_subset(L)
    return rows, [reference(q[b], k[b], v[b], rows) for b in range(B)]


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 127, 128, 129, 1000, 2500])
@pytest.mark.parametrize("pattern", PREFILL_PATTERNS)
def test_prefill_attention_peaked(gpu, pattern, L):
    """evo_attn_fwd_ws, variants 1 and 0, B = 2, H = 2, and the CUDA-core comparator the other attention tests trust."""
    q, k, v = prefill_case(pattern, L)
    rows, refs = _prefill_refs(pattern, L)
    for variant in (1, 0, "simple"):
        out = _attn(q, k, v, 0, 0 if variant == "simple" else variant, simple=variant == "simple")
        for b in range(2):
            check(out[b, rows], refs[b], (pattern, L, variant, b))


@pytest.mark.gpu
@pytest.mark.parametrize("q_pos0", [127, 255])
@pytest.mark.parametrize("pattern", ["ladder8.5", "ladder130", "falling", "sink", "diagonal", "tie"])
def test_prefill_attention_peaked_kv_cache_form(gpu, pattern, q_pos0):
    """Queries [q_pos0, q_pos0 + 200) -- two query blocks -- against a 640-row cache holding keys [0, q_pos0 + 200), NaN after."""
    Lq = 200
    L = q_pos0 + Lq
    q, k, v = prefill_case(pattern, L)
    rows = list(range(Lq))
    for variant in (1, 0):
        out = _attn(q[:, q_pos0:], k, v, q_pos0, variant, cache_rows=640)
        for b in range(2):
            ref = reference(q[b, q_pos0:], k[b], v[b], rows, pos0=q_pos0)
            check(out[b], ref, (pattern, q_pos0, variant, b))


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", ["ladder8.5", "ladder130", "diagonal", "random"])
def test_prefill_attention_peaked_8193(gpu, pattern):
    """L = 8193 (8192 nt + BOS): the wgmma kernel against the CUDA-core comparator on every row, and both against fp64 on
    the row subset (first 130 rows, rows around every tile boundary, last 130 rows)."""
    L = 8193
    q, k, v = prefill_case(pattern, L, B=1)
    rows, refs = _prefill_refs(pattern, L, B=1)
    a = _attn(q, k, v, 0, 1)
    c = _attn(q, k, v, 0, 0, simple=True)
    assert not torch.isnan(a.float()).any() and not torch.isnan(c.float()).any()
    vmax = v[0].abs().amax(-1).double().cummax(0).values                   # (L, H): max|v| over the keys each row sees
    assert ((a[0].double() - c[0].double()).abs().amax(-1) <= 4 * BF16_EPS * vmax).all()
    check(a[0, rows], refs[0], (pattern, "wgmma"))
    check(c[0, rows], refs[0], (pattern, "comparator"))


def _cu(lengths):
    return [0] + list(np.cumsum(lengths))


@pytest.mark.gpu
def test_varlen_attention_peaked_sequences_stay_apart(gpu):
    """evo_attn_fwd_varlen on lengths 1, 129, 700, 2500 packed together, each with its own pattern: a sink (129) next to a
    diagonal one-hot (700) must not leak into it, and every sequence meets its own fp64 reference."""
    H = 2
    seqs = [("random", 1), ("sink", 129), ("diagonal", 700), ("ladder30", 2500)]
    parts = [_prefill_seq(p, L, H, seed=50 + i) for i, (p, L) in enumerate(seqs)]
    lengths = [L for _, L in seqs]
    T, d = sum(lengths), H * HD
    qkv = torch.cat([torch.stack([q, k, v], 1) for q, k, v in parts]).reshape(T, 3 * d)     # (T, 3, H, 128) rows
    qd = qkv.to(DEV)
    cu = torch.tensor(_cu(lengths), dtype=torch.int64, device=DEV)
    out = torch.full((T, d), NAN, dtype=torch.bfloat16, device=DEV)
    ap = _lib.AttnVarlenParams(q=qd.data_ptr(), k=qd.data_ptr() + d * 2, v=qd.data_ptr() + 2 * d * 2, out=out.data_ptr(),
                               q_tok_stride=3 * d, kv_tok_stride=3 * d, cu_seqlens=cu.data_ptr(), n_seq=len(lengths), T=T,
                               max_seqlen=max(lengths), H=H, hd=HD, softmax_scale=SCALE)
    _lib.check(_lib.lib().evo_attn_fwd_varlen(C.byref(ap), stream()), "evo_attn_fwd_varlen")
    torch.cuda.synchronize()
    out = out.view(T, H, HD).cpu()
    c = _cu(lengths)
    for (pat, L), (q, k, v), a in zip(seqs, parts, c):
        rows = _rows_subset(L)
        check(out[a:a + L][rows], reference(q, k, v, rows), (pat, L))


# ------------------------------------------------------------------ decode
def _decode(qkv, cache, pos, S, nsplit, rows):
    lib = _lib.lib()
    B, _, H, _ = qkv.shape
    n = lib.evo_decode_attn_workspace(B, H, nsplit)
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    out = torch.full((B, H * HD), NAN, dtype=torch.bfloat16, device=DEV)
    fn = lib.evo_decode_attn_rows if rows else lib.evo_decode_attn
    _lib.check(fn(_lib.ptr(qkv), _lib.ptr(cache), _lib.ptr(out), _lib.ptr(pos), B, H, HD, S, nsplit, SCALE, _lib.ptr(ws), n, stream()),
               "evo_decode_attn_rows" if rows else "evo_decode_attn")
    torch.cuda.synchronize()
    return out.view(B, H, HD).cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("S", [640, 600])          # 640: the TMA-fed kernel (64-key tiles); 600: the per-thread-row kernel
def test_decode_attention_peaked(gpu, S):
    """evo_decode_attn (one position for the batch) at positions 0, 63, 64, 599 and evo_decode_attn_rows (a position per row),
    nsplit 1, 3, 4: the peak in the first split only, in the last split only, a sink with every other split's merge weight
    exactly 0, and q, k ~ N(0, 4^2).  Cache rows past each position hold NaN."""
    for pos in (0, 63, 64, 599):
        qkv, cache = decode_case(DECODE_PATTERNS, [pos] * 4, S, seed=pos)
        ref = decode_reference(qkv, cache, [pos] * 4)
        qd, cd = qkv.to(DEV), cache.to(DEV)
        posd = torch.tensor([pos], dtype=torch.int64, device=DEV)
        for nsplit in (1, 3, 4):
            check(_decode(qd, cd, posd, S, nsplit, rows=False), ref, (S, pos, nsplit))
    positions = [0, 63, 64, 599, 599, 130, 599, 64]
    pats = DECODE_PATTERNS + ["sink", "first", "last", "random"]
    qkv, cache = decode_case(pats, positions, S, seed=S)
    ref = decode_reference(qkv, cache, positions)
    qd, cd = qkv.to(DEV), cache.to(DEV)
    posd = torch.tensor(positions, dtype=torch.int64, device=DEV)
    for nsplit in (1, 3, 4):
        check(_decode(qd, cd, posd, S, nsplit, rows=True), ref, (S, "rows", nsplit))


@pytest.mark.gpu
@pytest.mark.parametrize("S", [320, 310])          # the two suffix kernels
def test_shared_prefix_attention_peaked(gpu, S):
    """evo_decode_attn_shared: the peak in the prefix only, in the suffix only (every prefix split then weighs exactly 0), or
    one key tied bitwise across prefix and suffix; prefix lengths 1, 128, 129, 2049; splits (1, 1) and (4, 3)."""
    c = shared_case(S, seed=S)
    lib = _lib.lib()
    d = {key: c[key].to(DEV) for key in ("pcache", "scache", "qkv")}
    offs = c["offs"].to(DEV)
    plen = torch.tensor([SH_PLEN[g] for g in range(c["G"])], dtype=torch.int64, device=DEV)
    spos = torch.tensor(c["spos"], dtype=torch.int64, device=DEV)
    for nsp_p, nsp_s in ((1, 1), (4, 3)):
        n = lib.evo_decode_attn_shared_workspace(c["B"], c["H"], nsp_p, nsp_s)
        ws = torch.empty(n, dtype=torch.uint8, device=DEV)
        out = torch.full((c["B"], c["H"] * HD), NAN, dtype=torch.bfloat16, device=DEV)
        _lib.check(lib.evo_decode_attn_shared(_lib.ptr(d["qkv"]), _lib.ptr(d["pcache"]), _lib.ptr(offs), _lib.ptr(plen), c["G"], c["P"],
                                              _lib.ptr(d["scache"]), _lib.ptr(spos), S, _lib.ptr(out), c["B"], c["H"], HD, nsp_p, nsp_s,
                                              SCALE, _lib.ptr(ws), n, stream()), "evo_decode_attn_shared")
        torch.cuda.synchronize()
        check(out.view(c["B"], c["H"], HD).cpu(), c["ref"], (S, nsp_p, nsp_s))


# ------------------------------------------------------------------ scoring head
@pytest.mark.gpu
@pytest.mark.parametrize("V", [256, 512])
@pytest.mark.parametrize("M", [1, 129, 1000])
def test_scoring_head_peaked_rows(gpu, M, V):
    """evo_unembed_score (fused: quad and 256-column-half merges of (max, sum e, sum e x)) and evo_logprobs on the same
    logits: rows whose max is in one half and target deep in the other, one-hot rows (entropy < 1e-6), uniform rows
    (entropy ln V), a +80 common offset."""
    lib = _lib.lib()
    sc = score_case(M, V)
    x, w, tg = sc["x"].to(DEV), sc["w"].to(DEV), sc["tg"].to(DEV)
    lp = torch.full((M,), NAN, dtype=torch.float32, device=DEV)
    ent = torch.full((M,), NAN, dtype=torch.float32, device=DEV)
    n = lib.evo_unembed_score_workspace(M, V)
    ws = torch.empty(max(n, 1), dtype=torch.uint8, device=DEV)
    sp = _lib.ScoreParams(x=x.data_ptr(), W=w.data_ptr(), targets=tg.data_ptr(), logprobs=lp.data_ptr(), entropy=ent.data_ptr(),
                          M=M, V=V, K=sc["K"], workspace=ws.data_ptr(), workspace_bytes=n)
    _lib.check(lib.evo_unembed_score(C.byref(sp), stream()), "evo_unembed_score")
    logits = sc["logits"].to(DEV)
    old = torch.full((M,), NAN, dtype=torch.float32, device=DEV)
    _lib.check(lib.evo_logprobs(_lib.ptr(logits), _lib.ptr(tg), _lib.ptr(old), M, V, stream()))
    torch.cuda.synchronize()
    lp, ent, old = lp.double().cpu(), ent.double().cpu(), old.double().cpu()
    lp_bar = 2e-5 + 2.0 ** -21 * sc["lse"].abs()
    ent_bar = 5e-5 + 2.0 ** -21 * sc["logits"].double().abs().amax(-1)
    kinds = [SCORE_KINDS[r % len(SCORE_KINDS)] for r in range(M)]
    for name, got, want, bar in (("logprob", lp, sc["lp"], lp_bar), ("entropy", ent, sc["ent"], ent_bar),
                                 ("evo_logprobs", old, sc["lp"], lp_bar), ("fused vs evo_logprobs", lp, old, lp_bar)):
        err = (got - want).abs()
        bad = ~(err <= bar)
        assert not bad.any(), (name, M, V, [(r, kinds[r], err[r].item(), bar[r].item()) for r in torch.nonzero(bad)[:5, 0].tolist()])
