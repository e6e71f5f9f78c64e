"""A plain fp64 reference for every GEMM epilogue (evo_gemm, evo_gemm_smallm, evo_unembed_score), with a rigorous interval per
output element and a report per tile.  Pure torch: it runs on the CPU or on the GPU, on whatever device its inputs live.

Rounding analysis.  The kernels compute acc = sum_k a[m,k] w[n,k] in fp32 (wgmma, then for stream-K a fix-up sum of fp32
partials), then an epilogue chain of IEEE fp32 operations and bf16 roundings.
  * Products of bf16 values are exact in fp32 and in fp64, so exact = a.double() @ w.double().T is the exact sum (fp64 sums of
    K <= 2^20 such products lose at most K 2^-53 S, below a millionth of the fp32 bound) and S = |a| @ |w|.T bounds every
    partial sum in any order.
  * Any fp32 summation of K terms -- any order, any split into ranges summed separately and then added, round-to-nearest or
    truncating adds -- returns a value within gamma S of exact, gamma = K u / (1 - K u) with u = 2^-23 (the unit roundoff of
    truncation; round-to-nearest has half of it).  Tensor-core accumulation is assumed to be at least as accurate as truncating
    fp32 adds; the GPU tests report the largest fraction of gamma S an output proves was used.
  * Every epilogue step except GELU is monotone non-decreasing in acc: fp32 and bf16 rounding, adding a bias or a residual.
    So the output of a linear epilogue lies in [chain(exact - gamma S), chain(exact + gamma S)].
  * GELU is not monotone.  l1 = bf16(acc) takes one of the bf16 values between the rounded ends, so the hull of bf16(GELU(l1))
    is taken over every one of them: bf16(GELU(v)) is tabulated once for all 2^16 bf16 values v (in fp32 with the kernels'
    order of operations, 0.5 x (1 + erf(x / sqrt 2)), and in fp64) and a sparse table answers the least and the greatest entry
    over any range of v exactly, with no assumption on where GELU turns.  The gate product bf16(gelu) * bf16(acc2) of two
    8-bit significands is exact in fp32 and monotone in each factor for a fixed sign of the other, so its hull is reached at
    the corners.
  * The rotary step x c - y s (x s + y c) of bf16 values: both products are exact in fp32, so with or without fma contraction
    the fp32 result is the exact value rounded once -- which fp64 computes exactly whenever the two products are within 2^36 of
    each other (rope_rotate returns a mask of those elements, and the tests assert only on them).
    Over the box of (x, y) the rotation is linear, so its hull is reached at the four corners.
  * In exact-integer mode (integer-valued inputs on a power-of-two grid with S below 2^24 grid units) every fp32 partial sum is
    exact, gamma is 0 and every interval collapses to chain(exact): the expected bits are known exactly.

The report gives, per tile of the kernel's output (row-block x column-block), the number of elements outside their interval and
the worst one, and the fraction of elements equal to chain(exact)."""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import torch

U32 = 2.0 ** -23                  # unit roundoff of truncating fp32 adds
EPIS = ("none", "bias", "resid", "bias_resid", "gelu_gate", "bias_rope")


def gamma(K: int) -> float:
    """The fp32 accumulation bound factor: |acc - exact| <= gamma(K) * S for any order of K terms."""
    ku = K * U32
    return ku / (1.0 - ku)


def exact_sums(a: torch.Tensor, w: torch.Tensor, rows_per_chunk: int | None = None):
    """(exact, S): a @ w.T and |a| @ |w|.T in fp64, row chunk by row chunk so that the temporaries stay bounded."""
    M, K = a.shape
    N = w.shape[0]
    wd = w.double()
    wa = wd.abs()
    exact = torch.empty(M, N, dtype=torch.float64, device=a.device)
    S = torch.empty_like(exact)
    step = rows_per_chunk or max(1, (64 << 20) // (8 * max(N, K)))
    for r0 in range(0, M, step):
        ad = a[r0:r0 + step].double()
        exact[r0:r0 + step] = ad @ wd.T
        S[r0:r0 + step] = ad.abs() @ wa.T
    return exact, S


def bf(x: torch.Tensor) -> torch.Tensor:
    """fp64/fp32 -> bf16 through fp32: the rounding of an fp32 accumulator (fp32 rounding is exact on fp32 inputs)."""
    return x.float().bfloat16()


def gelu32(x: torch.Tensor) -> torch.Tensor:
    """F.gelu (erf form) in fp32 with the kernels' order of operations; x bf16 or fp32, result fp32."""
    x = x.float()
    return (0.5 * x) * (1.0 + torch.erf(x * 0.7071067811865476))


def gelu64(x: torch.Tensor) -> torch.Tensor:
    x = x.double()
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


_GELU_TABLES = {}


def _gelu_tables(device):
    """All finite bf16 values in increasing order, and sparse tables of the least / greatest bf16(GELU(v)) (fp32 and fp64
    GELU together) over every run of 2^j consecutive values."""
    key = str(device)
    if key not in _GELU_TABLES:
        bits = torch.arange(-32768, 32768, dtype=torch.int32, device=device).to(torch.int16)
        v = bits.view(torch.bfloat16).float()
        v = torch.sort(v[torch.isfinite(v)]).values
        g32, g64 = bf(gelu32(v)).float(), bf(gelu64(v)).float()
        mins, maxs = [torch.minimum(g32, g64)], [torch.maximum(g32, g64)]
        j = 1
        while (1 << j) <= v.numel():
            h = 1 << (j - 1)
            mins.append(torch.minimum(mins[-1][:-h], mins[-1][h:]))
            maxs.append(torch.maximum(maxs[-1][:-h], maxs[-1][h:]))
            j += 1
        _GELU_TABLES[key] = (v, mins, maxs)
    return _GELU_TABLES[key]


def gelu_range_hull(lo: torch.Tensor, hi: torch.Tensor):
    """(least, greatest) of bf16(GELU(v)), GELU in fp32 or fp64, over every bf16 v with lo <= v <= hi (lo, hi bf16): fp32."""
    v, mins, maxs = _gelu_tables(lo.device)
    shape = lo.shape
    i0 = torch.searchsorted(v, lo.float().reshape(-1).contiguous(), right=False)
    i1 = torch.searchsorted(v, hi.float().reshape(-1).contiguous(), right=True) - 1
    n = (i1 - i0 + 1).clamp(min=1)
    j = torch.floor(torch.log2(n.double())).long()
    while True:                         # guard the float log2 at exact powers of two
        over = (1 << j) > n
        if not over.any():
            break
        j = j - over.long()
    out_lo = torch.empty(i0.shape, dtype=torch.float32, device=lo.device)
    out_hi = torch.empty_like(out_lo)
    for lvl in torch.unique(j).tolist():
        m = j == lvl
        a, b = i0[m], i1[m] - (1 << lvl) + 1
        out_lo[m] = torch.minimum(mins[lvl][a], mins[lvl][b])
        out_hi[m] = torch.maximum(maxs[lvl][a], maxs[lvl][b])
    return out_lo.view(shape), out_hi.view(shape)


def linear_chain(acc: torch.Tensor, bias=None, resid=None) -> torch.Tensor:
    """none / bias / resid / bias_resid: bf16(bf16(fp32(acc) + bias) + r), the roundings of include/evo_b200.h."""
    x = acc.float()
    if bias is not None:
        x = x + bias.float()
    if resid is not None:
        x = x.bfloat16().float() + resid.float()
    return x.bfloat16()


def gate_split(acc: torch.Tensor):
    """The w12 layout: weight rows interleaved [l1 | l2] in 128-row groups -> (acc1, acc2), each (M, N / 2)."""
    M, N = acc.shape
    v = acc.view(M, N // 256, 2, 128)
    return v[:, :, 0].reshape(M, N // 2), v[:, :, 1].reshape(M, N // 2)


def gelu_gate_values(l1: torch.Tensor, l2: torch.Tensor):
    """bf16(bf16(gelu(l1)) * l2) with GELU in fp32 and in fp64: (out32, out64)."""
    outs = []
    for g in (gelu32(l1), gelu64(l1)):
        outs.append((bf(g).float() * l2.float()).bfloat16())
    return outs[0], outs[1]


def rope_tables_rows(cos, sin, M, rope_L, row0=0):
    rows = (torch.arange(M, device=cos.device) + row0) % rope_L
    return cos[rows].double(), sin[rows].double()


def rope_rotate(x: torch.Tensor, rope_cols: int, c: torch.Tensor, s: torch.Tensor):
    """NeoX rotation of head columns [0, 64) against [64, 128) for the heads below rope_cols; x (M, N) bf16 -> bf16.
    Returns (out, exact_mask): exact_mask is False where fp64 cannot represent x c - y s exactly."""
    M, N = x.shape
    out = x.clone()
    ok = torch.ones(M, N, dtype=torch.bool, device=x.device)
    nh = rope_cols // 128
    if nh == 0:
        return out, ok
    h = x[:, :rope_cols].view(M, nh, 2, 64).double()
    xa, ya = h[:, :, 0], h[:, :, 1]
    cc, ss = c[:, None, :], s[:, None, :]
    p1, p2, p3, p4 = xa * cc, ya * ss, xa * ss, ya * cc
    ox, oy = bf(p1 - p2), bf(p3 + p4)

    def fine(u, v):    # both products within 2^36 of each other (or one of them zero): the fp64 difference is exact
        au, av = u.abs(), v.abs()
        return (au == 0) | (av == 0) | ((au <= av * 2.0 ** 36) & (av <= au * 2.0 ** 36))
    out[:, :rope_cols] = torch.stack([ox, oy], 2).reshape(M, rope_cols)
    ok[:, :rope_cols] = torch.stack([fine(p1, p2), fine(p3, p4)], 2).reshape(M, rope_cols)
    return out, ok


def rope_hull(xlo: torch.Tensor, xhi: torch.Tensor, rope_cols: int, c, s):
    """Hull of the rotation over the box [xlo, xhi] (per element, bf16): the corners (x, y) in {lo, hi}^2."""
    M, N = xlo.shape
    lo, hi = xlo.clone(), xhi.clone()
    nh = rope_cols // 128
    if nh == 0:
        return lo, hi
    hl = xlo[:, :rope_cols].view(M, nh, 2, 64).double()
    hh = xhi[:, :rope_cols].view(M, nh, 2, 64).double()
    cc, ss = c[:, None, :], s[:, None, :]
    rx, ry = [], []
    for xv in (hl[:, :, 0], hh[:, :, 0]):
        for yv in (hl[:, :, 1], hh[:, :, 1]):
            rx.append(bf(xv * cc - yv * ss).float())
            ry.append(bf(xv * ss + yv * cc).float())
    rx, ry = torch.stack(rx), torch.stack(ry)
    lo[:, :rope_cols] = torch.stack([rx.min(0).values, ry.min(0).values], 2).reshape(M, rope_cols).bfloat16()
    hi[:, :rope_cols] = torch.stack([rx.max(0).values, ry.max(0).values], 2).reshape(M, rope_cols).bfloat16()
    return lo, hi


@dataclass
class Expected:
    lo: torch.Tensor          # bf16, per element
    hi: torch.Tensor
    mid: torch.Tensor         # chain(exact): what a correctly rounded fp32 accumulation gives
    z: torch.Tensor | None = None      # fp64 input of the last rounding (none / bias): for the gamma S used
    S: torch.Tensor | None = None
    g: float = 0.0
    mask: torch.Tensor | None = None   # elements the interval is asserted on (all when None)


def expect(epi: str, exact, S, g: float, bias=None, resid=None, rope=None) -> Expected:
    """The interval of every output element of epilogue `epi` for accumulators within g * S of exact (g = 0: exact-integer
    mode).  rope = dict(cos, sin, rope_L, rope_cols[, row0]) for bias_rope."""
    lo_acc, hi_acc = (exact - g * S, exact + g * S) if g else (exact, exact)
    if epi in ("none", "bias", "resid", "bias_resid"):
        b = bias if epi in ("bias", "bias_resid") else None
        r = resid if epi in ("resid", "bias_resid") else None
        z = exact + b.double() if b is not None and r is None else (exact if b is None and r is None else None)
        return Expected(linear_chain(lo_acc, b, r), linear_chain(hi_acc, b, r), linear_chain(exact, b, r), z, S, g)
    if epi == "gelu_gate":
        (e1, e2), (l1a, l2a), (l1b, l2b) = gate_split(exact), gate_split(lo_acc), gate_split(hi_acc)
        m32, m64 = gelu_gate_values(bf(e1), bf(e2))
        L1lo, L1hi, L2lo, L2hi = bf(l1a), bf(l1b), bf(l2a), bf(l2b)
        glo, ghi = gelu_range_hull(L1lo, L1hi)
        corners = torch.stack([(gv * lv.float()).bfloat16().float() for gv in (glo, ghi) for lv in (L2lo, L2hi)])
        lo = torch.minimum(corners.min(0).values, torch.minimum(m32.float(), m64.float())).bfloat16()
        hi = torch.maximum(corners.max(0).values, torch.maximum(m32.float(), m64.float())).bfloat16()
        return Expected(lo, hi, m32, None, None, g)
    if epi == "bias_rope":
        M = exact.shape[0]
        c, s = rope_tables_rows(rope["cos"], rope["sin"], M, rope["rope_L"], rope.get("row0", 0))
        mid, ok = rope_rotate(linear_chain(exact, bias), rope["rope_cols"], c, s)
        lo, hi = rope_hull(linear_chain(lo_acc, bias), linear_chain(hi_acc, bias), rope["rope_cols"], c, s)
        return Expected(lo, hi, mid, None, None, g, ok)
    raise ValueError(epi)


def gamma_used(out: torch.Tensor, e: Expected) -> float:
    """Lower bound on the accumulation error, as a fraction of gamma S, that an output proves (none / bias only): an element
    that differs from chain(exact) had an accumulator at least as far from exact as the rounding boundary it crossed."""
    if e.z is None or e.S is None or not e.g:
        return 0.0
    o = out.double()
    diff = (out != e.mid) & torch.isfinite(o)
    if not diff.any():
        return 0.0
    z, o, S = e.z[diff], o[diff], e.S[diff]
    mant, ex = torch.frexp(o)                          # |o| = |mant| 2^ex, |mant| in [0.5, 1)
    ulp = torch.ldexp(torch.ones_like(o), ex - 8)
    toward_zero = (z.abs() < o.abs())
    at_pow2 = mant.abs() == 0.5
    half = torch.where(toward_zero & at_pow2, ulp / 4, ulp / 2)
    need = ((z - o).abs() - half).clamp(min=0)
    return float((need / (e.g * S).clamp(min=1e-300)).max().item())


@dataclass
class Report:
    name: str
    tile: tuple
    n_viol: int
    bad: dict = field(default_factory=dict)     # (row-block, col-block) -> (count, worst (row, col, got, lo, hi))
    match_min: float = 1.0                      # least per-tile fraction of elements equal to chain(exact)
    match_min_tile: tuple = (0, 0)
    match_all: float = 1.0
    n_checked: int = 0

    @property
    def bad_tiles(self):
        return sorted(self.bad)

    def __str__(self):
        s = (f"{self.name}: {self.n_viol} of {self.n_checked} elements outside their interval in {len(self.bad)} tile(s) of "
             f"{self.tile[0]}x{self.tile[1]}; exact-match fraction {self.match_all:.4f} overall, {self.match_min:.4f} at worst "
             f"(tile {self.match_min_tile})")
        for k in self.bad_tiles[:8]:
            n, (r, c, got, lo, hi) = self.bad[k]
            s += f"\n  tile {k}: {n} bad, worst at ({r}, {c}): got {got!r}, interval [{lo!r}, {hi!r}]"
        if len(self.bad) > 8:
            s += f"\n  ... and {len(self.bad) - 8} more tiles"
        return s

    def assert_ok(self, floor: float = 0.0):
        assert self.n_viol == 0, str(self)
        assert self.match_min >= floor, f"per-tile exact-match fraction below {floor}: " + str(self)


def check(name: str, out: torch.Tensor, e: Expected, tile=(128, 256)) -> Report:
    """Per-tile report of out (bf16, M x n_out) against the intervals e."""
    M, N = e.lo.shape
    out = out[:M, :N]
    o, lo, hi = out.float(), e.lo.float(), e.hi.float()
    ok = (o >= lo) & (o <= hi)                        # NaN fails
    if e.mask is not None:
        ok = ok | ~e.mask
    tr, tc = tile
    nr, nc = -(-M // tr), -(-N // tc)
    rows = torch.arange(M, device=o.device)[:, None] // tr
    cols = torch.arange(N, device=o.device)[None, :] // tc
    tid = (rows * nc + cols).expand(M, N).reshape(-1)
    counts = torch.bincount(tid, minlength=nr * nc)
    bad_counts = torch.bincount(tid, weights=(~ok).reshape(-1).double(), minlength=nr * nc)
    eq = (out.view(torch.int16) == e.mid.view(torch.int16)) | ((o == 0) & (e.mid.float() == 0))
    eq_counts = torch.bincount(tid, weights=eq.reshape(-1).double(), minlength=nr * nc)
    frac = (eq_counts / counts.clamp(min=1)).cpu()
    t = int(frac.argmin())
    rep = Report(name, tile, int((~ok).sum().item()), {}, float(frac[t]), (t // nc, t % nc),
                 float(eq.double().mean().item()) if eq.numel() else 1.0, M * N)
    excess = torch.maximum(lo - o, o - hi)
    excess = torch.where(torch.isnan(o), torch.full_like(o, float("inf")), excess)
    for t in torch.nonzero(bad_counts > 0).flatten().tolist()[:64]:
        i, j = divmod(t, nc)
        sl = excess[i * tr:(i + 1) * tr, j * tc:(j + 1) * tc].masked_fill(ok[i * tr:(i + 1) * tr, j * tc:(j + 1) * tc], -1.0)
        k = int(sl.reshape(-1).argmax())
        r, c = i * tr + k // sl.shape[1], j * tc + k % sl.shape[1]
        rep.bad[(i, j)] = (int(bad_counts[t].item()), (r, c, o[r, c].item(), lo[r, c].item(), hi[r, c].item()))
    if len(rep.bad) < int((bad_counts > 0).sum().item()):     # more failing tiles than listed: count them all
        for t in torch.nonzero(bad_counts > 0).flatten().tolist()[64:]:
            rep.bad[divmod(t, nc)] = (int(bad_counts[t].item()), (-1, -1, float("nan"), float("nan"), float("nan")))
    return rep


# ------------------------------------------------------------------ exact-integer inputs
def int_exponent(K: int) -> int:
    """e such that sums of K products of integers in [-15, 15] times 2^-e have a standard deviation of about 1 (the variance of
    a uniform integer in [-15, 15] is 80)."""
    return int(round(math.log2(80.0 * math.sqrt(K))))


def int_inputs(M, N, K, gen, device, ldr=None):
    """A in [-15, 15]; W in [-15, 15] 2^-e; bias in [-128, 128] 2^-e (on the accumulator's grid); residual in [-128, 128] 2^-7.
    Every product is below 2^8 grid units, so S stays below 225 K grid units (< 2^22 for K <= 11008): every fp32 partial sum
    of any order is exact."""
    e = int_exponent(K)
    ri = lambda *shape, lo=-15, hi=15: torch.randint(lo, hi + 1, shape, generator=gen, device=device).float()
    a = ri(M, K).bfloat16()
    w = (ri(N, K) * 2.0 ** -e).bfloat16()
    bias = (ri(N, lo=-128, hi=128) * 2.0 ** -e).bfloat16()
    resid = (ri(M, ldr or N, lo=-128, hi=128) * 2.0 ** -7).bfloat16()
    return a, w, bias, resid, e


def real_inputs(M, N, K, gen, device, ldr=None):
    """The model's scales: activations of standard deviation 0.5, weights 1/sqrt(K), bias 0.2, residual 1."""
    rn = lambda *shape: torch.randn(*shape, generator=gen, device=device)
    return ((rn(M, K) * 0.5).bfloat16(), (rn(N, K) / math.sqrt(K)).bfloat16(), (rn(N) * 0.2).bfloat16(),
            rn(M, ldr or N).bfloat16())


def int_preconditions(a, w, S, e: int, exact):
    """Exact-integer mode holds: S (which bounds every partial sum) is below 2^24 grid units.  Returns the fraction of sums
    that are not bf16-representable (so that the chain's rounding points are exercised): about half at K = 64, where sums
    carry 9-10 significant bits, and more for longer K."""
    assert float(S.max().item()) * 2.0 ** e < 2.0 ** 24, "partial sums may exceed fp32's exact-integer range"
    return float((bf(exact).double() != exact).double().mean().item())


# ------------------------------------------------------------------ the scoring head
U24 = 2.0 ** -24


def score_reference(logits: torch.Tensor, targets: torch.Tensor):
    """fp64 log-probability of the target (0 for a target < 0 or >= V) and entropy over bf16 logits; plus (lse, A, |mean|)
    for the error bounds."""
    x = logits.double()
    V = x.shape[1]
    lse = torch.logsumexp(x, 1)
    p = torch.exp(x - lse[:, None])
    mean = (p * x).sum(1)
    ent = lse - mean
    valid = (targets >= 0) & (targets < V)
    lp = torch.where(valid, x.gather(1, targets.clamp(0, V - 1)[:, None])[:, 0] - lse, torch.zeros_like(lse))
    tl = torch.where(valid, x.gather(1, targets.clamp(0, V - 1)[:, None])[:, 0], torch.zeros_like(lse))
    return lp, ent, dict(lse=lse, absmean=(p * x.abs()).sum(1), mean=mean, tlogit=tl, valid=valid, p=p, x=x,
                         max=x.max(1).values, disp=(p * (x - mean[:, None]).abs()).sum(1))


def _chain_sum_error(t: torch.Tensor, u: float) -> torch.Tensor:
    """Rounding bound of the per-thread sums of the scoring epilogue, relative to the row total S: thread `quad` of a 256-column
    half adds the 64 columns 8 i + 2 quad + e (i < 32, e < 2) one after another, in that order, and the add of a term t_k errs
    by at most u |P_k| (P_k the partial sum it produces) and at most |t_k| (the partial before it is a float, no farther than
    |t_k| from the exact P_k): sum_k min(u |P_k|, |t_k|).  t (rows, V): the terms over S."""
    rows, V = t.shape
    ch = t.reshape(rows, V // 256, 32, 4, 2).permute(0, 1, 3, 2, 4).reshape(rows, V // 256 * 4, 64)
    return torch.minimum(u * ch.cumsum(2)[:, :, 1:].abs(), ch[:, :, 1:].abs()).sum((1, 2))


def score_bounds(aux, V: int):
    """Error bounds of the fp32 statistics over exactly known logits x (fp64 p = softmax(x), mean = sum p x, A = sum p |x|,
    D = sum p |x - mean|).  Relative to the row's sum S of e^(x - max):
      * the per-thread sums (see _chain_sum_error): eS over the terms p, eW over the terms p x;
      * two lane merges and the fold over V / 256 halves: (4 + V / 256) u of S (of A S for W);
      * __expf (ex2.approx plus the fp32 rounding of its argument) errs by 2^-21 relative, once per term and once per merge
        level (three levels): 4 2^-21 on S; in the ratio W / S the common factors cancel and leave 4 2^-21 D.
    logf adds 2^-22 absolute, and each of max + log S, t - lse, lse - W / S one fp32 rounding (u = 2^-24 of its operands):
        |dlogprob| <= eS + (4 + V/256) u + 4 2^-21 + 2^-22 + u (|max| + 2 |lse| + |t|)
        |dentropy| <= that without |t|, + eW + (4 + V/256) u A + |mean| (eS + (4 + V/256) u) + 4 2^-21 D + 2 u (|lse| + |mean|)."""
    u = U24
    lev = (4 + V / 256) * u
    eS = _chain_sum_error(aux["p"], u) + lev
    eW = _chain_sum_error(aux["p"] * aux["x"], u) + lev * aux["absmean"]
    lse, mean = aux["lse"].abs(), aux["mean"].abs()
    mx = aux["max"].abs()
    base = eS + 4 * 2.0 ** -21 + 2.0 ** -22 + u * (mx + 2 * lse)
    tol_lp = base + u * aux["tlogit"].abs()
    tol_ent = base + eW + mean * eS + 4 * 2.0 ** -21 * aux["disp"] + 2 * u * (lse + mean)
    return tol_lp, tol_ent
