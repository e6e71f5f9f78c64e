"""Every implementation and mode of the Hyena operator against the oracle.

evo_hyena_fwd has two scan kernels: the mode-split TMA kernel (hyena_ms.cuh), taken when head_dim == 128 and
D % 256 == 0, and the scalar kernel (hyena_scan_kernel in hyena.cu) for every other geometry.  Both claim the
reference's bf16 rounding points, so both are held to the bars of
tests/test_gpu_parity.py::test_hyena_operator_vs_oracle.  On top of the plain prefill this file covers the history
inputs (halo, state_in), the carry passes the sequence-parallel forward chains (state_only with its fold kernel,
evo_hyena_combine_states, reuse_segment_states), the decode step at the 7B width and at head_dim != 128, and the calls
the launcher must reject.

References: the oracle's bf16 FFT operator (the reference's rounding points) and the fp64 time-domain recurrence
O.hyena_operator_time_domain (the truth; it takes a halo and a modal state).  Where the FFT operator cannot express an
input (a modal state entering row 0), a call on z that continues a prefix is checked against the tail of one GPU pass
over [prefix, z]."""
import ctypes as C
import math
import os
import sys
from functools import lru_cache
from types import SimpleNamespace

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

from oracle import stripedhyena_oracle as O          # noqa: E402
from evo_b200 import _lib                             # noqa: E402

DEV = "cuda:0"
BF16_EPS = 2.0 ** -7

# implementation -> (D, heads).  The kernel is selected by geometry: the scalar kernel runs head_dim 64, and head_dim 128
# with D % 256 != 0.
IMPLS = {"ms": (256, 2), "scalar_hd64": (256, 4), "scalar_d384": (384, 3)}
LENGTHS = (1, 2, 3, 15, 16, 17, 130, 1025, 4099)      # 16-token TMA stage, 8-token group, ragged last tiles
FORCES = (0, 1, 3, 7)                                 # 0 = the launcher's choice (8 x 513 tokens at B = 1, L = 4099)
PREFIX = 37                                           # rows before z in the continuation checks
NEAR_UNIT = (0.9, 0.9999)                             # pole magnitudes where carries matter: memories of ~10^4 tokens


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    _lib.lib()
    torch.set_num_threads(min(64, os.cpu_count() or 1))


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def maxerr(a, b):
    return (a.double().cpu() - b.double().cpu()).abs().max().item()


def meanerr(a, b):
    return (a.double().cpu() - b.double().cpu()).abs().mean().item()


def cplx(st):
    """(B, D, 8, 2) fp32 state -> (B, D, 8) complex on the host."""
    return torch.view_as_complex(st.float().cpu().contiguous())


# ------------------------------------------------------------------ helpers
@lru_cache(maxsize=8)
def _filter_sd(D, seed=1, pole_mag=None):
    """Filter parameters of one Hyena layer: sd on the host in the oracle's layout, f on the device.  They are drawn for
    max(D, 384) channels and sliced, so the D = 256 set is the first two heads of the D = 384 set."""
    W = max(D, 384)
    g = torch.Generator().manual_seed(seed)
    lo, hi = pole_mag or (0.5, 0.95)
    mag = lo + (hi - lo) * torch.rand(W, 8, 1, generator=g)
    ang = (torch.rand(W, 8, 1, generator=g) * 2 - 1) * math.pi
    sd = {"w": (torch.randn(3 * W, 1, 3, generator=g) * 0.3).bfloat16()[:3 * D],
          "b": (torch.randn(3 * W, generator=g) * 0.1).bfloat16()[:3 * D],
          "D": torch.randn(W, generator=g).bfloat16()[:D],
          "p": torch.stack([mag * torch.cos(ang), mag * torch.sin(ang)], dim=-1)[:D],
          "r": (torch.randn(W, 8, 1, 2, generator=g) * 0.3)[:D]}
    sd = {k: v.contiguous() for k, v in sd.items()}
    return sd, {k: v.to(DEV) for k, v in sd.items()}


def _hyena_call(z, f, H, force=0, halo=None, state_in=None, want_state=False, state_only=False, reuse=False, ws=None):
    """One evo_hyena_fwd launch on z (B, L, 3D).  ws: a caller-owned workspace (a carry pass's per-segment states are
    kept there for an output pass with reuse_segment_states = 1); allocated to the queried size when None.
    Returns (y, state_out, fir_state_out, ws); the outputs not requested are None."""
    lib = _lib.lib()
    B, L, C3 = z.shape
    D = C3 // 3
    y = None if state_only else torch.empty(B, L, D, dtype=torch.bfloat16, device=DEV)
    st = torch.empty(B, D, 8, 2, dtype=torch.float32, device=DEV) if want_state else None
    fs = torch.empty(B, C3, 2, dtype=torch.bfloat16, device=DEV) if want_state else None
    hp = _lib.HyenaParams(z=z.data_ptr(), y=y.data_ptr() if y is not None else None, fir_w=f["w"].data_ptr(), fir_b=f["b"].data_ptr(),
                          Dskip=f["D"].data_ptr(), poles=f["p"].data_ptr(), residues=f["r"].data_ptr(), B=B, L=L, D=D, S=8, nheads=H,
                          halo=halo.data_ptr() if halo is not None else None,
                          state_in=state_in.data_ptr() if state_in is not None else None,
                          state_out=st.data_ptr() if st is not None else None, fir_state_out=fs.data_ptr() if fs is not None else None,
                          force_segments=force, state_only=int(state_only), reuse_segment_states=int(reuse))
    need = lib.evo_hyena_fwd_workspace(C.byref(hp))
    if ws is None:
        ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
    _lib.check(lib.evo_hyena_fwd(C.byref(hp), _lib.ptr(ws), ws.numel(), stream()), "evo_hyena_fwd")
    torch.cuda.synchronize()
    return y, st, fs, ws


def _bf16_oracle(sd, z, H, halo=None, want_state=False):
    """The reference's FFT operator with its bf16 rounding points, one head at a time.  With a halo the short FIR runs
    over [halo, z] and the long convolution starts from a zero modal state at row 0 of z."""
    B, L, C3 = z.shape
    D = C3 // 3
    hd = D // H
    zz = z if halo is None else torch.cat([halo, z], 1)
    ys, sts = [], []
    for h in range(H):
        c3, c1 = slice(h * 3 * hd, (h + 1) * 3 * hd), slice(h * hd, (h + 1) * hd)
        z_pre, _ = O.fir_parallel(zz[:, :, c3], sd["w"][c3], sd["b"][c3])
        z_pre = z_pre[..., zz.shape[1] - L:].contiguous()
        y, st = O.iir_parallel(z_pre, O.hyena_filter(sd["p"][c1], sd["r"][c1], L), sd["D"][c1], sd["p"][c1], 1, hd, want_state)
        ys.append(y)
        sts.append(st)
    return torch.cat(ys, -1), (torch.cat(sts, 1) if want_state else None)


def _fp64_oracle(sd, z, H, halo=None, state_in=None):
    """fp64 time-domain operator: y (B, L, D) and the end state (B, D, 8) complex128."""
    D = z.shape[-1] // 3
    return O.hyena_operator_time_domain(z.double(), sd["w"], sd["b"], sd["D"], sd["p"], sd["r"], H, D // H,
                                        halo=None if halo is None else halo.double(),
                                        state_in=None if state_in is None else cplx(state_in).to(torch.complex128))


def _assert_vs_oracle(y, yb, yt, what):
    """The bars of test_hyena_operator_vs_oracle: the reference's rounding points are reproduced, only the fp32 scan
    vs fp32 FFT summation differs."""
    assert torch.isfinite(y.float()).all(), what
    frac = (y.cpu() == yb).float().mean().item()
    assert frac > 0.995, (what, frac)
    err, lim = maxerr(y, yb), 2 * BF16_EPS * max(1.0, yb.abs().max().item())
    assert err <= lim, (what, err, lim)
    eg, eb = meanerr(y, yt), meanerr(yb, yt)
    assert eg <= 1.25 * eb + 1e-6, (what, eg, eb)


def _assert_same_bf16(y, y_ref, what, frac_min):
    frac = (y == y_ref).float().mean().item()
    assert frac > frac_min, (what, frac)
    err, lim = maxerr(y, y_ref), 2 * BF16_EPS * max(1.0, y_ref.abs().max().item())
    assert err <= lim, (what, err, lim)


def _assert_state(st, ref, rel, what):
    ref = ref.to(torch.complex128)
    err, scale = (cplx(st).to(torch.complex128) - ref).abs().max().item(), max(1.0, ref.abs().max().item())
    assert err <= rel * scale, (what, err / scale, rel)


# ------------------------------------------------------------------ A. prefill scan matrix
def _matrix():
    return [pytest.param(impl, B, L, id=f"{impl}-B{B}-L{L}") for B in (1, 3) for L in LENGTHS for impl in IMPLS]


@lru_cache(maxsize=2)
def _prefill_refs(D, H, B, L):
    """Inputs and the GPU-independent references of one (geometry, B, L) cell."""
    sd, _ = _filter_sd(D)
    g = torch.Generator().manual_seed(7919 * L + B)
    z = torch.randn(B, L, 3 * D, generator=g).bfloat16()
    zp = torch.randn(B, PREFIX, 3 * D, generator=g).bfloat16()
    zp0 = zp.clone()
    zp0[:, -2:] = 0                                        # a prefix whose continuation needs no halo
    halo = zp[:, -2:].contiguous()
    yb, stb = _bf16_oracle(sd, z, H, want_state=True)
    yt, stt = _fp64_oracle(sd, z, H)
    return SimpleNamespace(
        z=z, zp=zp, zp0=zp0, halo=halo, yb=yb, stb=stb, yt=yt, stt=stt,
        fsb=z.permute(0, 2, 1)[..., -2:],                  # engine.parallel_fir keeps u[..., -2:]
        yb_halo=_bf16_oracle(sd, z, H, halo=halo)[0], yt_halo=_fp64_oracle(sd, z, H, halo=halo)[0],
        # bf16 oracle over [prefix, z]: its error against the truth sets the bar for a continued call
        yb_cont={"state_in": _bf16_oracle(sd, torch.cat([zp0, z], 1), H)[0][:, PREFIX:],
                 "halo+state_in": _bf16_oracle(sd, torch.cat([zp, z], 1), H)[0][:, PREFIX:]})


@pytest.mark.parametrize("impl,B,L", _matrix())
def test_prefill_scan_matrix(impl, B, L):
    """One implementation at one (B, L), every segment count (auto, 1, 3, 7: segments shorter than a group, lengths that
    are no multiple of 16, more segments than tokens) and every mode: plain; state_out + fir_state_out; halo; state_in;
    halo + state_in."""
    D, H = IMPLS[impl]
    sd, f = _filter_sd(D)
    o = _prefill_refs(D, H, B, L)
    z, halo = o.z.to(DEV), o.halo.to(DEV)
    # continuations: state_in = the GPU's end state of the prefix; reference = the tail of one sequential pass over
    # [prefix, z], and the fp64 operator started from the same halo and state
    cont = {}
    for name, pre, h in (("state_in", o.zp0, None), ("halo+state_in", o.zp, o.halo)):
        pre = pre.to(DEV)
        _, s_pre, _, _ = _hyena_call(pre, f, H, force=1, want_state=True)
        y_w, s_w, fs_w, _ = _hyena_call(torch.cat([pre, z], 1), f, H, force=1, want_state=True)
        yt_c, st_c = _fp64_oracle(sd, o.z, H, halo=h, state_in=s_pre)
        cont[name] = (h, s_pre, y_w[:, PREFIX:], s_w, fs_w, yt_c, st_c)
    for force in FORCES:
        tag = f"{impl} B={B} L={L} force={force}"
        y, _, _, ws = _hyena_call(z, f, H, force=force)
        _assert_vs_oracle(y, o.yb, o.yt, tag + " plain")
        if force == 0 and (B, L) == (1, 4099):
            assert ws.numel() == B * 8 * D * 8 * 2 * 4, tag      # auto: 8 segments of 513 tokens

        y2, st, fs, _ = _hyena_call(z, f, H, force=force, want_state=True)
        assert torch.equal(y2, y), tag
        # the reference keeps only L history columns when L < 2; the kernel zero-fills the missing one
        assert torch.equal(fs.cpu()[..., -o.fsb.shape[-1]:], o.fsb), tag
        if L < 2:
            assert fs.cpu()[..., 0].abs().sum() == 0, tag
        _assert_state(st, o.stb, 2e-4, tag + " state vs bf16 oracle")      # same bf16 inputs: fp32-level agreement
        _assert_state(st, o.stt, 1e-2, tag + " state vs fp64")              # truth uses unrounded x1v

        yh, _, _, _ = _hyena_call(z, f, H, force=force, halo=halo)
        _assert_vs_oracle(yh, o.yb_halo, o.yt_halo, tag + " halo")

        for name, (h, s_pre, y_w, s_w, fs_w, yt_c, st_c) in cont.items():
            what = f"{tag} {name}"
            yc, sc, fc, _ = _hyena_call(z, f, H, force=force, halo=None if h is None else h.to(DEV), state_in=s_pre, want_state=True)
            # the bars of test_hyena_continuation_and_sequence_sharding_are_exact
            _assert_same_bf16(yc, y_w, what, 0.9995)
            if force == 1:       # one segment: the same fp32 operations as the uninterrupted pass
                assert torch.equal(yc, y_w), what
            eg, eb = meanerr(yc, yt_c), meanerr(o.yb_cont[name], yt_c)
            assert eg <= 1.25 * eb + 1e-6, (what, eg, eb)
            assert maxerr(sc, s_w) <= 1e-4 * max(1.0, s_w.abs().max().item()), what
            _assert_state(sc, st_c, 1e-2, what + " state vs fp64")
            assert torch.equal(fc, fs_w), what


@pytest.mark.parametrize("B,L", [pytest.param(B, L, id=f"B{B}-L{L}") for B in (1, 3) for L in LENGTHS])
def test_prefill_implementations_agree(B, L):
    """The two kernels on the same two heads: the TMA kernel at D = 256, the scalar kernel as heads 0-1 of D = 384 (whose
    first 768 z columns and 256 channels are the D = 256 problem).  They differ only in the fp32 order of the residue sum."""
    _, f256 = _filter_sd(256)
    _, f384 = _filter_sd(384)
    torch.manual_seed(31 * L + B)
    z = torch.randn(B, L, 3 * 384, device=DEV).bfloat16()
    z256 = z[..., :768].contiguous()
    for force in FORCES:
        ms = _hyena_call(z256, f256, 2, force=force)[0]
        scalar = _hyena_call(z, f384, 3, force=force)[0][..., :256]
        _assert_same_bf16(ms, scalar, f"ms vs scalar B={B} L={L} force={force}", 0.995)


# ------------------------------------------------------------------ B. carry passes
def _carry_inputs(D, B, L, seed):
    g = torch.Generator().manual_seed(seed)
    z = (torch.randn(B, L, 3 * D, generator=g) * 0.5).bfloat16()
    halo = (torch.randn(B, 2, 3 * D, generator=g) * 0.5).bfloat16()
    s_in = torch.randn(B, D, 8, 2, generator=g) * 2
    return z, halo, s_in


@pytest.mark.parametrize("nseg", [1, 3, 8])
@pytest.mark.parametrize("impl", list(IMPLS))
def test_state_only_pass_and_fold(impl, nseg):
    """state_only: per-segment zero-start end states, folded by hyena_fold_states_kernel (3 segments: 334 + 334 + 333
    tokens; 8 segments: 7 x 126 + 119), with and without halo and state_in, against the fp64 end state and against the
    end state of an output pass at the same geometry."""
    D, H = IMPLS[impl]
    sd, f = _filter_sd(D, seed=2, pole_mag=NEAR_UNIT)
    B, L = 2, 1001
    z, halo, s_in = _carry_inputs(D, B, L, seed=nseg)
    zd = z.to(DEV)
    for use_halo in (False, True):
        for use_state in (False, True):
            what = f"{impl} nseg={nseg} halo={use_halo} state_in={use_state}"
            h = halo.to(DEV) if use_halo else None
            si = s_in.to(DEV) if use_state else None
            _, e, _, _ = _hyena_call(zd, f, H, force=nseg, halo=h, state_in=si, want_state=True, state_only=True)
            _, s_out, _, _ = _hyena_call(zd, f, H, force=nseg, halo=h, state_in=si, want_state=True)
            _, stt = _fp64_oracle(sd, z, H, halo=halo if use_halo else None, state_in=s_in if use_state else None)
            _assert_state(e, stt, 1e-2, what + " vs fp64")
            assert maxerr(e, s_out) <= 1e-3 * max(1.0, s_out.abs().max().item()), what


@pytest.mark.parametrize("force", [0, 3, 8])
@pytest.mark.parametrize("impl", list(IMPLS))
def test_output_pass_reusing_carry_states_is_bit_identical(impl, force):
    """state_only, then an output pass with reuse_segment_states = 1 on the same workspace (the order of
    evo_b200/parallel.py): the state kernel computes the same segment states as inside a plain output pass, so y and the
    end state are bit-identical to it.  A zeroed workspace must change y: the flag really reads the kept states."""
    D, H = IMPLS[impl]
    _, f = _filter_sd(D, seed=2, pole_mag=NEAR_UNIT)
    B, L = 1, 4099
    z, halo, s_in = (t.to(DEV) for t in _carry_inputs(D, B, L, seed=force))
    _, _, _, ws = _hyena_call(z, f, H, force=force, halo=halo, state_in=s_in, want_state=True, state_only=True)
    y_r, st_r, fs_r, _ = _hyena_call(z, f, H, force=force, halo=halo, state_in=s_in, want_state=True, reuse=True, ws=ws)
    y_p, st_p, fs_p, _ = _hyena_call(z, f, H, force=force, halo=halo, state_in=s_in, want_state=True)
    assert torch.equal(y_r, y_p) and torch.equal(st_r, st_p) and torch.equal(fs_r, fs_p)
    assert ws.numel() // (B * D * 8 * 2 * 4) > 1             # segments of the workspace
    y_z, _, _, _ = _hyena_call(z, f, H, force=force, halo=halo, state_in=s_in, reuse=True, ws=torch.zeros_like(ws))
    assert not torch.equal(y_z, y_p)


@pytest.mark.parametrize("nranks", [2, 4, 8])
def test_combine_states_every_rank(nranks):
    """evo_hyena_combine_states against fp64 sum_{q<r} p^((r-1-q) seg_len) E_q from the same fp32 inputs.  cpow_int
    squares in fp32, and every squaring doubles the relative error of the power, so p^n carries a relative error of
    order n * 2^-24, applied up to r - 1 times.  Bound: |err| <= 4 * r * seg_len * 2^-24 * sum_q |p^((r-1-q) seg_len) E_q|
    (+ 4 * 2^-24 of the same scale for the additions at seg_len = 1).  Measured on an H100: at most 0.14 of it."""
    lib = _lib.lib()
    D, B = 256, 2
    sd, f = _filter_sd(D, seed=9, pole_mag=(0.99, 0.9999))
    g = torch.Generator().manual_seed(nranks)
    ends = torch.randn(nranks, B, D, 8, 2, generator=g)
    ends_d = ends.to(DEV)
    E = torch.view_as_complex(ends.double())                              # (nranks, B, D, 8)
    p = torch.view_as_complex(sd["p"].double())[..., 0]                   # (D, 8)
    worst = 0.0
    for seg_len in (1, 300, 16384):
        for r in range(nranks):
            out = torch.full((B, D, 8, 2), float("nan"), device=DEV)
            _lib.check(lib.evo_hyena_combine_states(_lib.ptr(ends_d), _lib.ptr(out), _lib.ptr(f["p"]), r, nranks, seg_len, B, D, 8, stream()))
            torch.cuda.synchronize()
            terms = [p ** ((r - 1 - q) * seg_len) * E[q] for q in range(r)]
            want = sum(terms) if terms else torch.zeros_like(E[0])
            scale = sum(t.abs() for t in terms) if terms else torch.zeros(B, D, 8, dtype=torch.float64)
            err = (cplx(out).to(torch.complex128) - want).abs()
            bound = (4 * r * seg_len + 4) * 2.0 ** -24 * scale + 1e-30
            assert (err <= bound).all(), (seg_len, r, (err / bound).max().item())
            worst = max(worst, (err / bound).max().item())
    print(f"combine_states nranks={nranks}: max |err| / bound = {worst:.3g}")


def test_sequence_parallel_chain_on_one_gpu():
    """evo_b200/parallel.py's Hyena layer with 4 shards of 8200 tokens emulated on one GPU, calls in its order: halo = the
    previous shard's last two z rows, state_only into a kept workspace (auto segmentation: 16 segments per shard), combine,
    output pass with state_in and reuse_segment_states = 1.  Poles up to |p| = 0.9999 carry across the shard boundaries."""
    lib = _lib.lib()
    D, H, B, P, Lr = 256, 2, 1, 4, 8200
    L = P * Lr
    sd, f = _filter_sd(D, seed=5, pole_mag=NEAR_UNIT)
    torch.manual_seed(5)
    z = (torch.randn(B, L, 3 * D) * 0.5).bfloat16()
    zd = z.to(DEV)
    shards = [zd[:, r * Lr:(r + 1) * Lr].contiguous() for r in range(P)]
    halos = [None] + [zd[:, r * Lr - 2:r * Lr].contiguous() for r in range(1, P)]
    ends = torch.empty(P, B, D, 8, 2, dtype=torch.float32, device=DEV)
    wss = []
    for r in range(P):
        _, e, _, ws = _hyena_call(shards[r], f, H, halo=halos[r], want_state=True, state_only=True)
        assert ws.numel() // (B * D * 8 * 2 * 4) > 1          # the shard is split into several segments
        ends[r] = e
        wss.append(ws)
    ys = []
    for r in range(P):
        s_in = torch.empty(B, D, 8, 2, dtype=torch.float32, device=DEV)
        _lib.check(lib.evo_hyena_combine_states(_lib.ptr(ends), _lib.ptr(s_in), _lib.ptr(f["p"]), r, P, Lr, B, D, 8, stream()))
        y, st, _, _ = _hyena_call(shards[r], f, H, halo=halos[r], state_in=s_in, want_state=r == P - 1, reuse=True, ws=wss[r])
        ys.append(y)
    y = torch.cat(ys, 1)
    y_full, _, _, _ = _hyena_call(zd, f, H, force=1)
    _assert_same_bf16(y, y_full, "sharded vs one pass", 0.995)
    yb, _ = _bf16_oracle(sd, z, H)
    yt, stt = _fp64_oracle(sd, z, H)
    _assert_vs_oracle(y, yb, yt, "sharded vs oracle")
    _assert_state(st, stt, 1e-2, "last shard's end state vs fp64")


# ------------------------------------------------------------------ C. decode step
def _oracle_step(sd, H, u, fir_state, state):
    """The oracle's decode step (engine.step_fir + step_iir) in bf16 with fp32 poles, residues and state."""
    z_pre, fir_state = O.fir_step(u, fir_state, sd["w"], sd["b"])
    x2, x1, v = O.column_split(z_pre, H, sd["D"].shape[0] // H)
    y, state = O.iir_step(x2, x1, v, sd["D"], sd["r"], sd["p"], state)
    return y.to(torch.bfloat16), fir_state, state


def _step(u, y, fs, st, f, B, D, H):
    _lib.check(_lib.lib().evo_hyena_step(_lib.ptr(u), _lib.ptr(y), _lib.ptr(fs), _lib.ptr(st), _lib.ptr(f["w"]), _lib.ptr(f["b"]),
                                         _lib.ptr(f["D"]), _lib.ptr(f["p"]), _lib.ptr(f["r"]), B, D, 8, H, stream()), "evo_hyena_step")


@pytest.mark.parametrize("D,H,B", [(4096, 32, 1), (4096, 32, 16), (4096, 32, 64), (256, 4, 3)])
def test_decode_step_vs_oracle(D, H, B):
    """evo_hyena_step from the states of a GPU prefill, 32 steps, against the oracle's step seeded with the same states
    (the bars of test_hyena_step_bit_exact), then against one evo_hyena_fwd over prefix + steps.  The step rounds the
    short FIR as engine.step_fir does (every product and sum to bf16), the prefill as the conv1d does (fp32 sum, one
    rounding), so x1v differs by a bf16 ulp at a few positions and the two end states part by up to ~7e-3 of their
    magnitude in the reference itself.  The GPU's two paths may part by no more than the oracle's step chain and the
    oracle's prefill over the same tokens do."""
    sd, f = _filter_sd(D, seed=3)
    P, T = 61, 32
    torch.manual_seed(D + B)
    z = torch.randn(B, P + T, 3 * D, device=DEV).bfloat16()
    _, st, fs, _ = _hyena_call(z[:, :P].contiguous(), f, H, want_state=True)
    ofs, ost = fs.cpu(), cplx(st)
    zc = z.cpu()
    y = torch.empty(B, D, dtype=torch.bfloat16, device=DEV)
    for t in range(P, P + T):
        yref, ofs, ost = _oracle_step(sd, H, zc[:, t], ofs, ost)
        _step(z[:, t].contiguous(), y, fs, st, f, B, D, H)
        torch.cuda.synchronize()
        frac = (y.cpu() == yref).float().mean().item()
        assert frac > 0.998 and maxerr(y, yref) <= 2 * BF16_EPS * max(1.0, yref.abs().max().item()), (t, frac)
        assert torch.equal(fs.cpu(), ofs), t
        _assert_state(st, ost, 1e-4, f"step {t}")
    _, st_f, fs_f, _ = _hyena_call(z, f, H, want_state=True)
    assert torch.equal(fs, fs_f)
    _, stb_f = _bf16_oracle(sd, zc, H, want_state=True)
    scale = max(1.0, stb_f.abs().max().item())
    e_gpu = maxerr(st, st_f) / scale
    e_ref = (ost - stb_f).abs().max().item() / scale
    print(f"step D={D} B={B}: steps vs one prefill, max |d state| / max |state|: GPU {e_gpu:.3g}, oracle {e_ref:.3g}")
    assert e_gpu <= 1.25 * e_ref + 1e-4


# ------------------------------------------------------------------ D. rejected calls
def test_rejected_calls_and_empty_sequence():
    lib = _lib.lib()
    D, H, B, L = 256, 2, 2, 100
    _, f = _filter_sd(D)
    z = torch.randn(B, L, 3 * D, device=DEV).bfloat16()
    y = torch.empty(B, L, D, dtype=torch.bfloat16, device=DEV)
    st = torch.empty(B, D, 8, 2, dtype=torch.float32, device=DEV)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)

    def fwd(ws_bytes=None, **kw):
        args = dict(z=z.data_ptr(), y=y.data_ptr(), fir_w=f["w"].data_ptr(), fir_b=f["b"].data_ptr(), Dskip=f["D"].data_ptr(),
                    poles=f["p"].data_ptr(), residues=f["r"].data_ptr(), B=B, L=L, D=D, S=8, nheads=H, force_segments=1)
        args.update(kw)
        hp = _lib.HyenaParams(**args)
        _lib.check(lib.evo_hyena_fwd(C.byref(hp), _lib.ptr(ws), ws.numel() if ws_bytes is None else ws_bytes, stream()), "evo_hyena_fwd")
        return hp

    with pytest.raises(_lib.EvoError, match="state_size 7"):
        fwd(S=7)
    with pytest.raises(_lib.EvoError, match="nheads"):
        fwd(nheads=3)
    with pytest.raises(_lib.EvoError, match="bad batch 0"):
        fwd(B=0)
    with pytest.raises(_lib.EvoError, match="bad batch 65536"):
        fwd(B=65536)
    hp = _lib.HyenaParams(B=B, L=L, D=D, S=8, nheads=H, force_segments=3)
    need = lib.evo_hyena_fwd_workspace(C.byref(hp))
    assert need > 0
    with pytest.raises(_lib.EvoError, match="workspace too small"):
        fwd(ws_bytes=need - 1, force_segments=3)
    with pytest.raises(_lib.EvoError, match="state_only needs state_out"):
        fwd(state_only=1)
    with pytest.raises(_lib.EvoError, match="y is NULL"):
        fwd(y=None, state_out=st.data_ptr())
    u = torch.zeros(B, 3 * 48, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(_lib.EvoError, match="multiple of 32"):
        _lib.check(lib.evo_hyena_step(_lib.ptr(u), _lib.ptr(y), _lib.ptr(u), _lib.ptr(st), _lib.ptr(f["w"]), _lib.ptr(f["b"]), _lib.ptr(f["D"]),
                                      _lib.ptr(f["p"]), _lib.ptr(f["r"]), B, 48, 8, 1, stream()), "evo_hyena_step")
    with pytest.raises(_lib.EvoError, match="bad rank"):
        _lib.check(lib.evo_hyena_combine_states(_lib.ptr(st), _lib.ptr(st), _lib.ptr(f["p"]), 2, 2, 10, B, D, 8, stream()))
    torch.cuda.synchronize()
    # L = 0: nothing to do, nothing written
    y.fill_(float("nan"))
    st.fill_(float("nan"))
    fs = torch.full((B, 3 * D, 2), float("nan"), dtype=torch.bfloat16, device=DEV)
    assert lib.evo_hyena_fwd_workspace(C.byref(_lib.HyenaParams(B=B, L=0, D=D, S=8, nheads=H))) == 0
    fwd(L=0, state_out=st.data_ptr(), fir_state_out=fs.data_ptr(), force_segments=0)
    fwd(L=0, state_out=st.data_ptr(), state_only=1, ws_bytes=0)
    torch.cuda.synchronize()
    assert torch.isnan(y.float()).all() and torch.isnan(st).all() and torch.isnan(fs.float()).all()
