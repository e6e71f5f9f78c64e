"""GPU bring-up / diagnostics harness (development tool, run under gpurun).

    python tests/harness/gpu_bringup.py                 # all stages, each in its own subprocess + timeout
    python tests/harness/gpu_bringup.py --stage gemm1   # one stage inline

Every stage compares the CUDA kernels with the CPU oracle (and with torch-on-GPU where that
is a useful second opinion) and appends JSON lines to gpurun_out/bringup.jsonl, so a hang
or crash in one stage cannot hide the results of the others."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "gpurun_out")
os.makedirs(OUT, exist_ok=True)

STAGES = ["elementwise", "hyena", "gemm1", "gemm2", "attn0", "attn1", "attn2", "model", "perf_gemm", "perf_hyena", "perf_attn"]


def emit(stage, **kw):
    rec = {"stage": stage, **kw}
    line = json.dumps(rec, default=float)
    print(line, flush=True)
    with open(os.path.join(OUT, "bringup.jsonl"), "a") as f:
        f.write(line + "\n")


def main_driver(stages, timeout):
    for st in stages:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--stage", st], timeout=timeout,
                               capture_output=True, text=True)
            tail = (r.stdout[-3000:] + "\n--stderr--\n" + r.stderr[-3000:])
            status = "ok" if r.returncode == 0 else f"rc={r.returncode}"
        except subprocess.TimeoutExpired as e:
            status, tail = "TIMEOUT", ((e.stdout or b"")[-2000:].decode(errors="replace") if isinstance(e.stdout, bytes) else str(e.stdout)[-2000:])
        print(f"===== stage {st}: {status} in {time.time() - t0:.1f}s\n{tail}\n", flush=True)
        with open(os.path.join(OUT, "bringup.jsonl"), "a") as f:
            f.write(json.dumps({"stage": st, "status": status, "seconds": time.time() - t0}) + "\n")


# ------------------------------------------------------------------------------------------
def _imports():
    global torch, O, _lib, StripedHyena, dotdict, model_mod
    import torch
    from oracle import stripedhyena_oracle as O
    from evo_b200 import _lib
    from evo_b200.stripedhyena import StripedHyena, dotdict
    from evo_b200.stripedhyena import model as model_mod
    torch.backends.cuda.matmul.allow_tf32 = False


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def err(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    d = (a - b).abs()
    return {"max_abs": d.max().item(), "mean_abs": d.mean().item(), "ref_max": b.abs().max().item(),
            "n_bad_nan": int(torch.isnan(a).sum())}


def timeit(fn, iters=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(iters + 1)]
    ev[0].record()
    for i in range(iters):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    ts = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(iters))
    return ts[len(ts) // 2]


# ------------------------------------------------------------------------------------------ stages
def stage_elementwise():
    lib = _lib.lib()
    dev = "cuda:0"
    torch.manual_seed(0)
    # rmsnorm
    for D in (256, 4096):
        x = (torch.randn(37, D) * 3).bfloat16()
        sc = (1 + 0.1 * torch.randn(D)).bfloat16()
        ref = O.rms_norm(x, sc, 1e-6)
        xd, sd, od = x.to(dev), sc.to(dev), torch.empty(37, D, dtype=torch.bfloat16, device=dev)
        _lib.check(lib.evo_rmsnorm(_lib.ptr(xd), _lib.ptr(sd), _lib.ptr(od), 37, D, 1e-6, stream()))
        e = err(od, ref)
        emit("elementwise", op="rmsnorm", D=D, exact_frac=(od.cpu() == ref).float().mean().item(), **e)
    # embed
    tab = torch.randn(512, 256).bfloat16()
    ids = torch.randint(0, 512, (3, 11))
    for dt in (torch.int64, torch.int32):
        od = torch.empty(33, 256, dtype=torch.bfloat16, device=dev)
        idd = ids.to(dt).to(dev)
        tabd = tab.to(dev)
        _lib.check(lib.evo_embed(_lib.ptr(idd), int(dt == torch.int64), _lib.ptr(tabd), _lib.ptr(od), 33, 256, 512, stream()))
        emit("elementwise", op="embed", dtype=str(dt), equal=bool(torch.equal(od.cpu().view(3, 11, 256), tab[ids])))
    # rope tables + rotary
    for scaling in (1.0, 16.0):
        Lr = 300
        cos_ref, sin_ref = O.rotary_tables(Lr, 128, scaling_factor=scaling, dtype=torch.bfloat16)
        inv = (1.0 / (10000 ** (torch.arange(0, 128, 2, dtype=torch.float32) / 128))).to(dev)
        cd = torch.empty(Lr, 64, dtype=torch.bfloat16, device=dev); sdv = torch.empty_like(cd)
        _lib.check(lib.evo_rope_tables(_lib.ptr(cd), _lib.ptr(sdv), _lib.ptr(inv), 0, Lr, 64, scaling, stream()))
        emit("elementwise", op="rope_tables", scaling=scaling, cos_exact=(cd.cpu() == cos_ref).float().mean().item(),
             sin_exact=(sdv.cpu() == sin_ref).float().mean().item(), **err(cd, cos_ref))
        qkv = torch.randn(2, Lr, 3, 2, 128).bfloat16()
        q_ref = O.apply_rotary(qkv[:, :, 0], cos_ref, sin_ref); k_ref = O.apply_rotary(qkv[:, :, 1], cos_ref, sin_ref)
        qd = qkv.to(dev).contiguous()
        cdev, sdev = cos_ref.to(dev), sin_ref.to(dev)      # keep alive: a temporary could be freed + reused before the launch
        _lib.check(lib.evo_rotary_qk(_lib.ptr(qd), _lib.ptr(cdev), _lib.ptr(sdev), 2, Lr, 2, 128, stream()))
        qc = qd.cpu()
        emit("elementwise", op="rotary", scaling=scaling, q=err(qc[:, :, 0], q_ref), k=err(qc[:, :, 1], k_ref),
             v_untouched=bool(torch.equal(qc[:, :, 2], qkv[:, :, 2])))
    # logprobs
    lg = (torch.randn(50, 512) * 3).bfloat16(); tg = torch.randint(0, 512, (50,)); tg[3] = -1
    od = torch.empty(50, dtype=torch.float32, device=dev)
    lgd, tgd = lg.to(dev), tg.to(dev)
    _lib.check(lib.evo_logprobs(_lib.ptr(lgd), _lib.ptr(tgd), _lib.ptr(od), 50, 512, stream()))
    ref = torch.log_softmax(lg.float(), -1).gather(1, tg.clamp(min=0)[:, None])[:, 0]; ref[3] = 0
    emit("elementwise", op="logprobs", **err(od, ref))
    # kv append
    qkv = torch.randn(2, 5, 3, 2, 128).bfloat16()
    cache = torch.zeros(3, 16, 2, 2, 128, dtype=torch.bfloat16, device=dev)
    qkvd = qkv.to(dev)
    _lib.check(lib.evo_kv_append(_lib.ptr(qkvd), _lib.ptr(cache), 2, 5, 2, 128, 4, 16, stream()))
    cc = cache.cpu()
    ok = torch.equal(cc[:2, 4:9, 0], qkv[:, :, 1]) and torch.equal(cc[:2, 4:9, 1], qkv[:, :, 2]) and cc[:, :4].abs().sum() == 0 and cc[2].abs().sum() == 0
    emit("elementwise", op="kv_append", equal=bool(ok))


def _hyena_call(z, f, B, L, D, H, force=0, halo=None, state_in=None, want_state=True, state_only=False):
    lib = _lib.lib()
    dev = z.device
    y = torch.empty(B, L, D, dtype=torch.bfloat16, device=dev)
    st = torch.empty(B, D, 8, 2, dtype=torch.float32, device=dev)
    fs = torch.empty(B, 3 * D, 2, dtype=torch.bfloat16, device=dev)
    hp = _lib.HyenaParams(z=z.data_ptr(), y=y.data_ptr(), fir_w=f["w"].data_ptr(), fir_b=f["b"].data_ptr(), Dskip=f["D"].data_ptr(),
                          poles=f["p"].data_ptr(), residues=f["r"].data_ptr(), B=B, L=L, D=D, S=8, nheads=H,
                          halo=halo.data_ptr() if halo is not None else None,
                          state_in=state_in.data_ptr() if state_in is not None else None,
                          state_out=st.data_ptr() if want_state else None, fir_state_out=fs.data_ptr() if want_state else None,
                          force_segments=force, state_only=int(state_only))
    n = lib.evo_hyena_fwd_workspace(C.byref(hp))
    ws = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
    _lib.check(lib.evo_hyena_fwd(C.byref(hp), _lib.ptr(ws), n, stream()), "hyena")
    torch.cuda.synchronize()
    return y, st, fs


def stage_hyena():
    dev = "cuda:0"
    D, H = 256, 2
    cfg = O.tiny_config(num_layers=1, attn_layer_idxs=(), hidden_size=D, num_heads=H)
    sd = O.random_state_dict(cfg, seed=1)
    pre = "blocks.0.filter."
    f = {"w": sd[pre + "short_filter_weight"].to(dev), "b": sd[pre + "short_filter_bias"].to(dev), "D": sd[pre + "D"].to(dev),
         "p": sd[pre + "poles"].to(dev), "r": sd[pre + "residues"].to(dev)}
    mb = O.OracleStripedHyena(cfg, sd, torch.bfloat16)
    mt = O.OracleStripedHyena(cfg, sd, torch.float64)
    for (B, L) in ((1, 1), (2, 2), (2, 7), (3, 130), (2, 1025), (1, 4099)):
        torch.manual_seed(L)
        z = torch.randn(B, L, 3 * D).bfloat16()
        ipb, ipt = mb.initialize_inference_params()["hyena"], mt.initialize_inference_params()["hyena"]
        yb = mb.hyena_operator(0, z, ipb)
        yt = mt.hyena_operator(0, z.double(), ipt)
        for force in (1, 3):
            if force > 1 and L < 8:
                continue
            y, st, fs = _hyena_call(z.to(dev), f, B, L, D, H, force=force)
            stc = torch.view_as_complex(st.cpu())
            emit("hyena", B=B, L=L, nseg=force, vs_bf16_oracle=err(y, yb), vs_truth=err(y, yt), oracle_vs_truth=err(yb, yt),
                 exact_frac=(y.cpu() == yb).float().mean().item(),
                 state_abs=(stc - ipt.state_dict[0].to(torch.complex64)).abs().max().item(),
                 state_ref=ipt.state_dict[0].abs().max().item(),
                 fir_equal=bool(torch.equal(fs.cpu(), ipb.fir_state_dict[0])))
    # continuation: two halves with halo + state_in == one pass
    B, L = 2, 600
    z = torch.randn(B, L, 3 * D).bfloat16().to(dev)
    y_full, st_full, fs_full = _hyena_call(z, f, B, L, D, H, force=1)
    a = z[:, :250].contiguous(); b = z[:, 250:].contiguous()
    ya, sta, fsa = _hyena_call(a, f, B, 250, D, H, force=1)
    yb2, stb, fsb = _hyena_call(b, f, B, 350, D, H, force=2, halo=a[:, -2:].contiguous(), state_in=sta)
    emit("hyena", op="continuation", y=err(torch.cat([ya, yb2], 1), y_full), state=err(stb, st_full), fir_equal=bool(torch.equal(fsb, fs_full)))
    # state_only pass + combine (sequence-parallel algebra)
    lib = _lib.lib()
    _, e0, _ = _hyena_call(z[:, :300].contiguous(), f, B, 300, D, H, state_only=True)
    _, e1, _ = _hyena_call(z[:, 300:].contiguous(), f, B, 300, D, H, state_only=True, halo=z[:, 298:300].contiguous())
    ends = torch.stack([e0, e1]).contiguous()
    sin1 = torch.empty_like(e0)
    _lib.check(lib.evo_hyena_combine_states(_lib.ptr(ends), _lib.ptr(sin1), _lib.ptr(f["p"]), 1, 2, 300, B, D, 8, stream()))
    y1, st1, _ = _hyena_call(z[:, 300:].contiguous(), f, B, 300, D, H, halo=z[:, 298:300].contiguous(), state_in=sin1)
    emit("hyena", op="seqpar_2way", y=err(y1, y_full[:, 300:]), state=err(st1, st_full), e0_vs_prefix=err(e0, _hyena_call(z[:, :300].contiguous(), f, B, 300, D, H)[1]))
    # step kernel
    ipb = mb.initialize_inference_params()["hyena"]
    zc = z[:, :40].cpu()
    mb.hyena_operator(0, zc, ipb)
    fs = ipb.fir_state_dict[0].clone().to(dev).contiguous(); st = torch.view_as_real(ipb.state_dict[0].clone()).contiguous().to(dev)
    u = z[:, 40].contiguous()
    yref = mb.hyena_operator(0, z[:, 40:41].cpu(), ipb)[:, 0]
    yd = torch.empty(B, D, dtype=torch.bfloat16, device=dev)
    _lib.check(lib.evo_hyena_step(_lib.ptr(u), _lib.ptr(yd), _lib.ptr(fs), _lib.ptr(st), _lib.ptr(f["w"]), _lib.ptr(f["b"]), _lib.ptr(f["D"]),
                                  _lib.ptr(f["p"]), _lib.ptr(f["r"]), B, D, 8, H, stream()))
    emit("hyena", op="step", y=err(yd, yref), exact_frac=(yd.cpu() == yref).float().mean().item(),
         state=err(st, torch.view_as_real(ipb.state_dict[0])), fir_equal=bool(torch.equal(fs.cpu(), ipb.fir_state_dict[0])))


def _gemm(a, w, M, N, K, epi, variant, bias=None, resid=None, ldc=None):
    out = torch.full((M, ldc or N), float("nan"), dtype=torch.bfloat16, device=a.device)
    p = _lib.GemmParams(A=a.data_ptr(), lda=K, W=w.data_ptr(), C=out.data_ptr(), ldc=ldc or N,
                        bias=bias.data_ptr() if bias is not None else None, residual=resid.data_ptr() if resid is not None else None,
                        ldr=ldc or N, M=M, N=N, K=K, epilogue=epi, variant=variant)
    _lib.check(_lib.lib().evo_gemm(C.byref(p), stream()), "evo_gemm")
    return out


def stage_gemm(variant):
    dev = "cuda:0"
    name = "gemm1" if variant == 1 else "gemm2"
    for (M, N, K) in ((128, 256, 64), (256, 256, 128), (300, 512, 256), (1000, 768, 256), (4096, 4096, 4096), (8200, 512, 1024)):
        torch.manual_seed(M)
        a = (torch.randn(M, K, device=dev) * 0.5).bfloat16()
        w = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
        bias = (torch.randn(N, device=dev) * 0.2).bfloat16()
        acc = a.float() @ w.float().T
        out = _gemm(a, w, M, N, K, _lib.EPI_NONE, variant); torch.cuda.synchronize()
        emit(name, epi="none", M=M, N=N, K=K, **err(out, acc.bfloat16()))
        out = _gemm(a, w, M, N, K, _lib.EPI_BIAS, variant, bias=bias); torch.cuda.synchronize()
        emit(name, epi="bias", M=M, N=N, K=K, **err(out, (acc + bias.float()).bfloat16()))
        resid = torch.randn(M, N, device=dev).bfloat16()
        out = _gemm(a, w, M, N, K, _lib.EPI_BIAS_RESID, variant, bias=bias, resid=resid); torch.cuda.synchronize()
        emit(name, epi="bias_resid", M=M, N=N, K=K, **err(out, ((acc + bias.float()).bfloat16().float() + resid.float()).bfloat16()))
        out = _gemm(a, w, M, N, K, _lib.EPI_RESID, variant, resid=resid); torch.cuda.synchronize()
        emit(name, epi="resid", M=M, N=N, K=K, **err(out, (acc.bfloat16().float() + resid.float()).bfloat16()))
        # gelu-gate: W rows = [l1 128 | l2 128] per 256 tile
        wv = w.view(N // 256, 2, 128, K)
        z1 = (a.float() @ wv[:, 0].reshape(-1, K).float().T).bfloat16()
        z2 = (a.float() @ wv[:, 1].reshape(-1, K).float().T).bfloat16()
        ref = (torch.nn.functional.gelu(z1.float()).bfloat16().float() * z2.float()).bfloat16()
        out = _gemm(a, w, M, N, K, _lib.EPI_GELU_GATE, variant, ldc=N // 2); torch.cuda.synchronize()
        emit(name, epi="gelu_gate", M=M, N=N, K=K, **err(out, ref))


def _attn(qkv, B, L, H, variant, simple=False, cache=None, off=0):
    dev = qkv.device
    d = H * 128
    out = torch.full((B, L, d), float("nan"), dtype=torch.bfloat16, device=dev)
    ap = _lib.AttnParams(out=out.data_ptr(), B=B, Lq=L, H=H, hd=128, q_pos0=off, softmax_scale=1 / math.sqrt(128))
    ap.q, ap.q_tok_stride, ap.q_batch_stride = qkv.data_ptr(), 3 * d, L * 3 * d
    if cache is None:
        ap.k, ap.v, ap.kv_tok_stride, ap.kv_batch_stride, ap.Lk = qkv.data_ptr() + 2 * d, qkv.data_ptr() + 4 * d, 3 * d, L * 3 * d, L
    else:
        ap.k, ap.v, ap.kv_tok_stride, ap.kv_batch_stride, ap.Lk = cache.data_ptr(), cache.data_ptr() + 2 * d, 2 * d, cache.shape[1] * 2 * d, off + L
    lib = _lib.lib()
    if simple:
        from tests import support as TS
        TS.check(TS.lib().evot_attn_fwd_simple(C.byref(ap), stream()), "attn_simple")
    else:
        n = lib.evo_attn_fwd_workspace(C.byref(ap), variant)
        ws = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        _lib.check(lib.evo_attn_fwd_ws(C.byref(ap), variant, _lib.ptr(ws), n, stream()), "attn")
    torch.cuda.synchronize()
    return out


def stage_attn(variant):
    dev = "cuda:0"
    name = f"attn{variant}"
    H = 2
    for (B, L) in ((1, 1), (2, 37), (1, 128), (2, 129), (1, 300), (2, 1000), (1, 2500)):
        torch.manual_seed(L)
        qkv = torch.randn(B, L, 3, H, 128).bfloat16()
        ref = O.causal_attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]).reshape(B, L, H * 128)
        truth = O.causal_attention(qkv[:, :, 0].double(), qkv[:, :, 1].double(), qkv[:, :, 2].double()).reshape(B, L, H * 128)
        qd = qkv.to(dev)
        s = _attn(qd, B, L, H, variant, simple=True)
        emit(name, kind="simple", B=B, L=L, vs_oracle=err(s, ref), vs_truth=err(s, truth))
        o = _attn(qd, B, L, H, variant)
        emit(name, kind="wgmma", B=B, L=L, vs_oracle=err(o, ref), vs_truth=err(o, truth), oracle_vs_truth=err(ref, truth))
    # KV-cache form: 1 and 5 new queries at offset 200 of a 512-row cache
    B, Lc = 2, 512
    full = torch.randn(B, 260, 3, H, 128).bfloat16()
    cache = torch.zeros(B, Lc, 2, H, 128, dtype=torch.bfloat16)
    cache[:, :260, 0] = full[:, :, 1]; cache[:, :260, 1] = full[:, :, 2]
    ref_full = O.causal_attention(full[:, :, 0], full[:, :, 1], full[:, :, 2]).reshape(B, 260, H * 128)
    for (off, Lq) in ((200, 1), (200, 5), (255, 5)):
        q = full[:, off:off + Lq].contiguous().to(dev)
        o = _attn(q, B, Lq, H, variant, cache=cache.to(dev), off=off)
        emit(name, kind="kvcache", off=off, Lq=Lq, **err(o, ref_full[:, off:off + Lq]))


def stage_model():
    dev = "cuda:0"
    cfg = O.tiny_config(num_layers=4, attn_layer_idxs=(1, 3), hidden_size=256, num_heads=2)
    sd = O.random_state_dict(cfg, seed=7)
    m = StripedHyena(dotdict(cfg)); m.load_state_dict(sd, strict=True); m.to_bfloat16_except_poles_residues(); m = m.to(dev)
    ob = O.OracleStripedHyena(cfg, sd, torch.bfloat16); ot = O.OracleStripedHyena(cfg, sd, torch.float64)
    torch.manual_seed(0)
    ids = torch.randint(0, 4, (2, 333)) * 3 + 65
    lg, _ = m(ids.to(dev)); torch.cuda.synchronize()
    lb, _ = ob(ids); lt, _ = ot(ids)
    lsm = lambda x: torch.log_softmax(x.double().cpu(), -1)
    emit("model", logits_vs_oracle=err(lg, lb), logits_vs_truth=err(lg, lt), oracle_vs_truth=err(lb, lt),
         logprob_mean_abs_vs_truth=(lsm(lg) - lsm(lt)).abs().mean().item(), oracle_logprob_mean_abs_vs_truth=(lsm(lb) - lsm(lt)).abs().mean().item(),
         argmax_agree=(lg.cpu().argmax(-1) == lt.argmax(-1)).float().mean().item())
    # stateful: prefill 300 then 33 steps, against the stateless logits
    d = m.initialize_inference_params(); d["mha"].max_batch_size = 2; d["mha"].max_seqlen = 512
    pre, d = m(ids[:, :300].to(dev), inference_params_dict=d)
    errs = [err(pre, lg[:, :300])["max_abs"]]
    d["mha"].seqlen_offset = d["hyena"].seqlen_offset = 300
    for t in range(300, 333):
        s, d = m(ids[:, t:t + 1].to(dev), inference_params_dict=d)
        errs.append((s[:, 0].float() - lg[:, t].float()).abs().max().item())
        d["mha"].seqlen_offset += 1; d["hyena"].seqlen_offset += 1
    emit("model", stateful_prefill_max=errs[0], stateful_step_max=max(errs[1:]), logit_scale=lg.float().abs().max().item())


def stage_perf_gemm():
    dev = "cuda:0"
    ws = torch.empty(64 << 20, dtype=torch.uint8, device=dev)
    for (M, N, K, epi) in ((8192, 12288, 4096, 1), (65536, 12288, 4096, 1), (65536, 4096, 4096, 2), (65536, 22016, 4096, 4), (65536, 4096, 11008, 3), (65536, 512, 4096, 0), (16, 12288, 4096, 1)):
        a = (torch.randn(M, K, device=dev) * 0.5).bfloat16(); w = (torch.randn(N, K, device=dev) / 64).bfloat16()
        bias = torch.randn(N, device=dev).bfloat16()
        nout = N // 2 if epi == 4 else N
        resid = torch.randn(M, nout, device=dev).bfloat16()
        flops = 2.0 * M * N * K
        rec = {"M": M, "N": N, "K": K, "epi": epi}
        for variant in (0, 1):
            try:
                fn = lambda: _gemm(a, w, M, N, K, epi, variant, bias=bias, resid=resid, ldc=nout)
                ms = timeit(fn)
                rec[f"wgmma_v{variant}_ms"] = ms; rec[f"wgmma_v{variant}_tflops"] = flops / ms / 1e9
            except Exception as e:  # noqa
                rec[f"wgmma_v{variant}_err"] = str(e)[:200]
        out = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
        p = _lib.GemmParams(A=a.data_ptr(), lda=K, W=w.data_ptr(), C=out.data_ptr(), ldc=N, bias=bias.data_ptr(), residual=None, ldr=N, M=M, N=N, K=K, epilogue=1, variant=0)
        from tests import support as TS
        fn = lambda: TS.check(TS.lib().evot_gemm_cublaslt(C.byref(p), _lib.ptr(ws), ws.numel(), stream()))
        ms = timeit(fn); rec["cublaslt_ms"] = ms; rec["cublaslt_tflops"] = flops / ms / 1e9
        ms = timeit(lambda: torch.matmul(a, w.T)); rec["torch_ms"] = ms; rec["torch_tflops"] = flops / ms / 1e9
        emit("perf_gemm", **rec)


def stage_perf_hyena():
    dev = "cuda:0"
    D, H = 4096, 32
    cfg = O.tiny_config(num_layers=1, attn_layer_idxs=(), hidden_size=D, num_heads=H)
    sd = O.random_state_dict(cfg, seed=1)
    pre = "blocks.0.filter."
    f = {"w": sd[pre + "short_filter_weight"].to(dev), "b": sd[pre + "short_filter_bias"].to(dev), "D": sd[pre + "D"].to(dev),
         "p": sd[pre + "poles"].to(dev), "r": sd[pre + "residues"].to(dev)}
    for (B, L, force) in ((8, 8193, 0), (8, 8193, 2), (1, 131072, 0), (1, 16384, 0), (16, 4096, 0)):
        z = torch.randn(B, L, 3 * D, device=dev).bfloat16()
        ms = timeit(lambda: _hyena_call(z, f, B, L, D, H, force=force, want_state=False), iters=5)
        emit("perf_hyena", B=B, L=L, force=force, ms=ms, algo_GBs=8.0 * B * L * D / ms / 1e6)


def stage_perf_attn():
    dev = "cuda:0"
    H = 32
    for (B, L) in ((1, 8192), (8, 8193), (1, 32768)):
        qkv = torch.randn(B, L, 3, H, 128, device=dev).bfloat16()
        flops = 2.0 * B * L * L * H * 128       # causal-effective: 4*B*L^2*H*d / 2
        for variant in (0, 1, 2):
            ms = timeit(lambda: _attn(qkv, B, L, H, variant), iters=3, warm=1)
            emit("perf_attn", B=B, L=L, variant=variant, ms=ms, tflops=flops / ms / 1e9)
        if L <= 8193:
            try:
                from flash_attn import flash_attn_qkvpacked_func
                ms = timeit(lambda: flash_attn_qkvpacked_func(qkv, causal=True), iters=3, warm=1)
                emit("perf_attn", B=B, L=L, variant="flash_attn2_library", ms=ms, tflops=flops / ms / 1e9)
            except Exception as e:  # noqa
                emit("perf_attn", B=B, L=L, variant="flash_attn2_library", error=str(e)[:200])


def stage_perf_decode():
    """BASELINE configs[3]: evo-1.5-8k-base generate, batch 16, prompt 4096 + decode (recurrent state path)."""
    from evo_b200.models import load_checkpoint
    dev = "cuda:0"
    m = load_checkpoint("evo-1.5-8k-base", device=dev, random_init=True, seed=0)
    B, P, N = 16, 4096, 96
    g = torch.Generator().manual_seed(0)
    ids = (torch.randint(0, 4, (B, P + N), generator=g) * 3 + 65).to(dev)
    d = m.initialize_inference_params()
    d["mha"].max_batch_size = B
    d["hyena"].max_batch_size = B
    torch.cuda.synchronize(); t0 = time.time()
    lg, d = m(ids[:, :P], inference_params_dict=d)
    torch.cuda.synchronize(); t_prefill = time.time() - t0
    d["mha"].seqlen_offset = d["hyena"].seqlen_offset = P
    outs = []
    times = []
    for t in range(P, P + N):
        torch.cuda.synchronize(); t0 = time.time()
        s, d = m(ids[:, t:t + 1], inference_params_dict=d)
        torch.cuda.synchronize(); times.append(time.time() - t0)
        outs.append(s[:, 0])
        d["mha"].seqlen_offset += 1; d["hyena"].seqlen_offset += 1
    steady = sorted(times[8:])[len(times[8:]) // 2]
    # per-kernel-class breakdown of one eager (non-graph) step with CUDA events
    m._prof = []
    s, d = m(ids[:, P + N - 1:P + N], inference_params_dict=d)
    torch.cuda.synchronize()
    agg = {}
    for kind, work, e0, e1 in m._prof:
        a_ = agg.setdefault(kind, [0, 0.0, 0.0]); a_[0] += 1; a_[1] += e0.elapsed_time(e1) * 1e3; a_[2] += work
    m._prof = None
    breakdown = {k: {"n": v[0], "us_total": round(v[1], 1), "us_each": round(v[1] / v[0], 1), "weight_GBs": round(v[2] / (2.0 * B) * 2 / (v[1] * 1e-6) / 1e9, 1)} for k, v in agg.items()}
    # sanity: teacher-forced decode logits vs one stateless forward over the same P+N tokens (last 8 positions)
    full, _ = m(ids[:2, :P + N])
    dec = torch.stack(outs, 1)[:2]
    e = (dec[:, -8:].float() - full[:, P + N - 8:].float()).abs()
    emit("perf_decode", B=B, prompt=P, steps=N, prefill_s=t_prefill, prefill_nt_s=B * P / t_prefill, first_step_ms=times[0] * 1e3, capture_step_ms=times[1] * 1e3,
         steady_ms_per_step=steady * 1e3, decode_nt_s=B / steady, decode_vs_stateless_max=e.max().item(), logit_scale=full.float().abs().max().item(),
         weight_stream_floor_ms=12.9e9 / 6566.4e9 * 1e3, eager_breakdown=breakdown,
         env={k: os.environ.get(k) for k in ("EVO_B200_DECODE_STREAMK", "EVO_B200_DECODE_PDL", "EVO_B200_DECODE_GRAPH")})


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--stage", default=None)
    ap.add_argument("--stages", default=",".join(STAGES))
    ap.add_argument("--timeout", type=int, default=240)
    a = ap.parse_args()
    if a.stage is None:
        main_driver(a.stages.split(","), a.timeout)
    else:
        _imports()
        {"elementwise": stage_elementwise, "hyena": stage_hyena, "gemm1": lambda: stage_gemm(1), "gemm2": lambda: stage_gemm(0),
         "attn0": lambda: stage_attn(0), "attn1": lambda: stage_attn(1), "attn2": lambda: stage_attn(2), "model": stage_model, "perf_gemm": stage_perf_gemm,
         "perf_hyena": stage_perf_hyena, "perf_attn": stage_perf_attn, "perf_decode": stage_perf_decode}[a.stage]()
