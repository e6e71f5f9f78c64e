"""Micro-benchmark of the decode-step kernels inside CUDA graphs (run on the GPU box).

For each linear-layer shape of the 7B decode step: a graph of back-to-back launches that rotates over several
weight copies (so L2 never holds the weights), replayed and timed with CUDA events -> us per launch including
the in-graph launch gap, GB/s of weight stream.  Also the small kernels and one synthetic layer chain.
    python tools/decode_micro.py [--pdl 0|1] [--m 16] [--out out/decode_micro.jsonl]
"""
import argparse
import ctypes as C
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from evo_b200 import _lib  # noqa: E402

DEV = "cuda:0"


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def graph_time(fn, reps=5):
    """fn() enqueues the work once; returns ms per replay of the captured graph."""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pdl", type=int, default=0)
    ap.add_argument("--m", type=int, default=16)
    ap.add_argument("--out", default="out/decode_micro.jsonl")
    ap.add_argument("--ncu", action="store_true", help="launch every kernel 3x eagerly and exit (for an ncu duration list)")
    a = ap.parse_args()
    lib = _lib.lib()
    M = a.m
    torch.manual_seed(0)
    ws = torch.zeros(lib.evo_gemm_smallm_workspace(M, 256, 64, 4), dtype=torch.uint8, device=DEV)
    recs = []

    def emit(**kw):
        kw.update(pdl=a.pdl, M=M)
        print(json.dumps(kw), flush=True)
        recs.append(kw)

    def mk_gemm(N, K, epi, kind, copies):
        n_out = N // 2 if epi == 4 else N
        A = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
        Ws = [(torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16() for _ in range(copies)]
        bias = torch.randn(N, device=DEV).bfloat16()
        resid = torch.randn(M, n_out, device=DEV).bfloat16()
        out = torch.empty(M, n_out, dtype=torch.bfloat16, device=DEV)
        keep = (A, Ws, bias, resid, out)

        def launch(i):
            w = Ws[i % copies]
            if kind == "streamk":
                p = _lib.GemmSmallMParams(A=A.data_ptr(), lda=K, W=w.data_ptr(), C=out.data_ptr(), ldc=n_out, bias=bias.data_ptr(), residual=resid.data_ptr(), ldr=n_out,
                                          M=M, N=N, K=K, epilogue=epi, workspace=ws.data_ptr(), workspace_bytes=ws.numel())
                _lib.check(lib.evo_gemm_smallm(C.byref(p), stream()), "evo_gemm_smallm")
            else:
                p = _lib.GemmParams(A=A.data_ptr(), lda=K, W=w.data_ptr(), C=out.data_ptr(), ldc=n_out, bias=bias.data_ptr(), residual=resid.data_ptr(), ldr=n_out,
                                    M=M, N=N, K=K, epilogue=0 if epi == 4 else epi, variant=2)
                _lib.check(lib.evo_gemm(C.byref(p), stream()), "evo_gemm")
        return launch, keep

    lib.evo_set_pdl(a.pdl)
    NL = 32
    shapes = [("in", 12288, 4096, 1), ("out", 4096, 4096, 2), ("w12", 22016, 4096, 4), ("w3", 4096, 11008, 3), ("unembed", 512, 4096, 0)]
    gemms = {}
    if a.ncu:
        for name, N, K, epi in shapes:
            for kind in ("streamk", "tile64"):
                launch, keep = mk_gemm(N, K, epi, kind, 3)
                for i in range(3):
                    launch(i)
                torch.cuda.synchronize()
        Bc, S, Hh = M, 8192, 32
        cache = torch.randn(Bc, S, 2, Hh, 128, device=DEV).bfloat16()
        qkv = torch.randn(Bc, 3, Hh, 128, device=DEV).bfloat16()
        ctxo = torch.empty(Bc, Hh * 128, dtype=torch.bfloat16, device=DEV)
        posd = torch.full((1,), 4095, dtype=torch.int64, device=DEV)
        nws = lib.evo_decode_attn_workspace(Bc, Hh, 3)
        wsa = torch.empty(nws, dtype=torch.uint8, device=DEV)
        for _ in range(2):
            _lib.check(lib.evo_decode_attn(_lib.ptr(qkv), _lib.ptr(cache), _lib.ptr(ctxo), _lib.ptr(posd), Bc, Hh, 128, S, 3, 1.0 / math.sqrt(128), _lib.ptr(wsa), nws, stream()))
        torch.cuda.synchronize()
        return
    for name, N, K, epi in shapes:
        copies = max(2, min(8, int(400e6 // (N * K * 2)) + 1))
        for kind in ("streamk", "tile64"):
            launch, keep = mk_gemm(N, K, epi, kind, copies)
            ms = graph_time(lambda: [launch(i) for i in range(NL)])
            emit(what=f"gemm_{name}", kind=kind, N=N, K=K, us_per_launch=ms * 1e3 / NL, weight_GBs=N * K * 2 / (ms * 1e-3 / NL) / 1e9, copies=copies)
            if kind == "streamk":
                gemms[name] = (launch, keep)

    # small kernels
    D, H = 4096, 32
    x = torch.randn(M, D, device=DEV).bfloat16()
    y = torch.empty_like(x)
    scale = torch.ones(D, device=DEV).bfloat16()
    ms = graph_time(lambda: [_lib.check(lib.evo_rmsnorm(_lib.ptr(x), _lib.ptr(scale), _lib.ptr(y), M, D, 1e-6, stream())) for _ in range(NL)])
    emit(what="rmsnorm", us_per_launch=ms * 1e3 / NL)
    z = torch.randn(M, 3 * D, device=DEV).bfloat16()
    fir_state = torch.randn(M, 3 * D, 2, device=DEV).bfloat16()
    state = torch.randn(M, D, 8, 2, device=DEV)
    fw = torch.randn(3 * D, 3, device=DEV).bfloat16(); fb = torch.randn(3 * D, device=DEV).bfloat16(); Dk = torch.randn(D, device=DEV).bfloat16()
    poles = torch.rand(D, 8, 2, device=DEV) * 0.5; res = torch.randn(D, 8, 2, device=DEV)

    def hy():
        _lib.check(lib.evo_hyena_step(_lib.ptr(z), _lib.ptr(y), _lib.ptr(fir_state), _lib.ptr(state), _lib.ptr(fw), _lib.ptr(fb), _lib.ptr(Dk),
                                      _lib.ptr(poles), _lib.ptr(res), M, D, 8, H, stream()))
    ms = graph_time(lambda: [hy() for _ in range(NL)])
    emit(what="hyena_step", us_per_launch=ms * 1e3 / NL)

    # decode attention: one query per sequence over a 4096-token KV cache (1.07 GB of K,V per launch at B=16)
    Bc, ctx, S = M, 4096, 8192
    cache = torch.randn(Bc, S, 2, H, 128, device=DEV).bfloat16()
    qkv = torch.randn(Bc, 3, H, 128, device=DEV).bfloat16()
    ctxo = torch.empty(Bc, H * 128, dtype=torch.bfloat16, device=DEV)
    posd = torch.full((1,), ctx - 1, dtype=torch.int64, device=DEV)
    for nsplit in (1, 2, 3, 4, 8):
        nws = lib.evo_decode_attn_workspace(Bc, H, nsplit)
        wsa = torch.empty(nws, dtype=torch.uint8, device=DEV)
        fn = lambda: [_lib.check(lib.evo_decode_attn(_lib.ptr(qkv), _lib.ptr(cache), _lib.ptr(ctxo), _lib.ptr(posd), Bc, H, 128, S, nsplit,
                                                     1.0 / math.sqrt(128), _lib.ptr(wsa), nws, stream())) for _ in range(4)]
        ms = graph_time(fn)
        kv_bytes = Bc * ctx * 2 * H * 128 * 2
        emit(what="decode_attn", nsplit=nsplit, ctx=ctx, us_per_launch=ms * 1e3 / 4, kv_GBs=kv_bytes / (ms * 1e-3 / 4) / 1e9)
    del cache

    # one synthetic Hyena layer chain x 32 (weights rotate): rmsnorm, in, step, out, rmsnorm, w12(gate), w3
    def chain():
        for i in range(NL):
            _lib.check(lib.evo_rmsnorm(_lib.ptr(x), _lib.ptr(scale), _lib.ptr(y), M, D, 1e-6, stream()))
            gemms["in"][0](i)
            hy()
            gemms["out"][0](i)
            _lib.check(lib.evo_rmsnorm(_lib.ptr(x), _lib.ptr(scale), _lib.ptr(y), M, D, 1e-6, stream()))
            gemms["w12"][0](i)
            gemms["w3"][0](i)
    ms = graph_time(chain)
    emit(what="layer_chain_x32", ms_per_step=ms, us_per_layer=ms * 1e3 / NL, floor_ms=NL * 402.8e6 / 6566.4e9 * 1e3)
    lib.evo_set_pdl(0)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "a") as f:
        for r in recs:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
