"""bf16 against FP8 weights for the decode step, timed alternately in one run (GPU only).

  * the four 7B decode GEMMs (Wqkv / projections 12288x4096 + bias, out 4096x4096 + bias + residual, packed w12 22016x4096 with
    the GELU gate, w3 4096x11008 + residual) at M = 1, 16 and 64: evo_gemm_smallm on the bf16 weights against
    evo_gemm_smallm_fp8 on their E4M3 copies.  Each measurement is a CUDA graph of back-to-back launches rotating over enough
    weight copies that L2 never holds them, timed with CUDA events after a warm-up; us per launch, GB/s of weight bytes and
    the share of the H100 SXM's 3.35 TB/s;
  * the decode step at bench.py's generation geometry (random-init 7B, B = 16, a 4096-token prompt): decode_loop in ms per
    step, FP8 against the same model's bf16 kernel on its rounded weights (equal bytes to a bf16 model).
The card's name and power limit are read in the same run.  One JSON line per measurement.
    python tools/decode_fp8_micro.py [--out out/decode_fp8_micro.jsonl] [--rounds 5] [--steps 64]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from evo_b200 import _lib  # noqa: E402

DEV = "cuda:0"
HBM = 3.35e12
SHAPES = [("qkv", 12288, 4096, _lib.EPI_BIAS), ("out", 4096, 4096, _lib.EPI_BIAS_RESID), ("w12", 22016, 4096, _lib.EPI_GELU_GATE),
          ("w3", 4096, 11008, _lib.EPI_RESID)]


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip() or torch.cuda.get_device_name(0)


def graph(fn):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    return g


def time_graph(g, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def gemm_graphs(name, N, K, epi, M, ws):
    lib = _lib.lib()
    gate = epi == _lib.EPI_GELU_GATE
    n_out = N // 2 if gate else N
    copies = max(2, -(-400 * 2 ** 20 // (2 * N * K)))             # > 4x the 50 MB L2 in bf16 bytes
    ws_ = [torch.randn(N, K, device=DEV).mul_(K ** -0.5).bfloat16() for _ in range(copies)]
    f8 = []
    for w in ws_:
        q = torch.empty(lib.evo_fp8_weight_bytes(N, K, epi), dtype=torch.uint8, device=DEV)
        e = torch.empty(N, dtype=torch.int8, device=DEV)
        st = torch.zeros(1, dtype=torch.int32, device=DEV)
        _lib.check(lib.evo_fp8_quantize_rows(w.data_ptr(), N, K, epi, q.data_ptr(), e.data_ptr(), st.data_ptr(), stream()), "quantize")
        f8.append((q, e))
    a = torch.randn(M, K, device=DEV).bfloat16()
    c = torch.empty(M, n_out, device=DEV, dtype=torch.bfloat16)
    bias = torch.randn(N, device=DEV).bfloat16()
    r = torch.randn(M, n_out, device=DEV).bfloat16()
    reps = 8

    def params(i, fp8):
        p = _lib.GemmSmallMParams(A=a.data_ptr(), lda=K, W=(f8[i][0] if fp8 else ws_[i]).data_ptr(), C=c.data_ptr(), ldc=n_out,
                                  bias=bias.data_ptr(), residual=r.data_ptr(), ldr=n_out, M=M, N=N, K=K, epilogue=epi,
                                  workspace=ws.data_ptr(), workspace_bytes=ws.numel())
        return _lib.GemmSmallMFp8Params(base=p, W_exp=f8[i][1].data_ptr()) if fp8 else p

    def run(fp8):
        ps = [params(i, fp8) for i in range(copies)]

        def fn():
            for _ in range(reps):
                for p in ps:
                    if fp8:
                        _lib.check(lib.evo_gemm_smallm_fp8(C.byref(p), stream()), "fp8")
                    else:
                        _lib.check(lib.evo_gemm_smallm(C.byref(p), stream()), "bf16")
        return graph(fn), reps * copies
    return {"bf16": run(False), "fp8": run(True)}


def step_states(model, B, P, steps):
    """Prefill B prompts of P tokens once; a decode_loop graph state per mode (bf16 kernel on W', FP8)."""
    d = model.initialize_inference_params()
    d["mha"].max_batch_size, d["mha"].max_seqlen = B, P + steps + 64
    ids = torch.randint(0, 4, (B, P), device=DEV) * 3 + 65
    with torch.inference_mode():
        logits, d = model(ids, inference_params_dict=d)
    first = logits[:, -1].float().argmax(-1)
    model._ensure_fp8()                       # the bf16 comparator's capture then records the same addresses as later calls
    st = {}
    for mode in ("bf16", "fp8"):
        model._fp8_decode_bf16 = mode == "bf16"
        model._loop = None
        with torch.inference_mode():
            model.decode_loop(first, d, steps, P, top_k=1)
        st[mode] = model._loop
    return d, first, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="out/decode_fp8_micro.jsonl")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--no-step", action="store_true", help="GEMMs only")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_fp8_micro.py measures on the GPU; no GPU here")
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    out = open(a.out, "w")
    dev_card = card()

    def emit(**kw):
        kw["card"] = dev_card
        line = json.dumps(kw)
        print(line, flush=True)
        out.write(line + "\n")

    lib = _lib.lib()
    torch.manual_seed(0)
    ws = torch.zeros(lib.evo_gemm_smallm_workspace(64, 22016, 4096, _lib.EPI_GELU_GATE), dtype=torch.uint8, device=DEV)
    for name, N, K, epi in SHAPES:
        for M in (1, 16, 64):
            gs = gemm_graphs(name, N, K, epi, M, ws)
            t = {"bf16": [], "fp8": []}
            for _ in range(a.rounds):                                  # alternate the two forms
                for mode in ("bf16", "fp8"):
                    g, n = gs[mode]
                    t[mode].append(time_graph(g, 3) * 1e3 / n)
            rec = {"kind": "gemm", "name": name, "N": N, "K": K, "M": M}
            for mode, bpw in (("bf16", 2), ("fp8", 1)):
                us = statistics.median(t[mode])
                rec[mode] = {"us": round(us, 2), "GBps": round(bpw * N * K / us / 1e3, 1), "hbm_share": round(bpw * N * K / us / 1e-6 / HBM, 3),
                             "spread_us": [round(min(t[mode]), 2), round(max(t[mode]), 2)]}
            rec["fp8_over_bf16"] = round(rec["fp8"]["us"] / rec["bf16"]["us"], 3)
            emit(**rec)
            del gs
            torch.cuda.empty_cache()
    if a.no_step:
        return
    from evo_b200.models import load_checkpoint
    model = load_checkpoint("evo-1.5-8k-base", random_init=True, device=DEV, weights="fp8")
    B, P = 16, 4096
    d, first, st = step_states(model, B, P, a.steps)
    t = {"bf16": [], "fp8": []}
    for _ in range(a.rounds):
        for mode in ("bf16", "fp8"):
            model._fp8_decode_bf16 = mode == "bf16"
            model._loop = st[mode]
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.inference_mode():
                e0.record()
                model.decode_loop(first, d, a.steps, P, top_k=1)
                e1.record()
            torch.cuda.synchronize()
            assert model._loop is st[mode], "the step was recaptured inside the timed window"
            t[mode].append(e0.elapsed_time(e1) / a.steps)
    rec = {"kind": "step", "model": "evo-1.5-8k-base random init", "B": B, "prompt": P, "steps": a.steps}
    for mode in ("bf16", "fp8"):
        rec[mode] = {"ms_per_step": round(statistics.median(t[mode]), 3), "spread": [round(min(t[mode]), 3), round(max(t[mode]), 3)]}
    rec["fp8_over_bf16"] = round(rec["fp8"]["ms_per_step"] / rec["bf16"]["ms_per_step"], 3)
    emit(**rec)


if __name__ == "__main__":
    main()
