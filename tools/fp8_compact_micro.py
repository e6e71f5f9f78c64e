"""Compact FP8 weights against the non-compact FP8 model, timed alternately in one run (GPU only; 7B, random weights).

  * memory: torch.cuda.memory_allocated() after loading the bf16, FP8 (with its one-byte decode copies built) and compact FP8
    models, each alone, against the linear-weight bytes computed from the shapes;
  * evo_fp8_dequant_rows alone at the four 7B shapes: CUDA graphs of back-to-back launches rotating over enough copies that L2
    never holds them, median us per launch and TB/s of N*K*3 + N bytes;
  * prefill: the 8k scoring forward at bench.py's geometry (score_tokens, 8 x 8193) and a 1 x 1025 stateful prefill, FP8 against
    compact (the compact model rebuilds every linear weight once per forward);
  * decode step: decode_loop at bench.py --workload gen's geometry (B = 16, 4096-token prompt: the same kernels on both) and at
    B = 128 (a 512-token prompt; above 64 rows the compact model rebuilds every linear weight on every step).
The FP8 and compact models hold the same weights (one seed), and every timed pair is checked to give the same bits.  The card's
name and power limit are read in the same run.  One JSON line per measurement.
    python tools/fp8_compact_micro.py [--out out/fp8_compact_micro.jsonl] [--rounds 5] [--steps 32]
"""
import argparse
import ctypes as C
import gc
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from evo_b200 import _lib  # noqa: E402

DEV = "cuda:0"
MODEL = "evo-1-8k-base"
SHAPES = [("qkv", 12288, 4096, False), ("out", 4096, 4096, False), ("w12", 22016, 4096, True), ("w3", 4096, 11008, False)]


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip() or torch.cuda.get_device_name(0)


def timed(fn):
    """ms of fn() between CUDA events, synchronised."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def load(weights):
    from evo_b200.models import load_checkpoint
    gc.collect()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    m = load_checkpoint(MODEL, random_init=True, device=DEV, weights=weights, seed=0)
    if weights == "fp8":
        m._ensure_fp8()                               # the one-byte decode copies an FP8 model holds once it generates
    torch.cuda.synchronize()
    return m, torch.cuda.memory_allocated() - base


def linear_bytes(m):
    shapes = [tuple(getattr(mod, attr).shape) for _, _, mod, attr, _ in m._fp8_slots()]
    return {"bf16_GB": sum(2 * n * k for n, k in shapes) / 1e9, "q_plus_e_GB": sum(n * k + n for n, k in shapes) / 1e9,
            "scratch_GB": 2 * max(n * k for n, k in shapes) / 1e9}


def dequant_graph(N, K, gate):
    lib = _lib.lib()
    epi = _lib.EPI_GELU_GATE if gate else _lib.EPI_NONE
    copies = max(2, -(-400 * 2 ** 20 // (3 * N * K)))
    bufs = []
    for _ in range(copies):
        w = torch.randn(N, K, device=DEV).mul_(K ** -0.5).bfloat16()
        q = torch.empty(N * K, dtype=torch.uint8, device=DEV)
        e = torch.empty(N, dtype=torch.int8, device=DEV)
        st = torch.zeros(1, dtype=torch.int32, device=DEV)
        _lib.check(lib.evo_fp8_quantize_rows(w.data_ptr(), N, K, epi, q.data_ptr(), e.data_ptr(), st.data_ptr(), stream()), "quantize")
        bufs.append((q, e, w))
    reps = 8

    def fn():
        for _ in range(reps):
            for q, e, w in bufs:
                _lib.check(lib.evo_fp8_dequant_rows(q.data_ptr(), e.data_ptr(), N, K, epi, w.data_ptr(), stream()), "dequant")
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g, reps * copies, bufs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="out/fp8_compact_micro.jsonl")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_compact_micro.py measures on the GPU; no GPU here")
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    out = open(a.out, "w")
    dev_card = card()

    def emit(**kw):
        kw["card"] = dev_card
        line = json.dumps(kw)
        print(line, flush=True)
        out.write(line + "\n")

    def alternate(fns, rounds):
        """{name: (median, min, max)} of the ms of each fn, alternating; asserts that the fns of one round return the same bits."""
        t = {k: [] for k in fns}
        for _ in range(rounds):
            ref = None
            for k, fn in fns.items():
                ms, res = timed(fn)
                t[k].append(ms)
                res = [x.contiguous().view(torch.uint8) for x in res if x is not None]
                if ref is None:
                    ref = res
                assert all(torch.equal(x, y) for x, y in zip(ref, res)), f"{k}: different bits"
        return {k: {"ms": round(statistics.median(v), 3), "spread": [round(min(v), 3), round(max(v), 3)]} for k, v in t.items()}

    # ---- memory
    mem = {}
    m, mem["bf16"] = load("bf16")
    lin = linear_bytes(m)
    del m
    fp8, mem["fp8"] = load("fp8")
    compact, mem["fp8-compact"] = load("fp8-compact")
    emit(kind="memory", model=f"{MODEL} random init", allocated_GB={k: round(v / 1e9, 3) for k, v in mem.items()},
         linear_weights={k: round(v, 3) for k, v in lin.items()})

    # ---- the dequant kernel alone
    for name, N, K, gate in SHAPES:
        g, n, bufs = dequant_graph(N, K, gate)
        t = []
        for _ in range(a.rounds):
            g.replay()
            ms, _ = timed(lambda: [g.replay() for _ in range(3)])
            t.append(ms * 1e3 / (3 * n))
        us = statistics.median(t)
        emit(kind="dequant", name=name, N=N, K=K, us=round(us, 2), TBps=round((3 * N * K + N) / us / 1e6, 3),
             spread_us=[round(min(t), 2), round(max(t), 2)])
        del g, bufs
        torch.cuda.empty_cache()

    # ---- prefill
    ids = torch.randint(0, 4, (8, 8193), device=DEV) * 3 + 65
    with torch.inference_mode():
        for m in (fp8, compact):                                   # warm-up
            m.score_tokens(ids)
        r = alternate({"fp8": lambda: fp8.score_tokens(ids), "compact": lambda: compact.score_tokens(ids)}, max(3, a.rounds // 2))
    emit(kind="prefill", what="score_tokens 8 x 8193 (bench.py 8k)", **r, compact_over_fp8=round(r["compact"]["ms"] / r["fp8"]["ms"], 4))
    ids1 = torch.randint(0, 4, (1, 1025), device=DEV) * 3 + 65

    def prefill(m):
        d = m.initialize_inference_params()
        return (m(ids1, inference_params_dict=d)[0],)
    with torch.inference_mode():
        for m in (fp8, compact):
            prefill(m)
        r = alternate({"fp8": lambda: prefill(fp8), "compact": lambda: prefill(compact)}, 4 * a.rounds)
    emit(kind="prefill", what="stateful prefill 1 x 1025", **r, compact_over_fp8=round(r["compact"]["ms"] / r["fp8"]["ms"], 4))
    del ids
    torch.cuda.empty_cache()

    # ---- decode steps
    for B, P in ((16, 4096), (128, 512)):
        states = {}
        for k, m in (("fp8", fp8), ("compact", compact)):
            d = m.initialize_inference_params()
            d["mha"].max_batch_size, d["mha"].max_seqlen = B, P + a.steps + 64
            with torch.inference_mode():
                logits, d = m(torch.randint(0, 4, (B, P), device=DEV, generator=torch.Generator(DEV).manual_seed(B)) * 3 + 65,
                              inference_params_dict=d)
                first = logits[:, -1].float().argmax(-1)
                m._loop = None
                m.decode_loop(first, d, a.steps, P, top_k=1)          # captures the step
            states[k] = (m, d, first, m._loop)

        def step(k):
            m, d, first, loop = states[k]
            with torch.inference_mode():
                picked, kept = m.decode_loop(first, d, a.steps, P, top_k=1)
            assert m._loop is loop, "the step was recaptured inside the timed window"
            return picked, kept
        r = alternate({k: (lambda k=k: step(k)) for k in states}, a.rounds)
        for k in r:
            r[k]["ms_per_step"] = round(r[k].pop("ms") / a.steps, 4)
            r[k]["spread"] = [round(x / a.steps, 4) for x in r[k]["spread"]]
        emit(kind="step", B=B, prompt=P, steps=a.steps, **r, compact_over_fp8=round(r["compact"]["ms_per_step"] / r["fp8"]["ms_per_step"], 4))
        del states
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
