"""Per-tile cost of every prefill GEMM epilogue (development tool, needs a GPU; writes JSON under out/).

    python tests/harness/gemm_epilogue_fit.py                                   # the library of this tree
    python tests/harness/gemm_epilogue_fit.py --lib A.so --lib B.so --rounds 2  # A/B: alternating subprocesses, then bitwise comparison

For each epilogue the forward uses, a K sweep at its layer's N (BIAS, BIAS_RESID and BIAS_ROPE at 12288, GELU_GATE at 22016,
RESID at l3's 4096 over K = 2752...11008; M = 65 544 rows) is fitted to
    time = tiles_per_CTA * (c0 + c1 * K/64)
as in gemm_shapes.py, whose operands, timing and fit it reuses; also the median time and TFLOP/s of the six launches of one 8k
scoring forward, with the card name, its power limit and the SM clock sampled while timing.  Given two libraries it compares
every launch's output bit for bit.

Store-path experiments: EVO_B200_GEMM_DIRECT_STORE=1 in the environment keeps the per-thread stores on the 256-column tile (the
library reads it per launch); a library built with NVCC_EXTRA=-DEVO_GEMM_NO_STORE runs the staged epilogue's arithmetic without
residual loads or C stores -- its outputs are garbage, its times bound what any store path can win."""
import argparse
import json
import math
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import gemm_shapes as GS  # noqa: E402  (operands, timing, fit, card and clock of the per-shape harness)

# (N, epilogue, K points): EPI_BIAS 1, BIAS_RESID 2, RESID 3, GELU_GATE 4, BIAS_ROPE 6
SWEEPS = [(12288, 1, GS.SWEEP_K), (12288, 2, GS.SWEEP_K), (12288, 6, GS.SWEEP_K), (22016, 4, GS.SWEEP_K),
          (4096, 3, (2752, 5504, 8256, 11008))]


def child(lib_path, iters, out_path):
    import torch
    from evo_b200 import _lib
    if lib_path:
        _lib.LIB_PATH = os.path.abspath(lib_path)
    lib = _lib.lib()
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    rec = {"lib": _lib.LIB_PATH, "card": GS.card(), "env": {k: v for k, v in os.environ.items() if k.startswith("EVO_B200_GEMM")},
           "shapes": {}, "k_sweep": {}}
    with GS.Clock() as clk:
        for name, N, K, epi in GS.SHAPES:
            pr = GS.Problem(N, K, epi)
            ms = GS.median_ms(lambda: pr.run(lib), iters)
            rec["shapes"][name] = {"N": N, "K": K, "epi": epi, "ms": round(ms, 4), "tflops": round(2.0 * GS.M * N * K / ms / 1e9, 1)}
            print(name, rec["shapes"][name], flush=True)
            del pr
        for N, epi, ks in SWEEPS:
            pts = []
            for K in ks:
                pr = GS.Problem(N, K, epi)
                pts.append((K, GS.median_ms(lambda: pr.run(lib), iters)))
                del pr
            rec["k_sweep"][f"{N}/epi{epi}"] = {"ms": {k: round(t, 4) for k, t in pts},
                                               "tiles_per_cta": math.ceil(math.ceil(GS.M / 128) * (N // 256) / n_sm)}
    rec["sm_mhz"] = clk.median()
    for v in rec["k_sweep"].values():
        v["fit"] = GS.fit([(int(k), t) for k, t in v["ms"].items()], v["tiles_per_cta"], rec["sm_mhz"])
    print(json.dumps({k: v["fit"] for k, v in rec["k_sweep"].items()}), "sm_mhz", rec["sm_mhz"], flush=True)
    with open(out_path, "w") as f:
        json.dump(rec, f, indent=1)


def compare(paths):
    import torch
    libs = [GS.load(p) for p in paths]
    res = {}
    for name, N, K, epi in GS.SHAPES + [(f"sweep_{N}_k{K}_epi{e}", N, K, e) for N, e, ks in SWEEPS for K in ks]:
        pr = GS.Problem(N, K, epi)
        first = pr.run(libs[0]).clone()
        same = True
        for h in libs[1:]:
            pr.c.fill_(float("nan"))
            same = same and torch.equal(first, pr.run(h))
        res[name] = same
        del pr, first
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="libevo_b200.so to time (default: this tree's); twice for an A/B")
    ap.add_argument("--rounds", type=int, default=1, help="A/B only: how many times each library is timed, alternating")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(GS.ROOT, "out", "gemm_epilogue_fit"))
    ap.add_argument("--child", help=argparse.SUPPRESS)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    if a.child is not None:
        child(a.lib[0] if a.lib else None, a.iters, a.child)
        return
    libs = a.lib or [None]
    stamp = time.strftime("%Y%m%d-%H%M%S")
    runs = []
    for r in range(a.rounds if len(libs) > 1 else 1):
        for i, lp in enumerate(libs):
            path = os.path.join(a.out, f"{stamp}_lib{i}_round{r}.json")
            cmd = [sys.executable, os.path.abspath(__file__), "--child", path, "--iters", str(a.iters)] + (["--lib", lp] if lp else [])
            runs.append({"lib": lp, "round": r, "rc": subprocess.run(cmd).returncode, "json": path})
    summary = {"runs": runs}
    if len(libs) > 1:
        summary["bit_identical"] = compare(libs)
    with open(os.path.join(a.out, f"{stamp}_summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
