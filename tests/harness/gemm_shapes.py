"""Per-shape timing of the prefill GEMMs (development tool, needs a GPU; writes JSON under out/).

    python tests/harness/gemm_shapes.py                                        # the library of this tree
    python tests/harness/gemm_shapes.py --lib out/base/evo_b200/libevo_b200.so # another build
    python tests/harness/gemm_shapes.py --lib A.so --lib B.so --rounds 2       # A/B: alternating subprocesses, then bitwise comparison

Records, for the six launches of one 8k scoring forward (M = 65 544 rows) with their real epilogues:
median kernel time over CUDA events (one event pair per launch) and TFLOP/s; cuBLASLt on the same shape with the NONE/BIAS
epilogue, timed in the same process; a K sweep of the 12288-wide projection at BIAS and BIAS_RESID fitted to
    time = tiles_per_CTA * (c0 + c1 * K/64)
(c1: mainloop cost of one 128 x 256 x 64 k-block, 1024 MMA clocks at the dense bf16 rate; c0: the per-tile fixed cost, epilogue
plus pipeline refill), with the card name, its power limit and the SM clock sampled while timing.  Given two libraries it also
compares every launch's output bit for bit.  Tile-walk experiments: set EVO_B200_GEMM_GROUP / EVO_B200_GEMM_RASTER_N in the
environment (the library reads them per launch)."""
import argparse
import ctypes as C
import json
import math
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

M = 65544
# name, N, K, epilogue (EPI_NONE 0, BIAS 1, BIAS_RESID 2, RESID 3, GELU_GATE 4, BIAS_ROPE 6)
SHAPES = [("proj", 12288, 4096, 1), ("wqkv_rope", 12288, 4096, 6), ("out", 4096, 4096, 2), ("gate", 22016, 4096, 4),
          ("l3", 4096, 11008, 3), ("unembed", 512, 4096, 0)]
SWEEP_K = (1024, 2048, 4096, 8192)
ROPE_L = 8193


class Clock:
    """nvidia-smi read-only queries (SM clock) every 100 ms while the block runs."""

    def __init__(self):
        self.mhz, self.proc = [], None

    def __enter__(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0], "--query-gpu=clocks.sm",
                                          "--format=csv,noheader,nounits", "-lms", "100"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=lambda: [self.mhz.append(float(x)) for x in self.proc.stdout if x.strip().replace(".", "").isdigit()], daemon=True).start()
        except OSError:
            self.proc = None
        return self

    def __exit__(self, *a):
        if self.proc:
            self.proc.terminate()
            self.proc.wait()

    def median(self):
        return statistics.median(self.mhz) if self.mhz else None


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power, smax = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_max": smax}
    except Exception as e:  # noqa: BLE001  (a missing nvidia-smi leaves the card unnamed, the timings stand)
        return {"name": None, "error": str(e)[:200]}


def load(path):
    h = C.CDLL(os.path.abspath(path))
    from evo_b200 import _lib
    h.evo_gemm.restype, h.evo_gemm.argtypes = C.c_int, [C.POINTER(_lib.GemmParams), C.c_void_p]
    h.evo_last_error.restype = C.c_char_p
    return h


class Problem:
    """Seeded operands of one launch; run(lib) writes C and returns it."""

    def __init__(self, N, K, epi, dev="cuda:0"):
        import torch
        from evo_b200 import _lib
        g = torch.Generator(device=dev).manual_seed(N * 7 + K + epi)
        self.N, self.K, self.epi = N, K, epi
        self.n_out = N // 2 if epi == _lib.EPI_GELU_GATE else N
        self.a = (torch.randn(M, K, device=dev, generator=g) * 0.5).bfloat16()
        self.w = (torch.randn(N, K, device=dev, generator=g) / math.sqrt(K)).bfloat16()
        self.bias = (torch.randn(N, device=dev, generator=g) * 0.2).bfloat16()
        self.resid = torch.randn(M, self.n_out, device=dev, generator=g).bfloat16() if epi in (_lib.EPI_BIAS_RESID, _lib.EPI_RESID) else None
        self.cos = torch.rand(ROPE_L, 64, device=dev, generator=g).bfloat16()
        self.sin = torch.rand(ROPE_L, 64, device=dev, generator=g).bfloat16()
        self.c = torch.empty(M, self.n_out, dtype=torch.bfloat16, device=dev)
        rope = dict(rope_cos=self.cos.data_ptr(), rope_sin=self.sin.data_ptr(), rope_L=ROPE_L, rope_cols=2 * N // 3) if epi == _lib.EPI_BIAS_ROPE else {}
        self.p = _lib.GemmParams(A=self.a.data_ptr(), lda=K, W=self.w.data_ptr(), C=self.c.data_ptr(), ldc=self.n_out,
                                 bias=self.bias.data_ptr() if epi in (1, 2, 6) else None,
                                 residual=self.resid.data_ptr() if self.resid is not None else None, ldr=self.n_out,
                                 M=M, N=N, K=K, epilogue=epi, variant=0, **rope)

    def run(self, lib):
        import torch
        rc = lib.evo_gemm(C.byref(self.p), C.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc:
            raise RuntimeError(f"evo_gemm: {lib.evo_last_error().decode()}")
        return self.c

    def cublaslt(self, ws):
        import torch
        from tests import support as TS
        from evo_b200 import _lib
        p = _lib.GemmParams(A=self.p.A, lda=self.K, W=self.p.W, C=self.c.data_ptr(), ldc=self.N, bias=self.p.bias, residual=None,
                            ldr=self.N, M=M, N=self.N, K=self.K, epilogue=1 if self.p.bias else 0, variant=0)
        if self.n_out != self.N:     # the gate shape writes the full-width pre-activation
            self._wide = torch.empty(M, self.N, dtype=torch.bfloat16, device=self.c.device)
            p.C = self._wide.data_ptr()
        return lambda: TS.check(TS.lib().evot_gemm_cublaslt(C.byref(p), C.c_void_p(ws.data_ptr()), ws.numel(), C.c_void_p(torch.cuda.current_stream().cuda_stream)))


def median_ms(fn, iters, warm=3):
    import torch
    for _ in range(warm):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for e0, e1 in ev:
        e0.record(); fn(); e1.record()
    torch.cuda.synchronize()
    return statistics.median(e0.elapsed_time(e1) for e0, e1 in ev)


def fit(points, tiles_per_cta, mhz):
    """least squares t = b + s * K/64 over the sweep; c0 = b / tiles, c1 = s / tiles, also in SM clocks"""
    xs, ys = [k / 64 for k, _ in points], [t for _, t in points]
    xm, ym = sum(xs) / len(xs), sum(ys) / len(ys)
    s = sum((x - xm) * (y - ym) for x, y in zip(xs, ys)) / sum((x - xm) ** 2 for x in xs)
    b = ym - s * xm
    c0_us, c1_us = b / tiles_per_cta * 1e3, s / tiles_per_cta * 1e3
    r = {"c0_us": round(c0_us, 4), "c1_us": round(c1_us, 5), "tiles_per_cta": tiles_per_cta}
    if mhz:
        r.update(c0_clk=round(c0_us * mhz), c1_clk=round(c1_us * mhz, 1), c1_vs_1024_mma_clk=round(c1_us * mhz / 1024, 3))
    return r


def child(lib_path, iters, out_path):
    import torch
    from evo_b200 import _lib
    if lib_path:
        _lib.LIB_PATH = os.path.abspath(lib_path)
    lib = _lib.lib()
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    ws = torch.empty(64 << 20, dtype=torch.uint8, device="cuda:0")
    rec = {"lib": _lib.LIB_PATH, "card": card(), "env": {k: v for k, v in os.environ.items() if k.startswith("EVO_B200_GEMM")}, "shapes": {}, "k_sweep": {}}
    with Clock() as clk:
        for name, N, K, epi in SHAPES:
            pr = Problem(N, K, epi)
            flop = 2.0 * M * N * K
            ms = median_ms(lambda: pr.run(lib), iters)
            ms_lt = median_ms(pr.cublaslt(ws), iters)
            rec["shapes"][name] = {"N": N, "K": K, "epi": epi, "ms": round(ms, 4), "tflops": round(flop / ms / 1e9, 1),
                                   "cublaslt_ms": round(ms_lt, 4), "cublaslt_tflops": round(flop / ms_lt / 1e9, 1)}
            print(name, rec["shapes"][name], flush=True)
            del pr
        for epi in (1, 2):
            pts = []
            for K in SWEEP_K:
                pr = Problem(12288, K, epi)
                pts.append((K, median_ms(lambda: pr.run(lib), iters)))
                del pr
            tiles = math.ceil(math.ceil(M / 128) * (12288 // 256) / n_sm)
            rec["k_sweep"][f"12288/epi{epi}"] = {"ms": {k: round(t, 4) for k, t in pts}}
            rec["k_sweep"][f"12288/epi{epi}"]["fit"] = fit(pts, tiles, None)
    rec["sm_mhz"] = clk.median()
    for v in rec["k_sweep"].values():
        v["fit"] = fit([(int(k), t) for k, t in v["ms"].items()], v["fit"]["tiles_per_cta"], rec["sm_mhz"])
    print(json.dumps(rec["k_sweep"]), "sm_mhz", rec["sm_mhz"], flush=True)
    with open(out_path, "w") as f:
        json.dump(rec, f, indent=1)


def compare(paths):
    import torch
    libs = [load(p) for p in paths]
    res = {}
    for name, N, K, epi in SHAPES + [(f"sweep_k{K}_epi{e}", 12288, K, e) for K in SWEEP_K for e in (1, 2)]:
        pr = Problem(N, K, epi)
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
    ap.add_argument("--out", default=os.path.join(ROOT, "out", "gemm_shapes"))
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
            rc = subprocess.run(cmd).returncode
            runs.append({"lib": lp, "round": r, "rc": rc, "json": path})
    summary = {"runs": runs}
    if len(libs) > 1:
        summary["bit_identical"] = compare(libs)
    with open(os.path.join(a.out, f"{stamp}_summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
