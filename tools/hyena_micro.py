"""Hyena scan micro-benchmark: times evo_hyena_fwd (CUDA events, L2 flushed by the 2+ GB working set) for the bench
shapes, its state-only carry pass, and a segment-count sweep at the sequence-parallel shard shape.
    python tools/hyena_micro.py [--out out/hyena_micro.jsonl]"""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from evo_b200 import _lib  # noqa: E402
from evo_b200._lib import HyenaParams, check, ptr  # noqa: E402


def run(z, f, B, L, D, H, state_only=0, force_segments=0, iters=10):
    lib = _lib.lib()
    dev = z.device
    y = torch.empty(B, L, D, dtype=torch.bfloat16, device=dev)
    st_out = torch.empty(B, D, 8, 2, dtype=torch.float32, device=dev)
    hp = HyenaParams(z=z.data_ptr(), y=y.data_ptr(), fir_w=f["w"].data_ptr(), fir_b=f["b"].data_ptr(), Dskip=f["D"].data_ptr(), poles=f["p"].data_ptr(),
                     residues=f["r"].data_ptr(), B=B, L=L, D=D, S=8, nheads=H, state_out=st_out.data_ptr(), force_segments=force_segments, state_only=state_only)
    n = lib.evo_hyena_fwd_workspace(C.byref(hp))
    ws = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    go = lambda: check(lib.evo_hyena_fwd(C.byref(hp), ptr(ws), n, s), "hyena")
    for _ in range(3):
        go()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        go()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="out/hyena_micro.jsonl")
    a = ap.parse_args()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    dev = "cuda:0"
    D, H = 4096, 32
    torch.manual_seed(0)
    mag = 0.5 + 0.499 * torch.rand(D, 8, 1)
    ang = (torch.rand(D, 8, 1) * 2 - 1) * 3.14159
    f = {"w": (torch.randn(3 * D, 3) * 0.3).bfloat16().to(dev), "b": (torch.randn(3 * D) * 0.1).bfloat16().to(dev), "D": torch.randn(D).bfloat16().to(dev),
         "p": torch.stack([mag * torch.cos(ang), mag * torch.sin(ang)], -1).squeeze(2).contiguous().to(dev), "r": (torch.randn(D, 8, 2) * 0.3).to(dev)}
    with open(a.out, "a") as out:
        for B, L in [(8, 8193), (1, 16384), (1, 131072), (16, 4096), (2, 32769)]:
            z = (torch.randn(B, L, 3 * D, device=dev) * 0.7).bfloat16()
            rec = {"what": "hyena_micro", "B": B, "L": L, "D": D, "algorithmic_GB": 8.0 * B * L * D / 1e9}
            rec["ms"] = run(z, f, B, L, D, H)
            rec["GBps"] = 8.0 * B * L * D / rec["ms"] / 1e6
            rec["state_only_ms"] = run(z, f, B, L, D, H, state_only=1)
            if B == 1 and L == 16384:     # segment-count sweep for the sequence-parallel shard shape
                for ns in (4, 8, 9, 10, 16, 18):
                    rec[f"nseg{ns}_ms"] = run(z, f, B, L, D, H, force_segments=ns)
            print(json.dumps(rec)); out.write(json.dumps(rec) + "\n"); out.flush()
            del z


if __name__ == "__main__":
    main()
