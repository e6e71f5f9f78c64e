"""Sequence embeddings against packed scoring, and the pooling kernel against its bandwidth bound (development tool, needs a GPU;
writes JSON under out/).

    python tests/harness/embedding_throughput.py                  # 512 sequences, 2 rounds
    python tests/harness/embedding_throughput.py --seqs 64 --rounds 1

The 7B configuration with random weights and the 512-sequence scoring set of tests/harness/packed_forward.py (lengths
log-uniform in [200, 8192], the same seed), arms alternating over --rounds, all with the same --max-tokens:
  score          frontend.score_many(packed=True): every block, the final norm and the fused scoring head
  final          embed_sequences(layers=["final"]): every block and the final norm, no unembedding
  layer16        embed_sequences(layers=[16]): blocks 0-16 only
  four_layers    embed_sequences(layers=[8, 16, 24, "final"])
Per arm: nucleotides/s over the whole call.  Then evo_pool_varlen alone (mean, skip 1) at T = 131072, D = 4096, as one
sequence and as 512 sequences of 256 rows: median time over --pool-iters launches (CUDA events) against the time the HBM
traffic (one read of the rows, the partials written and read once, the output) takes at the data sheet's 3.35 TB/s.
The card's name, power limit and the SM clock sampled while timing are recorded beside the numbers."""
import argparse
import ctypes as C
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.harness.gemm_shapes import Clock, card, median_ms  # noqa: E402
from tests.harness.packed_forward import timed  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def pool_kernel(T, D, lengths, iters):
    import torch
    from evo_b200 import _lib
    lib = _lib.lib()
    x = torch.randn(T, D, device="cuda:0").bfloat16()
    cu = torch.tensor([0] + list(lengths), dtype=torch.int64).cumsum(0).to("cuda:0")
    out = torch.empty(len(lengths), D, dtype=torch.float32, device="cuda:0")
    pp = _lib.PoolVarlenParams(x=x.data_ptr(), ldx=D, cu_seqlens=cu.data_ptr(), n_seq=len(lengths), T=T, max_seqlen=max(lengths), D=D,
                               skip_first=1, mode=_lib.POOL_MEAN, out=out.data_ptr(), ldo=D)
    need = lib.evo_pool_varlen_workspace(C.byref(pp))
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device="cuda:0")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ms = median_ms(lambda: _lib.check(lib.evo_pool_varlen(C.byref(pp), _lib.ptr(ws), need, st), "evo_pool_varlen"), iters)
    chunks = sum(math.ceil((n - 1) / 512) for n in lengths if n - 1 > 512)
    traffic = T * D * 2 + 2 * chunks * D * 4 + len(lengths) * D * 4
    bound_ms = traffic / HBM_BYTES_PER_S * 1e3
    return {"T": T, "D": D, "sequences": len(lengths), "workspace_bytes": need, "median_ms": round(ms, 4), "bytes": traffic,
            "bound_ms": round(bound_ms, 4), "share_of_bound": round(bound_ms / ms, 3), "GB_per_s": round(traffic / ms / 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seqs", type=int, default=512)
    ap.add_argument("--min-len", type=int, default=200)
    ap.add_argument("--max-len", type=int, default=8192)
    ap.add_argument("--max-tokens", type=int, default=1 << 17)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--pool-iters", type=int, default=50)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=os.path.join(ROOT, "out", "embedding_throughput"))
    a = ap.parse_args()
    import random
    import torch
    from evo_b200 import CharLevelTokenizer, embed_sequences
    from evo_b200.frontend import packs, score_many
    from evo_b200.models import load_checkpoint
    if not torch.cuda.is_available():
        raise SystemExit("embedding_throughput.py measures on a GPU; none is visible")
    rng = random.Random(a.seed)                                   # packed_forward.py's scoring set: same draws, same order
    s_len = [int(math.exp(rng.uniform(math.log(a.min_len), math.log(a.max_len)))) for _ in range(a.seqs)]
    seqs = ["".join(rng.choice("ACGT") for _ in range(n)) for n in s_len]
    model = load_checkpoint("evo-1-8k-base", device="cuda:0", random_init=True)
    model.eval()
    tok = CharLevelTokenizer(512)
    nt = sum(s_len)
    rec = {"card": card(), "config": "evo-1-8k-base (7B), random weights", "max_tokens": a.max_tokens, "sequences": a.seqs,
           "nucleotides": nt, "lengths": f"log-uniform [{a.min_len}, {a.max_len}]", "forwards": len(packs(s_len, a.max_tokens)),
           "rounds": []}
    os.makedirs(a.out, exist_ok=True)
    path = os.path.join(a.out, time.strftime("%Y%m%d-%H%M%S") + ".json")

    def save():
        with open(path, "w") as f:
            json.dump(rec, f, indent=1)

    arms = {"score": lambda s: score_many(s, model, tok, max_tokens=a.max_tokens, device="cuda:0", packed=True),
            "final": lambda s: embed_sequences(s, model, tok, layers=["final"], max_tokens=a.max_tokens),
            "layer16": lambda s: embed_sequences(s, model, tok, layers=[16], max_tokens=a.max_tokens),
            "four_layers": lambda s: embed_sequences(s, model, tok, layers=[8, 16, 24, "final"], max_tokens=a.max_tokens)}
    for fn in arms.values():                                      # warm-up: module loads, allocator growth
        fn(seqs[:8])
    names = list(arms)
    with Clock() as clk:
        for r in range(a.rounds):
            res = {}
            rec["rounds"].append(res)
            for name in (names if r % 2 == 0 else names[::-1]):
                _, dt = timed(lambda: arms[name](seqs))
                res[name] = {"seconds": round(dt, 3), "nt_per_s": round(nt / dt, 1)}
                rec["sm_mhz"] = clk.median()
                print(r, name, json.dumps(res[name]), flush=True)
                save()
        del model
        torch.cuda.empty_cache()
        T = 1 << 17
        rec["pool_kernel"] = [pool_kernel(T, 4096, [T], a.pool_iters), pool_kernel(T, 4096, [256] * (T // 256), a.pool_iters)]
        rec["sm_mhz_incl_pool"] = clk.median()
    for p in rec["pool_kernel"]:
        print("pool", json.dumps(p), flush=True)
    save()
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
