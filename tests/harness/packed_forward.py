"""Packed variable-length forward against today's padded / grouped forwards (development tool, needs a GPU; writes JSON
under out/).

    python tests/harness/packed_forward.py                       # 512 scored sequences, 64 prompts, 3 rounds
    python tests/harness/packed_forward.py --score-seqs 64 --prompts 8 --tokens 16 --rounds 1

The 7B configuration with random weights, one seeded input set, arms alternating over --rounds:
  scoring   512 sequences with lengths log-uniform in [200, 8192] through frontend.score_many, bucketed (length-sorted
            batches of <= 32 with <= 10 % padding, scripts/score.py's defaults) and packed, both with the same --max-tokens.
            Per arm: nucleotides/s over the whole call and the number of forwards; across arms the largest |score difference|.
  prefill   the DESIGN.md section 6 workload, 64 prompts with lengths uniform in [256, 4096]: StripedHyena.prefill_ragged
            grouped (one forward per distinct length) and packed (one forward), then generate(ragged=True) end to end with each
            prefill and --tokens new tokens (top-k 4, top-p 1, temperature 1).  Across the prefill arms the largest |head logit|
            difference relative to the row's largest |logit|.
The card's name, power limit and the SM clock sampled while timing are recorded beside the numbers."""
import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.harness.gemm_shapes import Clock, card  # noqa: E402


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--score-seqs", type=int, default=512)
    ap.add_argument("--score-min", type=int, default=200)
    ap.add_argument("--score-max", type=int, default=8192)
    ap.add_argument("--max-tokens", type=int, default=1 << 17)
    ap.add_argument("--prompts", type=int, default=64)
    ap.add_argument("--min-len", type=int, default=256)
    ap.add_argument("--max-len", type=int, default=4096)
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=os.path.join(ROOT, "out", "packed_forward"))
    a = ap.parse_args()
    import random
    import torch
    from evo_b200 import CharLevelTokenizer, generate
    from evo_b200.frontend import length_buckets, packs, ragged_batches, score_many
    from evo_b200.models import load_checkpoint
    if not torch.cuda.is_available():
        raise SystemExit("packed_forward.py measures on a GPU; none is visible")
    rng = random.Random(a.seed)
    s_len = [int(math.exp(rng.uniform(math.log(a.score_min), math.log(a.score_max)))) for _ in range(a.score_seqs)]
    seqs = ["".join(rng.choice("ACGT") for _ in range(n)) for n in s_len]
    p_len = [rng.randint(a.min_len, a.max_len) for _ in range(a.prompts)]
    prompts = ["".join(rng.choice("ACGT") for _ in range(n)) for n in p_len]
    model = load_checkpoint("evo-1-8k-base", device="cuda:0", random_init=True)
    model.eval()
    tok = CharLevelTokenizer(512)
    rec = {"card": card(), "config": "evo-1-8k-base (7B), random weights", "max_tokens": a.max_tokens,
           "scoring": {"sequences": a.score_seqs, "nucleotides": sum(s_len), "lengths": f"log-uniform [{a.score_min}, {a.score_max}]",
                       "forwards": {"bucketed": len(length_buckets(seqs, batch_size=32, mode="sorted", max_tokens=a.max_tokens)),
                                    "packed": len(packs(s_len, a.max_tokens))}},
           "prefill": {"prompts": a.prompts, "tokens": sum(p_len), "distinct_lengths": len(set(p_len)),
                       "lengths": f"uniform [{a.min_len}, {a.max_len}]", "new_tokens": a.tokens},
           "rounds": []}
    os.makedirs(a.out, exist_ok=True)
    path = os.path.join(a.out, time.strftime("%Y%m%d-%H%M%S") + ".json")

    def save():
        with open(path, "w") as f:
            json.dump(rec, f, indent=1)

    ids = [tok.tokenize(p) for p in prompts]          # generate()'s prompt ids (prepend_bos=False)
    rows, cache_len = ragged_batches([len(t) for t in ids], a.tokens, batch_size=len(ids))[0]
    batch = [ids[r] for r in rows]
    gen_kw = dict(top_k=4, top_p=1.0, temperature=1.0, cached_generation=True, verbose=0, device="cuda:0", ragged=True, batch_size=64)

    def score_arm(packed, s):
        return score_many(s, model, tok, max_tokens=a.max_tokens, device="cuda:0", packed=packed)

    def prefill_arm(packed, b, cl):
        with torch.inference_mode():
            return model.prefill_ragged(b, cl, packed=packed)[0]

    def gen_arm(packed, p, n):
        torch.manual_seed(0)
        return generate(p, model, tok, n_tokens=n, packed_prefill=packed, **gen_kw)

    for packed in (False, True):                       # warm-up: module loads, graph captures, allocator growth
        score_arm(packed, seqs[:8])
        prefill_arm(packed, batch[:3], cache_len)
        gen_arm(packed, prompts[:3], 8)
    arms = [("score", False), ("score", True), ("prefill", False), ("prefill", True), ("generate", False), ("generate", True)]
    with Clock() as clk:
        for r in range(a.rounds):
            res, out = {}, {}
            rec["rounds"].append(res)
            for kind, packed in (arms if r % 2 == 0 else arms[::-1]):
                name = f"{kind}_{'packed' if packed else ('bucketed' if kind == 'score' else 'grouped')}"
                if kind == "score":
                    out[name], dt = timed(lambda: score_arm(packed, seqs))
                    res[name] = {"seconds": round(dt, 3), "nt_per_s": round(sum(s_len) / dt, 1)}
                elif kind == "prefill":
                    out[name], dt = timed(lambda: prefill_arm(packed, batch, cache_len))
                    res[name] = {"seconds": round(dt, 3), "tok_per_s": round(sum(p_len) / dt, 1)}
                else:
                    _, dt = timed(lambda: gen_arm(packed, prompts, a.tokens))
                    res[name] = {"seconds": round(dt, 3), "new_tok_per_s": round(a.prompts * a.tokens / dt, 1)}
                rec["sm_mhz"] = clk.median()
                print(r, name, json.dumps(res[name]), flush=True)
                save()
            res["max_abs_score_diff"] = max(abs(x - y) for x, y in zip(out["score_bucketed"], out["score_packed"]))
            hg, hp = out["prefill_grouped"].double(), out["prefill_packed"].double()
            res["max_head_logit_diff_rel"] = ((hg - hp).abs().max(-1).values / hg.abs().max(-1).values.clamp(min=1.0)).max().item()
            save()
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
