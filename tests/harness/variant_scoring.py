"""Variant scoring from reference checkpoints against scoring every full variant string (development tool, needs a GPU;
writes JSON under out/).

    python tests/harness/variant_scoring.py                          # 3 * 1024 + 3072 variants, 2 rounds
    python tests/harness/variant_scoring.py --first 768 --second 768 --rounds 2

The 7B configuration with random weights, a seeded 1024-nt and a seeded 4096-nt reference; the variants are single-nucleotide
substitutions: --first of the 3 * 1024 of the first reference (all by default; a seeded subset otherwise) and a seeded
--second of the 3 * 4096 of the second.  Two arms, alternating over --rounds after a warm-up on a few variants:
  full       frontend.score_many(full variant strings + references, packed=True)
  resumed    evo_b200.score_variants (one checkpointed forward per reference group, then the resumed passes)
Per arm: wall time (the resumed arm includes its reference pass), tokens run and variants/s; across arms the largest |score
difference|.  The card's name, power limit and the SM clock sampled while timing are recorded beside the numbers."""
import argparse
import json
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
    ap.add_argument("--first", type=int, default=3 * 1024, help="variants of the 1024-nt reference")
    ap.add_argument("--second", type=int, default=3072, help="variants of the 4096-nt reference")
    ap.add_argument("--stride", type=int, default=128)
    ap.add_argument("--max-tokens", type=int, default=1 << 17)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=os.path.join(ROOT, "out", "variant_scoring"))
    a = ap.parse_args()
    import random
    import torch
    from evo_b200 import CharLevelTokenizer, saturation_variants, score_variants
    from evo_b200.frontend import score_many
    from evo_b200.models import load_checkpoint
    if not torch.cuda.is_available():
        raise SystemExit("variant_scoring.py measures on a GPU; none is visible")
    rng = random.Random(a.seed)
    refs = ["".join(rng.choice("ACGT") for _ in range(n)) for n in (1024, 4096)]
    sat = [saturation_variants(r) for r in refs]
    picks = [sorted(rng.sample(range(len(s)), min(n, len(s)))) for s, n in zip(sat, (a.first, a.second))]
    variants = [(r, sat[r][i][1]) for r in (0, 1) for i in picks[r]]
    seqs = [s for _, s in variants]
    model = load_checkpoint("evo-1-8k-base", device="cuda:0", random_init=True)
    model.eval()
    tok = CharLevelTokenizer(512)
    full_tokens = sum(len(s) + 1 for s in seqs) + sum(len(r) + 1 for r in refs)
    rec = {"card": card(), "config": "evo-1-8k-base (7B), random weights", "max_tokens": a.max_tokens, "stride": a.stride,
           "variants": {"reference_1024": len(picks[0]), "reference_4096": len(picks[1])}, "rounds": []}
    os.makedirs(a.out, exist_ok=True)
    path = os.path.join(a.out, time.strftime("%Y%m%d-%H%M%S") + ".json")

    def save():
        with open(path, "w") as f:
            json.dump(rec, f, indent=1)

    def full_arm(vs):
        return score_many([s for _, s in vs] + refs, model, tok, max_tokens=a.max_tokens, device="cuda:0", packed=True), {"tokens": None}

    def resumed_arm(vs):
        stats = {}
        v, r = score_variants(refs, vs, model, tok, checkpoint_stride=a.stride, max_tokens=a.max_tokens, device="cuda:0", stats=stats)
        return v + r, stats

    warm = variants[:4] + variants[-4:]
    full_arm(warm)
    resumed_arm(warm)
    arms = ["full", "resumed"]
    with Clock() as clk:
        for r in range(a.rounds):
            res, out = {}, {}
            rec["rounds"].append(res)
            for name in (arms if r % 2 == 0 else arms[::-1]):
                (scores, stats), dt = timed(lambda: (full_arm if name == "full" else resumed_arm)(variants))
                out[name] = scores
                tokens = full_tokens if name == "full" else stats["reference_tokens"] + stats["variant_tokens"]
                res[name] = {"seconds": round(dt, 3), "tokens": tokens, "variants_per_s": round(len(variants) / dt, 1),
                             "tokens_per_s": round(tokens / dt, 1)}
                if name == "resumed":
                    res[name].update(reference_tokens=stats["reference_tokens"], variant_tokens=stats["variant_tokens"],
                                     passes=stats["passes"], checkpoint_stride=stats["checkpoint_stride"])
                rec["sm_mhz"] = clk.median()
                print(r, name, json.dumps(res[name]), flush=True)
                save()
            res["max_abs_score_diff"] = max(abs(x - y) for x, y in zip(out["full"], out["resumed"]))
            res["speedup"] = round(res["full"]["seconds"] / res["resumed"]["seconds"], 3)
            save()
    # where the resumed arm's time goes: its reference pass alone (both references, one checkpointed forward)
    from evo_b200.frontend import packed_ids
    ids = packed_ids(refs, tok, device="cuda:0")
    _, dt = timed(lambda: model.prefill_checkpoints(ids, [0, len(refs[0]) + 1, len(refs[0]) + len(refs[1]) + 2], a.stride))
    rec["reference_pass_seconds"] = round(dt, 3)
    save()
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
