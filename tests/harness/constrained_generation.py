"""Cost of constrained generation (development tool, needs a GPU; writes JSON under out/).

    python tests/harness/constrained_generation.py                           # B = 16 and 64, 1024-token prompts, 1000 new tokens
    python tests/harness/constrained_generation.py --batches 4 --tokens 64 --rounds 1

The 7B configuration with random weights generates from seeded random ACGT prompts with the reference CLI's sampling settings
(top-k 4, top-p 1, temperature 1), three arms per batch size, alternating order between rounds after a warm-up of each:
  unconstrained  generate(ragged=True)
  masked         the same with Constraints(forbid=(GGTCTC, CGTCTC), max_homopolymer=10): every step masked, no stops
  stop           masked plus stop=(TAA, TAG, TGA), stop_in_frame=True: rows end at their first in-frame stop codon and the loop
                 ends once every row of the batch has stopped
Per arm: milliseconds per decode step (decode-loop wall time over the steps it ran), the steps run against the steps asked
for, and the whole call's seconds.  Random weights say nothing about how soon a trained model emits a stop codon, so the
steps saved here only show the early exit working.  The card's name, power limit and the SM clock sampled while timing are
recorded beside the numbers."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.harness.gemm_shapes import Clock, card  # noqa: E402


def arm_constraints(arm):
    from evo_b200 import Constraints
    if arm == "unconstrained":
        return None
    if arm == "masked":
        return Constraints(forbid=("GGTCTC", "CGTCTC"), max_homopolymer=10)
    return Constraints(forbid=("GGTCTC", "CGTCTC"), max_homopolymer=10, stop=("TAA", "TAG", "TGA"), stop_in_frame=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="16,64")
    ap.add_argument("--prompt-len", type=int, default=1024)
    ap.add_argument("--tokens", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--arms", default="unconstrained,masked,stop")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=os.path.join(ROOT, "out", "constrained_generation"))
    a = ap.parse_args()
    import random
    import torch
    from evo_b200 import CharLevelTokenizer, generate
    from evo_b200.models import load_checkpoint
    if not torch.cuda.is_available():
        raise SystemExit("constrained_generation.py measures on a GPU; none is visible")
    model = load_checkpoint("evo-1-8k-base", device="cuda:0", random_init=True)
    model.eval()
    tok = CharLevelTokenizer(512)
    loops = []                                          # (seconds, steps run, steps asked) of every decode loop
    inner = model.decode_loop

    def timed(token, state, n_steps, starts, **kw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = inner(token, state, n_steps, starts, **kw)
        torch.cuda.synchronize()
        ran = int(state["mha"].seqlen_offset) - int(starts.max()) + 1
        loops.append((time.perf_counter() - t0, ran, n_steps))
        return out
    model.decode_loop = timed

    def run(arm, prompts, n_tokens):
        loops.clear()
        torch.manual_seed(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        texts, _ = generate(prompts, model, tok, n_tokens=n_tokens, top_k=4, top_p=1.0, temperature=1.0, cached_generation=True, verbose=0,
                            device="cuda:0", ragged=True, batch_size=len(prompts), constraints=arm_constraints(arm))
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        dt, ran, asked = (sum(x[i] for x in loops) for i in range(3))
        return {"seconds": round(wall, 3), "ms_per_step": round(dt / max(ran, 1) * 1e3, 3), "steps_run": ran, "steps_asked": asked,
                "mean_output_len": round(statistics.mean(len(t) for t in texts), 1)}

    rng = random.Random(a.seed)
    arms = a.arms.split(",")
    batches = [int(b) for b in a.batches.split(",")]
    rec = {"card": card(), "config": "evo-1-8k-base (7B), random weights", "prompt_len": a.prompt_len, "new_tokens": a.tokens,
           "sampling": {"top_k": 4, "top_p": 1.0, "temperature": 1.0}, "rounds": []}
    os.makedirs(a.out, exist_ok=True)
    path = os.path.join(a.out, time.strftime("%Y%m%d-%H%M%S") + ".json")
    prompts = {b: ["".join(rng.choice("ACGT") for _ in range(a.prompt_len)) for _ in range(b)] for b in batches}
    for b in batches:                                   # warm-up: module loads, graph captures, allocator growth
        for arm in arms:
            run(arm, prompts[b], 20)
    with Clock() as clk:
        for r in range(a.rounds):
            res = {}
            rec["rounds"].append(res)
            for b in batches:
                for arm in (arms if r % 2 == 0 else arms[::-1]):
                    res[f"B{b}_{arm}"] = run(arm, prompts[b], a.tokens)
                    rec["sm_mhz"] = clk.median()
                    print(r, b, arm, json.dumps(res[f"B{b}_{arm}"]), flush=True)
                    with open(path, "w") as f:
                        json.dump(rec, f, indent=1)
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
