"""Generation throughput for prompts of different lengths (development tool, needs a GPU; writes JSON under out/).

    python tests/harness/ragged_generation.py                      # 64 prompts, lengths uniform in [256, 4096], 256 new tokens
    python tests/harness/ragged_generation.py --prompts 8 --tokens 32 --rounds 2

The 7B configuration with random weights generates from one seeded mix of prompts with the reference CLI's sampling settings
(top-k 4, top-p 1, temperature 1), three ways, in one process, after a warm-up of each:
  one_at_a_time  today's generate() on the mixed list: every prompt is its own batch of one
  exact_groups   prompts grouped by identical length (semantic_design's read_prompts policy), one generate() per group
  ragged         generate(ragged=True): length-sorted batches of up to --batch-size, one position per row while decoding
Every arm prefills each prompt whole (force_prompt_threshold above the longest prompt), so the arms differ only in batching.
Per arm: generated tokens/s over the whole call, prefill seconds, and milliseconds per decode step for each batch size the
arm ran (median over its decode loops).  With --rounds > 1 the arms alternate.  The card's name, power limit and the SM clock
sampled while timing are recorded beside the numbers."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.harness.gemm_shapes import Clock, card  # noqa: E402


class Timers:
    """Wall time (ended by a device synchronise) of every prefill and decode loop the model runs."""

    def __init__(self, model):
        import torch
        self.prefill_s, self.steps = 0.0, []          # steps: (batch, n_steps, seconds)

        def timed(fn, record):
            def wrapper(*a, **kw):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = fn(*a, **kw)
                torch.cuda.synchronize()
                record(a, time.perf_counter() - t0)
                return out
            return wrapper
        self.depth = 0                                # prefill_ragged calls forward once per length group: count the outer call only
        inner_forward, inner_ragged = model.forward, model.prefill_ragged

        def ragged(*a, **kw):
            self.depth += 1
            try:
                return inner_ragged(*a, **kw)
            finally:
                self.depth -= 1
        model.forward = timed(inner_forward, lambda a, dt: self._add_prefill(dt) if self.depth == 0 else None)
        model.prefill_ragged = timed(ragged, lambda a, dt: self._add_prefill(dt))
        model.decode_loop = timed(model.decode_loop, lambda a, dt: self.steps.append((int(a[0].reshape(-1).shape[0]), int(a[2]), dt)))

    def _add_prefill(self, dt):
        self.prefill_s += dt

    def reset(self):
        self.prefill_s, self.steps = 0.0, []

    def step_ms(self):
        by_b = {}
        for b, n, dt in self.steps:
            by_b.setdefault(b, []).append(dt / n * 1e3)
        return {str(b): {"ms_per_step": round(statistics.median(v), 3), "loops": len(v)} for b, v in sorted(by_b.items())}


def run_arm(arm, prompts, model, tok, n_tokens, batch_size, timers):
    import torch
    from evo_b200 import generate
    from evo_b200.frontend import length_buckets
    kw = dict(n_tokens=n_tokens, top_k=4, top_p=1.0, temperature=1.0, cached_generation=True, verbose=0, device="cuda:0",
              force_prompt_threshold=max(len(p) for p in prompts) + 1)
    timers.reset()
    torch.manual_seed(0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if arm == "one_at_a_time":
        texts, _ = generate(prompts, model, tok, batched=True, **kw)        # different lengths: one prompt per batch
    elif arm == "exact_groups":
        texts = []
        for idx in length_buckets(prompts, batch_size=batch_size, mode="exact"):
            texts += generate([prompts[i] for i in idx], model, tok, batched=True, **kw)[0]
    else:
        texts, _ = generate(prompts, model, tok, ragged=True, batch_size=batch_size, **kw)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    assert len(texts) == len(prompts) and all(len(t) == n_tokens for t in texts)
    return {"seconds": round(wall, 3), "tokens_per_s": round(len(prompts) * n_tokens / wall, 1), "prefill_s": round(timers.prefill_s, 3),
            "decode_s": round(sum(dt for _, _, dt in timers.steps), 3), "decode_steps": timers.step_ms()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--prompts", type=int, default=64)
    ap.add_argument("--min-len", type=int, default=256)
    ap.add_argument("--max-len", type=int, default=4096)
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--arms", default="one_at_a_time,exact_groups,ragged")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=os.path.join(ROOT, "out", "ragged_generation"))
    a = ap.parse_args()
    import random
    import torch
    from evo_b200 import CharLevelTokenizer
    from evo_b200.models import load_checkpoint
    if not torch.cuda.is_available():
        raise SystemExit("ragged_generation.py measures on a GPU; none is visible")
    rng = random.Random(a.seed)
    lengths = [rng.randint(a.min_len, a.max_len) for _ in range(a.prompts)]
    prompts = ["".join(rng.choice("ACGT") for _ in range(n)) for n in lengths]
    model = load_checkpoint("evo-1-8k-base", device="cuda:0", random_init=True)
    model.eval()
    tok = CharLevelTokenizer(512)
    timers = Timers(model)
    arms = a.arms.split(",")
    rec = {"card": card(), "config": "evo-1-8k-base (7B), random weights", "prompts": a.prompts, "lengths": lengths,
           "distinct_lengths": len(set(lengths)), "new_tokens": a.tokens, "batch_size": a.batch_size,
           "sampling": {"top_k": 4, "top_p": 1.0, "temperature": 1.0}, "rounds": []}
    os.makedirs(a.out, exist_ok=True)
    path = os.path.join(a.out, time.strftime("%Y%m%d-%H%M%S") + ".json")

    def save():                                        # after every arm: a run cut short keeps what it measured
        with open(path, "w") as f:
            json.dump(rec, f, indent=1)
    for arm in arms:                                   # warm-up: module loads, graph captures, allocator growth
        run_arm(arm, prompts[:2] + prompts[:1], model, tok, 8, a.batch_size, timers)
    with Clock() as clk:
        for r in range(a.rounds):
            res = {}
            rec["rounds"].append(res)
            for arm in (arms if r % 2 == 0 else arms[::-1]):
                res[arm] = run_arm(arm, prompts, model, tok, a.tokens, a.batch_size, timers)
                rec["sm_mhz"] = clk.median()
                print(r, arm, json.dumps(res[arm]), flush=True)
                save()
    print(json.dumps({k: v for k, v in rec.items() if k != "lengths"}), flush=True)


if __name__ == "__main__":
    main()
