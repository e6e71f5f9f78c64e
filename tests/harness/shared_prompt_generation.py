"""Many samples of one prompt: replicated rows against a shared K,V prefix (development tool, needs a GPU; writes JSON under out/).

    python tests/harness/shared_prompt_generation.py                     # B in {16, 64} x P in {1024, 4096, 8000}, 256 new tokens
    python tests/harness/shared_prompt_generation.py --batches 4 --lengths 512 --tokens 32 --rounds 1 --no-131k

The 7B configuration with random weights generates B samples of one random P-nucleotide prompt with the reference CLI's
sampling settings (top-k 4, top-p 1, temperature 1), two ways, alternating over --rounds, after a warm-up of each:
  replicated  generate([p] * B, ragged=True, packed_prefill=True): B copies of the prompt prefilled and cached (today's best path)
  shared      generate([p] * B, ragged=True, share_prompts=True): one prefill, one prefix cache read once per step for all rows
Per arm: prefill seconds, milliseconds per decode step (median over the decode loops), generated tokens/s over the whole call,
and peak torch.cuda.max_memory_allocated.  Per case, the largest difference between the arms' logits under teacher forcing
(greedy decoding of 32 tokens from the same first token, compared up to the first token where the arms pick differently),
relative to the row's largest |logit|.  A case that does not fit in memory is recorded as such.  Then one run of the shared arm
alone on evo-1-131k-base: a 100 000-nt prompt, 16 samples of 256 tokens, with its peak memory.  The card's name, power limit
and the SM clock sampled while timing are recorded beside the numbers."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.harness.gemm_shapes import Clock, card  # noqa: E402

SAMPLING = dict(top_k=4, top_p=1.0, temperature=1.0)


class Timers:
    """Wall time (ended by a device synchronise) of the prefills and decode loops generate() runs."""

    def __init__(self, model):
        import torch
        self.prefill_s, self.steps = 0.0, []

        def timed(fn, record):
            def wrapper(*a, **kw):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = fn(*a, **kw)
                torch.cuda.synchronize()
                record(a, time.perf_counter() - t0)
                return out
            return wrapper
        for name in ("prefill_ragged", "prefill_prefixes", "shared_decode_state"):
            setattr(model, name, timed(getattr(model, name), self._add_prefill))
        model.decode_loop = timed(model.decode_loop, lambda a, dt: self.steps.append((int(a[2]), dt)))

    def _add_prefill(self, a, dt):
        self.prefill_s += dt

    def reset(self):
        self.prefill_s, self.steps = 0.0, []


def run_arm(arm, prompt, B, model, tok, n_tokens, timers):
    import torch
    from evo_b200 import generate
    kw = dict(n_tokens=n_tokens, cached_generation=True, verbose=0, device="cuda:0", ragged=True, batch_size=64, **SAMPLING)
    kw.update(packed_prefill=True) if arm == "replicated" else kw.update(share_prompts=True)
    timers.reset()
    torch.manual_seed(0)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    try:
        texts, _ = generate([prompt] * B, model, tok, **kw)
    except torch.cuda.OutOfMemoryError as e:
        return {"fits": False, "error": str(e).splitlines()[0][:200]}
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    assert len(texts) == B and all(len(t) == n_tokens for t in texts)
    return {"seconds": round(wall, 3), "tokens_per_s": round(B * n_tokens / wall, 1), "prefill_s": round(timers.prefill_s, 3),
            "decode_ms_per_step": round(statistics.median(dt / n * 1e3 for n, dt in timers.steps), 3) if timers.steps else None,
            "peak_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2)}


def teacher_forced_difference(model, prompt_ids, B, n=32):
    """Greedy decoding of B copies of one prompt from prefill_ragged(packed=True) and from prefill_shared, fed the same first
    token: the largest |logit difference| / max|logit| over every row, up to the first step where the arms pick differently."""
    import torch
    L = len(prompt_ids)
    starts = torch.full((B,), L, dtype=torch.int64)
    out = []
    with torch.inference_mode():
        head_s, ipd_s = model.prefill_shared([prompt_ids], [B], n)
        first = head_s.float().argmax(-1)
    for arm in ("shared", "replicated"):
        if arm == "replicated":
            del ipd_s
            with torch.inference_mode():
                head, ipd = model.prefill_ragged([prompt_ids] * B, (L + n + 63) // 64 * 64, packed=True)
        else:
            head, ipd = head_s, ipd_s
        model._loop = None
        got, kept = model.decode_loop(first, ipd, n, starts, top_k=1)
        out.append((torch.cat([head.float()[:, None], kept], 1).cpu(), torch.cat([first[:, None], got], 1).cpu()))
        del ipd
    (ls, ids_s), (lr, ids_r) = out
    worst = 0.0
    for b in range(B):
        scale = max(1.0, lr[b].abs().max().item())
        for t in range(ls.shape[1]):
            worst = max(worst, (ls[b, t] - lr[b, t]).abs().max().item() / scale)
            if ids_s[b, t] != ids_r[b, t]:
                break
    return worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="16,64")
    ap.add_argument("--lengths", default="1024,4096,8000")
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--long-prompt", type=int, default=100_000)
    ap.add_argument("--long-samples", type=int, default=16)
    ap.add_argument("--no-131k", action="store_true")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=os.path.join(ROOT, "out", "shared_prompt_generation"))
    a = ap.parse_args()
    import random
    import torch
    from evo_b200 import CharLevelTokenizer
    from evo_b200.models import load_checkpoint
    if not torch.cuda.is_available():
        raise SystemExit("shared_prompt_generation.py measures on a GPU; none is visible")
    rng = random.Random(a.seed)
    batches = [int(x) for x in a.batches.split(",") if x]
    lengths = [int(x) for x in a.lengths.split(",") if x]
    tok = CharLevelTokenizer(512)
    model = load_checkpoint("evo-1-8k-base", device="cuda:0", random_init=True)
    model.eval()
    timers = Timers(model)
    rec = {"card": card(), "config": "evo-1-8k-base (7B), random weights", "new_tokens": a.tokens, "sampling": SAMPLING, "cases": []}
    os.makedirs(a.out, exist_ok=True)
    path = os.path.join(a.out, time.strftime("%Y%m%d-%H%M%S") + ".json")

    def save():                                        # after every arm: a run cut short keeps what it measured
        with open(path, "w") as f:
            json.dump(rec, f, indent=1)
    arms = ["replicated", "shared"]
    warm = "".join(rng.choice("ACGT") for _ in range(300))
    for arm in arms:                                   # warm-up: module loads, graph captures, allocator growth
        run_arm(arm, warm, 4, model, tok, 8, timers)
    with Clock() as clk:
        for P in lengths:
            prompt = "".join(rng.choice("ACGT") for _ in range(P))
            for B in batches:
                case = {"B": B, "P": P, "rounds": []}
                rec["cases"].append(case)
                for r in range(a.rounds):
                    res = {}
                    case["rounds"].append(res)
                    for arm in (arms if r % 2 == 0 else arms[::-1]):
                        res[arm] = run_arm(arm, prompt, B, model, tok, a.tokens, timers)
                        rec["sm_mhz"] = clk.median()
                        print(P, B, r, arm, json.dumps(res[arm]), flush=True)
                        save()
                torch.cuda.empty_cache()
                try:
                    case["teacher_forced_max_rel_diff"] = teacher_forced_difference(model, tok.tokenize(prompt), min(B, 16))
                except torch.cuda.OutOfMemoryError as e:
                    case["teacher_forced_max_rel_diff"] = "out of memory: " + str(e).splitlines()[0][:120]
                print(P, B, "teacher-forced max rel diff", case["teacher_forced_max_rel_diff"], flush=True)
                save()
        if not a.no_131k:
            del model, timers
            torch.cuda.empty_cache()
            model = load_checkpoint("evo-1-131k-base", device="cuda:0", random_init=True)
            model.eval()
            model.config["max_seqlen"] = 131072          # generate()'s prompt limit: the config leaves it unset (8192 by default)
            timers = Timers(model)
            prompt = "".join(rng.choice("ACGT") for _ in range(a.long_prompt))
            L, S = a.long_prompt, a.long_samples
            cfg = model.config
            kv_row = 2 * cfg.hidden_size * 2 * len(model._attn_idxs)        # K and V, bf16, every attention layer
            run_arm("shared", warm, 2, model, tok, 8, timers)
            res = run_arm("shared", prompt, S, model, tok, a.tokens, timers)
            rec["long_131k"] = {"config": "evo-1-131k-base, random weights", "prompt": L, "samples": S, "shared": res,
                                "replicated_kv_cache_gb_arithmetic": round(S * ((L + a.tokens + 63) // 64 * 64) * kv_row / 1e9, 1),
                                "shared_kv_cache_gb_arithmetic": round((((L + 63) // 64 * 64) + S * ((a.tokens + 63) // 64 * 64)) * kv_row / 1e9, 2)}
            rec["sm_mhz"] = clk.median()
            print("131k", json.dumps(rec["long_131k"]), flush=True)
            save()
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
