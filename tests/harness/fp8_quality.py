"""What FP8 weights cost in model quality (needs a GPU; writes JSON under out/ unless --out says otherwise).

    python tests/harness/fp8_quality.py --model-dir DIR [--model-name evo-1-8k-base] [--fasta examples/example_seqs.fasta]
    python tests/harness/fp8_quality.py --random-init          # plumbing only: random weights say nothing about quality

One model is loaded in bf16, scored and used for greedy generation; then the same model is rounded to FP8 weights
(quantize_fp8) and the same is done again.  Reported per sequence of the FASTA file: the mean log-likelihood per nucleotide
under each (scoring runs the prefill path on the rounded weights W') and its difference; and, from the sequence's first
--prompt-len nucleotides, how many of --n-tokens greedy tokens the FP8 model generates before it first departs from the bf16
model (the agreement length)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def agreement(a: str, b: str) -> int:
    n = 0
    for x, y in zip(a, b):
        if x != y:
            break
        n += 1
    return n


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--model-dir", default=None)
    ap.add_argument("--model-name", default="evo-1-8k-base")
    ap.add_argument("--random-init", action="store_true")
    ap.add_argument("--fasta", default=os.path.join(ROOT, "examples", "example_seqs.fasta"))
    ap.add_argument("--prompt-len", type=int, default=64)
    ap.add_argument("--n-tokens", type=int, default=128)
    ap.add_argument("--out", default="out/fp8_quality.json")
    a = ap.parse_args(argv)
    if a.model_dir is None and not a.random_init:
        ap.error("--model-dir DIR (a downloaded snapshot) or --random-init")

    import torch
    import evo_b200
    from evo_b200.frontend import read_fasta, score_many
    from tests.harness.gemm_shapes import card

    _, seqs = read_fasta(a.fasta)
    ev = evo_b200.Evo(a.model_name, device="cuda:0", model_dir=a.model_dir, random_init=a.random_init)
    model, tok = ev.model, ev.tokenizer
    model.eval()
    prompts = [s[:a.prompt_len] for s in seqs]
    kw = dict(n_tokens=a.n_tokens, temperature=1.0, top_k=1, cached_generation=True, verbose=0, device="cuda:0", ragged=True)
    res = {}
    for mode in ("bf16", "fp8"):
        if mode == "fp8":
            model.quantize_fp8()
        with torch.inference_mode():
            res[mode] = {"scores": score_many(seqs, model, tok), "generated": evo_b200.generate(prompts, model, tok, **kw)[0]}
    rows = [{"seq": i, "length": len(s), "ll_bf16": res["bf16"]["scores"][i], "ll_fp8": res["fp8"]["scores"][i],
             "ll_diff": res["fp8"]["scores"][i] - res["bf16"]["scores"][i],
             "greedy_agreement": agreement(res["bf16"]["generated"][i], res["fp8"]["generated"][i])} for i, s in enumerate(seqs)]
    diffs = [abs(r["ll_diff"]) for r in rows]
    report = {"model": a.model_name, "weights": "random init" if a.random_init else a.model_dir, "card": card(),
              "n_tokens": a.n_tokens, "prompt_len": a.prompt_len, "mean_abs_ll_diff": sum(diffs) / len(diffs),
              "max_abs_ll_diff": max(diffs), "mean_greedy_agreement": sum(r["greedy_agreement"] for r in rows) / len(rows), "per_sequence": rows}
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps({k: v for k, v in report.items() if k != "per_sequence"}))


if __name__ == "__main__":
    main()
