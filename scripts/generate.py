"""
Usage: python -m scripts.generate \
           --model-name evo-1-131k-base \
           --prompt ACGT \
           --n-samples 10 \
           --n-tokens 100 \
           --temperature 1. \
           --top-k 4 \
           --device cuda:0

Generates sequences from a prompt with the reference's sampling arguments (scripts/generate.py of evo-design/evo), on the
evo_b200 engine.  With --cached-generation (the default) the token loop runs on the GPU (one CUDA graph per token, device
sampler); --seed makes a sampled run reproducible.  --prompts-csv reads the prompts from the first column of a CSV with a
header row (semantic_design's format) and generates them all in batches of up to --batch-size, whatever their lengths
(ragged generation: the whole prompt is prefilled, one position per row while decoding); outputs come in file order.
--samples-per-prompt K repeats each CSV prompt K times, prompt-major (semantic_design's n_sample_per_prompt).
--share-prompts sends the samples of one prompt (--prompt with --n-samples, or repeated CSV prompts) through shared-prompt
sampling: each distinct prompt is prefilled once and its samples decode against one shared copy of its K,V.  The boolean
flags keep the reference's `type=bool` parsing (any non-empty value is True).  --fp8-weights generates with an FP8-weight
model (Evo(weights="fp8")); scripts/score.py --fp8-weights scores under the same model.  --fp8-compact uses the same FP8
model holding only its one-byte weights (Evo(weights="fp8-compact")): the same tokens in about half the bf16 weight memory.
--acgt-only, --forbid, --max-homopolymer, --stop and --stop-in-frame constrain what is sampled (evo_b200.Constraints): any of
them keeps the outputs to A, C, G and T; they need the ragged paths (--prompts-csv or --share-prompts).
"""
import argparse

import torch

from evo_b200 import Constraints, Evo, generate
from evo_b200.frontend import read_prompts_csv


def build_parser():
    parser = argparse.ArgumentParser(description='Generate sequences with an Evo model on the evo_b200 engine.')
    parser.add_argument('--model-name', type=str, default='evo-1-131k-base', help='Evo model name')
    parser.add_argument('--prompt', type=str, default='ACGT', help='Prompt for generation')
    parser.add_argument('--n-samples', type=int, default=3, help='Number of sequences to sample at once')
    parser.add_argument('--n-tokens', type=int, default=100, help='Number of tokens to generate')
    parser.add_argument('--temperature', type=float, default=1.0, help='Temperature during sampling')
    parser.add_argument('--top-k', type=int, default=4, help='Top K during sampling')
    parser.add_argument('--top-p', type=float, default=1., help='Top P during sampling')
    parser.add_argument('--cached-generation', type=bool, default=True, help='Use KV caching during generation')
    parser.add_argument('--batched', type=bool, default=True, help='Use batched generation')
    parser.add_argument('--prepend-bos', type=bool, default=False, help='Prepend BOS token')
    parser.add_argument('--device', type=str, default='cuda:0', help='Device for generation')
    parser.add_argument('--verbose', type=int, default=1, help='Verbosity level')
    parser.add_argument('--seed', type=int, default=None, help='torch.manual_seed before sampling')
    parser.add_argument('--random-init', action='store_true', help='Skip the checkpoint download (random weights; smoke runs offline)')
    parser.add_argument('--model-dir', type=str, default=None, help='Directory of an already downloaded HF snapshot')
    parser.add_argument('--fp8-weights', action='store_true',
                        help='Round the linear-layer weights onto an FP8 (E4M3) grid, one power-of-two scale per row (Evo(weights="fp8"))')
    parser.add_argument('--fp8-compact', action='store_true',
                        help='The --fp8-weights model keeping only its one-byte weights: same outputs, less memory (Evo(weights="fp8-compact"); '
                             'takes precedence over --fp8-weights)')
    parser.add_argument('--prompts-csv', type=str, default=None,
                        help='CSV whose first column (after a header row) holds the prompts; generates every prompt once, batched whatever their lengths')
    parser.add_argument('--batch-size', type=int, default=64, help='Prompts per decode batch with --prompts-csv')
    parser.add_argument('--samples-per-prompt', type=int, default=1, help='Samples of each --prompts-csv prompt, prompt-major')
    parser.add_argument('--share-prompts', action='store_true',
                        help='Prefill each distinct prompt once and decode its samples against one shared K,V prefix')
    parser.add_argument('--acgt-only', action='store_true', help='Sample only the bytes A, C, G and T')
    parser.add_argument('--forbid', type=str, default=None,
                        help='Comma-separated motifs that must not appear in the output, on either strand (e.g. GGTCTC,CGTCTC)')
    parser.add_argument('--max-homopolymer', type=int, default=None, help='Longest run of one base allowed in the output')
    parser.add_argument('--stop', type=str, default=None,
                        help='Comma-separated motifs that end a sample when generated (e.g. TAA,TAG,TGA); the motif is kept')
    parser.add_argument('--stop-in-frame', action='store_true',
                        help='--stop motifs count only at codon boundaries, counted from the prompt\'s first nucleotide')
    return parser


def constraints_arg(args):
    """The Constraints the constraint flags describe, or None when none is given."""
    split = lambda v: tuple(m.strip() for m in v.split(',') if m.strip()) if v else ()
    if not (args.acgt_only or args.forbid or args.max_homopolymer is not None or args.stop or args.stop_in_frame):
        return None
    if args.prompts_csv is None and not args.share_prompts:
        raise SystemExit('constraint flags need --prompts-csv or --share-prompts')
    return Constraints(forbid=split(args.forbid), max_homopolymer=args.max_homopolymer, stop=split(args.stop),
                       stop_in_frame=args.stop_in_frame)


def weights_arg(args):
    """The Evo(weights=...) value the FP8 flags select."""
    return 'fp8-compact' if args.fp8_compact else 'fp8' if args.fp8_weights else 'bf16'


def main(argv=None):
    args = build_parser().parse_args(argv)
    constraints = constraints_arg(args)
    evo_model = Evo(args.model_name, device=args.device, random_init=args.random_init, model_dir=args.model_dir,
                    weights=weights_arg(args))
    model, tokenizer = evo_model.model, evo_model.tokenizer
    model.eval()
    if args.seed is not None:
        torch.manual_seed(args.seed)
    print('Generated sequences:')
    if args.samples_per_prompt < 1:
        raise SystemExit('--samples-per-prompt must be >= 1')
    if args.prompts_csv is not None:
        prompts = [p for p in read_prompts_csv(args.prompts_csv) for _ in range(args.samples_per_prompt)]
        return generate(prompts, model, tokenizer, n_tokens=args.n_tokens, temperature=args.temperature,
                        top_k=args.top_k, top_p=args.top_p, cached_generation=True, prepend_bos=args.prepend_bos, device=args.device,
                        verbose=args.verbose, ragged=True, batch_size=args.batch_size, share_prompts=args.share_prompts,
                        constraints=constraints)
    if args.share_prompts:
        return generate([args.prompt] * args.n_samples, model, tokenizer, n_tokens=args.n_tokens, temperature=args.temperature,
                        top_k=args.top_k, top_p=args.top_p, cached_generation=True, prepend_bos=args.prepend_bos, device=args.device,
                        verbose=args.verbose, ragged=True, batch_size=args.batch_size, share_prompts=True, constraints=constraints)
    return generate([args.prompt] * args.n_samples, model, tokenizer, n_tokens=args.n_tokens, temperature=args.temperature,
                    top_k=args.top_k, top_p=args.top_p, cached_generation=args.cached_generation, batched=args.batched,
                    prepend_bos=args.prepend_bos, device=args.device, verbose=args.verbose)


if __name__ == '__main__':
    main()
