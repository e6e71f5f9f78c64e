"""
Usage: python -m scripts.score \
           --input-fasta examples/example_seqs.fasta \
           --output-tsv scores.tsv \
           --model-name evo-1-131k-base \
           --device cuda:0

Scores the sequences of a FASTA file (mean log-likelihood per nucleotide) and writes `seqs<TAB>scores`.
Same arguments as the reference's scripts/score.py; what runs underneath is the evo_b200 engine: FASTA read without
Biopython (evo_b200.frontend.read_fasta), sequences scored in LENGTH BUCKETS (--batch-size sequences or --max-tokens padded
tokens per batch, whichever is hit first; the reference pads every file-order batch to its longest member), scores returned
in file order.  --packed lays the sequences end to end without any padding instead (packs of --max-tokens tokens, one
forward each).  --random-init / --model-dir are for boxes without network.  --fp8-weights scores under the FP8-weight model
(Evo(weights="fp8")), the model scripts/generate.py --fp8-weights samples from; --fp8-compact scores under that model
held as one-byte weights only (Evo(weights="fp8-compact")): the same scores in less device memory.
"""
import argparse

import numpy as np

from evo_b200 import Evo
from evo_b200.frontend import read_fasta, score_many


def build_parser():
    parser = argparse.ArgumentParser(description='Score sequences with an Evo model on the evo_b200 engine.')
    parser.add_argument('--input-fasta', required=True, help='Input FASTA file path')
    parser.add_argument('--output-tsv', required=True, help='Output path to save tab-separated values')
    parser.add_argument('--model-name', type=str, default='evo-1-131k-base', help='Evo model name')
    parser.add_argument('--batch-size', type=int, default=32, help='Number of sequences to evaluate at a time')
    parser.add_argument('--max-tokens', type=int, default=1 << 17, help='Padded tokens per batch (bounds the activation footprint)')
    parser.add_argument('--packed', action='store_true', help='Score sequences packed end to end (no padding) in packs of --max-tokens tokens')
    parser.add_argument('--device', type=str, default='cuda:0', help='Device for scoring')
    parser.add_argument('--random-init', action='store_true', help='Skip the checkpoint download (random weights; smoke runs offline)')
    parser.add_argument('--model-dir', type=str, default=None, help='Directory of an already downloaded HF snapshot')
    parser.add_argument('--fp8-weights', action='store_true',
                        help='Round the linear-layer weights onto an FP8 (E4M3) grid, one power-of-two scale per row (Evo(weights="fp8"))')
    parser.add_argument('--fp8-compact', action='store_true',
                        help='The --fp8-weights model keeping only its one-byte weights: same outputs, less memory (Evo(weights="fp8-compact"); '
                             'takes precedence over --fp8-weights)')
    return parser


def weights_arg(args):
    """The Evo(weights=...) value the FP8 flags select."""
    return 'fp8-compact' if args.fp8_compact else 'fp8' if args.fp8_weights else 'bf16'


def main(argv=None):
    args = build_parser().parse_args(argv)
    evo_model = Evo(args.model_name, device=args.device, random_init=args.random_init, model_dir=args.model_dir,
                    weights=weights_arg(args))
    model, tokenizer = evo_model.model, evo_model.tokenizer
    model.eval()
    _, seqs = read_fasta(args.input_fasta)
    print(f'Scoring {len(seqs)} sequences...')
    scores = score_many(seqs, model, tokenizer, batch_size=args.batch_size, max_tokens=args.max_tokens, device=args.device,
                        packed=args.packed)
    with open(args.output_tsv, 'w') as f:
        f.write('seqs\tscores\n')
        for s, v in zip(seqs, scores):
            f.write(f'{s}\t{_tsv_float(v)}\n')
    return scores


def _tsv_float(v):
    """The text pandas' to_csv writes for a float32 score column (the reference's scripts/score.py:57-58): the shortest decimal
    that round-trips the float32, an empty field for NaN."""
    v32 = np.float32(v)
    return '' if np.isnan(v32) else str(v32)


if __name__ == '__main__':
    main()
