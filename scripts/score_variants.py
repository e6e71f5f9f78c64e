"""
Usage: python -m scripts.score_variants \
           --reference-fasta wt.fasta \
           --variants-csv variants.csv \
           --output-tsv scores.tsv \
           --model-name evo-1-8k-base \
           --device cuda:0

Zero-shot variant-effect scoring against one reference (a FASTA file with exactly one record).  The variants come from
--variants-csv (a `sequence` column of full variant sequences, or a `mutant` column of 1-based substitution strings such as
`A123G:T130C`) or from --saturation (every single-nucleotide substitution, position-major, alternatives in A, C, G, T order).
Writes `variant<TAB>score<TAB>delta` in input order: the variant (its mutation string, or its sequence), its mean
log-likelihood (--reduce-method) and that score minus the reference's.  Every variant is scored from the reference's last
checkpoint before its first change (evo_b200.score_variants); the scores are those of scoring the full sequences.
"""
import argparse
import csv
import sys

from evo_b200 import Evo, apply_mutations, saturation_variants, score_variants
from evo_b200.frontend import read_fasta

from scripts.score import _tsv_float


def build_parser():
    parser = argparse.ArgumentParser(description='Score the variants of one reference with an Evo model on the evo_b200 engine.')
    parser.add_argument('--reference-fasta', required=True, help='FASTA file holding exactly one reference sequence')
    src = parser.add_mutually_exclusive_group(required=True)
    src.add_argument('--variants-csv', help='CSV with a `sequence` or a `mutant` column (e.g. A123G:T130C, 1-based)')
    src.add_argument('--saturation', action='store_true', help='Score every single-nucleotide substitution of the reference')
    parser.add_argument('--output-tsv', required=True, help='Output path of variant<TAB>score<TAB>delta')
    parser.add_argument('--reduce-method', choices=['mean', 'sum'], default='mean', help='Reduction of the per-token log-likelihoods')
    parser.add_argument('--checkpoint-stride', type=int, default=128, help='Tokens between reference checkpoints (a multiple of 128)')
    parser.add_argument('--max-tokens', type=int, default=1 << 17, help='Tokens per packed forward')
    parser.add_argument('--model-name', type=str, default='evo-1-131k-base', help='Evo model name')
    parser.add_argument('--device', type=str, default='cuda:0', help='Device for scoring')
    parser.add_argument('--random-init', action='store_true', help='Skip the checkpoint download (random weights; smoke runs offline)')
    parser.add_argument('--model-dir', type=str, default=None, help='Directory of an already downloaded HF snapshot')
    return parser


def read_variants(path, reference):
    """(names, sequences) of a variants CSV: a `sequence` column is taken as is (named by itself), a `mutant` column is applied
    to the reference (apply_mutations: a wrong reference base raises)."""
    with open(path, encoding='utf-8-sig', newline='') as f:
        rows = list(csv.DictReader(f))
    cols = rows[0].keys() if rows else []
    if 'mutant' in cols:
        names = [r['mutant'] for r in rows]
        return names, [apply_mutations(reference, m) for m in names]
    if 'sequence' in cols:
        seqs = [r['sequence'].strip() for r in rows]
        return seqs, seqs
    raise ValueError(f"{path}: needs a 'sequence' or a 'mutant' column")


def main(argv=None):
    args = build_parser().parse_args(argv)
    _, refs = read_fasta(args.reference_fasta)
    if len(refs) != 1:
        raise ValueError(f'{args.reference_fasta}: expected exactly one reference record, found {len(refs)}')
    reference = refs[0]
    if args.saturation:
        names, seqs = map(list, zip(*saturation_variants(reference))) if reference else ([], [])
    else:
        names, seqs = read_variants(args.variants_csv, reference)
    evo_model = Evo(args.model_name, device=args.device, random_init=args.random_init, model_dir=args.model_dir)
    model, tokenizer = evo_model.model, evo_model.tokenizer
    model.eval()
    print(f'Scoring {len(seqs)} variants of a {len(reference)}-nt reference...')
    stats = {}
    scores, (ref_score,) = score_variants(reference, seqs, model, tokenizer, reduce_method=args.reduce_method,
                                          checkpoint_stride=args.checkpoint_stride, max_tokens=args.max_tokens, device=args.device,
                                          stats=stats)
    if stats['checkpoint_stride'] != args.checkpoint_stride:
        print(f"checkpoint stride raised to {stats['checkpoint_stride']} to fit the checkpoint budget", file=sys.stderr)
    with open(args.output_tsv, 'w') as f:
        f.write('variant\tscore\tdelta\n')
        for n, v in zip(names, scores):
            f.write(f'{n}\t{_tsv_float(v)}\t{_tsv_float(v - ref_score)}\n')
    return scores, ref_score


if __name__ == '__main__':
    main()
