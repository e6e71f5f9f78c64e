"""
Usage: python -m scripts.embed \
           --input-fasta examples/example_seqs.fasta \
           --output-npz embeddings.npz \
           --layers final,16 \
           --pool mean \
           --model-name evo-1-131k-base \
           --device cuda:0

Embeds the sequences of a FASTA file: one float32 vector per sequence and requested layer (evo_b200.embed_sequences).  The
npz holds `names` (the FASTA headers, in file order) and one (n, D) float32 array per layer, named `layer_final`, `layer_16`,
`layer_-1` and so on, rows in file order.  --layers is a comma list of block indices (negative ones count from the end) and
`final` (the final-norm output); only the blocks up to the deepest one run.  --pool mean|max|last pools each sequence's
nucleotide rows (--include-bos adds the BOS row).  --random-init / --model-dir are for boxes without network.
"""
import argparse

import numpy as np

from evo_b200 import Evo, embed_sequences
from evo_b200.embeddings import parse_layers
from evo_b200.frontend import read_fasta


def build_parser():
    parser = argparse.ArgumentParser(description='Embed sequences with an Evo model on the evo_b200 engine.')
    parser.add_argument('--input-fasta', required=True, help='Input FASTA file path')
    parser.add_argument('--output-npz', required=True, help='Output .npz path')
    parser.add_argument('--layers', type=parse_layers, default=['final'], help='Comma list of block indices and/or `final`')
    parser.add_argument('--pool', choices=['mean', 'max', 'last'], default='mean', help='Pooling over each sequence\'s rows')
    parser.add_argument('--include-bos', action='store_true', help='Pool the BOS row too')
    parser.add_argument('--max-tokens', type=int, default=1 << 17, help='Tokens per packed forward')
    parser.add_argument('--model-name', type=str, default='evo-1-131k-base', help='Evo model name')
    parser.add_argument('--device', type=str, default='cuda:0', help='Device for the forward')
    parser.add_argument('--random-init', action='store_true', help='Skip the checkpoint download (random weights; smoke runs offline)')
    parser.add_argument('--model-dir', type=str, default=None, help='Directory of an already downloaded HF snapshot')
    return parser


def npz_arrays(names, embeddings):
    """The arrays of the output file: `names` and `layer_<layer>` per layer."""
    arrays = {'names': np.array(names, dtype=str)}
    for layer, emb in embeddings.items():
        arrays[f'layer_{layer}'] = emb
    return arrays


def main(argv=None):
    args = build_parser().parse_args(argv)
    names, seqs = read_fasta(args.input_fasta)
    evo_model = Evo(args.model_name, device=args.device, random_init=args.random_init, model_dir=args.model_dir)
    model, tokenizer = evo_model.model, evo_model.tokenizer
    model.eval()
    print(f'Embedding {len(seqs)} sequences at layers {",".join(map(str, args.layers))}...')
    emb = embed_sequences(seqs, model, tokenizer, layers=args.layers, pool=args.pool, include_bos=args.include_bos,
                          max_tokens=args.max_tokens, device=args.device)
    np.savez(args.output_npz, **npz_arrays(names, emb))
    return emb


if __name__ == '__main__':
    main()
