"""Sequence embeddings: one fp32 vector per sequence from any block of the model, for classifiers, clustering or retrieval.

The sequences run as packed forwards (frontend.packs of at most `max_tokens` tokens, BOS + bytes each, no padding), one
StripedHyena.embed_packed call per pack.  Each requested layer's rows are pooled per sequence on the GPU (evo_pool_varlen),
and only the blocks up to the deepest requested layer run: layer 16 of a 32-block model costs about half a forward.

Layers: a block index in [0, num_layers), a negative index counted from the end (-1 = the last block), or "final" (the
final-norm output, what the unembedding sees).  Pools: "mean" and "max" over the sequence's rows, "last" = its last row.  Row
t of a sequence is the hidden state after its BOS and first t nucleotides; include_bos=False (the default) leaves the BOS row
out of the pool."""
from __future__ import annotations

from typing import Dict, List, Sequence, Union

import numpy as np
import torch

from .stripedhyena.model import POOL_MODES, resolve_layers
from .tokenizer import CharLevelTokenizer

Layer = Union[int, str]


def parse_layers(text: str) -> List[Layer]:
    """The layers of a comma list such as 'final,16,-1' (what scripts/embed.py --layers takes)."""
    out: List[Layer] = []
    for part in text.split(","):
        part = part.strip()
        if part == "final":
            out.append(part)
        else:
            try:
                out.append(int(part))
            except ValueError:
                raise ValueError(f"unknown layer {part!r}: an integer block index or 'final'") from None
    return out


def embed_sequences(seqs: Sequence[str], model, tokenizer: CharLevelTokenizer, layers: Sequence[Layer] = ("final",),
                    pool: str = "mean", include_bos: bool = False, max_tokens: int = 1 << 17,
                    device: str = "cuda:0") -> Dict[Layer, np.ndarray]:
    """{layer: (n, D) float32 array} of the sequences' embeddings, rows in input order, keyed by the layers as given.  An empty
    sequence, a non-ASCII one, a model that is not on `device` (a CUDA device), an unknown layer or pool, or max_tokens < 1
    raise ValueError before anything is launched."""
    from . import _lib
    from .frontend import packed_ids, packs
    if pool not in POOL_MODES:
        raise ValueError(f"unknown pool {pool!r}: one of {sorted(POOL_MODES)}")
    try:
        resolve_layers(layers, model.config.num_layers)
    except _lib.EvoError as e:
        raise ValueError(str(e)) from None
    if max_tokens < 1:
        raise ValueError("max_tokens must be >= 1")
    seqs = list(seqs)
    if any(not isinstance(s, str) or not s for s in seqs):
        raise ValueError("every sequence must be a non-empty string")
    if any(len(s.encode()) != len(s) for s in seqs):
        raise ValueError("non-ASCII characters: the byte-level tokenizer would not give one token per character")
    dev = torch.device(device)
    mdev = model.embedding_layer.weight.device
    if dev.type != "cuda" or mdev != dev:
        raise ValueError(f"embed_sequences runs on a CUDA device: model on {mdev}, device {device!r}")
    keys = list(dict.fromkeys(layers if not isinstance(layers, (str, int)) else [layers]))
    d = model.config.hidden_size
    out = {k: np.empty((len(seqs), d), dtype=np.float32) for k in keys}
    for rows, cu in packs([len(s) for s in seqs], max_tokens):
        ids = packed_ids([seqs[i] for i in rows], tokenizer, device=device)
        got = model.embed_packed(ids, cu, layers=keys, pool=pool, skip_bos=not include_bos)
        for k in keys:
            out[k][rows] = got[k].cpu().numpy()
    return out
