"""Zero-shot variant-effect scoring: many variants of a reference scored from the reference's prefix checkpoints.

A variant's score is its log-likelihood (mean or sum over its nucleotides, as score_sequences reduces it); its effect is that
score minus the reference's.  Scoring every variant from token 0 repeats the reference's forward up to the first changed
token.  Here each reference runs once (StripedHyena.prefill_checkpoints) and keeps its full model state every `stride`
tokens; each variant then runs only from the last checkpoint at or before the row that predicts its first changed token
(StripedHyena.score_tokens_resumed).  That is exact: the model is causal, so rows before the checkpoint see the same context
in the variant as in the reference, and their logprobs are the reference's.

Positions are counted in BOS-prepended ids: row t of a sequence predicts ids[t + 1].
  first difference f   the first index where a variant's ids differ from its reference's (>= 1); len(ids_v) when there is
                       none (the variant equals the reference or is a prefix of it)
  resume point c       stride * floor((f - 1) / stride): the largest checkpoint that still lets the pass compute row f - 1
  score                reference logprobs over rows [0, c) + the variant pass's over rows [c, len(ids_v) - 1)"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .tokenizer import CharLevelTokenizer

BASES = "ACGT"
# Checkpoint tables above this many bytes raise the stride (see choose_stride); 8 GiB keeps a 131k reference at the 7B width
# within one H100 next to the weights and its K,V.
CHECKPOINT_BUDGET_BYTES = 8 << 30


# ----------------------------------------------------------------------------- variants
def saturation_variants(reference: str) -> List[Tuple[str, str]]:
    """Every single-nucleotide substitution of `reference` as (mutation, sequence), position-major (1-based positions in
    order), and at each position the alternatives in A, C, G, T order without the reference base: 3 * L variants for an
    ACGT reference.  Mutations are written like apply_mutations reads them, e.g. 'A1C'."""
    out = []
    for i, ref in enumerate(reference):
        for alt in BASES:
            if alt != ref:
                out.append((f"{ref}{i + 1}{alt}", reference[:i] + alt + reference[i + 1:]))
    return out


def apply_mutations(reference: str, mutant: str) -> str:
    """The sequence of a mutation string 'A123G:T130C' (substitutions, 1-based positions, ':'-separated; '' or '_wt' = the
    reference itself).  A reference base that does not match, a position outside the reference or a malformed entry raises
    ValueError."""
    seq = list(reference)
    if mutant in ("", "_wt", "WT", "wt"):
        return reference
    for m in mutant.split(":"):
        m = m.strip()
        if len(m) < 3 or not m[1:-1].isdigit():
            raise ValueError(f"malformed mutation {m!r} (expected e.g. A123G)")
        ref, pos, alt = m[0], int(m[1:-1]), m[-1]
        if not 1 <= pos <= len(reference):
            raise ValueError(f"mutation {m}: position {pos} outside the reference (length {len(reference)})")
        if reference[pos - 1] != ref:
            raise ValueError(f"mutation {m}: the reference has {reference[pos - 1]!r} at position {pos}, not {ref!r}")
        seq[pos - 1] = alt
    return "".join(seq)


# ----------------------------------------------------------------------------- plan
def first_difference(reference: str, variant: str) -> int:
    """f: the first index of the BOS-prepended ids where `variant` differs from `reference` (>= 1), or len(variant) + 1 =
    len(ids_v) when it does not (equal, or a prefix of the reference).  An extension of the reference differs at
    len(reference) + 1."""
    a = np.frombuffer(reference.encode(), dtype=np.uint8)
    b = np.frombuffer(variant.encode(), dtype=np.uint8)
    m = min(a.shape[0], b.shape[0])
    d = np.flatnonzero(a[:m] != b[:m])
    if d.size:
        return int(d[0]) + 1
    return b.shape[0] + 1 if b.shape[0] <= a.shape[0] else a.shape[0] + 1


def resume_point(f: int, stride: int) -> int:
    """c = stride * floor((f - 1) / stride): the last checkpoint at or before row f - 1 (0 = from the start)."""
    return stride * ((f - 1) // stride)


def checkpoint_bytes(config) -> int:
    """Bytes of one checkpoint: per Hyena layer the fp32 modal state (D, state_size, 2) and two bf16 z rows (2, 3D)."""
    d, s = config["hidden_size"], config["state_size"]
    n_hyena = config["num_layers"] - len(config.get("attn_layer_idxs") or [])
    return n_hyena * (d * s * 2 * 4 + 2 * 3 * d * 2)


def choose_stride(ref_lengths: Sequence[int], stride: int, per_checkpoint: int, budget: int = CHECKPOINT_BUDGET_BYTES) -> int:
    """The stride to use: `stride` (a positive multiple of 128) if the checkpoint tables of references with these nucleotide
    counts fit `budget` bytes, else the next multiple of 128 at which they do."""
    if isinstance(stride, bool) or not isinstance(stride, int) or stride <= 0 or stride % 128:
        raise ValueError(f"checkpoint_stride must be a positive multiple of 128, got {stride!r}")
    while sum(n // stride for n in ref_lengths) * per_checkpoint > budget:      # (n + 1 ids - 1) // stride checkpoints each
        stride += 128
    return stride


def reference_prefix_sums(logprobs: np.ndarray) -> np.ndarray:
    """p[c] = sum of rows [0, c) of one reference's logprobs, in float64."""
    out = np.zeros(logprobs.shape[0] + 1, dtype=np.float64)
    np.cumsum(logprobs, dtype=np.float64, out=out[1:])
    return out


def _normalise(references, variants) -> Tuple[List[str], List[Tuple[int, str]]]:
    refs = [references] if isinstance(references, str) else list(references)
    if not refs or any(not isinstance(r, str) or not r for r in refs):
        raise ValueError("score_variants needs at least one non-empty reference string")
    out = []
    for v in variants:
        if isinstance(v, str):
            if len(refs) != 1:
                raise ValueError("with several references every variant must be a (reference_index, sequence) pair")
            out.append((0, v))
        else:
            r, s = v
            if isinstance(r, bool) or not isinstance(r, (int, np.integer)) or not 0 <= r < len(refs):
                raise ValueError(f"reference index {r!r} outside the {len(refs)} references")
            out.append((int(r), s))
    for _, s in out:
        if not isinstance(s, str) or not s:
            raise ValueError("every variant must be a non-empty string")
    for s in refs + [s for _, s in out]:
        if len(s.encode()) != len(s):
            raise ValueError("non-ASCII characters: the byte-level tokenizer would not give one token per character")
    return refs, out


def plan_variants(refs: Sequence[str], variants: Sequence[Tuple[int, str]], stride: int, max_tokens: int):
    """(first differences, resume points, packs) of the variant passes: packs = frontend.packs over the pass lengths
    len(ids_v) - c of the variants that differ from their reference, as lists of variant indices and pass offsets."""
    from .frontend import packs
    f = [first_difference(refs[r], s) for r, s in variants]
    c = [resume_point(fv, stride) for fv in f]
    run = [k for k, (_, s) in enumerate(variants) if f[k] < len(s) + 1]
    out = []
    for rows, cu in packs([len(variants[k][1]) + 1 - c[k] for k in run], max_tokens, bos=0):
        out.append(([run[i] for i in rows], cu))
    return f, c, out


# ----------------------------------------------------------------------------- scoring
def _pass_ids(variants, idx, c, tokenizer, device):
    """Packed (T,) ids of the variant passes idx: ids_v[c_v:] each."""
    parts = []
    for k in idx:
        s = variants[k][1].encode()
        ids = np.empty(len(s) + 1, dtype=np.int64)
        ids[0] = tokenizer.eod_id
        ids[1:] = np.frombuffer(s, dtype=np.uint8)
        parts.append(ids[c[k]:])
    return torch.from_numpy(np.concatenate(parts)).pin_memory().to(device, non_blocking=True)


def score_variants(references: Union[str, Sequence[str]], variants: Sequence, model, tokenizer: CharLevelTokenizer,
                   reduce_method: str = "mean", checkpoint_stride: int = 128, max_tokens: int = 1 << 17, device: str = "cuda:0",
                   checkpoint_budget_bytes: int = CHECKPOINT_BUDGET_BYTES, stats: Optional[Dict] = None) -> Tuple[List[float], List[float]]:
    """(variant_scores, reference_scores) in input order.  references: one string or a list; variants: strings (one
    reference) or (reference_index, string) pairs.  Substitutions, insertions and deletions all work: only the first
    difference matters.  Each reference group (frontend.packs of the references, <= max_tokens tokens) runs one checkpointed
    forward; its variants that differ from it run in packs of <= max_tokens tokens from their resume points, and variants
    that do not differ need no pass.  If the checkpoint tables at `checkpoint_stride` would exceed `checkpoint_budget_bytes`
    the stride is raised to the next multiple of 128 that fits (choose_stride).  `stats`, if given, receives the stride used,
    the tokens run by the reference and the variant passes, and the number of passes."""
    from .frontend import packs
    if reduce_method not in ("mean", "sum"):
        raise ValueError(f"Invalid reduce_method {reduce_method}")
    if max_tokens < 1:
        raise ValueError("max_tokens must be >= 1")
    refs, var = _normalise(references, variants)
    stride = choose_stride([len(r) for r in refs], checkpoint_stride, checkpoint_bytes(model.config), checkpoint_budget_bytes)
    f, c, _ = plan_variants(refs, var, stride, max_tokens)
    by_ref: Dict[int, List[int]] = {}
    for k, (r, _) in enumerate(var):
        by_ref.setdefault(r, []).append(k)
    ref_scores = [0.0] * len(refs)
    var_scores = [0.0] * len(var)
    n_ref_tokens = n_var_tokens = n_passes = 0
    dev = torch.device(device)
    for group, _ in packs([len(r) for r in refs], max_tokens):
        ids = _pass_ids([(g, refs[g]) for g in group], range(len(group)), [0] * len(group), tokenizer, dev)
        cu = [0]
        for g in group:
            cu.append(cu[-1] + len(refs[g]) + 1)
        ck = model.prefill_checkpoints(ids, cu, stride)
        n_ref_tokens += cu[-1]
        n_passes += 1
        lp = ck.logprobs.cpu().numpy()
        prefix = {}
        for j, g in enumerate(group):
            rows = lp[cu[j]:cu[j + 1] - 1]
            prefix[g] = reference_prefix_sums(rows)
            ref_scores[g] = float(rows.sum(dtype=np.float64) / (1 if reduce_method == "sum" else rows.shape[0]))
        slot = {g: j for j, g in enumerate(group)}
        mine = [k for g in group for k in by_ref.get(g, [])]
        run = [k for k in mine if f[k] < len(var[k][1]) + 1]
        for k in mine:
            if f[k] == len(var[k][1]) + 1:                 # no difference: the reference's own rows
                n = len(var[k][1])
                var_scores[k] = float(prefix[var[k][0]][n] / (1 if reduce_method == "sum" else n))
        for rows, pcu in packs([len(var[k][1]) + 1 - c[k] for k in run], max_tokens, bos=0):
            idx = [run[i] for i in rows]
            ids = _pass_ids(var, idx, c, tokenizer, dev)
            pref_seq = [slot[var[k][0]] for k in idx]
            plen = [c[k] for k in idx]
            start = [ck.base[p] + pl // stride - 1 if pl else -1 for p, pl in zip(pref_seq, plen)]
            vlp = model.score_tokens_resumed(ck, ids, pcu, start, pref_seq, plen).cpu().numpy()
            n_var_tokens += pcu[-1]
            n_passes += 1
            for j, k in enumerate(idx):
                n = len(var[k][1])
                total = prefix[var[k][0]][c[k]] + vlp[pcu[j]:pcu[j + 1] - 1].sum(dtype=np.float64)
                var_scores[k] = float(total / (1 if reduce_method == "sum" else n))
        del ck
    if stats is not None:
        stats.update(checkpoint_stride=stride, reference_tokens=n_ref_tokens, variant_tokens=n_var_tokens, passes=n_passes)
    return var_scores, ref_scores
