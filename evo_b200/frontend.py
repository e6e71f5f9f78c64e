"""Batch front-end (SURVEY.md 8f-4): sequences on disk -> padded id matrices on the GPU, in length buckets.

What it replaces in the reference:
  * scripts/score.py:40-55       Bio.SeqIO FASTA parse + fixed-size batches in file order (one pad-to-longest per batch)
  * evo/scoring.py:9-33          prepare_batch: Python-list tokenisation, one int64 tensor and one H2D copy PER SEQUENCE
  * semantic_design.py:82-100    read_prompts: group prompts of identical length into batches of <= batch_size
Here: a FASTA / CSV reader with no dependencies, `length_buckets` (identical-length groups like read_prompts, or a
sorted token-budget packing that bounds the padding waste), and `device_batch`: the sequences' bytes travel to the GPU
ONCE as uint8 (1 byte per nucleotide, pinned staging) and evo_tokenize_pad writes the (B, width) id matrix there."""
from __future__ import annotations

import csv
import ctypes as C
from typing import Dict, Iterable, Iterator, List, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .tokenizer import CharLevelTokenizer


# ----------------------------------------------------------------------------- readers
def read_fasta(path: str) -> Tuple[List[str], List[str]]:
    """(names, sequences) of a FASTA file; sequence lines are joined, whitespace dropped (what str(record.seq) of
    Bio.SeqIO gives, scripts/score.py:40)."""
    names, seqs, cur = [], [], None
    with open(path, "r", encoding="utf-8-sig") as f:
        for line in f:
            line = line.strip()
            if not line:
                continue
            if line.startswith(">"):
                if cur is not None:
                    seqs.append("".join(cur))
                names.append(line[1:].split()[0] if len(line) > 1 else "")
                cur = []
            elif cur is not None:
                cur.append(line)
            else:
                raise ValueError(f"{path}: sequence data before the first '>' header")
    if cur is not None:
        seqs.append("".join(cur))
    return names, seqs


def read_prompts_csv(path: str) -> List[str]:
    """First column of a CSV with a header row (semantic_design.py:72-75)."""
    with open(path, encoding="utf-8-sig", newline="") as f:
        reader = csv.reader(f)
        next(reader)
        return [row[0] for row in reader]


# ----------------------------------------------------------------------------- bucketing
def length_buckets(seqs: Sequence[str], batch_size: int = 32, mode: str = "exact", max_tokens: int = 0,
                   max_waste: float = 0.1) -> List[List[int]]:
    """Index batches.
    mode "exact":  sequences of identical length share a batch of <= batch_size (read_prompts' rule, in first-seen order
                   of the lengths; a length seen once is its own batch) -- zero padding, what batched generation needs.
    mode "sorted": sort by length, then cut a batch when it would exceed batch_size sequences, `max_tokens` padded tokens
                   (0 = no budget) or a padding waste above `max_waste` -- what scoring wants: bounded padding FLOPs and
                   a bounded activation footprint whatever the length mix."""
    if batch_size < 1:
        raise ValueError("batch_size must be >= 1")
    if mode == "exact":
        groups: Dict[int, List[int]] = {}
        for i, s in enumerate(seqs):
            groups.setdefault(len(s), []).append(i)
        out = []
        for idx in groups.values():
            out.extend(idx[k:k + batch_size] for k in range(0, len(idx), batch_size))
        return out
    if mode != "sorted":
        raise ValueError(f"unknown bucketing mode {mode!r}")
    order = sorted(range(len(seqs)), key=lambda i: (len(seqs[i]), i))
    out, cur, cur_tokens = [], [], 0
    for i in order:
        n = len(seqs[i])                                      # ascending, so n is the width of the batch if i joins it
        width_tokens = n * (len(cur) + 1)
        waste = 1.0 - (cur_tokens + n) / max(width_tokens, 1)
        if cur and (len(cur) >= batch_size or (max_tokens and width_tokens > max_tokens) or waste > max_waste):
            out.append(cur)
            cur, cur_tokens = [], 0
        cur.append(i)
        cur_tokens += n
    if cur:
        out.append(cur)
    return out


def ragged_batches(lengths: Sequence[int], n_new: int, batch_size: int = 64, align: int = 64) -> List[Tuple[List[int], int]]:
    """Plan of ragged generation: [(row indices, KV-cache length)] per decode batch.  Indices are sorted by (length, index),
    so prompts of equal length are adjacent rows (what StripedHyena.prefill_ragged needs), and cut into batches of at most
    `batch_size`; a batch's cache holds its longest prompt plus `n_new` tokens, rounded up to `align` (64: the length the
    TMA-fed decode attention takes)."""
    if batch_size < 1:
        raise ValueError("batch_size must be >= 1")
    order = sorted(range(len(lengths)), key=lambda i: (lengths[i], i))
    out = []
    for k in range(0, len(order), batch_size):
        rows = order[k:k + batch_size]
        need = lengths[rows[-1]] + n_new
        out.append((rows, (need + align - 1) // align * align))
    return out


def shared_batches(prompts: Sequence, n_new: int, batch_size: int = 64, align: int = 64):
    """Plan of shared-prompt generation: (groups, batches).  groups[g] = the input indices of distinct prompt g (identical
    prompts, strings or token sequences, form one group), in first-seen order.  batches = [(parts, prefill, suffix_len)] per
    decode batch: parts = [(g, input indices)] with each group's rows contiguous and at most `batch_size` rows in all, groups
    in order, so a large group continues into the next batch(es); prefill = the groups whose rows first appear in this batch
    (each prompt is prefilled once, before its first batch, and its prefix lives until its last); suffix_len = the generated
    tokens' cache length, n_new rounded up to `align`."""
    if batch_size < 1:
        raise ValueError("batch_size must be >= 1")
    index: Dict = {}
    for i, p in enumerate(prompts):
        index.setdefault(p if isinstance(p, str) else tuple(p), []).append(i)
    groups = list(index.values())
    cut, cur, n = [], [], 0
    for g, idx in enumerate(groups):
        k = 0
        while k < len(idx):
            take = min(batch_size - n, len(idx) - k)
            cur.append((g, idx[k:k + take]))
            n, k = n + take, k + take
            if n == batch_size:
                cut.append(cur)
                cur, n = [], 0
    if cur:
        cut.append(cur)
    suffix_len = (n_new + align - 1) // align * align
    batches, seen = [], set()
    for parts in cut:
        fresh = [g for g, _ in parts if g not in seen]
        seen.update(fresh)
        batches.append((parts, fresh, suffix_len))
    return groups, batches


def packs(lengths: Sequence[int], max_tokens: int, bos: int = 1) -> List[Tuple[List[int], List[int]]]:
    """Plan of packed forwards: [(row indices, cu_seqlens)].  Sequences are taken longest first and cut into packs of at most
    `max_tokens` tokens, `bos` extra token per sequence included; inside a pack they stay longest first, so the longest
    sequences' blocks launch first.  A sequence longer than `max_tokens` gets a pack of its own.  cu_seqlens is the pack's
    n + 1 offsets in tokens (flash-attn varlen convention)."""
    if max_tokens < 1:
        raise ValueError("max_tokens must be >= 1")
    order = sorted(range(len(lengths)), key=lambda i: (-lengths[i], i))
    out, rows, cu = [], [], [0]
    for i in order:
        n = lengths[i] + bos
        if rows and cu[-1] + n > max_tokens:
            out.append((rows, cu))
            rows, cu = [], [0]
        rows.append(i)
        cu.append(cu[-1] + n)
    if rows:
        out.append((rows, cu))
    return out


# ----------------------------------------------------------------------------- host bytes -> device ids
def device_batch(seqs: Sequence[str], tokenizer: CharLevelTokenizer, prepend_bos: bool = True, device: str = "cuda:0",
                 dtype: torch.dtype = torch.long) -> Tuple[torch.Tensor, List[int]]:
    """(B, bos + max_len) ids on `device`, right-padded with pad_id, BOS = eod_id -- prepare_batch's result -- from ONE
    pinned uint8 transfer (the bytes) plus B+1 offsets; the id matrix is written by evo_tokenize_pad on the GPU."""
    lengths = [len(s) for s in seqs]
    raw = [s.encode() for s in seqs]
    blens = [len(r) for r in raw]
    if blens != lengths:
        raise ValueError("non-ASCII characters: the byte-level tokenizer would not give one token per character")
    total = sum(blens)
    stage = torch.empty(max(total, 1) + 8 * (len(seqs) + 1), dtype=torch.uint8).pin_memory()
    view = stage.numpy()
    offs = np.zeros(len(seqs) + 1, dtype=np.int64)
    np.cumsum(blens, out=offs[1:])
    obytes = 8 * (len(seqs) + 1)
    view[:obytes] = offs.view(np.uint8)                       # offsets first (8-byte aligned), bytes behind them
    pos = obytes
    for r in raw:
        view[pos:pos + len(r)] = np.frombuffer(r, dtype=np.uint8)
        pos += len(r)
    dev = torch.device(device)
    on_dev = stage.to(dev, non_blocking=True)
    width = (max(lengths) if lengths else 0) + int(prepend_bos)
    ids = torch.empty(len(seqs), width, dtype=dtype, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().evo_tokenize_pad(C.c_void_p(on_dev.data_ptr() + obytes), C.c_void_p(on_dev.data_ptr()), _lib.ptr(ids), int(dtype == torch.long),
                                               len(seqs), width, int(prepend_bos), tokenizer.eod_id, tokenizer.pad_id,
                                               C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "evo_tokenize_pad")
    return ids, lengths


def packed_ids(seqs: Sequence[str], tokenizer: CharLevelTokenizer, device: str = "cuda:0") -> torch.Tensor:
    """(T,) int64 ids on `device` of the sequences end to end, each as [BOS] + bytes: device_batch's one pinned uint8 transfer,
    then the padding of its (n, width) matrix dropped on the device."""
    ids, lengths = device_batch(seqs, tokenizer, prepend_bos=True, device=device)
    keep = torch.arange(ids.shape[1], device=ids.device)[None, :] <= torch.tensor(lengths, device=ids.device)[:, None]
    return ids[keep]


def score_many(seqs: Sequence[str], model, tokenizer: CharLevelTokenizer, batch_size: int = 32, max_tokens: int = 1 << 17,
               reduce_method: str = "mean", device: str = "cuda:0", packed: bool = False) -> List[float]:
    """score_sequences over an arbitrary list in length buckets; scores come back in input order (the loop of
    scripts/score.py:45-55 with bounded padding).

    packed=True: no padding at all -- the sequences (BOS + bytes each) are laid end to end in packs of at most `max_tokens`
    tokens (`packs`) and each pack is one model.score_tokens_packed call; `batch_size` does not apply."""
    from .scoring import score_sequences
    scores: List[float] = [0.0] * len(seqs)
    if packed:
        if reduce_method not in ("mean", "sum"):
            raise ValueError(f"Invalid reduce_method {reduce_method}")
        if any(len(s) == 0 for s in seqs):
            raise ValueError("packed scoring: empty sequence")
        reduce = np.mean if reduce_method == "mean" else np.sum
        for rows, cu in packs([len(s) for s in seqs], max_tokens):
            ids = packed_ids([seqs[i] for i in rows], tokenizer, device=device)
            lp = model.score_tokens_packed(ids, cu, want_logprobs=True)[0].cpu().numpy()
            for k, i in enumerate(rows):
                scores[i] = float(reduce(lp[cu[k]:cu[k + 1] - 1]))
        return scores
    for idx in length_buckets(seqs, batch_size=batch_size, mode="sorted", max_tokens=max_tokens):
        got = score_sequences([seqs[i] for i in idx], model, tokenizer, reduce_method=reduce_method, device=device)
        for i, g in zip(idx, got):
            scores[i] = float(g)
    return scores
