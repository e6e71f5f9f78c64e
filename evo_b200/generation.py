"""Token-by-token generation on top of the stateful call `model(x, inference_params_dict=d)`.

Same entry points, arguments and observable behaviour as the reference's evo/generation.py
(class Generator :38-204, function generate :207-297):
  * the first `force_prompt_threshold` prompt tokens go through one parallel forward, the rest of
    the prompt is teacher-forced one step at a time, then `num_tokens` tokens are sampled;
  * the position bookkeeping the caller-visible state objects expose (`seqlen_offset` on both
    holders) follows the reference, including its jump to the full prompt length after a
    truncated prefill (quirk Q1) and its report-only EOS check (Q2);
  * the per-sequence "scores" keep the reference's one-off alignment (Q3, SURVEY.md 8c).
What differs is underneath: the Hyena prefill state comes out of the scan kernel, so a prompt of
any length can be prefilled in one pass (`force_prompt_threshold >= len(prompt)`); there is no
(B, D, 8, 2L) FFT temporary that forces the 128-token cap."""
from __future__ import annotations

import os
import sys
from typing import List, Optional, Tuple

import numpy as np
import torch

from .scoring import logits_to_logprobs, prepare_batch
from .stripedhyena.sample import sample
from .tokenizer import CharLevelTokenizer


def _gb(device) -> float:
    return torch.cuda.memory_allocated(device=device) / 1e9 if torch.cuda.is_available() else 0.0


class Generator:
    def __init__(self, model, tokenizer: CharLevelTokenizer, top_k: int = 50, top_p: float = 0.7, temperature: float = 1.0):
        self.model, self.tokenizer = model, tokenizer
        self.top_k, self.top_p, self.temperature = top_k, top_p, temperature
        self.untils = ["\n\n"]
        # the token loop runs on the GPU (model.decode_loop) whenever generation is cached; "0" keeps the per-token host loop
        self.device_loop = os.environ.get("EVO_B200_DEVICE_LOOP", "1") != "0"

    # -- pieces of generate() -------------------------------------------------------------
    def _state_for(self, batch: int, device, cached: bool, given: Optional[dict]):
        """(state dict or None, cached?, already prefilled?).  A caller-held state is moved to the
        prompt's device and resumed (evo/generation.py:105-114); otherwise a fresh one is made."""
        if given is not None:
            holders = (given["mha"].key_value_memory_dict, given["hyena"].fir_state_dict, given["hyena"].state_dict)
            for store in holders:
                for key in list(store):
                    store[key] = store[key].to(device)
            return given, True, True
        if not cached:
            return None, False, False
        fresh = self.model.initialize_inference_params()
        for holder in (fresh["mha"], fresh["hyena"]):
            holder.max_batch_size = batch
        return fresh, True, False

    @staticmethod
    def _advance(state: dict, full_prompt_len: int) -> None:
        attn, rec = state["mha"], state["hyena"]
        if attn.seqlen_offset == 0:
            # first step after the prefill: the reference sets the FULL prompt length even if only
            # `force_prompt_threshold` tokens were prefilled (Q1) -- reproduced, not repaired
            attn.seqlen_offset = rec.seqlen_offset = full_prompt_len
        else:
            attn.seqlen_offset += 1
            rec.seqlen_offset += 1

    def _pick(self, last_logits: torch.Tensor) -> torch.Tensor:
        return sample(last_logits, top_k=self.top_k, top_p=self.top_p, temperature=self.temperature)

    def _generate_on_device(self, window, full_prompt, x, tail, num_tokens, state, resumed, stop_at_eos, print_generation, verbose, input_string):
        """Same token sequence as the per-token loop below, with the loop itself on the GPU (SURVEY 8f-2): the prompt goes
        through one parallel forward, then ONE captured CUDA graph per token runs all blocks, picks the token
        (evo_sample_step: forced prompt tail first, then top-k/top-p/temperature or argmax), records it and its logits and
        feeds it back -- no host synchronisation until the end.  Differences from the reference, all report-only: the
        per-token print and the EOS notice (Q2) come out after the loop instead of during it."""
        tk = self.tokenizer
        n_seq, n_tail = window.shape[0], tail.shape[1]
        dev = window.device
        total = n_tail + num_tokens
        picked = torch.empty(n_seq, num_tokens, dtype=torch.long, device=dev)
        kept_logits = torch.empty(n_seq, num_tokens, tk.vocab_size, dtype=torch.float, device=dev)
        pick_args = dict(top_k=self.top_k, top_p=self.top_p, temperature=self.temperature)
        first = 0
        if resumed:
            token = x[:, -1]
            attn = state["mha"]
            start = full_prompt.shape[-1] if attn.seqlen_offset == 0 else attn.seqlen_offset + 1
            forced, n_loop = tail, total
        else:
            with torch.inference_mode():
                logits, state = self.model(x, inference_params_dict=state)
            head = logits[:, -1].contiguous()
            if n_tail:
                token = tail[:, 0]
            else:
                token = self._pick_device(head)
                kept_logits[:, 0], picked[:, 0] = head, token
                first = 1
            start = full_prompt.shape[-1]                      # the reference's jump to the full prompt length (Q1)
            forced, n_loop = tail[:, 1:], total - 1
        if n_loop > 0:
            got, got_logits = self.model.decode_loop(token, state, n_loop, start, forced=forced if forced.shape[1] else None,
                                                     n_out=num_tokens - first, **pick_args)
            picked[:, first:], kept_logits[:, first:] = got, got_logits
        if stop_at_eos and num_tokens >= 2 and bool((picked[0, -2:] == tk.eos).all()):
            print("Stopping generation at EOS")              # report only, as in the reference (Q2)
        if print_generation and verbose and n_seq == 1:
            for t in torch.cat([tail[0], picked[0]]).tolist():
                print(tk.detokenize([t]), end=" ")
        if verbose:
            shown = tk.detokenize_batch(picked)
            shown = [t.split(stop)[0] if stop in t else t for t in shown for stop in self.untils[:1]]
            print(f"\n[generate] in: {input_string} | out: {shown} | {_gb(dev):.2f} GB allocated")
        return picked, kept_logits, state

    def _pick_device(self, head: torch.Tensor, constraints=None) -> torch.Tensor:
        """One call of the device sampler (evo_sample) on (B, V) bf16 logits; under a constraints.RowConstraints, one call of
        evo_sample_constrained, which also advances its rows."""
        import ctypes as C
        from . import _lib
        out = torch.empty(head.shape[0], dtype=torch.long, device=head.device)
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        head = head.to(torch.bfloat16).contiguous()
        stream = C.c_void_p(torch.cuda.current_stream(head.device).cuda_stream)
        if constraints is None:
            _lib.check(_lib.lib().evo_sample(_lib.ptr(head), _lib.ptr(out), head.shape[0], head.shape[1], int(self.top_k), float(self.top_p), float(self.temperature),
                                             seed, 0, stream), "evo_sample")
            return out
        cp = constraints.params()
        cp_dev = torch.frombuffer(bytearray(C.string_at(C.addressof(cp), C.sizeof(cp))), dtype=torch.uint8).to(head.device)
        _lib.check(_lib.lib().evo_sample_constrained(_lib.ptr(head), _lib.ptr(out), head.shape[0], head.shape[1], int(self.top_k), float(self.top_p),
                                                     float(self.temperature), seed, 0, _lib.ptr(cp_dev), stream), "evo_sample_constrained")
        constraints.index0 += 1
        return out

    # -- public ---------------------------------------------------------------------------
    def generate(self, device: str, input_string: str = None, input_ids: torch.Tensor = None, num_tokens: int = 32,
                 cached_generation: bool = True, force_prompt_threshold: int = 128, print_generation: bool = True,
                 verbose: bool = False, skip_special_tokens: bool = False, stop_at_eos: bool = True,
                 max_seqlen: int = None, inference_params_dict: dict = None) -> Tuple[torch.Tensor, torch.Tensor, dict]:
        tk = self.tokenizer
        full_prompt = input_ids if input_ids is not None else torch.tensor(tk.tokenize(input_string), dtype=torch.long, device=device)[None]
        window = full_prompt if max_seqlen is None else full_prompt[:, -max_seqlen:]
        num_tokens = int(num_tokens)
        n_seq, n_prompt = window.shape
        dev = window.device

        # prompt split: [prefilled in parallel | teacher-forced step by step]
        tail = window[:, force_prompt_threshold:] if n_prompt > force_prompt_threshold else window[:, :0]
        x = window[:, :force_prompt_threshold] if tail.shape[1] else window
        n_tail = tail.shape[1]

        picked = torch.empty(n_seq, num_tokens, dtype=torch.long, device=dev)
        kept_logits = torch.empty(n_seq, num_tokens, tk.vocab_size, dtype=torch.float, device=dev)
        eos = torch.tensor([tk.eos], dtype=torch.long, device=device)
        state, cached_generation, resumed = self._state_for(n_seq, dev, cached_generation, inference_params_dict)

        if verbose:
            what = f"prompt {input_string!r}" if input_string is not None else f"prompt ids {tuple(input_ids.shape)}"
            print(f"[generate] {what}; {_gb(dev):.2f} GB allocated; prefill {x.shape[1]} + forced {n_tail} + new {num_tokens}")

        if cached_generation and self.device_loop and hasattr(self.model, "decode_loop") and window.is_cuda and n_tail + num_tokens > 0:
            return self._generate_on_device(window, full_prompt, x, tail, num_tokens, state, resumed, stop_at_eos, print_generation, verbose, input_string)

        last_step = -1
        for last_step in range(n_tail + num_tokens):
            one_token = resumed or (cached_generation and last_step > 0)
            if one_token:
                x = x[:, -1:]
                self._advance(state, full_prompt.shape[-1])
            with torch.inference_mode():
                logits, state = self.model(x, inference_params_dict=state)
            head = logits[:, -1]
            token = tail[:, last_step] if last_step < n_tail else self._pick(head)

            if stop_at_eos and num_tokens >= 2 and bool((picked[0, -2:] == eos).all()):
                print("Stopping generation at EOS")              # report only, as in the reference (Q2)
            if print_generation and verbose and n_seq == 1:
                print(tk.detokenize([token.item()]), end=" ")

            k = last_step - n_tail
            if k >= 0:
                kept_logits[:, k], picked[:, k] = head, token
            x = token[:, None] if one_token else torch.cat([x, token[:, None]], dim=-1)

        done = last_step + 1
        if verbose:
            shown = tk.detokenize_batch(picked[:, :done])
            shown = [t.split(stop)[0] if stop in t else t for t in shown for stop in self.untils[:1]]
            print(f"\n[generate] in: {input_string} | out: {shown} | {_gb(dev):.2f} GB allocated")
        return picked[:, :done], kept_logits[:, :done], state


def _ragged_ids(prompt_seqs, model, tokenizer, n_tokens, prepend_bos):
    """The checks of ragged generation, all before anything is launched; returns (token ids per prompt, device)."""
    from . import _lib
    if n_tokens < 1:
        raise ValueError("ragged generation needs n_tokens >= 1")
    if not hasattr(model, "prefill_ragged"):
        raise ValueError("ragged generation needs the evo_b200 StripedHyena model")
    p0 = next(model.parameters(), None)
    if p0 is None or p0.device.type != "cuda":
        raise ValueError("ragged generation runs on CUDA only: move the model with .to('cuda:N')")
    ids = [([tokenizer.eod_id] if prepend_bos else []) + tokenizer.tokenize(p) for p in prompt_seqs]
    if any(len(p) == 0 for p in prompt_seqs):
        raise ValueError("ragged generation: empty prompt")
    limit = model.config.get("max_seqlen") or 8192
    too_long = [i for i, t in enumerate(ids) if len(t) > limit]
    if too_long:
        raise _lib.EvoError(f"prompt {too_long[0]} has {len(ids[too_long[0]])} tokens, above the model's max_seqlen {limit}")
    return ids, p0.device


def _initial_states(automaton, ids):
    """Each prompt's automaton state (None without constraints); raises ValueError before anything is launched when a
    prompt has no live continuation."""
    if automaton is None:
        return None
    return [automaton.initial_state(t) for t in ids]


def _decode_batch(model, engine, tokenizer, head, state, starts, n_tokens, automaton=None, init_states=None):
    """First pick from the prefill's head logits, then n_tokens - 1 steps of the on-device loop at per-row positions `starts`;
    returns (texts, mean log-likelihood scores) of the batch's rows, scored with the reference's alignment (Q3).
    With an automaton (constraints.compile) every pick is masked by it, rows start in `init_states`, and each row's text and
    score end at its stop motif; the loop is skipped, or ends early, once every row has stopped."""
    from .constraints import RowConstraints
    dev = head.device
    B = head.shape[0]
    picked = torch.empty(B, n_tokens, dtype=torch.long, device=dev)
    kept_logits = torch.empty(B, n_tokens, tokenizer.vocab_size, dtype=torch.float, device=dev)
    rows = None if automaton is None else RowConstraints(automaton, init_states, dev)
    token = engine._pick_device(head, rows)
    kept_logits[:, 0], picked[:, 0] = head, token
    loop_args = dict(n_out=n_tokens - 1, top_k=engine.top_k, top_p=engine.top_p, temperature=engine.temperature)
    if rows is None:
        if n_tokens > 1:
            got, got_logits = model.decode_loop(token, state, n_tokens - 1, starts, **loop_args)
            picked[:, 1:], kept_logits[:, 1:] = got, got_logits
        decoded = tokenizer.detokenize_batch(picked)
        # logits_to_logprobs(trim_bos=True) pairs logits[i] with token[i+1]: the reference's alignment (Q3)
        per_token = logits_to_logprobs(kept_logits, picked).float().cpu().numpy()
        return decoded, [float(np.mean(row)) for row in per_token]
    if n_tokens > 1 and not (automaton.has_stop and int(rows.n_stopped.item()) == B):
        got, got_logits, _ = model.decode_loop(token, state, n_tokens - 1, starts, constraints=rows, **loop_args)
        picked[:, 1:], kept_logits[:, 1:] = got, got_logits
    lengths = [n if n >= 0 else n_tokens for n in rows.length.tolist()]
    # columns past a row's length were never written: zero their token ids so the gather stays in range; their pairs are dropped
    keep = torch.arange(n_tokens, device=dev)[None, :] < torch.tensor(lengths, device=dev)[:, None]
    picked = torch.where(keep, picked, 0)
    per_token = logits_to_logprobs(kept_logits, picked).float().cpu().numpy()
    texts = [tokenizer.detokenize(row[:n]) for row, n in zip(picked.tolist(), lengths)]
    return texts, [float(np.mean(row[:n - 1])) if n > 1 else float("nan") for row, n in zip(per_token, lengths)]


def _generate_shared(prompt_seqs, model, tokenizer, engine, n_tokens, prepend_bos, batch_size, verbose, automaton=None):
    """generate(ragged=True, share_prompts=True): identical prompts form one group; each distinct prompt is prefilled once
    (StripedHyena.prefill_prefixes, packed) and its rows decode against its K,V as one shared prefix
    (StripedHyena.shared_decode_state + decode_loop), in batches of <= batch_size rows (frontend.shared_batches).  Texts and
    scores come back in input order."""
    from .frontend import shared_batches
    ids, _ = _ragged_ids(prompt_seqs, model, tokenizer, n_tokens, prepend_bos)
    init = _initial_states(automaton, ids)
    groups, plan = shared_batches(ids, n_tokens, batch_size)
    last_batch = {g: k for k, (parts, _, _) in enumerate(plan) for g, _ in parts}
    live = {}                                     # group -> (its prefill's prefixes, its index there), until its last batch
    texts: List[str] = [""] * len(ids)
    scores: List[float] = [0.0] * len(ids)
    for k, (parts, fresh, suffix_len) in enumerate(plan):
        with torch.inference_mode():
            if fresh:
                pre = model.prefill_prefixes([ids[groups[g][0]] for g in fresh])
                live.update((g, (pre, j)) for j, g in enumerate(fresh))
                del pre
            head, state = model.shared_decode_state([live[g] + (len(rows),) for g, rows in parts], suffix_len)
        for g, _ in parts:
            if last_batch[g] == k:
                del live[g]
        rows = [r for _, rr in parts for r in rr]
        starts = torch.tensor([len(ids[r]) for r in rows], dtype=torch.int64)
        decoded, got = _decode_batch(model, engine, tokenizer, head, state, starts, n_tokens, automaton,
                                     None if init is None else [init[r] for r in rows])
        del state, head
        if verbose > 1:
            print(f"[generate] shared-prompt batch of {len(rows)} rows in {len(parts)} groups, {len(fresh)} prefilled")
        for j, r in enumerate(rows):
            texts[r], scores[r] = decoded[j], got[j]
    return texts, scores


def _generate_ragged(prompt_seqs, model, tokenizer, engine, n_tokens, prepend_bos, batch_size, verbose, packed_prefill=False, automaton=None):
    """generate(ragged=True): prompts sorted by length and cut into batches of <= batch_size; per batch one ragged prefill
    (StripedHyena.prefill_ragged), one first pick (evo_sample) and one on-device loop with per-row positions.  Texts and
    scores come back in input order."""
    from .frontend import ragged_batches
    ids, _ = _ragged_ids(prompt_seqs, model, tokenizer, n_tokens, prepend_bos)
    init = _initial_states(automaton, ids)
    texts: List[str] = [""] * len(ids)
    scores: List[float] = [0.0] * len(ids)
    for rows, cache_len in ragged_batches([len(t) for t in ids], n_tokens, batch_size):
        with torch.inference_mode():
            head, state = model.prefill_ragged([ids[r] for r in rows], cache_len, packed=packed_prefill)
        starts = torch.tensor([len(ids[r]) for r in rows], dtype=torch.int64)
        decoded, got = _decode_batch(model, engine, tokenizer, head, state, starts, n_tokens, automaton,
                                     None if init is None else [init[r] for r in rows])
        del state, head
        if verbose > 1:
            print(f"[generate] ragged batch of {len(rows)}: prompt lengths {len(ids[rows[0]])}..{len(ids[rows[-1]])}, cache {cache_len}")
        for k, r in enumerate(rows):
            texts[r], scores[r] = decoded[k], got[k]
    return texts, scores


def generate(prompt_seqs: List[str], model, tokenizer: CharLevelTokenizer, n_tokens: int = 100, temperature: float = 0.0,
             top_k: int = 1, top_p: float = 1.0, batched: bool = True, prepend_bos: bool = False,
             cached_generation: bool = False, force_prompt_threshold: int = 128, verbose: int = 1,
             device: str = "cuda:0", ragged: bool = False, batch_size: int = 64, packed_prefill: bool = False, share_prompts: bool = False,
             constraints=None, **kwargs) -> Tuple[List[str], List[float]]:
    """Sequences and mean log-likelihood "scores" for a list of prompts.  Prompts of one common
    length run as one batch; anything else falls back to one prompt at a time (with a note on stderr).

    ragged=True batches prompts of different lengths: they are sorted by length and cut into batches of at most
    `batch_size` (64 keeps the stream-K decode GEMMs; larger batches take the 128x64 tiles), and each batch decodes with a
    position per row.  Every prompt is prefilled whole, so `force_prompt_threshold` does not apply and the reference's
    jump to the full prompt length (Q1) never happens.  Needs cached_generation=True, a CUDA model, non-empty prompts no
    longer than the model's max_seqlen, and n_tokens >= 1; texts and scores come back in input order.  packed_prefill=True
    prefills each batch with one packed forward (StripedHyena.prefill_ragged(packed=True)) instead of one forward per
    distinct prompt length.

    share_prompts=True (with ragged=True) draws many samples of a prompt from one prefill: identical prompts form a group,
    each distinct prompt is prefilled once per call, and the group's rows decode against its K,V as one shared prefix
    instead of holding and re-reading a copy each (frontend.shared_batches keeps a group's rows contiguous in batches of at
    most `batch_size` rows).  Texts and scores come back in input order, scored as with ragged=True.

    constraints (a constraints.Constraints, with ragged=True) controls what is sampled: only A, C, G and T, none of its
    forbidden motifs, no homopolymer above its limit, and each row ends at its first (in-frame) stop motif, which is kept.
    The device sampler masks every pick with the compiled automaton; a row's text ends at its stop, its score is the mean
    log-likelihood over its kept tokens under the model's unmasked logits, and a batch stops decoding once all its rows
    have stopped."""
    if constraints is not None and not ragged:
        raise ValueError("constraints need ragged=True: the reference-shaped path keeps the reference's sampling")
    automaton = None
    if constraints is not None:
        from .constraints import compile as compile_constraints
        automaton = compile_constraints(constraints)
    model.eval()
    engine = Generator(model, tokenizer, top_k=top_k, top_p=top_p, temperature=temperature)
    if share_prompts and not ragged:
        raise ValueError("share_prompts=True needs ragged=True")
    if ragged:
        if not cached_generation:
            raise ValueError("ragged generation needs cached_generation=True")
        if batch_size < 1:
            raise ValueError("batch_size must be >= 1")
        if share_prompts:
            texts, scores = _generate_shared(list(prompt_seqs), model, tokenizer, engine, int(n_tokens), prepend_bos, int(batch_size), verbose,
                                             automaton=automaton)
        else:
            texts, scores = _generate_ragged(list(prompt_seqs), model, tokenizer, engine, int(n_tokens), prepend_bos, int(batch_size), verbose,
                                             packed_prefill=bool(packed_prefill), automaton=automaton)
        if verbose:
            for prompt, text, score in zip(prompt_seqs, texts, scores):
                print(f'Prompt: "{prompt}",\tOutput: "{text}",\tScore: {score}')
        return texts, scores
    uniform = len({len(p) for p in prompt_seqs}) <= 1
    if batched and uniform:
        work = [list(prompt_seqs)]
    else:
        if verbose and not uniform:
            sys.stderr.write("Note: Prompts are of different lengths.\n")
        if verbose:
            sys.stderr.write("Note: Will not do batched generation.\n")
        work = [[p] for p in prompt_seqs]

    chatty = verbose > 1
    texts: List[str] = []
    scores: List[float] = []
    for group in work:
        ids, _ = prepare_batch(group, tokenizer, prepend_bos=prepend_bos, device=device)
        new_ids, new_logits, _ = engine.generate(device=device, input_ids=ids, num_tokens=n_tokens, stop_at_eos=False,
                                                 cached_generation=cached_generation, force_prompt_threshold=force_prompt_threshold,
                                                 print_generation=chatty, verbose=chatty)
        if chatty:
            print(f"[generate] ids {tuple(ids.shape)} -> new ids {tuple(new_ids.shape)}, logits {tuple(new_logits.shape)}")
        decoded = tokenizer.detokenize_batch(new_ids)
        if len(decoded) != ids.shape[0]:
            raise AssertionError("batch size mismatch after detokenisation")
        texts.extend(decoded)
        # logits_to_logprobs(trim_bos=True) pairs logits[i] with token[i+1]: the reference's alignment (Q3)
        per_token = logits_to_logprobs(new_logits, new_ids).float().cpu().numpy()
        scores.extend(float(np.mean(row)) for row in per_token)

    if verbose:
        for prompt, text, score in zip(prompt_seqs, texts, scores):
            print(f'Prompt: "{prompt}",\tOutput: "{text}",\tScore: {score}')
    return texts, scores
