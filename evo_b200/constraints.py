"""Constrained generation: what the device sampler may pick, as one deterministic automaton over {A, C, G, T}.

`Constraints` describes the rules; `compile()` turns them into the tables `evo_sample_constrained` /
`evo_sample_step_constrained` read (include/evo_b200.h).  Any `Constraints` restricts generated tokens to the bytes
A, C, G and T; on top of that:
  * forbid: motifs that must not END inside the generated region (a match straddling the prompt and the generated region
    counts, one wholly inside the prompt does not); with both_strands each motif's reverse complement is forbidden too;
  * max_homopolymer: no run of one base longer than this, a run that starts in the prompt's tail included;
  * stop: a row is finished at the first generated token that completes one of these motifs, which stays in its output;
    with stop_in_frame only occurrences starting at a codon boundary count, codons counted from the prompt's first
    nucleotide (after a leading BOS).

The automaton's state is the product of an Aho-Corasick state over the forbidden and stop motifs, the (last base, run
length) pair when max_homopolymer is set, and the codon phase when stop_in_frame is set.  A state is a violation when the
symbol that entered it completed a forbidden motif or a run above the limit.  Liveness is the greatest fixed point of
"not a violation, and a stop state or at least one live successor"; `allow[s]` holds the symbols whose successor is live.
So a row that starts from a state with some allowed symbol can never reach a state with nothing to sample.

The same module holds the host reference the tests compare the kernels with: `Automaton.walk` applies the automaton to a
token list and `Automaton.masked` sets the disallowed logits of a state to -inf."""
from __future__ import annotations

import collections
from dataclasses import dataclass
from typing import Iterable, Optional, Sequence, Tuple

import numpy as np

ALPHABET = "ACGT"
SYMBOL = {c: i for i, c in enumerate(ALPHABET)}
COMPLEMENT = str.maketrans("ACGT", "TGCA")
N_TOKENS = 512              # the byte-level tokenizer's vocabulary
BOS = 0                     # CharLevelTokenizer.eod_id, what prepend_bos puts in front of a prompt
MAX_STATES = 1 << 16        # 1 MiB of next-state table; far above what realistic motif sets need


def reverse_complement(s: str) -> str:
    return s.translate(COMPLEMENT)[::-1]


def _motifs(name: str, motifs) -> Tuple[str, ...]:
    if isinstance(motifs, str):
        motifs = (motifs,)
    out = tuple(str(m).upper() for m in motifs)
    for m in out:
        if not m or any(c not in SYMBOL for c in m):
            raise ValueError(f"{name} motif {m!r} must be a non-empty string of A, C, G and T")
    return out


def _longest_run(s: str) -> int:
    best = run = 0
    for i, c in enumerate(s):
        run = run + 1 if i and s[i - 1] == c else 1
        best = max(best, run)
    return best


@dataclass(frozen=True)
class Constraints:
    """What generated tokens must satisfy; immutable.  See the module docstring for each field's meaning."""
    forbid: Tuple[str, ...] = ()
    both_strands: bool = True
    max_homopolymer: Optional[int] = None
    stop: Tuple[str, ...] = ()
    stop_in_frame: bool = False

    def __post_init__(self):
        object.__setattr__(self, "forbid", _motifs("forbidden", self.forbid))
        object.__setattr__(self, "stop", _motifs("stop", self.stop))
        object.__setattr__(self, "both_strands", bool(self.both_strands))
        object.__setattr__(self, "stop_in_frame", bool(self.stop_in_frame))
        if self.max_homopolymer is not None:
            if int(self.max_homopolymer) != self.max_homopolymer or self.max_homopolymer < 1:
                raise ValueError(f"max_homopolymer must be an integer >= 1, got {self.max_homopolymer!r}")
            object.__setattr__(self, "max_homopolymer", int(self.max_homopolymer))
        for m in self.stop:
            bad = [f for f in self.forbidden_motifs() if f in m]
            if bad:
                raise ValueError(f"stop motif {m!r} contains the forbidden motif {bad[0]!r}: no row could ever stop on it")
            if self.max_homopolymer is not None and _longest_run(m) > self.max_homopolymer:
                raise ValueError(f"stop motif {m!r} has a run longer than max_homopolymer={self.max_homopolymer}")

    def forbidden_motifs(self) -> Tuple[str, ...]:
        """The forbidden motifs with, under both_strands, their reverse complements."""
        out = list(self.forbid)
        if self.both_strands:
            out += [reverse_complement(m) for m in self.forbid]
        return tuple(dict.fromkeys(out))


class _AhoCorasick:
    """goto (nodes, 4), per node: does a forbidden motif end here, and the lengths of the stop motifs ending here."""

    def __init__(self, forbidden: Sequence[str], stops: Sequence[str]):
        children = [{}]
        forb, stop_lens = [False], [set()]
        for kind, motifs in (("f", forbidden), ("s", stops)):
            for m in motifs:
                node = 0
                for c in m:
                    a = SYMBOL[c]
                    if a not in children[node]:
                        children[node][a] = len(children)
                        children.append({})
                        forb.append(False)
                        stop_lens.append(set())
                    node = children[node][a]
                if kind == "f":
                    forb[node] = True
                else:
                    stop_lens[node].add(len(m))
        n = len(children)
        goto = np.zeros((n, 4), dtype=np.int64)
        fail = [0] * n
        queue = collections.deque()
        for a in range(4):
            child = children[0].get(a)
            if child is None:
                goto[0, a] = 0
            else:
                goto[0, a] = child
                queue.append(child)
        while queue:                                # breadth first: a node's failure target is complete before it
            u = queue.popleft()
            forb[u] = forb[u] or forb[fail[u]]
            stop_lens[u] = stop_lens[u] | stop_lens[fail[u]]
            for a in range(4):
                child = children[u].get(a)
                if child is None:
                    goto[u, a] = goto[fail[u], a]
                else:
                    fail[child] = int(goto[fail[u], a])
                    goto[u, a] = child
                    queue.append(child)
        self.goto, self.forb, self.stop_lens = goto, forb, [frozenset(s) for s in stop_lens]


class Automaton:
    """The compiled tables (what `compile()` returns).
    next (S, 4) int32, allow (S,) uint8 bitmask of the symbols whose successor is live, stop (S,) uint8 flags,
    token_symbol (512,) int8: the symbol of each token, -1 for every byte other than A, C, G, T."""

    def __init__(self, constraints: Constraints, next_, allow, stop, violation, resets):
        self.constraints = constraints
        self.next, self.allow, self.stop = next_, allow, stop
        self.violation = violation
        self._resets = resets                       # phase -> the state a non-ACGT byte leads to
        self.token_symbol = np.full(N_TOKENS, -1, dtype=np.int8)
        for c, a in SYMBOL.items():
            self.token_symbol[ord(c)] = a

    @property
    def n_states(self) -> int:
        return int(self.next.shape[0])

    @property
    def has_stop(self) -> bool:
        return bool(self.constraints.stop)

    def initial_state(self, ids: Sequence[int]) -> int:
        """The state after a prompt's token ids, walked from the root.  Every byte outside ACGT (a BOS included) resets the
        motif and run trackers; every byte except a leading BOS advances the codon phase.  Matches inside the prompt do not
        count.  Raises ValueError when no continuation is live from it."""
        ids = [int(t) for t in ids]
        body = ids[1:] if ids and ids[0] == BOS else ids
        s = self._resets[0]
        phase = 0
        for t in body:
            a = int(self.token_symbol[t]) if 0 <= t < N_TOKENS else -1
            s = self._resets[(phase + 1) % 3 if self.constraints.stop_in_frame else 0] if a < 0 else int(self.next[s, a])
            phase += 1
        if self.allow[s] == 0:
            raise ValueError("no continuation of this prompt satisfies the constraints "
                             f"(prompt tail {bytes(t & 0xFF for t in body[-16:])!r})")
        return s

    def allowed_tokens(self, state: int) -> np.ndarray:
        """(512,) bool: the tokens a row in `state` may pick."""
        sym = self.token_symbol.astype(np.int64)
        return (sym >= 0) & ((int(self.allow[state]) >> np.maximum(sym, 0)) & 1).astype(bool)

    def masked(self, logits, state: int):
        """A copy of a (V,) torch logits row with every entry the state disallows set to -inf."""
        import torch
        ok = torch.zeros(logits.shape[-1], dtype=torch.bool)
        ok[:N_TOKENS] = torch.from_numpy(self.allowed_tokens(state)[:logits.shape[-1]])
        return logits.masked_fill(~ok.to(logits.device), float("-inf"))

    def walk(self, state: int, tokens: Iterable[int]):
        """Apply the automaton to generated tokens from `state`: (the state after each token, length, ok).  The walk ends
        at the first token that reaches a stop state (length = its 1-based index; None when no token does) or at the first
        token the state does not allow (ok = False)."""
        states = []
        for n, t in enumerate(tokens):
            t = int(t)
            if not (0 <= t < N_TOKENS and self.allowed_tokens(state)[t]):
                return states, None, False
            state = int(self.next[state, int(self.token_symbol[t])])
            states.append(state)
            if self.stop[state]:
                return states, n + 1, True
        return states, None, True

    def device_tables(self, device):
        """(next, allow, stop, token_symbol) as device tensors, in the layout evo_constraint_params points at."""
        import torch
        return (torch.from_numpy(self.next).to(device), torch.from_numpy(self.allow).to(device),
                torch.from_numpy(self.stop).to(device), torch.from_numpy(self.token_symbol).to(device))


def compile(constraints: Constraints) -> Automaton:  # noqa: A001 -- the issue's and the docs' name for it
    """Build the automaton of `constraints` (see the module docstring).  Raises ValueError when it would need more than
    MAX_STATES states."""
    if not isinstance(constraints, Constraints):
        raise TypeError("compile() takes a Constraints")
    c = constraints
    ac = _AhoCorasick(c.forbidden_motifs(), c.stop)
    hp = c.max_homopolymer
    phases = 3 if c.stop_in_frame else 1
    # product state: (Aho-Corasick node, last base or -1, run length capped at hp + 1, phase of the next position)
    index, keys = {}, []

    def intern(key):
        i = index.get(key)
        if i is None:
            if len(keys) >= MAX_STATES:
                raise ValueError(f"the constraints need more than {MAX_STATES} automaton states")
            i = index[key] = len(keys)
            keys.append(key)
        return i

    resets = [intern((0, -1, 0, p)) for p in range(phases)]
    next_rows, violation, stop = [], [], []
    k = 0
    while k < len(keys):                                     # breadth first over every state reachable from a reset
        node, last, run, phase = keys[k]
        row = []
        for a in range(4):
            n2 = int(ac.goto[node, a])
            if hp is None:
                l2, r2 = -1, 0
            else:
                l2, r2 = a, min(run + 1 if a == last else 1, hp + 1)
            row.append(intern((n2, l2, r2, (phase + 1) % phases)))
        next_rows.append(row)
        k += 1
    for node, last, run, phase in keys:
        violation.append(ac.forb[node] or (hp is not None and run > hp))
        # the symbol that entered this state sat at position phase - 1; a stop motif of length L ending there starts at a
        # codon boundary when (phase - 1 - (L - 1)) % 3 == 0
        lens = ac.stop_lens[node]
        stop.append(bool(lens) and (not c.stop_in_frame or any((phase - L) % 3 == 0 for L in lens)))
    nxt = np.asarray(next_rows, dtype=np.int32).reshape(-1, 4)
    viol = np.asarray(violation, dtype=bool)
    stp = np.asarray(stop, dtype=bool) & ~viol
    live = ~viol
    while True:                                              # greatest fixed point
        succ_live = live[nxt].any(axis=1)
        new = live & (stp | succ_live)
        if (new == live).all():
            break
        live = new
    allow = (live[nxt] * (1 << np.arange(4))).sum(axis=1).astype(np.uint8)
    return Automaton(c, nxt, allow, stp.astype(np.uint8), viol, resets)



class RowConstraints:
    """The device side of one constrained decode batch: the automaton's tables and each row's state, length and the
    stopped-row counter, with the evo_constraint_params that point at them.  `index0` is the generated index of the next
    pick; the sampling calls that use this object advance it."""

    def __init__(self, automaton: Automaton, states: Sequence[int], device):
        import torch
        self.automaton = automaton
        self.tables = automaton.device_tables(device)
        self.state = torch.tensor([int(s) for s in states], dtype=torch.int32, device=device)
        self.length = torch.full((len(states),), -1, dtype=torch.int64, device=device)
        self.n_stopped = torch.zeros(1, dtype=torch.int32, device=device)
        self.index0 = 0

    def params(self):
        from . import _lib
        nxt, allow, stop, sym = self.tables
        return _lib.ConstraintParams(next=nxt.data_ptr(), allow=allow.data_ptr(), stop=stop.data_ptr(), token_symbol=sym.data_ptr(),
                                     n_states=int(nxt.shape[0]), n_tokens=int(sym.shape[0]), state=self.state.data_ptr(),
                                     length=self.length.data_ptr(), n_stopped=self.n_stopped.data_ptr(), index0=int(self.index0))
