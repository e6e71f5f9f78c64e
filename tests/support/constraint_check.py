"""Plain-string statement of the generation constraints, written independently of the automaton in evo_b200/constraints.py:
the CPU tests compare the compiled automaton with it and the GPU tests check generated outputs with it."""
from typing import Optional, Tuple


def _revcomp(s: str) -> str:
    return "".join({"A": "T", "C": "G", "G": "C", "T": "A"}[ch] for ch in reversed(s))


def check_text(prompt: str, text: str, constraints) -> Tuple[bool, Optional[int]]:
    """(every rule held, the 1-based index of the generated character that completes the first stop motif, or None) for a
    generated `text` that followed `prompt` (the prompt's characters, without a BOS).  Checking ends at that stop."""
    c = constraints
    forbidden = list(c.forbid) + ([_revcomp(m) for m in c.forbid] if c.both_strands else [])
    full = prompt + text
    p = len(prompt)
    # matches and runs may reach back into the prompt, but not past its last byte outside ACGT
    clean = max((i + 1 for i, ch in enumerate(prompt) if ch not in "ACGT"), default=0)
    for end in range(p, len(full)):
        if full[end] not in "ACGT":
            return False, None
        window = full[clean:end + 1]
        if any(window.endswith(m) for m in forbidden):
            return False, None
        if c.max_homopolymer is not None and window.endswith(window[-1] * (c.max_homopolymer + 1)):
            return False, None
        for m in c.stop:
            # codons count from the prompt's first character
            if window.endswith(m) and (not c.stop_in_frame or (end - len(m) + 1) % 3 == 0):
                return True, end - p + 1
    return True, None
