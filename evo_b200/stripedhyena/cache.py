"""Inference-state holders.  Attribute names are the contract: evo/generation.py:109-119
and :140-148 read and WRITE them (max_batch_size, seqlen_offset, the three dicts)."""
from dataclasses import dataclass, field
from typing import Optional

from torch import Tensor


@dataclass
class InferenceParams:
    """Attention side: KV cache per layer, (max_batch, max_seqlen, 2, heads, head_dim) bf16
    (flash_attn/modules/mha.py:344-370 layout).

    Shared-prompt decoding (StripedHyena.prefill_shared) adds one prefix per group of rows that sample the same prompt:
    prefix_key_value_memory_dict[layer] (G, P, 2, heads, head_dim) bf16, group_offsets (G + 1) int64 row offsets and
    prefix_len (G) int64 prompt lengths, both on the device; key_value_memory_dict then holds each row's generated tokens only."""
    max_seqlen: int
    max_batch_size: int
    seqlen_offset: int = 0
    batch_size_offset: int = 0
    key_value_memory_dict: dict = field(default_factory=dict)
    lengths_per_sample: Optional[Tensor] = None
    prefix_key_value_memory_dict: Optional[dict] = None
    group_offsets: Optional[Tensor] = None
    prefix_len: Optional[Tensor] = None

    def reset(self, max_seqlen, max_batch_size):
        self.max_seqlen = max_seqlen
        self.max_batch_size = max_batch_size
        self.seqlen_offset = 0
        if self.lengths_per_sample is not None:
            self.lengths_per_sample.zero_()


@dataclass
class RecurrentInferenceParams:
    """Hyena side: fir_state_dict[layer] (B, 3D, 2) bf16 = last two pre-FIR inputs;
    state_dict[layer] (B, D, 8) complex64 = modal state."""
    fir_filter_length: int = 3
    state_dim: int = 16
    seqlen_offset: int = 0
    fir_state_dict: dict = field(default_factory=dict)
    state_dict: dict = field(default_factory=dict)

    def reset(self):
        self.fir_filter_length = 3
        self.state_dim = 16
        self.seqlen_offset = 0
