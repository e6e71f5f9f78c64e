"""`StripedHyena` with the object protocol evo-design/evo relies on, executed by libevo_b200.so.

Boundary obligations (SURVEY.md section 8b), each pinned by a reference call site:
  StripedHyena(cfg)                                  evo/models.py:146
  .load_state_dict(sd, strict=True) with HF names    evo/models.py:124-147
  .to_bfloat16_except_poles_residues(); .to(device)  evo/models.py:148-150
  model(ids) -> (logits, None)                       evo/scoring.py:81,116
  model(x, inference_params_dict=d) -> (logits, d)   evo/generation.py:152
  model.initialize_inference_params()                evo/generation.py:117

The module tree only exists to carry parameters under the checkpoint's key names; `forward`
never calls a torch op on activations.  torch supplies device memory and the stream.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import math
import numbers
import os
from dataclasses import dataclass, field
from itertools import accumulate
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib
from .._lib import (EPI_BIAS, EPI_BIAS_RESID, EPI_BIAS_ROPE, EPI_GELU_GATE, EPI_NONE, EPI_RESID, AttnParams, AttnVarlenParams,
                    AttnVarlenPrefixParams, GemmParams, GemmSmallMParams, HyenaParams, HyenaVarlenCkptParams, HyenaVarlenParams, check, ptr)
from .cache import InferenceParams, RecurrentInferenceParams

# attention variant passed to evo_attn_fwd_ws: every variant runs the same kernel, and 2 also accepts peer-scattered output
ATTN_VARIANT = 2


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def packed_lengths(cu_seqlens, T: int):
    """Host check of a packed batch's sequence boundaries (flash-attn varlen convention): cu_seqlens holds n + 1 offsets,
    cu[0] = 0, strictly increasing (no empty sequence), cu[n] = T.  Returns the n lengths; raises EvoError otherwise."""
    cu = [int(c) for c in (cu_seqlens.tolist() if torch.is_tensor(cu_seqlens) else cu_seqlens)]
    if len(cu) < 2 or cu[0] != 0:
        raise _lib.EvoError(f"cu_seqlens must hold n + 1 >= 2 offsets starting at 0, got {cu[:4]}")
    lengths = [b - a for a, b in zip(cu[:-1], cu[1:])]
    if min(lengths) <= 0:
        raise _lib.EvoError(f"cu_seqlens must be strictly increasing (every sequence non-empty); sequence {lengths.index(min(lengths))} has length {min(lengths)}")
    if cu[-1] != T:
        raise _lib.EvoError(f"cu_seqlens ends at {cu[-1]}, the packed ids hold {T} tokens")
    if len(lengths) > 65535:
        raise _lib.EvoError(f"{len(lengths)} sequences in one pack; at most 65535")
    return lengths


POOL_MODES = {"mean": _lib.POOL_MEAN, "max": _lib.POOL_MAX, "last": _lib.POOL_LAST}


def resolve_layers(layers, num_layers: int):
    """{layer: block index or "final"} of an embedding request: a layer is an int in [0, num_layers), a negative int counted
    from the end (-1 = the last block), or "final" (the final-norm output the unembedding sees).  Raises EvoError otherwise."""
    if isinstance(layers, (str, int)):
        layers = [layers]
    out = {}
    for k in layers:
        if isinstance(k, str) and k == "final":
            out[k] = "final"
        elif isinstance(k, numbers.Integral) and not isinstance(k, bool) and -num_layers <= k < num_layers:
            out[k] = int(k) % num_layers
        else:
            raise _lib.EvoError(f"unknown layer {k!r}: an int in [{-num_layers}, {num_layers}) or 'final'")
    if not out:
        raise _lib.EvoError("no layer requested")
    return out


class PrefixCheckpoints:
    """What StripedHyena.prefill_checkpoints keeps of n references: logprobs (T,) fp32 of the packed references (cu: n + 1 host
    offsets, lengths), the checkpoint stride, base (n + 1 host offsets: reference b's checkpoints are table rows
    [base[b], base[b + 1]), row base[b] + k - 1 = the state after its first k * stride tokens), and per layer: state[i]
    (n_ckpt, D, S, 2) fp32 and halo[i] (n_ckpt, 2, 3D) bf16 for Hyena layers, kv[i] (n, longest, 2, H, 128) bf16 for
    attention layers."""

    def __init__(self, logprobs, lengths, cu, stride, base, state, halo, kv):
        self.logprobs, self.lengths, self.cu, self.stride, self.base = logprobs, lengths, cu, stride, base
        self.state, self.halo, self.kv = state, halo, kv

    @property
    def n_ckpt(self) -> int:
        return self.base[-1]


@dataclass
class _Capture:
    """What a packed pass keeps for prefill_checkpoints (see PrefixCheckpoints), filled layer by layer into state, halo and kv;
    base and halo_rows (the z rows c - 2, c - 1 of every checkpoint c) are on the device."""
    n: int
    stride: int
    base: torch.Tensor
    halo_rows: torch.Tensor
    state: dict = field(default_factory=dict)
    halo: dict = field(default_factory=dict)
    kv: dict = field(default_factory=dict)


@dataclass
class _Resume:
    """Where a packed pass resumes its sequences from (score_tokens_resumed): the three tensors are on the device, plen holds
    prefix_len on the host."""
    ckpts: PrefixCheckpoints
    start_idx: torch.Tensor
    prefix_seq: torch.Tensor
    prefix_len: torch.Tensor
    plen: list


@dataclass
class _Pack:
    """A checked packed batch (StripedHyena._varlen): n sequences end to end as T rows, their offsets cu on the device and
    cu_host on the host; ckpt / resume: what the pass also captures or resumes from."""
    cu: torch.Tensor
    cu_host: list
    n: int
    T: int
    max_len: int
    lengths: list
    rope: Optional[tuple] = None
    ckpt: Optional[_Capture] = None
    resume: Optional[_Resume] = None


# ----------------------------------------------------------------------------- parameter carriers
class _Scale(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.scale = nn.Parameter(torch.ones(dim))


class _Linear(nn.Module):
    def __init__(self, fan_in, fan_out, bias):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(fan_out, fan_in).normal_(0.0, 1.0 / math.sqrt(fan_in)))
        self.bias = nn.Parameter(torch.zeros(fan_out)) if bias else None


def pack_w12(l1: torch.Tensor, l2: torch.Tensor, ipad: int) -> torch.Tensor:
    """(inner, K) x 2 -> (2*ipad, K): rows interleaved in 128-row groups [l1 rows g*128.. | l2 rows g*128..], zero rows past
    `inner`, so one 128x256 accumulator tile holds l1.x and l2.x of the same 128 inner features (gate fused in the epilogue)."""
    inner, k = l1.shape
    out = l1.new_zeros(ipad // 128, 2, 128, k)
    out[:, 0] = F.pad(l1, (0, 0, 0, ipad - inner)).view(ipad // 128, 128, k)
    out[:, 1] = F.pad(l2, (0, 0, 0, ipad - inner)).view(ipad // 128, 128, k)
    return out.view(2 * ipad, k)


def fp8_round_rows(w: torch.Tensor):
    """Host reference of the FP8 weight rounding (evo_fp8_quantize_rows): an (N, K) bf16 matrix -> (W', q, e) with
    W'[n, k] = q[n, k] 2^e[n], q torch.float8_e4m3fn (round to nearest even), e[n] = ceil(log2(amax_n / 448)) but at least -124
    (so that W' is exactly a bf16 number), e = 0 for an all-zero row.  amax = m 2^p, m in [0.5, 1), 448 = 0.875 2^9."""
    a = w.float().abs().amax(dim=1)
    m, p = torch.frexp(a)
    e = torch.where(m <= 0.875, p - 9, p - 8).clamp_min(-124)
    e = torch.where(a > 0, e, torch.zeros_like(e))
    q = torch.ldexp(w.float(), -e[:, None].float()).to(torch.float8_e4m3fn)
    return torch.ldexp(q.float(), e[:, None].float()).to(torch.bfloat16), q, e.to(torch.int8)


def _fp8_view(N: int, K: int, R: int):
    """Axes of an (N, K) matrix as the FP8 decode layout sees them (csrc/gemm_smallm.cu): rows (tile, r, warpgroup, warp,
    fragment row half, lane / 4), columns (k-block, 32-wide half, k16 step, fragment k half, lane % 4, pair element)."""
    return (N // (128 * R), R, 2, 4, 2, 8, K // 64, 2, 2, 2, 4, 2)


_FP8_ORDER = (0, 6, 1, 2, 3, 7, 5, 10, 8, 9, 4, 11)   # -> (tile, k-block, r, warpgroup, warp, half, lane, step, register, pair)


def fp8_layout(q: torch.Tensor, gate: bool = False) -> torch.Tensor:
    """(N, K) E4M3 weights -> the flat byte order evo_gemm_smallm_fp8 streams (gate: a packed w12, two 128-row groups per tile)."""
    N, K = q.shape
    return q.view(torch.uint8).reshape(_fp8_view(N, K, 2 if gate else 1)).permute(_FP8_ORDER).reshape(-1)


def fp8_unlayout(flat: torch.Tensor, N: int, K: int, gate: bool = False) -> torch.Tensor:
    """Inverse of fp8_layout: the flat bytes back to an (N, K) torch.float8_e4m3fn matrix."""
    view = _fp8_view(N, K, 2 if gate else 1)
    inv = sorted(range(len(_FP8_ORDER)), key=_FP8_ORDER.__getitem__)
    return flat.view(torch.uint8).reshape([view[i] for i in _FP8_ORDER]).permute(inv).reshape(N, K).view(torch.float8_e4m3fn)


def unpack_w12(w12: torch.Tensor, inner: int):
    ipad, k = w12.shape[0] // 2, w12.shape[1]
    v = w12.view(ipad // 128, 2, 128, k)
    return v[:, 0].reshape(ipad, k)[:inner], v[:, 1].reshape(ipad, k)[:inner]


class _GatedMLP(nn.Module):
    """ParallelGatedMLP parameters, held ONLY in the layouts the GEMMs read (SURVEY 8f-3: no second copy):
      w12 (2*ipad, D)  l1 / l2 interleaved per 128 rows, zero-padded 10928 -> 11008 (pack_w12)
      w3  (D, ipad)    l3 zero-padded along K
    The checkpoint's key names (mlp.l1.weight, mlp.l2.weight, mlp.l3.weight; evo/models.py:124-147) are what state_dict()
    shows and what load_state_dict() accepts: two hooks translate at the module boundary."""

    def __init__(self, cfg):
        super().__init__()
        d = cfg.hidden_size
        mult = cfg.get("inner_size_multiple_of", 64) * (cfg.get("model_parallel_size") or 1)
        inner = mult * ((int(2 * d * 4 / 3) + mult - 1) // mult)
        if cfg.get("inner_mlp_size") is not None:
            inner = cfg.get("inner_mlp_size")
        if (cfg.get("mlp_activation") or "silu") != "gelu":
            raise NotImplementedError("evo_b200 implements the Evo configs' exact-erf GELU gate only")
        self.inner, self.ipad = inner, _round_up(inner, 128)
        mk = lambda fo, fi: torch.empty(fo, fi).normal_(0.0, 1.0 / math.sqrt(fi))
        self.w12 = nn.Parameter(pack_w12(mk(inner, d), mk(inner, d), self.ipad))
        self.w3 = nn.Parameter(F.pad(mk(d, inner), (0, self.ipad - inner)))
        self._register_state_dict_hook(self._export_reference_keys)
        self._register_load_state_dict_pre_hook(self._import_reference_keys)

    @staticmethod
    def _export_reference_keys(module, state_dict, prefix, local_metadata):
        w12, w3 = state_dict.pop(prefix + "w12"), state_dict.pop(prefix + "w3")
        l1, l2 = unpack_w12(w12, module.inner)
        state_dict[prefix + "l1.weight"], state_dict[prefix + "l2.weight"] = l1.contiguous(), l2.contiguous()
        state_dict[prefix + "l3.weight"] = w3[:, :module.inner].contiguous()

    def _import_reference_keys(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        names = [prefix + n for n in ("l1.weight", "l2.weight", "l3.weight")]
        have = [n in state_dict for n in names]
        d = self.w3.shape[0]
        for n, ok, shape in zip(names, have, ((self.inner, d), (self.inner, d), (d, self.inner))):
            if not ok:
                missing_keys.append(n)
            elif tuple(state_dict[n].shape) != shape:
                error_msgs.append(f"size mismatch for {n}: copying a param with shape {tuple(state_dict[n].shape)} from checkpoint, the shape in current model is {shape}.")
                have = [False] * 3
        if have[0] and have[1]:
            state_dict[prefix + "w12"] = pack_w12(state_dict[names[0]], state_dict[names[1]], self.ipad)
        else:
            state_dict[prefix + "w12"] = self.w12.data         # reported above under the reference's own key names
        state_dict[prefix + "w3"] = F.pad(state_dict[names[2]], (0, self.ipad - self.inner)) if have[2] else self.w3.data
        for n in names:
            state_dict.pop(n, None)


class _HyenaFilter(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        d, s, k = cfg.hidden_size, cfg.state_size, cfg.short_filter_length
        if k != 3 or s != 8:
            raise NotImplementedError("kernels are specialised for short_filter_length=3, state_size=8 (the Evo configs)")
        if (cfg.get("hyena_filter_groups") or 1) != 1:
            raise NotImplementedError("hyena_filter_groups != 1")
        self.short_filter_weight = nn.Parameter(torch.randn(3 * d, 1, k) * 0.3)
        self.short_filter_bias = nn.Parameter(torch.randn(3 * d) * 0.1)
        self.D = nn.Parameter(torch.zeros(d))
        mag = 0.5 + 0.45 * torch.rand(d, s, 1)
        ang = (torch.rand(d, s, 1) * 2 - 1) * math.pi
        self.poles = nn.Parameter(torch.stack([mag * torch.cos(ang), mag * torch.sin(ang)], dim=-1))
        self.residues = nn.Parameter(torch.randn(d, s, 1, 2) * 0.3)

    def ptrs(self):
        """Device addresses of the five filter tensors under the field names every Hyena entry point takes, in its order."""
        return {"fir_w": self.short_filter_weight.data_ptr(), "fir_b": self.short_filter_bias.data_ptr(), "Dskip": self.D.data_ptr(),
                "poles": self.poles.data_ptr(), "residues": self.residues.data_ptr()}


class _Rotary(nn.Module):
    """Carrier of `inv_freq`.  flash_attn registers it as a NON-persistent buffer (layers/rotary.py:366); stripedhyena re-registers it
    as a persistent one, so its checkpoints carry `...rotary_emb.inv_freq`.  That second fact is recalled, not verified here (SURVEY.md
    A.7), so loading accepts both: a checkpoint value is used when present, the constructor's analytic value when absent -- what the
    reference ends up with in either world."""

    def __init__(self, head_dim, base):
        super().__init__()
        self.head_dim, self.base = head_dim, base
        self.register_buffer("inv_freq", self.analytic())

    def analytic(self, device=None):
        return 1.0 / (self.base ** (torch.arange(0, self.head_dim, 2, dtype=torch.float32, device=device) / self.head_dim))

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        if prefix + "inv_freq" not in state_dict:
            state_dict = {**state_dict, prefix + "inv_freq": self.inv_freq if self.inv_freq.device.type != "meta" else self.analytic()}
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)


class _MHA(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        d = cfg.hidden_size
        if (cfg.get("proj_groups") or 1) != 1:
            raise NotImplementedError("proj_groups != 1 (GQA) is not an Evo configuration")
        self.Wqkv = _Linear(d, 3 * d, bool(cfg.get("qkv_proj_bias", True)))
        self.out_proj = _Linear(d, d, bool(cfg.get("mha_out_proj_bias", True)))
        self.rotary_emb = _Rotary(d // cfg.num_attention_heads, cfg.get("rotary_emb_base") or 10000)


class _HyenaBlock(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        d = cfg.hidden_size
        self.pre_norm, self.post_norm = _Scale(d), _Scale(d)
        self.filter = _HyenaFilter(cfg)
        self.projections = _Linear(d, 3 * d, True)
        self.out_filter_dense = _Linear(d, d, True)
        self.mlp = _GatedMLP(cfg)


class _AttentionBlock(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        d = cfg.hidden_size
        self.pre_norm, self.post_norm = _Scale(d), _Scale(d)
        self.inner_mha_cls = _MHA(cfg)
        self.mlp = _GatedMLP(cfg)


class _Embedding(nn.Module):
    def __init__(self, vocab, dim):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(vocab, dim) * (2.5 / math.sqrt(dim)))


# ----------------------------------------------------------------------------- the model
class StripedHyena(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        d = config.hidden_size
        self.embedding_layer = _Embedding(config.vocab_size, d)
        self.norm = _Scale(d) if config.get("final_norm", True) else None
        self.unembed = self.embedding_layer if config.tie_embeddings else _Embedding(config.vocab_size, d)
        attn = set(config.attn_layer_idxs or [])
        self.blocks = nn.ModuleList(
            _AttentionBlock(config) if i in attn else _HyenaBlock(config) for i in range(config.num_layers))
        self._attn_idxs = attn
        self._packed = None
        self._rope = None
        self.decode_graph = os.environ.get("EVO_B200_DECODE_GRAPH", "1") != "0"
        # tile-major weight copies for decode (GEMM variant 3): bit-identical to variant 2; off unless measured faster
        self.decode_tiled = os.environ.get("EVO_B200_DECODE_TILED", "0") != "0"
        # decode-step GEMMs: stream-K weight-streaming kernel (csrc/gemm_smallm.cu) for batch <= 64; "0" = the 128x64 tiles
        self.decode_streamk = os.environ.get("EVO_B200_DECODE_STREAMK", "1") != "0"
        # programmatic dependent launch inside a decode step (evo_set_pdl): 0 off, 1 every kernel, 2 weight-streaming GEMMs only
        self.decode_pdl = int(os.environ.get("EVO_B200_DECODE_PDL", "4"))
        self._smallm_ws = None
        # FP8 weights (quantize_fp8): the linear layers' parameters hold W' = q 2^e and the decode-step GEMMs stream (q, e), a
        # cache built from W' like _packed.  _fp8_decode_bf16 runs those GEMMs on W' with the bf16 kernel instead (the tests'
        # comparator: the two are bit-identical)
        self._fp8_mode = False
        self._fp8_decode_bf16 = False
        self._fp8 = None
        # compact FP8 weights (quantize_fp8(compact=True)): the linear layers' (q, e) are the weights, held as non-persistent
        # buffers <attr>_q / <attr>_exp beside an empty parameter; linear_weight() rebuilds W' into _w_scratch before each GEMM
        self._fp8_compact = False
        self._w_scratch = None
        self._tiled = None   # tile-major weight copies for the weight-streaming decode GEMMs
        self._decode = None  # cached CUDA graph of one decode step (see _decode_forward)
        self._loop = None    # cached CUDA graph of one step of the on-device generation loop (see decode_loop)
        self._prof = None   # set to a list to record (kind, algorithmic work, start event, end event) per kernel call

    # ---- reference API ------------------------------------------------------------------
    def to_bfloat16_except_poles_residues(self):
        for name, p in self.named_parameters():
            if "poles" not in name and "residues" not in name:
                p.data = p.data.to(torch.bfloat16)
        self._packed = None
        return self

    def initialize_inference_params(self):
        return {
            "mha": InferenceParams(max_seqlen=self.config.get("max_seqlen") or 8192,
                                   max_batch_size=self.config.get("max_batch_size") or 1, seqlen_offset=0),
            "hyena": RecurrentInferenceParams(fir_filter_length=self.config.short_filter_length,
                                              state_dim=self.config.state_size, seqlen_offset=0),
        }

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        if self._fp8_compact:
            return self._load_compact(state_dict, strict, **kw)
        out = super().load_state_dict(state_dict, strict=strict, **kw)
        self._invalidate()
        if self._fp8_mode:
            self._round_fp8()       # an FP8 model stays one: loaded weights are rounded onto the grid at once
        return out

    def state_dict(self, *args, **kw):
        """The reference's keys and layouts.  A compact FP8 model exports W' (the bits a non-compact FP8 model holds), rebuilt
        on the model's device from (q, e): the call allocates the bf16 size of the linear weights, which the returned tensors
        then hold."""
        if not self._fp8_compact:
            return super().state_dict(*args, **kw)
        with self._materialized():
            return super().state_dict(*args, **kw)

    def _apply(self, fn, *a, **kw):
        out = super()._apply(fn, *a, **kw)
        self._invalidate()
        return out

    def _invalidate(self):
        """Drop everything built from the parameters or buffers (rotary tables from inv_freq) and the steps that captured it."""
        self._packed = self._rope = self._tiled = self._decode = self._loop = self._fp8 = self._w_scratch = None

    # ---- FP8 weights ----------------------------------------------------------------------------
    def _slot(self, i, name):
        """(owning module, attribute, gate layout) of block i's linear layer `name`: "in" (Wqkv / projections), "out" (out_proj /
        out_filter_dense), "w12" (the packed l1 / l2) or "w3"."""
        blk = self.blocks[i]
        if name in ("w12", "w3"):
            return blk.mlp, name, name == "w12"
        if i in self._attn_idxs:
            return (blk.inner_mha_cls.Wqkv if name == "in" else blk.inner_mha_cls.out_proj), "weight", False
        return (blk.projections if name == "in" else blk.out_filter_dense), "weight", False

    def _fp8_slots(self):
        """(block, name, owning module, attribute, gate layout) of every linear layer whose weight is held on the FP8 grid."""
        for i in range(len(self.blocks)):
            for name in ("in", "out", "w12", "w3"):
                yield (i, name) + self._slot(i, name)

    def _fp8_weights(self):
        """(block, name, parameter, gate layout) of every linear layer whose weight is held on the FP8 grid."""
        for i, name, mod, attr, gate in self._fp8_slots():
            yield i, name, getattr(mod, attr), gate

    @staticmethod
    def _compact_qe(mod, attr):
        """The (q, e) buffers a compact FP8 model holds for mod.<attr>."""
        return getattr(mod, attr + "_q"), getattr(mod, attr + "_exp")

    def _dequant(self, q, e, gate, out):
        """evo_fp8_dequant_rows: W' = q 2^e into out (N, K) bf16 on the current stream."""
        N, K = e.numel(), q.numel() // e.numel()
        self._record(f"fp8_dequant/{N}x{K}", 0.0, lambda: check(_lib.lib().evo_fp8_dequant_rows(
            ptr(q), ptr(e), N, K, EPI_GELU_GATE if gate else EPI_NONE, ptr(out), self._stream()), "evo_fp8_dequant_rows"))
        return out

    def linear_weight(self, i, name):
        """W' of block i's linear layer `name` ("in", "out", "w12" or "w3"; see _slot) as the GEMMs read it: (N, K) bf16 row-major,
        w12 in its packed order.  A bf16 or FP8 model returns the parameter.  A compact FP8 model rebuilds W' from (q, e) into
        one scratch buffer on the current stream and returns that buffer: it holds this matrix until the next call, so the GEMM
        that reads it must be the next kernel to touch it on the same stream."""
        mod, attr, gate = self._slot(i, name)
        if not self._fp8_compact:
            return getattr(mod, attr)
        q, e = self._compact_qe(mod, attr)
        if self._w_scratch is None:
            n = max(self._compact_qe(m, a)[0].numel() for _, _, m, a, _ in self._fp8_slots())
            self._w_scratch = torch.empty(n, dtype=torch.bfloat16, device=q.device)
        return self._dequant(q, e, gate, self._w_scratch[:q.numel()].view(e.numel(), -1))

    def _hold_compact(self, mod, attr, q, e):
        """Keep (q, e) as mod.<attr>'s weights and free its bf16 storage (the parameter stays, empty, under its key)."""
        mod.register_buffer(attr + "_q", q, persistent=False)
        mod.register_buffer(attr + "_exp", e, persistent=False)
        getattr(mod, attr).data = torch.empty(0, dtype=torch.bfloat16, device=q.device)

    @contextlib.contextmanager
    def _materialized(self):
        """A compact model whose linear parameters hold W' (new tensors, rebuilt from (q, e)) inside the block, empty again after."""
        slots = list(self._fp8_slots())
        if self.embedding_layer.weight.device.type != "cuda":
            raise _lib.EvoError("a compact FP8 model rebuilds its weights on CUDA (sm_90a): move it with .to('cuda:N') first")
        try:
            with torch.no_grad(), torch.cuda.device(self.embedding_layer.weight.device):
                for _, _, mod, attr, gate in slots:
                    q, e = self._compact_qe(mod, attr)
                    getattr(mod, attr).data = self._dequant(q, e, gate, torch.empty(e.numel(), q.numel() // e.numel(), dtype=torch.bfloat16,
                                                                                    device=q.device))
            yield
        finally:
            for _, _, mod, attr, _ in slots:
                getattr(mod, attr).data = torch.empty(0, dtype=torch.bfloat16, device=self._compact_qe(mod, attr)[0].device)

    def _load_compact(self, state_dict, strict, **kw):
        """load_state_dict into a compact FP8 model: a non-finite linear weight is refused before anything changes; otherwise
        the parameters hold W' for the load (a key the load does not fill keeps its value), and what is loaded is rounded and
        kept as (q, e) again.  Peak: the bf16 size of the linear weights."""
        names = {id(m): n for n, m in self.named_modules()}
        for _, _, mod, attr, _ in self._fp8_slots():
            p = names[id(mod)]
            for k in ([f"{p}.l1.weight", f"{p}.l2.weight"] if attr == "w12" else [f"{p}.l3.weight"] if attr == "w3" else [f"{p}.weight"]):
                v = state_dict.get(k)
                if torch.is_tensor(v) and v.is_floating_point() and not bool(torch.isfinite(v).all()):
                    raise _lib.EvoError(f"load_state_dict: {k} has a weight that is not finite; the model is unchanged")
        with self._materialized():
            out = super().load_state_dict(state_dict, strict=strict, **kw)
            self._round_fp8(compact=True)
        self._invalidate()
        return out

    def _quantize_rows(self, w, gate):
        """evo_fp8_quantize_rows on one parameter: rounds it in place to W' and returns (q in the decode layout, e)."""
        lib = _lib.lib()
        N, K = w.shape
        epi = EPI_GELU_GATE if gate else EPI_NONE
        nbytes = lib.evo_fp8_weight_bytes(N, K, epi)
        if nbytes == 0:
            raise _lib.EvoError(lib.evo_last_error().decode())
        q = torch.empty(nbytes, dtype=torch.uint8, device=w.device)
        e = torch.empty(N, dtype=torch.int8, device=w.device)
        status = torch.zeros(1, dtype=torch.int32, device=w.device)
        check(lib.evo_fp8_quantize_rows(ptr(w), N, K, epi, ptr(q), ptr(e), ptr(status), self._stream()), "evo_fp8_quantize_rows")
        if int(status.item()) != 0:
            raise _lib.EvoError("evo_fp8_quantize_rows: a weight is not finite; the matrix was left unchanged")
        return q, e

    def _round_fp8(self, compact=False):
        """Round every linear weight in place to W'; compact: then keep its (q, e) instead of W' (_hold_compact)."""
        with torch.no_grad():
            ws = list(self._fp8_slots())
            for _, _, mod, attr, _ in ws:
                w = getattr(mod, attr)
                if w.device.type != "cuda" or w.dtype != torch.bfloat16:
                    raise _lib.EvoError("quantize_fp8 runs on CUDA (sm_90a) with bf16 weights: move the model with .to('cuda:N') and call "
                                        "to_bfloat16_except_poles_residues() first")
            # refuse before anything is rounded, so that a refused model keeps every parameter
            for i, name, mod, attr, _ in ws:
                if not bool(torch.isfinite(getattr(mod, attr)).all()):
                    raise _lib.EvoError(f"quantize_fp8: block {i} {name} has a weight that is not finite; the model is unchanged")
            with torch.cuda.device(getattr(ws[0][2], ws[0][3]).device):
                for _, _, mod, attr, gate in ws:
                    q, e = self._quantize_rows(getattr(mod, attr).data, gate)
                    if compact:
                        self._hold_compact(mod, attr, q, e)
        self._invalidate()

    def quantize_fp8(self, compact: bool = False):
        """Make this an FP8 model: round the weight of every linear layer of every block (Wqkv / projections, out_proj /
        out_filter_dense, the packed w12 and w3) onto an E4M3 grid with one power-of-two scale per output row, in place (see
        fp8_round_rows).  Every path runs unchanged on the rounded bf16 weights W'; the decode-step GEMMs (batch <= 64) stream
        the one-byte E4M3 copies instead, bit-identical to the bf16 kernel on W'.  The embedding stays bf16.  Idempotent;
        state_dict() exports W' (an ordinary bf16 checkpoint), and load_state_dict() into an FP8 model rounds what it loads.

        compact=True: keep only the one-byte weights q and the row exponents e of those layers (about half the bf16 bytes, a
        third of the non-compact FP8 model's) and free their bf16 storage.  Since W' = q 2^e exactly, every path that reads W'
        gets it rebuilt bit for bit into one scratch buffer (linear_weight, sized for the largest matrix) just before its GEMM:
        the outputs are the non-compact FP8 model's on every path.  A compact model stays compact (quantize_fp8 leaves it
        unchanged, load_state_dict rounds what it loads)."""
        if self._fp8_compact:
            return self
        self._round_fp8(compact=compact)
        self._fp8_mode, self._fp8_compact = True, compact
        return self

    def _fp8_active(self):
        return self._fp8_mode and not self._fp8_decode_bf16

    def _ensure_fp8(self):
        """The decode copies {block: {name: (q, e)}} of W' (quantizing W' again leaves it unchanged); a compact model's own."""
        if self._fp8 is None:
            cache = {}
            with torch.no_grad(), torch.cuda.device(self.embedding_layer.weight.device):
                for i, name, mod, attr, gate in self._fp8_slots():
                    cache.setdefault(i, {})[name] = (self._compact_qe(mod, attr) if self._fp8_compact
                                                     else self._quantize_rows(getattr(mod, attr).data, gate))
            cache["ptrs"] = tuple(t.data_ptr() for i in range(len(self.blocks)) for q in cache[i].values() for t in q)
            self._fp8 = cache
        return self._fp8

    # ---- weight packing (once per load / move) ---------------------------------------------
    def _ensure_packed(self):
        if self._packed is not None:
            return self._packed
        dev = self.embedding_layer.weight.device
        if dev.type != "cuda":
            raise _lib.EvoError("evo_b200 runs on CUDA (sm_90a) only: move the model with .to('cuda:N'); there is no CPU path")
        for name, p in self.named_parameters():
            want = torch.float32 if ("poles" in name or "residues" in name) else torch.bfloat16
            if p.dtype != want:
                raise _lib.EvoError(f"parameter {name} is {p.dtype}; call to_bfloat16_except_poles_residues() (evo/models.py:148)")
            if p.device != dev:
                raise _lib.EvoError(f"parameter {name} is on {p.device}, expected {dev}")
        if self._fp8_compact:       # the linear parameters are empty: their (q, e) buffers are the weights
            for i, name, mod, attr, _ in self._fp8_slots():
                q, e = self._compact_qe(mod, attr)
                if q.device != dev or e.device != dev or q.dtype != torch.uint8 or e.dtype != torch.int8:
                    raise _lib.EvoError(f"block {i} {name}: FP8 weights {q.dtype} / {e.dtype} on {q.device}, expected uint8 / int8 on {dev}")
        packed = {}
        for i, blk in enumerate(self.blocks):
            # the MLP parameters already live in the GEMM layouts (see _GatedMLP): nothing is copied here; linear_weight reads them
            packed[i] = {"ipad": blk.mlp.ipad}
        hd = self.config.hidden_size // self.config.num_attention_heads
        base = self.config.get("rotary_emb_base") or 10000
        # flash_attn keeps the checkpoint's inv_freq buffer when it is fp32 and recomputes it in fp32 otherwise
        # (layers/rotary.py:386-401); one table per model: every attention block must then agree
        analytic = (1.0 / (base ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd))).to(dev)
        bufs = [self.blocks[i].inner_mha_cls.rotary_emb.inv_freq for i in sorted(self._attn_idxs)]
        if bufs and bufs[0].dtype == torch.float32:
            for b_ in bufs[1:]:
                if b_.dtype != torch.float32 or not torch.equal(b_, bufs[0]):
                    raise _lib.EvoError("attention blocks carry different rotary inv_freq buffers; one rope table per model is supported")
            packed["inv_freq"] = bufs[0].detach().to(dev).contiguous()
        else:
            packed["inv_freq"] = analytic
        self._packed = packed
        return packed

    # ---- thin wrappers over the C ABI ------------------------------------------------------------
    @staticmethod
    def _stream():
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def _record(self, kind, work, launch):
        """Run `launch()`; when profiling is on, bracket it with CUDA events on the launch stream."""
        if self._prof is None:
            return launch()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        launch()
        e1.record()
        self._prof.append((kind, work, e0, e1))

    def _gemm(self, a, w, out, M, N, K, epi, bias=None, resid=None, ldc=None, variant=0, rope=None, peers=None):
        """rope = (cos_ptr, sin_ptr, tokens_per_sequence, rotated_columns) for EPI_BIAS_ROPE;
        peers = (ctypes array of peer pointers, n, period, inner, row0): peer-scattered output (see evo_gemm_params), out may be None."""
        p = GemmParams(A=a.data_ptr(), lda=K, W=w.data_ptr(), C=out.data_ptr() if out is not None else None, ldc=ldc or N,
                       bias=bias.data_ptr() if bias is not None else None,
                       residual=resid.data_ptr() if resid is not None else None, ldr=ldc or N,
                       M=M, N=N, K=K, epilogue=epi, variant=variant)
        if rope is not None:
            p.rope_cos, p.rope_sin, p.rope_L, p.rope_cols = rope
        if peers is not None:
            arr, n, period, inner, row0 = peers
            p.c_peers, p.n_c_peers, p.peer_period, p.peer_inner, p.peer_row0 = C.cast(arr, C.c_void_p), n, period, inner, row0
        self._record(f"gemm/{N}x{K}/e{epi}/v{variant}", 2.0 * M * N * K, lambda: check(_lib.lib().evo_gemm(C.byref(p), self._stream()), "evo_gemm"))

    def _gemm_smallm(self, a, w, out, M, N, K, epi, bias=None, resid=None, fp8=None):
        """Decode-step linear layer (M <= 64): stream-K weight-streaming kernel, gate epilogue fused.  fp8 = (q, e) of W
        (_ensure_fp8): the FP8-weight form streams those instead of w."""
        lib = _lib.lib()
        need = lib.evo_gemm_smallm_workspace(M, N, K, epi)
        ws = self._smallm_ws
        if ws is None or ws.numel() < need or ws.device != a.device:
            self._decode = None      # a captured decode graph holds the old workspace address
            ws = self._smallm_ws = torch.zeros(max(need, lib.evo_gemm_smallm_workspace(M, 256, 64, EPI_GELU_GATE)),
                                               dtype=torch.uint8, device=a.device)
        n_out = N // 2 if epi == EPI_GELU_GATE else N
        p = GemmSmallMParams(A=a.data_ptr(), lda=K, W=(w if fp8 is None else fp8[0]).data_ptr(), C=out.data_ptr(), ldc=n_out,
                             bias=bias.data_ptr() if bias is not None else None,
                             residual=resid.data_ptr() if resid is not None else None, ldr=n_out,
                             M=M, N=N, K=K, epilogue=epi, workspace=ws.data_ptr(), workspace_bytes=ws.numel())
        if fp8 is not None:
            p8 = _lib.GemmSmallMFp8Params(base=p, W_exp=fp8[1].data_ptr())
            self._record(f"gemm/{N}x{K}/e{epi}/streamk_fp8", 2.0 * M * N * K,
                         lambda: check(lib.evo_gemm_smallm_fp8(C.byref(p8), self._stream()), "evo_gemm_smallm_fp8"))
            return
        self._record(f"gemm/{N}x{K}/e{epi}/streamk", 2.0 * M * N * K, lambda: check(lib.evo_gemm_smallm(C.byref(p), self._stream()), "evo_gemm_smallm"))

    def _rmsnorm(self, x, scale, out, rows):
        self._record("rmsnorm", 4.0 * rows * self.config.hidden_size, lambda: check(_lib.lib().evo_rmsnorm(
            ptr(x), ptr(scale), ptr(out), rows, self.config.hidden_size, float(self.config.eps), self._stream()), "evo_rmsnorm"))

    def _rope_tables(self, n_pos, dev):
        if self._rope is None or self._rope[0].shape[0] < n_pos:
            hd2 = self.config.hidden_size // self.config.num_attention_heads // 2
            scaling = float(self.config.get("rotary_emb_scaling_factor") or 1.0) if self.config.get("use_interpolated_rotary_pos_emb") else 1.0
            n = max(n_pos, 2048)
            cos = torch.empty(n, hd2, dtype=torch.bfloat16, device=dev)
            sin = torch.empty_like(cos)
            check(_lib.lib().evo_rope_tables(ptr(cos), ptr(sin), ptr(self._packed["inv_freq"]), 0, n, hd2, scaling, self._stream()), "evo_rope_tables")
            self._rope = (cos, sin)
            self._decode = None      # a captured decode graph holds the old tables' addresses
        return self._rope

    def _mlp_residual(self, i, blk, u, M):
        """out = l3(gelu(l1 n) * l2 n) + u with n = post_norm(u); returns a new (M, D) tensor."""
        d = self.config.hidden_size
        pk = self._packed[i]
        xn = torch.empty_like(u)
        self._rmsnorm(u, blk.post_norm.scale, xn, M)
        g = torch.empty(M, pk["ipad"], dtype=torch.bfloat16, device=u.device)
        self._gemm(xn, self.linear_weight(i, "w12"), g, M, 2 * pk["ipad"], d, EPI_GELU_GATE, ldc=pk["ipad"])
        out = xn  # reuse
        self._gemm(g, self.linear_weight(i, "w3"), out, M, d, pk["ipad"], EPI_RESID, resid=u)
        return out

    def _launch_ws(self, kind, work, what, size, fn, p, *args):
        """_record one launch of fn(&p, *args, workspace, bytes, stream) on a new workspace of size(&p, *args) bytes (at
        least one byte is allocated, so its address is never NULL).  Returns (workspace, bytes) for a launch that reuses it."""
        n = size(C.byref(p), *args)
        ws = torch.empty(max(n, 1), dtype=torch.uint8, device=self.embedding_layer.weight.device)
        self._record(kind, work, lambda: check(fn(C.byref(p), *args, ptr(ws), n, self._stream()), what))
        return ws, n

    def _hyena_state_out(self, p, n, dev):
        """n new end states as the outputs of the scan p: (n, D, S, 2) fp32 modal states, (n, 3D, 2) bf16 FIR history."""
        d = self.config.hidden_size
        st = torch.empty(n, d, self.config.state_size, 2, dtype=torch.float32, device=dev)
        fs = torch.empty(n, 3 * d, 2, dtype=torch.bfloat16, device=dev)
        p.state_out, p.fir_state_out = st.data_ptr(), fs.data_ptr()
        return st, fs

    @staticmethod
    def _contiguous_state(hy, i):
        """Layer i's Hyena states in `hy`, made contiguous in place (a step reads and writes them by address): (fir, state)."""
        st = hy.state_dict[i] = hy.state_dict[i].contiguous()
        fs = hy.fir_state_dict[i] = hy.fir_state_dict[i].contiguous()
        return fs, st

    def _hyena_block(self, i, blk, u, B, L, ip: Optional[RecurrentInferenceParams], varlen=None):
        cfg = self.config
        d, H = cfg.hidden_size, cfg.num_attention_heads
        M = B * L
        dev = u.device
        f = blk.filter
        xn = torch.empty_like(u)
        self._rmsnorm(u, blk.pre_norm.scale, xn, M)
        z = torch.empty(M, 3 * d, dtype=torch.bfloat16, device=dev)
        self._gemm(xn, self.linear_weight(i, "in"), z, M, 3 * d, d, EPI_BIAS, bias=blk.projections.bias)
        y = xn  # (M, D) buffer reuse
        lib = _lib.lib()
        have_state = ip is not None and i in ip.fir_state_dict
        if varlen is not None:
            self._hyena_varlen(i, f, z, y, varlen, ip)
        elif have_state and L == 1:
            fs, st = self._contiguous_state(ip, i)
            check(lib.evo_hyena_step(ptr(z), ptr(y), ptr(fs), ptr(torch.view_as_real(st)), *map(C.c_void_p, f.ptrs().values()),
                                     B, d, cfg.state_size, H, self._stream()), "evo_hyena_step")
        else:
            hp = HyenaParams(z=z.data_ptr(), y=y.data_ptr(), **f.ptrs(), B=B, L=L, D=d, S=cfg.state_size, nheads=H, force_segments=0, state_only=0)
            if have_state:  # continued prefill: history = stored states
                halo = ip.fir_state_dict[i].permute(0, 2, 1).contiguous()
                sin_ = torch.view_as_real(ip.state_dict[i].contiguous()).contiguous()
                hp.halo, hp.state_in = halo.data_ptr(), sin_.data_ptr()
            if ip is not None:
                st_out, fs_out = self._hyena_state_out(hp, B, dev)
            self._launch_ws("hyena", 8.0 * B * L * d, "evo_hyena_fwd", lib.evo_hyena_fwd_workspace, lib.evo_hyena_fwd, hp)
            if ip is not None:
                ip.state_dict[i], ip.fir_state_dict[i] = torch.view_as_complex(st_out), fs_out
        u2 = torch.empty_like(u)
        self._gemm(y, self.linear_weight(i, "out"), u2, M, d, d, EPI_BIAS_RESID, bias=blk.out_filter_dense.bias, resid=u)
        return self._mlp_residual(i, blk, u2, M)

    def _hyena_varlen(self, i, f, z, y, vl, ip):
        """Packed sequences: one scan over all T rows (evo_hyena_fwd_varlen); with `ip`, each sequence's end states become
        state_dict[i] (n, D, S) and fir_state_dict[i] (n, 3D, 2) as they are.  With vl.ckpt or vl.resume the checkpointed scan
        (evo_hyena_fwd_varlen_ckpt) runs instead.  vl.ckpt: store this layer's (n_ckpt, D, S, 2) state table and its
        (n_ckpt, 2, 3D) FIR history table -- z rows c - 2 and c - 1 of every checkpoint c, gathered as they are.
        vl.resume: start each sequence from its start_idx row of the tables prefill_checkpoints stored for this layer."""
        cfg, lib = self.config, _lib.lib()
        d, n = cfg.hidden_size, vl.n
        p = HyenaVarlenParams(z=z.data_ptr(), y=y.data_ptr(), **f.ptrs(), cu_seqlens=vl.cu.data_ptr(), n_seq=n, T=vl.T, max_seqlen=vl.max_len,
                              D=d, S=cfg.state_size, nheads=cfg.num_attention_heads, seg_len=0)
        if ip is not None:
            st_out, fs_out = self._hyena_state_out(p, n, z.device)
        what, size, fn = "evo_hyena_fwd_varlen", lib.evo_hyena_fwd_varlen_workspace, lib.evo_hyena_fwd_varlen
        ck, rs = vl.ckpt, vl.resume
        if ck is not None or rs is not None:
            p = HyenaVarlenCkptParams(base=p)
            what, size, fn = "evo_hyena_fwd_varlen_ckpt", lib.evo_hyena_fwd_varlen_ckpt_workspace, lib.evo_hyena_fwd_varlen_ckpt
        if ck is not None and ck.n > 0:
            st = torch.empty(ck.n, d, cfg.state_size, 2, dtype=torch.float32, device=z.device)
            p.ckpt_states, p.ckpt_base, p.ckpt_stride, p.n_ckpt = st.data_ptr(), ck.base.data_ptr(), ck.stride, ck.n
            ck.state[i] = st
            ck.halo[i] = z.index_select(0, ck.halo_rows).view(ck.n, 2, 3 * d)
        if rs is not None and rs.ckpts.n_ckpt > 0:
            src = rs.ckpts
            p.start_idx, p.state_table, p.halo_table, p.n_table = rs.start_idx.data_ptr(), src.state[i].data_ptr(), src.halo[i].data_ptr(), src.n_ckpt
        self._launch_ws("hyena", 8.0 * vl.T * d, what, size, fn, p)
        if ip is not None:
            ip.state_dict[i], ip.fir_state_dict[i] = torch.view_as_complex(st_out), fs_out

    def _rope_at(self, pos0, L, dev):
        """(cos, sin) addresses of the rotary tables' rows for positions pos0 .. pos0 + L - 1."""
        cos, sin = self._rope_tables(pos0 + L, dev)
        off = pos0 * cos.stride(0) * cos.element_size()
        return cos.data_ptr() + off, sin.data_ptr() + off

    def _rope_fused(self, mha):
        """Whether the Wqkv GEMM applies rotary in its epilogue (EVO_EPI_BIAS_ROPE: bias + rotary, head_dim 128), where
        flash_attn's MHA applies it (mha.py:635-648); otherwise a second pass over qkv does."""
        hd = self.config.hidden_size // self.config.num_attention_heads
        return mha.Wqkv.bias is not None and hd == 128

    def _qkv_rope(self, i, xn, mha, qkv, B, L, rope):
        """qkv (B*L, 3D) = Wqkv xn (+ bias) of block i, rotary on q and k from rope = (cos, sin) addresses of each sequence's L rows."""
        cfg, lib = self.config, _lib.lib()
        d, H = cfg.hidden_size, cfg.num_attention_heads
        M = B * L
        if self._rope_fused(mha):
            self._gemm(xn, self.linear_weight(i, "in"), qkv, M, 3 * d, d, EPI_BIAS_ROPE, bias=mha.Wqkv.bias, rope=(*rope, L, 2 * d))
        else:
            self._gemm(xn, self.linear_weight(i, "in"), qkv, M, 3 * d, d, EPI_BIAS if mha.Wqkv.bias is not None else EPI_NONE, bias=mha.Wqkv.bias)
            self._record("rotary", 8.0 * M * d, lambda: check(lib.evo_rotary_qk(ptr(qkv), C.c_void_p(rope[0]), C.c_void_p(rope[1]), B, L, H, d // H,
                                                                                self._stream()), "evo_rotary_qk"))

    def _out_proj(self, i, mha, ctx, u):
        """u + out_proj(ctx) of block i as a new (M, D) tensor."""
        d = self.config.hidden_size
        u2 = torch.empty_like(u)
        self._gemm(ctx, self.linear_weight(i, "out"), u2, u.shape[0], d, d, EPI_BIAS_RESID if mha.out_proj.bias is not None else EPI_RESID,
                   bias=mha.out_proj.bias, resid=u)
        return u2

    def _kv_cache(self, ip, i, rows):
        """Layer i's KV cache in `ip`, made on first use with `rows` rows (flash_attn/modules/mha.py:344-353; zeros instead of
        empty: quirk Q1)."""
        if i not in ip.key_value_memory_dict:
            H = self.config.num_attention_heads
            ip.key_value_memory_dict[i] = torch.zeros(rows, ip.max_seqlen, 2, H, self.config.hidden_size // H, dtype=torch.bfloat16,
                                                      device=self.embedding_layer.weight.device)
        return ip.key_value_memory_dict[i]

    def _attention_block(self, i, blk, u, B, L, ip: Optional[InferenceParams], varlen=None):
        cfg = self.config
        d, H = cfg.hidden_size, cfg.num_attention_heads
        hd = d // H
        M = B * L
        dev = u.device
        mha = blk.inner_mha_cls
        lib = _lib.lib()
        xn = torch.empty_like(u)
        self._rmsnorm(u, blk.pre_norm.scale, xn, M)
        qkv = torch.empty(M, 3 * d, dtype=torch.bfloat16, device=dev)
        off = int(ip.seqlen_offset) if ip is not None else 0
        # packed: the (T, 64) tables of each row's in-sequence position, read as one sequence of L = T rows
        rope = tuple(t.data_ptr() for t in varlen.rope) if varlen is not None else self._rope_at(off, L, dev)
        self._qkv_rope(i, xn, mha, qkv, B, L, rope)
        ctx = xn  # reuse
        if varlen is not None:
            self._attention_varlen(i, qkv, ctx, varlen, ip)
        else:
            ap = AttnParams(out=ctx.data_ptr(), B=B, Lq=L, H=H, hd=hd, q_pos0=off, softmax_scale=1.0 / math.sqrt(hd))
            ap.q, ap.q_tok_stride, ap.q_batch_stride = qkv.data_ptr(), 3 * d, L * 3 * d
            if ip is None:
                ap.k, ap.v = qkv.data_ptr() + d * 2, qkv.data_ptr() + 2 * d * 2
                ap.kv_tok_stride, ap.kv_batch_stride, ap.Lk = 3 * d, L * 3 * d, L
            else:
                cache = self._kv_cache(ip, i, ip.max_batch_size)
                if B > cache.shape[0] or off + L > cache.shape[1]:
                    raise _lib.EvoError(f"KV cache too small: batch {B} > {cache.shape[0]} or length {off + L} > {cache.shape[1]} (mha.py:366-367)")
                check(lib.evo_kv_append(ptr(qkv), ptr(cache), B, L, H, hd, off, cache.shape[1], self._stream()), "evo_kv_append")
                ap.k, ap.v = cache.data_ptr(), cache.data_ptr() + d * 2
                ap.kv_tok_stride, ap.kv_batch_stride, ap.Lk = 2 * d, cache.shape[1] * 2 * d, off + L
            causal_flops = 4.0 * B * H * hd * (L * (off + (L + 1) / 2.0))   # QK^T + PV over the visible (query, key) pairs
            self._launch_ws("attn", causal_flops, "evo_attn_fwd", lib.evo_attn_fwd_workspace, lib.evo_attn_fwd_ws, ap, ATTN_VARIANT)
        return self._mlp_residual(i, blk, self._out_proj(i, mha, ctx, u), M)

    def _attention_varlen(self, i, qkv, ctx, vl, ip):
        """Packed sequences: causal attention within each sequence (evo_attn_fwd_varlen) on the packed qkv rows; with `ip`,
        sequence b's k, v also go to rows [0, len_b) of batch row b of the layer's KV cache (evo_kv_append_varlen)."""
        cfg = self.config
        d, H = cfg.hidden_size, cfg.num_attention_heads
        hd = d // H
        lib = _lib.lib()
        cu, n, T, mx = vl.cu, vl.n, vl.T, vl.max_len
        if vl.ckpt is not None:         # the references' K,V, once per reference: the prefix every variant of it attends to
            cache = torch.empty(n, mx, 2, H, hd, dtype=torch.bfloat16, device=qkv.device)
            check(lib.evo_kv_append_varlen(ptr(qkv), ptr(cache), ptr(cu), n, T, mx, H, hd, mx, self._stream()), "evo_kv_append_varlen")
            vl.ckpt.kv[i] = cache
        if vl.resume is not None:
            rs = vl.resume
            cache = rs.ckpts.kv[i]
            ap = AttnVarlenPrefixParams(qkv=qkv.data_ptr(), out=ctx.data_ptr(), cu_seqlens=cu.data_ptr(), n_seq=n, T=T, max_seqlen=mx,
                                        cache=cache.data_ptr(), n_cache=cache.shape[0], cache_len=cache.shape[1],
                                        prefix_seq=rs.prefix_seq.data_ptr(), prefix_len=rs.prefix_len.data_ptr(),
                                        H=H, hd=hd, softmax_scale=1.0 / math.sqrt(hd))
            flops = 4.0 * H * hd * sum(L * (P + (L + 1) / 2.0) for L, P in zip(vl.lengths, rs.plen))
            self._record("attn", flops, lambda: check(lib.evo_attn_fwd_varlen_prefix(C.byref(ap), self._stream()), "evo_attn_fwd_varlen_prefix"))
            return
        if ip is not None:
            cache = self._kv_cache(ip, i, max(ip.max_batch_size, n))
            if n > cache.shape[0] or mx > cache.shape[1] or not cache.is_contiguous():
                raise _lib.EvoError(f"KV cache {tuple(cache.shape)} cannot hold {n} sequences of up to {mx} tokens")
            check(lib.evo_kv_append_varlen(ptr(qkv), ptr(cache), ptr(cu), n, T, mx, H, hd, cache.shape[1], self._stream()), "evo_kv_append_varlen")
        ap = AttnVarlenParams(q=qkv.data_ptr(), k=qkv.data_ptr() + d * 2, v=qkv.data_ptr() + 2 * d * 2, out=ctx.data_ptr(),
                              q_tok_stride=3 * d, kv_tok_stride=3 * d, cu_seqlens=cu.data_ptr(), n_seq=n, T=T, max_seqlen=mx,
                              H=H, hd=hd, softmax_scale=1.0 / math.sqrt(hd))
        causal_flops = 4.0 * H * hd * sum(L * (L + 1) / 2.0 for L in vl.lengths)
        self._record("attn", causal_flops, lambda: check(lib.evo_attn_fwd_varlen(C.byref(ap), self._stream()), "evo_attn_fwd_varlen"))

    # ---- forward ---------------------------------------------------------------------------------
    def forward(self, x, inference_params_dict=None, padding_mask=None):
        if padding_mask is not None:
            raise NotImplementedError("padding_mask is never passed by evo (evo/scoring.py:81); not implemented")
        if x.dim() != 2:
            raise ValueError("input ids must be (batch, length)")
        if x.dtype not in (torch.int32, torch.int64):
            raise TypeError("input ids must be int32 or int64")
        self._ensure_packed()
        dev = self.embedding_layer.weight.device
        if x.device != dev:
            raise _lib.EvoError(f"input ids on {x.device}, model on {dev}")
        x = x.contiguous()
        B, L = x.shape
        if L == 1 and inference_params_dict is not None and self._can_step(inference_params_dict, B):
            with torch.cuda.device(dev), torch.no_grad():
                return self._decode_forward(x, inference_params_dict), inference_params_dict
        with torch.cuda.device(dev), torch.no_grad():
            logits = self._logits(self._backbone(x, B, L, inference_params_dict))
        return logits.view(B, L, self.config.vocab_size), inference_params_dict

    def _embed(self, x):
        """(x.numel(), D) bf16 embedding rows of the token ids x."""
        M, d, V = x.numel(), self.config.hidden_size, self.config.vocab_size
        u = torch.empty(M, d, dtype=torch.bfloat16, device=x.device)
        check(_lib.lib().evo_embed(ptr(x), int(x.dtype == torch.int64), ptr(self.embedding_layer.weight), ptr(u), M, d, V, self._stream()), "evo_embed")
        return u

    def _final_norm(self, u):
        """The final norm of u (M, D) as a new tensor; u itself when the model has none."""
        if self.norm is None:
            return u
        xn = torch.empty_like(u)
        self._rmsnorm(u, self.norm.scale, xn, u.shape[0])
        return xn

    def _logits(self, u):
        """(M, V) bf16 logits of the final-norm output u (M, D)."""
        M, d, V = u.shape[0], self.config.hidden_size, self.config.vocab_size
        logits = torch.empty(M, V, dtype=torch.bfloat16, device=u.device)
        self._gemm(u, self.unembed.weight, logits, M, V, d, EPI_NONE)
        return logits

    def _backbone(self, x, B, L, inference_params_dict=None, varlen=None, *, taps=None, last_block=None):
        """embed -> all blocks -> final norm: the (B*L, D) bf16 input of the unembedding.  varlen (from _varlen): x is a packed
        (T,) batch run as B = 1, L = T; only the two token-mixing calls differ.
        taps: {block index or "final": fn}; fn(u) is called on that block's (M, D) output (a new tensor no later block writes)
        or on the final-norm output.  last_block: the deepest block to run.  With taps, the final norm runs only for a "final"
        tap; the defaults run every block and the final norm, as every other caller needs."""
        u = self._embed(x)
        for i, blk in enumerate(self.blocks):
            if last_block is not None and i > last_block:
                break
            if i in self._attn_idxs:
                ip = inference_params_dict["mha"] if inference_params_dict is not None else None
                u = self._attention_block(i, blk, u, B, L, ip, varlen)
            else:
                ip = inference_params_dict["hyena"] if inference_params_dict is not None else None
                u = self._hyena_block(i, blk, u, B, L, ip, varlen)
            if taps is not None and i in taps:
                taps[i](u)
        if taps is not None and "final" not in taps:
            return u
        u = self._final_norm(u)
        if taps is not None:
            taps["final"](u)
        return u

    def score_tokens(self, input_ids, want_logprobs=True, want_entropy=False):
        """Fused scoring head (SURVEY 8f-1): what evo/scoring.py computes from `model(input_ids)` -- log_softmax of the
        logits gathered at the NEXT token (logits_to_logprobs, :36-59) and the per-position entropy (:119-121) -- without
        the (B, L, 512) logits ever reaching HBM: the unembed GEMM's epilogue keeps max / sum-exp / sum-exp*logit / target
        logit per row (evo_unembed_score).  Returns (logprobs (B, L) fp32 or None, entropy (B, L) fp32 or None);
        logprobs[b, t] = log p(ids[b, t+1] | ids[b, :t+1]), 0 at the last position."""
        if input_ids.dim() != 2 or input_ids.dtype not in (torch.int32, torch.int64):
            raise TypeError("input ids must be (batch, length) int32/int64")
        self._ensure_packed()
        dev = self.embedding_layer.weight.device
        if input_ids.device != dev:
            raise _lib.EvoError(f"input ids on {input_ids.device}, model on {dev}")
        x = input_ids.contiguous()
        B, L = x.shape
        with torch.cuda.device(dev), torch.no_grad():
            u = self._backbone(x, B, L, None)
            targets = torch.full((B, L), -1, dtype=torch.long, device=dev)
            targets[:, :-1] = x[:, 1:]
            return self._score_head(u, targets, (B, L), want_logprobs, want_entropy)

    def _score_head(self, u, targets, shape, want_logprobs, want_entropy):
        """evo_unembed_score over the rows of u (the final-norm output): (logprobs, entropy) of `shape`, either None if unwanted."""
        d, V = self.config.hidden_size, self.config.vocab_size
        M, dev, lib = u.shape[0], u.device, _lib.lib()
        lp = torch.empty(shape, dtype=torch.float32, device=dev) if want_logprobs else None
        ent = torch.empty(shape, dtype=torch.float32, device=dev) if want_entropy else None
        n = lib.evo_unembed_score_workspace(M, V)
        ws = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        sp = _lib.ScoreParams(x=u.data_ptr(), W=self.unembed.weight.data_ptr(), targets=targets.data_ptr(), logprobs=lp.data_ptr() if lp is not None else None,
                              entropy=ent.data_ptr() if ent is not None else None, M=M, V=V, K=d, workspace=ws.data_ptr(), workspace_bytes=n)
        self._record(f"gemm/{V}x{d}/score", 2.0 * M * V * d, lambda: check(lib.evo_unembed_score(C.byref(sp), self._stream()), "evo_unembed_score"))
        return lp, ent

    # ---- packed variable-length sequences: n sequences end to end as one (T,) batch, no padding ----------------------
    def _varlen(self, ids, cu_seqlens, pos0=None):
        """Checks a packed call on the host before anything is launched and returns its _Pack: what its blocks need, with
        the (T, 64) rotary tables built once per forward and shared by every attention layer.  pos0: n host ints, sequence
        b's row t then sits at position pos0[b] + t (rows resumed behind a prefix)."""
        cfg = self.config
        d, H = cfg.hidden_size, cfg.num_attention_heads
        if d % H or d // H != 128 or d % 256:
            raise _lib.EvoError(f"packed sequences need head_dim 128 and hidden_size % 256 == 0 (hidden_size {d}, {H} heads)")
        if not torch.is_tensor(ids) or ids.dim() != 1 or ids.dtype not in (torch.int32, torch.int64):
            raise _lib.EvoError("packed ids must be a 1-D int32/int64 tensor")
        self._ensure_packed()
        dev = self.embedding_layer.weight.device
        if ids.device != dev:
            raise _lib.EvoError(f"input ids on {ids.device}, model on {dev}")
        T = ids.shape[0]
        lengths = packed_lengths(cu_seqlens, T)
        cu_host = list(accumulate(lengths, initial=0))
        vl = _Pack(cu=torch.tensor(cu_host, dtype=torch.int64).to(dev), cu_host=cu_host, n=len(lengths), T=T, max_len=max(lengths), lengths=lengths)
        if pos0 is not None and len(pos0) != len(lengths):
            raise _lib.EvoError(f"{len(pos0)} start positions for {len(lengths)} sequences")
        if self._attn_idxs:
            with torch.cuda.device(dev):
                first = vl.cu[:-1] if pos0 is None else vl.cu[:-1] - torch.tensor(pos0, dtype=torch.int64).to(dev)
                cos, sin = self._rope_tables(vl.max_len if pos0 is None else max(p + n for p, n in zip(pos0, lengths)), dev)
                pos = torch.arange(T, device=dev) - torch.repeat_interleave(first, torch.tensor(lengths, device=dev), output_size=T)
                vl.rope = (cos[pos].contiguous(), sin[pos].contiguous())
        return vl

    def _packed_pass(self, ids, vl, head=None, ipd=None, *, taps=None, last_block=None):
        """_backbone over the packed ids of vl on the model's device without autograd; returns head(u, x) of its output u and
        the contiguous ids x, run in the same scope (u itself without a head)."""
        with torch.cuda.device(ids.device), torch.no_grad():
            x = ids.contiguous()
            u = self._backbone(x, 1, vl.T, ipd, vl, taps=taps, last_block=last_block)
            return u if head is None else head(u, x)

    def _packed_score(self, u, x, vl, want_logprobs=True, want_entropy=False):
        """_score_head over the packed rows u of ids x: row r's target is the next token of its own sequence; the last row of
        each sequence has none (-1: logprob 0)."""
        targets = torch.empty(vl.T, dtype=torch.long, device=x.device)
        targets[:-1] = x[1:]
        targets[vl.cu[1:] - 1] = -1
        return self._score_head(u, targets, (vl.T,), want_logprobs, want_entropy)

    def forward_packed(self, ids, cu_seqlens):
        """Logits (T, V) bf16 of n sequences packed end to end: ids (T,), cu_seqlens n + 1 offsets (cu[0] = 0, cu[n] = T, no
        empty sequence).  Row r holds what `forward` gives at that token of its sequence alone; equal lengths give the bits of
        `forward` on the (n, L) batch.  One backbone pass over T rows: no padding, one GEMM of M = T per linear layer."""
        vl = self._varlen(ids, cu_seqlens)
        return self._packed_pass(ids, vl, lambda u, x: self._logits(u))

    def score_tokens_packed(self, ids, cu_seqlens, want_logprobs=True, want_entropy=False):
        """score_tokens for packed sequences: (logprobs (T,) fp32 or None, entropy (T,) fp32 or None).  The target of row r is
        the next token of the same sequence; the last row of each sequence has none (logprob 0)."""
        vl = self._varlen(ids, cu_seqlens)
        return self._packed_pass(ids, vl, lambda u, x: self._packed_score(u, x, vl, want_logprobs, want_entropy))

    # ---- embeddings: block outputs of a packed forward, pooled per sequence, stopping after the deepest block asked for ----
    def _pool(self, u, vl, skip_first, mode, out):
        """evo_pool_varlen: out (n, D) fp32 = the pooled rows of each packed sequence of u (T, D) bf16."""
        d, lib = self.config.hidden_size, _lib.lib()
        pp = _lib.PoolVarlenParams(x=u.data_ptr(), ldx=u.stride(0), cu_seqlens=vl.cu.data_ptr(), n_seq=vl.n, T=vl.T,
                                   max_seqlen=vl.max_len, D=d, skip_first=skip_first, mode=mode, out=out.data_ptr(), ldo=out.stride(0))
        self._launch_ws("pool", 2.0 * vl.T * d, "evo_pool_varlen", lib.evo_pool_varlen_workspace, lib.evo_pool_varlen, pp)

    def embed_packed(self, ids, cu_seqlens, layers=("final",), pool="mean", skip_bos=True):
        """Sequence embeddings of n packed sequences (ids (T,), cu_seqlens as forward_packed): {layer: tensor}, keyed by the
        layers as given (resolve_layers: block indices, negative ones counted from the end, or "final" = the final-norm output).
        pool "mean" / "max" / "last": (n, D) fp32 per layer, over each sequence's rows without its first (the BOS) when
        skip_bos; pool None: the (T, D) bf16 rows of the layer, every row.  Only the blocks up to the deepest layer asked for
        run; the final norm runs only for "final", the unembedding never.  Row r holds what the full forward computes at that
        block for that row.  Bad arguments raise EvoError before anything is launched."""
        want = resolve_layers(layers, len(self.blocks))
        if pool is not None and pool not in POOL_MODES:
            raise _lib.EvoError(f"unknown pool {pool!r}: one of {sorted(POOL_MODES)} or None")
        skip = int(bool(skip_bos)) if pool is not None else 0
        if skip and torch.is_tensor(ids) and ids.dim() == 1 and min(packed_lengths(cu_seqlens, ids.shape[0])) <= skip:
            raise _lib.EvoError("a sequence keeps no row to pool: every sequence needs a token after its BOS")
        vl = self._varlen(ids, cu_seqlens)
        d, dev = self.config.hidden_size, ids.device
        blocks = set(want.values())
        got = {}

        def tap(key):
            def keep(u):
                if pool is None:
                    got[key] = u
                else:
                    got[key] = torch.empty(vl.n, d, dtype=torch.float32, device=dev)
                    self._pool(u, vl, skip, POOL_MODES[pool], got[key])
            return keep
        self._packed_pass(ids, vl, taps={b: tap(b) for b in blocks},
                          last_block=len(self.blocks) - 1 if "final" in blocks else max(blocks))
        return {k: got[b] for k, b in want.items()}

    # ---- variant scoring: a reference's state at every stride-th row, and packed passes resumed from those states --------
    def prefill_checkpoints(self, ids, cu_seqlens, stride):
        """One packed forward over n references (score_tokens_packed's path) that also keeps their state every `stride` rows.
        Checkpoint k of reference b is the model state after its first c = k * stride tokens (k >= 1, c < its length): per
        Hyena layer the modal state and the FIR history (z rows c - 2, c - 1), stored at table row base[b] + k - 1; per
        attention layer the reference's K,V, once, in an (n, longest, 2, H, 128) cache.  Returns a PrefixCheckpoints holding
        them with the references' per-row logprobs (T,) fp32 (row r: the next token of its reference; 0 at each end)."""
        if isinstance(stride, bool) or not isinstance(stride, int) or stride <= 0 or stride % 128:
            raise _lib.EvoError(f"checkpoint stride must be a positive multiple of 128, got {stride!r}")
        vl = self._varlen(ids, cu_seqlens)
        dev = ids.device
        counts = [(n - 1) // stride for n in vl.lengths]
        base = list(accumulate(counts, initial=0))
        rows = [vl.cu_host[b] + k * stride + dr for b, c in enumerate(counts) for k in range(1, c + 1) for dr in (-2, -1)]
        ck = vl.ckpt = _Capture(n=base[-1], stride=stride, base=torch.tensor(base[:-1], dtype=torch.int64, device=dev),
                                halo_rows=torch.tensor(rows, dtype=torch.int64, device=dev))
        lp, _ = self._packed_pass(ids, vl, lambda u, x: self._packed_score(u, x, vl))
        return PrefixCheckpoints(logprobs=lp, lengths=vl.lengths, cu=vl.cu_host, stride=stride, base=base, state=ck.state,
                                 halo=ck.halo, kv=ck.kv)

    def score_tokens_resumed(self, ckpts, ids, cu_seqlens, start_idx, prefix_seq, prefix_len):
        """Per-row logprobs (T,) fp32 of n packed sequences, each resumed behind a prefix of a reference of `ckpts`
        (prefill_checkpoints): sequence b holds the tokens at positions [prefix_len[b], prefix_len[b] + len_b) of a sequence
        whose first prefix_len[b] tokens are those of reference prefix_seq[b].  Its Hyena layers start from checkpoint row
        start_idx[b] (-1 = from zero: prefix_len[b] must then be 0), its attention layers attend the reference's cached K,V
        rows [0, prefix_len[b]) before its own; row t's target is the sequence's next token (0 at its last row)."""
        n_ref = len(ckpts.lengths)
        start_idx, prefix_seq, prefix_len = ([int(v) for v in (a.tolist() if torch.is_tensor(a) else a)] for a in (start_idx, prefix_seq, prefix_len))
        if not len(start_idx) == len(prefix_seq) == len(prefix_len):
            raise _lib.EvoError("start_idx, prefix_seq and prefix_len need one entry per sequence")
        for b, (si, ps, pl) in enumerate(zip(start_idx, prefix_seq, prefix_len)):
            if not 0 <= ps < n_ref:
                raise _lib.EvoError(f"sequence {b}: prefix_seq {ps} outside the {n_ref} references")
            if not 0 <= pl < ckpts.lengths[ps]:
                raise _lib.EvoError(f"sequence {b}: prefix_len {pl} not below reference {ps}'s length {ckpts.lengths[ps]}")
            if si == -1:
                if pl != 0:
                    raise _lib.EvoError(f"sequence {b}: a zero start (start_idx -1) needs prefix_len 0, got {pl}")
            elif not ckpts.base[ps] <= si < ckpts.base[ps + 1] or (si - ckpts.base[ps] + 1) * ckpts.stride != pl:
                raise _lib.EvoError(f"sequence {b}: start_idx {si} is not reference {ps}'s checkpoint at prefix_len {pl}")
        vl = self._varlen(ids, cu_seqlens, pos0=prefix_len)
        if len(start_idx) != vl.n:
            raise _lib.EvoError(f"{len(start_idx)} start indices for {vl.n} sequences")
        on_dev = lambda v: torch.tensor(v, dtype=torch.int64, device=ids.device)
        vl.resume = _Resume(ckpts=ckpts, start_idx=on_dev(start_idx), prefix_seq=on_dev(prefix_seq), prefix_len=on_dev(prefix_len), plen=prefix_len)
        return self._packed_pass(ids, vl, lambda u, x: self._packed_score(u, x, vl))[0]

    # ---- decode step: small-M weight-streaming GEMM tiles + device-side position + CUDA graph ------
    def _can_step(self, ipd, B):
        mha, hy = ipd["mha"], ipd["hyena"]
        for i in range(len(self.blocks)):
            if i in self._attn_idxs:
                c = mha.key_value_memory_dict.get(i)
                if c is None or c.shape[0] < B:
                    return False
            elif i not in hy.fir_state_dict or i not in hy.state_dict:
                return False
        return True

    @staticmethod
    def _tile64(w):
        """(N, K) row-major -> (N/64, K/64, 64, 64): each 64x64 tile is one contiguous 8 KB block, so the decode GEMM's TMA
        boxes use every DRAM page they open (row-major tiles touch 64 pages for 128 bytes each: measured 2.2-3.5 TB/s)."""
        n, k = w.shape
        return w.view(n // 64, 64, k // 64, 64).permute(0, 2, 1, 3).contiguous()

    def _ensure_tiled(self):
        if self._tiled is not None:
            return self._tiled
        t = {}
        with torch.no_grad():
            for i, blk in enumerate(self.blocks):
                t[i] = {name: self._tile64(self.linear_weight(i, name).data) for name in ("in", "out", "w12", "w3")}
            t["unembed"] = self._tile64(self.unembed.weight.data)
        self._tiled = t
        return t

    def _decode_body(self, x, pos_dev, ipd, B, per_row=False, shared=None):
        """One token per sequence through all blocks; every launch reads the position from pos_dev: one shared int64, or
        (per_row) one per row, pos_dev[b] for row b (the _rows entry points).  shared (a shared-prompt state, see
        prefill_shared): {"spos": (B,) suffix positions on the device, "chunks": 64-row chunks of the groups}; the _shared entry
        points then read each group's prefix once and append to the rows' suffix caches."""
        lib = _lib.lib()
        prev = lib.evo_set_pdl(int(self.decode_pdl))
        try:
            return self._decode_body_impl(x, pos_dev, ipd, B, per_row, shared)
        finally:
            lib.evo_set_pdl(prev)

    def _decode_body_impl(self, x, pos_dev, ipd, B, per_row=False, shared=None):
        cfg = self.config
        d, H, V = cfg.hidden_size, cfg.num_attention_heads, cfg.vocab_size
        hd = d // H
        dev = x.device
        lib = _lib.lib()
        mha_ip, hy_ip = ipd["mha"], ipd["hyena"]
        streamk = self.decode_streamk and B <= 64
        # a compact FP8 model never builds the tile-major copies: they would hold W' again (variant 2 gives variant 3's bits)
        tiled = self._ensure_tiled() if (self.decode_tiled and not streamk and not self._fp8_compact) else None
        G2 = 3 if tiled is not None else 2       # weight-streaming tiles (3: tile-major weights)
        qkv_prep = lib.evo_decode_qkv_prep_rows if per_row else lib.evo_decode_qkv_prep
        decode_attn = lib.evo_decode_attn_rows if per_row else lib.evo_decode_attn
        fp8 = self._ensure_fp8() if (streamk and self._fp8_active()) else None

        def lin(a, w, out, N, K, epi, bias=None, resid=None):
            """w: a weight, or (block, name) of a linear layer: its (q, e) when the FP8 kernel streams them, otherwise its tile-major
            copy or W' (linear_weight: for a compact model, rebuilt just now into the scratch)."""
            q, scratch = None, False
            if isinstance(w, tuple):
                if fp8 is not None:
                    q, w = fp8[w[0]][w[1]], None
                elif tiled is not None:
                    w = tiled[w[0]][w[1]]
                else:
                    w, scratch = self.linear_weight(*w), self._fp8_compact
            if not streamk:
                self._gemm(a, w, out, B, N, K, epi, bias=bias, resid=resid, variant=G2)
            elif scratch:
                # the stream-K kernel fetches its first weight tiles before griddepcontrol.wait: under programmatic dependent
                # launch it could read the scratch before the dequant in front of it has finished writing it
                prev = lib.evo_set_pdl(0)
                try:
                    self._gemm_smallm(a, w, out, B, N, K, epi, bias=bias, resid=resid)
                finally:
                    lib.evo_set_pdl(prev)
            else:
                self._gemm_smallm(a, w, out, B, N, K, epi, bias=bias, resid=resid, fp8=q)

        u = self._embed(x)
        n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
        nsplit = max(1, min(16, -(-8 * n_sm // (H * B))))   # >= ~4 waves of 2 CTAs/SM
        for i, blk in enumerate(self.blocks):
            xn = torch.empty_like(u)
            self._rmsnorm(u, blk.pre_norm.scale, xn, B)
            u2 = torch.empty_like(u)
            if i in self._attn_idxs:
                mha = blk.inner_mha_cls
                qkv = torch.empty(B, 3 * d, dtype=torch.bfloat16, device=dev)
                lin(xn, (i, "in"), qkv, 3 * d, d, EPI_BIAS if mha.Wqkv.bias is not None else EPI_NONE, bias=mha.Wqkv.bias)
                cache = mha_ip.key_value_memory_dict[i]
                ctx = xn
                if shared is not None:
                    self._decode_attn_shared(i, qkv, ctx, pos_dev, shared, mha_ip, B, n_sm, nsplit)
                else:
                    cos, sin = self._rope_tables(cache.shape[1], dev)
                    check(qkv_prep(ptr(qkv), ptr(cache), ptr(cos), ptr(sin), ptr(pos_dev), B, H, hd, cache.shape[1], self._stream()), "evo_decode_qkv_prep")
                    nws = lib.evo_decode_attn_workspace(B, H, nsplit)
                    ws = torch.empty(nws, dtype=torch.uint8, device=dev)
                    check(decode_attn(ptr(qkv), ptr(cache), ptr(ctx), ptr(pos_dev), B, H, hd, cache.shape[1], nsplit,
                                              1.0 / math.sqrt(hd), ptr(ws), nws, self._stream()), "evo_decode_attn")
                lin(ctx, (i, "out"), u2, d, d, EPI_BIAS_RESID if mha.out_proj.bias is not None else EPI_RESID, bias=mha.out_proj.bias, resid=u)
            else:
                z = torch.empty(B, 3 * d, dtype=torch.bfloat16, device=dev)
                lin(xn, (i, "in"), z, 3 * d, d, EPI_BIAS, bias=blk.projections.bias)
                y = xn
                check(lib.evo_hyena_step(ptr(z), ptr(y), ptr(hy_ip.fir_state_dict[i]), ptr(torch.view_as_real(hy_ip.state_dict[i])),
                                         *map(C.c_void_p, blk.filter.ptrs().values()), B, d, cfg.state_size, H, self._stream()), "evo_hyena_step")
                lin(y, (i, "out"), u2, d, d, EPI_BIAS_RESID, bias=blk.out_filter_dense.bias, resid=u)
            pk = self._packed[i]
            xn2 = xn
            self._rmsnorm(u2, blk.post_norm.scale, xn2, B)
            g = torch.empty(B, pk["ipad"], dtype=torch.bfloat16, device=dev)
            if streamk:
                lin(xn2, (i, "w12"), g, 2 * pk["ipad"], d, EPI_GELU_GATE)
            else:
                t = torch.empty(B, 2 * pk["ipad"], dtype=torch.bfloat16, device=dev)
                lin(xn2, (i, "w12"), t, 2 * pk["ipad"], d, EPI_NONE)
                check(lib.evo_gelu_gate_interleaved(ptr(t), ptr(g), B, pk["ipad"], self._stream()), "evo_gelu_gate_interleaved")
            u = torch.empty_like(u2)
            lin(g, (i, "w3"), u, d, pk["ipad"], EPI_RESID, resid=u2)
        u = self._final_norm(u)
        logits = torch.empty(B, V, dtype=torch.bfloat16, device=dev)
        lin(u, tiled["unembed"] if tiled is not None else self.unembed.weight, logits, V, d, EPI_NONE)
        return logits

    def _decode_attn_shared(self, i, qkv, ctx, pos_dev, shared, mha_ip, B, n_sm, nsplit):
        """Attention of one decode step of a shared-prompt batch: rotary at pos[b], k,v appended at the row's suffix position,
        then one query per row over its group's prefix (read once per 64-row chunk) and its own suffix."""
        H = self.config.num_attention_heads
        hd = self.config.hidden_size // H
        lib, dev = _lib.lib(), qkv.device
        cache, pcache = mha_ip.key_value_memory_dict[i], mha_ip.prefix_key_value_memory_dict[i]
        S, P, G = cache.shape[1], pcache.shape[1], pcache.shape[0]
        cos, sin = self._rope_tables(P + S, dev)
        spos = shared["spos"]
        check(lib.evo_decode_qkv_prep_shared(ptr(qkv), ptr(cache), ptr(cos), ptr(sin), ptr(pos_dev), ptr(spos), B, H, hd, S, self._stream()),
              "evo_decode_qkv_prep_shared")
        # prefix: one wave of single-CTA-per-SM blocks, at least two 128-key tiles per split; suffix: no split past its 64-key tiles
        nsp_p = max(1, min(64, n_sm // (H * shared["chunks"]), -(-P // 256)))
        nsp_s = max(1, min(nsplit, -(-S // 64)))
        nws = lib.evo_decode_attn_shared_workspace(B, H, nsp_p, nsp_s)
        ws = torch.empty(nws, dtype=torch.uint8, device=dev)
        check(lib.evo_decode_attn_shared(ptr(qkv), ptr(pcache), ptr(mha_ip.group_offsets), ptr(mha_ip.prefix_len), G, P, ptr(cache), ptr(spos), S,
                                         ptr(ctx), B, H, hd, nsp_p, nsp_s, 1.0 / math.sqrt(hd), ptr(ws), nws, self._stream()), "evo_decode_attn_shared")

    # ---- prefill of prompts of different lengths into one decode batch ------------------------------------------------
    def prefill_ragged(self, prompts, cache_len, packed=False):
        """Prefill B prompts of different lengths into one state that decode_loop steps with per-row positions.

        packed=True: one packed forward over all prompts end to end (forward_packed's path with state emission): the KV
        caches are written by evo_kv_append_varlen, each prompt's Hyena end states come straight out of the varlen scan, and
        only the B last rows are unembedded.  Rows may then be in any order.  Equal-length prompts give the grouped path's
        bits.  Otherwise:

        prompts: B non-empty 1-D token sequences (lists or int tensors); rows of equal length must be adjacent (sort by
        length).  The rows are grouped by exact length (frontend.length_buckets) and each group runs the stateful forward
        once.  Every attention layer gets one (B, cache_len, 2, H, 128) KV cache; a group's InferenceParams holds its row
        slice cache[r0:r1], which is contiguous (the cache is batch-major), so the prefill writes and reads it in place.
        The groups' Hyena states are concatenated along the batch.  No row is padded: each row's state is its own prefill's.
        Returns (head (B, V) bf16: each row's logits at its last prompt position, the inference params dict).  Step 0 of
        decode_loop then runs at start_pos = the prompt lengths."""
        from ..frontend import length_buckets
        cfg = self.config
        B = len(prompts)
        lengths = [len(p) for p in prompts]
        if packed:
            return self._prefill_packed(prompts, lengths, cache_len)
        if B == 0 or min(lengths) == 0:
            raise ValueError("prefill_ragged needs at least one prompt and no empty prompt")
        if max(lengths) > cache_len:
            raise _lib.EvoError(f"prompt length {max(lengths)} exceeds the KV cache ({cache_len})")
        groups = length_buckets(prompts, batch_size=B, mode="exact")
        for idx in groups:
            if idx != list(range(idx[0], idx[0] + len(idx))):
                raise ValueError("prefill_ragged: prompts of equal length must be adjacent rows (sort the prompts by length)")
        self._ensure_packed()
        dev = self.embedding_layer.weight.device
        d, H, V = cfg.hidden_size, cfg.num_attention_heads, cfg.vocab_size
        with torch.cuda.device(dev), torch.no_grad():
            caches = {i: torch.zeros(B, cache_len, 2, H, d // H, dtype=torch.bfloat16, device=dev) for i in sorted(self._attn_idxs)}
            head = torch.empty(B, V, dtype=torch.bfloat16, device=dev)
            fir, state = {}, {}
            for idx in sorted(groups, key=lambda g: g[0]):
                r0, r1 = idx[0], idx[-1] + 1
                ids = torch.stack([torch.as_tensor(prompts[r], dtype=torch.long).to(dev) for r in idx])
                ip = {"mha": InferenceParams(max_seqlen=cache_len, max_batch_size=r1 - r0, seqlen_offset=0,
                                             key_value_memory_dict={i: c[r0:r1] for i, c in caches.items()}),
                      "hyena": RecurrentInferenceParams(fir_filter_length=cfg.short_filter_length, state_dim=cfg.state_size, seqlen_offset=0)}
                logits, ip = self.forward(ids, inference_params_dict=ip)
                head[r0:r1] = logits[:, -1]
                for i in ip["hyena"].state_dict:
                    state.setdefault(i, []).append(ip["hyena"].state_dict[i])
                    fir.setdefault(i, []).append(ip["hyena"].fir_state_dict[i])
            hy = RecurrentInferenceParams(fir_filter_length=cfg.short_filter_length, state_dim=cfg.state_size, seqlen_offset=0)
            hy.state_dict = {i: torch.cat(v, 0) for i, v in state.items()}
            hy.fir_state_dict = {i: torch.cat(v, 0) for i, v in fir.items()}
            mha = InferenceParams(max_seqlen=cache_len, max_batch_size=B, seqlen_offset=0, key_value_memory_dict=caches,
                                  lengths_per_sample=torch.tensor(lengths, dtype=torch.int64, device=dev))
        return head, {"mha": mha, "hyena": hy}

    def _prefill_packed(self, prompts, lengths, cache_len):
        cfg = self.config
        B = len(prompts)
        d, H = cfg.hidden_size, cfg.num_attention_heads
        if lengths and max(lengths) > cache_len:
            raise _lib.EvoError(f"prompt length {max(lengths)} exceeds the KV cache ({cache_len})")
        dev = self.embedding_layer.weight.device
        ids = torch.cat([torch.as_tensor(p, dtype=torch.long) for p in prompts] or [torch.zeros(0, dtype=torch.long)]).to(dev)
        vl = self._varlen(ids, list(accumulate(lengths, initial=0)))      # raises on an empty prompt, before anything is launched
        caches = {i: torch.zeros(B, cache_len, 2, H, d // H, dtype=torch.bfloat16, device=dev) for i in sorted(self._attn_idxs)}
        mha = InferenceParams(max_seqlen=cache_len, max_batch_size=B, seqlen_offset=0, key_value_memory_dict=caches,
                              lengths_per_sample=torch.tensor(lengths, dtype=torch.int64, device=dev))
        hy = RecurrentInferenceParams(fir_filter_length=cfg.short_filter_length, state_dim=cfg.state_size, seqlen_offset=0)
        # the last row of each prompt through the full-logits unembed: the same bits per row
        head = self._packed_pass(ids, vl, lambda u, x: self._logits(u.index_select(0, vl.cu[1:] - 1)), {"mha": mha, "hyena": hy})
        return head, {"mha": mha, "hyena": hy}

    # ---- shared-prompt sampling: many rows decode from one prefill of their prompt -----------------------------------
    def prefill_shared(self, prompts, rows_per_prompt, n_new):
        """Prefill G distinct prompts once and set up a decode batch in which prompt g has rows_per_prompt[g] contiguous rows
        (a group) that share its K,V as one prefix.  Returns (head (B, V) bf16: each row's logits at its prompt's last
        position, the inference params dict) with B = sum(rows_per_prompt); decode_loop steps it at start_pos = each row's
        prompt length.  The attention holder carries the (G, P, 2, H, 128) prefix caches (P = the longest prompt rounded up
        to 64), group_offsets and prefix_len; its key_value_memory_dict holds (B, round_up(n_new, 64), 2, H, 128) caches for
        the generated tokens.  Every row gets its own contiguous copy of its group's Hyena states."""
        if len(rows_per_prompt) != len(prompts):
            raise ValueError("prefill_shared: one row count per prompt")
        pre = self.prefill_prefixes(prompts)
        return self.shared_decode_state([(pre, g, n) for g, n in enumerate(rows_per_prompt)], n_new)

    def prefill_prefixes(self, prompts):
        """One packed prefill (prefill_ragged(packed=True)) of G distinct non-empty prompts: a dict of their head logits
        (G, V), (G, P, 2, H, 128) KV caches, Hyena end states and lengths, for shared_decode_state."""
        lengths = [len(p) for p in prompts]
        if not lengths or min(lengths) == 0:
            raise ValueError("prefill_prefixes needs at least one prompt and no empty prompt")
        head, ipd = self._prefill_packed(prompts, lengths, _round_up(max(lengths), 64))
        hy = ipd["hyena"]
        return {"head": head, "caches": ipd["mha"].key_value_memory_dict, "state": hy.state_dict, "fir": hy.fir_state_dict, "lengths": lengths}

    def shared_decode_state(self, parts, n_new):
        """Decode state of one shared-prompt batch: parts = [(prefix from prefill_prefixes, group index in it, rows)], one group
        per entry in row order.  Groups that are consecutive in one prefix keep its caches as a view; otherwise their prefix
        rows are copied into one (G, P, 2, H, 128) cache.  Returns (head (B, V), inference params dict) like prefill_shared."""
        if not parts or min(n for _, _, n in parts) < 1 or n_new < 1:
            raise ValueError("shared_decode_state needs at least one group, every group at least one row, and n_new >= 1")
        cfg = self.config
        d, H = cfg.hidden_size, cfg.num_attention_heads
        dev = self.embedding_layer.weight.device
        counts = [n for _, _, n in parts]
        B, G = sum(counts), len(parts)
        plen = [pre["lengths"][g] for pre, g, _ in parts]
        P = _round_up(max(plen), 64)
        pre0, g0 = parts[0][0], parts[0][1]
        as_view = all(pre is pre0 and g == g0 + k for k, (pre, g, _) in enumerate(parts))

        def per_row(get):                        # each group's (1, ...) slice repeated over its rows: one new contiguous tensor
            return torch.cat([get(pre)[g:g + 1].expand(n, *get(pre).shape[1:]) for pre, g, n in parts]).contiguous()

        with torch.cuda.device(dev), torch.no_grad():
            prefix = {}
            for i in sorted(self._attn_idxs):
                if as_view:
                    prefix[i] = pre0["caches"][i][g0:g0 + G]
                else:
                    prefix[i] = torch.zeros(G, P, 2, H, d // H, dtype=torch.bfloat16, device=dev)
                    for k, (pre, g, _) in enumerate(parts):
                        prefix[i][k, :plen[k]] = pre["caches"][i][g, :plen[k]]
            hy = RecurrentInferenceParams(fir_filter_length=cfg.short_filter_length, state_dim=cfg.state_size, seqlen_offset=0)
            for i in pre0["state"]:
                hy.state_dict[i] = per_row(lambda pre: pre["state"][i])
                hy.fir_state_dict[i] = per_row(lambda pre: pre["fir"][i])
            head = per_row(lambda pre: pre["head"])
            S = _round_up(n_new, 64)
            suffix = {i: torch.zeros(B, S, 2, H, d // H, dtype=torch.bfloat16, device=dev) for i in sorted(self._attn_idxs)}
            offs = torch.tensor([0] + counts, dtype=torch.int64).cumsum_(0)
            rows_len = torch.tensor(plen, dtype=torch.int64).repeat_interleave(torch.tensor(counts))
            mha = InferenceParams(max_seqlen=S, max_batch_size=B, seqlen_offset=0, key_value_memory_dict=suffix,
                                  lengths_per_sample=rows_len.to(dev), prefix_key_value_memory_dict=prefix,
                                  group_offsets=offs.to(dev), prefix_len=torch.tensor(plen, dtype=torch.int64, device=dev))
        return head, {"mha": mha, "hyena": hy}

    # ---- on-device generation loop (SURVEY 8f-2): token pick + bookkeeping + feedback inside the captured step ------
    # a constrained loop with stop motifs replays this many steps between reads of its stopped-row counter
    STOP_CHECK_STEPS = 16

    def decode_loop(self, first_token, ipd, n_steps, start_pos, *, top_k=1, top_p=0.0, temperature=1.0, forced=None, n_out=None, seed=None,
                    constraints=None):
        """Run `n_steps` single-token steps without returning to the host in between.

        first_token (B,) or (B, 1): the input of step 0; ipd: populated state (after a prefill); start_pos: sequence
        position of step 0 (the reference sets the FULL prompt length here, evo/generation.py:143), an int shared by every
        row, or a (B,) int64 tensor of per-row positions (prompts of different lengths, see prefill_ragged).  Step i feeds the
        token of step i-1; the token of step i is forced[:, i] while i < forced.shape[1] (teacher-forced prompt tail,
        evo/generation.py:156-160), afterwards it is picked on the device by evo_sample_step.
        Returns (picked (B, n_out) int64, kept_logits (B, n_out, V) fp32) for the sampled steps; the state holders'
        seqlen_offset end at the value the per-token protocol would leave (per-row positions: the largest row's, and the
        attention holder's lengths_per_sample holds every row's).
        One CUDA graph = one whole step (all blocks + sampler + counters); the host only replays it.

        constraints: a constraints.RowConstraints of the batch.  Its automaton masks every sampled pick and advances each row
        (evo_sample_step_constrained), and the call returns (picked, kept_logits, lengths), lengths (B,) int64 being each row's
        generated tokens up to and including its stop motif (-1: not stopped; the loop's first pick is generated token number
        constraints.index0).  Columns of a stopped row past its length are not written.  When the automaton has stop motifs
        the loop replays STOP_CHECK_STEPS steps at a time and ends once every row has stopped; the state holders then
        reflect the steps that ran."""
        lib = _lib.lib()
        dev = self.embedding_layer.weight.device
        x = first_token.reshape(-1, 1).contiguous()
        B = x.shape[0]
        V = self.config.vocab_size
        if not self._can_step(ipd, B):
            raise _lib.EvoError("decode_loop needs populated inference params (run the prefill first)")
        mha_ip, hy_ip = ipd["mha"], ipd["hyena"]
        n_forced = 0 if forced is None else int(forced.shape[1])
        n_out = n_steps - n_forced if n_out is None else n_out
        if n_out < 0:
            raise ValueError("more forced tokens than steps")
        per_row = torch.is_tensor(start_pos) and start_pos.dim() > 0
        if per_row:
            if tuple(start_pos.shape) != (B,):
                raise ValueError(f"per-row start_pos must have shape ({B},), got {tuple(start_pos.shape)}")
            starts = start_pos.detach().to("cpu", torch.int64)
            if int(starts.min()) < 0:
                raise ValueError("negative start position")
            last = int(starts.max())
        else:
            last = start_pos = int(start_pos)
        shared = None
        if mha_ip.prefix_len is not None:      # shared-prompt state (prefill_shared): the suffix caches hold the generated tokens only
            if not per_row:
                raise ValueError("a shared-prompt state needs per-row start positions (each row's prompt length)")
            counts = torch.diff(mha_ip.group_offsets.cpu())
            sstarts = starts - mha_ip.prefix_len.cpu().repeat_interleave(counts)
            if int(sstarts.min()) < 0:
                raise ValueError("a start position lies inside its row's shared prompt")
            shared = {"chunks": int(((counts + 63) // 64).sum())}
        fill = last if shared is None else int(sstarts.max())     # the last cache row a step writes is fill + n_steps - 1
        for i in mha_ip.key_value_memory_dict:
            if fill + n_steps > mha_ip.key_value_memory_dict[i].shape[1]:
                raise _lib.EvoError(f"sequence length {fill + n_steps} exceeds the KV cache ({mha_ip.key_value_memory_dict[i].shape[1]}) (mha.py:367)")
        with torch.cuda.device(dev), torch.no_grad():
            self._ensure_packed()
            key = ("loop_rows" if per_row else "loop", B) + self._step_key(ipd)
            picked = torch.empty(B, max(n_out, 1), dtype=torch.long, device=dev)
            kept = torch.empty(B, max(n_out, 1), V, dtype=torch.float32, device=dev)
            forced_c = forced.to(dev, torch.long).contiguous() if n_forced else None
            if seed is None:
                seed = int(torch.randint(0, 2 ** 62, (1,)).item())          # torch.manual_seed() governs reproducibility
            lp = _lib.LoopParams(forced=forced_c.data_ptr() if n_forced else None, n_forced=n_forced, forced_stride=n_forced,
                                 picked=picked.data_ptr(), picked_stride=picked.shape[1], kept_logits=kept.data_ptr(), n_out=n_out,
                                 top_k=int(top_k), top_p=float(top_p), temperature=float(temperature), seed=seed, step0=0)
            if shared is not None:
                pre = mha_ip.prefix_key_value_memory_dict
                key = ("loop_shared",) + key[1:] + (tuple((pre[i].data_ptr(), tuple(pre[i].shape)) for i in sorted(pre)),
                                                    mha_ip.group_offsets.data_ptr(), mha_ip.prefix_len.data_ptr(), shared["chunks"])
            if constraints is not None:
                key = ("constrained",) + key
            st = self._loop
            if st is None or st["key"] != key:
                st = {"key": key, "graph": None, "x": torch.empty(B, 1, dtype=torch.long, device=dev),
                      "pos": torch.zeros(B if per_row else 1, dtype=torch.int64, device=dev),
                      "step": torch.zeros(1, dtype=torch.int64, device=dev), "lp": torch.zeros(C.sizeof(_lib.LoopParams), dtype=torch.uint8, device=dev),
                      "lp_host": torch.zeros(C.sizeof(_lib.LoopParams), dtype=torch.uint8).pin_memory()}
                if shared is not None:
                    st["spos"] = torch.zeros(B, dtype=torch.int64, device=dev)
                if constraints is not None:
                    # the tables and per-row arrays go in through this device-resident struct, so the graph serves every call
                    st["cp"] = torch.zeros(C.sizeof(_lib.ConstraintParams), dtype=torch.uint8, device=dev)
                    st["cp_host"] = torch.zeros(C.sizeof(_lib.ConstraintParams), dtype=torch.uint8).pin_memory()
                    st["stopped_host"] = torch.zeros(1, dtype=torch.int32).pin_memory()
                self._loop = st
            if st.get("lp_copied") is not None:
                st["lp_copied"].synchronize()       # a previous call's async copy may not have left the pinned staging buffer yet
            C.memmove(st["lp_host"].data_ptr(), C.addressof(lp), C.sizeof(lp))
            st["lp"].copy_(st["lp_host"], non_blocking=True)
            if constraints is not None:
                cp = constraints.params()
                C.memmove(st["cp_host"].data_ptr(), C.addressof(cp), C.sizeof(cp))
                st["cp"].copy_(st["cp_host"], non_blocking=True)
            st["lp_copied"] = torch.cuda.Event()
            st["lp_copied"].record()
            if per_row:
                st["pos"].copy_(starts)
                if shared is not None:
                    st["spos"].copy_(sstarts)
                    shared["spos"] = st["spos"]
            else:
                st["pos"].fill_(int(start_pos))
            st["step"].zero_()
            st["x"].copy_(x.to(torch.long))

            def one_step():
                logits = self._decode_body(st["x"], st["pos"], ipd, B, per_row, shared)
                prev = lib.evo_set_pdl(int(self.decode_pdl))
                try:
                    if constraints is None:
                        check(lib.evo_sample_step(ptr(logits), ptr(st["x"]), B, V, ptr(st["lp"]), ptr(st["step"]), self._stream()), "evo_sample_step")
                    else:
                        check(lib.evo_sample_step_constrained(ptr(logits), ptr(st["x"]), B, V, ptr(st["lp"]), ptr(st["cp"]), ptr(st["step"]),
                                                              self._stream()), "evo_sample_step_constrained")
                    if shared is not None:
                        check(lib.evo_advance_positions(ptr(st["spos"]), B, 1, self._stream()), "evo_advance_positions")
                    if per_row:
                        check(lib.evo_advance_positions(ptr(st["pos"]), B, 1, self._stream()), "evo_advance_positions")
                        check(lib.evo_advance_counters(None, ptr(st["step"]), 1, self._stream()), "evo_advance_counters")
                    else:
                        check(lib.evo_advance_counters(ptr(st["pos"]), ptr(st["step"]), 1, self._stream()), "evo_advance_counters")
                finally:
                    lib.evo_set_pdl(prev)

            done = 0
            if st["graph"] is None or st.get("ptrs") != self._graph_ptrs():
                one_step()                      # eager step: allocates rope tables / workspaces the capture must not
                done = 1
                if self.decode_graph and n_steps > 1:
                    st["graph"], st["launches"], _ = self._capture(one_step)
                    st["ptrs"] = self._graph_ptrs()
            early_exit = constraints is not None and constraints.automaton.has_stop
            ran = done
            while ran < n_steps:
                n = min(n_steps - ran, self.STOP_CHECK_STEPS) if early_exit else n_steps - ran
                for _ in range(n):
                    if st["graph"] is not None:
                        self._replay(st)
                    else:
                        one_step()
                ran += n
                if early_exit and ran < n_steps:
                    st["stopped_host"].copy_(constraints.n_stopped, non_blocking=True)
                    read = torch.cuda.Event()
                    read.record()
                    read.synchronize()
                    if int(st["stopped_host"][0]) == B:
                        n_steps = ran
                        break
            if per_row:
                mha_ip.lengths_per_sample = (starts + n_steps - 1).to(dev)
                end = last + n_steps - 1
            else:
                end = int(start_pos) + n_steps - 1          # the position the last step ran at (what the per-token protocol leaves)
            mha_ip.seqlen_offset = hy_ip.seqlen_offset = end
            # the captured graph and its buffers stay alive in self._loop; the outputs are this call's own tensors
            if constraints is None:
                return picked[:, :n_out], kept[:, :n_out]
            constraints.index0 += max(n_steps - n_forced, 0)
            return picked[:, :n_out], kept[:, :n_out], constraints.length.clone()

    def _graph_ptrs(self):
        """Addresses a captured step bakes in besides the state tensors: rope tables, the stream-K workspace and, for an FP8
        model, its decode copies (none when _fp8_decode_bf16 selects the bf16 kernel); for a compact one, its (q, e) and the
        scratch W' is rebuilt into."""
        fp8 = self._ensure_fp8() if self._fp8_compact else self._fp8
        return (tuple(t.data_ptr() for t in (self._rope or ())), self._smallm_ws.data_ptr() if self._smallm_ws is not None else 0,
                self._fp8_active(), fp8["ptrs"] if fp8 is not None else (),
                self._w_scratch.data_ptr() if self._w_scratch is not None else 0)

    def _step_key(self, ipd):
        """The state addresses a captured step bakes in, after making every Hyena state contiguous in place: each layer's
        modal and FIR state, and each KV cache with its length."""
        hy_ip, kv = ipd["hyena"], ipd["mha"].key_value_memory_dict
        for i in list(hy_ip.state_dict):
            self._contiguous_state(hy_ip, i)
        return (tuple(hy_ip.state_dict[i].data_ptr() for i in sorted(hy_ip.state_dict)),
                tuple(hy_ip.fir_state_dict[i].data_ptr() for i in sorted(hy_ip.fir_state_dict)),
                tuple((kv[i].data_ptr(), kv[i].shape[1]) for i in sorted(kv)))

    @staticmethod
    def _capture(step):
        """Capture step() into a CUDA graph: (graph, launches per replay, what step returned).  The library counts the
        launches made while capturing, when nothing ran: they are taken back here and counted again at each _replay."""
        lib = _lib.lib()
        g = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        n0 = lib.evo_launch_count()
        with torch.cuda.graph(g):
            out = step()
        n = lib.evo_launch_count() - n0
        lib.evo_note_graph_replay(-n)
        return g, n, out

    @staticmethod
    def _replay(st):
        st["graph"].replay()
        _lib.lib().evo_note_graph_replay(st["launches"])

    def _decode_forward(self, x, ipd):
        """L == 1 with populated states.  Step 1 after a prefill runs eagerly (and makes the state
        tensors contiguous / resident); step 2 captures the whole step into a CUDA graph; later
        steps replay it: one host call per token instead of ~15 launches per block."""
        mha_ip = ipd["mha"]
        dev = x.device
        B = x.shape[0]
        key = (B, x.dtype) + self._step_key(ipd) + self._graph_ptrs()
        off = int(mha_ip.seqlen_offset)
        for i in mha_ip.key_value_memory_dict:
            if off >= mha_ip.key_value_memory_dict[i].shape[1]:
                raise _lib.EvoError(f"sequence length {off + 1} exceeds the KV cache ({mha_ip.key_value_memory_dict[i].shape[1]}) (mha.py:367)")
        st = self._decode
        if st is None or st["key"] != key:
            st = {"key": key, "graph": None, "x": torch.empty_like(x), "pos": torch.zeros(1, dtype=torch.int64, device=dev), "logits": None, "steps": 0}
            self._decode = st
        st["pos"].fill_(off)
        st["x"].copy_(x)
        if not self.decode_graph or self._prof is not None or st["steps"] == 0:
            st["steps"] += 1
            return self._decode_body(st["x"], st["pos"], ipd, B).view(B, 1, -1)
        if st["graph"] is None:
            st["graph"], st["launches"], st["logits"] = self._capture(lambda: self._decode_body(st["x"], st["pos"], ipd, B))
        self._replay(st)
        st["steps"] += 1
        return st["logits"].clone().view(B, 1, -1)
