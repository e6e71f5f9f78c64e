"""Streaming checkpoint ingest (SURVEY.md 8f-3): safetensors shards -> the model's device tensors, tensor by tensor.

The reference (evo/models.py:96-150) materialises the whole checkpoint as a host state dict (`load_file` per shard),
builds the model on the CPU, `load_state_dict`s (a second full copy), casts to bf16 on the CPU and only then moves
everything to the GPU: ~3x the checkpoint in host memory and a single-threaded cast.  Here
  * the model is constructed directly on the target device WITHOUT initialising its parameters (meta -> empty);
  * every shard is memory-mapped; each tensor's bytes go through a small ring of pinned staging buffers and one
    asynchronous H2D copy (the next tensor's page-in overlaps the previous copy);
  * dtype policy (evo/models.py:148: bf16 except poles/residues) and layout (MLP weights straight into the GEMM-packed
    w12 / w3 buffers, see stripedhyena.model._GatedMLP) are applied ON THE DEVICE, so no tensor exists twice;
  * strict-mode semantics are kept: missing / unexpected / mis-shaped keys raise RuntimeError like
    load_state_dict(strict=True) (evo/models.py:147).
Peak host memory: the staging ring (2 x the largest tensor); peak device memory: the model plus one staged tensor.

compact=True (weights="fp8-compact"): the linear-layer weights are never resident in bf16.  Each one is rounded to FP8 and kept
as (q, e) (StripedHyena.quantize_fp8(compact=True)) as soon as it is complete on the device, and its bf16 staging is freed; a
packed w12 is held in bf16 only until both of its halves (l1, l2) have arrived.  Peak device memory: the compact model plus the
matrices still being assembled and one staged tensor."""
from __future__ import annotations

import json
import mmap
import os
import struct
from typing import Dict, Iterator, List, Tuple

import numpy as np
import torch
import torch.nn.functional as F

_DTYPES = {"BF16": (torch.bfloat16, 2), "F16": (torch.float16, 2), "F32": (torch.float32, 4), "F64": (torch.float64, 8),
           "I64": (torch.int64, 8), "I32": (torch.int32, 4), "U8": (torch.uint8, 1), "I8": (torch.int8, 1), "BOOL": (torch.bool, 1)}


def shard_files(model_dir: str) -> List[str]:
    index = os.path.join(model_dir, "model.safetensors.index.json")
    single = os.path.join(model_dir, "model.safetensors")
    if os.path.exists(index):
        with open(index) as f:
            return [os.path.join(model_dir, s) for s in sorted(set(json.load(f)["weight_map"].values()))]
    if os.path.exists(single):
        return [single]
    raise FileNotFoundError(f"No safetensors files found in {model_dir}. Expected model.safetensors.index.json or model.safetensors.")


def iter_safetensors(path: str) -> Iterator[Tuple[str, torch.dtype, Tuple[int, ...], memoryview]]:
    """(name, dtype, shape, raw bytes) for every tensor of one .safetensors file, in file order, zero-copy (mmap).
    Format: u64 little-endian header length, JSON header {name: {dtype, shape, data_offsets}}, then the data."""
    with open(path, "rb") as f:
        mm = mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ)
    (hlen,) = struct.unpack("<Q", mm[:8])
    header = json.loads(bytes(mm[8:8 + hlen]).decode("utf-8"))
    base = 8 + hlen
    view = memoryview(mm)
    entries = sorted(((v["data_offsets"][0], k, v) for k, v in header.items() if k != "__metadata__"))
    for off, name, meta in entries:
        if meta["dtype"] not in _DTYPES:
            raise RuntimeError(f"{path}: tensor {name} has unsupported dtype {meta['dtype']}")
        dt, size = _DTYPES[meta["dtype"]]
        shape = tuple(int(s) for s in meta["shape"])
        n = int(np.prod(shape, dtype=np.int64)) * size if shape else size
        lo, hi = meta["data_offsets"]
        if hi - lo != n:
            raise RuntimeError(f"{path}: tensor {name}: {hi - lo} bytes on disk, shape {shape} x {meta['dtype']} needs {n}")
        yield name, dt, shape, view[base + lo: base + hi]


class _Staging:
    """Ring of pinned host buffers; each slot is reused only after the H2D copy that read it has completed."""

    def __init__(self, device: torch.device, slots: int = 2):
        self.device, self.cuda = device, device.type == "cuda"
        self.slots = [None] * slots
        self.events = [None] * slots
        self.k = 0

    def to_device(self, raw: memoryview, dtype: torch.dtype, shape) -> torch.Tensor:
        n = len(raw)
        if not self.cuda:
            return torch.frombuffer(bytearray(raw), dtype=dtype).view(shape) if n else torch.empty(shape, dtype=dtype)
        k = self.k
        self.k = (k + 1) % len(self.slots)
        if self.events[k] is not None:
            self.events[k].synchronize()
        buf = self.slots[k]
        if buf is None or buf.numel() < n:
            buf = self.slots[k] = torch.empty(max(n, 1 << 20), dtype=torch.uint8).pin_memory()
        buf.numpy()[:n] = np.frombuffer(raw, dtype=np.uint8)           # page-in from the mmap: the only host copy
        out = torch.empty(n, dtype=torch.uint8, device=self.device)
        out.copy_(buf[:n], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self.events[k] = ev
        return out.view(dtype).view(shape)


def _targets(model) -> Dict[str, tuple]:
    """checkpoint key -> (destination tensor, kind) for every key the model's state_dict() shows."""
    from .stripedhyena.model import _GatedMLP
    out: Dict[str, tuple] = {}
    mlps = {name: mod for name, mod in model.named_modules() if isinstance(mod, _GatedMLP)}
    for name, p in list(model.named_parameters()) + list(model.named_buffers()):
        owner = name.rsplit(".", 1)[0]
        if owner in mlps:
            continue
        out[name] = (p, "plain")
    for mname, mod in mlps.items():
        out[f"{mname}.l1.weight"] = (mod, "l1")
        out[f"{mname}.l2.weight"] = (mod, "l2")
        out[f"{mname}.l3.weight"] = (mod, "l3")
    if getattr(model, "unembed", None) is getattr(model, "embedding_layer", None):
        out["unembed.weight"] = out["embedding_layer.weight"]          # tied: the checkpoint may carry either or both
    return out


def _want_dtype(name: str) -> torch.dtype:
    return torch.float32 if ("poles" in name or "residues" in name) else torch.bfloat16      # evo/models.py:148


@torch.no_grad()
def _place(dst, kind: str, name: str, src: torch.Tensor, errors: List[str]) -> None:
    want = _want_dtype(name)
    if kind == "plain":
        if tuple(dst.shape) != tuple(src.shape):
            errors.append(f"size mismatch for {name}: copying a param with shape {tuple(src.shape)} from checkpoint, the shape in current model is {tuple(dst.shape)}.")
            return
        dst.data.copy_(src.to(want) if dst.dtype == want else src.to(dst.dtype))
        return
    mod = dst
    d, inner, ipad = mod.w3.shape[0], mod.inner, mod.ipad
    shape = (d, inner) if kind == "l3" else (inner, d)
    if tuple(src.shape) != shape:
        errors.append(f"size mismatch for {name}: copying a param with shape {tuple(src.shape)} from checkpoint, the shape in current model is {shape}.")
        return
    src = src.to(mod.w3.dtype)
    if kind == "l3":
        mod.w3.data[:, :inner].copy_(src)
        mod.w3.data[:, inner:].zero_()
        return
    half = 0 if kind == "l1" else 1
    v = mod.w12.data.view(ipad // 128, 2, 128, d)[:, half]             # (groups, 128, d) strided view into the packed buffer
    full = inner // 128
    v[:full].copy_(src[:full * 128].view(full, 128, d))
    if inner % 128:
        v[full, :inner % 128].copy_(src[full * 128:])
        v[full, inner % 128:].zero_()
    v[full + (1 if inner % 128 else 0):].zero_()


class _CompactSink:
    """Linear-layer weights of a compact FP8 model (their parameters already empty): checkpoint key -> the weight's slot.  Each
    matrix is rounded and kept as (q, e) once complete; w12 is assembled in a packed bf16 buffer until l1 and l2 are both in."""

    def __init__(self, model):
        self.model, self.slots, self.pending = model, {}, {}
        names = {id(m): n for n, m in model.named_modules()}
        d = model.config.hidden_size
        for _, name, mod, attr, gate in model._fp8_slots():
            p = names[id(mod)]
            if attr == "w12":
                self.slots[f"{p}.l1.weight"] = (mod, attr, gate, 0, (mod.inner, d))
                self.slots[f"{p}.l2.weight"] = (mod, attr, gate, 1, (mod.inner, d))
            elif attr == "w3":
                self.slots[f"{p}.l3.weight"] = (mod, attr, gate, None, (d, mod.inner))
            else:
                self.slots[f"{p}.weight"] = (mod, attr, gate, None, (3 * d if name == "in" else d, d))

    @torch.no_grad()
    def place(self, key: str, src: torch.Tensor, errors: List[str]) -> None:
        mod, attr, gate, half, shape = self.slots[key]
        if tuple(src.shape) != shape:
            errors.append(f"size mismatch for {key}: copying a param with shape {tuple(src.shape)} from checkpoint, the shape in current model is {shape}.")
            return
        src = src.to(torch.bfloat16)
        if attr == "w3":
            w = F.pad(src, (0, mod.ipad - mod.inner))
        elif attr == "w12":
            w = self.pending.get(id(mod))
            if w is None:
                w = self.pending[id(mod)] = (src.new_zeros(2 * mod.ipad, shape[1]), set())
            _, got = w
            v = w[0].view(mod.ipad // 128, 2, 128, shape[1])[:, half]
            full = mod.inner // 128
            v[:full].copy_(src[:full * 128].view(full, 128, shape[1]))
            if mod.inner % 128:
                v[full, :mod.inner % 128].copy_(src[full * 128:])
            got.add(half)
            if len(got) < 2:
                return
            w = self.pending.pop(id(mod))[0]
        else:
            w = src.contiguous()
        with torch.cuda.device(w.device):
            self.model._hold_compact(mod, attr, *self.model._quantize_rows(w, gate))


def load_streaming(model, model_dir: str, device, compact: bool = False) -> Dict[str, int]:
    """Fill `model` (already on `device`, parameters uninitialised) from the safetensors files in model_dir.  compact: the
    model's linear-layer parameters are empty and their weights arrive as compact FP8 (see the module docstring).
    Returns {"tensors", "bytes"}; raises RuntimeError on any strict-mode violation."""
    device = torch.device(device)
    targets = _targets(model)
    sink = _CompactSink(model) if compact else None
    if sink is not None:
        targets.update({k: (sink, "fp8") for k in sink.slots})
    seen, unexpected, errors = set(), [], []
    stage = _Staging(device)
    nbytes = 0
    for path in shard_files(model_dir):
        for name, dt, shape, raw in iter_safetensors(path):
            key = name[len("backbone."):] if name.startswith("backbone.") else name      # evo/models.py:124-131
            if key not in targets:
                unexpected.append(key)
                continue
            dst, kind = targets[key]
            if kind == "fp8":
                sink.place(key, stage.to_device(raw, dt, shape), errors)
            else:
                _place(dst, kind, key, stage.to_device(raw, dt, shape), errors)
            seen.add(key)
            nbytes += len(raw)
    if "embedding_layer.weight" in seen or "unembed.weight" in seen:                         # tied embeddings: either name fills both
        if targets.get("unembed.weight", (None,))[0] is targets.get("embedding_layer.weight", (1,))[0]:
            seen.update(("embedding_layer.weight", "unembed.weight"))
    if "unembed.weight" in targets and "unembed.weight" not in seen and "embedding_layer.weight" in seen:
        # untied model, checkpoint without unembed.weight: the reference fills it from the embedding whatever the config says
        # (evo/models.py:133-137)
        with torch.no_grad():
            targets["unembed.weight"][0].data.copy_(targets["embedding_layer.weight"][0].data)
        seen.add("unembed.weight")
    for key in [k for k in targets if k.endswith("rotary_emb.inv_freq") and k not in seen]:
        # optional in a checkpoint (see stripedhyena.model._Rotary): absent -> the analytic value the constructor would hold
        rot = model.get_submodule(key.rsplit(".", 1)[0])
        with torch.no_grad():
            targets[key][0].data.copy_(rot.analytic(device))
        seen.add(key)
    missing = [k for k in targets if k not in seen]
    if missing or unexpected or errors:
        msg = [f"Error(s) in loading state_dict for {type(model).__name__}:"]
        if missing:
            msg.append("\tMissing key(s) in state_dict: " + ", ".join(f'"{k}"' for k in missing) + ".")
        if unexpected:
            msg.append("\tUnexpected key(s) in state_dict: " + ", ".join(f'"{k}"' for k in unexpected) + ".")
        msg.extend("\t" + e for e in errors)
        raise RuntimeError("\n".join(msg))
    if device.type == "cuda":
        torch.cuda.synchronize(device)
    return {"tensors": len(seen), "bytes": nbytes}
