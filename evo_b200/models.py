"""`Evo` front door and checkpoint ingest: the reference's evo/models.py (Evo :21-62,
load_checkpoint :73-152) re-expressed for the evo_b200 engine.  Checkpoint key names after
the 'backbone.' strip, the tied unembed, strict loading and the bf16-except-poles/residues
dtype policy are the contract (evo/models.py:124-148)."""
from __future__ import annotations

import json
import os
from typing import Optional

import torch
import yaml

from .configs import MODEL_NAMES, MODELS, get_config
from .stripedhyena import StripedHyena, dotdict
from .tokenizer import CharLevelTokenizer

HF_MODEL_NAME_MAP = {name: spec[1] for name, spec in MODELS.items()}


def _read_safetensors(model_dir: str) -> dict:
    from safetensors.torch import load_file
    index = os.path.join(model_dir, "model.safetensors.index.json")
    single = os.path.join(model_dir, "model.safetensors")
    if os.path.exists(index):
        with open(index) as f:
            shards = sorted(set(json.load(f)["weight_map"].values()))
        tensors = {}
        for shard in shards:
            tensors.update(load_file(os.path.join(model_dir, shard)))
        return tensors
    if os.path.exists(single):
        return load_file(single)
    raise FileNotFoundError(f"No safetensors files found in {model_dir}. Expected model.safetensors.index.json or model.safetensors.")


# the reference resolves config_path relative to its package (pkgutil.get_data, evo/models.py:141); those two names
# map to the built-in dicts of evo_b200/configs.py, which hold the same keys and values
_PACKAGE_CONFIGS = {"evo-1-8k-base_inference.yml": "evo-1-8k-base", "evo-1-131k-base_inference.yml": "evo-1-131k-base"}


def _resolve_config(model_name: str, config_path: Optional[str]) -> dict:
    if config_path is None:
        return get_config(model_name)
    if os.path.isfile(config_path):
        with open(config_path) as f:
            return yaml.safe_load(f)
    base = os.path.basename(config_path)
    if base in _PACKAGE_CONFIGS and os.path.dirname(config_path) in ("configs", "evo/configs"):
        return get_config(_PACKAGE_CONFIGS[base])
    raise FileNotFoundError(f"config file {config_path!r} does not exist (and is not one of the package configs "
                            f"{sorted('configs/' + k for k in _PACKAGE_CONFIGS)})")


def load_checkpoint(model_name: str = "evo-1-8k-base", config_path: Optional[str] = None, device: str = None,
                    model_dir: Optional[str] = None, random_init: bool = False, seed: int = 0, streaming: bool = True, *args,
                    weights: str = "bf16", **kwargs):
    """HF snapshot -> safetensors -> StripedHyena on `device`.

    model_dir: use an already-downloaded snapshot directory instead of huggingface_hub.
    random_init: skip the checkpoint (benchmarks / tests on boxes without network) and keep the
    constructor's random initialisation, seeded.
    streaming: True (default) = tensor-by-tensor ingest straight into the device layouts; False = the reference's
    host-state-dict sequence (kept as the comparator for the ingest tests).
    weights: "bf16" (default) or "fp8": the model's linear-layer weights rounded onto an E4M3 grid with a power-of-two scale per
    row, on the device after loading (StripedHyena.quantize_fp8): generation then streams one byte per weight.
    "fp8-compact": the same model holding only the one-byte weights and row exponents of those layers (quantize_fp8(compact=True)),
    the same outputs on every path in about a third of the FP8 model's linear-weight memory.  The streaming ingest never holds
    those layers in bf16 (each is compacted as soon as it is loaded); random_init and streaming=False build the bf16 model
    first and compact it afterwards, so their peak device memory is the bf16 model's."""
    if weights not in WEIGHTS:
        raise ValueError(f"weights={weights!r}: should be one of {', '.join(WEIGHTS)}")
    compact = weights == "fp8-compact"
    model = _load(model_name, config_path, device, model_dir, random_init, seed, streaming, compact)
    return model.quantize_fp8(compact=compact) if weights != "bf16" else model


WEIGHTS = ("bf16", "fp8", "fp8-compact")


def _load(model_name, config_path, device, model_dir, random_init, seed, streaming, compact=False):
    cfg = dotdict(_resolve_config(model_name, config_path))

    if random_init:
        # build straight on the target device: no 26 GB fp32 host copy of a 7B model
        torch.manual_seed(seed)
        with torch.device(device if device is not None else "cpu"):
            model = StripedHyena(cfg)
        model.to_bfloat16_except_poles_residues()
        return model if device is None else model.to(device)
    if model_dir is None:
        from huggingface_hub import snapshot_download
        _, repo, revision = MODELS[model_name]
        model_dir = snapshot_download(repo, revision=revision)
    if not streaming:
        # the reference's own sequence (evo/models.py:96-150): host state dict -> strict load -> bf16 -> device
        state = {}
        for key, value in _read_safetensors(model_dir).items():
            state[key[len("backbone."):] if key.startswith("backbone.") else key] = value
        if "unembed.weight" not in state and "embedding_layer.weight" in state:
            state["unembed.weight"] = state["embedding_layer.weight"]
        model = StripedHyena(cfg)
        model.load_state_dict(state, strict=True)
        model.to_bfloat16_except_poles_residues()
        return model if device is None else model.to(device)
    # streaming ingest (SURVEY 8f-3): parameters are allocated once, on the target device, in their final dtype and layout;
    # each checkpoint tensor goes mmap -> pinned staging -> device and is cast / packed there (evo_b200/ingest.py)
    from .ingest import load_streaming
    dev = torch.device(device) if device is not None else torch.device("cpu")
    compact = compact and dev.type == "cuda"        # elsewhere quantize_fp8 refuses the model after an ordinary load
    with torch.device("meta"):
        model = StripedHyena(cfg)
    model.to_bfloat16_except_poles_residues()
    if compact:                                     # the linear weights arrive as (q, e): their parameters are never allocated
        for _, _, mod, attr, _ in model._fp8_slots():
            getattr(mod, attr).data = torch.empty(0, dtype=torch.bfloat16, device="meta")
    model = model.to_empty(device=dev)
    model.ingest_stats = load_streaming(model, model_dir, dev, compact=compact)
    if compact:
        model._fp8_mode = model._fp8_compact = True
        model._invalidate()
    return model


class Evo:
    """Evo('evo-1-8k-base') -> .model (StripedHyena protocol), .tokenizer.  Evo(name, weights="fp8"): an FP8-weight model;
    weights="fp8-compact": the same model keeping only the one-byte weights (see load_checkpoint)."""

    def __init__(self, model_name: str = "evo-1-8k-base", device: str = None, **load_kwargs):
        if model_name not in MODEL_NAMES:
            raise ValueError(f"Invalid model name {model_name}. Should be one of: {', '.join(MODEL_NAMES)}.")
        self.device = device
        self.model = load_checkpoint(model_name=model_name, device=device, **load_kwargs)
        self.tokenizer = CharLevelTokenizer(512)
