"""``load_model`` — dynamic sharding loader.

Reference: ``shard/utils.py:33-68``.  Differences (SURVEY §2.8, all deliberate):
* ``start_layer`` / ``end_layer`` may be given independently; missing bounds come from ``config.json``
  (pre-sharded dirs written by ``sharding_weight.py``) or default to ``0`` / ``num_hidden_layers``;
* only the tensors of this stage are read from disk (the reference ``mx.load``s every file lazily);
* quantised checkpoints keep their int4/int8 payload — dequantisation happens inside the kernels.
"""
from __future__ import annotations

import json
import logging
import os
from typing import Optional

import torch

from ..config import ModelConfig
from ..models import build_stage
from .checkpoint import get_model_path, key_in_shard, iter_safetensors, random_state_dict, shard_expert_tensors

log = logging.getLogger(__name__)


def load_model(path_or_hf_repo: str, start_layer: Optional[int] = None, end_layer: Optional[int] = None,
               dtype: Optional[torch.dtype] = None, device: Optional[str] = None, backend: Optional[str] = None,
               spec=None, expert_shard=None, adapter_path: Optional[str] = None):
    """``spec`` (a ``ShardSpec``, e.g. from ``parallel.partition.balanced_split``) overrides the layer bounds.
    ``expert_shard=(rank, world)`` keeps only this rank's ``E / world`` routed experts of every MoE layer (expert
    parallelism, ``parallel/ep.py::enable_expert_parallel``).  ``adapter_path``: an mlx_lm LoRA adapter directory
    (``utils/adapters.py``); the stage applies it to the layers it loads."""
    model_path = get_model_path(path_or_hf_repo)
    cfg = ModelConfig.from_path(model_path)
    spec = spec or cfg.shard(start_layer, end_layer)
    adapter = None
    if adapter_path is not None:
        from .adapters import load_adapter

        adapter = load_adapter(adapter_path)
    marker = os.path.join(model_path, "synthetic.json")
    if os.path.exists(marker):   # ``synthetic:<name>``: random-init weights of that architecture, built on the device
        with open(os.path.join(model_path, "config.json")) as f:
            cfgd = json.load(f)
        with open(marker) as f:
            seed = int(json.load(f).get("seed", 1))
        dev = device or ("cuda" if torch.cuda.is_available() else "cpu")
        dt = dtype or (torch.bfloat16 if torch.device(dev).type == "cuda" else torch.float32)
        model = random_model(cfgd, dtype=dt, device=dev, backend=backend, seed=seed, spec=spec, expert_shard=expert_shard,
                             adapter=adapter)
        log.info("built synthetic %s layers %s (%.2f GB) on %s", cfg.model_type, spec.describe(), model.weight_bytes() / 1e9, dev)
        return model
    device = device or ("cuda" if torch.cuda.is_available() else "cpu")
    if dtype is None:
        dtype = torch.bfloat16 if torch.device(device).type == "cuda" else torch.float32
    model = build_stage(cfg, spec, dtype, device, backend)
    model.expert_shard = expert_shard
    tied = cfg.tie_word_embeddings
    # HF-style per-expert keys also belong to the layer range, key_in_shard handles them by prefix
    sd = dict(shard_expert_tensors(iter_safetensors(model_path, lambda k: key_in_shard(k, spec, tied, cfg.model_type)),
                                   cfg.n_routed_experts or 0, expert_shard))
    if not sd:
        raise ValueError(f"no tensors for layers [{spec.start_layer}, {spec.end_layer}) in {model_path}")
    model.load_state(sd, adapter=adapter)
    log.info("loaded %s layers %s of %s (%.2f GB) on %s", cfg.model_type, spec.describe(),
             model_path, model.weight_bytes() / 1e9, device)
    return model


def random_model(config: dict, start_layer: Optional[int] = None, end_layer: Optional[int] = None,
                 dtype=torch.bfloat16, device="cpu", backend: Optional[str] = None, seed: int = 0,
                 quantization: Optional[dict] = None, spec=None, expert_shard=None, adapter=None):
    """Random-init stage directly on ``device`` (no disk round trip) — used by the benchmarks on the
    offline GPU box; key layout and shapes are identical to an mlx-community checkpoint.  ``adapter``: a parsed LoRA
    adapter (``utils/adapters.py::load_adapter``)."""
    config = dict(config)
    if quantization is not None:
        config["quantization"] = dict(quantization)
    cfg = ModelConfig.from_dict(config)
    spec = spec or cfg.shard(start_layer, end_layer)
    model = build_stage(cfg, spec, dtype, device, backend)
    model.expert_shard = expert_shard
    sd = dict(shard_expert_tensors(random_state_dict(cfg, spec, dtype=dtype, device=device, seed=seed, quantization=quantization),
                                   cfg.n_routed_experts or 0, expert_shard))
    model.load_state(sd, adapter=adapter)
    return model
