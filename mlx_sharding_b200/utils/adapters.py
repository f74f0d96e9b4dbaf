"""mlx_lm LoRA adapters (``mlx_lm.lora`` output), one per server, applied at load.

An adapter directory holds ``adapter_config.json`` (``fine_tune_type``, ``num_layers`` or the older ``lora_layers``,
``lora_parameters = {rank, scale, dropout, keys}``) and ``adapters.safetensors`` with ``model.layers.{i}.<module>.lora_a``
``[in, r]`` and ``.lora_b`` ``[r, out]``.  An adapted layer computes ``y = x W^T (+ bias) + scale * (x A) B``; ``scale``
multiplies the update directly (it is not alpha / rank) and ``dropout`` does nothing at inference.

Where the update goes (``attach``, called from ``StageModel._lin`` for every linear weight a stage loads):
* dense (bf16) weight: folded once, ``W + scale * (A B)^T`` in fp32 with one rounding -- what ``mlx_lm.fuse`` does for
  unquantised layers; the forward pass is unchanged;
* packed int4 / int8 weight: kept unfused on the ``LinearWeight`` (``lora_a``, ``lora_b_scaled``, rank zero-padded to a multiple
  of 8), because re-quantising would change the base weights; the CUDA backend runs it as a shrink launch plus a term in the
  quantised GEMM epilogue.
"""
from __future__ import annotations

import json
import os
import re
from typing import Dict, Tuple

import torch

from ..ops.weights import LinearWeight

CONFIG_FILE = "adapter_config.json"
WEIGHTS_FILE = "adapters.safetensors"
_KEY_RE = re.compile(r"^model\.layers\.(\d+)\.(.+)\.(lora_a|lora_b)$")


class LoraAdapter(dict):
    """``{module_prefix: (A [in, r], B [r, out])}`` (fp32, mlx_lm orientation; ``B`` without the scale), plus the adapter's
    ``scale``, ``rank``, ``num_layers`` and weights file."""

    def __init__(self, entries: Dict[str, Tuple[torch.Tensor, torch.Tensor]], scale: float, rank: int, num_layers: int,
                 path: str = ""):
        super().__init__(entries)
        self.scale, self.rank, self.num_layers, self.path = float(scale), int(rank), int(num_layers), path

    def subset(self, keep) -> "LoraAdapter":
        return LoraAdapter({k: v for k, v in self.items() if keep(k)}, self.scale, self.rank, self.num_layers, self.path)

    def check_layers(self, num_hidden_layers: int):
        """mlx_lm adapts the last ``num_layers`` blocks of the model (``model.layers[-max(num_layers, 0):]``: ``-1``, which
        ``mlx_lm.lora --num-layers -1`` writes, or any count >= the model's means every block): refuse an entry outside them."""
        n = self.num_layers
        lo = max(num_hidden_layers - n, 0) if 0 < n < num_hidden_layers else 0
        for prefix in sorted(self):
            i = int(prefix.split(".")[2])
            if not lo <= i < num_hidden_layers:
                raise ValueError(f"{self.path}: tensor '{prefix}.lora_a' is in layer {i}, outside the adapted layers "
                                 f"[{lo}, {num_hidden_layers}) (num_layers={n}) of the {num_hidden_layers}-layer model")


def load_adapter(path: str) -> LoraAdapter:
    """Parse and validate an adapter directory (the layer range is checked against the model by ``check_layers``)."""
    from safetensors import safe_open

    cfg_path, w_path = os.path.join(path, CONFIG_FILE), os.path.join(path, WEIGHTS_FILE)
    if not os.path.isfile(cfg_path):
        raise ValueError(f"{cfg_path}: adapter config not found")
    if not os.path.isfile(w_path):
        raise ValueError(f"{w_path}: adapter weights not found")
    with open(cfg_path) as f:
        cfg = json.load(f)
    ftype = cfg.get("fine_tune_type", "dora" if cfg.get("use_dora") else "lora")
    if ftype != "lora" or cfg.get("use_dora"):
        raise ValueError(f"{cfg_path}: fine_tune_type '{'dora' if cfg.get('use_dora') else ftype}' is not supported "
                         "(only 'lora' adapters can be served)")
    num_layers = cfg.get("num_layers", cfg.get("lora_layers"))
    if num_layers is None:
        raise ValueError(f"{cfg_path}: neither 'num_layers' nor 'lora_layers' is set")
    lp = cfg.get("lora_parameters")
    if not isinstance(lp, dict) or "rank" not in lp or "scale" not in lp:
        raise ValueError(f"{cfg_path}: 'lora_parameters' needs 'rank' and 'scale'")
    rank, scale = int(lp["rank"]), float(lp["scale"])

    halves: Dict[str, Dict[str, torch.Tensor]] = {}
    with safe_open(w_path, framework="pt") as f:
        for key in f.keys():
            m = _KEY_RE.match(key)
            if m is None:
                raise ValueError(f"{w_path}: tensor '{key}' is not a 'model.layers.<i>.<module>.lora_a|lora_b' adapter tensor")
            i, module, which = m.group(1), m.group(2), m.group(3)
            if module.startswith(("mlp.switch_mlp", "mlp.experts")):
                raise ValueError(f"{w_path}: tensor '{key}': LoRA on routed experts is not supported")
            t = f.get_tensor(key).float()
            if t.dim() != 2 or t.shape[1 if which == "lora_a" else 0] != rank:
                raise ValueError(f"{w_path}: tensor '{key}' has shape {tuple(t.shape)}, which does not match the config's rank {rank}")
            prefix = f"model.layers.{i}.{module}"
            halves.setdefault(prefix, {})[which] = t
    entries = {}
    for prefix, d in halves.items():
        for have, miss in (("lora_a", "lora_b"), ("lora_b", "lora_a")):
            if have in d and miss not in d:
                raise ValueError(f"{w_path}: tensor '{prefix}.{have}' has no partner '{prefix}.{miss}'")
        entries[prefix] = (d["lora_a"], d["lora_b"])
    return LoraAdapter(entries, scale, rank, int(num_layers), w_path)


def attach(W: LinearWeight, prefix: str, A: torch.Tensor, B: torch.Tensor, scale: float, source: str = "") -> LinearWeight:
    """``W`` with the adapter ``(A [in, r], B [r, out])`` applied: folded into a dense weight, unfused on a packed one.
    ``source`` (the adapter file) names the culprit in errors."""
    if (W.wq if W.is_quantized else W.weight).dim() != 2:
        raise ValueError(f"{source}: tensor '{prefix}.lora_a': only 2-D linear weights take an adapter")
    if A.shape[0] != W.in_features or B.shape[1] != W.out_features:
        raise ValueError(f"{source}: tensor '{prefix}.lora_a' {tuple(A.shape)} / '{prefix}.lora_b' {tuple(B.shape)} do not fit "
                         f"the base weight [out {W.out_features}, in {W.in_features}]")
    if W.is_quantized:
        # rank padded with zeros to a multiple of 8 (exact): the CUDA kernels read 16-byte rows of both tensors
        pad = -A.shape[1] % 8
        W.lora_a = torch.nn.functional.pad(A.t(), (0, 0, 0, pad)).contiguous().to(device=W.device, dtype=torch.bfloat16)
        W.lora_b_scaled = torch.nn.functional.pad(B.t() * scale, (0, pad)).contiguous().to(device=W.device, dtype=torch.bfloat16)
        return W
    dev = W.weight.device
    delta = (A.to(dev, torch.float32) @ B.to(dev, torch.float32)).t() * scale
    W.weight = (W.weight.float() + delta).to(W.weight.dtype).contiguous()
    return W
