"""Op API.  Two interchangeable implementations of the same function set:

* ``reference`` – pure PyTorch (CPU path, numerical oracle, and — on CUDA tensors — the cuBLAS baseline)
* ``b200``      – hand-written sm_90a CUDA kernels (``ops/csrc``; wgmma/TMA GEMMs, paged flash
                  attention, MoE, sampler, fused P2P stage boundary)

There is no silent fallback: asking for ``b200`` on a box whose extension is missing raises.
"""
from __future__ import annotations

import importlib

from .meta import BatchMeta  # noqa: F401
from .weights import LinearWeight, RopeSpec  # noqa: F401

_BACKENDS = {"reference": ".reference", "b200": ".b200"}


def get_backend(name: str):
    if name not in _BACKENDS:
        raise ValueError(f"unknown ops backend '{name}' (have {list(_BACKENDS)})")
    return importlib.import_module(_BACKENDS[name], __name__)


def default_backend_name(device) -> str:
    import torch

    dev = torch.device(device)
    return "b200" if dev.type == "cuda" else "reference"
