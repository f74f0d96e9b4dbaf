"""Weight containers shared by the PyTorch oracle and the sm_90a kernels.

``LinearWeight`` holds either a dense ``[N, K]`` matrix (row = output feature, K contiguous — the
K-major layout TMA/UMMA want) or the MLX affine-quantised triple (SURVEY U10).  A leading expert
dimension ``[E, N, K]`` is allowed for the stacked ``switch_mlp`` weights of DeepSeek MoE blocks
(reference deepseek_v2.py:101-111 stacks them the same way).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional

import torch

from ..utils import quant


@dataclass
class LinearWeight:
    weight: Optional[torch.Tensor] = None       # dense [.., N, K]
    wq: Optional[torch.Tensor] = None           # uint32/int32 [.., N, K*bits/32]
    scales: Optional[torch.Tensor] = None       # [.., N, K/g]
    biases: Optional[torch.Tensor] = None       # [.., N, K/g]
    bias: Optional[torch.Tensor] = None         # additive bias [N]
    group_size: int = 64
    bits: int = 4

    @property
    def is_quantized(self) -> bool:
        return self.wq is not None

    @property
    def out_features(self) -> int:
        return (self.wq if self.is_quantized else self.weight).shape[-2]

    @property
    def in_features(self) -> int:
        if self.is_quantized:
            return quant.quantized_in_features(self.wq, self.bits)
        return self.weight.shape[-1]

    @property
    def device(self):
        return (self.wq if self.is_quantized else self.weight).device

    def dense(self, dtype: torch.dtype = torch.float32) -> torch.Tensor:
        if self.is_quantized:
            return quant.dequantize(self.wq, self.scales, self.biases, self.group_size, self.bits, dtype)
        return self.weight.to(dtype)

    def dense_cached(self, dtype: torch.dtype) -> torch.Tensor:
        """Dense weight in ``dtype``; quantised weights are expanded once and kept."""
        if not self.is_quantized:
            return self.weight if self.weight.dtype == dtype else self.weight.to(dtype)
        c = getattr(self, "_dense_cache", None)
        if c is None or c.dtype != dtype:
            c = self.dense(dtype)
            self._dense_cache = c
        return c

    def to(self, device=None, dtype=None) -> "LinearWeight":
        def mv(t, cast):
            if t is None:
                return None
            if cast and dtype is not None and t.is_floating_point():
                return t.to(device=device, dtype=dtype)
            return t.to(device=device)

        return LinearWeight(mv(self.weight, True), mv(self.wq, False), mv(self.scales, True),
                            mv(self.biases, True), mv(self.bias, True), self.group_size, self.bits)

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size()
                   for t in (self.weight, self.wq, self.scales, self.biases, self.bias) if t is not None)

    @staticmethod
    def from_state(sd: Dict[str, torch.Tensor], prefix: str, qcfg: Optional[Dict[str, int]] = None,
                   dtype: Optional[torch.dtype] = None, device=None, pop: bool = True) -> "LinearWeight":
        """Build from checkpoint tensors ``{prefix}.weight[/scales/biases/bias]``.

        A module is quantised iff its ``.scales`` key exists (the reference's ``class_predicate``,
        shard/utils.py:56-59)."""
        get = sd.pop if pop else sd.get
        w = get(prefix + ".weight")
        s = get(prefix + ".scales", None)
        b = get(prefix + ".biases", None)
        bias = get(prefix + ".bias", None)

        def cast(t):
            if t is None:
                return None
            if dtype is not None and t.is_floating_point():
                return t.to(device=device, dtype=dtype)
            return t.to(device=device)

        if s is not None:
            if qcfg is None:
                raise ValueError(f"{prefix}: quantised tensors found but config has no 'quantization'")
            if w.dtype == torch.uint32:
                w = w.view(torch.int32)
            # scales / biases keep their stored precision (mlx-community 4/8-bit checkpoints carry fp16 tables; casting them to
            # the bf16 model dtype would cost ~0.4 % per dequantised weight on top of the quantisation error, and the reference
            # dequantises with the stored values)
            return LinearWeight(wq=w.to(device=device), scales=s.to(device=device), biases=b.to(device=device), bias=cast(bias),
                                group_size=int(qcfg["group_size"]), bits=int(qcfg["bits"]))
        return LinearWeight(weight=cast(w), bias=cast(bias))

    @staticmethod
    def concat(ws, dim: int = -2) -> "LinearWeight":
        """Concatenate along the output-feature axis (horizontal GEMM fusion, SURVEY K3/K4)."""
        ws = list(ws)
        q = ws[0].is_quantized
        assert all(w.is_quantized == q for w in ws)
        bias = None
        if any(w.bias is not None for w in ws):
            bias = torch.cat([w.bias if w.bias is not None else
                              torch.zeros(w.out_features, dtype=ws[0].bias.dtype if ws[0].bias is not None
                                          else torch.float32, device=w.device) for w in ws])
        if q:
            return LinearWeight(wq=torch.cat([w.wq for w in ws], dim), scales=torch.cat([w.scales for w in ws], dim),
                                biases=torch.cat([w.biases for w in ws], dim), bias=bias,
                                group_size=ws[0].group_size, bits=ws[0].bits)
        return LinearWeight(weight=torch.cat([w.weight for w in ws], dim), bias=bias)

    def slice_out(self, start: int, end: int) -> "LinearWeight":
        sl = (Ellipsis, slice(start, end), slice(None))
        if self.is_quantized:
            return LinearWeight(wq=self.wq[sl], scales=self.scales[sl], biases=self.biases[sl],
                                bias=None if self.bias is None else self.bias[start:end],
                                group_size=self.group_size, bits=self.bits)
        return LinearWeight(weight=self.weight[sl], bias=None if self.bias is None else self.bias[start:end])

    def slice_experts(self, lo: int, hi: int) -> "LinearWeight":
        """Experts ``[lo, hi)`` of a stacked ``[E, out, in]`` bank (expert parallelism)."""
        if self.is_quantized:
            return LinearWeight(wq=self.wq[lo:hi].contiguous(), scales=self.scales[lo:hi].contiguous(),
                                biases=self.biases[lo:hi].contiguous(), group_size=self.group_size, bits=self.bits)
        return LinearWeight(weight=self.weight[lo:hi].contiguous())

    def select_expert(self, e: int) -> "LinearWeight":
        if self.is_quantized:
            return LinearWeight(wq=self.wq[e], scales=self.scales[e], biases=self.biases[e],
                                group_size=self.group_size, bits=self.bits)
        return LinearWeight(weight=self.weight[e])


@dataclass
class RopeSpec:
    """Rotary embedding description: ``angle = position / freqs`` (MLX convention: ``freqs`` are the
    reciprocals of ``inv_freq``), ``interleaved`` = MLX ``traditional=True`` pair layout."""

    inv_freq: torch.Tensor          # fp32 [rot_dim / 2]
    rot_dim: int
    interleaved: bool = False
    mscale: float = 1.0             # YaRN magnitude scale applied to the rotated slice
