"""MLX affine group quantisation (the on-disk format of ``*-4bit-mlx`` / ``*-8bit`` checkpoints).

Format (SURVEY U10; consumed by the reference through ``nn.quantize`` at shard/utils.py:54-65):

* ``weight``  : ``uint32[out, in * bits / 32]`` – ``32 / bits`` codes per word, **LSB first**
* ``scales``  : ``fp16|bf16[out, in / group_size]``
* ``biases``  : ``fp16|bf16[out, in / group_size]``
* ``w[o, i] = scales[o, i // g] * q[o, i] + biases[o, i // g]``

These helpers are the CPU oracle for the in-kernel dequantisation done by the sm_90a GEMM /
embedding kernels (``ops/csrc``) and are used by the synthetic-checkpoint generator.
"""
from __future__ import annotations

from typing import Tuple

import torch

_SUPPORTED_BITS = (2, 4, 8)


def _as_u32(t: torch.Tensor) -> torch.Tensor:
    """uint32 storage viewed as int64 values in [0, 2^32) (torch has poor uint32 op coverage)."""
    if t.dtype == torch.uint32:
        return t.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    if t.dtype == torch.int32:
        return t.to(torch.int64) & 0xFFFFFFFF
    if t.dtype == torch.int64:
        return t & 0xFFFFFFFF
    raise TypeError(f"packed weight must be uint32/int32, got {t.dtype}")


def unpack_codes(wq: torch.Tensor, bits: int) -> torch.Tensor:
    """``uint32[..., n_words]`` -> ``uint8[..., n_words * 32 / bits]`` integer codes."""
    assert bits in _SUPPORTED_BITS
    per = 32 // bits
    w = _as_u32(wq)
    shifts = torch.arange(per, device=w.device, dtype=torch.int64) * bits
    codes = (w.unsqueeze(-1) >> shifts) & ((1 << bits) - 1)
    return codes.reshape(*wq.shape[:-1], wq.shape[-1] * per).to(torch.uint8)


def pack_codes(codes: torch.Tensor, bits: int) -> torch.Tensor:
    """Inverse of :func:`unpack_codes`; returns an ``int32`` tensor holding the uint32 bit pattern."""
    assert bits in _SUPPORTED_BITS
    per = 32 // bits
    assert codes.shape[-1] % per == 0
    c = codes.to(torch.int64).reshape(*codes.shape[:-1], codes.shape[-1] // per, per)
    shifts = torch.arange(per, device=c.device, dtype=torch.int64) * bits
    words = (c << shifts).sum(-1)
    words = torch.where(words >= 2 ** 31, words - 2 ** 32, words)
    return words.to(torch.int32)


def quantize(w: torch.Tensor, group_size: int = 64, bits: int = 4,
             out_dtype: torch.dtype = torch.float16) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Affine-quantise ``w[..., in]`` the way ``mx.quantize`` does.

    Returns ``(wq uint32-as-int32, scales, biases)``.
    """
    assert w.shape[-1] % group_size == 0, "in-features must be a multiple of group_size"
    n_bins = float((1 << bits) - 1)
    wf = w.float().reshape(*w.shape[:-1], w.shape[-1] // group_size, group_size)
    w_max = wf.amax(-1, keepdim=True)
    w_min = wf.amin(-1, keepdim=True)
    eps = 1e-7
    scale = ((w_max - w_min) / n_bins).clamp_min(eps)
    side = w_min.abs() > w_max.abs()
    scale = torch.where(side, scale, -scale)
    edge = torch.where(side, w_min, w_max)
    q0 = torch.round(edge / scale)
    scale = torch.where(q0 != 0, edge / q0, scale)
    bias = torch.where(q0 == 0, torch.zeros_like(edge), edge)
    # round-trip scale/bias through the storage dtype so dequantisation is exactly reproducible
    scale = scale.to(out_dtype).float()
    bias = bias.to(out_dtype).float()
    safe = torch.where(scale == 0, torch.ones_like(scale), scale)
    q = torch.round((wf - bias) / safe).clamp_(0, n_bins)
    codes = q.to(torch.uint8).reshape(w.shape)
    wq = pack_codes(codes, bits)
    return wq, scale.squeeze(-1).to(out_dtype), bias.squeeze(-1).to(out_dtype)


def dequantize(wq: torch.Tensor, scales: torch.Tensor, biases: torch.Tensor, group_size: int = 64,
               bits: int = 4, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    codes = unpack_codes(wq, bits).float()
    g = codes.reshape(*codes.shape[:-1], codes.shape[-1] // group_size, group_size)
    w = g * scales.float().unsqueeze(-1) + biases.float().unsqueeze(-1)
    return w.reshape(codes.shape).to(dtype)


def quantized_in_features(wq: torch.Tensor, bits: int) -> int:
    return wq.shape[-1] * (32 // bits)


def repack_int4_pairs(wq: torch.Tensor) -> torch.Tensor:
    """Kernel-friendly nibble order for the in-kernel dequant GEMM (same bits, different order): nibble ``j`` of each
    word <- code ``2j``, nibble ``4 + j`` <- code ``2j + 1``, so ``(w >> 4i) & 0x000F000F`` isolates the adjacent pair
    ``(v_2i, v_2i+1)`` as two 16-bit lanes.  Works word-wise (no per-code expansion)."""
    w = _as_u32(wq)
    out = torch.zeros_like(w)
    for j in range(4):
        out |= ((w >> (8 * j)) & 0xF) << (4 * j)
        out |= ((w >> (8 * j + 4)) & 0xF) << (16 + 4 * j)
    out = torch.where(out >= 2 ** 31, out - 2 ** 32, out)
    return out.to(torch.int32)


# ------------------------------------------------------------------------------------------------ MXFP8 (OCP microscaling)
def to_mxfp8(w: torch.Tensor):
    """``w [..., K]`` (any float dtype, ``K % 32 == 0``) -> ``(q uint8 [..., K], sf uint8 [..., K / 32])``: e4m3 elements with one
    shared power-of-two scale (ue8m0, ``2^(sf - 127)``) per 32 consecutive ``K`` values, ``scale = 2^ceil(log2(amax / 448))``.
    The load-time format of weights for ``ops/csrc/gemm_fp8.cu`` (wgmma e4m3 with per-32 block scales); the activation side
    is produced by ``elementwise.cu::quant_mxfp8_kernel`` with the same rule, bit for bit."""
    K = w.shape[-1]
    assert K % 32 == 0
    wf = w.float().reshape(*w.shape[:-1], K // 32, 32)
    v = wf.abs().amax(-1) * (1.0 / 448.0)
    bits = v.contiguous().view(torch.int32)
    e = ((bits >> 23) & 0xFF) + ((bits & 0x7FFFFF) != 0).to(torch.int32)      # biased exponent of the next power of two >= v
    e = e.clamp(max=254)
    inv = ((254 - e) << 23).view(torch.float32)                                # 2^-(e - 127)
    q = (wf * inv.unsqueeze(-1)).to(torch.float8_e4m3fn).view(torch.uint8).reshape(w.shape)
    return q.contiguous(), e.to(torch.uint8).contiguous()


def from_mxfp8(q: torch.Tensor, sf: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """Inverse of :func:`to_mxfp8` (exact: every MXFP8 value is representable in fp32)."""
    K = q.shape[-1]
    scale = ((sf.to(torch.int32)) << 23).view(torch.float32)                   # 2^(sf - 127); sf == 0 -> 0 (block of zeros)
    x = q.view(torch.float8_e4m3fn).float().reshape(*q.shape[:-1], K // 32, 32) * scale.unsqueeze(-1)
    return x.reshape(q.shape).to(dtype)
