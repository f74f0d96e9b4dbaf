"""Tier T0: fused peer-to-peer stage boundary over NVLink 5 / NVSwitch (SURVEY §5.8, call sites X1/X3).

Every rank owns a *resident inbox* per micro-batch group — hidden states ``[G, max_tokens, H]`` bf16, a
token inbox ``[G, max_seqs]`` int64 (stage 0 only receives into it) and one counting flag per group —
allocated with ``cudaMalloc`` and exported through CUDA IPC.  After the handle exchange
(``torch.distributed`` object all-gather on the control group) stage ``i`` holds a device pointer into
stage ``i+1``'s inbox, and the last stage one into stage 0's token inbox.

Hand-off = the *last kernel of the stage* (the down-proj wgmma GEMM epilogue for dense layers, the
MoE weighted-combine for DeepSeek MoE layers) stores its output rows straight into the peer inbox and
the last CTA bumps the peer's flag with a system-scope release (``models/base.py::_final_kwargs``,
``csrc/gemm_splitk.cu``, ``csrc/moe.cu``).  The consumer's step begins with a one-thread
``wait_flag_counter`` kernel (acquire.sys spin, bounded) — so a decode step is a single CUDA-graph
launch per stage with **no NCCL call, no host hop and no host->device traffic**.  Compare with the
reference: one blocking gRPC unary call per stage per token, host-staged fp16 (shard/utils.py:71-90,162-164).

Flags count completed hand-offs (``atomicAdd.sys``) and consumers keep their own arrival counter in
device memory, which makes the captured graphs replay-safe without baked step numbers.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List

import torch
import torch.distributed as dist


@dataclass
class _Region:
    ptr: int
    nbytes: int


class FusedP2PBoundary:
    """IPC-mapped inboxes + flags for a chain of ``world`` stages on one NVSwitch domain."""

    FLAG_STRIDE = 32  # uint32 elements between flags: one flag per 128 B line

    def __init__(self, hidden_size: int, num_groups: int, max_tokens: int, max_seqs: int, group=None,
                 dtype=torch.bfloat16, result_bytes: int = 0):
        """``result_bytes``: size of stage 0's per-group result inbox (sampled ids + log-probs [+ top-k], see
        ``graph_decode.ResultLayout``); defaults to the bare token ids (``max_seqs`` int64)."""
        from ..ops import b200

        self.C = b200.load_extension()
        self.group = group
        self.rank = dist.get_rank()
        self.world = dist.get_world_size()
        self.dev = torch.cuda.current_device()
        self.H, self.G, self.max_tokens, self.max_seqs = hidden_size, num_groups, max_tokens, max_seqs
        itemsize = torch.empty((), dtype=dtype).element_size()
        self.hidden_bytes = num_groups * max_tokens * hidden_size * itemsize
        self.result_stride = max((max(result_bytes, max_seqs * 8) + 255) // 256 * 256, 256)
        self.token_bytes = num_groups * self.result_stride
        self.flag_bytes = 2 * num_groups * self.FLAG_STRIDE * 4   # [hidden flags | token flags]
        total = self.hidden_bytes + self.token_bytes + self.flag_bytes
        total = (total + 255) // 256 * 256
        self.base, handle = self.C.ipc_alloc(total)
        handles: List = [None] * self.world
        dist.all_gather_object(handles, (handle, self.dev), group=group)
        self.peer_base = {}
        nxt = (self.rank + 1) % self.world
        for peer in {nxt, 0} - {self.rank}:
            h, pdev = handles[peer]
            if pdev != self.dev:
                self.C.enable_peer_access(pdev)
            self.peer_base[peer] = self.C.ipc_open(h)
        self.peer_base[self.rank] = self.base
        self.next_rank = nxt
        # device-resident arrival counters (consumer side) + error word
        self.counters = torch.zeros(2 * num_groups + 1, dtype=torch.int32, device="cuda")
        # host-visible mirror of the error word (mapped pinned memory): a wait kernel that times out sets it, ``error()`` is a plain
        # load — no device synchronisation on the serving path
        self.err_host = torch.zeros(4, dtype=torch.int32).pin_memory()
        dist.barrier(group=group)

    # -- address helpers ---------------------------------------------------------------------------
    def _hidden_ptr(self, base: int, g: int) -> int:
        return base + g * self.max_tokens * self.H * 2

    def _token_ptr(self, base: int, g: int) -> int:
        return base + self.hidden_bytes + g * self.result_stride

    def _flag_ptr(self, base: int, g: int, kind: int) -> int:
        return base + self.hidden_bytes + self.token_bytes + (kind * self.G + g) * self.FLAG_STRIDE * 4

    # my inbox (consumer views)
    def hidden_inbox(self, g: int, rows: int) -> torch.Tensor:
        return self.C.tensor_from_ptr(self._hidden_ptr(self.base, g), [rows, self.H], "bfloat16", self.dev)

    def token_inbox(self, g: int, n: int) -> torch.Tensor:
        return self.C.tensor_from_ptr(self._token_ptr(self.base, g), [n], "int64", self.dev)

    # peer inbox (producer views)
    def next_hidden(self, g: int, rows: int) -> torch.Tensor:
        return self.C.tensor_from_ptr(self._hidden_ptr(self.peer_base[self.next_rank], g), [rows, self.H], "bfloat16", self.dev)

    def next_hidden_flag(self, g: int) -> int:
        return self._flag_ptr(self.peer_base[self.next_rank], g, 0)

    def first_token_ptr(self, g: int) -> int:
        return self._token_ptr(self.peer_base[0], g)

    def first_token_flag(self, g: int) -> int:
        return self._flag_ptr(self.peer_base[0], g, 1)

    # -- stream-ordered primitives -------------------------------------------------------------------
    def wait_hidden(self, g: int):
        self.C.wait_flag_counter(self._flag_ptr(self.base, g, 0), self.counters[g].data_ptr(), self.counters[-1].data_ptr(),
                                 self.err_host.data_ptr())

    def wait_tokens(self, g: int):
        self.C.wait_flag_counter(self._flag_ptr(self.base, g, 1), self.counters[self.G + g].data_ptr(),
                                 self.counters[-1].data_ptr(), self.err_host.data_ptr())

    def send_tokens(self, tokens: torch.Tensor, g: int):
        """Last stage -> stage 0: sampled token ids (8 B per sequence instead of the reference's full
        ``[1, T, V]`` logits, SURVEY X3)."""
        assert tokens.dtype == torch.int64 and tokens.is_contiguous() and (tokens.numel() * 8) % 16 == 0
        self.C.copy_signal(tokens, self.first_token_ptr(g), self.first_token_flag(g), 0)

    def result_inbox(self, g: int, nbytes: int) -> torch.Tensor:
        return self.C.tensor_from_ptr(self._token_ptr(self.base, g), [nbytes], "uint8", self.dev)

    def wait_result(self, g: int):
        self.wait_tokens(g)

    def send_result(self, res: torch.Tensor, g: int):
        """Last stage -> stage 0: the result message of a step (tag, sampled ids, log-probs [, top-k]) in one copy + flag bump."""
        assert res.dtype == torch.uint8 and res.is_contiguous() and res.numel() % 16 == 0 and res.numel() <= self.result_stride
        self.C.copy_signal(res, self.first_token_ptr(g), self.first_token_flag(g), 0)

    def send_hidden(self, x: torch.Tensor, g: int):
        """Un-fused fallback (e.g. Gemma-2, whose last op is a norm): copy kernel + signal."""
        self.C.copy_signal(x.contiguous(), self._hidden_ptr(self.peer_base[self.next_rank], g), self.next_hidden_flag(g), 0)

    def error(self, sync: bool = False) -> bool:
        """True once a flag wait on this device timed out.  Default: read the mapped host mirror (no device sync)."""
        if sync:
            return bool(self.counters[-1].item())
        return bool(self.err_host[0])
