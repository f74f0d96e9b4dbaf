"""Expert parallelism for DeepSeek MoE blocks with a fused all-to-all over NVSwitch peer memory
(BASELINE config 5; SURVEY §2.4 "EP", K11-EP).

The reference executes all routed experts of a layer on the stage that owns the layer (``mx.gather_qmm``).
``ExpertParallelMoE`` shards the ``E`` routed experts of a layer across the ``world`` ranks of one NVSwitch
domain: rank ``r`` keeps experts ``[r*E/world, (r+1)*E/world)`` (1/world of the MoE weights — the dominant
HBM stream of a decode step) and every rank routes *its own* tokens.  Token exchange is done by the kernels
in ``ops/csrc/ep.cu`` — dispatch rows are written straight into the owner's receive region, expert outputs
are stored straight into the source's return buffer by the down-projection GEMM epilogue, publication words /
flags use release/acquire at system scope; there is no NCCL call and no host involvement on the path.

``forward(x, idx, w, residual)`` == ``ops.moe_experts`` on the un-sharded weights (verified in
``tests/test_multigpu.py``).
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.distributed as dist

from ..ops.weights import LinearWeight


class EPBuffers:
    """IPC-mapped receive / return buffers of one rank (shared by all MoE layers of that rank).

    Layout of the mapped region: ``[E_local][world * max_tokens][H]`` bf16 receive rows (expert-major, written by the senders) |
    their return addresses (u64) | ``[2][E_local]`` int32 row counters (double-buffered by step parity) | one u64 arrival word per
    source (the step's sequence number, released by the source's dispatch) | the fp32 return rows of this rank's own pairs |
    flags (the return flag every destination's down-projection bumps)."""

    def __init__(self, hidden: int, max_tokens: int, top_k: int, experts_per_rank: int, group=None):
        from ..ops import b200

        self.C = b200.load_extension()
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self.dev = torch.cuda.current_device()
        self.H, self.top_k = hidden, top_k
        self.max_tokens = max_tokens
        self.E_local = experts_per_rank
        self.cap = max_tokens * top_k                      # pairs one rank can route per step
        W, cap, H = self.world, self.cap, hidden
        rows = experts_per_rank * W * max_tokens
        self.off_recv_x = 0
        self.off_row_dst = self.off_recv_x + rows * H * 2
        self.off_cnt = self.off_row_dst + rows * 8
        self.off_arrive = (self.off_cnt + 2 * experts_per_rank * 4 + 255) // 256 * 256
        self.off_ret_y = (self.off_arrive + W * 8 + 255) // 256 * 256
        self.off_flags = self.off_ret_y + cap * H * 4
        self.off_ret_flag = self.off_flags + 128
        total = self.off_flags + 256
        self.base, handle = self.C.ipc_alloc(total)
        handles: List = [None] * W
        dist.all_gather_object(handles, (handle, self.dev), group=group)
        self.peer = []
        for r, (h, pdev) in enumerate(handles):
            if r == self.rank:
                self.peer.append(self.base)
            else:
                if pdev != self.dev:
                    self.C.enable_peer_access(pdev)
                self.peer.append(self.C.ipc_open(h))
        # tables of peer addresses, one per rank
        self.t_recv_x = [p + self.off_recv_x for p in self.peer]
        self.t_row_dst = [p + self.off_row_dst for p in self.peer]
        self.t_cnt = [p + self.off_cnt for p in self.peer]
        self.t_arrive = [p + self.off_arrive for p in self.peer]
        # my return buffer as mapped by every destination (the address a destination's down-projection epilogue stores to)
        peers_all: List = [None] * W
        dist.all_gather_object(peers_all, list(self.peer), group=group)
        self.t_my_ret = [peers_all[d][self.rank] + self.off_ret_y for d in range(W)]
        self.cnt = self.C.tensor_from_ptr(self.base + self.off_cnt, [2 * experts_per_rank], "int32", self.dev)
        self.arrive = self.base + self.off_arrive          # the W arrival words the grouped gate/up GEMM acquires
        self.ret_flag = self.base + self.off_ret_flag      # my return flag, bumped by every destination's down-projection
        self.ret_flags_dev = torch.tensor([p + self.off_ret_flag for p in self.peer], dtype=torch.int64, device="cuda")
        self._views = {}
        # device-resident step state; every field is a one-element view, passed to the kernels by pointer
        self.state = torch.zeros(5, dtype=torch.int32, device="cuda")
        self.send_seq = self.state[0:1]          # dispatch step sequence number (also what the arrival wait expects)
        self.done_counter = self.state[1:2]      # dispatch CTAs arrived (the last one publishes)
        self.down_tiles = self.state[2:3]        # down-projection tiles stored (the last CTA signals every source)
        self.ret_expected = self.state[3:4]      # return-flag value the combine of this step waits for
        self.error_word = self.state[4:5]        # set by any wait that times out
        self.error_ptr = self.error_word.data_ptr()
        self.ret_y = self.C.tensor_from_ptr(self.base + self.off_ret_y, [cap, H], "float32", self.dev)
        dist.barrier(group=group)

    def error(self) -> bool:
        return bool(self.error_word.item())

    def recv_views(self, stride: int):
        """(rows [E_local * stride, H] bf16, row_dst [E_local * stride] int64) over the receive buffer for this step's stride."""
        v = self._views.get(stride)
        if v is None:
            R = self.E_local * stride
            v = self._views[stride] = (self.C.tensor_from_ptr(self.base + self.off_recv_x, [R, self.H], "bfloat16", self.dev),
                                       self.C.tensor_from_ptr(self.base + self.off_row_dst, [R], "int64", self.dev))
        return v

    def dispatch_args(self, stride: int):
        """Arguments of both dispatch launches after ``experts_per_rank, my_rank``: receive stride, peer tables, step state."""
        return (stride, self.t_recv_x, self.t_row_dst, self.t_cnt, self.t_arrive, self.t_my_ret, self.send_seq, self.done_counter,
                self.ret_expected)


class ExpertParallelMoE:
    """One MoE layer's routed experts, sharded over the ranks of ``bufs``.  A step is four launches: dispatch (slot reservation at
    the sender; on its own, or folded into the router by ``route_forward``) -> grouped gate/up GEMM (acquires the arrivals itself)
    -> grouped down GEMM (its epilogue returns the rows) -> combine."""

    def __init__(self, bufs: EPBuffers, Wg: LinearWeight, Wu: LinearWeight, Wd: LinearWeight, num_experts: int,
                 act: str = "silu", weights_are_local: bool = False):
        from ..ops import b200

        self.b = bufs
        self.ops = b200
        self.E = num_experts
        assert num_experts % bufs.world == 0
        self.E_local = num_experts // bufs.world
        lo, hi = bufs.rank * self.E_local, (bufs.rank + 1) * self.E_local
        pick = (lambda W: b200._dense(W)) if weights_are_local else (lambda W: b200._dense(W)[lo:hi].contiguous())
        self.wg, self.wu, self.wd = pick(Wg), pick(Wu), pick(Wd)
        self.act = b200.ACT_IDS[act]

    def _stride(self, Tmax: int) -> int:
        """Receive rows per expert this step: ``world * Tmax`` rounded up to 64 (every rank computes the same value: ranks step in
        lock-step with equal batch shapes, or pass ``peer_tokens``)."""
        b = self.b
        return min(b.world * b.max_tokens, (b.world * Tmax + 63) // 64 * 64)

    def forward(self, x: torch.Tensor, idx: torch.Tensor, w: torch.Tensor, residual: Optional[torch.Tensor] = None,
                out: Optional[torch.Tensor] = None, peer_tokens: Optional[int] = None, join=None) -> torch.Tensor:
        """``peer_tokens``: upper bound of the tokens *any* rank routes in this step (default: this rank's own ``T`` —
        ranks stepping in lockstep with equal batch shapes); only sizes the receive stride and the local expert GEMMs."""
        b = self.b
        T, k = idx.shape
        assert T * k <= b.cap, "token batch exceeds the EP buffer capacity"
        Tmax = max(T, peer_tokens or getattr(self, "peer_tokens_default", 0) or 0)
        stride = self._stride(Tmax)
        b.C.ep_dispatch_scatter(x, idx, self.E_local, b.rank, *b.dispatch_args(stride))
        return self._experts_and_combine(T * k, Tmax, stride, w, residual, out, join)

    def route_forward(self, h, gate_w, route_kw: dict, pre_norm, residual_fn, out=None, next_norm=None):
        """The whole expert-parallel block as FOUR kernels (1 <= T <= 1024): router with the pre-MoE RMSNorm and the dispatch
        folded in (``moe.cu``: the token's CTA reserves its pairs' slots on the owners with remote atomics, stores the normalised
        row there and takes part in the publication) -> grouped gate/up GEMM -> grouped down GEMM -> combine with the next layer's
        input norm folded in.

        ``h``: un-normalised residual stream; ``pre_norm = (weight, eps)``; ``residual_fn(normed)`` -> ``(residual, join)``: called
        right after the router so the shared-expert branch (which consumes ``normed``) forks onto the side stream behind it;
        ``next_norm = (weight, eps)`` or None.  Returns ``out`` or ``(out, normed_next)``."""
        b, C = self.b, self.b.C
        from ..ops import b200 as O

        T = h.shape[0]
        k = int(route_kw["top_k"])
        assert 1 <= T <= 1024 and T * k <= b.cap
        Tmax = max(T, getattr(self, "peer_tokens_default", 0) or 0)
        stride = self._stride(Tmax)
        rk = dict(route_kw)
        if rk.pop("method", "greedy") != "group_limited_greedy":
            rk["n_group"], rk["topk_group"] = 1, 1
        normed = torch.empty_like(h)
        idx, w = C.ep_route_dispatch(h, O._bf16(gate_w), k, int(rk["n_group"]), int(rk["topk_group"]), float(rk["scaling"]),
                                     bool(rk["norm_topk"]), self.E_local, b.rank, *b.dispatch_args(stride),
                                     O._bf16(pre_norm[0]), float(pre_norm[1]), normed)
        residual, join = residual_fn(normed)
        fuse_norm = next_norm is not None and h.shape[1] <= 8192
        nxt = torch.empty_like(h) if fuse_norm else None
        res = self._experts_and_combine(T * k, Tmax, stride, w, residual, out, join, next_norm if fuse_norm else None, nxt)
        if next_norm is None:
            return res
        return res, (nxt if fuse_norm else O.rmsnorm(res, next_norm[0], next_norm[1]))

    def _experts_and_combine(self, npairs, Tmax, stride, w, residual, out, join, norm=None, normed=None):
        """Grouped gate/up (waits for every source's arrival word) -> grouped down (its epilogue stores each output row into the
        source's return buffer and the last CTA bumps every source's return flag) -> combine (waits for all returns; + residual,
        + ``norm = (weight, eps)`` into ``normed``)."""
        b, C = self.b, self.b.C
        rows, row_dst = b.recv_views(stride)
        max_rows = min(b.world * Tmax, stride)   # upper bound of rows one expert can receive (every rank sends <= Tmax)
        exp_rows = npairs                        # balanced routing: a rank receives about as many pairs as it sends
        wait = (stride, b.arrive, b.send_seq, b.error_ptr, b.world)
        h = C.grouped_linear(rows, self.wg, self.wu, b.cnt, max_rows, self.act, False, None, None, None, exp_rows, *wait, True)
        C.grouped_linear(h, self.wd, None, b.cnt, max_rows, 0, True, row_dst, b.ret_flags_dev, b.down_tiles, exp_rows, *wait, False)
        if join is not None:
            join.wait()   # ``residual`` (shared-expert branch) is produced on the side stream
        if norm is None:
            return C.ep_combine(b.ret_flag, b.ret_expected, b.error_ptr, b.ret_y, w, residual, out)
        return C.ep_combine(b.ret_flag, b.ret_expected, b.error_ptr, b.ret_y, w, residual, out, self.ops._bf16(norm[0]),
                            float(norm[1]), normed)


class ExpertParallelMoERef:
    """Backend-agnostic expert parallelism: the same exchange expressed with ``torch.distributed.all_to_all_single`` (gloo on
    CPU, NCCL on GPU) and the ``ops.reference`` expert math.  It is the CPU path of ``enable_expert_parallel`` (tests, plumbing
    without a GPU) and the NCCL baseline the fused kernels of ``ops/csrc/ep.cu`` are compared against.

    Same contract as :class:`ExpertParallelMoE`: ``forward(x, idx, w, residual)`` == ``ops.moe_experts`` on the un-sharded
    weights; every rank must call it the same number of times (token counts may differ per rank)."""

    def __init__(self, Wg: LinearWeight, Wu: LinearWeight, Wd: LinearWeight, num_experts: int, act: str = "silu",
                 weights_are_local: bool = False, group=None):
        from ..ops import reference as R

        self.R, self.group, self.act = R, group, act
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        assert num_experts % self.world == 0
        self.E, self.E_local = num_experts, num_experts // self.world
        lo, hi = self.rank * self.E_local, (self.rank + 1) * self.E_local
        pick = (lambda W: W) if weights_are_local else (lambda W: W.slice_experts(lo, hi))
        self.wg, self.wu, self.wd = pick(Wg), pick(Wu), pick(Wd)

    def _a2a(self, send: torch.Tensor, send_counts: List[int], recv_counts: List[int]) -> torch.Tensor:
        recv = send.new_empty((sum(recv_counts),) + tuple(send.shape[1:]))
        dist.all_to_all_single(recv, send.contiguous(), recv_counts, send_counts, group=self.group)
        return recv

    def forward(self, x: torch.Tensor, idx: torch.Tensor, w: torch.Tensor, residual: Optional[torch.Tensor] = None,
                out: Optional[torch.Tensor] = None, peer_tokens: Optional[int] = None, join=None) -> torch.Tensor:
        T, k = idx.shape
        W, R = self.world, self.R
        flat = idx.reshape(-1).long()
        dst = flat // self.E_local
        order = torch.argsort(dst, stable=True)                       # pairs grouped by destination rank
        send_counts = torch.bincount(dst, minlength=W)
        recv_counts = torch.empty_like(send_counts)
        dist.all_to_all_single(recv_counts, send_counts, group=self.group)
        sc, rc = send_counts.tolist(), recv_counts.tolist()
        rows = self._a2a(x[order // k], sc, rc)                       # token rows, one per (token, expert) pair
        local_e = self._a2a((flat[order] % self.E_local).to(torch.int64), sc, rc)
        # my experts on what I received (fp32 output rows, weight 1: the routing weight is applied by the source)
        y = torch.zeros(rows.shape[0], x.shape[1], dtype=torch.float32, device=x.device)
        for e in range(self.E_local):
            sel = torch.where(local_e == e)[0]
            if sel.numel():
                h = R.gated_up(rows[sel], self.wg.select_expert(e), self.wu.select_expert(e), self.act)
                y[sel] = R.linear(h, self.wd.select_expert(e), out_dtype=torch.float32)
        back = self._a2a(y, rc, sc)                                    # rows return in the order they were sent
        pair_y = torch.empty_like(back)
        pair_y[order] = back
        res = (pair_y.view(T, k, -1) * w.float().unsqueeze(-1)).sum(1)
        if residual is not None:
            res = res + residual.float()
        res = res.to(x.dtype)
        if out is not None:
            out.copy_(res)
            return out
        return res


def enable_expert_parallel(model, max_tokens: int = 256, group=None):
    """Switch a DeepSeek-V2 stage model (every rank holding the *same* layers, data-parallel over tokens) to
    expert-parallel execution: each MoE layer keeps only its ``E / world`` local experts and routes tokens through the
    expert all-to-all — the fused NVLink kernels (:class:`ExpertParallelMoE`) on the ``b200`` backend, ``all_to_all`` collectives
    (:class:`ExpertParallelMoERef`) on the reference backend.  Models loaded with ``expert_shard=(rank, world)``
    (``utils/loader.py``) already hold just their slice; otherwise the full banks are sliced here and dropped from this rank
    afterwards (1/world of the MoE memory).  Returns the :class:`EPBuffers` (``None`` on the reference backend)."""
    cfg = model.cfg
    local = getattr(model, "expert_shard", None) is not None
    if local:
        assert tuple(model.expert_shard) == (dist.get_rank(group), dist.get_world_size(group)), \
            "model was loaded for a different expert shard"
    if hasattr(model, "unfuse_shared_experts"):
        model.unfuse_shared_experts()     # shared experts were appended to the (un-sharded) routed bank: split them off again
    fused = model.backend_name == "b200"
    world = dist.get_world_size(group)
    bufs = EPBuffers(cfg.hidden_size, max_tokens, cfg.num_experts_per_tok, cfg.n_routed_experts // world, group=group) if fused else None
    model.ep_layers = {}
    for i, w in model.layer_weights.items():
        if "router" not in w:
            continue
        if fused:
            model.ep_layers[i] = ExpertParallelMoE(bufs, w["e_gate"], w["e_up"], w["e_down"], cfg.n_routed_experts,
                                                   weights_are_local=local)
        else:
            model.ep_layers[i] = ExpertParallelMoERef(w["e_gate"], w["e_up"], w["e_down"], cfg.n_routed_experts,
                                                      weights_are_local=local, group=group)
        for k in ("e_gate", "e_up", "e_down"):
            w[k] = None  # the (sliced) bank lives on in the expert-parallel layer object
    if fused:
        torch.cuda.empty_cache()
    return bufs
