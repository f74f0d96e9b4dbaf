"""``parallel/decode_loop.py`` on CPU (gloo): the device-resident decode loop in its eager / send-recv form — the code path of
``bench.py --impl baseline`` — must produce the tokens of a single-process greedy run, for whole-layer and half-layer splits."""
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

from helpers import TINY_DSV2, TINY_LLAMA, run_sequence


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, C, half, q):
    import torch.distributed as dist

    from mlx_sharding_b200.config import ModelConfig
    from mlx_sharding_b200.ops.meta import BatchMeta
    from mlx_sharding_b200.parallel.decode_loop import DecodeLoop
    from mlx_sharding_b200.parallel.partition import balanced_split
    from mlx_sharding_b200.parallel.pipeline import StageExecutor
    from mlx_sharding_b200.utils.loader import random_model

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    cfg = ModelConfig.from_dict(C)
    spec = balanced_split(cfg, world, half_layers=half)[rank]
    model = random_model(C, dtype=torch.float32, spec=spec)
    G, B, S, PS, steps = world, 3, 6, 4, 4
    pages_per_seq = (S + steps + 2 + PS - 1) // PS
    stage = StageExecutor(model, G * B * pages_per_seq + 1, PS)
    prompts = torch.randint(3, cfg.vocab_size - 1, (G, B, S), generator=torch.Generator().manual_seed(3))
    bts = [[[1 + (g * B + b) * pages_per_seq + i for i in range(pages_per_seq)] for b in range(B)] for g in range(G)]
    firsts = []
    for g in range(G):                                    # prefill through the chain with plain send / recv
        meta = BatchMeta.build([S] * B, [0] * B, bts[g], PS)
        x = prompts[g].reshape(-1) if rank == 0 else torch.empty(B * S, cfg.hidden_size)
        if rank > 0:
            dist.recv(x, rank - 1)
        out = stage.forward(x, meta)
        if rank < world - 1:
            dist.send(out, rank + 1)
            toks = torch.empty(B, dtype=torch.int64)
        else:
            toks = out.argmax(-1)
        dist.broadcast(toks, world - 1)
        firsts.append(toks)
    loop = DecodeLoop(stage, G, B, pages_per_seq, transport="nccl", use_graphs=False)   # "nccl" = torch.distributed send/recv
    for g in range(G):
        loop.groups[g].load(torch.full((B,), S, dtype=torch.int32), torch.tensor(bts[g], dtype=torch.int32), firsts[g], S + steps + 2)
    loop.capture()
    hist = [[firsts[g].clone()] for g in range(G)]
    for s in range(steps):
        loop.step_all()
        if rank == 0 and s > 0:                          # after step s, stage 0 has received the tokens of step s-1
            for g in range(G):
                hist[g].append(loop.groups[g].tokens.clone())
    loop.drain()
    if rank == 0:
        for g in range(G):
            hist[g].append(loop.groups[g].tokens.clone())
        # numpy arrays travel by value; a tensor put on the queue is handed over as a shared-memory file descriptor, which the
        # parent can only fetch from this process while it is alive, and it exits right after the barrier below
        q.put((prompts.numpy(), [torch.stack(h).numpy() for h in hist]))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(240)
@pytest.mark.parametrize("C,world,half", [(TINY_LLAMA, 2, False), (TINY_DSV2, 3, True)], ids=["llama-pp2", "dsv2-pp3-half"])
def test_decode_loop_send_recv_matches_single_process(C, world, half):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, C, half, q)) for r in range(world)]
    for p in procs:
        p.start()
    prompts, hist = q.get(timeout=200)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    from mlx_sharding_b200.utils.loader import random_model

    full = random_model(C, dtype=torch.float32)
    G, B, _ = prompts.shape
    for g in range(G):
        for b in range(B):
            ref = [int(o.argmax()) for o in run_sequence([full], prompts[g, b].tolist(), hist[g].shape[0] - 1, page_size=4)]
            assert hist[g][:, b].tolist() == ref, (g, b)
