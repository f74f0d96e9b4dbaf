#!/usr/bin/env python
"""Greedy CLI generator that drives a sharded model (reference ``generate.py``).

Same flags as the reference (``generate.py:12-20``): ``--model`` (the first shard), ``--prompt``,
``--max_tokens`` (512), ``--server_address`` (comma list of the remaining stages, in pipeline order),
``--start_layer`` / ``--end_layer``.  Differences: remote stages are optional (a single process holding
every layer works — the reference raises without at least one stub, generate.py:72-80); under
``torchrun`` the remaining stages are the other ranks (native chain, no gRPC).

Prints the generated text as it streams, then ``Prompt: X tokens-per-sec`` and
``Generation: Y tokens-per-sec`` like the reference (generate.py:114-122).
"""
import argparse
import os
import sys
import time

from mlx_sharding_b200.engine.core import LLMEngine
from mlx_sharding_b200.engine.sampler import SamplingParams
from mlx_sharding_b200.engine.tokenizer import load_tokenizer


def build_engine(model, server_address, num_pages=None, page_size=64):
    from mlx_sharding_b200.parallel.pipeline import ChainPipeline, LocalPipeline, StageExecutor

    num_pages = num_pages or 1024
    stage = StageExecutor(model, num_pages, page_size)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        # native chain: shared-memory launch ring + fused P2P hand-off on CUDA (gloo / NCCL send-recv elsewhere)
        return LLMEngine(ChainPipeline.build(stage, num_groups=1, max_tokens=2048, max_seqs=64), num_pages, page_size,
                         num_groups=1, max_prefill_tokens=2048)
    if not model.spec.is_last:
        from mlx_sharding_b200.parallel.grpc_compat import GrpcRelayPipeline, connect_stubs

        stubs = connect_stubs(server_address)
        if not stubs:
            raise ValueError("No gRPC stubs provided but the local model does not hold the last layer")
        for s in stubs:
            s.reset_cache()
        return LLMEngine(GrpcRelayPipeline(stage, stubs), num_pages, page_size, num_groups=1, max_seqs_per_group=1)
    return LLMEngine(LocalPipeline([stage]), num_pages, page_size, num_groups=1)


def stream_generate(engine, tokenizer, prompt: str, max_tokens: int):
    """Yield text segments; prints prompt / generation tokens-per-sec at the end (reference :90-122)."""
    ids = tokenizer.encode(prompt)
    detok = tokenizer.new_detokenizer()
    tic = time.perf_counter()
    req = engine.submit(ids, SamplingParams(temperature=0.0), max_tokens=max_tokens,
                        eos_token_id=tokenizer.eos_token_id)
    n, prompt_time = 0, None
    while not req.finished:
        engine.step()
        while not req.events.empty():
            ev = req.events.get()
            if ev is None or ev.token < 0:
                break
            if n == 0:
                prompt_time = time.perf_counter() - tic
                tic = time.perf_counter()
            n += 1
            if ev.finished and ev.finish_reason == "stop":
                break
            detok.add_token(ev.token)
            yield detok.last_segment
    if req.error:
        raise req.error
    detok.finalize()
    yield detok.last_segment
    gen_time = time.perf_counter() - tic
    print("\n" + "=" * 10)
    if n == 0:
        print("No tokens generated for this prompt")
        return
    print(f"Prompt: {len(ids) / max(prompt_time, 1e-9):.3f} tokens-per-sec")
    print(f"Generation: {(n - 1) / max(gen_time, 1e-9):.3f} tokens-per-sec")


def main(argv=None):
    parser = argparse.ArgumentParser(description="Generate text with a sharded model")
    parser.add_argument("--model", type=str, default="shard_0", help="Path to the (first shard of the) model")
    parser.add_argument("--prompt", type=str, default="Hello, how are you?", help="Input prompt")
    parser.add_argument("--max_tokens", type=int, default=512, help="Maximum number of tokens to generate")
    parser.add_argument("--server_address", type=str, default="localhost:50051",
                        help="Comma-separated addresses of the remaining pipeline stages")
    parser.add_argument("--start_layer", type=int, default=None, help="Start layer index")
    parser.add_argument("--end_layer", type=int, default=None, help="End layer index")
    parser.add_argument("--device", type=str, default=None)
    parser.add_argument("--no_chat_template", action="store_true", help="feed the raw prompt")
    parser.add_argument("--expert_parallel", action="store_true",
                        help="under torchrun, MoE models: every rank runs all layers (attention replicated) and holds E/world routed "
                             "experts of every MoE layer, exchanged with the fused all-to-all (parallel/ep.py) instead of a layer pipeline")
    args = parser.parse_args(argv)

    from mlx_sharding_b200.utils.checkpoint import get_model_path
    from mlx_sharding_b200.utils.loader import load_model

    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1 and args.expert_parallel:
        return main_expert_parallel(args)
    if world > 1:
        from mlx_sharding_b200.parallel.transport import init_distributed

        rank, _ = init_distributed(device=args.device)
        if rank != 0:
            from mlx_sharding_b200.server.shard_server import serve_chain

            return serve_chain(args.model, args.start_layer, args.end_layer, args.device)
        if args.start_layer is None and args.end_layer is None:
            from mlx_sharding_b200.config import ModelConfig
            from mlx_sharding_b200.parallel.partition import balanced_split

            cfg = ModelConfig.from_path(get_model_path(args.model))
            if cfg.start_layer is None:
                spec = balanced_split(cfg, world)[0]  # same rule as server/shard_server.py::serve_chain on the other ranks
                args.start_layer, args.end_layer = spec.start_layer, spec.end_layer
    tokenizer = load_tokenizer(get_model_path(args.model))
    model = load_model(args.model, args.start_layer, args.end_layer, device=args.device)
    prompt = args.prompt
    if not args.no_chat_template and getattr(tokenizer, "chat_template", None):
        prompt = tokenizer.apply_chat_template([{"role": "user", "content": args.prompt}], tokenize=False,
                                               add_generation_prompt=True)
    engine = build_engine(model, args.server_address)
    for seg in stream_generate(engine, tokenizer, prompt, args.max_tokens):
        print(seg, end="", flush=True)
    if hasattr(engine.pipe, "shutdown"):
        engine.pipe.shutdown()


def main_expert_parallel(args):
    """Expert-parallel generation (BASELINE config 5 as a user path): all ranks decode the *same* request in lockstep — the
    per-rank work is the replicated attention plus 1/world of every expert bank; rank 0 prints."""
    import torch
    import torch.distributed as dist

    from mlx_sharding_b200.parallel.ep import enable_expert_parallel
    from mlx_sharding_b200.parallel.pipeline import LocalPipeline, StageExecutor
    from mlx_sharding_b200.parallel.transport import init_distributed
    from mlx_sharding_b200.utils.checkpoint import get_model_path
    from mlx_sharding_b200.utils.loader import load_model

    rank, world = init_distributed(device=args.device)      # NCCL + one GPU per rank, or gloo on CPU
    dev = f"cuda:{torch.cuda.current_device()}" if dist.get_backend() == "nccl" else "cpu"
    tokenizer = load_tokenizer(get_model_path(args.model))
    model = load_model(args.model, device=dev, expert_shard=(rank, world))
    max_prefill = 2048
    enable_expert_parallel(model, max_tokens=max_prefill)
    num_pages, page_size = 1024, 64
    engine = LLMEngine(LocalPipeline([StageExecutor(model, num_pages, page_size)]), num_pages, page_size, num_groups=1,
                       max_prefill_tokens=max_prefill)
    prompt = args.prompt
    if not args.no_chat_template and getattr(tokenizer, "chat_template", None):
        prompt = tokenizer.apply_chat_template([{"role": "user", "content": args.prompt}], tokenize=False,
                                               add_generation_prompt=True)
    out = sys.stdout if rank == 0 else open(os.devnull, "w")
    stdout, sys.stdout = sys.stdout, out   # stream_generate prints its statistics: rank 0 only
    try:
        for seg in stream_generate(engine, tokenizer, prompt, args.max_tokens):
            print(seg, end="", flush=True)
    finally:
        sys.stdout = stdout
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1:])
