"""``mlx-sharding-server`` — run one non-primary pipeline stage.

Reference: ``shard/main.py:1-17`` (CLI: ``--model`` required, ``-s/--start-layer``, ``-e/--end-layer``) and
``shard/server/server.py:74-93`` (load shard, reset cache, start gRPC on an ephemeral port, print it,
block).  Same flags and behaviour in compat mode (default); extra flags select the native modes:

* ``--port`` (default 0 = ephemeral like the reference), ``--device``, ``--dtype``, ``--wire-dtype``;
* ``--rank/--world-size/--master-addr/--master-port`` (or a torchrun environment): join the native
  chain pipeline (NCCL / fused-P2P on GPUs, gloo on CPU) instead of serving gRPC.
"""
from __future__ import annotations

import argparse
import logging
import os
import sys

import torch

log = logging.getLogger("mlx_sharding_b200.shard_server")


def serve(model_path: str, start_layer=None, end_layer=None, port: int = 0, device=None, dtype=None,
          wire_dtype: str = "float16", num_pages: int = 512, page_size: int = 64, block: bool = True):
    """Compat mode: gRPC ``MLXTensorService`` for one stage (reference ``serve``)."""
    from ..parallel.grpc_compat import DTYPES, StageServicer, start_server
    from ..utils.loader import load_model

    model = load_model(model_path, start_layer, end_layer, dtype=dtype, device=device)
    servicer = StageServicer(model, num_pages=num_pages, page_size=page_size, wire_dtype=DTYPES[wire_dtype])
    server, bound = start_server(servicer, port)
    # the reference prints the port it picked (server.py:90); scripts parse this line
    print(f"Server started, listening on port {bound}", flush=True)
    log.info("stage layers [%d, %d) of %s on %s", model.spec.start_layer, model.spec.end_layer, model_path, model.device)
    if block:
        server.wait_for_termination()
    return server, bound, servicer


def serve_chain(model_path: str, start_layer=None, end_layer=None, device=None, dtype=None, num_pages: int = 2048,
                page_size: int = 64, num_groups=None, max_tokens: int = 2048, max_seqs: int = 64, transport: str = "auto"):
    """Native mode: this process is rank r > 0 of the chain pipeline (see parallel/pipeline.py)."""
    from ..config import ModelConfig
    from ..parallel.partition import balanced_split
    from ..parallel.pipeline import StageExecutor, build_chain, worker_loop
    from ..parallel.transport import init_distributed
    from ..utils.checkpoint import get_model_path
    from ..utils.loader import load_model

    rank, world = init_distributed(device=device)
    if start_layer is None and end_layer is None:
        cfg = ModelConfig.from_path(get_model_path(model_path))
        if cfg.start_layer is None:
            spec = balanced_split(cfg, world)[rank]  # cost-balanced whole layers (LM head / dense layers weighted)
            start_layer, end_layer = spec.start_layer, spec.end_layer
    dev = device or (f"cuda:{torch.cuda.current_device()}" if torch.cuda.is_available() else "cpu")
    model = load_model(model_path, start_layer, end_layer, dtype=dtype, device=dev)
    stage = StageExecutor(model, num_pages, page_size)
    # collective with the front end (openai_api.py / generate.py): same geometry on every rank
    ctl, plane = build_chain(stage, num_groups=num_groups, max_tokens=max_tokens, max_seqs=max_seqs, transport=transport)
    log.info("rank %d/%d serving layers [%d, %d) (hand-off: %s)", rank, world, model.spec.start_layer, model.spec.end_layer, plane.name)
    worker_loop(stage, ctl, plane)


def main(argv=None):
    parser = argparse.ArgumentParser(description="Pipeline-stage server (H100-native mlx-sharding-server)")
    parser.add_argument("--model", type=str, required=True, help="Path to the model or HF repo")
    parser.add_argument("-s", "--start-layer", type=int, default=None, help="Start layer index for model sharding")
    parser.add_argument("-e", "--end-layer", type=int, default=None, help="End layer index for model sharding")
    # extensions
    parser.add_argument("--port", type=int, default=0, help="gRPC port (0 = ephemeral, printed at start-up)")
    parser.add_argument("--device", type=str, default=None)
    parser.add_argument("--dtype", type=str, default=None, choices=["bfloat16", "float16", "float32"])
    parser.add_argument("--wire-dtype", type=str, default="float16", choices=["float16", "bfloat16", "float32"],
                        help="dtype of hidden states on the gRPC wire (reference peers expect float16)")
    parser.add_argument("--kv-pages", type=int, default=None,
                        help="KV pool pages (default 512 for the gRPC servicer; 2048 in the native chain, where every stage must "
                             "use the same pool geometry as the front end because block ids are global)")
    parser.add_argument("--page-size", type=int, default=64)
    parser.add_argument("--log-level", type=str, default="INFO")
    parser.add_argument("--rank", type=int, default=None, help="join the native chain pipeline as this rank")
    parser.add_argument("--world-size", type=int, default=None)
    parser.add_argument("--master-addr", type=str, default="127.0.0.1")
    parser.add_argument("--master-port", type=int, default=29511)
    args = parser.parse_args(argv)
    logging.basicConfig(level=getattr(logging, args.log_level.upper(), logging.INFO),
                        format="%(asctime)s - %(levelname)s - %(message)s")
    dtype = getattr(torch, args.dtype) if args.dtype else None
    native = args.rank is not None or ("RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1)
    if native:
        if args.rank is not None:
            os.environ.update(RANK=str(args.rank), WORLD_SIZE=str(args.world_size or 1),
                              MASTER_ADDR=args.master_addr, MASTER_PORT=str(args.master_port))
        serve_chain(args.model, args.start_layer, args.end_layer, args.device, dtype, args.kv_pages or 2048, args.page_size)
    else:
        serve(args.model, args.start_layer, args.end_layer, args.port, args.device, dtype, args.wire_dtype,
              args.kv_pages or 512, args.page_size)


if __name__ == "__main__":
    main(sys.argv[1:])
