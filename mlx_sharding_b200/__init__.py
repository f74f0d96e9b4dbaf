"""mlx_sharding_b200 — a Hopper (H100 / sm_90a) native pipeline-parallel LLM
inference engine with the capabilities of ``mzbac/mlx_sharding``.

Layer map (ours; see SURVEY.md §7.1):

* ``models/``   – config parsing, layer-range shard spec, Llama / Gemma-2 / DeepSeek-V2 stage models
* ``ops/``      – op API with two implementations: pure-PyTorch oracle and hand-written sm_90a CUDA
* ``engine/``   – paged KV cache, sampler, scheduler, generation driver, tokenizer utilities
* ``parallel/`` – stage-to-stage transports (fused P2P, NCCL, gloo, gRPC-compat), pipeline runtime, EP
* ``server/``   – ``mlx-sharding-server`` / ``mlx-sharding-api`` entry points, OpenAI HTTP API, web UI
* ``utils/``    – MLX-layout checkpoint IO, affine int4/int8 (un)packing, pre-splitter, timing
"""

__version__ = "0.1.0"

from .config import ModelConfig, ShardSpec  # noqa: F401
