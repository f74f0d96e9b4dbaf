# Convenience targets (everything here also works as the plain command shown).
PY ?= python

build:            ## compile the sm_90a extension in-tree (nvcc cross-compiles without a GPU)
	$(PY) -m mlx_sharding_b200.ops.build

test:             ## CPU test suite (models vs HF, engine, gloo chains, expert parallelism over gloo, gRPC, HTTP API, CLIs)
	$(PY) -m pytest tests -q -m "not gpu"

test-gpu:         ## on an H100: kernels vs fp32 oracles, models, multi-GPU parity
	$(PY) -m pytest tests -q -m gpu

bench:            ## headline benchmark on 1 GPU (see bench.py for N > 1 under torchrun)
	$(PY) bench.py

harness:          ## standalone GEMM test binaries (no torch)
	bash tests/cuda/build.sh

.PHONY: build test test-gpu bench harness
