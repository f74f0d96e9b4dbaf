"""Packaging (reference setup.py: package ``mlx-sharding``, console scripts ``mlx-sharding-server`` and
``mlx-sharding-api``, proto + static UI shipped as package data).  The CUDA extension is built in-tree by
``python -m mlx_sharding_b200.ops.build`` (or ``__graft_entry__.build()``), not by setuptools."""
from setuptools import find_packages, setup

setup(
    name="mlx-sharding-b200",
    version="0.1.0",
    description="Hopper-native pipeline-parallel LLM inference engine with the capabilities of mlx_sharding",
    packages=find_packages(include=["mlx_sharding_b200", "mlx_sharding_b200.*", "shard", "shard.*"]),
    py_modules=["generate", "sharding_weight"],
    python_requires=">=3.10",
    install_requires=["torch", "numpy", "safetensors", "transformers", "grpcio", "protobuf"],
    # optional: ``response_format`` (structured output) on the OpenAI server; --model <hub repo id>
    extras_require={"structured": ["xgrammar>=0.2"], "hub": ["huggingface_hub"]},
    entry_points={
        "console_scripts": [
            "mlx-sharding-server=shard.main:main",
            "mlx-sharding-api=shard.openai_api:main",
        ]
    },
    package_data={
        "mlx_sharding_b200": ["server/protos/*.proto", "server/static/*", "ops/csrc/*", "ops/*.so"],
    },
)
