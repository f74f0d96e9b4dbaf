"""Import-path compatibility with mzbac/mlx_sharding: ``shard.main:main`` and ``shard.openai_api:main``
(the reference's console-script targets, setup.py:27-32) resolve to the H100-native implementations."""
