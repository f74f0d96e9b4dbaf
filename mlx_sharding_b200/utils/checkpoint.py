"""MLX-community checkpoint IO: shard-aware safetensors loading, the offline pre-splitter and a
synthetic (random-init) checkpoint generator for the offline GPU box.

Reference behaviour being matched:

* key filter by layer range / embed / norm / lm_head — ``shard/server/model/llama.py:92-107``,
  ``gemma2.py:88-102``, ``deepseek_v2.py:86-99`` and ``sharding_weight.py:16-24``;
* pre-split output layout ``model-{start:05d}-{end:05d}.safetensors`` (+ ``.index.json``), ``config.json``
  with ``start_layer`` / ``end_layer``, copied tokenizer files — ``sharding_weight.py:26-71``;
* safetensors metadata ``{"format": "mlx"}`` — ``sharding_weight.py:28``.

Fixed on purpose (SURVEY §2.8): tied-embedding checkpoints keep ``model.embed_tokens`` on the last
shard as well (the reference's splitter forgets the Gemma-2 case).
"""
from __future__ import annotations

import glob
import json
import os
import re
import shutil
from typing import Callable, Dict, Iterable, Iterator, Optional, Tuple

import torch

from ..config import ModelConfig, ShardSpec
from . import quant

_LAYER_RE = re.compile(r"^model\.layers\.(\d+)\.")


_SYNTH_DIRS: Dict[str, str] = {}


def synthetic_model_dir(name: str) -> str:
    """``synthetic:<name>`` model ids (offline boxes, benchmarks): a directory with the canned ``config.json`` of a known
    architecture, a self-contained byte-level tokenizer and a ``synthetic.json`` marker — no weight files.  ``utils/loader.py``
    sees the marker and builds random-init weights of that architecture directly on the device (same key layout / shapes as the
    mlx-community checkpoint), so ``mlx-sharding-api --model synthetic:llama3-8b`` serves a full-size model without a download."""
    import tempfile

    from ..config import deepseek_v2_lite_config, gemma2_9b_config, llama3_8b_config

    tiny = lambda: dict(model_type="llama", vocab_size=320, hidden_size=64, intermediate_size=128, num_hidden_layers=4,
                        num_attention_heads=4, num_key_value_heads=2, rms_norm_eps=1e-5, rope_theta=10000.0,
                        max_position_embeddings=512, tie_word_embeddings=False)
    canned = {"deepseek-v2-lite": deepseek_v2_lite_config, "llama3-8b": llama3_8b_config, "gemma2-9b": gemma2_9b_config,
              "tiny-llama": tiny}
    if name not in canned:
        raise FileNotFoundError(f"unknown synthetic model '{name}' (known: {sorted(canned)})")
    d = _SYNTH_DIRS.get(name)
    if d is None:
        from ..engine.tokenizer import write_byte_tokenizer

        d = tempfile.mkdtemp(prefix=f"mlxb200_synth_{name}_")
        cfg = canned[name]()
        with open(os.path.join(d, "config.json"), "w") as f:
            json.dump(cfg, f)
        with open(os.path.join(d, "synthetic.json"), "w") as f:
            json.dump({"name": name, "seed": 1}, f)
        write_byte_tokenizer(d, vocab_size=min(int(cfg["vocab_size"]), 4096))
        _SYNTH_DIRS[name] = d
    return d


def get_model_path(path_or_hf_repo: str) -> str:
    """Local directory if it exists, else a HF hub snapshot (reference utils.py:34 via mlx_lm); ``synthetic:<name>`` -> see
    :func:`synthetic_model_dir`."""
    if str(path_or_hf_repo).startswith("synthetic:"):
        return synthetic_model_dir(str(path_or_hf_repo).split(":", 1)[1])
    if os.path.isdir(path_or_hf_repo):
        return path_or_hf_repo
    try:
        from huggingface_hub import snapshot_download

        return snapshot_download(
            repo_id=path_or_hf_repo,
            allow_patterns=["*.json", "*.safetensors", "*.py", "tokenizer.model", "*.tiktoken", "*.txt"],
        )
    except Exception as e:  # offline box
        raise FileNotFoundError(
            f"model path '{path_or_hf_repo}' is not a local directory and could not be downloaded: {e}"
        ) from e


def is_attn_key(key: str, model_type: str = "") -> bool:
    """True if a per-layer tensor belongs to the layer's *attention* block (else: its MLP block).  Gemma-2's
    ``post_attention_layernorm`` normalises the attention output; for Llama / DeepSeek that name is the pre-MLP norm."""
    if ".self_attn." in key or ".input_layernorm." in key:
        return True
    return model_type == "gemma2" and ".post_attention_layernorm." in key


def key_in_shard(key: str, spec: ShardSpec, tied_embeddings: bool = False, model_type: str = "") -> bool:
    """True if checkpoint tensor ``key`` belongs to stage ``spec`` (half-layer boundaries included)."""
    if "rotary_emb.inv_freq" in key:
        return False
    m = _LAYER_RE.match(key)
    if m:
        i = int(m.group(1))
        if not spec.owns_layer(i):
            return False
        return spec.runs_attn(i) if is_attn_key(key, model_type) else spec.runs_mlp(i)
    if key.startswith("model.embed_tokens"):
        return spec.is_first or (spec.is_last and tied_embeddings)
    if key.startswith("model.norm") or key.startswith("lm_head"):
        return spec.is_last
    return False


_SWITCH_RE = re.compile(r"\.mlp\.switch_mlp\.(gate_proj|up_proj|down_proj)\.")
_EXPERT_ID_RE = re.compile(r"\.mlp\.experts\.(\d+)\.")


def shard_expert_tensors(items, num_experts: int, expert_shard: Optional[Tuple[int, int]]):
    """Expert parallelism at load time (parallel/ep.py): of every routed-expert bank keep only the experts
    ``[r * E / world, (r + 1) * E / world)`` of rank ``r`` — stacked ``switch_mlp.*`` tensors are sliced as they stream by
    (so a rank never holds more than one full bank at a time), HF-style per-expert tensors of other ranks are dropped."""
    if expert_shard is None:
        yield from items
        return
    r, world = expert_shard
    assert num_experts % world == 0, "n_routed_experts must be divisible by the expert-parallel world size"
    lo, hi = r * num_experts // world, (r + 1) * num_experts // world
    for k, v in items:
        if _SWITCH_RE.search(k):
            yield k, v[lo:hi].clone() if v.is_cuda else v[lo:hi].contiguous()
            continue
        m = _EXPERT_ID_RE.search(k)
        if m is not None and not (lo <= int(m.group(1)) < hi):
            continue
        yield k, v


def iter_safetensors(model_path: str, keep: Optional[Callable[[str], bool]] = None,
                     device: str = "cpu") -> Iterator[Tuple[str, torch.Tensor]]:
    """Yield ``(key, tensor)`` for every tensor of every ``*.safetensors`` under ``model_path`` that
    passes ``keep`` — only those tensors are read from disk (mmap + per-key fetch)."""
    from safetensors import safe_open

    files = sorted(glob.glob(os.path.join(model_path, "*.safetensors")))
    if not files:
        raise FileNotFoundError(f"No safetensors found in {model_path}")
    for fpath in files:
        with safe_open(fpath, framework="pt", device=device) as f:
            for k in f.keys():
                if keep is None or keep(k):
                    yield k, f.get_tensor(k)


def load_shard_tensors(model_path: str, spec: ShardSpec, tied: bool = False,
                       device: str = "cpu", model_type: str = "") -> Dict[str, torch.Tensor]:
    return dict(iter_safetensors(model_path, lambda k: key_in_shard(k, spec, tied, model_type), device=device))


def save_safetensors(path: str, tensors: Dict[str, torch.Tensor]):
    from safetensors.torch import save_file

    out = {}
    for k, t in tensors.items():
        t = t.detach().cpu().contiguous()
        out[k] = t
    save_file(out, path, metadata={"format": "mlx"})


# ---------------------------------------------------------------------------------------------
# Offline pre-splitter (sharding_weight.py equivalent)
# ---------------------------------------------------------------------------------------------
def save_sharded_weights(model: str, output_dir: str, start_layer: int, end_layer: int,
                         total_layers: int) -> str:
    """Write stage ``[start_layer, end_layer)`` of ``model`` into ``output_dir``.

    Layout parity: reference ``sharding_weight.py:11-58``.  Returns the weights file path.
    """
    model_path = get_model_path(model)
    os.makedirs(output_dir, exist_ok=True)
    with open(os.path.join(model_path, "config.json")) as f:
        config = json.load(f)
    spec = ShardSpec(start_layer, end_layer, total_layers)
    tied = bool(config.get("tie_word_embeddings", False)) or config.get("model_type") == "gemma2"
    # a tied head is only needed when no explicit lm_head exists in the checkpoint
    shard = load_shard_tensors(model_path, spec, tied=tied)
    fname = f"model-{start_layer:05d}-{end_layer:05d}.safetensors"
    out_file = os.path.join(output_dir, fname)
    save_safetensors(out_file, shard)

    index_path = os.path.join(model_path, "model.safetensors.index.json")
    if os.path.exists(index_path):
        with open(index_path) as f:
            index = json.load(f)
        new_index = {
            "metadata": index.get("metadata", {}),
            "weight_map": {k: fname for k in index.get("weight_map", {}) if k in shard},
        }
        with open(out_file + ".index.json", "w") as f:
            json.dump(new_index, f, indent=2)

    config["start_layer"] = start_layer
    config["end_layer"] = end_layer
    with open(os.path.join(output_dir, "config.json"), "w") as f:
        json.dump(config, f, indent=2)
    return out_file


def copy_other_files(model: str, output_dir: str):
    """Copy tokenizer / auxiliary files (everything but weights, the index and config.json);
    reference ``sharding_weight.py:63-71``."""
    model_path = get_model_path(model)
    for name in os.listdir(model_path):
        if name.endswith(".safetensors") or name in ("model.safetensors.index.json", "config.json"):
            continue
        src, dst = os.path.join(model_path, name), os.path.join(output_dir, name)
        if os.path.isdir(src):
            shutil.copytree(src, dst, dirs_exist_ok=True)
        else:
            shutil.copy2(src, dst)


# ---------------------------------------------------------------------------------------------
# Synthetic checkpoints (random init in the exact mlx-community key layout)
# ---------------------------------------------------------------------------------------------
def _linear_entries(prefix: str, out_f: int, in_f: int, gen, dtype, device, qcfg, std=0.02,
                    bias: bool = False, lead: Tuple[int, ...] = ()) -> Iterable[Tuple[str, torch.Tensor]]:
    w = torch.randn(*lead, out_f, in_f, generator=gen, device=device, dtype=torch.float32) * std
    if qcfg is not None and in_f % qcfg["group_size"] == 0:
        wq, s, b = quant.quantize(w, qcfg["group_size"], qcfg["bits"], out_dtype=dtype
                                  if dtype in (torch.float16, torch.bfloat16) else torch.float16)
        yield prefix + ".weight", wq.view(torch.uint32)
        yield prefix + ".scales", s
        yield prefix + ".biases", b
    else:
        yield prefix + ".weight", w.to(dtype)
    if bias:
        yield prefix + ".bias", (torch.randn(*lead, out_f, generator=gen, device=device) * std).to(dtype)


def random_state_dict(cfg: ModelConfig, spec: Optional[ShardSpec] = None, dtype=torch.bfloat16,
                      device="cpu", seed: int = 0, quantization: Optional[Dict[str, int]] = None,
                      stacked_experts: bool = True) -> Iterator[Tuple[str, torch.Tensor]]:
    """Yield random-init tensors for stage ``spec`` with mlx-community key names.

    ``quantization={"group_size":64,"bits":4}`` emits ``weight/scales/biases`` triples for every
    Linear / Embedding except norms and the MoE router (which mlx leaves unquantised, SURVEY U10).
    """
    spec = spec or cfg.shard()
    gen = torch.Generator(device=device)
    H = cfg.hidden_size
    q = quantization
    tied = cfg.tie_word_embeddings

    def lin(prefix, out_f, in_f, layer_seed, **kw):
        gen.manual_seed(seed * 1000003 + layer_seed)
        return _linear_entries(prefix, out_f, in_f, gen, dtype, device, q, **kw)

    def norm(prefix, n, layer_seed):
        gen.manual_seed(seed * 1000003 + layer_seed)
        base = 0.0 if cfg.model_type == "gemma2" else 1.0
        yield prefix + ".weight", (base + 0.1 * torch.randn(n, generator=gen, device=device)).to(dtype)

    if spec.is_first or (spec.is_last and tied):
        yield from lin("model.embed_tokens", cfg.vocab_size, H, 1)
    for i in spec.layers():
        p = f"model.layers.{i}"
        s0 = 100 + i * 50
        ra, rm = spec.runs_attn(i), spec.runs_mlp(i)
        gem = cfg.model_type == "gemma2"
        if ra:
            yield from norm(p + ".input_layernorm", H, s0)
        if (ra if gem else rm):
            yield from norm(p + ".post_attention_layernorm", H, s0 + 1)
        if gem and rm:
            yield from norm(p + ".pre_feedforward_layernorm", H, s0 + 2)
            yield from norm(p + ".post_feedforward_layernorm", H, s0 + 3)
        a = p + ".self_attn"
        if not ra:
            pass
        elif cfg.model_type == "deepseek_v2":
            nh = cfg.num_attention_heads
            qd = cfg.qk_nope_head_dim + cfg.qk_rope_head_dim
            if cfg.q_lora_rank is None:
                yield from lin(a + ".q_proj", nh * qd, H, s0 + 4)
            else:
                yield from lin(a + ".q_a_proj", cfg.q_lora_rank, H, s0 + 4)
                yield from norm(a + ".q_a_layernorm", cfg.q_lora_rank, s0 + 5)
                yield from lin(a + ".q_b_proj", nh * qd, cfg.q_lora_rank, s0 + 6)
            yield from lin(a + ".kv_a_proj_with_mqa", cfg.kv_lora_rank + cfg.qk_rope_head_dim, H, s0 + 7)
            yield from norm(a + ".kv_a_layernorm", cfg.kv_lora_rank, s0 + 8)
            yield from lin(a + ".kv_b_proj", nh * (cfg.qk_nope_head_dim + cfg.v_head_dim),
                           cfg.kv_lora_rank, s0 + 9)
            yield from lin(a + ".o_proj", H, nh * cfg.v_head_dim, s0 + 10)
        else:
            hd = cfg.head_dim
            yield from lin(a + ".q_proj", cfg.num_attention_heads * hd, H, s0 + 4, bias=cfg.attention_bias)
            yield from lin(a + ".k_proj", cfg.num_key_value_heads * hd, H, s0 + 5, bias=cfg.attention_bias)
            yield from lin(a + ".v_proj", cfg.num_key_value_heads * hd, H, s0 + 6, bias=cfg.attention_bias)
            yield from lin(a + ".o_proj", H, cfg.num_attention_heads * hd, s0 + 7, bias=cfg.attention_bias)
        m = p + ".mlp"
        if not rm:
            continue
        if cfg.is_moe_layer(i):
            E, I = cfg.n_routed_experts, cfg.moe_intermediate_size
            gen.manual_seed(seed * 1000003 + s0 + 11)
            # router stays unquantised
            yield m + ".gate.weight", (torch.randn(E, H, generator=gen, device=device) * 0.02).to(dtype)
            if stacked_experts:
                yield from lin(m + ".switch_mlp.gate_proj", I, H, s0 + 12, lead=(E,))
                yield from lin(m + ".switch_mlp.up_proj", I, H, s0 + 13, lead=(E,))
                yield from lin(m + ".switch_mlp.down_proj", H, I, s0 + 14, lead=(E,))
            else:
                for e in range(E):
                    yield from lin(f"{m}.experts.{e}.gate_proj", I, H, s0 + 12 + 1000 * (e + 1))
                    yield from lin(f"{m}.experts.{e}.up_proj", I, H, s0 + 13 + 1000 * (e + 1))
                    yield from lin(f"{m}.experts.{e}.down_proj", H, I, s0 + 14 + 1000 * (e + 1))
            if cfg.n_shared_experts:
                Is = I * cfg.n_shared_experts
                yield from lin(m + ".shared_experts.gate_proj", Is, H, s0 + 15)
                yield from lin(m + ".shared_experts.up_proj", Is, H, s0 + 16)
                yield from lin(m + ".shared_experts.down_proj", H, Is, s0 + 17)
        else:
            I = cfg.intermediate_size
            yield from lin(m + ".gate_proj", I, H, s0 + 12, bias=cfg.mlp_bias)
            yield from lin(m + ".up_proj", I, H, s0 + 13, bias=cfg.mlp_bias)
            yield from lin(m + ".down_proj", H, I, s0 + 14, bias=cfg.mlp_bias)
    if spec.is_last:
        yield from norm("model.norm", H, 7)
        if not tied:
            yield from lin("lm_head", cfg.vocab_size, H, 9)


def write_synthetic_checkpoint(path: str, config: Dict, dtype=torch.bfloat16, seed: int = 0,
                               quantization: Optional[Dict[str, int]] = None, stacked_experts: bool = True,
                               shards: int = 1, with_tokenizer: bool = True) -> str:
    """Materialise a random-init checkpoint directory in the mlx-community layout (config.json,
    ``model*.safetensors`` [+ index], tokenizer files)."""
    os.makedirs(path, exist_ok=True)
    config = dict(config)
    if quantization is not None:
        config["quantization"] = dict(quantization)
    cfg = ModelConfig.from_dict(config)
    tensors = dict(random_state_dict(cfg, cfg.shard(0, cfg.num_hidden_layers), dtype=dtype, seed=seed,
                                     quantization=quantization, stacked_experts=stacked_experts))
    keys = list(tensors)
    if shards <= 1:
        save_safetensors(os.path.join(path, "model.safetensors"), tensors)
    else:
        weight_map = {}
        per = (len(keys) + shards - 1) // shards
        for si in range(shards):
            fname = f"model-{si + 1:05d}-of-{shards:05d}.safetensors"
            part = {k: tensors[k] for k in keys[si * per:(si + 1) * per]}
            if part:
                save_safetensors(os.path.join(path, fname), part)
                weight_map.update({k: fname for k in part})
        with open(os.path.join(path, "model.safetensors.index.json"), "w") as f:
            json.dump({"metadata": {"total_size": sum(t.numel() * t.element_size() for t in tensors.values())},
                       "weight_map": weight_map}, f)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(config, f, indent=2)
    if with_tokenizer:
        from ..engine.tokenizer import write_byte_tokenizer

        write_byte_tokenizer(path, vocab_size=cfg.vocab_size)
    return path


# ---------------------------------------------------------------------------------------------
# Synthetic LoRA adapters (mlx_lm layout, see utils/adapters.py)
# ---------------------------------------------------------------------------------------------
def _module_shapes(cfg, i: int) -> Dict[str, Tuple[int, int]]:
    """``module path -> (in, out)`` of the linear layers of block ``i`` that mlx_lm can adapt."""
    H = cfg.hidden_size
    if cfg.model_type == "deepseek_v2":
        nh, qd = cfg.num_attention_heads, cfg.qk_nope_head_dim + cfg.qk_rope_head_dim
        s = {"self_attn.kv_a_proj_with_mqa": (H, cfg.kv_lora_rank + cfg.qk_rope_head_dim),
             "self_attn.kv_b_proj": (cfg.kv_lora_rank, nh * (cfg.qk_nope_head_dim + cfg.v_head_dim)),
             "self_attn.o_proj": (nh * cfg.v_head_dim, H)}
        if cfg.q_lora_rank is None:
            s["self_attn.q_proj"] = (H, nh * qd)
        else:
            s.update({"self_attn.q_a_proj": (H, cfg.q_lora_rank), "self_attn.q_b_proj": (cfg.q_lora_rank, nh * qd)})
        if cfg.is_moe_layer(i):
            Is = cfg.moe_intermediate_size * (cfg.n_shared_experts or 0)
            if Is:
                s.update({"mlp.shared_experts.gate_proj": (H, Is), "mlp.shared_experts.up_proj": (H, Is),
                          "mlp.shared_experts.down_proj": (Is, H)})
        else:
            I = cfg.intermediate_size
            s.update({"mlp.gate_proj": (H, I), "mlp.up_proj": (H, I), "mlp.down_proj": (I, H)})
        return s
    hd, I = cfg.head_dim, cfg.intermediate_size
    return {"self_attn.q_proj": (H, cfg.num_attention_heads * hd), "self_attn.k_proj": (H, cfg.num_key_value_heads * hd),
            "self_attn.v_proj": (H, cfg.num_key_value_heads * hd), "self_attn.o_proj": (cfg.num_attention_heads * hd, H),
            "mlp.gate_proj": (H, I), "mlp.up_proj": (H, I), "mlp.down_proj": (I, H)}


def write_synthetic_adapter(path: str, cfg, rank: int = 8, scale: float = 20.0, num_layers: Optional[int] = None,
                            modules: Optional[Iterable[str]] = None, seed: int = 0, zero_b: bool = False,
                            std: float = 0.02) -> str:
    """Write a random adapter in the mlx_lm layout for the last ``num_layers`` blocks (-1: all) of the model ``cfg`` (config dict or
    ``ModelConfig``).  ``modules``: module paths inside a block (default: every adaptable linear, e.g. ``self_attn.q_proj``).
    ``zero_b``: ``B = 0``, mlx_lm's initial state (the adapted model equals the base model)."""
    from .adapters import CONFIG_FILE, WEIGHTS_FILE

    cfg = cfg if isinstance(cfg, ModelConfig) else ModelConfig.from_dict(dict(cfg))
    L = cfg.num_hidden_layers
    num_layers = L if num_layers is None else int(num_layers)
    gen = torch.Generator().manual_seed(seed)
    tensors = {}
    for i in range(L - num_layers if 0 < num_layers < L else 0, L):   # -1: every block, as mlx_lm writes it
        shapes = _module_shapes(cfg, i)
        for mod in (modules if modules is not None else shapes):
            if mod not in shapes:
                continue   # e.g. shared-expert modules on DeepSeek's dense layer
            k_in, n_out = shapes[mod]
            p = f"model.layers.{i}.{mod}"
            tensors[p + ".lora_a"] = torch.randn(k_in, rank, generator=gen) * (1.0 / k_in ** 0.5)
            tensors[p + ".lora_b"] = torch.zeros(rank, n_out) if zero_b else torch.randn(rank, n_out, generator=gen) * std
    os.makedirs(path, exist_ok=True)
    save_safetensors(os.path.join(path, WEIGHTS_FILE), tensors)
    keys = sorted({m for m in (modules if modules is not None else _module_shapes(cfg, L - 1))})
    with open(os.path.join(path, CONFIG_FILE), "w") as f:
        json.dump({"fine_tune_type": "lora", "num_layers": num_layers,
                   "lora_parameters": {"rank": rank, "scale": scale, "dropout": 0.0, "keys": keys}}, f, indent=2)
    return path
