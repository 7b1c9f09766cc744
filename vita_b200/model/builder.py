"""`load_pretrained_model` with the reference's signature and return value (vita/model/builder.py:14-24,306).

Checkpoint ingestion streams the HF safetensors shards of `model_path` and packs them into the kernel-native layout
(vita_b200/weights.py).  The tokenizer and the CPU image / audio pre-processors are the reference's own (out of
scope for the kernel tier) and are returned when their files are present next to the checkpoint.

`model_path="synthetic:tiny"` / `"synthetic:full[:L]"` builds seeded random weights instead (tests, demos, bench).
"""
from __future__ import annotations

import json
import os
from pathlib import Path

import torch

from .. import weights as W
from ..config import VitaConfig, LLMConfig, VisionConfig, AudioConfig
from .vita_mixtral import VITAMixtralForCausalLM


def config_from_hf(cfg_json: dict) -> VitaConfig:
    """config.json of the shipped checkpoint (web_demo/vllm_tools/model_weight_file/config.json) -> VitaConfig."""
    t = cfg_json.get("text_config", cfg_json)
    llm = LLMConfig(vocab_size=t.get("vocab_size", 51760), hidden_size=t.get("hidden_size", 4096),
                    intermediate_size=t.get("intermediate_size", 14336),
                    num_hidden_layers=t.get("num_hidden_layers", 32),
                    num_attention_heads=t.get("num_attention_heads", 32),
                    num_key_value_heads=t.get("num_key_value_heads", 8),
                    num_local_experts=t.get("num_local_experts", 8),
                    num_experts_per_tok=t.get("num_experts_per_tok", 2), rms_norm_eps=t.get("rms_norm_eps", 1e-5),
                    rope_theta=t.get("rope_theta", 1e6),
                    max_position_embeddings=t.get("max_position_embeddings", 32768),
                    tokenizer_model_max_length=cfg_json.get("tokenizer_model_max_length", 4600))
    v = cfg_json.get("vision_config", {})
    vision = VisionConfig(hidden_size=v.get("hidden_size", 1024), intermediate_size=v.get("intermediate_size", 4096),
                          num_hidden_layers=v.get("num_hidden_layers", 24),
                          num_attention_heads=v.get("num_attention_heads", 16), image_size=v.get("image_size", 448),
                          patch_size=v.get("patch_size", 14), layer_norm_eps=v.get("layer_norm_eps", 1e-6))
    a = cfg_json.get("audio_config", {})
    audio = AudioConfig(input_dim=a.get("num_mel_bins", 80), hidden_size=a.get("hidden_size", 1024),
                        num_attention_heads=a.get("num_attention_heads", 16),
                        linear_units=a.get("intermediate_size", 4096), num_blocks=a.get("num_hidden_layers", 24))
    return VitaConfig(llm=llm, vision=vision, audio=audio)


class LazySafetensors:
    """Read-only mapping over the `*.safetensors` shards of a checkpoint directory that reads a tensor only when it is
    asked for.  `weights.pack` walks the model layer by layer and moves every tensor to the GPU as soon as it has it,
    so the host never holds more than one layer of the 93.7 GB checkpoint (SURVEY.md section 8f rank 4) instead of the
    whole state dict.  Uses `model.safetensors.index.json` when present, else the shards' own key lists."""

    def __init__(self, path: Path, prefix: str = ""):
        from safetensors import safe_open
        self._open = safe_open
        self._prefix = prefix
        self._where = {}
        index = path / "model.safetensors.index.json"
        if index.exists():
            for k, shard in json.loads(index.read_text())["weight_map"].items():
                self._where[prefix + k] = path / shard
        else:
            for shard in sorted(path.glob("*.safetensors")):
                with safe_open(str(shard), framework="pt", device="cpu") as f:
                    for k in f.keys():
                        self._where[prefix + k] = shard
        if not self._where:
            raise ValueError(f"no *.safetensors shards under {path}")
        self._handles = {}

    def __contains__(self, key) -> bool:
        return key in self._where

    def __iter__(self):
        return iter(self._where)

    def __len__(self) -> int:
        return len(self._where)

    def keys(self):
        return self._where.keys()

    def __getitem__(self, key):
        shard = self._where[key]                       # KeyError for unknown names, like a dict
        f = self._handles.get(shard)
        if f is None:
            f = self._handles[shard] = self._open(str(shard), framework="pt", device="cpu").__enter__()
        return f.get_tensor(key[len(self._prefix):])

    def close(self):
        for f in self._handles.values():
            f.__exit__(None, None, None)
        self._handles.clear()


class _Overlay:
    """`primary` wins over `base` for the keys it has (the reference's separate vision-tower checkpoint override,
    vita/model/builder.py:245-257)."""

    def __init__(self, primary, base):
        self.primary, self.base = primary, base

    def __contains__(self, key):
        return key in self.primary or key in self.base

    def __getitem__(self, key):
        return self.primary[key] if key in self.primary else self.base[key]

    def __iter__(self):
        yield from self.primary
        yield from (k for k in self.base if k not in self.primary)


def _load_safetensors_dir(path: Path) -> LazySafetensors:
    return LazySafetensors(path)


class LoraMerged:
    """Read-only mapping that returns `W + (alpha / r) * B @ A` for every weight that has a LoRA pair in a PEFT adapter
    and the base tensor otherwise -- what `PeftModel.from_pretrained(...).merge_and_unload()` leaves behind
    (vita/model/builder.py:138-145), computed tensor by tensor while `weights.pack` streams the checkpoint, so the
    merged model is never materialised on the host."""

    def __init__(self, base, adapter: dict, lora_alpha: float, r: int, use_rslora: bool = False):
        self.base = base
        self.scale = lora_alpha / (r ** 0.5 if use_rslora else r)
        self.pairs = {}
        for k, a in adapter.items():
            if ".lora_A." not in k:
                continue
            kb = k.replace(".lora_A.", ".lora_B.")
            target = k.split(".lora_A.")[0]
            for pre in ("base_model.model.", "base_model."):
                if target.startswith(pre):
                    target = target[len(pre):]
                    break
            self.pairs[target + ".weight"] = (a, adapter[kb])

    def __contains__(self, key):
        return key in self.base

    def __iter__(self):
        return iter(self.base)

    def keys(self):
        return self.base.keys() if hasattr(self.base, "keys") else list(self.base)

    def __getitem__(self, key):
        w = self.base[key]
        pair = self.pairs.get(key)
        if pair is None:
            return w
        a, b = pair
        return (w.float() + self.scale * (b.float() @ a.float())).to(w.dtype)


def _load_adapter(path: Path):
    """PEFT adapter of a LoRA checkpoint directory: (tensors, lora_alpha, r, use_rslora)."""
    cfg = json.loads((path / "adapter_config.json").read_text())
    if (path / "adapter_model.safetensors").exists():
        from safetensors.torch import load_file
        tensors = load_file(str(path / "adapter_model.safetensors"))
    else:
        tensors = torch.load(str(path / "adapter_model.bin"), map_location="cpu")
    return tensors, float(cfg["lora_alpha"]), int(cfg["r"]), bool(cfg.get("use_rslora", False))


def _non_lora_trainables(path: Path) -> dict:
    """vita/model/builder.py:108-137: extra full tensors saved next to the adapter, with the trainer's prefixes."""
    f = path / "non_lora_trainables.bin"
    if not f.exists():
        return {}
    t = torch.load(str(f), map_location="cpu")
    t = {(k[11:] if k.startswith("base_model.") else k): v for k, v in t.items()}
    if any(k.startswith("model.model.") for k in t):
        t = {(k[6:] if k.startswith("model.") else k): v for k, v in t.items()}
    return t


def load_pretrained_model(model_path, model_base=None, model_name=None, model_type="mixtral-8x7b", load_8bit=False,
                          load_4bit=False, device_map="auto", device="cuda", **kwargs):
    """-> (tokenizer, model, image_processor, context_len), as vita/model/builder.py:306."""
    if model_type not in {"mixtral-8x7b"}:
        raise ValueError(f"Unknown Model Type {model_type}")                      # builder.py:25-26
    if load_8bit or load_4bit:
        raise ValueError("vita_b200 runs bf16 only (bitsandbytes paths are out of scope)")
    dev = torch.device(device if device != "cuda" else "cuda:0")
    model_kwargs = {k: kwargs[k] for k in ("max_batch", "max_seq_len", "max_new_tokens", "kv_cache_dtype", "k_scale",
                                           "v_scale") if k in kwargs}
    if str(model_path).startswith("synthetic:"):
        parts = str(model_path).split(":")
        cfg = VitaConfig.tiny() if parts[1] == "tiny" else VitaConfig.full(int(parts[2]) if len(parts) > 2 else 32)
        seed = int(kwargs.get("seed", 0))
        packed = W.pack(W.synthetic_state(cfg, seed), cfg, dev) if parts[1] == "tiny" else W.random_packed(cfg, dev, seed)
        return None, VITAMixtralForCausalLM(cfg, packed, dev, **model_kwargs), None, cfg.llm.tokenizer_model_max_length
    path = Path(model_path)
    cfg = config_from_hf(json.loads((path / "config.json").read_text()))
    is_lora = model_name is not None and "lora" in model_name.lower()
    if is_lora and model_base is None:
        import warnings                                                           # builder.py:47-50
        warnings.warn("There is `lora` in model name but no `model_base` is provided. If you are loading a LoRA "
                      "model, please provide the `model_base` argument.")
    if is_lora and model_base is not None:
        # builder.py:51-145: base weights, the non-LoRA trainables saved next to the adapter, then the merged adapter
        base_dir = Path(model_base) if any(Path(model_base).glob("*.safetensors")) else path
        state = _load_safetensors_dir(base_dir)
        extra = _non_lora_trainables(path)
        if extra:
            state = _Overlay(extra, state)
        adapter, alpha, r, rs = _load_adapter(path)
        state = LoraMerged(state, adapter, alpha, r, rs)
    elif model_base is not None:
        # builder.py:146-176 ("this may be mm projector only"): language model from model_base, whatever tensors
        # model_path holds (projector / encoders) on top
        state = _load_safetensors_dir(Path(model_base))
        if any(path.glob("*.safetensors")):
            state = _Overlay(_load_safetensors_dir(path), state)
        proj = path / "mm_projector.bin"
        if proj.exists():
            state = _Overlay(torch.load(str(proj), map_location="cpu"), state)
    else:
        state = _load_safetensors_dir(path)
    vt = kwargs.get("vision_tower_path")
    if vt:                                                                        # builder.py:245-257 override
        state = _Overlay(LazySafetensors(Path(vt), prefix=W.PREFIX_VISION), state)
    model = VITAMixtralForCausalLM(cfg, W.pack(state, cfg, dev), dev, **model_kwargs)
    def _close(m):
        for part in (getattr(m, "primary", None), getattr(m, "base", None)):
            if part is not None:
                _close(part)
        if hasattr(m, "close"):
            m.close()
    _close(state)
    tokenizer = image_processor = None
    try:
        from transformers import AutoTokenizer
        tokenizer = AutoTokenizer.from_pretrained(str(path), use_fast=True)
    except Exception:
        pass
    try:
        from transformers import CLIPImageProcessor
        image_processor = CLIPImageProcessor.from_pretrained(str(path))
        model.get_vision_tower().image_processor = image_processor
    except Exception:
        pass
    context_len = getattr(cfg.llm, "max_position_embeddings", 2048)               # builder.py:295-304
    return tokenizer, model, image_processor, context_len
