"""vLLM-facing model class on the CUDA kernels (SURVEY.md section 8f rank 1, reference path B).

Mirrors `MixtralForConditionalGeneration` of the reference's vLLM fork
(web_demo/vllm_tools/vllm_file/mixtral.py:897-1330): `forward` over FLATTENED tokens with the engine's paged KV cache
(:1130-1172), `merge_multimodal_embeddings` (:1084-1128, placeholder ids -> feature rows, in place), `compute_logits`
(:1174-1178), `sample` (:1180-1186; greedy or sampled per sequence group; `sample_with_logprobs` adds the logprobs
vLLM's Sampler returns: chosen token, top-N and prompt logprobs) and `load_weights` with the checkpoint -> kernel name map (:1189-1330).

What the engine hands the model per step is captured by `TokenBatch` (the fields of vLLM's flash-attention metadata:
slot mapping, block tables, sequence / query lengths); the engine's block tables and KV tensors are used as they are --
`kv_caches[l]` is vLLM's flash layout [2, num_blocks, block_size, n_kv_heads, head_dim], which is exactly the layout
`vita_gemm_qkv_rope` / `vita_decode_attention` address (page = block).  A step may mix fresh prompts (attention over the
prompt itself, FlashAttention kernel), single-token decodes (paged decode kernel) and multi-token continuations of
cached pages -- chunked-prefill chunks and prompts whose prefix the engine found in its prefix cache -- which take the
paged-KV FlashAttention kernel, all of them in one launch per layer.

The reference class was written against vLLM 0.5.5, whose model API no longer exists in the installed 0.22 (probed,
SURVEY.md section 8b).  `register()` registers this class under the reference's architecture name with the installed
`ModelRegistry`; the 0.22 engine drives models through `vllm_config` / forward-context objects that cannot be
exercised without a live engine on a GPU, so the tested contract is the call sequence above
(tests/test_vllm_adapter_gpu.py), not an engine run.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Iterable, List, Optional, Sequence, Tuple

import torch

from . import ops, weights as W
from .config import VitaConfig
from .sampling import TokenLogprobs, check_logprobs, from_vllm, logprob_records, row_tensors
from .model.internvit import InternViTVisionTower, VisionProjector
from .model.mixtral import FP8, LayerAttention, MixtralDecoder
from .model.whale import AudioEncoder

BF16 = torch.bfloat16

# vLLM's CacheConfig.cache_dtype -> the decoder's kv_cache_dtype
CACHE_DTYPES = {"auto": "bf16", "bfloat16": "bf16", "fp8": "fp8", "fp8_e4m3": "fp8"}


def kv_cache_dtype_of(cache_config) -> str:
    """`cache_config.cache_dtype` ("auto" when absent) -> "bf16" or "fp8" (e4m3).  "fp8_e5m2" and every other name
    raise NotImplementedError: the engine would otherwise allocate pages in a format the kernels misread."""
    name = getattr(cache_config, "cache_dtype", "auto") if cache_config is not None else "auto"
    name = "auto" if name is None else str(name)
    if name not in CACHE_DTYPES:
        raise NotImplementedError(f"cache_dtype {name!r} is not supported (supported: {sorted(CACHE_DTYPES)})")
    return CACHE_DTYPES[name]


@dataclass
class TokenBatch:
    """One engine step over T flattened tokens of B sequences (vLLM FlashAttentionMetadata, reduced to what is used)."""
    slot_mapping: torch.Tensor          # int32 [T] device: KV slot (block * block_size + offset) of every token
    block_tables: torch.Tensor          # int32 [B, max_blocks] device
    query_start_loc: Sequence[int]      # host, B + 1 entries: tokens of sequence i are rows [qsl[i], qsl[i + 1])
    seq_lens: Sequence[int]             # host, B entries: context length of sequence i including this step's tokens

    @staticmethod
    def from_vllm(md) -> "TokenBatch":
        """Best-effort view of a vLLM attention-metadata object (field names of the flash-attention backend)."""
        qsl = md.query_start_loc.tolist() if torch.is_tensor(md.query_start_loc) else list(md.query_start_loc)
        sl = md.seq_lens.tolist() if torch.is_tensor(md.seq_lens) else list(md.seq_lens)
        bt = getattr(md, "block_table", None)
        if bt is None:
            bt = md.block_tables
        return TokenBatch(md.slot_mapping.to(torch.int32), bt.to(torch.int32), qsl, sl)


@dataclass
class GroupLogprobs:
    """Logprobs of one sequence group (vLLM 0.5.5's SamplerOutput fields): `sample` for the token it sampled (logprob,
    rank, top-`SamplingParams.logprobs`), `prompt` for its prompt-logprob rows in order (each scores the next prompt
    token, with top-`SamplingParams.prompt_logprobs`)."""
    sample: Optional[TokenLogprobs] = None
    prompt: List[TokenLogprobs] = field(default_factory=list)


class MixtralForConditionalGeneration:
    """Reference path-B surface; weights arrive through `load_weights` (or pre-packed for tests)."""

    def __init__(self, config: VitaConfig, multimodal_config=None, cache_config=None, lora_config=None,
                 quant_config=None, device="cuda", image_token_index: int = 51000, audio_token_index: int = 51001,
                 packed: Optional[dict] = None):
        if lora_config is not None or quant_config is not None:
            raise ValueError("vita_b200 serves bf16 weights without LoRA / quantisation")
        self.config = config
        self.device = torch.device(device)
        self.image_token_index, self.audio_token_index = image_token_index, audio_token_index
        self.block_size = getattr(cache_config, "block_size", 16) if cache_config is not None else 16
        self.kv_cache_dtype = kv_cache_dtype_of(cache_config)
        self.packed = None
        self._dec_ws = {}
        if packed is not None:
            self._bind(packed)

    # ------------------------------------------------------------------------------------------ weights
    @staticmethod
    def checkpoint_name(name: str) -> Optional[str]:
        """Name found in a checkpoint / handed over by vLLM's loader -> the shipped checkpoint's own name (what
        vita_b200.weights.pack consumes).  Returns None for tensors the kernels do not use (mixtral.py:1247-1258)."""
        if "rotary_emb.inv_freq" in name:
            return None
        for a, b in (("language_model.lm_head.", "lm_head."), ("language_model.model.", "model.")):
            if name.startswith(a):
                name = b + name[len(a):]
        return name

    def load_weights(self, weights: Iterable[Tuple[str, torch.Tensor]]):
        """mixtral.py:1189-1330: consumes (name, tensor) pairs, stacks q|k|v and the experts' w1|w3 / w2 into the
        kernel-native layout.  Returns the set of consumed names."""
        state, used = {}, set()
        for name, t in weights:
            key = self.checkpoint_name(name)
            if key is None:
                continue
            state[key] = t
            used.add(name)
        if not any("global_cmvn" in k for k in state):
            # path B applies CMVN in the feature extractor (processor_whale.py:385-393) and skips these buffers
            # (mixtral.py:1257-1258): identity statistics
            a = self.config.audio
            state[W.PREFIX_AUDIO + "encoder.global_cmvn.mean"] = torch.zeros(a.input_dim)
            state[W.PREFIX_AUDIO + "encoder.global_cmvn.istd"] = torch.ones(a.input_dim)
        self._bind(W.pack(state, self.config, self.device))
        return used

    def _bind(self, packed: dict):
        cfg = self.config
        self.packed = packed
        # the decoder object supplies the layer loop + workspaces; its own (1-slot) KV cache is unused: the engine owns KV
        self.llm = MixtralDecoder(cfg.llm, packed["llm"], self.device, max_batch=1, max_seq_len=64, max_new_tokens=8,
                                  kv_cache_dtype=self.kv_cache_dtype)
        self.vision_tower = InternViTVisionTower(cfg.vision, packed["vision"], self.device) if "vision" in packed else None
        self.vision_projector = VisionProjector(packed["projector"]) if "projector" in packed else None
        self.audio_tower = AudioEncoder(cfg.audio, cfg.llm.hidden_size, packed["audio"], self.device) \
            if "audio" in packed else None

    # ------------------------------------------------------------------------------------------ multimodal
    def _validate_pixel_values(self, data: torch.Tensor) -> torch.Tensor:                       # mixtral.py:964-981
        h = self.config.vision.image_size
        for d in data:
            if tuple(d.shape) != (3, h, h):
                raise ValueError("The expected shape of pixel values per image per batch  per patch is "
                                 f"{(3, h, h)}. You supplied {tuple(d.shape)}.")
        return data

    @torch.no_grad()
    def merge_multimodal_embeddings(self, input_ids: torch.Tensor, input_embeds: torch.Tensor, embeddings,
                                    masks: Optional[torch.Tensor], token_id: int) -> torch.Tensor:
        """mixtral.py:1084-1128: overwrite the rows of `input_embeds` at the positions of `token_id` with the feature
        rows (only the valid ones when a mask is given).  In place, one device row-copy."""
        H = input_embeds.shape[-1]
        dst = (input_ids.reshape(-1) == token_id).nonzero().reshape(-1).to(torch.int32)
        feats = embeddings.reshape(-1, H) if torch.is_tensor(embeddings) else torch.cat(list(embeddings)).reshape(-1, H)
        src = None
        if masks is not None:
            src = masks.reshape(-1).bool().nonzero().reshape(-1).to(torch.int32)
        n = feats.shape[0] if src is None else src.numel()
        if dst.numel() != n:
            raise ValueError(f"Attempted to assign {n} multimodal tokens to {dst.numel()} placeholders")
        if n:
            ops.row_copy(feats.contiguous(), src, dst.to(self.device), input_embeds.view(-1, H), n)
        return input_embeds

    # ------------------------------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, positions: torch.Tensor, kv_caches: List[torch.Tensor], attn_metadata,
                intermediate_tensors=None, **kwargs) -> torch.Tensor:
        """-> hidden states [T, H] after the final norm (what `compute_logits` consumes), mixtral.py:1130-1172."""
        meta = attn_metadata if isinstance(attn_metadata, TokenBatch) else TokenBatch.from_vllm(attn_metadata)
        dev, H = self.device, self.config.llm.hidden_size
        ids = input_ids.reshape(-1).to(dev)
        T = ids.numel()
        emb = torch.empty(T, H, dtype=BF16, device=dev)
        ops.row_copy(self.packed["llm"]["embed"], ids.to(torch.int32), None, emb, T)       # embed_tokens, :1139
        pixel_values = kwargs.pop("pixel_values", None)
        if pixel_values is not None:                                                        # :1141-1150
            if not isinstance(pixel_values, torch.Tensor):
                raise ValueError(f"Incorrect type of pixel values. Got type: {type(pixel_values)}")
            px = self._validate_pixel_values(pixel_values.reshape(-1, *pixel_values.shape[-3:]))
            feats = self.vision_projector(self.vision_tower(px))
            self.merge_multimodal_embeddings(ids, emb, feats, None, self.image_token_index)
        audio_input = kwargs.pop("audio_input", None)
        if audio_input is not None:                                                         # :1152-1161
            audio_mask = kwargs.pop("audio_mask", None)
            lengths = audio_mask.sum(-1) if audio_mask is not None else \
                torch.full((audio_input.shape[0],), audio_input.shape[1])
            out = self.audio_tower(audio_input, lengths)
            self.merge_multimodal_embeddings(ids, emb, out["inputs_embeds"], out["attention_mask"],
                                             self.audio_token_index)
        return self._language_model(emb, positions.reshape(-1).to(device=dev, dtype=torch.int32), kv_caches, meta)

    __call__ = forward

    def _language_model(self, h: torch.Tensor, positions: torch.Tensor, kv_caches, meta: TokenBatch) -> torch.Tensor:
        c = self.config.llm
        qsl, seq_lens = list(meta.query_start_loc), list(meta.seq_lens)
        assert qsl[-1] == h.shape[0] and len(seq_lens) == len(qsl) - 1
        attention = LayerAttention.of_batch(qsl, seq_lens, meta.block_tables, self.block_size, self._decode_workspace)
        slots = meta.slot_mapping.to(device=self.device, dtype=torch.int32)
        # engine-owned pages, vLLM flash layout; fp8 caches may come as uint8 views of the e4m3 bytes
        k = [self._kv_view(kv[0]) for kv in kv_caches]
        v = [self._kv_view(kv[1]) for kv in kv_caches]
        return self.llm.run_layers(h, positions, slots, k, v, attention, final_norm=True).clone()   # final RMSNorm(h)

    def _kv_view(self, t: torch.Tensor) -> torch.Tensor:
        c = self.config.llm
        if self.kv_cache_dtype == "fp8":
            if t.dtype == torch.uint8:
                t = t.view(FP8)
            if t.dtype != FP8:
                raise ValueError(f"cache_dtype fp8 needs uint8 or float8_e4m3fn KV caches, got {t.dtype}")
        elif t.dtype != BF16:
            raise ValueError(f"cache_dtype auto / bfloat16 needs bf16 KV caches, got {t.dtype}")
        return t.reshape(-1, c.num_key_value_heads, c.head_dim)

    def _decode_workspace(self, n: int) -> torch.Tensor:
        if n not in self._dec_ws:
            nkv = self.config.llm.num_key_value_heads
            self._dec_ws[n] = ops.decode_attention_workspace(n, nkv, self.llm.decode_splits, self.device)
        return self._dec_ws[n]

    # ------------------------------------------------------------------------------------------ logits / sampling
    @torch.no_grad()
    def compute_logits(self, hidden_states: torch.Tensor, sampling_metadata=None) -> torch.Tensor:
        """mixtral.py:1174-1178.  `sampling_metadata.selected_token_indices` (if given) picks the rows to score."""
        sel = getattr(sampling_metadata, "selected_token_indices", None)
        if sel is not None:
            hidden_states = hidden_states[sel.to(hidden_states.device)]
        return ops.linear(hidden_states.contiguous(), self.packed["llm"]["lm_head"])

    @torch.no_grad()
    def sample(self, logits: torch.Tensor, sampling_metadata=None) -> torch.Tensor:
        """Next token per logits row.  With vLLM 0.5.5's SamplingMetadata, each sequence group that samples
        (`do_sample`, default True) draws the rows `sample_indices` points at (its position in `seq_groups` when the
        field is absent and there is one row per group) from `sampling_params`: temperature < 1e-5 is greedy,
        otherwise the row is drawn (vita_b200/sampling.py) with the request's seed as key and counter = the output
        length of its sequence (`seq_data[id].get_output_len()`); unseeded rows take one key each from torch's default
        generator.  Every other row -- a group that does not sample (a chunked-prefill chunk), prompt-logprob rows --
        and every row of a call without metadata (or without `seq_groups`) gets the greedy arg-max, as before (the
        reference demos sample with temperature 0.001 / 0.01, web_interactive_demo.py:132, web_ability_demo.py:351)."""
        B = logits.shape[0]
        best = torch.zeros(B, dtype=torch.int64, device=logits.device)
        groups = getattr(sampling_metadata, "seq_groups", None)
        if groups is None:
            ops.argmax_rows(logits.contiguous(), best)
            return (0xFFFFFFFF - (best & 0xFFFFFFFF)).to(torch.int64)
        params, counter, _ = self._sampled_rows(groups, B)
        T, K, P, S = row_tensors(params, logits.device)
        cnt = torch.tensor(counter, dtype=torch.int32).to(logits.device, non_blocking=True)
        ops.sample_rows(logits.contiguous(), T, K, P, S, cnt, best)
        return (0xFFFFFFFF - (best & 0xFFFFFFFF)).to(torch.int64)

    @staticmethod
    def _sampled_rows(groups, B: int):
        """-> per-row SamplingParams (None = greedy) and counters of the rows the groups sample, and per group its
        sampled row (or None) with its parameters."""
        params, counter, sampled = [None] * B, [0] * B, [None] * len(groups)
        for i, sg in enumerate(groups):
            if not getattr(sg, "do_sample", True):
                continue
            rows = getattr(sg, "sample_indices", None)
            if rows is None:
                if len(groups) != B:
                    raise ValueError(f"{len(groups)} sequence groups without sample_indices for {B} logits rows")
                rows = [i]
            rows = [int(r) for r in rows]
            if not rows:
                continue
            ids = list(sg.seq_ids)
            if len(ids) != 1 or len(rows) != 1:
                raise NotImplementedError("sequence groups with several sequences (n > 1, beam search)")
            if not 0 <= rows[0] < B:
                raise ValueError(f"sample index {rows[0]} outside the {B} logits rows")
            params[rows[0]] = from_vllm(sg.sampling_params)
            counter[rows[0]] = int(sg.seq_data[ids[0]].get_output_len())
            sampled[i] = (rows[0], params[rows[0]])
        return params, counter, sampled

    @torch.no_grad()
    def sample_with_logprobs(self, logits: torch.Tensor, sampling_metadata):
        """`sample()` plus the logprobs of vLLM 0.5.5's Sampler: -> (ids [B] as `sample()` returns them, one
        GroupLogprobs per sequence group).  A group that samples gets its token's logprob and rank over the processed
        row (vita_b200/sampling.py) with the top-`sampling_params.logprobs`.  With `sampling_params.prompt_logprobs`
        set, its `prompt_logprob_indices` rows score the next prompt token -- row j of a chunk that starts after
        `seq_data.get_num_computed_tokens()` tokens scores prompt token computed + j + 1 -- with the group's
        parameters, chunked-prefill chunks included.  One kernel launch for all rows."""
        B = logits.shape[0]
        groups = getattr(sampling_metadata, "seq_groups", None)
        if groups is None:
            raise ValueError("sample_with_logprobs needs SamplingMetadata with seq_groups")
        params, counter, sampled = self._sampled_rows(groups, B)
        target = [-1] * B
        used = {g[0] for g in sampled if g is not None}        # every row belongs to at most one group
        n_top, prompt_rows = 0, [None] * len(groups)
        for i, sg in enumerate(groups):
            sp = sg.sampling_params
            n = check_logprobs(getattr(sp, "logprobs", None), "logprobs")
            if sampled[i] is not None:
                n_top = max(n_top, n or 0)
            n_prompt = check_logprobs(getattr(sp, "prompt_logprobs", None), "prompt_logprobs")
            rows = [int(r) for r in (getattr(sg, "prompt_logprob_indices", None) or [])]
            if n_prompt is None or not rows:
                continue
            data = sg.seq_data[list(sg.seq_ids)[0]]
            prompt, done = list(data.prompt_token_ids), int(data.get_num_computed_tokens())
            if done + len(rows) >= len(prompt):
                raise ValueError(f"{len(rows)} prompt-logprob rows after {done} computed tokens of a "
                                 f"{len(prompt)}-token prompt")
            # the group's parameters; a scoring row draws nothing, so it never takes a key from torch's generator
            p = sampled[i][1] if sampled[i] is not None else from_vllm(sp, draws=False)
            for j, r in enumerate(rows):
                if not 0 <= r < B or r in used:
                    raise ValueError(f"prompt-logprob row {r} is outside the {B} logits rows or used twice")
                used.add(r)
                params[r], target[r] = p, prompt[done + 1 + j]
            prompt_rows[i] = (rows, n_prompt)
            n_top = max(n_top, n_prompt)
        dev = logits.device
        T, K, P, S = row_tensors(params, dev)
        cnt = torch.tensor(counter, dtype=torch.int32).to(dev, non_blocking=True)
        tgt = torch.tensor(target, dtype=torch.int32).to(dev, non_blocking=True)
        best = torch.zeros(B, dtype=torch.int64, device=dev)
        lp = torch.empty(B, dtype=torch.float32, device=dev)
        rank = torch.empty(B, dtype=torch.int32, device=dev)
        top_ids = torch.empty(B, max(n_top, 1), dtype=torch.int32, device=dev)
        top_lp = torch.empty(B, max(n_top, 1), dtype=torch.float32, device=dev)
        ops.sample_logprobs(logits.contiguous(), T, K, P, S, cnt, best, lp, rank, top_ids, top_lp, n_top, target=tgt)
        ids = (0xFFFFFFFF - (best & 0xFFFFFFFF)).to(torch.int64)
        toks = [t if t >= 0 else w for t, w in zip(target, ids.tolist())]
        lp, rank, top_ids, top_lp = lp.cpu(), rank.cpu(), top_ids.cpu(), top_lp.cpu()
        rec = lambda rows, n: logprob_records([toks[r] for r in rows], lp[rows], rank[rows], top_ids[rows],
                                              top_lp[rows], n)
        out = []
        for i, sg in enumerate(groups):
            g = GroupLogprobs()
            if sampled[i] is not None:
                n = check_logprobs(getattr(sg.sampling_params, "logprobs", None)) or 0
                g.sample = rec([sampled[i][0]], n)[0]
            if prompt_rows[i] is not None:
                g.prompt = rec(*prompt_rows[i])
            out.append(g)
        return ids, out


def register() -> bool:
    """Register the class with the installed vLLM under the reference's architecture name
    (web_demo/vllm_tools/vllm_file/__init__.py:83-84).  Returns False when vLLM is not importable."""
    try:
        from vllm import ModelRegistry
    except Exception:
        return False
    ModelRegistry.register_model("MixtralForConditionalGeneration", "vita_b200.vllm_adapter:MixtralForConditionalGeneration")
    return True
