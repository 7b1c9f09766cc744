"""`VITAMixtralForCausalLM` on the CUDA kernels -- the reference's Python surface for the omni forward path.

Mirrors vita/model/language_model/vita_mixtral.py:232-415 + vita/model/vita_arch.py:111-407:
`forward`, `generate`, `encode_images`, `encode_audios`, `prepare_inputs_labels_for_multimodal`, `get_vision_tower`,
`get_audio_encoder`, `process_images`.  The Python per-sample splice loop of the reference becomes host-side index
arithmetic (`plan_splice`, pure Python, unit-tested on CPU) + three device row-copies.
"""
from __future__ import annotations

import weakref
from dataclasses import dataclass
from typing import List, Optional, Sequence

import torch

from .. import ops
from ..beam import BeamSearch, check_beam_args, pack_outputs
from ..config import VitaConfig, IMAGE_TOKEN_INDEX, AUDIO_TOKEN_INDEX
from .internvit import InternViTVisionTower, VisionProjector
from ..sampling import MAX_LOGPROBS, check_logprobs, from_hf
from .mixtral import MixtralDecoder
from .whale import AudioEncoder

BF16 = torch.bfloat16


# ------------------------------------------------------------------------------------------------ splice planning
@dataclass
class SplicePlan:
    lengths: List[int]            # spliced length per sample (after truncation)
    text_src: List[int]           # token ids to gather from embed_tokens
    text_dst: List[int]           # flat destination row (sample * max_len + position)
    img_src: List[int]            # flat row in image_features.view(-1, H)
    img_dst: List[int]
    aud_src: List[int]            # flat row in audio_features.view(-1, H)
    aud_dst: List[int]
    max_len: int


def plan_splice(input_ids: Sequence[Sequence[int]], n_image_features: int, image_tokens: int, n_audio_features: int,
                audio_tokens: int, max_model_len: Optional[int]) -> SplicePlan:
    """Index arithmetic of prepare_inputs_labels_for_multimodal (vita/model/vita_arch.py:227-392), inference subset.

    Every IMAGE (-200) / AUDIO (-500) placeholder is replaced by the next unused feature block
    (`image_tokens` / `audio_tokens` rows each); samples lacking a modality still consume one (dummy) feature block
    of it (:240-251, :309-316); the result is truncated to `max_model_len` (:326-329) and right-padded (:372-392).
    Raises AssertionError on the same count mismatches the reference asserts (:227-236, :323-324)."""
    n_img_ph = sum(sum(1 for t in row if t == IMAGE_TOKEN_INDEX) for row in input_ids)
    n_aud_ph = sum(sum(1 for t in row if t == AUDIO_TOKEN_INDEX) for row in input_ids)
    no_img = sum(1 for row in input_ids if IMAGE_TOKEN_INDEX not in row)
    no_aud = sum(1 for row in input_ids if AUDIO_TOKEN_INDEX not in row)
    assert n_img_ph + no_img == n_image_features, "image placeholder / feature count mismatch (vita_arch.py:227-231)"
    assert n_aud_ph + no_aud == n_audio_features, "audio placeholder / feature count mismatch (vita_arch.py:232-236)"
    per_sample = []
    ii = ai = 0
    for row in input_ids:
        items = []   # (kind, value): ("t", token) | ("i", feature idx) | ("a", feature idx)
        has_i = has_a = False
        for t in row:
            if t == IMAGE_TOKEN_INDEX:
                items.append(("i", ii)); ii += 1; has_i = True
            elif t == AUDIO_TOKEN_INDEX:
                items.append(("a", ai)); ai += 1; has_a = True
            else:
                items.append(("t", int(t)))
        if not has_i:
            ii += 1      # a dummy image feature is consumed as a zero-length slice
        if not has_a:
            ai += 1
        per_sample.append(items)
    assert ii == n_image_features and ai == n_audio_features
    plan = SplicePlan([], [], [], [], [], [], [], 0)
    rows_per_sample = []
    for items in per_sample:
        rows = []
        for kind, v in items:
            if kind == "t":
                rows.append(("t", v))
            elif kind == "i":
                rows.extend(("i", v * image_tokens + j) for j in range(image_tokens))
            else:
                rows.extend(("a", v * audio_tokens + j) for j in range(audio_tokens))
        if max_model_len is not None:
            rows = rows[:max_model_len]
        rows_per_sample.append(rows)
        plan.lengths.append(len(rows))
    plan.max_len = max(plan.lengths) if plan.lengths else 0
    for s, rows in enumerate(rows_per_sample):
        for p, (kind, v) in enumerate(rows):
            dst = s * plan.max_len + p
            if kind == "t":
                plan.text_src.append(v); plan.text_dst.append(dst)
            elif kind == "i":
                plan.img_src.append(v); plan.img_dst.append(dst)
            else:
                plan.aud_src.append(v); plan.aud_dst.append(dst)
    return plan


@dataclass
class CausalLMOutput:
    logits: Optional[torch.Tensor]
    past_key_values: object = None


@dataclass
class GenerateOutput:
    sequences: torch.Tensor
    scores: Optional[tuple] = None
    logprobs: Optional[tuple] = None      # generate(logprobs=N): one sampling.TokenLogprobs per generated token
    sequences_scores: Optional[torch.Tensor] = None   # beam search: [R] fp32 length-penalised hypothesis scores
    beam_indices: Optional[torch.Tensor] = None       # beam search: [R, n] running beam of each token (-1: padding)


class CapturedEncoders:
    """Both encoders as ONE CUDA graph per input geometry: InternViT + projector on the capture stream, Whale + adapter
    on a forked stream (the two are independent until the splice), ~430 launches replayed with one call.  Inputs are
    copied into static buffers; the returned feature tensors are the graph's own outputs and are overwritten by the
    next call with the same geometry (the splice consumes them right away).  The model owns this object and is held
    weakly here, so dropping the last reference to a model frees its device memory at once, not at the next garbage
    collection of the cycle."""

    def __init__(self, model):
        self._model = weakref.ref(model)
        self.graphs = {}
        self.replayed_launches = 0     # kernels executed through graph replays (bench.py's gpu_launches)

    @torch.no_grad()
    def __call__(self, images: torch.Tensor, feats: torch.Tensor, lengths):
        m = self._model()
        if feats.dim() == 2:
            feats = feats.unsqueeze(0)
        lengths = torch.as_tensor(lengths).reshape(-1)
        key = (tuple(images.shape), tuple(feats.shape))
        ent = self.graphs.get(key)
        if ent is None:
            with torch.inference_mode(False):
                dev = m.device
                s_img = torch.empty(images.shape, dtype=BF16, device=dev)
                s_feat = torch.empty(feats.shape, dtype=torch.float32, device=dev)
                s_len = torch.empty(lengths.shape, dtype=torch.int64, device=dev)
                s_img.copy_(images); s_feat.copy_(feats); s_len.copy_(lengths)
                m.mm_projector(m.vision_tower(s_img))        # eager warm-up: one-time kernel attributes, length caches
                m.audio_encoder(s_feat, s_len)
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                cap, side = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
                cap.wait_stream(torch.cuda.current_stream())
                n0 = ops.launch_count()
                with torch.cuda.graph(g, stream=cap):
                    side.wait_stream(cap)
                    with torch.cuda.stream(side):
                        aud = m.audio_encoder(s_feat, s_len)
                    img = m.mm_projector(m.vision_tower(s_img))
                    cap.wait_stream(side)
                torch.cuda.current_stream().wait_stream(cap)
                ent = self.graphs[key] = (g, s_img, s_feat, s_len, img, aud, ops.launch_count() - n0)
        g, s_img, s_feat, s_len, img, aud, n_launch = ent
        s_img.copy_(images, non_blocking=True)
        s_feat.copy_(feats, non_blocking=True)
        s_len.copy_(lengths, non_blocking=True)
        g.replay()
        self.replayed_launches += n_launch
        return img, aud


class VITAMixtralForCausalLM:
    """Inference-only drop-in for the reference class of the same name (no nn.Module: weights live in the packed
    kernel-native layout)."""

    def __init__(self, cfg: VitaConfig, packed: dict, device="cuda", max_batch: int = 1,
                 max_seq_len: Optional[int] = None, max_new_tokens: int = 1024, shuffle_pages: bool = False,
                 kv_cache_dtype: str = "auto", k_scale=1.0, v_scale=1.0):
        """`kv_cache_dtype` "fp8" / "fp8_e4m3": e4m3 paged KV cache with per-layer k_scale / v_scale (MixtralDecoder);
        "auto" / "bf16" (default): bf16.  generate(), beam search and the serving engine run on whichever it is."""
        self.config = cfg
        self.device = torch.device(device)
        self.dtype = BF16
        self.packed = packed
        self.llm = MixtralDecoder(cfg.llm, packed["llm"], device, max_batch, max_seq_len, max_new_tokens,
                                  shuffle_pages=shuffle_pages, kv_cache_dtype=kv_cache_dtype, k_scale=k_scale,
                                  v_scale=v_scale)
        self.vision_tower = InternViTVisionTower(cfg.vision, packed["vision"], device) if "vision" in packed else None
        self.mm_projector = VisionProjector(packed["projector"]) if "projector" in packed else None
        self.audio_encoder = AudioEncoder(cfg.audio, cfg.llm.hidden_size, packed["audio"], device) \
            if "audio" in packed else None
        import os
        self._captured = CapturedEncoders(self) if os.environ.get("VITA_B200_ENC_GRAPH", "1") == "1" else None

    # -- surface helpers ------------------------------------------------------------------------------------
    def eval(self):
        return self

    def get_model(self):
        return self

    def get_vision_tower(self):
        return self.vision_tower

    def get_audio_encoder(self):
        return self.audio_encoder

    def resize_token_embeddings(self, n: int):
        assert n == self.config.llm.vocab_size, "vita_b200 does not resize packed embeddings"

    @property
    def image_processor(self):
        if getattr(self, "_image_processor", None) is None:
            from ..image_frontend import ImageProcessor
            self._image_processor = ImageProcessor(self.device)
        return self._image_processor

    def process_images(self, images, model_cfg=None):
        """vita_mixtral.py:397-415 / mm_utils.py:30-43: the tiles `dynamic_preprocess` cut on the host (448 x 448 PIL
        images or uint8 arrays) -> [N, 3, 448, 448]; rescale + normalise run on the GPU (csrc/image.cu), bit-equal to
        CLIPImageProcessor followed by the demo's cast to the model dtype.  Tensors pass through unchanged."""
        if torch.is_tensor(images):
            return images
        if isinstance(images, (list, tuple)) and len(images) and torch.is_tensor(images[0]) and images[0].is_floating_point():
            return torch.stack([torch.as_tensor(im) for im in images])
        return self.image_processor.process_tiles(list(images))

    def preprocess_image(self, image, min_num: int = 1, max_num: int = 12, use_thumbnail: bool = True):
        """dynamic_preprocess + process_images (video_audio_demo.py:214-221) as one device-side pipeline: a decoded
        RGB image (PIL / [H, W, 3] uint8) -> (pixel_values [N, 3, 448, 448] bf16, N)."""
        return self.image_processor.preprocess(image, min_num, max_num, use_thumbnail)

    # -- encoders --------------------------------------------------------------------------------------------
    @torch.no_grad()
    def encode_images(self, images: torch.Tensor) -> torch.Tensor:
        """vita_arch.py:131-134: vision tower + mm_projector -> [N, 256, H]."""
        return self.mm_projector(self.vision_tower(images))

    @torch.no_grad()
    def encode_audios(self, audios: torch.Tensor, lengths: torch.Tensor) -> dict:
        """The call north_star names `encode_audios` (reference call site vita_arch.py:186-191)."""
        return self.audio_encoder(audios, lengths)

    # -- splice ----------------------------------------------------------------------------------------------
    @torch.no_grad()
    def prepare_inputs_labels_for_multimodal(self, input_ids, position_ids, attention_mask, past_key_values, labels,
                                             images, audios):
        """vita_arch.py:151-407.  Returns (None, position_ids, attention_mask, past_key_values, inputs_embeds, labels)."""
        if self.vision_tower is None or images is None or input_ids.shape[1] == 1:       # :155-175
            return input_ids, position_ids, attention_mask, past_key_values, None, labels
        if isinstance(images, (list, tuple)) or images.ndim == 5:                          # :177-181
            images = torch.cat([im for im in images], dim=0)
        assert audios is not None, "the reference subscripts audio_features unconditionally (vita_arch.py:232-236)"
        if self._captured is not None and self.audio_encoder is not None and torch.is_tensor(audios["audios"]):
            image_features, audio_out = self._captured(images, audios["audios"], audios["lengths"])   # one graph replay
        else:
            image_features = self.encode_images(images)                                    # [N, 256, H]
            audio_out = self.encode_audios(audios["audios"], audios["lengths"])            # :186-189
        audio_features = audio_out["inputs_embeds"]
        ids = input_ids.tolist() if torch.is_tensor(input_ids) else [list(r) for r in input_ids]
        if attention_mask is not None:                                                     # :213-216
            am = attention_mask.bool().tolist()
            ids = [[t for t, m in zip(row, mrow) if m] for row, mrow in zip(ids, am)]
        inputs_embeds, plan = self.splice_features(ids, image_features, audio_features)
        B, S = inputs_embeds.shape[:2]
        dev = self.device
        lens = torch.tensor(plan.lengths)
        new_mask = None
        if attention_mask is not None:
            new_mask = (torch.arange(S)[None, :] < lens[:, None]).to(attention_mask.dtype).to(dev)
        new_pos = None
        if position_ids is not None:
            new_pos = (torch.arange(S)[None, :] * (torch.arange(S)[None, :] < lens[:, None])).to(dev)
        self._last_lengths = plan.lengths
        return None, new_pos, new_mask, past_key_values, inputs_embeds, labels

    @torch.no_grad()
    def splice_features(self, ids, image_features, audio_features):
        """The splice proper (vita_arch.py:227-392) from already-encoded features: `ids` list of token-id lists,
        image_features [N, 256, H], audio_features [B_a, T3, H] -> (inputs_embeds [B, S, H], SplicePlan)."""
        H = self.config.llm.hidden_size
        plan = plan_splice(ids, image_features.shape[0], image_features.shape[1], audio_features.shape[0],
                           audio_features.shape[1], self.config.llm.tokenizer_model_max_length)
        B, S = len(ids), plan.max_len
        out = torch.zeros(B * S, H, dtype=BF16, device=self.device)
        dev = self.device

        def idx(v):
            return torch.tensor(v, dtype=torch.int32).to(dev, non_blocking=True)

        if plan.text_src:
            ops.row_copy(self.packed["llm"]["embed"], idx(plan.text_src), idx(plan.text_dst), out, len(plan.text_src))
        if plan.img_src:
            ops.row_copy(image_features.view(-1, H), idx(plan.img_src), idx(plan.img_dst), out, len(plan.img_src))
        if plan.aud_src:
            ops.row_copy(audio_features.reshape(-1, H), idx(plan.aud_src), idx(plan.aud_dst), out, len(plan.aud_src))
        return out.view(B, S, H), plan

    # -- forward / generate ----------------------------------------------------------------------------------
    @torch.no_grad()
    def _embeds_for(self, input_ids, images, audios):
        if images is None or input_ids.shape[1] == 1:
            if input_ids.shape[1] > self.llm.cache.max_seq_len:
                raise ValueError(f"prompt of {input_ids.shape[1]} tokens exceeds the KV capacity "
                                 f"{self.llm.cache.max_seq_len}")
            ids = input_ids.to(torch.int32).reshape(-1).to(self.device)
            out = torch.empty(ids.numel(), self.config.llm.hidden_size, dtype=BF16, device=self.device)
            ops.row_copy(self.packed["llm"]["embed"], ids, None, out, ids.numel())
            return out.view(*input_ids.shape, -1), [input_ids.shape[1]] * input_ids.shape[0]
        emb = self.prepare_inputs_labels_for_multimodal(input_ids, None, None, None, None, images, audios)[4]
        return emb, self._last_lengths

    @torch.no_grad()
    def forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None,
                inputs_embeds=None, labels=None, use_cache=None, images=None, audios=None, **kw) -> CausalLMOutput:
        """vita_mixtral.py:249-289.  Prefill (any length) computes logits on all positions like the reference
        (`custom_forward` :171-173); a single-token call with `past_key_values` set runs one decode step on the
        paged cache owned by this object (the returned `past_key_values` is an opaque handle to it)."""
        assert labels is None, "training is out of scope"
        if inputs_embeds is None and input_ids is not None and input_ids.shape[1] == 1 and past_key_values is not None:
            B = input_ids.shape[0]
            if int(self.llm.cache.cache_len[:B].max()) + 1 > self.llm.cache.max_seq_len:
                raise ValueError("the paged KV cache of this sequence is full (max_seq_len reached)")
            # teacher-forceable decode step: feed the given token (not necessarily the arg-max)
            packed = (0xFFFFFFFF - input_ids.reshape(-1).to(torch.int64)).to(self.device)
            self.llm.best[:B].copy_(packed)
            self.llm.decode_step(B, use_graph=False, want_logits=True)
            return CausalLMOutput(self.llm.d_logits[:B].clone().unsqueeze(1), past_key_values)
        if inputs_embeds is None:
            inputs_embeds, lens = self._embeds_for(input_ids, images, audios)
        else:
            inputs_embeds = inputs_embeds.to(device=self.device, dtype=BF16)
            lens = [inputs_embeds.shape[1]] * inputs_embeds.shape[0]
        B, S, _ = inputs_embeds.shape
        assert B <= self.llm.max_batch
        self.llm.reset()
        rows = []
        for b in range(B):
            lg = self.llm.prefill(inputs_embeds[b, : lens[b]].contiguous(), slot=b, all_logits=True)
            if lens[b] < S:   # right padding (vita_arch.py:372-392): padded rows carry no information
                lg = torch.cat([lg, torch.zeros(S - lens[b], lg.shape[1], dtype=lg.dtype, device=lg.device)])
            rows.append(lg)
        return CausalLMOutput(torch.stack(rows), "vita_b200-paged-kv")

    __call__ = forward

    @torch.no_grad()
    def generate_batch(self, requests, max_new_tokens: int = 16, use_graph: bool = True, step_callback=None):
        """Concurrent decode of several independent requests (BASELINE configs[4]: duplex / bs=16 streaming).

        `requests`: list of dicts {"input_ids": [1, L], "images": ..., "audios": ...}, optionally with
        "sampling": {"temperature", "top_k", "top_p", "seed"} (as for generate(do_sample=True)); the others are greedy.
        A request with "logprobs": N (0 .. 20) receives "token_logprobs": one sampling.TokenLogprobs per returned token
        (as generate(logprobs=N)).  Each request is prefilled into its own paged-KV slot, then all of them advance one token per step through the
        batched decode step.  Returns the list of generated token lists.  `step_callback(step_index)` is called after
        every step launch (latency harnesses record CUDA events there)."""
        B = len(requests)
        if not 1 <= B <= self.llm.max_batch:
            raise ValueError(f"{B} requests do not fit max_batch = {self.llm.max_batch}")
        params = [None if r.get("sampling") is None else from_hf(True, **r["sampling"]) for r in requests]
        n_top = [check_logprobs(r.get("logprobs")) for r in requests]
        if any(params) and self.llm.ep_world > 1:
            raise ValueError("sampled decoding is single-GPU (the expert-parallel mode serves greedy requests)")
        if any(n is not None for n in n_top) and self.llm.ep_world > 1:
            raise ValueError("logprobs are single-GPU (the expert-parallel mode serves greedy requests)")
        self.llm.reset()
        for b, r in enumerate(requests):
            emb, lens = self._embeds_for(r["input_ids"], r.get("images"), r.get("audios"))
            self.llm.check_capacity(lens[0], max_new_tokens)
            self.llm.sampling.set(b, params[b], n_top[b])
            self.llm.prefill(emb[0, : lens[0]].contiguous(), slot=b, sampled=params[b] is not None,
                             logprobs=self.llm.sampling.log_width(b, 1))
        sampled = any(p is not None for p in params)
        logprobs = self.llm.sampling.log_width(0, B)
        for step in range(max_new_tokens):
            self.llm.decode_step_batched(B, use_graph=use_graph, sampled=sampled, logprobs=logprobs)
            if step_callback is not None:
                step_callback(step)
        out = [self.llm.generated_tokens(b)[:max_new_tokens] for b in range(B)]
        for b, r in enumerate(requests):
            if n_top[b] is not None:
                r["token_logprobs"] = self.llm.read_logprobs(b, out[b], n_top[b])
        return out

    def prepare_inputs_for_generation_original(self, input_ids, past_key_values=None, attention_mask=None,
                                               inputs_embeds=None, output_router_logits=False, **kwargs):
        """vita_mixtral.py:291-352 (host-side bookkeeping of HF `generate`): keep only the tokens the KV cache has not
        seen, derive position_ids from the mask.  `past_key_values` here is the opaque handle `forward` returns; the
        number of cached tokens is the length of this object's paged cache (slot 0 ... B-1 advance together)."""
        if past_key_values is not None:
            past_length = int(self.llm.cache.cache_len[0])
            if attention_mask is not None and attention_mask.shape[1] > input_ids.shape[1]:       # :311-312
                input_ids = input_ids[:, -(attention_mask.shape[1] - past_length):]
            elif past_length < input_ids.shape[1]:                                                # :315-316
                input_ids = input_ids[:, past_length:]
            else:                                                                                 # :318-320
                input_ids = input_ids[:, input_ids.shape[1] - 1:]
        position_ids = kwargs.get("position_ids", None)
        if attention_mask is not None and position_ids is None:                                   # :330-335
            position_ids = attention_mask.long().cumsum(-1) - 1
            position_ids.masked_fill_(attention_mask == 0, 1)
            if past_key_values:
                position_ids = position_ids[:, -input_ids.shape[1]:]
        if inputs_embeds is not None and past_key_values is None:                                 # :338-341
            model_inputs = {"inputs_embeds": inputs_embeds}
        else:
            model_inputs = {"input_ids": input_ids}
        model_inputs.update({"position_ids": position_ids, "past_key_values": past_key_values,
                             "use_cache": kwargs.get("use_cache"), "attention_mask": attention_mask,
                             "output_router_logits": output_router_logits})
        return model_inputs

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, inputs_embeds=None, attention_mask=None,
                                      output_router_logits=False, **kwargs):
        """vita_mixtral.py:354-382: the original bookkeeping + `images` / `audios` re-attached."""
        images = kwargs.pop("images", None)
        audios = kwargs.pop("audios", None)
        _inputs = self.prepare_inputs_for_generation_original(
            input_ids, past_key_values=past_key_values, inputs_embeds=inputs_embeds, attention_mask=attention_mask,
            output_router_logits=output_router_logits, **kwargs)
        if images is not None:
            _inputs["images"] = images
        if audios is not None:
            _inputs["audios"] = audios
        return _inputs

    @torch.no_grad()
    def generate(self, input_ids, images=None, audios=None, do_sample=False, temperature=None, top_p=None,
                 num_beams=1, output_scores=False, return_dict_in_generate=True, max_new_tokens=16, use_cache=True,
                 stopping_criteria=None, eos_token_id: Optional[int] = None, use_graph: bool = True, sync_every: int = 16,
                 top_k=None, seed: Optional[int] = None, logprobs: Optional[int] = None, length_penalty: float = 1.0,
                 early_stopping=False, num_return_sequences: int = 1, **kw):
        """Greedy or sampled decode with the call signature of video_audio_demo.py:257-270.  `sequences` (on
        `input_ids.device`) echoes the prompt ids, placeholders included, followed by the new tokens
        (video_audio_demo.py:272-276).

        `do_sample=True` draws every token, the first one included, with `temperature`, `top_k`, `top_p` (None = HF
        4.41's defaults 1.0, 50, 1.0; the policy is vita_b200/sampling.py).  `seed` (an extension) is the 64-bit stream
        key; without it one key is drawn from torch's default CPU generator, so `torch.manual_seed` makes a call
        reproducible.  With `output_scores` the scores are the warped rows, as HF returns them when sampling.
        `logprobs=N` (an extension, 0 .. 20) fills `logprobs` with one sampling.TokenLogprobs per generated token: its
        logprob and rank over the row it was chosen from and the N most likely tokens, computed on the GPU next to the
        choice (greedy tokens are unchanged).

        The decode step replays as one CUDA graph whether or not `output_scores` is set: with scores the step appends
        its logits row to a device-resident log, and `scores` are views of that log (valid until the next call).
        Tokens are read back every `sync_every` steps; stopping criteria see each new token exactly once.

        `num_beams` > 1 (at most 10 and at most the model's `max_batch`): beam search as HF transformers runs it with
        `length_penalty`, `early_stopping` and `num_return_sequences` (vita_b200/beam.py).  `sequences` holds the best
        `num_return_sequences` hypotheses, padded with `eos_token_id`, with `sequences_scores` and `beam_indices`;
        `scores` (with `output_scores`) holds one [num_beams, V] block of the running beams' log-softmax rows per step.
        The beams share their KV pages copy-on-write and advance together through the batched decode step.

        `do_sample=True` with `num_return_sequences` = N > 1 (at most the model's `max_batch`): N independent samples
        of the prompt, as HF 4.41 returns them.  The prompt is prefilled once and its KV pages are shared by the N
        sequences; sequence i draws from stream i of the call's key, so sequence 0 starts with the token the call with
        one sequence draws.  `sequences` is [N, L + T], T the longest row; a row is finished at its EOS or when a
        stopping criterion marks it (a bool result marks every row), and finished rows are padded with
        `eos_token_id`.  `scores` holds one [N, V] block of warped rows per step, `logprobs` one tuple of
        TokenLogprobs per sequence."""
        if num_beams != 1:
            return self._beam_search(input_ids, images, audios, num_beams, num_return_sequences, length_penalty,
                                     early_stopping, do_sample, logprobs, output_scores, return_dict_in_generate,
                                     max_new_tokens, stopping_criteria, eos_token_id, use_graph)
        N = num_return_sequences
        if isinstance(N, bool) or not isinstance(N, int) or N < 1:
            raise ValueError(f"num_return_sequences has to be a positive integer, got {N!r}")
        params = from_hf(do_sample, temperature, top_k, top_p, seed, **kw)
        sampled = params is not None
        if N > 1 and not sampled:
            raise ValueError(f"greedy decoding without beam search does not support num_return_sequences different "
                             f"than 1 (got {N})")
        n_top = check_logprobs(logprobs)
        want_lp = n_top is not None
        if sampled and self.llm.ep_world > 1:
            raise ValueError("sampled decoding is single-GPU (the expert-parallel mode serves greedy requests)")
        if want_lp and self.llm.ep_world > 1:
            raise ValueError("logprobs are single-GPU (the expert-parallel mode serves greedy requests)")
        if N > self.llm.max_batch:
            raise ValueError(f"num_return_sequences={N} exceeds the model's max_batch ({self.llm.max_batch}): the "
                             f"sequences run in decoder slots; build the model with max_batch >= {N}")
        if input_ids.shape[0] != 1:
            raise ValueError("generate() is single-sequence like the demo; use generate_batch() for more")
        if N > 1 and max_new_tokens < 1:
            raise ValueError("num_return_sequences > 1 needs max_new_tokens >= 1")
        emb, lens = self._embeds_for(input_ids, images, audios)
        llm = self.llm
        llm.check_capacity(lens[0], max_new_tokens)
        if N > 1:
            llm.reset()
            try:
                return self._run_samples(emb[0, : lens[0]].contiguous(), input_ids, N, params, n_top, output_scores,
                                         return_dict_in_generate, max_new_tokens, stopping_criteria, eos_token_id,
                                         use_graph, sync_every)
            finally:
                llm.cache.unshare()      # the static slot tables again, a full pool, greedy slots on stream 0
                for b in range(N):
                    llm.sampling.set(b, None)
        llm.reset()
        llm.sampling.set(0, params, n_top)
        width = llm.sampling.log_width(0, 1)                  # top entries the logprob log records (None: no log)
        score_log = llm.enable_score_log() if output_scores else None
        if want_lp:
            llm.enable_logprob_log()
        first = llm.prefill(emb[0, : lens[0]].contiguous(), slot=0, want_last_logits=output_scores, sampled=sampled,
                            scores=score_log, logprobs=width)
        if output_scores and not sampled:
            score_log[0].copy_(first[0])
        prompt = input_ids[0].tolist()
        L = len(prompt)
        seq_host = torch.empty(1, L + max_new_tokens, dtype=torch.long)      # one buffer; criteria get prefix views
        seq_host[0, :L] = torch.tensor(prompt, dtype=torch.long)
        n_new = checked = step = 0
        done = False
        while step < max_new_tokens and not done:
            n = min(sync_every, max_new_tokens - step)
            for _ in range(n):
                llm.decode_step(1, use_graph=use_graph, want_logits=output_scores, sampled=sampled,
                                logprobs=width)
            step += n
            toks = llm.generated_tokens(0)[:max_new_tokens]     # one host sync per `sync_every` tokens
            n_new = len(toks)
            seq_host[0, L + checked: L + n_new] = torch.tensor(toks[checked:], dtype=torch.long)
            for i in range(checked, n_new):                     # only the tokens added since the last sync
                stop = eos_token_id is not None and toks[i] == eos_token_id
                if not stop and stopping_criteria:
                    view = seq_host[:, : L + i + 1]
                    stop = any(bool(sc(view, None)) for sc in stopping_criteria)
                if stop:
                    n_new = i + 1
                    done = True
                    break
            checked = n_new
        seq = seq_host[:, : L + n_new].to(input_ids.device)
        if not return_dict_in_generate:
            return seq
        scores = tuple(score_log[i: i + 1] for i in range(n_new)) if output_scores else None
        lps = tuple(llm.read_logprobs(0, seq_host[0, L: L + n_new].tolist(), n_top)) if want_lp else None
        return GenerateOutput(seq, scores, lps)

    def _run_samples(self, emb, input_ids, N, params, n_top, output_scores, return_dict_in_generate, max_new_tokens,
                     stopping_criteria, eos_token_id, use_graph, sync_every):
        """generate(do_sample=True, num_return_sequences=N > 1), HF 4.41's `_sample` loop over the prompt expanded N
        times: prefill into slot 0, fork it into slots 1 .. N - 1 (MixtralDecoder.fork_sampled), then one batched
        step for all N per token.  Tokens are read back every `sync_every` steps; the stopping rules then run once per
        step on the [N, L + i + 1] view, in which finished rows hold the pad id."""
        llm = self.llm
        S = emb.shape[0]
        llm.sampling.set(0, params, n_top)
        width = llm.sampling.log_width(0, 1)
        score_log = llm.enable_beam_score_log(N, max_new_tokens) if output_scores else None
        if width is not None:
            llm.enable_logprob_log()
        llm.prefill(emb, slot=0, sampled=True, scores=score_log[0] if output_scores else None, logprobs=width)
        llm.fork_sampled(0, N, S, -(-(S + max_new_tokens) // llm.cache.page_size), score_log)
        prompt = input_ids[0].tolist()
        L, pad = len(prompt), eos_token_id               # HF pads with eos_token_id when no pad id is given
        seq_host = torch.empty(N, L + max_new_tokens, dtype=torch.long)
        seq_host[:, :L] = torch.tensor(prompt, dtype=torch.long)
        finished = torch.zeros(N, dtype=torch.bool)
        ends = [max_new_tokens] * N                      # tokens of each row before its padding
        t = step = 0
        while t < max_new_tokens and not bool(finished.all()):
            n = min(sync_every, max_new_tokens - step)
            for _ in range(n):
                llm.decode_step_batched(N, use_graph=use_graph, sampled=True, logprobs=width,
                                        warped_scores=output_scores)
            step += n
            t0, new = t, llm.token_log[:N, t:step].to("cpu", torch.long)   # one host sync per `sync_every` tokens
            for i in range(t0, step):
                col = new[:, i - t0].clone()
                if pad is not None:
                    col[finished] = pad
                seq_host[:, L + i] = col
                was = finished.clone()
                if eos_token_id is not None:
                    finished |= col == eos_token_id
                if stopping_criteria:
                    view = seq_host[:, : L + i + 1]
                    for sc in stopping_criteria:
                        finished |= torch.as_tensor(sc(view, None), dtype=torch.bool).reshape(-1).expand(N)
                for b in torch.nonzero(finished & ~was).flatten().tolist():
                    ends[b] = i + 1
                t = i + 1
                if bool(finished.all()):
                    break
        seq = seq_host[:, : L + t].to(input_ids.device)
        if not return_dict_in_generate:
            return seq
        scores = tuple(score_log[:N, i] for i in range(t)) if output_scores else None
        lps = None
        if n_top is not None:                           # without a pad id a finished row keeps its tokens
            lps = tuple(tuple(llm.read_logprobs(b, seq_host[b, L: L + (min(ends[b], t) if pad is not None else t)]
                                                .tolist(), n_top)) for b in range(N))
        return GenerateOutput(seq, scores, lps)

    @torch.no_grad()
    def _beam_search(self, input_ids, images, audios, N, R, length_penalty, early_stopping, do_sample, logprobs,
                     output_scores, return_dict_in_generate, max_new_tokens, stopping_criteria, eos_token_id,
                     use_graph):
        """generate(num_beams=N > 1): prefill once into slot 0, fork it into slots 1 .. N - 1 after the first choice,
        then one batched step over the N running beams per token.  Each step reads back every beam's top 2N
        logprobs (one host sync), lets BeamSearch choose, and moves the beams' KV rows to their new parents."""
        llm = self.llm
        check_beam_args(N, R, early_stopping)
        if do_sample:
            raise ValueError("beam-sample decoding (num_beams > 1 with do_sample=True) is not supported")
        if logprobs is not None:
            raise ValueError("logprobs= is not supported with num_beams > 1")
        if llm.ep_world > 1:
            raise ValueError("beam search is single-GPU (the expert-parallel mode serves greedy requests)")
        if N > llm.max_batch:
            raise ValueError(f"num_beams={N} exceeds the model's max_batch ({llm.max_batch}): the beams run in "
                             f"decoder slots; build the model with max_batch >= num_beams")
        if input_ids.shape[0] != 1:
            raise ValueError("generate() is single-sequence like the demo; use generate_batch() for more")
        if max_new_tokens < 1:
            raise ValueError("beam search needs max_new_tokens >= 1")
        emb, lens = self._embeds_for(input_ids, images, audios)
        llm.check_capacity(lens[0], max_new_tokens)
        llm.reset()
        try:
            return self._run_beams(emb[0, :lens[0]].contiguous(), input_ids, N, R, length_penalty, early_stopping,
                                   output_scores, return_dict_in_generate, max_new_tokens, stopping_criteria,
                                   eos_token_id, use_graph)
        finally:
            # the decoder leaves beam search as every other path expects it: block_table rows that agree with
            # slot_map's again (the engine's prefill writes through slot_map, the batched step reads block_table), a
            # full pool, greedy slots
            llm.cache.unshare()
            for b in range(N):
                llm.sampling.set(b, None)

    def _run_beams(self, emb, input_ids, N, R, length_penalty, early_stopping, output_scores,
                   return_dict_in_generate, max_new_tokens, stopping_criteria, eos_token_id, use_graph):
        llm = self.llm
        for b in range(N):
            llm.sampling.set(b, None, MAX_LOGPROBS)
        lp = llm.enable_logprob_log()
        score_log = llm.enable_beam_score_log(N, max_new_tokens) if output_scores else None
        S = emb.shape[0]
        llm.prefill(emb, slot=0, scores=score_log[0] if output_scores else None, logprobs=MAX_LOGPROBS,
                    log_softmax_scores=output_scores)
        if output_scores:
            score_log[1:N, 0].copy_(score_log[0, 0])          # step 0: HF's N identical rows of the expanded prompt
        prompt = input_ids[0].tolist()
        L, K = len(prompt), 2 * N
        seq_host = torch.empty(N, L + max_new_tokens, dtype=torch.long)      # the running beams, for the criteria
        seq_host[:, :L] = torch.tensor(prompt, dtype=torch.long)
        ids_h = torch.empty(N, K, dtype=torch.int32, pin_memory=True)
        lps_h = torch.empty(N, K, dtype=torch.float32, pin_memory=True)
        search = BeamSearch(N, max_new_tokens, eos_token_id, length_penalty, early_stopping)
        t, rows = 0, 1                 # t: tokens each running beam holds; rows: slots whose logprob row is current
        while True:
            ids_h[:rows].copy_(lp[2][:rows, t, :K], non_blocking=True)
            lps_h[:rows].copy_(lp[3][:rows, t, :K], non_blocking=True)
            torch.cuda.current_stream().synchronize()                       # the one host sync per step
            parents = search.step(ids_h[:rows].tolist(), lps_h[:rows].numpy())
            t += 1
            stop = False
            if stopping_criteria:      # every step, the last one included, as HF 4.41's beam search calls them
                for i, beam in enumerate(search.running):
                    seq_host[i, L:L + t] = torch.tensor(beam.tokens, dtype=torch.long)
                scores = tuple(score_log[:N, i] for i in range(t)) if output_scores else None
                stop = _criteria_stop(stopping_criteria, seq_host[:len(search.running), :L + t], scores)
            if search.done:
                break
            if stop:
                search.finalize()
                break
            if t == 1:                 # every first choice continues slot 0: fork it
                llm.fork(0, range(1, N), S)
            else:
                llm.cache.reorder(parents, S + t - 1)
            words = [0xFFFFFFFF - beam.tokens[-1] for beam in search.running]    # packed words decode_embed consumes
            llm.best[:N].copy_(torch.tensor(words, dtype=torch.int64))
            llm.decode_step_batched(N, use_graph=use_graph, logprobs=MAX_LOGPROBS, scores=output_scores)
            rows = N
        hyps = search.best(R)
        seq, seq_scores, beam_idx = pack_outputs(hyps, prompt, eos_token_id if eos_token_id is not None else 0)
        seq = torch.from_numpy(seq).to(input_ids.device)
        if not return_dict_in_generate:
            return seq
        scores = tuple(score_log[:N, i] for i in range(t)) if output_scores else None
        return GenerateOutput(seq, scores, None, torch.from_numpy(seq_scores), torch.from_numpy(beam_idx))


def _criteria_stop(stopping_criteria, view: torch.Tensor, scores) -> bool:
    """HF 4.41's StoppingCriteriaList over the running beams: a row is done when any criterion says so (a criterion
    may return one bool for all rows); the search stops when every row is done.  `scores`: the score blocks so far
    (output_scores) or None, as HF passes them."""
    done = torch.zeros(view.shape[0], dtype=torch.bool)
    for sc in stopping_criteria:
        done |= torch.as_tensor(sc(view, scores), dtype=torch.bool).reshape(-1).expand(view.shape[0])
    return bool(done.all())
