"""Whale audio encoder + CNNSubsampling adapter on the CUDA kernels.

Mirrors `audioEncoder.forward` (vita/model/multimodal_encoder/whale/init_model.py:114-139): fbank features
[B, T, 80] + lengths [B] -> {"inputs_embeds": [B, T''', H_llm], "attention_mask": [B, T''']} with the shipped stack
(GlobalCMVN -> Conv2dSubsampling4 -> 24-layer rel-pos Transformer -> CNNSubsampling adapter).  The random
dynamic-chunk mask of the reference's training default is off (parity note 8 of SURVEY.md section 8a): plain padding mask.
"""
from __future__ import annotations

import math

import torch

from .. import ops
from ..config import AudioConfig

BF16 = torch.bfloat16


class AudioEncoder:
    def __init__(self, cfg: AudioConfig, llm_hidden: int, weights: dict, device):
        self.cfg = cfg
        self.w = weights
        self.llm_hidden = llm_hidden
        self.device = torch.device(device)
        self.dtype = BF16
        # `.audio_processor.process(path) -> (fbank [T, 80], n_llm_tokens)` as the demo uses it
        # (video_audio_demo.py:183-187); the filterbank itself runs on the GPU (csrc/fbank.cu)
        from ..audio_frontend import AudioProcessor
        self.audio_processor = AudioProcessor(device)
        self._pos_proj = {}     # T2 -> per-layer linear_pos(pos_emb): input independent, computed once per length

    def to(self, *args, **kwargs):  # the demo calls audio_encoder.to(dtype=torch.float16) (video_audio_demo.py:176)
        return self

    @torch.no_grad()
    def encode(self, feats: torch.Tensor, lengths: torch.Tensor):
        """Encoder output before the adapter: ([B, T'', C] bf16, valid lengths int32 [B])."""
        c, w = self.cfg, self.w
        feat = feats.to(device=self.device, dtype=torch.float32).contiguous()
        B, T, Fd = feat.shape
        C = c.hidden_size
        T1, F1 = (T - 1) // 2, (Fd - 1) // 2
        T2, F2 = (T1 - 1) // 2, (F1 - 1) // 2
        assert F2 == c.freq_bins and T2 >= 1, "input too short / wrong feature dimension"
        lens = lengths.to(device=self.device).to(torch.int64).clamp(max=T)
        lens2 = (((lens - 1) // 2 - 1) // 2).clamp(min=0).to(torch.int32)   # mask[:, :, 2::2][:, :, 2::2]
        x1 = torch.empty(B, T1, F1, C, dtype=BF16, device=self.device)
        ops.whale_conv1(feat, w["cmvn_mean"], w["cmvn_istd"], w["conv1_w"], w["conv1_b"], x1)
        col = torch.empty(B * T2 * F2, 9 * C, dtype=BF16, device=self.device)
        ops.whale_im2col2(x1, col, B, T1, F1, C)
        x2 = ops.linear(col, w["conv2_w"], w["conv2_b"], act=ops.ACT_RELU)          # [B*T2*F2, C] == [B*T2, F2*C]
        x = ops.linear(x2.view(B * T2, F2 * C), w["sub_out_w"], w["sub_out_b"])
        x = ops.linear(x, w["embed_w"], w["embed_b"])
        x = ops.layernorm(x, w["embed_ln_w"], w["embed_ln_b"], c.layer_norm_eps, ops.ACT_RELU, math.sqrt(C))
        assert T2 < c.max_len
        if T2 not in self._pos_proj:      # attention.py:381 p = linear_pos(pos_emb): depends on the length only
            with torch.inference_mode(False):
                self._pos_proj[T2] = [ops.linear(w["pos_table"][:T2], lw["pos_w"]) for lw in w["layers"]]
        pos_proj = self._pos_proj[T2]
        nh, dk = c.num_attention_heads, c.head_dim
        y = torch.empty_like(x)
        qkv = torch.empty(B * T2, 3 * C, dtype=BF16, device=self.device)
        q2 = torch.empty(B * T2, nh, 2 * dk, dtype=BF16, device=self.device)
        k2 = torch.empty_like(q2)
        attn = torch.empty_like(x)
        mid = torch.empty(B * T2, c.linear_units, dtype=BF16, device=self.device)
        for lw, p in zip(w["layers"], pos_proj):
            ops.layernorm(x, lw["ln1_w"], lw["ln1_b"], c.layer_norm_eps, out=y)
            ops.linear(y, lw["qkv_w"], lw["qkv_b"], out=qkv)
            ops.whale_qk_prep(qkv, p, lw["bias_u"], lw["bias_v"], q2, k2, B, T2, nh, dk)
            ops.attention(q2, k2, qkv[:, 2 * C:], attn, (T2 * nh * 2 * dk, nh * 2 * dk, 2 * dk),
                          (T2 * nh * 2 * dk, nh * 2 * dk, 2 * dk), (T2 * 3 * C, 3 * C, dk), (T2 * C, C, dk), B, nh, nh,
                          T2, T2, 2 * dk, dk, lens2, False, dk ** -0.5)
            ops.linear(attn, lw["out_w"], lw["out_b"], residual=x, out=x)
            ops.layernorm(x, lw["ln2_w"], lw["ln2_b"], c.layer_norm_eps, out=y)
            ops.linear(y, lw["w1"], lw["b1"], act=ops.ACT_RELU, out=mid)
            ops.linear(mid, lw["w2"], lw["b2"], residual=x, out=x)
        x = ops.layernorm(x, w["after_w"], w["after_b"], c.layer_norm_eps)
        return x.view(B, T2, C), lens2

    @torch.no_grad()
    def forward(self, audios: torch.Tensor, lengths: torch.Tensor):
        c, w = self.cfg, self.w
        if audios.dim() == 2:
            audios = audios.unsqueeze(0)
        lengths = torch.as_tensor(lengths).reshape(-1)
        x, lens2 = self.encode(audios, lengths)
        B, T2, C = x.shape
        T3 = (T2 - 1) // 2 + 1
        k = c.adapter_kernel
        col = torch.empty(B * T3, k * C, dtype=BF16, device=self.device)
        ops.whale_adapter_im2col(x, lens2, col, B, T2, C, k)
        y = ops.linear(col, w["ad_conv_w"], w["ad_conv_b"])
        y = ops.layernorm(y, w["ad_ln_w"], w["ad_ln_b"], c.adapter_ln_eps, ops.ACT_GELU)
        out = ops.linear(y, w["ad_proj_w"], w["ad_proj_b"]).view(B, T3, self.llm_hidden)
        lens3 = (lens2 + 1) // 2                                                       # mask_pad[:, :, 0::2]
        mask = torch.arange(T3, device=self.device)[None, :] < lens3[:, None]
        return {"inputs_embeds": out, "attention_mask": mask}

    __call__ = forward
