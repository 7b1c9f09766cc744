"""InternViT-300M vision tower on the CUDA kernels.

Mirrors `InternViTVisionTower` (vita/model/multimodal_encoder/internvit/internvit_encoder.py:8-106) over
`InternVisionModel` (modeling_intern_vit.py:321-394): same call signature and output ([N, 256, 4096] for 448 px tiles),
select_layer = -1, CLS dropped, x0.5, pixel-shuffle.  All arithmetic runs in libvita_b200.so.
"""
from __future__ import annotations

import torch

from .. import ops
from ..config import VisionConfig

BF16 = torch.bfloat16


class InternViTVisionTower:
    def __init__(self, cfg: VisionConfig, weights: dict, device):
        self.cfg = cfg
        self.w = weights
        self.device = torch.device(device)
        self.dtype = BF16
        self.is_loaded = True
        self.select_layer = -1
        self.scale_pix_shuffle = cfg.scale_pix_shuffle
        self.image_processor = None  # set by the builder (CLIPImageProcessor constants, CPU preprocessing)

    def load_model(self):
        self.is_loaded = True

    @property
    def hidden_size(self) -> int:
        return self.cfg.out_dim

    @property
    def num_patches(self) -> int:
        return self.cfg.num_patches

    @torch.no_grad()
    def hidden_states(self, images: torch.Tensor) -> torch.Tensor:
        """Last hidden state [N, 1 + grid^2, hidden] (output of layer 24 == hidden_states[-1])."""
        c, w = self.cfg, self.w
        x = images.to(device=self.device, dtype=BF16).contiguous()
        n = x.shape[0]
        assert x.shape[1:] == (c.num_channels, c.image_size, c.image_size), "expected [N, 3, image, image] tiles"
        H, S = c.hidden_size, c.num_patches + 1
        col = torch.empty(n * c.num_patches, c.patch_k_pad, dtype=BF16, device=self.device)
        ops.vit_im2col(x, col, c.patch_size, c.patch_k_pad)
        patches = ops.linear(col, w["patch_w"], w["patch_b"])
        h = torch.empty(n, S, H, dtype=BF16, device=self.device)
        ops.vit_assemble(patches, w["cls"], w["pos"], h, n, c.num_patches, H)
        h2 = h.view(n * S, H)
        xn = torch.empty_like(h2)
        qkv = torch.empty(n * S, 3 * H, dtype=BF16, device=self.device)
        attn = torch.empty_like(h2)
        mid = torch.empty(n * S, c.intermediate_size, dtype=BF16, device=self.device)
        nh, D = c.num_attention_heads, H // c.num_attention_heads
        for lw in w["layers"]:
            ops.layernorm(h2, lw["ln1_w"], lw["ln1_b"], c.layer_norm_eps, out=xn)
            ops.linear(xn, lw["qkv_w"], lw["qkv_b"], out=qkv)
            ops.attention(qkv, qkv[:, H:], qkv[:, 2 * H:], attn, (S * 3 * H, 3 * H, D), (S * 3 * H, 3 * H, D),
                          (S * 3 * H, 3 * H, D), (S * H, H, D), n, nh, nh, S, S, D, D, None, False, D ** -0.5)
            ops.linear(attn, lw["proj_w"], lw["proj_b"], colscale=lw["ls1"], residual=h2, out=h2)
            ops.layernorm(h2, lw["ln2_w"], lw["ln2_b"], c.layer_norm_eps, out=xn)
            ops.linear(xn, lw["fc1_w"], lw["fc1_b"], act=ops.ACT_GELU, out=mid)
            ops.linear(mid, lw["fc2_w"], lw["fc2_b"], colscale=lw["ls2"], residual=h2, out=h2)
        return h

    @torch.no_grad()
    def forward(self, images) -> torch.Tensor:
        if isinstance(images, (list, tuple)):
            images = torch.stack([im for im in images])
        c = self.cfg
        h = self.hidden_states(images)
        n = h.shape[0]
        g = c.grid
        assert g * g == c.num_patches  # internvit_encoder.py:72
        out = torch.empty(n, c.out_tokens, c.out_dim, dtype=BF16, device=self.device)
        ops.vit_pixel_shuffle(h, out, n, g, c.hidden_size, c.scale_pix_shuffle)
        return out

    __call__ = forward


class VisionProjector:
    """mlp2x_gelu (vita/model/multimodal_projector/builder.py:160-168)."""

    def __init__(self, weights: dict):
        self.w = weights

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        y = ops.linear(x, self.w["w0"], self.w["b0"], act=ops.ACT_GELU)
        return ops.linear(y, self.w["w2"], self.w["b2"])
