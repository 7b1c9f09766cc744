"""Bring-up / benchmark aid for the wgmma FlashAttention (flash_tc.cu): one case per process so that a device trap
in one case does not take the others down.  usage: python scripts/fa_check.py <kind> <S> [bench]
kind: mix (causal GQA 32/8 x 128), vit (16 x 64, batch 8), whale (16 heads, 128/64, padded batch of 2)"""
import sys
import time

import torch

sys.path.insert(0, ".")
from vita_b200 import ops  # noqa: E402

BF16 = torch.bfloat16


def ref_attn(q, k, v, scale, causal, kv_lens=None):
    B, Hq, Sq, _ = q.shape
    Hkv, Skv = k.shape[1], k.shape[2]
    k = k.repeat_interleave(Hq // Hkv, 1)
    v = v.repeat_interleave(Hq // Hkv, 1)
    out = torch.empty(B, Hq, Sq, v.shape[-1], device=q.device)
    for h in range(Hq):      # per head: keeps the fp32 score tensor small
        s = torch.matmul(q[:, h].float(), k[:, h].float().transpose(-1, -2)) * scale
        if causal:
            s = s.masked_fill(torch.arange(Skv, device=q.device)[None, :] > torch.arange(Sq, device=q.device)[:, None],
                              float("-inf"))
        if kv_lens is not None:
            s = s.masked_fill((torch.arange(Skv, device=q.device)[None, :] >= kv_lens[:, None])[:, None, :], float("-inf"))
        out[:, h] = torch.matmul(torch.softmax(s, -1), v[:, h].float())
    return out


def main():
    kind, S = sys.argv[1], int(sys.argv[2])
    bench = len(sys.argv) > 3
    torch.manual_seed(0)
    dev = "cuda"
    if kind == "mix":
        nq, nkv, D = 32, 8, 128
        W = (nq + 2 * nkv) * D
        qkv = (torch.randn(S, W, device=dev)).to(BF16)
        out = torch.zeros(S, nq * D, dtype=BF16, device=dev)
        run = lambda: ops.attention(qkv, qkv[:, nq * D:], qkv[:, (nq + nkv) * D:], out, (0, W, D), (0, W, D), (0, W, D),
                                    (0, nq * D, D), 1, nq, nkv, S, S, D, D, None, True, D ** -0.5)
        q = qkv[:, :nq * D].view(S, nq, D).transpose(0, 1)[None]
        k = qkv[:, nq * D:(nq + nkv) * D].view(S, nkv, D).transpose(0, 1)[None]
        v = qkv[:, (nq + nkv) * D:].view(S, nkv, D).transpose(0, 1)[None]
        ref = lambda: ref_attn(q, k, v, D ** -0.5, True)[0].transpose(0, 1).reshape(S, nq * D)
        flops = 4 * S * S * D * nq / 2
    elif kind == "vit":
        N, nh, D = 8, 16, 64
        H = nh * D
        qkv = torch.randn(N, S, 3 * H, device=dev).to(BF16)
        out = torch.zeros(N, S, H, dtype=BF16, device=dev)
        run = lambda: ops.attention(qkv, qkv[..., H:], qkv[..., 2 * H:], out, (S * 3 * H, 3 * H, D), (S * 3 * H, 3 * H, D),
                                    (S * 3 * H, 3 * H, D), (S * H, H, D), N, nh, nh, S, S, D, D, None, False, D ** -0.5)
        t = qkv.view(N, S, 3, nh, D).permute(2, 0, 3, 1, 4)
        ref = lambda: ref_attn(t[0], t[1], t[2], D ** -0.5, False).transpose(1, 2).reshape(N, S, H)
        flops = 4 * S * S * D * nh * N
    else:
        B, nh, dk = 2, 16, 64
        q2 = torch.randn(B, S, nh, 2 * dk, device=dev).to(BF16)
        k2 = torch.randn(B, S, nh, 2 * dk, device=dev).to(BF16)
        qkv = torch.randn(B, S, 3 * nh * dk, device=dev).to(BF16)
        lens = torch.tensor([S, max(1, S - 29)], dtype=torch.int32, device=dev)
        out = torch.zeros(B, S, nh * dk, dtype=BF16, device=dev)
        run = lambda: ops.attention(q2, k2, qkv[..., 2 * nh * dk:], out, (S * nh * 2 * dk, nh * 2 * dk, 2 * dk),
                                    (S * nh * 2 * dk, nh * 2 * dk, 2 * dk), (S * 3 * nh * dk, 3 * nh * dk, dk),
                                    (S * nh * dk, nh * dk, dk), B, nh, nh, S, S, 2 * dk, dk, lens, False, dk ** -0.5)
        vv = qkv[..., 2 * nh * dk:].view(B, S, nh, dk).transpose(1, 2)
        ref = lambda: ref_attn(q2.transpose(1, 2), k2.transpose(1, 2), vv, dk ** -0.5, False, lens.long()) \
            .transpose(1, 2).reshape(B, S, nh * dk)
        flops = 4 * S * S * 3 * dk * nh * B / 1.5
    run()
    torch.cuda.synchronize()
    r = ref()
    err = (out.float() - r).abs()
    rel = err.max().item() / r.abs().max().item()
    bad = (err > 2e-2 * r.abs().max()).float().mean().item()
    print(f"[fa_check] {kind} S={S}: max err {err.max().item():.4e} max|ref| {r.abs().max().item():.3f} rel {rel:.3e} "
          f"frac bad {bad:.4f} finite {bool(torch.isfinite(out.float()).all())}", flush=True)
    if rel > 2e-2:
        fl = out.float().flatten()
        print("   got ", fl[:8].tolist(), "\n   want", r.flatten()[:8].tolist(), flush=True)
    if bench:
        for _ in range(3):
            run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 20
        e0.record()
        for _ in range(n):
            run()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / n
        print(f"[fa_bench] {kind} S={S}: {us:.1f} us  {flops / us / 1e6:.1f} TFLOP/s (algorithmic)", flush=True)


if __name__ == "__main__":
    main()
