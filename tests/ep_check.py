"""Expert-parallel prefill vs the single-GPU model with identical weights.  Run with torchrun (>= 2 GPUs):

    torchrun --nproc-per-node 2 tests/ep_check.py [--layers 2] [--seq 300] [--time-seq 4096 --time-layers 8]
"""
import argparse
import os
import sys
from pathlib import Path

import torch
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from vita_b200 import weights as W, parallel  # noqa: E402
from vita_b200.config import VitaConfig  # noqa: E402
from vita_b200.model.mixtral import MixtralDecoder  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--seq", type=int, default=300)
    ap.add_argument("--time-seq", type=int, default=0)
    ap.add_argument("--time-layers", type=int, default=8)
    args = ap.parse_args()
    world, rank, local = parallel.env_world()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    parallel.init("nccl", dev)
    cfg = VitaConfig.full(args.layers)
    ep_w = W.random_packed(cfg, dev, seed=3, parts=("llm",), ep=(rank, world))["llm"]
    dec = MixtralDecoder(cfg.llm, ep_w, dev, max_seq_len=args.seq + 64, max_new_tokens=8)
    g = torch.Generator(device=dev).manual_seed(11)
    emb = (torch.randn(args.seq, cfg.llm.hidden_size, device=dev, generator=g) * 0.05).to(torch.bfloat16)
    logits_ep = dec.prefill(emb.clone(), slot=0, all_logits=True).float()
    tok_ep = int(0xFFFFFFFF - (int(dec.best[0]) & 0xFFFFFFFF))
    # every rank returns the logits of its own token chunk, the owner of the last token holds the arg-max
    chunk = dec.ep_chunk(args.seq)
    pad = torch.zeros(chunk, logits_ep.shape[1], device=dev)
    pad[: logits_ep.shape[0]] = logits_ep
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad)
    logits_ep = torch.cat(parts)[: args.seq]
    t = torch.tensor([tok_ep if dec.best[0] != 0 else -1], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    tok_ep = int(t)
    ok = True
    if rank == 0:
        full_w = W.random_packed(cfg, dev, seed=3, parts=("llm",))["llm"]
        ref = MixtralDecoder(cfg.llm, full_w, dev, max_seq_len=args.seq + 64, max_new_tokens=8)
        logits_1 = ref.prefill(emb.clone(), slot=0, all_logits=True).float()
        tok_1 = int(0xFFFFFFFF - (int(ref.best[0]) & 0xFFFFFFFF))
        row_err = (logits_ep - logits_1).abs().amax(-1) / logits_1.abs().max()
        print(f"EP x{world} vs single GPU: median row err {row_err.median():.3e}, max {row_err.max():.3e}; "
              f"first token {tok_ep} vs {tok_1}")
        # every (token, k) row is produced once and summed in the single-GPU order -> bit-identical
        ok = bool(torch.equal(logits_ep, logits_1)) and tok_ep == tok_1
        print(f"bit-identical logits: {bool(torch.equal(logits_ep, logits_1))}")
        del ref, full_w
    if args.time_seq:
        cfg_t = VitaConfig.full(args.time_layers)
        w_t = W.random_packed(cfg_t, dev, seed=5, parts=("llm",), ep=(rank, world))["llm"]
        dec_t = MixtralDecoder(cfg_t.llm, w_t, dev, max_seq_len=args.time_seq + 64, max_new_tokens=8)
        emb_t = (torch.randn(args.time_seq, cfg_t.llm.hidden_size, device=dev) * 0.05).to(torch.bfloat16)
        for _ in range(2):
            dec_t.reset(); dec_t.prefill(emb_t.clone(), slot=0)
        dist.barrier(); torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 3
        a.record()
        for _ in range(n):
            dec_t.reset(); dec_t.prefill(emb_t.clone(), slot=0)
        b.record(); torch.cuda.synchronize()
        ms = parallel.reduce_max(a.elapsed_time(b) / n, dev)
        if rank == 0:
            S, L = args.time_seq, args.time_layers
            flops = (25.235e9 / 32 * L) * S + 2.62e5 / 32 * L * S * S + 0.424e9
            print(f"EP x{world} prefill S={S} L={L}: {ms:.2f} ms -> {flops / ms / 1e9:.1f} TFLOP/s aggregate "
                  f"({ms / L * 1e3:.0f} us/layer)")
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.broadcast(flag, 0)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if int(flag) == 1 else 1)


if __name__ == "__main__":
    main()
