"""Chunked prefill and prefix reuse: (a) the paged-KV attention kernel alone, (b) time to first token of a second turn.

(a) CUDA events around --iters launches of ops.attention_prefill_paged (Mixtral GQA 32 / 8 heads of 128, page size 16,
    shuffled pages, one sequence) at P cached in {0, 1024, 4096} x C new in {64, 512, 2048}; achieved TFLOP/s from the
    causal FLOP count 4 C (P + C / 2) 128 32.  At P = 0 the contiguous kernel (ops.attention) at the same shape too.
(b) A second conversation turn at configs[3] geometry: P = 4160 tokens already in the cache (turn 1) plus 64 new
    tokens, prefilled as a continuation (prefill(start = 4160)) against re-prefilling all 4224 tokens, full layer
    width, --layers deep (24: what one 80 GB H100 holds, as bench.py), synthetic weights; CUDA events, median of
    --rounds, the two alternating.

Prints one JSON line with the card's name and power limit.
Usage: python scripts/paged_prefill_bench.py [--iters 200] [--layers 24] [--rounds 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vita_b200 import ops, weights as W           # noqa: E402
from vita_b200.config import VitaConfig            # noqa: E402
from vita_b200.model.mixtral import MixtralDecoder  # noqa: E402

NQ, NKV, D, PS = 32, 8, 128, 16


def power_limit() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True,
                              timeout=30).stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def timed(fn, iters):
    for _ in range(10):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def kernel(iters):
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    rows = []
    for P in (0, 1024, 4096):
        for C in (64, 512, 2048):
            n = P + C
            n_pg = (n + PS - 1) // PS
            perm = torch.randperm(n_pg, generator=torch.Generator().manual_seed(P + C)).to(torch.int32)
            kc = torch.randn(n_pg * PS, NKV, D, generator=g, device=dev).to(torch.bfloat16)
            vc = torch.randn_like(kc)
            q = torch.randn(C, (NQ + 2 * NKV) * D, generator=g, device=dev).to(torch.bfloat16)
            out = torch.empty(C, NQ * D, dtype=torch.bfloat16, device=dev)
            plan = ops.PagedPrefill([0, C], [n], perm.view(1, -1).to(dev), PS)
            ms = timed(lambda: ops.attention_prefill_paged(q[:, :NQ * D], kc, vc, plan, out, NQ, NKV, D, D ** -0.5),
                       iters)
            flops = 4.0 * C * (P + C / 2) * D * NQ
            row = {"P": P, "C": C, "paged_us": round(ms * 1e3, 2), "paged_tflops": round(flops / ms / 1e9, 1)}
            if P == 0:
                k, v = q[:, NQ * D:(NQ + NKV) * D], q[:, (NQ + NKV) * D:]
                W_ = q.stride(0)
                ms0 = timed(lambda: ops.attention(q, k, v, out, (0, W_, D), (0, W_, D), (0, W_, D), (0, NQ * D, D), 1,
                                                  NQ, NKV, C, C, D, D, None, True, D ** -0.5), iters)
                row.update(contiguous_us=round(ms0 * 1e3, 2), contiguous_tflops=round(flops / ms0 / 1e9, 1))
            rows.append(row)
    return rows


def second_turn(layers, rounds, P=4160, C=64):
    dev = torch.device("cuda")
    cfg = VitaConfig.full(layers)
    packed = W.random_packed(cfg, dev, seed=0, parts=("llm",))
    llm = MixtralDecoder(cfg.llm, packed["llm"], dev, max_batch=1, max_seq_len=P + C + 64, max_new_tokens=8)
    ids = torch.randint(0, cfg.llm.vocab_size, (P + C,), generator=torch.Generator().manual_seed(1)).to(dev)
    emb = packed["llm"]["embed"][ids].contiguous()

    def run(cont):
        x = emb[P:].clone() if cont else emb.clone()
        if cont:
            llm.cache.cache_len.fill_(P)     # turn 1 is in the cache; the continuation rewrites rows P.. identically
        else:
            llm.reset()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        if cont:
            llm.prefill(x, slot=0, start=P)
        else:
            llm.prefill(x, slot=0)
        b.record()
        b.synchronize()
        return a.elapsed_time(b), int(llm.best[0])

    run(False)
    cont, full = [], []
    for _ in range(rounds):
        full.append(run(False))
        cont.append(run(True))
    med = lambda v: sorted(t for t, _ in v)[len(v) // 2]
    same = len({tok for _, tok in cont + full}) == 1
    return {"layers": layers, "cached": P, "new": C, "continue_ms": round(med(cont), 3),
            "reprefill_ms": round(med(full), 3), "first_token_equal": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("paged_prefill_bench.py needs a CUDA device")
    res = {"gpu": torch.cuda.get_device_name(), "power_limit": power_limit(), "kernel": kernel(args.iters),
           "second_turn": second_turn(args.layers, args.rounds)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
