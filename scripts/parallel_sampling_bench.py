"""Parallel sampling against separate requests at full layer width (synthetic weights, --layers deep).

For each prompt length S in --ctx (506: a text prompt; 4160: the row count of the video prompt, whose decoder cost is
the same whatever the rows hold) and N in {2, 4, 8} sampled sequences of one prompt, interleaved over --rounds rounds
(round 0 warms up and captures the CUDA graphs):
  * fork: one prefill into slot 0, then MixtralDecoder.fork_sampled into slots 1 .. N - 1 (what
    generate(num_return_sequences=N) and a Request with n = N do);
  * separate: N prefills of the same prompt into slots 0 .. N - 1 (N requests, no prefix cache);
each followed by --new-tokens sampled batched steps over the N slots.  Reported per (S, N, mode): the time to all N
first tokens (host clock around the prefills and the fork, ending in a device synchronise), within it the fork alone,
ms per batched step (CUDA events over the steps), and the KV pages the N sequences hold after their last step.
Medians over the rounds.  The card's name and power limit are read in the same run.

Usage: python scripts/parallel_sampling_bench.py [--rounds 3] [--new-tokens 64] [--layers 24] [--ctx 506,4160]
                                                  [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vita_b200 import weights as W                               # noqa: E402
from vita_b200.config import VitaConfig                          # noqa: E402
from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM  # noqa: E402
from vita_b200.sampling import SamplingParams                    # noqa: E402

NS = (2, 4, 8)
SP = SamplingParams(0.8, 50, 0.95, 1234)


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True,
                              timeout=30).stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def _med(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def run(model, emb, N, new, fork):
    """One (N, mode) measurement: ms to all N first tokens, ms of the fork, ms per batched step, pages held."""
    llm = model.llm
    S, ps = emb.shape[0], llm.cache.page_size
    rows = [emb.clone() for _ in range(1 if fork else N)]          # prefill consumes its rows
    llm.reset()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if fork:
        llm.sampling.set(0, SP)
        llm.prefill(rows[0], slot=0, sampled=True)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        llm.fork_sampled(0, N, S, -(-(S + new + 1) // ps))
    else:
        for b in range(N):
            llm.sampling.set(b, SP)
            llm.sampling.stream[b] = b
            llm.prefill(rows[b], slot=b, sampled=True)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(new):
        llm.decode_step_batched(N, use_graph=True, sampled=True)
    b.record()
    b.synchronize()
    n_pages = -(-(S + new) // ps)                                  # pages covering what each sequence wrote
    if fork:
        pages = len({pg for row in llm.cache.pool.table[:N] for pg in row[:n_pages]})
    else:
        pages = N * n_pages
    for s in range(N):
        llm.sampling.set(s, None)
    llm.reset()
    return (t2 - t0) * 1e3, (t2 - t1) * 1e3 if fork else 0.0, a.elapsed_time(b) / new, pages


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--new-tokens", type=int, default=64)
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--ctx", default="506,4160")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "parallel_sampling_bench measures on the GPU"
    dev = torch.device("cuda")
    info = gpu_info()
    print(f"gpu: {info}", flush=True)
    ctxs = [int(x) for x in args.ctx.split(",")]
    cfg = VitaConfig.full(args.layers)
    packed = W.random_packed(cfg, dev, seed=0, parts=("llm",))
    model = VITAMixtralForCausalLM(cfg, packed, dev, max_batch=max(NS), max_seq_len=max(ctxs) + args.new_tokens + 64,
                                   max_new_tokens=args.new_tokens + 16)
    results = []
    for S in ctxs:
        ids = torch.randint(3, cfg.llm.vocab_size, (1, S), generator=torch.Generator().manual_seed(S))
        emb = model._embeds_for(ids, None, None)[0][0, :S].contiguous()
        rec = {(n, f): [] for n in NS for f in (True, False)}
        for r in range(args.rounds + 1):
            for n in NS:
                for f in (True, False):
                    m = run(model, emb, n, args.new_tokens, f)
                    if r:
                        rec[(n, f)].append(m)
        for n in NS:
            for f in (True, False):
                ms = rec[(n, f)]
                row = {"ctx": S, "n": n, "mode": "fork" if f else "separate",
                       "first_tokens_ms": round(_med([m[0] for m in ms]), 3),
                       "fork_ms": round(_med([m[1] for m in ms]), 3),
                       "step_ms": round(_med([m[2] for m in ms]), 4), "kv_pages": ms[0][3]}
                results.append(row)
                print(json.dumps(row), flush=True)
    out = {"gpu": info, "layers": args.layers, "new_tokens": args.new_tokens, "rounds": args.rounds,
           "results": results}
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
