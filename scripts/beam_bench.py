"""Cost of beam search per decoded step at full layer width (synthetic weights, --layers deep, a prompt of --ctx
tokens, --new-tokens steps without EOS so every call runs all steps).

For N = 1 (today's greedy generate()) and N in {2, 4, 8} (generate(num_beams=N)), interleaved over --rounds rounds
(round 0 warms up and captures the CUDA graphs):
  * end-to-end: host clock around generate() ending in a device synchronise, minus a max_new_tokens=1 call (the
    prefill and one step) timed in the same round, over --new-tokens;
  * split (N > 1), from a loop that repeats generate()'s beam loop: the batched step (CUDA events), the host gap
    between the end of the [N, 2N] readback and the next launch (bookkeeping, copy-on-write update, token upload),
    and within it the copy-on-write update; the kv_copy_pages kernel alone (CUDA events over 200 launches of N - 1
    page pairs over every layer's K and V cache, with the bytes it moves).
Medians over the rounds.  The card's name and power limit are read in the same run.

Usage: python scripts/beam_bench.py [--rounds 3] [--new-tokens 128] [--layers 24] [--ctx 506] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vita_b200 import ops, weights as W                          # noqa: E402
from vita_b200.beam import BeamSearch                            # noqa: E402
from vita_b200.config import VitaConfig                          # noqa: E402
from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM  # noqa: E402
from vita_b200.sampling import MAX_LOGPROBS                      # noqa: E402

BEAMS = (1, 2, 4, 8)


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


def split_loop(model, ids, N, steps):
    """generate()'s beam loop with timers, means per step: the batched step (CUDA events), the host gap from the end of
    the readback synchronise to the next step's launch (BeamSearch.step, the copy-on-write update, the token upload),
    and the copy-on-write update alone (host clock around MixtralDecoder.fork / PagedKVCache.reorder, which ends with
    enqueuing kv_copy_pages)."""
    llm = model.llm
    emb = model._embeds_for(ids, None, None)[0][0].contiguous()
    S = emb.shape[0]
    llm.reset()
    for b in range(N):
        llm.sampling.set(b, None, MAX_LOGPROBS)
    lp = llm.enable_logprob_log()
    llm.prefill(emb, slot=0, logprobs=MAX_LOGPROBS)
    ids_h = torch.empty(N, 2 * N, dtype=torch.int32, pin_memory=True)
    lps_h = torch.empty(N, 2 * N, dtype=torch.float32, pin_memory=True)
    search = BeamSearch(N, steps)
    rec = {"step": [], "host_gap": [], "cow_host": []}
    t, rows, pending = 0, 1, None
    while True:
        ids_h[:rows].copy_(lp[2][:rows, t, :2 * N], non_blocking=True)
        lps_h[:rows].copy_(lp[3][:rows, t, :2 * N], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        h0 = time.perf_counter()
        if pending is not None:                      # the previous step's events are complete now
            rec["step"].append(pending[0].elapsed_time(pending[1]))
        parents = search.step(ids_h[:rows].tolist(), lps_h[:rows].numpy())
        t += 1
        if search.done:
            break
        h1 = time.perf_counter()
        if t == 1:
            llm.fork(0, range(1, N), S)
        else:
            llm.cache.reorder(parents, S + t - 1)
        rec["cow_host"].append((time.perf_counter() - h1) * 1e3)
        llm.best[:N].copy_(torch.tensor([0xFFFFFFFF - b.tokens[-1] for b in search.running], dtype=torch.int64))
        rec["host_gap"].append((time.perf_counter() - h0) * 1e3)
        pending = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        pending[0].record()
        llm.decode_step_batched(N, use_graph=True, logprobs=MAX_LOGPROBS)
        pending[1].record()
        rows = N
    return {k: sum(v) / len(v) for k, v in rec.items() if v}


def kv_copy_time(model, N, iters=200):
    """kv_copy_pages alone: N - 1 page pairs over the K and V caches of every layer (one step of N beams that all
    continue one parent), CUDA events over `iters` launches; ms per launch and the bytes moved (read + write)."""
    cache = model.llm.cache
    n_pages = cache.k[0].shape[0] // cache.page_size
    page_bytes = cache.page_size * cache.k[0][0].numel() * cache.k[0].element_size()
    base = torch.tensor([t.data_ptr() for t in cache.k + cache.v], dtype=torch.int64, device="cuda")
    pairs = torch.tensor([(0, n_pages - 1 - i) for i in range(N - 1)], dtype=torch.int32, device="cuda")
    launch = lambda: ops.kv_copy_pages(base, pairs, n_pages, page_bytes)
    for _ in range(20):
        launch()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        launch()
    b.record()
    b.synchronize()
    ms = a.elapsed_time(b) / iters
    nbytes = 2 * (N - 1) * len(cache.k + cache.v) * page_bytes
    return ms, nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--new-tokens", type=int, default=128)
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--ctx", type=int, default=506)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "beam_bench measures on the GPU"
    dev = torch.device("cuda")
    info = gpu_info()
    print(f"gpu: {info}", flush=True)
    cfg = VitaConfig.full(args.layers)
    packed = W.random_packed(cfg, dev, seed=0, parts=("llm",))
    model = VITAMixtralForCausalLM(cfg, packed, dev, max_batch=max(BEAMS), max_seq_len=args.ctx + args.new_tokens + 64,
                                   max_new_tokens=args.new_tokens + 16)
    ids = torch.randint(3, cfg.llm.vocab_size, (1, args.ctx), generator=torch.Generator().manual_seed(0))
    e2e = {n: [] for n in BEAMS}
    split = {n: [] for n in BEAMS if n > 1}
    prefill = []
    for r in range(args.rounds + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.generate(ids, max_new_tokens=1)
        torch.cuda.synchronize()
        pre = (time.perf_counter() - t0) * 1e3
        for n in BEAMS:
            kw = {} if n == 1 else dict(num_beams=n)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model.generate(ids, max_new_tokens=args.new_tokens, **kw)
            torch.cuda.synchronize()
            ms = ((time.perf_counter() - t0) * 1e3 - pre) / args.new_tokens
            if n > 1:
                sp = split_loop(model, ids, n, args.new_tokens)
            if r > 0:
                prefill.append(pre)
                e2e[n].append(ms)
                if n > 1:
                    split[n].append(sp)
    res = {"gpu": info, "layers": args.layers, "ctx": args.ctx, "new_tokens": args.new_tokens,
           "prefill_ms_med": round(_med(prefill), 3)}
    for n in BEAMS:
        row = {"ms_per_step_med": round(_med(e2e[n]), 3), "all": [round(x, 3) for x in e2e[n]]}
        if n > 1:
            for k in split[n][0]:
                row[f"{k}_ms_med"] = round(_med([s[k] for s in split[n]]), 4)
            ms, nbytes = kv_copy_time(model, n)
            row["kv_copy_kernel_ms"] = round(ms, 4)
            row["kv_copy_GB_per_s"] = round(nbytes / ms / 1e6, 1)
        res[f"N={n}"] = row
        print(f"N={n}: {row}", flush=True)
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
