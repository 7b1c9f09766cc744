"""Cost of log-probabilities: (a) the sampler kernel with logprob outputs, (b) ms per decoded token, greedy with and
without logprobs.

(a) CUDA events around --iters launches at V = 51760 for B in {1, 16, 64}, N in {0, 5, 20}, with T = 0 (greedy rows)
    and T 0.7 / top-k 50 / top-p 0.9; `ops.sample_rows` (no logprobs) is timed on the same rows as the baseline.
    Every configuration is timed in --repeats interleaved passes over all of them; the median and the spread are
    reported.
(b) bs = 1 decode at full layer width (synthetic weights, --layers deep, prompt of --ctx tokens), greedy without
    logprobs, with logprobs=0 and with logprobs=5, alternating inside one process like scripts/sampling_bench.py; each
    step's CUDA graph is captured once in the warm-up round and replayed after that; every turn times --new-tokens
    steps with CUDA events.  All variants must produce the same tokens (the logprob step takes the arg-max word of the
    same bf16 logits).

Usage: python scripts/logprobs_bench.py [--rounds 3] [--new-tokens 128] [--layers 24] [--ctx 506] [--repeats 5]
                                      [--out FILE]
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
from vita_b200.sampling import MAX_LOGPROBS        # noqa: E402

PARAM_SETS = {"greedy": (0.0, 0, 1.0), "T0.7+k50+p0.9": (0.7, 50, 0.9)}


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True,
                              timeout=30).stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def _time(fn, iters):
    for _ in range(20):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def kernel_times(V: int, iters: int, repeats: int):
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    runs = {}                                        # name -> launch closure
    for B in (1, 16, 64):
        logits = (torch.randn(B, V, device=dev, generator=g) * 2.5).to(torch.bfloat16)
        best = torch.zeros(B, dtype=torch.int64, device=dev)
        seed = torch.arange(B, dtype=torch.int64, device=dev) + 12345
        cnt = torch.zeros(B, dtype=torch.int32, device=dev)
        lp = torch.zeros(B, dtype=torch.float32, device=dev)
        rank = torch.zeros(B, dtype=torch.int32, device=dev)
        ids = torch.zeros(B, MAX_LOGPROBS, dtype=torch.int32, device=dev)
        tl = torch.zeros(B, MAX_LOGPROBS, dtype=torch.float32, device=dev)
        for name, (t, k, p) in PARAM_SETS.items():
            T = torch.full((B,), t, dtype=torch.float32, device=dev)
            K = torch.full((B,), k, dtype=torch.int32, device=dev)
            P = torch.full((B,), p, dtype=torch.float32, device=dev)
            a = (logits, T, K, P, seed, cnt, best)
            runs[f"B{B}_{name}_no_logprobs"] = lambda a=a: ops.sample_rows(*a)
            for N in (0, 5, 20):
                o = (lp, rank, ids, tl)
                runs[f"B{B}_{name}_N{N}"] = lambda a=a, o=o, N=N: ops.sample_logprobs(*a, *o, N)
    times = {k: [] for k in runs}
    for _ in range(repeats):
        for k, fn in runs.items():
            times[k].append(_time(fn, iters))
    out = {}
    for k, ts in times.items():
        ts = sorted(ts)
        out[k] = {"med": round(ts[len(ts) // 2], 2), "min": round(ts[0], 2), "max": round(ts[-1], 2)}
        print(f"sampler V={V} {k:32s} med {out[k]['med']:8.2f} us  [{out[k]['min']:.2f}, {out[k]['max']:.2f}]",
              flush=True)
    return out


def decode_times(args):
    dev = torch.device("cuda")
    cfg = VitaConfig.full(args.layers)
    packed = W.random_packed(cfg, dev, seed=0, parts=("llm",))
    llm = MixtralDecoder(cfg.llm, packed["llm"], dev, max_batch=1, max_seq_len=args.ctx + args.new_tokens + 64,
                         max_new_tokens=args.new_tokens + 16)
    g = torch.Generator(device=dev).manual_seed(1)
    emb = (torch.randn(args.ctx, cfg.llm.hidden_size, device=dev, generator=g) * 0.5).to(torch.bfloat16)
    variants = {"greedy": None, "greedy+logprobs0": 0, "greedy+logprobs5": 5}
    times = {n: [] for n in variants}
    toks = {}
    for r in range(args.rounds + 1):              # round 0 = warm-up + capture
        for name, n_top in variants.items():
            llm.reset()
            llm.sampling.set(0, None, n_top)
            width = llm.sampling.log_width(0, 1)
            llm.prefill(emb.clone(), slot=0, logprobs=width)
            llm.decode_step(1, use_graph=True, logprobs=width)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.new_tokens):
                llm.decode_step(1, use_graph=True, logprobs=width)
            b.record()
            b.synchronize()
            if r > 0:
                times[name].append(a.elapsed_time(b) / args.new_tokens)
            t = llm.token_log[0, : args.new_tokens + 1].tolist()
            toks.setdefault(name, t)
            assert toks[name] == t, f"{name}: tokens changed between rounds"
    assert toks["greedy"] == toks["greedy+logprobs0"] == toks["greedy+logprobs5"], "logprobs changed the tokens"
    out = {}
    for name, ts in times.items():
        ts = sorted(ts)
        out[name] = {"ms_per_token_min": round(ts[0], 4), "ms_per_token_med": round(ts[len(ts) // 2], 4),
                     "all": [round(t, 4) for t in times[name]]}
        print(f"decode {name:17s} min {ts[0]:.4f} ms  med {ts[len(ts) // 2]:.4f} ms  all {out[name]['all']}",
              flush=True)
    for n in ("greedy+logprobs0", "greedy+logprobs5"):
        out[f"{n}_over_greedy_med"] = round(out[n]["ms_per_token_med"] / out["greedy"]["ms_per_token_med"], 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--new-tokens", type=int, default=128)
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--ctx", type=int, default=506)
    ap.add_argument("--vocab", type=int, default=51760)
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--skip-decode", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("logprobs_bench.py needs a CUDA device")
    res = {"device": torch.cuda.get_device_name(), "gpu_name_power_limit": gpu_info()}
    print(f"device {res['device']}  (nvidia-smi: {res['gpu_name_power_limit']})", flush=True)
    res["sampler_us"] = kernel_times(args.vocab, args.iters, args.repeats)
    if not args.skip_decode:
        res["decode"] = decode_times(args)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
