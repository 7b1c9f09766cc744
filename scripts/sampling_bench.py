"""Cost of sampled decoding: (a) the sampler kernel alone, (b) ms per decoded token, greedy against sampled.

(a) CUDA events around >= 1000 launches of ops.sample_rows at V = 51760 for B in {1, 16, 64} and the parameter sets
    T only / T + top-k 50 / T + top-p 0.9 / T + top-k 50 + top-p 0.9 (T = 0.7).
(b) bs = 1 decode at full layer width (synthetic weights, --layers deep, prompt of --ctx tokens), the greedy and the
    sampled (T 0.7, top-k 50, top-p 0.9) step alternating inside one process like scripts/decode_ab.py; each step's
    CUDA graph is captured once in the warm-up round and replayed after that; every turn times --new-tokens steps with
    CUDA events.  The token logs of the greedy rounds must be equal (and so must those of the sampled rounds: same
    key, same counters).

Usage: python scripts/sampling_bench.py [--rounds 3] [--new-tokens 128] [--layers 24] [--ctx 506] [--out FILE]
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
from vita_b200.sampling import SamplingParams      # noqa: E402

PARAM_SETS = {"T": (0.7, 0, 1.0), "T+k50": (0.7, 50, 1.0), "T+p0.9": (0.7, 0, 0.9), "T+k50+p0.9": (0.7, 50, 0.9)}


def power_limit() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True,
                              timeout=30).stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def kernel_times(V: int, iters: int):
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    out = {}
    for B in (1, 16, 64):
        logits = (torch.randn(B, V, device=dev, generator=g) * 2.5).to(torch.bfloat16)
        best = torch.zeros(B, dtype=torch.int64, device=dev)
        seed = torch.arange(B, dtype=torch.int64, device=dev) + 12345
        cnt = torch.zeros(B, dtype=torch.int32, device=dev)
        for name, (t, k, p) in PARAM_SETS.items():
            T = torch.full((B,), t, dtype=torch.float32, device=dev)
            K = torch.full((B,), k, dtype=torch.int32, device=dev)
            P = torch.full((B,), p, dtype=torch.float32, device=dev)
            for _ in range(20):
                ops.sample_rows(logits, T, K, P, seed, cnt, best)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                ops.sample_rows(logits, T, K, P, seed, cnt, best)
            b.record()
            b.synchronize()
            us = a.elapsed_time(b) * 1e3 / iters
            out[f"B{B}_{name}"] = round(us, 2)
            print(f"sampler V={V} B={B:3d} {name:12s} {us:8.2f} us", flush=True)
    return out


def decode_times(args):
    dev = torch.device("cuda")
    cfg = VitaConfig.full(args.layers)
    packed = W.random_packed(cfg, dev, seed=0, parts=("llm",))
    llm = MixtralDecoder(cfg.llm, packed["llm"], dev, max_batch=1, max_seq_len=args.ctx + args.new_tokens + 64,
                         max_new_tokens=args.new_tokens + 16)
    g = torch.Generator(device=dev).manual_seed(1)
    emb = (torch.randn(args.ctx, cfg.llm.hidden_size, device=dev, generator=g) * 0.5).to(torch.bfloat16)
    params = {"greedy": None, "sampled": SamplingParams(0.7, 50, 0.9, 0xABCDEF)}
    times = {n: [] for n in params}
    toks = {}
    for r in range(args.rounds + 1):              # round 0 = warm-up + capture
        for name, sp in params.items():
            sampled = sp is not None
            llm.reset()
            llm.sampling.set(0, sp)
            llm.prefill(emb.clone(), slot=0, sampled=sampled)
            llm.decode_step(1, use_graph=True, sampled=sampled)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.new_tokens):
                llm.decode_step(1, use_graph=True, sampled=sampled)
            b.record()
            b.synchronize()
            if r > 0:
                times[name].append(a.elapsed_time(b) / args.new_tokens)
            t = llm.token_log[0, : args.new_tokens + 1].tolist()
            toks.setdefault(name, t)
            assert toks[name] == t, f"{name}: tokens changed between rounds"
    out = {}
    for name, ts in times.items():
        ts = sorted(ts)
        out[name] = {"ms_per_token_min": round(ts[0], 4), "ms_per_token_med": round(ts[len(ts) // 2], 4),
                     "all": [round(t, 4) for t in times[name]]}
        print(f"decode {name:8s} min {ts[0]:.4f} ms  med {ts[len(ts) // 2]:.4f} ms  all {out[name]['all']}", flush=True)
    out["sampled_over_greedy_med"] = round(out["sampled"]["ms_per_token_med"] / out["greedy"]["ms_per_token_med"], 4)
    out["sampled_tokens_differ_from_greedy"] = toks["sampled"] != toks["greedy"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--new-tokens", type=int, default=128)
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--ctx", type=int, default=506)
    ap.add_argument("--vocab", type=int, default=51760)
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--skip-decode", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sampling_bench.py needs a CUDA device")
    res = {"device": torch.cuda.get_device_name(), "power_limit": power_limit()}
    print(f"device {res['device']}  power limit {res['power_limit']}", flush=True)
    res["sampler_us"] = kernel_times(args.vocab, args.iters)
    if not args.skip_decode:
        res["decode"] = decode_times(args)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
