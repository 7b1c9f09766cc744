"""FP8 (e4m3) against bf16 KV cache, one process, the two alternating in every round (medians over --rounds).

(a) decode attention kernel alone (page 16, 16 splits): contexts 506 and 4160 at B = 1 and 16, CUDA events around
    --iters launches; GB/s of KV bytes read (2 x ctx x 8 heads x 128 x element size per row).  The launches cycle over
    enough copies of the cache (>= 256 MB of bf16 pages) that each one reads its pages from HBM, not from the 50 MB L2,
    as in a decode step, where the layer's weights pass through L2 between two attention launches.
(b) paged prefill: P = 4096 cached + C = 512 new rows, one sequence.  The e4m3 path's staging kernel alone and the whole
    e4m3 call (staging + FlashAttention over the scratch), next to the bf16 paged FlashAttention.
(c) bs = 1 greedy decode (CUDA graph), ms/token at S = 506 and 4160, --layers deep at full width, synthetic weights.
(d) the batched step at B = 16 with 4096-token contexts (GEMM path + paged decode attention), ms/step.  The two caches
    do not fit next to the weights together, so this part runs bf16 then fp8 (not interleaved).
(e) the largest max_batch at configs[4] geometry (--layers, max_seq_len --capacity-seq) whose decoder allocates, per
    dtype, from torch.cuda.mem_get_info with the weights resident, confirmed by allocating it.

Prints one JSON line with the card's name and power limit.
Usage: python scripts/kv_fp8_bench.py [--layers 24] [--rounds 5] [--iters 200] [--out FILE]
"""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vita_b200 import _lib, ops, weights as W      # noqa: E402
from vita_b200.config import VitaConfig            # noqa: E402
from vita_b200.model.mixtral import MixtralDecoder  # noqa: E402

NQ, NKV, D, PS = 32, 8, 128, 16
DTYPES = ("bf16", "fp8")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    return q or torch.cuda.get_device_name()


def med(xs):
    xs = sorted(xs)
    return round(xs[len(xs) // 2], 5)


def events(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def to_cache(x, dt):
    return x if dt == "bf16" else x.clamp(-448, 448).to(torch.float8_e4m3fn)


def attention_kernel(rounds, iters):
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    out = {}
    for ctx in (506, 4160):
        for B in (1, 16):
            n_pg = B * ((ctx + PS - 1) // PS)
            n_copies = -(-(256 << 20) // (2 * n_pg * PS * NKV * D * 2))
            kc = torch.randn(n_copies, n_pg * PS, NKV, D, generator=g, device=dev).to(torch.bfloat16)
            vc = torch.randn(n_copies, n_pg * PS, NKV, D, generator=g, device=dev).to(torch.bfloat16)
            caches = {dt: (to_cache(kc, dt), to_cache(vc, dt)) for dt in DTYPES}
            bt = torch.randperm(n_pg, generator=torch.Generator().manual_seed(ctx + B)).to(torch.int32).view(B, -1).to(dev)
            cur = torch.full((B,), ctx - 1, dtype=torch.int32, device=dev)
            q = torch.randn(B, NQ * D, generator=g, device=dev).to(torch.bfloat16)
            o = torch.empty_like(q)
            ws = ops.decode_attention_workspace(B, NKV, 16, dev)
            t = {dt: [] for dt in DTYPES}
            for r in range(rounds + 1):
                for dt in DTYPES:
                    k, v = caches[dt]
                    it = iter(range(1 << 30))

                    def f():
                        c = next(it) % n_copies
                        ops.decode_attention(q, k[c], v[c], bt, cur, o, ws, NQ, NKV, D, PS, 16, D ** -0.5)
                    ms = events(f, iters)
                    if r:
                        t[dt].append(ms)
            row = {}
            for dt in DTYPES:
                byts = 2 * B * ctx * NKV * D * (2 if dt == "bf16" else 1)
                row[dt] = {"us": round(med(t[dt]) * 1e3, 2), "GBps_kv": round(byts / (med(t[dt]) * 1e-3) / 1e9, 1)}
            row["cache_copies"] = n_copies
            out[f"ctx{ctx}_B{B}"] = row
            print("attention", ctx, B, row, flush=True)
    return out


def paged_prefill(rounds, iters):
    dev = torch.device("cuda")
    P, C = 4096, 512
    n = P + C
    n_pg = (n + PS - 1) // PS
    g = torch.Generator(device=dev).manual_seed(1)
    kc = torch.randn(n_pg * PS, NKV, D, generator=g, device=dev).to(torch.bfloat16)
    vc = torch.randn(n_pg * PS, NKV, D, generator=g, device=dev).to(torch.bfloat16)
    caches = {dt: (to_cache(kc, dt), to_cache(vc, dt)) for dt in DTYPES}
    bt = torch.randperm(n_pg, generator=torch.Generator().manual_seed(5)).to(torch.int32).view(1, -1).to(dev)
    q = torch.randn(C, NQ * D, generator=g, device=dev).to(torch.bfloat16)
    o = torch.empty_like(q)
    plan = ops.PagedPrefill([0, C], [n], bt, PS)
    work, _, k16, v16 = plan.fp8_stage(caches["fp8"][0])
    k8, v8 = caches["fp8"]
    stage = lambda: _lib.call("vita_kv_fp8_stage_pages", ops._p(k8), ops._p(v8), ops._p(bt), bt.stride(0),
                              ops._p(plan.ctx), ops._p(work), work.shape[0], ops._p(k16), ops._p(v16), NKV, D, PS,
                              1.0, 1.0, ops._stream())
    fns = {"bf16_flash": lambda: ops.attention_prefill_paged(q, kc, vc, plan, o, NQ, NKV, D, D ** -0.5),
           "fp8_stage_only": stage,
           "fp8_stage_plus_flash": lambda: ops.attention_prefill_paged(q, k8, v8, plan, o, NQ, NKV, D, D ** -0.5)}
    t = {k: [] for k in fns}
    for r in range(rounds + 1):
        for k, f in fns.items():
            ms = events(f, iters)
            if r:
                t[k].append(ms)
    res = {k: {"us": round(med(v) * 1e3, 2)} for k, v in t.items()}
    staged = 2 * n_pg * PS * NKV * D * 3          # 1 byte read + 2 bytes written per element, K and V
    res["fp8_stage_only"]["GBps"] = round(staged / (med(t["fp8_stage_only"]) * 1e-3) / 1e9, 1)
    res["scratch_bytes"] = 2 * n_pg * PS * NKV * D * 2
    res["shape"] = {"P": P, "C": C}
    print("paged prefill", res, flush=True)
    return res


def decode_bs1(packed, cfg, rounds, new_tokens):
    dev = torch.device("cuda")
    out = {}
    for S in (506, 4160):
        decs = {dt: MixtralDecoder(cfg.llm, packed["llm"], dev, max_batch=1, max_seq_len=S + new_tokens + 64,
                                   max_new_tokens=new_tokens + 16, kv_cache_dtype=dt) for dt in DTYPES}
        g = torch.Generator(device=dev).manual_seed(S)
        emb = (torch.randn(S, cfg.llm.hidden_size, device=dev, generator=g) * 0.5).to(torch.bfloat16)
        t = {dt: [] for dt in DTYPES}
        for r in range(rounds + 1):
            for dt, llm in decs.items():
                llm.reset()
                llm.prefill(emb.clone(), slot=0)
                llm.decode_step(1, use_graph=True)
                torch.cuda.synchronize()
                ms = events(lambda: llm.decode_step(1, use_graph=True), new_tokens)
                if r:
                    t[dt].append(ms)
        out[f"S{S}"] = {dt: {"ms_per_token": med(t[dt])} for dt in DTYPES}
        print("decode bs=1", S, out[f"S{S}"], flush=True)
        del decs
        gc.collect()
        torch.cuda.empty_cache()
    return out


def batched_step(packed, cfg, rounds, steps):
    dev = torch.device("cuda")
    B, S = 16, 4096
    out = {}
    for dt in DTYPES:
        llm = MixtralDecoder(cfg.llm, packed["llm"], dev, max_batch=B, max_seq_len=S + steps * (rounds + 2) + 64,
                             max_new_tokens=steps * (rounds + 2) + 16, kv_cache_dtype=dt)
        g = torch.Generator(device=dev).manual_seed(2)
        for b in range(B):
            emb = (torch.randn(S - 8 * b, cfg.llm.hidden_size, device=dev, generator=g) * 0.5).to(torch.bfloat16)
            llm.prefill(emb, slot=b)
        llm.decode_step_batched(B, use_graph=True)
        torch.cuda.synchronize()
        t = [events(lambda: llm.decode_step_batched(B, use_graph=True), steps) for _ in range(rounds)]
        out[dt] = {"ms_per_step": med(t)}
        print("batched step", dt, out[dt], flush=True)
        del llm
        gc.collect()
        torch.cuda.empty_cache()
    out["shape"] = {"B": B, "ctx": S}
    return out


def _allocates(cfg, packed, mb, seq, dt) -> bool:
    try:
        llm = MixtralDecoder(cfg.llm, packed["llm"], torch.device("cuda"), max_batch=mb, max_seq_len=seq,
                             max_new_tokens=64, kv_cache_dtype=dt)
        del llm
        return True
    except torch.OutOfMemoryError:
        return False


def capacity(packed, cfg, seq):
    """binary search on max_batch; each attempt builds the whole decoder (KV pages plus the per-slot decode state)"""
    out = {}
    per_tok = cfg.llm.num_hidden_layers * 2 * cfg.llm.num_key_value_heads * cfg.llm.head_dim
    for dt in DTYPES:
        gc.collect()
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info()
        per_seq = per_tok * ((seq + PS - 1) // PS * PS) * (2 if dt == "bf16" else 1)
        lo, hi = 0, int(free // per_seq) + 1            # lo allocates, hi does not
        while hi - lo > 1:
            mid = (lo + hi) // 2
            ok = _allocates(cfg, packed, mid, seq, dt)
            gc.collect()
            torch.cuda.empty_cache()
            lo, hi = (mid, hi) if ok else (lo, mid)
        out[dt] = {"max_batch": lo, "kv_bytes_per_seq": per_seq, "free_bytes_before": free}
        print("capacity", dt, out[dt], flush=True)
    out["max_seq_len"] = seq
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--new-tokens", type=int, default=64)
    ap.add_argument("--capacity-seq", type=int, default=4224)
    ap.add_argument("--out", default=None)
    ap.add_argument("--only", default="", help="comma-separated parts: attention,prefill,decode,batched,capacity")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    want = lambda part: not args.only or part in args.only.split(",")
    res = {"card": card(), "layers": args.layers}
    if want("attention"):
        res["decode_attention"] = attention_kernel(args.rounds, args.iters)
    if want("prefill"):
        res["paged_prefill"] = paged_prefill(args.rounds, args.iters // 4)
    cfg = VitaConfig.full(args.layers)
    packed = W.random_packed(cfg, torch.device("cuda"), seed=0, parts=("llm",))
    if want("decode"):
        res["decode_bs1"] = decode_bs1(packed, cfg, args.rounds, args.new_tokens)
    if want("batched"):
        res["batched_step_B16"] = batched_step(packed, cfg, args.rounds, 16)
    if want("capacity"):
        res["capacity"] = capacity(packed, cfg, args.capacity_seq)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
