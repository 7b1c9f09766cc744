#!/usr/bin/env python
"""BASELINE configs[4] on one GPU: B concurrent audio queries (10 s audio + short prompt each), paged-KV batched
greedy decode; reports p50 / p99 inter-token latency and tokens/s.  (8 x H100 = 8 such replicas.)

    python scripts/bench_cfg5.py [--batch 16] [--new-tokens 256] [--layers 32]
    python scripts/bench_cfg5.py --arrivals 12          # staggered arrivals (mean gap in decode steps) through the
                                                        # continuous batcher, with duplex events (negative-audio abort,
                                                        # barge-in interrupt); under torchrun the 16 queries are sharded
                                                        # over the ranks (request parallel) and the latencies gathered
    python scripts/bench_cfg5.py --arrivals 12 --prefill-chunk 512   # the same mix plus one video-length (4096-token)
                                                        # arrival, run without and with chunked admission (one GPU)
"""
import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from vita_b200 import weights as W  # noqa: E402
from vita_b200.config import VitaConfig, AUDIO_TOKEN_INDEX  # noqa: E402
from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM  # noqa: E402


def run_arrivals(args):
    """configs[4] as specified: concurrent audio queries ARRIVING over time, one weight copy per GPU, continuous
    batching over the paged KV cache; p50 / p99 inter-token latency as seen by the running requests (a step that also
    admits a new query includes that query's encoder + prefill: this is the latency a user hears), time to first token,
    and what the duplex events did."""
    import random
    import torch.distributed as dist
    from vita_b200 import parallel
    from vita_b200.engine import ContinuousBatcher, DecoderEngine, Request
    world, rank, local = parallel.env_world()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    parallel.init("nccl", dev)
    cfg = VitaConfig.full(args.layers)
    B, NT = args.batch, args.new_tokens
    mine = parallel.shard_requests(B, rank, world)
    packed = W.random_packed(cfg, dev, seed=0, parts=("llm", "vision", "projector", "audio"))
    long_len = 4096 if args.prefill_chunk else 0
    model = VITAMixtralForCausalLM(cfg, packed, dev, max_batch=max(len(mine), 1) + (1 if long_len else 0),
                                   max_seq_len=max(512, long_len) + NT + 16, max_new_tokens=NT + 16)
    rng = random.Random(7)
    g = torch.Generator().manual_seed(0)
    reqs, t = [], 0
    dummy_image = torch.zeros(1, 3, cfg.vision.image_size, cfg.vision.image_size)      # video_audio_demo.py:227
    for b in range(B):
        t += int(rng.expovariate(1.0 / args.arrivals)) if b else 0
        ids = torch.randint(0, cfg.llm.vocab_size - 8, (1, 140 + 2 * b), generator=g)
        ids[0, 3] = AUDIO_TOKEN_INDEX
        payload = {"input_ids": ids, "images": dummy_image,
                   "audios": {"audios": torch.randn(1, 998, 80, generator=g), "lengths": torch.tensor([998])}}
        # sessions of 2 queries each: the second query of a session barges in on the first one's answer
        reqs.append(Request(b, payload, NT, None, arrival_step=t, session=b // 2, negative_token_id=cfg.llm.vocab_size - 1))
    if long_len:
        # an 8-frame video conversation turn (S ~ 4096; text rows stand in for the spliced frame features, the prefill
        # cost is the same), arriving in the middle of the mix
        assert world == 1, "--prefill-chunk measures one GPU"
        ids = torch.randint(0, cfg.llm.vocab_size - 8, (1, long_len), generator=g)
        reqs.append(Request(B, {"input_ids": ids}, NT, None, arrival_step=reqs[B // 2].arrival_step))
        mine = list(mine) + [B]
    my_reqs = [r for r in reqs if r.rid in mine]
    eng = DecoderEngine(model, use_graph=True, overrun=8, lone_fast_path=True)
    # warm-up: every batch size this rank will see gets its graph captured outside the measurement
    warm = [Request(100 + i, r.payload, 4, None, 0) for i, r in enumerate(my_reqs)]
    ContinuousBatcher(eng, max(len(mine), 1), sync_every=4).run(warm)
    model.llm.reset()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()

    def measure(chunk):
        marks = []
        start = torch.cuda.Event(enable_timing=True)
        start.record()

        def on_step(step, n_active):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            marks.append((step, n_active, e))

        for r in my_reqs:
            r.steps, r.tokens, r.outcome = 0, [], ""
        out = ContinuousBatcher(eng, max(len(mine), 1), sync_every=8, prefill_chunk=chunk).run(my_reqs, on_step=on_step)
        torch.cuda.synchronize()
        ts = [(st, n, start.elapsed_time(e)) for st, n, e in marks]
        itl = []                                            # one sample per (step, active request)
        for (s0, n0, t0), (s1, n1, t1) in zip(ts, ts[1:]):
            itl += [t1 - t0] * n1
        total_tokens = sum(len(v) for v in out.values())
        wall_ms = ts[-1][2] if ts else 0.0
        return {"itl": itl, "tokens": total_tokens, "wall_ms": wall_ms,
                "outcomes": [r.outcome for r in my_reqs], "steps": len(ts)}

    if long_len:
        q = lambda v, p: sorted(v)[min(len(v) - 1, int(len(v) * p))]
        res = {}
        for chunk in (None, args.prefill_chunk):
            r = measure(chunk)
            res["whole" if chunk is None else f"chunk_{chunk}"] = {
                "p50_itl_ms": q(r["itl"], 0.5), "p99_itl_ms": q(r["itl"], 0.99), "max_itl_ms": max(r["itl"]),
                "tokens_per_s": r["tokens"] / (r["wall_ms"] / 1e3), "steps": r["steps"]}
        print(json.dumps({
            "workload": f"configs[4] arrivals (mean gap {args.arrivals} steps) plus one {long_len}-token arrival, "
                        f"{NT} new tokens each, {args.layers} layers, 1 GPU: arrivals prefilled whole vs. chunked "
                        f"admission with a budget of {args.prefill_chunk} tokens per step",
            "gpu": torch.cuda.get_device_name(), "power_limit": _power_limit(), **res}))
        return
    rec = measure(None)
    allrec = [None] * world
    if world > 1:
        dist.all_gather_object(allrec, rec)
    else:
        allrec = [rec]
    if rank == 0:
        itl_all = sorted(x for r in allrec for x in r["itl"])
        oc = [o for r in allrec for o in r["outcomes"]]
        q = lambda p: itl_all[min(len(itl_all) - 1, int(len(itl_all) * p))] if itl_all else None
        print(json.dumps({
            "workload": f"configs[4]: {B} audio queries (10 s audio + ~140-170 text tokens each) arriving with mean gap "
                        f"{args.arrivals} decode steps, {NT} new tokens each, {args.layers} layers, {world} GPU(s), "
                        "request parallel (queries sharded over GPUs, full weight copy per GPU), continuous batching",
            "n_gpus": world, "p50_itl_ms": q(0.5), "p90_itl_ms": q(0.9), "p99_itl_ms": q(0.99),
            "tokens_per_s_aggregate": sum(r["tokens"] for r in allrec) / (max(r["wall_ms"] for r in allrec) / 1e3),
            "tokens_per_s_per_gpu": sum(r["tokens"] for r in allrec) / (max(r["wall_ms"] for r in allrec) / 1e3) / world,
            "duplex_outcomes": {k: oc.count(k) for k in sorted(set(oc))},
            "itl_samples": len(itl_all),
            "note": "a step that admits an arrival includes its Whale encoder + prefill (what the running requests "
                    "wait for); CUDA events after every batched decode step"}))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def _power_limit() -> str:
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True,
                              timeout=30).stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--new-tokens", type=int, default=256)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--arrivals", type=float, default=0.0, help="mean gap between arrivals in decode steps (0 = all at step 0)")
    ap.add_argument("--prefill-chunk", type=int, default=None,
                    help="with --arrivals: add a 4096-token arrival and compare whole against chunked admission")
    args = ap.parse_args()
    if args.arrivals > 0:
        return run_arrivals(args)
    dev = torch.device("cuda", 0)
    cfg = VitaConfig.full(args.layers)
    B, NT = args.batch, args.new_tokens
    packed = W.random_packed(cfg, dev, seed=0, parts=("llm", "audio"))
    model = VITAMixtralForCausalLM(cfg, packed, dev, max_batch=B, max_seq_len=512 + NT, max_new_tokens=NT + 8)
    g = torch.Generator().manual_seed(0)
    reqs = []
    for b in range(B):
        ids = torch.randint(0, cfg.llm.vocab_size, (1, 140 + 2 * b), generator=g)
        ids[0, 3] = AUDIO_TOKEN_INDEX
        reqs.append({"input_ids": ids, "audios": {"audios": torch.randn(1, 998, 80, generator=g),
                                                   "lengths": torch.tensor([998])}})
    # audio-only requests: the splice needs the (dummy) image feature slot like the demo passes (video_audio_demo.py:227)
    for r in reqs:
        r["images"] = None
    def embeds(r):
        a = model.encode_audios(r["audios"]["audios"], r["audios"]["lengths"])["inputs_embeds"]
        ids = r["input_ids"][0].tolist()
        k = ids.index(AUDIO_TOKEN_INDEX)
        tok = lambda t: model._embeds_for(torch.tensor([t]), None, None)[0][0]
        return torch.cat([tok(ids[:k]), a[0], tok(ids[k + 1:])]).contiguous()
    model.llm.reset()
    events = []
    def run(record):
        model.llm.reset()
        for b, r in enumerate(reqs):
            model.llm.prefill(embeds(r), slot=b)
        for s in range(NT):
            model.llm.decode_step_batched(B, use_graph=True)
            if record:
                e = torch.cuda.Event(enable_timing=True); e.record(); events.append(e)
    run(False)
    torch.cuda.synchronize()
    start = torch.cuda.Event(enable_timing=True)
    model.llm.reset()
    for b, r in enumerate(reqs):
        model.llm.prefill(embeds(r), slot=b)
    start.record()
    for s in range(NT):
        model.llm.decode_step_batched(B, use_graph=True)
        e = torch.cuda.Event(enable_timing=True); e.record(); events.append(e)
    torch.cuda.synchronize()
    ts = [start.elapsed_time(e) for e in events]
    itl = sorted(b - a for a, b in zip([0.0] + ts[:-1], ts))
    toks = [model.llm.generated_tokens(b) for b in range(B)]
    assert all(len(t) == NT for t in toks)
    out = {"workload": f"configs[4] on 1 GPU: {B} concurrent audio queries (S0~264-294), {NT} decode steps, "
                       f"{args.layers} layers", "batch": B, "p50_itl_ms": itl[len(itl) // 2],
           "p99_itl_ms": itl[int(len(itl) * 0.99) - 1], "tokens_per_s": B * NT / (ts[-1] / 1e3),
           "launches_per_step": model.llm.launches_per_batched_step}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
