"""Prefix caching in the continuous batcher: K questions about one video at configs[3] geometry, cache off and on.

Every request is the system prompt, then the frame and audio feature rows of one video (the same rows for every
question), then its question: S = 4160 prompt rows for K = 8 questions, 64 new tokens each, --layers deep (24: what
one 80 GB H100 holds, as bench.py), full layer width, synthetic weights.  The encoders are not run: the feature rows are
fixed synthetic rows spliced between the text embeddings (the encoders cost the same with the cache off and on).
All questions arrive at step 0; --max-batch of them decode together.  The two modes alternate for --rounds.

Reported per mode (median and spread over the rounds): time to first token of each request (its prefill call: digest,
admission and prefill, ended by a device synchronise; the requests are admitted one after another, so request i's
wait for requests < i is not included), whole-run tokens/s, and cached_tokens per request; plus the page-digest
kernel alone over S rows (CUDA events over --iters launches) and whether both modes produced the same tokens.
Prints one JSON line with the card's name and power limit.
Usage: python scripts/prefix_cache_bench.py [--layers 24] [--rounds 3] [--questions 8] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vita_b200 import ops, weights as W                       # noqa: E402
from vita_b200.config import VitaConfig                        # noqa: E402
from vita_b200.engine import ContinuousBatcher, DecoderEngine, Request  # noqa: E402
from vita_b200.model.mixtral import MixtralDecoder             # noqa: E402


def power_limit() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True,
                              timeout=30).stdout.strip() or "unknown"
    except Exception:
        return "unknown"


class VideoQuestions:
    """The model side DecoderEngine needs: `llm` and `_embeds_for`, here splicing fixed feature rows (payload
    "images") between the embeddings of the system prompt and of the question."""

    def __init__(self, llm, embed):
        self.llm, self.embed = llm, embed

    def _embeds_for(self, input_ids, images, audios):
        sys_ids, q_ids = input_ids
        emb = torch.cat([self.embed[sys_ids], images, self.embed[q_ids]])[None]
        return emb, torch.tensor([emb.shape[1]])


class TimedEngine(DecoderEngine):
    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.ttft = []

    def prefill(self, slot, request):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        P = super().prefill(slot, request)
        torch.cuda.synchronize()
        self.ttft.append((time.perf_counter() - t0) * 1e3)
        return P


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--questions", type=int, default=8)
    ap.add_argument("--max-batch", type=int, default=4)
    ap.add_argument("--new-tokens", type=int, default=64)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prefix_cache_bench.py needs a CUDA device")
    dev = torch.device("cuda")
    n_sys, n_feat, n_q = 64, 4064, 32                # S = 4160 rows: system prompt, frame + audio features, question
    S = n_sys + n_feat + n_q
    cfg = VitaConfig.full(args.layers)
    packed = W.random_packed(cfg, dev, seed=0, parts=("llm",))
    llm = MixtralDecoder(cfg.llm, packed["llm"], dev, max_batch=args.max_batch, max_seq_len=S + args.new_tokens + 16,
                         max_new_tokens=args.new_tokens)
    model = VideoQuestions(llm, packed["llm"]["embed"])
    g = torch.Generator().manual_seed(1)
    V = cfg.llm.vocab_size
    sys_ids = torch.randint(0, V, (n_sys,), generator=g).to(dev)
    feats = (torch.randn(n_feat, cfg.llm.hidden_size, generator=g) * 0.02).to(dev, torch.bfloat16)
    questions = [torch.randint(0, V, (n_q,), generator=g).to(dev) for _ in range(args.questions)]

    def requests():
        return [Request(i, {"input_ids": (sys_ids, q), "images": feats}, args.new_tokens)
                for i, q in enumerate(questions)]

    def run(prefix_cache):
        llm.reset()
        eng = TimedEngine(model, prefix_cache=prefix_cache)
        reqs = requests()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = ContinuousBatcher(eng, args.max_batch).run(reqs)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        return {"ttft_ms": eng.ttft, "tok_s": sum(len(t) for t in out.values()) / wall,
                "cached": [r.cached_tokens for r in reqs]}, out

    run(False)                                        # warm-up: graphs of every batch size, workspaces
    run(True)
    res = {False: [], True: []}
    outs = {}
    for _ in range(args.rounds):
        for mode in (False, True):
            r, outs[mode] = run(mode)
            res[mode].append(r)

    rows = torch.randn(S, cfg.llm.hidden_size, generator=g).to(dev, torch.bfloat16)
    for _ in range(10):
        ops.page_digest(rows, llm.cache.page_size)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.iters):
        ops.page_digest(rows, llm.cache.page_size)
    b.record()
    b.synchronize()

    def summary(rs):
        med = lambda v: sorted(v)[len(v) // 2]
        ttft = list(zip(*[r["ttft_ms"] for r in rs]))            # per request, over the rounds
        return {"ttft_ms_median": [round(med(t), 2) for t in ttft],
                "ttft_ms_min_max": [[round(min(t), 2), round(max(t), 2)] for t in ttft],
                "tok_s": [round(r["tok_s"], 1) for r in rs], "cached_tokens": rs[-1]["cached"]}

    line = json.dumps({"gpu": torch.cuda.get_device_name(), "power_limit": power_limit(), "layers": args.layers,
                       "prompt_rows": S, "questions": args.questions, "new_tokens": args.new_tokens,
                       "max_batch": args.max_batch, "cache_off": summary(res[False]), "cache_on": summary(res[True]),
                       "digest_us": round(a.elapsed_time(b) / args.iters * 1e3, 2),
                       "same_tokens": outs[False] == outs[True]})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
