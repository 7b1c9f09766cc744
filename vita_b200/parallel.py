"""Multi-GPU plumbing: one process per GPU, torch.distributed for rendezvous and the few scalar reductions.

Two ways the omni forward path shards (SURVEY.md section 8e):
* by *request* (decode, short prompts): a 24-layer cut (70 GB bf16) fits one 80 GB H100, so each rank owns
  complete requests and their KV cache and the data path needs no collective; the only exchanges are bookkeeping
  (max-over-ranks timings, gathering generated token lists on rank 0);
* by *expert and token* (one long sequence, BASELINE configs[3]): rank r holds experts [r E/N, (r+1) E/N) and owns the
  token chunk `token_range(S, r, N)` of the residual stream; `MixtralDecoder._prefill_ep_seq` moves K/V rows, routed
  activations and expert outputs between ranks with P2P stores over NVLink symmetric memory.
"""
from __future__ import annotations

import os
from typing import List, Sequence

import torch
import torch.distributed as dist


def env_world():
    return int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))


def init(backend: str, device=None):
    world, rank, local = env_world()
    if world > 1 and not dist.is_initialized():
        kw = {"device_id": device} if (backend == "nccl" and device is not None) else {}
        dist.init_process_group(backend, **kw)
    return world, rank, local


def shard_requests(n_requests: int, rank: int, world: int) -> List[int]:
    """Round-robin request ownership: request i runs on rank i % world (balanced to within one request)."""
    return list(range(rank, n_requests, world))


def sequence_chunk(S: int, world: int) -> int:
    """Tokens per rank of a sequence-sharded residual stream: ceil(S / world) rounded up to a multiple of 8 (keeps the
    8-byte routing records of a chunk 16-byte aligned for the P2P all-gather)."""
    return ((S + world - 1) // world + 7) // 8 * 8


def token_range(S: int, rank: int, world: int):
    """[t0, t1) owned by `rank`; trailing ranks may own nothing when S is short."""
    chunk = sequence_chunk(S, world)
    return min(rank * chunk, S), min((rank + 1) * chunk, S)


def reduce_max(x: float, device="cpu") -> float:
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return float(x)
    t = torch.tensor([x], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def reduce_sum(x: float, device="cpu") -> float:
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return float(x)
    t = torch.tensor([x], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t)


def gather_token_lists(local: Sequence[Sequence[int]], owned: Sequence[int], n_requests: int):
    """Collect per-request token lists on every rank (object all-gather; host side, after generation)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        out = [None] * n_requests
        for i, toks in zip(owned, local):
            out[i] = list(toks)
        return out
    parts = [None] * dist.get_world_size()
    dist.all_gather_object(parts, (list(owned), [list(t) for t in local]))
    out = [None] * n_requests
    for own, toks in parts:
        for i, t in zip(own, toks):
            out[i] = t
    return out
