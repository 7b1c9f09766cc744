"""Sampled decoding: the one place that maps generation parameters to the per-row sampler parameters.

The kernel (csrc/sample.cu, `ops.sample_rows`) takes, per row, `temperature` (0 = greedy), `top_k` (<= 0: off),
`top_p` (>= 1: off), a 64-bit Philox key `seed`, and the index `n` of the token being drawn within its request (the
decoder passes its device-resident `gen_count`, so a request draws the same tokens in any slot, batch or graph).

Warping follows HF transformers 4.41 (`TemperatureLogitsWarper` -> `TopKLogitsWarper` -> `TopPLogitsWarper`, the
version the reference pins), which is also what vLLM does: x = l / T in fp32 from the bf16 logits; top-k keeps every
token >= the k-th largest logit; top-p keeps a top-k survivor iff the softmax mass of the survivors with a strictly
greater logit is < top_p (tied logits are kept or dropped together; the largest always stays).  The draw is a
Gumbel-max over the kept set, an exact sample of the renormalised warped distribution; it matches the distribution
of HF and vLLM, not their torch RNG streams.

Parameters come from two surfaces:
  * HF `generate(do_sample=True, temperature=, top_k=, top_p=, seed=)` -> `from_hf`;
  * vLLM `SamplingParams` (per sequence group) -> `from_vllm`.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch

# HF transformers 4.41 GenerationConfig defaults (what `None` means with do_sample=True)
HF_DEFAULT_TEMPERATURE, HF_DEFAULT_TOP_K, HF_DEFAULT_TOP_P = 1.0, 50, 1.0
# vLLM samples when temperature >= _SAMPLING_EPS (vllm/sampling_params.py); below it the request is greedy
VLLM_SAMPLING_EPS = 1e-5
U64 = (1 << 64) - 1

# sampling-only kwargs of HF generate() this library does not implement: name -> value that leaves the output as is
_HF_UNSUPPORTED = {"typical_p": 1.0, "min_p": None, "epsilon_cutoff": 0.0, "eta_cutoff": 0.0,
                   "repetition_penalty": 1.0, "no_repeat_ngram_size": 0}


@dataclass(frozen=True)
class SamplingParams:
    """One row's sampler parameters (already normalised: top_k 0 = off, top_p 1.0 = off)."""
    temperature: float
    top_k: int = 0
    top_p: float = 1.0
    seed: int = 0

    def __post_init__(self):
        if not self.temperature > 0:
            raise ValueError(f"temperature must be > 0 for a sampled row, got {self.temperature}")
        if self.top_k < 0:
            raise ValueError(f"top_k must be >= 0 (0 = off), got {self.top_k}")
        if not 0.0 <= self.top_p <= 1.0:
            raise ValueError(f"top_p must be in [0, 1], got {self.top_p}")
        if not 0 <= self.seed <= U64:
            raise ValueError(f"seed must be in [0, 2**64), got {self.seed}")


def draw_key(generator: Optional[torch.Generator] = None) -> int:
    """A 64-bit stream key from torch's default CPU generator (or `generator`): two draws of
    `torch.randint(0, 2**32, (2,))`, key = w[0] | w[1] << 32.  `torch.manual_seed(s)` therefore makes it
    reproducible, as HF users expect of generate(do_sample=True)."""
    w = torch.randint(0, 1 << 32, (2,), dtype=torch.int64, generator=generator).tolist()
    return int(w[0]) | (int(w[1]) << 32)


def from_hf(do_sample: bool, temperature=None, top_k=None, top_p=None, seed: Optional[int] = None,
            **kw) -> Optional[SamplingParams]:
    """HF generate() kwargs -> SamplingParams, or None for greedy (do_sample=False: the warpers are not applied).
    None means the GenerationConfig default; out-of-range values raise ValueError like HF's warpers do; sampling
    kwargs this library cannot honour raise instead of being ignored.  Without `seed` one key is drawn (draw_key)."""
    if not do_sample:
        return None
    for name, neutral in _HF_UNSUPPORTED.items():
        if name in kw and kw[name] is not None and kw[name] != neutral:
            raise ValueError(f"{name}={kw[name]!r} is not supported by vita_b200's sampler")
    t = HF_DEFAULT_TEMPERATURE if temperature is None else temperature
    k = HF_DEFAULT_TOP_K if top_k is None else top_k
    p = HF_DEFAULT_TOP_P if top_p is None else top_p
    if isinstance(t, bool) or not isinstance(t, (int, float)) or not t > 0:
        raise ValueError(f"`temperature` (={t}) has to be a strictly positive float with do_sample=True")
    if isinstance(k, bool) or not isinstance(k, int) or k < 0:
        raise ValueError(f"`top_k` has to be a strictly positive integer (or 0 = off), but is {k}")
    p = float(p)
    if p < 0 or p > 1.0:
        raise ValueError(f"`top_p` has to be a float >= 0 and <= 1, but is {p}")
    return SamplingParams(float(t), int(k), p, draw_key() if seed is None else int(seed))


def from_vllm(sp) -> Optional[SamplingParams]:
    """vLLM SamplingParams -> SamplingParams, or None for greedy (temperature < 1e-5).  top_k -1 or 0 is off.
    Unseeded sampled rows get a fresh key from torch's default generator (call order = row order).  Features outside
    this sampler raise NotImplementedError."""
    g = lambda name, default: getattr(sp, name, default)
    if g("n", 1) > 1 or (g("best_of", None) or 1) > 1:
        raise NotImplementedError("n > 1 / best_of > 1 (several sequences per request) is not supported")
    if g("use_beam_search", False):
        raise NotImplementedError("beam search is not supported")
    if g("presence_penalty", 0.0) != 0.0 or g("frequency_penalty", 0.0) != 0.0 or g("repetition_penalty", 1.0) != 1.0:
        raise NotImplementedError("presence / frequency / repetition penalties are not supported")
    if (g("min_p", 0.0) or 0.0) > 0.0:
        raise NotImplementedError("min_p is not supported")
    t = float(g("temperature", 1.0))
    if t < VLLM_SAMPLING_EPS:
        return None
    k = int(g("top_k", -1))
    if k < -1:
        raise ValueError(f"top_k must be -1 (disable) or at least 1, got {k}")
    seed = g("seed", None)
    return SamplingParams(t, max(k, 0), float(g("top_p", 1.0)), draw_key() if seed is None else int(seed) & U64)


def _i64(u: int) -> int:
    """u64 bit pattern as the int64 the device tensor stores."""
    return u - (1 << 64) if u >= (1 << 63) else u


def row_tensors(rows: List[Optional[SamplingParams]], device):
    """Per-row kernel parameters (temperature f32, top_k i32, top_p f32, seed i64; None = greedy) for a whole batch,
    built on the host and moved with one copy per tensor."""
    ps = [p or SamplingParams(1.0) for p in rows]
    t = torch.tensor([p.temperature if r is not None else 0.0 for p, r in zip(ps, rows)], dtype=torch.float32)
    k = torch.tensor([p.top_k for p in ps], dtype=torch.int32)
    tp = torch.tensor([p.top_p for p in ps], dtype=torch.float32)
    s = torch.tensor([_i64(p.seed) for p in ps], dtype=torch.int64)
    return tuple(x.to(device, non_blocking=True) for x in (t, k, tp, s))


class SlotSampling:
    """Per-slot sampler parameters of a decoder: [max_batch] device tensors (what the kernel reads, moved with their
    slot) plus a host mirror of which slots sample (to pick the greedy or the sampled step)."""

    def __init__(self, max_batch: int, device):
        dev = torch.device(device)
        self.temperature = torch.zeros(max_batch, dtype=torch.float32, device=dev)
        self.top_k = torch.zeros(max_batch, dtype=torch.int32, device=dev)
        self.top_p = torch.ones(max_batch, dtype=torch.float32, device=dev)
        self.seed = torch.zeros(max_batch, dtype=torch.int64, device=dev)
        self.sampled: List[bool] = [False] * max_batch

    @property
    def tensors(self):
        return [self.temperature, self.top_k, self.top_p, self.seed]

    def set(self, slot: int, params: Optional[SamplingParams]) -> None:
        """params None = greedy."""
        p = params or SamplingParams(1.0)
        row = slice(slot, slot + 1)
        self.temperature[row] = p.temperature if params is not None else 0.0
        self.top_k[row] = p.top_k
        self.top_p[row] = p.top_p
        self.seed[row] = _i64(p.seed)
        self.sampled[slot] = params is not None

    def swap(self, i: int, j: int) -> None:
        self.sampled[i], self.sampled[j] = self.sampled[j], self.sampled[i]

    def any_sampled(self, n: int) -> bool:
        return any(self.sampled[:n])
