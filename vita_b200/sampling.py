"""Sampled decoding: the one place that maps generation parameters to the per-row sampler parameters.

The kernel (csrc/sample.cu, `ops.sample_rows`) takes, per row, `temperature` (0 = greedy), `top_k` (<= 0: off),
`top_p` (>= 1: off), a 64-bit Philox key `seed`, the index `n` of the token being drawn within its request (the
decoder passes its device-resident `gen_count`, so a request draws the same tokens in any slot, batch or graph), and a
stream index `s`: the noise of token n comes from Philox counter (r >> 2, n, s, 0).

Parallel sampling (`generate(do_sample=True, num_return_sequences=N)`, `Request.n` / `Request.best_of`): the N
sequences of one request share its key and draw from streams 0 .. N-1 (`SlotSampling.fork`), so they are independent
samples, reproducible from one seed, and sequence 0 draws exactly what the same request with one sequence draws.

Warping follows HF transformers 4.41 (`TemperatureLogitsWarper` -> `TopKLogitsWarper` -> `TopPLogitsWarper`, the
version the reference pins), which is also what vLLM does: x = l / T in fp32 from the bf16 logits; top-k keeps every
token >= the k-th largest logit; top-p keeps a top-k survivor iff the softmax mass of the survivors with a strictly
greater logit is < top_p (tied logits are kept or dropped together; the largest always stays).  The draw is a
Gumbel-max over the kept set, an exact sample of the renormalised warped distribution; it matches the distribution
of HF and vLLM, not their torch RNG streams.

Parameters come from two surfaces:
  * HF `generate(do_sample=True, temperature=, top_k=, top_p=, seed=)` -> `from_hf`;
  * vLLM `SamplingParams` (per sequence group) -> `from_vllm`.

Log-probabilities (`ops.sample_logprobs`; `generate(logprobs=N)`, `Request.logprobs`, the vLLM adapter's
`sample_with_logprobs`).  For a row with parameters (T, top_k, top_p) the processed row is the bf16 logits as fp32
when T = 0 (greedy), and otherwise x = l / T over the kept set of the warp above and -inf outside it: the row the score
log holds and the token was chosen from.
  * logprob(r) = x_r - logsumexp(processed row), -inf outside the kept set: HF's
    `compute_transition_scores(sequences, scores, normalize_logits=True)` over this library's scores, and vLLM 0.5.5's
    Sampler (one log_softmax over the processed logits, for sampled and prompt rows alike);
  * rank(r) = 1 + #{tokens with a strictly greater processed value} (vLLM's `Logprob.rank`);
  * top-N (0 <= N <= 20, vLLM's default `max_logprobs`): the N tokens ordered by (logit descending, index ascending)
    with their logprobs; ids are compared on the bf16 logits, so they are exact;
  * the log-sum-exp is fp32 with Z = sum of the fixed-point masses exp(x - x_max) * 2^40 as u64 integers, like the
    top-p pass: independent of summation order and of batch position.
A row with a target token (vLLM prompt-logprob rows: the next prompt token) is scored with its parameters and nothing
is drawn.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch

# HF transformers 4.41 GenerationConfig defaults (what `None` means with do_sample=True)
HF_DEFAULT_TEMPERATURE, HF_DEFAULT_TOP_K, HF_DEFAULT_TOP_P = 1.0, 50, 1.0
# vLLM samples when temperature >= _SAMPLING_EPS (vllm/sampling_params.py); below it the request is greedy
VLLM_SAMPLING_EPS = 1e-5
U64 = (1 << 64) - 1
# most top-N entries a row can return (vLLM 0.5.5's default max_logprobs)
MAX_LOGPROBS = 20

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


@dataclass(frozen=True)
class TokenLogprobs:
    """Log-probability record of one token: its id, logprob and rank over the processed row, and the top-N as
    (id, logprob) pairs, highest logit first."""
    token: int
    logprob: float
    rank: int
    top: Tuple[Tuple[int, float], ...] = ()


def check_logprobs(n, name: str = "logprobs") -> Optional[int]:
    """A requested top-N count: None (no logprobs) or an int in [0, MAX_LOGPROBS]; anything else raises ValueError."""
    if n is None:
        return None
    if isinstance(n, bool) or not isinstance(n, int):
        raise ValueError(f"`{name}` must be an int in [0, {MAX_LOGPROBS}] or None, got {n!r}")
    if not 0 <= n <= MAX_LOGPROBS:
        raise ValueError(f"`{name}` must be in [0, {MAX_LOGPROBS}], got {n}")
    return n


def logprob_records(tokens, logprob, rank, top_ids, top_logprobs, n_top: int) -> List[TokenLogprobs]:
    """Host records from the kernel's outputs (row i of each array belongs to tokens[i]; n_top <= their width)."""
    lp, rk = logprob.tolist(), rank.tolist()
    ti, tl = top_ids[:, :n_top].tolist(), top_logprobs[:, :n_top].tolist()
    return [TokenLogprobs(int(t), lp[i], rk[i], tuple(zip(ti[i], tl[i]))) for i, t in enumerate(tokens)]


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


def from_vllm(sp, draws: bool = True) -> Optional[SamplingParams]:
    """vLLM SamplingParams -> SamplingParams, or None for greedy (temperature < 1e-5).  top_k -1 or 0 is off.
    Unseeded sampled rows get a fresh key from torch's default generator (call order = row order); with `draws` False
    (rows that are only scored, e.g. prompt-logprob rows) they get key 0 and the generator does not advance.  Features
    outside this sampler raise NotImplementedError."""
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
    key = (draw_key() if draws else 0) if seed is None else int(seed) & U64
    return SamplingParams(t, max(k, 0), float(g("top_p", 1.0)), key)


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
        self.stream = torch.zeros(max_batch, dtype=torch.int32, device=dev)  # stream index of the slot's sequence
        self.sampled: List[bool] = [False] * max_batch
        self.logprobs: List[Optional[int]] = [None] * max_batch     # top-N a slot's request asked for (None: none)

    @property
    def tensors(self):
        return [self.temperature, self.top_k, self.top_p, self.seed, self.stream]

    def set(self, slot: int, params: Optional[SamplingParams], logprobs: Optional[int] = None) -> None:
        """params None = greedy; `logprobs` = the request's top-N (None: no logprobs).  The slot draws from stream 0."""
        self.logprobs[slot] = check_logprobs(logprobs)
        p = params or SamplingParams(1.0)
        row = slice(slot, slot + 1)
        self.temperature[row] = p.temperature if params is not None else 0.0
        self.top_k[row] = p.top_k
        self.top_p[row] = p.top_p
        self.seed[row] = _i64(p.seed)
        self.stream[row] = 0
        self.sampled[slot] = params is not None

    def fork(self, src: int, count: int) -> None:
        """Slots src + 1 .. src + count - 1 take the parameters of slot src (stream 0) with streams 1 .. count - 1."""
        dst = slice(src + 1, src + count)
        for t in (self.temperature, self.top_k, self.top_p, self.seed):
            t[dst] = t[src].clone()
        self.stream[dst] = torch.arange(1, count, dtype=torch.int32, device=self.stream.device)
        for i in range(src + 1, src + count):
            self.sampled[i], self.logprobs[i] = self.sampled[src], self.logprobs[src]

    def swap(self, i: int, j: int) -> None:
        self.sampled[i], self.sampled[j] = self.sampled[j], self.sampled[i]
        self.logprobs[i], self.logprobs[j] = self.logprobs[j], self.logprobs[i]

    def any_sampled(self, n: int) -> bool:
        return any(self.sampled[:n])

    def log_width(self, s0: int, n: int) -> Optional[int]:
        """Top entries a step over slots [s0, s0 + n) records: None (no slot asks for logprobs), 0 (only logprob and
        rank: no slot asks for top entries) or MAX_LOGPROBS."""
        asked = [x for x in self.logprobs[s0:s0 + n] if x is not None]
        if not asked:
            return None
        return MAX_LOGPROBS if any(asked) else 0
