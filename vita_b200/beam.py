"""Beam search bookkeeping of `generate(num_beams=N)`: host code over each step's top candidates.

The rules are those of HF transformers 5.5.0 (`GenerationMixin._beam_search`, `_get_top_k_continuations`,
`_get_running_beams_for_next_iteration`, `_update_finished_beams`, `_check_early_stop_heuristic`,
`_beam_search_has_unfinished_sequences`) for one prompt, `do_sample=False` and one EOS id, restated per candidate:

  * a running beam b with score s_b proposes (b, t) with the fp32 score s_b + logprob(b, t); the 2N best proposals
    over all beams are the step's candidates, ordered by score descending, then beam ascending, then the order of the
    beam's row (logit descending, index ascending).  A beam's score is constant across its row, so each beam's own
    top 2N is enough;
  * a candidate "hits" when its token is the EOS id or it reaches max_new_tokens (HF's EosTokenCriteria and
    MaxLengthCriteria).  A hit ranked below N becomes a finished hypothesis scored fp32(s / n ** length_penalty), n =
    generated tokens including its last, unless the early-stop heuristic has closed or (early_stopping is True) N
    hypotheses are already finished; hits ranked N or lower are dropped.  The N best hypotheses are kept;
  * the first N candidates that are not EOS become the next running beams;
  * the heuristic closes when the best running score over the best hypothetical length (n, or max_new_tokens with
    early_stopping "never" and a positive penalty) no longer beats the worst of N finished hypotheses; the search ends
    when it has closed, when early_stopping is True and N hypotheses are finished, or when every candidate hit.

Ties between equal fp32 scores keep the earlier candidate (HF leaves their order to torch.topk).  Known differences
from transformers 4.41 (the version the reference pins): 4.41 takes the log-softmax of the bf16 logits in bf16, here
it is fp32; 4.41 finalizes the N running beams after the last step, 5.5.0 (and this module) finalizes the top N
candidates of the last step.  User stopping criteria are called once per step, the last one included, with the
running beams (at the last step: its first N candidates that are not EOS, 4.41's running beams then), and a true
result ends the search with the running beams added as hypotheses.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np

from .sampling import MAX_LOGPROBS

NEG = np.float32(-1e9)
MAX_BEAMS = MAX_LOGPROBS // 2      # each beam's candidates are its own top 2N, read from the top-20 logprob log


@dataclass
class Hypothesis:
    score: np.float32
    tokens: List[int]
    beam_indices: List[int]


@dataclass
class Beam:
    score: np.float32
    tokens: List[int] = field(default_factory=list)
    beam_indices: List[int] = field(default_factory=list)


def check_beam_args(num_beams, num_return_sequences, early_stopping) -> None:
    if isinstance(num_beams, bool) or not isinstance(num_beams, int) or num_beams < 1:
        raise ValueError(f"num_beams must be a positive int, got {num_beams!r}")
    if num_beams > MAX_BEAMS:
        raise ValueError(f"num_beams={num_beams} exceeds {MAX_BEAMS}: each beam's candidates are its top "
                         f"2 * num_beams tokens and the logprob log holds the top MAX_LOGPROBS = {MAX_LOGPROBS}")
    if not 1 <= num_return_sequences <= num_beams:
        raise ValueError(f"num_return_sequences must be in [1, num_beams = {num_beams}], got {num_return_sequences}")
    if early_stopping not in (True, False, "never"):
        raise ValueError(f"early_stopping must be True, False or 'never', got {early_stopping!r}")


class BeamSearch:
    """One search: `step(top_ids, top_logprobs)` per decoding step, `finalize()` for a stop from outside."""

    def __init__(self, num_beams: int, max_new_tokens: int, eos_token_id: Optional[int] = None,
                 length_penalty: float = 1.0, early_stopping: Union[bool, str] = False):
        self.N = num_beams
        self.max_new_tokens = max_new_tokens
        self.eos = eos_token_id
        self.length_penalty = float(length_penalty)
        self.early_stopping = early_stopping
        self.running: List[Beam] = [Beam(np.float32(0.0))]   # HF's start state: only beam 0 proposes at step 0
        self.finished: List[Hypothesis] = []                 # best first, at most N
        self.heuristic_open = True
        self.done = False

    def _penalized(self, score: np.float32, n: int) -> np.float32:
        return np.float32(score / np.float32(n ** self.length_penalty))

    def _full(self) -> bool:
        return len(self.finished) == self.N and self.early_stopping is True

    def _add(self, hyps: Sequence[Hypothesis]) -> None:
        """Keep the N best of the finished and `hyps` (stable: earlier ones first among equal scores)."""
        merged = self.finished + list(hyps)
        order = sorted(range(len(merged)), key=lambda i: (-float(merged[i].score), i))
        self.finished = [merged[i] for i in order[:self.N]]

    def step(self, top_ids: Sequence[Sequence[int]], top_logprobs: Sequence[Sequence[float]]) -> List[int]:
        """top_ids / top_logprobs [len(running), >= 2N]: each running beam's most likely tokens in row order with
        their fp32 logprobs.  Returns the parents (indices into the previous running beams) of the new running beams;
        empty when the search is done (`running` then keeps the step's last running beams)."""
        assert not self.done and len(top_ids) == len(self.running)
        N, K = self.N, 2 * self.N
        n = len(self.running[0].tokens) + 1                  # generated tokens of every candidate
        cands = []                                           # (score, beam, rank in row, token)
        for b, beam in enumerate(self.running):
            ids, lps = top_ids[b], np.asarray(top_logprobs[b], dtype=np.float32)
            assert len(ids) >= K, "each running beam needs its top 2 * num_beams tokens"
            for j in range(K):
                cands.append((np.float32(beam.score + lps[j]), b, j, int(ids[j])))
        cands.sort(key=lambda c: (-float(c[0]), c[1], c[2]))
        cands = cands[:K]
        at_max = n >= self.max_new_tokens
        hits = [at_max or c[3] == self.eos for c in cands]
        new = []
        if self.heuristic_open and not self._full():
            for (score, b, _, tok), hit in zip(cands[:N], hits[:N]):
                if hit:
                    parent = self.running[b]
                    new.append(Hypothesis(self._penalized(score, n), parent.tokens + [tok], parent.beam_indices + [b]))
        self._add(new)
        # the first N candidates that are not EOS; they run on unless every candidate hit (max_new_tokens), and then
        # remain as the last step's running beams (what stopping criteria see)
        survivors = [(c, i) for i, c in enumerate(cands) if c[3] != self.eos][:N]
        parents = [c[1] for c, _ in survivors]
        self.running = [Beam(score, self.running[b].tokens + [tok], self.running[b].beam_indices + [b])
                        for (score, b, _, tok), _ in survivors]
        if self.running:
            never = self.early_stopping == "never" and self.length_penalty > 0.0
            best = self._penalized(self.running[0].score, self.max_new_tokens if never else n)
            worst = self.finished[-1].score if len(self.finished) == N else NEG
            self.heuristic_open = self.heuristic_open and bool(best > worst)
        self.done = not self.heuristic_open or self._full() or all(hits)
        return [] if self.done else parents

    def finalize(self) -> None:
        """End the search now (a stopping criterion fired): the running beams become hypotheses."""
        if not self.done and self.running and self.heuristic_open and not self._full():
            n = len(self.running[0].tokens)
            self._add([Hypothesis(self._penalized(b.score, n), b.tokens, b.beam_indices) for b in self.running])
        self.running = []
        self.done = True

    def best(self, R: int) -> List[Hypothesis]:
        return self.finished[:R]


def pack_outputs(hyps: Sequence[Hypothesis], prompt: Sequence[int], pad: int) -> Tuple[np.ndarray, np.ndarray,
                                                                                          np.ndarray]:
    """HF's output layout: sequences [R, L + n] (prompt + tokens, padded with `pad`), sequences_scores [R] fp32,
    beam_indices [R, n] (padded with -1); n = the longest hypothesis."""
    n = max(len(h.tokens) for h in hyps)
    L = len(prompt)
    seq = np.full((len(hyps), L + n), pad, dtype=np.int64)
    idx = np.full((len(hyps), n), -1, dtype=np.int64)
    seq[:, :L] = np.asarray(prompt, dtype=np.int64)
    for r, h in enumerate(hyps):
        seq[r, L:L + len(h.tokens)] = h.tokens
        idx[r, :len(h.beam_indices)] = h.beam_indices
    return seq, np.array([h.score for h in hyps], dtype=np.float32), idx
