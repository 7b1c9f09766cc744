"""fp64 numpy restatement of the logprob contract (vita_b200/sampling.py, the LOGPROBS variant of
vita_b200/csrc/sample.cu), on top of oracle/sampling_oracle.warp.

  processed row:  T = 0: the logits; otherwise x = l / T over the kept set of the warp, -inf outside it
  logprob(r) = x_r - logsumexp(processed row);  rank(r) = 1 + #{processed values strictly greater than r's}
  top-N: the N tokens ordered by (logit descending, index ascending)

Test infrastructure only: the product never imports it.
"""
from __future__ import annotations

import numpy as np

from oracle import sampling_oracle as SO


def processed(logits, temperature: float, top_k: int, top_p: float):
    """-> (x [V] fp64, kept [V] bool, top-p boundary distance as in sampling_oracle.warp)."""
    l = np.asarray(logits, dtype=np.float64)
    if temperature == 0:
        return l.copy(), np.ones(l.size, dtype=bool), np.inf
    return SO.warp(l, temperature, top_k, top_p)


def logprobs(logits, temperature: float, top_k: int, top_p: float, n_top: int, target: int):
    """-> dict(logprob, rank of `target`; top_ids, top_logprobs [n_top]; row: every token's logprob; kept; dist)."""
    l = np.asarray(logits, dtype=np.float64)
    x, kept, dist = processed(l, temperature, top_k, top_p)
    xs = x[kept]
    m = xs.max()
    lse = m + np.log(np.exp(xs - m).sum())
    row = np.where(kept, x - lse, -np.inf)
    proc = np.where(kept, x, -np.inf)
    rank = 1 + int(np.count_nonzero(proc > proc[target]))
    order = np.lexsort((np.arange(l.size), -l))[:n_top]         # logit descending, index ascending
    return dict(logprob=float(row[target]), rank=rank, top_ids=order.astype(np.int64), top_logprobs=row[order],
                row=row, kept=kept, dist=dist)
