"""The sampling oracle (oracle/sampling_oracle.py) with the per-row stream index of parallel sampling: the noise of
token n of stream s is word (r & 3) of Philox4x32-10(counter (r >> 2, n, s, 0), key).  Stream 0 is the oracle's own
draw.  Test infrastructure only."""
from __future__ import annotations

import numpy as np

from oracle import sampling_oracle as SO


def gumbel(V: int, seed: int, n: int, stream: int = 0) -> np.ndarray:
    """g_r for r in [0, V) of the draw with key `seed`, counter `n` and stream index `stream` (fp64)."""
    r = np.arange(V, dtype=np.uint64)
    words = SO.philox4x32_10((r >> np.uint64(2), np.full(V, n, dtype=np.uint64), np.full(V, stream, dtype=np.uint64),
                              0), (seed & 0xFFFFFFFF, seed >> 32))
    w = np.choose((r & np.uint64(3)).astype(np.int64), words).astype(np.uint64)
    u = ((w >> np.uint64(8)).astype(np.float64) + 0.5) * 2.0 ** -24
    return -np.log(-np.log(u))


def choose(logits, temperature: float, top_k: int, top_p: float, seed: int, n: int, stream: int = 0):
    """SO.choose with a stream index: -> (token, gap between the best and second-best perturbed scores, top-p
    boundary distance)."""
    if temperature == 0 or stream == 0:
        return SO.choose(logits, temperature, top_k, top_p, seed, n)
    l = np.asarray(logits, dtype=np.float64)
    x, kept, dist = SO.warp(l, temperature, top_k, top_p)
    s = np.where(kept, x + gumbel(l.size, seed, n, stream), -np.inf)
    tok = int(np.argmax(s))
    rest = np.delete(s, tok)
    gap = float(s[tok] - rest.max()) if rest.size and np.isfinite(rest.max()) else np.inf
    return tok, gap, dist
