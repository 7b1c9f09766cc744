"""fp64 numpy restatement of the sampling contract (vita_b200/sampling.py, vita_b200/csrc/sample.cu).

  warp:   x = l / T; top-k keeps l >= the k-th largest l; top-p keeps a top-k survivor r iff the softmax mass of the
          survivors with l > l_r is < top_p (the largest logit always stays)
  noise:  u_r = ((w >> 8) + 0.5) * 2^-24, w = word (r & 3) of Philox4x32-10(counter (r >> 2, n, 0, 0),
          key (seed & 0xffffffff, seed >> 32)); g_r = -log(-log(u_r))
  draw:   argmax over the kept set of x_r + g_r, lowest index on ties

Test infrastructure only: the product never imports it.
"""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: 4 arrays (or ints) of uint32 words, key: 2 ints.  Returns the 4 output words as uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & MASK32 for x in ctr]
    c = np.broadcast_arrays(*c)
    c = [x.copy() for x in c]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
        p0, p1 = M0 * c[0], M1 * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & MASK32
        hi1, lo1 = p1 >> np.uint64(32), p1 & MASK32
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
    return [x.astype(np.uint32) for x in c]


def gumbel(V: int, seed: int, n: int) -> np.ndarray:
    """g_r for r in [0, V) of the draw with key `seed` and counter `n` (fp64)."""
    r = np.arange(V, dtype=np.uint64)
    words = philox4x32_10((r >> np.uint64(2), np.full(V, n, dtype=np.uint64), 0, 0), (seed & 0xFFFFFFFF, seed >> 32))
    w = np.choose((r & np.uint64(3)).astype(np.int64), words).astype(np.uint64)
    u = ((w >> np.uint64(8)).astype(np.float64) + 0.5) * 2.0 ** -24
    return -np.log(-np.log(u))


def warp(logits, temperature: float, top_k: int, top_p: float):
    """-> (x [V] fp64, kept [V] bool, boundary distance: the smallest |mass above r - top_p| over the top-k
    survivors (inf when top-p is off); a token that close to the boundary may fall either way in fp32)."""
    l = np.asarray(logits, dtype=np.float64)
    V = l.shape[0]
    x = l / float(temperature)
    kept = np.ones(V, dtype=bool)
    if 0 < top_k < V:
        kth = np.sort(l)[::-1][top_k - 1]
        kept = l >= kth
    dist = np.inf
    if top_p < 1.0:
        xs = x[kept]
        e = np.exp(xs - xs.max())
        prob = e / e.sum()
        vals = l[kept]
        order = np.argsort(-vals, kind="stable")
        sv, sp = vals[order], prob[order]
        # mass strictly above each distinct value
        uniq, first = np.unique(-sv, return_index=True)        # ascending -v = descending v
        csum = np.concatenate([[0.0], np.cumsum(sp)])
        above_u = csum[first]                                   # mass of the entries before the first of each value
        above = np.empty_like(vals)
        idx = np.searchsorted(uniq, -vals)
        above[:] = above_u[idx]
        keep_p = above < top_p
        if not keep_p.any():
            keep_p = vals == vals.max()
        dist = float(np.min(np.abs(above - top_p)))
        k2 = kept.copy()
        k2[np.flatnonzero(kept)] = keep_p
        kept = k2
    return x, kept, dist


def probs(logits, temperature: float, top_k: int, top_p: float) -> np.ndarray:
    """Renormalised warped distribution (what a draw samples from)."""
    x, kept, _ = warp(logits, temperature, top_k, top_p)
    p = np.zeros_like(x)
    e = np.exp(x[kept] - x[kept].max())
    p[kept] = e / e.sum()
    return p


def choose(logits, temperature: float, top_k: int, top_p: float, seed: int, n: int):
    """-> (token, gap between the best and second-best perturbed scores, top-p boundary distance).
    temperature 0 = greedy (first index of the largest logit; gap = top-1 minus top-2 logit)."""
    l = np.asarray(logits, dtype=np.float64)
    if temperature == 0:
        order = np.argsort(-l, kind="stable")
        gap = l[order[0]] - l[order[1]] if l.size > 1 else np.inf
        return int(order[0]), float(gap), np.inf
    x, kept, dist = warp(l, temperature, top_k, top_p)
    s = np.where(kept, x + gumbel(l.size, seed, n), -np.inf)
    tok = int(np.argmax(s))
    rest = np.delete(s, tok)
    gap = float(s[tok] - rest.max()) if rest.size and np.isfinite(rest.max()) else np.inf
    return tok, gap, dist
