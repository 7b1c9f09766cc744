"""Inputs of the sampler tests (tests/test_sample_shapes_gpu.py), built on the CPU from seeded generators so that the
CPU checks of tests/test_sample_shapes.py see the same bits, plus the host side of the kernel's key map and of its
top-p tolerance.

Every row is bf16-exact (float32 arrays holding bf16 values).  The oracle gets what the kernel sees: T and p rounded
to fp32.  Families (V = 4096 unless stated; `V` is a parameter of every builder):

  topk      the k-th largest key at low byte 0x00 (0.5) and 0xFF (1.992) of its high bin, in the highest populated
            bin, on each side of the sign change (high bins 0x7F / 0x80: the smallest normal values of either sign),
            and a tie group of 5 that straddles k; k in {1, 2, 255, 256, 257, V-1, V, V+1} (V and V+1: off).  The key
            just below the threshold (in the same bin unless the threshold is at low byte 0x00) is always present.
  topp      a normal row shifted until the oracle's lowest kept key is a chosen key (0.5 / 1.992 / 4.0), for
            p in {0.5, 0.9, 0.999, 0.99999994} (the last is the largest fp32 below 1), with no token closer to the
            boundary than the tolerance; p in {0, 1e-6} keep the largest logit only.  Each placed row also runs with
            a top-k floor a few keys below the top-p threshold inside its high bin (the mass histogram's floor_key).
  zeros     -0.0 and +0.0 at the top-k threshold, at the top-p threshold and as the row maximum, in both orders of
            index.  The contract keeps or drops equal values together, so both signs are kept.
  masked    4000 of 4096 logits at -inf (a logits processor's mask) and 96 finite ones; top-k reaches the -inf group.
  prune     V = 51760: one maximum, every other token at x_max - d (d in {8, 12, 16}) and some at x_max - 24.5; the
            counter n is searched (SO.gumbel) until the oracle's winner is a sub-maximum token with a clear gap.
  division  logits at T_DIV whose bf16(fp32(l) / T) differs from bf16(fp32(l) * fp32(1 / T)): at the six temperatures
            above no bf16 logit tells the two apart, and about one fp32 temperature in 3000 has such logits.
  top-N     V = 51760: a tie group at the N-th largest value with members in 1024-wide chunks 0, 17 and 50 and at V-1
            (fewer than N in chunk 0), with and without -0.0 / +0.0 in the group; N in {1, 19, 20}.
Temperatures cycle through T_SAMPLED; T_GREEDY are the values that select the greedy path.
"""
from __future__ import annotations

import dataclasses
import functools

import numpy as np
import torch

from oracle import sampling_oracle as SO

BF16 = torch.bfloat16
T_SAMPLED = (1e-5, 0.05, 0.7, 1.0, 1.5, 100.0)     # 1e-5: the smallest temperature vLLM still samples with
T_GREEDY = (0.0, -1.0, -0.0)
P_PLACED = (0.5, 0.9, 0.999, 0.99999994)
KEY_FINITE = (0x0080, 0xFF7F)                     # keys of -max .. +max (0x007F is -inf, 0xFF80 is +inf)
CHUNK = 1024                                      # the sampler's block: the top-N tie loop takes one chunk per pass
DRAW_TOL = 1e-4                                   # perturbed-score gap a draw needs to be compared (fp32 x + g)


# ------------------------------------------------------------------------------------------------ the kernel's key map
def bf16_key(bits):
    """bf16 bit patterns -> 16-bit keys whose unsigned order is the numeric order (csrc/sample.cu: bf16_key)."""
    u = np.asarray(bits, dtype=np.uint32)
    return np.where(u & 0x8000, ~u & 0xFFFF, u | 0x8000).astype(np.uint32)


def canon_key(k):
    """-0.0's key (0x7FFF) read as +0.0's (0x8000): equal values, equal keys."""
    k = np.asarray(k, dtype=np.uint32)
    return np.where(k == 0x7FFF, 0x8000, k).astype(np.uint32)


def key_value(k) -> np.ndarray:
    """16-bit keys -> float32 values (bf16-exact)."""
    k = np.asarray(k, dtype=np.uint32)
    u = np.where(k & 0x8000, k & 0x7FFF, ~k & 0xFFFF).astype(np.uint32)
    return (u << 16).view(np.float32)


def keys_of(row) -> np.ndarray:
    return bf16_key(np.asarray(row, dtype=np.float32).view(np.uint32) >> 16)


def to_bf16(x) -> np.ndarray:
    """round to bf16 (RNE), returned as float32"""
    return torch.from_numpy(np.asarray(x, dtype=np.float32)).to(BF16).float().numpy()


def f32(v: float) -> float:
    return float(np.float32(v))


def pack_word(row, idx: int) -> int:
    """the packed (logit, ~index) word of csrc/sample.cu's pack_score, as the signed int64 torch holds"""
    u = int(np.asarray(row[idx], dtype=np.float32).view(np.uint32))
    if u == 0x80000000:
        u = 0
    u = (~u & 0xFFFFFFFF) if u & 0x80000000 else (u | 0x80000000)
    w = (u << 32) | (0xFFFFFFFF - idx)
    return w - (1 << 64) if w >= 1 << 63 else w


# ------------------------------------------------------------------------------------------------ oracle side
@dataclasses.dataclass
class Case:
    family: str
    name: str
    row: np.ndarray               # float32, bf16-exact, [V]
    T: float
    k: int
    p: float
    seed: int = 0
    n: int = 0                    # Philox counter
    meta: dict = dataclasses.field(default_factory=dict)

    @property
    def V(self) -> int:
        return self.row.size

    @property
    def greedy(self) -> bool:
        return not f32(self.T) > 0

    def warp(self):
        """SO.warp on the values the kernel sees: (x, kept, dist); greedy rows keep every token"""
        l = self.row.astype(np.float64)
        if self.greedy:
            return l.copy(), np.ones(self.V, dtype=bool), np.inf
        return SO.warp(l, f32(self.T), self.k, f32(self.p))


def survivors(row, k: int) -> np.ndarray:
    l = np.asarray(row, dtype=np.float64)
    if 0 < k < l.size:
        return l >= np.sort(l)[::-1][k - 1]
    return np.ones(l.size, dtype=bool)


def above_mass(row, T: float, k: int):
    """-> (above [V]: the softmax mass of the top-k survivors whose logit is strictly greater, as a fraction of their
    total, NaN outside the survivors; survivors [V] bool).  fp64, with T rounded to fp32."""
    l = np.asarray(row, dtype=np.float64)
    surv = survivors(l, k)
    x = l / f32(T)
    e = np.zeros(l.size)
    e[surv] = np.exp(x[surv] - x[surv].max())
    order = np.argsort(-l, kind="stable")
    sl = -l[order]                                            # ascending; -0.0 and +0.0 compare equal
    cs = np.concatenate([[0.0], np.cumsum(e[order])])
    first = np.searchsorted(sl, sl, side="left")             # first position of each value's group
    above = np.empty(l.size)
    above[order] = cs[first] / cs[-1]
    above[~surv] = np.nan
    return above, surv


def topp_tol(row, T: float, k: int, above) -> np.ndarray:
    """Per-token tolerance on |above - p| within which the kernel's fixed-point top-p may decide either way.

    The kernel sums u64 masses w_r = rint(expf(x_r - x_max) * 2^40).  Two errors separate its fraction A'/Z' from the
    fp64 one:
      - rounding each mass to an integer moves it by <= 1/2 while Z' >= 2^40 (the maximum alone weighs 2^40), so the
        fraction moves by at most V * 2^-41;
      - x = fp32(l / T), x - x_max in fp32 and expf (2 ulp) give every mass a relative error
        delta <= 2^-22 * (1 + max |x|); a common relative error cancels in A / Z, and the rest moves the fraction
        f = A / Z by at most 2 * delta * f * (1 - f) (d(A / (A + C)) = f (1 - f) (dA / A - dC / C)).
    Tokens whose mass rounds to 0 (x < x_max - 28.4) add nothing to any bin or to Z: the mass above them is the
    whole of Z, which is >= p * Z for every p < 1, so they are dropped; the oracle gives them less than 2^-41 of Z
    each, inside the first term.  p * Z is formed in fp64 from fp32 p (the oracle gets the same p)."""
    surv = np.isfinite(above)
    x = np.asarray(row, dtype=np.float64)[surv] / f32(T)
    delta = 2.0 ** -22 * (1.0 + np.abs(x[np.isfinite(x)]).max())
    a = np.where(surv, above, 0.0)
    return np.asarray(row).size * 2.0 ** -41 + 2.0 * delta * a * (1.0 - a)


def topp_exempt(case: Case) -> np.ndarray:
    """tokens whose top-p decision the kernel may take either way (|above - p| < tol); none when top-p is off"""
    if case.greedy or not 0.0 < f32(case.p) < 1.0:              # p = 0 keeps the largest logit, whatever the masses
        return np.zeros(case.V, dtype=bool)
    above, surv = above_mass(case.row, case.T, case.k)
    tol = topp_tol(case.row, case.T, case.k, above)
    return surv & (np.abs(np.where(surv, above, 0.0) - f32(case.p)) < tol)


def expected_scores(case: Case, kept) -> torch.Tensor:
    """the plain variant's score log row: the logits for greedy rows, else bf16(fp32(l) / fp32(T)) on the kept set
    and -inf outside it (torch CPU fp32 division and the bf16 conversion both round to nearest even)"""
    l = torch.from_numpy(case.row.astype(np.float32))
    if case.greedy:
        return l.to(BF16)
    x = (l / torch.tensor(f32(case.T), dtype=torch.float32)).to(BF16)
    return torch.where(torch.from_numpy(np.asarray(kept)), x, torch.tensor(float("-inf"), dtype=BF16))


def draw(case: Case, kept):
    """the oracle's draw over `kept`: (token, gap to the second perturbed score); greedy: first arg-max, inf"""
    l = case.row.astype(np.float64)
    if case.greedy:
        return int(np.argmax(l)), np.inf
    x = l / f32(case.T)
    s = np.where(kept, x + SO.gumbel(case.V, case.seed, case.n), -np.inf)
    tok = int(np.argmax(s))
    rest = np.delete(s, tok)
    gap = float(s[tok] - rest.max()) if rest.size and np.isfinite(rest.max()) else np.inf
    return tok, gap


def draw_tol(case: Case) -> float:
    """fp32 rounding of x + g at |x| = |l| / T (the rule of test_sampling_gpu)"""
    fin = np.isfinite(case.row)
    return max(DRAW_TOL, 4e-7 * float(np.abs(case.row[fin]).max()) / f32(case.T))


# ------------------------------------------------------------------------------------------------ builders
def _clip_keys(k):
    return np.clip(k, *KEY_FINITE).astype(np.uint32)


TOPK_PLACES = {                                   # name -> threshold key, largest key above it
    "lo00": (0xBF00, 0xBF00 + 600),               # 0.5: the key below is 0xBEFF, in the next bin down
    "loFF": (0xBFFF, 0xBFFF + 600),               # 1.992: the low pass ends at its last bin
    "topbin": (0xC040, 0xC0FF),                   # the threshold's high bin is the highest populated one
    "neg7F": (0x7F10, 0x7F10 + 400),              # -2.2e-38 (normal): the keys above cross -0 / +0
    "pos80": (0x80F0, 0x80F0 + 400),              # +2.2e-38 (normal): the keys below cross +0 / -0
}


def topk_k_values(V: int):
    return (1, 2, 255, 256, 257, V - 1, V, V + 1)


def topk_row(V: int, k: int, place: str, tie: int, seed: int) -> np.ndarray:
    """keys: `tie` tokens at the threshold, enough above it that the k-th largest is at the threshold (the tie group
    straddles k when tie > 1 and k allows), the key just below the threshold, the rest below; shuffled"""
    thr, top = TOPK_PLACES[place]
    rng = np.random.default_rng(seed)
    kk = min(k, V - 1)
    n_above = max(0, kk - 1 - tie // 2)
    tie = max(1, min(tie, V - n_above - 1))              # keep one token below the threshold
    above = rng.integers(thr + 1, top + 1, n_above)
    n_below = V - n_above - tie
    below = rng.integers(max(KEY_FINITE[0], thr - 700), thr, n_below)
    if n_below:
        below[0] = thr - 1
    keys = np.concatenate([above, np.full(tie, thr), below])
    return key_value(_clip_keys(rng.permutation(keys)))


def topk_cases(V: int = 4096):
    out = []
    for pi, place in enumerate(TOPK_PLACES):
        for tie in (1, 5):
            for ki, k in enumerate(topk_k_values(V)):
                # the placements across the sign change run at T = 1, where x keeps the logit's bits
                T = 1.0 if place in ("neg7F", "pos80") else T_SAMPLED[(pi + ki + tie) % len(T_SAMPLED)]
                row = topk_row(V, k, place, tie, 1000 + 97 * pi + 13 * ki + tie)
                out.append(Case("topk", f"{place}-tie{tie}-k{k}", row, T, k, 1.0, seed=7 + ki, n=pi,
                                meta=dict(thr_key=TOPK_PLACES[place][0], tie=tie)))
    return out


def _lowest_kept_key(row, T, k, p) -> int:
    _, kept, _ = SO.warp(row.astype(np.float64), f32(T), k, f32(p))
    return int(canon_key(keys_of(row[kept])).min())


TOPP_TARGETS = (0xBF00, 0xBFFF, 0xC080)           # 0.5, 1.992, 4.0


def topp_row(V: int, T: float, p: float, target: int, seed: int, k: int = 0):
    """a normal row shifted until the oracle's lowest kept key is `target` and no token is within the tolerance of
    the boundary; None if no seed of a few works"""
    for attempt in range(8):
        rng = np.random.default_rng(seed + 7919 * attempt)
        row = to_bf16(rng.normal(0.0, 1.5, V))
        for _ in range(8):
            got = _lowest_kept_key(row, T, k, p)
            if got == target:
                break
            row = to_bf16(row + (key_value(target) - key_value(got)))
        if _lowest_kept_key(row, T, k, p) != target:
            continue
        c = Case("topp", "", row, T, k, p)
        if not topp_exempt(c).any():
            return row
    return None


def topp_cases(V: int = 4096):
    out = []
    i = 0
    for p in P_PLACED:
        for target in TOPP_TARGETS:
            T = (0.7, 1.0, 1.5)[i % 3]
            row = topp_row(V, T, p, target, 5000 + i)
            i += 1
            if row is None:
                continue
            out.append(Case("topp", f"p{p}-key{target:04X}", row, T, 0, p, seed=31 + i, n=i,
                            meta=dict(thr_key=target)))
            # a top-k floor a few keys below the top-p threshold, inside its high bin
            keys = canon_key(keys_of(row))
            floor = next((f for f in range(target - 1, (target & 0xFF00) - 1, -1)
                          if (keys == f).any() and f >= (target & 0xFF00)), None)
            if floor is not None:
                k = int((keys >= floor).sum())
                c = Case("topp", f"p{p}-key{target:04X}-k{k}", row, T, k, p, seed=41 + i, n=i,
                         meta=dict(floor_key=floor))
                if not topp_exempt(c).any():
                    out.append(c)
    for p in (0.0, 1e-6):
        for j, T in enumerate((1e-5, 0.05, 100.0)):
            row = to_bf16(np.random.default_rng(6000 + j).normal(0, 2, V))
            out.append(Case("topp", f"p{p}-T{T}", row, T, 0, p, seed=51 + j, n=j))
            out.append(Case("topp", f"p{p}-T{T}-k50", row, T, 50, p, seed=61 + j, n=j))
    return out


def zeros_cases(V: int = 4096):
    """-0.0 and +0.0 as one tie group at the top-k threshold, at the top-p threshold and as the maximum"""
    out = []
    for order in ("neg-first", "pos-first"):
        rng = np.random.default_rng(7000 + len(order))
        n_pos, n_z = 100, 12
        zeros = np.concatenate([np.full(n_z // 2, -0.0), np.full(n_z // 2, 0.0)]).astype(np.float32)
        if order == "pos-first":
            zeros = zeros[::-1].copy()
        pos = to_bf16(rng.uniform(0.5, 3.0, n_pos))
        neg = to_bf16(-rng.uniform(0.5, 6.0, V - n_pos - n_z))
        # zeros at indices n_pos .. n_pos + n_z - 1 in the chosen order; the rest shuffled around them
        rest = rng.permutation(np.concatenate([pos, neg]))
        row = np.concatenate([rest[:n_pos], zeros, rest[n_pos:]]).astype(np.float32)
        # top-k: the k-th largest is zero (its first, a middle and its last member)
        for k in (n_pos + 1, n_pos + n_z // 2, n_pos + n_z):
            out.append(Case("zeros", f"topk-{order}-k{k}", row, 0.7, k, 1.0, seed=3, n=k))
        # top-p: the mass above zero is below p, the mass above zero plus the +0.0 tokens is not.  The kernel's high
        # pass puts +0.0 in bin 0x80 and -0.0 in bin 0x7F: a threshold over raw keys keeps one sign only
        # ("split": p * Z at the mass above zero plus 3 of the 6 +0.0 tokens; "inside": plus 11.5 of the 12 zeros, so
        # that a top-p that is not tie-aware, HF's, keeps the whole group too)
        zi = np.flatnonzero(row == 0)
        for k in (0, n_pos + n_z):
            above, surv = above_mass(row, 1.0, k)
            a0 = float(above[zi[0]])
            u = float(np.exp(-row.astype(np.float64).max()) / np.exp(row[surv].astype(np.float64) - row.max()).sum())
            for zs, tag in ((3.0, "split"), (n_z - 0.5, "inside")):
                out.append(Case("zeros", f"topp-{tag}-{order}-k{k}", row, 1.0, k, f32(a0 + zs * u), seed=5 + k,
                                n=int(zs)))
        # zero as the maximum, both signs present
        mrow = np.where(row > 0, -row, row).astype(np.float32)
        for k, p in ((0, 0.0), (1, 1.0), (0, 0.5), (3, 0.9)):
            out.append(Case("zeros", f"max-{order}-k{k}-p{p}", mrow, 1.0, k, p, seed=8, n=k))
    return out


def masked_cases(V: int = 4096):
    rng = np.random.default_rng(8000)
    out = []
    row = np.full(V, -np.inf, dtype=np.float32)
    live = rng.choice(V, 96, replace=False)
    live[0] = V - 1
    row[live] = to_bf16(rng.normal(0, 2, 96))
    for j, (k, p) in enumerate(((50, 1.0), (96, 1.0), (97, 1.0), (200, 1.0), (V - 1, 1.0), (0, 0.9), (200, 0.9),
                                (0, 0.0))):
        out.append(Case("masked", f"k{k}-p{p}", row, (0.7, 1.0, 1.5)[j % 3], k, p, seed=9, n=j))
    return out


PRUNE_D = (8.0, 12.0, 16.0)
PRUNE_V = 51760


@functools.lru_cache(maxsize=None)
def _prune_search(d: float, V: int, seed: int):
    """the first counter n whose oracle winner is a sub-maximum token with a gap above the draw tolerance"""
    row = prune_row(d, V)
    x = row.astype(np.float64)
    for n in range(20000):
        s = x + SO.gumbel(V, seed, n)
        tok = int(np.argmax(s))
        if tok != 0:
            rest = np.delete(s, tok)
            if s[tok] - rest.max() > 4 * DRAW_TOL:
                return n
    raise AssertionError(f"no qualifying draw for d = {d}")


def prune_row(d: float, V: int = PRUNE_V) -> np.ndarray:
    """T = 1: token 0 at x_max = 4, the others at 4 - d, every 97th at 4 - 24.5 (below the prune floor)"""
    row = np.full(V, 4.0 - d, dtype=np.float32)
    row[0] = 4.0
    row[1::97] = 4.0 - 24.5
    return row


def prune_cases(V: int = PRUNE_V):
    out = []
    for d in PRUNE_D:
        seed = 0x9E3779B97F4A7C15 ^ int(d)
        n = _prune_search(d, V, seed)
        out.append(Case("prune", f"d{d:g}", prune_row(d, V), 1.0, 0, 1.0, seed=seed, n=n, meta=dict(d=d)))
    return out


TIE_CHUNKS = (0, 17, 50)


def topn_tie_row(V: int, N: int, zeros: bool, seed: int):
    """-> (row, tie indices): N - 6 tokens above the tie value (or none when N < 7), a tie group of 12 with 3 members
    in each of chunks 0, 17 and 50 plus index V - 1, the rest below"""
    rng = np.random.default_rng(seed)
    tv = 0.0 if zeros else 1.5
    row = to_bf16(rng.uniform(tv - 6.0, tv - 0.5, V))
    ties = []
    for c in TIE_CHUNKS:
        lo = c * CHUNK
        ties += [int(i) for i in rng.choice(np.arange(lo, min(lo + CHUNK, V - 1)), 3, replace=False)]
    ties.append(V - 1)
    ties = np.array(sorted(ties))
    vals = np.full(ties.size, tv, dtype=np.float32)
    if zeros:
        vals[::2] = -0.0
    row[ties] = vals
    n_above = max(0, N - 6) if N > 1 else 0
    free = np.setdiff1d(np.arange(V), ties)
    row[rng.choice(free, n_above, replace=False)] = to_bf16(rng.uniform(tv + 0.5, tv + 3.0, n_above))
    return row, ties


def topn_cases(V: int = PRUNE_V):
    """(case, N, tie indices) for the LOGPROBS variant"""
    out = []
    for zeros in (False, True):
        for N in (1, 19, 20):
            row, ties = topn_tie_row(V, N, zeros, 9000 + N + 100 * zeros)
            for j, (T, k, p) in enumerate(((0.0, 0, 1.0), (0.7, 0, 1.0), (1.0, 20, 0.9))):
                c = Case("topn", f"N{N}-{'zeros' if zeros else 'ties'}-T{T}", row, T, k, p, seed=11 + j, n=N,
                         meta=dict(N=N, ties=ties))
                out.append(c)
    return out


T_DIV = 0.45542171597480774                       # fp32; 26 logits in (0.01, 64) round differently there


def division_sensitive(T: float) -> np.ndarray:
    """the bf16 values l with 0.01 < |l| < 64 for which bf16(fp32(l) / T) != bf16(fp32(l) * fp32(1 / T))"""
    bits = np.arange(1 << 16, dtype=np.uint32)
    v = (bits << 16).view(np.float32)
    v = v[np.isfinite(v) & (np.abs(v) > 0.01) & (np.abs(v) < 64)]
    t = np.float32(T)
    a = torch.from_numpy(v / t).to(BF16).view(torch.int16)
    b = torch.from_numpy(v * (np.float32(1) / t)).to(BF16).view(torch.int16)
    return v[(a != b).numpy()]


def division_cases(V: int = 4096):
    rng = np.random.default_rng(8500)
    row = to_bf16(rng.normal(0, 2, V))
    sens = division_sensitive(T_DIV)
    at = rng.choice(V, min(V, 8 * sens.size), replace=False)
    row[at] = np.resize(sens, at.size)
    return [Case("division", f"T{T_DIV:.6f}-k{k}", row, T_DIV, k, 1.0, seed=71 + k, n=1, meta=dict(sensitive=sens))
            for k in (0, V // 2)]


def all_cases(V: int = 4096):
    return topk_cases(V) + topp_cases(V) + zeros_cases(V) + masked_cases(V) + division_cases(V)


def stack(cases) -> torch.Tensor:
    return torch.from_numpy(np.stack([c.row for c in cases])).to(BF16)
