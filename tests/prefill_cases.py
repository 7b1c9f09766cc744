"""Inputs of the prefill FlashAttention tests (tests/test_prefill_shapes_gpu.py) and a host model of the kernel's lazy
softmax rescale, which tests/test_prefill_shapes.py uses to prove that the late-jump inputs reach it.

flash_tc.cu walks a row's keys in tiles of 128 and keeps a reference max m_ref in log2 units (s * scale * log2 e).  A
tile whose largest score m exceeds m_ref + 8 moves the reference and multiplies the row sum and, past the first tile,
the O accumulator by 2^(m_ref - m); a smaller rise is absorbed: probabilities up to 2^8 are summed as they are.

Three input regimes, built on the CPU from seeded generators so that both test files see the same bits:
  randn  q, k, v ~ N(0, 1): q.k.D^-0.5 has a standard deviation of about 1, every softmax is nearly flat and a row's
         max after its first tile never rises by 8 again;
  sharp  the same with q scaled by 4;
  late   randn with planted keys.  The last 8 dimensions of q and k become spike channels (zero everywhere else).  Per KV
         head, a key gets a spike value in one channel and chosen query rows of its group (all query heads) a channel
         weight such that their score at that key is m_ref + delta, where m_ref is the reference the kernel holds
         before that key's tile (the model below) and delta in DELTAS is chosen per KV head.  7.9 stays under the
         threshold (P = 2^7.9 ~ 239 enters the sum unscaled), 8.1 just crosses it.  Placements: the first key of tile
         1, a key in a middle tile, the last key of a row's causal window (two rows, one channel each), a key of the
         last, partial tile, and a staircase of three jumps, each above 8, in tiles 1, 2 and 3.
"""
import math

import torch

BF16 = torch.bfloat16
LOG2E = 1.4426950408889634
TILE = 128
THRESH = 8.0
DELTAS = (7.9, 8.1, 20.0, 60.0)
STAIRS = (8.1, 20.0, 60.0)   # ascending: the small step's channel weight is the small one (bf16 rounding of q)
SPIKE = 4.0                  # the spike key's value in its channel
N_CH = 8

REGIMES = ("randn", "sharp", "late")

# shapes of the serving path
MIXTRAL_S = (1, 2, 127, 128, 129, 255, 256, 257, 1000, 4096, 4600)
NQ, NKV, D = 32, 8, 128
QKV_W = (NQ + 2 * NKV) * D
VIT_CASES = ((1, 1025), (13, 1025), (1, 65))
VIT_H, VIT_NH, VIT_D = 1024, 16, 64
WHALE_T2 = (70, 248)
WHALE_B, WHALE_NH, WHALE_DK = 6, 16, 64
PAGED_CASES = [(p, c) for p in (0, 100, 1000, 4000) for c in (1, 129, 500)]


def token_ranges(S=4600, worlds=(2, 4, 8)):
    """distinct (t0, t1) of parallel.token_range with t0 > 0 (t0 = 0 is the plain causal prompt)"""
    from vita_b200 import parallel
    out = []
    for w in worlds:
        for r in range(w):
            t0, t1 = parallel.token_range(S, r, w)
            if 0 < t0 < t1 and (t0, t1) not in out:
                out.append((t0, t1))
    return out


def whale_lengths(T2):
    return [0, 1, 127, 128, 129, T2]


def randn(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(BF16)


# ------------------------------------------------------------------------------------------------ kernel model
def row_limit(r, causal, q_pos0, kv_len):
    """keys [0, limit) of query row r"""
    return min(kv_len, q_pos0 + r + 1) if causal else kv_len


def rescale_tiles(s_log2, lim):
    """The kernel's decision for one row: s_log2 [>= lim] fp64 scores in log2 units, keys >= lim masked.  Returns the
    tiles at which the reference moves and the reference held before each tile."""
    m = -math.inf
    moved, before = [], []
    for j in range((lim + TILE - 1) // TILE):
        before.append(m)
        mx = float(s_log2[j * TILE:min((j + 1) * TILE, lim)].max())
        m_new = max(m, mx)
        if m_new > m + THRESH:
            moved.append(j)
            m = m_new
    return moved, before


def row_scores(q, k64, r, h, sl2, lim):
    """fp64 log2-unit scores of query row r, head h over keys [0, lim): q [Sq, Hq, D], k64 [Skv, D] fp64 keys of h's
    KV head"""
    return (k64[:lim] @ q[r, h].double()) * sl2


# ------------------------------------------------------------------------------------------------ late jumps
def _placements(Sq, causal, q_pos0, kv_len):
    """(name, [keys], [deltas or None = the head's delta], channel per key, rows) of one KV head"""
    nt = (kv_len + TILE - 1) // TILE
    lim = [row_limit(r, causal, q_pos0, kv_len) for r in range(Sq)]
    sees = lambda t: [r for r in range(Sq) if lim[r] > t]
    out = []
    if nt >= 2:
        out.append(("tile 1, first key", [TILE], [None], [0], sees(TILE)))
    if nt >= 3:
        t = TILE * (nt // 2) + 37
        out.append(("middle tile", [t], [None], [1], sees(t)))
    for ch in (2, 3):                     # the last key of a row's window, one row per channel
        if causal:
            rows = [r for r in range(Sq) if lim[r] - 1 >= TILE]
            out.append(("window's last key", None, [None], [ch], rows))
        elif nt >= 2 and ch == 2:
            out.append(("last valid key", [kv_len - 1], [None], [ch], sees(kv_len - 1)))
    if nt >= 2 and kv_len % TILE:
        t = TILE * (nt - 1) + (kv_len - 1 - TILE * (nt - 1)) // 2
        out.append(("last, partial tile", [t], [None], [4], sees(t)))
    if nt >= 4:
        ts = [TILE + 5, 2 * TILE + 9, 3 * TILE + 13]
        out.append(("staircase", ts, list(STAIRS), [5, 6, 7], sees(ts[-1])))
    return out


def plant_late_jumps(q, k, *, group, scale, causal, q_pos0, kv_len):
    """The late-jump regime on one batch entry, in place: q [Sq, Hq, D], k [Skv, Hkv, D] bf16 (views are written
    through).  Returns the targets (kv head, query head, row, key, delta, placement)."""
    Sq, Hq, Dqk = q.shape
    c0 = Dqk - N_CH
    q[..., c0:] = 0
    k[..., c0:] = 0
    sl2 = scale * LOG2E
    targets = []
    if kv_len <= TILE:
        return targets
    plan = _placements(Sq, causal, q_pos0, kv_len)
    for g in range(k.shape[1]):
        delta = DELTAS[g % len(DELTAS)]
        k64 = k[:, g].double()
        used = set()
        for name, keys, deltas, chans, rows in plan:
            free = [r for r in rows if r not in used]
            if not free:
                continue
            pick = [free[-1]] if keys is None else sorted({free[-1], free[len(free) // 2]})
            for r in pick:
                used.add(r)
                ks = [row_limit(r, causal, q_pos0, kv_len) - 1] if keys is None else keys
                ds = [delta] if deltas[0] is None else deltas
                for t, d, ch in zip(ks, ds, chans):
                    k[t, g, c0 + ch] = k64[t, c0 + ch] = SPIKE
                    lim = row_limit(r, causal, q_pos0, kv_len)
                    for h in range(g * group, (g + 1) * group):
                        q[r, h, c0 + ch] = 0
                        s = row_scores(q, k64, r, h, sl2, lim)
                        _, before = rescale_tiles(s, lim)
                        need = (before[t // TILE] + d) / sl2          # raw score at key t
                        q[r, h, c0 + ch] = (need - float(s[t]) / sl2) / SPIKE
                        targets.append((g, h, r, t, d, name))
    return targets


def check_targets(q, k, targets, *, group, scale, causal, q_pos0, kv_len):
    """Runs the model on the built inputs.  Returns (problems, number of rescales past the first tile at the targets):
    a target with delta > 8 must move the reference at its key's tile, one with delta < 8 must not, and its planted
    key must be the largest of its tile and rise by delta within the bf16 rounding of q."""
    sl2 = scale * LOG2E
    bad, late, k64 = [], 0, {}
    for g, h, r, t, d, name in targets:
        lim = row_limit(r, causal, q_pos0, kv_len)
        if g not in k64:
            k64[g] = k[:, g].double()
        s = row_scores(q, k64[g], r, h, sl2, lim)
        moved, before = rescale_tiles(s, lim)
        j = t // TILE
        tile = s[j * TILE:min((j + 1) * TILE, lim)]
        rise = float(s[t]) - before[j]
        what = f"{name}: kv head {g}, head {h}, row {r}, key {t}, delta {d}"
        if float(tile.max()) != float(s[t]):
            bad.append(f"{what}: the planted key is not its tile's max")
        if abs(rise - d) > (0.09 if d < 10 else 0.02 * d):      # bf16 rounding of the channel weight
            bad.append(f"{what}: rises by {rise:.3f}")
        if (d > THRESH) != (j in moved):
            bad.append(f"{what}: rescale at tile {j} is {j in moved}")
        late += j in moved and j > 0
    return bad, late


# ------------------------------------------------------------------------------------------------ cases
def _regime(q, k, regime, **kw):
    if regime == "sharp":
        q.mul_(4)
        return []
    if regime == "late":
        return plant_late_jumps(q, k, **kw)
    return []


def mixtral_case(S, regime, seed=0):
    """packed qkv [S, (32 + 16) * 128] as the qkv GEMM writes it; q / k / v are views of it"""
    qkv = randn((S, QKV_W), 1000 + S + seed)
    q, k = qkv[:, :NQ * D].view(S, NQ, D), qkv[:, NQ * D:(NQ + NKV) * D].view(S, NKV, D)
    kw = dict(group=NQ // NKV, scale=D ** -0.5, causal=True, q_pos0=0, kv_len=S)
    return qkv, _regime(q, k, regime, **kw), kw


def sharded_case(t0, t1, regime, seed=0):
    """a sequence shard: q rows [t0, t1) in a packed qkv buffer, K / V [t1, 8, 128] in the cache layout"""
    Sq = t1 - t0
    qkv = randn((Sq, QKV_W), 2000 + t0 + seed)
    kc = randn((t1, NKV, D), 3000 + t0 + seed)
    vc = randn((t1, NKV, D), 4000 + t0 + seed)
    kw = dict(group=NQ // NKV, scale=D ** -0.5, causal=True, q_pos0=t0, kv_len=t1)
    return (qkv, kc, vc), _regime(qkv[:, :NQ * D].view(Sq, NQ, D), kc, regime, **kw), kw


def vit_case(B, S, regime, seed=0):
    """packed qkv [B, S, 3 * 1024]"""
    qkv = randn((B, S, 3 * VIT_H), 5000 + B + S + seed)
    kw = dict(group=1, scale=VIT_D ** -0.5, causal=False, q_pos0=0, kv_len=S)
    targets = []
    for b in range(B):
        q = qkv[b, :, :VIT_H].view(S, VIT_NH, VIT_D)
        k = qkv[b, :, VIT_H:2 * VIT_H].view(S, VIT_NH, VIT_D)
        targets.append(_regime(q, k, regime, **kw))
    return qkv, targets, kw


def whale_case(T2, regime, seed=0):
    """q2 = [q + u | q + v] and k2 = [k | p] [B, T2, 16, 128], qkv [B, T2, 3 * 1024] (v heads in the last third).
    K and V rows past each length hold +-2^60."""
    B, C = WHALE_B, WHALE_NH * WHALE_DK
    q2 = randn((B, T2, WHALE_NH, 2 * WHALE_DK), 6000 + T2 + seed)
    k2 = randn((B, T2, WHALE_NH, 2 * WHALE_DK), 7000 + T2 + seed)
    qkv = randn((B, T2, 3 * C), 8000 + T2 + seed)
    lens = whale_lengths(T2)
    g = torch.Generator().manual_seed(9000 + T2)
    targets, kws = [], []
    for b, n in enumerate(lens):
        n = min(n, T2)
        kw = dict(group=1, scale=WHALE_DK ** -0.5, causal=False, q_pos0=0, kv_len=n)
        targets.append(_regime(q2[b], k2[b], regime, **kw))
        kws.append(kw)
        for t in (k2[b, n:], qkv[b, n:, 2 * C:]):
            sign = torch.randint(0, 2, t.shape, generator=g).to(BF16) * 2 - 1
            t.copy_(sign * 2.0 ** 60)
    return (q2, k2, qkv, lens), targets, kws


def paged_case(regime, seed=0):
    """PAGED_CASES: q [T, (32 + 16) * 128] packed (only the q columns are read), per sequence K / V [P + C, 8, 128]"""
    T = sum(c for _, c in PAGED_CASES)
    q = randn((T, QKV_W), 10000 + seed)
    kv, targets, kws = [], [], []
    r0 = 0
    for i, (p, c) in enumerate(PAGED_CASES):
        k, v = randn((p + c, NKV, D), 11000 + 2 * i + seed), randn((p + c, NKV, D), 11001 + 2 * i + seed)
        kw = dict(group=NQ // NKV, scale=D ** -0.5, causal=True, q_pos0=p, kv_len=p + c)
        targets.append(_regime(q[r0:r0 + c, :NQ * D].view(c, NQ, D), k, regime, **kw))
        kv.append((k, v))
        kws.append(kw)
        r0 += c
    return (q, kv), targets, kws
