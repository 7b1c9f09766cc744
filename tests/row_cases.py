"""Inputs of the prefill row-kernel tests (tests/test_row_shapes_gpu.py), built on the CPU from seeded generators so that
the CPU checks of tests/test_row_shapes.py see the same bits, and a host model of the qkv GEMM's tail-split schedule.

A. Norms.  RMSNorm rows carry per-row scales 2^-40 .. 2^40 (exact powers of two) and one all-zero row; the weight has
   mixed signs.  LayerNorm rows are randn at scales 2^-8 .. 2^8 with per-row means, rows with a common offset of 2^10,
   and a constant row.  bf16 holds only 1016, 1024 and 1032 around 2^10, so an offset row is 2^10 with a sparse set of
   +-8 steps: a variance of 0.008 .. 4 under a squared mean of 2^20.  A one-pass variance E[x^2] - mean^2 in fp32 loses
   about 2^20 * 2^-24 = 0.06 there, which the two-pass kernel does not.
B. qkv projection with the RoPE + paged-KV epilogue.  Positions 0, a run ending at 32767, a shuffled permutation of
   [0, 32768) and duplicates; slots on shuffled pages of 16 or 128 with spare pages, rows with slot -1, or no slots.
C. Router.  A generic gate (the random regime) and a crafted gate whose rows 2 and 5 are identical (exact ties) and
   whose rows 3 and 4 differ in one element only (near-ties), with crafted tokens: a tie for first place, a tie for
   second place, a zero row, a dominant logit (> 104 above the rest: the others' expf underflows to 0), and near-ties
   just above the accumulation bound, both for first and for second place.  The scatter uses "same pair" tokens that
   all choose experts (6, 1).
D. MoE combine.  Residual rows about 2^8 times the expert outputs, and expert outputs that cancel the residual.
"""
import math

import torch

BF16 = torch.bfloat16
E = 8
D = 128

# ------------------------------------------------------------------------------------------------ A. norms
RMS_H = (8, 4088, 4096, 4104, 12288, 16384)
RMS_ROWS = (1, 129, 4600)
RMS_EPS = (1e-5, 1e-6)
ACT_NONE, ACT_GELU, ACT_RELU = 0, 1, 2
# (caller, H, eps, act, out_scale): every LayerNorm the encoders run, and the largest H the kernel takes
LN_CASES = (("internvit", 1024, 1e-6, ACT_NONE, 1.0), ("whale", 1024, 1e-5, ACT_NONE, 1.0),
            ("whale embed", 1024, 1e-5, ACT_RELU, math.sqrt(1024)), ("adapter", 2048, 1e-3, ACT_GELU, 1.0),
            ("bound", 8192, 1e-5, ACT_NONE, 1.0))
LN_ROWS = (1, 129, 4600)
OFFSET = 1024.0


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def rms_case(rows, H, seed=0):
    """x [rows, H] bf16, w [H] bf16 with mixed signs, the per-row exponent (x = randn * 2^e).  Row rows // 2 is all
    zero when rows > 1; exponents -40 and 40 both occur when rows > 2."""
    g = _gen(100 + rows * 7 + H + seed)
    e = torch.randint(-40, 41, (rows,), generator=g)
    if rows > 2:
        e[0], e[-1] = -40, 40
    elif rows == 1:
        e[0] = 40
    x = torch.randn(rows, H, generator=g) * torch.pow(2.0, e.double()).float()[:, None]
    if rows > 1:
        x[rows // 2] = 0
        e[rows // 2] = 0
    sign = torch.randint(0, 2, (H,), generator=g) * 2 - 1
    w = sign * (0.25 + torch.rand(H, generator=g))
    return x.to(BF16), w.to(BF16), e


def ln_case(rows, H, seed=0):
    """x [rows, H], w [H] (mixed signs), b [H] bf16 and the kind of every row: "randn" (scale 2^-8 .. 2^8, a per-row mean
    of up to 4 scales), "offset k" (2^10 with k elements moved by +-8) and "constant" (row rows // 2 when rows > 1)"""
    g = _gen(200 + rows * 3 + H + seed)
    x = torch.empty(rows, H)
    kinds = []
    steps = (1, 4, H // 64, H // 16)
    for r in range(rows):
        if rows > 1 and r == rows // 2:
            x[r] = -3.25
            kinds.append("constant")
        elif r % 4 == 1:
            k = steps[(r // 4) % len(steps)]
            row = torch.full((H,), OFFSET)
            idx = torch.randperm(H, generator=g)[:k]
            row[idx] += 8.0 * (torch.randint(0, 2, (k,), generator=g) * 2 - 1)
            x[r] = row
            kinds.append(f"offset {k}")
        else:
            s = 2.0 ** int(torch.randint(-8, 9, (1,), generator=g))
            x[r] = (torch.randn(H, generator=g) + 4 * (torch.rand(1, generator=g) * 2 - 1)) * s
            kinds.append("randn")
    sign = torch.randint(0, 2, (H,), generator=g) * 2 - 1
    w = sign * (0.25 + torch.rand(H, generator=g))
    b = torch.randn(H, generator=g) * 0.5
    return x.to(BF16), w.to(BF16), b.to(BF16), kinds


def rms_ref(x, w, eps):
    """MixtralRMSNorm's fp32 formula in fp64: x * rsqrt(mean(x^2) + eps) * w (x, w on any device)"""
    x = x.double()
    return x * torch.rsqrt((x * x).mean(-1, keepdim=True) + eps) * w.double()


def ln_ref(x, w, b, eps, act, out_scale):
    """torch.nn.LayerNorm (biased variance) -> act -> * out_scale, in fp64"""
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    y = (x - mu) * torch.rsqrt(((x - mu) ** 2).mean(-1, keepdim=True) + eps) * w.double() + b.double()
    if act == ACT_GELU:
        y = 0.5 * y * (1.0 + torch.erf(y / math.sqrt(2.0)))
    elif act == ACT_RELU:
        y = y.clamp_min(0.0)
    return y * out_scale


def one_pass_var32(x, threads, vpt):
    """what a one-pass variance E[x^2] - mean^2 gives in fp32, summed as layernorm_kernel<threads, vpt> sums: each
    thread its 8 * vpt elements in order, then the 32 lanes of a warp by butterfly, then the warp totals.  x [rows, H]"""
    x = x.float()
    rows, H = x.shape
    nvec = H // 8

    def butterfly(t):                                  # warp_sum over the last dim (32 lanes)
        for o in (16, 8, 4, 2, 1):
            t = t + t[..., torch.arange(32) ^ o]
        return t[..., 0]

    def reduce(v):                                     # v [rows, H] fp32 -> block_sum in the kernel's order
        t = torch.zeros(rows, threads)
        for i in range(vpt):
            for j in range(8):
                cols = [(tid + i * threads) * 8 + j for tid in range(threads) if tid + i * threads < nvec]
                t[:, :len(cols)] += v[:, cols]
        w = butterfly(t.view(rows, threads // 32, 32))
        return butterfly(torch.cat([w, torch.zeros(rows, 32 - threads // 32)], -1))

    mean = reduce(x) / H
    return reduce(x * x) / H - mean * mean


# ------------------------------------------------------------------------------------------------ B. qkv + RoPE
ROPE_LEN, ROPE_THETA = 32768, 1e6
QKV_GEOMS = {"mixtral": (32, 8, 4096), "tiny": (4, 1, 512), "odd": (3, 2, 512)}
QKV_M = {"mixtral": (1, 127, 128, 129, 4600), "tiny": (1, 129, 4600), "odd": (1, 129, 4600)}
# (positions, slots) pairs run at every (geometry, M)
QKV_INPUTS = (("zero", "pages 16"), ("end", "pages 128"), ("perm", "pages 16, holes"), ("dup", "none"),
              ("end", "pages 128, holes"))
TILE_M, TILE_N = 128, 256


def qkv_cases():
    return [(geom, M) for geom in QKV_GEOMS for M in QKV_M[geom]]


def qkv_schedule(M, N, sms, tail_split=True):
    """(grid, whole tiles, split) of linear_qkv_rope: launch_gemm's grid min(SMs, 4 * max_tiles) with max_tiles =
    (M // 128 + 1) * ceil(N / 256), and make_sched's split of the R = tiles % grid tiles of the last wave into 2 pieces
    (one head each) when 2 R <= grid (gemm_sm90.cu).  split 1: every tile is processed whole."""
    num_n = (N + TILE_N - 1) // TILE_N
    max_tiles = (M // TILE_M + 1) * num_n
    grid = max(1, min(sms, max_tiles * (4 if tail_split else 1)))
    total = (M + TILE_M - 1) // TILE_M * num_n
    R = total % grid
    split = 2 if tail_split and R > 0 and 2 * R <= grid else 1
    return grid, total, split


def qkv_positions(kind, M, seed=0):
    g = _gen(300 + M + seed)
    if kind == "zero":
        p = torch.zeros(M, dtype=torch.int64)
    elif kind == "end":
        p = torch.arange(ROPE_LEN - M, ROPE_LEN)
    elif kind == "perm":
        p = torch.randperm(ROPE_LEN, generator=g)[:M]
    elif kind == "dup":
        p = torch.randint(0, ROPE_LEN, ((M + 1) // 2,), generator=g)
        p = torch.cat([p, p.flip(0)])[:M]
        p[0] = ROPE_LEN - 1
        p = p[torch.randperm(M, generator=g)]
    else:
        raise ValueError(kind)
    return p.to(torch.int32)


def qkv_slots(kind, M, seed=0):
    """slot_mapping [M] int32 (or None) and the number of cache slots: the sequence's pages in shuffled order among two
    spare pages that no row writes; "holes" gives every seventh row slot -1"""
    if kind == "none":
        return None, 0
    ps = 16 if "16" in kind else 128
    g = _gen(400 + M + ps + seed)
    n_pages = (M + ps - 1) // ps + 2
    perm = torch.randperm(n_pages, generator=g)
    t = torch.arange(M)
    slots = perm[t // ps] * ps + t % ps
    if "holes" in kind:
        slots[t % 7 == 3] = -1
    return slots.to(torch.int32), n_pages * ps


def qkv_case(geom, M, seed=0):
    """x [M, K], w [(n_q + 2 n_kv) * 128, K] bf16: projections of about unit size"""
    n_q, n_kv, K = QKV_GEOMS[geom]
    g = _gen(500 + M + K + n_q + seed)
    x = torch.randn(M, K, generator=g).to(BF16)
    w = (torch.randn((n_q + 2 * n_kv) * D, K, generator=g) * K ** -0.5).to(BF16)
    return x, w


def rope_ref(P, pos, table, n_rot):
    """P [M, heads, 128] fp64 projections; rotates heads [0, n_rot) by the fp32 table rows in fp64 (rotate_half form)"""
    cs = table[pos.long().to(table.device)].double().to(P.device)          # [M, 2, 64]
    c, s = cs[:, None, 0], cs[:, None, 1]
    out = P.clone()
    x1, x2 = P[:, :n_rot, :64], P[:, :n_rot, 64:]
    out[:, :n_rot, :64] = x1 * c - x2 * s
    out[:, :n_rot, 64:] = x2 * c + x1 * s
    return out


# ------------------------------------------------------------------------------------------------ C. router
ROUTER_H = (512, 4096)
ROUTER_T = (1, 2, 127, 128, 129, 4600)
SCATTER_T = (1, 129, 4600)
# Bound on the fp32 error of one router logit: the kernel sums exact products of bf16 values, 32 in order per thread,
# then 5 butterfly levels and 2 levels over the warps, so <= 39 roundings of at most 2^-24 each: < 2^-18.7 * sum|xn w|.
# 2^-16 leaves a factor of 6.5.
LOGIT_BOUND = 2.0 ** -16
LOGIT_ABS = 2.0 ** -21       # added to the bound: expf's relative error (<= 2 ulp) on the kernel's probabilities
SECOND_MAX_GAP = 80.0        # past this gap the second probability is below fp32's normal range: no order is defined
GATE_L1 = 150.0              # sum |g| of a full-scale gate row: a token aligned with it gets a logit of about 150
TIE, NEAR_A, NEAR_B, DOM = (2, 5), 3, 4, 6
NEAR_GAP = 3.0               # a near-tie's gap in bounds; `decided` needs more than 2
DOMINANT_GAP = 106.0         # expf(-104) < 2^-150 / 2 rounds to 0: the second weight is exactly 0
SAME_PAIR = (6, 1)


def _gate_sigma(H):
    return GATE_L1 / (0.8 * H)


def router_gate(H, crafted, seed=0):
    """gate [8, H] bf16.  crafted: row 5 = row 2, and row 4 = row 3 but for element 0, which is larger by near_d(H)"""
    g = _gen(600 + H + seed)
    gate = torch.randn(E, H, generator=g) * _gate_sigma(H)
    if crafted:
        gate[TIE[1]] = gate[TIE[0]]
        gate[NEAR_B] = gate[NEAR_A]
        gate[NEAR_B, 0] = gate[NEAR_A, 0] + near_d(H)
    return gate.to(BF16)


def near_d(H):
    """a power of two near the gate's scale"""
    return 2.0 ** round(math.log2(_gate_sigma(H)))


def router_norm_w(H, seed=0):
    g = _gen(700 + H + seed)
    return (0.5 + torch.rand(H, generator=g)).to(BF16)


def xn_host(h, nw, eps=1e-5):
    """the router's normed row as the CPU sees it: fp64 RMSNorm rounded to bf16 (the kernel's xn may differ by an ulp
    where its fp32 product lands on a rounding boundary)"""
    return rms_ref(h, nw, eps).to(BF16)


def logits64(xn, gate):
    """fp64 logits [T, 8] and the per-token bound LOGIT_BOUND * max_e sum_k |xn_k g_ek|.  Identical gate rows give
    identical logits (each row's dot product is computed alone)."""
    x, gd = xn.double(), gate.double().to(xn.device)
    lg = torch.stack([(x * gd[e]).sum(-1) for e in range(E)], -1)
    l1 = torch.stack([(x.abs() * gd[e].abs()).sum(-1) for e in range(E)], -1).amax(-1)
    return lg, LOGIT_BOUND * l1 + LOGIT_ABS


def top2_ref(lg, bound):
    """the kernel's rule on fp64 logits: descending, the first index wins exact ties.  Returns ids [T, 2], weights
    [T, 2] (fp64 softmax renormalised over the pair) and `decided` [T]: the top-1/top-2 and top-2/top-3 gaps are either
    exact ties or larger than twice the bound (each logit is off by at most the bound), and the top-1/top-2 gap is at
    most SECOND_MAX_GAP"""
    T = lg.shape[0]
    order = torch.sort(-lg, dim=-1, stable=True).indices
    srt = lg.gather(-1, order)
    ok = torch.ones(T, dtype=torch.bool, device=lg.device)
    for a in (0, 1):
        gap = srt[:, a] - srt[:, a + 1]
        ok &= (gap == 0) | (gap > 2 * bound)
    ok &= srt[:, 0] - srt[:, 1] <= SECOND_MAX_GAP
    ids = order[:, :2]
    d = (srt[:, 1] - srt[:, 0])
    w1 = torch.exp(d) / (1 + torch.exp(d))
    return ids, torch.stack([1 - w1, w1], -1), ok


def _aligned(gate_row_f):
    """a hidden row whose normed form lines up with a gate row: sign(g) (RMSNorm removes the scale)"""
    return torch.sign(gate_row_f)


# the ids each crafted token must get ("dominant": the top expert, then the lowest other index: every other
# probability underflows to exactly 0 and the first index wins ties)
CRAFTED_IDS = {"tie for first": TIE, "tie for second": (0, TIE[0]), "zero row": (0, 1), "dominant": (DOM, 0),
               "near-tie for first": (NEAR_B, NEAR_A), "near-tie for second": (7, NEAR_B)}


def crafted_tokens(H, nw, gate):
    """[(name, h [H] fp32)]: crafted hidden rows for the crafted gate, named as in CRAFTED_IDS"""
    gf, nwf = gate.float(), nw.float()
    out = [("tie for first", _aligned(gf[TIE[0]]) / nwf),                    # rows 2 and 5 are identical
           ("tie for second", _aligned(gf[0] + 0.6 * gf[TIE[0]]) / nwf),      # row 0 first, rows 2 / 5 tied behind
           ("zero row", torch.zeros(H)),                                     # eight equal logits
           ("dominant", _aligned(gf[DOM]) / nwf)]                            # the others' expf(l - m) underflows
    # near-ties: rows 3 / 4 differ in element 0 only, so l4 - l3 = xn_0 * (g4_0 - g3_0); xn_0 sets the gap to
    # NEAR_GAP bounds (just past the two bounds of `decided`), with the higher index 4 ahead of 3
    dd = float(gf[NEAR_B, 0] - gf[NEAR_A, 0])
    for name, base in (("near-tie for first", gf[NEAR_A]), ("near-tie for second", gf[7] + 0.6 * gf[NEAR_A])):
        h = _aligned(base) / nwf
        h[0] = 0.0
        x64 = h.double()
        inv = float(torch.rsqrt((x64 * x64).mean() + 1e-5))
        _, b = logits64(xn_host(h[None], nw), gate)
        h[0] = NEAR_GAP * float(b[0]) / dd / (inv * float(nwf[0]))
        out.append((name, h))
    return out


def router_case(T, H, regime, seed=0):
    """h [T, H] bf16, norm_w, gate and the name of every token.  "random": randn rows (scales 2^-4 .. 2^4) over the
    generic gate.  "crafted": the crafted tokens first (as many as fit), then randn rows, over the crafted gate."""
    nw = router_norm_w(H, seed)
    gate = router_gate(H, regime == "crafted", seed)
    g = _gen(800 + T + H + seed)
    s = torch.pow(2.0, torch.randint(-4, 5, (T,), generator=g).double()).float()[:, None]
    h = torch.randn(T, H, generator=g) * s
    names = ["randn"] * T
    if regime == "crafted":
        for i, (name, row) in enumerate(crafted_tokens(H, nw, gate)[:T]):
            h[i] = row
            names[i] = name
    elif regime == "same pair":
        a, b = SAME_PAIR
        gf = gate.float()
        h = (_aligned(gf[a] + 0.6 * gf[b]) / nw.float())[None] * (1 + 0.2 * torch.randn(T, H, generator=g)) * s
        names = ["same pair"] * T
    return h.to(BF16), nw, gate, names


# ------------------------------------------------------------------------------------------------ D. combine
COMBINE_H = (512, 4096)
COMBINE_T = (1, 129, 4600)


def combine_case(T, H, seed=0):
    """h, y0, y1 [T, H] bf16 in token order, ids [T, 2] int32 (distinct experts) and the kind of every row: "big h"
    (|h| ~ 2^8 |y|) or "cancel" (y0 ~ -0.3 h, y1 ~ -0.7 h: h + y0 + y1 is about 2^-6 of h).  Even rows are "big h"."""
    g = _gen(900 + T + H + seed)
    s = torch.pow(2.0, torch.randint(-3, 4, (T,), generator=g).double()).float()[:, None]
    h = (torch.randn(T, H, generator=g) * s).to(BF16).float()
    y0 = torch.randn(T, H, generator=g) * s * 2.0 ** -8
    y1 = torch.randn(T, H, generator=g) * s * 2.0 ** -8
    cancel = torch.arange(T) % 2 == 1
    e = torch.randn(T, H, generator=g) * s * 2.0 ** -6
    y0c = (-0.3 * h).to(BF16).float()
    y0[cancel] = y0c[cancel]
    y1[cancel] = (-h - y0c + e)[cancel]
    kinds = ["cancel" if c else "big h" for c in cancel.tolist()]
    a = torch.randint(0, E, (T,), generator=g)
    b = (a + torch.randint(1, E, (T,), generator=g)) % E
    ids = torch.stack([a, b], -1).to(torch.int32)
    return h.to(BF16), y0.to(BF16), y1.to(BF16), ids, kinds
