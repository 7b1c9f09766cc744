"""The decode-step kernels at the shapes that serve, against plain fp64 references.

A. Paged decode attention (Mixtral geometry: 32 query heads, 8 KV heads, D = 128) over batches whose rows have very
   different contexts (empty splits, splits of fewer than 16 keys, exactly 64 keys, the first pipelined key, long
   tails), shuffled block tables, every cache slot outside a row's context poisoned with NaN, q compact or as a strided
   view of the qkv rows, both split merges (tagged all-to-all and ticket).
B. The tensor-core decode GEMVs: qkv + RoPE + KV append (exactly one slot per row written), router + gate|up + down with
   the routing forced onto every ordered expert pair, the stream-K o-proj at its contributor extremes.
C. The arg-max contract of the LM head and of argmax_rows: the first index on ties, like torch.argmax, including
   ties between -0.0 and +0.0.  NaN logits are out of scope: their order is not specified.

After every launch the cross-CTA scratch must be all-zero again, and results must not depend on the batch a row runs
in: row b gives the same bits at B = 1 as inside a larger batch.
"""
import math

import pytest
import torch

from tests.util import BF16, close_rows, matmul64, same_bits

pytestmark = pytest.mark.gpu

NQ, NKV, D = 32, 8, 128
SCALE = D ** -0.5
EPS = 1e-5


def _cpu_randn(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=torch.float64) * scale).to(BF16)


def _gpu_randn(shape, seed, scale):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(BF16)


def _perm(n, seed):
    return torch.randperm(n, generator=torch.Generator().manual_seed(seed))


def _rmsnorm64(h, nw):
    h = h.double().cpu()
    return h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + EPS) * nw.double().cpu()


@pytest.fixture
def lib_options():
    """Sets library tunables for one test and restores their values afterwards."""
    from vita_b200 import ops
    names = ("attn_tagged", "attn_early")
    before = {n: ops.get_option(n) for n in names}
    yield ops.set_option
    for n, v in before.items():
        ops.set_option(n, v)


# ================================================================================================ A. paged attention
def _contexts(splits):
    return [1, 2, 15, 16, 17, 64, 65, 64 * splits - 1, 64 * splits, 64 * splits + 1, 1000, 4161]


def _attn_cases():
    pages = (16, 32, 128)
    cases = []
    # B = 16: every context of the list in one batch, at every split count (ticket merge: the 16 x 8 x splits CTAs are
    # more than the tagged all-to-all may keep resident)
    for i, s in enumerate((1, 2, 3, 4, 8, 12, 16)):
        cases.append((s, pages[i % 3], _contexts(s) + [3, 100, 2048, 63]))
    # the serving shape of the batched step, B = 3 at 16 splits: 384 CTAs, ticket merge
    cases.append((16, 16, [4161, 1, 64 * 16 + 1]))
    cases.append((16, 128, [64 * 16, 2, 1000]))
    # the largest batches that fit the tagged merge on a 132-SM H100 (two resident CTAs per SM): 8 / 4 / 2 rows at
    # 4 / 8 / 16 splits; the list of contexts in chunks, so that each one also runs through the tagged merge
    for s in (4, 8, 16):
        n = 264 // (NKV * s)
        ctx = _contexts(s)
        for j in range(0, len(ctx), n):
            cases.append((s, pages[(j // n + s) % 3], ctx[j:j + n]))
    for s, page, c in ((16, 128, [4161]), (4, 16, [257]), (12, 32, [4161]), (1, 16, [1000]), (2, 128, [129])):
        cases.append((s, page, c))
    return cases


ATTN_CASES = _attn_cases()


def _paged_cache(ctxs, page, seed):
    """K/V caches with every slot outside a row's context set to NaN, shuffled (non-monotone) block tables whose unused
    entries point at valid pages that hold NaN only, and the fp32 K/V rows of each context."""
    B = len(ctxs)
    need = [(c + page - 1) // page for c in ctxs]
    max_pages = max(need) + 2                      # the page after the last one is always a poisoned one
    n_poison = 3
    n_pages = sum(need) + n_poison
    perm = _perm(n_pages, seed)
    poison = perm[sum(need):]
    bt = torch.empty(B, max_pages, dtype=torch.int32)
    kc = torch.full((n_pages * page, NKV, D), float("nan"), dtype=BF16)
    vc = kc.clone()
    ks, vs = [], []
    off = 0
    for b, c in enumerate(ctxs):
        bt[b, :need[b]] = perm[off:off + need[b]]
        off += need[b]
        bt[b, need[b]:] = poison[_perm(max_pages - need[b], seed + 1 + b) % n_poison]
        k = _cpu_randn((c, NKV, D), 1000 * seed + 2 * b)
        v = _cpu_randn((c, NKV, D), 1000 * seed + 2 * b + 1)
        t = torch.arange(c)
        slots = bt[b, t // page].long() * page + t % page
        kc[slots], vc[slots] = k, v
        ks.append(k)
        vs.append(v)
    return bt, kc, vc, ks, vs


def _attn_ref(q, k, v):
    """explicit softmax attention in fp64: q [NQ, D], k / v [ctx, NKV, D] -> [NQ, D]"""
    qg = q.double().view(NKV, NQ // NKV, D)
    s = torch.einsum("gjd,tgd->gjt", qg, k.double()) * SCALE
    p = torch.softmax(s, dim=-1)
    return torch.einsum("gjt,tgd->gjd", p, v.double()).reshape(NQ, D)


@pytest.mark.parametrize("splits,page,ctxs", ATTN_CASES,
                         ids=[f"s{s}-p{p}-B{len(c)}-ctx{c[0]}" for s, p, c in ATTN_CASES])
def test_decode_attention_shapes(lib_options, splits, page, ctxs):
    from vita_b200 import ops
    B = len(ctxs)
    seed = 7 * splits + page + B
    bt, kc, vc, ks, vs = _paged_cache(ctxs, page, seed)
    q = _cpu_randn((B, NQ * D), seed + 500)
    ref = torch.stack([_attn_ref(q[b].view(NQ, D), ks[b], vs[b]) for b in range(B)])    # [B, NQ, D]
    kc_d, vc_d, bt_d = kc.cuda(), vc.cuda(), bt.cuda()
    cur = torch.tensor([c - 1 for c in ctxs], dtype=torch.int32, device="cuda")
    q_d = q.cuda()
    W = (NQ + 2 * NKV) * D
    qkv = torch.full((B, W), float("nan"), dtype=BF16, device="cuda")   # the K / V part of the rows stays NaN
    qkv[:, :NQ * D] = q_d
    ws = ops.decode_attention_workspace(B, NKV, splits, "cuda")
    sentinel = torch.full((NQ * D,), -7.25, dtype=BF16, device="cuda")

    def run(q_arg, q_stride, rows=slice(None)):
        n = len(range(B)[rows])
        out = torch.empty(n + 1, NQ * D, dtype=BF16, device="cuda")
        out[n] = sentinel
        ops.decode_attention(q_arg, kc_d, vc_d, bt_d[rows].contiguous(), cur[rows].contiguous(), out[:n], ws, NQ, NKV,
                             D, page, splits, SCALE, q_stride=q_stride)
        torch.cuda.synchronize()
        assert int(ws.count_nonzero()) == 0, f"workspace not all-zero after the launch (B={n})"
        same_bits(out[n], sentinel, f"out row {n} past the batch")
        return out[:n].clone()

    label = lambda i: f"row {i[0]} (ctx {ctxs[i[0]]}), head {i[1]}" if len(i) == 2 else f"row {i}"
    for tagged in (1, 0):
        lib_options("attn_tagged", tagged)
        path = ops.decode_attention_merge(B, NKV, splits)
        got = {}
        for layout, (q_arg, stride) in (("compact", (q_d, 0)), ("strided", (qkv[:, :NQ * D], W))):
            lib_options("attn_early", 1)
            o = run(q_arg, stride)
            same_bits(run(q_arg, stride), o, f"{path} merge, {layout} q: second launch on the same workspace")
            lib_options("attn_early", 0)
            same_bits(run(q_arg, stride), o, f"{path} merge, {layout} q: attn_early 0 vs 1")
            lib_options("attn_early", 1)
            close_rows(o.view(B, NQ, D), ref, f"decode attention, {path} merge, {layout} q, splits {splits}, "
                        f"page {page}", label)
            got[layout] = o
        same_bits(got["strided"], got["compact"], f"{path} merge: strided vs compact q")
        if B > 1:
            if ops.decode_attention_merge(1, NKV, splits) != path:
                continue
            for b in range(B):
                o1 = run(q_d[b:b + 1], 0, slice(b, b + 1))
                same_bits(o1[0], got["compact"][b], f"{path} merge: row {b} (ctx {ctxs[b]}) at B = 1 vs in B = {B}")


# ================================================================================================ B. tensor-core GEMVs
def _ws(B, rb):
    from vita_b200 import ops
    return ops.TcWorkspace(B, rb, "cuda")


def _ws_clean(ws, what):
    torch.cuda.synchronize()
    assert int(ws.buf.count_nonzero()) == 0, f"{what}: stream-K scratch not all-zero after the launch"


QKV_CASES = [("small", 16), ("small", 128), ("full", 16), ("full", 128)]


@pytest.mark.parametrize("geom,page", QKV_CASES, ids=[f"{g}-p{p}" for g, p in QKV_CASES])
def test_tc_qkv_rope_kv_append(geom, page):
    """q rows and exactly one K / V slot per row: RoPE'd projections against fp64; every other byte untouched"""
    from vita_b200 import ops, weights
    H = 512 if geom == "small" else 4096
    positions = [0, 15, 16, page - 1, page, 4095] if geom == "small" else [15, page, 4095]
    B = len(positions)
    R = (NQ + 2 * NKV) * D
    seed = H + page
    h = _cpu_randn((B, H), seed, 1.5)
    nw = _cpu_randn((H,), seed + 1)
    w = _gpu_randn((R, H), seed + 2, 1.0 / math.sqrt(H))
    table = weights.rope_table(4096, D, 1e6)
    max_pages = 4096 // page
    bt = _perm(B * max_pages, seed + 3).view(B, max_pages).to(torch.int32)
    cur = torch.tensor(positions, dtype=torch.int32)
    slots = [int(bt[b, p // page]) * page + p % page for b, p in enumerate(positions)]
    ws = _ws(B, NQ + 2 * NKV)

    # fp64 reference: bf16(rmsnorm) . W, rounded to bf16 before RoPE (as the kernel and the GEMM path do)
    x = _rmsnorm64(h, nw).to(BF16)
    y = matmul64(w, x).to(BF16).double()                                                 # [B, R]
    cs = table.double().view(4096, 128)
    heads = y.view(B, NQ + 2 * NKV, D)
    rot = heads.clone()
    for b, p in enumerate(positions):
        c, s = cs[p, :64], cs[p, 64:]
        lo, hi = heads[b, :NQ + NKV, :64], heads[b, :NQ + NKV, 64:]
        rot[b, :NQ + NKV, :64] = lo * c - hi * s
        rot[b, :NQ + NKV, 64:] = hi * c + lo * s
    q_ref, k_ref, v_ref = rot[:, :NQ], rot[:, NQ:NQ + NKV], rot[:, NQ + NKV:]

    n_slots = B * max_pages * page
    fill = 0x7FA5                   # a NaN with a payload the kernel never writes: compared bit for bit

    def run(rows):
        n = len(rows)
        q = torch.full((n + 1, NQ * D), fill, dtype=torch.int16, device="cuda").view(BF16)
        kc = torch.full((n_slots, NKV, D), fill, dtype=torch.int16, device="cuda").view(BF16)
        vc = kc.clone()
        ops.decode_tc_qkv_rope(h[rows].cuda(), nw.cuda(), w, table.cuda(), cur[rows].cuda(), bt[rows].cuda(), q[:n],
                               kc, vc, ws, NQ, NKV, D, page, EPS)
        _ws_clean(ws, f"qkv B={n}")
        assert (q[n].view(torch.int16) == fill).all(), f"q row {n} past the batch was written"
        mask = torch.ones(n_slots, dtype=torch.bool, device="cuda")
        mask[[slots[r] for r in rows]] = False
        for name, cc in (("k", kc), ("v", vc)):
            assert (cc.view(torch.int16)[mask] == fill).all(), \
                f"{name} cache: a byte outside the appended slots changed"
        return q[:n].clone(), kc, vc

    rows = list(range(B))
    q, kc, vc = run(rows)
    label = lambda i: f"row {i[0]} (pos {positions[i[0]]}), head {i[1]}"
    close_rows(q.view(B, NQ, D), q_ref, f"qkv q (page {page})", label)
    idx = torch.tensor(slots, device="cuda")
    close_rows(kc[idx], k_ref, f"qkv k cache append (page {page})", label)
    close_rows(vc[idx], v_ref, f"qkv v cache append (page {page})", label)
    q2, kc2, vc2 = run(rows)
    for a, b_, n in ((q, q2, "q"), (kc, kc2, "k cache"), (vc, vc2, "v cache")):
        same_bits(b_, a, f"qkv {n}: second launch on the same workspace")
    if geom == "full":
        for b in rows:
            q1, kc1, vc1 = run([b])
            same_bits(q1[0], q[b], f"qkv q row {b} at B = 1 vs in B = {B}")
            same_bits(kc1[slots[b]], kc[slots[b]], f"qkv k slot of row {b} at B = 1 vs in B = {B}")
            same_bits(vc1[slots[b]], vc[slots[b]], f"qkv v slot of row {b} at B = 1 vs in B = {B}")


def _forced_moe_inputs(H, pairs, n_blocks, seed):
    """Tokens with disjoint supports (mutually orthogonal normalised rows) and a router whose weight rows are built from
    those directions, so that token b's logits are 2.0 for pairs[b][0], 1.25 for pairs[b][1] and -0.5 .. -2.0 for the
    other experts: the chosen pair is set with wide margins."""
    B = len(pairs)
    blk = H // n_blocks
    h = torch.zeros(B, H, dtype=torch.float64)
    for b in range(B):
        h[b, b * blk:(b + 1) * blk] = _cpu_randn((blk,), seed + b, 1.5).double()
    h = h.to(BF16)
    g = torch.Generator().manual_seed(seed + 99)
    nw = (1.0 + 0.25 * torch.randn(H, generator=g, dtype=torch.float64)).to(BF16)
    xn = _rmsnorm64(h, nw)
    gw = torch.zeros(8, H, dtype=torch.float64)
    for b, (e0, e1) in enumerate(pairs):
        t = torch.linspace(-0.5, -2.0, 8, dtype=torch.float64)
        t[e0], t[e1] = 2.0, 1.25
        gw += t[:, None] * (xn[b] / (xn[b] @ xn[b]))[None, :]
    return h, nw, gw.to(BF16)


def _moe_check(h, nw, gw, w13, w2, pairs, resid, what, runs_at_b1=False):
    from vita_b200 import ops
    B, H = h.shape
    I = w13.shape[1] // 2
    ws = _ws(B, max(2 * (I // 128), H // 128))
    # fp64 router (HF order: softmax, top-2, renormalise)
    xn = _rmsnorm64(h, nw)
    probs = torch.softmax(xn @ gw.double().T, dim=-1)
    top_v, top_i = torch.topk(probs, 2, dim=-1)
    top_v = top_v / top_v.sum(-1, keepdim=True)
    assert top_i.tolist() == [list(p) for p in pairs], f"{what}: the forced routing is not what the reference picks"
    x = xn.to(BF16)

    def run(rows):
        n = len(rows)
        act = torch.full((n, 2, I), float("nan"), dtype=BF16, device="cuda")
        ids = torch.full((n, 2), -1, dtype=torch.int32, device="cuda")
        tw = torch.zeros(n, 2, dtype=torch.float32, device="cuda")
        hd = h[rows].cuda()
        ops.decode_tc_moe_gate_up(hd, nw.cuda(), gw.cuda(), w13, ids, tw, act, ws, EPS)
        _ws_clean(ws, f"{what}: gate|up B={n}")
        out = resid[rows].cuda()
        ops.decode_tc_moe_down(act, w2, ids, tw, out, ws)
        _ws_clean(ws, f"{what}: down B={n}")
        return act, ids, tw, out

    rows = list(range(B))
    act, ids, tw, out = run(rows)
    assert ids.cpu().tolist() == [list(p) for p in pairs], f"{what}: topk_ids {ids.cpu().tolist()}"
    assert (tw.cpu().double() - top_v).abs().max() < 1e-4, f"{what}: top-2 weights {tw.cpu().tolist()}"
    act_ref = torch.empty(B, 2, I, dtype=torch.float64)
    down_ref = resid.double().clone()
    for e in sorted({e for p in pairs for e in p}):          # only the experts in use, each matrix converted once
        uses = [(b, k) for b, p in enumerate(pairs) for k in range(2) if p[k] == e]
        gu = matmul64(w13[e], torch.stack([x[b] for b, _ in uses]))
        dn = matmul64(w2[e], torch.stack([act[b, k] for b, k in uses]))   # the down projection of the kernel's act
        for n, (b, k) in enumerate(uses):
            act_ref[b, k] = torch.nn.functional.silu(gu[n, :I]) * gu[n, I:]
            down_ref[b] += top_v[b, k] * dn[n]
    close_rows(act, act_ref, f"{what}: gate|up activations",
                lambda i: f"token {i[0]} (experts {pairs[i[0]]}), slot {i[1]}")
    close_rows(out, down_ref, f"{what}: down + residual", lambda i: f"token {i[0]} (experts {pairs[i[0]]})")
    again = run(rows)
    for a, b_, n in zip((act, ids, tw, out), again, ("act", "ids", "weights", "out")):
        same_bits(b_, a, f"{what}: {n}, second launch on the same workspace")
    if runs_at_b1:
        for b in rows:
            for a, b_, n in zip((act, ids, tw, out), run([b]), ("act", "ids", "weights", "out")):
                same_bits(b_[0], a[b], f"{what}: {n} of token {b} at B = 1 vs in B = {B}")


ALL_PAIRS = [(i, j) for i in range(8) for j in range(8) if i != j]


@pytest.mark.parametrize("group", range(7))
def test_tc_moe_every_expert_pair_small(group):
    """H = 512, I = 1024: 8 tokens per launch, 7 launches cover the 56 ordered expert pairs"""
    H, I = 512, 1024
    pairs = ALL_PAIRS[8 * group:8 * group + 8]
    h, nw, gw = _forced_moe_inputs(H, pairs, 8, 40 + group)
    w13 = _gpu_randn((8, 2 * I, H), 11, 0.05)
    w2 = _gpu_randn((8, H, I), 12, 0.05)
    resid = _cpu_randn((len(pairs), H), 50 + group, 0.25)
    _moe_check(h, nw, gw, w13, w2, pairs, resid, f"moe pairs {pairs}")


def test_tc_moe_full_geometry_edge_experts():
    """H = 4096, I = 14336: the first and the last expert of w13 / w2 (expert 7's rows end at the tensor maps' edge),
    B = 3 and each token alone"""
    H, I = 4096, 14336
    pairs = [(7, 0), (0, 7), (3, 6)]
    h, nw, gw = _forced_moe_inputs(H, pairs, 4, 70)
    w13 = _gpu_randn((8, 2 * I, H), 21, 0.02)
    w2 = _gpu_randn((8, H, I), 22, 0.015)
    resid = _cpu_randn((len(pairs), H), 71, 0.25)
    _moe_check(h, nw, gw, w13, w2, pairs, resid, "moe full geometry", runs_at_b1=True)


OPROJ_CASES = [(n, k) for n in (1000, 4096) for k in (64, 384, 448, 4096)]


@pytest.mark.parametrize("N,K", OPROJ_CASES, ids=[f"N{n}-K{k}" for n, k in OPROJ_CASES])
def test_tc_oproj_stream_k_extremes(N, K):
    """K = 64: one k-block, no partial row block; K = 384: one unit per CTA, up to 6 contributors per row block;
    K = 448: 7 k-blocks over CTAs of 2 units; K = 4096: the serving shape"""
    from vita_b200 import ops
    B = 3
    x = _cpu_randn((B, K), N + K)
    h = _cpu_randn((B, N), N + K + 1)
    w = _gpu_randn((N, K), N + K + 2, 1.0 / math.sqrt(K))
    ws = _ws(B, (N + 127) // 128)
    ref = h.double() + matmul64(w, x)

    def run(rows):
        out = h[rows].cuda()
        ops.decode_tc_oproj(x[rows].cuda(), w, out, ws)
        _ws_clean(ws, f"oproj N={N} K={K} B={len(rows)}")
        return out

    rows = list(range(B))
    out = run(rows)
    close_rows(out, ref, f"oproj N={N} K={K}", lambda i: f"row {i[0]}")
    same_bits(run(rows), out, f"oproj N={N} K={K}: second launch on the same workspace")
    for b in rows:
        same_bits(run([b])[0], out[b], f"oproj N={N} K={K}: row {b} at B = 1 vs in B = {B}")


# ================================================================================================ C. arg-max contract
def _unpack(words):
    return [int(0xFFFFFFFF - (int(w) & 0xFFFFFFFF)) for w in words.cpu().tolist()]


def _tie_pairs(V):
    rb = (V + 127) // 128
    return [
        (128 * (rb // 4) + 3, 128 * (rb // 4) + 29),       # one warp, two lanes
        (128 * (rb // 3) + 7, 128 * (rb // 3 + 1) + 7),    # one lane, neighbouring row blocks
        (128 * (rb // 2) + 10, 128 * (rb // 2) + 100),     # two warps of one row block
        (V // 50, V - V // 5),                             # far apart: different CTAs
        (0, V - 1),                                        # first row, last row of the partial last row block
        (128 * 5 + 120, 128 * 6 + 2),                      # lower index in a higher warp
    ]


def _greedy_words(logits):
    """argmax_rows and the sampler's greedy word (temperature 0) over the same rows"""
    from vita_b200 import ops
    B = logits.shape[0]
    a = torch.zeros(B, dtype=torch.int64, device="cuda")
    ops.argmax_rows(logits, a)
    s = torch.zeros(B, dtype=torch.int64, device="cuda")
    f = lambda v, dt: torch.full((B,), v, dtype=dt, device="cuda")
    ops.sample_rows(logits, f(0.0, torch.float32), f(0, torch.int32), f(1.0, torch.float32), f(1, torch.int64),
                    f(0, torch.int32), s)
    torch.cuda.synchronize()
    return a, s


def _lm_head(h, nw, w):
    from vita_b200 import ops
    V, H = w.shape
    B = h.shape[0]
    ws = _ws(B, (V + 127) // 128)
    logits = torch.empty(B, V, dtype=BF16, device="cuda")
    best = torch.zeros(B, dtype=torch.int64, device="cuda")
    ops.tc_lm_head_argmax(h, H, nw, w, logits, best, B, ws, EPS)
    _ws_clean(ws, f"lm head V={V} B={B}")
    return logits, best


def _check_argmax(logits, best, what):
    want = torch.argmax(logits.float(), dim=-1).tolist()
    got = _unpack(best)
    assert got == want, f"{what}: LM head picks {got}, torch.argmax of its logits {want}"
    a, s = _greedy_words(logits)
    assert torch.equal(a, best), f"{what}: argmax_rows {_unpack(a)} vs the LM head's word {got}"
    assert torch.equal(s, a), f"{what}: sampler greedy word {_unpack(s)} vs argmax_rows {_unpack(a)}"


@pytest.mark.parametrize("H,V", [(4096, 51760), (512, 2047)])
def test_lm_head_argmax_ties(H, V):
    """Pairs of identical W rows hold the maximum of one row each (exact ties: one non-zero weight per pair row, so the
    logits are exact products); placed in one warp, in two warps, in two CTAs, and at 0 / V - 1."""
    pairs = _tie_pairs(V)
    B = len(pairs)
    cols = [7 + 64 * p for p in range(B)]
    h = _cpu_randn((B, H), V, 1.5).double()
    nw = _cpu_randn((H,), V + 1).double()
    for b in range(B):
        h[b, cols] = 0.0
        h[b, cols[b]] = 4.0
    nw[cols] = 1.0
    h, nw = h.to(BF16).cuda(), nw.to(BF16).cuda()
    Vp = (V + 7) // 8 * 8
    w_full = _gpu_randn((Vp, H), V + 2, 0.03)
    for p, (i, j) in enumerate(pairs):
        for r in (i, j):
            w_full[r] = 0.0
            w_full[r, cols[p]] = 8.0
    w = w_full[:V]
    logits, best = _lm_head(h, nw, w)
    x = _rmsnorm64(h, nw).to(BF16)
    ref = matmul64(w, x)
    close_rows(logits, ref, f"lm head logits V={V}", lambda i: f"row {i[0]}")
    for b, (i, j) in enumerate(pairs):
        assert logits[b, i].item() == logits[b, j].item() == logits[b].float().max().item(), \
            f"row {b}: the tie at ({i}, {j}) is not the maximum"
    _check_argmax(logits, best, f"lm head ties V={V}")
    assert _unpack(best) == [i for i, _ in pairs]
    l1, b1 = _lm_head(h[:1], nw, w)
    same_bits(l1[0], logits[0], f"lm head logits row 0 at B = 1 vs in B = {B}")
    assert torch.equal(b1[0], best[0]), f"lm head: arg-max word of row 0 at B = 1 vs in B = {B}"


@pytest.mark.parametrize("H,V", [(4096, 51760), (512, 2047)])
def test_lm_head_argmax_zero_maximum(H, V):
    """Every logit is negative except those of two W rows, one all -0.0 and one all +0.0: the maximum is zero, its key
    has to rank above every negative one, and the lower of the two indices wins.  On the H100 both zero logits come out
    as +0.0 (the tensor cores sum the -0.0 products to +0.0, and stream-K partial sums start from +0.0), so this is a
    tie of two +0.0 today; the LM head is held to torch.argmax whatever signs it returns."""
    g = torch.Generator().manual_seed(V)
    h = (torch.rand(2, H, generator=g, dtype=torch.float64) + 0.1).to(BF16).cuda()
    nw = (torch.rand(H, generator=g, dtype=torch.float64) + 0.5).to(BF16).cuda()
    Vp = (V + 7) // 8 * 8
    w_full = -_gpu_randn((Vp, H), V + 3, 0.03).abs()
    i, j = V // 50, V - V // 5
    w_full[i] = -0.0
    w_full[j] = 0.0
    logits, best = _lm_head(h, nw, w_full[:V])
    assert (logits.float().max(-1).values == 0).all()
    _check_argmax(logits, best, f"lm head zero maximum V={V}")
    assert _unpack(best) == [i, i]


@pytest.mark.parametrize("V", [51760, 2047])
def test_argmax_rows_signed_zero_and_ties(V):
    """argmax_rows and the sampler's greedy word on crafted rows: the maximum is -0.0 and +0.0 in both orders, or an
    exact tie, at index pairs in one thread, in two threads and far apart.  Expected: torch.argmax (first index)."""
    spots = [(5, 6), (5, 5 + 256), (100, V - 1), (0, V // 2 + 3)]
    rows, want = [], []
    g = torch.Generator().manual_seed(V)
    for i, j in spots:
        for a, b in ((-0.0, 0.0), (0.0, -0.0), (1.5, 1.5)):
            r = -1.0 - torch.rand(V, generator=g, dtype=torch.float64)
            r[i], r[j] = a, b
            rows.append(r)
            want.append(i)
    logits = torch.stack(rows).to(BF16).cuda()
    assert torch.argmax(logits.float(), dim=-1).tolist() == want
    a, s = _greedy_words(logits)
    assert _unpack(a) == want, f"argmax_rows {_unpack(a)} vs torch.argmax {want}"
    assert torch.equal(s, a), f"sampler greedy word {_unpack(s)} vs argmax_rows {_unpack(a)}"


@pytest.mark.parametrize("V", [51760, 2047])
def test_sampler_keeps_a_zero_maximum(V):
    """Sampled rows (T > 0) whose largest logit is zero: top_p = 0 and top_k = 1 keep the largest logit.  A lone -0.0
    maximum is the only token kept; -0.0 and +0.0 together are one value, both stay, and the draw between them follows
    the fp64 sampling oracle."""
    import numpy as np
    from oracle import sampling_oracle as SO
    from vita_b200 import ops
    g = torch.Generator().manual_seed(V + 1)
    rows, params, lone = [], [], []
    for i in (5, 300, V - 1):
        for T, k, p in ((0.7, 0, 0.0), (0.7, 1, 1.0), (1.3, 1, 0.0)):
            r = -1.0 - torch.rand(V, generator=g, dtype=torch.float64)
            r[i] = -0.0
            rows.append(r)
            params.append((T, k, p))
            lone.append(i)
    for i, j in ((5, 6), (0, V - 1)):
        for a, b in ((-0.0, 0.0), (0.0, -0.0)):
            for n in range(4):
                r = -1.0 - torch.rand(V, generator=g, dtype=torch.float64)
                r[i], r[j] = a, b
                rows.append(r)
                params.append((0.7, 0, 0.0))
                lone.append(None)
    B = len(rows)
    logits = torch.stack(rows).to(BF16).cuda()
    f = lambda col, dt: torch.tensor([x[col] for x in params], dtype=dt, device="cuda")
    seeds = [1234567 + b for b in range(B)]
    counters = [b % 4 for b in range(B)]
    best = torch.zeros(B, dtype=torch.int64, device="cuda")
    ops.sample_rows(logits, f(0, torch.float32), f(1, torch.int32), f(2, torch.float32),
                    torch.tensor(seeds, dtype=torch.int64, device="cuda"),
                    torch.tensor(counters, dtype=torch.int32, device="cuda"), best)
    got = _unpack(best)
    lf = logits.float().cpu().numpy()
    for b in range(B):
        T, k, p = params[b]
        if lone[b] is not None:
            assert got[b] == lone[b], f"row {b} (T {T}, top_k {k}, top_p {p}): drew {got[b]}, the only kept token is {lone[b]}"
            continue
        tok, gap, _ = SO.choose(lf[b], T, k, p, seeds[b], counters[b])
        zeros = set(np.flatnonzero(lf[b] == 0).tolist())
        assert got[b] in zeros, f"row {b}: drew {got[b]}, outside the zero maximum {sorted(zeros)}"
        if gap > 1e-4:
            assert got[b] == tok, f"row {b}: drew {got[b]}, the oracle draws {tok} (gap {gap:.3g})"
