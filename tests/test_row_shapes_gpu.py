"""The prefill layer's row kernels at the shapes that serve, against plain fp64 references, row by row
(inputs: tests/row_cases.py; their CPU checks: tests/test_row_shapes.py).

A. ops.rmsnorm at H in {8, 4088, 4096, 4104, 12288, 16384} (both instantiations, and nvec not a multiple of the block)
   over rows of scale 2^-40 .. 2^40 and an all-zero row; ops.layernorm at every (H, eps, act, out_scale) the encoders
   use, with offset rows that a one-pass variance gets wrong and a constant row (output act(bias) * scale).
B. ops.linear_qkv_rope (RoPE + paged-KV append in the GEMM epilogue) in the 32/8, 4/1 and 3/2 head geometries at
   positions up to 32767, duplicates and holes (slot -1): q and k heads against an fp64 rotation by the fp32 table, v
   heads unrotated, cache rows bit-identical to the k / v heads of the output and nothing else written.  The tail-split
   schedule is modelled on the host (row_cases.qkv_schedule); switching it off gives the same bits.
C. ops.moe_router / ops.moe_route_scatter: exact ids and weights within the accumulation bound on every decided token,
   the tie rule, the zero row, a dominant logit, near-ties; bits independent of the batch and equal between the two
   kernels; the scatter at capacity = T with two experts exactly full, compared through perm_row.
D. ops.moe_combine over the dense (moe_align) and slot (moe_route_scatter) layouts, with residuals 2^8 times the expert
   outputs and outputs that cancel the residual, with and without the next RMSNorm.
E. The embedding splice (ops.row_copy) at [51760, 4096] and past the grid's row count, and the encoders' glue at serving
   geometry (InternViT im2col / assemble / pixel shuffle, Whale conv1 / im2col / adapter im2col / qk prep): exact
   copies and single roundings bit for bit, Whale's conv1 against fp64.

Every output is a contiguous slice of a larger buffer filled with a canary; only the bytes the kernel is meant to write
may change, and a second launch gives the same bits.  Relative errors are per row: max |got - ref| / max |ref|.
"""
import functools

import pytest
import torch

from tests import row_cases as RC
from tests.util import BF16, close_rows, same_bits

pytestmark = pytest.mark.gpu

FILL = 0x7FA5                    # bf16 canary: a NaN with a payload no kernel writes
FILL32 = 0x7FC0BEEF              # fp32 / int32 canary: a NaN, and a row index no kernel writes
E = RC.E
WORST = {}                       # section -> worst per-row relative error seen


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(WORST):
        print(f"row kernels worst rel error {key}: {WORST[key]:.3e}")


def _note(key, r):
    WORST[key] = max(WORST.get(key, 0.0), r)


@functools.lru_cache(maxsize=4)
def _cached(build, *args):
    """the CPU-built inputs of a case (callers copy them to the GPU)"""
    return build(*args)


def _canary(shape, dtype=BF16):
    if dtype == BF16:
        return torch.full(shape, FILL, dtype=torch.int16, device="cuda").view(BF16)
    return torch.full(shape, FILL32, dtype=torch.int32, device="cuda").view(dtype)


def _raw(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32)


def _is_canary(t):
    return _raw(t) == (FILL if t.dtype == BF16 else FILL32)


def _untouched(buf, inside, what):
    """every element of buf outside the index `inside` (along the first dimension) still holds the canary"""
    mask = torch.ones(buf.shape[0], dtype=torch.bool, device=buf.device)
    mask[inside] = False
    n = int((~_is_canary(buf[mask])).sum())
    assert n == 0, f"{what}: {n} elements outside the output were written"


def _padded(rows, *shape, dtype=BF16):
    """(buffer, view): rows [1, rows + 1) of a canary buffer with one spare row on each side"""
    buf = _canary((rows + 2, *shape), dtype)
    return buf, buf[1:rows + 1]


def _close(got, want, what, labels, rel=1.6e-2):
    """close_rows on rows brought to [1, 2) by an exact power of two each: a row of scale 2^-40 gets the same relative
    test as one of scale 1 (close_rows alone floors max|ref| at 1e-6)"""
    want = want.double()
    m = want.abs().amax(-1, keepdim=True)
    p = torch.where(m > 0, torch.exp2(torch.floor(torch.log2(m))), torch.ones_like(m))
    return close_rows(got.to(want.device).double() / p, want / p, what, labels, rel)


# ================================================================================================ A. norms
@pytest.mark.parametrize("H", RC.RMS_H)
@pytest.mark.parametrize("rows", RC.RMS_ROWS)
def test_rmsnorm(rows, H):
    from vita_b200 import ops
    x, w, e = _cached(RC.rms_case, rows, H)
    x, w = x.cuda(), w.cuda()
    for eps in RC.RMS_EPS:
        what = f"rmsnorm rows={rows} H={H} eps={eps}"
        outs = []
        for _ in range(2):
            buf, out = _padded(rows, H)
            ops.rmsnorm(x, w, eps, out=out)
            torch.cuda.synchronize()
            _untouched(buf, slice(1, rows + 1), what)
            outs.append(out.clone())
        same_bits(outs[1], outs[0], f"{what}: second launch")
        got = outs[0]
        if rows > 1:
            assert (got[rows // 2].float() == 0).all(), f"{what}: the zero row gives {got[rows // 2][:8].tolist()}"
        _note("A rmsnorm", _close(got, RC.rms_ref(x, w, eps), what, lambda i: f"row {i[0]} (x ~ 2^{int(e[i[0]])})"))


@pytest.mark.parametrize("rows", RC.LN_ROWS)
@pytest.mark.parametrize("case", RC.LN_CASES, ids=[c[0] for c in RC.LN_CASES])
def test_layernorm(case, rows):
    from vita_b200 import ops
    name, H, eps, act, scale = case
    x, w, b, kinds = _cached(RC.ln_case, rows, H)
    x, w, b = x.cuda(), w.cuda(), b.cuda()
    what = f"layernorm {name} rows={rows}"
    outs = []
    for _ in range(2):
        buf, out = _padded(rows, H)
        ops.layernorm(x, w, b, eps, act, scale, out=out)
        torch.cuda.synchronize()
        _untouched(buf, slice(1, rows + 1), what)
        outs.append(out.clone())
    same_bits(outs[1], outs[0], f"{what}: second launch")
    got = outs[0]
    if rows > 1 and act == RC.ACT_NONE and scale == 1.0:
        same_bits(got[rows // 2], b, f"{what}: the constant row must give the bias")
    _note("A layernorm", _close(got, RC.ln_ref(x, w, b, eps, act, scale), what, lambda i: f"row {i[0]} ({kinds[i[0]]})"))


# ================================================================================================ B. qkv + RoPE + KV append
@functools.lru_cache(maxsize=1)
def _table():
    from vita_b200 import weights
    return weights.rope_table(RC.ROPE_LEN, RC.D, RC.ROPE_THETA).cuda()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _qkv_run(x, w, pos, slots, n_slots, n_q, n_kv):
    """linear_qkv_rope into rows [1, M + 1) of a canary buffer and canary caches of n_slots slots"""
    from vita_b200 import ops
    M, N = x.shape[0], w.shape[0]
    buf, out = _padded(M, N)
    kc = vc = None
    if slots is not None:
        kc, vc = _canary((n_slots, n_kv, RC.D)), _canary((n_slots, n_kv, RC.D))
        slots = slots.cuda()
    ops.linear_qkv_rope(x, w, out, pos.cuda(), slots, _table(), kc, vc, n_q, n_kv, RC.D)
    torch.cuda.synchronize()
    _untouched(buf, slice(1, M + 1), "qkv_out")
    return out.clone(), kc, vc


def _check_caches(out, kc, vc, slots, n_q, n_kv, what):
    D = RC.D
    if slots is None:
        return
    s = slots.cuda().long()
    live = s >= 0
    k_rows = out[live, n_q * D:(n_q + n_kv) * D].reshape(-1, n_kv, D)
    v_rows = out[live, (n_q + n_kv) * D:].reshape(-1, n_kv, D)
    same_bits(kc[s[live]], k_rows, f"{what}: k cache rows vs the k heads of qkv_out")
    same_bits(vc[s[live]], v_rows, f"{what}: v cache rows vs the v heads of qkv_out")
    for c, name in ((kc, "k"), (vc, "v")):
        _untouched(c, s[live], f"{what}: {name} cache (slot -1 rows and spare pages)")


@pytest.mark.parametrize("geom,M", RC.qkv_cases())
def test_qkv_rope_kv_append(geom, M, monkeypatch):
    n_q, n_kv, _ = RC.QKV_GEOMS[geom]
    heads = n_q + 2 * n_kv
    x, w = _cached(RC.qkv_case, geom, M)
    x, w = x.cuda(), w.cuda()
    P = (x.double() @ w.double().T).view(M, heads, RC.D)
    grid, tiles, split = RC.qkv_schedule(M, w.shape[0], _sms())
    sched = f"{tiles} tiles on {grid} CTAs, " + ("tail split in 2" if split == 2 else "no split")
    first = None
    for pos_kind, slot_kind in RC.QKV_INPUTS:
        pos = RC.qkv_positions(pos_kind, M)
        slots, n_slots = RC.qkv_slots(slot_kind, M)
        what = f"qkv {geom} M={M}, positions {pos_kind}, slots {slot_kind} ({sched})"
        runs = [_qkv_run(x, w, pos, slots, n_slots, n_q, n_kv) for _ in range(2)]
        for a, b in zip(runs[1], runs[0]):
            if a is not None:
                same_bits(a, b, f"{what}: second launch")
        out, kc, vc = runs[0]
        ref = RC.rope_ref(P, pos, _table(), n_q + n_kv)
        label = lambda i: f"row {i[0]} (position {int(pos[i[0]])}), head {i[1]}"
        _note("B qkv rope", close_rows(out.view(M, heads, RC.D), ref, what, label))
        _check_caches(out, kc, vc, slots, n_q, n_kv, what)
        if first is None:
            first = (pos, slots, n_slots, runs[0])
    monkeypatch.setenv("VITA_B200_GEMM_TAIL_SPLIT", "0")           # read at every dispatch
    pos, slots, n_slots, want = first
    got = _qkv_run(x, w, pos, slots, n_slots, n_q, n_kv)
    for a, b, name in zip(got, want, ("qkv_out", "k cache", "v cache")):
        if a is not None:
            same_bits(a, b, f"qkv {geom} M={M}: {name} without the tail split vs {sched}")


def test_qkv_schedules_take_both_paths():
    """on this GPU's SM count, at least one case of B cuts its last wave and one does not"""
    sms = _sms()
    splits = {}
    for geom, M in RC.qkv_cases():
        n_q, n_kv, _ = RC.QKV_GEOMS[geom]
        splits[(geom, M)] = RC.qkv_schedule(M, (n_q + 2 * n_kv) * RC.D, sms)
    print(f"qkv schedules on {sms} SMs (grid, tiles, split): {splits}")
    assert {s[2] for s in splits.values()} == {1, 2}, splits


# ================================================================================================ C. router + scatter
EPS = 1e-5


def _router_run(h, nw, gate):
    """moe_router into canary-padded outputs: (xn [T, H], ids [T, 2], w [T, 2])"""
    from vita_b200 import ops
    T, H = h.shape
    xb, xn = _padded(T, H)
    ib, ids = _padded(2 * T, dtype=torch.int32)
    wb, tw = _padded(2 * T, dtype=torch.float32)
    ops.moe_router(h, nw, gate, xn, ids.view(T, 2), tw.view(T, 2), EPS)
    torch.cuda.synchronize()
    for buf, n, name in ((xb, T, "xn"), (ib, 2 * T, "topk_ids"), (wb, 2 * T, "topk_w")):
        _untouched(buf, slice(1, n + 1), f"router {name}")
    return xn.clone(), ids.view(T, 2).clone(), tw.view(T, 2).clone()


def _check_router(h, nw, gate, names, what, xn, ids, tw):
    T = h.shape[0]
    label = lambda i: f"token {i[0]} ({names[i[0]]})"
    _note("C router xn", _close(xn, RC.rms_ref(h, nw, EPS), f"{what}: xn", label))
    lg, bound = RC.logits64(xn, gate)
    want_ids, want_w, decided = RC.top2_ref(lg, bound)
    ids, tw = ids.long(), tw.double()
    assert torch.isfinite(tw).all(), f"{what}: non-finite weights"
    crafted = {n: t for t, n in enumerate(names) if n != "randn"}
    for name, t in crafted.items():
        tag = f"{what}: {name} (token {t})"
        got = ids[t].tolist()
        assert got == list(RC.CRAFTED_IDS[name]), f"{tag}: ids {got}, want {list(RC.CRAFTED_IDS[name])}"
        if name == "dominant":
            assert tw[t].tolist() == [1.0, 0.0], f"{tag}: weights {tw[t].tolist()}"
            continue
        assert bool(decided[t]), f"{tag}: not decided on the kernel's xn"
        if name in ("tie for first", "zero row"):
            assert tw[t].tolist() == [0.5, 0.5], f"{tag}: weights {tw[t].tolist()}"
        if name == "zero row":
            assert not xn[t].float().any(), f"{tag}: xn is not zero"
    bad = decided & (ids != want_ids).any(-1)
    if bad.any():
        t = int(bad.nonzero()[0])
        pytest.fail(f"{what}: token {t} ({names[t]}) routed to {ids[t].tolist()}, fp64 says {want_ids[t].tolist()} "
                    f"(logits {lg[t].tolist()})")
    err = ((tw - want_w).abs().amax(-1) - bound)[decided]                  # weight error <= bound / 2 + a few ulps
    assert err.numel() == 0 or float(err.max()) <= 2.0 ** -20, f"{what}: a weight is off by more than the bound"
    if decided.any():
        _note("C router weights (abs)", float((tw - want_w).abs().amax(-1)[decided].max()))
    assert ((tw.sum(-1) - 1).abs() <= 2.0 ** -22).all(), f"{what}: weights do not sum to 1"
    return decided


@pytest.mark.parametrize("regime", ["random", "crafted"])
@pytest.mark.parametrize("T", RC.ROUTER_T)
@pytest.mark.parametrize("H", RC.ROUTER_H)
def test_router(H, T, regime):
    h, nw, gate, names = _cached(RC.router_case, T, H, regime)
    h, nw, gate = h.cuda(), nw.cuda(), gate.cuda()
    what = f"router H={H} T={T} {regime}"
    runs = [_router_run(h, nw, gate) for _ in range(2)]
    for a, b, n in zip(runs[1], runs[0], ("xn", "ids", "weights")):
        same_bits(a, b, f"{what}: {n}, second launch")
    decided = _check_router(h, nw, gate, names, what, *runs[0])
    if regime == "random":
        assert float(decided.double().mean()) >= 0.95, f"{what}: only {float(decided.double().mean()):.3f} decided"


def _scatter_run(h, nw, gate, cap, with_topk):
    """moe_route_scatter into canary buffers: (x_slots, counts, perm_row [T, 2], row_weight, ids, w)"""
    from vita_b200 import ops
    T, H = h.shape
    xb, xs = _padded(E * cap, H)
    rb, rw = _padded(E * cap, dtype=torch.float32)
    pb, perm = _padded(2 * T, dtype=torch.int32)
    cnt = torch.zeros(E, dtype=torch.int32, device="cuda")
    ids = tw = None
    if with_topk:
        ids, tw = torch.empty(T, 2, dtype=torch.int32, device="cuda"), torch.empty(T, 2, device="cuda")
    ops.moe_route_scatter(h, nw, gate, xs, cnt, perm, rw, EPS, ids, tw)
    torch.cuda.synchronize()
    for buf, n, name in ((xb, E * cap, "x_slots"), (rb, E * cap, "row_weight"), (pb, 2 * T, "perm_row")):
        _untouched(buf, slice(1, n + 1), f"scatter {name}")
    return xs, cnt, perm.view(T, 2).long(), rw, ids, tw


@pytest.mark.parametrize("regime", ["random", "same pair"])
@pytest.mark.parametrize("T", RC.SCATTER_T)
@pytest.mark.parametrize("H", RC.ROUTER_H)
def test_route_scatter_at_capacity(H, T, regime):
    """capacity = T, the least the API allows; "same pair" fills experts 6 and 1 exactly"""
    h, nw, gate, names = _cached(RC.router_case, T, H, regime)
    h, nw, gate = h.cuda(), nw.cuda(), gate.cuda()
    what = f"scatter H={H} T={T} {regime}, capacity {T}"
    xn, ids_r, tw_r = _router_run(h, nw, gate)
    xs, cnt, p, rw, ids, tw = _scatter_run(h, nw, gate, T, True)
    same_bits(ids, ids_r, f"{what}: topk_ids vs moe_router")
    same_bits(tw, tw_r, f"{what}: topk_w vs moe_router")
    want_cnt = torch.bincount(ids.reshape(-1).long(), minlength=E)
    assert cnt.tolist() == want_cnt.tolist(), f"{what}: counts {cnt.tolist()} vs {want_cnt.tolist()}"
    if regime == "same pair":
        assert ids.long().eq(torch.tensor(RC.SAME_PAIR, device="cuda")).all(), f"{what}: a token left the pair"
        assert sorted(cnt.tolist())[-2:] == [T, T], f"{what}: counts {cnt.tolist()}"
    assert torch.equal(p // T, ids.long()), f"{what}: perm_row // capacity is not the expert"
    assert p.unique().numel() == 2 * T, f"{what}: a row is claimed twice"
    assert ((p % T) < cnt.long()[ids.long()]).all(), f"{what}: a claimed row lies past its expert's count"
    for k in (0, 1):
        same_bits(xs[p[:, k]], xn, f"{what}: slot rows of choice {k} vs the router's xn")
    same_bits(rw[p], tw, f"{what}: row_weight at the claimed rows vs topk_w")
    claimed = torch.zeros(E * T, dtype=torch.bool, device="cuda")
    claimed[p.reshape(-1)] = True
    assert _is_canary(xs[~claimed]).all(), f"{what}: an unclaimed slot row changed"
    assert _is_canary(rw[~claimed]).all(), f"{what}: an unclaimed row_weight changed"
    # without topk outputs (the expert-parallel form): the same per-token rows and weights, wherever they landed
    xs2, cnt2, p2, rw2, _, _ = _scatter_run(h, nw, gate, T, False)
    assert cnt2.tolist() == cnt.tolist() and torch.equal(p2 // T, p // T), f"{what}: topk_ids = None moves tokens"
    same_bits(xs2[p2], xs[p], f"{what}: slot rows with topk_ids = None")
    same_bits(rw2[p2], rw[p], f"{what}: row weights with topk_ids = None")


@pytest.mark.parametrize("regime", ["random", "crafted"])
@pytest.mark.parametrize("H", RC.ROUTER_H)
def test_router_batch_invariance(H, regime):
    """tokens of a T = 4600 launch: the same bits alone (T = 1), and from moe_route_scatter (capacity T + 5)"""
    T = 4600
    h, nw, gate, names = _cached(RC.router_case, T, H, regime)
    h, nw, gate = h.cuda(), nw.cuda(), gate.cuda()
    xn, ids, tw = _router_run(h, nw, gate)
    picks = sorted({t for t, n in enumerate(names) if n != "randn"} | set(range(0, T, 233)) | {T - 1})
    for t in picks:
        x1, i1, w1 = _router_run(h[t:t + 1], nw, gate)
        tag = f"router H={H} {regime}: token {t} ({names[t]}) alone vs in a batch of {T}"
        same_bits(x1[0], xn[t], f"{tag}: xn")
        same_bits(i1[0], ids[t], f"{tag}: ids")
        same_bits(w1[0], tw[t], f"{tag}: weights")
    xs, _, p, _, ids2, tw2 = _scatter_run(h, nw, gate, T + 5, True)
    same_bits(ids2, ids, f"router H={H} {regime}: moe_route_scatter ids vs moe_router")
    same_bits(tw2, tw, f"router H={H} {regime}: moe_route_scatter weights vs moe_router")
    same_bits(xs[p[:, 0]], xn, f"router H={H} {regime}: moe_route_scatter rows vs moe_router xn")


# ================================================================================================ D. combine
def _perm_rows(layout, T, H, ids):
    """perm_row [T, 2] int32 of the layout and the number of expert-output rows it addresses"""
    from vita_b200 import ops
    if layout == "dense":
        i32 = lambda n: torch.empty(n, dtype=torch.int32, device="cuda")
        offs, perm, rtok = i32(E + 1), i32(2 * T), i32(2 * T)
        rw = torch.empty(2 * T, device="cuda")
        ops.moe_align(ids.cuda(), torch.rand(T, 2, device="cuda"), offs, perm, rtok, rw, T, E)
        return perm, 2 * T
    cap = T + 5
    h, nw, gate, _ = _cached(RC.router_case, T, H, "random")
    _, _, p, _, _, _ = _scatter_run(h.cuda(), nw.cuda(), gate.cuda(), cap, False)
    return p.to(torch.int32).reshape(-1).contiguous(), E * cap


@pytest.mark.parametrize("layout", ["dense", "slots"])
@pytest.mark.parametrize("T", RC.COMBINE_T)
@pytest.mark.parametrize("H", RC.COMBINE_H)
def test_moe_combine(H, T, layout):
    from vita_b200 import ops
    h, y0, y1, ids, kinds = _cached(RC.combine_case, T, H)
    h, y0, y1 = h.cuda(), y0.cuda(), y1.cuda()
    perm, rows = _perm_rows(layout, T, H, ids)
    p = perm.view(T, 2).long()
    y = _canary((rows, H))                       # rows no token points at stay NaN: the kernel must not read them
    y[p[:, 0]] = y0
    y[p[:, 1]] = y1
    g = torch.Generator().manual_seed(H + T)
    nw = ((torch.randint(0, 2, (H,), generator=g) * 2 - 1) * (0.25 + torch.rand(H, generator=g))).to(BF16).cuda()
    want_h = h.double() + y0.double() + y1.double()
    label = lambda i: f"token {i[0]} ({kinds[i[0]]})"
    res = {}
    for norm in ("next norm", "no norm"):
        for rep in range(2):
            what = f"combine H={H} T={T} {layout}, {norm}"
            hb, hv = _padded(T, H)
            hv.copy_(h)
            xb, xv = _padded(T, H)
            ops.moe_combine(hv, y, perm, nw if norm == "next norm" else None, xv, EPS)
            torch.cuda.synchronize()
            _untouched(hb, slice(1, T + 1), f"{what}: h")
            if norm == "no norm":
                assert _is_canary(xb).all(), f"{what}: xn_out was written without a norm weight"
            else:
                _untouched(xb, slice(1, T + 1), f"{what}: xn_out")
            if rep == 1:
                same_bits(hv, res[norm][0], f"{what}: h, second launch")
                same_bits(xv, res[norm][1], f"{what}: xn, second launch")
            res[norm] = (hv.clone(), xv.clone())
        # one rounding of the exact fp32 sum to bf16: 2^-9 of the row's largest value, with a factor of 2
        _note("D combine h", _close(res[norm][0], want_h, f"{what}: h", label, rel=2.0 ** -8))
    same_bits(res["no norm"][0], res["next norm"][0], f"combine H={H} T={T} {layout}: h without the norm")
    hk = res["next norm"][0]
    _note("D combine xn", _close(res["next norm"][1], RC.rms_ref(hk, nw, EPS), f"combine H={H} T={T} {layout}: xn",
                                 label))


# ================================================================================================ E. splice and encoder glue
def test_row_copy_embedding_splice():
    """embedding rows of a [51760, 4096] table into a permuted destination: ids 0 and 51759, placeholders -200 / -500
    skipped (their destination rows keep the canary)"""
    from vita_b200 import ops
    V, H, n = 51760, 4096, 4600
    g = torch.Generator(device="cuda").manual_seed(61)
    table = torch.randn(V, H, device="cuda", generator=g).to(BF16)
    src = torch.randint(0, V, (n,), device="cuda", generator=g, dtype=torch.int32)
    src[0], src[1], src[7::97], src[11::97] = 0, V - 1, -200, -500
    dst = torch.randperm(n, device="cuda", generator=g).to(torch.int32)
    buf, out = _padded(n, H)
    ops.row_copy(table, src, dst, out, n)
    torch.cuda.synchronize()
    live = src >= 0
    d = dst.long() + 1
    same_bits(buf[d[live]], table[src[live].long()], "row_copy: copied rows")
    _untouched(buf, d[live], "row_copy: placeholder rows and padding")


def test_row_copy_grid_stride():
    """more rows than the grid's 65535 * 16 CTAs: the grid-stride loop copies the rest"""
    from vita_b200 import ops
    n, H = 65535 * 16 + 1001, 8
    g = torch.Generator(device="cuda").manual_seed(62)
    table = torch.randn(n, H, device="cuda", generator=g).to(BF16)
    src = torch.randperm(n, device="cuda", generator=g).to(torch.int32)
    buf, out = _padded(n, H)
    ops.row_copy(table, src, None, out, n)
    torch.cuda.synchronize()
    _untouched(buf, slice(1, n + 1), "row_copy grid stride")
    same_bits(out, table[src.long()], "row_copy grid stride")


def test_vit_im2col_448():
    """13 tiles of 448 x 448 px, 14 px patches, rows padded from 588 to the config's 592 columns with zeros"""
    from vita_b200 import ops
    from vita_b200.config import VisionConfig
    v = VisionConfig()
    P, HW, n, k_pad = v.patch_size, v.image_size, 13, v.patch_k_pad
    assert (P, HW, k_pad) == (14, 448, 592)
    img = torch.randn(n, 3, HW, HW, generator=torch.Generator().manual_seed(63)).to(BF16)
    rows = n * (HW // P) ** 2
    buf, col = _padded(rows, k_pad)
    ops.vit_im2col(img.cuda(), col, P, k_pad)
    torch.cuda.synchronize()
    _untouched(buf, slice(1, rows + 1), "vit_im2col")
    want = torch.nn.functional.unfold(img.float(), P, stride=P).transpose(1, 2).reshape(rows, 3 * P * P)
    same_bits(col[:, :3 * P * P].cpu(), want.to(BF16), "vit_im2col: patches")
    assert not col[:, 3 * P * P:].float().any(), "vit_im2col: padding columns are not zero"


def test_vit_assemble_and_pixel_shuffle():
    """cat([cls, patches]) + pos at 1024 + 1 tokens, H = 1024 (one fp32 add, rounded once: the bits of torch's bf16
    add); pixel shuffle of the 32 x 32 grid at C = 1024 with the x0.5 scale (exact)"""
    from oracle import vita_oracle as O
    from vita_b200 import ops
    n, g, H = 2, 32, 1024
    gen = torch.Generator().manual_seed(64)
    patches, cls = torch.randn(n * g * g, H, generator=gen).to(BF16), torch.randn(H, generator=gen).to(BF16)
    pos = torch.randn(g * g + 1, H, generator=gen).to(BF16)
    buf, out = _padded(n * (g * g + 1), H)
    ops.vit_assemble(patches.cuda(), cls.cuda(), pos.cuda(), out, n, g * g, H)
    torch.cuda.synchronize()
    _untouched(buf, slice(1, n * (g * g + 1) + 1), "vit_assemble")
    want = (torch.cat([cls.expand(n, 1, H), patches.view(n, g * g, H)], 1).float() + pos.float()).to(BF16)
    same_bits(out.view(n, g * g + 1, H).cpu(), want, "vit_assemble")
    hfull = torch.randn(n, g * g + 1, H, generator=gen).to(BF16)
    rows = n * (g // 2) ** 2
    buf, ps = _padded(rows, 4 * H)
    ops.vit_pixel_shuffle(hfull.cuda(), ps, n, g, H, 0.5)
    torch.cuda.synchronize()
    _untouched(buf, slice(1, rows + 1), "vit_pixel_shuffle")
    want = O.pixel_shuffle(hfull[:, 1:].float().reshape(n, g, g, H) * 0.5).reshape(rows, 4 * H).to(BF16)
    same_bits(ps.cpu(), want, "vit_pixel_shuffle")


WHALE_T, WHALE_F, WHALE_C = 998, 80, 1024


def test_whale_conv1_against_fp64():
    """GlobalCMVN + Conv2d(1, 1024, 3, 2) + ReLU at T = 998 frames of 80 bins, per output row (b, t1, f1)"""
    from vita_b200 import ops
    B, T, F, C = 2, WHALE_T, WHALE_F, WHALE_C
    gen = torch.Generator().manual_seed(65)
    feat = torch.randn(B, T, F, generator=gen) * 3 + 1
    mean, istd = torch.randn(F, generator=gen), 0.5 + torch.rand(F, generator=gen)
    w, b = (torch.randn(C, 9, generator=gen) * 0.3).to(BF16), (torch.randn(C, generator=gen) * 0.1).to(BF16)
    T1, F1 = (T - 1) // 2, (F - 1) // 2
    buf, out = _padded(B * T1, F1, C)
    ops.whale_conv1(feat.cuda(), mean.cuda(), istd.cuda(), w.cuda(), b.cuda(), out)
    torch.cuda.synchronize()
    _untouched(buf, slice(1, B * T1 + 1), "whale_conv1")
    xin = ((feat - mean) * istd).to(BF16).double().unsqueeze(1)              # the bf16 cast of the normalised input
    ref = torch.nn.functional.conv2d(xin, w.double().view(C, 1, 3, 3), b.double(), stride=2).clamp_min(0)
    ref = ref.permute(0, 2, 3, 1).reshape(B * T1 * F1, C)
    _note("E whale conv1", _close(out.reshape(B * T1 * F1, C), ref, "whale_conv1",
                                  lambda i: f"(b, t1, f1) = {divmod(i[0], T1 * F1)[0]}, {divmod(i[0] % (T1 * F1), F1)}"))


def test_whale_im2col2_and_adapter_im2col():
    """Conv2d(C, C, 3, 2) im2col on the [B, 498, 39, 1024] map; the adapter's Conv1d(k = 5, stride 2) im2col with
    lengths {T2, 1, 0}: frames past a length are zero"""
    from vita_b200 import ops
    B, C = 2, WHALE_C
    T1, F1 = (WHALE_T - 1) // 2, (WHALE_F - 1) // 2
    T2, F2 = (T1 - 1) // 2, (F1 - 1) // 2
    gen = torch.Generator().manual_seed(66)
    x1 = torch.randn(B, T1, F1, C, generator=gen).to(BF16)
    rows = B * T2 * F2
    buf, col = _padded(rows, 9 * C)
    ops.whale_im2col2(x1.cuda(), col, B, T1, F1, C)
    torch.cuda.synchronize()
    _untouched(buf, slice(1, rows + 1), "whale_im2col2")
    pat = x1.unfold(1, 3, 2).unfold(2, 3, 2)                                 # [B, T2, F2, C, kt, kf]
    want = pat.permute(0, 1, 2, 4, 5, 3).reshape(rows, 9 * C)
    same_bits(col.cpu(), want, "whale_im2col2")

    k, nb = 5, 3
    x = torch.randn(nb, T2, C, generator=gen).to(BF16)
    lens = torch.tensor([T2, 1, 0], dtype=torch.int32)
    T3 = (T2 - 1) // 2 + 1
    buf, colA = _padded(nb * T3, k * C)
    ops.whale_adapter_im2col(x.cuda(), lens.cuda(), colA, nb, T2, C, k)
    torch.cuda.synchronize()
    _untouched(buf, slice(1, nb * T3 + 1), "whale_adapter_im2col")
    xm = x.clone()
    for b_, n_ in enumerate(lens.tolist()):
        xm[b_, n_:] = 0
    xp = torch.cat([xm, torch.zeros(nb, k - 1, C, dtype=BF16)], 1)         # right pad k - 1 zero frames
    want = xp.unfold(1, k, 2).permute(0, 1, 3, 2).reshape(nb * T3, k * C)
    same_bits(colA.cpu(), want, "whale_adapter_im2col")


def test_whale_qk_prep_16_heads():
    """[q + u | q + v] (one fp32 add each, rounded once) and [k | p] (copies) for 16 heads x 64, 6 x 248 rows"""
    from vita_b200 import ops
    B, T, heads, dk = 6, 248, 16, 64
    C = heads * dk
    gen = torch.Generator().manual_seed(67)
    qkv, p = torch.randn(B * T, 3 * C, generator=gen).to(BF16), torch.randn(T, C, generator=gen).to(BF16)
    bu, bv = (torch.randn(C, generator=gen) * 0.2).to(BF16), (torch.randn(C, generator=gen) * 0.2).to(BF16)
    qb, q2 = _padded(B * T, heads, 2 * dk)
    kb, k2 = _padded(B * T, heads, 2 * dk)
    ops.whale_qk_prep(qkv.cuda(), p.cuda(), bu.cuda(), bv.cuda(), q2, k2, B, T, heads, dk)
    torch.cuda.synchronize()
    for buf, name in ((qb, "q2"), (kb, "k2")):
        _untouched(buf, slice(1, B * T + 1), f"whale_qk_prep {name}")
    q = qkv[:, :C].float().view(B * T, heads, dk)
    want_q = torch.cat([q + bu.float().view(heads, dk), q + bv.float().view(heads, dk)], -1).to(BF16)
    want_k = torch.cat([qkv[:, C:2 * C].view(B * T, heads, dk), p.repeat(B, 1).view(B * T, heads, dk)], -1)
    same_bits(q2.cpu(), want_q, "whale_qk_prep q2")
    same_bits(k2.cpu(), want_k, "whale_qk_prep k2")
