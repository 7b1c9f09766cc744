"""The inputs of tests/test_row_shapes_gpu.py do what they claim, checked on the same bits without a GPU: the RoPE table
against fp64, the host model of the qkv GEMM's schedule, norm rows that a one-pass variance gets wrong, crafted router
tokens (exact ties, zero row, dominant logit, near-ties just past the accumulation bound), and combine rows that
cancel."""
import math

import pytest
import torch

from tests import row_cases as RC


def test_rope_table_matches_fp64_angles():
    """weights.rope_table(32768, 128, 1e6) is (cos, sin) of pos * theta^(-2i/128) within what an fp32 inv_freq and an
    fp32 product allow (the pow, the reciprocal and the product round: at most 2^-22 of the angle) plus the fp32
    cos / sin rounding.  A wrong layout, dtype or theta is off by far more."""
    from vita_b200 import weights
    t = weights.rope_table(RC.ROPE_LEN, RC.D, RC.ROPE_THETA)
    assert t.dtype == torch.float32 and t.shape == (RC.ROPE_LEN, 2, RC.D // 2) and t.is_contiguous()
    pos = torch.arange(RC.ROPE_LEN, dtype=torch.float64)[:, None]
    ang = pos * RC.ROPE_THETA ** (-torch.arange(0, RC.D, 2, dtype=torch.float64) / RC.D)
    bound = ang * 2.0 ** -22 + 2.0 ** -22
    for k, f in ((0, torch.cos), (1, torch.sin)):
        err = (t[:, k].double() - f(ang)).abs()
        assert (err <= bound).all(), f"{f.__name__}: worst excess {float((err - bound).max()):.3e}"
    assert float((t[-1, 0].double() - torch.cos(ang[-1])).abs().max()) > 0      # the bound is not vacuous at 32767


def test_qkv_schedule_model():
    """gemm_sm90.cu on 132 SMs: Mixtral's M = 1, 128 and 129 cut their last wave in halves, M = 4600 (864 tiles,
    remainder 72) does not; without the tail split nothing is cut"""
    N = (32 + 2 * 8) * RC.D
    assert RC.qkv_schedule(1, N, 132) == (96, 24, 2)
    assert RC.qkv_schedule(128, N, 132) == (132, 24, 2)
    assert RC.qkv_schedule(129, N, 132) == (132, 48, 2)
    assert RC.qkv_schedule(4600, N, 132) == (132, 864, 1)
    assert all(RC.qkv_schedule(M, N, 132, tail_split=False)[2] == 1 for M in (1, 128, 129, 4600))
    assert RC.qkv_schedule(4600, 7 * RC.D, 132) == (132, 144, 2)       # the 3/2 geometry: last tile holds one head


@pytest.mark.parametrize("kind", ["zero", "end", "perm", "dup"])
def test_qkv_positions(kind):
    for M in (1, 129, 4600):
        p = RC.qkv_positions(kind, M)
        assert p.dtype == torch.int32 and p.shape == (M,) and 0 <= int(p.min()) and int(p.max()) < RC.ROPE_LEN
        if kind == "end":
            assert int(p[-1]) == RC.ROPE_LEN - 1
        if kind == "perm":
            assert p.unique().numel() == M
        if kind == "dup" and M > 1:
            assert p.unique().numel() < M and int(p.max()) == RC.ROPE_LEN - 1


@pytest.mark.parametrize("kind", ["pages 16", "pages 128", "pages 16, holes", "pages 128, holes"])
def test_qkv_slots(kind):
    for M in (1, 129, 4600):
        s, n = RC.qkv_slots(kind, M)
        live = s[s >= 0]
        assert live.unique().numel() == live.numel() and int(live.max()) < n
        assert n - live.numel() >= 2 * (16 if "16" in kind else 128)                  # two spare pages
        assert ("holes" in kind) == bool((s < 0).any()) or M < 4
    assert RC.qkv_slots("none", 5) == (None, 0)


@pytest.mark.parametrize("rows", RC.RMS_ROWS)
def test_rms_rows(rows):
    x, w, e = RC.rms_case(rows, 4096)
    assert (w.float() > 0).any() and (w.float() < 0).any()
    if rows > 2:
        assert int(e.min()) == -40 and int(e.max()) == 40
        assert not x[rows // 2].float().any()
        nz = torch.ones(rows, dtype=torch.bool)
        nz[rows // 2] = False
        m = x[nz].float().abs().amax(-1) / torch.pow(2.0, e[nz].double()).float()
        assert ((m > 0.5) & (m < 8)).all()                 # each row is randn at its scale


def test_layernorm_offset_rows_defeat_a_one_pass_variance():
    """E[x^2] - mean^2 in fp32, summed as the kernel sums, moves 1 / sqrt(var + eps) of some offset row of every case by
    more than the 1.6e-2 tolerance; the two-pass variance is exact to fp32 there.  The constant row has variance 0."""
    for name, H, eps, _, _ in RC.LN_CASES:
        x, _, _, kinds = RC.ln_case(129, H)
        thr, vpt = (128, 1) if H <= 1024 else (256, 4)
        xd = x.double()
        var = ((xd - xd.mean(-1, keepdim=True)) ** 2).mean(-1)
        off = torch.tensor([k.startswith("offset") for k in kinds])
        one = RC.one_pass_var32(x[off], thr, vpt).double()
        rel = ((one + eps).clamp_min(1e-30).rsqrt() / (var[off] + eps).rsqrt() - 1).abs()
        assert float(rel.max()) > 0.1, f"{name}: a one-pass variance is off by at most {float(rel.max()):.3e}"
        assert float(var[kinds.index("constant")]) == 0.0
        assert ((var[off] > 0.007) & (var[off] < 4.1)).all()


def test_router_crafted_tokens():
    """on the host's xn, every crafted token gets its CRAFTED_IDS, is decided, and has the gap it claims"""
    for H in RC.ROUTER_H:
        h, nw, gate, names = RC.router_case(16, H, "crafted")
        assert torch.equal(gate[RC.TIE[0]], gate[RC.TIE[1]])
        assert int((gate[RC.NEAR_A] != gate[RC.NEAR_B]).sum()) == 1
        lg, b = RC.logits64(RC.xn_host(h, nw), gate)
        ids, w, ok = RC.top2_ref(lg, b)
        srt = lg.sort(-1, descending=True).values
        for t, name in enumerate(names):
            if name == "randn":
                continue
            what = f"H={H} {name}"
            if name == "dominant":
                assert int(ids[t, 0]) == RC.DOM and float(srt[t, 0] - srt[t, 1]) > RC.DOMINANT_GAP, what
                assert math.exp(-float(srt[t, 0] - srt[t, 1])) < 2.0 ** -151, what      # rounds to 0 in fp32
                continue
            assert ok[t] and tuple(ids[t].tolist()) == RC.CRAFTED_IDS[name], f"{what}: {ids[t].tolist()}"
            if name.startswith("near-tie"):
                a = 0 if name.endswith("first") else 1
                r = float((srt[t, a] - srt[t, a + 1]) / b[t])
                assert 2.5 < r < 3.5, f"{what}: gap of {r:.3f} bounds"
            if name in ("tie for first", "zero row"):
                assert w[t].tolist() == [0.5, 0.5], what
        assert ok[len(RC.CRAFTED_IDS):].all()


@pytest.mark.parametrize("H", RC.ROUTER_H)
def test_router_random_regime_is_decided(H):
    h, nw, gate, _ = RC.router_case(4600, H, "random")
    lg, b = RC.logits64(RC.xn_host(h, nw), gate)
    _, _, ok = RC.top2_ref(lg, b)
    assert float(ok.double().mean()) >= 0.98


@pytest.mark.parametrize("H", RC.ROUTER_H)
def test_same_pair_tokens_fill_two_experts(H):
    h, nw, gate, _ = RC.router_case(4600, H, "same pair")
    lg, b = RC.logits64(RC.xn_host(h, nw), gate)
    ids, _, ok = RC.top2_ref(lg, b)
    assert ok.all() and (ids == torch.tensor(RC.SAME_PAIR)).all()


def test_logit_bound_covers_the_kernel_sum():
    """39 fp32 roundings (32 in a thread, 5 butterfly levels, 2 over the warps) stay below LOGIT_BOUND"""
    assert 39 * 2.0 ** -24 * (1 + 2.0 ** -20) < RC.LOGIT_BOUND / 6


def test_combine_rows():
    h, y0, y1, ids, kinds = RC.combine_case(129, 4096)
    hd, s = h.double(), (h.double() + y0.double() + y1.double())
    for t, k in enumerate(kinds):
        ratio = float(s[t].abs().max() / hd[t].abs().max())
        if k == "cancel":
            assert ratio < 2.0 ** -4, (t, ratio)
            assert float(y0[t].double().abs().max()) > 0.2 * float(hd[t].abs().max())
        else:
            y = float(torch.maximum(y0[t].double().abs(), y1[t].double().abs()).max() / hd[t].abs().max())
            assert 2.0 ** -11 < y < 2.0 ** -6, (t, y)
    assert (ids[:, 0] != ids[:, 1]).all() and int(ids.min()) >= 0 and int(ids.max()) < RC.E
