"""CPU checks of the sampler test inputs (tests/sample_cases.py): each crafted row is where it claims to be, so that
tests/test_sample_shapes_gpu.py tests what it says it tests.  No GPU."""
import numpy as np
import pytest
import torch

from oracle import sampling_oracle as SO
from tests import sample_cases as C


def test_key_map_matches_the_value_order():
    bits = np.arange(1 << 16, dtype=np.uint32)
    keys = C.bf16_key(bits)
    assert np.array_equal(np.sort(keys), bits)                               # a bijection on 16 bits
    vals = torch.from_numpy((bits << 16).view(np.float32)).numpy()
    fin = np.isfinite(vals)
    order = np.argsort(keys[fin])
    assert np.all(np.diff(vals[fin][order].astype(np.float64)) >= 0)         # key order = value order
    assert np.array_equal(C.key_value(keys).view(np.uint32), bits << 16)    # and back
    assert C.bf16_key(0x8000) == 0x7FFF and C.bf16_key(0x0000) == 0x8000     # -0.0 just below +0.0
    assert C.canon_key(0x7FFF) == 0x8000
    assert C.bf16_key(0xFF80) == 0x007F and C.bf16_key(0x7F80) == 0xFF80     # -inf, +inf
    assert C.bf16_key(0x7FC0) > C.bf16_key(0x7F80)                           # a NaN sorts above +inf (the canary)
    row = np.array([1.0, -0.0, 0.0, -2.5], dtype=np.float32)
    assert C.pack_word(row, 1) == C.pack_word(row, 2) + 1                    # equal values, index breaks the tie


@pytest.mark.parametrize("case", C.topk_cases(), ids=lambda c: c.name)
def test_topk_placements(case):
    keys = C.keys_of(case.row)
    thr = case.meta["thr_key"]
    k = case.k
    if k >= case.V:
        return                                                               # top-k is off
    kth = int(np.sort(keys)[::-1][k - 1])
    assert kth == thr, (hex(kth), hex(thr))
    assert (keys == thr - 1).any()                                           # the next key down is populated
    n_above, n_tie = int((keys > thr).sum()), int((keys == thr).sum())
    assert n_above < k <= n_above + n_tie
    if case.meta["tie"] > 1 and 3 <= k <= case.V - 3:
        assert n_above < k - 1 and n_above + n_tie > k                       # the tie group straddles k
    if case.name.startswith("topbin"):
        assert keys.max() >> 8 == thr >> 8
    assert np.all((keys >= C.KEY_FINITE[0]) & (keys <= C.KEY_FINITE[1]))
    _, kept, _ = case.warp()
    assert np.array_equal(kept, keys >= thr)


@pytest.mark.parametrize("case", C.topp_cases(), ids=lambda c: c.name)
def test_topp_placements(case):
    x, kept, dist = case.warp()
    assert not C.topp_exempt(case).any()                                    # every token is compared exactly
    keys = C.canon_key(C.keys_of(case.row))
    low = int(keys[kept].min())
    if "thr_key" in case.meta:
        assert low == case.meta["thr_key"]
        surv = keys[C.survivors(case.row, case.k)]
        hb = low >> 8
        if C.f32(case.p) <= 0.999:                                           # both passes in play
            assert ((surv >> 8 == hb) & (surv > low)).any() or low & 0xFF == 0xFF
            assert ((surv >> 8 == hb) & (surv < low)).any() or low & 0xFF == 0
    if "floor_key" in case.meta:
        f = case.meta["floor_key"]
        assert int(np.sort(keys)[::-1][case.k - 1]) == f                    # the k-th largest is the floor
        _, kept_all, _ = SO.warp(case.row.astype(np.float64), C.f32(case.T), 0, C.f32(case.p))
        assert f >> 8 == int(C.canon_key(C.keys_of(case.row[kept_all])).min()) >> 8
        # the floor changes the top-p decision: top-p over all tokens would keep more, top-k alone more again
        assert kept.sum() < (kept_all & (keys >= f)).sum() or kept.sum() < (keys >= f).sum()
    if C.f32(case.p) < 1e-5:
        assert np.array_equal(kept, case.row == case.row.max())
        assert C.topp_exempt(case).sum() == 0


def test_topp_tolerance_is_small():
    for case in C.topp_cases():
        above, surv = C.above_mass(case.row, case.T, case.k)
        tol = C.topp_tol(case.row, case.T, case.k, above)
        assert tol.max() < 1e-4, (case.name, tol.max())


@pytest.mark.parametrize("case", C.zeros_cases(), ids=lambda c: c.name)
def test_zeros_kept_together(case):
    x, kept, _ = case.warp()
    z = case.row == 0
    assert np.signbit(case.row[z]).any() and (~np.signbit(case.row[z])).any()
    assert kept[z].all() or not kept[z].any()                                # one value, one decision
    if case.name.startswith("topk"):
        assert kept[z].all()
    if "split" in case.name:
        # the bug this row catches: the mass above zero is < p * Z but that plus the +0.0 tokens' mass is not
        above, surv = C.above_mass(case.row, case.T, case.k)
        assert kept[z].all()
        zi = np.flatnonzero(z)
        a0 = above[zi[0]]
        xs = case.row[surv].astype(np.float64)
        u = np.exp(-xs.max()) / np.exp(xs - xs.max()).sum()
        assert a0 < C.f32(case.p) <= a0 + 6 * u
    assert not C.topp_exempt(case).any()


@pytest.mark.parametrize("case", [c for c in C.zeros_cases() if c.name.startswith(("topk", "topp-inside"))],
                         ids=lambda c: c.name)
def test_zeros_rows_agree_with_transformers(case):
    """HF's warpers agree with the oracle on these rows: TopK removes only logits strictly below the k-th largest, and
    the "inside" top-p rows keep the whole zero group even with the group's members taken one by one in sort order
    (HF's top-p is not tie-aware, so on the "split" rows it splits the group: it is no reference there)."""
    from transformers import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = torch.from_numpy(case.row.astype(np.float32))[None]
    ids = torch.zeros(1, 1, dtype=torch.long)
    s = TemperatureLogitsWarper(C.f32(case.T))(ids, s)
    if 0 < case.k < case.V:
        s = TopKLogitsWarper(case.k)(ids, s)
    if C.f32(case.p) < 1.0:
        s = TopPLogitsWarper(C.f32(case.p))(ids, s)
    _, kept, _ = case.warp()
    assert np.array_equal(torch.isfinite(s[0]).numpy(), kept)


def test_division_rows():
    """the division rows hold logits where l * (1 / T) and l / T round to different bf16 values"""
    for case in C.division_cases():
        sens = case.meta["sensitive"]
        assert sens.size >= 20
        t = np.float32(case.T)
        a = torch.from_numpy(case.row / t).to(torch.bfloat16).view(torch.int16)
        b = torch.from_numpy(case.row * (np.float32(1) / t)).to(torch.bfloat16).view(torch.int16)
        assert int((a != b).sum()) >= 8 * sens.size
        for T in C.T_SAMPLED:
            assert C.division_sensitive(T).size == 0


def test_masked_rows():
    for case in C.masked_cases():
        fin = np.isfinite(case.row)
        assert fin.sum() == 96 and (~fin).sum() == case.V - 96
        _, kept, _ = case.warp()
        if 96 < case.k < case.V and C.f32(case.p) >= 1.0:
            assert kept.all()                                                # top-k reaches the -inf group
        assert not C.topp_exempt(case).any()


def test_prune_draws():
    for case in C.prune_cases():
        d = case.meta["d"]
        l = case.row.astype(np.float64)
        assert l[0] == l.max() and np.all((l[1:] == l[0] - d) | (l[1:] == l[0] - 24.5))
        assert (l == l[0] - 24.5).any()
        tok, gap = C.draw(case, np.ones(case.V, dtype=bool))
        assert tok != 0 and l[tok] == l[0] - d
        assert gap > C.draw_tol(case)
        assert SO.choose(l, 1.0, 0, 1.0, case.seed, case.n)[0] == tok


def test_topn_tie_rows():
    for case in C.topn_cases():
        N, ties = case.meta["N"], case.meta["ties"]
        l = case.row.astype(np.float64)
        assert sorted({int(i) // C.CHUNK for i in ties}) == list(C.TIE_CHUNKS) and ties[-1] == case.V - 1
        assert np.all(l[ties] == l[ties[0]])
        nth = np.sort(l)[::-1][N - 1]
        assert nth == l[ties[0]]                                             # the N-th largest is the tie value
        n_above = int((l > nth).sum())
        assert n_above + ties.size > N
        if N > 1:
            assert int((ties < C.CHUNK).sum()) < N - n_above                 # chunk 0 alone cannot fill top-N
        if "zeros" in case.name:
            assert np.signbit(case.row[ties]).any() and (~np.signbit(case.row[ties])).any()
