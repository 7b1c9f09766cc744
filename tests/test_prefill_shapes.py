"""The late-jump inputs of tests/test_prefill_shapes_gpu.py reach the lazy rescale of flash_tc.cu: a host model of the
kernel's per-tile decision (128-key tiles, causal limit, m_new > m_ref + 8 in log2 units) run on the very bits the GPU
tests use.  Runs without a GPU."""
import pytest

from tests import prefill_cases as PC


def _check(q, k, targets, kw, what, need_late):
    bad, late = PC.check_targets(q, k, targets, **kw)
    assert not bad, f"{what}: " + "; ".join(bad[:5])
    if need_late:
        assert late > 0, f"{what}: no target rescales past the first tile"
    deltas = {t[4] for t in targets}
    if need_late:
        assert {7.9, 8.1, 20.0, 60.0} <= deltas | set(PC.STAIRS) and 7.9 in deltas, f"{what}: deltas {sorted(deltas)}"
    return late


@pytest.mark.parametrize("S", PC.MIXTRAL_S)
def test_mixtral_late_jumps_take_the_rescale(S):
    qkv, targets, kw = PC.mixtral_case(S, "late")
    q = qkv[:, :PC.NQ * PC.D].view(S, PC.NQ, PC.D)
    k = qkv[:, PC.NQ * PC.D:(PC.NQ + PC.NKV) * PC.D].view(S, PC.NKV, PC.D)
    _check(q, k, targets, kw, f"mixtral S={S}", S > PC.TILE)
    if S > 3 * PC.TILE:
        names = {t[5] for t in targets}
        assert names == {"tile 1, first key", "middle tile", "window's last key", "last, partial tile", "staircase"} \
            or (S % PC.TILE == 0 and "last, partial tile" not in names), names


@pytest.mark.parametrize("t0,t1", PC.token_ranges())
def test_sharded_late_jumps_take_the_rescale(t0, t1):
    (qkv, kc, _), targets, kw = PC.sharded_case(t0, t1, "late")
    _check(qkv[:, :PC.NQ * PC.D].view(t1 - t0, PC.NQ, PC.D), kc, targets, kw, f"shard [{t0}, {t1})", True)


@pytest.mark.parametrize("B,S", PC.VIT_CASES)
def test_vit_late_jumps_take_the_rescale(B, S):
    qkv, targets, kw = PC.vit_case(B, S, "late")
    H = PC.VIT_H
    for b in range(B):
        q = qkv[b, :, :H].view(S, PC.VIT_NH, PC.VIT_D)
        k = qkv[b, :, H:2 * H].view(S, PC.VIT_NH, PC.VIT_D)
        _check(q, k, targets[b], kw, f"vit B={B} S={S} image {b}", S > PC.TILE)


@pytest.mark.parametrize("T2", PC.WHALE_T2)
def test_whale_late_jumps_take_the_rescale(T2):
    (q2, k2, _, lens), targets, kws = PC.whale_case(T2, "late")
    for b in range(PC.WHALE_B):
        _check(q2[b], k2[b], targets[b], kws[b], f"whale T2={T2} length {lens[b]}", kws[b]["kv_len"] > PC.TILE)


def test_paged_late_jumps_take_the_rescale():
    (q, kv), targets, kws = PC.paged_case("late")
    r0 = 0
    for i, (p, c) in enumerate(PC.PAGED_CASES):
        qv = q[r0:r0 + c, :PC.NQ * PC.D].view(c, PC.NQ, PC.D)
        _check(qv, kv[i][0], targets[i], kws[i], f"paged P={p} C={c}", p + c > PC.TILE)
        r0 += c


def test_model_matches_the_kernel_rule():
    """the rule itself: a rise of 7.9 is absorbed, 8.1 moves the reference, at any tile"""
    import torch
    s = torch.zeros(4 * PC.TILE, dtype=torch.float64)
    s[PC.TILE + 3] = 7.9
    s[2 * PC.TILE] = 8.1 + 0.0
    s[3 * PC.TILE + 5] = 16.3
    moved, before = PC.rescale_tiles(s, s.numel())
    assert moved == [0, 2, 3] and before == [float("-inf"), 0.0, 0.0, 8.1]
    assert PC.rescale_tiles(s, 2 * PC.TILE)[0] == [0]            # the masked tail never counts
