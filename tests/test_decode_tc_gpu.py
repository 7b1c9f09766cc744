"""Decode-step linears on wgmma (swap-AB GEMV, stream-K with tagged partial slots) vs the oracle's functions.
Each kernel is launched twice on the same workspace to exercise the self-clearing slot tags."""
import pytest
import torch
import torch.nn.functional as F

from tests.util import randn, to_dev, assert_close, bf16_round, BF16
from oracle import vita_oracle as O

pytestmark = pytest.mark.gpu


def _gpu_randn(shape, seed, scale):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(BF16)


def _ws(B, rb):
    from vita_b200 import ops
    return ops.TcWorkspace(B, rb, "cuda")


@pytest.mark.parametrize("H,nq,nkv", [(512, 4, 1), (4096, 32, 8)])
def test_tc_qkv_rope(H, nq, nkv):
    from vita_b200 import ops, weights
    B, D, page = 2, 128, 16
    h = randn((B, H), 1, 1.5)
    nw = randn((H,), 2)
    w = _gpu_randn(((nq + 2 * nkv) * D, H), 3, 0.03)
    table = weights.rope_table(256, D, 1e6)
    cur = torch.tensor([37, 5], dtype=torch.int32)
    bt = torch.tensor([[3, 1, 4, 0, 5, 2, 6, 7], [15, 14, 13, 12, 11, 10, 9, 8]], dtype=torch.int32)
    ws = _ws(B, nq + 2 * nkv)
    xn = bf16_round(O.rmsnorm(h, nw, 1e-5))
    qkv = bf16_round(O.linear(xn, w.float().cpu()))
    for rep in range(2):
        q = torch.zeros(B, nq * D, dtype=BF16, device="cuda")
        kc = torch.zeros(16 * page, nkv, D, dtype=BF16, device="cuda")
        vc = torch.zeros_like(kc)
        ops.decode_tc_qkv_rope(to_dev(h), to_dev(nw), w, table.cuda(), cur.cuda(), bt.cuda(), q, kc, vc, ws, nq, nkv,
                               D, page, 1e-5)
        for b in range(B):
            qq = qkv[b, : nq * D].view(1, nq, 1, D)
            kk = qkv[b, nq * D: (nq + nkv) * D].view(1, nkv, 1, D)
            vv = qkv[b, (nq + nkv) * D:].view(nkv, D)
            cos, sin = O.rope_cos_sin(cur[b].view(1, 1).long(), D, 1e6)
            qr, kr = O.apply_rope(qq, kk, cos, sin)
            slot = int(bt[b, int(cur[b]) // page]) * page + int(cur[b]) % page
            assert_close(q[b], qr.reshape(-1), rel=2e-2, what=f"tc decode q (rep {rep})")
            assert_close(kc[slot], kr.reshape(nkv, D), rel=2e-2, what="tc decode k cache")
            assert_close(vc[slot], vv, rel=2e-2, what="tc decode v cache")
        assert int((kc.float().abs().sum(-1).sum(-1) > 0).sum()) == B


@pytest.mark.parametrize("N,K", [(512, 512), (4096, 4096)])
def test_tc_oproj(N, K):
    from vita_b200 import ops
    B = 2
    x, h = randn((B, K), 1), randn((B, N), 2)
    w = _gpu_randn((N, K), 3, 0.03)
    ws = _ws(B, (N + 127) // 128)
    want = h + O.linear(x, w.float().cpu())
    for rep in range(2):
        hd = to_dev(h)
        ops.decode_tc_oproj(to_dev(x), w, hd, ws)
        assert_close(hd, want, rel=1.2e-2, what=f"tc decode oproj (rep {rep})")


@pytest.mark.parametrize("H,I", [(512, 1024), (4096, 14336)])
def test_tc_moe(H, I):
    from vita_b200 import ops
    B, E = 2, 8
    h = randn((B, H), 1, 1.5)
    nw = randn((H,), 2)
    gw = randn((E, H), 3, 0.05)
    w13 = _gpu_randn((E, 2 * I, H), 4, 0.03)
    w2 = _gpu_randn((E, H, I), 5, 0.03)
    ws = _ws(B, max(2 * (I // 128), H // 128))
    xn = O.rmsnorm(h, nw, 1e-5)
    _, top_v, top_i = O.router_topk(xn, gw)
    ref_xn = bf16_round(xn)
    want = h.clone()
    acts = {}
    for b in range(B):
        for k in range(2):
            e = int(top_i[b, k])
            gu = O.linear(ref_xn[b], w13[e].float().cpu())
            acts[(b, k)] = bf16_round(F.silu(gu[:I]) * gu[I:])
            want[b] += top_v[b, k] * O.linear(acts[(b, k)], w2[e].float().cpu())
    for rep in range(2):
        hd = to_dev(h)
        act = torch.empty(B, 2, I, dtype=BF16, device="cuda")
        ids = torch.full((B, 2), -1, dtype=torch.int32, device="cuda")
        tw = torch.zeros(B, 2, dtype=torch.float32, device="cuda")
        ops.decode_tc_moe_gate_up(hd, to_dev(nw), to_dev(gw), w13, ids, tw, act, ws, 1e-5)
        assert torch.equal(ids.cpu().long(), top_i)
        assert (tw.cpu() - top_v).abs().max() < 5e-3
        for (b, k), a in acts.items():
            assert_close(act[b, k], a, rel=2e-2, what=f"tc decode act (rep {rep})")
        ops.decode_tc_moe_down(act, w2, ids, tw, hd, ws)
        assert_close(hd, want, rel=1.5e-2, what=f"tc decode moe out (rep {rep})")


@pytest.mark.parametrize("H,V", [(512, 2047), (4096, 51760)])
def test_tc_lm_head_argmax(H, V):
    from vita_b200 import ops
    B = 2
    hrows = randn((B, 3, H), 1, 1.5)
    nw = randn((H,), 2)
    Vp = (V + 7) // 8 * 8
    w_full = _gpu_randn((Vp, H), 3, 0.03)
    w = w_full[:V]
    hd = to_dev(hrows)
    ws = _ws(B, (V + 127) // 128)
    xn = bf16_round(O.rmsnorm(hrows[:, 2], nw, 1e-5))
    ref = O.linear(xn, w.float().cpu())
    for rep in range(2):
        logits = torch.empty(B, V, dtype=BF16, device="cuda")
        best = torch.zeros(B, dtype=torch.int64, device="cuda")
        ops.tc_lm_head_argmax(hd[:, 2], 3 * H, to_dev(nw), w, logits, best, B, ws, 1e-5)
        assert_close(logits, ref, what=f"tc logits (rep {rep})")
        got_idx = (0xFFFFFFFF - (best.cpu() & 0xFFFFFFFF)).long()
        lg = logits.float().cpu()
        for b in range(B):
            first = int((lg[b] == lg[b].max()).nonzero()[0])
            assert int(got_idx[b]) == first


@pytest.fixture
def tc_options():
    """Sets library tunables for one test and restores the defaults afterwards."""
    from vita_b200 import ops
    names = ("tc_wide_route", "tc_l2_ahead", "tc_trigger_lead", "pdl")
    before = {n: ops.get_option(n) for n in names}
    yield ops.set_option
    for n, v in before.items():
        ops.set_option(n, v)


def _moe_pair(ops, h, nw, gw, w13, w2, ws, I):
    B = h.shape[0]
    hd = h.clone()
    act = torch.empty(B, 2, I, dtype=BF16, device="cuda")
    ids = torch.full((B, 2), -1, dtype=torch.int32, device="cuda")
    tw = torch.zeros(B, 2, dtype=torch.float32, device="cuda")
    ops.decode_tc_moe_gate_up(hd, nw, gw, w13, ids, tw, act, ws, 1e-5)
    ops.decode_tc_moe_down(act, w2, ids, tw, hd, ws)
    return hd, act, ids, tw


def test_tc_tunables_keep_the_bits(tc_options):
    """Programmatic launch, the L2 look-ahead and the trigger placement only move work in time: outputs must be
    bit-identical.  The wide router changes the summation order of the 8 logits, so the narrow one is held to the same
    expert choice and to float tolerance on the weights."""
    from vita_b200 import ops
    B, H, I, E, V = 2, 4096, 14336, 8, 51760
    h = to_dev(randn((B, H), 1, 1.5))
    nw, gw = to_dev(randn((H,), 2)), to_dev(randn((E, H), 3, 0.05))
    w13, w2 = _gpu_randn((E, 2 * I, H), 4, 0.03), _gpu_randn((E, H, I), 5, 0.03)
    wo = _gpu_randn((H, H), 6, 0.03)
    wl = _gpu_randn((V, H), 7, 0.03)
    x = to_dev(randn((B, H), 8))
    ws = _ws(B, max(2 * (I // 128), (V + 127) // 128))

    def run_all():
        out = list(_moe_pair(ops, h, nw, gw, w13, w2, ws, I))
        ho = h.clone()
        ops.decode_tc_oproj(x, wo, ho, ws)
        out.append(ho)
        logits = torch.empty(B, V, dtype=BF16, device="cuda")
        best = torch.zeros(B, dtype=torch.int64, device="cuda")
        ops.tc_lm_head_argmax(h, H, nw, wl, logits, best, B, ws, 1e-5)
        out += [logits, best.clone()]
        return out

    base = run_all()
    for name, value, restore in (("pdl", 0, 1), ("tc_l2_ahead", 6, 0), ("tc_trigger_lead", 3, 0)):
        tc_options(name, value)
        for rep in range(2):
            got = run_all()
            for a, b in zip(base, got):
                assert torch.equal(a, b), f"{name}={value} changed an output (rep {rep})"
        tc_options(name, restore)
    tc_options("tc_wide_route", 0)
    hd, act, ids, tw = _moe_pair(ops, h, nw, gw, w13, w2, ws, I)
    assert torch.equal(ids, base[2])
    assert (tw - base[3]).abs().max() < 1e-5
    assert_close(act, base[1], rel=1e-3, what="narrow-router activations")
    assert_close(hd, base[0], rel=1e-3, what="narrow-router MoE output")


def test_tc_early_route_handover_keeps_the_bits(tc_options):
    """gate|up publishes the expert pair as one tagged word and the down projection streams its rows early: same bits as
    the hand-over through topk_ids, with and without programmatic launch, over consecutive "layers" sharing the word."""
    from vita_b200 import ops
    B, H, I, E = 2, 4096, 14336, 8
    nw, gw = to_dev(randn((H,), 2)), to_dev(randn((E, H), 3, 0.05))
    w13, w2 = _gpu_randn((E, 2 * I, H), 4, 0.03), _gpu_randn((E, H, I), 5, 0.03)
    ws = _ws(B, 2 * (I // 128))
    hs = [to_dev(randn((B, H), 10 + i, 1.5)) for i in range(3)]
    base = [_moe_pair(ops, h, nw, gw, w13, w2, ws, I) for h in hs]
    word = torch.zeros(B, dtype=torch.int64, device="cuda")
    for pdl in (1, 0):
        tc_options("pdl", pdl)
        for rep in range(2):
            for layer, h in enumerate(hs):
                hd = h.clone()
                act = torch.empty(B, 2, I, dtype=BF16, device="cuda")
                ids = torch.full((B, 2), -1, dtype=torch.int32, device="cuda")
                tw = torch.zeros(B, 2, dtype=torch.float32, device="cuda")
                ops.decode_tc_moe_gate_up(hd, nw, gw, w13, ids, tw, act, ws, 1e-5, word, layer + 1)
                ops.decode_tc_moe_down(act, w2, ids, tw, hd, ws, word, layer + 1)
                for a, b in zip(base[layer], (hd, act, ids, tw)):
                    assert torch.equal(a, b), f"early route changed an output (pdl={pdl}, rep {rep}, layer {layer})"
                w = word.cpu().tolist()
                assert [x >> 32 for x in w] == [layer + 1] * B
                assert [[(x >> 8) & 0xff, x & 0xff] for x in w] == ids.cpu().tolist()
    tc_options("pdl", 1)
