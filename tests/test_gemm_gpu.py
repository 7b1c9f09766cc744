"""wgmma GEMM (vita_gemm_bf16 + grouped MoE variants) against the oracle's `linear` on the same bf16 inputs."""
import pytest
import torch
import torch.nn.functional as F

from tests.util import randn, to_dev, assert_close, bf16_round
from oracle import vita_oracle as O

pytestmark = pytest.mark.gpu


def _run(M, N, K, bias=False, act=0, colscale=False, residual=False, lda_pad=0, seed=0):
    from vita_b200 import ops
    x = randn((M, K + lda_pad), seed, 1.0)
    w = randn((N, K), seed + 1, 0.05)
    b = randn((N,), seed + 2, 0.5) if bias else None
    cs = randn((N,), seed + 3, 1.0) if colscale else None
    r = randn((M, N), seed + 4, 1.0) if residual else None
    xd = to_dev(x)
    xv = xd[:, :K] if lda_pad else xd
    y = ops.linear(xv, to_dev(w), None if b is None else to_dev(b), act, None if cs is None else to_dev(cs),
                   None if r is None else to_dev(r))
    torch.cuda.synchronize()
    ref = O.linear(x[:, :K], w, b)
    if act == 1:
        ref = F.gelu(ref)
    elif act == 2:
        ref = F.relu(ref)
    if cs is not None:
        ref = ref * cs
    if r is not None:
        ref = ref + r
    assert_close(y, ref, what=f"gemm M={M} N={N} K={K} bias={bias} act={act} cs={colscale} res={residual}")


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 256, 128), (256, 512, 256), (300, 520, 200), (1, 128, 64),
                                   (77, 8, 512), (129, 1000, 72)])
def test_gemm_plain_shapes(M, N, K):
    _run(M, N, K)


def test_gemm_epilogues():
    _run(260, 384, 320, bias=True, act=1)
    _run(260, 384, 320, bias=True, act=2)
    _run(260, 392, 320, bias=True, colscale=True, residual=True)
    _run(200, 256, 128, residual=True, lda_pad=64)


def test_gemm_model_shapes():
    _run(1025, 3072, 1024, bias=True)            # InternViT qkv
    _run(512, 6144, 4096)                        # Mixtral qkv, S=512 (BLOCK_N=128 path)
    _run(2048, 4096, 4096, residual=True)        # o_proj with residual (BLOCK_N=256 path)
    _run(256, 4096, 4096, bias=True, act=1)      # projector


def test_gemm_tail_split_shapes(monkeypatch):
    # tiles of the last partial wave are cut along N (gemm_sm90.cu Sched); tile counts as chosen on 132 SMs
    _run(2048, 5120, 512, bias=True)             # 256-wide: 320 tiles = 2 waves + 56 -> pieces of 128 columns
    _run(2048, 2560, 512, bias=True)             # 160 tiles = 1 wave + 28 -> pieces of 64 columns
    _run(2048, 3328, 512, residual=True)         # 208 tiles = 1 wave + 76: too many for a cut, whole tiles
    _run(1025, 3072, 256, bias=True, act=1)      # 108 tiles of 256 columns, one partial wave, ragged last row tile
    _run(4096, 4096, 1024, residual=True)        # o_proj at S=4096: 512 tiles = 3 waves + 116, whole tiles
    monkeypatch.setenv("VITA_B200_GEMM_BN", "128")
    _run(2048, 4352, 512, bias=True)             # 128-wide: 544 tiles = 4 waves + 16 -> pieces of 32 columns


def test_gemm_tail_split_is_bit_identical_to_whole_tiles(monkeypatch):
    import os
    from vita_b200 import ops
    x, w = to_dev(randn((2048, 1024), 5, 1.0)), to_dev(randn((5120, 1024), 6, 0.05))
    monkeypatch.setenv("VITA_B200_GEMM_TAIL_SPLIT", "0")
    whole = ops.linear(x, w).clone()
    monkeypatch.setenv("VITA_B200_GEMM_TAIL_SPLIT", "1")
    cut = ops.linear(x, w)
    torch.cuda.synchronize()
    assert torch.equal(whole, cut)


def test_gemm_many_tiles_persistent():
    # more tiles than SMs -> every CTA loops (smem ring phase wrap across tiles)
    _run(1536, 8192, 512, bias=True)


def _moe_case(H, I, E, counts, seed=0):
    from vita_b200 import ops
    rows = sum(counts)
    offs = torch.tensor([0] + list(torch.tensor(counts).cumsum(0)), dtype=torch.int32)
    x = randn((rows, H), seed, 1.0)
    w13 = randn((E, 2 * I, H), seed + 1, 0.05)
    w2 = randn((E, H, I), seed + 2, 0.05)
    rw = torch.rand(rows, generator=torch.Generator().manual_seed(seed + 3))
    xd, w13d, w2d = to_dev(x), to_dev(w13), to_dev(w2)
    offs_d = offs.cuda()
    act = torch.full((rows, I), float("nan"), dtype=torch.bfloat16, device="cuda")
    ops.moe_gate_up(xd, w13d, act, offs_d, rows)
    y = torch.full((rows, H), float("nan"), dtype=torch.bfloat16, device="cuda")
    ops.moe_down(act, w2d, y, offs_d, rw.cuda(), rows)
    torch.cuda.synchronize()
    ref_act = torch.zeros(rows, I)
    ref_y = torch.zeros(rows, H)
    for e in range(E):
        a, b = int(offs[e]), int(offs[e + 1])
        if a == b:
            continue
        gu = O.linear(x[a:b], w13[e])
        ref_act[a:b] = F.silu(gu[:, :I]) * gu[:, I:]
        ref_y[a:b] = O.linear(bf16_round(ref_act[a:b]), w2[e]) * rw[a:b, None]
    assert_close(act, ref_act, what="moe gate_up silu")
    assert_close(y, ref_y, rel=2.5e-2, what="moe down")


def test_moe_grouped_small():
    _moe_case(512, 1024, 8, [100, 0, 160, 129, 1, 128, 70, 56])


def test_moe_grouped_full_width():
    _moe_case(4096, 14336, 8, [130, 90, 128, 0, 260, 64, 127, 225])


@pytest.mark.parametrize("M,K,n_q,n_kv", [(37, 256, 4, 1), (506, 4096, 32, 8), (300, 512, 3, 2), (4096, 512, 32, 8)])
def test_qkv_gemm_with_rope_and_kv_append_epilogue(M, K, n_q, n_kv):
    """vita_gemm_qkv_rope == vita_gemm_bf16 followed by vita_rope_kv_write, bit for bit (qkv rows and both caches)."""
    from vita_b200 import ops, weights
    D = 128
    N = (n_q + 2 * n_kv) * D
    x, w = to_dev(randn((M, K), 1, 1.0)), to_dev(randn((N, K), 2, 0.05))
    pos = (torch.arange(M, dtype=torch.int32) * 3 % 1000 + 5).cuda()
    page, n_slots = 16, (M + 15) // 16 * 16
    perm = torch.randperm(n_slots // page, generator=torch.Generator().manual_seed(0))
    slots = torch.tensor([int(perm[p // page]) * page + p % page for p in range(M)], dtype=torch.int32).cuda()
    table = weights.rope_table(1024, D, 1e6).cuda()
    kc1 = torch.zeros(n_slots, n_kv, D, dtype=torch.bfloat16, device="cuda"); vc1 = torch.zeros_like(kc1)
    kc2, vc2 = torch.zeros_like(kc1), torch.zeros_like(kc1)
    two = ops.linear(x, w)
    ops.rope_kv_write(two, pos, slots, table, kc1, vc1, n_q, n_kv, D)
    one = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    ops.linear_qkv_rope(x, w, one, pos, slots, table, kc2, vc2, n_q, n_kv, D)
    torch.cuda.synchronize()
    assert torch.equal(one, two)
    assert torch.equal(kc1, kc2) and torch.equal(vc1, vc2)
    # no cache write
    three = torch.empty_like(one)
    ops.linear_qkv_rope(x, w, three, pos, None, table, None, None, n_q, n_kv, D)
    assert torch.equal(three, one)


@pytest.mark.parametrize("T,H,I", [(301, 512, 1024), (1000, 4096, 14336), (16, 4096, 14336)])
def test_fused_router_permute_slot_layout_equals_align_gather_flow(T, H, I):
    """vita_moe_route_scatter + the *_slots grouped GEMMs + combine == router + align + gather + grouped GEMMs + combine,
    bit for bit (the slot layout only moves rows)."""
    from vita_b200 import ops
    E = 8
    dev = "cuda"
    h0 = to_dev(randn((T, H), 1, 1.5))
    nw, gw = to_dev(randn((H,), 2)), to_dev(randn((E, H), 3, 0.05))
    g = torch.Generator(device=dev).manual_seed(4)
    w13 = (torch.randn(E, 2 * I, H, device=dev, generator=g) * 0.03).to(torch.bfloat16)
    w2 = (torch.randn(E, H, I, device=dev, generator=g) * 0.03).to(torch.bfloat16)
    nxt = to_dev(randn((H,), 5))
    i32 = lambda *s: torch.empty(*s, dtype=torch.int32, device=dev)
    bf = lambda *s: torch.empty(*s, dtype=torch.bfloat16, device=dev)
    # (a) align + gather flow
    ha = h0.clone()
    xn, ids, tw = bf(T, H), i32(T, 2), torch.empty(T, 2, device=dev)
    ops.moe_router(ha, nw, gw, xn, ids, tw, 1e-5)
    offs, perm, rtok, rw = i32(E + 1), i32(2 * T), i32(2 * T), torch.empty(2 * T, device=dev)
    ops.moe_align(ids, tw, offs, perm, rtok, rw, T, E)
    xp, act, yp = bf(2 * T, H), bf(2 * T, I), bf(2 * T, H)
    ops.row_copy(xn, rtok, None, xp, 2 * T)
    ops.moe_gate_up(xp, w13, act, offs, 2 * T)
    ops.moe_down(act, w2, yp, offs, rw, 2 * T)
    xa = bf(T, H)
    ops.moe_combine(ha, yp, perm, nxt, xa, 1e-5)
    # (b) fused router + permute over slots (capacity > T, buffers poisoned with NaN)
    cap = T + 5
    hb = h0.clone()
    nanbf = lambda *s: torch.full(s, float("nan"), dtype=torch.bfloat16, device=dev)
    xs, acts, ys = nanbf(E * cap, H), nanbf(E * cap, I), nanbf(E * cap, H)
    cnt, perm2, rws = torch.zeros(E, dtype=torch.int32, device=dev), i32(2 * T), torch.empty(E * cap, device=dev)
    ids2, tw2 = i32(T, 2), torch.empty(T, 2, device=dev)
    ops.moe_route_scatter(hb, nw, gw, xs, cnt, perm2, rws, 1e-5, ids2, tw2)
    assert torch.equal(ids2, ids) and torch.equal(tw2, tw)
    assert cnt.cpu().tolist() == torch.bincount(ids.cpu().reshape(-1).long(), minlength=E).tolist()
    p2 = perm2.view(T, 2).long()
    assert torch.equal(p2 // cap, ids.long())                                  # every row sits in its expert's range
    assert p2.reshape(-1).unique().numel() == 2 * T                            # and no row is claimed twice
    assert torch.equal(xs[p2[:, 0]], xn) and torch.equal(xs[p2[:, 1]], xn)
    assert torch.equal(rws[p2.reshape(-1)].view(T, 2), tw)
    ops.moe_gate_up_slots(xs, w13, acts, cnt, 2 * T)
    ops.moe_down_slots(acts, w2, ys, cnt, rws, 2 * T)
    xb = bf(T, H)
    ops.moe_combine(hb, ys, perm2, nxt, xb, 1e-5)
    torch.cuda.synchronize()
    assert torch.equal(ha, hb) and torch.equal(xa, xb)
