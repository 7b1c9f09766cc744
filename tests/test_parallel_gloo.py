"""world_size-2 gloo test of the request-parallel plumbing (the N>1 path of bench.py / serving)."""
import os
import socket

import torch
import torch.multiprocessing as mp


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE=str(world), RANK=str(rank),
                      LOCAL_RANK=str(rank))
    from vita_b200 import parallel
    w, r, _ = parallel.init("gloo")
    assert (w, r) == (world, rank)
    owned = parallel.shard_requests(5, rank, world)
    toks = [[100 * i + k for k in range(i + 1)] for i in owned]          # stand-in for generated tokens
    everything = parallel.gather_token_lists(toks, owned, 5)
    tmax = parallel.reduce_max(10.0 + rank)
    tsum = parallel.reduce_sum(float(len(owned)))
    q.put((rank, owned, everything, tmax, tsum))
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


def test_request_sharding_and_reductions_two_ranks():
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert res[0][1] == [0, 2, 4] and res[1][1] == [1, 3]
    want = [[100 * i + k for k in range(i + 1)] for i in range(5)]
    for _, _, everything, tmax, tsum in res:
        assert everything == want
        assert tmax == 11.0 and tsum == 5.0


def test_single_process_degenerates():
    from vita_b200 import parallel
    assert parallel.shard_requests(3, 0, 1) == [0, 1, 2]
    assert parallel.reduce_max(3.5) == 3.5
    assert parallel.gather_token_lists([[1], [2, 3]], [0, 1], 2) == [[1], [2, 3]]


def _ep_worker(rank, world, port, q):
    """Expert-parallel decomposition of the MoE block: the ranks' expert ranges (weights.expert_range) split the
    experts so that the sum over ranks of the local experts' weighted outputs equals the full MixtralSparseMoeBlock of
    the oracle.  (The expert-parallel prefill sums these rows at each token's owning rank; an all-reduce here stands
    for that exchange.)"""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE=str(world), RANK=str(rank),
                      LOCAL_RANK=str(rank))
    import torch.nn.functional as F
    from oracle import vita_oracle as O
    from vita_b200 import parallel, weights as W
    from vita_b200.config import VitaConfig
    parallel.init("gloo")
    cfg = VitaConfig.tiny()
    state = W.synthetic_state(cfg, 0, parts=("llm",))
    lo, hi = W.expert_range(cfg.llm.num_local_experts, rank, world)
    xn = torch.randn(37, cfg.llm.hidden_size, generator=torch.Generator().manual_seed(5))
    full, top_i, top_v = O.sparse_moe(state, cfg.llm, 0, xn)
    part = torch.zeros_like(xn)
    for e in range(lo, hi):
        tok, kpos = torch.where(top_i == e)
        if tok.numel():
            w1, w3, w2 = O.expert_weights(state, cfg.llm, 0, e)
            y = O.linear(F.silu(O.linear(xn[tok], w1)) * O.linear(xn[tok], w3), w2) * top_v[tok, kpos, None]
            part.index_add_(0, tok, y)
    torch.distributed.all_reduce(part)
    q.put((rank, (lo, hi), float((part - full).abs().max())))
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


def test_expert_parallel_decomposition_two_ranks():
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_ep_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert [r[1] for r in res] == [(0, 4), (4, 8)]
    assert all(r[2] < 1e-5 for r in res)


def _seq_worker(rank, world, port, q):
    """Sequence-sharded expert-parallel decoder layer (MixtralDecoder._prefill_ep_seq), restated with the oracle's
    functions and gloo collectives: own-token qkv + RoPE, all-gathered K/V, causal attention with the chunk's position
    offset, own-token o-proj + router, all-gathered routed rows, local experts over all tokens, rows returned to the
    token owners -> must equal the oracle's full decoder layer on the owner's rows."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE=str(world), RANK=str(rank),
                      LOCAL_RANK=str(rank))
    import torch.distributed as dist
    import torch.nn.functional as F
    from oracle import vita_oracle as O
    from vita_b200 import parallel, weights as W
    from vita_b200.config import VitaConfig
    parallel.init("gloo")
    cfg = VitaConfig.tiny()
    c = cfg.llm
    state = W.synthetic_state(cfg, 0, parts=("llm",))
    S, H = 37, c.hidden_size
    nq, nkv, D = c.num_attention_heads, c.num_key_value_heads, c.head_dim
    h = torch.randn(1, S, H, generator=torch.Generator().manual_seed(9)) * 0.5
    want, _ = O.decoder_layer(state, c, 0, h, torch.arange(S)[None])
    chunk = parallel.sequence_chunk(S, world)
    t0, t1 = parallel.token_range(S, rank, world)
    n = t1 - t0
    p = "model.layers.0."
    ho = h[:, t0:t1]
    x = O.rmsnorm(ho, state[p + "input_layernorm.weight"], c.rms_norm_eps)
    qh = O.linear(x, state[p + "self_attn.q_proj.weight"]).view(1, n, nq, D).transpose(1, 2)
    kh = O.linear(x, state[p + "self_attn.k_proj.weight"]).view(1, n, nkv, D).transpose(1, 2)
    vh = O.linear(x, state[p + "self_attn.v_proj.weight"]).view(1, n, nkv, D).transpose(1, 2)
    cos, sin = O.rope_cos_sin(torch.arange(t0, t1)[None], D, c.rope_theta)
    qh, kh = O.apply_rope(qh, kh, cos, sin)
    # exchange 1: all-gather of the K/V rows (fixed-size chunks, the tail rank pads)
    def gather_rows(t, width):
        pad = torch.zeros(chunk, width)
        pad[:n] = t
        parts = [torch.zeros(chunk, width) for _ in range(world)]
        dist.all_gather(parts, pad)
        return torch.cat(parts)[:S]
    k_all = gather_rows(kh.transpose(1, 2).reshape(n, nkv * D), nkv * D).view(S, nkv, D).transpose(0, 1)[None]
    v_all = gather_rows(vh.transpose(1, 2).reshape(n, nkv * D), nkv * D).view(S, nkv, D).transpose(0, 1)[None]
    kk = k_all[:, :, :t1].repeat_interleave(nq // nkv, dim=1)
    vv = v_all[:, :, :t1].repeat_interleave(nq // nkv, dim=1)
    sc = torch.matmul(qh, kk.transpose(2, 3)) * D ** -0.5
    mask = torch.arange(t1)[None, :] > (t0 + torch.arange(n))[:, None]          # keys <= q_pos0 + row
    attn = F.softmax(sc.masked_fill(mask[None, None], float("-inf")), dim=-1)
    o = torch.matmul(attn, vv).transpose(1, 2).reshape(1, n, nq * D)
    ho = ho + O.linear(o, state[p + "self_attn.o_proj.weight"])
    xn2_own = O.rmsnorm(ho, state[p + "post_attention_layernorm.weight"], c.rms_norm_eps)[0]
    # exchange 2: all-gather of the routed rows; every rank routes all tokens identically
    xn2 = gather_rows(xn2_own, H)
    _, top_v, top_i = O.router_topk(xn2, state[p + "block_sparse_moe.gate.weight"], c.num_experts_per_tok)
    lo, hi = W.expert_range(c.num_local_experts, rank, world)
    part = torch.zeros(world * chunk, H)
    for e in range(lo, hi):
        tok, kpos = torch.where(top_i == e)
        if tok.numel():
            w1, w3, w2 = O.expert_weights(state, c, 0, e)
            y = O.linear(F.silu(O.linear(xn2[tok], w1)) * O.linear(xn2[tok], w3), w2) * top_v[tok, kpos, None]
            part.index_add_(0, tok, y)
    # exchange 3: expert outputs go to the token owners (the fused P2P combine; here an all-reduce + slice)
    dist.all_reduce(part)
    got = ho[0] + part[t0:t1]
    q.put((rank, (t0, t1), float((got - want[0, t0:t1]).abs().max()) if n else 0.0))
    dist.barrier()
    dist.destroy_process_group()


def test_sequence_sharded_expert_parallel_layer_two_ranks():
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_seq_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert [r[1] for r in res] == [(0, 24), (24, 37)]
    assert all(r[2] < 2e-5 for r in res), res


def test_sequence_sharded_expert_parallel_layer_four_ranks():
    """The same decomposition with 4 ranks and S = 37: chunks of 16 tokens, the last rank owns none (the case the
    epoch-keeping branch of MixtralDecoder._prefill_ep_seq exists for) and every rank holds two experts."""
    world, port = 4, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_seq_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=240) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    ranges = [r[1] for r in res]
    assert ranges[0][0] == 0 and ranges[-1][1] == 37 and all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
    assert all(r[2] < 2e-5 for r in res), res


def test_token_ranges_cover_the_sequence():
    from vita_b200 import parallel
    for S in (1, 7, 8, 37, 300, 4096, 4097):
        for world in (1, 2, 4, 8):
            rs = [parallel.token_range(S, r, world) for r in range(world)]
            assert rs[0][0] == 0 and rs[-1][1] == S
            assert all(a[1] == b[0] for a, b in zip(rs, rs[1:]))
            assert all(t0 % 8 == 0 or t0 == S for t0, _ in rs)
