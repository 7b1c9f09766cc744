"""FP8 (e4m3) KV cache on the GPU.

Every kernel that writes the cache must store quantize(bf16 row) (tests/test_kv_fp8.py) and leave every other byte
alone; every kernel that reads it must give the bits of its bf16 twin run on dequantize(cache).  On top of that the
model with an fp8 cache follows the fp32 oracle (oracle/vita_oracle.py, through `quantized_kv_oracle`, whose cached
rows go through the same quantizer) at the tiny config and at the PR1 geometry, and the serving surfaces (graph replay,
the continuous batcher, the vLLM adapter, beam search) agree with the decoder bit for bit.
"""
import contextlib
import math

import pytest
import torch

from tests.test_decode_shapes_gpu import (ATTN_CASES, D, EPS, NKV, NQ, SCALE, _attn_ref, _cpu_randn, _gpu_randn,
                                          _paged_cache, _perm)
from tests.test_kv_fp8 import BF16, FP8, dequantize, qdq, quantize
from tests.util import close_rows, same_bits
from vita_b200 import weights as W
from vita_b200.config import VitaConfig

pytestmark = pytest.mark.gpu

CANARY = 0xA5
SCALE_PAIRS = [(1.0, 1.0), (2.0 ** -3, 0.37), (0.37, 2.0 ** -3)]


@pytest.fixture
def lib_options():
    from vita_b200 import ops
    names = ("attn_tagged", "attn_early")
    before = {n: ops.get_option(n) for n in names}
    yield ops.set_option
    for n, v in before.items():
        ops.set_option(n, v)


def _u8(t):
    return t.view(torch.uint8)


def _check_store(kc16, vc16, kc8, vc8, slots, ks, vs, what):
    """e4m3 bytes at the slots == quantize(bf16 rows); every other byte still the canary"""
    idx = torch.tensor(slots, device="cuda")
    for name, c16, c8, s in (("k", kc16, kc8, ks), ("v", vc16, vc8, vs)):
        want = _u8(quantize(c16[idx].cpu(), s))
        got = _u8(c8[idx]).cpu()
        if not torch.equal(got, want):
            bad = (got != want).nonzero()[0].tolist()
            pytest.fail(f"{what}: {name} byte {bad} is {int(got[tuple(bad)]):#04x}, quantize gives "
                        f"{int(want[tuple(bad)]):#04x} (bf16 {float(c16[idx][tuple(bad)]):.6g}, scale {s})")
        mask = torch.ones(c8.shape[0], dtype=torch.bool, device="cuda")
        mask[idx] = False
        assert (_u8(c8)[mask] == CANARY).all(), f"{what}: {name} cache byte outside the written rows changed"
    sat = [(_u8(c[idx]) & 0x7F == 0x7E).any().item() for c in (kc8, vc8)]
    return any(sat)


# ------------------------------------------------------------------------------------------------ writes
@pytest.mark.parametrize("ks,vs", SCALE_PAIRS)
@pytest.mark.parametrize("M", [5, 300])
def test_gemm_qkv_rope_store(M, ks, vs):
    """prefill (M = 300) and batched-step (M = 5) shapes of the qkv GEMM: q / qkv rows identical to the bf16 path"""
    from vita_b200 import ops
    K, R, page = 512, (NQ + 2 * NKV) * D, 16
    seed = M + int(ks * 100)
    x = _gpu_randn((M, K), seed, 1.0)
    x[::7] = (x[::7].float() * 300).to(BF16)                      # rows whose K / V saturate
    w = _gpu_randn((R, K), seed + 1, 1.0 / math.sqrt(K))
    n_slots = ((M + page - 1) // page + 3) * page
    slots = _perm(n_slots, seed + 2)[:M].tolist()
    pos = torch.randint(0, 4096, (M,), generator=torch.Generator().manual_seed(seed + 3), dtype=torch.int32).cuda()
    sm = torch.tensor(slots, dtype=torch.int32, device="cuda")
    table = W.rope_table(4096, D, 1e6).cuda()
    kc = torch.full((n_slots, NKV, D), 0x7FA5, dtype=torch.int16, device="cuda").view(BF16)
    vc = kc.clone()
    kc8 = torch.full((n_slots, NKV, D), CANARY, dtype=torch.uint8, device="cuda").view(FP8)
    vc8 = kc8.clone()
    out, out8 = (torch.empty(M, R, dtype=BF16, device="cuda") for _ in range(2))
    ops.linear_qkv_rope(x, w, out, pos, sm, table, kc, vc, NQ, NKV, D)
    ops.linear_qkv_rope(x, w, out8, pos, sm, table, kc8, vc8, NQ, NKV, D, ks, vs)
    torch.cuda.synchronize()
    same_bits(out8, out, "qkv rows")
    assert _check_store(kc, vc, kc8, vc8, slots, ks, vs, f"qkv GEMM M={M}"), "no saturating row was stored"


@pytest.mark.parametrize("ks,vs", SCALE_PAIRS)
@pytest.mark.parametrize("B", [1, 4])
def test_tc_qkv_rope_store(B, ks, vs):
    """the bs = 1 chain's qkv GEMV (and its batched form): q identical, one e4m3 slot per row"""
    from vita_b200 import ops
    H, page, R = 512, 16, (NQ + 2 * NKV) * D
    seed = 10 * B + int(ks * 100)
    h = _gpu_randn((B, H), seed, 1.5)
    h[0] = (h[0].float() * 300).to(BF16)                            # rmsnorm undoes the scale: saturate by weight
    nw = _gpu_randn((H,), seed + 1, 1.0)
    w = _gpu_randn((R, H), seed + 2, 1.0 / math.sqrt(H))
    w[NQ * D:NQ * D + 64] *= 400                                    # k head 0, first half: saturates
    table = W.rope_table(4096, D, 1e6).cuda()
    max_pages = 4096 // page
    bt = _perm(B * max_pages, seed + 3).view(B, max_pages).to(torch.int32)
    positions = [0, 15, 16, 4095][:B] if B > 1 else [1000]
    cur = torch.tensor(positions, dtype=torch.int32)
    slots = [int(bt[b, p // page]) * page + p % page for b, p in enumerate(positions)]
    n_slots = B * max_pages * page
    ws = ops.TcWorkspace(B, NQ + 2 * NKV, "cuda")
    kc = torch.full((n_slots, NKV, D), 0x7FA5, dtype=torch.int16, device="cuda").view(BF16)
    vc = kc.clone()
    kc8 = torch.full((n_slots, NKV, D), CANARY, dtype=torch.uint8, device="cuda").view(FP8)
    vc8 = kc8.clone()
    q, q8 = (torch.empty(B, NQ * D, dtype=BF16, device="cuda") for _ in range(2))
    args = (table, cur.cuda(), bt.cuda())
    ops.decode_tc_qkv_rope(h, nw, w, *args, q, kc, vc, ws, NQ, NKV, D, page, EPS)
    ops.decode_tc_qkv_rope(h, nw, w, *args, q8, kc8, vc8, ws, NQ, NKV, D, page, EPS, ks, vs)
    torch.cuda.synchronize()
    assert int(ws.buf.count_nonzero()) == 0
    same_bits(q8, q, "q rows")
    assert _check_store(kc, vc, kc8, vc8, slots, ks, vs, f"qkv GEMV B={B}"), "no saturating row was stored"


def test_rope_kv_write_refuses_fp8():
    from vita_b200 import ops, _lib
    qkv = torch.zeros(1, (NQ + 2 * NKV) * D, dtype=BF16, device="cuda")
    c8 = torch.zeros(16, NKV, D, dtype=FP8, device="cuda")
    pos = torch.zeros(1, dtype=torch.int32, device="cuda")
    with pytest.raises(_lib.VitaB200Error, match="e4m3"):
        ops.rope_kv_write(qkv, pos, pos, W.rope_table(64, D, 1e6).cuda(), c8, c8, NQ, NKV, D)
    with pytest.raises(_lib.VitaB200Error):       # a mixed pair
        ops.linear_qkv_rope(torch.zeros(1, 512, dtype=BF16, device="cuda"),
                            torch.zeros((NQ + 2 * NKV) * D, 512, dtype=BF16, device="cuda"), qkv, pos, pos,
                            W.rope_table(64, D, 1e6).cuda(), c8, torch.zeros(16, NKV, D, dtype=BF16, device="cuda"),
                            NQ, NKV, D)


# ------------------------------------------------------------------------------------------------ decode attention
@pytest.mark.parametrize("splits,page,ctxs", ATTN_CASES,
                         ids=[f"s{s}-p{p}-B{len(c)}-ctx{c[0]}" for s, p, c in ATTN_CASES])
def test_decode_attention_fp8(lib_options, splits, page, ctxs):
    """bits of the bf16 kernel on the dequantized cache, through both merges and both fetch orders; fp64 on the
    dequantized rows within the bf16 bar"""
    from vita_b200 import ops
    B = len(ctxs)
    seed = 7 * splits + page + B
    ks, vs = (0.37, 2.0 ** -3) if seed % 2 else (2.0 ** -3, 0.37)
    bt, kc, vc, krows, vrows = _paged_cache(ctxs, page, seed)       # NaN outside every context
    k8, v8 = quantize(kc, ks), quantize(vc, vs)
    kd, vd = dequantize(k8, ks).cuda(), dequantize(v8, vs).cuda()
    k8, v8 = k8.cuda(), v8.cuda()
    q = _cpu_randn((B, NQ * D), seed + 500).cuda()
    ref = torch.stack([_attn_ref(q[b].cpu().view(NQ, D), qdq(krows[b], ks), qdq(vrows[b], vs)) for b in range(B)])
    bt_d = bt.cuda()
    cur = torch.tensor([c - 1 for c in ctxs], dtype=torch.int32, device="cuda")
    ws = ops.decode_attention_workspace(B, NKV, splits, "cuda")

    def run(kcache, vcache, **kw):
        out = torch.empty(B, NQ * D, dtype=BF16, device="cuda")
        ops.decode_attention(q, kcache, vcache, bt_d, cur, out, ws, NQ, NKV, D, page, splits, SCALE, **kw)
        torch.cuda.synchronize()
        assert int(ws.count_nonzero()) == 0, "workspace not all-zero after the launch"
        return out

    label = lambda i: f"row {i[0]} (ctx {ctxs[i[0]]}), head {i[1]}"
    for tagged in (1, 0):
        lib_options("attn_tagged", tagged)
        path = ops.decode_attention_merge(B, NKV, splits)
        for early in (1, 0):
            lib_options("attn_early", early)
            want = run(kd, vd)
            got = run(k8, v8, k_scale=ks, v_scale=vs)
            same_bits(got, want, f"{path} merge, attn_early {early}: fp8 vs bf16 on dequant(cache)")
        close_rows(got.view(B, NQ, D), ref, f"fp8 decode attention, {path} merge", label)


# ------------------------------------------------------------------------------------------------ paged prefill
@pytest.mark.parametrize("page", [16, 32, 128])
@pytest.mark.parametrize("P", [0, 16, 1000, 4000])
def test_paged_prefill_fp8(P, page):
    """continuations of C = 1, 129, 500 rows after P cached keys over shuffled e4m3 pages: the bits of the bf16 paged
    kernel on dequant(pages); the bytes past each context change nothing"""
    from vita_b200 import ops
    ks, vs = 0.37, 2.0 ** -3
    Cs = [1, 129, 500]
    ctx = [P + c for c in Cs]
    need = [(n + page - 1) // page for n in ctx]
    max_pages = max(need) + 1
    n_pages = sum(need) + 2
    perm = _perm(n_pages, P + page)
    bt = torch.full((len(Cs), max_pages), int(perm[-1]), dtype=torch.int32)
    off = 0
    for i, n in enumerate(need):
        bt[i, :n] = perm[off:off + n]
        off += n
    g = torch.Generator().manual_seed(P)
    k8 = quantize(torch.randn(n_pages * page, NKV, D, generator=g).to(BF16) * 4, ks)
    v8 = quantize(torch.randn(n_pages * page, NKV, D, generator=g).to(BF16) * 4, vs)
    live = torch.zeros(n_pages * page, dtype=torch.bool)
    for i, n in enumerate(ctx):
        t = torch.arange(n)
        live[bt[i, t // page].long() * page + t % page] = True

    def garbage(c, seed):
        c = c.clone()
        junk = torch.randint(0, 256, (int((~live).sum()), NKV, D), generator=torch.Generator().manual_seed(seed),
                             dtype=torch.int32).to(torch.uint8)
        junk[:, :, ::9] = 0x7F                                   # NaN codes among them
        _u8(c)[~live] = junk
        return c

    T = sum(Cs)
    qsl = [0]
    for c in Cs:
        qsl.append(qsl[-1] + c)
    q = _cpu_randn((T, NQ * D), P + 7).cuda()
    plan = ops.PagedPrefill(qsl, ctx, bt.cuda(), page)
    results = []
    for seed in (1, 2):
        kg, vg = garbage(k8, seed), garbage(v8, seed + 10)
        kd, vd = dequantize(kg, ks).cuda(), dequantize(vg, vs).cuda()
        want = torch.empty(T, NQ * D, dtype=BF16, device="cuda")
        got = torch.empty_like(want)
        ops.attention_prefill_paged(q, kd, vd, plan, want, NQ, NKV, D, SCALE)
        ops.attention_prefill_paged(q, kg.cuda(), vg.cuda(), plan, got, NQ, NKV, D, SCALE, ks, vs)
        torch.cuda.synchronize()
        assert torch.isfinite(got.float()).all()
        same_bits(got, want, f"P={P}: fp8 paged prefill vs bf16 on dequant(pages)")
        results.append(got)
    same_bits(results[1], results[0], f"P={P}: bytes past the contexts changed the output")


# ------------------------------------------------------------------------------------------------ model
def _model(cfg, packed, **kw):
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    return VITAMixtralForCausalLM(cfg, packed, "cuda", **kw)


@pytest.fixture(scope="module")
def tiny():
    cfg = VitaConfig.tiny()
    state = W.synthetic_state(cfg, 0, parts=("llm",))
    packed = {"llm": W.pack_llm(state, cfg, "cuda")}
    L = cfg.llm.num_hidden_layers
    ks = [0.37 if l % 2 else 2.0 ** -3 for l in range(L)]
    vs = [2.0 ** -3 if l % 2 else 0.37 for l in range(L)]
    model = _model(cfg, packed, max_batch=4, max_seq_len=512, max_new_tokens=32, kv_cache_dtype="fp8", k_scale=ks,
                   v_scale=vs)
    yield cfg, state, packed, model, ks, vs
    del model
    torch.cuda.empty_cache()


@contextlib.contextmanager
def quantized_kv_oracle(ks, vs, cache=None, slot=0, stats=None):
    """oracle/vita_oracle.py with the fp8 cache's reads, for the duration of the block.  `decoder_layer` (which
    `mixtral_forward`, `greedy_generate` and tests/full_depth.py's StreamedOracle call) is wrapped: a whole prompt (no
    cache yet) attends its own rows as they are; a call that continues a cache (decode steps, chunks) reads every key,
    its own new rows included, as the cache holds it -- the decode kernel and the paged prefill read every key from the
    cache.  The layer arithmetic is the oracle's: only its K (after RoPE) and V outputs are replaced.

    The cached rows are the oracle's own quantize -> dequantize of their bf16 rounding (scales ks[l] / vs[l]), or, with
    `cache` (a PagedKVCache the CUDA path filled for the same tokens), the CUDA path's e4m3 rows at the same positions
    of `slot`, dequantized: "cache-aligned", as tests/full_depth.py aligns the routing.  Rounding to e4m3 is a discrete
    decision: an element whose value sits within bf16 noise of a rounding boundary lands one e4m3 step (6-12 %) apart
    in the two computations, which is quantization noise, not kernel error.  Aligned, the comparison measures the
    arithmetic; `stats` then collects every decision where the CUDA code differs from the oracle's own, with its
    distance to the rounding boundary (relative to the value)."""
    from oracle import vita_oracle as O
    layer, linear, rope = O.decoder_layer, O.linear, O.apply_rope

    def cached(x, l, which, positions, judge):
        """the rows the cache serves for x [B, n_kv, S, D] (K) or [B, S, n_kv * D] (V projection) at positions"""
        s = ks[l] if which == "k" else vs[l]
        if cache is None:
            return qdq(x, s).to(x.dtype)
        pos = positions.reshape(-1).to(cache.slot_map.device)
        c8 = (cache.k if which == "k" else cache.v)[l][cache.slot_map[slot, pos].long()]     # [S, n_kv, D]
        c8 = c8.permute(1, 0, 2)[None] if which == "k" else c8.reshape(1, pos.numel(), -1)
        if judge:
            own = quantize(x, s).view(torch.uint8).to(c8.device)
            cu = c8.view(torch.uint8)
            diff = own != cu
            stats["decisions"] += own.numel()
            stats["differ"] += int(diff.sum())
            if diff.any():
                xs = (x.to(BF16).float() / s).to(c8.device)
                if which == "v":
                    xs = xs.unflatten(-1, (-1, 128))
                    diff = diff.unflatten(-1, (-1, 128))
                    own, cu = own.unflatten(-1, (-1, 128)), cu.unflatten(-1, (-1, 128))
                rowmax = xs.abs().amax(-1, keepdim=True).clamp_min(2.0 ** -9).expand_as(xs)
                a, b = own[diff].view(FP8).float(), cu[diff].view(FP8).float()
                # distance of the value to the midpoint of the two codes, in units of its head row's largest value
                stats["dist"].append(((xs[diff] - (a + b) / 2).abs() / rowmax[diff]).cpu())
        return dequantize(c8, s).to(device=x.device, dtype=x.dtype)

    def quantized_layer(state, lcfg, l, h, positions, past_kv=None, trace=None, route=None):
        judge = stats is not None and route is not None     # decisions are judged where the routing is aligned
        if past_kv is None:
            h, (k, v) = layer(state, lcfg, l, h, positions, None, trace, route)
            B, nkv, S, D_ = v.shape
            vq = cached(v.transpose(1, 2).reshape(B, S, nkv * D_), l, "v", positions, judge)
            return h, (cached(k, l, "k", positions, judge), vq.view(B, S, nkv, D_).transpose(1, 2))
        wv = state[f"model.layers.{l}.self_attn.v_proj.weight"]

        def q_linear(x, w, b=None):
            y = linear(x, w, b)
            return cached(y, l, "v", positions, judge) if w is wv else y

        def q_rope(q, k, cos, sin):
            q, k = rope(q, k, cos, sin)
            return q, cached(k, l, "k", positions, judge)
        O.linear, O.apply_rope = q_linear, q_rope
        try:
            return layer(state, lcfg, l, h, positions, past_kv, trace, route)
        finally:
            O.linear, O.apply_rope = linear, rope

    O.decoder_layer = quantized_layer
    try:
        yield O
    finally:
        O.decoder_layer = layer


def _new_stats():
    return {"decisions": 0, "differ": 0, "dist": []}


def _check_decisions(st, what):
    """the CUDA path's e4m3 codes: where they differ from the oracle's own, the value lies within bf16-level noise
    (relative to its head row) of the midpoint between the two codes: a rounding decision, not a wrong row.  How many
    differ depends on how many elements are small against their row (e4m3 codes are dense near zero), so that count is
    reported, not bounded."""
    frac = st["differ"] / max(1, st["decisions"])
    d = torch.cat(st["dist"]) if st["dist"] else torch.zeros(1)
    p99 = float(d.quantile(0.99)) if d.numel() > 1 else float(d.max())
    print(f"{what}: {st['differ']} of {st['decisions']} e4m3 codes differ from the oracle's ({frac:.4f}), distance "
          f"to the boundary (per head row) p99 {p99:.4f}, max {float(d.max()):.4f}")
    assert p99 < 0.02 and float(d.max()) < 0.0625, (what, frac, p99, float(d.max()))


def _row_errors(got, ref):
    return (got - ref).abs().amax(-1) / ref.abs().amax(-1)


def test_generate_fp8_against_quantized_oracle(tiny):
    cfg, state, _, model, ks, vs = tiny
    ids = torch.randint(0, cfg.llm.vocab_size, (1, 40), generator=torch.Generator().manual_seed(3))
    N = 12
    out = model.generate(ids, max_new_tokens=N, output_scores=True)
    toks = out.sequences[0, ids.shape[1]:].tolist()
    got = torch.cat(list(out.scores)).float().cpu()
    with quantized_kv_oracle(ks, vs) as O:
        _, ref = O.greedy_generate(state, cfg, ids, max_new_tokens=N, teacher=toks)
    ref = ref.float()
    err = _row_errors(got, ref)
    assert float(err.median()) < 3.5e-2 and float(err.max()) < 0.1, f"row errors {err.tolist()}"
    top = ref.topk(2, -1)
    margin = (top.values[:, 0] - top.values[:, 1]) / ref.abs().amax(-1)
    for i, t in enumerate(toks):
        if margin[i] > err[i]:
            assert t == int(top.indices[i, 0]), f"step {i}: {t} vs oracle {int(top.indices[i, 0])}"


def test_chunked_prefill_fp8_against_quantized_oracle(tiny):
    """a prompt prefilled in three chunks: the first attends its own rows, the later ones read every key through the
    cache; every logits row against the oracle with the same reads, aligned on the CUDA path's e4m3 codes and expert
    pairs (tests/full_depth.py's reasoning: both are discrete decisions)"""
    from vita_b200.model.mixtral import MixtralDecoder
    cfg, state, packed, _, ks, vs = tiny
    c = cfg.llm
    llm = MixtralDecoder(c, packed["llm"], "cuda", max_batch=1, max_seq_len=256, max_new_tokens=8,
                         kv_cache_dtype="fp8", k_scale=ks, v_scale=vs)
    ids = torch.randint(0, c.vocab_size, (150,), generator=torch.Generator().manual_seed(12))
    cuts = [0, 40, 97, 150]
    emb = packed["llm"]["embed"][ids.cuda()]
    llm.route_trace = []
    got = torch.cat([llm.prefill(emb[a:b].clone(), slot=0, all_logits=True, start=a, final=b == cuts[-1])
                     for a, b in zip(cuts, cuts[1:])]).float().cpu()
    trace, llm.route_trace = llm.route_trace, None
    L = c.num_hidden_layers
    stats = _new_stats()
    with quantized_kv_oracle(ks, vs, cache=llm.cache, stats=stats) as O:
        e = O._f(state["model.embed_tokens.weight"])[ids][None]
        past, rows = [None] * L, []
        for n, (a, b) in enumerate(zip(cuts, cuts[1:])):
            h, pos = e[:, a:b], torch.arange(a, b)[None]
            for l in range(L):
                h, past[l] = O.decoder_layer(state, c, l, h, pos, past[l], None, {"ids": trace[n * L + l][0].cpu()})
            rows.append(O.linear(O.rmsnorm(h, state["model.norm.weight"], c.rms_norm_eps), state["lm_head.weight"])[0])
    err = _row_errors(got, torch.cat(rows).float())
    assert float(err.median()) < 3.5e-2 and float(err.max()) < 0.1, f"row errors {err.tolist()}"
    _check_decisions(stats, "chunked prefill")


@pytest.fixture(scope="module")
def pr1_fp8():
    """PR1 geometry (oracle/pr1.py: full layer width, 32 / 8 heads, 8 experts, depth 4, routers at scale 1 as the
    any-seed test uses them) with an fp8 cache at vLLM's default scales (1.0; the kernel tests and the tiny-config model
    tests cover other scales)"""
    from oracle import pr1
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = pr1.config()
    state = pr1.build_state(cfg, 1.0)
    L = cfg.llm.num_hidden_layers
    ks = vs = [1.0] * L
    model = VITAMixtralForCausalLM(cfg, {"llm": W.pack_llm(state, cfg, "cuda")}, "cuda", max_seq_len=256,
                                   max_new_tokens=pr1.NEW_TOKENS + 1, kv_cache_dtype="fp8", k_scale=ks, v_scale=vs)
    del state
    yield cfg, model, ks, vs
    del model
    torch.cuda.empty_cache()


@pytest.mark.parametrize("prompt_seed", [0, 1, 2])
def test_pr1_geometry_against_the_routing_aligned_quantized_oracle(pr1_fp8, prompt_seed):
    """fp8 cache at the serving head geometry: prefill + 32 free-running greedy tokens through the bs = 1 chain against
    tests/full_depth.py's routing-aligned fp32 oracle with the fp8 reads, aligned on the CUDA path's e4m3 codes as well,
    at PR1's any-seed bars; the codes themselves are judged against the oracle's own quantization"""
    from oracle import pr1
    from tests.full_depth import check_mixtral
    cfg, model, ks, vs = pr1_fp8
    assert cfg.llm.num_key_value_heads == 8 and cfg.llm.hidden_size == 4096
    ids = pr1.prompt(prompt_seed, cfg.llm.vocab_size)
    emb = model.packed["llm"]["embed"][ids[0].cuda()].contiguous()
    stats = _new_stats()
    with quantized_kv_oracle(ks, vs, cache=model.llm.cache, stats=stats):
        r = check_mixtral(model, emb, n_tokens=pr1.NEW_TOKENS)
    print({k: v for k, v in r.items() if k not in ("oracle_top2_rel_gap",)})
    rows = sorted(r["row_rel_err"])
    assert rows[len(rows) // 2] < 3.5e-2 and rows[-1] < 0.1, r
    assert r["ids_equal_where_decided"] == r["ids_decided"], r
    _check_decisions(stats, f"PR1 seed {prompt_seed}")


def test_graph_replay_equals_eager(tiny):
    cfg, _, _, model, _, _ = tiny
    ids = torch.randint(0, cfg.llm.vocab_size, (1, 70), generator=torch.Generator().manual_seed(4))
    a = model.generate(ids, max_new_tokens=10, output_scores=True, use_graph=True)
    a_scores = [s.clone() for s in a.scores]
    b = model.generate(ids, max_new_tokens=10, output_scores=True, use_graph=False)
    assert torch.equal(a.sequences, b.sequences)
    assert all(torch.equal(x, y) for x, y in zip(a_scores, b.scores))


def test_batcher_equals_solo(tiny):
    from vita_b200.engine import ContinuousBatcher, DecoderEngine, Request
    cfg, _, _, model, _, _ = tiny
    spec = [(0, 40, 12), (1, 300, 8), (2, 9, 10), (3, 130, 6)]

    def requests():
        g = torch.Generator().manual_seed(21)
        return [Request(rid, {"input_ids": torch.randint(0, cfg.llm.vocab_size, (1, plen), generator=g)}, n, None,
                        arrival_step=arr) for rid, (arr, plen, n) in enumerate(spec)]
    eng = DecoderEngine(model)
    together = ContinuousBatcher(eng, 3).run(requests())
    chunked = ContinuousBatcher(eng, 3, prefill_chunk=64).run(requests())
    for r in requests():
        r.arrival_step = 0
        solo = ContinuousBatcher(eng, 1).run([r])
        assert together[r.rid] == solo[r.rid], f"request {r.rid}: batched {together[r.rid]} vs solo {solo[r.rid]}"
    assert len(together) == len(spec) and all(len(chunked[k]) == len(together[k]) for k in together)


def test_adapter_equals_fp8_decoder(tiny):
    """the adapter over engine-owned uint8 pages: a whole prompt, a continuation of cached pages and a decode step of
    two sequences give the fp8 decoder's logits bit for bit"""
    import types
    from vita_b200.model.mixtral import MixtralDecoder
    from vita_b200.vllm_adapter import MixtralForConditionalGeneration, TokenBatch
    cfg, _, packed, _, _, _ = tiny
    c, dev = cfg.llm, torch.device("cuda")
    m = MixtralForConditionalGeneration(cfg, device=dev, packed=packed,
                                        cache_config=types.SimpleNamespace(cache_dtype="fp8", block_size=16))
    llm = MixtralDecoder(c, packed["llm"], dev, max_batch=2, max_seq_len=128, max_new_tokens=8, kv_cache_dtype="fp8")
    cache, bs = llm.cache, llm.cache.page_size
    g = torch.Generator().manual_seed(6)
    prompts = [torch.randint(3, 1900, (n,), generator=g).tolist() for n in (37, 20)]
    embeds = lambda ids: packed["llm"]["embed"][torch.tensor(ids, device=dev)]
    as_engine = lambda: [torch.stack([k.view(torch.uint8), v.view(torch.uint8)]).view(2, -1, bs, c.num_key_value_heads,
                                                                                      c.head_dim)
                         for k, v in zip(cache.k, cache.v)]

    # whole prompt of 37, then a continuation of 21 more rows over its pages
    p = prompts[0]
    want = llm.prefill(embeds(p[:20]), slot=0, all_logits=True)
    kv = [torch.zeros(2, k.shape[0] // bs, bs, c.num_key_value_heads, c.head_dim, dtype=torch.uint8, device=dev)
          for k in cache.k]
    meta = TokenBatch(cache.slot_map[0, :20].contiguous(), cache.block_table[:1], [0, 20], [20])
    got = m.compute_logits(m.forward(torch.tensor(p[:20]), torch.arange(20), kv, meta))
    assert torch.equal(got, want), "prompt logits differ"
    for a, b in zip(kv, as_engine()):
        assert torch.equal(a[:, :b.shape[1]], b), "engine pages differ from the decoder's"
    want = llm.prefill(embeds(p[20:]), slot=0, all_logits=True, start=20)
    meta = TokenBatch(cache.slot_map[0, 20:37].contiguous(), cache.block_table[:1], [0, 17], [37])
    got = m.compute_logits(m.forward(torch.tensor(p[20:]), torch.arange(20, 37), kv, meta))
    assert torch.equal(got, want), "continuation logits differ"

    # one decode step of two sequences
    llm.reset()
    for b, p in enumerate(prompts):
        llm.prefill(embeds(p), slot=b)
    kv = as_engine()
    toks = (0xFFFFFFFF - (llm.best[:2] & 0xFFFFFFFF)).tolist()
    lens = [len(p) for p in prompts]
    meta = TokenBatch(torch.stack([cache.slot_map[b, n] for b, n in enumerate(lens)]), cache.block_table[:2], [0, 1, 2],
                      [n + 1 for n in lens])
    got = m.compute_logits(m.forward(torch.tensor(toks), torch.tensor(lens), kv, meta))
    llm.decode_step_batched(2, use_graph=False)
    assert torch.equal(got, llm.d_logits[:2]), "decode-step logits differ"
    with pytest.raises(ValueError, match="fp8"):
        m.forward(torch.tensor(toks), torch.tensor(lens), [t.view(torch.int16)[..., :64] for t in kv], meta)


def test_beam_search_on_fp8_pages(tiny):
    from vita_b200 import ops
    cfg, _, _, model, _, _ = tiny
    # kv_copy_pages moves e4m3 pages byte for byte
    pages, ps, row = 6, 16, NKV * D
    bufs = [torch.randint(0, 256, (pages * ps, NKV, D), dtype=torch.int32, device="cuda").to(torch.uint8).view(FP8)
            for _ in range(4)]
    before = [_u8(b).clone() for b in bufs]
    base = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device="cuda")
    ops.kv_copy_pages(base, torch.tensor([[1, 4], [3, 0]], dtype=torch.int32, device="cuda"), pages, ps * row)
    torch.cuda.synchronize()
    for b, old in zip(bufs, before):
        want = old.clone().view(pages, ps, NKV, D)
        want[4], want[0] = want[1].clone(), want[3].clone()
        assert torch.equal(_u8(b).view(pages, ps, NKV, D), want)
    # beam search over the model's fp8 pages: graph == eager, and the page table is at rest afterwards
    ids = torch.randint(0, cfg.llm.vocab_size, (1, 33), generator=torch.Generator().manual_seed(9))
    kw = dict(num_beams=3, num_return_sequences=2, max_new_tokens=12, output_scores=True)
    a = model.generate(ids, use_graph=True, **kw)
    b = model.generate(ids, use_graph=False, **kw)
    assert torch.equal(a.sequences, b.sequences) and torch.equal(a.sequences_scores, b.sequences_scores)
    pool = model.llm.cache.pool
    pool.check()
    assert pool.table == pool.static.tolist() and pool.free == [] and all(r == 1 for r in pool.refs)
    assert torch.equal(model.llm.cache.block_table.cpu(), pool.static)
