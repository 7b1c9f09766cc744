"""Chunked prefill and prefix reuse: the paged-KV FlashAttention variant (vita_attention_prefill_paged) and everything
built on it -- MixtralDecoder.prefill(start, final), the vLLM adapter's continuation sequences, the batcher's chunked
admission.

The bar is bit-identity: the paged kernel runs the consumer code of the contiguous kernel on a byte-identical
shared-memory image, so it must equal ops.attention over the gathered keys; every other prefill kernel works row by
row (no split-K in the GEMMs), so a prompt prefilled in chunks must equal the one-shot prefill."""
import numpy as np
import pytest
import torch

from tests.util import assert_close
from vita_b200 import _lib, ops
from vita_b200 import weights as W
from vita_b200.config import VitaConfig

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
NQ, NKV, D = 32, 8, 128
SCALE = D ** -0.5


# ------------------------------------------------------------------------------------------------ kernel level
def _case_data(cases, seed):
    """Per sequence (P cached + C new): K / V of all P + C keys, and a packed q buffer [T, (NQ + 2 NKV) D] (the qkv
    layout: only the first NQ * D columns are read)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    T = sum(c for _, c in cases)
    q = torch.randn(T, (NQ + 2 * NKV) * D, generator=g, device="cuda").to(BF16)
    kv = [(torch.randn(p + c, NKV, D, generator=g, device="cuda").to(BF16),
           torch.randn(p + c, NKV, D, generator=g, device="cuda").to(BF16)) for p, c in cases]
    return q, kv


def _paged(cases, kv, ps, seed, stale):
    """Shuffled pages.  `stale`: every slot no sequence owns is NaN (the unused tail of each last page included) and
    the unused block-table entries are garbage page ids."""
    g = torch.Generator().manual_seed(seed)
    n_pg = [(p + c + ps - 1) // ps for p, c in cases]
    n_pages = sum(n_pg) + 4
    perm = torch.randperm(n_pages, generator=g).tolist()
    width = max(n_pg) + 3
    table = torch.full((len(cases), width), 0, dtype=torch.int32)
    if stale:
        table.random_(1 << 20, 1 << 30, generator=g)
    fill = float("nan") if stale else 0.0
    kc = torch.full((n_pages * ps, NKV, D), fill, dtype=BF16, device="cuda")
    vc = torch.full_like(kc, fill)
    slots = []
    o = 0
    for i, (p, c) in enumerate(cases):
        pages = perm[o:o + n_pg[i]]
        o += n_pg[i]
        table[i, :n_pg[i]] = torch.tensor(pages, dtype=torch.int32)
        pos = torch.arange(p + c)
        s = (torch.tensor(pages)[pos // ps] * ps + pos % ps).cuda()
        kc[s], vc[s] = kv[i]
        slots.append(s)
    return kc, vc, table.cuda(), slots


def _qsl(cases):
    qsl = [0]
    for _, c in cases:
        qsl.append(qsl[-1] + c)
    return qsl


def _run_paged(q, kc, vc, table, cases, ps, seqs=None):
    qsl = _qsl(cases)
    plan = ops.PagedPrefill(qsl, [p + c for p, c in cases], table, ps, seqs)
    out = torch.zeros(qsl[-1], NQ * D, dtype=BF16, device="cuda")
    ops.attention_prefill_paged(q[:, : NQ * D], kc, vc, plan, out, NQ, NKV, D, SCALE)
    return out


def _run_contiguous(q, kv, cases):
    """ops.attention(Sq = C, Skv = P + C, causal, q_pos0 = P) per sequence over its gathered keys."""
    qsl = _qsl(cases)
    out = torch.zeros(qsl[-1], NQ * D, dtype=BF16, device="cuda")
    for i, (p, c) in enumerate(cases):
        k, v = kv[i]
        ops.attention(q[qsl[i]:qsl[i + 1]], k, v, out[qsl[i]:qsl[i + 1]], (0, q.stride(0), D), (0, NKV * D, D),
                      (0, NKV * D, D), (0, NQ * D, D), 1, NQ, NKV, c, p + c, D, D, None, True, SCALE, q_pos0=p)
    return out


def _fp32(q, k, v, p):
    c = q.shape[0]
    qf = q[:, : NQ * D].float().view(c, NQ, D).transpose(0, 1)                      # [NQ, C, D]
    kf = k.float().repeat_interleave(NQ // NKV, dim=1).transpose(0, 1)            # [NQ, P + C, D]
    vf = v.float().repeat_interleave(NQ // NKV, dim=1).transpose(0, 1)
    s = qf @ kf.transpose(1, 2) * SCALE
    mask = torch.arange(p + c, device=q.device)[None, :] > (p + torch.arange(c, device=q.device))[:, None]
    s.masked_fill_(mask, float("-inf"))
    return (s.softmax(-1) @ vf).transpose(0, 1).reshape(c, NQ * D)


GRID = [(p, c) for p in (0, 16, 100, 1000, 4000) for c in (1, 7, 128, 129, 500)]


@pytest.mark.parametrize("ps", [16, 32])
def test_paged_equals_contiguous_bitwise_and_fp32(ps):
    q, kv = _case_data(GRID, ps)
    want = _run_contiguous(q, kv, GRID)
    kc, vc, table, _ = _paged(GRID, kv, ps, ps, stale=False)
    got = _run_paged(q, kc, vc, table, GRID, ps)          # every (P, C) of the grid in one launch
    torch.cuda.synchronize()
    qsl = _qsl(GRID)
    bad = [GRID[i] for i in range(len(GRID)) if not torch.equal(got[qsl[i]:qsl[i + 1]], want[qsl[i]:qsl[i + 1]])]
    assert not bad, f"page_size {ps}: paged != contiguous for (P, C) in {bad}"
    for i, (p, c) in enumerate(GRID):
        assert_close(got[qsl[i]:qsl[i + 1]], _fp32(q[qsl[i]:qsl[i + 1]], *kv[i], p), rel=2e-2, what=f"P={p} C={c}")


@pytest.mark.parametrize("ps", [16, 32, 64, 128])
def test_stale_page_tails_and_table_entries_never_reach_the_output(ps):
    cases = [(0, 7), (16, 129), (100, 1), (1000, 500), (37, 91)]
    q, kv = _case_data(cases, 3)
    clean = _run_paged(q, *_paged(cases, kv, ps, 4, stale=False)[:3], cases, ps)
    dirty = _run_paged(q, *_paged(cases, kv, ps, 4, stale=True)[:3], cases, ps)
    torch.cuda.synchronize()
    assert torch.isfinite(dirty.float()).all()
    assert torch.equal(dirty, clean)


def test_batch_independence():
    cases = [(4000, 500), (0, 129), (100, 7), (1000, 128), (16, 1)]
    q, kv = _case_data(cases, 5)
    kc, vc, table, _ = _paged(cases, kv, 16, 6, stale=True)
    together = _run_paged(q, kc, vc, table, cases, 16)
    qsl = _qsl(cases)
    for i in range(len(cases)):
        alone = _run_paged(q, kc, vc, table, cases, 16, seqs=[i])
        assert torch.equal(alone[qsl[i]:qsl[i + 1]], together[qsl[i]:qsl[i + 1]]), cases[i]
        others = torch.cat([alone[:qsl[i]], alone[qsl[i + 1]:]])
        assert not others.any(), "rows of sequences outside the plan were written"


def test_unsupported_page_size_is_rejected_without_launch():
    cases = [(24, 40)]
    q, kv = _case_data(cases, 7)
    kc, vc, table, _ = _paged(cases, kv, 8, 8, stale=False)
    plan = ops.PagedPrefill(_qsl(cases), [64], table, 8)
    out = torch.full((40, NQ * D), 3.0, dtype=BF16, device="cuda")
    before = ops.launch_count()
    with pytest.raises(_lib.VitaB200Error, match="page_size"):
        ops.attention_prefill_paged(q[:, : NQ * D], kc, vc, plan, out, NQ, NKV, D, SCALE)
    torch.cuda.synchronize()
    assert ops.launch_count() == before and bool((out == 3.0).all())
    with pytest.raises(_lib.VitaB200Error):
        ops.PagedPrefill([0, 40], [30], table, 16)        # fewer keys than new rows


# ------------------------------------------------------------------------------------------------ decoder level
def _one_shot_vs_chunked(llm, emb, chunks):
    """KV rows of every layer, last-row logits and first token: one-shot prefill against prefill in `chunks`."""
    S = emb.shape[0]
    def snapshot():
        s = llm.cache.slot_map[0, :S].long()
        return ([k[s].clone() for k in llm.cache.k] + [v[s].clone() for v in llm.cache.v],
                llm.d_logits[0].clone(), int(llm.best[0]))
    llm.reset()
    llm.prefill(emb.clone(), slot=0, want_last_logits=True)
    want = snapshot()
    for chunk in chunks:
        llm.reset()
        llm.best[0] = 12345
        for s0 in range(0, S, chunk):
            n = min(chunk, S - s0)
            final = s0 + n == S
            llm.prefill(emb[s0:s0 + n].clone(), slot=0, start=s0, final=final, want_last_logits=True)
            if not final:     # a non-final chunk leaves the first token and the sampler counter alone
                assert int(llm.best[0]) == 12345 and int(llm.gen_count[0]) == 0
        assert int(llm.cache.cache_len[0]) == S
        got = snapshot()
        kv_bad = [i for i, (a, b) in enumerate(zip(got[0], want[0])) if not torch.equal(a, b)]
        assert not kv_bad, f"chunk {chunk}: KV rows of tensors {kv_bad} differ"
        assert torch.equal(got[1], want[1]), f"chunk {chunk}: last-row logits differ"
        assert got[2] == want[2]


def test_decoder_chunked_prefill_tiny():
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = VitaConfig.tiny()
    model = VITAMixtralForCausalLM(cfg, {"llm": W.pack_llm(W.synthetic_state(cfg, 0, parts=("llm",)), cfg, "cuda")},
                                   "cuda", max_seq_len=1024, max_new_tokens=8)
    ids = torch.randint(0, cfg.llm.vocab_size, (1, 700), generator=torch.Generator().manual_seed(1))
    emb = model._embeds_for(ids, None, None)[0][0].contiguous()
    _one_shot_vs_chunked(model.llm, emb, [64, 128, 129, 500])
    with pytest.raises(ValueError):
        model.llm.prefill(emb[:400].clone(), slot=0, start=700)          # past the KV capacity


@pytest.fixture(scope="module")
def pr1_model():
    from oracle import pr1
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = pr1.config()
    state = pr1.build_state(cfg)
    model = VITAMixtralForCausalLM(cfg, {"llm": W.pack_llm(state, cfg, "cuda")}, "cuda", max_seq_len=1024,
                                   max_new_tokens=pr1.NEW_TOKENS + 1)
    del state
    return cfg, model


def test_decoder_chunked_prefill_pr1_geometry(pr1_model):
    cfg, model = pr1_model
    ids = torch.randint(0, cfg.llm.vocab_size, (1, 700), generator=torch.Generator().manual_seed(2))
    emb = model._embeds_for(ids, None, None)[0][0].contiguous()
    _one_shot_vs_chunked(model.llm, emb, [64, 128, 129, 500])


def test_chunked_prefill_keeps_the_pr1_free_running_trajectory(pr1_model):
    from pathlib import Path
    from oracle import pr1
    cfg, model = pr1_model
    g = np.load(Path(__file__).resolve().parent / "golden" / "pr1_l4.npz")
    ids = pr1.prompt(int(g["prompt_seed"]), cfg.llm.vocab_size)
    emb = model._embeds_for(ids, None, None)[0][0].contiguous()
    llm = model.llm
    llm.reset()
    S = emb.shape[0]
    for s0 in range(0, S, 64):
        llm.prefill(emb[s0:s0 + 64].clone(), slot=0, start=s0, final=s0 + 64 >= S)
    for _ in range(pr1.NEW_TOKENS):
        llm.decode_step(1)
    assert llm.generated_tokens(0)[: pr1.NEW_TOKENS] == g["tokens"].tolist()


# ------------------------------------------------------------------------------------------------ vLLM adapter
class _Engine:
    """Engine-side bookkeeping of the adapter test: shuffled blocks, vLLM flash KV layout, greedy sampling."""

    def __init__(self, cfg, bs=16, n_blocks=96, seed=0):
        c = cfg.llm
        self.bs = bs
        self.kv = [torch.zeros(2, n_blocks, bs, c.num_key_value_heads, c.head_dim, dtype=BF16, device="cuda")
                   for _ in range(c.num_hidden_layers)]
        self.free = torch.randperm(n_blocks, generator=torch.Generator().manual_seed(seed)).tolist()

    def blocks(self, n_tokens, shared=()):
        n = (n_tokens + 8 + self.bs - 1) // self.bs           # (room for the decode steps that follow)
        return list(shared) + [self.free.pop() for _ in range(n - len(shared))]

    def step(self, m, items):
        """items: (table, token ids, first position) per sequence; returns the greedy next token of each."""
        ids, pos, slots, qsl, lens = [], [], [], [0], []
        for table, toks, p0 in items:
            ps = list(range(p0, p0 + len(toks)))
            ids += toks; pos += ps
            slots += [table[p // self.bs] * self.bs + p % self.bs for p in ps]
            qsl.append(qsl[-1] + len(toks)); lens.append(p0 + len(toks))
        width = max(len(t) for t, _, _ in items)
        bt = torch.tensor([t + [0] * (width - len(t)) for t, _, _ in items], dtype=torch.int32, device="cuda")
        from vita_b200.vllm_adapter import TokenBatch
        meta = TokenBatch(torch.tensor(slots, dtype=torch.int32, device="cuda"), bt, qsl, lens)
        hidden = m.forward(torch.tensor(ids), torch.tensor(pos), self.kv, meta)

        class Sel:
            selected_token_indices = torch.tensor([q - 1 for q in qsl[1:]])
        logits = m.compute_logits(hidden, Sel)
        return m.sample(logits).tolist(), logits


@pytest.fixture(scope="module")
def adapter():
    from vita_b200.vllm_adapter import MixtralForConditionalGeneration
    cfg = VitaConfig.tiny()
    m = MixtralForConditionalGeneration(cfg, device="cuda", packed=W.pack(W.synthetic_state(cfg, 0), cfg, "cuda"))
    return cfg, m


def _decode(eng, m, seqs, n):
    """n greedy decode steps of every (table, tokens) sequence, one flattened batch per step."""
    for _ in range(n):
        nxt, _ = eng.step(m, [(t, [s[-1]], len(s) - 1) for t, s in seqs])
        for (t, s), x in zip(seqs, nxt):
            s.append(x)


def test_adapter_chunked_prefill_alongside_decodes(adapter):
    cfg, m = adapter
    g = torch.Generator().manual_seed(3)
    a = torch.randint(3, 1900, (70,), generator=g).tolist()
    b = torch.randint(3, 1900, (23,), generator=g).tolist()
    N = 6
    # unchunked: both prompts whole in one step, then decodes
    e1 = _Engine(cfg, seed=1)
    ta, tb = e1.blocks(len(a) + N), e1.blocks(len(b) + 3 + N)
    nxt, ref_logits = e1.step(m, [(ta, a, 0), (tb, b, 0)])
    ra, rb = [ta, a + [nxt[0]]], [tb, b + [nxt[1]]]
    _decode(e1, m, [rb], 3)                      # b runs ahead by three tokens, as in the chunked schedule
    _decode(e1, m, [ra, rb], N)
    # chunked: b alone, then a over three forward calls that also carry b's decodes
    e2 = _Engine(cfg, seed=2)
    ta, tb = e2.blocks(len(a) + N), e2.blocks(len(b) + 3 + N)
    nxt, _ = e2.step(m, [(tb, b, 0)])
    sb = b + [nxt[0]]
    for lo, hi in ((0, 30), (30, 55), (55, 70)):
        nxt, logits = e2.step(m, [(ta, a[lo:hi], lo), (tb, [sb[-1]], len(sb) - 1)])
        sb.append(nxt[1])
    sa = a + [nxt[0]]
    assert torch.equal(logits[0], ref_logits[0]), "first-token logits of the chunked prompt differ"
    # b took 3 decodes in the chunk steps: it is now where the reference's b was before the joint decodes
    sb_ref_prefix = rb[1][: len(sb)]
    assert sb == sb_ref_prefix
    _decode(e2, m, [[ta, sa], [tb, sb]], N)
    assert sa == ra[1] and sb == rb[1]


def test_adapter_prefix_caching(adapter):
    cfg, m = adapter
    g = torch.Generator().manual_seed(4)
    x = torch.randint(3, 1900, (40,), generator=g).tolist()          # 2 full blocks + 8
    y = torch.randint(3, 1900, (21,), generator=g).tolist()
    second = x[:32] + y
    N = 5
    # reference: the second prompt prefilled whole on its own
    e1 = _Engine(cfg, seed=5)
    t = e1.blocks(len(second) + N)
    nxt, ref_logits = e1.step(m, [(t, second, 0)])
    ref = [t, second + nxt]
    _decode(e1, m, [ref], N)
    # cached: the first request fills its blocks, the second shares its two full blocks and sends only the suffix
    e2 = _Engine(cfg, seed=6)
    t1 = e2.blocks(len(x) + 1)
    e2.step(m, [(t1, x, 0)])
    t2 = e2.blocks(len(second) + N, shared=t1[:2])
    nxt, logits = e2.step(m, [(t2, y, 32)])
    assert torch.equal(logits[0], ref_logits[0]), "first-token logits after prefix reuse differ"
    got = [t2, second + nxt]
    _decode(e2, m, [got], N)
    assert got[1] == ref[1]


# ------------------------------------------------------------------------------------------------ batcher
@pytest.mark.parametrize("sampled", [False, True])
def test_batcher_chunked_admission_gives_the_same_tokens(sampled):
    from vita_b200.engine import ContinuousBatcher, DecoderEngine, Request
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    from vita_b200.sampling import from_hf
    cfg = VitaConfig.tiny()
    packed = {"llm": W.pack_llm(W.synthetic_state(cfg, 0, parts=("llm",)), cfg, "cuda")}
    model = VITAMixtralForCausalLM(cfg, packed, "cuda", max_batch=4, max_seq_len=512, max_new_tokens=24)
    spec = [(0, 40, 16), (1, 300, 8), (2, 9, 12), (3, 200, 10), (5, 130, 6)]

    def requests():
        g = torch.Generator().manual_seed(21)
        out = []
        for rid, (arr, plen, n) in enumerate(spec):
            ids = torch.randint(0, cfg.llm.vocab_size, (1, plen), generator=g)
            sp = from_hf(True, temperature=0.9, top_k=40, top_p=0.9, seed=1000 + rid) if sampled and rid % 2 == 0 \
                else None
            out.append(Request(rid, {"input_ids": ids}, n, None, arrival_step=arr, sampling=sp))
        return out
    eng = DecoderEngine(model)
    whole = ContinuousBatcher(eng, 3).run(requests())
    chunked = ContinuousBatcher(eng, 3, prefill_chunk=64).run(requests())
    assert chunked == whole
