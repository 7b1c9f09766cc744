"""Prefix caching in the continuous batcher on the H100 (vita_b200/engine.py, DecoderEngine(prefix_cache=True)): the
page-digest kernel against its numpy reference, bit-identical KV rows and logits after a hit, and batcher schedules
whose tokens and logprob records equal the cache-off run."""
import numpy as np
import pytest
import torch

from tests.test_prefix_cache import digest_ref
from vita_b200 import ops
from vita_b200 import weights as W
from vita_b200.config import AUDIO_TOKEN_INDEX, IMAGE_TOKEN_INDEX, VitaConfig
from vita_b200.engine import ContinuousBatcher, DecoderEngine, Request
from vita_b200.sampling import from_hf

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ digest kernel
@pytest.mark.parametrize("S,H,ld,ps", [(15, 64, 64, 16), (16, 64, 72, 16), (17, 64, 128, 16), (80, 40, 48, 32),
                                       (4160, 4096, 4096, 16), (4160, 4096, 4104, 32)])
def test_page_digest_matches_numpy_reference(S, H, ld, ps):
    g = torch.Generator().manual_seed(S + ld)
    full = torch.randn(S, ld, generator=g).bfloat16()
    rows = full.cuda()[:, :H]
    got = ops.page_digest(rows, ps).cpu().numpy().view(np.uint64)
    want = digest_ref(full[:, :H], ps)
    assert got.shape == (S // ps, 2)
    assert np.array_equal(got, want)


# ------------------------------------------------------------------------------------------------ models
def _tiny(max_batch=3, max_seq_len=512, max_new_tokens=24, parts=("llm",), **kw):
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = VitaConfig.tiny()
    state = W.synthetic_state(cfg, 0, parts=parts) if parts != "all" else W.synthetic_state(cfg, 0)
    packed = W.pack(state, cfg, "cuda") if parts == "all" else {"llm": W.pack_llm(state, cfg, "cuda")}
    return cfg, VITAMixtralForCausalLM(cfg, packed, "cuda", max_batch=max_batch, max_seq_len=max_seq_len,
                                       max_new_tokens=max_new_tokens, shuffle_pages=True, **kw)


@pytest.fixture(scope="module")
def pr1_model():
    from oracle import pr1
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = pr1.config()
    state = pr1.build_state(cfg)
    model = VITAMixtralForCausalLM(cfg, {"llm": W.pack_llm(state, cfg, "cuda")}, "cuda", max_batch=3,
                                   max_seq_len=1024, max_new_tokens=16, shuffle_pages=True)
    del state
    return cfg, model


# ------------------------------------------------------------------------------------------------ same request twice
def _same_request_twice(model, cfg, S):
    llm = model.llm
    llm.reset()
    ids = torch.randint(0, cfg.llm.vocab_size, (1, S), generator=torch.Generator().manual_seed(S))
    eng = DecoderEngine(model, prefix_cache=True)
    ps = llm.cache.page_size

    def admit(slot):
        eng.reset_slot(slot)
        r = Request(slot, {"input_ids": ids}, 4, logprobs=0)      # logprobs: the last-row logits land in d_logits
        P = eng.prefill(slot, r)
        rows = llm.cache.slot_map[slot, :S].long()
        kv = [t[rows].clone() for t in llm.cache.k + llm.cache.v]
        return P, kv, llm.d_logits[slot].clone(), int(llm.best[slot])

    P0, kv0, lg0, b0 = admit(0)
    P1, kv1, lg1, b1 = admit(1)
    assert P0 == 0 and P1 == ps * ((S - 1) // ps)
    table = llm.cache.pool.table
    assert table[1][:P1 // ps] == table[0][:P1 // ps]              # the hit pages are shared, not copied
    bad = [i for i, (a, b) in enumerate(zip(kv0, kv1)) if not torch.equal(a[P1:], b[P1:])]
    assert not bad, f"newly written KV rows of tensors {bad} differ from the cold prefill"
    assert torch.equal(lg0, lg1) and b0 == b1
    llm.cache.pool.check()
    llm.reset()


@pytest.mark.parametrize("S", [16, 17, 100, 300])
def test_same_request_twice_is_bit_identical_tiny(S):
    cfg, model = _tiny(max_batch=2)
    _same_request_twice(model, cfg, S)


def test_same_request_twice_is_bit_identical_pr1_geometry(pr1_model):
    cfg, model = pr1_model
    _same_request_twice(model, cfg, 700)


# ------------------------------------------------------------------------------------------------ batcher schedules
def _requests(cfg, n=7, prefix_len=150, stagger=2, negative=None, sessions=False):
    """Questions over two shared prefixes (and one unrelated prompt): greedy, sampled and logprobs requests mixed,
    arriving staggered with different lengths, so retirements swap slots."""
    g = torch.Generator().manual_seed(5)
    prefixes = [torch.randint(0, cfg.llm.vocab_size, (prefix_len,), generator=g) for _ in range(2)]
    out = []
    for rid in range(n):
        q = torch.randint(0, cfg.llm.vocab_size, (5 + 7 * rid,), generator=g)
        ids = torch.cat([prefixes[rid % 2], q]) if rid != 3 else q
        sp = from_hf(True, temperature=0.8, top_k=30, top_p=0.9, seed=500 + rid) if rid % 3 == 1 else None
        r = Request(rid, {"input_ids": ids[None]}, 4 + 3 * (rid % 4), None, arrival_step=stagger * rid, sampling=sp,
                    logprobs=2 if rid % 3 == 2 else None)
        if sessions:
            r.session, r.negative_token_id = rid % 2, -1
        if negative is not None and rid in negative:
            r.negative_token_id = negative[rid]
        out.append(r)
    return out


def _run(model, cfg, prefix_cache, chunk=None, max_batch=3, **kw):
    model.llm.reset()
    eng = DecoderEngine(model, prefix_cache=prefix_cache)
    reqs = _requests(cfg, **kw)
    out = ContinuousBatcher(eng, max_batch, sync_every=2, prefill_chunk=chunk).run(reqs)
    model.llm.cache.pool.check()
    return out, reqs, eng


def _assert_same(model, cfg, **kw):
    """Tokens and logprob records bit-identical to the cache-off run when admission is not chunked.  A chunked
    admission that hits needs fewer chunks, so the steps after it run at other batch sizes, and a duplex interrupt
    lands at another step, than in the cache-off run: there the tokens are the same, an interrupted answer stops
    at another length (one is a prefix of the other), and logprob values may round differently."""
    want, wreqs, _ = _run(model, cfg, False, **kw)
    got, greqs, eng = _run(model, cfg, True, **kw)
    if kw.get("chunk") is None:
        assert got == want
    for a, b in zip(wreqs, greqs):
        assert a.outcome == b.outcome, a.rid
        if kw.get("chunk") is None:
            assert a.token_logprobs == b.token_logprobs, a.rid
        else:
            n = min(len(a.tokens), len(b.tokens))
            assert a.tokens[:n] == b.tokens[:n], a.rid
            assert a.outcome == "interrupted" or a.tokens == b.tokens, a.rid
            assert [t.token for t in a.token_logprobs[:n]] == [t.token for t in b.token_logprobs[:n]], a.rid
    assert sum(r.cached_tokens for r in greqs) > 0 and eng.prefix_stats["hit_pages"] > 0
    return greqs, eng


@pytest.mark.parametrize("chunk", [None, 64])
def test_batcher_tokens_equal_the_cache_off_run_tiny(chunk):
    cfg, model = _tiny()
    _assert_same(model, cfg, chunk=chunk)


def test_batcher_tokens_equal_the_cache_off_run_pr1_geometry(pr1_model):
    cfg, model = pr1_model
    _assert_same(model, cfg)
    _assert_same(model, cfg, chunk=64)


def test_batcher_with_eviction():
    # 2 slots of 16 pages: 32 pages in all, each request reserves up to 14, so indexed prefixes get evicted
    cfg, model = _tiny(max_batch=2, max_seq_len=256)
    reqs, eng = _assert_same(model, cfg, max_batch=2, n=9, prefix_len=150, stagger=0)
    assert eng.evictions > 0
    reqs, eng = _assert_same(model, cfg, max_batch=2, n=9, prefix_len=150, stagger=0, chunk=64)


def test_batcher_duplex_interrupts_and_negative_queries():
    cfg, model = _tiny()
    firsts, _, _ = _run(model, cfg, False)
    negative = {rid: firsts[rid][0] for rid in (0, 2, 4)}         # these queries answer with their "state token"
    reqs, _ = _assert_same(model, cfg, negative=negative, sessions=True)
    assert [r.outcome for r in reqs if r.rid in negative] == ["negative"] * 3
    assert any(r.outcome == "interrupted" for r in reqs)
    # request 2 shares prefix 0 with the dropped negative query 0 (and arrives after it)
    assert reqs[2].cached_tokens >= 144
    reqs, _ = _assert_same(model, cfg, negative=negative, sessions=True, chunk=64)


# ------------------------------------------------------------------------------------------------ multimodal
def test_multimodal_requests_share_the_feature_pages():
    cfg, model = _tiny(max_batch=2, max_seq_len=1024, parts="all")
    g = torch.Generator().manual_seed(9)
    ps = model.llm.cache.page_size
    img = lambda: torch.randn(1, 3, cfg.vision.image_size, cfg.vision.image_size, generator=g).bfloat16().float()
    image, other_image = img(), img()
    audios = {"audios": torch.randn(1, 100, 80, generator=g).bfloat16().float(), "lengths": torch.tensor([100])}
    head = torch.randint(0, cfg.llm.vocab_size, (40,), generator=g)

    def req(rid, image, q_seed):
        q = torch.randint(0, cfg.llm.vocab_size, (9,), generator=torch.Generator().manual_seed(q_seed))
        ids = torch.cat([head, torch.tensor([IMAGE_TOKEN_INDEX, 5, AUDIO_TOKEN_INDEX]), q])[None]
        return Request(rid, {"input_ids": ids, "images": image, "audios": audios}, 6, None, arrival_step=rid)

    def run(prefix_cache):
        model.llm.reset()
        reqs = [req(0, image, 1), req(1, image, 2), req(2, other_image, 1)]
        eng = DecoderEngine(model, prefix_cache=prefix_cache)
        return ContinuousBatcher(eng, 2).run(reqs), reqs, eng

    want, _, _ = run(False)
    got, reqs, eng = run(True)
    assert got == want
    S = int(model._embeds_for(reqs[1].payload["input_ids"], image, audios)[1][0])
    assert reqs[1].cached_tokens == ps * ((S - 9) // ps) and reqs[1].cached_tokens > 40     # image + audio rows
    assert reqs[2].cached_tokens == ps * (40 // ps)                 # only the pages before the other image


# ------------------------------------------------------------------------------------------------ fp8 KV
def test_fp8_kv_cache_hits_and_clear_margin_tokens():
    cfg, model = _tiny(kv_cache_dtype="fp8")
    want, wreqs, _ = _run(model, cfg, False)
    got, greqs, eng = _run(model, cfg, True)
    assert eng.prefix_stats["hit_pages"] > 0
    for a, b in zip(wreqs, greqs):
        if a.sampling is not None or a.logprobs is None:
            continue
        for i, (ta, tb) in enumerate(zip(a.tokens, b.tokens)):
            top = a.token_logprobs[i].top
            if len(top) < 2 or top[0][1] - top[1][1] < 0.05:
                break                                               # past an unclear margin the runs may part
            assert ta == tb, (a.rid, i)


# ------------------------------------------------------------------------------------------------ invalidation
def test_generate_between_batcher_runs_leaves_no_stale_hits():
    cfg, model = _tiny()
    fresh, _, _ = _run(model, cfg, False)
    model.llm.reset()
    eng = DecoderEngine(model, prefix_cache=True)
    first = ContinuousBatcher(eng, 3, sync_every=2).run(_requests(cfg))
    other = torch.randint(0, cfg.llm.vocab_size, (1, 170), generator=torch.Generator().manual_seed(77))
    model.generate(other, max_new_tokens=8)                        # rewrites the KV cache from slot 0's static row
    reqs = _requests(cfg)
    second = ContinuousBatcher(eng, 3, sync_every=2).run(reqs)
    assert first == fresh and second == fresh
    assert reqs[0].cached_tokens == 0                              # nothing survives the reset of generate()


def test_expert_parallel_is_refused():
    cfg, model = _tiny(max_batch=1, max_seq_len=128)
    model.llm.ep_world = 2
    with pytest.raises(ValueError):
        DecoderEngine(model, prefix_cache=True)
