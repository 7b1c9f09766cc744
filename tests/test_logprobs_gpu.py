"""Log-probabilities on the GPU (the LOGPROBS variant of csrc/sample.cu, `ops.sample_logprobs`): the kernel against the
fp64 oracle, tokens unchanged, batch invariance, and the three surfaces -- generate(logprobs=N), the continuous batcher
and the vLLM adapter's sample_with_logprobs."""
import gc
import types

import numpy as np
import pytest
import torch

from tests.logprobs_oracle import logprobs as oracle_logprobs
from vita_b200 import ops, weights as W
from vita_b200.config import VitaConfig
from vita_b200.sampling import MAX_LOGPROBS, SamplingParams

pytestmark = pytest.mark.gpu

DEV = "cuda"
ATOL = 1e-4


@pytest.fixture(autouse=True, scope="module")
def _free_models():
    """The models built here hold CUDA graphs in reference cycles: free them when the module ends."""
    yield
    gc.collect()


def _unpack(words):
    return [int(0xFFFFFFFF - (int(w) & 0xFFFFFFFF)) for w in words]


def _rows(rng, B, V):
    """scaled-normal rows plus crafted ones: exact ties, one dominant logit, a flat row"""
    out = []
    for i in range(B):
        kind = i % 4
        if kind == 1:
            r = np.round(rng.normal(0, 2, V) * 2) / 2            # many exact ties
        elif kind == 2:
            r = rng.normal(0, 1, V)
            r[rng.integers(V)] = 25.0                             # one dominant logit
        elif kind == 3:
            r = np.full(V, 0.5 * (i % 3))                         # flat
        else:
            r = rng.normal(0, float(rng.choice([0.5, 2.0, 5.0])), V)
        out.append(r)
    return torch.tensor(np.stack(out), dtype=torch.float32).to(torch.bfloat16)


def _params(B, T, k, p, seeds, n):
    f = lambda v, dt: torch.as_tensor(v, dtype=dt).to(DEV)
    return (f([T] * B, torch.float32), f([k] * B, torch.int32), f([p] * B, torch.float32),
            f([s - 2**64 if s >= 2**63 else s for s in seeds], torch.int64), f(n, torch.int32))


def _launch_lp(logits, prm, n_top, target=None, log_rows=0):
    B = logits.shape[0]
    shape = (B, log_rows) if log_rows else (B,)
    best = torch.zeros(B, dtype=torch.int64, device=DEV)
    lp = torch.full(shape, 7.0, dtype=torch.float32, device=DEV)
    rank = torch.full(shape, -7, dtype=torch.int32, device=DEV)
    ids = torch.full(shape + (MAX_LOGPROBS,), -7, dtype=torch.int32, device=DEV)
    tl = torch.full(shape + (MAX_LOGPROBS,), 7.0, dtype=torch.float32, device=DEV)
    tg = None if target is None else torch.tensor(target, dtype=torch.int32, device=DEV)
    ops.sample_logprobs(logits, *prm, best, lp, rank, ids, tl, n_top, target=tg)
    return best, lp, rank, ids, tl


def _close(got, want):
    """equal -inf pattern, finite values within ATOL"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.array_equal(np.isfinite(got), np.isfinite(want)), (got, want)
    fin = np.isfinite(want)
    assert np.all(np.abs(got[fin] - want[fin]) <= ATOL), np.abs(got[fin] - want[fin]).max()


GRID = [(0.0, 0, 1.0)] + [(T, k, p) for T in (0.7, 1.3) for k in (0, 50) for p in (1.0, 0.9)]


@pytest.mark.parametrize("V", [2048, 51760])
def test_kernel_matches_oracle(V):
    rng = np.random.default_rng(V)
    B = 16
    checked = 0
    for T, k, p in GRID:
        logits = _rows(rng, B, V).to(DEV)
        lf = logits.float().cpu().numpy()
        seeds = [int(s) for s in rng.integers(0, 2**63, B)]
        cnt = [int(c) for c in rng.integers(0, 1000, B)]
        prm = _params(B, T, k, p, seeds, cnt)
        # even rows draw (or take the arg-max), odd rows score a target: the arg-max, a random token, a low one
        target = [-1 if b % 2 == 0 else int((np.argmax(lf[b]), rng.integers(V), np.argmin(lf[b]))[b // 2 % 3])
                  for b in range(B)]
        for N in (0, 1, 5, 20):
            best, lp, rank, ids, tl = (t.cpu() for t in _launch_lp(logits, prm, N, target))
            toks = _unpack(best)
            for b in range(B):
                tok = target[b] if target[b] >= 0 else toks[b]
                want = oracle_logprobs(lf[b], T, k, p, N, tok)
                if want["dist"] <= 1e-6:            # a token that close to the top-p boundary may fall either way
                    continue
                assert want["kept"][tok] or target[b] >= 0
                _close([lp[b].item()], [want["logprob"]])
                assert rank[b].item() == want["rank"], (T, k, p, N, b)
                assert ids[b, :N].tolist() == want["top_ids"].tolist(), (T, k, p, N, b)
                _close(tl[b, :N].numpy(), want["top_logprobs"])
                assert (ids[b, N:] == -7).all()               # columns past N are not written
                if target[b] >= 0:
                    assert toks[b] == int(np.lexsort((np.arange(V), -lf[b]))[0])   # best keeps the greedy word
                checked += 1
    assert checked > 0.9 * len(GRID) * B * 4


def test_tokens_unchanged_and_greedy_rows_equal_argmax_rows():
    rng = np.random.default_rng(1)
    B, V = 32, 51760
    for T, k, p in GRID:
        logits = _rows(rng, B, V).to(DEV)
        seeds = [int(s) for s in rng.integers(0, 2**64, B, dtype=np.uint64)]
        prm = _params(B, T, k, p, seeds, [int(c) for c in rng.integers(0, 50, B)])
        ref = torch.zeros(B, dtype=torch.int64, device=DEV)
        ops.sample_rows(logits, *prm, ref)
        for N in (0, 5, 20):
            best = _launch_lp(logits, prm, N)[0]
            assert torch.equal(best, ref), (T, k, p, N)
        if T == 0:
            am = torch.zeros(B, dtype=torch.int64, device=DEV)
            ops.argmax_rows(logits, am)
            assert torch.equal(ref, am)


def test_batch_invariance_and_counter_rows():
    rng = np.random.default_rng(2)
    V, B = 51760, 12
    logits = _rows(rng, B, V).to(DEV)
    seeds = [int(s) for s in rng.integers(0, 2**63, B)]
    cnt = [int(c) for c in rng.integers(0, 6, B)]
    T = [0.0, 0.7, 1.3] * 4
    K = [0, 50, 0, 50] * 3
    P = [1.0, 0.9, 0.9, 1.0, 1.0, 0.9] * 2
    target = [-1, -1, 5, -1, 17, -1] * 2
    f = lambda v, dt: torch.as_tensor(v, dtype=dt).to(DEV)

    def run(order, log_rows=0):
        prm = (f([T[i] for i in order], torch.float32), f([K[i] for i in order], torch.int32),
               f([P[i] for i in order], torch.float32), f([seeds[i] for i in order], torch.int64),
               f([cnt[i] for i in order], torch.int32))
        return _launch_lp(logits[order].contiguous(), prm, 20, [target[i] for i in order], log_rows)

    ref = run(list(range(B)))
    for perm in (list(range(B))[::-1], [int(i) for i in rng.permutation(B)]):
        out = run(perm)
        for j, i in enumerate(perm):
            for a, r in zip(out, ref):
                assert torch.equal(a[j], r[i]), (i, j)          # bit-identical at any batch position
    # a device-resident log: request b writes row counter[b] and nothing else
    log = run(list(range(B)), log_rows=6)
    for b in range(B):
        for a, r in zip(log[1:], ref[1:]):
            assert torch.equal(a[b, cnt[b]], r[b])
            others = [x for x in range(6) if x != cnt[b]]
            assert (a[b, others] == (7.0 if a.dtype == torch.float32 else -7)).all()


def test_parameter_checks():
    logits = torch.zeros(2, 64, dtype=torch.bfloat16, device=DEV)
    prm = _params(2, 0.0, 0, 1.0, [0, 0], [0, 0])
    from vita_b200 import _lib
    with pytest.raises(_lib.VitaB200Error):
        _launch_lp(logits, prm, 21)
    small = torch.zeros(2, 8, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(_lib.VitaB200Error):
        _launch_lp(small, prm, 9)                               # more top entries than tokens


# ------------------------------------------------------------------------------------------------ generate
@pytest.fixture(scope="module")
def tiny():
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = VitaConfig.tiny()
    return cfg, VITAMixtralForCausalLM(cfg, W.pack(W.synthetic_state(cfg, 0), cfg, DEV), DEV, max_new_tokens=32)


def _omni(golden):
    inp, _ = golden
    t = torch.from_numpy
    return t(inp["omni_ids"]), dict(images=t(inp["images"])[:1],
                                     audios={"audios": t(inp["feats"])[:1], "lengths": t(inp["lengths"])[:1]})


def _host_logprobs(score_row, tok, n):
    x = score_row.double().cpu()
    lsm = torch.log_softmax(x, -1)
    order = np.lexsort((np.arange(x.numel()), -x.numpy()))[:n]
    rank = 1 + int((x > x[tok]).sum())
    return lsm[tok].item(), rank, order.tolist(), lsm[order].numpy()


@pytest.mark.parametrize("sample", [None, dict(do_sample=True, temperature=1.0, top_k=40, top_p=0.9, seed=99)])
def test_generate_logprobs(tiny, golden, sample):
    cfg, model = tiny
    ids, mm = _omni(golden)
    L, N = ids.shape[1], 12
    kw = dict(max_new_tokens=N, **mm, **(sample or {}))
    plain = model.generate(ids, **kw)
    out = model.generate(ids, logprobs=5, output_scores=True, **kw)
    eager = model.generate(ids, logprobs=5, use_graph=False, **kw)
    toks = out.sequences[0, L:].tolist()
    assert toks == plain.sequences[0, L:].tolist() and plain.logprobs is None
    assert eager.logprobs == out.logprobs and eager.sequences.tolist() == out.sequences.tolist()
    assert len(out.logprobs) == N
    for i, (t, rec) in enumerate(zip(toks, out.logprobs)):
        # greedy scores are the logits, sampled ones at T = 1 are l itself (-inf outside the kept set): exact in bf16
        lp, rank, top, top_lp = _host_logprobs(out.scores[i][0], t, 5)
        assert rec.token == t and rec.rank == rank
        _close([rec.logprob], [lp])
        _close([b for _, b in rec.top], top_lp)
        kept = int(np.isfinite(top_lp).sum())       # past the kept set the log has no logits to order the ids by
        assert [a for a, _ in rec.top][:kept] == top[:kept]
    # logprobs=0 records only the logprob and rank, the same ones
    zero = model.generate(ids, logprobs=0, **kw)
    assert [(e.token, e.logprob, e.rank, e.top) for e in zero.logprobs] == \
        [(e.token, e.logprob, e.rank, ()) for e in out.logprobs]
    with pytest.raises(ValueError):
        model.generate(ids, logprobs=21, **kw)


def test_generate_batch_logprobs(tiny):
    cfg, _ = tiny
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    model = VITAMixtralForCausalLM(cfg, {"llm": W.pack_llm(W.synthetic_state(cfg, 0, parts=("llm",)), cfg, DEV)}, DEV,
                                   max_batch=3, max_seq_len=128, max_new_tokens=16)
    g = torch.Generator().manual_seed(4)
    ids = [torch.randint(0, cfg.llm.vocab_size, (1, 9 + 4 * i), generator=g) for i in range(3)]
    smp = {"temperature": 0.9, "top_k": 30, "seed": 77}
    reqs = [{"input_ids": ids[0], "logprobs": 3}, {"input_ids": ids[1], "sampling": smp, "logprobs": 0},
            {"input_ids": ids[2]}]
    got = model.generate_batch(reqs, max_new_tokens=8)
    plain = model.generate_batch([{k: v for k, v in r.items() if k != "logprobs"} for r in reqs], max_new_tokens=8)
    assert got == plain and "token_logprobs" not in reqs[2]
    for r, toks in zip(reqs[:2], got):
        assert [e.token for e in r["token_logprobs"]] == toks
        assert all(len(e.top) == r["logprobs"] and np.isfinite(e.logprob) for e in r["token_logprobs"])
    solo = [{"input_ids": ids[0], "logprobs": 3}]
    model.generate_batch(solo, max_new_tokens=8)
    assert solo[0]["token_logprobs"] == reqs[0]["token_logprobs"]


# ------------------------------------------------------------------------------------------------ serving engine
def test_continuous_batching_logprobs_match_solo_runs():
    from vita_b200.engine import ContinuousBatcher, DecoderEngine, Request
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = VitaConfig.tiny()
    packed = {"llm": W.pack_llm(W.synthetic_state(cfg, 0, parts=("llm",)), cfg, DEV)}
    model = VITAMixtralForCausalLM(cfg, packed, DEV, max_batch=4, max_seq_len=128, max_new_tokens=24)
    spec = [(0, 9, 10), (0, 17, 4), (1, 5, 12), (2, 30, 6), (3, 12, 9), (9, 7, 5), (40, 21, 7)]
    sampled = {1: SamplingParams(0.8, 50, 0.9, 11), 4: SamplingParams(0.7, 20, 0.95, 42)}
    asks = {0: 5, 1: 20, 3: 0, 4: 2, 6: 1}

    def reqs():
        g = torch.Generator().manual_seed(11)
        out = []
        for rid, (arr, plen, n_new) in enumerate(spec):
            ids = torch.randint(0, cfg.llm.vocab_size, (1, plen), generator=g)
            out.append(Request(rid, {"input_ids": ids}, n_new, None, arrival_step=arr, sampling=sampled.get(rid),
                               logprobs=asks.get(rid)))
        return out

    eng = DecoderEngine(model)
    solo = {}
    for r in reqs():
        r.arrival_step = 0
        ContinuousBatcher(eng, 1).run([r])
        solo[r.rid] = r
    rs = reqs()
    out = ContinuousBatcher(eng, 3, sync_every=2).run(rs)
    for r in rs:
        assert out[r.rid] == solo[r.rid].tokens
        assert r.token_logprobs == solo[r.rid].token_logprobs, f"request {r.rid}: logprobs changed under batching"
        if r.logprobs is not None:
            assert len(r.token_logprobs) == len(r.tokens) and all(len(e.top) == r.logprobs for e in r.token_logprobs)
        else:
            assert r.token_logprobs == []


def test_negative_query_logprobs():
    """a duplex query dropped as negative right after its prefill keeps the record of its state token"""
    from vita_b200.engine import ContinuousBatcher, DecoderEngine, Request
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = VitaConfig.tiny()
    packed = {"llm": W.pack_llm(W.synthetic_state(cfg, 0, parts=("llm",)), cfg, DEV)}
    model = VITAMixtralForCausalLM(cfg, packed, DEV, max_batch=2, max_seq_len=128, max_new_tokens=16)
    g = torch.Generator().manual_seed(5)
    ids = [torch.randint(0, cfg.llm.vocab_size, (1, n), generator=g) for n in (11, 14)]
    eng = DecoderEngine(model)
    solo = Request(1, {"input_ids": ids[1]}, 4, logprobs=3)
    ContinuousBatcher(eng, 1).run([solo])
    state = solo.tokens[0]                               # the query's first token, taken as its `<2>` state token
    reqs = [Request(0, {"input_ids": ids[0]}, 8, logprobs=2),
            Request(1, {"input_ids": ids[1]}, 4, arrival_step=3, negative_token_id=state, logprobs=3)]
    ContinuousBatcher(eng, 2).run(reqs)
    neg = reqs[1]
    assert neg.outcome == "negative" and neg.tokens == [state]
    assert [e.token for e in neg.token_logprobs] == neg.tokens
    assert neg.token_logprobs == solo.token_logprobs[:1]
    assert [e.token for e in reqs[0].token_logprobs] == reqs[0].tokens


# ------------------------------------------------------------------------------------------------ vLLM adapter
def _vsp(**kw):
    base = dict(n=1, best_of=1, use_beam_search=False, presence_penalty=0.0, frequency_penalty=0.0,
                repetition_penalty=1.0, min_p=0.0, temperature=1.0, top_k=-1, top_p=1.0, seed=None, logprobs=None,
                prompt_logprobs=None)
    base.update(kw)
    return types.SimpleNamespace(**base)


def _group(sp, sid, out_len=0, prompt=(), computed=0, sample_indices=None, prompt_rows=None, do_sample=True):
    data = types.SimpleNamespace(get_output_len=lambda: out_len, prompt_token_ids=list(prompt),
                                 get_num_computed_tokens=lambda: computed)
    sg = types.SimpleNamespace(sampling_params=sp, seq_ids=[sid], seq_data={sid: data}, do_sample=do_sample)
    if sample_indices is not None:
        sg.sample_indices = sample_indices
    if prompt_rows is not None:
        sg.prompt_logprob_indices = prompt_rows
    return sg


@pytest.fixture(scope="module")
def adapter():
    from vita_b200.vllm_adapter import MixtralForConditionalGeneration
    cfg = VitaConfig.tiny()
    return cfg, MixtralForConditionalGeneration(cfg, device=DEV, packed={"llm": W.pack_llm(
        W.synthetic_state(cfg, 0, parts=("llm",)), cfg, DEV)})


def _check_rec(rec, lf, T, k, p, n, tok):
    want = oracle_logprobs(lf, T, k, p, n, tok)
    if want["dist"] <= 1e-6:
        return 0
    assert rec.token == tok and rec.rank == want["rank"]
    assert [a for a, _ in rec.top] == want["top_ids"].tolist()
    _close([rec.logprob] + [b for _, b in rec.top], [want["logprob"]] + want["top_logprobs"].tolist())
    return 1


def test_vllm_sample_with_logprobs(adapter):
    cfg, m = adapter
    rng = np.random.default_rng(5)
    B, V = 10, cfg.llm.vocab_size
    hidden = torch.tensor(rng.normal(0, 1, (B, cfg.llm.hidden_size)), dtype=torch.bfloat16, device=DEV)
    logits = m.compute_logits(hidden)
    lf = logits.float().cpu().numpy()
    prompt = [int(t) for t in rng.integers(0, V, 12)]
    sps = [_vsp(temperature=0.8, top_k=40, top_p=0.9, seed=7, logprobs=5),
           _vsp(temperature=0.0, logprobs=20, prompt_logprobs=3),
           _vsp(temperature=1.3, seed=8),
           _vsp(temperature=0.7, top_p=0.9, seed=9, prompt_logprobs=20)]
    meta = lambda: types.SimpleNamespace(seq_groups=[
        _group(sps[0], 1, out_len=4, sample_indices=[0]),
        _group(sps[1], 2, prompt=prompt, computed=3, sample_indices=[5], prompt_rows=[1, 2, 3, 4]),
        _group(sps[2], 3, out_len=9, sample_indices=[6]),
        _group(sps[3], 4, prompt=prompt, computed=6, sample_indices=[], prompt_rows=[7, 8, 9], do_sample=False)])
    ids, groups = m.sample_with_logprobs(logits, meta())
    assert ids.tolist() == m.sample(logits, meta()).tolist()          # sample() keeps its tokens
    n = 0
    for gi, row, (T, k, p), N in ((0, 0, (0.8, 40, 0.9), 5), (1, 5, (0.0, 0, 1.0), 20), (2, 6, (1.3, 0, 1.0), 0)):
        rec = groups[gi].sample
        assert rec.token == ids[row].item()
        n += _check_rec(rec, lf[row], T, k, p, N, rec.token)
    assert groups[0].prompt == [] and groups[2].prompt == [] and groups[3].sample is None
    for gi, rows, done, (T, k, p), N in ((1, [1, 2, 3, 4], 3, (0.0, 0, 1.0), 3), (3, [7, 8, 9], 6, (0.7, 0, 0.9), 20)):
        assert len(groups[gi].prompt) == len(rows)
        for j, (row, rec) in enumerate(zip(rows, groups[gi].prompt)):
            n += _check_rec(rec, lf[row], T, k, p, N, prompt[done + 1 + j])
    assert n >= 10


def test_vllm_unseeded_keys_match_sample(adapter):
    """a group that only scores prompt rows takes no key: unseeded sampling groups draw what sample() draws"""
    cfg, m = adapter
    rng = np.random.default_rng(6)
    V = cfg.llm.vocab_size
    logits = m.compute_logits(torch.tensor(rng.normal(0, 1, (4, cfg.llm.hidden_size)), dtype=torch.bfloat16,
                                           device=DEV))
    prompt = [int(t) for t in rng.integers(0, V, 8)]
    meta = lambda: types.SimpleNamespace(seq_groups=[
        _group(_vsp(temperature=0.9, prompt_logprobs=1), 1, prompt=prompt, computed=2, sample_indices=[],
               prompt_rows=[0, 1], do_sample=False),
        _group(_vsp(temperature=1.0), 2, out_len=3, sample_indices=[2]),
        _group(_vsp(temperature=1.0, logprobs=1), 3, out_len=5, sample_indices=[3])])
    torch.manual_seed(3)
    want = m.sample(logits, meta()).tolist()
    next_want = torch.randint(0, 1 << 30, (1,)).item()
    torch.manual_seed(3)
    ids, groups = m.sample_with_logprobs(logits, meta())
    assert ids.tolist() == want and [r.token for r in groups[0].prompt] == prompt[3:5]
    assert torch.randint(0, 1 << 30, (1,)).item() == next_want       # the generator advanced as far as in sample()


def test_vllm_prompt_logprobs_chunked_equal_whole(adapter):
    from vita_b200.vllm_adapter import TokenBatch
    cfg, m = adapter
    c = cfg.llm
    bs, n_blocks = 16, 16
    g = torch.Generator().manual_seed(3)
    prompt = torch.randint(3, 1900, (70,), generator=g).tolist()
    sp = _vsp(temperature=0.7, top_k=50, seed=5, logprobs=2, prompt_logprobs=4)

    def run(chunks):
        kv = [torch.zeros(2, n_blocks, bs, c.num_key_value_heads, c.head_dim, dtype=torch.bfloat16, device=DEV)
              for _ in range(c.num_hidden_layers)]
        table = torch.randperm(n_blocks, generator=torch.Generator().manual_seed(1)).tolist()
        recs, first = [], None
        for lo, hi in chunks:
            pos = list(range(lo, hi))
            slots = torch.tensor([table[q // bs] * bs + q % bs for q in pos], dtype=torch.int32, device=DEV)
            meta = TokenBatch(slots, torch.tensor([table], dtype=torch.int32, device=DEV), [0, hi - lo], [hi])
            hidden = m.forward(torch.tensor(prompt[lo:hi]), torch.tensor(pos), kv, meta)
            logits = m.compute_logits(hidden)
            final = hi == len(prompt)
            n_rows = hi - lo - (1 if final else 0)
            sg = _group(sp, 1, prompt=prompt, computed=lo, sample_indices=[hi - lo - 1] if final else [],
                        prompt_rows=list(range(n_rows)), do_sample=final)
            ids, groups = m.sample_with_logprobs(logits, types.SimpleNamespace(seq_groups=[sg]))
            recs += groups[0].prompt
            if final:
                first = groups[0].sample
        return recs, first

    whole, first = run([(0, 70)])
    chunked, first_c = run([(0, 30), (30, 55), (55, 70)])
    assert len(whole) == 69 and [r.token for r in whole] == prompt[1:]
    assert chunked == whole and first_c == first
