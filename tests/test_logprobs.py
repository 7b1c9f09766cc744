"""Logprob contract on the CPU: the fp64 oracle against torch.log_softmax over the installed transformers' warpers, the
top-N / rank definitions, parameter checks of every surface, and the batcher's logprob hand-over with a stand-in
engine."""
import types

import numpy as np
import pytest
import torch

from tests.logprobs_oracle import logprobs as oracle_logprobs
from tests.test_engine import FakeEngine, stream
from vita_b200 import sampling as S
from vita_b200.engine import ContinuousBatcher, Request


def _hf_log_softmax(l32, T, k, p):
    """HF 4.41's warpers applied to the fp32 upcast of a bf16 row, then log_softmax in float64."""
    from transformers.generation.logits_process import (TemperatureLogitsWarper, TopKLogitsWarper,
                                                        TopPLogitsWarper)
    s = torch.tensor(l32, dtype=torch.float64)[None]
    ids = torch.zeros(1, 1, dtype=torch.long)
    if T > 0:
        s = TemperatureLogitsWarper(T)(ids, s)
        if k:
            s = TopKLogitsWarper(k)(ids, s)
        if p < 1.0:
            s = TopPLogitsWarper(p)(ids, s)
    return torch.log_softmax(s, -1)[0].numpy()


def _boundary_tie(l, k, p):
    """a value tie at the top-k or top-p boundary: HF breaks it by sort order, the contract keeps / drops ties together"""
    sv = np.sort(l)[::-1]
    if 0 < k < l.size and sv[k - 1] == sv[k]:
        return True
    return bool(np.any(np.diff(sv[: (k or l.size) + 1]) == 0)) if p < 1.0 else False


def test_oracle_matches_log_softmax_over_transformers_warpers():
    rng = np.random.default_rng(11)
    checked = 0
    for trial in range(300):
        V = int(rng.choice([7, 64, 500]))
        l32 = torch.tensor(rng.normal(0, rng.choice([0.5, 2.0, 6.0]), V), dtype=torch.float32) \
            .to(torch.bfloat16).float().numpy()
        T = float(rng.choice([0.0, 0.3, 0.7, 1.0, 1.5]))
        k = int(rng.choice([0, 1, 5, 50])) if T > 0 else 0
        p = float(rng.choice([1.0, 0.5, 0.9, 0.95])) if T > 0 else 1.0
        if _boundary_tie(l32, k, p):
            continue
        want = _hf_log_softmax(l32, T, k, p)
        got = oracle_logprobs(l32, T, k, p, 5, int(rng.integers(V)))["row"]
        assert np.array_equal(np.isfinite(got), np.isfinite(want)), (trial, V, T, k, p)
        fin = np.isfinite(want)
        np.testing.assert_allclose(got[fin], want[fin], rtol=0, atol=1e-12)
        checked += 1
    assert checked > 200


def test_oracle_rank_and_top_n():
    l = np.array([1.0, 3.0, 3.0, -2.0, 0.5, 3.0])
    r = oracle_logprobs(l, 0.0, 0, 1.0, 4, 4)
    assert r["top_ids"].tolist() == [1, 2, 5, 0]          # logit descending, index ascending on ties
    assert r["rank"] == 5                                  # 1 + four tokens strictly above 0.5
    assert oracle_logprobs(l, 0.0, 0, 1.0, 0, 2)["rank"] == 1    # ties share the best rank
    # outside the kept set: -inf, and the rank counts every kept token
    r = oracle_logprobs(l, 0.7, 3, 1.0, 6, 0)
    assert r["logprob"] == -np.inf and r["rank"] == 4
    assert np.isfinite(r["top_logprobs"][:3]).all() and not np.isfinite(r["top_logprobs"][3:]).any()


@pytest.mark.parametrize("bad", [-1, 21, 2.0, "5", True])
def test_logprobs_range_and_type(bad):
    with pytest.raises(ValueError):
        S.check_logprobs(bad)


def test_logprobs_accepted_values():
    assert S.check_logprobs(None) is None
    assert [S.check_logprobs(n) for n in (0, 1, 20)] == [0, 1, 20]
    sl = S.SlotSampling(3, "cpu")
    sl.set(1, None, 5)
    sl.set(2, S.SamplingParams(0.7, 50, 0.9, 3), None)
    assert sl.log_width(0, 2) == S.MAX_LOGPROBS and sl.log_width(0, 1) is None and sl.log_width(2, 1) is None
    sl.set(0, None, 0)
    assert sl.log_width(0, 1) == 0 and sl.log_width(0, 3) == S.MAX_LOGPROBS
    sl.swap(1, 2)
    assert sl.logprobs == [0, None, 5] and sl.sampled == [False, True, False]
    with pytest.raises(ValueError):
        sl.set(0, None, 21)


def test_logprob_records():
    lp = torch.tensor([-0.5, -1.5])
    rank = torch.tensor([1, 3], dtype=torch.int32)
    ids = torch.tensor([[4, 7, 9], [7, 4, 2]], dtype=torch.int32)
    tl = torch.tensor([[-0.5, -1.0, -2.0], [-0.25, -1.0, -1.5]])
    recs = S.logprob_records([4, 2], lp, rank, ids, tl, 2)
    assert recs[0] == S.TokenLogprobs(4, -0.5, 1, ((4, -0.5), (7, -1.0)))
    assert recs[1].token == 2 and recs[1].rank == 3 and recs[1].top == ((7, -0.25), (4, -1.0))


def _vsp(**kw):
    base = dict(n=1, best_of=1, use_beam_search=False, presence_penalty=0.0, frequency_penalty=0.0,
                repetition_penalty=1.0, min_p=0.0, temperature=1.0, top_k=-1, top_p=1.0, seed=None, logprobs=None,
                prompt_logprobs=None)
    base.update(kw)
    return types.SimpleNamespace(**base)


def test_scoring_params_draw_no_key():
    torch.manual_seed(5)
    a = S.from_vllm(_vsp(temperature=0.7, top_k=40))
    torch.manual_seed(5)
    s = S.from_vllm(_vsp(temperature=0.7, top_k=40), draws=False)
    assert s == S.SamplingParams(0.7, 40, 1.0, 0)
    assert S.from_vllm(_vsp(temperature=0.7, top_k=40)) == a          # the generator did not advance
    assert S.from_vllm(_vsp(temperature=0.7, seed=9), draws=False).seed == 9


def test_vllm_adapter_rejects_a_row_claimed_twice():
    from vita_b200.config import VitaConfig
    from vita_b200.vllm_adapter import MixtralForConditionalGeneration
    m = MixtralForConditionalGeneration(VitaConfig.tiny(), device="cpu")

    def group(sp, sid, **kw):
        data = types.SimpleNamespace(get_output_len=lambda: 0, prompt_token_ids=list(range(10)),
                                     get_num_computed_tokens=lambda: 0)
        return types.SimpleNamespace(sampling_params=sp, seq_ids=[sid], seq_data={sid: data}, **kw)
    meta = types.SimpleNamespace(seq_groups=[
        group(_vsp(seed=1), 1, sample_indices=[0], do_sample=True),
        group(_vsp(prompt_logprobs=2), 2, sample_indices=[], do_sample=False, prompt_logprob_indices=[1, 0])])
    with pytest.raises(ValueError):
        m.sample_with_logprobs(torch.zeros(2, 64, dtype=torch.bfloat16), meta)


def test_vllm_adapter_rejects_out_of_range_logprobs():
    from vita_b200.config import VitaConfig
    from vita_b200.vllm_adapter import MixtralForConditionalGeneration
    m = MixtralForConditionalGeneration(VitaConfig.tiny(), device="cpu")
    sp = types.SimpleNamespace(n=1, best_of=1, use_beam_search=False, presence_penalty=0.0, frequency_penalty=0.0,
                               repetition_penalty=1.0, min_p=0.0, temperature=1.0, top_k=-1, top_p=1.0, seed=1,
                               logprobs=21, prompt_logprobs=None)
    data = types.SimpleNamespace(get_output_len=lambda: 0)
    sg = types.SimpleNamespace(sampling_params=sp, seq_ids=[0], seq_data={0: data})
    meta = types.SimpleNamespace(seq_groups=[sg])
    with pytest.raises(ValueError):
        m.sample_with_logprobs(torch.zeros(1, 64, dtype=torch.bfloat16), meta)
    with pytest.raises(ValueError):
        m.sample_with_logprobs(torch.zeros(1, 64, dtype=torch.bfloat16), None)


def _lp(seed, i):
    """the stand-in's logprob of token i of the request with `seed`"""
    return -(seed * 100 + i) / 1000.0


class LogprobEngine(FakeEngine):
    """The stand-in engine plus `read_logprobs`.  Like the real engine it pairs the rows of its per-slot log (here a
    function of the slot's request and the row) with the tokens the batcher holds: its token log, like the real one,
    does not hold a first token before a step has consumed it."""

    def __init__(self, max_batch, cap):
        super().__init__(max_batch, cap)
        self.reads = []

    def read_logprobs(self, slot, tokens, n_top):
        seed = int(self.seed[slot])
        self.reads.append(seed)
        return [S.TokenLogprobs(t, _lp(seed, i), 1, tuple((t + j, -1.0 - j) for j in range(n_top)))
                for i, t in enumerate(tokens)]


def test_batcher_reads_logprobs_only_for_requests_that_ask():
    reqs = []
    for rid in range(7):
        reqs.append(Request(rid, {"seed": 100 + rid}, 4 + rid % 4, arrival_step=rid // 2,
                            eos_token_id=stream(100 + rid, 8)[2] if rid == 3 else None,
                            logprobs=(rid % 3 or None) if rid % 2 else None))
    eng = LogprobEngine(3, 64)
    out = ContinuousBatcher(eng, 3, sync_every=2).run(reqs)
    asked = {r.rid for r in reqs if r.logprobs is not None}
    assert sorted(eng.reads) == sorted(100 + rid for rid in asked)
    for r in reqs:
        assert out[r.rid] == r.tokens
        if r.logprobs is None:
            assert r.token_logprobs == []
        else:
            assert [e.token for e in r.token_logprobs] == r.tokens
            assert [e.logprob for e in r.token_logprobs] == [_lp(r.payload["seed"], i) for i in range(len(r.tokens))]
            assert all(len(e.top) == r.logprobs for e in r.token_logprobs)
    # the stand-in engine without read_logprobs keeps working for requests that do not ask
    plain = [Request(r.rid, r.payload, r.max_new_tokens, r.eos_token_id, arrival_step=r.arrival_step) for r in reqs]
    assert ContinuousBatcher(FakeEngine(3, 64), 3, sync_every=2).run(plain) == out


def test_negative_query_keeps_its_first_token_record():
    """a query dropped as negative right after its prefill: its one record carries the state token"""
    first = stream(7, 1)[0]
    reqs = [Request(0, {"seed": 3}, 6, logprobs=2),
            Request(1, {"seed": 7}, 5, arrival_step=2, negative_token_id=first, logprobs=4)]
    eng = LogprobEngine(2, 64)
    ContinuousBatcher(eng, 2).run(reqs)
    neg = reqs[1]
    assert neg.outcome == "negative" and neg.tokens == [first]
    assert [e.token for e in neg.token_logprobs] == [first] and neg.token_logprobs[0].logprob == _lp(7, 0)
    assert len(neg.token_logprobs[0].top) == 4
