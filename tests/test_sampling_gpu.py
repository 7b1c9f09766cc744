"""Sampled decoding on the GPU: the sampler kernel against the fp64 oracle (oracle/sampling_oracle.py), its
distribution, determinism, and the three surfaces that use it -- generate(do_sample=True), the continuous batcher and
the vLLM adapter's sample()."""
import types

import numpy as np
import pytest
import torch

from oracle import sampling_oracle as SO
from vita_b200 import ops, weights as W
from vita_b200.config import VitaConfig
from vita_b200.sampling import SamplingParams

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _unpack(words):
    return [int(0xFFFFFFFF - (int(w) & 0xFFFFFFFF)) for w in words]


def _rows(rng, B, V):
    """scaled-normal rows plus crafted ones: exact ties, one dominant logit, a flat row"""
    out = []
    for i in range(B):
        kind = i % 8
        if kind == 5:
            r = np.round(rng.normal(0, 2, V) * 2) / 2            # many exact ties
        elif kind == 6:
            r = rng.normal(0, 1, V)
            r[rng.integers(V)] = 25.0                             # one dominant logit
        elif kind == 7:
            r = np.full(V, 0.5 * (i % 3))                         # flat
        else:
            r = rng.normal(0, float(rng.choice([0.5, 2.0, 5.0])), V)
        out.append(r)
    return torch.tensor(np.stack(out), dtype=torch.float32).to(torch.bfloat16)


def _launch(logits, T, k, p, seed, n, scores=None):
    B = logits.shape[0]
    best = torch.zeros(B, dtype=torch.int64, device=DEV)
    f = lambda v, dt: torch.as_tensor(v, dtype=dt).to(DEV)
    seeds = [s - 2**64 if s >= 2**63 else s for s in seed]
    ops.sample_rows(logits, f(T, torch.float32), f(k, torch.int32), f(p, torch.float32), f(seeds, torch.int64),
                    f(n, torch.int32), best, scores)
    return best


@pytest.mark.parametrize("V,B", [(2048, 64), (51760, 16)])
def test_kernel_matches_oracle(V, B):
    rng = np.random.default_rng(V)
    qualified = total = 0
    for T in (0.001, 0.7, 1.0, 1.5):
        for k in (0, 1, 50):
            for p in (1.0, 0.5, 0.9):
                logits = _rows(rng, B, V).to(DEV)
                seeds = [int(s) for s in rng.integers(0, 2**63, B)]
                seeds = [s | (int(rng.integers(0, 2)) << 63) for s in seeds]
                ns = [int(c) for c in rng.integers(0, 5000, B)]
                got = _unpack(_launch(logits, [T] * B, [k] * B, [p] * B, seeds, ns).tolist())
                lf = logits.float().cpu().numpy()
                for b in range(B):
                    tok, gap, dist = SO.choose(lf[b], T, k, p, seeds[b], ns[b])
                    total += 1
                    # fp32 rounding of x + g at |x| = |l| / T, and fp32 top-p masses near the boundary
                    tol = max(1e-4, 4e-7 * np.abs(lf[b]).max() / T)
                    if gap > tol and dist > 1e-6:
                        qualified += 1
                        assert got[b] == tok, (T, k, p, b, got[b], tok, gap)
    assert qualified >= 0.99 * total, (qualified, total)


def test_greedy_rows_bit_identical_to_argmax_rows():
    rng = np.random.default_rng(1)
    for V in (2048, 51760, 1000):
        B = 24
        logits = _rows(rng, B, V).to(DEV)
        ref = torch.zeros(B, dtype=torch.int64, device=DEV)
        ops.argmax_rows(logits, ref)
        T = [0.0 if b % 2 == 0 else 0.8 for b in range(B)]
        got = _launch(logits, T, [50] * B, [0.9] * B, list(range(B)), [3] * B)
        assert got[0::2].tolist() == ref[0::2].tolist()
        assert torch.equal(_launch(logits, [0.0] * B, [0] * B, [1.0] * B, [0] * B, [0] * B), ref)


def test_distribution_chi_square():
    from scipy.stats import chisquare
    V, N = 2048, 1 << 16
    rng = np.random.default_rng(7)
    row = torch.tensor(rng.normal(0, 1.0, V), dtype=torch.float32).to(torch.bfloat16)
    T, k, p, seed = 0.8, 40, 0.9, 0xC0FFEE
    probs = SO.probs(row.float().numpy(), T, k, p)
    kept = np.flatnonzero(probs > 0)
    assert 20 <= kept.size <= 60, kept.size
    logits = row.to(DEV)[None].repeat(N, 1)
    toks = np.array(_unpack(_launch(logits, [T] * N, [k] * N, [p] * N, [seed] * N, list(range(N))).tolist()))
    assert np.isin(toks, kept).all()
    counts = np.bincount(toks, minlength=V)[kept]
    exp = probs[kept] * N
    big = exp >= 5
    f_obs = np.append(counts[big], counts[~big].sum())
    f_exp = np.append(exp[big], exp[~big].sum())
    if f_exp[-1] == 0:
        f_obs, f_exp = f_obs[:-1], f_exp[:-1]
    assert chisquare(f_obs, f_exp).pvalue > 1e-3


def test_determinism_and_batch_invariance():
    rng = np.random.default_rng(2)
    V, B = 51760, 64
    logits = _rows(rng, B, V).to(DEV)
    T = [float(t) for t in rng.choice([0.0, 0.7, 1.0], B)]
    k = [int(x) for x in rng.choice([0, 50], B)]
    p = [float(x) for x in rng.choice([1.0, 0.9], B)]
    seeds = [int(s) for s in rng.integers(0, 2**62, B)]
    ns = list(range(B))
    a = _launch(logits, T, k, p, seeds, ns)
    assert torch.equal(a, _launch(logits, T, k, p, seeds, ns))
    for b in (0, 17, 63):
        one = _launch(logits[b:b + 1], T[b:b + 1], k[b:b + 1], p[b:b + 1], seeds[b:b + 1], ns[b:b + 1])
        assert one.item() == a[b].item()


# ------------------------------------------------------------------------------------------------ generate()
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


def test_generate_sampled(tiny, golden):
    cfg, model = tiny
    ids, mm = _omni(golden)
    L, N = ids.shape[1], 12
    kw = dict(do_sample=True, temperature=0.7, top_k=20, top_p=0.9, max_new_tokens=N, **mm)
    seed = 0x5EED_0123_4567_89AB
    out = model.generate(ids, seed=seed, output_scores=True, **kw)
    toks = out.sequences[0, L:].tolist()
    assert len(toks) == N and len(out.scores) == N
    # every token, the first one included, is the oracle's draw from the logged warped row with counter n = i
    qualified = 0
    for i, t in enumerate(toks):
        row = out.scores[i][0].float().cpu().numpy().astype(np.float64)
        fin = np.isfinite(row)
        assert fin.sum() >= 1 and fin[t]
        s = np.where(fin, row, -np.inf) + SO.gumbel(row.size, seed, i)
        order = np.argsort(-s, kind="stable")
        # the log holds x = l / T rounded to bf16: exempt draws whose perturbed-score gap is within that rounding
        tol = 2 * 2.0 ** -8 * np.abs(row[fin]).max() + 1e-4
        if not fin.sum() > 1 or s[order[0]] - s[order[1]] > tol:
            qualified += 1
            assert t == int(order[0]), (i, t, int(order[0]))
    assert qualified >= N // 2
    eager = model.generate(ids, seed=seed, use_graph=False, **kw)
    assert eager.sequences.tolist() == out.sequences.tolist()
    again = model.generate(ids, seed=seed, sync_every=5, **kw)
    assert again.sequences.tolist() == out.sequences.tolist()
    assert model.generate(ids, seed=seed + 1, **kw).sequences.tolist() != out.sequences.tolist()
    # the library's launch options change timing, never the tokens.  chain_wait = 0 lets a chain kernel trigger its
    # dependent before its own predecessor has completed: the sampler must still see this step's counter (gen_count,
    # written by decode_embed after its trigger); attn_early relies on chain_wait and goes off with it
    names = ("pdl", "chain_counters", "chain_wait", "attn_early")
    saved = {n: ops.get_option(n) for n in names}
    try:
        for opts in [(pdl, cc, 1, 1) for pdl in (0, 1) for cc in (0, 1)] + [(1, 0, 0, 0), (1, 1, 0, 0)]:
            for n, v in zip(names, opts):
                ops.set_option(n, v)
            for use_graph in (True, False):
                model.llm._graphs = {}
                got = model.generate(ids, seed=seed, use_graph=use_graph, **kw)
                assert got.sequences.tolist() == out.sequences.tolist(), (opts, use_graph)
    finally:
        for n, v in saved.items():
            ops.set_option(n, v)
        model.llm._graphs = {}
    # torch.manual_seed makes an unseeded call reproducible
    torch.manual_seed(99)
    a = model.generate(ids, **kw).sequences.tolist()
    torch.manual_seed(99)
    assert model.generate(ids, **kw).sequences.tolist() == a


def test_generate_low_temperature_is_greedy_on_clear_margins(tiny, golden):
    cfg, model = tiny
    ids, mm = _omni(golden)
    L = ids.shape[1]
    greedy = model.generate(ids, max_new_tokens=10, output_scores=True, **mm)
    rows = torch.cat(list(greedy.scores)).float()
    top = rows.topk(2, dim=-1).values
    clear = ((top[:, 0] - top[:, 1]) > 0.0025).tolist()      # Gumbel spread (20.2) x T (1e-4), plus slack
    n = 0
    while n < len(clear) and clear[n]:
        n += 1
    assert n >= 1
    s = model.generate(ids, max_new_tokens=10, do_sample=True, temperature=1e-4, top_k=0, seed=3, **mm)
    assert s.sequences[0, L:L + n].tolist() == greedy.sequences[0, L:L + n].tolist()


def test_sampled_step_launch_count(tiny, golden):
    cfg, model = tiny
    ids, mm = _omni(golden)
    model.generate(ids, max_new_tokens=2, do_sample=True, seed=1, output_scores=True, **mm)
    llm = model.llm
    for want_logits in (False, True):
        n0 = ops.launch_count()
        llm.decode_step(1, use_graph=False, want_logits=want_logits, sampled=True)
        torch.cuda.synchronize()
        assert ops.launch_count() - n0 == llm.launches_per_decode_step_sampled
    assert llm.launches_per_decode_step_sampled == llm.launches_per_decode_step + 1


def test_generate_batch_mixes_sampled_and_greedy(tiny, golden):
    cfg, _ = tiny
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    model = VITAMixtralForCausalLM(cfg, {"llm": W.pack_llm(W.synthetic_state(cfg, 0, parts=("llm",)), cfg, DEV)}, DEV,
                                   max_batch=3, max_seq_len=128, max_new_tokens=16)
    g = torch.Generator().manual_seed(4)
    ids = [torch.randint(0, cfg.llm.vocab_size, (1, 9 + 4 * i), generator=g) for i in range(3)]
    smp = {"temperature": 0.9, "top_k": 30, "seed": 77}
    mixed = model.generate_batch([{"input_ids": ids[0]}, {"input_ids": ids[1], "sampling": smp},
                                  {"input_ids": ids[2]}], max_new_tokens=8)
    greedy = model.generate_batch([{"input_ids": i} for i in ids], max_new_tokens=8)
    assert mixed[0] == greedy[0] and mixed[2] == greedy[2]
    solo = model.generate_batch([{"input_ids": ids[1], "sampling": smp}], max_new_tokens=8)
    assert solo[0] == mixed[1]


# ------------------------------------------------------------------------------------------------ serving engine
def test_continuous_batching_sampled_requests_match_solo_runs():
    from vita_b200.engine import ContinuousBatcher, DecoderEngine, Request
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = VitaConfig.tiny()
    packed = {"llm": W.pack_llm(W.synthetic_state(cfg, 0, parts=("llm",)), cfg, DEV)}
    model = VITAMixtralForCausalLM(cfg, packed, DEV, max_batch=4, max_seq_len=128, max_new_tokens=24)
    spec = [(0, 9, 10), (0, 17, 4), (1, 5, 12), (2, 30, 6), (3, 12, 9), (9, 7, 5), (40, 21, 7)]
    sampled = {1: SamplingParams(0.8, 50, 0.9, 11), 2: SamplingParams(1.2, 0, 1.0, 2**64 - 5),
               4: SamplingParams(0.7, 20, 0.95, 42), 6: SamplingParams(1.0, 5, 1.0, 7)}

    def reqs(all_greedy=False):
        g = torch.Generator().manual_seed(11)
        out = []
        for rid, (arr, plen, n_new) in enumerate(spec):
            ids = torch.randint(0, cfg.llm.vocab_size, (1, plen), generator=g)
            out.append(Request(rid, {"input_ids": ids}, n_new, None, arrival_step=arr,
                               sampling=None if all_greedy else sampled.get(rid)))
        return out

    eng = DecoderEngine(model)
    solo = {}
    for r in reqs():
        r.arrival_step = 0
        solo.update(ContinuousBatcher(eng, 1).run([r]))
    out = ContinuousBatcher(eng, 3, sync_every=2).run(reqs())
    greedy = ContinuousBatcher(eng, 3, sync_every=2).run(reqs(all_greedy=True))
    for rid in solo:
        assert len(out[rid]) == spec[rid][2]
        assert out[rid] == solo[rid], f"request {rid} changed under continuous batching"
        if rid not in sampled:
            assert out[rid] == greedy[rid]
    assert any(out[rid] != greedy[rid] for rid in sampled)
    # a lone sampled request on the bs = 1 chain draws exactly what generate(do_sample=True) draws
    r = reqs()[2]
    r.arrival_step = 0
    lone = ContinuousBatcher(DecoderEngine(model, lone_fast_path=True), 1).run([r])[2]
    sp = sampled[2]
    gen = model.generate(r.payload["input_ids"], do_sample=True, temperature=sp.temperature, top_k=sp.top_k,
                         top_p=sp.top_p, seed=sp.seed, max_new_tokens=spec[2][2])
    assert gen.sequences[0, spec[2][1]:].tolist() == lone


# ------------------------------------------------------------------------------------------------ vLLM adapter
def _meta(params, out_lens, sample_indices=None, do_sample=None):
    groups = []
    for i, (sp, n) in enumerate(zip(params, out_lens)):
        data = types.SimpleNamespace(get_output_len=lambda n=n: n)
        sg = types.SimpleNamespace(sampling_params=sp, seq_ids=[100 + i], seq_data={100 + i: data})
        if sample_indices is not None:
            sg.sample_indices = sample_indices[i]
            sg.do_sample = do_sample[i]
        groups.append(sg)
    return types.SimpleNamespace(seq_groups=groups)


def _vsp(**kw):
    base = dict(n=1, best_of=1, use_beam_search=False, presence_penalty=0.0, frequency_penalty=0.0,
                repetition_penalty=1.0, min_p=0.0, temperature=1.0, top_k=-1, top_p=1.0, seed=None)
    base.update(kw)
    return types.SimpleNamespace(**base)


def test_vllm_adapter_sample():
    from vita_b200.vllm_adapter import MixtralForConditionalGeneration
    cfg = VitaConfig.tiny()
    m = MixtralForConditionalGeneration(cfg, device=DEV, packed={"llm": W.pack_llm(
        W.synthetic_state(cfg, 0, parts=("llm",)), cfg, DEV)})
    rng = np.random.default_rng(5)
    B, V = 12, cfg.llm.vocab_size
    hidden = torch.tensor(rng.normal(0, 1, (B, cfg.llm.hidden_size)), dtype=torch.bfloat16, device=DEV)
    logits = m.compute_logits(hidden)
    lf = logits.float().cpu().numpy()
    greedy = m.sample(logits, None).tolist()
    assert greedy == m.sample(logits, types.SimpleNamespace(selected_token_indices=None)).tolist()
    params = [_vsp(temperature=0.001) if i % 3 == 0 else _vsp(temperature=0.8, top_k=(-1, 40)[i % 2], top_p=0.9,
                                                               seed=1000 + i) for i in range(B)]
    lens = [int(x) for x in rng.integers(0, 300, B)]
    got = m.sample(logits, _meta(params, lens)).tolist()
    for i in range(B):
        if i % 3 == 0:
            top = np.sort(lf[i])[::-1]
            if top[0] - top[1] > 0.025:               # Gumbel spread (20.2) x T (0.001), plus slack
                assert got[i] == greedy[i]
        else:
            sp = params[i]
            tok, gap, dist = SO.choose(lf[i], sp.temperature, max(sp.top_k, 0), sp.top_p, sp.seed, lens[i])
            if gap > 1e-4 and dist > 1e-6:
                assert got[i] == tok, i
    # unseeded rows draw one key each from torch's default generator
    torch.manual_seed(3)
    a = m.sample(logits, _meta([_vsp(temperature=1.0)] * B, lens)).tolist()
    torch.manual_seed(3)
    assert m.sample(logits, _meta([_vsp(temperature=1.0)] * B, lens)).tolist() == a
    # vLLM 0.5.5 layout: groups point at their rows through sample_indices; a chunked-prefill chunk does not sample
    # (do_sample False) and prompt-logprob rows are not sampled -- those rows keep the greedy arg-max
    sp = [_vsp(temperature=0.8, top_k=40, seed=7), _vsp(temperature=0.9, seed=8), _vsp(temperature=0.7, seed=9)]
    got = m.sample(logits, _meta(sp, [3, 0, 11], sample_indices=[[4], [], [9]], do_sample=[True, False, True])).tolist()
    for row, s, n in ((4, sp[0], 3), (9, sp[2], 11)):
        tok, gap, dist = SO.choose(lf[row], s.temperature, max(s.top_k, 0), s.top_p, s.seed, n)
        if gap > 1e-4 and dist > 1e-6:
            assert got[row] == tok, row
    assert [got[r] for r in range(B) if r not in (4, 9)] == [greedy[r] for r in range(B) if r not in (4, 9)]
    for bad in (dict(n=2), dict(best_of=3), dict(use_beam_search=True), dict(presence_penalty=0.1),
                dict(frequency_penalty=0.2), dict(repetition_penalty=1.3), dict(min_p=0.1)):
        with pytest.raises(NotImplementedError):
            m.sample(logits, _meta([_vsp(temperature=0.5, **bad)] * B, lens))
