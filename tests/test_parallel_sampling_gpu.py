"""Parallel sampling on the GPU: the sampler's stream index against the old entry points and the stream oracle
(tests/stream_oracle.py), the fork of a prefilled slot (MixtralDecoder.fork_sampled), generate(do_sample=True,
num_return_sequences=N) and the batcher's n / best_of groups."""
import numpy as np
import pytest
import torch

from oracle import sampling_oracle as SO
from tests import stream_oracle as SSO
from vita_b200 import _lib, ops, weights as W
from vita_b200.config import VitaConfig
from vita_b200.engine import ContinuousBatcher, DecoderEngine, Request
from vita_b200.sampling import SamplingParams

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _unpack(words):
    return [int(0xFFFFFFFF - (int(w) & 0xFFFFFFFF)) for w in words]


def _i64(s):
    return s - 2**64 if s >= 2**63 else s


def _params(rng, B, greedy=True):
    T = [float(t) for t in rng.choice([0.0, 0.7, 1.0, 1.5] if greedy else [0.7, 1.0, 1.5], B)]
    k = [int(x) for x in rng.choice([0, 1, 50], B)]
    p = [float(x) for x in rng.choice([1.0, 0.9, 0.5], B)]
    seeds = [int(s) | (int(rng.integers(0, 2)) << 63) for s in rng.integers(0, 2**63, B)]
    ns = [int(c) for c in rng.integers(0, 5000, B)]
    f = lambda v, dt: torch.as_tensor(v, dtype=dt).to(DEV)
    return (f(T, torch.float32), f(k, torch.int32), f(p, torch.float32), f([_i64(s) for s in seeds], torch.int64),
            f(ns, torch.int32)), (T, k, p, seeds, ns)


def _rows(rng, B, V):
    r = rng.normal(0, 1, (B, V)) * rng.choice([0.5, 2.0, 5.0], (B, 1))
    r[::5] = np.round(r[::5] * 2) / 2                     # exact ties
    return torch.tensor(r, dtype=torch.float32).to(torch.bfloat16).to(DEV)


# ------------------------------------------------------------------------------------------------ kernel
def _old_entry(entry, logits, prm, best, scores, lp, target):
    """The entry points as they were before the stream index (external ctypes callers use them)."""
    B, V = logits.shape
    T, k, p, seed, n = prm
    rows = scores.shape[1] if scores is not None else 0
    sp = scores.data_ptr() if scores is not None else None
    s = torch.cuda.current_stream().cuda_stream
    if entry == "vita_sample_rows":
        _lib.call(entry, logits.data_ptr(), V, B, V, T.data_ptr(), k.data_ptr(), p.data_ptr(), seed.data_ptr(),
                  n.data_ptr(), best.data_ptr(), sp, V, rows, s)
    else:
        logprob, rank, ids, lps = lp
        _lib.call(entry, logits.data_ptr(), V, B, V, T.data_ptr(), k.data_ptr(), p.data_ptr(), seed.data_ptr(),
                  n.data_ptr(), target.data_ptr() if target is not None else None, best.data_ptr(), sp, V, rows,
                  logprob.data_ptr(), rank.data_ptr(), ids.data_ptr(), lps.data_ptr(), 5, ids.shape[1], 0, s)


@pytest.mark.parametrize("variant", ["plain", "logprobs", "logsoftmax"])
@pytest.mark.parametrize("V", [2048, 51760, 1000])
def test_stream_zero_is_bit_identical_to_the_old_entry_points(variant, V):
    rng = np.random.default_rng(V)
    B = 48
    logits = _rows(rng, B, V)
    prm, _ = _params(rng, B)
    prm[4].copy_(torch.arange(B, device=DEV, dtype=torch.int32) % 4)   # counters inside the score log's rows
    target = torch.where(torch.arange(B, device=DEV) % 7 == 3, 5, -1).to(torch.int32)

    def outs():
        lp = (torch.full((B,), 7.0, device=DEV), torch.full((B,), -3, dtype=torch.int32, device=DEV),
              torch.full((B, 8), -3, dtype=torch.int32, device=DEV), torch.full((B, 8), 7.0, device=DEV))
        return torch.zeros(B, dtype=torch.int64, device=DEV), torch.full((B, 4, V), 3.0, dtype=torch.bfloat16,
                                                                            device=DEV), lp

    entry = {"plain": "vita_sample_rows", "logprobs": "vita_sample_rows_logprobs",
             "logsoftmax": "vita_sample_rows_logsoftmax"}[variant]
    ref = outs()
    _old_entry(entry, logits, prm, ref[0], ref[1], ref[2], None if variant == "plain" else target)
    for streams in (None, torch.zeros(B, dtype=torch.int32, device=DEV)):
        got = outs()
        if variant == "plain":
            ops.sample_rows(logits, *prm, got[0], got[1], streams=streams)
        else:
            ops.sample_logprobs(logits, *prm, got[0], *got[2], 5, target=target, scores=got[1],
                                log_softmax_scores=variant == "logsoftmax", streams=streams)
        torch.cuda.synchronize()
        assert torch.equal(got[0], ref[0])
        assert torch.equal(got[1].view(torch.int16), ref[1].view(torch.int16))
        for a, b in zip(got[2], ref[2]):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("V,B", [(2048, 64), (51760, 16)])
def test_streams_match_the_oracle(V, B):
    rng = np.random.default_rng(V + 1)
    qualified = total = 0
    for rep in range(12):
        logits = _rows(rng, B, V)
        prm, (T, k, p, seeds, ns) = _params(rng, B, greedy=False)
        streams = [int(s) for s in rng.integers(0, 2**31, B)]
        streams[:4] = [0, 1, 2, 3]
        best = torch.zeros(B, dtype=torch.int64, device=DEV)
        if rep % 2:
            lp = (torch.zeros(B, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV))
            ops.sample_logprobs(logits, *prm, best, *lp, None, None, 0,
                                streams=torch.tensor(streams, dtype=torch.int32, device=DEV))
        else:
            ops.sample_rows(logits, *prm, best, streams=torch.tensor(streams, dtype=torch.int32, device=DEV))
        got = _unpack(best.tolist())
        lf = logits.float().cpu().numpy()
        for b in range(B):
            tok, gap, dist = SSO.choose(lf[b], T[b], k[b], p[b], seeds[b], ns[b], streams[b])
            total += 1
            tol = max(1e-4, 4e-7 * np.abs(lf[b]).max() / T[b])
            if gap > tol and dist > 1e-6:
                qualified += 1
                assert got[b] == tok, (b, streams[b], got[b], tok, gap)
    assert qualified >= 0.98 * total, (qualified, total)


def _first_tokens(row, T, k, p, seeds, streams):
    N = len(seeds)
    f = lambda v, dt: torch.as_tensor(v, dtype=dt).to(DEV)
    best = torch.zeros(N, dtype=torch.int64, device=DEV)
    ops.sample_rows(row.to(DEV)[None].repeat(N, 1), f([T] * N, torch.float32), f([k] * N, torch.int32),
                    f([p] * N, torch.float32), f([_i64(s) for s in seeds], torch.int64), f([0] * N, torch.int32),
                    best, streams=f(streams, torch.int32))
    return np.array(_unpack(best.tolist()))


def test_first_tokens_over_keys_and_streams_chi_square():
    from scipy.stats import chisquare
    V, N = 2048, 1 << 16
    rng = np.random.default_rng(8)
    row = torch.tensor(rng.normal(0, 1.0, V), dtype=torch.float32).to(torch.bfloat16)
    T, k, p = 0.8, 40, 0.9
    probs = SO.probs(row.float().numpy(), T, k, p)
    kept = np.flatnonzero(probs > 0)
    seeds = [int(s) for s in rng.integers(0, 2**63, N // 16) for _ in range(16)]
    toks = _first_tokens(row, T, k, p, seeds, [i % 16 for i in range(N)])     # 16 streams of each key
    assert np.isin(toks, kept).all()
    counts = np.bincount(toks, minlength=V)[kept]
    exp = probs[kept] * N
    big = exp >= 5
    f_obs = np.append(counts[big], counts[~big].sum())
    f_exp = np.append(exp[big], exp[~big].sum())
    if f_exp[-1] == 0:
        f_obs, f_exp = f_obs[:-1], f_exp[:-1]
    assert chisquare(f_obs, f_exp).pvalue > 1e-3


def test_two_streams_of_one_key_are_not_correlated():
    from scipy.stats import chi2_contingency
    V, N = 512, 1 << 15
    rng = np.random.default_rng(9)
    row = torch.tensor(rng.normal(0, 1.0, V), dtype=torch.float32).to(torch.bfloat16)
    T, k, p = 1.0, 6, 1.0
    probs = SO.probs(row.float().numpy(), T, k, p)
    seeds = [int(s) for s in rng.integers(0, 2**63, N)]
    a = _first_tokens(row, T, k, p, seeds, [0] * N)
    b = _first_tokens(row, T, k, p, seeds, [1] * N)
    match, want = float(np.mean(a == b)), float(np.sum(probs ** 2))
    assert abs(match - want) < 5 * np.sqrt(want * (1 - want) / N), (match, want)
    kept = np.flatnonzero(probs > 0)
    table = np.array([[np.sum((a == i) & (b == j)) for j in kept] for i in kept])
    assert chi2_contingency(table).pvalue > 1e-3


# ------------------------------------------------------------------------------------------------ models
def _tiny(max_batch=8, max_seq_len=512, max_new_tokens=32):
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = VitaConfig.tiny()
    packed = {"llm": W.pack_llm(W.synthetic_state(cfg, 0, parts=("llm",)), cfg, DEV)}
    return cfg, VITAMixtralForCausalLM(cfg, packed, DEV, max_batch=max_batch, max_seq_len=max_seq_len,
                                       max_new_tokens=max_new_tokens, shuffle_pages=True)


@pytest.fixture(scope="module")
def tiny():
    return _tiny()


def _pr1():
    from oracle import pr1
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = pr1.config()
    state = pr1.build_state(cfg)
    model = VITAMixtralForCausalLM(cfg, {"llm": W.pack_llm(state, cfg, DEV)}, DEV, max_batch=4, max_seq_len=512,
                                   max_new_tokens=16, shuffle_pages=True)
    del state
    return cfg, model


def _ids(cfg, n, seed):
    return torch.randint(0, cfg.llm.vocab_size, (1, n), generator=torch.Generator().manual_seed(seed))


SP = SamplingParams(0.9, 40, 0.95, 0x1234_5678_9ABC_DEF0)


def _kv_rows(cache, slot, S):
    pos = torch.arange(S)
    ps = cache.page_size
    pages = cache.block_table[slot].cpu()[pos // ps].to(torch.int64)
    return (pages * ps + pos % ps).to(DEV)


@pytest.mark.parametrize("which", ["tiny", "pr1"])
def test_fork_is_exact(which):
    """Prompt K/V of every fork is bit-identical (full pages physically shared, the partial page copied), and the
    forked run's tokens equal N separate prefills of the prompt advanced in one batch with the same keys and
    streams."""
    cfg, model = _tiny(max_batch=4) if which == "tiny" else _pr1()
    llm, N, S, steps = model.llm, 4, 37, 12
    emb, lens = model._embeds_for(_ids(cfg, S, 1), None, None)
    rows = emb[0, :S].contiguous()
    ps = llm.cache.page_size

    llm.reset()
    llm.sampling.set(0, SP, 0)
    llm.prefill(rows.clone(), slot=0, sampled=True, logprobs=0)
    llm.fork_sampled(0, N, S, -(-(S + steps + 1) // ps))
    llm.cache.pool.check()
    full = S // ps
    bt = llm.cache.block_table.cpu()
    for d in range(1, N):
        assert torch.equal(bt[d, :full], bt[0, :full])
        assert bt[d, full] != bt[0, full]
        for l in range(cfg.llm.num_hidden_layers):
            for t in (llm.cache.k[l], llm.cache.v[l]):
                assert torch.equal(t[_kv_rows(llm.cache, d, S)].view(torch.int16),
                                   t[_kv_rows(llm.cache, 0, S)].view(torch.int16))
    assert llm.sampling.stream[:N].tolist() == list(range(N))
    for _ in range(steps):
        llm.decode_step_batched(N, sampled=True, logprobs=0)
    forked = [llm.generated_tokens(b) for b in range(N)]
    forked_lp = llm.lp_log[0][:N, :steps].clone()

    llm.reset()
    for b in range(N):
        llm.sampling.set(b, SP, 0)
        llm.sampling.stream[b] = b
        llm.prefill(rows.clone(), slot=b, sampled=True, logprobs=0)
    for _ in range(steps):
        llm.decode_step_batched(N, sampled=True, logprobs=0)
    solo = [llm.generated_tokens(b) for b in range(N)]
    assert forked == solo
    assert torch.equal(forked_lp, llm.lp_log[0][:N, :steps])
    if which == "tiny":                                  # (PR1's synthetic logits are too peaked to tell apart)
        assert len({tuple(t) for t in forked}) == N        # the streams are different samples
    for b in range(N):
        llm.sampling.set(b, None)
    llm.reset()


# ------------------------------------------------------------------------------------------------ generate()
class _Stop:
    """Marks every row (a bool) once the view is `at` columns wide, or only `rows` (a [N] tensor)."""

    def __init__(self, at, rows=None):
        self.at, self.rows, self.calls = at, rows, 0

    def __call__(self, ids, scores):
        self.calls += 1
        hit = ids.shape[1] >= self.at
        if self.rows is None:
            return hit
        out = torch.zeros(ids.shape[0], dtype=torch.bool)
        out[self.rows] = hit
        return out


def _gen(model, ids, **kw):
    args = dict(do_sample=True, temperature=0.9, top_k=40, top_p=0.95, seed=77, num_return_sequences=4,
                max_new_tokens=12, sync_every=5)
    args.update(kw)
    return model.generate(ids, **args)


def test_generate_shapes_eos_and_criteria(tiny):
    cfg, model = tiny
    ids = _ids(cfg, 21, 2)
    L = ids.shape[1]
    free = _gen(model, ids)
    rows = free.sequences[:, L:].tolist()
    assert free.sequences.shape == (4, L + 12) and torch.equal(free.sequences[:, :L], ids.repeat(4, 1))
    assert len({tuple(r) for r in rows}) > 1
    assert model.llm.cache.pool is not None and not model.llm.cache.shared
    # EOS: a token of row 1; every row stops at its first EOS and is padded with it until the last row stops
    eos = rows[1][3]
    out = _gen(model, ids, eos_token_id=eos)
    ends = [r.index(eos) + 1 if eos in r else 12 for r in rows]
    T = max(ends)
    assert out.sequences.shape == (4, L + T)
    for b in range(4):
        assert out.sequences[b, L:].tolist() == rows[b][:ends[b]] + [eos] * (T - ends[b])
    # a bool criterion stops every row
    stop = _Stop(L + 5)
    out = _gen(model, ids, stopping_criteria=[stop])
    assert out.sequences[:, L:].tolist() == [r[:5] for r in rows] and stop.calls == 5
    # a per-row criterion finishes the rows it marks: padded with the EOS id, or kept without one
    absent = next(t for t in range(cfg.llm.vocab_size) if all(t not in r for r in rows))
    out = _gen(model, ids, stopping_criteria=[_Stop(L + 3, rows=[2])], eos_token_id=absent)
    assert out.sequences.shape == (4, L + 12)
    assert out.sequences[2, L:].tolist() == rows[2][:3] + [absent] * 9
    assert [out.sequences[b, L:].tolist() for b in (0, 1, 3)] == [rows[b] for b in (0, 1, 3)]
    out = _gen(model, ids, stopping_criteria=[_Stop(L + 3, rows=[0, 1, 2, 3])])
    assert out.sequences[:, L:].tolist() == [r[:3] for r in rows]
    out = _gen(model, ids, stopping_criteria=[_Stop(L + 3, rows=[2])])
    assert out.sequences[:, L:].tolist() == rows


def test_generate_reproducible_first_token_and_graph(tiny):
    cfg, model = tiny
    ids = _ids(cfg, 33, 3)
    L = ids.shape[1]
    a = _gen(model, ids)
    assert torch.equal(a.sequences, _gen(model, ids).sequences)
    assert torch.equal(a.sequences, _gen(model, ids, use_graph=False).sequences)
    assert torch.equal(a.sequences, _gen(model, ids, sync_every=1).sequences)
    torch.manual_seed(5)
    m1 = _gen(model, ids, seed=None)
    torch.manual_seed(5)
    assert torch.equal(m1.sequences, _gen(model, ids, seed=None).sequences)
    one = model.generate(ids, do_sample=True, temperature=0.9, top_k=40, top_p=0.95, seed=77, max_new_tokens=4)
    assert a.sequences[0, L].item() == one.sequences[0, L].item()


def test_generate_scores_and_logprobs(tiny):
    cfg, model = tiny
    ids = _ids(cfg, 40, 4)
    L, N, T = ids.shape[1], 4, 0.9
    out = _gen(model, ids, output_scores=True, logprobs=3)
    plain = _gen(model, ids)
    assert torch.equal(out.sequences, plain.sequences)
    n_new = out.sequences.shape[1] - L
    assert len(out.scores) == n_new and all(s.shape == (N, cfg.llm.vocab_size) for s in out.scores)
    one = model.generate(ids, do_sample=True, temperature=0.9, top_k=40, top_p=0.95, seed=77, max_new_tokens=1,
                         output_scores=True, logprobs=3)
    for b in range(N):                                   # every sequence's first row comes from the prompt's logits
        assert torch.equal(out.scores[0][b].view(torch.int16), one.scores[0][0].view(torch.int16))
    qualified = total = 0
    for i, s in enumerate(out.scores):                   # the warped rows the tokens were drawn from
        rows = s.float().cpu().numpy()
        for b in range(N):
            t = int(out.sequences[b, L + i])
            assert np.isfinite(rows[b, t])
            tok, gap, _ = SSO.choose(rows[b] * T, T, 0, 1.0, 77, i, b)
            total += 1
            if gap > 2e-2 * max(1.0, np.abs(rows[b][np.isfinite(rows[b])]).max()):
                qualified += 1
                assert tok == t, (i, b)
    assert qualified >= total // 2
    assert len(out.logprobs) == N
    for b in range(N):
        recs = out.logprobs[b]
        assert [r.token for r in recs] == out.sequences[b, L:].tolist()
        assert all(len(r.top) == 3 and r.rank >= 1 and r.logprob <= 0 for r in recs)
    assert out.logprobs[0][0] == one.logprobs[0]


# ------------------------------------------------------------------------------------------------ batcher
def _requests(cfg, chunky=False):
    g = torch.Generator().manual_seed(12)
    prefix = torch.randint(0, cfg.llm.vocab_size, (150,), generator=g)
    out = []
    for rid in range(6):
        q = torch.randint(0, cfg.llm.vocab_size, (4 + 5 * rid,), generator=g)
        ids = torch.cat([prefix, q])[None]
        sp = SamplingParams(0.8 + 0.1 * (rid % 3), 30, 0.9, 900 + rid) if rid != 4 else None
        kw = dict(n=4, best_of=6, logprobs=None) if rid == 2 else dict(logprobs=1 if rid == 3 else None)
        if rid == 5:
            kw = dict(n=2, logprobs=2)
        out.append(Request(rid, {"input_ids": ids}, 6 + 2 * rid, None, arrival_step=3 * rid, sampling=sp, **kw))
    return out


def _solo(model, r, stream):
    """The request alone in slot 0, drawing from `stream` of its key (batched step: batch-invariant on tiny)."""
    llm = model.llm
    llm.reset()
    emb, lens = model._embeds_for(r.payload["input_ids"], None, None)
    width = 0
    llm.sampling.set(0, r.sampling, width)
    llm.sampling.stream[0] = stream
    llm.prefill(emb[0, :lens[0]].contiguous(), slot=0, sampled=r.sampling is not None, logprobs=width)
    for _ in range(r.max_new_tokens):
        llm.decode_step_batched(1, sampled=r.sampling is not None, logprobs=width)
    toks = llm.generated_tokens(0)[:r.max_new_tokens]
    lp = sum(llm.lp_log[0][0, :len(toks)].tolist())      # in token order, as the batcher sums
    llm.sampling.set(0, None)
    return toks, lp


def test_batcher_groups_among_staggered_arrivals(tiny):
    cfg, model = tiny
    runs = {}
    for cache in (False, True):
        for chunk in (None, 32):
            model.llm.reset()
            eng = DecoderEngine(model, prefix_cache=cache)
            for rep in range(2):                         # the second run reuses the slots: no page leaks
                reqs = _requests(cfg)
                done = ContinuousBatcher(eng, 8, sync_every=3, prefill_chunk=chunk).run(reqs)
                model.llm.cache.pool.check()
                res = (done, [[(q.index, q.tokens) for q in r.sequences] for r in reqs])
                if rep:
                    assert res == runs[(cache, chunk)]
                runs[(cache, chunk)] = res
            pool = model.llm.cache.pool
            held = {pg for row in pool.table for pg in row if pg >= 0}
            assert len(held) + len(pool.free) + len(pool.index.lru) == len(pool.refs)
            if cache:
                assert eng.prefix_stats["hit_pages"] > 0
    assert runs[(False, None)] == runs[(True, None)]
    assert runs[(False, 32)] == runs[(True, 32)]
    reqs = _requests(cfg)
    done, seqs = runs[(False, None)]
    group = reqs[2]
    assert len(seqs[2]) == 4 and len(seqs[5]) == 2
    solo = {s: _solo(model, group, s) for s in range(6)}
    for i, toks in seqs[2]:
        assert toks == solo[i][0], i
    ranked = sorted(range(6), key=lambda s: (-solo[s][1], s))[:4]
    assert [i for i, _ in seqs[2]] == ranked
    assert done[2] == seqs[2][0][1]
    for i, toks in seqs[5]:
        assert toks == _solo(model, reqs[5], i)[0]
    assert seqs[5][0][1] != seqs[5][1][1]
    for rid in (0, 1, 3):
        assert done[rid] == _solo(model, reqs[rid], 0)[0]
    model.llm.reset()
