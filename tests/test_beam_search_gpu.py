"""Beam search on the GPU: `kv_copy_pages`, copy-on-write KV pages bit for bit against solo replays, the decisions
against the oracle (tests/beam_oracle.py) fed with the kernel's logprobs, graph against eager, the log-softmax score
rows, and the demo's generate() kwargs with num_beams=4."""
import gc

import numpy as np
import pytest
import torch

from tests.beam_oracle import beam_search as oracle_beam_search
from vita_b200 import ops, weights as W
from vita_b200.beam import BeamSearch
from vita_b200.config import VitaConfig
from vita_b200.sampling import MAX_LOGPROBS

pytestmark = pytest.mark.gpu

DEV = "cuda"
N = 4


@pytest.fixture(autouse=True, scope="module")
def _free_models():
    yield
    gc.collect()


def test_kv_copy_pages_bit_exact():
    g = torch.Generator(device="cpu").manual_seed(0)
    n_pages, ps, nkv, D, layers = 24, 16, 8, 128, 3
    caches = [torch.randn(n_pages * ps, nkv, D, generator=g).to(torch.bfloat16).to(DEV) for _ in range(2 * layers)]
    pairs = [(3, 7), (3, 9), (0, 23), (11, 2)]
    canary = {5, 6, 12}                                      # pages in no pair: NaN, must stay NaN
    for c in caches:
        for pg in canary:
            c[pg * ps:(pg + 1) * ps] = float("nan")
    before = [c.clone() for c in caches]
    base = torch.tensor([c.data_ptr() for c in caches], dtype=torch.int64, device=DEV)
    ops.kv_copy_pages(base, torch.tensor(pairs, dtype=torch.int32, device=DEV), n_pages, ps * nkv * D * 2)
    torch.cuda.synchronize()
    for c, b in zip(caches, before):
        want = b.clone()
        for s, d in pairs:
            want[d * ps:(d + 1) * ps] = b[s * ps:(s + 1) * ps]
        assert torch.equal(c.view(torch.int16), want.view(torch.int16))
        for pg in canary:
            assert torch.isnan(c[pg * ps:(pg + 1) * ps].float()).all()


# ------------------------------------------------------------------------------------------------ decoder driver
def _packed(tokens):
    return torch.tensor([0xFFFFFFFF - t for t in tokens], dtype=torch.int64)


def _drive(model, ids, steps, eos=None, use_graph=True):
    """The loop of VITAMixtralForCausalLM._beam_search, recording per step each running beam's logits row and the
    kernel's top 20.  Returns (search, records {history: (logits, top ids, top logprobs)}, histories per step)."""
    llm = model.llm
    emb = model._embeds_for(ids, None, None)[0][0].contiguous()
    S = emb.shape[0]
    llm.reset()
    for b in range(N):
        llm.sampling.set(b, None, MAX_LOGPROBS)
    lp = llm.enable_logprob_log()
    llm.prefill(emb, slot=0, logprobs=MAX_LOGPROBS)
    search = BeamSearch(N, steps, eos)
    recs, per_step = {}, []
    t, rows = 0, 1
    while True:
        torch.cuda.synchronize()
        logits = llm.d_logits[:rows].float().cpu()
        top_i, top_l = lp[2][:rows, t].cpu(), lp[3][:rows, t].cpu()
        hist = [tuple(b.tokens) for b in search.running]
        per_step.append(hist)
        for b, h in enumerate(hist):
            recs[h] = (logits[b], top_i[b], top_l[b])
        parents = search.step(top_i[:, :2 * N].tolist(), top_l[:, :2 * N].numpy())
        t += 1
        if search.done:
            break
        if t == 1:
            llm.fork(0, range(1, N), S)
        else:
            llm.cache.reorder(parents, S + t - 1)
        llm.best[:N].copy_(_packed([b.tokens[-1] for b in search.running]))
        llm.decode_step_batched(N, use_graph=use_graph, logprobs=MAX_LOGPROBS)
        rows = N
    return search, recs, per_step


def _solo_replays(model, ids, recs):
    """Every recorded history replayed alone in slot 0 (static pages): prefill, then its tokens forced through
    decode_step_batched(1).  Returns the histories compared."""
    llm = model.llm
    emb = model._embeds_for(ids, None, None)[0][0].contiguous()
    leaves = [h for h in recs if not any(len(o) > len(h) and o[:len(h)] == h for o in recs)]
    compared = set()
    for leaf in leaves:
        llm.reset()
        llm.sampling.set(0, None, None)
        llm.prefill(emb.clone(), slot=0, want_last_logits=True)
        for i in range(len(leaf) + 1):
            h = leaf[:i]
            if h in recs:
                got = llm.d_logits[0].float().cpu()
                assert torch.equal(got, recs[h][0]), f"beam history of {len(h)} tokens: logits differ from its replay"
                compared.add(h)
            if i < len(leaf):
                llm.best[:1].copy_(_packed([leaf[i]]))
                llm.decode_step_batched(1, use_graph=False)
    return compared


def _batch_replays(model, ids, recs, per_step):
    """The N histories of every step replayed together on the static table: each prompt prefilled into its own slot,
    then the tokens forced through decode_step_batched(N).  Returns the histories compared."""
    llm = model.llm
    emb = model._embeds_for(ids, None, None)[0][0].contiguous()
    compared = set()
    for t, hist in enumerate(per_step[1:], start=1):
        llm.reset()
        for b in range(N):
            llm.sampling.set(b, None, None)
            llm.prefill(emb.clone(), slot=b)
        for i in range(t):
            llm.best[:N].copy_(_packed([h[i] for h in hist]))
            llm.decode_step_batched(N, use_graph=False)
        got = llm.d_logits[:N].float().cpu()
        for b, h in enumerate(hist):
            assert torch.equal(got[b], recs[h][0]), f"step {t}, slot {b}: logits differ from the static-page replay"
            compared.add(h)
    return compared


@pytest.fixture(scope="module")
def tiny():
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = VitaConfig.tiny()
    model = VITAMixtralForCausalLM(cfg, W.pack(W.synthetic_state(cfg, 0), cfg, DEV), DEV, max_batch=N,
                                   max_new_tokens=64, shuffle_pages=True)
    return cfg, model


@pytest.fixture(scope="module")
def pr1_model():
    from oracle import pr1
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = pr1.config()
    state = pr1.build_state(cfg)
    model = VITAMixtralForCausalLM(cfg, {"llm": W.pack_llm(state, cfg, DEV)}, DEV, max_batch=N, max_seq_len=512,
                                   max_new_tokens=64, shuffle_pages=True)
    del state
    return cfg, model


def _prompt(cfg, n, seed):
    return torch.randint(0, cfg.llm.vocab_size, (1, n), generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("which", ["tiny", "pr1"])
def test_beam_kv_bit_exact_against_replay(request, which):
    """Copy-on-write pages change nothing: every running beam's logits row equals a replay of its history on the
    static page table, for the N beams of a step run as one batch.  On the tiny config it also equals a solo
    replay at B = 1; at PR1 geometry the batched step is not batch-size invariant (the same histories on static
    pages give different rows at B = 1 and B = 4), so there only the batch replay is bit for bit."""
    cfg, model = request.getfixturevalue("tiny" if which == "tiny" else "pr1_model")
    ids = _prompt(cfg, 27, 5)                     # 27 + 40 tokens: crosses the 16-row page boundary 3 times
    search, recs, per_step = _drive(model, ids, 40)
    assert _batch_replays(model, ids, recs, per_step) == set(recs) - {()}
    if which == "tiny":
        assert _solo_replays(model, ids, recs) == set(recs)
    model.llm.reset()


def _eos_for(recs):
    """A token the beams propose often but not first: EOS then finishes hypotheses along the way."""
    counts = {}
    for h, (_, ti, _) in recs.items():
        if len(h) in (3, 4):
            for t in ti[1:4].tolist():
                counts[t] = counts.get(t, 0) + 1
    return max(counts, key=counts.get)


@pytest.mark.parametrize("lp,es", [(1.0, False), (0.0, True), (2.0, "never")])
def test_decisions_against_oracle(tiny, lp, es):
    cfg, model = tiny
    ids = _prompt(cfg, 19, 8)
    _, recs0, _ = _drive(model, ids, 24)
    eos = _eos_for(recs0)
    out = model.generate(ids, num_beams=N, num_return_sequences=N, max_new_tokens=24, eos_token_id=eos,
                         length_penalty=lp, early_stopping=es, output_scores=True)
    search, recs, per_step = _drive(model, ids, 24, eos)
    V = cfg.llm.vocab_size

    def kernel_rows(tokens, step):
        rows = torch.full((N, V), float("-inf"))
        for b, t in enumerate(tokens.tolist()):
            _, ti, tl = recs[tuple(t)]
            rows[b, ti.long()] = tl
        return rows

    seqs, scores, idx, steps = oracle_beam_search(kernel_rows, N, 24, eos, lp, es, N)
    L = ids.shape[1]
    assert torch.equal(out.sequences[:, :L].cpu(), ids.repeat(N, 1))
    assert torch.equal(out.sequences[:, L:].cpu(), seqs)
    assert torch.equal(out.sequences_scores, scores)
    assert torch.equal(out.beam_indices, idx)
    assert len(out.scores) == steps == len(per_step)
    # fp64 log_softmax of the same logits rows: each step's choice of running beams agrees unless within 2e-4
    lsm64 = {h: torch.log_softmax(r[0].double(), -1) for h, r in recs.items()}
    run64 = lambda h: sum(float(lsm64[h[:i]][h[i]]) for i in range(len(h)))
    for t, hist in enumerate(per_step[:-1]):
        cands = []
        for h in hist:
            ti = recs[h][1][:2 * N].long()
            assert (lsm64[h][ti] - recs[h][2][:2 * N].double()).abs().max() < 1e-4
            cands += [(run64(h) + float(lsm64[h][x]), h + (int(x),)) for x in ti if int(x) != eos]
        cands.sort(key=lambda c: -c[0])
        if {c[1] for c in cands[:N]} != set(per_step[t + 1]):
            assert cands[N - 1][0] - cands[N][0] < 2e-4
    # output_scores: the kernel's logprobs rounded to bf16, and fp64 log_softmax within bf16 rounding
    for t, hist in enumerate(per_step):
        blk = out.scores[t]
        assert blk.shape == (N, V) and blk.dtype == torch.bfloat16
        for b in range(N):
            h = hist[b] if t else ()
            logits, ti, tl = recs[h]
            row = blk[b].float().cpu()
            assert torch.equal(row[ti.long()], tl.to(torch.bfloat16).float())
            lsm = torch.log_softmax(logits.double(), -1)
            fin = torch.isfinite(row)
            assert fin.all()
            assert ((row.double() - lsm).abs() <= lsm.abs() * 2 ** -8 + 1e-4).all()


def test_graph_equals_eager(tiny):
    cfg, model = tiny
    ids = _prompt(cfg, 33, 9)
    kw = dict(num_beams=N, num_return_sequences=2, max_new_tokens=20, eos_token_id=7, output_scores=True)
    a = model.generate(ids, use_graph=True, **kw)
    a_scores = [s.clone() for s in a.scores]
    b = model.generate(ids, use_graph=False, **kw)
    assert torch.equal(a.sequences, b.sequences) and torch.equal(a.sequences_scores, b.sequences_scores)
    assert torch.equal(a.beam_indices, b.beam_indices)
    assert all(torch.equal(x, y) for x, y in zip(a_scores, b.scores))
    # num_beams=1 is still the greedy path
    g = model.generate(ids, max_new_tokens=5)
    assert g.sequences_scores is None and g.beam_indices is None


class _LengthStop:
    def __init__(self, L, n):
        self.L, self.n, self.calls = L, n, 0

    def __call__(self, ids, scores):
        self.calls += 1
        assert ids.shape[0] == N and len(scores) == ids.shape[1] - self.L and scores[-1].shape[0] == N
        return ids.shape[1] >= self.L + self.n


class _Boom:
    def __call__(self, ids, scores):
        if ids.shape[1] > self.at:
            raise RuntimeError("criterion failed")
        return False


def _assert_static(model):
    """The decoder holds its table at rest and a full pool (nothing reset it since generate returned)."""
    pool = model.llm.cache.pool
    pool.check()
    assert pool.table == pool.static.tolist() and pool.free == [] and all(r == 1 for r in pool.refs)
    assert torch.equal(model.llm.cache.block_table.cpu(), pool.static)


def test_demo_kwargs_with_beams():
    from tests.test_demo_replay_gpu import KeywordsStoppingCriteria, ToyTokenizer, _demo_inputs
    from vita_b200.model.builder import load_pretrained_model
    _, model, _, _ = load_pretrained_model("synthetic:tiny", None, "vita-tiny", "mixtral-8x7b", max_new_tokens=96,
                                           max_batch=N)
    tok = ToyTokenizer()
    input_ids, image_tensor, audios = _demo_inputs(model, True)
    L = input_ids.shape[1]
    kwargs = dict(images=image_tensor, audios=audios, do_sample=False, temperature=0.01, top_p=None, num_beams=N,
                  output_scores=True, return_dict_in_generate=True, use_cache=True)
    never = KeywordsStoppingCriteria([tok.glyph(model.config.llm.vocab_size - 1) * 3], tok, input_ids)
    with torch.inference_mode():
        out = model.generate(input_ids, max_new_tokens=12, stopping_criteria=[never], **kwargs)
    assert out.sequences.device == input_ids.device and out.sequences.shape == (1, L + 12)
    assert (input_ids != out.sequences[:, :L]).sum().item() == 0
    assert len(out.scores) == 12 and never.calls == 12            # every step exactly once, the last one included
    _assert_static(model)
    stop = _LengthStop(L, 5)
    with torch.inference_mode():
        out = model.generate(input_ids, max_new_tokens=12, stopping_criteria=[stop], **kwargs)
    assert stop.calls == 5 and out.sequences.shape == (1, L + 5) and len(out.scores) == 5
    _assert_static(model)
    boom = _Boom()
    boom.at = L + 3
    with pytest.raises(RuntimeError, match="criterion failed"):
        model.generate(input_ids, max_new_tokens=12, stopping_criteria=[boom], **kwargs)
    _assert_static(model)


def test_batcher_after_beam_search():
    """A beam search leaves nothing behind that the continuous batcher could trip over: the batcher's tokens after a
    generate(num_beams=4) on the same model equal those of a run before it."""
    from vita_b200.engine import ContinuousBatcher, DecoderEngine, Request
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = VitaConfig.tiny()
    packed = {"llm": W.pack_llm(W.synthetic_state(cfg, 0, parts=("llm",)), cfg, DEV)}
    model = VITAMixtralForCausalLM(cfg, packed, DEV, max_batch=N, max_seq_len=128, max_new_tokens=24,
                                   shuffle_pages=True)
    g = torch.Generator().manual_seed(4)
    spec = [(0, 9, 10), (0, 23, 8), (1, 5, 12), (2, 30, 6)]

    def requests():
        return [Request(rid, {"input_ids": torch.randint(0, cfg.llm.vocab_size, (1, plen),
                                                         generator=torch.Generator().manual_seed(100 + rid))},
                        n_new, None, arrival_step=arr) for rid, (arr, plen, n_new) in enumerate(spec)]

    eng = DecoderEngine(model)
    before = ContinuousBatcher(eng, 3).run(requests())
    beams_ids = torch.randint(0, cfg.llm.vocab_size, (1, 40), generator=g)
    beams = model.generate(beams_ids, num_beams=N, max_new_tokens=20, num_return_sequences=2)
    assert beams.sequences.shape[0] == 2
    _assert_static(model)
    after = ContinuousBatcher(eng, 3).run(requests())
    assert after == before
    # and the batcher's row swaps do not disturb a beam search: same result as on a fresh model
    again = model.generate(beams_ids, num_beams=N, max_new_tokens=20, num_return_sequences=2)
    fresh = VITAMixtralForCausalLM(cfg, packed, DEV, max_batch=N, max_seq_len=128, max_new_tokens=24,
                                   shuffle_pages=True).generate(beams_ids, num_beams=N, max_new_tokens=20,
                                                                num_return_sequences=2)
    for out in (beams, again):
        assert torch.equal(out.sequences, fresh.sequences) and torch.equal(out.sequences_scores, fresh.sequences_scores)
