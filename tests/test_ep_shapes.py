"""The expert-parallel prefill's cases, host references and flag discipline, without a GPU: the case tables are where
they claim to be, the receive-slot map is a bijection, the reduce + norm reference agrees with the oracle, and the
real rank generators (MixtralDecoder._prefill_ep_seq_steps, kernels stubbed) never issue a wait the host flag model
does not allow when stepped round-robin, while fakes that break the discipline are refused."""
import dataclasses
from collections import Counter

import pytest
import torch

from oracle import vita_oracle as O
from tests import ep_cases as C
from vita_b200 import ops
from vita_b200 import weights as W
from vita_b200.config import VitaConfig
from vita_b200.parallel import sequence_chunk

BF16 = torch.bfloat16


# ------------------------------------------------------------------------------------------------ case tables
@pytest.mark.parametrize("N,S", C.SEQ_CASES)
def test_seq_case_geometry(N, S):
    chunk = sequence_chunk(S, N)
    rt = C.rank_tokens(S, N)
    assert chunk % 8 == 0 and rt[0][0] == 0 and rt[-1][1] == S
    assert all(a[1] == b[0] for a, b in zip(rt, rt[1:]))
    assert all(t1 - t0 <= chunk for t0, t1 in rt)
    # every receive slot of every (t, k) lies inside its owner's 2 * chunk rows
    for t in range(S):
        for k in range(2):
            o, row = C.recv_slot(t, k, chunk)
            assert 0 <= o < N and 0 <= row < 2 * (rt[o][1] - rt[o][0])


def test_seq_cases_cover_the_edges():
    assert C.empty_ranks(37, 4) == [3] and C.empty_ranks(37, 8) == [5, 6, 7]
    assert C.rank_tokens(37, 2)[1] == (24, 37) and C.odd_ranks(37, 2) == [1]
    assert (13 * 8) % 16 == 8                             # rank 1's routing records end in two 4-byte words
    assert sequence_chunk(4096, 8) == 512 and not C.empty_ranks(4096, 8)
    assert sequence_chunk(300, 2) == 152 and C.rank_tokens(300, 2)[1] == (152, 300)


@pytest.mark.parametrize("N,S", C.SEQ_CASES)
def test_receive_slot_map_is_a_bijection(N, S):
    chunk = sequence_chunk(S, N)
    got = sorted(C.recv_slot(t, k, chunk) for t in range(S) for k in range(2))
    want = sorted((o, j) for o, (t0, t1) in enumerate(C.rank_tokens(S, N)) for j in range(2 * (t1 - t0)))
    assert got == want


@pytest.mark.parametrize("kind,S", [("empty+full", 37), ("empty+full", 300), ("empty+full", 4096),
                                    ("near128", 300), ("near128", 4096), ("random", 300)])
def test_routing_cases(kind, S):
    ids, tw = C.routing(kind, S, seed=1)
    assert ids.shape == (S, 2) and ids.dtype == torch.int32 and bool((ids[:, 0] != ids[:, 1]).all())
    assert bool(((ids >= 0) & (ids < C.E)).all())
    assert torch.equal(tw.sum(1), torch.ones(S)) and bool((tw > 0).all())
    counts = torch.bincount(ids.reshape(-1).long(), minlength=C.E).tolist()
    if kind == "empty+full":
        assert counts[2] == S and counts[5] == 0           # an expert with every token, a local expert with none
    if kind == "near128":
        assert counts == C.COUNTS_NEAR_128[S]
        assert sum(c % 128 not in (127, 0, 1) for c in counts) <= 1 and 0 in counts     # one count balances the sum
    offs, perm, rtok, rw, assign = C.align_ref(ids, tw)
    assert offs.tolist()[1:] == torch.cumsum(torch.tensor(counts), 0).tolist()
    flat = ids.reshape(-1)
    for i in range(2 * S):
        r = int(perm[i])
        assert int(assign[r]) == i and int(rtok[r]) == i // 2 and float(rw[r]) == float(tw.reshape(-1)[i])
        e = int(flat[i])
        assert int(offs[e]) <= r < int(offs[e + 1])
    for e in range(C.E):                                   # stable: assignment order inside each expert
        a = assign[int(offs[e]):int(offs[e + 1])]
        assert bool((a[1:] > a[:-1]).all())


# ------------------------------------------------------------------------------------------------ references
@pytest.mark.parametrize("H", [512, 4096])
def test_reduce_norm_reference_matches_the_oracle(H):
    g = torch.Generator().manual_seed(H)
    h = (torch.randn(9, H, generator=g) * 0.5).to(BF16)
    s0 = (torch.randn(9, H, generator=g) * 0.1).to(BF16)
    s1 = (torch.randn(9, H, generator=g) * 0.1).to(BF16)
    w = (1.0 + 0.1 * torch.randn(H, generator=g)).to(BF16)
    hp = C.reduce_ref(h, s0, s1)
    assert torch.equal(hp.float(), (h.float() + (s0.float() + s1.float())).to(BF16).float())
    got = C.rmsnorm64(hp, w, 1e-5)
    want = O.rmsnorm(hp, w, 1e-5).double()
    assert float(((got - want).abs().amax(-1) / want.abs().amax(-1)).max()) < 1e-6


def test_random_packed_ep_equals_sliced_full_weights():
    cfg = VitaConfig.tiny()
    full = W.random_packed(cfg, "cpu", seed=3, parts=("llm",))["llm"]
    for N in (2, 4, 8):
        for r in range(N):
            part = W.random_packed(cfg, "cpu", seed=3, parts=("llm",), ep=(r, N))["llm"]
            want = C.rank_weights(full, r, N)
            assert part["ep"] == want["ep"] == (r, N)
            for lp, lw in zip(part["layers"], want["layers"]):
                assert lp.keys() == lw.keys()
                for k in lp:
                    assert torch.equal(lp[k], lw[k]), (N, r, k)
                    assert lw[k].is_contiguous()
            for k in ("embed", "norm", "lm_head"):
                assert torch.equal(part[k], full[k])


# ------------------------------------------------------------------------------------------------ flag model
class Launches:
    """Stand-in for the real EP ops: records what would have been launched."""

    def __init__(self):
        self.log = []

    def ep_signal(self, ptrs, which, n_ranks, my_rank, epoch):
        self.log.append(("signal", my_rank, which, epoch))

    def ep_wait(self, flags, which, n_ranks, epoch, n_wait=None):
        self.log.append(("wait", flags, which, epoch))

    def ep_reduce_norm_gather(self, rs, flags, hp, xp, w, tok0, n_owned, n_ranks, my_rank, epoch, H, eps, gather=True):
        self.log.append(("reduce", my_rank, n_owned, epoch))


def fake_rank(ops_, r, N, S, L, fault=None):
    """A rank that follows the yield structure of MixtralDecoder._prefill_ep_seq_steps (flags handle = rank), or,
    with `fault`, breaks it: waits for the routed rows before yielding, waits for an epoch ahead, never signals that
    its expert rows have landed, or signals the routed rows in the K/V group."""
    t0, t1 = C.rank_tokens(S, N)[r]
    n = t1 - t0
    for li in range(L):
        ep = li + 1
        ops_.ep_signal(None, 2, N, r, ep)
        yield
        ops_.ep_wait(r, 2, N, ep + (fault == "epoch_ahead"), n_wait=r)
        ops_.ep_signal(None, 2 if fault == "wrong_group" else 3, N, r, ep)
        if fault != "wait_before_yield":
            yield
        ops_.ep_wait(r, 3, N, ep)
        if fault != "no_signal":
            ops_.ep_signal(None, 0, N, r, ep)
        yield
        ops_.ep_reduce_norm_gather(None, r, None, None, None, t0, n, N, r, ep, 512, 1e-5, gather=False)
        if n == 0:
            ops_.ep_wait(r, 0, N, ep)
        if fault == "wait_before_yield":
            yield
    return r


@pytest.mark.parametrize("N,S", C.SEQ_CASES)
def test_round_robin_fakes_satisfy_every_wait(N, S):
    model, rec = C.FlagModel(N), Launches()
    g = C.guarded_ops(model, rec, rank_of=lambda f: f)
    ops_ = type("Guarded", (), {k: staticmethod(v) for k, v in g.items()})
    assert C.step_round_robin([fake_rank(ops_, r, N, S, 2) for r in range(N)]) == list(range(N))
    want = torch.zeros(N, 4 * N, dtype=torch.int32)
    for which in C.WHICH:
        want[:, which * N:(which + 1) * N] = 2
    assert torch.equal(model.table(), want)
    waits = [e for e in rec.log if e[0] == "wait"]
    assert len(waits) == N * 2 * 2 + 2 * len(C.empty_ranks(S, N))


@pytest.mark.parametrize("fault", ["wait_before_yield", "epoch_ahead", "no_signal", "wrong_group"])
@pytest.mark.parametrize("N,S", [(2, 37), (4, 37), (8, 300)])
def test_guard_refuses_a_broken_rank_before_launch(N, S, fault):
    """One rank breaks the discipline (rank N - 1 for the epoch, whose K/V wait needs every other rank; rank 0, which
    runs first in every phase, otherwise): the guard raises and the wait it refused is not in the launch log."""
    model, rec = C.FlagModel(N), Launches()
    g = C.guarded_ops(model, rec, rank_of=lambda f: f)
    tries = []

    def counted(fn):
        return lambda *a, **k: (tries.append(a), fn(*a, **k))
    ops_ = type("Guarded", (), {k: staticmethod(v if k == "ep_signal" else counted(v)) for k, v in g.items()})
    bad = N - 1 if fault in ("epoch_ahead", "no_signal") else 0
    gens = [fake_rank(ops_, r, N, S, 2, fault if r == bad else None) for r in range(N)]
    with pytest.raises(C.FlagNotSet):
        C.step_round_robin(gens)
    launched = [e for e in rec.log if e[0] != "signal"]
    assert len(launched) == len(tries) - 1, "the refused wait was launched"


# ---- the real rank generators, every kernel stubbed
EP_OPS = ("ep_signal", "ep_wait", "ep_reduce_norm_gather")
STUBBED = ("rmsnorm", "linear_qkv_rope", "ep_push", "attention", "linear", "moe_router", "moe_align", "row_copy",
           "moe_gate_up", "moe_down_ep", "tc_lm_head_argmax")


def _stub_decoders(monkeypatch, cfg, N, S):
    from vita_b200.model.mixtral import MixtralDecoder
    monkeypatch.setattr(ops, "decode_attention_workspace", lambda B, nkv, sp, dev: torch.zeros(1, dtype=torch.uint8))
    monkeypatch.setattr(ops, "TcWorkspace", lambda B, rb, dev: None)
    pushes = []
    for name in STUBBED:
        monkeypatch.setattr(ops, name, (lambda *a, **k: pushes.append(a)) if name == "ep_push" else
                            (lambda *a, **k: None))
    c, L = cfg, cfg.num_hidden_layers
    z = lambda *s: torch.zeros(*s, dtype=BF16)
    w = {"embed": z(1, 1), "norm": z(1), "lm_head": z(1, 1), "rope": W.rope_table(S + 64, c.head_dim, c.rope_theta),
         "layers": [{"ln1": z(1), "wqkv": z(1, 1), "wo": z(1, 1), "ln2": z(1), "gate": z(1, 1),
                     "w13": z(C.E, 1, 1), "w2": z(C.E, 1, 1)} for _ in range(L)]}
    peers = C.LocalPeers(N, "cpu")
    decs = [MixtralDecoder(c, C.rank_weights(w, r, N), "cpu", max_seq_len=S + 64, max_new_tokens=8,
                           ep_alloc=peers.alloc(r)) for r in range(N)]
    return decs, pushes


@pytest.mark.parametrize("N,S", C.SEQ_CASES)
def test_real_rank_generators_keep_the_flag_discipline(monkeypatch, N, S):
    """MixtralDecoder._prefill_ep_seq_steps of N ranks with stubbed kernels, stepped round-robin under the guard: no
    wait is refused, three phases per layer, and the host flags end at the last epoch in every group; the pushes of
    all ranks tile each all-gathered region (K/V pages of every layer, xn2, ids, tw) exactly once."""
    cfg = dataclasses.replace(VitaConfig.tiny().llm, max_position_embeddings=8192)
    decs, pushes = _stub_decoders(monkeypatch, cfg, N, S)
    model, rec = C.FlagModel(N), Launches()
    by_ptr = {d.ep_p2p["flags"].data_ptr(): r for r, d in enumerate(decs)}
    for name, fn in C.guarded_ops(model, rec, lambda f: by_ptr[f.data_ptr()]).items():
        monkeypatch.setattr(ops, name, fn)
    gens = [d._prefill_ep_seq_steps(torch.zeros(S, cfg.hidden_size, dtype=BF16), 0, True, False) for d in decs]
    out = C.step_round_robin(gens)
    # (the stubbed LM head returns None; a token-less rank returns its empty logits without one)
    assert [o is not None and o.shape[0] == 0 for o in out] == [t1 == t0 for t0, t1 in C.rank_tokens(S, N)]
    L = cfg.num_hidden_layers
    want = torch.zeros(N, 4 * N, dtype=torch.int32)
    for which in C.WHICH:
        want[:, which * N:(which + 1) * N] = L
    assert torch.equal(model.table(), want)
    signals = [e for e in rec.log if e[0] == "signal"]
    assert len(signals) == 3 * L * N
    # the pushed byte ranges: every region exactly covered, rank by rank
    sy, H = decs[0].ep_p2p, cfg.hidden_size
    off, kvl, kvr = sy["off"], sy["kv_layer"], sy["kv_row"]
    regions = {"xn2": (off["xn2"], S * H * 2), "ids": (off["ids"], S * 8), "tw": (off["tw"], S * 8)}
    for li in range(L):
        ko = off["kv"] + 2 * li * kvl
        regions[f"k{li}"], regions[f"v{li}"] = (ko, S * kvr), (ko + kvl, S * kvr)
    got = Counter()
    for base_ptrs, ranges, n_ranks, my_rank in pushes:
        assert n_ranks == N and len(ranges) <= 4 and ranges
        got.update((o, b) for o, b in ranges)
    assert all(b > 0 for _, b in got)                       # a token-less rank pushes nothing
    for name, (o0, nb) in regions.items():
        mine = sorted(r for r in got if o0 <= r[0] < o0 + nb)
        assert all(got[r] == (1 if name[0] in "kv" else L) for r in mine), name     # K/V once, routed rows per layer
        pos = o0
        for o, b in mine:
            assert o == pos and o % 16 == 0 and b % 4 == 0, (name, o, b, pos)
            pos += b
        assert pos == o0 + nb, (name, pos - o0, nb)
    assert sum(got.values()) == 5 * L * (N - len(C.empty_ranks(S, N)))     # nothing pushed outside the regions
