"""The expert-parallel prefill on one H100.

A. Its kernels against host references, with every "peer" an ordinary allocation on the one device:
   moe_down_ep (every (token, k) row in its owner's receive slot, bit for bit moe_down over the same offsets, close to
   fp64), ep_push (exact bytes in every peer, canaries intact), ep_signal / ep_wait, ep_reduce_norm_gather (gather=0:
   h bit-exact against the fp32 host sum, xn against fp64 RMSNorm) and the refusals that launch nothing.
B. The whole sequence-sharded prefill with N emulated ranks (tests/ep_cases.run_ep_prefill) against the single-GPU
   MixtralDecoder with the same weights: logits, first token, K/V pages, the all-gathered routed rows and the flags.

Every wait is launched only on flags that are already set (the host flag model of ep_cases refuses anything else),
so no kernel here can spin."""
import pytest
import torch

from tests import ep_cases as C
from tests.util import close_rows, same_bits
from vita_b200 import _lib, ops
from vita_b200 import weights as W
from vita_b200.config import VitaConfig
from vita_b200.model.mixtral import MixtralDecoder
from vita_b200.parallel import sequence_chunk
from vita_b200.weights import expert_range

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
DEV = "cuda"
E = C.E
NAN = float("nan")
# one bf16 rounding (unit roundoff 2^-8 of the largest element of a row) plus room for the fp32 accumulation
ROW_REL = 2.0 ** -8 * 1.03


def _ptrs(bufs):
    return torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device=DEV)


def _i32(t):
    return t.to(DEV, torch.int32).contiguous()


# ------------------------------------------------------------------------------------------------ A. moe_down_ep
DOWN_CASES = [("tiny", 37, "empty+full"), ("tiny", 300, "near128"), ("tiny", 300, "random"),
              ("full", 4096, "near128"), ("full", 4096, "empty+full")]
WIDTH = {"tiny": (512, 1024), "full": (4096, 14336)}


@pytest.fixture(scope="module")
def down_weights():
    """w2 [E, H, I] and activations [8192, I] per width, drawn once (bf16, |w| ~ 0.02, |act| ~ 1)."""
    out = {}

    def get(width):
        if width not in out:
            H, I = WIDTH[width]
            g = torch.Generator(device=DEV).manual_seed(H)
            w2 = (torch.randn(E, H, I, device=DEV, generator=g) * 0.02).to(BF16)
            act = torch.randn(8192, I, device=DEV, generator=g).to(BF16)
            out[width] = (w2, act)
        return out[width]
    yield get
    out.clear()


def _down_ep(act, w2l, offs_l, rw, assign, chunk, N, rows, H):
    """One rank's moe_down_ep into N NaN-filled receive buffers of 2 * chunk + 8 rows (the last 8: canaries)."""
    recv = [torch.full((2 * chunk + 8, H), NAN, dtype=BF16, device=DEV) for _ in range(N)]
    ops.moe_down_ep(act, w2l, offs_l, rw, assign, _ptrs(recv), rows, chunk)
    torch.cuda.synchronize()
    return recv


@pytest.mark.parametrize("width,S,kind", DOWN_CASES)
def test_moe_down_ep_rows_land_in_their_owners_slots(width, S, kind, down_weights, monkeypatch):
    H, I = WIDTH[width]
    w2, act_all = down_weights(width)
    rows = 2 * S
    act = act_all[:rows]
    ids, tw = C.routing(kind, S, seed=S)
    offs, perm, rtok, rw, assign = C.align_ref(ids, tw)
    # the kernel's own align gives the same plan
    d = dict(offs=torch.empty(E + 1, dtype=torch.int32, device=DEV), perm=torch.empty(rows, dtype=torch.int32, device=DEV),
             rtok=torch.empty(rows, dtype=torch.int32, device=DEV), rw=torch.empty(rows, dtype=torch.float32, device=DEV),
             assign=torch.empty(rows, dtype=torch.int32, device=DEV))
    ops.moe_align(_i32(ids), tw.to(DEV), d["offs"], d["perm"], d["rtok"], d["rw"], S, E, row_assign=d["assign"])
    for k, v in zip(("offs", "perm", "rtok", "rw", "assign"), (offs, perm, rtok, rw, assign)):
        assert torch.equal(d[k].cpu(), v), k
    ref64, ref_rows = C.down_ref64(act, w2, offs, d["rw"], 0, E)
    row64 = torch.full((rows, H), NAN, dtype=torch.float64, device=DEV)
    row64[ref_rows.to(DEV)] = ref64
    t, k = (assign // 2).long(), (assign % 2).long()
    worst = 0.0
    for N in (2, 4, 8):
        chunk = sequence_chunk(S, N)
        owner = t // chunk
        slot = (t - owner * chunk) * 2 + k
        for r in range(N):
            lo, hi = expert_range(E, r, N)
            r0, r1 = int(offs[lo]), int(offs[hi])
            w2l, offs_l = w2[lo:hi], d["offs"][lo:]
            y = torch.full((rows, H), NAN, dtype=BF16, device=DEV)
            ops.moe_down(act, w2l, y, offs_l, d["rw"], rows)
            recv = _down_ep(act, w2l, offs_l, d["rw"], d["assign"], chunk, N, rows, H)
            # expected receive buffers: NaN except the slots of this rank's rows, which hold moe_down's rows
            want = [torch.full_like(b, NAN) for b in recv]
            for o in range(N):
                m = (owner[r0:r1] == o).nonzero().view(-1) + r0
                want[o][slot[m].to(DEV)] = y[m.to(DEV)]
            for o in range(N):
                same_bits(recv[o], want[o], f"{width} S={S} {kind} N={N} rank {r}: receive buffer of rank {o}")
            if r1 > r0:
                worst = max(worst, close_rows(y[r0:r1], row64[r0:r1], f"{width} S={S} {kind} N={N} rank {r}",
                                              lambda i: f"row {r0 + i[0]}", rel=ROW_REL))
            # the same bits without the tail split and with the 128-wide tile
            for env, val in (("VITA_B200_GEMM_TAIL_SPLIT", "0"), ("VITA_B200_GEMM_BN", "128")):
                with monkeypatch.context() as mp:
                    mp.setenv(env, val)
                    again = _down_ep(act, w2l, offs_l, d["rw"], d["assign"], chunk, N, rows, H)
                for o in range(N):
                    same_bits(again[o], recv[o], f"{env}={val} N={N} rank {r} -> rank {o}")
    print(f"\nEPSTAT down_ep {width} S={S} {kind}: worst row err vs fp64 {worst:.3e}")


# ------------------------------------------------------------------------------------------------ A. ep_push
PUSH_SETS = {
    "empty": [0],
    "words": [4, 8, 12],
    "tails": [16, 16 * 5 + 4, 16 * 9 + 8, 16 * 3 + 12],
    "xn2+records": [300 * 4096 * 2, 13 * 8, 13 * 8, 0],       # several MB of rows, then odd-count routing records
    "one-long": [16 * 1000 + 12],
}


def _layout(sizes):
    """16-byte aligned offsets with a 64-byte canary gap before each range."""
    offs, pos = [], 64
    for b in sizes:
        offs.append(pos)
        pos = (pos + b + 15) // 16 * 16 + 64
    return list(zip(offs, sizes)), pos + 64


@pytest.mark.parametrize("n_ranks", [2, 3, 8, 32])
@pytest.mark.parametrize("name", list(PUSH_SETS))
def test_ep_push_copies_exact_bytes_into_every_peer(n_ranks, name):
    ranges, total = _layout(PUSH_SETS[name])
    g = torch.Generator(device=DEV).manual_seed(n_ranks)
    orig = [torch.randint(0, 256, (total,), dtype=torch.uint8, device=DEV, generator=g) for _ in range(n_ranks)]
    bufs = [o.clone() for o in orig]
    ptrs = _ptrs(bufs)
    for me in range(n_ranks):
        for b, o in zip(bufs, orig):
            b.copy_(o)
        ops.ep_push(ptrs, ranges, n_ranks, me)
        torch.cuda.synchronize()
        for p in range(n_ranks):
            want = orig[p].clone()
            if p != me:
                for o, nb in ranges:
                    want[o:o + nb] = orig[me][o:o + nb]
            assert torch.equal(bufs[p], want), f"{name}: rank {me} -> rank {p}" + (" (own buffer)" if p == me else "")


# ------------------------------------------------------------------------------------------------ A. signal / wait
@pytest.mark.parametrize("n_ranks", [2, 3, 8, 32])
def test_ep_signal_sets_one_flag_in_every_peer(n_ranks):
    N = n_ranks
    flags = [torch.full((4 * N + 8,), -7, dtype=torch.int32, device=DEV) for _ in range(N)]
    for f in flags:
        f[:4 * N] = 0
    model = C.FlagModel(N)
    by_ptr = {f.data_ptr(): r for r, f in enumerate(flags)}
    g = C.guarded_ops(model, ops, lambda f: by_ptr[f.data_ptr()])
    ptrs = _ptrs(flags)
    want = torch.zeros(N, 4 * N + 8, dtype=torch.int32)
    want[:, 4 * N:] = -7
    for which in C.WHICH:
        epoch = 3 + which
        for me in range(N):
            g["ep_signal"](ptrs, which, N, me, epoch)
            want[:, which * N + me] = epoch
            assert torch.equal(torch.stack(flags).cpu(), want), f"which {which}, rank {me}"
        for r in range(N):                      # every flag of the group is set now: these waits return at once
            g["ep_wait"](flags[r], which, N, epoch)
            g["ep_wait"](flags[r], which, N, epoch, n_wait=r)
        torch.cuda.synchronize()
        with pytest.raises(C.FlagNotSet):       # ... and one for the next epoch is refused before launch
            g["ep_wait"](flags[0], which, N, epoch + 1)
    assert torch.equal(torch.stack(flags).cpu()[:, :4 * N], model.table())


# ------------------------------------------------------------------------------------------------ A. reduce + norm
# (N, my_rank, tok0, n_owned): one token; the 13 odd tokens of rank 1 at S = 37, N = 2; a full chunk of 512
REDUCE_CASES = [(2, 1, 24, 1), (2, 1, 24, 13), (8, 1, 512, 512), (4, 3, 48, 7)]


@pytest.mark.parametrize("H", [512, 4096])
@pytest.mark.parametrize("N,me,tok0,n", REDUCE_CASES)
@pytest.mark.parametrize("norm", [True, False], ids=["norm", "no-norm"])
def test_ep_reduce_norm_gather_owner_rows(H, N, me, tok0, n, norm):
    eps, epoch = 1e-5, 5
    rows = tok0 + n + 16                           # rows past the owned ones: canaries
    g = torch.Generator(device=DEV).manual_seed(H + n)
    # every other owned token (the last one included) is tiny, so that eps carries weight in its norm
    tiny = torch.ones(rows, 1, device=DEV)
    tiny[tok0 + (n - 1) % 2:tok0 + n:2] = 1e-3
    h0 = [(torch.randn(rows, H, device=DEV, generator=g) * tiny).to(BF16) for _ in range(N)]
    h = [x.clone() for x in h0]
    xn = [torch.full((rows, H), NAN, dtype=BF16, device=DEV) for _ in range(N)]
    slot_scale = tiny[tok0:tok0 + n].repeat_interleave(2, 0)
    rs = (torch.randn(2 * n + 4, H, device=DEV, generator=g) * 0.5)
    rs[:2 * n] *= slot_scale
    rs = rs.to(BF16)
    rs[1:2 * n:2][:, ::3] = -rs[0:2 * n:2][:, ::3]         # slot sums that cancel exactly
    w = (1.0 + 0.1 * torch.randn(H, device=DEV, generator=g)).to(BF16) if norm else None
    flags = [torch.zeros(4 * N, dtype=torch.int32, device=DEV) for _ in range(N)]
    model = C.FlagModel(N)
    flags[me][:N] = epoch                          # preset: every rank's expert rows of this epoch have landed
    for src in range(N):
        model.flags[me][src] = epoch
    by_ptr = {f.data_ptr(): r for r, f in enumerate(flags)}
    gd = C.guarded_ops(model, ops, lambda f: by_ptr[f.data_ptr()])
    gd["ep_reduce_norm_gather"](rs, flags[me], _ptrs(h), _ptrs(xn), w, tok0, n, N, me, epoch, H, eps, gather=False)
    torch.cuda.synchronize()
    hp = C.reduce_ref(h0[me][tok0:tok0 + n].cpu(), rs[0:2 * n:2].cpu(), rs[1:2 * n:2].cpu())
    want_h = h0[me].clone()
    want_h[tok0:tok0 + n] = hp.to(DEV)
    same_bits(h[me], want_h, "owner's h rows (and the rows around them)")
    for r in range(N):
        if r != me:
            same_bits(h[r], h0[r], f"h of rank {r}")
            assert bool(xn[r].isnan().all()), f"xn of rank {r} was written"
    if norm:
        want = C.rmsnorm64(hp.to(DEV), w, eps)
        err = close_rows(xn[me][tok0:tok0 + n], want, "xn", lambda i: f"token {tok0 + i[0]}", rel=ROW_REL)
        print(f"\nEPSTAT reduce H={H} N={N} n={n}: worst xn row err vs fp64 {err:.3e}")
        outside = torch.cat([xn[me][:tok0], xn[me][tok0 + n:]])
        assert bool(outside.isnan().all()), "xn written outside the owned rows"
    else:
        assert bool(xn[me].isnan().all()), "xn written without a norm weight"


# ------------------------------------------------------------------------------------------------ A. refusals
def test_ep_refusals_launch_nothing():
    """Bad arguments raise before any launch.  Every flag is already far past the epoch and every buffer is large, so
    even a launch that slipped through would neither spin nor leave its buffers."""
    n_max = 40
    bufs = [torch.zeros(1 << 20, dtype=torch.uint8, device=DEV) for _ in range(n_max)]
    snap = [b.clone() for b in bufs]
    ptrs = _ptrs(bufs)
    flags = torch.full((4 * n_max,), 1 << 20, dtype=torch.int32, device=DEV)
    h = torch.zeros(64, 8192, dtype=BF16, device=DEV)
    hp = _ptrs([h] * n_max)
    refused = [
        ("more than 4 ranges", lambda: ops.ep_push(ptrs, [(0, 16)] * 5, 2, 0)),
        ("unaligned offset", lambda: ops.ep_push(ptrs, [(8, 16)], 2, 0)),
        ("bytes % 4", lambda: ops.ep_push(ptrs, [(0, 6)], 2, 0)),
        ("negative bytes", lambda: ops.ep_push(ptrs, [(0, -4)], 2, 0)),
        ("push to 0 ranks", lambda: ops.ep_push(ptrs, [(0, 16)], 0, 0)),
        ("push to 33 ranks", lambda: ops.ep_push(ptrs, [(0, 16)], 33, 0)),
        ("signal 0 ranks", lambda: ops.ep_signal(ptrs, 0, 0, 0, 1)),
        ("signal 33 ranks", lambda: ops.ep_signal(ptrs, 0, 33, 0, 1)),
        ("wait 0 ranks", lambda: ops.ep_wait(flags, 0, 0, 1)),
        ("wait 33 ranks", lambda: ops.ep_wait(flags, 0, 33, 1)),
        ("n_wait > n_ranks", lambda: ops.ep_wait(flags, 0, 2, 1, n_wait=3)),
        ("reduce 0 ranks", lambda: ops.ep_reduce_norm_gather(h, flags, hp, hp, None, 0, 1, 0, 0, 1, 512, 1e-5, False)),
        ("reduce 33 ranks", lambda: ops.ep_reduce_norm_gather(h, flags, hp, hp, None, 0, 1, 33, 0, 1, 512, 1e-5, False)),
        ("H % 8", lambda: ops.ep_reduce_norm_gather(h, flags, hp, hp, None, 0, 1, 2, 0, 1, 516, 1e-5, False)),
        ("H > 4096", lambda: ops.ep_reduce_norm_gather(h, flags, hp, hp, None, 0, 1, 2, 0, 1, 4104, 1e-5, False)),
    ]
    torch.cuda.synchronize()
    before = ops.launch_count()
    for what, call in refused:
        with pytest.raises(_lib.VitaB200Error):
            call()
        assert ops.launch_count() == before, f"{what}: launched"
    torch.cuda.synchronize()
    assert all(torch.equal(b, s) for b, s in zip(bufs, snap)) and bool((h == 0).all())


# ------------------------------------------------------------------------------------------------ B. whole prefill
PREFILL_CASES = [("tiny", N, S) for N in (2, 4, 8) for S in (37, 300)] + [("full2", 2, 300), ("full1", 8, 4096)]
CONFIGS = {"tiny": VitaConfig.tiny, "full2": lambda: VitaConfig.full(2), "full1": lambda: VitaConfig.full(1)}


@pytest.mark.parametrize("name,N,S", PREFILL_CASES)
def test_emulated_ep_prefill_matches_single_gpu(name, N, S, monkeypatch):
    cfg = CONFIGS[name]().llm
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    w = W.random_packed(CONFIGS[name](), DEV, seed=3, parts=("llm",))["llm"]
    g = torch.Generator(device=DEV).manual_seed(11)
    emb = (torch.randn(S, cfg.hidden_size, device=DEV, generator=g) * 0.05).to(BF16)
    ref = MixtralDecoder(cfg, w, DEV, max_seq_len=S + 64, max_new_tokens=8)
    want = ref.prefill(emb.clone(), slot=0, all_logits=True)
    best = int(ref.best[0])
    ref_kv = [(ref.cache.k[l][:S], ref.cache.v[l][:S]) for l in range(cfg.num_hidden_layers)]
    del ref
    got = C.run_ep_prefill(cfg, w, N, emb, monkeypatch)
    same_bits(torch.cat(got["logits"]), want, f"{name} N={N} S={S}: logits of the own rows")
    owner = [r for r, (t0, t1) in enumerate(C.rank_tokens(S, N)) if t0 <= S - 1 < t1]
    assert got["best"] == [best if r in owner else 0 for r in range(N)], "first token"
    for r in range(N):
        for l, (k, v) in enumerate(ref_kv):
            same_bits(got["kv"][r][l][0], k, f"rank {r} layer {l}: K pages")
            same_bits(got["kv"][r][l][1], v, f"rank {r} layer {l}: V pages")
        for key in ("xn2", "ids", "tw"):
            same_bits(got[key][r], got[key][0], f"rank {r}: {key} differs from rank 0's")
        assert torch.equal(got["flags"][r], got["model"].table()[r]), f"rank {r}: device flags vs host model"
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"\nEPSTAT prefill {name} N={N} S={S}: bit-identical, peak {peak:.2f} GiB")
