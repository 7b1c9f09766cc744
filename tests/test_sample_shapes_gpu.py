"""The sampler (csrc/sample.cu: ops.sample_rows / ops.sample_logprobs) at the shapes and edges that serve, against the
fp64 oracle (oracle/sampling_oracle.py, tests/logprobs_oracle.py) token by token (inputs: tests/sample_cases.py; their
CPU checks: tests/test_sample_shapes.py).

Most checks read the plain variant's score log.  There, a kept token holds bf16(fp32(l) / fp32(T)) and a dropped one
-inf; the kernel divides with __fdiv_rn and the host with torch's CPU fp32 division, and both round to bf16 to nearest
even, so the log is compared bit for bit.  Greedy rows log the logits' bits.

A. Top-k kept sets, exact, at every placement of the k-th largest key and k in {1, 2, 255, 256, 257, V-1, V, V+1};
   -0.0 / +0.0 at the threshold; rows masked to -inf; logits whose bf16(l / T) a reciprocal multiply would change.
B. Top-p kept sets, token by token: only tokens with |above - p| < tol (sample_cases.topp_tol) may differ, and equal
   values are kept or dropped together.  Thresholds at chosen keys, with and without a top-k floor in the same bin.
C. Draws: the packed best word against the oracle's draw where the perturbed-score gap is clear; the prune rows
   (sub-maximum winners up to 16 below x_max) always.
D. Layouts: V from 1 to the shared-memory limit V_max (read from the refusal at an oversize V), rows as views into a
   NaN-filled buffer (ld = V + 8: the vectorised staging path; ld = V + 1 and a one-element offset: the scalar path),
   bit-identical to the contiguous launch; V_max against the oracle, V_max + 8 refused.
E. Logprobs: logprob, rank and top-N on tie rows whose group spans chunks 0, 17 and 50 and V - 1, with -0.0 / +0.0
   inside; the LSM score row against logprobs_oracle's row; targets at 0, V - 1, outside the kept set and >= V; a
   canary-filled score log written at row counter[b] only.
F. One launch of B = 64 and of B = 256 mixing all of the above with per-row parameters and streams: every row has the
   bits of its solo launch, and the plain, LOGPROBS and LSM variants agree on the best word and the kept set.
"""
import functools

import numpy as np
import pytest
import torch

from tests import sample_cases as C
from tests.logprobs_oracle import logprobs as oracle_logprobs
from vita_b200 import _lib, ops

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF16 = torch.bfloat16
NAN16 = 0x7FC1                     # bf16 NaN: its key sorts above +inf, so a read past V becomes the row maximum
FILL = 0x7FA5                      # score-log canary: a NaN with a payload no kernel writes
ATOL = 1e-4                        # logprobs (fp32 x - x_max - log Z) against fp64, plus fp32_slack
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(WORST):
        print(f"sampler worst {key}: {WORST[key]:.3e}")


def _note(key, v):
    WORST[key] = max(WORST.get(key, 0.0), float(v))


@functools.lru_cache(maxsize=None)
def _cases(family, V=4096):
    return {"topk": C.topk_cases, "topp": C.topp_cases, "zeros": C.zeros_cases, "masked": C.masked_cases,
            "prune": C.prune_cases, "topn": C.topn_cases, "division": C.division_cases}[family](V)


def _prm(cases, streams=None):
    f = lambda v, dt: torch.as_tensor(v, dtype=dt).to(DEV)
    seeds = [c.seed - 2 ** 64 if c.seed >= 2 ** 63 else c.seed for c in cases]
    return (f([C.f32(c.T) for c in cases], torch.float32), f([c.k for c in cases], torch.int32),
            f([C.f32(c.p) for c in cases], torch.float32), f(seeds, torch.int64), f([c.n for c in cases], torch.int32))


def _log_rows(cases):
    return max(c.n for c in cases) + 1


def _canary(shape):
    return torch.full(shape, FILL, dtype=torch.int16, device=DEV).view(BF16)


def _plain(logits, cases, streams=None):
    """-> (best [B] int64, score log rows [B, V] (row counter[b] of each request)"""
    B = len(cases)
    prm = _prm(cases)
    best = torch.zeros(B, dtype=torch.int64, device=DEV)
    rows = _log_rows(cases)
    log = _canary((B, rows, logits.shape[1]))
    st = None if streams is None else torch.tensor(streams, dtype=torch.int32, device=DEV)
    ops.sample_rows(logits, *prm, best, log, streams=st)
    n = torch.tensor([c.n for c in cases], device=DEV)
    return best.cpu(), log[torch.arange(B, device=DEV), n].cpu(), log


def _lp(logits, cases, n_top=0, target=None, lsm=False, streams=None, scores=True):
    B = len(cases)
    prm = _prm(cases)
    best = torch.zeros(B, dtype=torch.int64, device=DEV)
    lp = torch.full((B,), 7.0, device=DEV)
    rank = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    ids = torch.full((B, 20), -7, dtype=torch.int32, device=DEV)
    tl = torch.full((B, 20), 7.0, device=DEV)
    log = _canary((B, _log_rows(cases), logits.shape[1])) if scores else None
    tg = None if target is None else torch.tensor(target, dtype=torch.int32, device=DEV)
    st = None if streams is None else torch.tensor(streams, dtype=torch.int32, device=DEV)
    ops.sample_logprobs(logits, *prm, best, lp, rank, ids, tl, n_top, target=tg, scores=log, log_softmax_scores=lsm,
                        streams=st)
    out = dict(best=best.cpu(), lp=lp.cpu(), rank=rank.cpu(), ids=ids.cpu(), tl=tl.cpu())
    if scores:
        n = torch.tensor([c.n for c in cases], device=DEV)
        out["srow"] = log[torch.arange(B, device=DEV), n].cpu()
    return out


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32) if t.dtype == torch.float32 else t


def _kept_of(case, srow):
    """the kernel's kept set from a plain score-log row (a -inf logit logs -inf either way: taken as the oracle's)"""
    got = torch.isfinite(srow.float()).numpy()
    masked = np.isneginf(case.row)
    _, kept, _ = case.warp()
    return np.where(masked, kept, got)


def _check_row(case, srow):
    """-> list of problems of one plain score-log row against the oracle (empty = pass)"""
    _, kept, _ = case.warp()
    exempt = C.topp_exempt(case)
    got = _kept_of(case, srow)
    bad = []
    diff = (got != kept) & ~exempt
    if diff.any():
        i = np.flatnonzero(diff)[:4]
        bad.append(f"{case.name}: kept set differs at {i.tolist()} (values {case.row[i].tolist()}, kernel "
                   f"{got[i].tolist()})")
    fin = np.isfinite(case.row)
    vals = np.where(case.row == 0, 0.0, case.row)                  # -0.0 and +0.0 are one value
    for v in np.unique(vals[fin & got]):
        grp = fin & (vals == v)
        if not got[grp].all():
            bad.append(f"{case.name}: tie group {v} split")
            break
    want = C.expected_scores(case, np.where(exempt, got, kept))
    if not torch.equal(_bits(srow), _bits(want)):
        i = torch.nonzero(_bits(srow) != _bits(want))[:4, 0].tolist()
        bad.append(f"{case.name}: score bits differ at {i}: {srow[i].tolist()} vs {want[i].tolist()}")
    _note("top-p exempt tokens per row", exempt.sum())
    return bad


def _run_family(cases):
    logits = C.stack(cases).to(DEV)
    best, srows, _ = _plain(logits, cases)
    return best, srows


# ------------------------------------------------------------------------------------------------ A / B. kept sets
@pytest.mark.parametrize("family", ["topk", "topp", "zeros", "masked", "division"])
def test_kept_sets(family):
    cases = _cases(family)
    _, srows = _run_family(cases)
    bad = [m for c, s in zip(cases, srows) for m in _check_row(c, s)]
    assert not bad, "\n".join(bad[:12])


@pytest.mark.parametrize("T", C.T_SAMPLED + C.T_GREEDY)
def test_kept_sets_every_temperature(T):
    """each placement family at every temperature, greedy ones included (the score log then holds the logits)"""
    cases = [C.Case(c.family, f"{c.name}-T{T}", c.row, T, c.k, c.p, c.seed, c.n, c.meta)
             for c in _cases("topk")[::3] + _cases("topp")[::2] + _cases("zeros")[::2]]
    best, srows = _run_family(cases)
    bad = [m for c, s in zip(cases, srows) for m in _check_row(c, s)]
    assert not bad, "\n".join(bad[:12])
    if not C.f32(T) > 0:
        am = torch.zeros(len(cases), dtype=torch.int64, device=DEV)
        ops.argmax_rows(C.stack(cases).to(DEV), am)
        assert torch.equal(best, am.cpu())                                # greedy = argmax_rows, bit for bit
        assert best.tolist() == [C.pack_word(c.row, int(np.argmax(np.where(c.row == 0, 0.0, c.row)))) for c in cases]


# ------------------------------------------------------------------------------------------------ C. draws
@pytest.mark.parametrize("family", ["topk", "topp", "zeros", "masked", "prune"])
def test_draws(family):
    cases = _cases(family, C.PRUNE_V) if family == "prune" else _cases(family)
    best, srows = _run_family(cases)
    checked = 0
    bad = []
    for b, c in enumerate(cases):
        _, kept, _ = c.warp()
        if (_kept_of(c, srows[b]) != kept).any():
            continue                                                       # a boundary token fell the other way
        tok, gap = C.draw(c, kept)
        if c.family != "prune" and gap <= C.draw_tol(c):
            continue
        checked += 1
        if int(best[b]) != C.pack_word(c.row, tok):
            got = 0xFFFFFFFF - (int(best[b]) & 0xFFFFFFFF)
            bad.append(f"{c.name}: drew {got} ({c.row[got]}), oracle {tok} ({c.row[tok]}, gap {gap:.3g})")
    assert not bad, "\n".join(bad[:12])
    assert checked >= 0.9 * len(cases), (checked, len(cases))


# ------------------------------------------------------------------------------------------------ D. layouts
V_LIST = (1, 2, 7, 8, 1000, 1023, 1024, 1025, 4097, 51760, 51761)


def _v_max(lsm=None):
    """the largest V the variant takes on this device, from the refusal at an oversize V (nothing is launched)"""
    logits = torch.zeros(1, 1 << 18, dtype=BF16, device=DEV)
    with pytest.raises(_lib.VitaB200Error) as e:
        if lsm is None:
            ops.sample_rows(logits, *_prm([C.Case("", "", np.zeros(1, np.float32), 1.0, 0, 1.0)]),
                            torch.zeros(1, dtype=torch.int64, device=DEV))
        else:
            _lp(logits, [C.Case("", "", np.zeros(1, np.float32), 1.0, 0, 1.0)], lsm=lsm, scores=False)
    msg = str(e.value)
    return int(msg.split("V <= ")[1].split(" ")[0])


def _layout_cases(V, seed):
    rng = np.random.default_rng(seed)
    row = C.to_bf16(rng.normal(0, 2, V))
    m = row.max()
    row[V - 1] = m                                                         # ties for the maximum: the first one
    row[min(5, V - 1)] = m                                                 # wins, and with V > 1029 one thread
    if V > 1029:                                                           # stages two of them
        row[5 + 1024] = m
    k = max(1, min(50, V - 1))
    return [C.Case("layout", f"V{V}-{i}", row, T, kk, p, seed=seed + i, n=i)
            for i, (T, kk, p) in enumerate(((0.0, 0, 1.0), (0.7, k, 1.0), (1.0, 0, 0.9), (1.5, k, 0.5),
                                            (0.05, 0, 0.0), (1e-5, 2, 1.0)))]


def _strided(logits, ld, offset):
    B, V = logits.shape
    buf = torch.full((B * ld + offset + 8,), NAN16, dtype=torch.int16, device=DEV).view(BF16)
    view = buf[offset:offset + B * ld].view(B, ld)[:, :V]
    view.copy_(logits)
    return view


def _all_outputs(logits, cases, n_top):
    best, srows, _ = _plain(logits, cases)
    lp = _lp(logits, cases, n_top=n_top)
    lsm = _lp(logits, cases, n_top=n_top, lsm=True)
    return [best, srows] + [lp[k] for k in ("best", "lp", "rank", "ids", "tl", "srow")] + [lsm["srow"], lsm["lp"]]


@pytest.mark.parametrize("V", V_LIST + ("max",))
def test_layouts_and_staging_paths(V):
    if V == "max":
        V = min(_v_max(), _v_max(False), _v_max(True))
    cases = _layout_cases(V, 100 + V % 1000)
    logits = C.stack(cases).to(DEV)
    n_top = min(5, V)
    ref = _all_outputs(logits, cases, n_top)
    for ld, off in ((V + 8, 0), (V + 1, 0), (V, 1)):
        got = _all_outputs(_strided(logits, ld, off), cases, n_top)
        for a, r in zip(got, ref):
            assert torch.equal(_bits(a), _bits(r)), (V, ld, off)
    bad = [m for c, s in zip(cases, ref[1]) for m in _check_row(c, s)]
    assert not bad, "\n".join(bad[:12])
    for b, c in enumerate(cases):
        _, kept, _ = c.warp()
        tok, gap = C.draw(c, kept)
        if c.greedy or gap > C.draw_tol(c):
            assert int(ref[0][b]) == C.pack_word(c.row, tok), (c.name, tok)


def test_vmax_refusal():
    for lsm in (None, False, True):
        vm = _v_max(lsm)
        assert 80000 < vm < 90000, vm                                      # about 82 288 on an H100
        cases = [C.Case("", "", np.zeros(vm + 8, np.float32), 1.0, 0, 1.0)]
        logits = torch.zeros(1, vm + 8, dtype=BF16, device=DEV)
        with pytest.raises(_lib.VitaB200Error):
            if lsm is None:
                ops.sample_rows(logits, *_prm(cases), torch.zeros(1, dtype=torch.int64, device=DEV))
            else:
                _lp(logits, cases, lsm=lsm, scores=False)
        torch.cuda.synchronize()   # a refusal launches nothing, leaves no error


# ------------------------------------------------------------------------------------------------ E. logprobs and LSM
def fp32_slack(c, idx):
    """fp32 rounding of x = l / T and x_max (relative 2^-24 each) and of the differences taken from them"""
    fin = np.isfinite(c.row)
    T = 1.0 if c.greedy else C.f32(c.T)
    return 2.0 ** -22 * (np.abs(np.where(fin, c.row, 0.0)[idx]) + np.abs(c.row[fin]).max()) / T


def _check_lp(c, out, b, N, target):
    tok = target if 0 <= target < c.V else 0xFFFFFFFF - (int(out["best"][b]) & 0xFFFFFFFF)
    want = oracle_logprobs(c.row, C.f32(c.T) if not c.greedy else 0.0, c.k, C.f32(c.p), N, tok)
    bad = []
    g, w = out["lp"][b].item(), want["logprob"]
    if not (np.isinf(g) and np.isinf(w) and g == w or abs(g - w) <= ATOL + fp32_slack(c, tok)):
        bad.append(f"{c.name} target {target}: logprob {g} vs {w}")
    elif np.isfinite(w):
        _note("logprob error / (ATOL + fp32 slack)", abs(g - w) / (ATOL + fp32_slack(c, tok)))
    if out["rank"][b].item() != want["rank"]:
        bad.append(f"{c.name} target {target}: rank {out['rank'][b].item()} vs {want['rank']}")
    if out["ids"][b, :N].tolist() != want["top_ids"].tolist():
        bad.append(f"{c.name}: top ids {out['ids'][b, :N].tolist()} vs {want['top_ids'].tolist()}")
    tw = want["top_logprobs"]
    tg = out["tl"][b, :N].numpy().astype(np.float64)
    fin = np.isfinite(tw)
    tol = ATOL + fp32_slack(c, want["top_ids"])
    if not (np.array_equal(np.isfinite(tg), fin) and np.all(np.abs(tg[fin] - tw[fin]) <= tol[fin])):
        bad.append(f"{c.name}: top logprobs {tg} vs {tw}")
    if (out["ids"][b, N:] != -7).any():
        bad.append(f"{c.name}: top ids written past N")
    return bad, want


def _check_lsm_row(c, srow, want):
    """LSM row: same -inf pattern as the oracle's row, finite values within one bf16 rounding (2^-8 relative) plus
    the fp32 error of the logprob itself"""
    g = srow.float().numpy().astype(np.float64)
    w = want["row"]
    if not np.array_equal(np.isfinite(g), np.isfinite(w)):
        return [f"{c.name}: LSM -inf pattern differs"]
    fin = np.isfinite(w)
    err = np.abs(g[fin] - w[fin]) - 2.0 ** -8 * np.abs(w[fin]) - fp32_slack(c, np.flatnonzero(fin))
    _note("LSM error beyond one bf16 rounding and fp32 slack", max(0.0, err.max()))
    return [] if err.max() <= ATOL else [f"{c.name}: LSM row off by {err.max()} beyond bf16"]


@pytest.mark.parametrize("family", ["topn", "zeros", "topk", "topp"])
def test_logprobs_ranks_topn_and_lsm(family):
    base = _cases(family, C.PRUNE_V) if family == "topn" else _cases(family)[::2]
    bad = []
    for N in sorted({c.meta.get("N", 20) for c in base} | {1}):
        cases = [c for c in base if c.meta.get("N", N) == N]
        logits = C.stack(cases).to(DEV)
        V = cases[0].V
        for target_kind in ("draw", "0", "last", "dropped", "V"):
            target = []
            for c in cases:
                _, kept, _ = c.warp()
                t = {"draw": -1, "0": 0, "last": V - 1, "V": V,
                     "dropped": int(np.flatnonzero(~kept)[0]) if (~kept).any() else V - 1}[target_kind]
                target.append(t)
            out = _lp(logits, cases, n_top=N, target=target)
            lsm = _lp(logits, cases, n_top=N, target=target, lsm=True)
            for b, c in enumerate(cases):
                for o in (out, lsm):
                    m, want = _check_lp(c, o, b, N, target[b])
                    bad += m
                bad += _check_lsm_row(c, lsm["srow"][b], want)
                if not c.greedy:
                    bad += _check_row(c, out["srow"][b])
            if target_kind in ("draw", "V"):                                 # target >= V draws, like no target
                plain, _, _ = _plain(logits, cases)
                assert torch.equal(out["best"], plain) and torch.equal(lsm["best"], plain)
    assert not bad, "\n".join(bad[:12])


def test_score_log_rows_and_counters():
    """only row counter[b] of a canary-filled score log changes; counter -1 and counter >= rows write nothing"""
    cases = _cases("topk")[:8]
    V, rows = cases[0].V, 4
    counters = [0, 3, -1, 4, 2, 100, 1, -5]
    cases = [C.Case(c.family, c.name, c.row, c.T, c.k, c.p, c.seed, n) for c, n in zip(cases, counters)]
    logits = C.stack(cases).to(DEV)
    prm = _prm(cases)
    for variant in ("plain", "logprobs", "lsm"):
        log = _canary((len(cases), rows, V))
        best = torch.zeros(len(cases), dtype=torch.int64, device=DEV)
        if variant == "plain":
            ops.sample_rows(logits, *prm, best, log)
        else:
            lp = torch.zeros(len(cases), device=DEV)
            rk = torch.zeros(len(cases), dtype=torch.int32, device=DEV)
            ops.sample_logprobs(logits, *prm, best, lp, rk, None, None, 0, scores=log,
                                log_softmax_scores=variant == "lsm")
        raw = log.view(torch.int16).cpu()
        for b, n in enumerate(counters):
            for r in range(rows):
                untouched = bool((raw[b, r] == FILL).all())
                assert untouched == (r != n), (variant, b, n, r)


# ------------------------------------------------------------------------------------------------ F. mixed batch
def _mixed(B, V=C.PRUNE_V):
    pool = (_cases("topk", V)[::4] + _cases("topp", V) + _cases("zeros", V) + _cases("masked", V)
            + _cases("prune", V) + _cases("topn", V) + _cases("division", V))
    rng = np.random.default_rng(B)
    Ts = C.T_SAMPLED + C.T_GREEDY
    out = []
    for i in range(B):
        c = pool[i % len(pool)]
        T = c.T if i < len(pool) else Ts[int(rng.integers(len(Ts)))]
        out.append(C.Case(c.family, f"{c.name}-{i}", c.row, T, c.k, c.p, int(rng.integers(0, 2 ** 64, dtype=np.uint64)),
                          c.n if i < len(pool) else int(rng.integers(0, 8)), c.meta))
    return out, [int(s) for s in rng.integers(0, 4, B)]


@pytest.mark.parametrize("B", [64, 256])
def test_mixed_batch_matches_solo_launches(B):
    cases, streams = _mixed(B)
    logits = C.stack(cases).to(DEV)
    best, srows, _ = _plain(logits, cases, streams)
    lp = _lp(logits, cases, n_top=20, streams=streams)
    lsm = _lp(logits, cases, n_top=20, streams=streams, lsm=True)
    assert torch.equal(lp["best"], best) and torch.equal(lsm["best"], best)
    assert torch.equal(_bits(lp["srow"]), _bits(srows))                  # the LOGPROBS variant logs the same row
    for b, c in enumerate(cases):
        kept = _kept_of(c, srows[b])
        if not c.greedy:
            lsm_kept = np.where(np.isneginf(c.row), kept, torch.isfinite(lsm["srow"][b].float()).numpy())
            assert np.array_equal(kept, lsm_kept), c.name
        one, srow1, _ = _plain(logits[b:b + 1], cases[b:b + 1], streams[b:b + 1])
        assert one.item() == best[b].item(), c.name
        assert torch.equal(_bits(srow1[0]), _bits(srows[b])), c.name
        one_lp = _lp(logits[b:b + 1], cases[b:b + 1], n_top=20, streams=streams[b:b + 1], scores=False)
        for key in ("best", "lp", "rank", "ids", "tl"):
            assert torch.equal(_bits(one_lp[key][0]), _bits(lp[key][b])), (c.name, key)
    if B == 64:
        bad = [m for c, s in zip(cases, srows) for m in _check_row(c, s)]
        assert not bad, "\n".join(bad[:12])
