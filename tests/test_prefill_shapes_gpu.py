"""The prefill kernels at the shapes that serve, against plain fp64 references, row by row.

A. FlashAttention (ops.attention) in its three head geometries: Mixtral causal GQA 32/8 x 128 over the packed qkv rows
   (whole prompts and the sequence shards of expert parallelism, q_pos0 > 0), InternViT 16 x 64 non-causal over the
   packed qkv of 1 and 13 tiles, Whale 128/64 with key lengths.  Each under three input regimes (tests/prefill_cases.py):
   randn, sharp (q x 4) and late jumps, which drive the lazy rescale of flash_tc.cu at tiles past the first; the
   host-side proof that they do is tests/test_prefill_shapes.py.  Both exp2 paths (fa_poly 0 and 1); the output goes to
   a NaN-filled buffer with a gap after the heads and extra rows, and nothing outside [Sq, heads * Dv] may change; a
   second launch gives the same bits.  Whale's keys and values past each length hold +-2^60: a masked key weighs
   exactly zero on the MUFU path.  With fa_poly = 1, ex2_poly clamps its argument at -126, so a masked key weighs about
   2^-126 rather than 0; against values of 2^60 that is about 2^-66 per key, invisible at bf16 output precision.
B. The paged variant (chunked prefill, cached prefixes) on the sharp and late-jump inputs over shuffled, NaN-stale
   pages: fp64 per row, bit identity with the contiguous kernel, and an e4m3 cache gives the bits of a bf16 cache
   holding the dequantized values.
C. The dense wgmma GEMM: in-place residual (out is residual) at the model's shapes, writes confined to [M, N] of a
   padded NaN buffer, odd N (single-column stores) with bias, GELU and residual, ragged K, the LM head.
D. The slot-layout grouped MoE GEMMs at H = 4096, I = 14336: per-expert counts whose row tiles straddle two experts,
   slots past each count stay NaN, the row hint only changes the tile shape (same bits), and the 128-wide SILU tile.
"""
import functools
import math

import pytest
import torch

from tests import prefill_cases as PC
from tests.test_kv_fp8 import dequantize, quantize
from tests.test_paged_prefill_gpu import _paged, _qsl, _run_contiguous
from tests.util import BF16, close_rows, same_bits

pytestmark = pytest.mark.gpu

FILL = 0x7FA5                    # a NaN with a payload no kernel writes: compared bit for bit
NQ, NKV, D, W = PC.NQ, PC.NKV, PC.D, PC.QKV_W
WORST = {}                       # (section, regime, fa_poly) -> worst per-row relative error seen


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(WORST, key=str):
        print(f"prefill worst rel error {key}: {WORST[key]:.3e}")


def _note(key, r):
    WORST[key] = max(WORST.get(key, 0.0), r)


@pytest.fixture
def fa_poly():
    """sets the fa_poly option for one test and restores it afterwards"""
    from vita_b200 import ops
    before = ops.get_option("fa_poly")
    yield lambda v: ops.set_option("fa_poly", v)
    ops.set_option("fa_poly", before)


def _nan_buffer(shape):
    return torch.full(shape, FILL, dtype=torch.int16, device="cuda").view(BF16)


def _untouched(buf, inside, what):
    """every element of buf outside the index `inside` still holds FILL"""
    mask = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    mask[inside] = False
    n = int((buf.view(torch.int16)[mask] != FILL).sum())
    assert n == 0, f"{what}: {n} elements outside the output were written"


# ================================================================================================ A. FlashAttention
REGIME = pytest.mark.parametrize("regime", PC.REGIMES)
POLY = pytest.mark.parametrize("poly", [0, 1], ids=["mufu", "poly"])


@functools.lru_cache(maxsize=8)
def _cached(build, *args):
    """the CPU-built inputs of a case, shared by its fa_poly variants (callers copy them to the GPU)"""
    return build(*args)


def _attn_ref(q, k, v, scale, causal, q_pos0, kv_len, group):
    """fp64 softmax attention of one batch entry on the GPU, one KV head group at a time: q [Sq, Hq, Dqk],
    k [Skv, Hkv, Dqk], v [Skv, Hkv, Dv] -> [Sq, Hq, Dv]"""
    Sq, Hq, _ = q.shape
    out = torch.zeros(Sq, Hq, v.shape[-1], dtype=torch.float64, device="cuda")
    if kv_len == 0:
        return out
    k, v = k[:kv_len], v[:kv_len]
    cols = torch.arange(kv_len, device="cuda")
    for g in range(k.shape[1]):
        qg = q[:, g * group:(g + 1) * group].cuda().double()
        s = torch.einsum("sgd,td->gst", qg, k[:, g].cuda().double()) * scale
        if causal:
            s.masked_fill_(cols[None, None, :] > (q_pos0 + torch.arange(Sq, device="cuda"))[None, :, None], -math.inf)
        out[:, g * group:(g + 1) * group] = torch.einsum("gst,td->sgd", torch.softmax(s, -1), v[:, g].cuda().double())
        del s
    return out


def _attend(q, k, v, strides, B, Hq, Hkv, Sq, Skv, Dqk, Dv, kv_lens, causal, scale, q_pos0, what):
    """ops.attention into a NaN-filled [B, Sq + 2, Hq * Dv + 64] buffer; checks that only [:, :Sq, :Hq * Dv] changed
    and that a second launch gives the same bits.  Returns [B, Sq, Hq, Dv]."""
    from vita_b200 import ops
    HD = Hq * Dv
    res = []
    for _ in range(2):
        buf = _nan_buffer((B, Sq + 2, HD + 64))
        out = buf[:, :Sq, :HD]
        ops.attention(q, k, v, out, *strides, (buf.stride(0), buf.stride(1), Dv), B, Hq, Hkv, Sq, Skv, Dqk, Dv,
                      kv_lens, causal, scale, q_pos0)
        torch.cuda.synchronize()
        _untouched(buf, (slice(None), slice(0, Sq), slice(0, HD)), what)
        res.append(out.clone())
    same_bits(res[1], res[0], f"{what}: second launch")
    return res[0].view(B, Sq, Hq, Dv)


def _check_attn(got, ref, key, what):
    """got / ref [B, Sq, H, Dv]"""
    label = lambda i: f"batch {i[0]}, row {i[1]}, head {i[2]}"
    _note(key, close_rows(got, ref, what, label))


@POLY
@REGIME
@pytest.mark.parametrize("S", PC.MIXTRAL_S)
def test_flash_mixtral_causal(fa_poly, S, regime, poly):
    """whole prompts over the packed qkv rows (mixtral.py LayerAttention): q, k and v are strided views of one buffer"""
    qkv, _, kw = _cached(PC.mixtral_case, S, regime)
    qkv = qkv.cuda()
    ref = _attn_ref(qkv[:, :NQ * D].view(S, NQ, D), qkv[:, NQ * D:(NQ + NKV) * D].view(S, NKV, D),
                    qkv[:, (NQ + NKV) * D:].view(S, NKV, D), kw["scale"], True, 0, S, NQ // NKV)[None]
    fa_poly(poly)
    what = f"mixtral S={S}, {regime}, fa_poly {poly}"
    got = _attend(qkv, qkv[:, NQ * D:], qkv[:, (NQ + NKV) * D:], ((0, W, D), (0, W, D), (0, W, D)), 1, NQ, NKV, S, S,
                  D, D, None, True, kw["scale"], 0, what)
    _check_attn(got, ref, ("A mixtral", regime, poly), what)


@POLY
@REGIME
@pytest.mark.parametrize("t0,t1", PC.token_ranges())
def test_flash_sequence_shard(fa_poly, t0, t1, regime, poly):
    """a shard's rows [t0, t1) against keys [0, t1) of the cache layout (mixtral.py, expert-parallel prefill)"""
    Sq = t1 - t0
    (qkv, kc, vc), _, kw = _cached(PC.sharded_case, t0, t1, regime)
    qkv, kc, vc = qkv.cuda(), kc.cuda(), vc.cuda()
    ref = _attn_ref(qkv[:, :NQ * D].view(Sq, NQ, D), kc, vc, kw["scale"], True, t0, t1, NQ // NKV)[None]
    fa_poly(poly)
    what = f"shard [{t0}, {t1}), {regime}, fa_poly {poly}"
    got = _attend(qkv, kc, vc, ((0, W, D), (0, NKV * D, D), (0, NKV * D, D)), 1, NQ, NKV, Sq, t1, D, D, None, True,
                  kw["scale"], t0, what)
    _check_attn(got, ref, ("A shard", regime, poly), what)


@POLY
@REGIME
@pytest.mark.parametrize("B,S", PC.VIT_CASES)
def test_flash_vit(fa_poly, B, S, regime, poly):
    """InternViT: non-causal 16 x 64 over the packed qkv of B tiles (internvit.py)"""
    H, nh, Dh = PC.VIT_H, PC.VIT_NH, PC.VIT_D
    qkv, _, kw = _cached(PC.vit_case, B, S, regime)
    qkv = qkv.cuda()
    t = qkv.view(B, S, 3, nh, Dh)
    ref = torch.stack([_attn_ref(t[b, :, 0], t[b, :, 1], t[b, :, 2], kw["scale"], False, 0, S, 1) for b in range(B)])
    st = (S * 3 * H, 3 * H, Dh)
    fa_poly(poly)
    what = f"vit B={B} S={S}, {regime}, fa_poly {poly}"
    got = _attend(qkv, qkv[..., H:], qkv[..., 2 * H:], (st, st, st), B, nh, nh, S, S, Dh, Dh, None, False, kw["scale"],
                  0, what)
    _check_attn(got, ref, ("A vit", regime, poly), what)


@POLY
@REGIME
@pytest.mark.parametrize("T2", PC.WHALE_T2)
def test_flash_whale_key_lengths(fa_poly, T2, regime, poly):
    """Whale: [q + u | q + v] against [k | p] (128) with 64-wide v heads, lengths {0, 1, 127, 128, 129, T2} clamped to
    T2; length 0 gives zeros, as softmax(...).masked_fill(mask, 0) does in the reference"""
    B, nh, dk = PC.WHALE_B, PC.WHALE_NH, PC.WHALE_DK
    C = nh * dk
    (q2, k2, qkv, lens), _, kws = _cached(PC.whale_case, T2, regime)
    q2, k2, qkv = q2.cuda(), k2.cuda(), qkv.cuda()
    v = qkv[..., 2 * C:].view(B, T2, nh, dk)
    ref = torch.stack([_attn_ref(q2[b], k2[b], v[b], kws[b]["scale"], False, 0, kws[b]["kv_len"], 1)
                       for b in range(B)])
    qs = (T2 * nh * 2 * dk, nh * 2 * dk, 2 * dk)
    kv_lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    fa_poly(poly)
    what = f"whale T2={T2}, {regime}, fa_poly {poly}"
    got = _attend(q2, k2, qkv[..., 2 * C:], (qs, qs, (T2 * 3 * C, 3 * C, dk)), B, nh, nh, T2, T2, 2 * dk, dk, kv_lens,
                  False, kws[0]["scale"], 0, what)
    assert not got[0].any(), f"{what}: length 0 must give zeros"
    _check_attn(got, ref, ("A whale", regime, poly), what)


# ================================================================================================ B. paged
def _paged_out(q, kc, vc, table, ps, ks=None, vs=None):
    from vita_b200 import ops
    cases = PC.PAGED_CASES
    qsl = _qsl(cases)
    plan = ops.PagedPrefill(qsl, [p + c for p, c in cases], table, ps)
    out = torch.zeros(qsl[-1], NQ * D, dtype=BF16, device="cuda")
    ops.attention_prefill_paged(q[:, :NQ * D], kc, vc, plan, out, NQ, NKV, D, D ** -0.5, ks, vs)
    torch.cuda.synchronize()
    return out


@POLY
@pytest.mark.parametrize("regime", ["sharp", "late"])
@pytest.mark.parametrize("ps", [16, 32, 64, 128])
def test_flash_paged(fa_poly, ps, regime, poly):
    cases = PC.PAGED_CASES
    qsl = _qsl(cases)
    (q, kv), _, kws = _cached(PC.paged_case, regime)
    q = q.cuda()
    kv = [(k.cuda(), v.cuda()) for k, v in kv]
    kc, vc, table, _ = _paged(cases, kv, ps, ps, stale=True)
    ks, vs = 0.37, 2.0 ** -3
    k8, v8 = quantize(kc, ks), quantize(vc, vs)
    kd, vd = dequantize(k8, ks), dequantize(v8, vs)
    refs = [_attn_ref(q[qsl[i]:qsl[i + 1], :NQ * D].view(c, NQ, D), *kv[i], D ** -0.5, True, p, p + c, NQ // NKV)
            for i, (p, c) in enumerate(cases)]
    fa_poly(poly)
    tag = f"page {ps}, {regime}, fa_poly {poly}"
    got = _paged_out(q, kc, vc, table, ps)
    want = _run_contiguous(q, kv, cases)
    torch.cuda.synchronize()
    for i, (p, c) in enumerate(cases):
        rows = slice(qsl[i], qsl[i + 1])
        r = close_rows(got[rows].view(c, NQ, D), refs[i], f"{tag}: P={p} C={c}", lambda j: f"row {j[0]}, head {j[1]}")
        _note(("B paged", regime, poly), r)
        same_bits(got[rows], want[rows], f"{tag}: P={p} C={c}, paged vs contiguous")
    same_bits(_paged_out(q, k8, v8, table, ps, ks, vs), _paged_out(q, kd, vd, table, ps),
              f"{tag}: e4m3 cache vs bf16 cache of the dequantized values")


# ================================================================================================ C. dense GEMMs
def _gemm_ref(x, w, bias=None, act=0, colscale=None, residual=None):
    """fp64 on the GPU: residual + colscale * act(x w^T + bias)"""
    y = x.cuda().double() @ w.cuda().double().T
    if bias is not None:
        y += bias.cuda().double()
    if act == 1:
        y = 0.5 * y * (1.0 + torch.erf(y / math.sqrt(2.0)))
    if colscale is not None:
        y *= colscale.cuda().double()
    if residual is not None:
        y += residual.cuda().double()
    return y


def _gpu_randn(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(BF16)


def _linear_case(M, N, K, *, bias=False, act=0, colscale=False, residual=False, in_place=False, pad=8, seed=0,
                 what=""):
    """ops.linear writing into rows [0, M) and columns [0, N) of a NaN-filled [M + 3, N + pad] buffer; in place: the
    same view is the residual (as every residual linear of the model runs)"""
    from vita_b200 import ops
    x = _gpu_randn((M, K), seed)
    w = _gpu_randn((N, K), seed + 1, K ** -0.5)
    b = _gpu_randn((N,), seed + 2, 0.5) if bias else None
    cs = _gpu_randn((N,), seed + 3) if colscale else None
    buf = _nan_buffer((M + 3, N + pad))
    out = buf[:M, :N]
    r = None
    if residual:
        r = _gpu_randn((M, N + pad), seed + 4)[:, :N]        # ldr = ldc: a multiple of 8 also for odd N
        if in_place:
            out.copy_(r)
            r = out
    ref = _gemm_ref(x, w, b, act, cs, r if not in_place else out.clone())
    ops.linear(x, w, b, act, cs, r, out=out)
    torch.cuda.synchronize()
    _untouched(buf, (slice(0, M), slice(0, N)), what)
    _note(("C gemm", "in place" if in_place else "out of place", 0),
          close_rows(out, ref, what, lambda i: f"row {i[0]}"))


@pytest.mark.parametrize("M", [1, 129, 4600])
def test_gemm_oproj_in_place(M):
    """o-proj, N = K = 4096, out is residual; M = 1 and 129 run cut tail tiles, 4600 a cut last wave"""
    _linear_case(M, 4096, 4096, residual=True, in_place=True, seed=M, what=f"o-proj M={M} in place")


@pytest.mark.parametrize("name,K", [("proj", 1024), ("fc2", 4096)])
def test_gemm_vit_layer_scale_in_place(name, K):
    """InternViT proj / fc2 with bias, layer scale and the residual in place, 13 tiles of 1025 rows"""
    _linear_case(13 * 1025, 1024, K, bias=True, colscale=True, residual=True, in_place=True, seed=K,
                 what=f"vit {name} in place")


@pytest.mark.parametrize("name,K", [("out", 1024), ("w2", 4096)])
def test_gemm_whale_in_place(name, K):
    """Whale out / w2 with bias and the residual in place, 6 x 248 rows"""
    _linear_case(6 * 248, 1024, K, bias=True, residual=True, in_place=True, seed=K + 1, what=f"whale {name} in place")


@pytest.mark.parametrize("M,N,K,pad", [(2048, 1000, 512, 24), (1, 4096, 4096, 8), (129, 6144, 4096, 64),
                                       (300, 520, 200, 8)])
def test_gemm_writes_stay_inside(M, N, K, pad):
    """(2048, 1000, 512): the partial last wave is cut in halves and the last half tile straddles N"""
    _linear_case(M, N, K, bias=True, pad=pad, seed=M + N, what=f"gemm M={M} N={N} K={K} ldc={N + pad}")


@pytest.mark.parametrize("N", [1, 3, 33, 1001])
def test_gemm_odd_n(N):
    """single-column stores: bias, GELU and residual on the last column"""
    _linear_case(129, N, 256, bias=True, act=1, residual=True, pad=8 - N % 8 + 8, seed=N, what=f"gemm odd N={N}")


@pytest.mark.parametrize("K", [8, 56, 64, 72])
def test_gemm_ragged_k(K):
    _linear_case(300, 392, K, bias=True, residual=True, seed=K, what=f"gemm K={K}")


def test_gemm_lm_head():
    _linear_case(129, 51760, 4096, seed=5, what="lm head")


# ================================================================================================ D. grouped MoE GEMMs
MOE_T = 300
MOE_CAP = MOE_T + 5                                  # not a multiple of 128
MOE_COUNTS = [0, 1, 127, 128, 129, MOE_CAP, 300, 2]


@pytest.fixture(scope="module")
def moe_weights():
    E, H, I = 8, 4096, 14336
    return _gpu_randn((E, 2 * I, H), 31, 0.02), _gpu_randn((E, H, I), 32, 0.015)


def _moe_run(x, w13, w2, cnt, rw, hint):
    from vita_b200 import ops
    E, I = w13.shape[0], w13.shape[1] // 2
    act = _nan_buffer((E * MOE_CAP, I))
    y = _nan_buffer((E * MOE_CAP, w2.shape[1]))
    ops.moe_gate_up_slots(x, w13, act, cnt, hint)
    ops.moe_down_slots(act, w2, y, cnt, rw, hint)
    torch.cuda.synchronize()
    return act, y


def _moe_check(x, w13, w2, rw, act, y, what):
    I = w13.shape[1] // 2
    for e, n in enumerate(MOE_COUNTS):
        r0 = e * MOE_CAP
        for t in (act, y):
            assert (t[r0 + n:r0 + MOE_CAP].view(torch.int16) == FILL).all(), f"{what}: expert {e}: a slot past {n} changed"
        if n == 0:
            continue
        gu = x[r0:r0 + n].double() @ w13[e].double().T
        ref = torch.nn.functional.silu(gu[:, :I]) * gu[:, I:]
        _note(("D moe", "gate|up", 0), close_rows(act[r0:r0 + n], ref, f"{what}: gate|up expert {e} ({n} rows)",
                                                  lambda i: f"slot {i[0]}"))
        dn = (act[r0:r0 + n].double() @ w2[e].double().T) * rw[r0:r0 + n, None].double()
        _note(("D moe", "down", 0), close_rows(y[r0:r0 + n], dn, f"{what}: down expert {e} ({n} rows)",
                                               lambda i: f"slot {i[0]}"))


def _moe_inputs():
    E = 8
    x = _nan_buffer((E * MOE_CAP, 4096))
    rw = torch.full((E * MOE_CAP,), float("nan"), device="cuda")
    g = torch.Generator(device="cuda").manual_seed(33)
    for e, n in enumerate(MOE_COUNTS):
        x[e * MOE_CAP:e * MOE_CAP + n] = _gpu_randn((n, 4096), 40 + e)
        rw[e * MOE_CAP:e * MOE_CAP + n] = torch.rand(n, device="cuda", generator=g)
    return x, rw, torch.tensor(MOE_COUNTS, dtype=torch.int32, device="cuda")


def test_moe_slots_counts_and_row_hints(moe_weights):
    """counts {0, 1, 127, 128, 129, cap, 300, 2} with cap = 305; rows_hint 1, the actual rows and E * cap"""
    w13, w2 = moe_weights
    x, rw, cnt = _moe_inputs()
    act, y = _moe_run(x, w13, w2, cnt, rw, sum(MOE_COUNTS))
    _moe_check(x, w13, w2, rw, act, y, "moe slots")
    for hint in (1, 8 * MOE_CAP):
        a2, y2 = _moe_run(x, w13, w2, cnt, rw, hint)
        same_bits(a2, act, f"moe gate|up: rows_hint {hint} vs {sum(MOE_COUNTS)}")
        same_bits(y2, y, f"moe down: rows_hint {hint} vs {sum(MOE_COUNTS)}")


def test_moe_slots_128_wide_tiles(moe_weights, monkeypatch):
    """VITA_B200_GEMM_BN=128: the 128-wide SILU tile (launch_gemm<128, true, 6>) and the 128-wide down tile"""
    monkeypatch.setenv("VITA_B200_GEMM_BN", "128")
    w13, w2 = moe_weights
    x, rw, cnt = _moe_inputs()
    act, y = _moe_run(x, w13, w2, cnt, rw, sum(MOE_COUNTS))
    _moe_check(x, w13, w2, rw, act, y, "moe slots, 128-wide tiles")
