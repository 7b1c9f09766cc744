"""FP8 (e4m3) KV cache, host side: the quantizer every kernel is held to, the kv_cache_dtype option on the three public
surfaces, the refusals, and the cache's footprint.

The write definition is c = e4m3_rn_satfinite(float(bf16(x)) / scale) and the read bf16(float(c) * scale)
(include/vita_b200.h, vita_gemm_qkv_rope_fp8).  `quantize` / `dequantize` below state it in torch (clamp, then cast);
`e4m3_reference` states it from the bit layout, and the two must agree on every bf16 input.
"""
import types

import numpy as np
import pytest
import torch

from vita_b200.config import VitaConfig

FP8 = torch.float8_e4m3fn
BF16 = torch.bfloat16
SCALES = (1.0, 2.0 ** -3, 0.37)


def quantize(x: torch.Tensor, scale: float) -> torch.Tensor:
    """bf16 rows -> e4m3 bytes: fp32 division by the fp32 scale, clamp to +-448, round to nearest even.  On x's
    device; the scale is a tensor there, so the division is a true elementwise division on either device."""
    s = torch.tensor(scale, dtype=torch.float32, device=x.device)
    return (x.to(BF16).float() / s).clamp(-448.0, 448.0).to(FP8)


def dequantize(c: torch.Tensor, scale: float) -> torch.Tensor:
    """e4m3 bytes -> their bf16 values: bf16(float(c) * scale), on c's device."""
    return (c.float() * torch.tensor(scale, dtype=torch.float32, device=c.device)).to(BF16)


def qdq(x: torch.Tensor, scale: float) -> torch.Tensor:
    """what a cached row reads back as (fp32)"""
    return dequantize(quantize(x, scale), scale).float()


def e4m3_reference(x: np.ndarray) -> np.ndarray:
    """cvt.rn.satfinite.e4m3 from the format: 1 sign, 4 exponent (bias 7), 3 mantissa bits; subnormals step 2^-9;
    finite saturation at 448 (0x7e); NaN -> 0x7f.  x: float64 values (already divided by the scale in fp32)."""
    out = np.zeros(x.shape, dtype=np.uint8)
    sign = np.signbit(x).astype(np.uint8) << 7
    a = np.abs(x)
    nan = np.isnan(x)
    sat = ~nan & (a >= 448.0)
    sub = ~nan & ~sat & (a < 2.0 ** -6)
    nrm = ~nan & ~sat & ~sub
    out[sat] = 0x7E
    out[sub] = np.rint(a[sub] / 2.0 ** -9).astype(np.uint8)          # 8 rounds up into the smallest normal: code 8
    e = np.floor(np.log2(a[nrm])).astype(np.int64)
    m = np.rint(a[nrm] / np.exp2(e - 3)).astype(np.int64)            # 8 .. 16, half to even
    e = np.where(m == 16, e + 1, e)
    m = np.where(m == 16, 8, m)
    code = ((e + 7) << 3) | (m - 8)
    assert (code <= 0x7E).all()
    out[nrm] = code.astype(np.uint8)
    out |= sign
    out[nan] = 0x7F
    return out


@pytest.mark.parametrize("scale", SCALES)
def test_quantizer_on_every_bf16_pattern(scale):
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    x = bits.view(BF16)
    got = quantize(x, scale).view(torch.uint8).numpy()
    q = (x.float() / torch.tensor(scale, dtype=torch.float32)).double().numpy()
    want = e4m3_reference(q)
    nan = np.isnan(q)
    assert (np.isnan(quantize(x, scale).float().numpy()) == nan).all(), "NaN in, NaN out"
    bad = np.nonzero((got != want) & ~nan)[0]
    assert bad.size == 0, (f"{bad.size} patterns differ, e.g. bf16 {int(bits[bad[0]]) & 0xffff:#06x}: "
                           f"{got[bad[0]]:#04x} vs {want[bad[0]]:#04x}")
    # the edges named by the contract
    edge = torch.tensor([448.0, -448.0, 464.0, 1e30, -1e30, float("inf"), 2.0 ** -9, 2.0 ** -10, -0.0, 0.0])
    e = quantize(edge * scale, scale).view(torch.uint8).tolist()
    assert e[:6] == [0x7E, 0xFE, 0x7E, 0x7E, 0xFE, 0x7E]
    assert e[8:] == [0x80, 0x00]
    # with a power-of-two scale the read is exact: every finite code survives the round trip
    if scale != 0.37:
        codes = torch.arange(256, dtype=torch.int32).to(torch.uint8)
        codes = codes[(codes & 0x7F) != 0x7F]
        assert torch.equal(quantize(dequantize(codes.view(FP8), scale), scale).view(torch.uint8), codes)


def test_option_names():
    from vita_b200.model.mixtral import parse_kv_cache_dtype
    from vita_b200.vllm_adapter import kv_cache_dtype_of
    for name, want in (("auto", "bf16"), ("bf16", "bf16"), ("bfloat16", "bf16"), ("fp8", "fp8"), ("fp8_e4m3", "fp8")):
        assert parse_kv_cache_dtype(name) == want
    with pytest.raises(NotImplementedError):
        parse_kv_cache_dtype("fp8_e5m2")
    with pytest.raises(ValueError):
        parse_kv_cache_dtype("int8")
    cc = lambda d: types.SimpleNamespace(cache_dtype=d, block_size=16)
    for name, want in (("auto", "bf16"), ("bfloat16", "bf16"), ("fp8", "fp8"), ("fp8_e4m3", "fp8")):
        assert kv_cache_dtype_of(cc(name)) == want
    assert kv_cache_dtype_of(None) == "bf16"
    assert kv_cache_dtype_of(types.SimpleNamespace(block_size=16)) == "bf16"
    for bad in ("fp8_e5m2", "fp8_inc", "half", "int8"):
        with pytest.raises(NotImplementedError):
            kv_cache_dtype_of(cc(bad))


def test_adapter_reads_cache_dtype():
    from vita_b200.vllm_adapter import MixtralForConditionalGeneration
    cfg = VitaConfig.tiny()
    for name, want in (("auto", "bf16"), ("fp8", "fp8"), ("fp8_e4m3", "fp8")):
        m = MixtralForConditionalGeneration(cfg, device="cpu",
                                            cache_config=types.SimpleNamespace(cache_dtype=name, block_size=32))
        assert m.kv_cache_dtype == want and m.block_size == 32
    with pytest.raises(NotImplementedError):
        MixtralForConditionalGeneration(cfg, device="cpu", cache_config=types.SimpleNamespace(cache_dtype="fp8_e5m2"))


def test_model_surfaces_pass_the_option(monkeypatch):
    """VITAMixtralForCausalLM(kv_cache_dtype=...) and load_pretrained_model(..., kv_cache_dtype=...) hand the option and
    the scales to the decoder"""
    from vita_b200.model import vita_mixtral, builder
    seen = []

    class Recorder:
        def __init__(self, *a, **kw):
            seen.append(kw)

    monkeypatch.setattr(vita_mixtral, "MixtralDecoder", Recorder)
    monkeypatch.setenv("VITA_B200_ENC_GRAPH", "0")
    cfg = VitaConfig.tiny()
    vita_mixtral.VITAMixtralForCausalLM(cfg, {"llm": {}}, "cpu", kv_cache_dtype="fp8", k_scale=0.5, v_scale=[0.25] * 2)
    assert seen[-1]["kv_cache_dtype"] == "fp8" and seen[-1]["k_scale"] == 0.5 and seen[-1]["v_scale"] == [0.25] * 2
    vita_mixtral.VITAMixtralForCausalLM(cfg, {"llm": {}}, "cpu")
    assert seen[-1]["kv_cache_dtype"] == "auto"
    monkeypatch.setattr(builder.W, "pack", lambda *a, **k: {"llm": {}})
    builder.load_pretrained_model("synthetic:tiny", device="cpu", kv_cache_dtype="fp8_e4m3", k_scale=0.125)
    assert seen[-1]["kv_cache_dtype"] == "fp8_e4m3" and seen[-1]["k_scale"] == 0.125


def test_expert_parallel_refuses_fp8():
    from vita_b200.model.mixtral import MixtralDecoder
    cfg = VitaConfig.tiny().llm
    w = {"ep": (0, 2), "rope": torch.zeros(1 << 16, 2, 64)}
    with pytest.raises(ValueError, match="fp8"):
        MixtralDecoder(cfg, w, "cpu", max_seq_len=64, max_new_tokens=8, kv_cache_dtype="fp8")


def test_fp8_cache_is_half_the_bytes():
    from vita_b200.model.mixtral import PagedKVCache
    cfg = VitaConfig.tiny().llm
    a = PagedKVCache(cfg, 3, 100, "cpu")
    b = PagedKVCache(cfg, 3, 100, "cpu", kv_cache_dtype="fp8", k_scale=0.5, v_scale=[0.25] * cfg.num_hidden_layers)
    nbytes = lambda c: sum(t.numel() * t.element_size() for t in c.k + c.v)
    assert all(t.dtype == FP8 for t in b.k + b.v) and all(t.dtype == BF16 for t in a.k + a.v)
    assert 2 * nbytes(b) == nbytes(a)
    assert b.k_scale == [0.5] * cfg.num_hidden_layers and b.v_scale == [0.25] * cfg.num_hidden_layers
    assert torch.equal(a.block_table, b.block_table) and torch.equal(a.slot_map, b.slot_map)
    with pytest.raises(ValueError):
        PagedKVCache(cfg, 1, 16, "cpu", kv_cache_dtype="fp8", k_scale=[1.0])          # one per layer
    with pytest.raises(ValueError):
        PagedKVCache(cfg, 1, 16, "cpu", kv_cache_dtype="fp8", v_scale=0.0)
    with pytest.raises(ValueError):
        PagedKVCache(cfg, 1, 16, "cpu", k_scale=0.5)                                   # bf16 has no scales
    with pytest.raises(NotImplementedError):
        PagedKVCache(cfg, 1, 16, "cpu", kv_cache_dtype="fp8_e5m2")

