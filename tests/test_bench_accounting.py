"""The algorithmic FLOP / byte counts bench.py divides by (SURVEY.md section 8d), checked on the CPU against their
closed forms, and the JSON-line helpers that need no GPU."""
import importlib.util
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def _bench():
    spec = importlib.util.spec_from_file_location("bench_module", ROOT / "bench.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_prefill_flops_and_decode_bytes_closed_forms():
    b = _bench()
    from vita_b200.config import VitaConfig
    cfg = VitaConfig.full(32)
    H, I, L, V, D, nq, nkv, E = 4096, 14336, 32, 51760, 128, 32, 8, 8
    per_tok_layer = 2 * H * (nq + 2 * nkv) * D + 2 * H * nq * D + 2 * H * E + 2 * 3 * 2 * H * I
    assert abs(per_tok_layer * L / 25.235e9 - 1) < 2e-3                       # SURVEY 8(d): 25.2 GFLOP per token
    S = 4096
    assert b.prefill_flops(S, cfg) == per_tok_layer * L * S + 2 * S * S * nq * D * L + 2 * H * V
    ctx = 634
    per_layer = ((nq + 2 * nkv) * D * H + H * nq * D) * 2 + E * H * 2 + 2 * 3 * H * I * 2 + 2 * H * 2
    assert b.decode_bytes(ctx, cfg) == L * (per_layer + 2 * nkv * D * 2 * ctx) + V * H * 2 + H * 2
    assert abs(b.decode_bytes(ctx, cfg) / 25.74e9 - 1) < 2e-3                  # 25.7 GB per decoded token at bs = 1


def test_workload_geometry_and_peaks():
    b = _bench()
    from vita_b200.config import VitaConfig
    cfg = VitaConfig.full(32)
    assert b.spliced_len(cfg) == 506                                           # 126 text + 256 visual + 124 audio tokens
    p = b.peaks()
    assert p["hbm_gbs"] > 1000 and p["tflops"] > 100
