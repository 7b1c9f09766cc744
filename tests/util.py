"""Shared helpers for the parity tests (the oracle is imported here as the checker only)."""
import pytest
import torch

BF16 = torch.bfloat16


def bf16_round(t: torch.Tensor) -> torch.Tensor:
    return t.to(BF16).to(torch.float32)


def randn(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return bf16_round(torch.randn(shape, generator=g) * scale)


def to_dev(t: torch.Tensor) -> torch.Tensor:
    return t.to(device="cuda", dtype=BF16).contiguous()


def assert_close(got: torch.Tensor, want: torch.Tensor, rel=1.6e-2, what=""):
    """bf16 tolerance: max |got - want| <= rel * max|want| (fp32 accumulate, one or two bf16 roundings)."""
    got = got.detach().float().cpu()
    want = want.detach().float().cpu()
    assert got.shape == want.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(want.shape)}"
    assert torch.isfinite(got).all(), f"{what}: non-finite values"
    err = (got - want).abs().max().item()
    ref = want.abs().max().item()
    assert err <= rel * max(ref, 1e-6), f"{what}: max err {err:.4e} vs max|ref| {ref:.4e} (rel {err / max(ref, 1e-6):.3e})"
    return err / max(ref, 1e-6)


# ------------------------------------------------------------------------------------------------ fp64 references
GPU_REF_ELEMS = 10 ** 8     # fp64 references of larger matrices run on the GPU


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int16) if t.dtype == BF16 else t


def same_bits(a: torch.Tensor, b: torch.Tensor, what: str) -> None:
    assert torch.equal(bits(a), bits(b)), f"{what}: bits differ"


def f64(w: torch.Tensor) -> torch.Tensor:
    """w as float64 where its fp64 products are cheap: on the GPU above GPU_REF_ELEMS elements, on the CPU below"""
    return w.double() if w.numel() > GPU_REF_ELEMS else w.cpu().double()


def matmul64(w: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """x [n, K] . w [N, K]^T in fp64 -> CPU float64 [n, N] (w bf16 on any device)"""
    w64 = f64(w)
    return (x.to(w64.device, torch.float64) @ w64.T).cpu()


def close_rows(got: torch.Tensor, want: torch.Tensor, what: str, labels, rel=1.6e-2) -> float:
    """assert_close applied to every leading index separately: got / want [..., n].  The comparison runs on want's
    device (a CUDA reference stays on the GPU).  Returns the worst relative error."""
    dev = want.device
    got = got.detach().to(dev, torch.float64)
    want = want.detach().to(torch.float64)
    assert got.shape == want.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(want.shape)}"
    bad = ~torch.isfinite(got).all(-1)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        pytest.fail(f"{what}: non-finite values at {labels(i)}")
    err = (got - want).abs().amax(-1)
    ref = want.abs().amax(-1).clamp_min(1e-6)
    r = err / ref
    worst = float(r.max()) if r.numel() else 0.0
    if worst > rel:
        i = [int(x) for x in torch.unravel_index(r.argmax(), r.shape)]
        pytest.fail(f"{what}: max err {float(err[tuple(i)]):.4e} vs max|ref| {float(ref[tuple(i)]):.4e} "
                    f"(rel {float(r[tuple(i)]):.3e} > {rel}) at {labels(i)}")
    return worst
