#!/usr/bin/env python
"""Times the wgmma GEMM on the shapes of the BASELINE prefill (S=506 and S=4096) with both tile widths."""
import json, os, subprocess, sys
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

def run(bn):
    import torch
    from vita_b200 import ops
    out = {}
    dev = "cuda"
    def timeit(fn, n=20):
        for _ in range(3): fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        tot = 0.0
        for _ in range(n):
            flush.zero_()
            a.record(); fn(); b.record(); b.synchronize()
            tot += a.elapsed_time(b)
        return tot / n * 1e3
    H, I, E = 4096, 14336, 8
    for S in (506, 4096):
        x = torch.randn(S, H, device=dev).bfloat16()
        wqkv = torch.randn(6144, H, device=dev).bfloat16() * 0.02
        wo = torch.randn(H, H, device=dev).bfloat16() * 0.02
        qkv = torch.empty(S, 6144, device=dev, dtype=torch.bfloat16)
        out[f"S{S}_qkv"] = (timeit(lambda: ops.linear(x, wqkv, out=qkv)), 2 * S * 6144 * H)
        o = torch.empty(S, H, device=dev, dtype=torch.bfloat16)
        out[f"S{S}_oproj"] = (timeit(lambda: ops.linear(x, wo, residual=x, out=o)), 2 * S * H * H)
        rows = 2 * S
        w13 = torch.empty(E, 2 * I, H, device=dev, dtype=torch.bfloat16).normal_(0, 0.02)
        w2 = torch.empty(E, H, I, device=dev, dtype=torch.bfloat16).normal_(0, 0.02)
        cnt = torch.full((E,), rows // E, dtype=torch.int64)
        cnt[0] += 37; cnt[1] -= 37
        offs = torch.cat([torch.zeros(1, dtype=torch.int64), cnt.cumsum(0)]).to(torch.int32).to(dev)
        xp = torch.randn(rows, H, device=dev).bfloat16()
        act = torch.empty(rows, I, device=dev, dtype=torch.bfloat16)
        yp = torch.empty(rows, H, device=dev, dtype=torch.bfloat16)
        rw = torch.rand(rows, device=dev)
        out[f"S{S}_moe_gate_up"] = (timeit(lambda: ops.moe_gate_up(xp, w13, act, offs, rows), 10), 2 * rows * 2 * I * H)
        out[f"S{S}_moe_down"] = (timeit(lambda: ops.moe_down(act, w2, yp, offs, rw, rows), 10), 2 * rows * H * I)
        del w13, w2
    print(json.dumps({k: {"us": v[0], "tflops": v[1] / v[0] / 1e6} for k, v in out.items()}))

if __name__ == "__main__":
    if len(sys.argv) > 1:
        run(sys.argv[1])
    else:
        for bn in ("128", "256", "auto"):
            env = dict(os.environ)
            if bn != "auto":
                env["VITA_B200_GEMM_BN"] = bn
            r = subprocess.run([sys.executable, __file__, bn], env=env, capture_output=True, text=True)
            print(bn, r.stdout.strip() or r.stderr[-500:])
