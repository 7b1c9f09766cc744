"""Expert-parallel prefill (sequence-sharded dense part + all-gathered K/V and routed rows + fused P2P combine) vs the
single-GPU model with identical weights, bit for bit; needs >= 2 GPUs."""
import subprocess
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent


@pytest.mark.gpu
@pytest.mark.parametrize("mode,port", [("seq", 29532)])
def test_ep2_prefill_matches_single_gpu(mode, port):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (run under gpurun --gpus 2)")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), str(ROOT / "tests" / "ep_check.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    print(res.stdout[-2000:], res.stderr[-2000:])
    assert res.returncode == 0
