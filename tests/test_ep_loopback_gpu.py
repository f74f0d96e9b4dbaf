"""Expert-parallel exchange on one GPU: the multi-GPU workers of ``tests/mgpu`` under torchrun with a single rank.  With one rank
every pair is dispatched to the rank's own receive buffer and returned to its own return buffer, so the dispatch, the arrival
wait in the grouped GEMM, the return epilogue and the combine run end to end on a one-GPU machine."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _torchrun_one(script, args, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=1", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(HERE, "mgpu", script), *args]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=420, env=dict(os.environ, CUDA_VISIBLE_DEVICES="0"))
    return r.stdout + r.stderr


def test_expert_parallel_moe_loopback():
    out = _torchrun_one("ep_parity.py", [], 29601)
    assert "EP_OK" in out, out[-3000:]


@pytest.mark.parametrize("mode,port", [("forward", 29602), ("fused", 29603)])
def test_expert_parallel_stress_loopback(mode, port):
    out = _torchrun_one("ep_stress.py", [mode], port)
    assert "EP_STRESS_OK " + mode in out, out[-3000:]
