"""Multi-GPU parity (BASELINE config 4 shape): TPC-H Q3 on 2 datanodes with two NCCL
redistributes, checked against the single-node oracle.  Needs >= 2 GPUs."""
import os
import socket
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpus():
    try:
        import ctypes
        cu = ctypes.CDLL("libcuda.so.1")
        if cu.cuInit(0) != 0:
            return 0
        n = ctypes.c_int()
        return n.value if cu.cuDeviceGetCount(ctypes.byref(n)) == 0 else 0
    except OSError:
        return 0


# the three ways a redistribute can travel: the peer windows (default), NCCL send/recv (windows switched off), and the
# fallback every rank takes together when a rank's region does not fit the window
@pytest.mark.gpu
@pytest.mark.skipif(_ngpus() < 2, reason="needs two GPUs (gpurun --gpus 2)")
@pytest.mark.parametrize("env,orders,want", [
    ({}, 30000, ("peer windows x2", "nccl all-to-all x0")),
    ({"GX_NO_PEER": "1"}, 30000, ("peer windows x0", "nccl all-to-all x2")),
    ({"GX_PEER_WINDOW_MB": "1"}, 200000, ("peer windows x1", "nccl all-to-all x1")),
], ids=["peer", "nccl", "window_too_small"])
def test_q3_two_datanodes_with_redistribute(env, orders, want):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "scripts", "q3_multi.py"), "--sf", "1", "--orders", str(orders)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT, env=dict(os.environ, **env))
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    assert "OK q3 parity vs oracle" in r.stdout, r.stdout[-2000:]
    for w in want:
        assert w in r.stdout, r.stdout[-2000:]


@pytest.mark.gpu
@pytest.mark.skipif(_ngpus() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("env", [{}, {"GX_NO_GATHER_COMBINE": "1"}], ids=["gathered", "records"])
def test_combine_float8_overflow_rule(env):
    """two finite partial sums overflowing in combine are GX_ERR_OVERFLOW; an infinite partial is not"""
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "scripts", "combine_fp_multi.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT, env=dict(os.environ, **env))
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    assert "OK combine overflow rule" in r.stdout, r.stdout[-2000:]
