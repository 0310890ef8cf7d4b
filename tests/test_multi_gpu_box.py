"""Multi-GPU tests on a real box (skipped unless >= 2 H100s are visible): bench.py under torchrun with every result-exchange
path (peer push from the sweep, peer push by the exchange kernel, NCCL all-reduce) must give the same Hessian slab checksum
as a single GPU."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _run(n, collective, port, push=None):
    cmd = [sys.executable]
    if n > 1:
        cmd += ["-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1", "--master-port", str(port)]
    cmd += [os.path.join(ROOT, "bench.py"), "--gpus", str(n), "--steps", "5", "--warmup", "3", "--scale", "0.25", "--no-cpu-baseline", "--collective", collective]
    env = dict(os.environ)
    if push:
        env["GB_PEER_PUSH"] = push  # fused: rows stored into the peers by the sweep; deferred: by the exchange kernel behind it
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    assert out.returncode == 0, out.stderr[-2000:]
    line = [l for l in out.stdout.splitlines() if l.startswith("{")][-1]
    return json.loads(line)


def test_two_gpu_exchange_paths_agree_with_one_gpu():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    one = _run(1, "fused", 29601)
    fused = _run(2, "fused", 29602, push="fused")
    deferred = _run(2, "fused", 29604, push="deferred")
    nccl = _run(2, "nccl", 29603)
    assert fused["slab_checksum"] == pytest.approx(one["slab_checksum"], rel=1e-6)
    assert deferred["slab_checksum"] == fused["slab_checksum"]  # same rows, only pushed by another kernel
    assert fused["parity_check"]["ok"] and deferred["parity_check"]["ok"]
    assert nccl["slab_checksum"] == pytest.approx(one["slab_checksum"], rel=1e-6)
    assert fused["n_gpus"] == 2 and nccl["n_gpus"] == 2
    # (no speed assertion: at this debug scale a step is ~0.2 ms and launch overheads dominate)
