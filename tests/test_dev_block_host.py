"""The pool block owner of glim_b200/csrc/gb_internal.cuh (gb_dev_block, gb_dev_carve), compiled for the host with nvcc against
a pool that records its calls (tests/cpp/dev_block_host.cu).  Every block goes back to the pool of the device its owner was made
for, including a block that an owner which was never carved takes over from a handle.  The carve sizes, takes and lays out one
block.  A move hands the block on, and an owner assigned to returns the block it held.  No device call: runs on the CPU-only box."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = "/usr/local/cuda/bin/nvcc"  # the toolkit glim_b200/csrc/Makefile builds with


def test_pool_blocks_return_to_their_owners_device(tmp_path):
    exe = str(tmp_path / "dev_block_host")
    subprocess.check_call([NVCC, "-std=c++17", "-ccbin", "/usr/bin/g++", "-o", exe, os.path.join(ROOT, "tests", "cpp", "dev_block_host.cu")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr
