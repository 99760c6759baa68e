"""Multi-GPU parity of the flat-bucket sharded data-parallel runtime over NCCL (SURVEY section 8 row a21 / e; reference:
distributed/__init__.py:126-230 wrapping, train_utils.py:18-116 accumulation under `no_sync`).

Each case launches `tools/ddp_parity.py` with `torch.distributed.run` on the GPUs of this box: every rank feeds its own
micro-batches to the sharded model while rank 0 also runs an unsharded copy over all of them; mean loss, every rank-0
gradient shard (reduce-scatter AVG) and the parameters the next all-gather delivers must agree for four optimizer steps.
Skipped on machines with fewer GPUs than the case needs."""

import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (ranks, environment of tools/ddp_parity.py)
CASES = {
    "resident_fp32": (2, dict(COMM_DTYPE="fp32", RESHARD="0")),
    "resident_bf16_accum2": (2, dict(COMM_DTYPE="bf16", RESHARD="0", ACCUM="2")),
    "stage3_reshard_bf16": (2, dict(COMM_DTYPE="bf16", RESHARD="1")),
    "stage3_reshard_fp32_accum2_ckpt": (2, dict(COMM_DTYPE="fp32", RESHARD="1", ACCUM="2", CKPT="2")),
    "hsdp_2x2_bf16": (4, dict(COMM_DTYPE="bf16", RESHARD="1", SHARD="2")),
    # MoE blocks: expert weight gradients are written by overwriting K-grouped GEMMs into the shared (stage 3) gradient buffers
    "moe_stage3_reshard_fp32_accum2": (2, dict(COMM_DTYPE="fp32", RESHARD="1", ACCUM="2", MOE="1")),
    "moe_resident_bf16_accum2": (2, dict(COMM_DTYPE="bf16", RESHARD="0", ACCUM="2", MOE="1")),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_sharded_equals_unsharded_over_nccl(name):
    ranks, env_add = CASES[name]
    if torch.cuda.device_count() < ranks:
        pytest.skip(f"needs {ranks} GPUs, this box has {torch.cuda.device_count()}")
    env = dict(os.environ)
    env.update(env_add)
    port = 29600 + (os.getpid() + sorted(CASES).index(name)) % 300
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={ranks}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tools", "ddp_parity.py")]
    proc = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    tail = (proc.stdout + proc.stderr)[-3000:]
    assert proc.returncode == 0, tail
    assert "DDP_PARITY OK" in proc.stdout, tail
