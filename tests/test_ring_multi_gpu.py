"""Multi-GPU parity of the sequence-parallel attention op (skipped unless >= 2 GPUs are visible), against the float64
ORACLE: (1) dense oracle at a small size — forward and all gradients, both work assignments, masks, fp32 and bf16
inputs, decode op; (2) the row-wise oracle at the benchmark length of the visible GPU count (32K tokens on 2 GPUs =
configs[1]; 128K on 8 = configs[2])."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _n_gpus():
    n = torch.cuda.device_count()
    return 8 if n >= 8 else 4 if n >= 4 else 2


def _launch(env_extra, port):
    env = dict(os.environ, **env_extra)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(_n_gpus()),
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(ROOT, "tests", "ring_multi_gpu_worker.py")], capture_output=True, text=True,
                       timeout=900, env=env)
    assert r.returncode == 0 and "RING_MULTI_GPU OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_ring_on_all_visible_gpus_dense_oracle():
    _launch({}, 29571)


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_ring_on_all_visible_gpus_nccl_transport_dense_oracle():
    """the two-sided executor (ring_exec.py) on real NCCL side streams: fp32 inputs reach it as bf16 operands, and the
    worker then holds their results to the bf16-result bound"""
    _launch({"LWM_RING_TRANSPORT": "nccl"}, 29573)


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_ring_on_all_visible_gpus_baseline_length_sampled_oracle():
    n = _n_gpus()
    _launch({"RING_TEST_MODE": "sampled", "RING_TEST_S": str(32768 if n == 2 else 65536 if n == 4 else 131072)}, 29572)
