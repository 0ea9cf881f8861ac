"""Sharded CCL through NCCL against a whole-volume oracle CCL: two ranks on two GPUs.  NCCL does
not put two ranks of one communicator on the same device, so a one-GPU machine runs the same path
with a single rank (communicator set-up, the all-gather, the replicated union-find and the
relabelling); the linking of two to eight ranks runs on one device in tests/test_ccl_multirank_gpu.py,
through the same ign_ccl6_volume_finish_gathered_dev, and over gloo in tests/test_multigpu_cpu.py."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sharded_ccl_over_nccl_matches_whole_volume(ctx):
  from igneous_b200 import _shim
  world = min(2, _shim.device_count())
  out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
                        "--master-addr", "127.0.0.1", "--master-port", "29571",
                        os.path.join(ROOT, "tools", "check_multigpu.py")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
  assert "MULTIGPU_CCL_PARITY OK" in out.stdout, out.stdout[-3000:]
