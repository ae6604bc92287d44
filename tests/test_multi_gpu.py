"""Row-sharded frames on real GPUs against the single-GPU frame, with both exchange paths of the C++
graph: peer-memory stores from the downsample kernel (default) and NCCL broadcasts + all-reduce.

The frame is split over 4 ranks where the machine has 4 GPUs, else over 2.  On a single GPU the two ranks
share it (see multi_gpu_worker.py): every sharded step still runs, on one device."""
import os
import signal
import subprocess
import sys

import pytest

from tests import common

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpu_count():
    import torch

    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
@pytest.mark.parametrize("fxaa", [0, 1])
def test_sharded_frame_is_bit_identical(cuda, fxaa, exchange):
    world = 4 if _gpu_count() >= 4 else 2
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(common.free_port()), os.path.join(ROOT, "tests", "multi_gpu_worker.py"), "1280", "768", "300", str(fxaa)]
    env = dict(os.environ, GRB_SHARD_EXCHANGE=exchange)
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, cwd=ROOT, env=env, start_new_session=True)
    try:
        out, err = proc.communicate(timeout=600)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)  # the launcher and every rank
        out, err = proc.communicate()
        pytest.fail("the sharded run did not finish in 600 s:\n" + out[-3000:] + err[-3000:])
    sys.stdout.write(out[-3000:])
    assert proc.returncode == 0, out[-3000:] + err[-3000:]
    assert out.count(f"sharded over {world} ranks == single GPU: True") == 3, out[-3000:]
    if exchange == "peer":
        assert "peer-memory exchange unavailable" not in out + err, "IPC works between the ranks: the peer path must be the one that ran"
