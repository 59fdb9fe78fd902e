"""The fused unpack+FFT gathering each line from 3, 5, 6 and 8 blocks (uneven splits, one row
per block, empty destinations), every staged schedule, and the refusals that must launch
nothing: processes sharing the GPU over the NCCL-free communicator (tests/mp_fft_worker.py)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.parametrize("world", [5, 6, 8])
def test_fused_fft_multi_block_gathers(world, tmp_path):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29751 + world),
           os.path.join(HERE, "mp_fft_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1", PA_TEST_TMPDIR=str(tmp_path))
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    assert f"MP_FFT_OK world={world}" in out.stdout, out.stdout[-2000:]
