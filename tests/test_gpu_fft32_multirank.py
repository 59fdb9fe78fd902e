"""Single-precision FFTs with 2, 3, 4 and 8 processes sharing the GPU over the NCCL-free
communicator (tests/mp_fft32_worker.py): the real Float32 3-d transform on 2 and 4 ranks, the
fused ComplexF32 gather from 3 and 8 ranks under every staged schedule, and a refused shape that
launches nothing on any rank."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_single_precision_ffts_ranks_sharing_the_gpu(world, tmp_path):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29811 + world),
           os.path.join(HERE, "mp_fft32_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1", PA_TEST_TMPDIR=str(tmp_path))
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    assert f"MP_FFT32_OK world={world}" in out.stdout, out.stdout[-2000:]
