"""Real-to-complex line transforms (`rfft_` / `brfft_`, `pa_rfft`) on the GPU against numpy.fft,
at the FFT's own tolerance 8 eps log2(N) max|X|: single-rank lines (one launch per call, `src`
untouched), the real 3-d transform of a PencilFFTs real-input plan on one rank, and the same with
2 and 4 processes sharing the GPU (tests/mp_rfft_worker.py)."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import pencilarrays_b200 as pa

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
EPS = np.finfo(np.float64).eps


def tol(n, ref):
    return 8 * EPS * np.log2(n) * np.abs(ref).max()


def line_pencils(dims, perm=None):
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    permute = pa.Permutation(*perm) if perm else None
    pr = pa.Pencil(topo, dims, (2, 3), permute=permute)
    ax = (perm or (1, 2, 3))[0] - 1
    pc = pa.Pencil(pr, size_global=tuple(n // 2 + 1 if d == ax else n for d, n in enumerate(dims)))
    return pr, pc, dims[ax]


@pytest.mark.parametrize("dims,perm,extra", [((16, 3, 5), None, ()), ((64, 12, 8), None, ()),
                                             ((512, 8, 4), None, (2,)), ((2048, 3, 2), None, ()),
                                             ((32, 5, 7), (1, 3, 2), ()), ((128, 6, 3), (1, 3, 2), (3,))])
def test_rfft_then_brfft_single_rank(dims, perm, extra):
    pr, pc, N = line_pencils(dims, perm)
    xr = pa.PencilArray.undef(torch.float64, pr, *extra)
    xc = pa.PencilArray.undef(torch.complex128, pc, *extra)
    xr.data.normal_()
    before = xr.data.clone()
    n0 = pa.launch_count()
    assert pa.rfft_(xc, xr) is xc
    torch.cuda.synchronize()
    assert pa.launch_count() - n0 == 1
    assert torch.equal(xr.data.view(torch.uint8), before.view(torch.uint8))  # src untouched
    # torch (row-major) shape of a parent: the first memory dim -- the transform axis -- is LAST
    ref = np.fft.rfft(before.cpu().numpy(), axis=-1)
    got = xc.data.cpu().numpy()
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= tol(N, ref)

    # backward, from a spectrum whose bins 0 and N/2 carry imaginary parts (ignored, like numpy)
    xc.data.view(torch.float64).normal_()
    spec = xc.data.clone()
    back = pa.PencilArray.undef(torch.float64, pr, *extra)
    n0 = pa.launch_count()
    assert pa.brfft_(back, xc) is back
    torch.cuda.synchronize()
    assert pa.launch_count() - n0 == 1
    assert torch.equal(xc.data.view(torch.uint8), spec.view(torch.uint8))  # src untouched
    ref_b = N * np.fft.irfft(spec.cpu().numpy(), n=N, axis=-1)
    assert np.abs(back.data.cpu().numpy() - ref_b).max() <= tol(N, ref_b)

    # round trip
    pa.rfft_(xc, xr)
    pa.brfft_(back, xc)
    torch.cuda.synchronize()
    assert (back.data / N - before).abs().max().item() <= tol(N, before.cpu().numpy())


@pytest.mark.parametrize("dims,perm,decomp", [((6, 32, 4), (2, 1, 3), (1, 3)),
                                              ((5, 3, 64), (3, 1, 2), (1, 2)),
                                              ((7, 128, 3), (2, 3, 1), (1, 3))])
def test_transform_axis_is_the_first_memory_dim_not_logical_dim_1(dims, perm, decomp):
    """The transform axis is perm[1]: compared with numpy on the LOGICAL arrays, along that axis."""
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    ax = perm[0] - 1
    N = dims[ax]
    pr = pa.Pencil(topo, dims, decomp, permute=pa.Permutation(*perm))
    pc = pa.Pencil(pr, size_global=tuple(n // 2 + 1 if d == ax else n for d, n in enumerate(dims)))
    xr = pa.PencilArray.undef(torch.float64, pr)
    xc = pa.PencilArray.undef(torch.complex128, pc)
    xr.data.normal_()
    G = xr.logical().cpu().numpy().copy()
    pa.rfft_(xc, xr)
    torch.cuda.synchronize()
    ref = np.fft.rfft(G, axis=ax)
    got = xc.logical().cpu().numpy()
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= tol(N, ref)
    back = pa.PencilArray.undef(torch.float64, pr)
    pa.brfft_(back, xc)
    torch.cuda.synchronize()
    assert np.abs(back.logical().cpu().numpy() - N * G).max() <= tol(N, N * G)


def test_empty_local_array_launches_nothing():
    pr, pc, _ = line_pencils((32, 0, 4))
    xr = pa.PencilArray.undef(torch.float64, pr)
    xc = pa.PencilArray.undef(torch.complex128, pc)
    n0 = pa.launch_count()
    pa.rfft_(xc, xr)
    pa.brfft_(xr, xc)
    torch.cuda.synchronize()
    assert pa.launch_count() == n0


def test_refusals_on_device_arrays():
    pr, pc, _ = line_pencils((64, 4, 4))
    xr = pa.PencilArray.undef(torch.float64, pr)
    xc = pa.PencilArray.undef(torch.complex128, pc)
    with pytest.raises(pa.ArgumentError):  # complex pencil of the wrong size
        pa.rfft_(pa.PencilArray.undef(torch.complex128, pr), xr)
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pr24 = pa.Pencil(topo, (24, 4, 4), (2, 3))
    pc24 = pa.Pencil(pr24, size_global=(13, 4, 4))
    with pytest.raises(pa.ArgumentError):  # N not a power of two
        pa.rfft_(pa.PencilArray.undef(torch.complex128, pc24), pa.PencilArray.undef(torch.float64, pr24))
    pa.rfft_(xc, xr)
    torch.cuda.synchronize()


def real_chain(dims):
    """x (real and complex), y and z pencils of a PencilFFTs real-input plan on one rank."""
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pxr = pa.Pencil(topo, dims, (2, 3))
    pxc = pa.Pencil(pxr, size_global=(dims[0] // 2 + 1,) + tuple(dims[1:]))
    pyc = pa.Pencil(pxc, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    return pxr, pxc, pyc, pzc


@pytest.mark.parametrize("dims", [(16, 32, 8), (64, 64, 64), (128, 16, 32)])
def test_real_three_dimensional_fft_like_pencilffts(dims):
    """rfft_ along x, then x->y and y->z with the next complex transform fused: the z-pencil
    array, read in logical order, is fftn(rfft(G, axis=0), axes=(1, 2)); the backward chain
    (fft_ along z, fused z->y, plain y->x, brfft_) returns prod(dims) times the input."""
    pxr, pxc, pyc, pzc = real_chain(dims)
    uxr = pa.PencilArray.undef(torch.float64, pxr)
    uxc, uyc, uzc = (pa.PencilArray.undef(torch.complex128, p) for p in (pxc, pyc, pzc))
    uxr.data.normal_()
    G = uxr.logical().cpu().numpy().copy()
    pa.rfft_(uxc, uxr)
    pa.transpose_(pa.Transposition(uyc, uxc), fft="forward")
    pa.transpose_(pa.Transposition(uzc, uyc), fft="forward")
    torch.cuda.synchronize()
    ref = np.fft.fftn(np.fft.rfft(G, axis=0), axes=(1, 2))
    n = math.prod(dims)
    assert np.abs(uzc.logical().cpu().numpy() - ref).max() <= tol(n, ref)
    pa.fft_(uzc, "backward")
    pa.transpose_(pa.Transposition(uyc, uzc), fft="backward")
    pa.transpose_(pa.Transposition(uxc, uyc))
    back = pa.PencilArray.undef(torch.float64, pxr)
    pa.brfft_(back, uxc)
    torch.cuda.synchronize()
    assert np.abs(back.logical().cpu().numpy() - n * G).max() <= tol(n, n * G)


@pytest.mark.parametrize("nproc", [2, 4])
def test_real_three_dimensional_fft_ranks_sharing_the_gpu(nproc, tmp_path):
    """2 / 4 processes over the NCCL-free communicator, PointToPoint and Alltoallv: the odd
    N/2+1 axis splits unevenly once the y and z pencils decompose it."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(29671 + nproc),
           os.path.join(HERE, "mp_rfft_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1", PA_TEST_TMPDIR=str(tmp_path))
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    assert f"MP_RFFT_OK world={nproc}" in out.stdout, out.stdout[-2000:]
