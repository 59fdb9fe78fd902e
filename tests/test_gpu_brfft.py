"""The fused y->x transpose + complex-to-real transform (`Transposition(..., brfft=True)`,
`pa_transpose_brfft`) on the GPU.  It runs the gather of the fused unpack+FFT and the backward
half of `brfft_`, so its output must be the bytes of `brfft_(transpose_(y->x))` -- in both
precisions, at every line length, through both gathers.  Plus: bins 0 and N/2 ignored, no side
effects, refusals that launch nothing, the 3-kernel real backward chain, caller streams, and 2, 3,
4 and 8 processes sharing the GPU (tests/mp_brfft_worker.py)."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200 import _lib
from pencilarrays_b200._lib import lib
from gpu_util import hold, stream_ptr

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
PREC = {"f64": (torch.float64, torch.complex128, np.finfo(np.float64).eps, 0),
        "f32": (torch.float32, torch.complex64, np.finfo(np.float32).eps, _lib.PA_FFT_F32)}


def chain(dims, xperm=None, yperm=(2, 1, 3)):
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pxr = pa.Pencil(topo, dims, (2, 3), permute=pa.Permutation(*xperm) if xperm else None)
    ax = (xperm or (1, 2, 3))[0] - 1
    pxc = pa.Pencil(pxr, size_global=tuple(n // 2 + 1 if d == ax else n for d, n in enumerate(dims)))
    pyc = pa.Pencil(pxc, decomp_dims=(1, 3), permute=pa.Permutation(*yperm) if yperm else pa.NoPermutation())
    pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    return pxr, pxc, pyc, pzc


def bits(u):
    return u.data.contiguous().view(torch.uint8).reshape(-1)


def fused_and_plain(pxr, pxc, src, rdt, cdt, extra=(), **kw):
    """(fused result, plain transpose + brfft_ result, launches of the fused call)."""
    fused = pa.PencilArray.undef(rdt, pxr, *extra)
    bits(fused).fill_(0x5A)
    t = pa.Transposition(fused, src, brfft=True)
    assert t.fft_fusable()
    n0 = pa.launch_count()
    pa.transpose_(t, **kw)
    torch.cuda.synchronize()
    n = pa.launch_count() - n0
    ux = pa.PencilArray.undef(cdt, pxc, *extra)
    pa.transpose_(pa.Transposition(ux, src), **kw)
    plain = pa.PencilArray.undef(rdt, pxr, *extra)
    pa.brfft_(plain, ux)
    torch.cuda.synchronize()
    return fused, plain, n


NS = [16, 32, 64, 128, 256, 512, 1024, 2048]


@pytest.mark.parametrize("prec", PREC)
@pytest.mark.parametrize("N", NS)
def test_bytes_equal_the_unfused_path_one_rank(prec, N):
    """y->x with one rank (transposing gather; 3 and 5 columns, not a multiple of C) and the
    identity plan x->x (linear gather).  With one rank the fused kernel reads the whole local array
    straight from src, with or without stage_self (only the unfused side stages it); the gather of
    a staged self block from the recv_buf tail is covered by the stage_self variant of
    tests/mp_brfft_worker.py."""
    rdt, cdt, _, _ = PREC[prec]
    pxr, pxc, pyc, _ = chain((N, 5, 3))
    uy = pa.PencilArray.undef(cdt, pyc)
    uy.data.view(rdt).normal_()
    before = uy.data.clone()
    for kw in (dict(), dict(stage_self=True)):
        fused, plain, n = fused_and_plain(pxr, pxc, uy, rdt, cdt, **kw)
        assert n == 1
        assert torch.equal(bits(fused), bits(plain)), (N, kw)
        assert torch.equal(uy.data.view(torch.uint8), before.view(torch.uint8))  # src untouched
    # identity plan: the complex x-pencil array itself (its own pencil object, same geometry)
    ux = pa.PencilArray.undef(cdt, pa.Pencil(pxr, size_global=pxc.size_global))
    ux.data.view(rdt).normal_()
    fused, plain, n = fused_and_plain(pxr, ux.pencil, ux, rdt, cdt)
    assert n == 1 and torch.equal(bits(fused), bits(plain)), N


@pytest.mark.parametrize("prec", PREC)
@pytest.mark.parametrize("dims,xperm,yperm,extra", [
    ((64, 7, 3), (1, 3, 2), (2, 1, 3), ()),
    ((32, 6, 5), None, (2, 3, 1), (3,)),
    ((256, 3, 2), (1, 3, 2), (3, 2, 1), (2, 1, 3)),
    ((16, 3, 2), None, None, (1, 2, 1, 3, 2)),          # 3 + 5 dims = PA_MAX_DIMS
    ((2048, 3, 1), None, (2, 1, 3), (2, 3)),
])
def test_bytes_equal_with_permutations_and_extra_dims(prec, dims, xperm, yperm, extra):
    rdt, cdt, _, _ = PREC[prec]
    pxr, pxc, pyc, _ = chain(dims, xperm, yperm)
    uy = pa.PencilArray.undef(cdt, pyc, *extra)
    uy.data.view(rdt).normal_()
    for kw in (dict(), dict(stage_self=True)):
        fused, plain, n = fused_and_plain(pxr, pxc, uy, rdt, cdt, extra, **kw)
        assert n == 1 and torch.equal(bits(fused), bits(plain)), (dims, kw)


@pytest.mark.parametrize("prec", PREC)
def test_imaginary_parts_of_bins_0_and_n_over_2_are_ignored(prec):
    rdt, cdt, _, _ = PREC[prec]
    N = 128
    pxr, pxc, pyc, _ = chain((N, 6, 5))
    uy = pa.PencilArray.undef(cdt, pyc)
    uy.data.view(rdt).normal_()
    a = pa.PencilArray.undef(rdt, pxr)
    pa.transpose_(pa.Transposition(a, uy, brfft=True))
    for k in (0, N // 2):
        uy.logical()[k].imag.normal_()
    b = pa.PencilArray.undef(rdt, pxr)
    pa.transpose_(pa.Transposition(b, uy, brfft=True))
    torch.cuda.synchronize()
    assert torch.equal(bits(a), bits(b))


def test_canaries_around_dst_and_empty_local_arrays():
    rdt, cdt = torch.float64, torch.complex128
    pxr, pxc, pyc, _ = chain((64, 5, 3))
    uy = pa.PencilArray.undef(cdt, pyc)
    uy.data.normal_()
    t = pa.Transposition(pa.PencilArray.undef(rdt, pxr), uy, brfft=True)
    nbytes = 64 * 5 * 3 * 8
    buf = torch.full((nbytes + 512,), 0xA5, dtype=torch.uint8, device="cuda")
    rc = lib.pa_transpose_brfft(t.plan.h, None, pxr._h, C.c_void_p(uy.data_ptr()),
                                C.c_void_p(buf.data_ptr() + 256), _lib.PA_WAITALL, stream_ptr())
    assert rc == _lib.PA_OK, lib.pa_last_error()
    torch.cuda.synchronize()
    assert bool((buf[:256] == 0xA5).all()) and bool((buf[256 + nbytes:] == 0xA5).all())
    ref = pa.PencilArray.undef(rdt, pxr)
    pa.transpose_(pa.Transposition(ref, uy, brfft=True))
    torch.cuda.synchronize()
    assert torch.equal(buf[256:256 + nbytes], bits(ref))
    # an empty local array: nothing launched
    exr, exc, eyc, _ = chain((64, 0, 3))
    ey = pa.PencilArray.undef(cdt, eyc)
    n0 = pa.launch_count()
    pa.transpose_(pa.Transposition(pa.PencilArray.undef(rdt, exr), ey, brfft=True))
    torch.cuda.synchronize()
    assert pa.launch_count() == n0


def test_refusals_launch_nothing_and_leave_dst_untouched():
    rdt, cdt = torch.float64, torch.complex128
    pxr, pxc, pyc, _ = chain((24, 4, 4))                 # N = 24: refused by the check
    uy = pa.PencilArray.undef(cdt, pyc)
    uy.data.normal_()
    out = pa.PencilArray.undef(rdt, pxr)
    bits(out).fill_(0x3C)
    torch.cuda.synchronize()
    before = out.data.clone()
    t = pa.Transposition(out, uy, brfft=True)
    assert not t.fft_fusable()
    n0 = pa.launch_count()
    with pytest.raises(pa.ArgumentError):
        pa.transpose_(t)
    # bad flags / precision / overlap through the ABI, on device pointers
    h, s, d, st = t.plan.h, C.c_void_p(uy.data_ptr()), C.c_void_p(out.data_ptr()), stream_ptr()
    good_r, good_c, good_y, _ = chain((32, 4, 4))
    gy = pa.PencilArray.undef(cdt, good_y)
    gx = pa.PencilArray.undef(rdt, good_r)
    bits(gx).fill_(0x3C)
    gbefore = gx.data.clone()
    gt = pa.Transposition(gx, gy, brfft=True)
    gs, gd = C.c_void_p(gy.data_ptr()), C.c_void_p(gx.data_ptr())
    for flags in (_lib.PA_FFT_BACKWARD, _lib.PA_FFT_F32, 64):
        assert lib.pa_transpose_brfft(gt.plan.h, None, good_r._h, gs, gd, flags, st) == _lib.PA_EINVAL
    assert lib.pa_transpose_brfft(gt.plan.h, None, good_r._h, gs, C.c_void_p(gy.data_ptr()), 0, st) \
        == _lib.PA_EINVAL                                 # overlap
    assert lib.pa_transpose_brfft(gt.plan.h, None, good_c._h, gs, gd, 0, st) == _lib.PA_EINCOMPAT
    assert lib.pa_transpose_brfft(h, None, pxr._h, s, d, 0, st) == _lib.PA_EINVAL
    torch.cuda.synchronize()
    assert pa.launch_count() == n0
    assert torch.equal(out.data.view(torch.uint8), before.view(torch.uint8))
    assert torch.equal(gx.data.view(torch.uint8), gbefore.view(torch.uint8))


@pytest.mark.parametrize("prec", PREC)
@pytest.mark.parametrize("dims", [(16, 32, 8), (64, 64, 64), (128, 16, 32)])
def test_real_backward_chain_is_three_kernels(prec, dims):
    """fft_ along z, fused z->y, fused y->x + brfft: prod(dims) times the field."""
    rdt, cdt, eps, _ = PREC[prec]
    pxr, pxc, pyc, pzc = chain(dims)
    uxr = pa.PencilArray.undef(rdt, pxr)
    uxr.data.normal_()
    G = uxr.logical().cpu().numpy().astype(np.float64)
    uxc, uyc, uzc = (pa.PencilArray.undef(cdt, p) for p in (pxc, pyc, pzc))
    pa.rfft_(uxc, uxr)
    pa.transpose_(pa.Transposition(uyc, uxc), fft="forward")
    pa.transpose_(pa.Transposition(uzc, uyc), fft="forward")
    back = pa.PencilArray.undef(rdt, pxr)
    t_zy, t_yx = pa.Transposition(uyc, uzc), pa.Transposition(back, uyc, brfft=True)
    torch.cuda.synchronize()
    n0 = pa.launch_count()
    pa.fft_(uzc, "backward")
    pa.transpose_(t_zy, fft="backward")
    pa.transpose_(t_yx)
    torch.cuda.synchronize()
    assert pa.launch_count() - n0 == 3
    n = math.prod(dims)
    err = np.abs(back.logical().cpu().numpy().astype(np.float64) - n * G).max()
    assert err <= 8 * eps * np.log2(n) * n * np.abs(G).max(), err


def test_ordered_on_a_held_caller_stream():
    """On a side stream held by a spin, the call returns before the spin ends, and its result
    (produced behind the hold) equals the default-stream result byte for byte."""
    rdt, cdt = torch.float64, torch.complex128
    pxr, pxc, pyc, _ = chain((512, 16, 8))
    uy = pa.PencilArray.undef(cdt, pyc)
    uy.data.normal_()
    ref = pa.PencilArray.undef(rdt, pxr)
    pa.transpose_(pa.Transposition(ref, uy, brfft=True))
    torch.cuda.synchronize()
    out = pa.PencilArray.undef(rdt, pxr)
    t = pa.Transposition(out, uy, brfft=True)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        held = hold()
        uy2 = uy.data.clone()      # the input, produced behind the hold
        src = pa.PencilArray(pyc, uy2)
        pa.transpose_(pa.Transposition(out, src, brfft=True))
        assert not held.query()
    side.synchronize()
    assert torch.equal(bits(out), bits(ref))
    del t


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_ranks_sharing_the_gpu(world, tmp_path):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29851 + world),
           os.path.join(HERE, "mp_brfft_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1", PA_TEST_TMPDIR=str(tmp_path))
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    assert f"MP_BRFFT_OK world={world}" in out.stdout, out.stdout[-2000:]
