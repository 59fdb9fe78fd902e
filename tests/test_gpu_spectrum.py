"""Shell-binned spectra on the GPU (pa_shell_spectrum, pa.shell_spectrum), one process, against the
NumPy reference of tests/spectrum_ref.py: bins bit for bit (the dropped modes included), each bin
within the rounding bound of DESIGN §3m against math.fsum; both element types, abs2 and realdot,
2-d, 3-d (every permutation) and 4-d pencils with and without extra dims, every r2c dim and none;
offset bases, NaN, empty arrays; determinism, one launch per call, refusals, stream ordering; and
Parseval through rfft_ and the two fused transposes.  tests/mp_spectrum_worker.py runs it with 2,
3, 4 and 8 processes sharing the GPU."""
import ctypes as C
import itertools
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
from reduce_dims_ref import logical_view
import spectrum_ref as R

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CTYPES = [torch.complex128, torch.complex64]


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def pencil(dims, perm=None):
    N = len(dims)
    grid, decomp = ((1,), (2,)) if N == 2 else ((1, 1), (2, 3))
    kw = {"permute": pa.Permutation(*perm)} if perm else {}
    return pa.Pencil(pa.MPITopology(pa.COMM_SELF, grid), dims, decomp, **kw)


def make(dtype, pen, extra=(), offset=0, seed=0):
    """A PencilArray `offset` elements into its allocation, and its logical-order numpy copy
    (spatial dims first, extra dims last)."""
    rng = np.random.default_rng(seed)
    mem = pa.size_local(pen, pa.MemoryOrder())
    shape = tuple(reversed(mem + tuple(extra)))
    n = math.prod(shape)
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 10.0 ** rng.integers(-2, 2, n)
    x = x.astype(np.complex128 if dtype == torch.complex128 else np.complex64)
    buf = torch.empty(n + offset, dtype=dtype, device="cuda")
    buf[offset:].copy_(torch.from_numpy(x))
    u = pa.PencilArray(pen, buf[offset:].view(shape), tuple(extra))
    return u, logical_view(u, u.data).cpu().numpy()


def check(u, x, v=None, y=None, what="", **kw):
    N = len(u.space_dims)
    got = pa.shell_spectrum(u, v, **kw)
    nb = kw.get("nbins") or R.default_nbins(x.shape[:N], kw.get("rfft_dim"), kw.get("scales"),
                                            kw.get("width", 1.0))
    assert got.shape == (nb,) and got.device == u.data.device
    assert got.dtype == (torch.float64 if u.dtype == torch.complex128 else torch.float32)
    exact, absum = R.spectrum(x, N, nb, y, kw.get("rfft_dim"), kw.get("rfft_n"), kw.get("scales"),
                              kw.get("width", 1.0))
    R.check_bins(got.cpu().numpy(), exact, absum, x.size, sms(), u.dtype == torch.complex64,
                 what=(what, kw))
    return got


CASES = [((9, 12), None), ((9, 12), (2, 1))] + \
        [((7, 6, 5), p) for p in itertools.permutations((1, 2, 3))] + \
        [((5, 4, 3, 6), None), ((5, 4, 3, 6), (4, 2, 3, 1))]


@pytest.mark.parametrize("size,perm", CASES)
@pytest.mark.parametrize("dtype", CTYPES)
def test_abs2_every_rfft_dim_against_numpy(size, perm, dtype):
    pen = pencil(size, perm)
    for extra in ((), (3,)):
        u, x = make(dtype, pen, extra, seed=len(extra))
        for rd in [None] + list(range(1, len(size) + 1)):
            check(u, x, what=(size, perm, extra), rfft_dim=rd)
        # anisotropic scales, a width off 1, odd rfft_n and fewer bins than the default
        check(u, x, what="scales", rfft_dim=1, rfft_n=2 * size[0] - 1,
              scales=tuple(0.5 + 0.25 * d for d in range(len(size))), width=0.7)
        nb = pa.spectrum_nbins(u)
        check(u, x, what="dropped", nbins=max(1, nb // 2))


@pytest.mark.parametrize("boff", [0, 1])
@pytest.mark.parametrize("dtype", CTYPES)
def test_realdot_at_equal_and_different_alignments(dtype, boff):
    pen = pencil((16, 6, 7), (2, 3, 1))
    u, x = make(dtype, pen, (2,), seed=1)
    v, y = make(dtype, pen, (2,), offset=boff, seed=2)
    for rd in (None, 1, 3):
        check(u, x, v, y, what=boff, rfft_dim=rd)
    # realdot of u with itself is the abs2 spectrum bit for bit
    a = pa.shell_spectrum(u, u, rfft_dim=2)
    b = pa.shell_spectrum(u, rfft_dim=2)
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


def test_complexf64_off_16_bytes():
    """ComplexF64 arrays at an odd 8 bytes (element loads), alone and against an aligned one."""
    pen = pencil((11, 6, 5))
    n = 11 * 6 * 5
    rng = np.random.default_rng(4)
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    y = (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    raw = torch.zeros(2 * n + 2, dtype=torch.float64, device="cuda")
    raw[1:2 * n + 1].copy_(torch.from_numpy(x.view(np.float64)))
    yb = torch.from_numpy(y).cuda()
    xl = x.reshape(5, 6, 11).transpose(2, 1, 0)
    yl = y.reshape(5, 6, 11).transpose(2, 1, 0)
    nb = R.default_nbins((11, 6, 5))
    for b, yy, m in ((None, None, _lib.PA_MAP_ABS2), (yb, yl, _lib.PA_MAP_DOT)):
        res = torch.empty(nb, dtype=torch.float64, device="cuda")
        assert lib.pa_shell_spectrum(pen._h, 0, None, None, _lib.PA_COMPLEXF64, m,
                                     C.c_void_p(raw.data_ptr() + 8),
                                     C.c_void_p(b.data_ptr()) if b is not None else None, 0, 0,
                                     None, 1.0, nb, C.c_void_p(res.data_ptr()), stream_ptr()) == 0
        exact, absum = R.spectrum(xl, 3, nb, yy)
        R.check_bins(res.cpu().numpy(), exact, absum, n, sms(), False, what=m)


@pytest.mark.parametrize("dtype", CTYPES)
def test_offset_bases_and_nan_confined_to_its_bin(dtype):
    pen = pencil((33, 9, 5), (3, 1, 2))
    for off in (1, 3):
        u, x = make(dtype, pen, (2,), offset=off, seed=off)
        check(u, x, what=off, rfft_dim=2)
    u, x = make(dtype, pen, seed=9)
    idx = (3, 4, 0)  # wavenumbers (3, 4, 0): |k| = 5
    x[idx] = np.nan
    logical_view(u, u.data)[idx] = complex(np.nan, 0.0)
    got = check(u, x, what="nan")
    assert np.isnan(got.cpu().numpy()).sum() == 1 and np.isnan(got[5].item())


def test_empty_local_and_global_arrays():
    pen = pencil((0, 5, 4))
    u = pa.PencilArray.undef(torch.complex128, pen)
    r = pa.shell_spectrum(u)
    assert r.shape == (pa.spectrum_nbins(u),) and bool((r == 0).all())
    r = pa.shell_spectrum(u, u, nbins=7, rfft_dim=2)
    assert r.shape == (7,) and bool((r == 0).all())
    torch.cuda.synchronize()


def test_two_calls_bitwise_equal_and_one_launch_each():
    pen = pencil((129, 256, 64), (3, 2, 1))
    for dtype in CTYPES:
        u, _ = make(dtype, pen, (2,))
        for kw in ({}, {"rfft_dim": 1}, {"nbins": 40, "width": 2.0}):
            a = pa.shell_spectrum(u, **kw)
            n0 = pa.launch_count()
            b = pa.shell_spectrum(u, **kw)
            assert pa.launch_count() - n0 == 1
            assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


def test_refused_call_launches_nothing_and_leaves_the_result_untouched():
    pen = pencil((16, 21, 41))
    u, _ = make(torch.complex128, pen)
    guard = torch.full((4096 * 8 + 64,), 0x5A, dtype=torch.uint8, device="cuda")
    res = C.c_void_p(guard.data_ptr() + 32)
    a = C.c_void_p(u.data_ptr())
    n0 = pa.launch_count()

    def call(dtype=_lib.PA_COMPLEXF64, m=_lib.PA_MAP_ABS2, b=None, rd=0, rn=0, w=1.0, nb=10,
             r=res, comm=None):
        return lib.pa_shell_spectrum(pen._h, 0, None, comm, dtype, m, a, b, rd, rn, None, w, nb, r,
                                     stream_ptr())
    for kw in ({"dtype": _lib.PA_FLOAT64}, {"m": _lib.PA_MAP_ABS}, {"b": a}, {"m": _lib.PA_MAP_DOT},
               {"rd": 4}, {"rd": 1, "rn": 3}, {"w": 0.0}, {"nb": 0}, {"nb": 4097},
               {"r": C.c_void_p(guard.data_ptr() + 33)}):
        assert call(**kw) == _lib.PA_EINVAL, kw
        assert lib.pa_last_error().decode().startswith("pa_shell_spectrum:")
    h = C.c_void_p()
    assert lib.pa_comm_init_local(2, 0, C.byref(h)) == 0
    try:
        assert call(comm=h) == _lib.PA_EINCOMPAT
    finally:
        lib.pa_comm_destroy(h)
    assert pa.launch_count() == n0
    torch.cuda.synchronize()
    assert bool((guard == 0x5A).all())


def test_stream_ordering_without_host_sync():
    pen = pencil((64, 32, 16))
    u = pa.PencilArray.undef(torch.complex128, pen)
    u.data.fill_(1.0)
    pa.shell_spectrum(u)  # warm-up
    nb = pa.spectrum_nbins(u)
    count = np.bincount(R.shells((64, 32, 16)).reshape(-1).astype(np.int64), minlength=nb)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        held = hold()
        u.data.fill_(2.0)          # produced behind the hold
        r = pa.shell_spectrum(u)
        m = pa.sum(u, pa.abs2)
        assert not held.query()    # the calls did not wait for the device
    torch.cuda.synchronize()
    assert np.array_equal(r.cpu().numpy(), 4.0 * count) and m.item() == 4.0 * 64 * 32 * 16


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_parseval_through_rfft_and_the_fused_transposes(dtype):
    """E of the forward transform of a real field sums to N_total * sum(u^2)."""
    dims = (64, 32, 16)
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    ctype = torch.complex128 if dtype == torch.float64 else torch.complex64
    pxr = pa.Pencil(topo, dims, (2, 3))
    pxc = pa.Pencil(pxr, size_global=(dims[0] // 2 + 1,) + dims[1:])
    pyc = pa.Pencil(pxc, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    ur = pa.PencilArray.undef(dtype, pxr)
    g = np.random.default_rng(3).standard_normal(dims)
    logical_view(ur, ur.data).copy_(torch.from_numpy(g))
    uxc, uyc, uzc = (pa.PencilArray.undef(ctype, p) for p in (pxc, pyc, pzc))
    pa.rfft_(uxc, ur)
    pa.transpose_(pa.Transposition(uyc, uxc), fft="forward")
    pa.transpose_(pa.Transposition(uzc, uyc), fft="forward")
    E = pa.shell_spectrum(uzc, rfft_dim=1, rfft_n=dims[0])
    s = pa.sum(ur, pa.abs2)
    ntot = math.prod(dims)
    total, want = math.fsum(E.double().cpu().numpy()), ntot * s.item()
    eps = 2.0 ** -53 if dtype == torch.float64 else 2.0 ** -24
    # the FFT's error (a few eps log2 n relative), the spectrum's and the sum's roundings
    tol = (8 * math.log2(ntot) + R.depth(uzc.data.numel(), sms()) + 64) * eps * want
    assert abs(total - want) <= tol, (total, want, tol)
    # every mode in some bin: the default nbins covers them
    assert E.numel() == R.default_nbins(pa.size_global(pzc, pa.LogicalOrder()), 1)


@pytest.mark.parametrize("nproc", [2, 3, 4, 8])
def test_ranks_sharing_the_gpu(nproc):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(29851 + nproc),
           os.path.join(HERE, "mp_spectrum_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1")
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    assert f"MP_SPECTRUM_OK world={nproc}" in out.stdout, out.stdout[-2000:]
