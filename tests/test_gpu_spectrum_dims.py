"""Spectra over chosen dims on the GPU (pa_shell_spectrum_dims, pa.shell_spectrum(dims=, keep=)),
one process, against the NumPy reference of tests/spectrum_dims_ref.py: every (bin subset, keep
subset) on 2-d, 3-d (every permutation) and 4-d pencils with and without extra dims, every r2c dim
and none, both element types, abs2 and realdot, each value within the bound of DESIGN §3n against
math.fsum; the unchanged pa_shell_spectrum path; kept sums against summed calls; misaligned and
offset bases, NaN, empty arrays, the partial-area refusal; determinism, one launch per call,
refusals, stream ordering; and E(k_h; y) through rfft_ and a fused transpose.
tests/mp_spectrum_dims_worker.py runs it with 2, 3, 4 and 8 processes sharing the GPU."""
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
import spectrum_dims_ref as RD

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
    """A PencilArray `offset` elements into its allocation, and its logical-order numpy copy."""
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


def as_logical(u, got, keep):
    """The library's result (u.data's layout, non-kept positions 1, bins last) as an array of the
    kept dims in logical order, bins last."""
    nb = got.shape[-1]
    if not keep:
        return got.cpu().numpy()
    lv = torch.stack([logical_view(u, got[..., b]) for b in range(nb)], -1).cpu().numpy()
    return lv.reshape(tuple(lv.shape[d - 1] for d in sorted(keep)) + (nb,))


def check(u, x, v=None, y=None, dims=None, keep=(), what="", **kw):
    N = len(u.space_dims)
    dims_ = tuple(range(1, N + 1)) if dims is None else tuple(dims)
    got = pa.shell_spectrum(u, v, dims=dims_, keep=keep, **kw)
    nb = kw.get("nbins") or RD.default_nbins(x.shape[:N], dims_, kw.get("rfft_dim"),
                                             kw.get("scales"), kw.get("width", 1.0))
    shape = [1] * u.data.dim()
    for d in keep:
        shape[d - 1] = x.shape[d - 1]
    assert got.dtype == (torch.float64 if u.dtype == torch.complex128 else torch.float32)
    assert got.shape[-1] == nb and got.numel() == math.prod(shape) * nb, (got.shape, what)
    exact, absum = RD.spectrum(x, N, nb, dims_, tuple(sorted(keep)), y, kw.get("rfft_dim"),
                               kw.get("rfft_n"), kw.get("scales"), kw.get("width", 1.0))
    nslab = x.size // max(1, math.prod(shape))
    RD.check(as_logical(u, got, keep), exact, absum, nslab, sms(), u.dtype == torch.complex64,
             what=(what, dims_, keep, kw))
    return got


def subsets(xs, lo=0):
    for r in range(lo, len(xs) + 1):
        yield from itertools.combinations(xs, r)


CASES = [((9, 12), None), ((9, 12), (2, 1))] + \
        [((7, 6, 5), p) for p in itertools.permutations((1, 2, 3))] + \
        [((5, 4, 3, 6), None), ((5, 4, 3, 6), (4, 2, 3, 1))]


@pytest.mark.parametrize("size,perm", CASES)
@pytest.mark.parametrize("dtype", CTYPES)
def test_every_bin_and_keep_subset_against_numpy(size, perm, dtype):
    N = len(size)
    pen = pencil(size, perm)
    for extra in ((), (3,)):
        u, x = make(dtype, pen, extra, seed=len(extra))
        nl = N + len(extra)
        for dims in subsets(range(1, N + 1), 1):
            rest = [d for d in range(1, nl + 1) if d not in dims]
            for keep in subsets(rest):
                rds = [None] + list(range(1, N + 1)) if len(size) < 4 or len(keep) < 2 else [None, 1]
                for rd in rds:
                    check(u, x, dims=dims, keep=keep, rfft_dim=rd, what=(size, perm, extra))
    # anisotropic scales, a width off 1, odd rfft_n and fewer bins than the default
    u, x = make(dtype, pen, (2,), seed=7)
    sc = tuple(0.5 + 0.25 * d for d in range(N))
    check(u, x, dims=(1,), keep=(N + 1,), rfft_dim=1, rfft_n=2 * size[0] - 1, scales=sc, width=0.7,
          what="scales")
    check(u, x, dims=(2,), keep=(1,), nbins=2, what="dropped")


@pytest.mark.parametrize("boff", [0, 1])
@pytest.mark.parametrize("dtype", CTYPES)
def test_realdot_at_equal_and_different_alignments(dtype, boff):
    pen = pencil((16, 6, 7), (2, 3, 1))
    u, x = make(dtype, pen, (2,), seed=1)
    v, y = make(dtype, pen, (2,), offset=boff, seed=2)
    for dims, keep in (((1, 3), (2,)), ((1,), ()), ((1, 2, 3), (4,)), ((2,), (1, 4)), ((3,), (1,))):
        for rd in (None, 1, 3):
            check(u, x, v, y, dims=dims, keep=keep, rfft_dim=rd, what=boff)
    a = pa.shell_spectrum(u, u, dims=(1, 3), keep=(2,), rfft_dim=1)
    b = pa.shell_spectrum(u, dims=(1, 3), keep=(2,), rfft_dim=1)
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


@pytest.mark.parametrize("dtype", CTYPES)
def test_every_dim_binned_nothing_kept_is_shell_spectrum(dtype):
    for size, perm in CASES[:4] + CASES[-1:]:
        pen = pencil(size, perm)
        u, _ = make(dtype, pen, (2,), seed=3)
        N = len(size)
        for kw in ({}, {"rfft_dim": 1}, {"nbins": 5, "width": 0.5}):
            a = pa.shell_spectrum(u, **kw)
            b = pa.shell_spectrum(u, dims=tuple(range(N, 0, -1)), keep=(), **kw)
            assert b.shape == a.shape and a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


@pytest.mark.parametrize("dtype", CTYPES)
def test_kept_sums_equal_the_summed_call(dtype):
    pen = pencil((24, 20, 18), (3, 2, 1))
    u, x = make(dtype, pen, (3,), seed=5)
    for dims, keep in (((1, 3), (2,)), ((1,), (2, 3)), ((1, 2, 3), (4,)), ((2, 3), (1,)),
                       ((3,), (1, 4))):
        got = pa.shell_spectrum(u, dims=dims, keep=keep, rfft_dim=1).double()
        summed = pa.shell_spectrum(u, dims=dims, rfft_dim=1).double()
        red = tuple(range(got.dim() - 1))
        tot = got.sum(dim=red) if red else got
        _, absum = RD.spectrum(x, 3, summed.numel(), dims, (), None, 1)
        tol = 2 * RD.depth(x.size, sms()) * 2.0 ** -53 * absum + \
            (np.abs(absum) * 2.0 ** -22 if dtype == torch.complex64 else 0)
        assert (np.abs(tot.cpu().numpy() - summed.cpu().numpy()) <= tol + 1e-300).all(), (dims, keep)


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
    for dims, keep in (((1, 3), (2,)), ((2, 3), (1,)), ((1,), ())):
        nb = RD.default_nbins((11, 6, 5), dims)
        nk = math.prod((11, 6, 5)[d - 1] for d in keep)
        for b, yy, m in ((None, None, _lib.PA_MAP_ABS2), (yb, yl, _lib.PA_MAP_DOT)):
            res = torch.empty(nk * nb, dtype=torch.float64, device="cuda")
            assert lib.pa_shell_spectrum_dims(
                pen._h, 0, None, None, _lib.PA_COMPLEXF64, m, C.c_void_p(raw.data_ptr() + 8),
                C.c_void_p(b.data_ptr()) if b is not None else None, 0, 0, None, 1.0, nb, len(dims),
                (C.c_int * len(dims))(*dims), len(keep), (C.c_int * max(1, len(keep)))(*keep),
                C.c_void_p(res.data_ptr()), stream_ptr()) == 0, lib.pa_last_error()
            exact, absum = RD.spectrum(xl, 3, nb, dims, keep, yy)
            got = res.cpu().numpy().reshape((nk, nb)).reshape(exact.shape)
            RD.check(got, exact, absum, n // nk, sms(), False, what=(dims, keep, m))


@pytest.mark.parametrize("dtype", CTYPES)
def test_offset_bases_and_nan_confined_to_its_value(dtype):
    pen = pencil((33, 9, 5), (3, 1, 2))
    for off in (1, 3):
        u, x = make(dtype, pen, (2,), offset=off, seed=off)
        check(u, x, dims=(1, 3), keep=(2,), rfft_dim=2, what=off)
        check(u, x, dims=(2,), keep=(1, 4), what=off)
    u, x = make(dtype, pen, seed=9)
    idx = (3, 4, 0)  # kept y = 4, wavenumbers (3, ., 0) over (x, z): |k_h| = 3
    x[idx] = np.nan
    logical_view(u, u.data)[idx] = complex(np.nan, 0.0)
    got = check(u, x, dims=(1, 3), keep=(2,), what="nan")
    g = as_logical(u, got, (2,))
    assert np.isnan(g).sum() == 1 and np.isnan(g[4, 3])


def test_empty_local_and_global_arrays():
    pen = pencil((0, 5, 4))
    u = pa.PencilArray.undef(torch.complex128, pen)
    r = pa.shell_spectrum(u, dims=(2, 3), keep=(1,))
    assert r.numel() == 0
    r = pa.shell_spectrum(u, dims=(2,), keep=(3,))
    assert r.shape[-1] == pa.spectrum_nbins(u, dims=(2,)) and bool((r == 0).all())
    r = pa.shell_spectrum(u, u, dims=(1,), nbins=7, rfft_dim=2)
    assert r.shape == (7,) and bool((r == 0).all())
    w = pa.PencilArray.undef(torch.complex64, pencil((6, 5, 4)), 0)
    r = pa.shell_spectrum(w, dims=(1, 3), keep=(2,))
    assert r.shape[-1] == pa.spectrum_nbins(w, dims=(1, 3)) and bool((r == 0).all())
    torch.cuda.synchronize()


def test_two_calls_bitwise_equal_and_one_launch_each():
    for size, perm in (((129, 256, 64), (3, 2, 1)), ((129, 256, 64), None)):
        pen = pencil(size, perm)
        for dtype in CTYPES:
            u, _ = make(dtype, pen, (2,))
            for kw in ({"dims": (1, 3), "keep": (2,), "rfft_dim": 1}, {"dims": (1,)},
                       {"dims": (2, 3), "keep": (1,)}, {"keep": (4,)},
                       {"dims": (1, 2), "keep": (3,), "nbins": 40, "width": 2.0}):
                a = pa.shell_spectrum(u, **kw)
                n0 = pa.launch_count()
                b = pa.shell_spectrum(u, **kw)
                assert pa.launch_count() - n0 == 1
                assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


def test_refused_call_launches_nothing_and_leaves_the_result_untouched():
    pen = pencil((16, 21, 41))
    u, _ = make(torch.complex128, pen)
    guard = torch.full((4096 * 8 * 21 + 64,), 0x5A, dtype=torch.uint8, device="cuda")
    res = C.c_void_p(guard.data_ptr() + 32)
    a = C.c_void_p(u.data_ptr())
    n0 = pa.launch_count()

    def call(dtype=_lib.PA_COMPLEXF64, m=_lib.PA_MAP_ABS2, b=None, rd=0, w=1.0, nb=10, dims=(1, 3),
             keep=(2,), r=res, comm=None):
        return lib.pa_shell_spectrum_dims(pen._h, 0, None, comm, dtype, m, a, b, rd, 0, None, w, nb,
                                          len(dims), (C.c_int * max(1, len(dims)))(*dims), len(keep),
                                          (C.c_int * max(1, len(keep)))(*keep), r, stream_ptr())
    for kw in ({"dtype": _lib.PA_FLOAT64}, {"m": _lib.PA_MAP_ABS}, {"b": a}, {"m": _lib.PA_MAP_DOT},
               {"dims": ()}, {"dims": (4,)}, {"keep": (3,)}, {"keep": (4,)}, {"rd": 4}, {"w": 0.0},
               {"nb": 0}, {"nb": 4097}, {"r": C.c_void_p(guard.data_ptr() + 33)}):
        assert call(**kw) == _lib.PA_EINVAL, kw
        assert lib.pa_last_error().decode().startswith("pa_shell_spectrum_dims:")
    h = C.c_void_p()
    assert lib.pa_comm_init_local(2, 0, C.byref(h)) == 0
    try:
        assert call(comm=h) == _lib.PA_EINCOMPAT
    finally:
        lib.pa_comm_destroy(h)
    # the partial area: two ranks splitting the kept dim, checked before the communicator
    big = pa.Pencil(pa.MPITopology(pa.Comm(0, 2), (2, 1)), (8, 512, 8), (2, 3))
    assert lib.pa_shell_spectrum_dims(big._h, 0, None, None, _lib.PA_COMPLEXF64, _lib.PA_MAP_ABS2, a,
                                      None, 0, 0, None, 1.0, 4096, 2, (C.c_int * 2)(1, 3), 1,
                                      (C.c_int * 1)(2), res, stream_ptr()) == _lib.PA_EINVAL
    assert "partial area" in lib.pa_last_error().decode()
    assert pa.launch_count() == n0
    torch.cuda.synchronize()
    assert bool((guard == 0x5A).all())


def test_stream_ordering_without_host_sync():
    pen = pencil((64, 32, 16))
    u = pa.PencilArray.undef(torch.complex128, pen)
    u.data.fill_(1.0)
    pa.shell_spectrum(u, dims=(1, 3), keep=(2,))  # warm-up
    nb = pa.spectrum_nbins(u, dims=(1, 3))
    count = np.bincount(RD.shells((64, 32, 16), (1, 3))[:, 0, :].reshape(-1).astype(np.int64),
                        minlength=nb)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        held = hold()
        u.data.fill_(2.0)          # produced behind the hold
        r = pa.shell_spectrum(u, dims=(1, 3), keep=(2,))
        e = pa.shell_spectrum(u, dims=(1,))
        assert not held.query()    # the calls did not wait for the device
    torch.cuda.synchronize()
    assert r.shape == (1, 32, 1, nb)
    assert np.array_equal(r.cpu().numpy()[0, :, 0, :], np.broadcast_to(4.0 * count, (32, nb)))
    cx = np.bincount(np.abs(np.fft.fftfreq(64, 1 / 64)).astype(np.int64), minlength=33)
    assert np.array_equal(e.cpu().numpy(), 4.0 * 32 * 16 * cx)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_horizontal_spectrum_through_rfft_and_a_fused_transpose(dtype):
    """E(k_h; y) of a real field of known modes: u = sum of cos(2 pi (a x / Lx + c z / Lz)) g(y),
    forward-transformed along x (rfft_) and z (a fused transpose + FFT)."""
    dims = (32, 12, 16)
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    ctype = torch.complex128 if dtype == torch.float64 else torch.complex64
    pxr = pa.Pencil(topo, dims, (2, 3))
    pxc = pa.Pencil(pxr, size_global=(dims[0] // 2 + 1,) + dims[1:])
    pzc = pa.Pencil(pxc, decomp_dims=(2, 1), permute=pa.Permutation(3, 2, 1))  # z contiguous
    X, Y, Z = np.meshgrid(*(np.arange(n) for n in dims), indexing="ij")
    modes = ((3, 4, 1.5), (5, 0, 0.5), (0, 2, 2.0))  # (a, c, amplitude); y profile 1 + y
    g = sum(A * np.cos(2 * np.pi * (a * X / dims[0] + c * Z / dims[2])) for a, c, A in modes) * (1 + Y)
    ur = pa.PencilArray.undef(dtype, pxr)
    logical_view(ur, ur.data).copy_(torch.from_numpy(g))
    uxc, uzc = pa.PencilArray.undef(ctype, pxc), pa.PencilArray.undef(ctype, pzc)
    pa.rfft_(uxc, ur)
    pa.transpose_(pa.Transposition(uzc, uxc), fft="forward")
    E = pa.shell_spectrum(uzc, dims=(1, 3), keep=(2,), rfft_dim=1, rfft_n=dims[0])
    E = as_logical(uzc, E, (2,))
    ntot = dims[0] * dims[2]
    want = np.zeros_like(E, dtype=np.float64)
    for a, c, A in modes:  # each cosine puts (A / 2)^2 ntot^2 into modes (a, c) and (-a, -c)
        b = int(math.floor(math.hypot(a, c) + 0.5))
        want[:, b] += 2 * (A / 2) ** 2 * ntot ** 2 * (1 + np.arange(dims[1])) ** 2
    eps = 2.0 ** -53 if dtype == torch.float64 else 2.0 ** -24
    tol = 64 * math.log2(ntot) * eps * want.max()
    assert np.abs(E - want).max() <= tol, (np.abs(E - want).max(), tol)


@pytest.mark.parametrize("nproc", [2, 3, 4, 8])
def test_ranks_sharing_the_gpu(nproc):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(29871 + nproc),
           os.path.join(HERE, "mp_spectrum_dims_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1")
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    assert f"MP_SPECTRUM_DIMS_OK world={nproc}" in out.stdout, out.stdout[-2000:]
