"""pa_shell_spectrum on the host (no GPU needed): every refusal in the order pa_b200.h states it
with its text, PA_ENOGPU for valid calls without a GPU, pa_shell_spectrum_nbins against the NumPy
reference (tests/spectrum_ref.py) over seeded geometries, the bin geometry of reduce_core.hpp bit
for bit against NumPy over every mode (tests/spectrum_host_check.cpp), and the Python mirror's
argument checks."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200 import _lib
from pencilarrays_b200._lib import lib, i64arr
import spectrum_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
F64, F32, C64, C32 = range(4)
ID, ABS, ABS2, DOT = range(4)
NO_GPU = lib.pa_device_count() == 0
BUF = (C.c_double * 64)()
P = C.cast(BUF, C.c_void_p)


def pencil(size, grid=None, perm=None):
    N = len(size)
    grid = grid or ((1,) if N == 2 else (1, 1))
    decomp = (2,) if len(grid) == 1 else (2, 3)
    kw = {"permute": pa.Permutation(*perm)} if perm else {}
    comm = pa.COMM_SELF if all(g == 1 for g in grid) else pa.Comm(0, int(np.prod(grid)))
    return pa.Pencil(pa.MPITopology(comm, grid), size, decomp, **kw)


def call(pen, dtype=C64, m=ABS2, a=P, b=None, extra=(), rd=0, rn=0, scales=None, width=1.0,
         nbins=10, result=P):
    sc = (C.c_double * len(scales))(*scales) if scales is not None else None
    return lib.pa_shell_spectrum(pen._h if pen else None, len(extra),
                                 i64arr(extra) if extra else None, None, dtype, m, a, b, rd, rn, sc,
                                 width, nbins, result, None)


def err():
    return lib.pa_last_error().decode()


def test_export_and_signature():
    for f in ("pa_shell_spectrum", "pa_shell_spectrum_nbins"):
        assert hasattr(lib, f) and f in _lib.SIGNATURES


def test_refusals_in_order():
    pen = pencil((8, 6, 5))
    odd = C.c_void_p(BUF and C.addressof(BUF) + 4)
    # each case also breaks every later check, so the earliest refusal must win
    cases = [
        (dict(pen=None, dtype=F64, b=P, extra=(-1,), rd=9, width=0.0, nbins=0, a=None,
              result=None), "null pencil"),
        (dict(dtype=F64, b=P, extra=(-1,), rd=9, width=0.0, nbins=0, a=None), "dtype 0, map 2"),
        (dict(m=ABS, b=P, extra=(-1,)), "map 1"),
        (dict(b=P, extra=(-1,), rd=9), "`b` goes with PA_MAP_DOT only"),
        (dict(m=DOT, extra=(-1,), rd=9), "`b` is missing"),
        (dict(extra=(-1,), rd=9, width=0.0), "negative extra dim"),
        (dict(rd=4, rn=3, width=0.0), "rfft_dim 4 out of range 0..3"),
        (dict(rd=-1), "rfft_dim -1 out of range"),
        (dict(rd=1, rn=13, width=0.0), "rfft_n 13 does not fit"),
        (dict(rd=1, rn=-2), "rfft_n -2"),
        (dict(rn=4, width=0.0), "without an r2c dim"),
        (dict(scales=(1.0, 0.0, 1.0), width=0.0, nbins=0), "scale 0 of dim 2"),
        (dict(scales=(1.0, 1.0, float("inf"))), "scale inf of dim 3"),
        (dict(width=float("nan"), nbins=0), "width nan"),
        (dict(width=-1.0), "width -1"),
        (dict(nbins=0, a=None), "nbins 0 out of range 1..4096"),
        (dict(nbins=4097, a=None), "nbins 4097"),
        (dict(a=None, result=None), "null array pointer"),
        (dict(m=DOT, b=odd, result=None), "aligned to 8 bytes"),
        (dict(result=None), "`result`"),
        (dict(result=odd), "`result`"),
    ]
    for kw, text in cases:
        pen_ = kw.pop("pen", pen)
        assert call(pen_, **kw) == _lib.PA_EINVAL, (kw, err())
        assert err().startswith("pa_shell_spectrum:") and text in err(), (kw, err())
    # ComplexF32: 4-byte arrays and results are fine, 2-byte ones are not
    two = C.c_void_p(C.addressof(BUF) + 2)
    assert call(pen, dtype=C32, a=two) == _lib.PA_EINVAL and "aligned to 4" in err()
    assert call(pen, dtype=C32, result=two) == _lib.PA_EINVAL and "`result`" in err()
    # rank count: a 1 x 2 grid without a communicator, after every argument check
    two_ranks = pencil((8, 6, 5), grid=(1, 2))
    assert call(two_ranks, nbins=0) == _lib.PA_EINVAL
    assert call(two_ranks) == _lib.PA_EINCOMPAT and "needs a communicator" in err()


@pytest.mark.skipif(not NO_GPU, reason="on a GPU machine valid calls run (tests/test_gpu_spectrum.py)")
def test_valid_calls_need_a_gpu():
    pen = pencil((8, 6, 5), perm=(3, 1, 2))
    for kw in (dict(), dict(dtype=C32), dict(m=DOT, b=P), dict(rd=1), dict(rd=1, rn=15),
               dict(rd=3, scales=(0.5, 2.0, 1.0), width=0.3, nbins=4096), dict(extra=(3, 2)),
               dict(nbins=1)):
        assert call(pen, **kw) == _lib.PA_ENOGPU, kw
    # an empty local array may have NULL pointers
    empty = pencil((0, 6, 5))
    assert call(empty, a=None) == _lib.PA_ENOGPU
    assert call(empty, m=DOT, a=None, b=None) == _lib.PA_ENOGPU


def geometries():
    """The reference cases and seeded random geometries: odd and even extents, every rfft_dim,
    odd rfft_n, anisotropic scales and widths that put |k| near bin boundaries."""
    out = [((8, 9, 10), None, None, None, 1.0), ((8, 9, 10), 1, None, None, 1.0),
           ((257, 512, 512), 1, None, None, 1.0), ((7, 6), 2, 11, None, 1.0),
           ((5, 4, 3, 6), 3, None, (0.5, 1.5, 2.0, 0.25), 0.5), ((1, 1, 1), None, None, None, 1.0),
           ((0, 4, 4), None, None, None, 1.0), ((16, 16, 16), None, None, (2 * np.pi / 3,) * 3, 1.0)]
    rng = np.random.default_rng(2024)
    for _ in range(40):
        N = int(rng.integers(2, 5))
        size = tuple(int(x) for x in rng.integers(1, 13 if N < 4 else 7, N))
        rd = int(rng.integers(0, N + 1)) or None
        rn = None
        if rd and rng.random() < 0.5:
            rn = 2 * size[rd - 1] - 1  # odd real length
        scales = tuple(float(x) for x in rng.choice([1.0, 0.5, 2 * np.pi / 7, 1 / 3, 3.7], N))
        width = float(rng.choice([1.0, 0.5, 1 / 3, 0.1, 2 * np.pi / 7, 0.7]))
        out.append((size, rd, rn, scales, width))
    return out


def test_nbins_against_the_reference():
    for size, rd, rn, scales, width in geometries():
        pen = pencil(size)
        got = C.c_int()
        sc = (C.c_double * len(size))(*scales) if scales else None
        assert lib.pa_shell_spectrum_nbins(pen._h, rd or 0, rn or 0, sc, width, C.byref(got)) == 0, err()
        assert got.value == R.default_nbins(size, rd, scales, width), (size, rd, scales, width)
    # the query refuses what the spectrum refuses, in the same words
    pen = pencil((8, 9, 10))
    assert lib.pa_shell_spectrum_nbins(pen._h, 1, 3, None, 1.0, None) == _lib.PA_EINVAL
    assert err().startswith("pa_shell_spectrum:") and "rfft_n 3" in err()
    assert lib.pa_shell_spectrum_nbins(None, 0, 0, None, 1.0, None) == _lib.PA_EINVAL


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = os.path.join(str(tmp_path_factory.mktemp("spectrum")), "spectrum_host_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", out,
                    os.path.join(HERE, "spectrum_host_check.cpp")], check=True)
    return out


def test_bins_bit_exact_against_numpy(exe):
    for size, rd, rn, scales, width in geometries():
        if np.prod(size) > 1 << 16:
            continue
        N = len(size)
        nbins = R.default_nbins(size, rd, scales, width)
        for nb in (nbins, max(1, nbins // 2)):
            args = [str(N)] + [str(n) for n in size] + [str(rd or 0), str(rn if rn is not None else
                    R.default_rfft_n(size, rd)), repr(width), str(nb)] + \
                   [repr(s) for s in (scales or (1.0,) * N)]
            out = subprocess.run([exe] + args, capture_output=True, check=True).stdout
            v = np.frombuffer(out, np.int32)
            total = int(np.prod(size))
            bins, wts = v[:total], v[total:]
            sh = R.shells(size, rd, scales, width).reshape(-1, order="F")
            want = np.where(sh < nb, sh, -1).astype(np.int32)
            assert np.array_equal(bins, want), (size, rd, scales, width, nb)
            w = R.mode_weights(size, rd, rn).reshape(-1, order="F")
            assert np.array_equal(wts, w.astype(np.int32)), (size, rd, rn)
            if nb == nbins and total:
                assert bins.max() == nbins - 1  # the default covers every mode, no more


def test_python_argument_checks():
    pen = pencil((8, 6, 5))
    u = pa.PencilArray(pen, torch.empty((5, 6, 8), dtype=torch.complex128))
    r = pa.PencilArray(pen, torch.empty((5, 6, 8), dtype=torch.float64))
    w = pa.PencilArray(pen, torch.empty((5, 6, 8), dtype=torch.complex64))
    other = pa.PencilArray(pencil((8, 6, 5)), torch.empty((5, 6, 8), dtype=torch.complex128))
    for args, kw in (((r,), {}), ((u, w), {}), ((u, other), {}), ((u, r), {}),
                     ((u,), {"rfft_dim": 1.0}), ((u,), {"rfft_dim": True}), ((u,), {"rfft_n": 3.5}),
                     ((u,), {"scales": (1.0, 2.0)}), ((u,), {"scales": "abc"}),
                     ((u,), {"width": "x"}), ((u,), {"nbins": 3.0}), ((u,), {"rfft_dim": 4}),
                     ((u,), {"nbins": 0}), ((u,), {"width": 0.0}), ((u,), {"rfft_n": 5})):
        with pytest.raises(pa.ArgumentError):
            pa.shell_spectrum(*args, **kw)
    assert pa.spectrum_nbins(u) == R.default_nbins((8, 6, 5))
    assert pa.spectrum_nbins(u, rfft_dim=1, scales=(1, 2, 3), width=0.5) == \
        R.default_nbins((8, 6, 5), 1, (1.0, 2.0, 3.0), 0.5)
