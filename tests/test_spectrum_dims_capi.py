"""pa_shell_spectrum_dims on the host (no GPU needed): the exports and signatures, every refusal in
the order pa_b200.h states it with its text, PA_ENOGPU for valid calls without a GPU,
pa_shell_spectrum_dims_nbins against the NumPy reference (tests/spectrum_dims_ref.py) for every bin
subset, the bins of every mode bit for bit against NumPy through reduce_core.hpp
(tests/spectrum_dims_host_check.cpp), and the Python mirror's argument checks."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200 import _lib
from pencilarrays_b200._lib import lib, i64arr
import spectrum_ref as R
import spectrum_dims_ref as RD

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


def ints(xs):
    return (C.c_int * max(1, len(xs)))(*xs) if xs is not None else None


def call(pen, dtype=C64, m=ABS2, a=P, b=None, extra=(), rd=0, rn=0, scales=None, width=1.0,
         nbins=10, dims=(1, 3), keep=(2,), n_bin=None, n_keep=None, result=P):
    sc = (C.c_double * len(scales))(*scales) if scales is not None else None
    return lib.pa_shell_spectrum_dims(
        pen._h if pen else None, len(extra), i64arr(extra) if extra else None, None, dtype, m, a, b,
        rd, rn, sc, width, nbins, len(dims) if n_bin is None else n_bin, ints(dims),
        len(keep or ()) if n_keep is None else n_keep, ints(keep), result, None)


def err():
    return lib.pa_last_error().decode()


def test_exports_and_signatures():
    for f in ("pa_shell_spectrum_dims", "pa_shell_spectrum_dims_nbins"):
        assert hasattr(lib, f) and f in _lib.SIGNATURES
    assert len(_lib.SIGNATURES["pa_shell_spectrum_dims"][1]) == 19
    assert len(_lib.SIGNATURES["pa_shell_spectrum_dims_nbins"][1]) == 8
    hdr = open(os.path.join(HERE, "..", "include", "pa_b200.h")).read()
    for f in ("pa_shell_spectrum_dims(", "pa_shell_spectrum_dims_nbins("):
        assert f in hdr


def test_refusals_in_order():
    pen = pencil((8, 6, 5))
    odd = C.c_void_p(C.addressof(BUF) + 4)
    # each case also breaks every later check, so the earliest refusal must win
    cases = [
        (dict(pen=None, dtype=F64, b=P, extra=(-1,), dims=(), rd=9, width=0.0, nbins=0, a=None,
              result=None), "null pencil"),
        (dict(dtype=F64, b=P, extra=(-1,), dims=(), rd=9, width=0.0, nbins=0, a=None), "dtype 0, map 2"),
        (dict(m=ABS, b=P, extra=(-1,)), "map 1"),
        (dict(b=P, extra=(-1,), dims=()), "`b` goes with PA_MAP_DOT only"),
        (dict(m=DOT, extra=(-1,), dims=()), "`b` is missing"),
        (dict(extra=(-1,), dims=(), rd=9, width=0.0), "negative extra dim"),
        (dict(extra=(1, 2, 3, 4, 5, 6), dims=()), "extra dims on a 3-d pencil"),
        (dict(dims=(), keep=(9,), rd=9), "at least one bin dim"),
        (dict(dims=None, n_bin=2, keep=(9,)), "at least one bin dim"),
        (dict(dims=(4,), keep=(9,), rd=9), "bin dim 4 out of range 1..3"),
        (dict(dims=(0,), keep=(9,)), "bin dim 0 out of range"),
        (dict(dims=(1, 1), keep=(9,)), "bin dim 1 given twice"),
        (dict(keep=None, n_keep=1, rd=9), "1 kept dims and no `keep_dims`"),
        (dict(keep=(), n_keep=-1, rd=9), "-1 kept dims"),
        (dict(keep=(4,), rd=9, width=0.0), "kept dim 4 out of range 1..3 (3 spatial dims, then 0 extra)"),
        (dict(extra=(2,), keep=(5,), rd=9), "kept dim 5 out of range 1..4"),
        (dict(keep=(2, 2), rd=9), "kept dim 2 given twice"),
        (dict(keep=(3,), rd=9, nbins=0), "dim 3 is both a bin dim and a kept dim"),
        (dict(rd=4, rn=3, width=0.0), "rfft_dim 4 out of range 0..3"),
        (dict(rd=1, rn=13, width=0.0), "rfft_n 13 does not fit"),
        (dict(rn=4, width=0.0), "without an r2c dim"),
        (dict(scales=(1.0, 0.0, 1.0), width=0.0, nbins=0), "scale 0 of dim 2"),
        (dict(width=float("nan"), nbins=0), "width nan"),
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
        assert err().startswith("pa_shell_spectrum_dims:") and text in err(), (kw, err())
    two = C.c_void_p(C.addressof(BUF) + 2)
    assert call(pen, dtype=C32, a=two) == _lib.PA_EINVAL and "aligned to 4" in err()
    assert call(pen, dtype=C32, result=two) == _lib.PA_EINVAL and "`result`" in err()
    # the partial area, from the global geometry: 2 ranks splitting y, y kept (512 / 2 outputs per
    # rank x 4096 bins > 524288), refused before the rank-count check; 2048 bins fit
    big = pencil((8, 512, 8), grid=(2, 1))
    assert call(big, nbins=4096) == _lib.PA_EINVAL and "partial area (524288" in err(), err()
    assert call(big, nbins=2048) == _lib.PA_EINCOMPAT and "needs a communicator" in err()
    # rank count: a 1 x 2 grid without a communicator, after every argument check
    two_ranks = pencil((8, 6, 5), grid=(1, 2))
    assert call(two_ranks, nbins=0) == _lib.PA_EINVAL
    assert call(two_ranks) == _lib.PA_EINCOMPAT and "needs a communicator" in err()


@pytest.mark.skipif(not NO_GPU, reason="on a GPU machine valid calls run (tests/test_gpu_spectrum_dims.py)")
def test_valid_calls_need_a_gpu():
    pen = pencil((8, 6, 5), perm=(3, 1, 2))
    for kw in (dict(), dict(dtype=C32), dict(m=DOT, b=P), dict(rd=2), dict(dims=(1,), keep=()),
               dict(dims=(2, 1, 3), keep=()), dict(dims=(3,), keep=(1, 2)),
               dict(extra=(3,), keep=(4, 2)), dict(extra=(3,), dims=(1, 2, 3), keep=(4,)),
               dict(rd=1, rn=15, scales=(0.5, 2.0, 1.0), width=0.3, nbins=4096)):
        assert call(pen, **kw) == _lib.PA_ENOGPU, (kw, err())
    # an empty local array may have NULL pointers, an empty local result a NULL result
    empty = pencil((0, 6, 5))
    assert call(empty, a=None) == _lib.PA_ENOGPU
    assert call(empty, m=DOT, a=None, b=None) == _lib.PA_ENOGPU
    assert call(empty, a=None, dims=(2,), keep=(1,), result=None) == _lib.PA_ENOGPU


def subsets(N):
    for r in range(1, N + 1):
        yield from itertools.combinations(range(1, N + 1), r)


def test_nbins_against_the_reference():
    for size, rd, rn, scales, width in _geometries():
        pen = pencil(size)
        sc = (C.c_double * len(size))(*scales) if scales else None
        for dims in subsets(len(size)):
            got = C.c_int()
            assert lib.pa_shell_spectrum_dims_nbins(pen._h, rd or 0, rn or 0, sc, width, len(dims),
                                                    ints(dims), C.byref(got)) == 0, err()
            assert got.value == RD.default_nbins(size, dims, rd, scales, width), (size, dims, rd)
        # every dim binned is pa_shell_spectrum_nbins
        full = C.c_int()
        assert lib.pa_shell_spectrum_nbins(pen._h, rd or 0, rn or 0, sc, width, C.byref(full)) == 0
        assert full.value == RD.default_nbins(size, range(1, len(size) + 1), rd, scales, width)
    pen = pencil((8, 9, 10))
    for args, text in (((1, 3, None, 1.0, 1, ints((1,))), "rfft_n 3"),
                       ((0, 0, None, 1.0, 0, ints(())), "at least one bin dim"),
                       ((0, 0, None, 1.0, 1, ints((4,))), "bin dim 4 out of range"),
                       ((0, 0, None, 0.0, 1, ints((1,))), "width 0")):
        assert lib.pa_shell_spectrum_dims_nbins(pen._h, *args, None) == _lib.PA_EINVAL
        assert err().startswith("pa_shell_spectrum_dims:") and text in err(), err()
    assert lib.pa_shell_spectrum_dims_nbins(None, 0, 0, None, 1.0, 1, ints((1,)), None) == _lib.PA_EINVAL


def _geometries():
    """Reference cases and seeded random geometries: odd and even extents, every rfft_dim, odd
    rfft_n, anisotropic scales and widths that put |k| near bin boundaries."""
    out = [((8, 9, 10), None, None, None, 1.0), ((8, 9, 10), 1, None, None, 1.0),
           ((257, 512, 512), 1, None, None, 1.0), ((7, 6), 2, 11, None, 1.0),
           ((5, 4, 3, 6), 3, None, (0.5, 1.5, 2.0, 0.25), 0.5), ((1, 1, 1), None, None, None, 1.0),
           ((0, 4, 4), None, None, None, 1.0), ((16, 16, 16), None, None, (2 * np.pi / 3,) * 3, 1.0)]
    rng = np.random.default_rng(2025)
    for _ in range(30):
        N = int(rng.integers(2, 5))
        size = tuple(int(x) for x in rng.integers(1, 13 if N < 4 else 7, N))
        rd = int(rng.integers(0, N + 1)) or None
        rn = 2 * size[rd - 1] - 1 if rd and rng.random() < 0.5 else None  # odd real length
        scales = tuple(float(x) for x in rng.choice([1.0, 0.5, 2 * np.pi / 7, 1 / 3, 3.7], N))
        width = float(rng.choice([1.0, 0.5, 1 / 3, 0.1, 2 * np.pi / 7, 0.7]))
        out.append((size, rd, rn, scales, width))
    return out


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = os.path.join(str(tmp_path_factory.mktemp("spectrum_dims")), "spectrum_dims_host_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", out,
                    os.path.join(HERE, "spectrum_dims_host_check.cpp")], check=True)
    return out


def test_bins_bit_exact_against_numpy(exe):
    for size, rd, rn, scales, width in _geometries():
        if np.prod(size) > 1 << 14:
            continue
        N = len(size)
        for dims in subsets(N):
            nbins = RD.default_nbins(size, dims, rd, scales, width)
            mask = sum(1 << (d - 1) for d in dims)
            for nb in (nbins, max(1, nbins // 2)):
                args = [str(N)] + [str(n) for n in size] + [
                    str(rd or 0), str(rn if rn is not None else R.default_rfft_n(size, rd)),
                    repr(width), str(nb), str(mask)] + [repr(s) for s in (scales or (1.0,) * N)]
                v = np.frombuffer(subprocess.run([exe] + args, capture_output=True,
                                                 check=True).stdout, np.int32)
                total = int(np.prod(size))
                bins, wts = v[:total], v[total:]
                sh = RD.shells(size, dims, rd, scales, width).reshape(-1, order="F")
                want = np.where(sh < nb, sh, -1).astype(np.int32)
                assert np.array_equal(bins, want), (size, dims, rd, scales, width, nb)
                w = R.mode_weights(size, rd, rn).reshape(-1, order="F")
                assert np.array_equal(wts, w.astype(np.int32)), (size, rd, rn)
                if nb == nbins and total:
                    assert bins.max() == nbins - 1  # the default covers every mode, no more


def test_python_argument_checks():
    pen = pencil((8, 6, 5))
    u = pa.PencilArray(pen, torch.empty((5, 6, 8), dtype=torch.complex128))
    u3 = pa.PencilArray(pen, torch.empty((3, 5, 6, 8), dtype=torch.complex128), (3,))
    for args, kw in (((u,), {"dims": ()}), ((u,), {"dims": (4,)}), ((u,), {"dims": (1, 1)}),
                     ((u,), {"dims": 1.0}), ((u,), {"dims": True}), ((u,), {"dims": "ab"}),
                     ((u,), {"keep": (4,)}), ((u,), {"keep": (2, 2)}), ((u,), {"keep": 0}),
                     ((u,), {"dims": (1, 2), "keep": (2,)}), ((u,), {"keep": (1, 2, 3)}),
                     ((u3,), {"dims": (4,)}), ((u3,), {"keep": (5,)}), ((u,), {"dims": (1, 3), "keep": (2,), "nbins": 0}),
                     ((u,), {"dims": (1,), "rfft_dim": 4}), ((u,), {"keep": None, "dims": (1,), "width": 0.0})):
        with pytest.raises(pa.ArgumentError):
            pa.shell_spectrum(*args, **kw)
    with pytest.raises(pa.ArgumentError, match="pa_shell_spectrum_dims: nbins"):
        pa.shell_spectrum(u, dims=(1, 3), keep=(2,), nbins=5000)
    with pytest.raises(pa.ArgumentError):
        pa.spectrum_nbins(u, dims=(4,))
    with pytest.raises(pa.ArgumentError):
        pa.spectrum_nbins(u, dims=())
    for dims in subsets(3):
        assert pa.spectrum_nbins(u, dims=dims) == RD.default_nbins((8, 6, 5), dims)
    assert pa.spectrum_nbins(u, dims=(1, 3), rfft_dim=1, scales=(1, 2, 3), width=0.5) == \
        RD.default_nbins((8, 6, 5), (1, 3), 1, (1.0, 2.0, 3.0), 0.5)
    assert pa.spectrum_nbins(u, dims=(1, 2, 3)) == pa.spectrum_nbins(u)
    assert pa.spectrum_nbins(u, dims=2) == RD.default_nbins((8, 6, 5), (2,))
