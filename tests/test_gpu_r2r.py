"""Real-to-real line transforms (`r2r_`, `pa_r2r`: DCT-II/III, DST-II/III) on the GPU.

* accuracy per line for each kind, every N and both precisions, against an extended-precision
  reference built here from `fft_ld`: max within eps log2(N) (eps32 for float32), RMS within 3x
  scipy.fft's on the same data in the same precision;
* known answers (constants, impulses, single-bin cosines / sines) and the round trips
  REDFT01(REDFT10(x)) = RODFT01(RODFT10(x)) = 2N x;
* byte-for-byte: in place = out of place, a batch = the same lines one launch at a time,
  permuted pencils = the unpermuted result, extra dims up to PA_MAX_DIMS;
* canaries around dst through the C ABI, src untouched, refusals and empty arrays launch nothing,
  a caller's held side stream;
* the mixed 3-d transform this exists for (DCT-II along x, rfft along y, fft along z) on one rank
  and on 2 and 4 processes sharing the GPU (tests/mp_r2r_worker.py)."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.fft as sf
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200 import _lib
from pencilarrays_b200._lib import lib

from fft_ref import CLD, LD, PI_LD, fft_ld, line_errors, scaled_lines
from gpu_util import hold, stream_ptr

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
NS = [1 << k for k in range(4, 12)]  # 16 ... 2048
KINDS = ["REDFT10", "REDFT01", "RODFT10", "RODFT01"]
TDT = {"d": torch.float64, "f": torch.float32}
NDT = {"d": np.float64, "f": np.float32}
EPS = {"d": float(np.finfo(np.float64).eps), "f": float(np.finfo(np.float32).eps)}


# ---- extended-precision references (long double, through fft_ld) ----
def _w(N, k, sign):
    a = PI_LD * np.asarray(k, dtype=LD) / LD(2 * N)
    return (np.cos(a) + LD(sign) * 1j * np.sin(a)).astype(CLD)


def redft10_ld(x):
    """DCT-II: Re(exp(-i pi k / 2N) FFT_2N([x, reversed x])[k])."""
    x = np.asarray(x).astype(LD)
    N = x.shape[-1]
    Y = fft_ld(np.concatenate((x, x[..., ::-1]), axis=-1), -1)[..., :N]
    return (_w(N, np.arange(N), -1) * Y).real


def redft01_ld(X):
    """DCT-III: Re(FFT^+_2N(a))[n], a[k] = c_k X[k] exp(i pi k / 2N) (c_0 = 1, else 2), a = 0 past N."""
    X = np.asarray(X).astype(LD)
    N = X.shape[-1]
    c = np.full(N, LD(2))
    c[0] = LD(1)
    a = np.concatenate((c * X * _w(N, np.arange(N), 1), np.zeros(X.shape, dtype=CLD)), axis=-1)
    return fft_ld(a, 1)[..., :N].real


def rodft10_ld(x):
    """DST-II(x)[k] = DCT-II((-1)^n x[n])[N-1-k]."""
    x = np.asarray(x)
    s = np.where(np.arange(x.shape[-1]) % 2 == 0, 1, -1)
    return redft10_ld(x * s)[..., ::-1]


def rodft01_ld(X):
    """DST-III(X)[n] = (-1)^n DCT-III(X reversed)[n]."""
    X = np.asarray(X)
    s = np.where(np.arange(X.shape[-1]) % 2 == 0, 1, -1)
    return redft01_ld(X[..., ::-1]) * s


REF = {"REDFT10": redft10_ld, "REDFT01": redft01_ld, "RODFT10": rodft10_ld, "RODFT01": rodft01_ld}


def scipy_r2r(x, kind):
    fn = sf.dct if kind.startswith("RE") else sf.dst
    return fn(x, type=2 if kind.endswith("10") else 3, axis=-1)


def line_pencil(dims, perm=None, decomp=(2, 3), topo=None):
    topo = topo or pa.MPITopology(pa.COMM_SELF, (1, 1))
    return pa.Pencil(topo, dims, decomp, permute=pa.Permutation(*perm) if perm else None)


def lines_array(x, prec):
    """A PencilArray holding the rows of x (nlines, N) as its lines."""
    nl, N = x.shape
    u = pa.PencilArray.undef(TDT[prec], line_pencil((N, nl, 1)))
    u.data.copy_(torch.from_numpy(np.ascontiguousarray(x, dtype=NDT[prec]).reshape(1, nl, N)))
    return u


def run_lines(x, prec, kind):
    u = lines_array(x, prec)
    out = pa.PencilArray.undef(TDT[prec], u.pencil)
    n0 = pa.launch_count()
    assert pa.r2r_(out, u, kind) is out
    torch.cuda.synchronize()
    assert pa.launch_count() - n0 == 1
    return out.data.cpu().numpy().reshape(x.shape)


def tol(N, ref, prec):
    return 8 * EPS[prec] * np.log2(N) * np.abs(ref).max()


# ---------------------------------------------------------------------------------- accuracy
@pytest.mark.parametrize("prec", ["d", "f"])
@pytest.mark.parametrize("N", NS)
def test_accuracy_per_line_against_extended_precision(N, prec):
    x = scaled_lines(np.random.default_rng(700 + N), 64, N, complex_=False).astype(NDT[prec])
    for kind in KINDS:
        got = run_lines(x, prec, kind)
        ref = REF[kind](x)
        mx, rms = line_errors(got, ref)
        _, rms_scipy = line_errors(scipy_r2r(x, kind), ref)
        assert mx <= EPS[prec] * np.log2(N), (kind, N, prec, mx / EPS[prec])
        assert rms <= 3 * rms_scipy, (kind, N, prec, rms / EPS[prec], rms_scipy / EPS[prec])


def test_reference_agrees_with_scipy():
    """The long-double references are scipy's transforms, to double precision."""
    x = np.random.default_rng(3).standard_normal((4, 64))
    for kind in KINDS:
        ref = np.asarray(REF[kind](x), dtype=np.float64)
        assert np.abs(ref - scipy_r2r(x, kind)).max() <= 64 * EPS["d"] * np.abs(ref).max(), kind


# ----------------------------------------------------------------------------- known answers
@pytest.mark.parametrize("prec", ["d", "f"])
@pytest.mark.parametrize("N", [16, 128, 2048])
def test_known_answers(N, prec):
    n = np.arange(N)
    ks = [0, 1, N // 4, N // 2, N - 2, N - 1]

    def cos(j, m):  # cos(pi j m / 2N), the integer product reduced mod 4N first: exact arguments
        return np.cos(np.pi * ((j * m) % (4 * N)) / (2 * N))

    def sin(j, m):
        return np.sin(np.pi * ((j * m) % (4 * N)) / (2 * N))

    # DCT-II: constants and cos(pi (2n+1) k0 / 2N) land in bin k0 (2N at k0 = 0, N otherwise)
    x = np.stack([np.ones(N)] + [cos(2 * n + 1, k0) for k0 in ks])
    want = np.zeros_like(x)
    want[0, 0] = 2 * N
    for i, k0 in enumerate(ks):
        want[i + 1, k0] = 2 * N if k0 == 0 else N
    got = run_lines(x, prec, "REDFT10")
    assert np.abs(got - want).max() <= tol(N, want, prec)
    # DST-II: sin(pi (2n+1)(k0+1) / 2N) lands in bin k0 (2N at k0 = N-1, where it is (-1)^n)
    x = np.stack([sin(2 * n + 1, k0 + 1) for k0 in ks])
    want = np.zeros_like(x)
    for i, k0 in enumerate(ks):
        want[i, k0] = 2 * N if k0 == N - 1 else N
    got = run_lines(x, prec, "RODFT10")
    assert np.abs(got - want).max() <= tol(N, want, prec)
    # DCT-III / DST-III of impulses: the basis functions
    X = np.zeros((len(ks), N))
    for i, k0 in enumerate(ks):
        X[i, k0] = 1
    want_c = np.stack([np.ones(N) if k0 == 0 else 2 * cos(2 * n + 1, k0) for k0 in ks])
    want_s = np.stack([(-1.0) ** n if k0 == N - 1 else 2 * sin(2 * n + 1, k0 + 1) for k0 in ks])
    assert np.abs(run_lines(X, prec, "REDFT01") - want_c).max() <= tol(N, want_c, prec)
    assert np.abs(run_lines(X, prec, "RODFT01") - want_s).max() <= tol(N, want_s, prec)


@pytest.mark.parametrize("prec", ["d", "f"])
@pytest.mark.parametrize("N", NS)
def test_round_trips_are_2N_times_the_input(N, prec):
    x = np.random.default_rng(N).standard_normal((24, N)).astype(NDT[prec])
    u = lines_array(x, prec)
    y = pa.PencilArray.undef(TDT[prec], u.pencil)
    for fwd, bwd in (("REDFT10", "REDFT01"), ("RODFT10", "RODFT01")):
        pa.r2r_(y, u, fwd)
        pa.r2r_(y, y, bwd)
        torch.cuda.synchronize()
        back = y.data.cpu().numpy().reshape(x.shape).astype(np.float64) / (2 * N)
        assert np.abs(back - x).max() <= tol(N, x, prec), (fwd, N, prec)


# ------------------------------------------------------------------------------ byte for byte
def raw(t):
    return t.view(torch.uint8)


@pytest.mark.parametrize("prec", ["d", "f"])
@pytest.mark.parametrize("N", NS)
def test_in_place_equals_out_of_place(N, prec):
    p = line_pencil((N, 37, 3))
    u = pa.PencilArray.undef(TDT[prec], p)
    u.data.normal_()
    before = u.data.clone()
    for kind in KINDS:
        out = pa.PencilArray.undef(TDT[prec], p)
        pa.r2r_(out, u, kind)
        inp = pa.PencilArray.undef(TDT[prec], p)
        inp.data.copy_(u.data)
        n0 = pa.launch_count()
        assert pa.r2r_(inp, inp, kind) is inp
        torch.cuda.synchronize()
        assert pa.launch_count() - n0 == 1
        assert torch.equal(raw(u.data), raw(before)), kind           # src untouched out of place
        assert torch.equal(raw(inp.data), raw(out.data)), (kind, N, prec)


@pytest.mark.parametrize("prec", ["d", "f"])
@pytest.mark.parametrize("N", [16, 512, 2048])
def test_batch_equals_one_line_per_launch(N, prec):
    nl = 21  # not a multiple of the lines per CTA
    x = scaled_lines(np.random.default_rng(N + 1), nl, N, complex_=False).astype(NDT[prec])
    one = line_pencil((N, 1, 1))
    for kind in KINDS:
        batch = run_lines(x, prec, kind)
        for i in range(nl):
            a = pa.PencilArray.undef(TDT[prec], one)
            a.data.copy_(torch.from_numpy(x[i].reshape(1, 1, N)))
            b = pa.PencilArray.undef(TDT[prec], one)
            pa.r2r_(b, a, kind)
            torch.cuda.synchronize()
            assert b.data.cpu().numpy().reshape(N).tobytes() == batch[i].tobytes(), (kind, i)


@pytest.mark.parametrize("prec", ["d", "f"])
@pytest.mark.parametrize("dims,perm,decomp", [((6, 32, 5), (2, 1, 3), (1, 3)),
                                              ((5, 3, 64), (3, 1, 2), (1, 2)),
                                              ((7, 256, 3), (2, 3, 1), (1, 3))])
def test_permuted_pencils_agree_with_the_unpermuted_result(dims, perm, decomp, prec):
    """Transform axis = perm[1] = logical dim 2 or 3: the logical result equals the unpermuted
    pencil's result with the axes moved, byte for byte."""
    ax = perm[0] - 1
    N = dims[ax]
    pp = line_pencil(dims, perm, decomp)
    u = pa.PencilArray.undef(TDT[prec], pp)
    u.data.normal_()
    G = u.logical().cpu().numpy().copy()              # logical order
    Gx = np.ascontiguousarray(np.moveaxis(G, ax, 0))  # the axis first
    qx = line_pencil(Gx.shape)
    ux = pa.PencilArray.undef(TDT[prec], qx)
    ux.logical().copy_(torch.from_numpy(Gx))
    for kind in KINDS:
        out = pa.PencilArray.undef(TDT[prec], pp)
        outx = pa.PencilArray.undef(TDT[prec], qx)
        pa.r2r_(out, u, kind)
        pa.r2r_(outx, ux, kind)
        torch.cuda.synchronize()
        got = np.moveaxis(out.logical().cpu().numpy(), ax, 0)
        want = outx.logical().cpu().numpy()
        assert np.ascontiguousarray(got).tobytes() == np.ascontiguousarray(want).tobytes(), kind
        ref = np.moveaxis(scipy_r2r(np.moveaxis(G.astype(np.float64), ax, -1), kind), -1, ax)
        assert np.abs(out.logical().cpu().numpy() - ref).max() <= tol(N, ref, prec)


@pytest.mark.parametrize("prec", ["d", "f"])
def test_extra_dims_up_to_pa_max_dims(prec):
    N = 64
    p = line_pencil((N, 3, 2))
    extra = (2, 1, 3, 2, 2)  # 3 + 5 = PA_MAX_DIMS
    u = pa.PencilArray.undef(TDT[prec], p, *extra)
    assert u.data.dim() == _lib.PA_MAX_DIMS
    u.data.normal_()
    flat = u.data.cpu().numpy().reshape(-1, N)
    for kind in KINDS:
        out = pa.PencilArray.undef(TDT[prec], p, *extra)
        n0 = pa.launch_count()
        pa.r2r_(out, u, kind)
        torch.cuda.synchronize()
        assert pa.launch_count() - n0 == 1
        assert out.data.cpu().numpy().reshape(-1, N).tobytes() == run_lines(flat, prec, kind).tobytes()


# ------------------------------------------------------------------ C ABI, refusals, streams
@pytest.mark.parametrize("prec", ["d", "f"])
def test_canaries_around_dst_and_src_untouched(prec):
    N, nl = 256, 19
    s = 8 if prec == "d" else 4
    p = line_pencil((N, nl, 1))
    pad = 4096
    src = torch.randn(nl * N, dtype=TDT[prec], device="cuda")
    before = src.clone()
    for kind, code in (("REDFT10", 5), ("REDFT01", 4), ("RODFT10", 9), ("RODFT01", 8)):
        buf = torch.full((2 * pad + nl * N * s,), 0xA5, dtype=torch.uint8, device="cuda")
        flags = 0 if prec == "d" else _lib.PA_FFT_F32
        pa.check(lib.pa_r2r(p._h, 0, None, code, flags, C.c_void_p(src.data_ptr()),
                            C.c_void_p(buf.data_ptr() + pad), stream_ptr()))
        torch.cuda.synchronize()
        b = buf.cpu()
        assert bool((b[:pad] == 0xA5).all()) and bool((b[-pad:] == 0xA5).all()), kind
        got = b[pad:-pad].view(TDT[prec]).numpy().reshape(nl, N)
        ref = scipy_r2r(before.cpu().numpy().reshape(nl, N).astype(np.float64), kind)
        assert np.abs(got - ref).max() <= tol(N, ref, prec), kind
        assert torch.equal(raw(src), raw(before)), kind


def test_refusals_and_empty_arrays_launch_nothing():
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    p = line_pencil((64, 4, 4), topo=topo)
    x = pa.PencilArray.undef(torch.float64, p)
    x.data.normal_()
    torch.cuda.synchronize()
    n0 = pa.launch_count()
    cases = [
        lambda: pa.r2r_(pa.PencilArray.undef(torch.float32, p), x, "REDFT10"),          # mixed dtypes
        lambda: pa.r2r_(pa.PencilArray.undef(torch.complex128, p),
                        pa.PencilArray.undef(torch.complex128, p), "REDFT10"),        # complex
        lambda: pa.r2r_(pa.PencilArray.undef(torch.float64, line_pencil((64, 4, 2), topo=topo)), x,
                        "REDFT01"),                                                   # other pencil
        lambda: pa.r2r_(pa.PencilArray.undef(torch.float64, p, 2), x, "RODFT10"),       # extra dims
        lambda: pa.r2r_(x, x, "REDFT00"),                                             # kind
    ]
    for n in (8, 24, 4096):                                                           # N
        q = line_pencil((n, 4, 4))
        cases.append(lambda q=q: pa.r2r_(*[pa.PencilArray.undef(torch.float64, q)] * 2, "REDFT10"))
    qd = line_pencil((64, 4, 4), decomp=(1, 3))                                        # decomposed axis
    cases.append(lambda: pa.r2r_(*[pa.PencilArray.undef(torch.float64, qd)] * 2, "REDFT10"))
    for case in cases:
        with pytest.raises(pa.ArgumentError):
            case()
    # C-level refusals on device pointers: bad kind / flags, partial overlap, misalignment
    buf = torch.zeros(2 * 64 * 16 + 64, dtype=torch.float64, device="cuda")
    a = buf.data_ptr()
    for kind, flags, s, d in ((3, 0, a, a), (5, _lib.PA_FFT_FORWARD, a, a), (5, 0, a, a + 64),
                              (5, 0, a + 8, a + 8 + 64 * 16 * 8)):
        assert lib.pa_r2r(p._h, 0, None, kind, flags, C.c_void_p(s), C.c_void_p(d),
                          stream_ptr()) == _lib.PA_EINVAL
    torch.cuda.synchronize()
    assert pa.launch_count() == n0
    for prec in ("d", "f"):
        e = line_pencil((32, 0, 4))
        ue = pa.PencilArray.undef(TDT[prec], e)
        for kind in KINDS:
            pa.r2r_(ue, ue, kind)
            pa.r2r_(pa.PencilArray.undef(TDT[prec], e), ue, kind)
    torch.cuda.synchronize()
    assert pa.launch_count() == n0


@pytest.mark.parametrize("prec", ["d", "f"])
def test_on_a_held_side_stream(prec):
    """On a caller's side stream behind a spin: the call returns before the spin ends (no host
    synchronisation), reads the input produced behind the spin, and gives the default-stream
    result byte for byte."""
    N = 512
    p = line_pencil((N, 64, 8))
    x_dev = torch.randn(8, 64, N, dtype=TDT[prec], device="cuda")
    for kind in KINDS:
        u = pa.PencilArray.undef(TDT[prec], p)
        out = pa.PencilArray.undef(TDT[prec], p)
        u.data.copy_(x_dev)
        pa.r2r_(out, u, kind)
        torch.cuda.synchronize()
        first = out.data.clone()
        raw(u.data).fill_(0xEE)
        raw(out.data).fill_(0xEE)
        s = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            held = hold()
            u.data.copy_(x_dev)
            pa.r2r_(out, u, kind)
            assert not held.query(), "r2r_ returned after the spin had ended: a host synchronisation"
            got = out.data.clone()
        torch.cuda.synchronize()
        assert torch.equal(raw(got), raw(first)), kind


# ----------------------------------------------------------------- the mixed 3-d transform
def mixed_chain(dims, topo):
    """x (real), y (real and complex) and z (complex) pencils: DCT-II along x, rfft along y, fft
    along z."""
    pxr = pa.Pencil(topo, dims, (2, 3))
    pyr = pa.Pencil(pxr, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    pyc = pa.Pencil(pyr, size_global=(dims[0], dims[1] // 2 + 1, dims[2]))
    pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    return pxr, pyr, pyc, pzc


@pytest.mark.parametrize("prec", ["d", "f"])
@pytest.mark.parametrize("dims", [(16, 32, 8), (64, 64, 64), (128, 16, 32)])
def test_mixed_three_dimensional_transform(dims, prec):
    """Forward: r2r_ DCT-II along x, plain real x->y, rfft_ along y, fused y->z + fft: the z-pencil
    array is fft(rfft(dct(G, 2, axis=0), axis=1), axis=2).  Backward inverts each step and returns
    2 Nx Ny Nz G."""
    rdt, cdt = (torch.float64, torch.complex128) if prec == "d" else (torch.float32, torch.complex64)
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pxr, pyr, pyc, pzc = mixed_chain(dims, topo)
    ux, ux2, uy = (pa.PencilArray.undef(rdt, p) for p in (pxr, pxr, pyr))
    uyc, uzc = pa.PencilArray.undef(cdt, pyc), pa.PencilArray.undef(cdt, pzc)
    ux.data.normal_()
    G = ux.logical().cpu().numpy().astype(np.float64)
    pa.r2r_(ux2, ux, "REDFT10")
    pa.transpose_(pa.Transposition(uy, ux2))
    pa.rfft_(uyc, uy)
    pa.transpose_(pa.Transposition(uzc, uyc), fft="forward")
    torch.cuda.synchronize()
    ref = np.fft.fft(np.fft.rfft(sf.dct(G, 2, axis=0), axis=1), axis=2)
    n = math.prod(dims)
    assert np.abs(uzc.logical().cpu().numpy() - ref).max() <= tol(n, ref, prec)
    pa.fft_(uzc, "backward")
    pa.transpose_(pa.Transposition(uyc, uzc))
    pa.brfft_(uy, uyc)
    pa.transpose_(pa.Transposition(ux2, uy))
    pa.r2r_(ux2, ux2, "REDFT01")
    torch.cuda.synchronize()
    want = 2 * n * G
    assert np.abs(ux2.logical().cpu().numpy() - want).max() <= tol(n, want, prec)


@pytest.mark.parametrize("world", [2, 4])
def test_mixed_three_dimensional_transform_ranks_sharing_the_gpu(world, tmp_path):
    """2 / 4 processes over the NCCL-free communicator, PointToPoint and Alltoallv, both
    precisions."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29891 + world),
           os.path.join(HERE, "mp_r2r_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1", PA_TEST_TMPDIR=str(tmp_path))
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    assert f"MP_R2R_OK world={world}" in out.stdout, out.stdout[-2000:]
