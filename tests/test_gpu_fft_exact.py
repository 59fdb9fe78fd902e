"""The FFT kernels against an extended-precision DFT (tests/fft_ref.py), per line, on one GPU.

* accuracy: `fft_` at every L in 8..1024 (both tunings of fft_lines), `rfft_` / `brfft_` at
  every N in 16..2048, both directions, on 64 lines scaled by 2^s (s cycling over -40..40): the
  worst line's relative error within eps log2(L), the RMS within 3x cuFFT's on the same data;
* known answers that catch index and digit-reversal slips (impulses, constants, alternating
  signs, bin-aligned exponentials; brfft_ ignoring the imaginary parts of bins 0 and N/2 bit for
  bit);
* invariant I1: `transpose_(t, fft=d)` is byte for byte `fft_` of the plain `transpose_` --
  partial column tiles, linear gather, extra dims up to PA_MAX_DIMS, fft_lines = 4 -- and rfft_
  of a batch is byte for byte the same lines one launch at a time;
* canaries around the destination through the C ABI, `src` untouched;
* one case past 2^32 bytes and 2^16 CTAs (skipped when the shared GPU lacks the memory)."""
import math

import numpy as np
import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200._lib import lib, check, i64arr
from fft_ref import EPS, brfft_ld, fft_ld, line_errors, rfft_ld, scaled_lines
from gpu_util import ptr, stream_ptr

pytestmark = pytest.mark.gpu
LS = [1 << k for k in range(3, 11)]
NS = [1 << k for k in range(4, 12)]
NLINES = 64


def _topo():
    return pa.MPITopology(pa.COMM_SELF, (1, 1))


def _lines_array(x):
    """complex lines (nl, L) -> a single-rank PencilArray (L, nl, 1) holding them"""
    nl, L = x.shape
    u = pa.PencilArray.undef(torch.complex128, pa.Pencil(_topo(), (L, nl, 1), (2, 3)))
    u.data.copy_(torch.from_numpy(np.ascontiguousarray(x).reshape(u.data.shape)))
    return u


def _with_fft_lines(v):
    pa.set_tunable("fft_lines", v)


@pytest.fixture
def fft_lines_default():
    yield
    pa.set_tunable("fft_lines", 0)


def fft_lines_on_gpu(x, sign):
    u = _lines_array(x)
    pa.fft_(u, "forward" if sign < 0 else "backward")
    torch.cuda.synchronize()
    return u.data.cpu().numpy().reshape(x.shape)


# ------------------------------------------------------------------------------- accuracy
@pytest.mark.parametrize("lines4", [0, 4])
@pytest.mark.parametrize("L", LS)
def test_fft_accuracy_per_line(L, lines4, fft_lines_default):
    _with_fft_lines(lines4)
    x = scaled_lines(np.random.default_rng(L), NLINES, L)
    dev = torch.from_numpy(x).cuda()
    for sign in (-1, 1):
        ref = fft_ld(x, sign)
        mx, rms = line_errors(fft_lines_on_gpu(x, sign), ref)
        cu = (torch.fft.fft(dev) if sign < 0 else torch.fft.ifft(dev, norm="forward")).cpu().numpy()
        _, rms_cu = line_errors(cu, ref)
        assert mx <= EPS * math.log2(L), (L, lines4, sign, mx, rms, rms_cu)
        assert rms <= 3 * rms_cu, (L, lines4, sign, mx, rms, rms_cu)


def _real_pencils(N, nl):
    pr = pa.Pencil(_topo(), (N, nl, 1), (2, 3))
    pc = pa.Pencil(pr, size_global=(N // 2 + 1, nl, 1))
    return pr, pc


def rfft_on_gpu(x):
    nl, N = x.shape
    pr, pc = _real_pencils(N, nl)
    xr = pa.PencilArray.undef(torch.float64, pr)
    xc = pa.PencilArray.undef(torch.complex128, pc)
    xr.data.copy_(torch.from_numpy(np.ascontiguousarray(x).reshape(xr.data.shape)))
    pa.rfft_(xc, xr)
    torch.cuda.synchronize()
    return xc.data.cpu().numpy().reshape(nl, N // 2 + 1)


def brfft_on_gpu(X, N):
    nl = X.shape[0]
    pr, pc = _real_pencils(N, nl)
    xc = pa.PencilArray.undef(torch.complex128, pc)
    xr = pa.PencilArray.undef(torch.float64, pr)
    xc.data.copy_(torch.from_numpy(np.ascontiguousarray(X).reshape(xc.data.shape)))
    pa.brfft_(xr, xc)
    torch.cuda.synchronize()
    return xr.data.cpu().numpy().reshape(nl, N)


def _hermitian_clean(X):
    Xc = X.copy()
    Xc[:, 0] = Xc[:, 0].real
    Xc[:, -1] = Xc[:, -1].real
    return Xc


@pytest.mark.parametrize("N", NS)
def test_rfft_and_brfft_accuracy_per_line(N):
    rng = np.random.default_rng(N)
    x = scaled_lines(rng, NLINES, N, complex_=False)
    ref = rfft_ld(x)
    mx, rms = line_errors(rfft_on_gpu(x), ref)
    _, rms_cu = line_errors(torch.fft.rfft(torch.from_numpy(x).cuda()).cpu().numpy(), ref)
    assert mx <= EPS * math.log2(N), (N, "r2c", mx, rms, rms_cu)
    assert rms <= 3 * rms_cu, (N, "r2c", mx, rms, rms_cu)

    X = scaled_lines(rng, NLINES, N // 2 + 1)
    ref = brfft_ld(X, N)
    got = brfft_on_gpu(X, N)
    mx, rms = line_errors(got, ref)
    cu = torch.fft.irfft(torch.from_numpy(_hermitian_clean(X)).cuda(), n=N, norm="forward").cpu().numpy()
    _, rms_cu = line_errors(cu, ref)
    assert mx <= EPS * math.log2(N), (N, "c2r", mx, rms, rms_cu)
    assert rms <= 3 * rms_cu, (N, "c2r", mx, rms, rms_cu)
    # bins 0 and N/2: their imaginary parts are ignored -- exactly, not approximately
    assert got.tobytes() == brfft_on_gpu(_hermitian_clean(X), N).tobytes()


# -------------------------------------------------------------------------- known answers
@pytest.mark.parametrize("lines4", [0, 4])
@pytest.mark.parametrize("L", LS)
def test_fft_known_answers(L, lines4, fft_lines_default):
    _with_fft_lines(lines4)
    n = np.arange(L)
    for sign in (-1, 1):
        # line m = delta[n - m]: its transform is W^(m k), a different line for every m
        imp = np.eye(L, dtype=np.complex128)
        got = fft_lines_on_gpu(imp, sign)
        mx, _ = line_errors(got, fft_ld(imp, sign))
        assert mx <= EPS * math.log2(L), (L, sign, "impulses", mx)
        assert np.all(got[0] == 1)                           # delta[n]: all ones, exactly
        # constant lines: L c at bin 0, exact zeros elsewhere
        c = np.array([1.0, -3.5, 2.0 ** -30, 1e6 + 1j])[:, None] * np.ones((1, L))
        got = fft_lines_on_gpu(c, sign)
        assert np.array_equal(got[:, 0], L * c[:, 0]) and not np.any(got[:, 1:]), (L, sign, "const")
        # alternating signs: everything in bin L/2
        alt = np.where(n % 2 == 0, 1.0, -1.0)[None, :].astype(np.complex128)
        got = fft_lines_on_gpu(alt, sign)
        assert abs(got[0, L // 2] - L) <= EPS * L and np.abs(np.delete(got[0], L // 2)).max() <= EPS * L * math.log2(L)
        # bin-aligned exponentials exp(-sign 2 pi i k0 n / L): L at bin k0
        k0 = np.array([1, 3, L // 2 - 1, L - 1])
        e = np.exp(-sign * 2j * np.pi * np.outer(k0, n) / L)
        got = fft_lines_on_gpu(e, sign)
        mx, _ = line_errors(got, fft_ld(e, sign))
        assert mx <= EPS * math.log2(L), (L, sign, "exp", mx)
        assert np.all(np.abs(got).argmax(axis=1) == k0)


@pytest.mark.parametrize("N", [16, 64, 2048])
def test_rfft_known_answers(N):
    n = np.arange(N)
    x = np.stack([np.ones(N), np.where(n % 2 == 0, 1.0, -1.0), np.cos(2 * np.pi * 3 * n / N),
                  np.eye(N)[1], np.eye(N)[N - 1]])
    got = rfft_on_gpu(x)
    mx, _ = line_errors(got, rfft_ld(x))
    assert mx <= EPS * math.log2(N), mx
    assert got[0, 0] == N and got[1, N // 2] == N
    # and back: N x
    back = brfft_on_gpu(got, N)
    mx, _ = line_errors(back, N * x)
    assert mx <= 2 * EPS * math.log2(N), mx


# ------------------------------------------------------------- I1: fused == fft_(plain), bytes
def _fill(u, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    u.data.view(torch.float64).copy_(torch.randn(u.data.view(torch.float64).shape, generator=g,
                                                 device="cuda", dtype=torch.float64))


def _i1(dst_pencil, src, extra, direction):
    fused = pa.PencilArray.undef(torch.complex128, dst_pencil, *extra)
    fused.data.view(torch.uint8).fill_(0x5A)
    n0 = pa.launch_count()
    pa.transpose_(pa.Transposition(fused, src), fft=direction)
    torch.cuda.synchronize()
    assert pa.launch_count() - n0 == 1
    plain = pa.PencilArray.undef(torch.complex128, dst_pencil, *extra)
    pa.transpose_(pa.Transposition(plain, src))
    pa.fft_(plain, direction)
    torch.cuda.synchronize()
    assert torch.equal(fused.data.view(torch.uint8), plain.data.view(torch.uint8)), \
        (dst_pencil.size_global, extra, direction)
    return fused


def _x_to_y(dims, extra=()):
    """x -> y with y contiguous in the destination: a transposing gather, ncol = dims[0]"""
    px = pa.Pencil(_topo(), dims, (2, 3))
    py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    return px, py


@pytest.mark.parametrize("L", [8, 64, 256, 1024])
@pytest.mark.parametrize("lines4", [0, 4])
def test_i1_transposing_gather_partial_tiles(L, lines4, fft_lines_default):
    _with_fft_lines(lines4)
    C_ = 4 if (L >= 1024 or (lines4 == 4 and L >= 256)) else 8
    for ncol in (2 * C_, 2 * C_ + 1, 2 * C_ + C_ - 1):
        px, py = _x_to_y((ncol, L, 3))
        ux = pa.PencilArray.undef(torch.complex128, px)
        _fill(ux, ncol + L)
        before = ux.data.clone()
        for d in ("forward", "backward"):
            _i1(py, ux, (), d)
        assert torch.equal(ux.data.view(torch.uint8), before.view(torch.uint8))


@pytest.mark.parametrize("extra", [(2,), (3, 2)])
@pytest.mark.parametrize("L", [16, 512])
def test_i1_extra_dims_and_linear_gather(L, extra):
    px, py = _x_to_y((11, L, 3), extra)
    ux = pa.PencilArray.undef(torch.complex128, px, *extra)
    _fill(ux, L)
    for d in ("forward", "backward"):
        _i1(py, ux, extra, d)
    # a local permute that keeps the contiguous dim (linear gather)
    qx = pa.Pencil(_topo(), (L, 5, 3), (2, 3))
    q2 = pa.Pencil(qx, decomp_dims=(2, 3), permute=pa.Permutation(1, 3, 2))
    vx = pa.PencilArray.undef(torch.complex128, qx, *extra)
    _fill(vx, L + 1)
    for d in ("forward", "backward"):
        _i1(q2, vx, extra, d)


def test_i1_four_dimensional_with_every_outer_dim():
    """4-d pencil + 4 extra dims = PA_MAX_DIMS dims: 6 outer dims (FFT_MAXO), every extent >= 2."""
    dims, extra = (3, 8, 2, 2), (2, 2, 2, 2)
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    p1 = pa.Pencil(topo, dims, (2, 3))
    p2 = pa.Pencil(p1, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3, 4))
    u = pa.PencilArray.undef(torch.complex128, p1, *extra)
    _fill(u, 4)
    for d in ("forward", "backward"):
        got = _i1(p2, u, extra, d)
    # and the transform itself, against the reference, line by line.  Torch shapes (reversed
    # memory order): u (e4, e3, e2, e1, w, z, y, x); got (e4, e3, e2, e1, w, z, x, y)
    lines = np.moveaxis(u.data.cpu().numpy(), -2, -1)
    g = got.data.cpu().numpy()
    assert g.shape == lines.shape
    mx, _ = line_errors(g, fft_ld(lines, 1))    # the last direction run: backward
    assert mx <= EPS * 3, mx


@pytest.mark.parametrize("N", [16, 256, 2048])
def test_rfft_batch_equals_lines_one_at_a_time(N):
    x = scaled_lines(np.random.default_rng(3), 24, N, complex_=False)
    batch = rfft_on_gpu(x)
    for j in (0, 1, 7, 8, 23):
        assert rfft_on_gpu(x[j:j + 1]).tobytes() == batch[j:j + 1].tobytes(), (N, j)
    X = scaled_lines(np.random.default_rng(4), 24, N // 2 + 1)
    batch = brfft_on_gpu(X, N)
    for j in (0, 5, 23):
        assert brfft_on_gpu(X[j:j + 1], N).tobytes() == batch[j:j + 1].tobytes(), (N, j)


# ----------------------------------------------------------------------------- canaries
PAD = 4096


def _canary_buffer(nbytes):
    buf = torch.empty(nbytes + 2 * PAD, dtype=torch.uint8, device="cuda")
    buf.copy_(torch.arange(buf.numel(), device="cuda", dtype=torch.int64).mul_(37).remainder_(251)
              .to(torch.uint8))
    return buf, buf.clone()


def _outside_unchanged(buf, pattern, nbytes):
    assert torch.equal(buf[:PAD], pattern[:PAD])
    assert torch.equal(buf[PAD + nbytes:], pattern[PAD + nbytes:])


@pytest.mark.parametrize("L,ncol", [(8, 9), (1024, 5), (64, 15)])
def test_canaries_fused_transpose_c_abi(L, ncol):
    px, py = _x_to_y((ncol, L, 3))
    ux = pa.PencilArray.undef(torch.complex128, px)
    _fill(ux, L)
    before = ux.data.clone()
    t = pa.Transposition(pa.PencilArray.undef(torch.complex128, py), ux)
    nbytes = t.plan.info.length_out * 16
    buf, pattern = _canary_buffer(nbytes)
    check(lib.pa_transpose(t.plan.h, None, ptr(ux.data), ptr(buf, PAD),
                           pa._lib.PA_WAITALL | pa._lib.PA_FFT_FORWARD, stream_ptr()))
    torch.cuda.synchronize()
    _outside_unchanged(buf, pattern, nbytes)
    assert torch.equal(ux.data.view(torch.uint8), before.view(torch.uint8))
    plain = pa.PencilArray.undef(torch.complex128, py)
    pa.transpose_(pa.Transposition(plain, ux))
    pa.fft_(plain, "forward")
    torch.cuda.synchronize()
    assert torch.equal(buf[PAD:PAD + nbytes], plain.data.view(torch.uint8).reshape(-1))


@pytest.mark.parametrize("N", [16, 2048])
def test_canaries_rfft_c_abi(N):
    nl = 13
    pr, pc = _real_pencils(N, nl)
    xr = pa.PencilArray.undef(torch.float64, pr)
    xr.data.normal_()
    before = xr.data.clone()
    nbytes = nl * (N // 2 + 1) * 16
    buf, pattern = _canary_buffer(nbytes)
    check(lib.pa_rfft(pr._h, pc._h, 0, i64arr([]), pa._lib.PA_FFT_FORWARD, ptr(xr.data), ptr(buf, PAD),
                      stream_ptr()))
    torch.cuda.synchronize()
    _outside_unchanged(buf, pattern, nbytes)
    assert torch.equal(xr.data, before)
    spec = buf[PAD:PAD + nbytes].clone()
    rbytes = nl * N * 8
    buf2, pattern2 = _canary_buffer(rbytes)
    check(lib.pa_rfft(pr._h, pc._h, 0, i64arr([]), pa._lib.PA_FFT_BACKWARD, ptr(spec), ptr(buf2, PAD),
                      stream_ptr()))
    torch.cuda.synchronize()
    _outside_unchanged(buf2, pattern2, rbytes)
    back = buf2[PAD:PAD + rbytes].view(torch.float64).reshape(before.shape)
    assert (back / N - before).abs().max().item() <= 2 * EPS * math.log2(N) * before.abs().max().item()


# --------------------------------------------------------------- past 2^32 bytes, 2^16 CTAs
def test_large_in_place_fft_past_4_gib():
    dims = (8, 8192, 4097)                    # 4.0002 GiB of ComplexF64, 4.2 M CTAs
    need = math.prod(dims) * 16
    free, _ = torch.cuda.mem_get_info()
    if free < 3 * need:
        pytest.skip(f"needs {3 * need / 2**30:.1f} GiB free on the shared GPU, {free / 2**30:.1f} free")
    u = pa.PencilArray.undef(torch.complex128, pa.Pencil(_topo(), dims, (2, 3)))
    g = torch.Generator(device="cuda").manual_seed(9)
    flat = u.data.view(torch.float64).reshape(-1)
    chunk = 1 << 27
    for i in range(0, flat.numel(), chunk):
        n = min(chunk, flat.numel() - i)
        flat[i:i + n].copy_(torch.randn(n, generator=g, device="cuda", dtype=torch.float64))
    lines = u.data.reshape(-1, 8)
    nl = lines.shape[0]
    pick = np.unique(np.concatenate(([0, 1, nl // 2, nl - 2, nl - 1],
                                     np.random.default_rng(1).integers(0, nl, 200))))
    idx = torch.from_numpy(pick).cuda()
    x = lines.index_select(0, idx).cpu().numpy()
    pa.fft_(u, "forward")
    torch.cuda.synchronize()
    got = lines.index_select(0, idx).cpu().numpy()
    del u, lines, flat
    torch.cuda.empty_cache()
    mx, _ = line_errors(got, fft_ld(x, -1))
    assert mx <= EPS * 3, mx
