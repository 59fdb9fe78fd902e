"""Single-precision FFTs (PA_FFT_F32: complex64 `fft_` / fused `transpose_(t, fft=...)`, float32
<-> complex64 `rfft_` / `brfft_`) on one GPU, against the extended-precision DFT per line.

The inputs are rounded to float32 first and exactly those values go to the reference, so the
error measured is the kernels' own, in units of eps32:
* accuracy: `fft_` at every L in 8..1024 and `rfft_` / `brfft_` at every N in 16..2048, both
  directions, 64 lines scaled by 2^s: worst line within eps32 log2(L), RMS within 3x cuFFT's
  complex64 / float32 transforms on the same data;
* known answers (impulses, constants, alternating signs, bin-aligned exponentials; brfft_ ignores
  the imaginary parts of bins 0 and N/2 bit for bit);
* the fused ComplexF32 transpose + FFT is byte for byte `fft_` of the plain transpose (partial
  column tiles, linear gather, extra dims up to PA_MAX_DIMS, odd source extents), and an rfft_
  batch is byte for byte its lines one launch at a time (complex lines that start only 8-byte
  aligned included);
* canaries around the destination through the C ABI; refusals launch nothing; one held side
  stream per entry point; the real Float32 3-d transform on one rank against numpy.fft."""
import math

import numpy as np
import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200._lib import lib, check, i64arr
from fft_ref import brfft_ld, fft_ld, line_errors, rfft_ld, scaled_lines
from gpu_util import hold, ptr, stream_ptr

pytestmark = pytest.mark.gpu
LS = [1 << k for k in range(3, 11)]
NS = [1 << k for k in range(4, 12)]
NLINES = 64
EPS32 = float(np.finfo(np.float32).eps)
F32 = pa._lib.PA_FFT_F32
SENTINEL = 0x5A


def _topo():
    return pa.MPITopology(pa.COMM_SELF, (1, 1))


def lines32(seed, nl, L, complex_=True):
    """scaled_lines rounded to single precision: the exact inputs of kernel and reference"""
    x = scaled_lines(np.random.default_rng(seed), nl, L, complex_=complex_)
    return x.astype(np.complex64 if complex_ else np.float32)


def fft_lines_on_gpu(x, sign):
    nl, L = x.shape
    u = pa.PencilArray.undef(torch.complex64, pa.Pencil(_topo(), (L, nl, 1), (2, 3)))
    u.data.copy_(torch.from_numpy(np.ascontiguousarray(x).reshape(u.data.shape)))
    n0 = pa.launch_count()
    pa.fft_(u, "forward" if sign < 0 else "backward")
    torch.cuda.synchronize()
    assert pa.launch_count() - n0 == 1
    return u.data.cpu().numpy().reshape(x.shape)


def _real_pencils(N, nl):
    pr = pa.Pencil(_topo(), (N, nl, 1), (2, 3))
    pc = pa.Pencil(pr, size_global=(N // 2 + 1, nl, 1))
    return pr, pc


def rfft_on_gpu(x):
    nl, N = x.shape
    pr, pc = _real_pencils(N, nl)
    xr = pa.PencilArray.undef(torch.float32, pr)
    xc = pa.PencilArray.undef(torch.complex64, pc)
    xr.data.copy_(torch.from_numpy(np.ascontiguousarray(x).reshape(xr.data.shape)))
    before = xr.data.clone()
    pa.rfft_(xc, xr)
    torch.cuda.synchronize()
    assert torch.equal(xr.data, before)
    return xc.data.cpu().numpy().reshape(nl, N // 2 + 1)


def brfft_on_gpu(X, N):
    nl = X.shape[0]
    pr, pc = _real_pencils(N, nl)
    xc = pa.PencilArray.undef(torch.complex64, pc)
    xr = pa.PencilArray.undef(torch.float32, pr)
    xc.data.copy_(torch.from_numpy(np.ascontiguousarray(X).reshape(xc.data.shape)))
    before = xc.data.clone()
    pa.brfft_(xr, xc)
    torch.cuda.synchronize()
    assert torch.equal(xc.data.view(torch.uint8), before.view(torch.uint8))
    return xr.data.cpu().numpy().reshape(nl, N)


def _hermitian_clean(X):
    Xc = X.copy()
    Xc[:, 0] = Xc[:, 0].real
    Xc[:, -1] = Xc[:, -1].real
    return Xc


# ------------------------------------------------------------------------------- accuracy
@pytest.mark.parametrize("L", LS)
def test_fft32_accuracy_per_line(L):
    x = lines32(L, NLINES, L)
    dev = torch.from_numpy(x).cuda()
    for sign in (-1, 1):
        ref = fft_ld(x, sign)
        got = fft_lines_on_gpu(x, sign)
        assert got.dtype == np.complex64
        mx, rms = line_errors(got, ref)
        cu = (torch.fft.fft(dev) if sign < 0 else torch.fft.ifft(dev, norm="forward")).cpu().numpy()
        assert cu.dtype == np.complex64
        _, rms_cu = line_errors(cu, ref)
        assert mx <= EPS32 * math.log2(L), (L, sign, mx / EPS32, rms / EPS32, rms_cu / EPS32)
        assert rms <= 3 * rms_cu, (L, sign, mx / EPS32, rms / EPS32, rms_cu / EPS32)


@pytest.mark.parametrize("N", NS)
def test_rfft32_and_brfft32_accuracy_per_line(N):
    x = lines32(N, NLINES, N, complex_=False)
    ref = rfft_ld(x)
    mx, rms = line_errors(rfft_on_gpu(x), ref)
    _, rms_cu = line_errors(torch.fft.rfft(torch.from_numpy(x).cuda()).cpu().numpy(), ref)
    assert mx <= EPS32 * math.log2(N), (N, "r2c", mx / EPS32, rms / EPS32, rms_cu / EPS32)
    assert rms <= 3 * rms_cu, (N, "r2c", mx / EPS32, rms / EPS32, rms_cu / EPS32)

    X = lines32(N + 1, NLINES, N // 2 + 1)
    ref = brfft_ld(X, N)
    got = brfft_on_gpu(X, N)
    assert got.dtype == np.float32
    mx, rms = line_errors(got, ref)
    cu = torch.fft.irfft(torch.from_numpy(_hermitian_clean(X)).cuda(), n=N, norm="forward").cpu().numpy()
    _, rms_cu = line_errors(cu, ref)
    assert mx <= EPS32 * math.log2(N), (N, "c2r", mx / EPS32, rms / EPS32, rms_cu / EPS32)
    assert rms <= 3 * rms_cu, (N, "c2r", mx / EPS32, rms / EPS32, rms_cu / EPS32)
    # bins 0 and N/2: their imaginary parts are ignored -- exactly, not approximately
    assert got.tobytes() == brfft_on_gpu(_hermitian_clean(X), N).tobytes()


# -------------------------------------------------------------------------- known answers
@pytest.mark.parametrize("L", LS)
def test_fft32_known_answers(L):
    n = np.arange(L)
    for sign in (-1, 1):
        imp = np.eye(L, dtype=np.complex64)
        got = fft_lines_on_gpu(imp, sign)
        mx, _ = line_errors(got, fft_ld(imp, sign))
        assert mx <= EPS32 * math.log2(L), (L, sign, "impulses", mx)
        assert np.all(got[0] == 1)
        c = (np.array([1.0, -3.5, 2.0 ** -30, 1e6 + 1j])[:, None] * np.ones((1, L))).astype(np.complex64)
        got = fft_lines_on_gpu(c, sign)
        assert np.array_equal(got[:, 0], L * c[:, 0]) and not np.any(got[:, 1:]), (L, sign, "const")
        alt = np.where(n % 2 == 0, 1.0, -1.0)[None, :].astype(np.complex64)
        got = fft_lines_on_gpu(alt, sign)
        assert abs(got[0, L // 2] - L) <= EPS32 * L
        assert np.abs(np.delete(got[0], L // 2)).max() <= EPS32 * L * math.log2(L)
        k0 = np.array([1, 3, L // 2 - 1, L - 1])
        e = np.exp(-sign * 2j * np.pi * np.outer(k0, n) / L).astype(np.complex64)
        got = fft_lines_on_gpu(e, sign)
        mx, _ = line_errors(got, fft_ld(e, sign))
        assert mx <= EPS32 * math.log2(L), (L, sign, "exp", mx)
        assert np.all(np.abs(got).argmax(axis=1) == k0)


@pytest.mark.parametrize("N", [16, 64, 2048])
def test_rfft32_known_answers(N):
    n = np.arange(N)
    x = np.stack([np.ones(N), np.where(n % 2 == 0, 1.0, -1.0), np.cos(2 * np.pi * 3 * n / N),
                  np.eye(N)[1], np.eye(N)[N - 1]]).astype(np.float32)
    got = rfft_on_gpu(x)
    mx, _ = line_errors(got, rfft_ld(x))
    assert mx <= EPS32 * math.log2(N), mx
    assert got[0, 0] == N and got[1, N // 2] == N
    back = brfft_on_gpu(got, N)
    mx, _ = line_errors(back, N * x.astype(np.float64))
    assert mx <= 2 * EPS32 * math.log2(N), mx


# ------------------------------------------------------------- fused == fft_(plain), bytes
def _fill(u, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    f = u.data.view(torch.float32)
    f.copy_(torch.randn(f.shape, generator=g, device="cuda", dtype=torch.float32))


def _fused_equals_unfused(dst_pencil, src, extra, direction):
    fused = pa.PencilArray.undef(torch.complex64, dst_pencil, *extra)
    fused.data.view(torch.uint8).fill_(SENTINEL)
    n0 = pa.launch_count()
    pa.transpose_(pa.Transposition(fused, src), fft=direction)
    torch.cuda.synchronize()
    assert pa.launch_count() - n0 == 1
    plain = pa.PencilArray.undef(torch.complex64, dst_pencil, *extra)
    pa.transpose_(pa.Transposition(plain, src))
    pa.fft_(plain, direction)
    torch.cuda.synchronize()
    assert torch.equal(fused.data.view(torch.uint8), plain.data.view(torch.uint8)), \
        (dst_pencil.size_global, extra, direction)
    return fused, plain


def _x_to_y(dims):
    px = pa.Pencil(_topo(), dims, (2, 3))
    py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    return px, py


@pytest.mark.parametrize("L", [8, 64, 256, 512, 1024])
def test_fused32_transposing_gather_partial_tiles(L):
    C_ = 8 if L >= 1024 else 16   # lines per CTA in single precision
    for ncol in (2 * C_, 2 * C_ + 1, 3 * C_ - 1):
        px, py = _x_to_y((ncol, L, 3))
        ux = pa.PencilArray.undef(torch.complex64, px)
        _fill(ux, ncol + L)
        before = ux.data.clone()
        for d in ("forward", "backward"):
            fused, _ = _fused_equals_unfused(py, ux, (), d)
        assert torch.equal(ux.data.view(torch.uint8), before.view(torch.uint8))
    # and the transform itself, per line, for the last case (backward)
    lines = np.moveaxis(ux.data.cpu().numpy(), -1, -2)   # torch (z, y, x) -> (z, x, y)
    mx, _ = line_errors(fused.data.cpu().numpy(), fft_ld(lines, 1))
    assert mx <= EPS32 * math.log2(L), mx


@pytest.mark.parametrize("dims", [(9, 64, 3), (33, 16, 5), (513, 8, 2), (17, 1024, 1)])
def test_fused32_odd_source_extent(dims):
    """x -> y with the x extent N/2+1 odd (the complex axis of a real-input plan)."""
    px, py = _x_to_y(dims)
    ux = pa.PencilArray.undef(torch.complex64, px)
    _fill(ux, dims[0])
    for d in ("forward", "backward"):
        _fused_equals_unfused(py, ux, (), d)


@pytest.mark.parametrize("extra", [(2,), (3, 2)])
@pytest.mark.parametrize("L", [16, 512])
def test_fused32_extra_dims_and_linear_gather(L, extra):
    px = pa.Pencil(_topo(), (11, L, 3), (2, 3))
    py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    ux = pa.PencilArray.undef(torch.complex64, px, *extra)
    _fill(ux, L)
    for d in ("forward", "backward"):
        _fused_equals_unfused(py, ux, extra, d)
    qx = pa.Pencil(_topo(), (L, 5, 3), (2, 3))
    q2 = pa.Pencil(qx, decomp_dims=(2, 3), permute=pa.Permutation(1, 3, 2))
    vx = pa.PencilArray.undef(torch.complex64, qx, *extra)
    _fill(vx, L + 1)
    for d in ("forward", "backward"):
        _fused_equals_unfused(q2, vx, extra, d)


def test_fused32_four_dimensional_with_every_outer_dim():
    """4-d pencil + 4 extra dims = PA_MAX_DIMS dims: 6 outer dims, every extent >= 2."""
    dims, extra = (3, 8, 2, 2), (2, 2, 2, 2)
    p1 = pa.Pencil(_topo(), dims, (2, 3))
    p2 = pa.Pencil(p1, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3, 4))
    u = pa.PencilArray.undef(torch.complex64, p1, *extra)
    _fill(u, 4)
    for d in ("forward", "backward"):
        got, _ = _fused_equals_unfused(p2, u, extra, d)
    lines = np.moveaxis(u.data.cpu().numpy(), -2, -1)
    g = got.data.cpu().numpy()
    assert g.shape == lines.shape
    mx, _ = line_errors(g, fft_ld(lines, 1))
    assert mx <= EPS32 * 3, mx


@pytest.mark.parametrize("N", [16, 256, 2048])
def test_rfft32_batch_equals_lines_one_at_a_time(N):
    """Complex line j starts at 8 (N/2+1) j bytes: the odd lines (1, 7, 23) are only 8-byte
    aligned inside the batch, 16-byte aligned alone."""
    x = lines32(3, 24, N, complex_=False)
    batch = rfft_on_gpu(x)
    for j in (0, 1, 7, 8, 23):
        assert rfft_on_gpu(x[j:j + 1]).tobytes() == batch[j:j + 1].tobytes(), (N, j)
    X = lines32(4, 24, N // 2 + 1)
    batch = brfft_on_gpu(X, N)
    for j in (0, 1, 5, 23):
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


@pytest.mark.parametrize("L,ncol", [(8, 17), (1024, 9), (64, 31)])
def test_canaries_fused32_transpose_c_abi(L, ncol):
    px, py = _x_to_y((ncol, L, 3))
    ux = pa.PencilArray.undef(torch.complex64, px)
    _fill(ux, L)
    before = ux.data.clone()
    t = pa.Transposition(pa.PencilArray.undef(torch.complex64, py), ux)
    nbytes = t.plan.info.length_out * 8
    buf, pattern = _canary_buffer(nbytes)
    check(lib.pa_transpose(t.plan.h, None, ptr(ux.data), ptr(buf, PAD),
                           pa._lib.PA_WAITALL | pa._lib.PA_FFT_FORWARD | F32, stream_ptr()))
    torch.cuda.synchronize()
    _outside_unchanged(buf, pattern, nbytes)
    assert torch.equal(ux.data.view(torch.uint8), before.view(torch.uint8))
    plain = pa.PencilArray.undef(torch.complex64, py)
    pa.transpose_(pa.Transposition(plain, ux))
    pa.fft_(plain, "forward")
    torch.cuda.synchronize()
    assert torch.equal(buf[PAD:PAD + nbytes], plain.data.view(torch.uint8).reshape(-1))


@pytest.mark.parametrize("N", [16, 2048])
def test_canaries_rfft32_c_abi(N):
    nl = 13
    pr, pc = _real_pencils(N, nl)
    xr = pa.PencilArray.undef(torch.float32, pr)
    xr.data.normal_()
    before = xr.data.clone()
    nbytes = nl * (N // 2 + 1) * 8
    buf, pattern = _canary_buffer(nbytes)
    check(lib.pa_rfft(pr._h, pc._h, 0, i64arr([]), pa._lib.PA_FFT_FORWARD | F32, ptr(xr.data),
                      ptr(buf, PAD), stream_ptr()))
    torch.cuda.synchronize()
    _outside_unchanged(buf, pattern, nbytes)
    assert torch.equal(xr.data, before)
    spec = buf[PAD:PAD + nbytes].clone()
    ref = rfft_ld(before.cpu().numpy().reshape(nl, N))
    mx, _ = line_errors(spec.view(torch.complex64).cpu().numpy().reshape(nl, N // 2 + 1), ref)
    assert mx <= EPS32 * math.log2(N), mx
    rbytes = nl * N * 4
    buf2, pattern2 = _canary_buffer(rbytes)
    check(lib.pa_rfft(pr._h, pc._h, 0, i64arr([]), pa._lib.PA_FFT_BACKWARD | F32, ptr(spec),
                      ptr(buf2, PAD), stream_ptr()))
    torch.cuda.synchronize()
    _outside_unchanged(buf2, pattern2, rbytes)
    back = buf2[PAD:PAD + rbytes].view(torch.float32).reshape(before.shape)
    assert (back / N - before).abs().max().item() <= 2 * EPS32 * math.log2(N) * before.abs().max().item()


# ------------------------------------------------------------------ refusals launch nothing
def test_refused_fused32_transposes_launch_nothing():
    # 48-point ComplexF32 lines: not a power of two
    px, py = _x_to_y((16, 48, 3))
    ux = pa.PencilArray.undef(torch.complex64, px)
    _fill(ux, 48)
    uy = pa.PencilArray.undef(torch.complex64, py)
    uy.data.view(torch.uint8).fill_(SENTINEL)
    t = pa.Transposition(uy, ux)
    assert not t.fft_fusable()
    torch.cuda.synchronize()
    n0 = pa.launch_count()
    with pytest.raises(pa.ArgumentError, match="power of two"):
        pa.transpose_(t, fft="forward")
    # a Float64 plan asked for an FFT: no flag is set for float64 arrays, and elsize 8 is refused
    qx, qy = _x_to_y((16, 64, 3))
    vx = pa.PencilArray.undef(torch.float64, qx)
    vx.data.normal_()
    vy = pa.PencilArray.undef(torch.float64, qy)
    vy.data.view(torch.uint8).fill_(SENTINEL)
    tq = pa.Transposition(vy, vx)
    assert not tq.fft_fusable()
    torch.cuda.synchronize()
    n1 = pa.launch_count()
    with pytest.raises(pa.ArgumentError, match="16-byte"):
        pa.transpose_(tq, fft="backward")
    # a ComplexF64 plan asked for a ComplexF32 FFT through the C ABI
    wx = pa.PencilArray.undef(torch.complex128, qx)
    wy = pa.PencilArray.undef(torch.complex128, qy)
    wy.data.view(torch.uint8).fill_(SENTINEL)
    tw = pa.Transposition(wy, wx)
    assert lib.pa_transpose(tw.plan.h, None, ptr(wx.data), ptr(wy.data),
                            pa._lib.PA_WAITALL | pa._lib.PA_FFT_FORWARD | F32, stream_ptr()) \
        == pa._lib.PA_EINVAL
    assert b"8-byte" in lib.pa_last_error()
    torch.cuda.synchronize()
    assert pa.launch_count() == n0 == n1
    for u in (uy, vy, wy):
        assert bool((u.data.view(torch.uint8) == SENTINEL).all())


# ------------------------------------------------------------------------ caller's stream
def on_side_stream(produce, call, consume):
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        held = hold()
        produce()
        call()
        assert not held.query(), "the call returned after the spin had ended: a host synchronisation"
        out = consume()
    torch.cuda.synchronize()
    return out


def _side_stream_equals_default(u_in, x_dev, call, u_out):
    u_in.data.copy_(x_dev)
    call()
    torch.cuda.synchronize()
    first = u_out.data.clone()
    u_in.data.view(torch.uint8).fill_(SENTINEL)
    u_out.data.view(torch.uint8).fill_(SENTINEL)
    got = on_side_stream(lambda: u_in.data.copy_(x_dev), call, lambda: u_out.data.clone())
    assert torch.equal(got.view(torch.uint8), first.view(torch.uint8))
    return first.cpu().numpy()


def _gate(got, ref, n):
    mx, _ = line_errors(got, ref)
    assert mx <= EPS32 * math.log2(n), (n, mx / EPS32)


@pytest.mark.parametrize("direction", ["forward", "backward"])
def test_fft32_on_a_side_stream(direction):
    L = 32
    u = pa.PencilArray.undef(torch.complex64, pa.Pencil(_topo(), (L, 12, 8), (2, 3)))
    rng = np.random.default_rng(21)
    x = (rng.standard_normal(u.data.shape) + 1j * rng.standard_normal(u.data.shape)).astype(np.complex64)
    got = _side_stream_equals_default(u, torch.from_numpy(x).cuda(), lambda: pa.fft_(u, direction), u)
    _gate(got, fft_ld(x, -1 if direction == "forward" else 1), L)


@pytest.mark.parametrize("direction", ["forward", "backward"])
def test_fused32_transpose_on_a_side_stream(direction):
    px, py = _x_to_y((17, 32, 8))
    ux, uy, plain = (pa.PencilArray.undef(torch.complex64, p) for p in (px, py, py))
    rng = np.random.default_rng(22)
    x = (rng.standard_normal(ux.data.shape) + 1j * rng.standard_normal(ux.data.shape)).astype(np.complex64)
    xd = torch.from_numpy(x).cuda()
    ux.data.copy_(xd)
    pa.transpose_(plain, ux)
    torch.cuda.synchronize()
    t = pa.Transposition(uy, ux)
    got = _side_stream_equals_default(ux, xd, lambda: pa.transpose_(t, fft=direction), uy)
    _gate(got, fft_ld(plain.data.cpu().numpy(), -1 if direction == "forward" else 1), 32)


def test_rfft32_and_brfft32_on_a_side_stream():
    N = 64
    pr, pc = _real_pencils(N, 12)
    xr, back = pa.PencilArray.undef(torch.float32, pr), pa.PencilArray.undef(torch.float32, pr)
    xc = pa.PencilArray.undef(torch.complex64, pc)
    rng = np.random.default_rng(23)
    x = rng.standard_normal(xr.data.shape).astype(np.float32)
    got = _side_stream_equals_default(xr, torch.from_numpy(x).cuda(), lambda: pa.rfft_(xc, xr), xc)
    _gate(got, rfft_ld(x), N)
    X = (rng.standard_normal(xc.data.shape) + 1j * rng.standard_normal(xc.data.shape)).astype(np.complex64)
    got = _side_stream_equals_default(xc, torch.from_numpy(X).cuda(), lambda: pa.brfft_(back, xc), back)
    _gate(got, brfft_ld(X, N), N)


# ------------------------------------------------------- the real Float32 3-d transform
def real_chain(dims):
    pxr = pa.Pencil(_topo(), dims, (2, 3))
    pxc = pa.Pencil(pxr, size_global=(dims[0] // 2 + 1,) + tuple(dims[1:]))
    pyc = pa.Pencil(pxc, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    return pxr, pxc, pyc, pzc


@pytest.mark.parametrize("dims", [(16, 32, 8), (64, 64, 64), (128, 16, 32), (2048, 8, 1024)])
def test_real32_three_dimensional_fft_like_pencilffts(dims):
    """rfft_ along x, fused x->y and y->z (complex64) against numpy.fft of the same float32 field,
    and back (fft_ along z, fused z->y, plain y->x, brfft_): prod(dims) times the input."""
    pxr, pxc, pyc, pzc = real_chain(dims)
    uxr = pa.PencilArray.undef(torch.float32, pxr)
    uxc, uyc, uzc = (pa.PencilArray.undef(torch.complex64, p) for p in (pxc, pyc, pzc))
    uxr.data.normal_()
    G = uxr.logical().cpu().numpy().astype(np.float64)
    n0 = pa.launch_count()
    pa.rfft_(uxc, uxr)
    pa.transpose_(pa.Transposition(uyc, uxc), fft="forward")
    pa.transpose_(pa.Transposition(uzc, uyc), fft="forward")
    torch.cuda.synchronize()
    assert pa.launch_count() - n0 == 3
    ref = np.fft.fftn(np.fft.rfft(G, axis=0), axes=(1, 2))
    n = math.prod(dims)
    tol = 8 * EPS32 * math.log2(n)
    got = uzc.logical().cpu().numpy()
    assert got.dtype == np.complex64
    assert np.abs(got - ref).max() <= tol * np.abs(ref).max()
    pa.fft_(uzc, "backward")
    pa.transpose_(pa.Transposition(uyc, uzc), fft="backward")
    pa.transpose_(pa.Transposition(uxc, uyc))
    back = pa.PencilArray.undef(torch.float32, pxr)
    pa.brfft_(back, uxc)
    torch.cuda.synchronize()
    assert np.abs(back.logical().cpu().numpy() - n * G).max() <= tol * n * np.abs(G).max()
