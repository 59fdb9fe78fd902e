"""The fused transposition of real arrays + DCT / DST (`Transposition(..., r2r=kind)`,
`pa_transpose_r2r`) and + real-to-complex FFT (`Transposition(..., rfft=True)`,
`pa_transpose_rfft`) on the GPU.  They run the real gather and the post-load stages of `r2r_` /
`rfft_`, so their output must be the bytes of `r2r_(transpose_(...))` / `rfft_(transpose_(...))`
-- in both precisions, at every line length, for all four kinds, through both gathers.  Plus: no
side effects, refusals that launch nothing, the wall-bounded 3-d chains in three kernels each
way, caller streams, and 2, 3, 4 and 8 processes sharing the GPU
(tests/mp_fused_real_worker.py)."""
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
from gpu_util import hold, stream_ptr

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
PREC = {"f64": (torch.float64, torch.complex128, np.finfo(np.float64).eps, 0),
        "f32": (torch.float32, torch.complex64, np.finfo(np.float32).eps, _lib.PA_FFT_F32)}
KINDS = ["REDFT10", "REDFT01", "RODFT10", "RODFT01"]
NS = [16, 32, 64, 128, 256, 512, 1024, 2048]


def real_xy(dims, xperm=None, yperm=(2, 1, 3)):
    """Real x- and y-pencils on one rank, the complex y-pencil (N/2+1 along y) and the complex
    z-pencil of a wall-bounded chain."""
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px = pa.Pencil(topo, dims, (2, 3), permute=pa.Permutation(*xperm) if xperm else None)
    py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(*yperm) if yperm else pa.NoPermutation())
    ay = (yperm or (1, 2, 3))[0] - 1
    pyc = pa.Pencil(py, size_global=tuple(n // 2 + 1 if d == ay else n for d, n in enumerate(dims)))
    return px, py, pyc


def bits(u):
    return u.data.contiguous().view(torch.uint8).reshape(-1)


def r2r_fused_and_plain(po, src, kind, extra=(), **kw):
    """(fused result, plain transpose + r2r_ result, launches of the fused call)."""
    fused = pa.PencilArray.undef(src.dtype, po, *extra)
    bits(fused).fill_(0x5A)
    t = pa.Transposition(fused, src, r2r=kind)
    assert t.fft_fusable()
    n0 = pa.launch_count()
    pa.transpose_(t, **kw)
    torch.cuda.synchronize()
    n = pa.launch_count() - n0
    mid = pa.PencilArray.undef(src.dtype, po, *extra)
    pa.transpose_(pa.Transposition(mid, src), **kw)
    plain = pa.PencilArray.undef(src.dtype, po, *extra)
    pa.r2r_(plain, mid, kind)
    torch.cuda.synchronize()
    return fused, plain, n


def rfft_fused_and_plain(pc, src, cdt, extra=(), **kw):
    """(fused result, plain transpose + rfft_ result, launches of the fused call)."""
    fused = pa.PencilArray.undef(cdt, pc, *extra)
    bits(fused).fill_(0x5A)
    t = pa.Transposition(fused, src, rfft=True)
    assert t.fft_fusable()
    n0 = pa.launch_count()
    pa.transpose_(t, **kw)
    torch.cuda.synchronize()
    n = pa.launch_count() - n0
    mid = pa.PencilArray.undef(src.dtype, t.Po, *extra)  # the real counterpart of pc
    pa.transpose_(pa.Transposition(mid, src), **kw)
    plain = pa.PencilArray.undef(cdt, pc, *extra)
    pa.rfft_(plain, mid)
    torch.cuda.synchronize()
    return fused, plain, n


@pytest.mark.parametrize("prec", PREC)
@pytest.mark.parametrize("N", NS)
def test_bytes_equal_the_unfused_path_one_rank(prec, N):
    """x->y with one rank (transposing gather; 5 and 3 columns, not a multiple of C) and an
    identity plan y->y (linear gather), with and without stage_self, all four kinds and rfft."""
    rdt, cdt, _, _ = PREC[prec]
    px, py, pyc = real_xy((5, N, 3))
    ux = pa.PencilArray.undef(rdt, px)
    ux.data.normal_()
    before = ux.data.clone()
    for kw in (dict(), dict(stage_self=True)):
        for kind in KINDS:
            fused, plain, n = r2r_fused_and_plain(py, ux, kind, **kw)
            assert n == 1
            assert torch.equal(bits(fused), bits(plain)), (N, kind, kw)
        fused, plain, n = rfft_fused_and_plain(pyc, ux, cdt, **kw)
        assert n == 1 and torch.equal(bits(fused), bits(plain)), (N, "rfft", kw)
        assert torch.equal(ux.data.view(torch.uint8), before.view(torch.uint8))  # src untouched
    # identity plan: the real y-pencil array itself (its own pencil object, same geometry)
    uy = pa.PencilArray.undef(rdt, pa.Pencil(py, size_global=py.size_global))
    uy.data.normal_()
    for kind in KINDS:
        fused, plain, n = r2r_fused_and_plain(py, uy, kind)
        assert n == 1 and torch.equal(bits(fused), bits(plain)), (N, kind, "linear")
    fused, plain, n = rfft_fused_and_plain(pyc, uy, cdt)
    assert n == 1 and torch.equal(bits(fused), bits(plain)), (N, "rfft linear")


@pytest.mark.parametrize("prec", PREC)
@pytest.mark.parametrize("dims,xperm,yperm,extra", [
    ((7, 64, 3), (1, 3, 2), (2, 1, 3), ()),
    ((6, 32, 5), None, (2, 3, 1), (3,)),
    ((3, 256, 2), (1, 3, 2), (2, 1, 3), (2, 1, 3)),
    ((3, 16, 2), None, (2, 1, 3), (1, 2, 1, 3, 2)),     # 3 + 5 dims = PA_MAX_DIMS
    ((3, 2048, 1), None, (2, 1, 3), (2, 3)),
])
def test_bytes_equal_with_permutations_and_extra_dims(prec, dims, xperm, yperm, extra):
    rdt, cdt, _, _ = PREC[prec]
    px, py, pyc = real_xy(dims, xperm, yperm)
    ux = pa.PencilArray.undef(rdt, px, *extra)
    ux.data.normal_()
    for kw in (dict(), dict(stage_self=True)):
        for kind in KINDS:
            fused, plain, n = r2r_fused_and_plain(py, ux, kind, extra, **kw)
            assert n == 1 and torch.equal(bits(fused), bits(plain)), (dims, kind, kw)
        fused, plain, n = rfft_fused_and_plain(pyc, ux, cdt, extra, **kw)
        assert n == 1 and torch.equal(bits(fused), bits(plain)), (dims, "rfft", kw)


def test_canaries_around_dst_and_empty_local_arrays():
    rdt, cdt = torch.float64, torch.complex128
    px, py, pyc = real_xy((5, 64, 3))
    ux = pa.PencilArray.undef(rdt, px)
    ux.data.normal_()
    t = pa.Transposition(pa.PencilArray.undef(rdt, py), ux, r2r="REDFT01")
    tc = pa.Transposition(pa.PencilArray.undef(cdt, pyc), ux, rfft=True)
    for nbytes, call, ref in (
            (5 * 64 * 3 * 8,
             lambda d: lib.pa_transpose_r2r(t.plan.h, None, _lib.PA_REDFT01, C.c_void_p(ux.data_ptr()),
                                            d, _lib.PA_WAITALL, stream_ptr()),
             lambda: pa.transpose_(t).Ao),
            (5 * 33 * 3 * 16,
             lambda d: lib.pa_transpose_rfft(tc.plan.h, None, pyc._h, C.c_void_p(ux.data_ptr()), d,
                                             _lib.PA_WAITALL, stream_ptr()),
             lambda: pa.transpose_(tc).Ao)):
        buf = torch.full((nbytes + 512,), 0xA5, dtype=torch.uint8, device="cuda")
        rc = call(C.c_void_p(buf.data_ptr() + 256))
        assert rc == _lib.PA_OK, lib.pa_last_error()
        torch.cuda.synchronize()
        assert bool((buf[:256] == 0xA5).all()) and bool((buf[256 + nbytes:] == 0xA5).all())
        r = ref()
        torch.cuda.synchronize()
        assert torch.equal(buf[256:256 + nbytes], bits(r))
    # empty local arrays: nothing launched
    ex, ey, eyc = real_xy((5, 64, 0))
    eu = pa.PencilArray.undef(rdt, ex)
    n0 = pa.launch_count()
    pa.transpose_(pa.Transposition(pa.PencilArray.undef(rdt, ey), eu, r2r="REDFT10"))
    pa.transpose_(pa.Transposition(pa.PencilArray.undef(cdt, eyc), eu, rfft=True))
    torch.cuda.synchronize()
    assert pa.launch_count() == n0


def test_refusals_launch_nothing_and_leave_dst_untouched():
    rdt, cdt = torch.float64, torch.complex128
    px, py, pyc = real_xy((4, 24, 4))                 # N = 24: refused by the check
    ux = pa.PencilArray.undef(rdt, px)
    ux.data.normal_()
    out = pa.PencilArray.undef(rdt, py)
    outc = pa.PencilArray.undef(cdt, pyc)
    bits(out).fill_(0x3C)
    bits(outc).fill_(0x3C)
    torch.cuda.synchronize()
    before, beforec = out.data.clone(), outc.data.clone()
    t = pa.Transposition(out, ux, r2r="REDFT10")
    tc = pa.Transposition(outc, ux, rfft=True)
    assert not t.fft_fusable() and not tc.fft_fusable()
    n0 = pa.launch_count()
    with pytest.raises(pa.ArgumentError):
        pa.transpose_(t)
    with pytest.raises(pa.ArgumentError):
        pa.transpose_(tc)
    # bad kinds / flags / precision / overlap through the ABI, on device pointers
    gx, gy, gyc = real_xy((4, 32, 4))
    gu = pa.PencilArray.undef(rdt, gx)
    go = pa.PencilArray.undef(rdt, gy)
    bits(go).fill_(0x3C)
    gbefore = go.data.clone()
    gt = pa.Transposition(go, gu, r2r="REDFT10")
    h, st = gt.plan.h, stream_ptr()
    gs, gd = C.c_void_p(gu.data_ptr()), C.c_void_p(go.data_ptr())
    for kind in (0, 3, 6, 10, -1):
        assert lib.pa_transpose_r2r(h, None, kind, gs, gd, 0, st) == _lib.PA_EINVAL
    for flags in (_lib.PA_FFT_FORWARD, _lib.PA_FFT_F32, 64):
        assert lib.pa_transpose_r2r(h, None, _lib.PA_REDFT10, gs, gd, flags, st) == _lib.PA_EINVAL
        assert lib.pa_transpose_rfft(h, None, gyc._h, gs, gd, flags, st) == _lib.PA_EINVAL
    assert lib.pa_transpose_r2r(h, None, _lib.PA_REDFT10, gs, gs, 0, st) == _lib.PA_EINVAL  # overlap
    assert lib.pa_transpose_rfft(h, None, gy._h, gs, gd, 0, st) == _lib.PA_EINCOMPAT
    assert lib.pa_transpose_r2r(t.plan.h, None, _lib.PA_REDFT10, C.c_void_p(ux.data_ptr()),
                                C.c_void_p(out.data_ptr()), 0, st) == _lib.PA_EINVAL
    torch.cuda.synchronize()
    assert pa.launch_count() == n0
    assert torch.equal(out.data.view(torch.uint8), before.view(torch.uint8))
    assert torch.equal(outc.data.view(torch.uint8), beforec.view(torch.uint8))
    assert torch.equal(go.data.view(torch.uint8), gbefore.view(torch.uint8))


def chain_pencils(dims):
    """x (real), y (real), y (complex, N/2+1 along y) and z (complex) pencils on one rank."""
    px, py, pyc = real_xy(dims)
    pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    pz = pa.Pencil(py, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    return px, py, pyc, pzc, pz


@pytest.mark.parametrize("prec", PREC)
@pytest.mark.parametrize("dims", [(16, 32, 8), (64, 64, 64), (32, 16, 128)])
def test_mixed_chain_is_three_kernels_each_way(prec, dims):
    """DCT-II along x, RFFT along y, FFT along z: r2r_, fused x->y + rfft, fused y->z + FFT; then
    fft_, fused z->y + brfft, fused y->x + DCT-III.  Byte-equal to the unfused chain, within
    8 eps log2(n) of scipy / numpy."""
    rdt, cdt, eps, _ = PREC[prec]
    px, py, pyc, pzc, _ = chain_pencils(dims)
    n = math.prod(dims)
    ux = pa.PencilArray.undef(rdt, px)
    ux.data.normal_()
    G = ux.logical().cpu().numpy().astype(np.float64)
    F = np.fft.fft(np.fft.rfft(sf.dct(G, 2, axis=0), axis=1), axis=2)
    u1 = pa.PencilArray.undef(rdt, px)
    uyc, uzc = pa.PencilArray.undef(cdt, pyc), pa.PencilArray.undef(cdt, pzc)
    t_xy = pa.Transposition(uyc, u1, rfft=True)
    t_yz = pa.Transposition(uzc, uyc)
    back_y = pa.PencilArray.undef(rdt, py)
    back = pa.PencilArray.undef(rdt, px)
    t_zy = pa.Transposition(back_y, uzc, brfft=True)
    t_yx = pa.Transposition(back, back_y, r2r="REDFT01")
    torch.cuda.synchronize()
    n0 = pa.launch_count()
    pa.r2r_(u1, ux, "REDFT10")
    pa.transpose_(t_xy)
    pa.transpose_(t_yz, fft="forward")
    torch.cuda.synchronize()
    assert pa.launch_count() - n0 == 3
    got = uzc.logical().cpu().numpy()
    assert np.abs(got - F).max() <= 8 * eps * np.log2(n) * np.abs(F).max()
    fwd_bits = bits(uzc).clone()
    n0 = pa.launch_count()
    pa.fft_(uzc, "backward")
    pa.transpose_(t_zy)
    pa.transpose_(t_yx)
    torch.cuda.synchronize()
    assert pa.launch_count() - n0 == 3
    err = np.abs(back.logical().cpu().numpy().astype(np.float64) - 2 * n * G).max()
    assert err <= 8 * eps * np.log2(n) * 2 * n * np.abs(G).max(), err

    # the unfused chains: 4 kernels forward, 5 backward
    v1, vy = pa.PencilArray.undef(rdt, px), pa.PencilArray.undef(rdt, py)
    vyc, vzc = pa.PencilArray.undef(cdt, pyc), pa.PencilArray.undef(cdt, pzc)
    pa.r2r_(v1, ux, "REDFT10")
    pa.transpose_(pa.Transposition(vy, v1))
    pa.rfft_(vyc, vy)
    pa.transpose_(pa.Transposition(vzc, vyc), fft="forward")
    torch.cuda.synchronize()
    assert torch.equal(bits(vzc), fwd_bits)
    pa.fft_(vzc, "backward")
    pa.transpose_(pa.Transposition(vyc, vzc))
    pa.brfft_(vy, vyc)
    vx = pa.PencilArray.undef(rdt, px)
    pa.transpose_(pa.Transposition(vx, vy))
    pa.r2r_(vx, vx, "REDFT01")
    torch.cuda.synchronize()
    assert torch.equal(bits(vx), bits(back))


@pytest.mark.parametrize("prec", PREC)
@pytest.mark.parametrize("dims", [(16, 32, 16), (64, 64, 64), (32, 16, 128)])
def test_all_walls_chain_is_three_kernels_each_way(prec, dims):
    """DCT-II along x, y and z: r2r_, fused x->y + DCT-II, fused y->z + DCT-II; then r2r_
    DCT-III, fused z->y + DCT-III, fused y->x + DCT-III.  Byte-equal to the unfused chain, within
    8 eps log2(n) of scipy.fft.dctn."""
    rdt, _, eps, _ = PREC[prec]
    px, py, _, _, pz = chain_pencils(dims)
    n = math.prod(dims)
    ux = pa.PencilArray.undef(rdt, px)
    ux.data.normal_()
    G = ux.logical().cpu().numpy().astype(np.float64)
    F = sf.dctn(G, 2)
    u1, uy, uz = (pa.PencilArray.undef(rdt, p) for p in (px, py, pz))
    t_xy = pa.Transposition(uy, u1, r2r="REDFT10")
    t_yz = pa.Transposition(uz, uy, r2r="REDFT10")
    wz, wy, wx = (pa.PencilArray.undef(rdt, p) for p in (pz, py, px))
    t_zy = pa.Transposition(wy, wz, r2r="REDFT01")
    t_yx = pa.Transposition(wx, wy, r2r="REDFT01")
    torch.cuda.synchronize()
    n0 = pa.launch_count()
    pa.r2r_(u1, ux, "REDFT10")
    pa.transpose_(t_xy)
    pa.transpose_(t_yz)
    torch.cuda.synchronize()
    assert pa.launch_count() - n0 == 3
    got = uz.logical().cpu().numpy().astype(np.float64)
    assert np.abs(got - F).max() <= 8 * eps * np.log2(n) * np.abs(F).max()
    n0 = pa.launch_count()
    pa.r2r_(wz, uz, "REDFT01")
    pa.transpose_(t_zy)
    pa.transpose_(t_yx)
    torch.cuda.synchronize()
    assert pa.launch_count() - n0 == 3
    scale = 8 * n
    err = np.abs(wx.logical().cpu().numpy().astype(np.float64) - scale * G).max()
    assert err <= 8 * eps * np.log2(n) * scale * np.abs(G).max(), err

    # the unfused chains: 5 kernels each way
    v = [pa.PencilArray.undef(rdt, p) for p in (px, py, py, pz, pz)]
    pa.r2r_(v[0], ux, "REDFT10")
    pa.transpose_(pa.Transposition(v[1], v[0]))
    pa.r2r_(v[2], v[1], "REDFT10")
    pa.transpose_(pa.Transposition(v[3], v[2]))
    pa.r2r_(v[4], v[3], "REDFT10")
    torch.cuda.synchronize()
    assert torch.equal(bits(v[4]), bits(uz))
    b = [pa.PencilArray.undef(rdt, p) for p in (pz, py, py, px, px)]
    pa.r2r_(b[0], v[4], "REDFT01")
    pa.transpose_(pa.Transposition(b[1], b[0]))
    pa.r2r_(b[2], b[1], "REDFT01")
    pa.transpose_(pa.Transposition(b[3], b[2]))
    pa.r2r_(b[4], b[3], "REDFT01")
    torch.cuda.synchronize()
    assert torch.equal(bits(b[4]), bits(wx))


@pytest.mark.parametrize("mode", ["r2r", "rfft"])
def test_ordered_on_a_held_caller_stream(mode):
    """On a side stream held by a spin, the call returns before the spin ends, and its result
    (produced behind the hold) equals the default-stream result byte for byte."""
    rdt, cdt = torch.float64, torch.complex128
    px, py, pyc = real_xy((16, 512, 8))
    ux = pa.PencilArray.undef(rdt, px)
    ux.data.normal_()
    po, dt, kw = (py, rdt, dict(r2r="RODFT10")) if mode == "r2r" else (pyc, cdt, dict(rfft=True))
    ref = pa.PencilArray.undef(dt, po)
    pa.transpose_(pa.Transposition(ref, ux, **kw))
    torch.cuda.synchronize()
    out = pa.PencilArray.undef(dt, po)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        held = hold()
        ux2 = ux.data.clone()      # the input, produced behind the hold
        src = pa.PencilArray(px, ux2)
        pa.transpose_(pa.Transposition(out, src, **kw))
        assert not held.query()
    side.synchronize()
    assert torch.equal(bits(out), bits(ref))


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_ranks_sharing_the_gpu(world, tmp_path):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29931 + world),
           os.path.join(HERE, "mp_fused_real_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1", PA_TEST_TMPDIR=str(tmp_path))
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    assert f"MP_FUSED_REAL_OK world={world}" in out.stdout, out.stdout[-2000:]
