"""The one-sided fused transpose + FFT (PeerGet, DESIGN §3h) on the GPU.

Single process: a grid line of ranks emulated as separate device tensors.  `pa_get_all_fft` of
every rank -- remote blocks read straight out of the other ranks' src tensors, the self block out
of its own -- must equal, byte for byte, `fft_` of the transposed array (pack / exchange / unpack
through the C ABI, itself checked against the global array).  Canary bytes around dst stay, every
src stays, and a refused geometry launches nothing.

Processes sharing the GPU over the NCCL-free communicator (tests/mp_fft_peerget_worker.py): the
whole `transpose_(t, fft=...)` with PeerGet against PointToPoint, the 3-d FFT against numpy, the
caller-stream ordering, and PeerPut's refusal."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200 import _lib
from pencilarrays_b200._lib import lib
from pencilarrays_b200.transpositions import _Plan
from gpu_util import emulate_transpose_gpu, stream_ptr
from util import make_ranks

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
FWD, BWD, F32 = _lib.PA_FFT_FORWARD, _lib.PA_FFT_BACKWARD, _lib.PA_FFT_F32
PAD = 256  # canary bytes on either side of dst


def local(A, p):
    return A[tuple(slice(r.start - 1, r.stop - 1) for r in pa.range_local(p))]


def make_line(grid, dims, sdec, extra=(), sperm=(2, 1, 3), dperm=None, dtype=torch.complex128):
    """Source pencils decomposed along sdec (x among them), destination pencils with x local and
    contiguous; the PeerGet plan, src array (loaded from one global field) and the transposed
    array (emulated exchange) of every rank."""
    ddec = tuple(2 if d == 1 else d for d in sdec)
    es = 16 if dtype == torch.complex128 else 8
    rng = np.random.default_rng(hash((grid, dims, sdec, extra)) % 2**32)
    G = (rng.standard_normal(dims + extra) + 1j * rng.standard_normal(dims + extra)).astype(
        np.complex128 if es == 16 else np.complex64)
    plans, srcs, plains = [], [], []
    for er in make_ranks(grid):
        ps = pa.Pencil(er.topo, dims, sdec, permute=pa.Permutation(*sperm) if sperm else None)
        pd = pa.Pencil(ps, decomp_dims=ddec, permute=pa.Permutation(*dperm) if dperm else pa.NoPermutation())
        plans.append(_Plan(ps, pd, extra, es, pa.PeerGet()))
        u = pa.PencilArray.undef(dtype, ps, *extra)
        u.logical().copy_(torch.from_numpy(np.ascontiguousarray(local(G, ps))))
        srcs.append(u)
        plains.append(pa.PencilArray.undef(dtype, pd, *extra))
    emulate_transpose_gpu(plans, [u.data for u in srcs], [v.data for v in plains])
    torch.cuda.synchronize()
    for v in plains:
        want = np.ascontiguousarray(local(G, v.pencil))
        assert v.logical().cpu().numpy().tobytes() == want.tobytes(), "emulated transpose"
    return plans, srcs, plains


def get_all_fft(plan, srcs, r, dst_ptr, flags):
    info = plan.info
    peers = [srcs[plan.peer(n).world_rank].data_ptr() or None for n in range(1, info.nproc + 1)]
    arr = (C.c_void_p * info.nproc)(*peers)
    return lib.pa_get_all_fft(plan.h, C.c_void_p(srcs[r].data_ptr() or None), arr,
                              C.c_void_p(dst_ptr), flags, stream_ptr())


def check_line(grid, dims, sdec, directions=("forward", "backward"), **kw):
    plans, srcs, plains = make_line(grid, dims, sdec, **kw)
    before = [u.data.clone() for u in srcs]
    prec = F32 if srcs[0].dtype == torch.complex64 else 0
    for r, (plan, plain) in enumerate(zip(plans, plains)):
        assert lib.pa_plan_fft_check_ex(plan.h, prec) == _lib.PA_OK, lib.pa_last_error()
        nout = plain.data.numel() * plain.elsize
        for direction in directions:
            ref = pa.PencilArray(plain.pencil, plain.data.clone(), plain.extra_dims)
            pa.fft_(ref, direction)
            raw = torch.full((nout + 2 * PAD,), 0x5A, dtype=torch.uint8, device="cuda")
            flags = (FWD if direction == "forward" else BWD) | prec
            st = get_all_fft(plan, srcs, r, raw.data_ptr() + PAD if nout else 0, flags)
            assert st == _lib.PA_OK, lib.pa_last_error()
            torch.cuda.synchronize()
            got = raw[PAD:PAD + nout]
            assert torch.equal(got, ref.data.reshape(-1).view(torch.uint8)), (grid, dims, r, direction, kw)
            assert bool((raw[:PAD] == 0x5A).all()) and bool((raw[PAD + nout:] == 0x5A).all()), "canary"
    for u, b in zip(srcs, before):
        assert torch.equal(u.data, b), "a src array changed"


@pytest.mark.parametrize("grid,dims,sdec", [
    ((2,), (16, 6, 3), (1,)),          # 2 blocks
    ((3,), (64, 7, 2), (1,)),          # 64/3 = 21/21/22
    ((5,), (8, 4, 3), (1,)),           # 8/5 = 1,2,1,2,2; y = 4 < 5: an empty destination
    ((6,), (1024, 7, 2), (1,)),        # 1024/6
    ((8,), (8, 9, 2), (1,)),           # one row per block
    ((8,), (64, 5, 3), (1,)),          # y = 5 < 8: three empty destinations
    ((3, 2), (64, 6, 4), (1, 3)),      # lines of 3 ranks in a 2-d grid
], ids=["2", "3_64", "5_8", "6_1024", "8_rows", "8_empty", "3x2"])
def test_blocks_per_line(grid, dims, sdec):
    check_line(grid, dims, sdec)


@pytest.mark.parametrize("kw", [
    dict(dims=(32, 13, 3)),                                     # partial tiles (13 columns)
    dict(dims=(16, 5, 3), extra=(2, 1, 1, 1, 2)),               # 3 + 5 = PA_MAX_DIMS dims
    dict(dims=(64, 6, 5), sperm=(3, 2, 1)),                     # z contiguous in the source
    dict(dims=(64, 6, 5), sperm=(3, 1, 2), dperm=(1, 3, 2)),
    dict(dims=(128, 6, 5), sperm=(2, 3, 1), dperm=(1, 3, 2)),
    dict(dims=(256, 9, 2), dtype=torch.complex64, extra=(3,)),
], ids=["partial", "max_dims", "src_zyx", "src_zxy", "perms", "f32_extra"])
def test_layouts(kw):
    dims = kw.pop("dims")
    check_line((3,), dims, (1,), **kw)


@pytest.mark.parametrize("dtype", [torch.complex128, torch.complex64], ids=["c128", "c64"])
@pytest.mark.parametrize("lines", [4, 0], ids=["lines4", "lines_default"])
@pytest.mark.parametrize("L", [8, 16, 32, 64, 128, 256, 512, 1024])
def test_every_line_length(L, lines, dtype):
    pa.set_tunable("fft_lines", lines)
    try:
        check_line((3,), (L, 11, 2), (1,), dtype=dtype)
    finally:
        pa.set_tunable("fft_lines", 0)


def test_refused_geometry_launches_nothing():
    for dims, prec, dtype in (((48, 5, 2), 0, torch.complex128), ((2048, 3, 2), F32, torch.complex64)):
        ranks = make_ranks((3,))
        plans, srcs = [], []
        for er in ranks:
            ps = pa.Pencil(er.topo, dims, (1,), permute=pa.Permutation(2, 1, 3))
            pd = pa.Pencil(ps, decomp_dims=(2,), permute=pa.NoPermutation())
            plans.append(_Plan(ps, pd, (), 16 if prec == 0 else 8, pa.PeerGet()))
            srcs.append(pa.PencilArray.undef(dtype, ps))
        for r, plan in enumerate(plans):
            n = plan.info.length_out * plan.info.elsize
            raw = torch.full((n + 2 * PAD,), 0x3C, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            n0 = pa.launch_count()
            assert get_all_fft(plan, srcs, r, raw.data_ptr() + PAD, FWD | prec) == _lib.PA_EINVAL
            assert pa.launch_count() == n0
            torch.cuda.synchronize()
            assert bool((raw == 0x3C).all())


@pytest.mark.parametrize("world", [2, 3, 4, 5, 6, 8])
def test_peerget_fused_transpose_across_processes(world, tmp_path):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29971 + world),
           os.path.join(HERE, "mp_fft_peerget_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1", PA_TEST_TMPDIR=str(tmp_path))
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    assert f"MP_FFT_PEERGET_OK world={world}" in out.stdout, out.stdout[-2000:]
