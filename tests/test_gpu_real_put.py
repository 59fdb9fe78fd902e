"""The send-side fused real line transforms + put (PeerPut, DESIGN §3j) on the GPU.

Single process: a grid line of ranks emulated as separate device tensors.  `pa_put_all_r2r` of
every rank must leave, byte for byte, what `r2r_` on a copy of src followed by the plain
transposition leaves; `pa_put_all_brfft` what `brfft_` followed by the transposition of the reals
leaves.  The blocks split a line at any real (N = 32 over 3 ranks: 11 / 11 / 10).  Canary bytes
around every dst stay, every src stays, and a refused call launches nothing.

Processes sharing the GPU over the NCCL-free communicator (tests/mp_real_put_worker.py): the whole
`r2r_first=` / `brfft_first=True` schedule against the unfused PeerPut pair, and the mixed and
all-walls 3-d chains against scipy / numpy and against the PointToPoint chains that fuse on the
receive side."""
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
from pencilarrays_b200.transpositions import _Plan, _brfft_pencil
from gpu_util import emulate_transpose_gpu, hold, stream_ptr
from util import make_ranks

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
F32 = _lib.PA_FFT_F32
PAD = 256  # canary bytes on either side of every dst
KINDS = ["REDFT10", "REDFT01", "RODFT10", "RODFT01"]
CPLX_OF = {torch.float64: torch.complex128, torch.float32: torch.complex64}


def local(A, p):
    return A[tuple(slice(r.start - 1, r.stop - 1) for r in pa.range_local(p))]


def make_line(grid, dims, sdec, mode, extra=(), sperm=None, dperm=(2, 1, 3), dtype=torch.float64):
    """Real source pencils with x local and first in memory (decomposed along sdec), destination
    pencils decomposed along x in place of y, the PeerPut real plan; the src arrays (real for an
    r2r kind, the complex counterpart for mode "c2r") and per rank the array the reference
    transform writes and the reference dst."""
    ddec = tuple(1 if d == 2 else d for d in sdec)
    es = 8 if dtype == torch.float64 else 4
    rng = np.random.default_rng(hash((grid, dims, sdec, extra, mode)) % 2**32)
    plans, srcs, cplx, refs = [], [], [], []
    for er in make_ranks(grid):
        ps = pa.Pencil(er.topo, dims, sdec, permute=pa.Permutation(*sperm) if sperm else None)
        pd = pa.Pencil(ps, decomp_dims=ddec, permute=pa.Permutation(*dperm) if dperm else pa.NoPermutation())
        plans.append(_Plan(ps, pd, extra, es, pa.PeerPut()))
        if mode == "c2r":
            pc = _brfft_pencil(ps)
            u = pa.PencilArray.undef(CPLX_OF[dtype], pc, *extra)
            cplx.append(pc)
        else:
            u = pa.PencilArray.undef(dtype, ps, *extra)
        v = torch.from_numpy(rng.standard_normal(tuple(u.data.shape)))
        if mode == "c2r":
            v = v + 1j * torch.from_numpy(rng.standard_normal(tuple(u.data.shape)))
        u.data.copy_(v.to(u.data.dtype))
        srcs.append(u)
        refs.append((pa.PencilArray.undef(dtype, ps, *extra), pa.PencilArray.undef(dtype, pd, *extra)))
    return plans, srcs, cplx, refs


def reference(plans, srcs, refs, mode):
    for u, (t, _) in zip(srcs, refs):
        if mode == "c2r":
            pa.brfft_(t, u)
        else:
            t.data.copy_(u.data)
            pa.r2r_(t, t, mode)
    emulate_transpose_gpu(plans, [t.data for t, _ in refs], [v.data for _, v in refs])
    torch.cuda.synchronize()
    return [v.data.reshape(-1).view(torch.uint8).clone() for _, v in refs]


def put_all(plan, cplx, srcs, dsts, r, flags, mode):
    info = plan.info
    peers = [dsts[plan.peer(n).world_rank] or None for n in range(1, info.nproc + 1)]
    arr = (C.c_void_p * info.nproc)(*peers)
    src = C.c_void_p(srcs[r].data_ptr() or None)
    if mode == "c2r":
        return lib.pa_put_all_brfft(plan.h, cplx[r]._h, src, arr, C.c_void_p(dsts[r] or None), flags,
                                    stream_ptr())
    return lib.pa_put_all_r2r(plan.h, getattr(_lib, "PA_" + mode), src, arr, C.c_void_p(dsts[r] or None),
                              flags, stream_ptr())


def check_line(grid, dims, sdec, modes=tuple(KINDS) + ("c2r",), **kw):
    prec = F32 if kw.get("dtype") == torch.float32 else 0
    for mode in modes:
        plans, srcs, cplx, refs = make_line(grid, dims, sdec, mode, **kw)
        before = [u.data.clone() for u in srcs]
        for plan in plans:
            assert lib.pa_plan_real_put_check(plan.h, prec) == _lib.PA_OK, lib.pa_last_error()
        want = reference(plans, srcs, refs, mode)
        raws = [torch.full((w.numel() + 2 * PAD,), 0x5A, dtype=torch.uint8, device="cuda") for w in want]
        dsts = [raw.data_ptr() + PAD if w.numel() else 0 for raw, w in zip(raws, want)]
        for r, plan in enumerate(plans):
            assert put_all(plan, cplx, srcs, dsts, r, prec, mode) == _lib.PA_OK, lib.pa_last_error()
        torch.cuda.synchronize()
        for r, (raw, w) in enumerate(zip(raws, want)):
            n = w.numel()
            assert torch.equal(raw[PAD:PAD + n], w), (grid, dims, r, mode, kw)
            assert bool((raw[:PAD] == 0x5A).all()) and bool((raw[PAD + n:] == 0x5A).all()), "canary"
        for u, b in zip(srcs, before):
            assert torch.equal(u.data, b), "a src array changed"


LINES = [
    ((2,), (16, 6, 3), (2,)),          # 2 blocks
    ((3,), (32, 7, 2), (2,)),          # 32/3 = 11/11/10: odd block boundaries
    ((5,), (16, 4, 3), (2,)),          # 16/5; y = 4 < 5: a rank without source lines
    ((6,), (2048, 7, 2), (2,)),        # 2048/6
    ((8,), (16, 8, 2), (2,)),          # 2 reals per block, one source row per rank
    ((8,), (64, 5, 3), (2,)),          # y = 5 < 8: three ranks without source lines
    ((3, 2), (64, 6, 4), (2, 3)),      # lines of 3 ranks in a 2-d grid
]
LINE_IDS = ["2", "3_odd", "5_empty", "6_2048", "8_rows", "8_empty", "3x2"]


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("grid,dims,sdec", LINES, ids=LINE_IDS)
def test_blocks_per_line(grid, dims, sdec, dtype):
    check_line(grid, dims, sdec, dtype=dtype)


@pytest.mark.parametrize("kw", [
    dict(dims=(32, 13, 3)),                                     # partial tiles (13 columns)
    dict(dims=(16, 5, 3), extra=(2, 1, 1, 1, 2)),               # 3 + 5 = PA_MAX_DIMS dims
    dict(dims=(64, 6, 5), dperm=None),                          # unpermuted: stores along the line
    dict(dims=(64, 6, 5), dperm=(3, 1, 2)),                     # z contiguous in the destination
    dict(dims=(128, 6, 5), sperm=(1, 3, 2), dperm=(2, 3, 1)),
    dict(dims=(256, 9, 2), dtype=torch.float32, extra=(3,)),
    dict(dims=(32, 9, 2), dtype=torch.float32, dperm=None),
], ids=["partial", "max_dims", "unpermuted", "dst_zxy", "perms", "f32_extra", "f32_unpermuted"])
def test_layouts(kw):
    kw = dict(kw)
    dims = kw.pop("dims")
    check_line((3,), dims, (2,), **kw)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("N", [16, 32, 64, 128, 256, 512, 1024, 2048])
def test_every_line_length(N, dtype):
    check_line((3,), (N, 11, 2), (2,), dtype=dtype)


@pytest.mark.parametrize("mode", ["REDFT01", "RODFT10", "c2r"])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
def test_local_plans_one_kernel_on_the_caller_stream(dtype, mode):
    """One-rank lines and plans without an exchange, any method: `r2r_first=` / `brfft_first=True`
    is one kernel, ordered behind a held caller stream, equal to the pair."""
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    dims = (128, 12, 6)
    rng = np.random.default_rng(11)
    for method in (pa.PointToPoint(), pa.PeerGet(), pa.PeerPut()):
        ps = pa.Pencil(topo, dims, (2, 3))
        for pd in (pa.Pencil(ps, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3)),
                   pa.Pencil(ps, decomp_dims=(2, 3), permute=pa.Permutation(3, 2, 1))):
            side = torch.cuda.Stream()
            with torch.cuda.stream(side):
                out = pa.PencilArray.undef(dtype, pd)
                want = pa.PencilArray.undef(dtype, pd)
                mid = pa.PencilArray.undef(dtype, ps)
                if mode == "c2r":
                    u = pa.PencilArray.undef(CPLX_OF[dtype], _brfft_pencil(ps))
                    t = pa.Transposition(out, u, method=method, brfft_first=True)
                    val = torch.from_numpy(rng.standard_normal(u.data.shape) +
                                           1j * rng.standard_normal(u.data.shape)).to(u.data.dtype)
                else:
                    u = pa.PencilArray.undef(dtype, ps)
                    t = pa.Transposition(out, u, method=method, r2r_first=mode)
                    val = torch.from_numpy(rng.standard_normal(u.data.shape)).to(dtype)
                assert t.fft_first_fusable()
                # (on the device before the hold: a pageable upload behind it would block the host)
                val = val.cuda()
                # (the first call on a plan creates its streams and events, which synchronises the
                #  device: done here, before the hold)
                pa.transpose_(t)
                torch.cuda.synchronize()
                out.data.fill_(0)
                held = hold()
                u.data.copy_(val)  # behind the hold
                n0 = pa.launch_count()
                pa.transpose_(t)
                assert pa.launch_count() - n0 == 1
                assert not held.query()
                if mode == "c2r":
                    pa.brfft_(mid, u)
                else:
                    pa.r2r_(mid, u, mode)
                pa.transpose_(want, mid, method=method)
                torch.cuda.current_stream().synchronize()
                assert torch.equal(out.data.view(torch.uint8), want.data.view(torch.uint8)), (method, pd.perm)


def test_refusals_launch_nothing():
    plans, srcs, cplx = [], [], []
    for er in make_ranks((3,)):
        ps = pa.Pencil(er.topo, (48, 5, 2), (2,))  # 48 reals is no power of two
        pd = pa.Pencil(ps, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
        plans.append(_Plan(ps, pd, (), 8, pa.PeerPut()))
        srcs.append(pa.PencilArray.undef(torch.float64, ps))
        cplx.append(_brfft_pencil(ps))
    for mode in ("REDFT10", "c2r"):
        for r, plan in enumerate(plans):
            n = plan.info.length_out * plan.info.elsize
            raw = torch.full((n + 2 * PAD,), 0x3C, dtype=torch.uint8, device="cuda")
            dsts = [raw.data_ptr() + PAD] * 3
            torch.cuda.synchronize()
            n0 = pa.launch_count()
            assert put_all(plan, cplx, srcs, dsts, r, 0, mode) == _lib.PA_EINVAL
            assert lib.pa_r2r_put(plan.h, None, _lib.PA_REDFT10, C.c_void_p(srcs[r].data_ptr()),
                                  C.c_void_p(dsts[0]), 0, stream_ptr()) == _lib.PA_EINVAL
            assert pa.launch_count() == n0
            torch.cuda.synchronize()
            assert bool((raw == 0x3C).all())
    # a PointToPoint transposition with an exchange: refused when built, before any launch
    er = make_ranks((2,))[0]
    ps = pa.Pencil(er.topo, (32, 4, 3), (2,))
    pd = pa.Pencil(ps, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
    u, v = pa.PencilArray.undef(torch.float64, ps), pa.PencilArray.undef(torch.float64, pd)
    n0 = pa.launch_count()
    with pytest.raises(pa.ArgumentError, match="receive side"):
        pa.Transposition(v, u, method=pa.PointToPoint(), r2r_first="REDFT10")
    assert pa.launch_count() == n0


@pytest.mark.parametrize("world", [2, 3, 4, 6, 8])
def test_real_put_across_processes(world, tmp_path):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29961 + world),
           os.path.join(HERE, "mp_real_put_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1", PA_TEST_TMPDIR=str(tmp_path))
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    assert f"MP_REAL_PUT_OK world={world}" in out.stdout, out.stdout[-2000:]
