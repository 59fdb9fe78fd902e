"""The send-side fused transform + put (PeerPut, DESIGN §3i) on the GPU.

Single process: a grid line of ranks emulated as separate device tensors.  `pa_put_all_fft` of
every rank -- its own bins stored into its dst, every other block straight into the other ranks'
dst tensors -- must leave, byte for byte, what `fft_` on a copy of src followed by the plain
transposition leaves (pack / exchange / unpack through the C ABI); `pa_put_all_rfft` what `rfft_`
followed by the transposition of the complex array leaves.  Canary bytes around every dst stay,
every src stays, and a refused call launches nothing.

Processes sharing the GPU over the NCCL-free communicator (tests/mp_fft_put_worker.py): the
whole `transpose_(t, fft_first=...)` / `rfft_first=True` schedule against the unfused PeerPut
pair, and the 3-d chains against numpy and against the PointToPoint `fft=` chains."""
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
FWD, BWD, F32 = _lib.PA_FFT_FORWARD, _lib.PA_FFT_BACKWARD, _lib.PA_FFT_F32
PAD = 256  # canary bytes on either side of every dst
REAL_OF = {torch.complex128: torch.float64, torch.complex64: torch.float32}


def local(A, p):
    return A[tuple(slice(r.start - 1, r.stop - 1) for r in pa.range_local(p))]


def make_line(grid, dims, sdec, extra=(), sperm=None, dperm=(2, 1, 3), dtype=torch.complex128,
              rfft=False):
    """Source pencils with x local and first in memory (decomposed along sdec), destination pencils
    decomposed along x in place of y; the PeerPut plan, the src arrays (one global field) and the
    reference dst of every rank: fft_ (rfft_) of src, then the emulated plain transposition."""
    ddec = tuple(1 if d == 2 else d for d in sdec)
    es = 16 if dtype == torch.complex128 else 8
    rng = np.random.default_rng(hash((grid, dims, sdec, extra, rfft)) % 2**32)
    if rfft:
        G = rng.standard_normal(dims + extra).astype(np.float64 if es == 16 else np.float32)
    else:
        G = (rng.standard_normal(dims + extra) + 1j * rng.standard_normal(dims + extra)).astype(
            np.complex128 if es == 16 else np.complex64)
    plans, srcs, reals, refs = [], [], [], []
    for er in make_ranks(grid):
        ps = pa.Pencil(er.topo, dims, sdec, permute=pa.Permutation(*sperm) if sperm else None)
        u = pa.PencilArray.undef(REAL_OF[dtype] if rfft else dtype, ps, *extra)
        u.logical().copy_(torch.from_numpy(np.ascontiguousarray(local(G, ps))))
        srcs.append(u)
        pc = _brfft_pencil(ps) if rfft else ps  # the plan's input pencil (rfft: N/2+1 bins)
        pd = pa.Pencil(pc, decomp_dims=ddec, permute=pa.Permutation(*dperm) if dperm else pa.NoPermutation())
        plans.append(_Plan(pc, pd, extra, es, pa.PeerPut()))
        reals.append(ps)
        t = pa.PencilArray.undef(dtype, pc, *extra)
        if rfft:
            pa.rfft_(t, u)
        else:
            t.data.copy_(u.data)
            pa.fft_(t, "forward")
        refs.append((t, pa.PencilArray.undef(dtype, pd, *extra)))
    return plans, srcs, reals, refs, G


def reference(plans, srcs, refs, direction, rfft):
    for u, (t, _) in zip(srcs, refs):
        if rfft:
            pa.rfft_(t, u)
        else:
            t.data.copy_(u.data)
            pa.fft_(t, direction)
    emulate_transpose_gpu(plans, [t.data for t, _ in refs], [v.data for _, v in refs])
    torch.cuda.synchronize()
    return [v.data.reshape(-1).view(torch.uint8).clone() for _, v in refs]


def put_all(plan, reals, srcs, dsts, r, flags, rfft):
    info = plan.info
    peers = [dsts[plan.peer(n).world_rank] or None for n in range(1, info.nproc + 1)]
    arr = (C.c_void_p * info.nproc)(*peers)
    src = C.c_void_p(srcs[r].data_ptr() or None)
    if rfft:
        return lib.pa_put_all_rfft(plan.h, reals[r]._h, src, arr, C.c_void_p(dsts[r] or None), flags,
                                   stream_ptr())
    return lib.pa_put_all_fft(plan.h, src, arr, C.c_void_p(dsts[r] or None), flags, stream_ptr())


def check_line(grid, dims, sdec, directions=("forward", "backward"), rfft=False, **kw):
    plans, srcs, reals, refs, _ = make_line(grid, dims, sdec, rfft=rfft, **kw)
    before = [u.data.clone() for u in srcs]
    prec = F32 if kw.get("dtype") == torch.complex64 else 0
    check_fn = lib.pa_plan_rfft_put_check if rfft else lib.pa_plan_fft_put_check
    for plan in plans:
        assert check_fn(plan.h, prec) == _lib.PA_OK, lib.pa_last_error()
    for direction in (("forward",) if rfft else directions):
        want = reference(plans, srcs, refs, direction, rfft)
        raws = [torch.full((w.numel() + 2 * PAD,), 0x5A, dtype=torch.uint8, device="cuda") for w in want]
        dsts = [raw.data_ptr() + PAD if w.numel() else 0 for raw, w in zip(raws, want)]
        flags = (0 if rfft else (FWD if direction == "forward" else BWD)) | prec
        for r, plan in enumerate(plans):
            assert put_all(plan, reals, srcs, dsts, r, flags, rfft) == _lib.PA_OK, lib.pa_last_error()
        torch.cuda.synchronize()
        for r, (raw, w) in enumerate(zip(raws, want)):
            n = w.numel()
            assert torch.equal(raw[PAD:PAD + n], w), (grid, dims, r, direction, rfft, kw)
            assert bool((raw[:PAD] == 0x5A).all()) and bool((raw[PAD + n:] == 0x5A).all()), "canary"
    for u, b in zip(srcs, before):
        assert torch.equal(u.data, b), "a src array changed"


LINES = [
    ((2,), (16, 6, 3), (2,)),          # 2 blocks
    ((3,), (64, 7, 2), (2,)),          # 64/3 = 21/21/22
    ((5,), (8, 4, 3), (2,)),           # 8/5 = 1,2,1,2,2; y = 4 < 5: a rank without source lines
    ((6,), (1024, 7, 2), (2,)),        # 1024/6
    ((8,), (8, 9, 2), (2,)),           # one row per block
    ((8,), (64, 5, 3), (2,)),          # y = 5 < 8: three ranks without source lines
    ((3, 2), (64, 6, 4), (2, 3)),      # lines of 3 ranks in a 2-d grid
]
LINE_IDS = ["2", "3_64", "5_8", "6_1024", "8_rows", "8_empty", "3x2"]


@pytest.mark.parametrize("grid,dims,sdec", LINES, ids=LINE_IDS)
def test_blocks_per_line(grid, dims, sdec):
    check_line(grid, dims, sdec)


@pytest.mark.parametrize("grid,dims,sdec", LINES, ids=LINE_IDS)
def test_rfft_blocks_per_line(grid, dims, sdec):
    N = max(16, 2 * (dims[0] // 2))
    check_line(grid, (N,) + dims[1:], sdec, rfft=True)


@pytest.mark.parametrize("rfft", [False, True], ids=["fft", "rfft"])
@pytest.mark.parametrize("kw", [
    dict(dims=(32, 13, 3)),                                     # partial tiles (13 columns)
    dict(dims=(16, 5, 3), extra=(2, 1, 1, 1, 2)),               # 3 + 5 = PA_MAX_DIMS dims
    dict(dims=(64, 6, 5), dperm=None),                          # unpermuted: stores along the line
    dict(dims=(64, 6, 5), dperm=(3, 1, 2)),                     # z contiguous in the destination
    dict(dims=(128, 6, 5), sperm=(1, 3, 2), dperm=(2, 3, 1)),
    dict(dims=(256, 9, 2), dtype=torch.complex64, extra=(3,)),
    dict(dims=(64, 9, 2), dtype=torch.complex64, dperm=None),
], ids=["partial", "max_dims", "unpermuted", "dst_zxy", "perms", "f32_extra", "f32_unpermuted"])
def test_layouts(kw, rfft):
    kw = dict(kw)
    dims = kw.pop("dims")
    check_line((3,), dims, (2,), rfft=rfft, **kw)


@pytest.mark.parametrize("dtype", [torch.complex128, torch.complex64], ids=["c128", "c64"])
@pytest.mark.parametrize("lines", [4, 8], ids=["lines4", "lines8"])
@pytest.mark.parametrize("L", [8, 16, 32, 64, 128, 256, 512, 1024])
def test_every_line_length(L, lines, dtype):
    pa.set_tunable("fft_lines", lines)
    try:
        check_line((3,), (L, 11, 2), (2,), dtype=dtype)
        check_line((3,), (2 * L, 11, 2), (2,), dtype=dtype, rfft=True)
    finally:
        pa.set_tunable("fft_lines", 0)


@pytest.mark.parametrize("rfft", [False, True], ids=["fft", "rfft"])
@pytest.mark.parametrize("dtype", [torch.complex128, torch.complex64], ids=["c128", "c64"])
def test_local_plans_one_kernel_on_the_caller_stream(dtype, rfft):
    """One-rank lines and plans without an exchange, any method: `transpose_(t, fft_first=...)` /
    `rfft_first=True` is one kernel, ordered behind a held caller stream, equal to the pair."""
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    dims = (128, 12, 6)
    rng = np.random.default_rng(7)
    for method in (pa.PointToPoint(), pa.PeerGet(), pa.PeerPut()):
        ps = pa.Pencil(topo, dims, (2, 3))
        for pd in (pa.Pencil(ps, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3)),
                   pa.Pencil(ps, decomp_dims=(2, 3), permute=pa.Permutation(3, 2, 1))):
            side = torch.cuda.Stream()
            with torch.cuda.stream(side):
                if rfft:
                    u = pa.PencilArray.undef(REAL_OF[dtype], ps)
                    pc = _brfft_pencil(ps)
                    cd = pa.Pencil(pc, decomp_dims=pd.decomp_dims, permute=pd.perm)
                    out = pa.PencilArray.undef(dtype, cd)
                    t = pa.Transposition(out, u, method=method, rfft_first=True)
                    assert t.fft_first_fusable()
                    mid = pa.PencilArray.undef(dtype, pc)
                    want = pa.PencilArray.undef(dtype, cd)
                else:
                    u = pa.PencilArray.undef(dtype, ps)
                    out = pa.PencilArray.undef(dtype, pd)
                    t = pa.Transposition(out, u, method=method)
                    assert t.fft_first_fusable()
                    mid = pa.PencilArray.undef(dtype, ps)
                    want = pa.PencilArray.undef(dtype, pd)
                # (on the device before the hold: a pageable upload behind it would block the host)
                val = (torch.from_numpy(rng.standard_normal(u.data.shape)).to(u.data.dtype)
                       if rfft else torch.from_numpy(rng.standard_normal(u.data.shape) +
                                                     1j * rng.standard_normal(u.data.shape)).to(dtype)).cuda()
                # (the first call on a plan creates its streams and events, which synchronises the
                #  device: done here, before the hold)
                pa.transpose_(t) if rfft else pa.transpose_(t, fft_first="backward")
                torch.cuda.synchronize()
                out.data.fill_(0)
                held = hold()
                u.data.copy_(val)  # behind the hold
                n0 = pa.launch_count()
                if rfft:
                    pa.transpose_(t)
                else:
                    pa.transpose_(t, fft_first="backward")
                assert pa.launch_count() - n0 == 1
                assert not held.query()
                if rfft:
                    pa.rfft_(mid, u)
                else:
                    mid.data.copy_(u.data)
                    pa.fft_(mid, "backward")
                pa.transpose_(want, mid, method=method)
                torch.cuda.current_stream().synchronize()
                assert torch.equal(out.data.view(torch.uint8), want.data.view(torch.uint8)), (method, pd.perm)


def test_refusals_launch_nothing():
    plans, srcs, reals = [], [], []
    for er in make_ranks((3,)):
        ps = pa.Pencil(er.topo, (48, 5, 2), (2,))
        pd = pa.Pencil(ps, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
        plans.append(_Plan(ps, pd, (), 16, pa.PeerPut()))
        srcs.append(pa.PencilArray.undef(torch.complex128, ps))
        reals.append(pa.Pencil(ps, size_global=(94, 5, 2)))  # 48 bins are no N/2+1 of a power of two
    for rfft in (False, True):
        for r, plan in enumerate(plans):
            n = plan.info.length_out * plan.info.elsize
            raw = torch.full((n + 2 * PAD,), 0x3C, dtype=torch.uint8, device="cuda")
            dsts = [raw.data_ptr() + PAD] * 3
            torch.cuda.synchronize()
            n0 = pa.launch_count()
            # 48 points is no power of two
            assert put_all(plan, reals, srcs, dsts, r, 0 if rfft else FWD, rfft) != _lib.PA_OK
            assert lib.pa_fft_put(plan.h, None, C.c_void_p(srcs[r].data_ptr()), C.c_void_p(dsts[0]),
                                  FWD, stream_ptr()) == _lib.PA_EINVAL
            assert pa.launch_count() == n0
            torch.cuda.synchronize()
            assert bool((raw == 0x3C).all())
    # a PointToPoint transposition with an exchange: refused by the Python mirror and the library
    er = make_ranks((2,))[0]
    ps = pa.Pencil(er.topo, (32, 4, 3), (2,))
    pd = pa.Pencil(ps, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
    u, v = pa.PencilArray.undef(torch.complex128, ps), pa.PencilArray.undef(torch.complex128, pd)
    t = pa.Transposition(v, u, method=pa.PointToPoint())
    assert not t.fft_first_fusable()
    n0 = pa.launch_count()
    with pytest.raises(pa.ArgumentError, match="receive side"):
        pa.transpose_(t, fft_first="forward")
    assert pa.launch_count() == n0


@pytest.mark.parametrize("world", [2, 3, 4, 5, 6, 8])
def test_fft_put_across_processes(world, tmp_path):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29991 + world),
           os.path.join(HERE, "mp_fft_put_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1", PA_TEST_TMPDIR=str(tmp_path))
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    assert f"MP_FFT_PUT_OK world={world}" in out.stdout, out.stdout[-2000:]
