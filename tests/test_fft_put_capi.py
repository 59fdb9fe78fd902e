"""The send-side fused transform + put (PeerPut, DESIGN §3i) on the host: its checks and the
refusals of `pa_fft_put`, `pa_rfft_put`, `pa_put_all_fft` and `pa_put_all_rfft`.  No device is
needed.

`pa_plan_fft_put_check` / `pa_plan_rfft_put_check` rebuild every rank's plan of the grid line, so
a refused geometry is refused on every rank alike -- a rank that refused while its peers went
ahead would leave them waiting on flags it never sets.  Asking them leaves every existing verdict
(tests/golden/fft_check_verdicts.json) exactly as recorded."""
import ctypes as C
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import pencilarrays_b200 as pa  # noqa: E402
from pencilarrays_b200 import _lib  # noqa: E402
from pencilarrays_b200._lib import lib, ArgumentError  # noqa: E402
from pencilarrays_b200.transpositions import _Plan, _brfft_pencil  # noqa: E402
from util import build_chain, make_ranks  # noqa: E402
from test_fft_check import ALL  # noqa: E402
from test_fft_peerget_capi import golden, HostBuf  # noqa: E402

OK, EINVAL, EINCOMPAT, ENOGPU = _lib.PA_OK, _lib.PA_EINVAL, _lib.PA_EINCOMPAT, _lib.PA_ENOGPU
F32, FWD, BWD, WAITALL = _lib.PA_FFT_F32, _lib.PA_FFT_FORWARD, _lib.PA_FFT_BACKWARD, _lib.PA_WAITALL
METHODS = [pa.PointToPoint(), pa.Alltoallv(), pa.PeerPut(), pa.PeerGet()]


def no_gpu():
    return lib.pa_device_count() == 0


def put_verdicts(case):
    """{(step, rank): "ffff rrrr"}: the fft and rfft put checks of the PeerPut plan in ComplexF64 and
    ComplexF32, plus the grid line of every rank per step; and the fft_check_ex table of every
    method, asked AFTER the put checks."""
    ranks, steps = build_chain(case)
    table, lines, gold_codes = {}, {}, {}
    for k in range(1, len(steps)):
        for r in range(len(ranks)):
            codes = ""
            for f32 in (False, True):
                plan = _Plan(steps[k - 1][r][0], steps[k][r][0], case["extra"], 8 if f32 else 16,
                             pa.PeerPut())
                for fn in (lib.pa_plan_fft_put_check, lib.pa_plan_rfft_put_check):
                    st = fn(plan.h, F32 if f32 else 0)
                    assert fn(plan.h, F32 if f32 else 0) == st  # cached
                    codes += str(st)
                info = plan.info
                lines[(k, r)] = tuple(sorted(plan.peer(n).world_rank for n in range(1, info.nproc + 1))) \
                    if info.dim else (r,)
            table[(k, r)] = codes
            ex = ""
            for method in METHODS:
                for f32 in (False, True):
                    plan = _Plan(steps[k - 1][r][0], steps[k][r][0], case["extra"], 8 if f32 else 16,
                                 method)
                    lib.pa_plan_fft_put_check(plan.h, F32 if f32 else 0)
                    lib.pa_plan_rfft_put_check(plan.h, F32 if f32 else 0)
                    ex += str(lib.pa_plan_fft_check_ex(plan.h, F32 if f32 else 0))
            gold_codes[f"{k}/{r}"] = ex
    return table, lines, gold_codes


@pytest.mark.parametrize("case", ALL, ids=[c["name"] for c in ALL])
def test_put_verdicts_are_uniform_and_fft_check_unchanged(case):
    table, lines, ex = put_verdicts(case)
    for (k, r), line in lines.items():
        for i in range(4):
            got = {table[(k, q)][i] for q in line}
            assert len(got) == 1, (case["name"], k, line, i, got)
            assert got <= {str(OK), str(EINVAL)}
    gold = golden()[case["name"]]
    assert set(ex) == set(gold)
    for key, codes in ex.items():
        assert codes[:6] == gold[key][:6], (case["name"], key, codes, gold[key])
        assert codes[6:8] == codes[0:2], (case["name"], key, codes)


def test_the_sets_exercise_both_put_verdicts():
    seen = set()
    for case in ALL:
        table, _, _ = put_verdicts(case)
        seen |= {c[0] for c in table.values()} | {c[2] for c in table.values()}
    assert seen == {str(OK), str(EINVAL)}


# ---- a grid line: x-pencil (x local, first memory dim) -> y-pencil decomposed along x ----------
def line_plans(nproc, L, other=(4, 3), extra=(), elsize=16, method=None, permuted=True):
    method = method or pa.PeerPut()
    out = []
    for er in make_ranks((nproc,)):
        px = pa.Pencil(er.topo, (L,) + other, (2,))
        py = pa.Pencil(px, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3) if permuted else None)
        out.append(_Plan(px, py, extra, elsize, method))
        out[-1].px = px  # (the input pencil: real_pencil derives the rfft source pencil from it)
    return out


def setup(nproc=3, L=64, elsize=16, method=None, n_real=None):
    plans = line_plans(nproc, L, other=(nproc + 1, 3), elsize=elsize, method=method)
    plan = plans[1]
    info = plan.info
    nin, nout = info.length_in * elsize, info.length_out * elsize
    if n_real is not None:
        nin = nin // L * n_real * elsize // 2
    ain, aout = (nin + 255) // 256 * 256, (nout + 255) // 256 * 256
    buf = HostBuf(ain + aout + nproc * aout * 4)
    src, dst = buf.at(0), buf.at(ain)
    peers = [buf.at(ain + aout + 4 * aout * n) for n in range(nproc)]
    return plan, src, peers, dst, buf


def real_pencil(plan, N):
    """The real x-pencil of N points beside the plan's input pencil (its N/2+1-bin counterpart when
    the input pencil has N/2+1 points along x)."""
    return pa.Pencil(plan.px, size_global=(N,) + tuple(plan.px.size_global[1:]))


def arr(peers):
    return (C.c_void_p * len(peers))(*[p.value if p is not None else None for p in peers]) \
        if peers is not None else None


def put_all(plan, src, peers, dst, flags):
    return lib.pa_put_all_fft(plan.h if plan else None, src, arr(peers), dst, flags, None)


@pytest.mark.parametrize("flags", [0, FWD | BWD, F32, FWD | WAITALL, BWD | _lib.PA_STAGE_SELF,
                                   FWD | _lib.PA_NO_OVERLAP, FWD | 64, 1 << 31])
def test_put_all_fft_bad_flags(flags):
    plan, src, peers, dst, _ = setup()
    assert put_all(plan, src, peers, dst, flags) == EINVAL
    assert lib.pa_last_error().startswith(b"pa_put_all_fft: ")


@pytest.mark.parametrize("flags", [0, FWD | BWD, F32, FWD | F32 | WAITALL | 64, _lib.PA_NO_OVERLAP])
def test_fft_put_bad_flags(flags):
    plan, src, _, dst, _ = setup()
    assert lib.pa_fft_put(plan.h, None, src, dst, flags, None) == EINVAL
    assert lib.pa_last_error().startswith(b"pa_fft_put: flags must be exactly")


def test_stage_self_is_refused_with_its_reason():
    plan, src, peers, dst, _ = setup()
    for st in (lib.pa_fft_put(plan.h, None, src, dst, FWD | _lib.PA_STAGE_SELF, None),
               put_all(plan, src, peers, dst, FWD | _lib.PA_STAGE_SELF)):
        assert st == EINVAL
        assert b"PA_STAGE_SELF does not apply" in lib.pa_last_error()


@pytest.mark.parametrize("method", [pa.PointToPoint(), pa.Alltoallv(), pa.PeerGet()], ids=repr)
def test_other_methods_are_refused_naming_the_receive_side_fusion(method):
    plan, src, peers, dst, _ = setup(method=method)
    p8 = setup(method=method, elsize=8)[0]
    for pl, f32 in ((plan, 0), (p8, F32)):
        for fn in (lib.pa_plan_fft_put_check, lib.pa_plan_rfft_put_check):
            assert fn(pl.h, f32) == EINVAL
            assert b"needs PeerPut" in lib.pa_last_error()
            assert b"PA_FFT_FORWARD" in lib.pa_last_error()
    assert lib.pa_fft_put(plan.h, None, src, dst, FWD, None) == EINVAL
    assert b"receive side" in lib.pa_last_error()
    assert put_all(plan, src, peers, dst, BWD) == EINVAL
    # ... yet a local plan of the same method runs (no device here: ENOGPU after the checks)
    topo = pa.MPITopology(pa.COMM_SELF, (1,))
    px = pa.Pencil(topo, (32, 4, 3), (2,))
    py = pa.Pencil(px, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
    local = _Plan(px, py, (), 16, method)
    assert lib.pa_plan_fft_put_check(local.h, 0) == OK
    big = HostBuf(2 * 32 * 4 * 3 * 16)
    if no_gpu():
        assert lib.pa_fft_put(local.h, None, big.at(0), big.at(32 * 4 * 3 * 16), FWD, None) == ENOGPU


def test_host_refusals():
    plan, src, peers, dst, _ = setup()
    assert lib.pa_fft_put(None, None, src, dst, FWD, None) == EINVAL
    assert put_all(None, src, peers, dst, FWD) == EINVAL
    # a purely local plan has nothing to put
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px = pa.Pencil(topo, (16, 8, 4), (2, 3))
    py = pa.Pencil(px, decomp_dims=(2, 3), permute=pa.Permutation(2, 1, 3))
    assert put_all(_Plan(px, py, (), 16, pa.PeerPut()), src, peers, dst, FWD) == EINVAL
    assert b"no exchange" in lib.pa_last_error()
    # lengths: the plan's verdict first
    for L in (4, 48, 2048):
        pl, s2, pe2, d2, _ = setup(L=L)
        assert put_all(pl, s2, pe2, d2, FWD) == EINVAL
        assert b"power of two in 8..1024" in lib.pa_last_error()
        assert lib.pa_fft_put(pl.h, None, s2, d2, BWD, None) == EINVAL
    # dtypes: a ComplexF32 flag on a ComplexF64 plan and the other way round
    assert put_all(plan, src, peers, dst, FWD | F32) == EINVAL
    assert b"ComplexF32" in lib.pa_last_error()
    p8, s8, pe8, d8, _ = setup(elsize=8)
    assert lib.pa_fft_put(p8.h, None, s8, d8, FWD, None) == EINVAL
    assert b"ComplexF64" in lib.pa_last_error()
    # pointers: a missing peer array, NULL src / dst, misalignment, overlap
    assert put_all(plan, src, None, dst, FWD) == EINVAL
    assert put_all(plan, src, [peers[0], peers[1], None], dst, FWD) == EINVAL
    assert b"peer 3" in lib.pa_last_error()
    assert put_all(plan, None, peers, dst, BWD) == EINVAL
    assert b"null array pointer" in lib.pa_last_error()
    assert lib.pa_fft_put(plan.h, None, src, None, FWD, None) == EINVAL
    assert put_all(plan, src, [C.c_void_p(peers[0].value + 8)] + peers[1:], dst, FWD) == EINVAL
    assert b"aligned" in lib.pa_last_error()
    assert lib.pa_fft_put(plan.h, None, src, C.c_void_p(dst.value + 8), FWD, None) == EINVAL
    assert b"aligned" in lib.pa_last_error()
    assert lib.pa_fft_put(plan.h, None, src, C.c_void_p(src.value + 16), FWD, None) == EINVAL
    assert b"overlap" in lib.pa_last_error()
    assert lib.pa_fft_put(plan.h, None, src, src, FWD, None) == EINVAL
    assert b"overlap" in lib.pa_last_error()
    # the self entry of `peers` is ignored (plan 1 is rank 2 of the line)
    if no_gpu():
        assert put_all(plan, src, [peers[0], None, peers[2]], dst, FWD) == ENOGPU


def test_a_decomposed_transform_axis_is_refused():
    for er in make_ranks((2,))[:1]:
        # x decomposed in the input pencil: the first memory dim of src is not whole
        px = pa.Pencil(er.topo, (32, 8, 4), (1,))
        py = pa.Pencil(px, decomp_dims=(2,), permute=pa.Permutation(2, 1, 3))
        plan = _Plan(px, py, (), 16, pa.PeerPut())
        for fn in (lib.pa_plan_fft_put_check, lib.pa_plan_rfft_put_check):
            assert fn(plan.h, 0) == EINVAL
            assert b"is decomposed" in lib.pa_last_error()


def test_rfft_put_refusals():
    N = 64
    plan, src, peers, dst, _ = setup(L=N // 2 + 1, n_real=N)
    real = real_pencil(plan, N)
    rfft_put = lambda p, r, s, d, f: lib.pa_rfft_put(p.h if p else None, None, r._h if r else None,  # noqa: E731
                                                     s, d, f, None)
    assert rfft_put(None, real, src, dst, 0) == EINVAL
    for flags in (FWD, BWD, _lib.PA_NO_OVERLAP, 64):
        assert rfft_put(plan, real, src, dst, flags) == EINVAL
        assert lib.pa_last_error().startswith(b"pa_rfft_put: flags may combine")
    assert rfft_put(plan, real, src, dst, _lib.PA_STAGE_SELF) == EINVAL
    assert b"PA_STAGE_SELF" in lib.pa_last_error()
    # dtype pairs: Float32 -> ComplexF32 needs an elsize-8 plan
    assert rfft_put(plan, real, src, dst, F32) == EINVAL
    assert b"ComplexF32" in lib.pa_last_error()
    # `real` must be the N-point counterpart of the plan's input pencil
    assert rfft_put(plan, None, src, dst, 0) == EINVAL
    assert rfft_put(plan, real_pencil(plan, 2 * N), src, dst, 0) == EINCOMPAT
    assert b"N/2+1" in lib.pa_last_error()
    # lengths: bins that are not N/2+1 for a power-of-two N (the plan's verdict)
    p64, s64, _, d64, _ = setup(L=64)
    assert rfft_put(p64, real_pencil(p64, 126), s64, d64, 0) == EINVAL
    assert b"N/2+1 with N a power of two" in lib.pa_last_error()
    # pointers
    assert rfft_put(plan, real, None, dst, 0) == EINVAL
    assert rfft_put(plan, real, src, C.c_void_p(dst.value + 8), 0) == EINVAL
    assert b"aligned" in lib.pa_last_error()
    assert rfft_put(plan, real, src, C.c_void_p(src.value + 16), WAITALL) == EINVAL
    assert b"overlap" in lib.pa_last_error()
    # pa_put_all_rfft: the same checks, flags 0 or PA_FFT_F32, and every peer array
    put_all_r = lambda f, pe=peers: lib.pa_put_all_rfft(plan.h, real._h, src, arr(pe), dst, f, None)  # noqa: E731
    assert put_all_r(WAITALL) == EINVAL
    assert lib.pa_last_error().startswith(b"pa_put_all_rfft: flags may combine PA_FFT_F32 only")
    assert put_all_r(0, [peers[0], peers[1], None]) == EINVAL
    assert b"peer 3" in lib.pa_last_error()
    if no_gpu():
        assert rfft_put(plan, real, src, dst, WAITALL) == ENOGPU
        assert put_all_r(0) == ENOGPU


def test_valid_arguments_without_a_device_give_enogpu():
    if not no_gpu():
        pytest.skip("GPU present")
    for elsize, prec in ((16, 0), (8, F32)):
        for L in (8, 1024):
            plan, src, peers, dst, _ = setup(nproc=6, L=L, elsize=elsize)
            for d in (FWD, BWD):
                assert put_all(plan, src, peers, dst, d | prec) == ENOGPU, (elsize, L, d)
                assert lib.pa_fft_put(plan.h, None, src, dst, d | prec | WAITALL, None) == ENOGPU
        for N in (16, 2048):
            plan, src, peers, dst, _ = setup(nproc=6, L=N // 2 + 1, elsize=elsize, n_real=N)
            real = real_pencil(plan, N)
            assert lib.pa_rfft_put(plan.h, None, real._h, src, dst, prec, None) == ENOGPU
            assert lib.pa_put_all_rfft(plan.h, real._h, src, arr(peers), dst, prec, None) == ENOGPU


def test_empty_source_accepts_null_pointers():
    """y = 3 over 4 ranks: rank 4 owns no source lines (its src is empty)."""
    if not no_gpu():
        pytest.skip("GPU present")
    plans = line_plans(4, 16, other=(3, 2))
    for plan in plans:
        info = plan.info
        peers = [None if plan.peer(n).send_count == 0 else C.c_void_p(1 << 20) for n in range(1, 5)]
        src = C.c_void_p(1 << 24) if info.length_in else None
        dst = C.c_void_p(1 << 28) if info.length_out else None
        assert put_all(plan, src, peers, dst, FWD) == ENOGPU, lib.pa_last_error()


def test_python_mirror_refuses_before_any_window_setup():
    er = make_ranks((2,))[0]
    pr = pa.Pencil(er.topo, (64, 4, 3), (2,))
    px = _brfft_pencil(pr)
    py = pa.Pencil(px, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
    cx = pa.PencilArray.undef(torch.complex128, px, device="cpu")
    cy = pa.PencilArray.undef(torch.complex128, py, device="cpu")
    rx = pa.PencilArray.undef(torch.float64, pr, device="cpu")
    # dtype pairs
    with pytest.raises(ArgumentError):
        pa.Transposition(cy, pa.PencilArray.undef(torch.float32, pr, device="cpu"), rfft_first=True)
    with pytest.raises(ArgumentError):
        pa.Transposition(cy, rx, rfft_first=True, rfft=True)
    # the method: refused by the check, before the collective window setup
    with pytest.raises(ArgumentError, match="needs PeerPut"):
        pa.Transposition(cy, rx, rfft_first=True, method=pa.PointToPoint())
    t = pa.Transposition(cy, cx, method=pa.PeerGet())
    assert not t.fft_first_fusable()
