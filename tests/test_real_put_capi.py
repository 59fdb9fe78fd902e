"""The send-side fused real line transforms + put (PeerPut, DESIGN §3j) on the host: the verdict
`pa_plan_real_put_check` and the refusals of `pa_r2r_put`, `pa_brfft_put`, `pa_put_all_r2r` and
`pa_put_all_brfft`.  No device is needed.

The verdict rebuilds every rank's plan of the grid line, so a refused geometry is refused on every
rank alike; it has its own cache, so asking it leaves every other verdict -- the pinned
tests/golden/fft_check_verdicts.json and the put verdicts of the complex plans -- as it was."""
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
KINDS = [_lib.PA_REDFT10, _lib.PA_REDFT01, _lib.PA_RODFT10, _lib.PA_RODFT01]
METHODS = [pa.PointToPoint(), pa.Alltoallv(), pa.PeerPut(), pa.PeerGet()]


def no_gpu():
    return lib.pa_device_count() == 0


def real_verdicts(case):
    """{(step, rank): "ab"}: the real put verdict of the PeerPut plan in Float64 and Float32, the
    grid line of every rank per step, and the fft_check_ex table of every method asked AFTER the
    real put checks of the same plans."""
    ranks, steps = build_chain(case)
    table, lines, gold_codes = {}, {}, {}
    for k in range(1, len(steps)):
        for r in range(len(ranks)):
            codes = ""
            for f32 in (False, True):
                plan = _Plan(steps[k - 1][r][0], steps[k][r][0], case["extra"], 4 if f32 else 8,
                             pa.PeerPut())
                st = lib.pa_plan_real_put_check(plan.h, F32 if f32 else 0)
                assert lib.pa_plan_real_put_check(plan.h, F32 if f32 else 0) == st  # cached
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
                    lib.pa_plan_real_put_check(plan.h, F32 if f32 else 0)
                    ex += str(lib.pa_plan_fft_check_ex(plan.h, F32 if f32 else 0))
            gold_codes[f"{k}/{r}"] = ex
    return table, lines, gold_codes


@pytest.mark.parametrize("case", ALL, ids=[c["name"] for c in ALL])
def test_real_put_verdicts_are_uniform_and_fft_check_unchanged(case):
    table, lines, ex = real_verdicts(case)
    for (k, r), line in lines.items():
        for i in range(2):
            got = {table[(k, q)][i] for q in line}
            assert len(got) == 1, (case["name"], k, line, i, got)
            assert got <= {str(OK), str(EINVAL)}
    gold = golden()[case["name"]]
    assert set(ex) == set(gold)
    for key, codes in ex.items():
        assert codes[:6] == gold[key][:6], (case["name"], key, codes, gold[key])


def test_the_sets_exercise_both_real_put_verdicts():
    seen = set()
    for case in ALL:
        table, _, _ = real_verdicts(case)
        seen |= {c[0] for c in table.values()} | {c[1] for c in table.values()}
    assert seen == {str(OK), str(EINVAL)}


# ---- a grid line: real x-pencil (x local, first memory dim) -> y-pencil decomposed along x -----
def line_plans(nproc, N, other=(4, 3), extra=(), elsize=8, method=None, permuted=True):
    method = method or pa.PeerPut()
    out = []
    for er in make_ranks((nproc,)):
        px = pa.Pencil(er.topo, (N,) + other, (2,))
        py = pa.Pencil(px, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3) if permuted else None)
        out.append(_Plan(px, py, extra, elsize, method))
        out[-1].px = px  # (the input pencil: its complex counterpart is brfft's source pencil)
    return out


@pytest.mark.parametrize("nproc", range(1, 10))
@pytest.mark.parametrize("N", [16, 32, 48, 2048, 4096])
def test_every_rank_of_a_line_agrees(nproc, N):
    """Lines of 1 ... 9 ranks: 8 blocks at most, a power of two N in 16..2048, any block boundary
    (N = 32 over 3 ranks: 11 / 11 / 10 reals)."""
    for elsize, f32 in ((8, 0), (4, F32)):
        got = {lib.pa_plan_real_put_check(p.h, f32) for p in line_plans(nproc, N, other=(5, 2),
                                                                           elsize=elsize)}
        assert len(got) == 1, (nproc, N, got)
        want = OK if (nproc <= 8 and N in (16, 32, 2048)) else EINVAL
        assert got == {want}, (nproc, N, lib.pa_last_error())


def test_refusal_reasons():
    p9 = line_plans(9, 64)[4]
    assert lib.pa_plan_real_put_check(p9.h, 0) == EINVAL
    assert b"more than 8 blocks" in lib.pa_last_error()
    p48 = line_plans(3, 48)[0]
    assert lib.pa_plan_real_put_check(p48.h, 0) == EINVAL
    assert b"power of two in 16..2048" in lib.pa_last_error()
    # the cached refusal keeps its reason
    assert lib.pa_plan_real_put_check(p48.h, 0) == EINVAL
    assert b"power of two in 16..2048" in lib.pa_last_error()
    # element sizes: a Float32 flag on a Float64 plan, a complex plan
    p = line_plans(3, 64)[1]
    assert lib.pa_plan_real_put_check(p.h, F32) == EINVAL
    assert b"Float32 (elsize 4)" in lib.pa_last_error()
    pc = line_plans(3, 64, elsize=16)[1]
    assert lib.pa_plan_real_put_check(pc.h, 0) == EINVAL
    assert b"Float64 (elsize 8)" in lib.pa_last_error()
    # a decomposed transform axis
    er = make_ranks((2,))[0]
    px = pa.Pencil(er.topo, (32, 8, 4), (1,))
    py = pa.Pencil(px, decomp_dims=(2,), permute=pa.Permutation(2, 1, 3))
    assert lib.pa_plan_real_put_check(_Plan(px, py, (), 8, pa.PeerPut()).h, 0) == EINVAL
    assert b"is decomposed" in lib.pa_last_error()


@pytest.mark.parametrize("method", [pa.PointToPoint(), pa.Alltoallv(), pa.PeerGet()], ids=repr)
def test_other_methods_are_refused_naming_the_receive_side_fusion(method):
    for elsize, f32 in ((8, 0), (4, F32)):
        for plan in line_plans(3, 64, elsize=elsize, method=method):
            assert lib.pa_plan_real_put_check(plan.h, f32) == EINVAL
            assert b"needs PeerPut" in lib.pa_last_error()
            assert b"pa_transpose_r2r" in lib.pa_last_error()
    # ... yet a local plan of the same method passes
    topo = pa.MPITopology(pa.COMM_SELF, (1,))
    px = pa.Pencil(topo, (32, 4, 3), (2,))
    py = pa.Pencil(px, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
    assert lib.pa_plan_real_put_check(_Plan(px, py, (), 8, method).h, 0) == OK


def test_caches_are_apart():
    """The real put verdict does not answer for the complex put verdicts or the receive-side real
    verdict of the same plan, nor they for it."""
    # a real PeerPut plan: its receive-side verdict refuses PeerPut, the send-side one accepts
    p = line_plans(3, 64)[0]
    assert lib.pa_plan_real_check(p.h, 0) == EINVAL
    assert lib.pa_plan_real_put_check(p.h, 0) == OK
    assert lib.pa_plan_real_check(p.h, 0) == EINVAL
    q = line_plans(3, 64)[0]
    assert lib.pa_plan_real_put_check(q.h, 0) == OK
    assert lib.pa_plan_real_check(q.h, 0) == EINVAL
    # complex put verdicts refuse an elsize-8 real plan as Float64 yet accept it as ComplexF32
    for first_real in (True, False):
        p = line_plans(3, 64)[1]
        if first_real:
            assert lib.pa_plan_real_put_check(p.h, 0) == OK
        assert lib.pa_plan_fft_put_check(p.h, 0) == EINVAL
        assert lib.pa_plan_rfft_put_check(p.h, 0) == EINVAL
        assert lib.pa_plan_fft_put_check(p.h, F32) == OK
        assert lib.pa_plan_real_put_check(p.h, 0) == OK
        assert lib.pa_plan_real_put_check(p.h, F32) == EINVAL


# ---- the entry points -----------------------------------------------------------------------
def setup(nproc=3, N=64, elsize=8, method=None, cplx=False):
    plans = line_plans(nproc, N, other=(nproc + 1, 3), elsize=elsize, method=method)
    plan = plans[1]
    info = plan.info
    nin, nout = info.length_in * elsize, info.length_out * elsize
    if cplx:
        nin = nin // N * (N // 2 + 1) * 2
    ain, aout = (nin + 255) // 256 * 256, (nout + 255) // 256 * 256
    buf = HostBuf(ain + aout + nproc * aout * 4)
    src, dst = buf.at(0), buf.at(ain)
    peers = [buf.at(ain + aout + 4 * aout * n) for n in range(nproc)]
    return plan, src, peers, dst, buf


def arr(peers):
    return (C.c_void_p * len(peers))(*[p.value if p is not None else None for p in peers]) \
        if peers is not None else None


def r2r_put(plan, kind, src, dst, flags):
    return lib.pa_r2r_put(plan.h if plan else None, None, kind, src, dst, flags, None)


def put_all_r2r(plan, kind, src, peers, dst, flags):
    return lib.pa_put_all_r2r(plan.h if plan else None, kind, src, arr(peers), dst, flags, None)


@pytest.mark.parametrize("flags", [FWD, BWD, _lib.PA_NO_OVERLAP, 64, 1 << 31])
def test_bad_flags(flags):
    plan, src, peers, dst, _ = setup()
    assert r2r_put(plan, _lib.PA_REDFT10, src, dst, flags) == EINVAL
    assert lib.pa_last_error().startswith(b"pa_r2r_put: flags may combine PA_WAITALL and PA_FFT_F32 only")
    assert put_all_r2r(plan, _lib.PA_REDFT10, src, peers, dst, flags | WAITALL) == EINVAL
    assert lib.pa_last_error().startswith(b"pa_put_all_r2r: flags may combine PA_FFT_F32 only")
    cp = _brfft_pencil(plan.px)
    assert lib.pa_brfft_put(plan.h, None, cp._h, src, dst, flags, None) == EINVAL
    assert lib.pa_last_error().startswith(b"pa_brfft_put: flags may combine")


@pytest.mark.parametrize("kind", [-1, 0, 3, 6, 7, 10, 11, 99])
def test_bad_kinds(kind):
    plan, src, peers, dst, _ = setup()
    assert r2r_put(plan, kind, src, dst, 0) == EINVAL
    assert b"is not PA_REDFT10, PA_REDFT01, PA_RODFT10 or PA_RODFT01" in lib.pa_last_error()
    assert put_all_r2r(plan, kind, src, peers, dst, 0) == EINVAL
    assert lib.pa_last_error().startswith(b"pa_put_all_r2r: kind")


def test_stage_self_is_refused_with_its_reason():
    plan, src, peers, dst, _ = setup()
    cp = _brfft_pencil(plan.px)
    for st in (r2r_put(plan, _lib.PA_REDFT01, src, dst, _lib.PA_STAGE_SELF),
               put_all_r2r(plan, _lib.PA_REDFT01, src, peers, dst, _lib.PA_STAGE_SELF),
               lib.pa_brfft_put(plan.h, None, cp._h, src, dst, _lib.PA_STAGE_SELF | WAITALL, None)):
        assert st == EINVAL
        assert b"PA_STAGE_SELF does not apply" in lib.pa_last_error()


def test_r2r_put_host_refusals():
    plan, src, peers, dst, _ = setup()
    K = _lib.PA_RODFT10
    assert r2r_put(None, K, src, dst, 0) == EINVAL
    assert put_all_r2r(None, K, src, peers, dst, 0) == EINVAL
    # a purely local plan has nothing to put
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px = pa.Pencil(topo, (16, 8, 4), (2, 3))
    py = pa.Pencil(px, decomp_dims=(2, 3), permute=pa.Permutation(2, 1, 3))
    assert put_all_r2r(_Plan(px, py, (), 8, pa.PeerPut()), K, src, peers, dst, 0) == EINVAL
    assert b"no exchange" in lib.pa_last_error()
    # lengths and block counts: the plan's verdict first
    for N in (8, 48, 4096):
        pl, s2, pe2, d2, _ = setup(N=N)
        assert put_all_r2r(pl, K, s2, pe2, d2, 0) == EINVAL
        assert b"power of two in 16..2048" in lib.pa_last_error()
        assert r2r_put(pl, K, s2, d2, 0) == EINVAL
    p9, s9, pe9, d9, _ = setup(nproc=9)
    assert r2r_put(p9, K, s9, d9, 0) == EINVAL
    assert b"more than 8 blocks" in lib.pa_last_error()
    # precision
    assert r2r_put(plan, K, src, dst, F32) == EINVAL
    assert b"Float32" in lib.pa_last_error()
    # pointers: a missing peer array, NULL src / dst, misalignment, overlap
    assert put_all_r2r(plan, K, src, None, dst, 0) == EINVAL
    assert put_all_r2r(plan, K, src, [peers[0], peers[1], None], dst, 0) == EINVAL
    assert b"peer 3" in lib.pa_last_error()
    assert put_all_r2r(plan, K, None, peers, dst, 0) == EINVAL
    assert b"null array pointer" in lib.pa_last_error()
    assert r2r_put(plan, K, src, None, 0) == EINVAL
    _, roomy, _, d_roomy, _b = setup(cplx=True)  # (room for a shifted src before dst)
    assert r2r_put(plan, K, C.c_void_p(roomy.value + 8), d_roomy, 0) == EINVAL  # loads pairs of reals
    assert b"aligned" in lib.pa_last_error()
    assert r2r_put(plan, K, src, C.c_void_p(dst.value + 4), 0) == EINVAL
    assert b"aligned" in lib.pa_last_error()
    assert put_all_r2r(plan, K, src, [C.c_void_p(peers[0].value + 4)] + peers[1:], dst, 0) == EINVAL
    assert b"aligned" in lib.pa_last_error()
    assert r2r_put(plan, K, src, C.c_void_p(src.value + 16), 0) == EINVAL
    assert b"overlap" in lib.pa_last_error()
    assert r2r_put(plan, K, src, src, WAITALL) == EINVAL
    assert b"overlap" in lib.pa_last_error()
    if no_gpu():
        # the self entry of `peers` is ignored (plan 1 is rank 2 of the line); the destination
        # may start at any real
        assert put_all_r2r(plan, K, src, [peers[0], None, peers[2]], C.c_void_p(dst.value + 8), 0) == ENOGPU
        assert r2r_put(plan, K, src, dst, WAITALL) == ENOGPU


def test_brfft_put_host_refusals():
    N = 64
    plan, src, peers, dst, _ = setup(N=N, cplx=True)
    cp = _brfft_pencil(plan.px)
    brfft_put = lambda p, c, s, d, f: lib.pa_brfft_put(p.h if p else None, None, c._h if c else None,  # noqa: E731
                                                       s, d, f, None)
    assert brfft_put(None, cp, src, dst, 0) == EINVAL
    # the precision of a Float64 plan
    assert brfft_put(plan, cp, src, dst, F32) == EINVAL
    assert b"Float32" in lib.pa_last_error()
    # `cplx` must be the N/2+1-bin counterpart of the plan's input pencil
    assert brfft_put(plan, None, src, dst, 0) == EINVAL
    other = pa.Pencil(plan.px, size_global=(N + 2,) + tuple(plan.px.size_global[1:]))
    assert brfft_put(plan, other, src, dst, 0) == EINCOMPAT
    assert b"N/2+1" in lib.pa_last_error()
    assert brfft_put(plan, plan.px, src, dst, 0) == EINCOMPAT
    # pointers
    assert brfft_put(plan, cp, None, dst, 0) == EINVAL
    assert brfft_put(plan, cp, C.c_void_p(src.value + 8), dst, 0) == EINVAL
    assert b"aligned" in lib.pa_last_error()
    assert brfft_put(plan, cp, src, C.c_void_p(src.value + 64), WAITALL) == EINVAL
    assert b"overlap" in lib.pa_last_error()
    put_all_b = lambda f, pe=peers: lib.pa_put_all_brfft(plan.h, cp._h, src, arr(pe), dst, f, None)  # noqa: E731
    assert put_all_b(WAITALL) == EINVAL
    assert lib.pa_last_error().startswith(b"pa_put_all_brfft: flags may combine PA_FFT_F32 only")
    assert put_all_b(0, [peers[0], peers[1], None]) == EINVAL
    assert b"peer 3" in lib.pa_last_error()
    if no_gpu():
        assert brfft_put(plan, cp, src, dst, WAITALL) == ENOGPU
        assert put_all_b(0) == ENOGPU


def test_valid_arguments_without_a_device_give_enogpu():
    if not no_gpu():
        pytest.skip("GPU present")
    for elsize, prec in ((8, 0), (4, F32)):
        for N in (16, 2048):
            plan, src, peers, dst, _ = setup(nproc=6, N=N, elsize=elsize, cplx=True)
            for kind in KINDS:
                assert put_all_r2r(plan, kind, src, peers, dst, prec) == ENOGPU, (elsize, N, kind)
                assert r2r_put(plan, kind, src, dst, prec | WAITALL) == ENOGPU
            cp = _brfft_pencil(plan.px)
            assert lib.pa_brfft_put(plan.h, None, cp._h, src, dst, prec, None) == ENOGPU
            assert lib.pa_put_all_brfft(plan.h, cp._h, src, arr(peers), dst, prec, None) == ENOGPU
        # local plans of any method
        topo = pa.MPITopology(pa.COMM_SELF, (1,))
        px = pa.Pencil(topo, (32, 4, 3), (2,))
        py = pa.Pencil(px, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
        big = HostBuf(2 * 32 * 4 * 3 * 16)
        for method in METHODS:
            local = _Plan(px, py, (), elsize, method)
            assert r2r_put(local, _lib.PA_REDFT01, big.at(0), big.at(32 * 4 * 3 * 16), prec) == ENOGPU


def test_empty_source_accepts_null_pointers():
    """y = 3 over 4 ranks: rank 4 owns no source lines (its src is empty)."""
    if not no_gpu():
        pytest.skip("GPU present")
    for plan in line_plans(4, 16, other=(3, 2)):
        info = plan.info
        peers = [None if plan.peer(n).send_count == 0 else C.c_void_p(1 << 20) for n in range(1, 5)]
        src = C.c_void_p(1 << 24) if info.length_in else None
        dst = C.c_void_p(1 << 28) if info.length_out else None
        assert put_all_r2r(plan, _lib.PA_REDFT10, src, peers, dst, 0) == ENOGPU, lib.pa_last_error()


def test_python_mirror():
    er = make_ranks((2,))[0]
    pr = pa.Pencil(er.topo, (64, 4, 3), (2,))
    prc = _brfft_pencil(pr)
    py = pa.Pencil(pr, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
    rx = pa.PencilArray.undef(torch.float64, pr, device="cpu")
    ry = pa.PencilArray.undef(torch.float64, py, device="cpu")
    cx = pa.PencilArray.undef(torch.complex128, prc, device="cpu")
    # dtypes
    with pytest.raises(ArgumentError, match="r2r_first: dest and src"):
        pa.Transposition(ry, pa.PencilArray.undef(torch.float32, pr, device="cpu"), r2r_first="REDFT10")
    with pytest.raises(ArgumentError, match="r2r_first must be one of"):
        pa.Transposition(ry, rx, r2r_first="REDFT00")
    with pytest.raises(ArgumentError, match="brfft_first: dest and src"):
        pa.Transposition(ry, pa.PencilArray.undef(torch.complex64, prc, device="cpu"), brfft_first=True)
    # the mode keywords exclude each other
    for kw in (dict(r2r_first="REDFT10", brfft_first=True), dict(r2r_first="REDFT10", r2r="REDFT10"),
               dict(brfft_first=True, rfft=True), dict(brfft_first=True, rfft_first=True),
               dict(r2r_first="REDFT01", brfft=True)):
        with pytest.raises(ArgumentError, match="exclude each other"):
            pa.Transposition(ry, rx, method=pa.PeerPut(), **kw)
    # the method: refused by the check, before the collective window setup
    for method in (pa.PointToPoint(), pa.Alltoallv(), pa.PeerGet()):
        with pytest.raises(ArgumentError, match="needs PeerPut"):
            pa.Transposition(ry, rx, r2r_first="RODFT10", method=method)
        with pytest.raises(ArgumentError, match="needs PeerPut"):
            pa.Transposition(ry, cx, brfft_first=True, method=method)
    # fft= / fft_first= with the new modes, on local transpositions (no window either)
    topo = pa.MPITopology(pa.COMM_SELF, (1,))
    lx = pa.Pencil(topo, (32, 4, 3), (2,))
    ly = pa.Pencil(lx, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
    a = pa.PencilArray.undef(torch.float64, lx, device="cpu")
    b = pa.PencilArray.undef(torch.float64, ly, device="cpu")
    c = pa.PencilArray.undef(torch.complex128, _brfft_pencil(lx), device="cpu")
    t = pa.Transposition(b, a, r2r_first="REDFT10", method=pa.PeerPut())
    tb = pa.Transposition(b, c, brfft_first=True, method=pa.PointToPoint())
    for tt in (t, tb):
        assert tt.fft_first_fusable()
        assert not tt.fft_fusable()
        with pytest.raises(ArgumentError, match="implies its transform"):
            pa.transpose_(tt, fft="forward")
        with pytest.raises(ArgumentError, match="implies its transform"):
            pa.transpose_(tt, fft_first="forward")
