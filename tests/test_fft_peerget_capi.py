"""The one-sided fused transpose + FFT (PeerGet, DESIGN §3h) on the host: its check and the
`pa_get_all_fft` refusals.  No device is needed.

A PeerGet plan's `pa_plan_fft_check_ex` verdict also covers the gather of `k_get_fft` -- the
peers' get blocks read from their src arrays plus the self block read from src.  It must be one
verdict per grid line, in both precisions, on every configuration of the suite; and on these it
is the PointToPoint verdict of the same geometry (the get configuration never refuses where the
staged ones accept).  The verdicts of every other method are pinned to a table recorded before
the one-sided path existed (tests/golden/fft_check_verdicts.json)."""
import ctypes as C
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import pencilarrays_b200 as pa  # noqa: E402
from pencilarrays_b200 import _lib  # noqa: E402
from pencilarrays_b200._lib import lib  # noqa: E402
from pencilarrays_b200.transpositions import _Plan  # noqa: E402
from util import build_chain, make_ranks  # noqa: E402
from test_fft_check import ALL  # noqa: E402

OK, EINVAL, ENOGPU = _lib.PA_OK, _lib.PA_EINVAL, _lib.PA_ENOGPU
F32, FWD, BWD = _lib.PA_FFT_F32, _lib.PA_FFT_FORWARD, _lib.PA_FFT_BACKWARD
GOLDEN = os.path.join(HERE, "golden", "fft_check_verdicts.json")
METHODS = [("p2p", pa.PointToPoint()), ("a2av", pa.Alltoallv()), ("put", pa.PeerPut()),
           ("get", pa.PeerGet())]


def verdict_table(case):
    """{"step/rank": 8 digits}: the fft check of every method (METHODS order) in ComplexF64 and
    ComplexF32 on every emulated rank, and the grid line of each rank per step."""
    ranks, steps = build_chain(case)
    table, lines = {}, {}
    for k in range(1, len(steps)):
        for r in range(len(ranks)):
            codes = ""
            for _, method in METHODS:
                for f32 in (False, True):
                    plan = _Plan(steps[k - 1][r][0], steps[k][r][0], case["extra"], 8 if f32 else 16,
                                 method)
                    st = lib.pa_plan_fft_check_ex(plan.h, F32 if f32 else 0)
                    assert lib.pa_plan_fft_check_ex(plan.h, F32 if f32 else 0) == st  # cached
                    codes += str(st)
                    info = plan.info
                    line = tuple(sorted(plan.peer(n).world_rank for n in range(1, info.nproc + 1))) \
                        if info.dim else (r,)
            table[f"{k}/{r}"] = codes
            lines[(k, r)] = line
    return table, lines


_GOLD = None


def golden():
    global _GOLD
    if _GOLD is None:
        with open(GOLDEN) as f:
            _GOLD = json.load(f)
    return _GOLD


@pytest.mark.parametrize("case", ALL, ids=[c["name"] for c in ALL])
def test_peerget_verdict_is_uniform_and_other_methods_unchanged(case):
    table, lines = verdict_table(case)
    gold = golden()[case["name"]]
    assert set(table) == set(gold)
    for key, codes in table.items():
        # PointToPoint, Alltoallv and PeerPut: exactly the recorded verdicts
        assert codes[:6] == gold[key][:6], (case["name"], key, codes, gold[key])
        # PeerGet: the get gather refuses nothing the staged gathers accept (and vice versa)
        assert codes[6:8] == codes[0:2], (case["name"], key, codes)
    for (k, r), line in lines.items():
        for prec in range(2):
            got = {table[f"{k}/{q}"][6 + prec] for q in line}
            assert len(got) == 1, (case["name"], k, line, prec, got)
            assert got <= {str(OK), str(EINVAL)}


def test_the_seeded_set_exercises_both_peerget_verdicts():
    seen = set()
    for case in ALL:
        table, _ = verdict_table(case)
        seen |= {c[6] for c in table.values()} | {c[7] for c in table.values()}
    assert seen == {str(OK), str(EINVAL)}


# ---- pa_get_all_fft refusals --------------------------------------------------------------
def line_plans(nproc, L, other=(4, 3), extra=(), elsize=16, method=None):
    """x-pencil decomposed along x over `nproc` ranks -> y-pencil with x local and contiguous:
    each destination line of L points is gathered from `nproc` blocks."""
    method = method or pa.PeerGet()
    out = []
    for er in make_ranks((nproc,)):
        px = pa.Pencil(er.topo, (L,) + other, (1,), permute=pa.Permutation(2, 1, 3))
        py = pa.Pencil(px, decomp_dims=(2,), permute=pa.NoPermutation())
        out.append(_Plan(px, py, extra, elsize, method))
    return out


class HostBuf:
    """Aligned host addresses: every refusal returns before the pointers are touched."""

    def __init__(self, nbytes):
        self.raw = C.create_string_buffer(nbytes + 256)
        self.base = (C.addressof(self.raw) + 255) // 256 * 256

    def at(self, off):
        return C.c_void_p(self.base + off)


def call(plan, src, peers, dst, flags):
    arr = (C.c_void_p * len(peers))(*[p.value if p is not None else None for p in peers]) \
        if peers is not None else None
    return lib.pa_get_all_fft(plan.h if plan else None, src, arr, dst, flags, None)


def setup(nproc=3, L=64, elsize=16, method=None):
    plans = line_plans(nproc, L, other=(nproc + 1, 3), elsize=elsize, method=method)
    plan = plans[1]
    info = plan.info
    nin, nout = info.length_in * elsize, info.length_out * elsize
    ain, aout = (nin + 255) // 256 * 256, (nout + 255) // 256 * 256  # keep every array 256-aligned
    buf = HostBuf(ain + aout + nproc * ain * 4)
    src, dst = buf.at(0), buf.at(ain)
    peers = [buf.at(ain + aout + 4 * ain * n) for n in range(nproc)]
    return plan, src, peers, dst, nin, nout


def no_gpu():
    return lib.pa_device_count() == 0


@pytest.mark.parametrize("flags", [0, FWD | BWD, F32, FWD | _lib.PA_WAITALL, BWD | _lib.PA_STAGE_SELF,
                                   FWD | 64, 1 << 31])
def test_bad_flags(flags):
    plan, src, peers, dst, _, _ = setup()
    assert call(plan, src, peers, dst, flags) == EINVAL
    assert lib.pa_last_error().startswith(b"pa_get_all_fft: flags")


def test_host_refusals():
    plan, src, peers, dst, nin, nout = setup()
    assert call(None, src, peers, dst, FWD) == EINVAL
    # a purely local plan has nothing to get
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px = pa.Pencil(topo, (16, 8, 4), (2, 3))
    py = pa.Pencil(px, decomp_dims=(2, 3), permute=pa.Permutation(2, 1, 3))
    assert call(_Plan(px, py, (), 16, pa.PeerGet()), src, peers, dst, FWD) == EINVAL
    assert b"no exchange" in lib.pa_last_error()
    # the plan's verdict first: lines of 48 points, ComplexF32 flag on a ComplexF64 plan
    p48, s48, pe48, d48, _, _ = setup(L=48)
    assert call(p48, s48, pe48, d48, FWD) == EINVAL
    assert b"power of two" in lib.pa_last_error()
    assert call(plan, src, peers, dst, FWD | F32) == EINVAL
    assert b"ComplexF32" in lib.pa_last_error()
    # pointers: a missing peer array, src of a non-empty self block, misalignment, overlap
    assert call(plan, src, None, dst, FWD) == EINVAL
    assert call(plan, src, [peers[0], peers[1], None], dst, FWD) == EINVAL
    assert b"peer 3" in lib.pa_last_error()
    assert call(plan, None, peers, dst, BWD) == EINVAL
    assert call(plan, src, [C.c_void_p(peers[0].value + 8)] + peers[1:], dst, FWD) == EINVAL
    assert b"aligned" in lib.pa_last_error()
    assert call(plan, src, peers, C.c_void_p(dst.value + 8), FWD) == EINVAL
    assert call(plan, src, peers, C.c_void_p(src.value + 16), FWD) == EINVAL
    assert b"overlap" in lib.pa_last_error()
    # the self entry of `peers` is ignored (plan 1 is rank 2 of the line)
    if no_gpu():
        assert call(plan, src, [peers[0], None, peers[2]], dst, FWD) == ENOGPU


def test_valid_arguments_without_a_device_give_enogpu():
    if not no_gpu():
        pytest.skip("GPU present")
    for elsize, prec in ((16, 0), (8, F32)):
        for method in (pa.PeerGet(), pa.PointToPoint()):
            plan, src, peers, dst, _, _ = setup(nproc=6, L=1024, elsize=elsize, method=method)
            for d in (FWD, BWD):
                assert call(plan, src, peers, dst, d | prec) == ENOGPU, (elsize, method, d)


def test_empty_destination_accepts_null_pointers():
    """y = 3 over 4 ranks: rank 1 owns no y-pencil lines and rank 4's src is empty."""
    if not no_gpu():
        pytest.skip("GPU present")
    plans = line_plans(4, 16, other=(3, 2))
    for plan in plans:
        info = plan.info
        peers = [None if plan.peer(n).recv_count == 0 else C.c_void_p(1 << 20)
                 for n in range(1, 5)]
        src = C.c_void_p(1 << 24) if info.length_in else None
        dst = C.c_void_p(1 << 28) if info.length_out else None
        assert call(plan, src, peers, dst, FWD) == ENOGPU, lib.pa_last_error()


if __name__ == "__main__":
    # record the verdict table with the library on sys.path (tests/golden/fft_check_verdicts.json)
    out = {c["name"]: verdict_table(c)[0] for c in ALL}
    with open(sys.argv[1], "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
