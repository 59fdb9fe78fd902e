"""The maps, ops and finalisation of the distributed reductions (pencilarrays.jl_b200/csrc/
reduce_core.hpp), run on the CPU through tests/reduce_host_check.cpp in the kernel's tree order
(per-thread runs, warp and CTA trees, the fold of the rank partials), against numpy."""
import math
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
F64, F32, C64, C32, I32, I64, BOOL = range(7)
ID, ABS, ABS2, DOT = range(4)
SUM, MAX, MIN, ANY, ALL = range(5)
EQ, NE, LT, LE, GT, GE, ISNAN, ISFINITE = (k << 4 for k in range(1, 9))
NP = {F64: np.float64, F32: np.float32, C64: np.complex128, C32: np.complex64, I32: np.int32,
      I64: np.int64}
RES = {F64: np.float64, F32: np.float32, I32: np.int32, I64: np.int64, BOOL: np.uint8}


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = os.path.join(str(tmp_path_factory.mktemp("reduce")), "reduce_host_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", out, os.path.join(HERE, "reduce_host_check.cpp")],
                   check=True)
    return out


def run(exe, dtype, f, op, a, b=None, ref=0, G=3, P=1, res=None):
    a = np.ascontiguousarray(a, dtype=NP[dtype])
    refb = np.zeros(16, np.uint8)
    if op >> 4 in range(1, 7):
        rv = np.asarray(ref, dtype=NP[dtype] if f == ID else np.real(a[:1]).dtype).tobytes()
        refb[:len(rv)] = np.frombuffer(rv, np.uint8)
    data = a.tobytes() + (np.ascontiguousarray(b, dtype=NP[dtype]).tobytes() if f == DOT else b"")
    out = subprocess.run([exe, str(dtype), str(f), str(op), str(G), str(P), str(len(a))],
                         input=data + refb.tobytes(), capture_output=True, check=True).stdout
    return np.frombuffer(out, dtype=res)[0]


def bits(x):
    return np.asarray(x).tobytes()


@pytest.mark.parametrize("dtype", [F64, F32])
def test_max_min_propagate_nan_and_order_signed_zeros(exe, dtype):
    t = NP[dtype]
    x = np.linspace(-3, 5, 3001).astype(t)
    x[1777] = np.nan
    for op in (MAX, MIN):
        for P in (1, 3):
            assert np.isnan(run(exe, dtype, ID, op, x, G=5, P=P, res=t))
            assert np.isnan(run(exe, dtype, ABS, op, x, G=5, P=P, res=t))
    for z in ([0.0, -0.0], [-0.0, 0.0], [-0.0] * 5 + [0.0] + [-0.0] * 7):
        z = np.array(z, t)
        for P in (1, 2):
            assert bits(run(exe, dtype, ID, MAX, z, P=P, res=t)) == bits(t(0.0))
            assert bits(run(exe, dtype, ID, MIN, z, P=P, res=t)) == bits(t(-0.0))
    y = np.random.default_rng(1).standard_normal(5000).astype(t)
    assert run(exe, dtype, ID, MAX, y, G=4, P=3, res=t) == y.max()
    assert run(exe, dtype, ID, MIN, y, G=4, P=3, res=t) == y.min()


def test_int32_abs2_wraps_and_sum_widens_to_int64(exe):
    x = np.array([50000, -3, 46341, 7] * 300 + [2 ** 31 - 1] * 5, np.int32)
    with np.errstate(over="ignore"):
        sq = x * x  # wraps in int32, as Julia's abs2(::Int32)
    assert run(exe, I32, ABS2, MAX, x, res=np.int32) == sq.max()
    assert run(exe, I32, ABS2, MIN, x, res=np.int32) == sq.min()
    assert run(exe, I32, ABS2, SUM, x, P=3, res=np.int64) == sq.astype(np.int64).sum()
    big = np.full(10000, 2 ** 30, np.int32)
    assert run(exe, I32, ID, SUM, big, P=2, res=np.int64) == 10000 * 2 ** 30  # > typemax(Int32)
    m = np.array([-2 ** 31, 5], np.int32)  # abs(typemin(Int32)) == typemin(Int32)
    assert run(exe, I32, ABS, MAX, m, res=np.int32) == 5
    assert run(exe, I32, ABS, MIN, m, res=np.int32) == -2 ** 31


def test_hypot_without_overflow_or_underflow(exe):
    for s in (1e300, 1e-300, 1.0, 1e-310):
        z = np.array([complex(s, s), complex(3 * s, 4 * s), complex(-s, 0.5 * s)], np.complex128)
        got = run(exe, C64, ABS, MAX, z, res=np.float64)
        assert np.isfinite(got) and got == np.abs(z).max(), (s, got, np.abs(z).max())
    rng = np.random.default_rng(7)
    z = (rng.standard_normal(20000) * 10.0 ** rng.integers(-300, 300, 20000)
         + 1j * rng.standard_normal(20000) * 10.0 ** rng.integers(-300, 300, 20000))
    for k in range(0, 20000, 1000):  # max over small groups: every abs is exercised; Borges'
        w = z[k:k + 1000]          # correction step is correctly rounded in all but rare cases
        for op, want in ((MAX, np.abs(w).max()), (MIN, np.abs(w).min())):
            got = run(exe, C64, ABS, op, w, res=np.float64)
            assert abs(got - want) <= np.spacing(want), (got, want)
    with np.errstate(over="ignore"):
        w = z.astype(np.complex64)
    w = w[np.isfinite(w)]
    assert run(exe, C32, ABS, MAX, w, res=np.float32) == np.abs(w).max()
    assert run(exe, C32, ABS, MIN, w, res=np.float32) == np.abs(w).min()


def test_float32_sums_accumulate_in_fp64(exe):
    x = np.concatenate([[1e8], np.ones(20000)]).astype(np.float32)  # fp32 steps would drop every 1
    want = np.float32(math.fsum(x.astype(np.float64)))
    assert run(exe, F32, ID, SUM, x, G=4, P=2, res=np.float32) == want
    z = (x + 1j * x[::-1]).astype(np.complex64)
    got = run(exe, C32, ID, SUM, z, G=4, P=2, res=np.complex64)
    assert got == np.complex64(complex(math.fsum(z.real.astype(np.float64)),
                                       math.fsum(z.imag.astype(np.float64))))


@pytest.mark.parametrize("dtype", [C64, C32, F64, F32, I32, I64])
def test_realdot_of_x_with_itself_is_abs2_bit_for_bit(exe, dtype):
    rng = np.random.default_rng(dtype)
    x = rng.standard_normal(4099) * 1e3
    if dtype in (C64, C32):
        x = x + 1j * rng.standard_normal(4099) * 1e3
    x = x.astype(NP[dtype])
    rt = {C64: np.float64, C32: np.float32, I32: np.int64}.get(dtype, NP[dtype])
    for op in (SUM, MAX, MIN):
        d = run(exe, dtype, DOT, op, x, x, G=3, P=2, res=rt if op == SUM else np.real(x[:1]).dtype)
        s = run(exe, dtype, ABS2, op, x, G=3, P=2, res=rt if op == SUM else np.real(x[:1]).dtype)
        assert bits(d) == bits(s), (op, d, s)


def test_float64_sum_within_the_documented_tree_depth(exe):
    rng = np.random.default_rng(3)
    x = rng.standard_normal(300001) * 10.0 ** rng.integers(-5, 5, 300001)
    G, P = 7, 3
    n_rank = len(x) // P + 1
    run_len = math.ceil(math.ceil(n_rank / 2 / G) / 256) * 2 + 2
    depth = run_len + 5 + 3 + math.ceil(G / 256) + 5 + 3 + (P - 1)
    for f, fx in ((ID, x), (ABS2, x * x)):
        got = run(exe, F64, f, SUM, x, G=G, P=P, res=np.float64)
        assert abs(got - math.fsum(fx)) <= depth * np.finfo(np.float64).eps * math.fsum(np.abs(fx))


def test_any_all_predicates(exe):
    x = np.arange(-50, 51, dtype=np.float64)
    assert run(exe, F64, ID, ANY | EQ, x, ref=7.0, res=np.uint8) == 1
    assert run(exe, F64, ID, ANY | EQ, x, ref=7.5, res=np.uint8) == 0
    assert run(exe, F64, ID, ALL | GE, x, ref=-50.0, P=3, res=np.uint8) == 1
    assert run(exe, F64, ID, ALL | GT, x, ref=-50.0, P=3, res=np.uint8) == 0
    assert run(exe, F64, ABS, ALL | LE, x, ref=50.0, res=np.uint8) == 1
    assert run(exe, F64, ID, ALL | ISFINITE, x, res=np.uint8) == 1
    y = x.copy()
    y[33] = np.inf
    assert run(exe, F64, ID, ALL | ISFINITE, y, res=np.uint8) == 0
    assert run(exe, F64, ID, ANY | ISNAN, y, res=np.uint8) == 0
    y[40] = np.nan
    assert run(exe, F64, ID, ANY | ISNAN, y, P=2, res=np.uint8) == 1
    assert run(exe, F64, ID, ANY | NE, np.full(9, np.nan), ref=np.nan, res=np.uint8) == 1  # NaN != NaN
    z = (x + 1j).astype(np.complex128)
    assert run(exe, C64, ID, ANY | EQ, z, ref=3 + 1j, res=np.uint8) == 1
    assert run(exe, C64, ID, ALL | NE, z, ref=3 + 2j, res=np.uint8) == 1
    assert run(exe, I32, ID, ALL | LT, np.arange(10, dtype=np.int32), ref=10, res=np.uint8) == 1
