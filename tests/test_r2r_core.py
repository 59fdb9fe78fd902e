"""The real-to-real pair steps (DCT-II post step, DCT-III pre step) of the shared host/device FFT
core (pencilarrays.jl_b200/csrc/fft_core.hpp), run on the CPU through tests/r2r_host_check.cpp in
the r2r kernel's order, in double and in float, for all four kinds and every N in 16..2048,
against scipy.fft.dct / dst per line."""
import os
import subprocess

import numpy as np
import pytest
import scipy.fft as sf

from fft_ref import line_errors, scaled_lines

HERE = os.path.dirname(os.path.abspath(__file__))
NS = [1 << k for k in range(4, 12)]  # 16 ... 2048
KINDS = {"REDFT10": 5, "REDFT01": 4, "RODFT10": 9, "RODFT01": 8}
EPS = {"d": float(np.finfo(np.float64).eps), "f": float(np.finfo(np.float32).eps)}
DT = {"d": np.float64, "f": np.float32}


def scipy_r2r(x, kind):
    fn = sf.dct if kind.startswith("RE") else sf.dst
    return fn(np.asarray(x, dtype=np.float64), type=2 if kind.endswith("10") else 3, axis=-1)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = os.path.join(str(tmp_path_factory.mktemp("r2r")), "r2r_host_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", out, os.path.join(HERE, "r2r_host_check.cpp")],
                   check=True)
    return out


def run(exe, prec, kind, x):
    x = np.ascontiguousarray(x, dtype=DT[prec])
    out = subprocess.run([exe, prec, str(KINDS[kind]), str(x.shape[-1])], input=x.tobytes(),
                         capture_output=True, check=True).stdout
    return np.frombuffer(out, dtype=DT[prec]).reshape(x.shape)


@pytest.mark.parametrize("prec", ["d", "f"])
@pytest.mark.parametrize("N", NS)
def test_every_kind_matches_scipy_per_line(exe, prec, N):
    """8 lines scaled by 2^s (the inputs rounded to the precision first, so the reference sees
    the same values): per-line relative 2-norm error within eps log2(N)."""
    x = scaled_lines(np.random.default_rng(500 + N), 8, N, complex_=False).astype(DT[prec])
    for kind in KINDS:
        got = run(exe, prec, kind, x)
        mx, _ = line_errors(got, scipy_r2r(x, kind))
        assert mx <= EPS[prec] * np.log2(N), (kind, N, prec, mx / EPS[prec])


@pytest.mark.parametrize("prec", ["d", "f"])
@pytest.mark.parametrize("N", [16, 256, 2048])
def test_round_trips_are_2N_times_the_input(exe, prec, N):
    x = np.random.default_rng(N).standard_normal((4, N)).astype(DT[prec])
    for fwd, bwd in (("REDFT10", "REDFT01"), ("RODFT10", "RODFT01")):
        back = run(exe, prec, bwd, run(exe, prec, fwd, x)).astype(np.float64) / (2 * N)
        assert np.abs(back - x).max() <= 4 * EPS[prec] * np.log2(N) * np.abs(x).max(), (fwd, N, prec)
