"""The single-precision instantiation of the shared FFT core (fft_core.hpp with T = float, the
code the PA_FFT_F32 kernels run) on the CPU through tests/fft32_host_check.cpp, per line against
the extended-precision reference (tests/fft_ref.py).  The inputs are rounded to float32 first and
those exact values go to the reference, so the error measured is the core's own."""
import os
import subprocess

import numpy as np
import pytest

from fft_ref import brfft_ld, extended_precision_available, fft_ld, line_errors, rfft_ld, scaled_lines

HERE = os.path.dirname(os.path.abspath(__file__))
LS = [1 << k for k in range(3, 11)]   # 8 ... 1024
NS = [1 << k for k in range(4, 12)]   # 16 ... 2048
EPS32 = float(np.finfo(np.float32).eps)

pytestmark = pytest.mark.skipif(not extended_precision_available(),
                                reason="np.longdouble is not extended precision on this platform")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = os.path.join(str(tmp_path_factory.mktemp("fft32")), "fft32_host_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", out, os.path.join(HERE, "fft32_host_check.cpp")],
                   check=True)
    return out


def run(exe, args, data, dtype):
    out = subprocess.run([exe] + [str(a) for a in args], input=np.ascontiguousarray(data).tobytes(),
                         capture_output=True, check=True).stdout
    return np.frombuffer(out, dtype=dtype)


@pytest.mark.parametrize("L", LS)
def test_complex_core_accuracy_per_line(exe, L):
    """Every L in 8..1024, both directions; at 1024 points also with a radix-16 first pass."""
    x = scaled_lines(np.random.default_rng(300 + L), 8, L).astype(np.complex64)
    for logR1 in [0] + ([4] if L == 1024 else []):
        for sign in (-1, 1):
            got = np.stack([run(exe, ["c", L, sign] + ([logR1] if logR1 else []), l, np.complex64)
                            for l in x])
            assert got.shape == x.shape
            mx, _ = line_errors(got, fft_ld(x, sign))
            assert mx <= EPS32 * np.log2(L), (L, sign, logR1, mx / EPS32)


@pytest.mark.parametrize("N", NS)
def test_real_core_accuracy_per_line(exe, N):
    rng = np.random.default_rng(400 + N)
    x = scaled_lines(rng, 8, N, complex_=False).astype(np.float32)
    got = np.stack([run(exe, ["r", N, -1], l, np.complex64) for l in x])
    assert got.shape == (8, N // 2 + 1)
    mx, _ = line_errors(got, rfft_ld(x))
    assert mx <= EPS32 * np.log2(N), (N, "r2c", mx / EPS32)
    X = scaled_lines(rng, 8, N // 2 + 1).astype(np.complex64)
    assert np.all(X[:, 0].imag != 0) and np.all(X[:, -1].imag != 0)
    got = np.stack([run(exe, ["r", N, 1], l, np.float32) for l in X])
    assert got.shape == (8, N)
    mx, _ = line_errors(got, brfft_ld(X, N))
    assert mx <= EPS32 * np.log2(N), (N, "c2r", mx / EPS32)
    # the imaginary parts of bins 0 and N/2 are ignored bit for bit
    Xr = X.copy()
    Xr[:, 0] = Xr[:, 0].real
    Xr[:, -1] = Xr[:, -1].real
    clean = np.stack([run(exe, ["r", N, 1], l, np.float32) for l in Xr])
    assert clean.tobytes() == got.tobytes()


def test_single_precision_is_not_double_precision(exe):
    """The fp32 core rounds like fp32: far from the reference in double-precision units, yet
    inside its own gate (a double-precision build behind the flag would pass the gates above
    without this)."""
    L = 256
    x = scaled_lines(np.random.default_rng(5), 8, L).astype(np.complex64)
    got = np.stack([run(exe, ["c", L, -1], l, np.complex64) for l in x])
    mx, rms = line_errors(got, fft_ld(x, -1))
    assert rms > 0.1 * EPS32 and mx <= EPS32 * np.log2(L)
