"""The r2c post-pass and c2r pre-pass of the real-line transforms (rfft_ / brfft_), from the
shared host/device FFT core (pencilarrays.jl_b200/csrc/fft_core.hpp), run on the CPU through
tests/rfft_host_check.cpp in the kernels' order, against numpy.fft.rfft / N * irfft."""
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
NS = [1 << k for k in range(4, 12)]  # 16 ... 2048


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = os.path.join(str(tmp_path_factory.mktemp("rfft")), "rfft_host_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", out, os.path.join(HERE, "rfft_host_check.cpp")],
                   check=True)
    return out


def run(exe, n, sign, data):
    out = subprocess.run([exe, str(n), str(sign)], input=data.tobytes(), capture_output=True,
                         check=True).stdout
    return np.frombuffer(out, dtype=np.float64 if sign > 0 else np.complex128)


def tol(n, ref):
    return 8 * np.finfo(np.float64).eps * np.log2(n) * np.abs(ref).max()


@pytest.mark.parametrize("n", NS)
def test_r2c_matches_numpy_rfft(exe, n):
    rng = np.random.default_rng(n)
    for x in (rng.standard_normal(n), np.cos(2 * np.pi * 3 * np.arange(n) / n) + 0.25):
        y = run(exe, n, -1, x)
        ref = np.fft.rfft(x)
        assert y.shape == (n // 2 + 1,)
        assert np.abs(y - ref).max() <= tol(n, ref)


@pytest.mark.parametrize("n", NS)
def test_c2r_matches_numpy_irfft_unnormalised(exe, n):
    rng = np.random.default_rng(1000 + n)
    X = rng.standard_normal(n // 2 + 1) + 1j * rng.standard_normal(n // 2 + 1)
    # bins 0 and N/2 carry non-zero imaginary parts: they must be ignored, as numpy ignores them
    assert X[0].imag != 0 and X[-1].imag != 0
    y = run(exe, n, 1, X)
    ref = n * np.fft.irfft(X, n=n)
    assert y.shape == (n,)
    assert np.abs(y - ref).max() <= tol(n, ref)
    # same answer as with those imaginary parts zeroed
    Xr = X.copy()
    Xr[0], Xr[-1] = X[0].real, X[-1].real
    assert np.abs(run(exe, n, 1, Xr) - y).max() <= tol(n, ref)


@pytest.mark.parametrize("n", [16, 256, 2048])
def test_round_trip(exe, n):
    x = np.random.default_rng(7).standard_normal(n)
    back = run(exe, n, 1, run(exe, n, -1, x)) / n
    assert np.abs(back - x).max() <= tol(n, x) * 2
