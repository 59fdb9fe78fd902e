"""Per-line accuracy of the FFT kernels against the extended-precision reference
(tests/fft_ref.py), beside cuFFT (torch.fft) on the same device tensors: the table of
DESIGN.md §3b / §3c.  64 lines per length, line j scaled by 2^s (s cycling over -40..40).
--single: the PA_FFT_F32 kernels beside cuFFT complex64 / float32, inputs rounded to float32
first, errors in units of eps32 = 2^-23 (DESIGN.md §3d).

    python profiles/fft_accuracy.py [--single]   # prints a markdown table (max / RMS per-line error)
"""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import pencilarrays_b200 as pa  # noqa: E402
from fft_ref import EPS, brfft_ld, fft_ld, line_errors, rfft_ld, scaled_lines  # noqa: E402
from test_gpu_fft_exact import brfft_on_gpu, fft_lines_on_gpu, rfft_on_gpu  # noqa: E402


def fmt(e):
    return f"{e[0] / EPS:.2f} / {e[1] / EPS:.2f}"


def main_single():
    from test_gpu_fft32 import EPS32, brfft_on_gpu as brfft32, fft_lines_on_gpu as fft32, lines32, \
        rfft_on_gpu as rfft32

    def f(e):
        return f"{e[0] / EPS32:.2f} / {e[1] / EPS32:.2f}"

    print(f"# {torch.cuda.get_device_name()}; single precision, errors in units of eps32 = 2^-23, "
          "max / RMS over 64 lines")
    print("| L | fft_ fwd | fft_ bwd | cuFFT fwd | cuFFT bwd | eps32 log2 L |")
    print("|---|---|---|---|---|---|")
    for k in range(3, 11):
        L = 1 << k
        x = lines32(L, 64, L)
        dev = torch.from_numpy(x).cuda()
        row = [line_errors(fft32(x, s), fft_ld(x, s)) for s in (-1, 1)]
        row.append(line_errors(torch.fft.fft(dev).cpu().numpy(), fft_ld(x, -1)))
        row.append(line_errors(torch.fft.ifft(dev, norm="forward").cpu().numpy(), fft_ld(x, 1)))
        print(f"| {L} | " + " | ".join(f(e) for e in row) + f" | {math.log2(L):.0f} |")
    print()
    print("| N | rfft_ | brfft_ | cuFFT rfft | cuFFT irfft (unnormalised) | eps32 log2 N |")
    print("|---|---|---|---|---|---|")
    for k in range(4, 12):
        N = 1 << k
        x = lines32(N, 64, N, complex_=False)
        X = lines32(N + 1, 64, N // 2 + 1)
        Xc = X.copy()
        Xc[:, 0] = Xc[:, 0].real
        Xc[:, -1] = Xc[:, -1].real
        rf, bf = rfft_ld(x), brfft_ld(X, N)
        row = [line_errors(rfft32(x), rf), line_errors(brfft32(X, N), bf),
               line_errors(torch.fft.rfft(torch.from_numpy(x).cuda()).cpu().numpy(), rf),
               line_errors(torch.fft.irfft(torch.from_numpy(Xc).cuda(), n=N, norm="forward").cpu().numpy(), bf)]
        print(f"| {N} | " + " | ".join(f(e) for e in row) + f" | {math.log2(N):.0f} |")


def main():
    if "--single" in sys.argv[1:]:
        return main_single()
    print(f"# {torch.cuda.get_device_name()}; errors in units of eps = 2^-52, max / RMS over 64 lines")
    print("| L | fft_ fwd | fft_ bwd | fft_ fwd, fft_lines=4 | cuFFT fwd | cuFFT bwd | eps log2 L |")
    print("|---|---|---|---|---|---|---|")
    for k in range(3, 11):
        L = 1 << k
        x = scaled_lines(np.random.default_rng(L), 64, L)
        dev = torch.from_numpy(x).cuda()
        row = []
        for sign in (-1, 1):
            row.append(line_errors(fft_lines_on_gpu(x, sign), fft_ld(x, sign)))
        pa.set_tunable("fft_lines", 4)
        row.append(line_errors(fft_lines_on_gpu(x, -1), fft_ld(x, -1)))
        pa.set_tunable("fft_lines", 0)
        row.append(line_errors(torch.fft.fft(dev).cpu().numpy(), fft_ld(x, -1)))
        row.append(line_errors(torch.fft.ifft(dev, norm="forward").cpu().numpy(), fft_ld(x, 1)))
        print(f"| {L} | " + " | ".join(fmt(e) for e in row) + f" | {math.log2(L):.0f} |")
    print()
    print("| N | rfft_ | brfft_ | cuFFT rfft | cuFFT irfft (unnormalised) | eps log2 N |")
    print("|---|---|---|---|---|---|")
    for k in range(4, 12):
        N = 1 << k
        rng = np.random.default_rng(N)
        x = scaled_lines(rng, 64, N, complex_=False)
        X = scaled_lines(rng, 64, N // 2 + 1)
        Xc = X.copy()
        Xc[:, 0] = Xc[:, 0].real
        Xc[:, -1] = Xc[:, -1].real
        rf, bf = rfft_ld(x), brfft_ld(X, N)
        row = [line_errors(rfft_on_gpu(x), rf), line_errors(brfft_on_gpu(X, N), bf),
               line_errors(torch.fft.rfft(torch.from_numpy(x).cuda()).cpu().numpy(), rf),
               line_errors(torch.fft.irfft(torch.from_numpy(Xc).cuda(), n=N, norm="forward").cpu().numpy(), bf)]
        print(f"| {N} | " + " | ".join(fmt(e) for e in row) + f" | {math.log2(N):.0f} |")


if __name__ == "__main__":
    main()
