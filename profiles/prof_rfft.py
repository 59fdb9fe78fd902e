#!/usr/bin/env python
"""Real-to-complex line transforms (rfft_ / brfft_) against cuFFT (torch.fft.rfft / irfft on the
same tensors -- library code, the baseline) and against this library's own complex fft_ at the
same complex line length L = N/2.  Then the real 3-d transform of a PencilFFTs real-input plan
(rfft_ + two fused transposes, and back) against torch.fft.rfftn / irfftn on the same array.
One GPU, CUDA events around back-to-back launches after warm-up, arrays >> L2.

Two numbers per cuFFT baseline:
  *_call_ms     one torch.fft call returning a fresh tensor (after warm-up the caching allocator
                makes the allocation free).  No `out=`: torch's CUDA out-variants run cuFFT into a
                temporary and copy it into `out`, an extra pass over the output.  The call still
                includes whatever torch itself adds (c2r: a copy of the input, which cuFFT's c2r
                overwrites);
  *_kernels_ms  the cuFFT kernels of that call alone (torch.profiler, CUDA activity only: every
                kernel outside torch's own `at::` kernels, memcpy / memset excluded).

HBM bytes per line: rfft_ / brfft_ 8 N + 16 (N/2+1) (no workspace); fft_ 2 * 16 L.
--single: Float32 <-> ComplexF32 (PA_FFT_F32) against cuFFT's float32 / complex64 transforms;
4 N + 8 (N/2+1) and 2 * 8 L bytes per line.

  python profiles/prof_rfft.py [--single] [--json out.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pencilarrays_b200 as pa  # noqa: E402

PEAK = 3350.0  # H100 SXM data-sheet HBM3 bandwidth (GB/s) unless MEASURED_PEAKS.json says otherwise
try:
    PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass


def timed(fn, reps=20):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def library_kernels_ms(fn, reps=10):
    """Device time per call of the kernels that are not torch's own (the cuFFT kernels), and
    their names; None when the profiler saw no such kernel."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us, names = 0.0, set()
    for e in prof.key_averages():
        k = e.key
        if "at::" in k or k.startswith("Memcpy") or k.startswith("Memset") or e.self_device_time_total <= 0:
            continue
        us += e.self_device_time_total
        names.add(k[:80])
    return (round(us / 1e3 / reps, 4) if us > 0 else None), sorted(names)


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return name, q.stdout.strip()
    except Exception as e:  # the numbers still stand, without the power limit beside them
        return name, f"unknown ({e})"


def frac(nbytes, ms):
    return round(nbytes / ms / 1e6 / PEAK, 3) if ms else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--single", action="store_true", help="Float32 / ComplexF32 instead of Float64 / ComplexF64")
    args = ap.parse_args()
    rt, ct, rs = (torch.float32, torch.complex64, 4) if args.single else (torch.float64, torch.complex128, 8)
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}; HBM peak used for fractions: {PEAK} GB/s",
          flush=True)
    rows = [dict(card=name, power_limit_and_max_sm_clock=power, peak_gbs=PEAK)]
    if args.single:
        rows[0]["precision"] = "single"
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    for dims in ((512, 512, 512), (2048, 512, 256)):
        N, L = dims[0], dims[0] // 2
        nlines = math.prod(dims[1:])
        pr = pa.Pencil(topo, dims, (2, 3))
        pc = pa.Pencil(pr, size_global=(L + 1,) + dims[1:])
        xr = pa.PencilArray.undef(rt, pr)
        xc = pa.PencilArray.undef(ct, pc)
        back = pa.PencilArray.undef(rt, pr)
        xr.data.normal_()
        pa.rfft_(xc, xr)
        nb = nlines * (rs * N + 2 * rs * (L + 1))
        ms_r = timed(lambda: pa.rfft_(xc, xr))
        ms_b = timed(lambda: pa.brfft_(back, xc))
        del back
        cr = lambda: torch.fft.rfft(xr.data, dim=-1)  # noqa: E731
        # norm="forward": the inverse unscaled, like brfft_
        cb = lambda: torch.fft.irfft(xc.data, n=N, dim=-1, norm="forward")  # noqa: E731
        ms_cr, ms_cb = timed(cr), timed(cb)
        (ms_kr, names_r), (ms_kb, names_b) = library_kernels_ms(cr), library_kernels_ms(cb)
        # the in-repo yardstick: the complex fft_ at the same line length L, same number of lines
        pl = pa.Pencil(topo, (L,) + dims[1:], (2, 3))
        u = pa.PencilArray.undef(ct, pl)
        u.data.view(rt).normal_()
        ms_f = timed(lambda: pa.fft_(u, "forward"))
        nb_f = nlines * 2 * 2 * rs * L
        del u
        r = dict(dims=dims, N=N, L=L, rfft_ms=round(ms_r, 4), rfft_frac_of_hbm=frac(nb, ms_r),
                 brfft_ms=round(ms_b, 4), brfft_frac_of_hbm=frac(nb, ms_b),
                 cufft_rfft_call_ms=round(ms_cr, 4), cufft_rfft_call_frac_of_hbm=frac(nb, ms_cr),
                 cufft_rfft_kernels_ms=ms_kr, cufft_rfft_kernels_frac_of_hbm=frac(nb, ms_kr),
                 cufft_irfft_call_ms=round(ms_cb, 4), cufft_irfft_call_frac_of_hbm=frac(nb, ms_cb),
                 cufft_irfft_kernels_ms=ms_kb, cufft_irfft_kernels_frac_of_hbm=frac(nb, ms_kb),
                 cufft_rfft_kernel_names=names_r, cufft_irfft_kernel_names=names_b,
                 fft_at_L_ms=round(ms_f, 4), fft_at_L_frac_of_hbm=frac(nb_f, ms_f))
        rows.append(r)
        print(r, flush=True)
        del xr, xc
        torch.cuda.empty_cache()

    # the real 3-d transform: rfft_ along x, then x->y and y->z with the complex transform fused;
    # backward: fft_ along z, fused z->y, plain y->x, brfft_ -- against cuFFT's own 3-d plans
    dims = (512, 512, 512)
    pxr = pa.Pencil(topo, dims, (2, 3))
    pxc = pa.Pencil(pxr, size_global=(dims[0] // 2 + 1,) + dims[1:])
    pyc = pa.Pencil(pxc, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    uxr = pa.PencilArray.undef(rt, pxr)
    uxc, uyc, uzc = (pa.PencilArray.undef(ct, p) for p in (pxc, pyc, pzc))
    uxr.data.normal_()
    t_xy, t_yz = pa.Transposition(uyc, uxc), pa.Transposition(uzc, uyc)
    t_zy, t_yx = pa.Transposition(uyc, uzc), pa.Transposition(uxc, uyc)
    ms_fwd = timed(lambda: (pa.rfft_(uxc, uxr), pa.transpose_(t_xy, fft="forward"),
                            pa.transpose_(t_yz, fft="forward")))
    ms_bwd = timed(lambda: (pa.fft_(uzc, "backward"), pa.transpose_(t_zy, fft="backward"),
                            pa.transpose_(t_yx), pa.brfft_(uxr, uxc)))
    uxr.data.normal_()
    spec = torch.fft.rfftn(uxr.data)  # (512, 512, 257): torch halves the LAST dim = x
    del uyc, uzc
    torch.cuda.empty_cache()
    cf = lambda: torch.fft.rfftn(uxr.data)  # noqa: E731
    cbk = lambda: torch.fft.irfftn(spec, s=uxr.data.shape, norm="forward")  # noqa: E731
    ms_cfwd, ms_cbwd = timed(cf), timed(cbk)
    (ms_kf, _), (ms_kbk, _) = library_kernels_ms(cf), library_kernels_ms(cbk)
    r = dict(dims=dims, what="real 3-d FFT", chain_forward_ms=round(ms_fwd, 4), chain_backward_ms=round(ms_bwd, 4),
             cufft_rfftn_call_ms=round(ms_cfwd, 4), cufft_rfftn_kernels_ms=ms_kf,
             cufft_irfftn_call_ms=round(ms_cbwd, 4), cufft_irfftn_kernels_ms=ms_kbk)
    rows.append(r)
    print(r, flush=True)
    if args.json:
        json.dump(rows, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
