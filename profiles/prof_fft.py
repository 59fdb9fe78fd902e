#!/usr/bin/env python
"""Fused unpack+FFT (PA_FFT_FORWARD) against the unfused pair it replaces:
transpose! (K3) followed by a batched 1-d FFT along the new contiguous dim
(cuFFT through torch.fft -- library code, the baseline).  One GPU, ComplexF64,
CUDA events around back-to-back launches, arrays >> L2.  --single: the same in
ComplexF32 (PA_FFT_F32) against cuFFT complex64; tunable fft_lines does not apply there.

  python profiles/prof_fft.py [--single] [--json out.json]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pencilarrays_b200 as pa  # noqa: E402

PEAK = 3350.0  # H100 SXM data-sheet HBM3 bandwidth (GB/s) unless MEASURED_PEAKS.json says otherwise
try:
    PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass


def timed(fn, reps=5):
    for _ in range(2):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--single", action="store_true", help="ComplexF32 instead of ComplexF64")
    args = ap.parse_args()
    ct, rt, es = (torch.complex64, torch.float32, 8) if args.single else (torch.complex128, torch.float64, 16)
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    rows = [dict(card=torch.cuda.get_device_name(), precision="single")] if args.single else []
    for dims in ((512, 512, 512), (256, 256, 256), (256, 1024, 256), (1024, 256, 256)):
        px = pa.Pencil(topo, dims, (2, 3))
        py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
        pz = pa.Pencil(py, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
        ux, uy, uz = (pa.PencilArray.undef(ct, p) for p in (px, py, pz))
        ux.data.view(rt).normal_()
        uy.data.view(rt).normal_()
        nb = 2 * ux.data.numel() * es
        for leg, dst, src in (("x->y", uy, ux), ("y->z", uz, uy)):
            t = pa.Transposition(dst, src)
            L = dst.data.shape[-1]
            tmp = torch.empty_like(dst.data)
            ms_t = timed(lambda: pa.transpose_(t))
            ms_f = timed(lambda: torch.fft.fft(dst.data, dim=-1, out=tmp))
            ms_tf = timed(lambda: (pa.transpose_(t), torch.fft.fft(dst.data, dim=-1, out=tmp)))
            ms_fused = timed(lambda: pa.transpose_(t, fft="forward"))
            ms_fused4 = None
            if not args.single:
                pa.set_tunable("fft_lines", 4)
                ms_fused4 = round(timed(lambda: pa.transpose_(t, fft="forward")), 4)
                pa.set_tunable("fft_lines", 0)
            r = dict(dims=dims, leg=leg, L=L, transpose_ms=round(ms_t, 4), cufft_ms=round(ms_f, 4),
                     unfused_ms=round(ms_tf, 4), fused_ms=round(ms_fused, 4), fused_4lines_ms=ms_fused4,
                     fused_frac_of_hbm=round(nb / ms_fused / 1e6 / PEAK, 3),
                     speedup_vs_unfused=round(ms_tf / ms_fused, 3))
            rows.append(r)
            print(r, flush=True)
    # a whole 3-d transform of a 512^3 ComplexF64 pencil set on one GPU: in-place fft along x,
    # then x->y and y->z with the next transform fused -- against cuFFT's own 3-d plan on the
    # same array (library code; it needs no pencil transposes on a single GPU)
    dims = (512, 512, 512)
    px = pa.Pencil(topo, dims, (2, 3))
    py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    pz = pa.Pencil(py, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    ux, uy, uz = (pa.PencilArray.undef(ct, p) for p in (px, py, pz))
    ux.data.view(rt).normal_()
    t1, t2 = pa.Transposition(uy, ux), pa.Transposition(uz, uy)
    tmp = torch.empty_like(ux.data)
    ms_line = timed(lambda: pa.fft_(ux, "forward"))
    ms_3d = timed(lambda: (pa.fft_(ux, "forward"), pa.transpose_(t1, fft="forward"),
                           pa.transpose_(t2, fft="forward")))
    ms_unfused = timed(lambda: (torch.fft.fft(ux.data, dim=-1, out=tmp), pa.transpose_(t1),
                                torch.fft.fft(uy.data, dim=-1, out=uy.data), pa.transpose_(t2),
                                torch.fft.fft(uz.data, dim=-1, out=uz.data)))
    ms_cufft3d = timed(lambda: torch.fft.fftn(ux.data, out=tmp))
    nb = 2 * ux.data.numel() * es
    r = dict(dims=dims, what="3-d FFT", in_place_line_fft_ms=round(ms_line, 4),
             in_place_line_fft_frac_of_hbm=round(nb / ms_line / 1e6 / PEAK, 3),
             fused_3d_ms=round(ms_3d, 4), unfused_pencil_3d_ms=round(ms_unfused, 4),
             cufft_fftn_single_gpu_ms=round(ms_cufft3d, 4))
    rows.append(r)
    print(r, flush=True)
    if args.json:
        json.dump(rows, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
