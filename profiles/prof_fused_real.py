#!/usr/bin/env python
"""The fused transpositions of real arrays (Transposition(..., r2r=kind) / pa_transpose_r2r and
Transposition(..., rfft=True) / pa_transpose_rfft) against the unfused pairs they replace (plain
transpose_ x->y, then r2r_ / rfft_ along y), for DCT-II, DCT-III and rfft; and the two
wall-bounded 3-d chains built with them against their unfused forms:

  mixed (DCT x, RFFT y, FFT z):  forward  3 kernels (r2r_, fused x->y + rfft, fused y->z + FFT)
                                          vs 4 (r2r_, plain x->y, rfft_, fused y->z + FFT);
                                 backward 3 kernels (fft_, fused z->y + brfft, fused y->x + DCT-III)
                                          vs 5 (fft_, plain z->y, brfft_, plain y->x, r2r_)
  all walls (DCT x, y, z):       3 kernels each way vs 5 (r2r_, then twice plain transpose + r2r_)

One GPU, one rank, both precisions, in one run; CUDA events around back-to-back calls after
warm-up (prof_rfft.timed).  The card and its power limit are printed with the numbers.  Sizes are
given as (x, y, z) with the transform of the fused step along y: 512^3 and (512, 2048, 256).

HBM bytes per line of N points, s bytes per real: 2 s N for the fused r2r and s N + 2 s (N/2+1)
for the fused rfft; the unfused pairs add a write and a read of the N reals.

  python profiles/prof_fused_real.py [--json out.json]
"""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import pencilarrays_b200 as pa  # noqa: E402
from prof_rfft import PEAK, card, frac, timed  # noqa: E402


def pencils(dims):
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px = pa.Pencil(topo, dims, (2, 3))
    py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    pyc = pa.Pencil(py, size_global=(dims[0], dims[1] // 2 + 1, dims[2]))
    pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    pz = pa.Pencil(py, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    return px, py, pyc, pzc, pz


def r(ms):
    return round(ms, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}; HBM peak used for fractions: {PEAK} GB/s",
          flush=True)
    rows = [dict(card=name, power_limit_and_max_sm_clock=power, peak_gbs=PEAK)]
    for prec, rt, ct, rs in (("double", torch.float64, torch.complex128, 8),
                             ("single", torch.float32, torch.complex64, 4)):
        for dims in ((512, 512, 512), (512, 2048, 256)):
            N = dims[1]
            nlines = dims[0] * dims[2]
            px, py, pyc, pzc, pz = pencils(dims)
            ux, u1, vx = (pa.PencilArray.undef(rt, px) for _ in range(3))
            uy, wy = pa.PencilArray.undef(rt, py), pa.PencilArray.undef(rt, py)
            uyc, uzc = pa.PencilArray.undef(ct, pyc), pa.PencilArray.undef(ct, pzc)
            ux.data.normal_()
            row = dict(precision=prec, dims=dims, N=N)

            # ---- fused step against its pair ----
            t_plain = pa.Transposition(uy, ux)
            for label, kind in (("dct2", "REDFT10"), ("dct3", "REDFT01")):
                tf = pa.Transposition(wy, ux, r2r=kind)
                ms_f = timed(lambda: pa.transpose_(tf))
                ms_p = timed(lambda: (pa.transpose_(t_plain), pa.r2r_(wy, uy, kind)))
                row[f"{label}_fused_ms"], row[f"{label}_pair_ms"] = r(ms_f), r(ms_p)
                row[f"{label}_speedup"] = round(ms_p / ms_f, 3)
                row[f"{label}_fused_frac_of_hbm"] = frac(nlines * 2 * rs * N, ms_f)
            tf = pa.Transposition(uyc, ux, rfft=True)
            ms_f = timed(lambda: pa.transpose_(tf))
            ms_p = timed(lambda: (pa.transpose_(t_plain), pa.rfft_(uyc, uy)))
            row["rfft_fused_ms"], row["rfft_pair_ms"] = r(ms_f), r(ms_p)
            row["rfft_speedup"] = round(ms_p / ms_f, 3)
            row["rfft_fused_frac_of_hbm"] = frac(nlines * (rs * N + 2 * rs * (N // 2 + 1)), ms_f)
            row["plain_xy_ms"] = r(timed(lambda: pa.transpose_(t_plain)))

            # ---- mixed chain: DCT x, RFFT y, FFT z ----
            t_yz = pa.Transposition(uzc, uyc)
            t_zy, t_yx = pa.Transposition(uyc, uzc), pa.Transposition(vx, uy)
            t_zy_b = pa.Transposition(wy, uzc, brfft=True)
            t_yx_r = pa.Transposition(vx, wy, r2r="REDFT01")
            row["mixed_fwd_3_ms"] = r(timed(lambda: (pa.r2r_(u1, ux, "REDFT10"), pa.transpose_(tf),
                                                     pa.transpose_(t_yz, fft="forward"))))
            t_xy1 = pa.Transposition(uy, u1)
            row["mixed_fwd_4_ms"] = r(timed(lambda: (pa.r2r_(u1, ux, "REDFT10"), pa.transpose_(t_xy1),
                                                     pa.rfft_(uyc, uy), pa.transpose_(t_yz, fft="forward"))))
            row["mixed_bwd_3_ms"] = r(timed(lambda: (pa.fft_(uzc, "backward"), pa.transpose_(t_zy_b),
                                                     pa.transpose_(t_yx_r))))
            row["mixed_bwd_5_ms"] = r(timed(lambda: (pa.fft_(uzc, "backward"), pa.transpose_(t_zy),
                                                     pa.brfft_(uy, uyc), pa.transpose_(t_yx),
                                                     pa.r2r_(vx, vx, "REDFT01"))))
            del uyc, uzc, t_yz, t_zy, t_zy_b, tf
            torch.cuda.empty_cache()

            # ---- all walls: DCT x, y, z ----
            uz, wz = pa.PencilArray.undef(rt, pz), pa.PencilArray.undef(rt, pz)
            t_xy_d, t_yz_d = pa.Transposition(wy, u1, r2r="REDFT10"), pa.Transposition(uz, wy, r2r="REDFT10")
            t_zy_d, t_yx_d = pa.Transposition(wy, uz, r2r="REDFT01"), pa.Transposition(vx, wy, r2r="REDFT01")
            t_yz_p, t_zy_p = pa.Transposition(wz, uy), pa.Transposition(uy, wz)
            row["walls_fwd_3_ms"] = r(timed(lambda: (pa.r2r_(u1, ux, "REDFT10"), pa.transpose_(t_xy_d),
                                                     pa.transpose_(t_yz_d))))
            row["walls_fwd_5_ms"] = r(timed(lambda: (pa.r2r_(u1, ux, "REDFT10"), pa.transpose_(t_xy1),
                                                     pa.r2r_(wy, uy, "REDFT10"), pa.transpose_(t_yz_p),
                                                     pa.r2r_(uz, wz, "REDFT10"))))
            row["walls_bwd_3_ms"] = r(timed(lambda: (pa.r2r_(wz, uz, "REDFT01"), pa.transpose_(t_zy_d),
                                                     pa.transpose_(t_yx_d))))
            row["walls_bwd_5_ms"] = r(timed(lambda: (pa.r2r_(wz, uz, "REDFT01"), pa.transpose_(t_zy_p),
                                                     pa.r2r_(wy, uy, "REDFT01"), pa.transpose_(t_yx),
                                                     pa.r2r_(vx, vx, "REDFT01"))))
            rows.append(row)
            print(row, flush=True)
            del ux, u1, vx, uy, wy, uz, wz
            del t_plain, t_yx, t_yx_r, t_xy1, t_xy_d, t_yz_d, t_zy_d, t_yx_d, t_yz_p, t_zy_p
            torch.cuda.empty_cache()
    if args.json:
        json.dump(rows, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
