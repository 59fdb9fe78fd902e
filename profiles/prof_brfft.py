#!/usr/bin/env python
"""The fused y->x transpose + complex-to-real transform (Transposition(..., brfft=True),
pa_transpose_brfft) against the unfused pair it replaces (plain transpose_ y->x, then brfft_),
and the real backward 3-d transform of a PencilFFTs real-input plan with it (3 kernels: fft_ z,
fused z->y, fused y->x + brfft) against today's 4 kernels and cuFFT irfftn(norm="forward").
One GPU, one rank, both precisions, in one run; CUDA events around back-to-back calls after
warm-up (prof_rfft.timed).  The card and its power limit are printed with the numbers.

HBM bytes per line of the fused step: 16 M + 8 N (Float64; M = N/2+1 bins in, N reals out) or
8 M + 4 N (Float32) -- the same as brfft_ alone; the unfused pair adds a complex write and read.

  python profiles/prof_brfft.py [--json out.json]
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
from prof_rfft import PEAK, card, frac, library_kernels_ms, timed  # noqa: E402


def chain(dims):
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pxr = pa.Pencil(topo, dims, (2, 3))
    pxc = pa.Pencil(pxr, size_global=(dims[0] // 2 + 1,) + dims[1:])
    pyc = pa.Pencil(pxc, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    return pxr, pxc, pyc, pzc


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
        for dims in ((512, 512, 512), (2048, 512, 256)):
            N, M = dims[0], dims[0] // 2 + 1
            nlines = math.prod(dims[1:])
            pxr, pxc, pyc, pzc = chain(dims)
            uxr = pa.PencilArray.undef(rt, pxr)
            uxc, uyc, uzc = (pa.PencilArray.undef(ct, p) for p in (pxc, pyc, pzc))
            uxr.data.normal_()
            pa.rfft_(uxc, uxr)
            t_xy, t_yz = pa.Transposition(uyc, uxc), pa.Transposition(uzc, uyc)
            pa.transpose_(t_xy, fft="forward")
            pa.transpose_(t_yz, fft="forward")
            t_zy, t_yx = pa.Transposition(uyc, uzc), pa.Transposition(uxc, uyc)
            t_fused = pa.Transposition(uxr, uyc, brfft=True)
            nb = nlines * (2 * rs * M + rs * N)
            ms_fused = timed(lambda: pa.transpose_(t_fused))
            ms_pair = timed(lambda: (pa.transpose_(t_yx), pa.brfft_(uxr, uxc)))
            ms_t = timed(lambda: pa.transpose_(t_yx))
            ms_b = timed(lambda: pa.brfft_(uxr, uxc))
            # the whole backward chain, z-pencil spectrum -> real x-pencil field
            ms_bwd4 = timed(lambda: (pa.fft_(uzc, "backward"), pa.transpose_(t_zy, fft="backward"),
                                     pa.transpose_(t_yx), pa.brfft_(uxr, uxc)))
            ms_bwd3 = timed(lambda: (pa.fft_(uzc, "backward"), pa.transpose_(t_zy, fft="backward"),
                                     pa.transpose_(t_fused)))
            r = dict(precision=prec, dims=dims, N=N, M=M,
                     fused_yx_brfft_ms=round(ms_fused, 4), fused_frac_of_hbm=frac(nb, ms_fused),
                     plain_yx_plus_brfft_ms=round(ms_pair, 4), plain_yx_ms=round(ms_t, 4),
                     brfft_ms=round(ms_b, 4), speedup=round(ms_pair / ms_fused, 3),
                     chain_backward_3_kernels_ms=round(ms_bwd3, 4),
                     chain_backward_4_kernels_ms=round(ms_bwd4, 4))
            # cuFFT's single-GPU inverse of the same real array (no pencil transposes needed)
            del uyc, uzc, t_xy, t_yz, t_zy, t_yx, t_fused
            torch.cuda.empty_cache()
            uxr.data.normal_()
            spec = torch.fft.rfftn(uxr.data)  # torch halves the LAST dim = x
            cbk = lambda: torch.fft.irfftn(spec, s=uxr.data.shape, norm="forward")  # noqa: E731
            r["cufft_irfftn_call_ms"] = round(timed(cbk), 4)
            r["cufft_irfftn_kernels_ms"] = library_kernels_ms(cbk)[0]
            del spec
            rows.append(r)
            print(r, flush=True)
            del uxr, uxc
            torch.cuda.empty_cache()
    if args.json:
        json.dump(rows, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
