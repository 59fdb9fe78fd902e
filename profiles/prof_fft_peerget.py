#!/usr/bin/env python
"""The one-sided fused transpose + FFT (PeerGet, DESIGN §3h) on one GPU, in one process: a grid
line of R = 2, 4 and 8 ranks emulated as separate device tensors, the x -> y step of a 512^3
ComplexF64 / ComplexF32 transform, forward.  Per R and precision, the whole emulated line back
to back (CUDA events after warm-up, prof_rfft.timed):

  (a) fused:    pa_get_all_fft for every rank -- ONE kernel per rank gathers every line from the
                other ranks' src tensors and its own, transforms and stores it;
  (b) unfused:  the one-sided path without fusion for every rank -- pa_get_all (the remote blocks)
                + pa_copy_self (the self block) + fft_ in place on dst;
  (c) local:    the single-rank fused transpose_(t, fft="forward") of one array of the same global
                size (the HBM reference: the same bytes through one kernel).

Fractions are of 3.35 TB/s (H100 SXM data sheet) for 2 s n bytes (n elements of s bytes).  The
"remote" loads of the emulation hit local HBM: NVLink rates are NOT measured here.

  python profiles/prof_fft_peerget.py [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import pencilarrays_b200 as pa  # noqa: E402
from pencilarrays_b200 import _lib  # noqa: E402
from pencilarrays_b200._lib import lib, check  # noqa: E402
from pencilarrays_b200.transpositions import _Plan  # noqa: E402
from prof_rfft import card, timed  # noqa: E402

PEAK = 3350.0  # GB/s, H100 SXM HBM3 data sheet
DIMS = (512, 512, 512)


def frac(nbytes, ms):
    return round(nbytes / ms / 1e6 / PEAK, 3)


def stream():
    check(lib.pa_set_device(torch.cuda.current_device()))
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def line(R, dtype, es):
    """x-pencil (y split over R ranks) -> y-pencil (x split, y contiguous) of every rank."""
    plans, srcs, dsts = [], [], []
    for r in range(R):
        topo = pa.MPITopology(pa.Comm(r, R), (R,))
        px = pa.Pencil(topo, DIMS, (2,))
        py = pa.Pencil(px, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
        plans.append(_Plan(px, py, (), es, pa.PeerGet()))
        u = pa.PencilArray.undef(dtype, px)
        u.data.view(torch.float32 if es == 8 else torch.float64).normal_()
        srcs.append(u)
        dsts.append(pa.PencilArray.undef(dtype, py))
    return plans, srcs, dsts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}; fractions of {PEAK} GB/s", flush=True)
    rows = [dict(card=name, power_limit_and_max_sm_clock=power, peak_gbs=PEAK)]
    n = DIMS[0] * DIMS[1] * DIMS[2]
    for prec, dtype, es, flag in (("double", torch.complex128, 16, 0),
                                  ("single", torch.complex64, 8, _lib.PA_FFT_F32)):
        # (c) one rank, one array of the same global size
        topo = pa.MPITopology(pa.COMM_SELF, (1,))
        px = pa.Pencil(topo, DIMS, (2,))
        py = pa.Pencil(px, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
        ux, uy = pa.PencilArray.undef(dtype, px), pa.PencilArray.undef(dtype, py)
        ux.data.view(torch.float32 if es == 8 else torch.float64).normal_()
        t = pa.Transposition(uy, ux)
        ms_local = timed(lambda: pa.transpose_(t, fft="forward"))
        del ux, uy, t
        torch.cuda.empty_cache()
        for R in (2, 4, 8):
            plans, srcs, dsts = line(R, dtype, es)
            peer_arrs = []
            for plan in plans:
                ptrs = [srcs[plan.peer(k).world_rank].data_ptr() for k in range(1, R + 1)]
                peer_arrs.append((C.c_void_p * R)(*ptrs))

            def fused():
                st = stream()
                for r, plan in enumerate(plans):
                    check(lib.pa_get_all_fft(plan.h, C.c_void_p(srcs[r].data_ptr()), peer_arrs[r],
                                             C.c_void_p(dsts[r].data_ptr()), _lib.PA_FFT_FORWARD | flag, st))

            def unfused():
                st = stream()
                for r, plan in enumerate(plans):
                    check(lib.pa_get_all(plan.h, peer_arrs[r], C.c_void_p(dsts[r].data_ptr()), 0, st))
                    check(lib.pa_copy_self(plan.h, C.c_void_p(srcs[r].data_ptr()),
                                           C.c_void_p(dsts[r].data_ptr()), st))
                    pa.fft_(dsts[r], "forward")

            ms_a, ms_b = timed(fused), timed(unfused)
            row = dict(precision=prec, dims=DIMS, ranks=R, fused_ms=round(ms_a, 4), unfused_ms=round(ms_b, 4),
                       local_fused_ms=round(ms_local, 4), speedup=round(ms_b / ms_a, 3),
                       fused_frac=frac(2 * es * n, ms_a), unfused_frac=frac(2 * es * n, ms_b),
                       local_frac=frac(2 * es * n, ms_local))
            rows.append(row)
            print(row, flush=True)
            del plans, srcs, dsts, peer_arrs
            torch.cuda.empty_cache()
    if args.json:
        json.dump(rows, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
