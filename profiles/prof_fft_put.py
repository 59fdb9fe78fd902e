#!/usr/bin/env python
"""The send-side fused transform + put (PeerPut, DESIGN §3i) on one GPU, in one process: a grid line
of R = 2, 4 and 8 ranks emulated as separate device tensors, the x -> y step of a 512^3 transform,
forward.  Per R and precision, the whole emulated line back to back, on the same tensors in one run
(CUDA events after warm-up, prof_rfft.timed):

  (a) fused:     pa_put_all_fft for every rank -- ONE kernel per rank loads its source lines,
                 transforms them and stores the bins into every rank's dst tensor;
  (b) unfused:   fft_ in place on src, then pa_put_all (the remote blocks) + pa_copy_self (the
                 self block) for every rank;
  (c) get:       pa_get_all_fft for every rank on the PeerGet plan of the same pencils (the
                 receive-side fusion of the NEXT transform: a different step of the chain, the same
                 bytes through one kernel);
  (d) r2c:       pa_put_all_rfft from real src tensors (N = 512) against rfft_ + pa_put_all +
                 pa_copy_self of the N/2+1-bin complex arrays.

Fractions are of 3.35 TB/s (H100 SXM data sheet) for the bytes read and written once.  The
"remote" stores of the emulation hit local HBM: NVLink rates are NOT measured here.

  python profiles/prof_fft_put.py [--json out.json]
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
from pencilarrays_b200.transpositions import _Plan, _brfft_pencil  # noqa: E402
from prof_rfft import card, timed  # noqa: E402

PEAK = 3350.0  # GB/s, H100 SXM HBM3 data sheet
DIMS = (512, 512, 512)
REAL = {torch.complex128: torch.float64, torch.complex64: torch.float32}


def frac(nbytes, ms):
    return round(nbytes / ms / 1e6 / PEAK, 3)


def stream():
    check(lib.pa_set_device(torch.cuda.current_device()))
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptrs(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def line(R, dtype, es, rfft):
    """x-pencil (y split over R ranks, x first in memory) -> y-pencil (x split, y contiguous) of
    every rank; rfft: real x-pencils of N = 512 and the complex plans of N/2+1 bins."""
    out = dict(put=[], get=[], src=[], mid=[], dst=[], real=[])
    for r in range(R):
        topo = pa.MPITopology(pa.Comm(r, R), (R,))
        px = pa.Pencil(topo, DIMS, (2,))
        pc = _brfft_pencil(px) if rfft else px
        py = pa.Pencil(pc, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
        out["put"].append(_Plan(pc, py, (), es, pa.PeerPut()))
        out["get"].append(_Plan(pc, py, (), es, pa.PeerGet()))
        u = pa.PencilArray.undef(REAL[dtype] if rfft else dtype, px)
        u.data.view(REAL[dtype]).normal_()
        out["src"].append(u)
        out["real"].append(px)
        out["mid"].append(pa.PencilArray.undef(dtype, pc) if rfft else u)
        out["dst"].append(pa.PencilArray.undef(dtype, py))
    return out


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
        for R in (2, 4, 8):
            L = line(R, dtype, es, False)
            dst_all = [ptrs([L["dst"][plan.peer(k).world_rank] for k in range(1, R + 1)]) for plan in L["put"]]
            src_all = [ptrs([L["src"][plan.peer(k).world_rank] for k in range(1, R + 1)]) for plan in L["get"]]

            def fused():
                st = stream()
                for r, plan in enumerate(L["put"]):
                    check(lib.pa_put_all_fft(plan.h, C.c_void_p(L["src"][r].data_ptr()), dst_all[r],
                                             C.c_void_p(L["dst"][r].data_ptr()), _lib.PA_FFT_FORWARD | flag, st))

            def unfused():
                st = stream()
                for r, plan in enumerate(L["put"]):
                    pa.fft_(L["src"][r], "forward")
                    check(lib.pa_put_all(plan.h, C.c_void_p(L["src"][r].data_ptr()), dst_all[r], 0, st))
                    check(lib.pa_copy_self(plan.h, C.c_void_p(L["src"][r].data_ptr()),
                                           C.c_void_p(L["dst"][r].data_ptr()), st))

            def get():
                st = stream()
                for r, plan in enumerate(L["get"]):
                    check(lib.pa_get_all_fft(plan.h, C.c_void_p(L["src"][r].data_ptr()), src_all[r],
                                             C.c_void_p(L["dst"][r].data_ptr()), _lib.PA_FFT_FORWARD | flag, st))

            ms_a, ms_b, ms_c = timed(fused), timed(unfused), timed(get)
            del L, dst_all, src_all
            torch.cuda.empty_cache()
            # (d) r2c: N = 512 reals -> 257 bins per line
            Lr = line(R, dtype, es, True)
            dst_all = [ptrs([Lr["dst"][plan.peer(k).world_rank] for k in range(1, R + 1)]) for plan in Lr["put"]]

            def rfused():
                st = stream()
                for r, plan in enumerate(Lr["put"]):
                    check(lib.pa_put_all_rfft(plan.h, Lr["real"][r]._h, C.c_void_p(Lr["src"][r].data_ptr()),
                                              dst_all[r], C.c_void_p(Lr["dst"][r].data_ptr()), flag, st))

            def runfused():
                st = stream()
                for r, plan in enumerate(Lr["put"]):
                    pa.rfft_(Lr["mid"][r], Lr["src"][r])
                    check(lib.pa_put_all(plan.h, C.c_void_p(Lr["mid"][r].data_ptr()), dst_all[r], 0, st))
                    check(lib.pa_copy_self(plan.h, C.c_void_p(Lr["mid"][r].data_ptr()),
                                           C.c_void_p(Lr["dst"][r].data_ptr()), st))

            ms_d, ms_e = timed(rfused), timed(runfused)
            del Lr, dst_all
            torch.cuda.empty_cache()
            rbytes = n * es // 2 + (DIMS[0] // 2 + 1) * (n // DIMS[0]) * es  # reals read, bins written
            row = dict(precision=prec, dims=DIMS, ranks=R,
                       fft_put_ms=round(ms_a, 4), fft_then_put_ms=round(ms_b, 4), get_fft_ms=round(ms_c, 4),
                       speedup=round(ms_b / ms_a, 3), fft_put_frac=frac(2 * es * n, ms_a),
                       fft_then_put_frac=frac(2 * es * n, ms_b), get_fft_frac=frac(2 * es * n, ms_c),
                       rfft_put_ms=round(ms_d, 4), rfft_then_put_ms=round(ms_e, 4),
                       rfft_speedup=round(ms_e / ms_d, 3), rfft_put_frac=frac(rbytes, ms_d))
            rows.append(row)
            print(row, flush=True)
    if args.json:
        json.dump(rows, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
