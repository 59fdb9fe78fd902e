#!/usr/bin/env python
"""The send-side fused real line transforms + put (PeerPut, DESIGN §3j) on one GPU, in one process:
a grid line of R = 2, 4 and 8 ranks emulated as separate device tensors, the x -> y step of a 512^3
real transform.  Per R and precision, the whole emulated line back to back, on the same tensors in
one run (CUDA events after warm-up, prof_rfft.timed), the method of prof_fft_put.py:

  DCT-II (REDFT10), DCT-III (REDFT01):
    fused:    pa_put_all_r2r for every rank -- ONE kernel per rank loads its source lines,
              transforms them and stores the reals into every rank's dst tensor;
    unfused:  r2r_ src -> mid, then pa_put_all (the remote blocks) + pa_copy_self (the self block)
              of mid for every rank;
  c2r (brfft, N = 512 from 257 bins):
    fused:    pa_put_all_brfft from the complex src tensors;
    unfused:  brfft_ src -> mid, then pa_put_all + pa_copy_self of the reals.

Fractions are of 3.35 TB/s (H100 SXM data sheet) for the bytes read and written once.  The
"remote" stores of the emulation hit local HBM: NVLink rates are NOT measured here.

  python profiles/prof_real_put.py [--json out.json]
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
CPLX = {torch.float64: torch.complex128, torch.float32: torch.complex64}


def frac(nbytes, ms):
    return round(nbytes / ms / 1e6 / PEAK, 3)


def stream():
    check(lib.pa_set_device(torch.cuda.current_device()))
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptrs(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def line(R, dtype, es, c2r):
    """Real x-pencil (y split over R ranks, x first in memory) -> real y-pencil (x split, y
    contiguous) of every rank, the PeerPut real plan; src real (c2r: its N/2+1-bin counterpart)."""
    out = dict(put=[], src=[], mid=[], dst=[], cplx=[])
    for r in range(R):
        topo = pa.MPITopology(pa.Comm(r, R), (R,))
        px = pa.Pencil(topo, DIMS, (2,))
        py = pa.Pencil(px, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
        out["put"].append(_Plan(px, py, (), es, pa.PeerPut()))
        pc = _brfft_pencil(px)
        out["cplx"].append(pc)
        u = pa.PencilArray.undef(CPLX[dtype] if c2r else dtype, pc if c2r else px)
        u.data.view(dtype).normal_()
        out["src"].append(u)
        out["mid"].append(pa.PencilArray.undef(dtype, px))
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
    for prec, dtype, es, flag in (("double", torch.float64, 8, 0),
                                  ("single", torch.float32, 4, _lib.PA_FFT_F32)):
        for R in (2, 4, 8):
            row = dict(precision=prec, dims=DIMS, ranks=R)
            for step in ("REDFT10", "REDFT01", "c2r"):
                c2r = step == "c2r"
                L = line(R, dtype, es, c2r)
                dst_all = [ptrs([L["dst"][plan.peer(k).world_rank] for k in range(1, R + 1)])
                           for plan in L["put"]]
                kind = None if c2r else getattr(_lib, "PA_" + step)

                def fused():
                    st = stream()
                    for r, plan in enumerate(L["put"]):
                        src, dst = C.c_void_p(L["src"][r].data_ptr()), C.c_void_p(L["dst"][r].data_ptr())
                        if c2r:
                            check(lib.pa_put_all_brfft(plan.h, L["cplx"][r]._h, src, dst_all[r], dst, flag, st))
                        else:
                            check(lib.pa_put_all_r2r(plan.h, kind, src, dst_all[r], dst, flag, st))

                def unfused():
                    st = stream()
                    for r, plan in enumerate(L["put"]):
                        if c2r:
                            pa.brfft_(L["mid"][r], L["src"][r])
                        else:
                            pa.r2r_(L["mid"][r], L["src"][r], step)
                        mid = C.c_void_p(L["mid"][r].data_ptr())
                        check(lib.pa_put_all(plan.h, mid, dst_all[r], 0, st))
                        check(lib.pa_copy_self(plan.h, mid, C.c_void_p(L["dst"][r].data_ptr()), st))

                ms_f, ms_u = timed(fused), timed(unfused)
                del L, dst_all
                torch.cuda.empty_cache()
                # bytes read and written once: c2r reads N/2+1 bins and writes N reals per line
                nbytes = (n * es + (DIMS[0] // 2 + 1) * (n // DIMS[0]) * 2 * es) if c2r else 2 * n * es
                key = step.lower()
                row.update({f"{key}_put_ms": round(ms_f, 4), f"{key}_then_put_ms": round(ms_u, 4),
                            f"{key}_speedup": round(ms_u / ms_f, 3), f"{key}_put_frac": frac(nbytes, ms_f),
                            f"{key}_then_put_frac": frac(nbytes, ms_u)})
            rows.append(row)
            print(row, flush=True)
    if args.json:
        json.dump(rows, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
