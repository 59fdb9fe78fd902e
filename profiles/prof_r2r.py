#!/usr/bin/env python
"""The real-to-real line transforms (r2r_, pa_r2r: DCT-II/III, DST-II/III) along x of real
(512, 512, 512) and (2048, 512, 256) arrays, each kind in place and out of place, against rfft_ /
brfft_ at the same N (the same N/2-point core and nearly the same bytes) and against the DCT a
user can build today from torch alone (Makhoul's reordering + torch.fft.rfft / irfft + twiddle,
eager).  One GPU, one rank, both precisions, in one run; CUDA events around back-to-back calls
after warm-up (prof_rfft.timed).  The card and its power limit are printed with the numbers.

HBM bytes per line: 2 s N (s = 8 for Float64, 4 for Float32): N reals in, N reals out.

  python profiles/prof_r2r.py [--json out.json]
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

KINDS = ["REDFT10", "REDFT01", "RODFT10", "RODFT01"]


def torch_dct2(x):
    """DCT-II (REDFT10) along the last dim from torch alone: reorder, rfft, twiddle."""
    N = x.shape[-1]
    v = torch.cat((x[..., ::2], x[..., 1::2].flip(-1)), dim=-1)
    k = torch.arange(N // 2 + 1, device=x.device, dtype=x.dtype)
    a = torch.polar(torch.ones_like(k), -math.pi * k / (2 * N)) * torch.fft.rfft(v)
    return torch.cat((2 * a.real, (-2 * a.imag[..., 1:N // 2]).flip(-1)), dim=-1)


def torch_dct3(X):
    """DCT-III (REDFT01) along the last dim from torch alone: twiddle, irfft, reorder."""
    N = X.shape[-1]
    k = torch.arange(N // 2 + 1, device=X.device, dtype=X.dtype)
    Xr = torch.cat((torch.zeros_like(X[..., :1]), X.flip(-1)[..., :N // 2]), dim=-1)  # X[N-k]
    V = torch.polar(torch.ones_like(k), math.pi * k / (2 * N)) * torch.complex(X[..., :N // 2 + 1], -Xr)
    v = torch.fft.irfft(V, n=N, norm="forward")
    return torch.stack((v[..., :N // 2], v.flip(-1)[..., :N // 2]), dim=-1).flatten(-2)


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
            N = dims[0]
            nlines = math.prod(dims[1:])
            nb = nlines * 2 * rs * N
            topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
            pr = pa.Pencil(topo, dims, (2, 3))
            pc = pa.Pencil(pr, size_global=(N // 2 + 1,) + dims[1:])
            x, y = pa.PencilArray.undef(rt, pr), pa.PencilArray.undef(rt, pr)
            x.data.normal_()
            r = dict(precision=prec, dims=dims, N=N)
            for kind in KINDS:
                ms_out = timed(lambda: pa.r2r_(y, x, kind))
                ms_in = timed(lambda: pa.r2r_(y, y, kind))
                r[f"{kind}_out_of_place_ms"] = round(ms_out, 4)
                r[f"{kind}_in_place_ms"] = round(ms_in, 4)
                r[f"{kind}_frac_of_hbm"] = frac(nb, ms_out)
            xc = pa.PencilArray.undef(ct, pc)
            ms_r = timed(lambda: pa.rfft_(xc, x))
            ms_b = timed(lambda: pa.brfft_(y, xc))
            r["rfft_ms"], r["brfft_ms"] = round(ms_r, 4), round(ms_b, 4)
            r["rfft_frac_of_hbm"] = frac(nlines * (rs * N + 2 * rs * (N // 2 + 1)), ms_r)
            del xc
            torch.cuda.empty_cache()
            # the same DCTs from torch alone, on the same parent array (lines along its last dim)
            xd = x.data
            r["torch_dct2_ms"] = round(timed(lambda: torch_dct2(xd)), 4)
            r["torch_dct3_ms"] = round(timed(lambda: torch_dct3(xd)), 4)
            pa.r2r_(y, x, "REDFT10")
            ref = torch_dct2(xd)
            r["torch_dct2_max_rel_diff"] = float((ref - y.data).abs().max() / ref.abs().max())
            del ref
            rows.append(r)
            print(r, flush=True)
            del x, y, xd
            torch.cuda.empty_cache()
    if args.json:
        json.dump(rows, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
