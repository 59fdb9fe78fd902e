"""Shell-binned spectra (pa.shell_spectrum, DESIGN §3m) on one GPU at 512^3-class r2c shapes
(257, 512, 512): ComplexF64 and ComplexF32, with and without 3 components.  CUDA events around
the library alternated with a torch composite (a precomputed int64 bin index and weight, built
outside the timed region, then bincount(idx, weights=w * |u|^2)); the HBM fraction of the bytes
read (3.35 TB/s); the last-CTA fold on its own (the same call on a one-element-per-CTA array of
the same CTA count and nbins).  Prints the card and its power limit, then one JSON line per case.
    python profiles/prof_spectrum.py [--iters 20]"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import pencilarrays_b200 as pa  # noqa: E402
import spectrum_ref as R  # noqa: E402

HBM = 3.35e12


def timed(fn, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("card:", q)
    dims = (257, 512, 512)
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    # the z-pencil of a real 3-d transform: logical x (the r2c dim) slowest in memory
    pen = pa.Pencil(topo, dims, (1, 2), permute=pa.Permutation(3, 2, 1))
    shell = torch.from_numpy(R.shells(dims, 1)).cuda()
    wgt = torch.from_numpy(R.mode_weights(dims, 1, 512)).cuda()
    nb = pa.spectrum_nbins(pa.PencilArray.undef(torch.complex64, pen), rfft_dim=1)
    for dtype in (torch.complex128, torch.complex64):
        for extra in ((), (3,)):
            u = pa.PencilArray.undef(dtype, pen, *extra)
            u.data.copy_(torch.randn(u.data.shape, dtype=dtype, device="cuda"))
            # torch composite: index and weight, built once; the z-pencil's torch dims are the
            # logical (x, y, z), components first
            idx, w = shell.long(), wgt
            if extra:
                idx, w = idx.unsqueeze(0).expand(u.data.shape), w.unsqueeze(0).expand(u.data.shape)
            idx, w = idx.contiguous().reshape(-1), w.contiguous().reshape(-1)

            def lib_call():
                return pa.shell_spectrum(u, rfft_dim=1)

            def torch_call():
                p = torch.view_as_real(u.data).double().square().sum(-1).reshape(-1)
                return torch.bincount(idx, weights=w * p, minlength=nb)

            for _ in range(3):
                lib_call(), torch_call()
            E, T = lib_call(), torch_call()
            torch.cuda.synchronize()
            rel = float((E.double() - T).abs().max() / T.abs().max())
            tl, tt = [], []
            for _ in range(a.rounds):
                tl.append(timed(lib_call, a.iters))
                tt.append(timed(torch_call, a.iters))
            nbytes = u.data.numel() * u.data.element_size()
            # the fold alone: an array of one element per CTA the big call launches
            n = u.data.numel()
            V = 16 // u.data.element_size()
            G = min(math.ceil(n / (V * 128 * 4)), 4 * torch.cuda.get_device_properties(0).multi_processor_count)
            small = pa.Pencil(topo, (G * V, 1, 512), (2, 3))
            us = pa.PencilArray.undef(dtype, small)
            us.data.zero_()
            tf = timed(lambda: pa.shell_spectrum(us, nbins=nb), a.iters)
            print(json.dumps({"dtype": str(dtype), "extra": list(extra), "nbins": nb,
                              "bytes": nbytes, "lib_ms": min(tl), "lib_ms_all": tl,
                              "torch_ms": min(tt), "torch_ms_all": tt,
                              "speedup": min(tt) / min(tl),
                              "hbm_fraction": nbytes / (min(tl) * 1e-3) / HBM,
                              "fold_probe_ms": tf, "max_rel_diff_vs_torch": rel}), flush=True)
            del u, idx, w


if __name__ == "__main__":
    main()
