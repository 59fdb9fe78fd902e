"""Reductions along dims (pa_reduce_dims, DESIGN §3l) on one GPU against torch's sum(dim=...) /
amax(abs(.), dim=...) on the local tensor: a 512^3 x-pencil of Float64, ComplexF64 and Float32,
keeping y (plane averages, also with 3 extra components), x, z, (y, z) and (x, y).  CUDA events,
the library and torch alternated, median of the rounds; read bytes over the 3.35 TB/s data-sheet
HBM bandwidth.  Prints the card and its power limit first.

    python profiles/prof_reduce_dims.py [--n 512] [--rounds 5] [--iters 10]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pencilarrays_b200 as pa  # noqa: E402

HBM = 3.35e12


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no GPU: nothing to measure")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"# {q}")
    n = args.n
    pen = pa.Pencil(pa.MPITopology(pa.COMM_SELF, (1, 1)), (n, n, n), (2, 3))  # an x-pencil
    cases = [("keep y", (1, 3), ()), ("keep y, 3 comps", (1, 3), (3,)), ("keep x", (2, 3), ()),
             ("keep z", (1, 2), ()), ("keep (y,z)", (1,), ()), ("keep (x,y)", (3,), ())]
    print("| dtype | case | sum ours ms | torch ms | ours / torch HBM | maximum(abs) ours ms | "
          "torch ms | ours / torch HBM |")
    print("|---|---|---|---|---|---|---|---|")
    for dtype in (torch.float64, torch.complex128, torch.float32):
        for name, dims, extra in cases:
            u = pa.PencilArray.undef(dtype, pen, *extra)
            u.data.copy_(torch.randn(u.data.shape, dtype=dtype, device="cuda"))
            nd = u.data.dim()
            axes = tuple(i for i in range(nd) if u.data.shape[i] != 1 and
                         pa.reductions.result_shape(u, dims)[1][i] == 1)
            x = u.data
            ours_s, torch_s, ours_m, torch_m = [], [], [], []
            for _ in range(args.rounds):
                ours_s.append(timed(lambda: pa.sum(u, dims=dims), args.iters))
                torch_s.append(timed(lambda: x.sum(dim=axes, keepdim=True), args.iters))
                ours_m.append(timed(lambda: pa.maximum(u, abs, dims=dims), args.iters))
                torch_m.append(timed(lambda: torch.amax(x.abs(), dim=axes, keepdim=True), args.iters))
            got = pa.sum(u, dims=dims)
            want = x.sum(dim=axes, keepdim=True)
            assert torch.allclose(got.to(want.dtype), want, rtol=1e-4, atol=1e-3 * n), name
            nbytes = x.numel() * x.element_size()
            med = [statistics.median(v) for v in (ours_s, torch_s, ours_m, torch_m)]
            fr = [nbytes / t / HBM for t in med]
            print(f"| {str(dtype)[6:]} | {name} | {med[0] * 1e3:.3f} | {med[1] * 1e3:.3f} | "
                  f"{fr[0]:.2f} / {fr[1]:.2f} | {med[2] * 1e3:.3f} | {med[3] * 1e3:.3f} | "
                  f"{fr[2]:.2f} / {fr[3]:.2f} |", flush=True)
            del u, x, got, want
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
