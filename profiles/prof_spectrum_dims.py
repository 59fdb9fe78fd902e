"""Spectra over chosen dims (pa.shell_spectrum(dims=, keep=), DESIGN §3n) on one GPU at the 512^3
r2c shape (257, 512, 512), x the r2c dim, ComplexF64 and ComplexF32:
  kh_y_zpencil   E(k_h; y): dims (1, 3), keep (2,) on the z-pencil (z fastest, y in the middle)
  kh_y_xpencil   the same on the x-pencil (x fastest): the kept dim is not the fastest either
  kyz_x_xpencil  dims (2, 3), keep (1,) on the x-pencil: the kept dim is the fastest memory dim
  kx_zpencil     E(k_x): dims (1,), y and z summed
  comp_zpencil   per-component E_i(k) of 3 components: dims (1, 2, 3), keep (4,)
CUDA events around the library call alternated with a torch composite (an int64 index
kept_index * nbins + bin and a weight, built outside the timed region, then bincount of
w * |u|^2) and with pa.shell_spectrum (every dim binned) on the same array.  Prints the card and
its power limit, then one JSON line per case.
    python profiles/prof_spectrum_dims.py [--iters 20] [--rounds 3]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import pencilarrays_b200 as pa  # noqa: E402
from reduce_dims_ref import logical_view  # noqa: E402

HBM = 3.35e12


def timed(fn, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def composite_index(u, dims, keep, rfft_dim, nb):
    """(index, weight) in u.data's layout: (row-major kept index over the kept dims in logical
    order) * nb + bin, dropped modes at the end (an extra slot), and the Hermitian weight."""
    N = len(u.space_dims)
    size = tuple(pa.size_global(u.pencil, pa.LogicalOrder())) + tuple(u.extra_dims)
    dev = u.data.device
    q = torch.zeros(size[:N], dtype=torch.float64, device=dev)
    wt = torch.ones(size[:N], dtype=torch.float64, device=dev)
    for d in range(N):
        n = size[d]
        i = torch.arange(n, device=dev)
        k = (i if d + 1 == rfft_dim else torch.where(i < (n + 1) // 2, i, i - n)).double()
        sh = [1] * N
        sh[d] = n
        if d + 1 in dims:
            q = q + (k * k).reshape(sh)
        if d + 1 == rfft_dim:
            w = torch.full((n,), 2.0, dtype=torch.float64, device=dev)
            w[0] = 1.0
            w[n - 1] = 1.0  # (the real length 2 (n - 1) is even)
            wt = wt * w.reshape(sh)
    b = torch.floor(torch.sqrt(q) + 0.5).long()
    pad = (1,) * (len(size) - N)
    b = b.reshape(b.shape + pad).expand(size)
    wt = wt.reshape(wt.shape + pad).expand(size)
    o = torch.zeros(size, dtype=torch.int64, device=dev)
    stride = 1
    for d in sorted(keep, reverse=True):
        sh = [1] * len(size)
        sh[d - 1] = size[d - 1]
        o = o + torch.arange(size[d - 1], device=dev).reshape(sh) * stride
        stride *= size[d - 1]
    idx = torch.where(b < nb, o * nb + b, stride * nb)
    it = torch.empty(u.data.shape, dtype=torch.int64, device=dev)
    wd = torch.empty(u.data.shape, dtype=torch.float64, device=dev)
    logical_view(u, it).copy_(idx)
    logical_view(u, wd).copy_(wt)
    return it.reshape(-1), wd.reshape(-1), stride


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("card:", q, flush=True)
    dims3 = (257, 512, 512)
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    zpen = pa.Pencil(topo, dims3, (1, 2), permute=pa.Permutation(3, 2, 1))
    xpen = pa.Pencil(topo, dims3, (2, 3))
    cases = [("kh_y_zpencil", zpen, (), (1, 3), (2,)), ("kh_y_xpencil", xpen, (), (1, 3), (2,)),
             ("kyz_x_xpencil", xpen, (), (2, 3), (1,)), ("kx_zpencil", zpen, (), (1,), ()),
             ("comp_zpencil", zpen, (3,), (1, 2, 3), (4,))]
    for dtype in (torch.complex128, torch.complex64):
        for name, pen, extra, dims, keep in cases:
            u = pa.PencilArray.undef(dtype, pen, *extra)
            u.data.copy_(torch.randn(u.data.shape, dtype=dtype, device="cuda"))
            nb = pa.spectrum_nbins(u, rfft_dim=1, dims=dims)
            idx, w, nk = composite_index(u, dims, keep, 1, nb)

            def lib_call():
                return pa.shell_spectrum(u, rfft_dim=1, dims=dims, keep=keep)

            def full_call():
                return pa.shell_spectrum(u, rfft_dim=1)

            def torch_call():
                p = torch.view_as_real(u.data).double().square().sum(-1).reshape(-1)
                return torch.bincount(idx, weights=w * p, minlength=nk * nb + 1)[:nk * nb]

            for _ in range(3):
                lib_call(), full_call(), torch_call()
            E, T = lib_call(), torch_call()
            torch.cuda.synchronize()
            if keep:
                E = torch.stack([logical_view(u, E[..., b]) for b in range(nb)], -1)
            E = E.reshape(-1).double()
            rel = float((E - T).abs().max() / T.abs().max())
            tl, tf, tt = [], [], []
            for _ in range(a.rounds):
                tl.append(timed(lib_call, a.iters))
                tf.append(timed(full_call, a.iters))
                tt.append(timed(torch_call, a.iters))
            nbytes = u.data.numel() * u.data.element_size()
            print(json.dumps({"case": name, "dtype": str(dtype), "dims": list(dims),
                              "keep": list(keep), "nbins": nb, "kept_outputs": nk, "bytes": nbytes,
                              "lib_ms": min(tl), "lib_ms_all": tl, "shell_ms": min(tf),
                              "shell_ms_all": tf, "torch_ms": min(tt), "torch_ms_all": tt,
                              "speedup_vs_torch": min(tt) / min(tl),
                              "ratio_to_shell": min(tl) / min(tf),
                              "hbm_fraction": nbytes / (min(tl) * 1e-3) / HBM,
                              "max_rel_diff_vs_torch": rel}), flush=True)
            del u, idx, w, E, T
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
