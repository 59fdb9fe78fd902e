#!/usr/bin/env python
"""Per-kernel roofline at the BASELINE shapes on ONE GPU.

Rank 0 of the 8-rank process grid is emulated for geometry only
(`Comm(0, 8)` -- no exchange happens): its pack (K1) and unpack (K2) blocks of
configs[3] (1024^3 ComplexF64, grid (4,2)) and configs[4]
(2048x1024x1024 Float32, perms None->(2,3,1)->(3,1,2)) are launched through the
C ABI exactly as `pa_transpose` launches them, each timed alone with CUDA
events (3 warm-ups, 10 timed launches, buffers >> L2).  configs[1]
(256^3 Float64, 1 GPU) runs as the fused K3 kernel for every permutation.

  python profiles/prof_kernels.py [--quick] [--json out.json]
Under ncu use --quick (one launch per kernel).
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pencilarrays_b200 as pa  # noqa: E402
from pencilarrays_b200._lib import lib, check  # noqa: E402
from pencilarrays_b200.transpositions import _Plan  # noqa: E402

PEAK = 3350.0  # H100 SXM data-sheet HBM3 bandwidth (GB/s) unless MEASURED_PEAKS.json says otherwise
try:
    PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass


def timed(fn, quick):
    if quick:
        fn()
        torch.cuda.synchronize()
        return float("nan")
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(10):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 10


def run_config(name, nranks, grid, dims, chain, elsize, quick, rows):
    comm = pa.Comm(0, nranks)
    topo = pa.MPITopology(comm, grid)
    pens = []
    for i, (d, p) in enumerate(chain):
        perm = pa.NoPermutation() if p is None else pa.Permutation(*p)
        pens.append(pa.Pencil(topo, dims, d, permute=perm) if i == 0 else
                    pa.Pencil(pens[0], decomp_dims=d, permute=perm))
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.pa_set_device(torch.cuda.current_device()))
    for k in range(1, len(pens)):
        plan = _Plan(pens[k - 1], pens[k], (), elsize, pa.PointToPoint())
        info = plan.info
        src = torch.empty(max(1, info.length_in * elsize), dtype=torch.uint8, device="cuda").random_()
        dst = torch.empty(max(1, info.length_out * elsize), dtype=torch.uint8, device="cuda")
        leg = f"{name} leg{k} {chain[k-1][1]}->{chain[k][1]}"
        if info.dim == 0 or info.nproc == 1:
            ms = timed(lambda: check(lib.pa_copy_self(plan.h, C.c_void_p(src.data_ptr()),
                                                      C.c_void_p(dst.data_ptr()), st)), quick)
            nb = 2 * info.length_in * elsize
            rows.append(dict(kernel="K3 fused", leg=leg, block="self", bytes=nb, ms=ms,
                             GBps=nb / ms / 1e6, frac=nb / ms / 1e6 / PEAK,
                             klass=plan.block(2).kernel_class))
            continue
        send = torch.empty(max(1, info.send_bytes), dtype=torch.uint8, device="cuda")
        recv = torch.empty(max(1, info.recv_bytes), dtype=torch.uint8, device="cuda").random_()
        for op, label in ((0, "K1 pack"), (1, "K2 unpack")):
            tot_b, tot_ms = 0, 0.0
            for p in range(1, info.nproc + 1):
                peer = plan.peer(p)
                if op == 0:
                    f = lambda: check(lib.pa_pack(plan.h, p, C.c_void_p(src.data_ptr()), C.c_void_p(
                        recv.data_ptr() if peer.is_self else send.data_ptr()), st))
                    nb = 2 * (peer.recv_count if peer.is_self else peer.send_count)
                else:
                    f = lambda: check(lib.pa_unpack(plan.h, p, C.c_void_p(recv.data_ptr()),
                                                    C.c_void_p(dst.data_ptr()), st))
                    nb = 2 * peer.recv_count
                ms = timed(f, quick)
                tot_b += nb
                tot_ms += ms
                rows.append(dict(kernel=label, leg=leg, block=f"peer{p}{'(self)' if peer.is_self else ''}",
                                 bytes=nb, ms=ms, GBps=nb / ms / 1e6, frac=nb / ms / 1e6 / PEAK,
                                 klass=plan.block(op, p).kernel_class))
            rows.append(dict(kernel=label, leg=leg, block="ALL", bytes=tot_b, ms=tot_ms,
                             GBps=tot_b / tot_ms / 1e6, frac=tot_b / tot_ms / 1e6 / PEAK, klass=-1))
        ms = timed(lambda: check(lib.pa_copy_self(plan.h, C.c_void_p(src.data_ptr()),
                                                  C.c_void_p(dst.data_ptr()), st)), quick)
        nb = 2 * info.length_self * elsize
        rows.append(dict(kernel="K3 fused", leg=leg, block="self", bytes=nb, ms=ms, GBps=nb / ms / 1e6,
                         frac=nb / ms / 1e6 / PEAK, klass=plan.block(2).kernel_class))
        del src, dst, send, recv
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--json", default=None)
    ap.add_argument("--only", default=None)
    ap.add_argument("--tunable", action="append", default=[], help="name=value for pa_set_tunable")
    a = ap.parse_args()
    for tv in a.tunable:
        k, v = tv.split("=")
        check(lib.pa_set_tunable(k.encode(), int(v)))
    rows = []
    X, Y, Z = (2, 3), (1, 3), (1, 2)
    cfgs = [
        ("cfg4 1024^3 c128 (4,2) fft-perms", 8, (4, 2), (1024,) * 3, [(X, None), (Y, (2, 1, 3)), (Z, (3, 2, 1))], 16),
        ("cfg4 1024^3 c128 (4,2) no-perm", 8, (4, 2), (1024,) * 3, [(X, None), (Y, None), (Z, None)], 16),
        ("cfg5 2048x1024x1024 f32 (4,2)", 8, (4, 2), (2048, 1024, 1024), [(X, None), (Y, (2, 3, 1)), (Z, (3, 1, 2))], 4),
        ("cfg3 512^3 c128 (2,1)", 2, (2, 1), (512,) * 3, [(X, None), (Y, (2, 1, 3)), (Z, (3, 2, 1))], 16),
    ]
    for p in [(2, 1, 3), (2, 3, 1), (3, 2, 1), (3, 1, 2), (1, 3, 2), None]:
        cfgs.append((f"cfg2 256^3 f64 1 GPU perm {p}", 1, (1, 1), (256,) * 3, [(X, None), (Y, p)], 8))
    for c in cfgs:
        if a.only and a.only not in c[0]:
            continue
        run_config(*c, a.quick, rows)
    for r in rows:
        print(f"{r['leg']:58s} {r['kernel']:10s} {r['block']:12s} class={r['klass']:2d} "
              f"{r['bytes']/2**20:9.1f} MiB  {r['ms']:8.4f} ms  {r['GBps']:8.1f} GB/s  {100*r['frac']:5.1f}% of measured HBM")
    if a.json:
        json.dump(dict(peak_GBps=PEAK, rows=rows), open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
