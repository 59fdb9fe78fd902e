#!/usr/bin/env python
"""Global reductions (pa_reduce): the local kernel on one rank against torch's best single-pass
equivalent on the same tensors, and the latency of the cross-rank combine.

1. One rank, arrays of 64 MiB .. 2 GiB of every element type, for sum, sum(abs2) and
   maximum(abs): CUDA events around back-to-back calls after warm-up, the library and torch
   alternated round by round (median of the rounds).  torch: torch.sum, torch.linalg.vector_norm(x)
   ** 2 (integers: torch.sum(x * x)), torch.amax(x.abs()).  HBM fraction = bytes read / time over
   the 3.35 TB/s data-sheet bandwidth of the H100 SXM.
2. The combine: a one-element-per-rank sum across 2 / 4 / 8 processes sharing the GPU on the
   NCCL-free communicator (torch.distributed.run), microseconds per call over 200 back-to-back calls.

The card and its power limit are printed with the numbers.

  python profiles/prof_reduce.py [--json out.json] [--skip-combine]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import pencilarrays_b200 as pa  # noqa: E402
from prof_rfft import card, timed  # noqa: E402

PEAK_GBS = 3350.0  # H100 SXM data sheet, HBM3
TYPES = [torch.float64, torch.float32, torch.complex128, torch.complex64, torch.int32, torch.int64]
SIZES_MIB = [64, 256, 1024, 2048]


def torch_best(op, x):
    if op == "sum":
        return lambda: torch.sum(x)
    if op == "sum(abs2)":
        if x.dtype.is_floating_point or x.dtype.is_complex:
            return lambda: torch.linalg.vector_norm(x) ** 2
        return lambda: torch.sum(x * x)
    return lambda: torch.amax(x.abs())


def ours(op, u):
    if op == "sum":
        return lambda: pa.sum(u)
    if op == "sum(abs2)":
        return lambda: pa.sum(u, pa.abs2)
    return lambda: pa.maximum(u, abs)


def local_kernel(rows, rounds):
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    for dtype in TYPES:
        es = torch.empty(0, dtype=dtype).element_size()
        for mib in SIZES_MIB:
            n = (mib << 20) // es
            pen = pa.Pencil(topo, (n // 1024, 32, 32), (2, 3))
            u = pa.PencilArray.undef(dtype, pen)
            if dtype.is_floating_point or dtype.is_complex:
                u.data.normal_()
            else:
                u.data.random_(-1000, 1000)
            for op in ("sum", "sum(abs2)", "maximum(abs)"):
                a, b = ours(op, u), torch_best(op, u.data)
                ta, tb = [], []
                for _ in range(rounds):  # alternate the two
                    ta.append(timed(a, reps=10))
                    tb.append(timed(b, reps=10))
                ma, mb = statistics.median(ta), statistics.median(tb)
                nbytes = n * es
                row = dict(dtype=str(dtype).replace("torch.", ""), MiB=mib, op=op, ms=round(ma, 4),
                           hbm_frac=round(nbytes / ma / 1e6 / PEAK_GBS, 3), torch_ms=round(mb, 4),
                           torch_hbm_frac=round(nbytes / mb / 1e6 / PEAK_GBS, 3),
                           speedup=round(mb / ma, 3))
                rows.append(row)
                print(json.dumps(row), flush=True)
            del u


COMBINE_WORKER = r"""
import os, sys, json, torch, torch.distributed as dist
sys.path.insert(0, os.environ["PA_ROOT"])
import pencilarrays_b200 as pa
comm = pa.comm_world(transport="ipc")
pen = pa.Pencil(pa.MPITopology(comm, (comm.size, 1)), (comm.size, 1, 1), (1, 2))
u = pa.PencilArray.undef(torch.float64, pen)
u.data.fill_(1.0)
for _ in range(20):
    pa.sum(u)
torch.cuda.synchronize()
dist.barrier()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
for _ in range(200):
    r = pa.sum(u)
b.record()
torch.cuda.synchronize()
assert r.item() == comm.size
us = a.elapsed_time(b) / 200 * 1e3
out = [None] * comm.size
dist.all_gather_object(out, us)
if comm.rank == 0:
    print("COMBINE " + json.dumps(dict(ranks=comm.size, us_per_call=[round(x, 1) for x in out])))
dist.destroy_process_group()
"""


def combine(rows, tmpdir):
    path = os.path.join(tmpdir, "prof_reduce_combine.py")
    with open(path, "w") as f:
        f.write(COMBINE_WORKER)
    for nproc in (2, 4, 8):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(29811 + nproc), path]
        env = dict(os.environ, OMP_NUM_THREADS="1", PA_ROOT=ROOT)
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
        line = [l for l in out.stdout.splitlines() if l.startswith("COMBINE ")]
        if out.returncode != 0 or not line:
            raise RuntimeError(out.stderr[-2000:])
        row = json.loads(line[0][len("COMBINE "):])
        rows.append(row)
        print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--skip-combine", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_reduce.py measures on the GPU; there is none here")
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}; HBM peak for fractions: {PEAK_GBS} GB/s",
          flush=True)
    rows = [dict(card=name, power_limit_and_max_sm_clock=power, peak_gbs=PEAK_GBS)]
    local_kernel(rows, args.rounds)
    if not args.skip_combine:
        import tempfile
        with tempfile.TemporaryDirectory() as d:
            combine(rows, d)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
