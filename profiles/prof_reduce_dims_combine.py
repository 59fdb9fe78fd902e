"""Combine latency of pa_reduce_dims (DESIGN §3l) with P processes on the NCCL-free communicator.
Run as ``python -m torch.distributed.run --nproc-per-node=P profiles/prof_reduce_dims_combine.py``.

Two results, each combined over all P ranks (z is decomposed and reduced, the kept dims are not):
a small one (64 outputs: keep y of a 64 x 64 x 8P Float64 pencil) and one at the partial area's
capacity (524288 outputs: keep (x, y) of a 1024 x 512 x P pencil, one plane per rank).  For each,
the time per call of 50 back-to-back calls (CUDA events, median of 5 rounds, max over ranks), and
the same call on a one-rank pencil over the local array (the local pass alone, no combine).  With
processes sharing one GPU the contexts are time-sliced, so the P > 1 numbers measure the slices.
"""
import os
import statistics
import subprocess
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pencilarrays_b200 as pa  # noqa: E402


def timed(fn, iters=50):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    dist.barrier()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    comm = pa.comm_world(transport="ipc")
    rank, P = comm.rank, comm.size
    if rank == 0:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True).stdout.strip()
        print(f"# {q}; {P} processes on GPU {torch.cuda.current_device()}", flush=True)
    for name, size, dims in (("small (64 outputs)", (64, 64, 8 * P), (1, 3)),
                             ("capacity (524288 outputs)", (1024, 512, P), (3,))):
        pen = pa.Pencil(pa.MPITopology(comm, (P,)), size, (3,))
        u = pa.PencilArray.undef(torch.float64, pen)
        u.data.normal_()
        mem = tuple(reversed(u.data.shape))
        one = pa.PencilArray(pa.Pencil(pa.MPITopology(pa.COMM_SELF, (1, 1)), mem, (2, 3)), u.data)
        full, local = [], []
        for _ in range(5):
            full.append(timed(lambda: pa.sum(u, dims=dims)))
            local.append(timed(lambda: pa.sum(one, dims=dims)))
        out = [None] * P
        dist.all_gather_object(out, (statistics.median(full), statistics.median(local)))
        if rank == 0:
            f = max(o[0] for o in out)
            l = max(o[1] for o in out)
            print(f"| {P} | {name} | {f:.3f} | {l:.3f} |", flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
