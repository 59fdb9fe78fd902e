"""Worker of tests/test_gpu_reduce.py (launched with torch.distributed.run): global reductions with
`world` processes on the NCCL-free communicator (they may share one GPU), or on an NCCL
communicator without its flag window when PA_REDUCE_NCCL=1 (the ncclAllGather fallback).

* the first reduction on the communicator returns without waiting for the device;
* the port of test/reductions.jl: Int32 filled with 2 myid; minimum, maximum, minimum(abs2),
  maximum(abs2); sum and sum(abs2) equal to the sum of the per-rank values; the complex
  two-array case (a == b, and a copy); any / all with == and >;
* Float64 and ComplexF64 results identical on every rank and equal to the rank-order fold of the
  per-rank one-rank results;
* a grid with ranks that own nothing;
* 100 back-to-back reductions with a different value each call, alternating two streams, no host
  waits, every result checked; the same interleaved with PeerPut transposes on the communicator.
"""
import math
import os
import struct
import sys

import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import pencilarrays_b200 as pa  # noqa: E402
from gpu_util import hold, hold_cycles  # noqa: E402


def gather(x):
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, x)
    return out


def bits(t):
    return t.cpu().numpy().tobytes()


def local_result(fn, u, *args):
    """The one-rank reduction of this rank's local array (a one-rank pencil over its parent)."""
    mem = tuple(reversed(u.data.shape))[:3]
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    p = pa.Pencil(topo, mem, (2, 3))
    return fn(pa.PencilArray(p, u.data, u.extra_dims), *args)


def jl_max(x, y):
    if math.isnan(x):
        return x
    if math.isnan(y):
        return y
    return y if (y > x or (math.copysign(1, y) < math.copysign(1, x))) else x


def main():
    nccl = os.environ.get("PA_REDUCE_NCCL") == "1"
    comm = pa.comm_world(transport="nccl" if nccl else "ipc")
    if nccl:
        pa.set_tunable("nccl_fences", 1)  # no flag window: the ncclAllGather fallback
    rank, world = comm.rank, comm.size
    myid = rank + 1
    checks = 0
    for r in range(world):  # calibrate the spin one process at a time: the GPU is shared
        if r == rank:
            hold_cycles()
        dist.barrier()

    # ---- the first reduction on the communicator (it sets up its workspace) does not wait for
    #      the device: it is queued behind a spin and returns while the spin still runs
    pen0 = pa.Pencil(pa.MPITopology(comm, (world, 1)), (16, 21, 41), (2, 3))
    f = pa.PencilArray.undef(torch.float64, pen0)
    f.data.fill_(0.0)
    # (CUDA loads a kernel's module at its first launch, and that load waits for the device: the
    #  same kernel runs once on a one-rank pencil first, which uses the device's own workspace)
    local_result(pa.sum, f)
    torch.cuda.synchronize()
    dist.barrier()
    held = hold()
    f.data.fill_(float(myid))
    first = pa.sum(f)
    assert not held.query(), "the first reduction synchronised the host"
    torch.cuda.synchronize()
    assert first.item() == sum(n * m for n, m in gather((f.data.numel(), myid)))
    checks += 1

    # ---- test/reductions.jl --------------------------------------------------------------
    pen = pa.Pencil((16, 32, 14), comm)
    u = pa.PencilArray.undef(torch.int32, pen)
    u.data.fill_(2 * myid)
    assert pa.minimum(u).item() == 2
    assert pa.maximum(u).item() == 2 * world
    assert pa.minimum(u, pa.abs2).item() == 4
    assert pa.maximum(u, pa.abs2).item() == (2 * world) ** 2
    s = pa.sum(u)
    assert s.dtype == torch.int64
    assert s.item() == sum(gather(int(u.data.to(torch.int64).sum())))
    assert pa.sum(u, pa.abs2).item() == sum(gather(int((u.data.to(torch.int64) ** 2).sum())))
    uh = pa.PencilArray(pen, u.data.to(torch.complex128) * (1 + 1j))
    vh = pa.PencilArray(pen, uh.data.clone())
    a = pa.sum(uh, pa.abs2)
    b = pa.mapreduce(pa.realdot, "+", uh, vh)
    c = pa.mapreduce(pa.realdot, "+", uh, uh)
    assert a.dtype == torch.float64 and bits(a) == bits(b) == bits(c)
    assert a.item() == sum(gather(2.0 * float((u.data.to(torch.float64) ** 2).sum())))
    assert pa.any(u, "==", 2).item() is True
    assert pa.any(u, "==", -2).item() is False
    assert pa.all(u, "==", 2).item() is (world == 1)
    assert pa.all(u, ">", 0).item() is True
    checks += 14

    # ---- Float64 / ComplexF64: same bits everywhere, = the rank-order fold of rank results ----
    pen2 = pa.Pencil(pa.MPITopology(comm, (world, 1)), (16, 21, 41), (2, 3),
                     permute=pa.Permutation(3, 1, 2))
    g = torch.Generator(device="cuda").manual_seed(100 + rank)
    x = pa.PencilArray.undef(torch.float64, pen2, 2)
    x.data.copy_(torch.randn(x.data.shape, generator=g, device="cuda", dtype=torch.float64))
    z = pa.PencilArray.undef(torch.complex128, pen2, 2)
    z.data.copy_(torch.randn(z.data.shape, generator=g, device="cuda", dtype=torch.complex128))
    for fn, arr, args in ((pa.sum, x, ()), (pa.sum, x, (pa.abs2,)), (pa.maximum, x, (abs,)),
                          (pa.minimum, x, ()), (pa.sum, z, ()), (pa.sum, z, (abs,)),
                          (pa.maximum, z, (abs,))):
        got = fn(arr, *args)
        allbits = gather(bits(got))
        assert all(bb == allbits[0] for bb in allbits), (fn.__name__, args)
        parts = gather(bits(local_result(fn, arr, *args)))
        if got.dtype == torch.complex128:
            vals = [complex(*struct.unpack("<2d", p)) for p in parts]
            acc = complex(0.0, 0.0)
            for v in vals:
                acc = complex(acc.real + v.real, acc.imag + v.imag)
            want = struct.pack("<2d", acc.real, acc.imag)
        else:
            vals = [struct.unpack("<d", p)[0] for p in parts]
            if fn is pa.sum:
                acc = 0.0
                for v in vals:
                    acc = acc + v
            else:
                acc = -math.inf if fn is pa.maximum else math.inf
                for v in vals:
                    acc = jl_max(acc, v) if fn is pa.maximum else -jl_max(-acc, -v)
            want = struct.pack("<d", acc)
        assert allbits[0] == want, (fn.__name__, args, allbits[0], want)
        checks += 1

    # ---- ranks that own nothing ------------------------------------------------------------
    pen3 = pa.Pencil(pa.MPITopology(comm, (world, 1)), (5, 7, 3), (3, 2))
    e = pa.PencilArray.undef(torch.float64, pen3)
    e.data.fill_(float(myid))
    owners = gather((e.data.numel(), myid))
    assert world < 4 or any(n == 0 for n, _ in owners)
    assert pa.sum(e).item() == sum(n * m for n, m in owners)
    assert pa.maximum(e).item() == max(m for n, m in owners if n)
    assert pa.minimum(e).item() == min(m for n, m in owners if n)
    assert pa.all(e, ">", 0).item() is True and pa.any(e, "isnan").item() is False
    checks += 4

    # ---- 100 back-to-back calls, two streams, no host waits -------------------------------------
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    arrs = [pa.PencilArray.undef(torch.int64, pen2) for _ in range(100)]
    lens = gather(arrs[0].data.numel())
    torch.cuda.synchronize()
    results = []
    for i, arr in enumerate(arrs):
        with torch.cuda.stream(streams[i % 2]):
            arr.data.fill_(i * 1000 + rank)
            results.append(pa.sum(arr))
    torch.cuda.synchronize()
    for i, r in enumerate(results):
        assert r.item() == sum(n * (i * 1000 + q) for q, n in enumerate(lens)), i
    checks += 100

    # ---- interleaved with PeerPut transposes on the same communicator ----------------------------
    if not nccl:
        py = pa.Pencil(pen2, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
        ux = pa.PencilArray.undef(torch.float64, pen2)
        uy = pa.PencilArray.undef(torch.float64, py)
        back = pa.PencilArray.undef(torch.float64, pen2)
        ux.data.copy_(torch.randn(ux.data.shape, generator=g, device="cuda", dtype=torch.float64))
        want_sum = pa.sum(ux)
        for i in range(20):
            with torch.cuda.stream(streams[i % 2]):
                pa.transpose_(uy, ux, method=pa.PeerPut())
                s1 = pa.sum(uy)
                pa.transpose_(back, uy, method=pa.PeerPut())
                s2 = pa.maximum(back, abs)
            torch.cuda.synchronize()
            assert torch.equal(back.data, ux.data), i
            assert abs(s1.item() - want_sum.item()) <= 1e-12 * pa.sum(ux, abs).item(), i
            assert s2.item() == max(gather(ux.data.abs().max().item())), i
            checks += 3

    dist.barrier()
    if rank == 0:
        print(f"MP_REDUCE_OK world={world} nccl={int(nccl)} checks={checks}")
    dist.destroy_process_group()


if __name__ == "__main__":
    try:
        main()
    except BaseException:
        import traceback
        tb = traceback.format_exc()
        sys.stderr.write("".join(f"WORKER-ERROR[{os.environ.get('RANK', '?')}] {l}\n"
                                 for l in tb.splitlines()))
        sys.stderr.flush()
        os._exit(1)
