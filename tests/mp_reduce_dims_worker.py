"""Worker of tests/test_gpu_reduce_dims.py (launched with torch.distributed.run): reductions along
dims with `world` processes on the NCCL-free communicator (they may share one GPU).

* 1-d and 2-d grids with uneven splits and ranks that own nothing, every subset of dims, sum,
  maximum(abs), any and the two-array realdot: each rank's result equals the global reduction sliced to its kept ranges, group members hold the same
  bits, and Float64 / Int64 results are the rank-order fold of the members' one-rank results;
* interleaved pa_reduce / pa_reduce_dims calls on two streams, no host waits, every result checked;
* refusals (bad dims, the partial-area capacity, no flag window) raise on every rank.
"""
import itertools
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import pencilarrays_b200 as pa  # noqa: E402
from reduce_dims_ref import expect, check, logical_view  # noqa: E402


def gather(x):
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, x)
    return out


def subsets(n):
    return [s for k in range(1, n + 1) for s in itertools.combinations(range(1, n + 1), k)]


def global_array(dtype, shape, seed):
    """The same global array (logical order, extra dims last) on every rank."""
    rng = np.random.default_rng(seed)
    n = int(np.prod(shape))
    if dtype.is_floating_point:
        x = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 3, n)
    else:
        x = rng.integers(-60000, 60000, n)
    return x.astype(torch.empty(0, dtype=dtype).numpy().dtype).reshape(shape)


def local_array(pen, dtype, xg, extra):
    """This rank's PencilArray of the global array xg, and its logical-order ranges."""
    rng = pa.range_local(pen, pa.LogicalOrder())
    u = pa.PencilArray.undef(dtype, pen, *extra)
    sl = tuple(slice(r.start - 1, r.stop - 1) for r in rng)  # (1-based ranges)
    view = logical_view(u, u.data)
    view.copy_(torch.from_numpy(np.ascontiguousarray(xg[sl])))
    return u, sl


def one_rank(u, fn, dims, *args):
    """The reduction of this rank's local array alone: a one-rank pencil over its parent, with the
    same memory layout (identity permutation, so logical dim m + 1 is memory dim m)."""
    N = len(u.space_dims)
    mem = tuple(reversed(u.data.shape))[:N]
    perm = pa.permutations.as_tuple(u.pencil.perm, N)
    p = pa.Pencil(pa.MPITopology(pa.COMM_SELF, (1, 1)), mem, (2, 3))
    d = tuple(perm.index(l) + 1 if l <= N else l for l in dims)
    return fn(pa.PencilArray(p, u.data, u.extra_dims), *args, dims=d)


def main():
    comm = pa.comm_world(transport="ipc")
    rank, world = comm.rank, comm.size
    checks = 0
    grids = [(world,)]
    if world in (4, 8):
        grids.append((2, world // 2))
    elif world in (2, 3):
        grids.append((1, world))
    for gi, grid in enumerate(grids):
        size = (13, 7, 5) if world < 8 else (13, 7, 3)  # uneven; with 8 ranks some own nothing
        decomp = (2,) if len(grid) == 1 else (2, 3)
        for perm, extra, dtype in (((2, 1, 3), (), torch.float64), (None, (2,), torch.int64),
                                   ((3, 2, 1), (3,), torch.float32)):
            topo = pa.MPITopology(comm, grid)
            kw = {"permute": pa.Permutation(*perm)} if perm else {}
            pen = pa.Pencil(topo, size, decomp, **kw)
            xg = global_array(dtype, size + extra, seed=10 * gi + len(extra))
            u, sl = local_array(pen, dtype, xg, extra)
            yg = global_array(dtype, size + extra, seed=10 * gi + len(extra) + 5)
            v, _ = local_array(pen, dtype, yg, extra)
            for dims in subsets(3 + len(extra)):
                # realdot of two arrays (an inner product along dims, e.g. a Reynolds stress)
                got = pa.mapreduce(pa.realdot, "+", u, v, dims=dims)
                want, tol = expect(xg, pa.realdot, "+", dims, y=yg)
                ksl = tuple(slice(0, 1) if (i + 1) in dims else s
                            for i, s in enumerate(sl + tuple(slice(0, e) for e in extra)))
                check(logical_view(u, got).cpu().numpy(), want[ksl],
                      tol[ksl] if tol is not None else None, (grid, perm, dims, "realdot"))
                checks += 1
                for fn, f, op, args in ((pa.sum, None, "+", ()), (pa.maximum, abs, "max", (abs,)),
                                        (pa.any, None, "any", (">", 10))):
                    got = fn(u, *args, dims=dims)
                    if op == "any":
                        want, tol = expect(xg, None, "any", dims, ">", 10)
                    else:
                        want, tol = expect(xg, f, op, dims)
                    ksl = tuple(slice(0, 1) if (i + 1) in dims else s
                                for i, s in enumerate(sl + tuple(slice(0, e) for e in extra)))
                    want = want[ksl]
                    tol = tol[ksl] if tol is not None else None
                    check(logical_view(u, got).cpu().numpy(), want, tol, (grid, perm, dims, op))
                    # group members (same kept ranges) hold the same bits
                    key = tuple(s for i, s in enumerate(ksl) if (i + 1) not in dims)
                    mine = got.cpu().numpy().tobytes()
                    for k2, b2 in gather((repr(key), mine)):
                        if k2 == repr(key):
                            assert b2 == mine, (grid, dims, op)
                    # the rank-order fold of the members' one-rank results (accumulator = result type)
                    if op == "+" and dtype != torch.float32:
                        parts = gather((repr(key), one_rank(u, fn, dims, *args).cpu().numpy()))
                        acc = np.zeros(got.shape, got.cpu().numpy().dtype)
                        for k2, p in parts:
                            if k2 == repr(key):
                                acc = acc + p
                        assert acc.tobytes() == mine, (grid, dims)
                    checks += 1

    # ---- interleaved pa_reduce / pa_reduce_dims on two streams, no host waits ----------------
    pen = pa.Pencil(pa.MPITopology(comm, (world,)), (16, 9, 10), (3,))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    arrs = [pa.PencilArray.undef(torch.int64, pen) for _ in range(40)]
    nz = gather(arrs[0].data.shape[0])  # local z extent per rank
    torch.cuda.synchronize()
    results = []
    for i, arr in enumerate(arrs):
        with torch.cuda.stream(streams[i % 2]):
            arr.data.fill_(i * 1000 + rank)
            results.append((pa.sum(arr), pa.sum(arr, dims=(3,)), pa.sum(arr, dims=(1, 2))))
    torch.cuda.synchronize()
    for i, (s, sz, sxy) in enumerate(results):
        assert s.item() == sum(16 * 9 * n * (i * 1000 + q) for q, n in enumerate(nz)), i
        assert bool((sz == sum(n * (i * 1000 + q) for q, n in enumerate(nz))).all()), i
        assert bool((sxy == 16 * 9 * (i * 1000 + rank)).all()), i
        checks += 3

    # ---- refusals on every rank ---------------------------------------------------------------
    u = pa.PencilArray.undef(torch.float64, pen)
    for bad in ((), (0,), (4,), (1, 1)):
        try:
            pa.sum(u, dims=bad)
            raise AssertionError(f"dims {bad} accepted")
        except pa.ArgumentError:
            checks += 1
    big = pa.Pencil(pa.MPITopology(comm, (world,)), (1030, 520, world), (3,))
    ub = pa.PencilArray.undef(torch.float64, big)
    try:
        pa.sum(ub, dims=(3,))
        raise AssertionError("partial larger than the area accepted")
    except pa.ArgumentError as e:
        assert "partial area" in str(e), e
        checks += 1
    pa.set_tunable("nccl_fences", 1)
    try:
        pa.sum(u, dims=(1,))
        raise AssertionError("no flag window accepted")
    except pa.PencilError as e:
        assert "flag window" in str(e), e
        checks += 1
    finally:
        pa.set_tunable("nccl_fences", 0)
    assert pa.sum(u, dims=(1,)).shape == (u.data.shape[0], 9, 1)

    dist.barrier()
    if rank == 0:
        print(f"MP_REDUCE_DIMS_OK world={world} checks={checks}")
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
