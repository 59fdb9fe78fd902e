"""Worker of tests/test_gpu_spectrum_dims.py (launched with torch.distributed.run): spectra over
chosen dims with `world` processes on the NCCL-free communicator (they may share one GPU).

* 1-d and 2-d grids with uneven splits and ranks that own nothing; kept dims decomposed and not;
  abs2 and realdot, with and without an r2c dim and extra dims: each rank's slice within the bound
  of DESIGN §3n against math.fsum over the gathered global array, and identical bits on every
  member of a combine group;
* calls interleaved with pa.sum, pa.sum(dims=...) and pa.shell_spectrum on two streams, no host
  waits: one shared sequence and serialisation;
* refusals (the partial area, no flag window) raise on every rank.
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import pencilarrays_b200 as pa  # noqa: E402
from reduce_dims_ref import logical_view  # noqa: E402
import spectrum_ref as R  # noqa: E402
import spectrum_dims_ref as RD  # noqa: E402


def gather(x):
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, x)
    return out


def global_array(dtype, shape, seed):
    rng = np.random.default_rng(seed)
    n = int(np.prod(shape))
    x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    return x.astype(np.complex128 if dtype == torch.complex128 else np.complex64).reshape(shape)


def local_array(pen, dtype, xg, extra):
    rng = pa.range_local(pen, pa.LogicalOrder())
    u = pa.PencilArray.undef(dtype, pen, *extra)
    sl = tuple(slice(r.start - 1, r.stop - 1) for r in rng)
    logical_view(u, u.data).copy_(torch.from_numpy(np.ascontiguousarray(xg[sl])))
    return u


def as_logical(u, got, keep):
    nb = got.shape[-1]
    if not keep:
        return got.cpu().numpy()
    lv = torch.stack([logical_view(u, got[..., b]) for b in range(nb)], -1).cpu().numpy()
    return lv.reshape(tuple(lv.shape[d - 1] for d in sorted(keep)) + (nb,))


def main():
    comm = pa.comm_world(transport="ipc")
    rank, world = comm.rank, comm.size
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    checks = 0
    grids = [(world,)]
    if world in (4, 8):
        grids.append((2, world // 2))
    elif world in (2, 3):
        grids.append((1, world))
    for gi, grid in enumerate(grids):
        size = (13, 7, 5) if world < 8 else (13, 7, 3)  # uneven; with 8 ranks some own nothing
        decomp = (2,) if len(grid) == 1 else (2, 3)
        topo = pa.MPITopology(comm, grid)
        for perm, extra, dtype in (((2, 1, 3), (), torch.complex128), (None, (2,), torch.complex64),
                                   ((3, 2, 1), (3,), torch.complex128)):
            kw = {"permute": pa.Permutation(*perm)} if perm else {}
            pen = pa.Pencil(topo, size, decomp, **kw)
            xg = global_array(dtype, size + extra, seed=10 * gi + len(extra))
            yg = global_array(dtype, size + extra, seed=10 * gi + len(extra) + 5)
            u, v = local_array(pen, dtype, xg, extra), local_array(pen, dtype, yg, extra)
            rng = pa.range_local(pen, pa.LogicalOrder())
            cases = [((1, 3), (2,)), ((1,), ()), ((2, 3), (1,)), ((1, 2), (3,))]
            if extra:
                cases += [((1, 2, 3), (4,)), ((1,), (2, 4))]
            for dims, keep in cases:
                # the group: the ranks that own the same ranges along every kept dim
                key = tuple((rng[d - 1].start, rng[d - 1].stop) if d <= 3 else None for d in keep)
                for rd in (None, 1, 3):
                    for vv, yy in ((None, None), (v, yg)):
                        got = pa.shell_spectrum(u, vv, dims=dims, keep=keep, rfft_dim=rd)
                        nb = RD.default_nbins(size, dims, rd)
                        exact, absum = RD.spectrum(xg, 3, nb, dims, keep, yy, rd)
                        sl = tuple(slice(rng[d - 1].start - 1, rng[d - 1].stop - 1) if d <= 3 else
                                   slice(None) for d in keep)
                        nslab = xg.size // max(1, int(np.prod(exact.shape[:-1])))
                        RD.check(as_logical(u, got, keep), exact[sl], absum[sl], nslab, sms,
                                 dtype == torch.complex64, P=world, what=(grid, perm, dims, keep, rd))
                        mine = (key, got.cpu().numpy().tobytes())
                        for k, b in gather(mine):
                            if k == key and got.numel() > 0:
                                assert b == mine[1], (grid, perm, dims, keep, rd, "group bits")
                        checks += 1

    # ---- interleaved with pa.sum, pa.sum(dims=...) and pa.shell_spectrum on two streams ----------
    pen = pa.Pencil(pa.MPITopology(comm, (world,)), (16, 9, 10), (3,))  # z decomposed
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    arrs = [pa.PencilArray.undef(torch.complex128, pen) for _ in range(24)]
    count = np.bincount(R.shells((16, 9, 10)).reshape(-1).astype(np.int64),
                        minlength=R.default_nbins((16, 9, 10)))
    nbh = RD.default_nbins((16, 9, 10), (1, 2))
    zr = pa.range_local(pen, pa.LogicalOrder())[2]
    counth = np.bincount(RD.shells((16, 9, 10), (1, 2))[:, :, 0].reshape(-1).astype(np.int64),
                         minlength=nbh)
    torch.cuda.synchronize()
    results = []
    for i, arr in enumerate(arrs):
        with torch.cuda.stream(streams[i % 2]):
            arr.data.fill_(float(i + 1))
            results.append((pa.sum(arr, pa.abs2), pa.shell_spectrum(arr, dims=(1, 2), keep=(3,)),
                            pa.sum(arr, pa.abs2, dims=(1, 2)), pa.shell_spectrum(arr),
                            pa.shell_spectrum(arr, dims=(1,))))
    torch.cuda.synchronize()
    for i, (s, Eh, sxy, E, Ex) in enumerate(results):
        c = float((i + 1) ** 2)
        assert s.item() == c * 16 * 9 * 10, i
        assert Eh.shape == (len(zr), 1, 1, nbh), Eh.shape
        assert np.array_equal(Eh.cpu().numpy().reshape(len(zr), nbh),
                              np.broadcast_to(c * counth, (len(zr), nbh))), i
        assert bool((sxy == c * 16 * 9).all()), i
        assert np.array_equal(E.cpu().numpy(), c * count), i
        cx = np.bincount(np.abs(R.wavenumbers(16)), minlength=9)
        assert np.array_equal(Ex.cpu().numpy(), c * 9 * 10 * cx), i
        checks += 5

    # ---- refusals on every rank -----------------------------------------------------------------
    u = pa.PencilArray.undef(torch.complex128, pen)
    for kw in ({"keep": (3,), "dims": (1, 3)}, {"dims": (4,)}, {"keep": (3,), "nbins": 5000}):
        try:
            pa.shell_spectrum(u, **kw)
            raise AssertionError(f"{kw} accepted")
        except pa.ArgumentError:
            checks += 1
    big = pa.Pencil(pa.MPITopology(comm, (world,)), (4, 1024 * world, 4), (2,))
    ub = pa.PencilArray.undef(torch.complex64, big)
    try:  # 1024 kept y per rank x 4096 bins > 524288 accumulators
        pa.shell_spectrum(ub, dims=(1, 3), keep=(2,), nbins=4096)
        raise AssertionError("partial area accepted")
    except pa.ArgumentError as e:
        assert "partial area" in str(e), e
        checks += 1
    pa.set_tunable("nccl_fences", 1)
    try:
        pa.shell_spectrum(u, dims=(1, 2), keep=(3,))
        raise AssertionError("no flag window accepted")
    except pa.PencilError as e:
        assert "flag window" in str(e), e
        checks += 1
    finally:
        pa.set_tunable("nccl_fences", 0)
    assert pa.shell_spectrum(u, dims=(1, 2), keep=(3,)).shape[-1] == nbh

    dist.barrier()
    if rank == 0:
        print(f"MP_SPECTRUM_DIMS_OK world={world} checks={checks}")
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
