"""Worker of tests/test_gpu_spectrum.py (launched with torch.distributed.run): shell-binned spectra
with `world` processes on the NCCL-free communicator (they may share one GPU).

* 1-d and 2-d grids with uneven splits and ranks that own nothing, abs2 and realdot, with and
  without an r2c dim and extra dims: every rank holds the same bits, each bin within the bound of
  DESIGN §3m against math.fsum over the gathered global array;
* spectra interleaved with pa_reduce / pa_reduce_dims on two streams, no host waits;
* Parseval through the distributed real chain (rfft_ and two fused transposes) on 2 and 4 ranks;
* refusals (bad nbins, no flag window) raise on every rank.
"""
import math
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
        for perm, extra, dtype in (((2, 1, 3), (), torch.complex128), (None, (2,), torch.complex64),
                                   ((3, 2, 1), (3,), torch.complex128)):
            topo = pa.MPITopology(comm, grid)
            kw = {"permute": pa.Permutation(*perm)} if perm else {}
            pen = pa.Pencil(topo, size, decomp, **kw)
            xg = global_array(dtype, size + extra, seed=10 * gi + len(extra))
            yg = global_array(dtype, size + extra, seed=10 * gi + len(extra) + 5)
            u, v = local_array(pen, dtype, xg, extra), local_array(pen, dtype, yg, extra)
            for rd in (None, 1, 3):
                for vv, yy in ((None, None), (v, yg)):
                    got = pa.shell_spectrum(u, vv, rfft_dim=rd)
                    nb = R.default_nbins(size, rd)
                    assert got.shape == (nb,)
                    exact, absum = R.spectrum(xg, 3, nb, yy, rd)
                    R.check_bins(got.cpu().numpy(), exact, absum, u.data.numel(), sms,
                                 dtype == torch.complex64, P=world, what=(grid, perm, rd))
                    mine = got.cpu().numpy().tobytes()
                    assert all(b == mine for b in gather(mine)), (grid, perm, rd, "bits")
                    checks += 1

    # ---- interleaved with pa_reduce / pa_reduce_dims on two streams, no host waits -------------
    pen = pa.Pencil(pa.MPITopology(comm, (world,)), (16, 9, 10), (3,))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    arrs = [pa.PencilArray.undef(torch.complex128, pen) for _ in range(30)]
    shell = R.shells((16, 9, 10))
    count = np.bincount(shell.reshape(-1).astype(np.int64), minlength=R.default_nbins((16, 9, 10)))
    torch.cuda.synchronize()
    results = []
    for i, arr in enumerate(arrs):
        with torch.cuda.stream(streams[i % 2]):
            arr.data.fill_(float(i + 1))
            results.append((pa.sum(arr, pa.abs2), pa.shell_spectrum(arr),
                            pa.sum(arr, pa.abs2, dims=(1, 2))))
    torch.cuda.synchronize()
    for i, (s, E, sxy) in enumerate(results):
        c = float((i + 1) ** 2)
        assert s.item() == c * 16 * 9 * 10, i
        assert np.array_equal(E.cpu().numpy(), c * count), i
        assert bool((sxy == c * 16 * 9).all()), i
        checks += 3

    # ---- Parseval through the distributed real chain ----------------------------------------------
    if world in (2, 4):
        dims = (32, 16, 32)
        grid = (2, world // 2)
        topo = pa.MPITopology(comm, grid)
        pxr = pa.Pencil(topo, dims, (2, 3))
        pxc = pa.Pencil(pxr, size_global=(dims[0] // 2 + 1,) + dims[1:])
        pyc = pa.Pencil(pxc, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
        pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
        g = np.random.default_rng(21).standard_normal(dims)
        ur = pa.PencilArray.undef(torch.float64, pxr)
        rng = pa.range_local(pxr, pa.LogicalOrder())
        sl = tuple(slice(r.start - 1, r.stop - 1) for r in rng)
        logical_view(ur, ur.data).copy_(torch.from_numpy(np.ascontiguousarray(g[sl])))
        uxc, uyc, uzc = (pa.PencilArray.undef(torch.complex128, p) for p in (pxc, pyc, pzc))
        pa.rfft_(uxc, ur)
        pa.transpose_(pa.Transposition(uyc, uxc), fft="forward")
        pa.transpose_(pa.Transposition(uzc, uyc), fft="forward")
        E = pa.shell_spectrum(uzc, rfft_dim=1)
        s = pa.sum(ur, pa.abs2)
        ntot = math.prod(dims)
        total, want = math.fsum(E.cpu().numpy()), ntot * s.item()
        tol = (8 * math.log2(ntot) + R.depth(uzc.data.numel(), sms, world) + 64) * 2.0 ** -53 * want
        assert abs(total - want) <= tol, (total, want)
        assert abs(want - ntot * float(np.sum(g * g))) <= 1e-9 * want
        checks += 1

    # ---- refusals on every rank -----------------------------------------------------------------
    u = pa.PencilArray.undef(torch.complex128, pen)
    for kw in ({"nbins": 0}, {"nbins": 5000}, {"rfft_dim": 4}, {"width": -1.0}):
        try:
            pa.shell_spectrum(u, **kw)
            raise AssertionError(f"{kw} accepted")
        except pa.ArgumentError as e:
            assert "pa_shell_spectrum:" in str(e), e
            checks += 1
    pa.set_tunable("nccl_fences", 1)
    try:
        pa.shell_spectrum(u)
        raise AssertionError("no flag window accepted")
    except pa.PencilError as e:
        assert "flag window" in str(e), e
        checks += 1
    finally:
        pa.set_tunable("nccl_fences", 0)
    assert pa.shell_spectrum(u).shape == (R.default_nbins((16, 9, 10)),)

    dist.barrier()
    if rank == 0:
        print(f"MP_SPECTRUM_OK world={world} checks={checks}")
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
