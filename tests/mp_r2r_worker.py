"""Worker of tests/test_gpu_r2r.py, launched with torch.distributed.run: the mixed 3-d transform
(r2r_ DCT-II along x, real x->y transpose, rfft_ along y, fused y->z + fft) and its inverse with
the ranks sharing the GPU through the NCCL-free communicator, both staged methods and both
precisions.  Every rank builds the same global field from a seed and compares its own part with
scipy.fft / numpy.fft."""
import math
import os
import sys

import numpy as np
import scipy.fft as sf
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import pencilarrays_b200 as pa  # noqa: E402


def local(A, p):
    return A[tuple(slice(r.start - 1, r.stop - 1) for r in pa.range_local(p))]


def main():
    comm = pa.comm_world(transport="ipc")
    assert comm.transport == "ipc" and comm.handle is not None
    rank, world = comm.rank, comm.size
    grid = {2: (2, 1), 4: (2, 2)}[world]
    ran = 0
    # Ny/2+1 = 17 and 9 points: uneven blocks once the z pencil decomposes dim 2
    for dims in ((16, 32, 8), (64, 16, 32)):
        topo = pa.MPITopology(comm, grid)
        pxr = pa.Pencil(topo, dims, (2, 3))
        pyr = pa.Pencil(pxr, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
        pyc = pa.Pencil(pyr, size_global=(dims[0], dims[1] // 2 + 1, dims[2]))
        pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
        n = math.prod(dims)
        for rdt, cdt, eps in ((torch.float64, torch.complex128, np.finfo(np.float64).eps),
                              (torch.float32, torch.complex64, np.finfo(np.float32).eps)):
            G = np.random.default_rng(13).standard_normal(dims).astype(
                np.float64 if rdt == torch.float64 else np.float32)
            F = np.fft.fft(np.fft.rfft(sf.dct(G.astype(np.float64), 2, axis=0), axis=1), axis=2)
            tol_f = 8 * eps * np.log2(n) * np.abs(F).max()
            tol_b = 8 * eps * np.log2(n) * 2 * n * np.abs(G).max()
            ux = pa.PencilArray.undef(rdt, pxr)
            ux.logical().copy_(torch.from_numpy(np.ascontiguousarray(local(G, pxr))))
            src_bytes = ux.data.clone()
            for method in (pa.PointToPoint(), pa.Alltoallv()):
                ux2, uy = pa.PencilArray.undef(rdt, pxr), pa.PencilArray.undef(rdt, pyr)
                uyc, uzc = pa.PencilArray.undef(cdt, pyc), pa.PencilArray.undef(cdt, pzc)
                n0 = pa.launch_count()
                pa.r2r_(ux2, ux, "REDFT10")
                torch.cuda.synchronize()
                assert pa.launch_count() - n0 == (1 if ux.data.numel() else 0)
                pa.transpose_(pa.Transposition(uy, ux2, method=method))
                pa.rfft_(uyc, uy)
                pa.transpose_(pa.Transposition(uzc, uyc, method=method), fft="forward")
                torch.cuda.synchronize()
                assert torch.equal(ux.data, src_bytes)
                got = uzc.logical().cpu().numpy()
                assert got.shape == local(F, pzc).shape
                err = np.abs(got - local(F, pzc)).max(initial=0)
                assert err <= tol_f, ("forward", dims, rdt, rank, method, err)
                pa.fft_(uzc, "backward")
                pa.transpose_(pa.Transposition(uyc, uzc, method=method))
                pa.brfft_(uy, uyc)
                pa.transpose_(pa.Transposition(ux2, uy, method=method))
                pa.r2r_(ux2, ux2, "REDFT01")
                torch.cuda.synchronize()
                err = np.abs(ux2.logical().cpu().numpy() - 2 * n * local(G, pxr)).max(initial=0)
                assert err <= tol_b, ("backward", dims, rdt, rank, method, err)
                ran += 1
    dist.barrier()
    if rank == 0:
        print(f"MP_R2R_OK world={world} runs={ran}")
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
