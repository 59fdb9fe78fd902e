"""Worker of tests/test_gpu_rfft.py, launched with torch.distributed.run: the real 3-d FFT of a
PencilFFTs real-input plan (rfft_ along x, fused x->y and y->z transposes) with the ranks sharing
the GPU through the NCCL-free communicator, both staged methods.  Every rank builds the same
global field from a seed and compares its own part with numpy.fft."""
import math
import os
import sys

import numpy as np
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
    # N/2+1 = 9 and 33 points: uneven blocks once the y and z pencils decompose dim 1
    for dims in ((16, 8, 16), (64, 16, 8)):
        topo = pa.MPITopology(comm, grid)
        pxr = pa.Pencil(topo, dims, (2, 3))
        pxc = pa.Pencil(pxr, size_global=(dims[0] // 2 + 1,) + dims[1:])
        pyc = pa.Pencil(pxc, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
        pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
        G = np.random.default_rng(11).standard_normal(dims)
        F = np.fft.fftn(np.fft.rfft(G, axis=0), axes=(1, 2))
        n = math.prod(dims)
        eps = np.finfo(np.float64).eps
        tol_f = 8 * eps * np.log2(n) * np.abs(F).max()
        tol_b = 8 * eps * np.log2(n) * n * np.abs(G).max()
        uxr = pa.PencilArray.undef(torch.float64, pxr)
        uxr.logical().copy_(torch.from_numpy(np.ascontiguousarray(local(G, pxr))))
        src_bytes = uxr.data.clone()
        for method in (pa.PointToPoint(), pa.Alltoallv()):
            uxc, uyc, uzc = (pa.PencilArray.undef(torch.complex128, p) for p in (pxc, pyc, pzc))
            n0 = pa.launch_count()
            pa.rfft_(uxc, uxr)
            torch.cuda.synchronize()
            assert pa.launch_count() - n0 == (1 if uxr.data.numel() else 0)
            pa.transpose_(pa.Transposition(uyc, uxc, method=method), fft="forward")
            pa.transpose_(pa.Transposition(uzc, uyc, method=method), fft="forward")
            torch.cuda.synchronize()
            assert torch.equal(uxr.data, src_bytes)
            got = uzc.logical().cpu().numpy()
            assert got.shape == local(F, pzc).shape
            assert np.abs(got - local(F, pzc)).max(initial=0) <= tol_f, ("forward", dims, rank, method)
            pa.fft_(uzc, "backward")
            pa.transpose_(pa.Transposition(uyc, uzc, method=method), fft="backward")
            pa.transpose_(pa.Transposition(uxc, uyc, method=method))
            back = pa.PencilArray.undef(torch.float64, pxr)
            pa.brfft_(back, uxc)
            torch.cuda.synchronize()
            err = np.abs(back.logical().cpu().numpy() - n * local(G, pxr)).max(initial=0)
            assert err <= tol_b, ("backward", dims, rank, method, err)
            ran += 1
    dist.barrier()
    if rank == 0:
        print(f"MP_RFFT_OK world={world} runs={ran}")
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
