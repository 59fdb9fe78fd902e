"""Worker of tests/test_gpu_fused_real.py, launched with torch.distributed.run: the fused
transposition of real arrays + DCT / DST (`Transposition(..., r2r=kind)`) and + RFFT
(`Transposition(..., rfft=True)`) with the ranks sharing the GPU through the NCCL-free
communicator.  Under PointToPoint and Alltoallv, with and without a staged self block and in both
precisions, every rank must hold the bytes of the plain transpose followed by `r2r_` / `rfft_`.
The wall-bounded mixed chain (DCT x, RFFT y, FFT z) in three kernels each way is compared with
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

# world size -> [(grid, global dims)]: the transform runs along y (N = dims[1]), split over the
# x-pencil's decomposition of y.  N = 32 over 3 ranks gives blocks of 11, 11 and 10 reals (odd
# boundaries: one complex slot filled from two blocks), 64 over 3 gives 22, 21, 21; with 8 ranks
# x = 4 leaves four ranks without any y-pencil data
SHAPES = {2: [((2, 1), (8, 32, 6)), ((2, 1), (6, 128, 4))],
          3: [((3, 1), (5, 32, 3)), ((3, 1), (4, 64, 2))],
          4: [((2, 2), (8, 32, 16)), ((4, 1), (3, 2048, 2))],
          8: [((8, 1), (4, 16, 6)), ((8, 1), (9, 256, 2))]}
# the mixed chain transforms along every dim: powers of two throughout
CHAIN = {2: ((2, 1), (16, 32, 8)), 3: ((3, 1), (16, 32, 8)), 4: ((2, 2), (16, 32, 8)),
         8: ((8, 1), (16, 32, 8))}
VARIANTS = [("p2p", pa.PointToPoint(), {}),
            ("a2av", pa.Alltoallv(), {}),
            ("p2p_stage_self", pa.PointToPoint(), {"stage_self": True}),
            ("a2av_stage_self", pa.Alltoallv(), {"stage_self": True})]
PREC = [(torch.float64, torch.complex128, np.finfo(np.float64).eps),
        (torch.float32, torch.complex64, np.finfo(np.float32).eps)]
KINDS = ["REDFT10", "REDFT01", "RODFT10", "RODFT01"]


def local(A, p):
    return A[tuple(slice(r.start - 1, r.stop - 1) for r in pa.range_local(p))]


def load(u, A):
    u.logical().copy_(torch.from_numpy(np.ascontiguousarray(local(A, u.pencil))))


def pencils(comm, grid, dims):
    topo = pa.MPITopology(comm, grid)
    px = pa.Pencil(topo, dims, (2, 3))
    py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    pyc = pa.Pencil(py, size_global=(dims[0], dims[1] // 2 + 1, dims[2]))
    pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    return px, py, pyc, pzc


def b(u):
    return u.data.view(torch.uint8)


def fused_vs_unfused(comm, rank, world):
    ran = 0
    for grid, dims in SHAPES[world]:
        px, py, pyc, _ = pencils(comm, grid, dims)
        G = np.random.default_rng(5).standard_normal(dims)
        for rdt, cdt, _ in PREC:
            ux = pa.PencilArray.undef(rdt, px)
            load(ux, G.astype(np.float32 if rdt == torch.float32 else np.float64))
            src_bytes = ux.data.clone()
            for name, method, kw in VARIANTS:
                mid = pa.PencilArray.undef(rdt, py)
                pa.transpose_(pa.Transposition(mid, ux, method=method), **kw)
                for kind in KINDS:
                    fused = pa.PencilArray.undef(rdt, py)
                    b(fused).fill_(0x5A)
                    t = pa.Transposition(fused, ux, method=method, r2r=kind)
                    assert t.fft_fusable(), (grid, dims, rank)
                    pa.transpose_(t, **kw)
                    plain = pa.PencilArray.undef(rdt, py)
                    pa.r2r_(plain, mid, kind)
                    torch.cuda.synchronize()
                    assert torch.equal(b(fused), b(plain)), ("r2r fused != unfused", kind, name, rdt,
                                                             grid, dims, rank)
                    ran += 1
                fused = pa.PencilArray.undef(cdt, pyc)
                b(fused).fill_(0x5A)
                t = pa.Transposition(fused, ux, method=method, rfft=True)
                assert t.fft_fusable(), (grid, dims, rank)
                pa.transpose_(t, **kw)
                plain = pa.PencilArray.undef(cdt, pyc)
                pa.rfft_(plain, mid)
                torch.cuda.synchronize()
                assert torch.equal(b(fused), b(plain)), ("rfft fused != unfused", name, rdt, grid,
                                                         dims, rank)
                assert torch.equal(b(ux), src_bytes.view(torch.uint8)), ("src", name)
                ran += 1
    return ran


def mixed_chain(comm, rank, world):
    """r2r_ DCT-II along x, fused x->y + rfft, fused y->z + FFT; then fft_, fused z->y + brfft,
    fused y->x + DCT-III, against scipy / numpy.  (Three transform kernels each way; the ranks
    also launch their pack kernels, so launches are counted on one rank only, in
    tests/test_gpu_fused_real.py.)"""
    ran = 0
    grid, dims = CHAIN[world]
    px, py, pyc, pzc = pencils(comm, grid, dims)
    n = math.prod(dims)
    for rdt, cdt, eps in PREC:
        G = np.random.default_rng(13).standard_normal(dims).astype(
            np.float64 if rdt == torch.float64 else np.float32)
        F = np.fft.fft(np.fft.rfft(sf.dct(G.astype(np.float64), 2, axis=0), axis=1), axis=2)
        tol_f = 8 * eps * np.log2(n) * np.abs(F).max()
        tol_b = 8 * eps * np.log2(n) * 2 * n * np.abs(G).max()
        for method in (pa.PointToPoint(), pa.Alltoallv()):
            ux = pa.PencilArray.undef(rdt, px)
            load(ux, G)
            u1 = pa.PencilArray.undef(rdt, px)
            uyc, uzc = pa.PencilArray.undef(cdt, pyc), pa.PencilArray.undef(cdt, pzc)
            back_y, back = pa.PencilArray.undef(rdt, py), pa.PencilArray.undef(rdt, px)
            ts = [pa.Transposition(uyc, u1, method=method, rfft=True),
                  pa.Transposition(uzc, uyc, method=method),
                  pa.Transposition(back_y, uzc, method=method, brfft=True),
                  pa.Transposition(back, back_y, method=method, r2r="REDFT01")]
            pa.r2r_(u1, ux, "REDFT10")
            pa.transpose_(ts[0])
            pa.transpose_(ts[1], fft="forward")
            torch.cuda.synchronize()
            got = uzc.logical().cpu().numpy()
            err = np.abs(got - local(F, pzc)).max(initial=0)
            assert err <= tol_f, ("forward", rdt, rank, method, err)
            pa.fft_(uzc, "backward")
            pa.transpose_(ts[2])
            pa.transpose_(ts[3])
            torch.cuda.synchronize()
            err = np.abs(back.logical().cpu().numpy() - 2 * n * local(G, px)).max(initial=0)
            assert err <= tol_b, ("backward", rdt, rank, method, err)
            ran += 1
    return ran


def main():
    comm = pa.comm_world(transport="ipc")
    assert comm.transport == "ipc" and comm.handle is not None
    rank, world = comm.rank, comm.size
    ran = fused_vs_unfused(comm, rank, world)
    ran += mixed_chain(comm, rank, world)
    dist.barrier()
    if rank == 0:
        print(f"MP_FUSED_REAL_OK world={world} runs={ran}")
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
