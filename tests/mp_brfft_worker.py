"""Worker of tests/test_gpu_brfft.py, launched with torch.distributed.run: the fused y->x transpose
+ complex-to-real transform (`Transposition(real_x, cplx_y, brfft=True)`) with the ranks sharing
the GPU through the NCCL-free communicator.  Every staged schedule must give, on every rank, the
bytes of the plain y->x transpose followed by `brfft_`; the whole real backward chain is compared
with numpy; a refused line length launches nothing on any rank."""
import math
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import pencilarrays_b200 as pa  # noqa: E402

# world size -> [(grid, real global dims)]: the N/2+1 bins split unevenly over the y-pencil's
# decomposition of x; with 8 ranks 9 bins give one-row blocks and y = 4 leaves four ranks
# without any x-pencil data
SHAPES = {2: [((2, 1), (16, 8, 16)), ((2, 1), (128, 6, 4))],
          3: [((3, 1), (64, 5, 3)), ((3, 1), (16, 2, 4))],
          4: [((2, 2), (32, 8, 16)), ((4, 1), (2048, 3, 2))],
          8: [((8, 1), (16, 4, 6)), ((8, 1), (256, 9, 2))]}
# the whole backward chain transforms along every dim: powers of two throughout
CHAIN = {2: ((2, 1), (16, 8, 16)), 3: ((3, 1), (64, 8, 16)), 4: ((2, 2), (32, 8, 16)),
         8: ((8, 1), (16, 16, 8))}
VARIANTS = [("p2p", pa.PointToPoint(), {}, {}),
            ("a2av", pa.Alltoallv(), {}, {}),
            ("stage_self", pa.PointToPoint(), {"stage_self": True}, {}),
            ("chunks3", pa.PointToPoint(), {}, {"p2p_chunks": 3}),
            ("no_overlap", pa.PointToPoint(), {"overlap": False}, {}),
            ("nowait", pa.Alltoallv(), {"waitall": False}, {})]
PREC = [(torch.float64, torch.complex128, np.finfo(np.float64).eps),
        (torch.float32, torch.complex64, np.finfo(np.float32).eps)]


def local(A, p):
    return A[tuple(slice(r.start - 1, r.stop - 1) for r in pa.range_local(p))]


def load(u, A):
    u.logical().copy_(torch.from_numpy(np.ascontiguousarray(local(A, u.pencil))))


def chain(comm, grid, dims):
    topo = pa.MPITopology(comm, grid)
    pxr = pa.Pencil(topo, dims, (2, 3))
    pxc = pa.Pencil(pxr, size_global=(dims[0] // 2 + 1,) + dims[1:])
    pyc = pa.Pencil(pxc, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    return pxr, pxc, pyc, pzc


def fused_vs_unfused(comm, rank, world):
    ran = 0
    for grid, dims in SHAPES[world]:
        pxr, pxc, pyc, pzc = chain(comm, grid, dims)
        rng = np.random.default_rng(5)
        S = rng.standard_normal((dims[0] // 2 + 1,) + dims[1:]) + \
            1j * rng.standard_normal((dims[0] // 2 + 1,) + dims[1:])
        for rdt, cdt, _ in PREC:
            uy = pa.PencilArray.undef(cdt, pyc)
            load(uy, S.astype(np.complex64 if cdt == torch.complex64 else np.complex128))
            src_bytes = uy.data.clone()
            for name, method, kw, tun in VARIANTS:
                for k, v in tun.items():
                    pa.set_tunable(k, v)
                try:
                    fused = pa.PencilArray.undef(rdt, pxr)
                    fused.data.view(torch.uint8).fill_(0x5A)
                    t = pa.Transposition(fused, uy, method=method, brfft=True)
                    assert t.fft_fusable(), (grid, dims, rank)
                    pa.transpose_(t, **kw)
                    if not kw.get("waitall", True):
                        pa.Waitall(t)
                    ux = pa.PencilArray.undef(cdt, pxc)
                    pa.transpose_(pa.Transposition(ux, uy, method=method), **kw)
                    if not kw.get("waitall", True):
                        pa.Waitall(pa.Transposition(ux, uy, method=method))
                    plain = pa.PencilArray.undef(rdt, pxr)
                    pa.brfft_(plain, ux)
                    torch.cuda.synchronize()
                    assert torch.equal(fused.data.view(torch.uint8), plain.data.view(torch.uint8)), \
                        ("fused != unfused", name, rdt, grid, dims, rank)
                    assert torch.equal(uy.data.view(torch.uint8), src_bytes.view(torch.uint8)), ("src", name)
                    ran += 1
                finally:
                    for k in tun:
                        pa.set_tunable(k, 1)
    return ran


def backward_chain(comm, rank, world):
    """fft_ along z, fused z->y, fused y->x + brfft: N times the field, against numpy."""
    ran = 0
    grid, dims = CHAIN[world]
    pxr, pxc, pyc, pzc = chain(comm, grid, dims)
    G = np.random.default_rng(11).standard_normal(dims)
    F = np.fft.fftn(np.fft.rfft(G, axis=0), axes=(1, 2))
    n = math.prod(dims)
    for rdt, cdt, eps in PREC:
        for method in (pa.PointToPoint(), pa.Alltoallv()):
            uz = pa.PencilArray.undef(cdt, pzc)
            load(uz, F.astype(np.complex64 if cdt == torch.complex64 else np.complex128))
            uy = pa.PencilArray.undef(cdt, pyc)
            back = pa.PencilArray.undef(rdt, pxr)
            pa.fft_(uz, "backward")
            pa.transpose_(pa.Transposition(uy, uz, method=method), fft="backward")
            pa.transpose_(pa.Transposition(back, uy, method=method, brfft=True))
            torch.cuda.synchronize()
            err = np.abs(back.logical().cpu().numpy() - n * local(G, pxr)).max(initial=0)
            assert err <= 8 * eps * np.log2(n) * n * np.abs(G).max(), (rdt, method, rank, err)
            ran += 1
    return ran


def refused(comm, rank, world):
    if world != 3:
        return 0
    pxr, pxc, pyc, _ = chain(comm, (3, 1), (24, 6, 4))  # 13 bins: N = 24 is not a power of two
    uy = pa.PencilArray.undef(torch.complex128, pyc)
    uy.data.normal_()
    ran = 0
    for method in (pa.PointToPoint(), pa.Alltoallv()):
        out = pa.PencilArray.undef(torch.float64, pxr)
        out.data.view(torch.uint8).fill_(0x3C)
        torch.cuda.synchronize()
        before = out.data.clone()
        t = pa.Transposition(out, uy, method=method, brfft=True)
        assert not t.fft_fusable(), rank
        n0 = pa.launch_count()
        try:
            pa.transpose_(t)
            raise AssertionError(f"fused brfft accepted N = 24 on rank {rank}")
        except pa.ArgumentError:
            pass
        torch.cuda.synchronize()
        assert pa.launch_count() == n0, ("launched", rank, pa.launch_count() - n0)
        assert torch.equal(out.data.view(torch.uint8), before.view(torch.uint8))
        ran += 1
    return ran


def main():
    comm = pa.comm_world(transport="ipc")
    assert comm.transport == "ipc" and comm.handle is not None
    rank, world = comm.rank, comm.size
    ran = fused_vs_unfused(comm, rank, world) + backward_chain(comm, rank, world) + refused(comm, rank, world)
    dist.barrier()
    if rank == 0:
        print(f"MP_BRFFT_OK world={world} runs={ran}")
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
