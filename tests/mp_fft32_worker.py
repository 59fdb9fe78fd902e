"""Worker of tests/test_gpu_fft32_multirank.py, launched with torch.distributed.run: single-precision
FFTs (PA_FFT_F32) with the ranks sharing one GPU over the NCCL-free communicator.

* world 2 and 4: the real Float32 3-d transform of a PencilFFTs real-input plan (rfft_ along x,
  fused complex64 x->y and y->z, and back), PointToPoint and Alltoallv, the odd N/2+1 axis split
  unevenly once the y and z pencils decompose it; against numpy.fft of the same float32 field;
* world 3 and 8: the fused ComplexF32 unpack+FFT gathering every line from 3 or 8 blocks (uneven
  splits, one row per block, ranks with an empty destination) under PointToPoint, Alltoallv,
  stage_self and p2p_chunks = 3, forward and backward: byte for byte `fft_` of the plain
  transpose, and per line within eps32 log2(L) of the extended-precision reference;
* world 3: L = 48 refused on every rank, nothing launched, dst untouched."""
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
from fft_ref import fft_ld, line_errors  # noqa: E402

EPS32 = float(np.finfo(np.float32).eps)
# world size -> [(grid, global dims (L, y, z), decomposed dims of the source pencil)]
GATHERS = {
    3: [((3,), (64, 5, 3), (1,)),            # 64/3 = 21/21/22
        ((3,), (16, 2, 4), (1,))],           # y = 2 < 3: one rank owns no destination
    8: [((8,), (8, 9, 2), (1,)),             # one row per block
        ((8,), (1024, 3, 2), (1,))],         # y = 3 < 8: five empty destinations
}
REFUSED = {3: [((3,), (48, 6, 4), (1,))]}
VARIANTS = [("p2p", pa.PointToPoint(), {}, {}),
            ("a2av", pa.Alltoallv(), {}, {}),
            ("stage_self", pa.PointToPoint(), {"stage_self": True}, {}),
            ("chunks3", pa.PointToPoint(), {}, {"p2p_chunks": 3})]


def local(A, p):
    return A[tuple(slice(r.start - 1, r.stop - 1) for r in pa.range_local(p))]


def load(u, A):
    u.logical().copy_(torch.from_numpy(np.ascontiguousarray(local(A, u.pencil))))


def real3d(comm, rank, world):
    grid = {2: (2, 1), 4: (2, 2)}[world]
    ran = 0
    for dims in ((16, 8, 16), (64, 16, 8)):
        topo = pa.MPITopology(comm, grid)
        pxr = pa.Pencil(topo, dims, (2, 3))
        pxc = pa.Pencil(pxr, size_global=(dims[0] // 2 + 1,) + dims[1:])
        pyc = pa.Pencil(pxc, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
        pzc = pa.Pencil(pyc, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
        G = np.random.default_rng(11).standard_normal(dims).astype(np.float32)
        F = np.fft.fftn(np.fft.rfft(G.astype(np.float64), axis=0), axes=(1, 2))
        n = math.prod(dims)
        tol_f = 8 * EPS32 * np.log2(n) * np.abs(F).max()
        tol_b = 8 * EPS32 * np.log2(n) * n * np.abs(G).max()
        uxr = pa.PencilArray.undef(torch.float32, pxr)
        load(uxr, G)
        src_bytes = uxr.data.clone()
        for method in (pa.PointToPoint(), pa.Alltoallv()):
            uxc, uyc, uzc = (pa.PencilArray.undef(torch.complex64, p) for p in (pxc, pyc, pzc))
            t_xy = pa.Transposition(uyc, uxc, method=method)
            t_yz = pa.Transposition(uzc, uyc, method=method)
            assert t_xy.fft_fusable() and t_yz.fft_fusable(), (dims, rank)
            pa.rfft_(uxc, uxr)
            pa.transpose_(t_xy, fft="forward")
            pa.transpose_(t_yz, fft="forward")
            torch.cuda.synchronize()
            assert torch.equal(uxr.data, src_bytes)
            got = uzc.logical().cpu().numpy()
            assert got.dtype == np.complex64 and got.shape == local(F, pzc).shape
            assert np.abs(got - local(F, pzc)).max(initial=0) <= tol_f, ("forward", dims, rank, method)
            pa.fft_(uzc, "backward")
            pa.transpose_(pa.Transposition(uyc, uzc, method=method), fft="backward")
            pa.transpose_(pa.Transposition(uxc, uyc, method=method))
            back = pa.PencilArray.undef(torch.float32, pxr)
            pa.brfft_(back, uxc)
            torch.cuda.synchronize()
            err = np.abs(back.logical().cpu().numpy() - n * local(G, pxr).astype(np.float64)).max(initial=0)
            assert err <= tol_b, ("backward", dims, rank, method, err)
            ran += 1
    return ran


def pencils(comm, grid, dims, decomp):
    topo = pa.MPITopology(comm, grid)
    src = pa.Pencil(topo, dims, decomp, permute=pa.Permutation(2, 1, 3))  # y contiguous
    dst_decomp = tuple(2 if d == 1 else d for d in decomp)
    dst = pa.Pencil(src, decomp_dims=dst_decomp, permute=pa.NoPermutation())  # x local, contiguous
    return src, dst


def global_field(dims, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(dims) + 1j * rng.standard_normal(dims)).astype(np.complex64)


def gathers(comm, rank, world):
    ran = 0
    for (grid, dims, decomp) in GATHERS.get(world, []):
        ps, pd = pencils(comm, grid, dims, decomp)
        G = global_field(dims, 17)
        u = pa.PencilArray.undef(torch.complex64, ps)
        load(u, G)
        src_bytes = u.data.clone()
        want_plain = np.ascontiguousarray(local(G, pd))
        L = dims[0]
        for name, method, kw, tun in VARIANTS:
            for k, v in tun.items():
                pa.set_tunable(k, v)
            try:
                fused = pa.PencilArray.undef(torch.complex64, pd)
                plain = pa.PencilArray.undef(torch.complex64, pd)
                t_f = pa.Transposition(fused, u, method=method)
                t_p = pa.Transposition(plain, u, method=method)
                assert t_f.fft_fusable(), (grid, dims, rank)
                for direction, sign in (("forward", -1), ("backward", 1)):
                    fused.data.view(torch.uint8).fill_(0x5A)
                    pa.transpose_(t_f, fft=direction, **kw)
                    pa.transpose_(t_p, **kw)
                    torch.cuda.synchronize()
                    got_plain = plain.logical().cpu().numpy()
                    assert got_plain.tobytes() == want_plain.tobytes(), ("plain", name, grid, dims, rank)
                    pa.fft_(plain, direction)
                    torch.cuda.synchronize()
                    assert torch.equal(fused.data.view(torch.uint8), plain.data.view(torch.uint8)), \
                        ("fused != unfused", name, direction, grid, dims, rank)
                    assert torch.equal(u.data, src_bytes), ("src", name, rank)
                    if name == "p2p" and plain.data.numel():
                        lines = np.moveaxis(want_plain, 0, -1)
                        got = np.moveaxis(fused.logical().cpu().numpy(), 0, -1)
                        mx, _ = line_errors(got, fft_ld(lines, sign))
                        assert mx <= EPS32 * math.log2(L), ("accuracy", grid, dims, rank, direction, mx)
                    ran += 1
            finally:
                for k in tun:
                    pa.set_tunable(k, 1)
    for (grid, dims, decomp) in REFUSED.get(world, []):
        ps, pd = pencils(comm, grid, dims, decomp)
        G = global_field(dims, 23)
        u = pa.PencilArray.undef(torch.complex64, ps)
        load(u, G)
        for method in (pa.PointToPoint(), pa.Alltoallv()):
            out = pa.PencilArray.undef(torch.complex64, pd)
            out.data.view(torch.uint8).fill_(0x3C)
            torch.cuda.synchronize()
            before = out.data.clone()
            t = pa.Transposition(out, u, method=method)
            assert not t.fft_fusable(), (grid, dims, rank)
            n0 = pa.launch_count()
            try:
                pa.transpose_(t, fft="forward")
                raise AssertionError(f"fused FFT accepted L = {dims[0]} on rank {rank}")
            except pa.ArgumentError:
                pass
            torch.cuda.synchronize()
            assert pa.launch_count() == n0, ("launched", grid, dims, rank, pa.launch_count() - n0)
            assert torch.equal(out.data.view(torch.uint8), before.view(torch.uint8))
            pa.transpose_(t)
            torch.cuda.synchronize()
            assert out.logical().cpu().numpy().tobytes() == np.ascontiguousarray(local(G, pd)).tobytes()
            ran += 1
    return ran


def main():
    comm = pa.comm_world(transport="ipc")
    assert comm.transport == "ipc" and comm.handle is not None
    rank, world = comm.rank, comm.size
    ran = real3d(comm, rank, world) if world in (2, 4) else 0
    ran += gathers(comm, rank, world)
    assert ran > 0
    dist.barrier()
    if rank == 0:
        print(f"MP_FFT32_OK world={world} runs={ran}")
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
