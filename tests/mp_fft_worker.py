"""Worker of tests/test_gpu_fft_multiblock.py, launched with torch.distributed.run: the fused
unpack+FFT gathering its lines from 3, 5, 6 and 8 blocks, with the ranks sharing one GPU over
the NCCL-free communicator.

Per configuration, an x-pencil decomposed along the transform axis x (y contiguous) goes to a
pencil with x local and contiguous, so every destination line of L points is assembled from one
block per rank of the line: uneven splits (64/3, 1024/6, 8/5), one row per block (8/8), and a
rank whose destination is empty.  Under PointToPoint, Alltoallv, stage_self, p2p_chunks = 3 and
overlap off, forward and backward, every rank requires

  * I1: transpose_(t, fft=d) == fft_(plain transpose_), byte for byte;
  * the plain transpose equal to its part of the global array, bit for bit;
  * its lines within eps log2(L) of the extended-precision reference (tests/fft_ref.py).

Then the refusals (L = 48 over 3 ranks, L = 2048): ArgumentError on every rank, no kernel
launched, dst untouched, and the next plain transpose on the same plan and arrays bit-exact."""
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
from fft_ref import EPS, fft_ld, line_errors  # noqa: E402

# world size -> [(grid, global dims (L, y, z), decomposed dims of the source pencil)]
CONFIGS = {
    5: [((5,), (8, 4, 3), (1,))],                        # 8/5 -> 1,2,1,2,2; y = 4 < 5: rank 0 owns nothing
    6: [((6,), (1024, 7, 2), (1,)),                      # 1024/6
        ((3, 2), (64, 6, 4), (1, 3))],                   # lines of 3 ranks: 64/3 = 21/21/22
    8: [((8,), (8, 9, 2), (1,)),                         # one row per block
        ((8,), (64, 5, 3), (1,))],                       # y = 5 < 8: three empty destinations
}
REFUSED = {5: [((5,), (2048, 6, 2), (1,))], 6: [((3, 2), (48, 6, 4), (1, 3))], 8: []}
VARIANTS = [("p2p", pa.PointToPoint(), {}, {}),
            ("a2av", pa.Alltoallv(), {}, {}),
            ("stage_self", pa.PointToPoint(), {"stage_self": True}, {}),
            ("chunks3", pa.PointToPoint(), {}, {"p2p_chunks": 3}),
            ("no_overlap", pa.PointToPoint(), {"overlap": False}, {}),
            ("a2av_stage_self", pa.Alltoallv(), {"stage_self": True}, {})]


def local(A, p):
    return A[tuple(slice(r.start - 1, r.stop - 1) for r in pa.range_local(p))]


def pencils(comm, grid, dims, decomp):
    topo = pa.MPITopology(comm, grid)
    src = pa.Pencil(topo, dims, decomp, permute=pa.Permutation(2, 1, 3))  # y contiguous
    dst_decomp = tuple(2 if d == 1 else d for d in decomp)
    dst = pa.Pencil(src, decomp_dims=dst_decomp, permute=pa.NoPermutation())  # x local, contiguous
    return src, dst


def global_field(dims, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(dims) + 1j * rng.standard_normal(dims)


def load(u, A):
    u.logical().copy_(torch.from_numpy(np.ascontiguousarray(local(A, u.pencil))))


def main():
    comm = pa.comm_world(transport="ipc")
    rank, world = comm.rank, comm.size
    ran = 0
    for (grid, dims, decomp) in CONFIGS[world]:
        ps, pd = pencils(comm, grid, dims, decomp)
        G = global_field(dims, 17)
        u = pa.PencilArray.undef(torch.complex128, ps)
        load(u, G)
        src_bytes = u.data.clone()
        want_plain = np.ascontiguousarray(local(G, pd))
        L = dims[0]
        for name, method, kw, tun in VARIANTS:
            for k, v in tun.items():
                pa.set_tunable(k, v)
            try:
                fused = pa.PencilArray.undef(torch.complex128, pd)
                plain = pa.PencilArray.undef(torch.complex128, pd)
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
                        ("I1", name, direction, grid, dims, rank)
                    assert torch.equal(u.data, src_bytes), ("src", name, rank)
                    if name == "p2p" and plain.data.numel():
                        # the lines along x of my part of the global array, against the reference
                        lines = np.moveaxis(want_plain, 0, -1)
                        got = np.moveaxis(fused.logical().cpu().numpy(), 0, -1)
                        mx, _ = line_errors(got, fft_ld(lines, sign))
                        assert mx <= EPS * math.log2(L), ("accuracy", grid, dims, rank, direction, mx)
                    ran += 1
            finally:
                for k in tun:
                    pa.set_tunable(k, 1)
    for (grid, dims, decomp) in REFUSED[world]:
        ps, pd = pencils(comm, grid, dims, decomp)
        G = global_field(dims, 23)
        u = pa.PencilArray.undef(torch.complex128, ps)
        load(u, G)
        for method in (pa.PointToPoint(), pa.Alltoallv()):
            out = pa.PencilArray.undef(torch.complex128, pd)
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
    dist.barrier()
    if rank == 0:
        print(f"MP_FFT_OK world={world} runs={ran}")
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
