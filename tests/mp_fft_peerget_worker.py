"""Worker of tests/test_gpu_fft_peerget.py, launched with torch.distributed.run: the one-sided
fused transpose + FFT (PeerGet) with the ranks sharing one GPU over the NCCL-free communicator.

  * transpose_(t, fft=d) with PeerGet == the same call with PointToPoint, byte for byte, under
    waitall True and False + Waitall, tunable multi_put 1 (protocol inside the kernel) and 0
    (standalone flag kernels around it), forward and backward, repeated so that the flag
    sequence numbers advance; lines from 2 ... 8 blocks, ranks with empty destinations;
  * on 2 and 4 processes the whole 3-d FFT (fft_ along x, fused x -> y, fused y -> z, all
    PeerGet, and back) against numpy.fft.fftn, in both precisions;
  * the caller-stream pattern: hold a side stream, produce the input behind the hold, run the
    fused PeerGet transpose there: the call returns before the hold ends, the result is right;
  * PeerPut + fft= is refused on every rank, launches nothing and leaves dst untouched."""
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
from gpu_util import hold  # noqa: E402

# world size -> [(grid, global dims (L, y, z), decomposed dims of the source pencil, dtype)]
CONFIGS = {
    2: [((2,), (16, 6, 4), (1,), torch.complex128), ((2,), (512, 3, 2), (1,), torch.complex64)],
    3: [((3,), (64, 7, 2), (1,), torch.complex128)],
    4: [((4,), (32, 8, 3), (1,), torch.complex128), ((2, 2), (16, 8, 4), (1, 3), torch.complex64)],
    5: [((5,), (8, 4, 3), (1,), torch.complex128)],   # y = 4 < 5: rank 0 has no destination lines
    6: [((6,), (1024, 7, 2), (1,), torch.complex128), ((3, 2), (64, 6, 4), (1, 3), torch.complex128)],
    8: [((8,), (8, 9, 2), (1,), torch.complex128), ((8,), (64, 5, 3), (1,), torch.complex64)],
}
EPS = {torch.complex128: np.finfo(np.float64).eps, torch.complex64: np.finfo(np.float32).eps}
NP = {torch.complex128: np.complex128, torch.complex64: np.complex64}


def local(A, p):
    return A[tuple(slice(r.start - 1, r.stop - 1) for r in pa.range_local(p))]


def load(u, A):
    u.logical().copy_(torch.from_numpy(np.ascontiguousarray(local(A, u.pencil))))


def global_field(dims, seed, dtype):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(dims) + 1j * rng.standard_normal(dims)).astype(NP[dtype])


def pencils(comm, grid, dims, decomp):
    topo = pa.MPITopology(comm, grid)
    src = pa.Pencil(topo, dims, decomp, permute=pa.Permutation(2, 1, 3))  # y contiguous
    dst_decomp = tuple(2 if d == 1 else d for d in decomp)
    dst = pa.Pencil(src, decomp_dims=dst_decomp, permute=pa.NoPermutation())  # x local, contiguous
    return src, dst


def equal_to_staged(comm):
    ran = 0
    for (grid, dims, decomp, dtype) in CONFIGS[comm.size]:
        ps, pd = pencils(comm, grid, dims, decomp)
        u = pa.PencilArray.undef(dtype, ps)
        load(u, global_field(dims, 31, dtype))
        src_bytes = u.data.clone()
        ref = pa.PencilArray.undef(dtype, pd)
        out = pa.PencilArray.undef(dtype, pd)
        t_ref = pa.Transposition(ref, u, method=pa.PointToPoint())
        t = pa.Transposition(out, u, method=pa.PeerGet())
        assert t.fft_fusable() and t_ref.fft_fusable(), (grid, dims, comm.rank)
        for multi in (1, 0):
            pa.set_tunable("multi_put", multi)
            try:
                for waitall in (True, False):
                    for it in range(3):
                        for direction in ("forward", "backward"):
                            out.data.view(torch.uint8).fill_(0x5A)
                            pa.transpose_(t_ref, fft=direction)
                            pa.transpose_(t, fft=direction, waitall=waitall)
                            if not waitall:
                                pa.Waitall(t)
                            torch.cuda.synchronize()
                            assert torch.equal(out.data.view(torch.uint8), ref.data.view(torch.uint8)), \
                                (grid, dims, multi, waitall, it, direction, comm.rank)
                            assert torch.equal(u.data, src_bytes), ("src", grid, dims, comm.rank)
                            ran += 1
            finally:
                pa.set_tunable("multi_put", 1)
    return ran


def fft3d(comm):
    if comm.size not in (2, 4):
        return 0
    ran = 0
    grid = (2, 1) if comm.size == 2 else (2, 2)
    dims = (16, 32, 8)
    for dtype in (torch.complex128, torch.complex64):
        topo = pa.MPITopology(comm, grid)
        px = pa.Pencil(topo, dims, (2, 3))
        py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
        pz = pa.Pencil(px, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
        G = global_field(dims, 41, dtype)
        ux, uy, uz = (pa.PencilArray.undef(dtype, p) for p in (px, py, pz))
        vy, vx = pa.PencilArray.undef(dtype, py), pa.PencilArray.undef(dtype, px)
        load(ux, G)
        t_xy = pa.Transposition(uy, ux, method=pa.PeerGet())
        t_yz = pa.Transposition(uz, uy, method=pa.PeerGet())
        t_zy = pa.Transposition(vy, uz, method=pa.PeerGet())
        t_yx = pa.Transposition(vx, vy, method=pa.PeerGet())
        pa.fft_(ux, "forward")
        pa.transpose_(t_xy, fft="forward")
        pa.transpose_(t_yz, fft="forward")
        torch.cuda.synchronize()
        X = np.fft.fftn(G.astype(np.complex128))
        tol = 8 * EPS[dtype] * math.log2(math.prod(dims)) * np.abs(X).max()
        err = np.abs(uz.logical().cpu().numpy() - local(X, pz)).max() if uz.data.numel() else 0.0
        assert err <= tol, ("forward", dtype, comm.rank, err, tol)
        pa.fft_(uz, "backward")
        pa.transpose_(t_zy, fft="backward")
        pa.transpose_(t_yx, fft="backward")
        torch.cuda.synchronize()
        back = math.prod(dims) * G.astype(np.complex128)
        err = np.abs(vx.logical().cpu().numpy() - local(back, px)).max() if vx.data.numel() else 0.0
        assert err <= 8 * EPS[dtype] * math.log2(math.prod(dims)) * np.abs(back).max() * 2, \
            ("backward", dtype, comm.rank, err)
        ran += 1
    return ran


def caller_stream(comm):
    grid, dims, decomp, dtype = CONFIGS[comm.size][0]
    ps, pd = pencils(comm, grid, dims, decomp)
    G = global_field(dims, 53, dtype)
    u = pa.PencilArray.undef(dtype, ps)
    fresh = pa.PencilArray.undef(dtype, ps)
    load(fresh, G)
    ref, out = pa.PencilArray.undef(dtype, pd), pa.PencilArray.undef(dtype, pd)
    u.data.copy_(fresh.data)
    pa.transpose_(pa.Transposition(ref, u, method=pa.PointToPoint()), fft="forward")
    t = pa.Transposition(out, u, method=pa.PeerGet())
    # (the first transpose on a plan creates its streams and events, which synchronises the
    #  device: done here, before the hold)
    pa.transpose_(t, fft="forward")
    torch.cuda.synchronize()
    u.data.zero_()
    out.data.view(torch.uint8).fill_(0x5A)
    torch.cuda.synchronize()
    dist.barrier()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        held = hold()
        u.data.copy_(fresh.data)  # the input is produced behind the hold
        pa.transpose_(t, fft="forward", waitall=False)
        returned_early = not held.query()
        got = out.data.clone()  # consumed on the same stream
        pa.Waitall(t)
    side.synchronize()
    assert returned_early, ("the fused PeerGet transpose waited for the caller's stream", comm.rank)
    assert torch.equal(got.view(torch.uint8), ref.data.view(torch.uint8)), ("caller stream", comm.rank)
    return 1


def put_refused(comm):
    grid, dims, decomp, dtype = CONFIGS[comm.size][0]
    ps, pd = pencils(comm, grid, dims, decomp)
    u = pa.PencilArray.undef(dtype, ps)
    load(u, global_field(dims, 61, dtype))
    out = pa.PencilArray.undef(dtype, pd)
    t = pa.Transposition(out, u, method=pa.PeerPut())
    out.data.view(torch.uint8).fill_(0x3C)
    torch.cuda.synchronize()
    before = out.data.clone()
    n0 = pa.launch_count()
    try:
        pa.transpose_(t, fft="forward")
        raise AssertionError(f"PeerPut + fft accepted on rank {comm.rank}")
    except pa.ArgumentError as e:
        assert "one-sided methods have no unpack pass" in str(e), str(e)
    torch.cuda.synchronize()
    assert pa.launch_count() == n0, ("launched", comm.rank)
    assert torch.equal(out.data.view(torch.uint8), before.view(torch.uint8))
    return 1


def main():
    comm = pa.comm_world(transport="ipc")
    ran = equal_to_staged(comm) + fft3d(comm) + caller_stream(comm) + put_refused(comm)
    dist.barrier()
    if comm.rank == 0:
        print(f"MP_FFT_PEERGET_OK world={comm.size} runs={ran}")
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
