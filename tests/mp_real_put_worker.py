"""Worker of tests/test_gpu_real_put.py, launched with torch.distributed.run: the send-side fused
real line transforms + put (PeerPut) with the ranks sharing one GPU over the NCCL-free communicator.

  * Transposition(..., r2r_first=kind) == r2r_ on a copy of src + the plain PeerPut transposition,
    and Transposition(..., brfft_first=True) == brfft_ + the plain PeerPut transposition of the
    reals, byte for byte, under waitall True and False + Waitall, tunable multi_put 1 (protocol
    inside the kernel) and 0 (standalone flag kernels around it), repeated so that the flag sequence
    numbers advance;
  * the PeerPut 3-d chains in three kernels each way -- mixed (DCT x, RFFT y, FFT z) and all walls
    (DCT x, y, z) -- in both precisions, against scipy.fft / numpy.fft, and byte for byte equal to
    the PointToPoint chains that fuse on the receive side (r2r= / rfft= / fft= / brfft=);
  * r2r_first= refused on every rank for PointToPoint, Alltoallv and PeerGet with an exchange."""
import math
import os
import sys

import numpy as np
import scipy.fft
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import pencilarrays_b200 as pa  # noqa: E402
from pencilarrays_b200.transpositions import _brfft_pencil  # noqa: E402

# world size -> [(grid, global dims (N, y, z), decomposed dims of the source pencil, dtype, dperm)]
CONFIGS = {
    2: [((2,), (16, 6, 4), (2,), torch.float64, (2, 1, 3)),
        ((2,), (1024, 3, 2), (2,), torch.float32, None)],
    3: [((3,), (32, 7, 2), (2,), torch.float64, (2, 1, 3))],      # 11 / 11 / 10 reals
    4: [((4,), (64, 8, 3), (2,), torch.float64, None),
        ((2, 2), (32, 8, 4), (2, 3), torch.float32, (2, 1, 3))],
    6: [((6,), (2048, 7, 2), (2,), torch.float64, (2, 1, 3)),
        ((3, 2), (64, 6, 4), (2, 3), torch.float64, None)],
    8: [((8,), (16, 9, 2), (2,), torch.float64, (2, 1, 3)),
        ((8,), (64, 5, 3), (2,), torch.float32, (2, 1, 3))],     # y = 5 < 8: ranks without lines
}
EPS = {torch.float64: np.finfo(np.float64).eps, torch.float32: np.finfo(np.float32).eps}
NPR = {torch.float64: np.float64, torch.float32: np.float32}
CPLX = {torch.float64: torch.complex128, torch.float32: torch.complex64}
KINDS = ["REDFT10", "REDFT01", "RODFT10", "RODFT01"]


def local(A, p):
    return A[tuple(slice(r.start - 1, r.stop - 1) for r in pa.range_local(p))]


def load(u, A):
    u.logical().copy_(torch.from_numpy(np.ascontiguousarray(local(A, u.pencil))))


def global_field(dims, seed, dtype, cplx=False):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal(dims)
    if cplx:
        A = A + 1j * rng.standard_normal(dims)
        return A.astype(np.complex128 if dtype == torch.float64 else np.complex64)
    return A.astype(NPR[dtype])


def same(a, b):
    return torch.equal(a.data.view(torch.uint8), b.data.view(torch.uint8))


def runs(t, ref_fn, out, check, what):
    ran = 0
    for multi in (1, 0):
        pa.set_tunable("multi_put", multi)
        try:
            for waitall in (True, False):
                for it in range(2):
                    ref_fn()
                    out.data.view(torch.uint8).fill_(0x5A)
                    pa.transpose_(t, waitall=waitall)
                    if not waitall:
                        pa.Waitall(t)
                    torch.cuda.synchronize()
                    check((what, multi, waitall, it))
                    ran += 1
        finally:
            pa.set_tunable("multi_put", 1)
    return ran


def equal_to_unfused(comm):
    ran = 0
    for (grid, dims, decomp, dtype, dperm) in CONFIGS[comm.size]:
        topo = pa.MPITopology(comm, grid)
        ddec = tuple(1 if d == 2 else d for d in decomp)
        ps = pa.Pencil(topo, dims, decomp)
        pd = pa.Pencil(ps, decomp_dims=ddec, permute=pa.Permutation(*dperm) if dperm else None)
        mid = pa.PencilArray.undef(dtype, ps)
        ref, out = pa.PencilArray.undef(dtype, pd), pa.PencilArray.undef(dtype, pd)
        t_ref = pa.Transposition(ref, mid, method=pa.PeerPut())
        # r2r: dst = transpose(r2r_(src, kind))
        x = pa.PencilArray.undef(dtype, ps)
        load(x, global_field(dims, 51, dtype))
        x_bytes = x.data.clone()
        for kind in KINDS:
            t = pa.Transposition(out, x, method=pa.PeerPut(), r2r_first=kind)
            assert t.fft_first_fusable(), (grid, dims, comm.rank)

            def unfused(kind=kind):
                pa.r2r_(mid, x, kind)
                pa.transpose_(t_ref)

            def check(key, kind=kind):
                assert same(out, ref), (grid, dims, kind, key, comm.rank)
                assert torch.equal(x.data, x_bytes), ("src", grid, dims, comm.rank)
            ran += runs(t, unfused, out, check, kind)
        # c2r: dst = transpose(brfft_(src)), src on the N/2+1-bin counterpart
        pc = _brfft_pencil(ps)
        c = pa.PencilArray.undef(CPLX[dtype], pc)
        load(c, global_field(pc.size_global, 53, dtype, cplx=True))
        c_bytes = c.data.clone()
        tb = pa.Transposition(out, c, method=pa.PeerPut(), brfft_first=True)
        assert tb.fft_first_fusable(), (grid, dims, comm.rank)

        def unfused_b():
            pa.brfft_(mid, c)
            pa.transpose_(t_ref)

        def check_b(key):
            assert same(out, ref), (grid, dims, "c2r", key, comm.rank)
            assert torch.equal(c.data, c_bytes), ("src", grid, dims, comm.rank)
        ran += runs(tb, unfused_b, out, check_b, "c2r")
    return ran


def refusals(comm):
    """r2r_first= with an exchanging plan of another method: refused on every rank, before any
    window or launch."""
    topo = pa.MPITopology(comm, (comm.size,))
    ps = pa.Pencil(topo, (32, 2 * comm.size, 3), (2,))
    pd = pa.Pencil(ps, decomp_dims=(1,), permute=pa.Permutation(2, 1, 3))
    u, v = pa.PencilArray.undef(torch.float64, ps), pa.PencilArray.undef(torch.float64, pd)
    for method in (pa.PointToPoint(), pa.Alltoallv(), pa.PeerGet()):
        n0 = pa.launch_count()
        try:
            pa.Transposition(v, u, method=method, r2r_first="REDFT10")
        except pa.ArgumentError as e:
            assert "needs PeerPut" in str(e), (method, str(e))
        else:
            raise AssertionError(f"r2r_first= accepted with {method} on rank {comm.rank}")
        assert pa.launch_count() == n0
    return 1


def chains(comm):
    grids = {2: (2, 1), 4: (2, 2), 6: (3, 2)}
    if comm.size not in grids:
        return 0
    grid = grids[comm.size]
    topo = pa.MPITopology(comm, grid)
    ran = 0
    put = lambda d, s, **k: pa.Transposition(d, s, method=pa.PeerPut(), **k)  # noqa: E731
    p2p = lambda d, s, **k: pa.Transposition(d, s, method=pa.PointToPoint(), **k)  # noqa: E731
    for dtype in (torch.float64, torch.float32):
        tol_of = lambda n, m: 8 * EPS[dtype] * math.log2(n) * m  # noqa: E731  (DESIGN §5)
        cdt = CPLX[dtype]
        real = lambda p: pa.PencilArray.undef(dtype, p)  # noqa: E731
        cmk = lambda p: pa.PencilArray.undef(cdt, p)  # noqa: E731
        # ---- mixed: DCT x, RFFT y, FFT z, and back (FFT z, c2r y, DCT-III x) ----
        dims = (32, 16, 8)
        rx = pa.Pencil(topo, dims, (2, 3))
        ry = pa.Pencil(rx, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
        cy = _brfft_pencil(ry)  # N/2+1 bins along y
        cz = pa.Pencil(cy, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
        R = global_field(dims, 61, dtype)
        x, x2 = real(rx), real(rx)
        load(x, R)
        load(x2, R)
        wy, wz = real(ry), cmk(cz)
        sy, sz = cmk(cy), cmk(cz)
        # PeerPut: r2r_put x -> y, rfft_put y -> z, fft_ z
        pa.transpose_(put(wy, x, r2r_first="REDFT10"))
        pa.transpose_(put(wz, wy, rfft_first=True))
        pa.fft_(wz, "forward")
        # PointToPoint, receive side: r2r_ x, x -> y + rfft, y -> z + fft
        pa.r2r_(x2, x2, "REDFT10")
        pa.transpose_(p2p(sy, x2, rfft=True))
        pa.transpose_(p2p(sz, sy), fft="forward")
        torch.cuda.synchronize()
        assert same(wz, sz), ("mixed forward chain != PointToPoint", dtype, comm.rank)
        X = np.fft.fft(np.fft.rfft(scipy.fft.dct(R.astype(np.float64), type=2, axis=0), axis=1), axis=2)
        err = np.abs(wz.logical().cpu().numpy() - local(X, cz)).max() if wz.data.numel() else 0.0
        assert err <= tol_of(math.prod(dims), np.abs(X).max()), ("mixed forward", dtype, comm.rank, err)
        # back: fft_put z -> y, brfft_put y -> x, r2r_ x
        qy, qx = cmk(cy), real(rx)
        pa.transpose_(put(qy, wz), fft_first="backward")
        pa.transpose_(put(qx, qy, brfft_first=True))
        pa.r2r_(qx, qx, "REDFT01")
        # receive side: bfft_ z, z -> y + brfft, y -> x + DCT-III
        ty, tx = real(ry), real(rx)
        pa.fft_(sz, "backward")
        pa.transpose_(p2p(ty, sz, brfft=True))
        pa.transpose_(p2p(tx, ty, r2r="REDFT01"))
        torch.cuda.synchronize()
        assert same(qx, tx), ("mixed backward chain != PointToPoint", dtype, comm.rank)
        back = 2 * math.prod(dims) * R.astype(np.float64)
        err = np.abs(qx.logical().cpu().numpy() - local(back, rx)).max() if qx.data.numel() else 0.0
        assert err <= 2 * tol_of(math.prod(dims), np.abs(back).max()), ("mixed backward", dtype, comm.rank, err)
        ran += 2
        # ---- all walls: DCT x, y, z and back ----
        dims = (32, 16, 16)
        rx = pa.Pencil(topo, dims, (2, 3))
        ry = pa.Pencil(rx, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
        rz = pa.Pencil(rx, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
        R = global_field(dims, 67, dtype)
        x, x2 = real(rx), real(rx)
        load(x, R)
        load(x2, R)
        wy, wz, sy, sz = real(ry), real(rz), real(ry), real(rz)
        pa.transpose_(put(wy, x, r2r_first="REDFT10"))
        pa.transpose_(put(wz, wy, r2r_first="REDFT10"))
        pa.r2r_(wz, wz, "REDFT10")
        pa.r2r_(x2, x2, "REDFT10")
        pa.transpose_(p2p(sy, x2, r2r="REDFT10"))
        pa.transpose_(p2p(sz, sy, r2r="REDFT10"))
        torch.cuda.synchronize()
        assert same(wz, sz), ("all-walls forward chain != PointToPoint", dtype, comm.rank)
        X = scipy.fft.dctn(R.astype(np.float64), type=2)
        err = np.abs(wz.logical().cpu().numpy() - local(X, rz)).max() if wz.data.numel() else 0.0
        assert err <= tol_of(math.prod(dims), np.abs(X).max()), ("walls forward", dtype, comm.rank, err)
        qy, qx, ty, tx = real(ry), real(rx), real(ry), real(rx)
        pa.transpose_(put(qy, wz, r2r_first="REDFT01"))
        pa.transpose_(put(qx, qy, r2r_first="REDFT01"))
        pa.r2r_(qx, qx, "REDFT01")
        pa.r2r_(sz, sz, "REDFT01")
        pa.transpose_(p2p(ty, sz, r2r="REDFT01"))
        pa.transpose_(p2p(tx, ty, r2r="REDFT01"))
        torch.cuda.synchronize()
        assert same(qx, tx), ("all-walls backward chain != PointToPoint", dtype, comm.rank)
        back = 8 * math.prod(dims) * R.astype(np.float64)
        err = np.abs(qx.logical().cpu().numpy() - local(back, rx)).max() if qx.data.numel() else 0.0
        assert err <= 2 * tol_of(math.prod(dims), np.abs(back).max()), ("walls backward", dtype, comm.rank, err)
        ran += 2
    return ran


def main():
    comm = pa.comm_world(transport="ipc")
    ran = equal_to_unfused(comm) + refusals(comm) + chains(comm)
    dist.barrier()
    if comm.rank == 0:
        print(f"MP_REAL_PUT_OK world={comm.size} runs={ran}")
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
