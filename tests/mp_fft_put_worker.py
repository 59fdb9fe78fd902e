"""Worker of tests/test_gpu_fft_put.py, launched with torch.distributed.run: the send-side fused
transform + put (PeerPut) with the ranks sharing one GPU over the NCCL-free communicator.

  * transpose_(t, fft_first=d) == fft_ on a copy of src + the plain PeerPut transposition, and
    Transposition(..., rfft_first=True) == rfft_ + the plain PeerPut transposition, byte for byte,
    under waitall True and False + Waitall, tunable multi_put 1 (protocol inside the kernel) and 0
    (standalone flag kernels around it), repeated so that the flag sequence numbers advance;
    lines from 2 ... 8 blocks, ranks without source lines, permuted and unpermuted destinations;
  * the PeerPut 3-d chains -- complex forward and backward, real forward (rfft x, fft y, fft z)
    and real backward (bfft z, bfft y, brfft x) -- in both precisions, against numpy.fft, and
    byte for byte equal to the PointToPoint chains that fuse on the receive side (fft= / brfft=)."""
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
from pencilarrays_b200.transpositions import _brfft_pencil  # noqa: E402

# world size -> [(grid, global dims (L, y, z), decomposed dims of the source pencil, dtype, dperm)]
CONFIGS = {
    2: [((2,), (16, 6, 4), (2,), torch.complex128, (2, 1, 3)),
        ((2,), (512, 3, 2), (2,), torch.complex64, None)],
    3: [((3,), (64, 7, 2), (2,), torch.complex128, (2, 1, 3))],
    4: [((4,), (32, 8, 3), (2,), torch.complex128, None),
        ((2, 2), (16, 8, 4), (2, 3), torch.complex64, (2, 1, 3))],
    5: [((5,), (8, 4, 3), (2,), torch.complex128, (2, 1, 3))],   # y = 4 < 5: a rank without source lines
    6: [((6,), (1024, 7, 2), (2,), torch.complex128, (2, 1, 3)),
        ((3, 2), (64, 6, 4), (2, 3), torch.complex128, None)],
    8: [((8,), (8, 9, 2), (2,), torch.complex128, (2, 1, 3)),
        ((8,), (64, 5, 3), (2,), torch.complex64, (2, 1, 3))],     # y = 5 < 8: three of them
}
EPS = {torch.complex128: np.finfo(np.float64).eps, torch.complex64: np.finfo(np.float32).eps}
NP = {torch.complex128: np.complex128, torch.complex64: np.complex64}
REAL = {torch.complex128: torch.float64, torch.complex64: torch.float32}
NPR = {torch.complex128: np.float64, torch.complex64: np.float32}


def local(A, p):
    return A[tuple(slice(r.start - 1, r.stop - 1) for r in pa.range_local(p))]


def load(u, A):
    u.logical().copy_(torch.from_numpy(np.ascontiguousarray(local(A, u.pencil))))


def global_field(dims, seed, dtype, real=False):
    rng = np.random.default_rng(seed)
    if real:
        return rng.standard_normal(dims).astype(NPR[dtype])
    return (rng.standard_normal(dims) + 1j * rng.standard_normal(dims)).astype(NP[dtype])


def same(a, b):
    return torch.equal(a.data.view(torch.uint8), b.data.view(torch.uint8))


def runs(t, ref_fn, out, check, what, **kw):
    ran = 0
    for multi in (1, 0):
        pa.set_tunable("multi_put", multi)
        try:
            for waitall in (True, False):
                for it in range(2):
                    ref_fn()
                    out.data.view(torch.uint8).fill_(0x5A)
                    pa.transpose_(t, waitall=waitall, **kw)
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
        # complex: dst = transpose(fft_(src))
        ps = pa.Pencil(topo, dims, decomp)
        pd = pa.Pencil(ps, decomp_dims=ddec, permute=pa.Permutation(*dperm) if dperm else None)
        u, mid = pa.PencilArray.undef(dtype, ps), pa.PencilArray.undef(dtype, ps)
        load(u, global_field(dims, 31, dtype))
        src_bytes = u.data.clone()
        ref, out = pa.PencilArray.undef(dtype, pd), pa.PencilArray.undef(dtype, pd)
        t_ref = pa.Transposition(ref, mid, method=pa.PeerPut())
        t = pa.Transposition(out, u, method=pa.PeerPut())
        assert t.fft_first_fusable(), (grid, dims, comm.rank)
        for direction in ("forward", "backward"):
            def unfused():
                mid.data.copy_(u.data)
                pa.fft_(mid, direction)
                pa.transpose_(t_ref)

            def check(key):
                assert same(out, ref), (grid, dims, direction, key, comm.rank)
                assert torch.equal(u.data, src_bytes), ("src", grid, dims, comm.rank)
            ran += runs(t, unfused, out, check, "fft", fft_first=direction)
        # real: dst = transpose(rfft_(src)), N = 2 L
        rdims = (2 * dims[0],) + dims[1:]
        pr = pa.Pencil(topo, rdims, decomp)
        pc = _brfft_pencil(pr)
        pcd = pa.Pencil(pc, decomp_dims=ddec, permute=pa.Permutation(*dperm) if dperm else None)
        x = pa.PencilArray.undef(REAL[dtype], pr)
        load(x, global_field(rdims, 37, dtype, real=True))
        x_bytes = x.data.clone()
        cmid = pa.PencilArray.undef(dtype, pc)
        cref, cout = pa.PencilArray.undef(dtype, pcd), pa.PencilArray.undef(dtype, pcd)
        tc_ref = pa.Transposition(cref, cmid, method=pa.PeerPut())
        tc = pa.Transposition(cout, x, method=pa.PeerPut(), rfft_first=True)
        assert tc.fft_first_fusable(), (grid, rdims, comm.rank)

        def unfused_r():
            pa.rfft_(cmid, x)
            pa.transpose_(tc_ref)

        def check_r(key):
            assert same(cout, cref), (grid, rdims, key, comm.rank)
            assert torch.equal(x.data, x_bytes), ("src", grid, rdims, comm.rank)
        ran += runs(tc, unfused_r, cout, check_r, "rfft")
    return ran


def chains(comm):
    grids = {2: (2, 1), 4: (2, 2), 6: (3, 2)}
    if comm.size not in grids:
        return 0
    grid = grids[comm.size]
    topo = pa.MPITopology(comm, grid)
    ran = 0
    for dtype in (torch.complex128, torch.complex64):
        tol_of = lambda n, m: 8 * EPS[dtype] * math.log2(n) * m  # noqa: E731  (DESIGN §5)
        # ---- complex, forward and backward ----
        dims = (16, 32, 8)
        px = pa.Pencil(topo, dims, (2, 3))
        py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
        pz = pa.Pencil(px, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
        G = global_field(dims, 41, dtype)
        mk = lambda p: pa.PencilArray.undef(dtype, p)  # noqa: E731
        ux, uy, uz, vy, vx = mk(px), mk(py), mk(pz), mk(py), mk(px)
        ax, ay, az, by, bx = mk(px), mk(py), mk(pz), mk(py), mk(px)
        load(ux, G)
        load(ax, G)
        put = lambda d, s: pa.Transposition(d, s, method=pa.PeerPut())  # noqa: E731
        p2p = lambda d, s, **k: pa.Transposition(d, s, method=pa.PointToPoint(), **k)  # noqa: E731
        pa.transpose_(put(uy, ux), fft_first="forward")
        pa.transpose_(put(uz, uy), fft_first="forward")
        pa.fft_(uz, "forward")
        pa.fft_(ax, "forward")
        pa.transpose_(p2p(ay, ax), fft="forward")
        pa.transpose_(p2p(az, ay), fft="forward")
        torch.cuda.synchronize()
        assert same(uz, az), ("complex forward chain != PointToPoint", dtype, comm.rank)
        X = np.fft.fftn(G.astype(np.complex128))
        err = np.abs(uz.logical().cpu().numpy() - local(X, pz)).max() if uz.data.numel() else 0.0
        assert err <= tol_of(math.prod(dims), np.abs(X).max()), ("forward", dtype, comm.rank, err)
        pa.transpose_(put(vy, uz), fft_first="backward")
        pa.transpose_(put(vx, vy), fft_first="backward")
        pa.fft_(vx, "backward")
        pa.fft_(az, "backward")
        pa.transpose_(p2p(by, az), fft="backward")
        pa.transpose_(p2p(bx, by), fft="backward")
        torch.cuda.synchronize()
        assert same(vx, bx), ("complex backward chain != PointToPoint", dtype, comm.rank)
        back = math.prod(dims) * G.astype(np.complex128)
        err = np.abs(vx.logical().cpu().numpy() - local(back, px)).max() if vx.data.numel() else 0.0
        assert err <= 2 * tol_of(math.prod(dims), np.abs(back).max()), ("backward", dtype, comm.rank, err)
        ran += 2
        # ---- real: rfft x, fft y, fft z and back (bfft z, bfft y, brfft x) ----
        rdims = (32, 16, 8)
        rx = pa.Pencil(topo, rdims, (2, 3))
        cx = _brfft_pencil(rx)
        cy = pa.Pencil(cx, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
        cz = pa.Pencil(cx, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
        R = global_field(rdims, 43, dtype, real=True)
        xr, xr2 = pa.PencilArray.undef(REAL[dtype], rx), pa.PencilArray.undef(REAL[dtype], rx)
        load(xr, R)
        wy, wz, qy, qx = mk(cy), mk(cz), mk(cy), mk(cx)
        sx, sy, sz, ty = mk(cx), mk(cy), mk(cz), mk(cy)
        pa.transpose_(pa.Transposition(wy, xr, method=pa.PeerPut(), rfft_first=True))
        pa.transpose_(put(wz, wy), fft_first="forward")
        pa.fft_(wz, "forward")
        pa.rfft_(sx, xr)
        pa.transpose_(p2p(sy, sx), fft="forward")
        pa.transpose_(p2p(sz, sy), fft="forward")
        torch.cuda.synchronize()
        assert same(wz, sz), ("real forward chain != PointToPoint", dtype, comm.rank)
        Xr = np.fft.rfftn(R.astype(np.float64), axes=(1, 2, 0))
        err = np.abs(wz.logical().cpu().numpy() - local(Xr, cz)).max() if wz.data.numel() else 0.0
        assert err <= tol_of(math.prod(rdims), np.abs(Xr).max()), ("real forward", dtype, comm.rank, err)
        pa.transpose_(put(qy, wz), fft_first="backward")
        pa.transpose_(put(qx, qy), fft_first="backward")
        pa.brfft_(xr2, qx)
        xr3 = pa.PencilArray.undef(REAL[dtype], rx)
        pa.fft_(sz, "backward")
        pa.transpose_(p2p(ty, sz), fft="backward")
        pa.transpose_(p2p(xr3, ty, brfft=True))
        torch.cuda.synchronize()
        assert same(xr2, xr3), ("real backward chain != PointToPoint", dtype, comm.rank)
        backr = math.prod(rdims) * R.astype(np.float64)
        err = np.abs(xr2.logical().cpu().numpy() - local(backr, rx)).max() if xr2.data.numel() else 0.0
        assert err <= 2 * tol_of(math.prod(rdims), np.abs(backr).max()), ("real backward", dtype, comm.rank, err)
        ran += 2
    return ran


def main():
    comm = pa.comm_world(transport="ipc")
    ran = equal_to_unfused(comm) + chains(comm)
    dist.barrier()
    if comm.rank == 0:
        print(f"MP_FFT_PUT_OK world={comm.size} runs={ran}")
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
