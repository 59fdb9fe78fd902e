"""Worker of tests/test_gpu_streams.py (launched with torch.distributed.run): ordering on the
caller's streams with `world` processes on the NCCL-free communicator (they may share a GPU).
Hold, then produce, as in test_gpu_streams.py; every operation is warmed up on the default
stream first and every check runs once.

On a (world, 1) grid x->y exchanges over the whole world while y->z is a one-rank line
(nproc == 1) sharing the family's arenas:
* shared arena, both orders: op A on a held stream s1, op B on s2 with no wait of its own --
  the x->y exchange (PointToPoint / Alltoallv, stage_self off and on) and the in-place y->z of a
  ManyPencilArray.  The second op must finish after the spin, both must match the oracle;
* the caller-stream pattern on a side stream: PointToPoint, Alltoallv, PeerPut, PeerGet,
  p2p_chunks = 3, waitall=false + Waitall on a third stream (which must then wait for the
  exchange), against the oracle; the fused FFT of the c128_pow2 cases per line against the
  extended-precision DFT and byte for byte equal to the same transpose on the default stream.
"""
import math
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import pencilarrays_b200 as pa  # noqa: E402
from oracle import pencil_oracle as O  # noqa: E402
from util import CASES, perm_of  # noqa: E402
from fft_ref import EPS, fft_ld, line_errors  # noqa: E402
from gpu_util import hold, hold_cycles, timing_event  # noqa: E402

DIMS = (16, 21, 41)
SPECS = [((2, 3), None), ((1, 3), (2, 3, 1)), ((1, 2), (3, 2, 1))]  # x, y, z
SENTINEL = 0x5A
DEFAULTS = {"p2p_chunks": 1}


def raw(u):
    return u.data.view(torch.uint8).reshape(-1)


def still_held(held, t0, tag):
    """The call came back while the spin still ran: no host synchronisation.  (The host time
    since the hold tells a slow host apart from a call that waited for the device.)"""
    assert not held.query(), tag + (f"{(time.perf_counter() - t0) * 1e3:.1f} ms since the hold",)


def main():
    comm = pa.comm_world(transport="ipc")
    assert comm.transport == "ipc" and comm.handle is not None
    rank, world = comm.rank, comm.size
    for r in range(world):  # calibrate the spin one process at a time: the GPU is shared
        if r == rank:
            hold_cycles()
        dist.barrier()

    grid = (world, 1)
    topo = pa.MPITopology(comm, grid)
    pens = []
    for d, p in SPECS:
        pens.append(pa.Pencil(topo, DIMS, d, permute=perm_of(p)) if not pens else
                    pa.Pencil(pens[-1], decomp_dims=d, permute=perm_of(p)))
    px, py, pz = pens
    opens = [[O.OPencil(O.OTopology(grid, r), DIMS, d, p) for r in range(world)] for d, p in SPECS]
    arrs = [O.scatter(O.global_pattern(DIMS, (), 8), opens[0], (), np.float64)]
    for k in (1, 2):
        nxt = [O.OArray.undef(np.float64, p) for p in opens[k]]
        O.transpose_all(nxt, arrs[-1])
        arrs.append(nxt)
    want = [np.ascontiguousarray(a[rank].data.reshape(-1, order="F")).view(np.uint8) for a in arrs]
    want_dev = [torch.from_numpy(w.copy()).cuda() for w in want]

    def put(u, k):
        raw(u).copy_(want_dev[k])

    def same(t, k):
        return t.view(torch.uint8).reshape(-1).cpu().numpy().tobytes() == want[k].tobytes()

    checks, failures = 0, []

    # ---- shared arena: the x->y exchange and a one-rank in-place y->z, both orders
    MB = pa.ManyPencilArray(torch.float64, py, pz)
    tB = pa.Transposition(MB[2], MB[1])
    assert tB.dim is not None and tB.plan.info.nproc == 1
    # (B's arena growth first: the exchange's recv windows are registered against the grown arena)
    put(MB[1], 1)
    pa.transpose_(tB)
    torch.cuda.synchronize()
    assert same(MB[2].data, 2)
    ux, uy = pa.PencilArray.undef(torch.float64, px), pa.PencilArray.undef(torch.float64, py)
    for method in (pa.PointToPoint(), pa.Alltoallv()):
        tA = pa.Transposition(uy, ux, method=method)
        assert tA.plan.info.nproc == world
        for stage_self in (False, True):
            # name -> (input, oracle index of the input, call, output, oracle index, storage)
            A = (ux, 0, lambda: pa.transpose_(tA, stage_self=stage_self), uy, 1, [ux.data, uy.data])
            B = (MB[1], 1, lambda: pa.transpose_(tB), MB[2], 2, [MB.data])
            for first, second in ((A, B), (B, A)):
                tag = (rank, method, stage_self, "exchange first" if first is A else "one-rank first")
                for op in (first, second):
                    put(op[0], op[1])
                    op[2]()
                    torch.cuda.synchronize()
                    assert same(op[3].data, op[4]), tag
                for op in (first, second):
                    for d in op[5]:
                        d.view(torch.uint8).fill_(SENTINEL)
                put(second[0], second[1])
                s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
                torch.cuda.synchronize()
                with torch.cuda.stream(s1):
                    held, t0 = hold(), time.perf_counter()
                    put(first[0], first[1])
                    first[2]()
                    still_held(held, t0, tag)
                    got1 = first[3].data.clone()
                with torch.cuda.stream(s2):
                    second[2]()
                    b_done = timing_event()
                    still_held(held, t0, tag)
                    got2 = second[3].data.clone()
                torch.cuda.synchronize()
                # (every order and method is reported, not only the first that fails)
                if not same(got1, first[4]):
                    failures.append(tag + ("first op: wrong bytes",))
                if not same(got2, second[4]):
                    failures.append(tag + ("second op: wrong bytes",))
                if not held.elapsed_time(b_done) > 0:
                    failures.append(tag + ("second op ran beside the held one on the shared arena",))
                checks += 1
    assert not failures, failures

    # ---- caller-stream pattern, x->y over the world
    variants = [(pa.PointToPoint(), {}, True), (pa.Alltoallv(), {}, True), (pa.PeerPut(), {}, True),
                (pa.PeerGet(), {}, True), (pa.PointToPoint(), {"p2p_chunks": 3}, True),
                (pa.PointToPoint(), {}, False), (pa.PeerGet(), {}, False)]
    for method, tun, waitall in variants:
        tag = (rank, method, tun, waitall)
        for name, v in tun.items():
            pa.set_tunable(name, v)
        vy = pa.PencilArray.undef(torch.float64, py)
        t = pa.Transposition(vy, ux, method=method)
        put(ux, 0)
        pa.transpose_(t, waitall=waitall)
        pa.Waitall(t)
        torch.cuda.synchronize()
        assert same(vy.data, 1), tag
        raw(ux).fill_(SENTINEL)
        raw(vy).fill_(SENTINEL)
        s, third = torch.cuda.Stream(), torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            held, t0 = hold(), time.perf_counter()
            put(ux, 0)
            pa.transpose_(t, waitall=waitall)
            still_held(held, t0, tag)
            if not waitall:
                with torch.cuda.stream(third):
                    pa.Waitall(t)
                    w_done = timing_event()
                still_held(held, t0, tag)
            got = vy.data.clone()
        torch.cuda.synchronize()
        assert same(got, 1), tag
        if not waitall:  # the third stream waited for the send side of the held exchange
            assert held.elapsed_time(w_done) > 0, tag
        for name in tun:
            pa.set_tunable(name, DEFAULTS[name])
        checks += 1

    # ---- fused FFT of the c128_pow2 case with this world size, on a side stream
    for case in [c for c in CASES if c["name"].startswith("c128_pow2") and math.prod(c["grid"]) == world]:
        extra = case["extra"]
        ctopo = pa.MPITopology(comm, case["grid"])
        (d0, p0), (d1, p1) = case["chain"][:2]
        c0 = pa.Pencil(ctopo, case["dims"], d0, permute=perm_of(p0))
        c1 = pa.Pencil(c0, decomp_dims=d1, permute=perm_of(p1))
        o0 = [O.OPencil(O.OTopology(case["grid"], r), case["dims"], d0, p0) for r in range(world)]
        o1 = [O.OPencil(O.OTopology(case["grid"], r), case["dims"], d1, p1) for r in range(world)]
        rng = np.random.default_rng(7)
        shape = tuple(case["dims"]) + tuple(extra)
        G = rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
        Gb = np.ascontiguousarray(G.reshape(-1, order="F")).view(np.uint8) \
            .reshape(-1, 16).reshape(shape + (16,), order="F")
        a_in = O.scatter(Gb, o0, extra, np.complex128)[rank].data
        a_out = O.scatter(Gb, o1, extra, np.complex128)[rank].data  # lines along axis 0
        x_dev = torch.from_numpy(np.ascontiguousarray(a_in.reshape(-1, order="F")).copy()).cuda()
        src = pa.PencilArray.undef(torch.complex128, c0, *extra)
        L = a_out.shape[0]
        for method in (pa.PointToPoint(), pa.Alltoallv()):
            for direction in ("forward", "backward"):
                tag = (rank, case["name"], method, direction)
                out = pa.PencilArray.undef(torch.complex128, c1, *extra)
                t = pa.Transposition(out, src, method=method)
                src.data.view(-1).copy_(x_dev)
                pa.transpose_(t, fft=direction)
                torch.cuda.synchronize()
                first = out.data.clone()
                got_mem = first.cpu().numpy().reshape(-1).reshape(a_out.shape, order="F")
                ref = fft_ld(np.moveaxis(a_out, 0, -1), -1 if direction == "forward" else 1)
                mx, _ = line_errors(np.moveaxis(got_mem, 0, -1), ref)
                assert mx <= EPS * math.log2(L), tag + (mx,)
                raw(src).fill_(SENTINEL)
                raw(out).fill_(SENTINEL)
                s = torch.cuda.Stream()
                torch.cuda.synchronize()
                with torch.cuda.stream(s):
                    held, t0 = hold(), time.perf_counter()
                    src.data.view(-1).copy_(x_dev)
                    pa.transpose_(t, fft=direction)
                    still_held(held, t0, tag)
                    got = out.data.clone()
                torch.cuda.synchronize()
                assert torch.equal(got.view(torch.uint8), first.view(torch.uint8)), tag
                checks += 1

    dist.barrier()
    if rank == 0:
        print(f"MP_STREAMS_OK world={world} checks={checks}")
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
