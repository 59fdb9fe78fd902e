"""Ordering on the caller's streams, checked deterministically: hold a stream with one bounded
spin (`gpu_util.hold`, about 50 ms), produce the real input behind it, call the library and
consume its output on the same stream.  A kernel that is not ordered behind the caller's
stream reads the sentinel the input held before, and the bytes differ from the reference on
every run; `held.query()` still False right after the call means the call did not synchronise
the host.  Every operation is warmed up first (plan state, arena growth and twiddle tables are
first-use costs).  No check runs twice.

* the caller-stream pattern on a side stream: `transpose_` (plain, stage_self, PointToPoint,
  Alltoallv, waitall=False + Waitall, Waitall on a third stream), in-place ManyPencilArray
  x->y->z, the aliased local permutation, `fft_`, the fused `transpose_(..., fft=...)`,
  `rfft_` / `brfft_` -- byte movers against the oracle, transforms per line against the
  extended-precision DFT (tests/fft_ref.py) and byte for byte against the default stream;
* shared arenas: op A on a held stream, op B of the same pencil family on a second stream
  with no wait of its own; B must finish after the spin (the arena's events order it behind
  A) and both must match the oracle;
* PencilIO through the C ABI (`pa_io_write` / `pa_io_read`) and the Python mirror: ordered
  after work queued on any stream;
* the same with 2 and 4 processes sharing the GPU (tests/mp_streams_worker.py)."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200._lib import lib, check, i64arr
from oracle import pencil_oracle as O
from fft_ref import EPS, brfft_ld, fft_ld, line_errors, rfft_ld
from gpu_util import hold, timing_event

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

DIMS = (16, 21, 41)
# (decomp, perm) of the x, y, z pencils of tests/util.py's ref_transpose cases, and x permuted
# locally (same decomposition: no exchange)
SPECS = {"x": ((2, 3), None), "y": ((1, 3), (2, 3, 1)), "z": ((1, 2), (3, 2, 1)),
         "xp": ((2, 3), (3, 2, 1))}
SENTINEL = 0x5A


def pencils():
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px = pa.Pencil(topo, DIMS, SPECS["x"][0])
    py = pa.Pencil(px, decomp_dims=SPECS["y"][0], permute=pa.Permutation(*SPECS["y"][1]))
    pz = pa.Pencil(py, decomp_dims=SPECS["z"][0], permute=pa.Permutation(*SPECS["z"][1]))
    pxp = pa.Pencil(px, permute=pa.Permutation(*SPECS["xp"][1]))
    return px, py, pz, pxp


_oracle = None


def oracle():
    """Oracle bytes of the x array (global bit pattern, NaN payloads included) and of its
    transposes: name -> (device uint8 tensor, host bytes)."""
    global _oracle
    if _oracle is None:
        t = O.OTopology((1, 1), 0)
        op = {k: O.OPencil(t, DIMS, d, p) for k, (d, p) in SPECS.items()}
        (ax,) = O.scatter(O.global_pattern(DIMS, (), 8), [op["x"]], (), np.float64)
        arrs = {"x": ax}
        for k, frm in (("y", "x"), ("z", "y"), ("xp", "x")):
            arrs[k] = O.OArray.undef(np.float64, op[k])
            O.transpose_all([arrs[k]], [arrs[frm]])
        _oracle = {}
        for k, a in arrs.items():
            raw = np.ascontiguousarray(a.data.reshape(-1, order="F")).view(np.uint8)
            _oracle[k] = (torch.from_numpy(raw.copy()).cuda(), raw.tobytes())
    return _oracle


def raw(u):
    return u.data.view(torch.uint8).reshape(-1)


def put(u, name):
    raw(u).copy_(oracle()[name][0])


def same(got: torch.Tensor, name) -> bool:
    return got.view(torch.uint8).reshape(-1).cpu().numpy().tobytes() == oracle()[name][1]


def file_holds(path, name) -> bool:
    return path.read_bytes() == oracle()[name][1]


def on_side_stream(produce, call, consume):
    """Hold a fresh side stream, then produce, call and consume on it; the call must come back
    while the spin still runs.  Returns what `consume` gave, after a device synchronisation."""
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        held = hold()
        produce()
        call()
        assert not held.query(), "the call returned after the spin had ended: a host synchronisation"
        out = consume()
    torch.cuda.synchronize()
    return out


# ---------------------------------------------------------------------------- caller's stream
VARIANTS = ["plain", "stage_self", "PointToPoint", "Alltoallv", "waitall_false", "waitall_third_stream"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_transpose_on_a_side_stream(variant):
    px, py, pz, _ = pencils()
    ux, uy, uz = (pa.PencilArray.undef(torch.float64, p) for p in (px, py, pz))
    method = pa.Alltoallv() if variant == "Alltoallv" else pa.PointToPoint()
    ts = [pa.Transposition(uy, ux, method=method), pa.Transposition(uz, uy, method=method)]
    waitall = not variant.startswith("waitall")
    third = torch.cuda.Stream()

    def call():
        for t in ts:
            pa.transpose_(t, waitall=waitall, stage_self=(variant == "stage_self"))
            if variant == "waitall_false":
                pa.Waitall(t)
            elif variant == "waitall_third_stream":
                with torch.cuda.stream(third):
                    pa.Waitall(t)

    put(ux, "x")
    call()
    torch.cuda.synchronize()
    assert same(uy.data, "y") and same(uz.data, "z")
    for u in (ux, uy, uz):
        raw(u).fill_(SENTINEL)
    gy, gz = on_side_stream(lambda: put(ux, "x"), call, lambda: (uy.data.clone(), uz.data.clone()))
    assert same(gy, "y"), variant
    assert same(gz, "z"), variant


def test_in_place_many_pencil_array_on_a_side_stream():
    px, py, pz, _ = pencils()
    A = pa.ManyPencilArray(torch.float64, px, py, pz)

    def call():
        pa.transpose_(A[2], A[1])
        pa.transpose_(A[3], A[2])

    put(A[1], "x")
    call()
    torch.cuda.synchronize()
    assert same(A[3].data, "z")
    A.data.view(torch.uint8).fill_(SENTINEL)
    got = on_side_stream(lambda: put(A[1], "x"), call, lambda: A[3].data.clone())
    assert same(got, "z")


def test_aliased_local_permutation_on_a_side_stream():
    px, _, _, pxp = pencils()
    A = pa.ManyPencilArray(torch.float64, px, pxp)
    t = pa.Transposition(A[2], A[1])
    assert t.dim is None  # same decomposition: a local permutation through the scratch arena
    put(A[1], "x")
    pa.transpose_(t)
    torch.cuda.synchronize()
    assert same(A[2].data, "xp")
    A.data.view(torch.uint8).fill_(SENTINEL)
    got = on_side_stream(lambda: put(A[1], "x"), lambda: pa.transpose_(t), lambda: A[2].data.clone())
    assert same(got, "xp")


def _gate(got, ref, n):
    """the per-line gate of tests/test_gpu_fft_exact.py: worst line within eps log2(n)"""
    mx, _ = line_errors(got, ref)
    assert mx <= EPS * math.log2(n), (n, mx)


def _side_stream_equals_default(u_in, x_dev, call, u_out):
    """Run `call` once on the default stream, then on a held side stream behind the production
    of its input: byte for byte the same result.  Returns the default-stream result."""
    u_in.data.copy_(x_dev)
    call()
    torch.cuda.synchronize()
    first = u_out.data.clone()
    raw(u_in).fill_(SENTINEL)
    raw(u_out).fill_(SENTINEL)
    got = on_side_stream(lambda: u_in.data.copy_(x_dev), call, lambda: u_out.data.clone())
    assert torch.equal(got.view(torch.uint8), first.view(torch.uint8))
    return first.cpu().numpy()


@pytest.mark.parametrize("direction", ["forward", "backward"])
def test_fft_on_a_side_stream(direction):
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    L = 32
    u = pa.PencilArray.undef(torch.complex128, pa.Pencil(topo, (L, 12, 8), (2, 3)))
    rng = np.random.default_rng(11)
    x = rng.standard_normal(u.data.shape) + 1j * rng.standard_normal(u.data.shape)
    got = _side_stream_equals_default(u, torch.from_numpy(x).cuda(), lambda: pa.fft_(u, direction), u)
    _gate(got, fft_ld(x, -1 if direction == "forward" else 1), L)


@pytest.mark.parametrize("direction", ["forward", "backward"])
def test_fused_transpose_fft_on_a_side_stream(direction):
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px = pa.Pencil(topo, (16, 32, 8), (2, 3))
    py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    ux, uy, plain = (pa.PencilArray.undef(torch.complex128, p) for p in (px, py, py))
    rng = np.random.default_rng(12)
    x = rng.standard_normal(ux.data.shape) + 1j * rng.standard_normal(ux.data.shape)
    xd = torch.from_numpy(x).cuda()
    ux.data.copy_(xd)
    pa.transpose_(plain, ux)
    torch.cuda.synchronize()
    t = pa.Transposition(uy, ux)
    got = _side_stream_equals_default(ux, xd, lambda: pa.transpose_(t, fft=direction), uy)
    _gate(got, fft_ld(plain.data.cpu().numpy(), -1 if direction == "forward" else 1), 32)


def test_rfft_and_brfft_on_a_side_stream():
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    N = 64
    pr = pa.Pencil(topo, (N, 12, 8), (2, 3))
    pc = pa.Pencil(pr, size_global=(N // 2 + 1, 12, 8))
    xr, back = pa.PencilArray.undef(torch.float64, pr), pa.PencilArray.undef(torch.float64, pr)
    xc = pa.PencilArray.undef(torch.complex128, pc)
    rng = np.random.default_rng(13)
    x = rng.standard_normal(xr.data.shape)
    got = _side_stream_equals_default(xr, torch.from_numpy(x).cuda(), lambda: pa.rfft_(xc, xr), xc)
    _gate(got, rfft_ld(x), N)
    X = rng.standard_normal(xc.data.shape) + 1j * rng.standard_normal(xc.data.shape)
    got = _side_stream_equals_default(xc, torch.from_numpy(X).cuda(), lambda: pa.brfft_(back, xc), back)
    _gate(got, brfft_ld(X, N), N)


# ---------------------------------------------------------------------------- shared arenas
PAIRS = [("many", "many2"), ("stage_self", "permute"), ("permute", "stage_self"),
         ("many", "stage_self")]


@pytest.mark.parametrize("a,b", PAIRS, ids=["-then-".join(p) for p in PAIRS])
def test_shared_arena_pair_serialises_across_streams(a, b):
    """Op A on a held stream s1, then op B on s2 with no wait of its own; every op stages
    through the family's one recv arena on a single rank (in-place ManyPencilArray transposes,
    a stage_self transpose, the aliased local permutation's scratch).  B must wait for A."""
    px, py, pz, pxp = pencils()
    assert len({p.buffers()[2] for p in (px, py, pz, pxp)}) == 1  # one family, one recv arena
    MA, MB = (pa.ManyPencilArray(torch.float64, px, py) for _ in range(2))
    ML = pa.ManyPencilArray(torch.float64, px, pxp)
    ux, uy = pa.PencilArray.undef(torch.float64, px), pa.PencilArray.undef(torch.float64, py)
    ops = {  # name -> (input, call, output, oracle name of the output, storage to clear)
        "many": (MA[1], lambda: pa.transpose_(MA[2], MA[1]), MA[2], "y", [MA.data]),
        "many2": (MB[1], lambda: pa.transpose_(MB[2], MB[1]), MB[2], "y", [MB.data]),
        "stage_self": (ux, lambda: pa.transpose_(uy, ux, stage_self=True), uy, "y", [ux.data, uy.data]),
        "permute": (ML[1], lambda: pa.transpose_(ML[2], ML[1]), ML[2], "xp", [ML.data]),
    }
    for name in (a, b):  # warm-up, and both ops correct on the default stream
        inp, call, out, want, _ = ops[name]
        put(inp, "x")
        call()
        torch.cuda.synchronize()
        assert same(out.data, want), name
    for name in (a, b):
        for d in ops[name][4]:
            d.view(torch.uint8).fill_(SENTINEL)
    put(ops[b][0], "x")  # B's input is ready; A's is produced behind the hold
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        held = hold()
        put(ops[a][0], "x")
        ops[a][1]()
        assert not held.query()
        got_a = ops[a][2].data.clone()
    with torch.cuda.stream(s2):
        ops[b][1]()
        b_done = timing_event()
        assert not held.query()
        got_b = ops[b][2].data.clone()
    torch.cuda.synchronize()
    assert same(got_a, ops[a][3]), (a, b, "A")
    assert same(got_b, ops[b][3]), (a, b, "B")
    assert held.elapsed_time(b_done) > 0, (a, b, "B ran beside A on the shared arena")


# ---------------------------------------------------------------------------- PencilIO
def _io(fn, u, path):
    return fn(u.pencil._h, 0, i64arr(()), 8, 0, C.c_void_p(u.data_ptr()), str(path).encode(), 0)


def test_pa_io_write_waits_for_work_on_other_streams(tmp_path):
    px = pencils()[0]
    u = pa.PencilArray.undef(torch.float64, px)
    path = tmp_path / "w.bin"
    put(u, "x")
    torch.cuda.synchronize()
    check(_io(lib.pa_io_write, u, path))  # warm-up; on one rank the file is the x array
    assert file_holds(path, "x")
    raw(u).fill_(SENTINEL)
    torch.cuda.synchronize()
    path.unlink()
    with torch.cuda.stream(torch.cuda.Stream()):
        hold()
        put(u, "x")
        check(_io(lib.pa_io_write, u, path))
    torch.cuda.synchronize()
    assert file_holds(path, "x")


def test_pa_io_read_waits_for_work_on_other_streams(tmp_path):
    px = pencils()[0]
    u = pa.PencilArray.undef(torch.float64, px)
    path = tmp_path / "r.bin"
    other = np.frombuffer(oracle()["y"][1], dtype=np.uint8)[::-1].tobytes()
    path.write_bytes(other)
    check(_io(lib.pa_io_read, u, path))  # warm-up
    torch.cuda.synchronize()
    assert np.array_equal(raw(u).cpu().numpy(), np.frombuffer(other, np.uint8))
    put(u, "x")
    torch.cuda.synchronize()
    with torch.cuda.stream(torch.cuda.Stream()):
        hold()
        snap = u.data.clone()  # still queued behind the spin when the read starts
        check(_io(lib.pa_io_read, u, path))
    torch.cuda.synchronize()
    assert same(snap, "x")
    assert np.array_equal(raw(u).cpu().numpy(), np.frombuffer(other, np.uint8))


def test_pencilio_mirror_on_a_held_stream(tmp_path):
    """The Python mirror relies on the library's ordering: no synchronisation of its own."""
    px = pencils()[0]
    u, v = pa.PencilArray.undef(torch.float64, px), pa.PencilArray.undef(torch.float64, px)
    fname = tmp_path / "m.bin"
    raw(u).fill_(SENTINEL)
    put(v, "y")
    torch.cuda.synchronize()
    with torch.cuda.stream(torch.cuda.Stream()):
        hold()
        put(u, "x")
        with pa.open_(pa.MPIIODriver(), fname, pa.COMM_SELF, write=True, create=True) as ff:
            ff.write("u", u)
    torch.cuda.synchronize()
    assert file_holds(fname, "x")
    with torch.cuda.stream(torch.cuda.Stream()):
        hold()
        snap = v.data.clone()
        with pa.open_(pa.MPIIODriver(), fname, pa.COMM_SELF, read=True) as ff:
            pa.read_(ff, v, "u")
    torch.cuda.synchronize()
    assert same(snap, "y")
    assert same(v.data, "x")


# ---------------------------------------------------------------------------- processes
@pytest.mark.parametrize("nproc", [2, 4])
def test_streams_ranks_sharing_the_gpu(nproc, tmp_path):
    """tests/mp_streams_worker.py: the multi-rank schedules on side streams, and a one-rank
    in-place transpose sharing the arena with an exchange over the grid line, both orders."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(29691 + nproc),
           os.path.join(HERE, "mp_streams_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1", PA_TEST_TMPDIR=str(tmp_path))
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    assert f"MP_STREAMS_OK world={nproc}" in out.stdout, out.stdout[-2000:]
