"""``Transpositions``: the reference module's public surface
(src/Transpositions/Transpositions.jl) over libpa_b200.

    t = Transposition(dest, src; method=PointToPoint())   # :93-118
    transpose_(t; waitall=True)                           # transpose!(t; waitall)   :170-179
    Waitall(t)                                            # MPI.Waitall(t)           :127-130
    transpose_(dest, src; method=...)                     # transpose!(dest, src)    :160-168
    t = Transposition(real_x, cplx_y; brfft=True)         # GPU extension: real = brfft(transpose)
    t = Transposition(real_y, real_x; r2r="REDFT10")      # GPU extension: real = r2r(transpose)
    t = Transposition(cplx_y, real_x; rfft=True)          # GPU extension: cplx = rfft(transpose)
    transpose_(t; fft_first="forward")                    # GPU extension: dest = transpose(fft(src))
    t = Transposition(cplx_y, real_x; rfft_first=True)    # GPU extension: cplx = transpose(rfft(src))
    t = Transposition(real_y, real_x; r2r_first="REDFT10")  # GPU extension: real = transpose(r2r(src))
    t = Transposition(real_x, cplx_y; brfft_first=True)   # GPU extension: real = transpose(brfft(src))

Python has no ``!`` in identifiers: ``transpose_`` (torch's in-place naming)
stands for ``transpose!``; ``transpose_bang`` is an alias.  Errors follow the
reference: incompatible pencils / extra dims raise ``ArgumentError``.

All work is enqueued on the CURRENT torch CUDA stream and is asynchronous with
respect to the host, like any other CUDA op.
"""
from __future__ import annotations

import ctypes as C
import threading
from typing import NamedTuple

import torch

from . import _lib
from ._lib import lib, check, i64arr, ArgumentError, PlanInfo, PeerInfo, Timings
from .arrays import PencilArray
from .pencils import Pencil
from .permutations import as_tuple


class AbstractTransposeMethod:
    def __repr__(self):
        return type(self).__name__

    def __eq__(self, other):
        return type(self) is type(other)

    def __hash__(self):
        return hash(type(self).__name__)


class PointToPoint(AbstractTransposeMethod):  # Transpositions.jl:18
    code = _lib.PA_POINT_TO_POINT


class Alltoallv(AbstractTransposeMethod):  # Transpositions.jl:19
    code = _lib.PA_ALLTOALLV


class PeerPut(AbstractTransposeMethod):
    """GPU extension (no reference counterpart): one-sided puts over NVLink.

    Each remote block is packed by a kernel that stores straight into the
    destination rank's ``dest`` array through a peer mapping -- no ``send_buf``,
    no ``recv_buf``, no unpack pass.  ``Transposition(dest, src; method=PeerPut())``
    is COLLECTIVE over the communicator (like ``MPI_Win_create``): it exchanges
    CUDA IPC handles of ``dest``.  Falls back to the staged PointToPoint
    schedule when ``src`` and ``dest`` alias (in-place transposes).
    ``transpose_(t, fft_first=...)`` and ``Transposition(..., rfft_first=True)`` (``r2r_first=``,
    ``brfft_first=True``) fuse the transform along ``src``'s first memory dimension into the put
    kernel: one kernel per rank loads every local source line, transforms it and stores the
    outputs into the peers' ``dest``.
    """
    code = _lib.PA_PEER_PUT


class PeerGet(AbstractTransposeMethod):
    """Pull flavour of :class:`PeerPut`: the unpack kernel of each remote block
    loads straight out of the source rank's ``src`` array over NVLink.  The
    window is on ``src``; ``waitall=False`` defers only the fence that guards
    the reuse of ``src`` -- the role ``MPI.Waitall(t)`` has in the reference.
    ``transpose_(t, fft=...)`` fuses the FFT here too: one kernel per rank gathers
    every line from the peers' ``src`` arrays and its own, transforms and stores it."""
    code = _lib.PA_PEER_GET


_tunables = {}


def set_tunable(name: str, value: int):
    """``pa_set_tunable`` + a host-side record (the mirror needs to know whether the
    staged methods run over this library's own NVLink copy kernels)."""
    check(lib.pa_set_tunable(name.encode(), int(value)))
    _tunables[name] = int(value)


class _Plan:
    """Owner of one ``pa_plan`` handle (geometry + launch descriptors + streams)."""

    def __init__(self, pin: Pencil, pout: Pencil, extra_dims, elsize: int, method):
        h = C.c_void_p()
        check(lib.pa_plan_create(pin._h, pout._h, len(extra_dims), i64arr(extra_dims), elsize,
                                 method.code, C.byref(h)))
        self.h = h
        info = PlanInfo()
        check(lib.pa_plan_get_info(h, C.byref(info)))
        self.info = info
        self._ipc_handles = []   # every pa_ipc_import this plan holds a reference for
        self._windows = {}       # key -> registered local pointer
        self._arena_ptr = None   # recv_buf the peers' arena windows were registered against

    def __del__(self):
        try:
            lib.pa_plan_destroy(self.h)  # (synchronises nothing: the mappings go after it)
            for hh in self._ipc_handles:
                lib.pa_ipc_release(hh)
        except Exception:
            pass

    def peer(self, n: int) -> PeerInfo:
        p = PeerInfo()
        check(lib.pa_plan_get_peer(self.h, n, C.byref(p)))
        return p

    def block(self, op: int, n: int = 1):
        d = _lib.BlockDesc()
        check(lib.pa_plan_get_block(self.h, op, n, C.byref(d)))
        return d


def _get_plan(pin: Pencil, pout: Pencil, extra_dims, elsize, method) -> _Plan:
    # plans are cached on the output pencil: `transpose!(dest, src)` builds a
    # fresh Transposition per call in the reference (:165); re-deriving the
    # geometry is cheap there, re-creating streams/events per call is not here.
    key = (id(pin), tuple(extra_dims), int(elsize), method.code)
    hit = pout._plans.get(key)
    if hit is not None and hit[0] is pin:
        return hit[1]
    plan = _Plan(pin, pout, extra_dims, elsize, method)
    pout._plans[key] = (pin, plan)
    return plan


_bound = threading.local()


def _stream_ptr():
    # keep the library's (statically linked) CUDA runtime on torch's current device
    dev = torch.cuda.current_device()
    if getattr(_bound, "dev", None) != dev:
        check(lib.pa_set_device(dev))
        _bound.dev = dev
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _exchange_windows(plan: _Plan, key, ptr: int, comm, setter):
    """Collective over the communicator (like ``MPI_Win_create``): expose the device
    allocation at ``ptr`` (0: this rank owns nothing -- it exports nothing but still
    maps its peers') to the peers of the plan's grid line, map theirs and hand each
    mapped pointer to ``setter(n, mapped)``.

    Whether anything has to be (re)mapped is decided COLLECTIVELY: a rank whose own
    pointer is unchanged still takes part when a peer re-allocated its array.
    Failures never leave ranks stuck in a collective: all raise together."""
    import torch.distributed as dist

    if not dist.is_initialized():
        raise ArgumentError(_lib.PA_EINVAL, "one-sided / peer-memory transposes need "
                            "torch.distributed for the handle exchange")
    _stream_ptr()  # binds the library to torch's current device
    changed = plan._windows.get(key) != ptr
    h = C.create_string_buffer(_lib.PA_IPC_HANDLE_BYTES)
    off = C.c_int64()
    err = None
    if ptr:
        st = lib.pa_ipc_export(C.c_void_p(ptr), h, C.byref(off))
        if st != _lib.PA_OK:
            err = f"rank {comm.rank}: export failed: {lib.pa_last_error().decode()}"
    allh = [None] * comm.size
    dist.all_gather_object(allh, (comm.rank, bytes(h.raw) if ptr else None, off.value, err, changed))
    errs = [e for (_, _, _, e, _) in allh if e]
    if not errs and not any(c for (_, _, _, _, c) in allh):
        return  # every rank still holds current mappings
    if not errs:
        byrank = {r: (hh, oo) for (r, hh, oo, _, _) in allh}
        for n in range(1, plan.info.nproc + 1):
            peer = plan.peer(n)
            if peer.is_self:
                continue
            hh, oo = byrank[peer.world_rank]
            if hh is None:
                continue  # that rank owns nothing: nothing will be put to / got from it
            mapped = C.c_void_p()
            st = lib.pa_ipc_import(hh, oo, C.byref(mapped))
            if st == _lib.PA_OK:
                plan._ipc_handles.append(hh)
                st = setter(n, mapped)
            if st != _lib.PA_OK:
                err = f"rank {comm.rank}: import from rank {peer.world_rank} failed: " \
                      f"{lib.pa_last_error().decode()}"
                break
    oks = [None] * comm.size
    dist.all_gather_object(oks, err)
    errs += [e for e in oks if e]
    if errs:
        raise _lib.DeviceError(_lib.PA_ECUDA, "peer window setup failed: " + "; ".join(errs[:3]))
    plan._windows[key] = ptr


def _register_window(plan: _Plan, Ao: PencilArray, Ai: PencilArray, comm):
    """Window of a one-sided method on ``Ao`` (``dest`` for PeerPut, ``src`` for
    PeerGet): ``pa_ipc_export`` / ``pa_ipc_import`` / ``pa_plan_set_window``."""
    lo, hi = Ao.data_ptr(), Ao.data_ptr() + Ao.data.numel() * Ao.elsize
    si, ei = Ai.data_ptr(), Ai.data_ptr() + Ai.data.numel() * Ai.elsize
    # same rule as libpa_b200 (same base pointer, or overlapping ranges); views of one
    # ManyPencilArray alias on every rank, empty ones included
    aliased = (lo < ei and si < hi) or (lo != 0 and lo == si) or \
        (Ao._owner is not None and Ao._owner is Ai._owner)
    if aliased:
        # in place: libpa_b200 takes the staged schedule.  (Aliasing is a property of the
        # ManyPencilArray, the same on every rank, so skipping the collective is symmetric.)
        return _register_arenas(plan, Ao.pencil if plan.info.method == _lib.PA_PEER_PUT
                                else Ai.pencil, comm)
    ptr = lo if Ao.data.numel() > 0 else 0
    _register_window_ptr(plan, ptr, comm)


def _register_window_ptr(plan: _Plan, ptr: int, comm):
    _exchange_windows(plan, ("win", ptr), ptr, comm,
                      lambda n, mapped: lib.pa_plan_set_window(plan.h, C.c_void_p(ptr), n, mapped))


def _uses_ipc_exchange(comm) -> bool:
    return comm.transport == "ipc" or bool(_tunables.get("ipc_exchange"))


def _register_arenas(plan: _Plan, Po: Pencil, comm):
    """Own-kernel exchange of the staged methods: reserve the arenas at the maximum
    size over the ranks (so that every rank re-allocates -- or not -- at the same
    call), then expose ``recv_buf`` to the peers (``pa_plan_set_recv_window``)."""
    import torch.distributed as dist

    if plan.info.dim == 0 or plan.info.nproc == 1 or not _uses_ipc_exchange(comm):
        return
    _stream_ptr()
    sizes = [None] * comm.size
    dist.all_gather_object(sizes, (plan.info.send_bytes, plan.info.recv_bytes))
    check(lib.pa_pencil_reserve(Po._h, max(1, max(s for s, _ in sizes)),
                                max(1, max(r for _, r in sizes))))
    fam = Po._family
    plans = fam.__dict__.setdefault("_ipc_plans", [])
    if not any(p is plan for p in plans):
        plans.append(plan)
    _, _, rp, _ = Po.buffers()
    for pl in plans:  # every plan sharing these arenas (same list, same order on every rank)
        _exchange_windows(pl, "arena", rp, comm,
                          lambda n, mapped, pl=pl: lib.pa_plan_set_recv_window(pl.h, n, mapped))


def _real_pencil_of(cplx: Pencil, n: int) -> Pencil:
    """The real counterpart of a complex pencil with ``n`` points along its first memory dim:
    :func:`_rfft_pencil` when ``n`` is even, else derived once per (pencil, ``n``) in the same
    family.  (An odd ``n`` is refused later, by the C verdict, as any other line length.)"""
    pr = _rfft_pencil(cplx)
    ax = as_tuple(cplx.perm, cplx.ndims)[0] - 1
    if pr.size_global[ax] == n:
        return pr
    odd = cplx.__dict__.setdefault("_rfft_real_n", {})
    if n not in odd:
        odd[n] = Pencil(cplx, size_global=tuple(n if d == ax else m
                                                for d, m in enumerate(cplx.size_global)))
    return odd[n]


def _brfft_pencil(real: Pencil) -> Pencil:
    """The complex counterpart of a real pencil -- N//2+1 points along its first memory dim --
    derived once per real pencil.  It is in the same family (shares the staging arenas), so
    repeated ``Transposition(..., brfft=True)`` reuse one plan cached on it."""
    pc = real.__dict__.get("_brfft_cplx")
    if pc is None:
        ax = as_tuple(real.perm, real.ndims)[0] - 1
        pc = Pencil(real, size_global=tuple(n // 2 + 1 if d == ax else n
                                            for d, n in enumerate(real.size_global)))
        real._brfft_cplx = pc
    return pc


def _rfft_pencil(cplx: Pencil) -> Pencil:
    """The real counterpart of a complex pencil of M points along its first memory dim -- N =
    2 (M - 1) points there -- derived once per complex pencil, in the same family, like
    :func:`_brfft_pencil`."""
    pr = cplx.__dict__.get("_rfft_real")
    if pr is None:
        ax = as_tuple(cplx.perm, cplx.ndims)[0] - 1
        pr = Pencil(cplx, size_global=tuple(2 * (n - 1) if d == ax else n
                                            for d, n in enumerate(cplx.size_global)))
        cplx._rfft_real = pr
    return pr


_BRFFT_PAIRS = {(torch.float64, torch.complex128), (torch.float32, torch.complex64)}
_REAL_DTYPES = (torch.float64, torch.float32)


class _Fused(NamedTuple):
    """One fused line transform, keyed by (side, mode) in :data:`_FUSED`."""
    kw: str          # the kwarg that asks for it, as the messages name it
    real: str        # the real array: "Ai" (src), "Ao" (dest), "both" or "" (complex on both sides)
    pencils: object  # (Ai, Ao) -> the plan's (Pi, Po): a derived pencil on the complex side
    elsize: str      # the array that gives the plan's element size
    verdict: str     # the pa_plan_*check* that answers whether the fused kernel can run
    call: object     # (t, comm, src, dst, flags, stream) -> status


def _own(Ai, Ao):
    return Ai.pencil, Ao.pencil


def _brfft_first_pencils(Ai, Ao):
    # the plan's input: the real counterpart of src, N points as in dest
    ax = as_tuple(Ai.pencil.perm, Ai.pencil.ndims)[0] - 1
    return _real_pencil_of(Ai.pencil, Ao.pencil.size_global[ax]), Ao.pencil


# receive side: dest = T(transpose(src)); send side: dest = transpose(T(src))
_FUSED = {
    ("unpack", "fft"): _Fused(
        "fft", "", _own, "Ai", "pa_plan_fft_check_ex",
        lambda t, comm, s, d, f, st: lib.pa_transpose(t.plan.h, comm, s, d, f, st)),
    ("unpack", "brfft"): _Fused(
        "brfft", "Ao", lambda Ai, Ao: (Ai.pencil, _brfft_pencil(Ao.pencil)), "Ai", "pa_plan_brfft_check",
        lambda t, comm, s, d, f, st: lib.pa_transpose_brfft(t.plan.h, comm, t.Ao.pencil._h, s, d, f, st)),
    ("unpack", "r2r"): _Fused(
        "r2r", "both", _own, "Ai", "pa_plan_real_check",
        lambda t, comm, s, d, f, st: lib.pa_transpose_r2r(t.plan.h, comm, _R2R_KINDS[t._op[2]], s, d, f, st)),
    ("unpack", "rfft"): _Fused(
        "rfft", "Ai", lambda Ai, Ao: (Ai.pencil, _rfft_pencil(Ao.pencil)), "Ai", "pa_plan_real_check",
        lambda t, comm, s, d, f, st: lib.pa_transpose_rfft(t.plan.h, comm, t.Ao.pencil._h, s, d, f, st)),
    ("put", "fft"): _Fused(
        "fft_first", "", _own, "Ai", "pa_plan_fft_put_check",
        lambda t, comm, s, d, f, st: lib.pa_fft_put(t.plan.h, comm, s, d, f, st)),
    ("put", "rfft"): _Fused(
        "rfft_first", "Ai", lambda Ai, Ao: (_brfft_pencil(Ai.pencil), Ao.pencil), "Ao",
        "pa_plan_rfft_put_check",
        lambda t, comm, s, d, f, st: lib.pa_rfft_put(t.plan.h, comm, t.Ai.pencil._h, s, d, f, st)),
    ("put", "r2r"): _Fused(
        "r2r_first", "both", _own, "Ai", "pa_plan_real_put_check",
        lambda t, comm, s, d, f, st: lib.pa_r2r_put(t.plan.h, comm, _R2R_KINDS[t._op[2]], s, d, f, st)),
    ("put", "brfft"): _Fused(
        "brfft_first", "Ao", _brfft_first_pencils, "Ao", "pa_plan_real_put_check",
        lambda t, comm, s, d, f, st: lib.pa_brfft_put(t.plan.h, comm, t.Ai.pencil._h, s, d, f, st)),
}


def _article(kw: str) -> str:
    return "a" if kw.startswith("b") else "an"


class Transposition:
    """Holds data for transposition between two pencil configurations (:69-119).

    ``brfft=True`` (GPU extension): ``Ao`` is float64 (float32) on a real x-pencil of N points
    along its first memory dim and ``Ai`` complex128 (complex64) on the complex y-pencil; the plan
    is the complex y -> x plan to the real pencil's N//2+1 counterpart, and ``transpose_(t)``
    writes ``Ao = brfft(transpose(Ai))`` in one kernel after the exchange (``pa_transpose_brfft``):
    the last step of a PencilFFTs real-input backward transform, without the complex x array.

    ``r2r="REDFT10"`` (``"REDFT01"``, ``"RODFT10"``, ``"RODFT01"``; GPU extension): ``Ao`` and
    ``Ai`` are float64 (float32) arrays on two real pencils, and ``transpose_(t)`` writes ``Ao =
    r2r_(transpose(Ai), kind)`` along ``Ao``'s first memory dim in one kernel after the exchange
    (``pa_transpose_r2r``).  ``rfft=True``: ``Ai`` is float64 (float32) on a real x-pencil and
    ``Ao`` complex128 (complex64) on the complex y-pencil of N//2+1 points along its first memory
    dim; the plan is the real x -> y plan to ``Ao``'s real counterpart, and ``transpose_(t)``
    writes ``Ao = rfft_(transpose(Ai))`` (``pa_transpose_rfft``).  Both are byte for byte the
    unfused pair, without the array in between.

    ``rfft_first=True`` (GPU extension, send side): ``Ai`` is float64 (float32) on a real pencil of
    N points along its first memory dim and ``Ao`` complex128 (complex64); the plan is the complex
    plan from ``Ai``'s N//2+1 counterpart to ``Ao``'s pencil, and ``transpose_(t)`` writes ``Ao =
    transpose(rfft_(Ai))`` in one kernel per rank (``pa_rfft_put``): ``PeerPut``, or a local
    transposition with any method.  Byte for byte ``rfft_`` followed by the plain transposition.
    ``brfft``, ``r2r``, ``rfft`` and ``rfft_first`` exclude each other.

    ``r2r_first="REDFT10"`` (``"REDFT01"``, ``"RODFT10"``, ``"RODFT01"``; GPU extension, send side):
    ``Ai`` and ``Ao`` are float64 (float32) arrays on two real pencils, and ``transpose_(t)`` writes
    ``Ao = transpose(r2r_(Ai, kind))`` along ``Ai``'s first memory dim in one kernel per rank
    (``pa_r2r_put``).  ``brfft_first=True``: ``Ai`` is complex128 (complex64) on a complex pencil
    and ``Ao`` float64 (float32); N comes from ``Ao``'s pencil, the plan is the real plan from
    ``Ai``'s N-point counterpart to ``Ao``'s pencil, and ``transpose_(t)`` writes ``Ao =
    transpose(brfft(Ai))`` (``pa_brfft_put``).  Both need ``PeerPut`` when the transposition
    exchanges data (any method when it is local) and are byte for byte the unfused pair.  Every
    one of ``brfft``, ``r2r``, ``rfft``, ``rfft_first``, ``r2r_first`` and ``brfft_first`` excludes
    the others."""

    def __init__(self, Ao: PencilArray, Ai: PencilArray, *, method=None, brfft=False, r2r=None,
                 rfft=False, rfft_first=False, r2r_first=None, brfft_first=False):
        method = PointToPoint() if method is None else method
        asked = [(("unpack", "brfft", None), bool(brfft)), (("unpack", "r2r", r2r), r2r is not None),
                 (("unpack", "rfft", None), bool(rfft)), (("put", "rfft", None), bool(rfft_first)),
                 (("put", "r2r", r2r_first), r2r_first is not None),
                 (("put", "brfft", None), bool(brfft_first))]
        ops = [op for op, on in asked if on]
        if len(ops) > 1:
            raise ArgumentError(_lib.PA_EINVAL, "brfft=, r2r=, rfft= and rfft_first= exclude each other"
                                if sum(on for _, on in asked[:4]) > 1 else
                                "brfft=, r2r=, rfft=, rfft_first=, r2r_first= and brfft_first= exclude "
                                "each other")
        # (side, mode, r2r kind) of the fused transform; None: a complex transposition, fft= /
        # fft_first= choose at transpose_
        self._op = ops[0] if ops else None
        if Ai.extra_dims != Ao.extra_dims:  # :99-103
            raise ArgumentError(_lib.PA_EINVAL,
                                "incompatible number of extra dimensions of PencilArrays: "
                                f"{Ai.extra_dims} != {Ao.extra_dims}")
        row = _FUSED[self._op[:2]] if self._op else _FUSED[("unpack", "fft")]
        kw = row.kw
        if row.real == "both":
            if self._op[2] not in _R2R_KINDS:
                raise ArgumentError(_lib.PA_EINVAL,
                                    f"{kw} must be one of {sorted(_R2R_KINDS)}: got {self._op[2]!r}")
            if Ai.dtype != Ao.dtype or Ai.dtype not in _REAL_DTYPES:
                raise ArgumentError(_lib.PA_EINVAL, f"{kw}: dest and src must be two float64 or two "
                                    f"float32 arrays: got {Ao.dtype} and {Ai.dtype}")
        elif row.real:
            real, cplx, names = (Ai, Ao, "src and dest") if row.real == "Ai" else (Ao, Ai, "dest and src")
            if (real.dtype, cplx.dtype) not in _BRFFT_PAIRS:
                raise ArgumentError(_lib.PA_EINVAL, f"{kw}: {names} must be float64 and complex128, "
                                    f"or float32 and complex64: got {real.dtype} and {cplx.dtype}")
        elif Ai.dtype != Ao.dtype:  # PencilArray{T,N} for both arguments
            raise ArgumentError(_lib.PA_EINVAL, f"element types differ: {Ai.dtype} != {Ao.dtype}")
        Pi, Po = row.pencils(Ai, Ao)
        if Pi.topology is not Po.topology:  # assert_compatible uses `!==` (:182-184)
            raise ArgumentError(_lib.PA_EINCOMPAT, "pencil topologies must be the same.")
        self.Pi, self.Po, self.Ai, self.Ao = Pi, Po, Ai, Ao
        self.method = method
        elsize = (Ao if row.elsize == "Ao" else Ai).elsize
        self._plan = _get_plan(Pi, Po, Ai.extra_dims, elsize, method)  # remaining checks in C
        d = self._plan.info.dim
        self.dim = None if d == 0 else d  # :110
        exchange = d != 0 and self._plan.info.nproc > 1
        if self._op and self._op[0] == "put":
            # (the same verdict on every rank of the line: refused before the collective window setup)
            check(getattr(lib, row.verdict)(self._plan.h, self._precision()))
        elif self._op and exchange and isinstance(method, (PeerPut, PeerGet)):
            # (the same on every rank of the line: refused before the collective window setup)
            raise ArgumentError(_lib.PA_EINVAL, f"{kw}: the one-sided methods have no unpack "
                                "pass to fuse with; use PointToPoint / Alltoallv")
        if exchange and Pi.topology.comm.handle is not None:
            comm = Pi.topology.comm
            if isinstance(method, PeerPut):
                _register_window(self._plan, Ao, Ai, comm)
            elif isinstance(method, PeerGet):
                _register_window(self._plan, Ai, Ao, comm)
            else:
                _register_arenas(self._plan, Po, comm)

    def _is(self, side, mode):
        return self._op is not None and self._op[:2] == (side, mode)

    brfft = property(lambda self: self._is("unpack", "brfft"))
    r2r = property(lambda self: self._op[2] if self._is("unpack", "r2r") else None)
    rfft = property(lambda self: self._is("unpack", "rfft"))
    rfft_first = property(lambda self: self._is("put", "rfft"))
    r2r_first = property(lambda self: self._op[2] if self._is("put", "r2r") else None)
    brfft_first = property(lambda self: self._is("put", "brfft"))

    def _precision(self) -> int:
        """PA_FFT_F32 for single precision: a plan only knows its element size, and 8 bytes is
        float64 as well as complex64.  A complex transposition is single precision for complex64
        arrays only."""
        single = (torch.complex64,) if self._op is None else (torch.float32, torch.complex64)
        return _lib.PA_FFT_F32 if self.Ai.dtype in single else 0

    def _fusable(self, side) -> bool:
        op = self._op or (side, "fft")
        if op[0] != side:
            return False
        return getattr(lib, _FUSED[op[:2]].verdict)(self._plan.h, self._precision()) == _lib.PA_OK

    @property
    def plan(self) -> _Plan:
        return self._plan

    def timings(self) -> Timings:
        t = Timings()
        check(lib.pa_plan_timings(self._plan.h, C.byref(t)))
        return t

    def enable_timing(self, on=True):
        check(lib.pa_plan_enable_timing(self._plan.h, 1 if on else 0))

    def fft_fusable(self) -> bool:
        """Whether ``transpose_(self, fft=...)`` can run the unpack and the 1-d FFT as one
        kernel (``pa_plan_fft_check``).  The answer depends on the global geometry only, so it
        is the same on every rank of the grid line; when it is False, transpose and transform
        separately.  complex64 arrays are asked about in single precision (``PA_FFT_F32``).
        With ``PeerGet`` the answer covers the one-sided fused kernel as well; ``PeerPut`` has
        nothing to fuse with, and ``transpose_(t, fft=...)`` refuses it whatever this says.
        For a ``brfft=True`` transposition: whether ``pa_transpose_brfft`` can run
        (``pa_plan_brfft_check``); for ``r2r=`` / ``rfft=True``: whether ``pa_transpose_r2r`` /
        ``pa_transpose_rfft`` can (``pa_plan_real_check``, one answer for both); for an
        ``rfft_first=True`` (``r2r_first=``, ``brfft_first=True``) one: False (see
        :meth:`fft_first_fusable`)."""
        return self._fusable("unpack")

    def fft_first_fusable(self) -> bool:
        """Whether the send-side fused kernel can run on this transposition: for a complex one
        ``transpose_(self, fft_first=...)`` (``pa_plan_fft_put_check``), for an ``rfft_first=True``
        one ``transpose_(self)`` (``pa_plan_rfft_put_check``), for an ``r2r_first=`` or
        ``brfft_first=True`` one ``transpose_(self)`` (``pa_plan_real_put_check``).  Needs ``PeerPut``
        when the transposition exchanges data; the answer is the same on every rank of the grid
        line."""
        return self._fusable("put")


def Waitall(t: Transposition):
    """``MPI.Waitall(t::Transposition)`` (:127-130): sends done => send_buf reusable."""
    check(lib.pa_wait(t.plan.h, _stream_ptr()))
    return None


def transpose_(*args, method=None, waitall=True, overlap=True, stage_self=False, fft=None,
               fft_first=None):
    """``transpose!(dest, src; method)`` or ``transpose!(t; waitall)`` (:160-179).

    ``fft="forward"`` / ``"backward"`` (GPU extension, SURVEY 8 f2): the unpack and the
    1-d complex FFT along ``dest``'s contiguous dimension -- the step a PencilFFTs-style
    plan runs next -- execute as one kernel; ``dest`` receives the transformed array.
    complex128 arrays are transformed in double precision, complex64 in single.  With the
    staged methods the fused kernel is the unpack; with ``PeerGet`` it reads every line straight
    out of the peers' ``src`` arrays (one kernel per rank, no staging; ``waitall=False`` defers
    only the fence that guards the reuse of ``src``).  ``PeerPut`` is refused.

    ``fft_first="forward"`` / ``"backward"`` (GPU extension, send side): ``dest`` receives the
    transposition of the 1-d FFT of ``src`` along ``src``'s first memory dimension, in one kernel
    per rank that loads the source lines, transforms them and stores every bin into the rank
    that owns it (``pa_fft_put``): ``PeerPut``, or a local transposition with any method.  Byte
    for byte ``fft_`` on a copy of ``src`` followed by the plain transposition; ``fft=`` and
    ``fft_first=`` exclude each other.

    A ``Transposition(..., brfft=True)`` (``r2r=``, ``rfft=True``, ``rfft_first=True``,
    ``r2r_first=``, ``brfft_first=True``) runs the fused transpose + complex-to-real (real-to-real,
    real-to-complex) transform; ``fft=`` and ``fft_first=`` do not apply to it."""
    if len(args) == 1 and isinstance(args[0], Transposition):
        t = args[0]
    elif len(args) == 2:
        dest, src = args
        if dest is src:  # same pencil & same data (:164)
            return dest
        t = Transposition(dest, src, method=method)
        waitall = True
    else:
        raise TypeError("transpose_(dest, src; method) or transpose_(t; waitall)")
    flags = (_lib.PA_WAITALL if waitall else 0) | (0 if overlap else _lib.PA_NO_OVERLAP) | (
        _lib.PA_STAGE_SELF if stage_self else 0)
    op = t._op
    if op is not None:
        kw = _FUSED[op[:2]].kw
        if op[0] == "put":
            if fft is not None or fft_first is not None:
                raise ArgumentError(_lib.PA_EINVAL, f"{_article(kw)} {kw} transposition implies its "
                                    "transform: transpose_(t) without fft= / fft_first=")
        elif fft_first is not None:
            raise ArgumentError(_lib.PA_EINVAL, "fft_first= applies to complex transpositions only")
        elif fft is not None:
            raise ArgumentError(_lib.PA_EINVAL, f"{_article(kw)} {kw} transposition implies its "
                                "transform: transpose_(t) without fft=")
    elif fft_first is not None:
        if fft is not None:
            raise ArgumentError(_lib.PA_EINVAL, "fft= and fft_first= exclude each other")
        op, flags = ("put", "fft"), flags | _direction("fft_first", fft_first)
    elif fft is not None:
        op, flags = ("unpack", "fft"), flags | _direction("fft", fft)
    if op is not None:
        flags |= t._precision()
    row = _FUSED[op[:2]] if op else _FUSED[("unpack", "fft")]
    # (an empty local array may have a null data pointer: the library accepts that)
    check(row.call(t, t.Pi.topology.comm.handle, C.c_void_p(t.Ai.data_ptr() or None),
                   C.c_void_p(t.Ao.data_ptr() or None), flags, _stream_ptr()))
    return t if len(args) == 1 else args[0]


def _direction(kw: str, value) -> int:
    if value in ("forward", -1):
        return _lib.PA_FFT_FORWARD
    if value in ("backward", 1):
        return _lib.PA_FFT_BACKWARD
    raise ArgumentError(_lib.PA_EINVAL, f"{kw} must be 'forward' or 'backward'")


transpose_bang = transpose_


def fft_(u: PencilArray, direction="forward"):
    """In-place 1-d complex FFT of ``u`` along its contiguous (first memory) dimension: the
    first step of a PencilFFTs-style 3-d transform (the other two are ``transpose_(t,
    fft=...)``).  Same kernel as the fused unpack+FFT, without a transposition.  complex128 or
    complex64 (single precision)."""
    t = Transposition(u, u)
    return transpose_(t, fft=direction).Ao


def _rfft(dest: PencilArray, src: PencilArray, forward: bool):
    real, cplx = (src, dest) if forward else (dest, src)
    pairs = {(torch.float64, torch.complex128): 0, (torch.float32, torch.complex64): _lib.PA_FFT_F32}
    if (real.dtype, cplx.dtype) not in pairs:
        raise ArgumentError(_lib.PA_EINVAL, "real and complex arrays must be float64 and complex128, "
                            f"or float32 and complex64: got {real.dtype} and {cplx.dtype}")
    if src.extra_dims != dest.extra_dims:
        raise ArgumentError(_lib.PA_EINVAL, "incompatible extra dimensions of PencilArrays: "
                            f"{src.extra_dims} != {dest.extra_dims}")
    ex = dest.extra_dims
    flags = (_lib.PA_FFT_FORWARD if forward else _lib.PA_FFT_BACKWARD) | pairs[(real.dtype, cplx.dtype)]
    check(lib.pa_rfft(real.pencil._h, cplx.pencil._h, len(ex), i64arr(ex), flags,
                      C.c_void_p(src.data_ptr() or None), C.c_void_p(dest.data_ptr() or None),
                      _stream_ptr()))
    return dest


def rfft_(dest: PencilArray, src: PencilArray):
    """Real-to-complex 1-d FFT along the first memory dimension (not decomposed): ``dest =
    numpy.fft.rfft(src)`` there.  ``src``: float64 (float32) on a pencil of global size (..., N,
    ...); ``dest``: complex128 (complex64) on ``Pencil(src.pencil, size_global=(..., N//2+1,
    ...))``; float32 / complex64 run in single precision.  Step 1 of a
    PencilFFTs real-input plan; the two complex steps are ``transpose_(t, fft=...)``."""
    return _rfft(dest, src, True)


def brfft_(dest: PencilArray, src: PencilArray):
    """Inverse of :func:`rfft_`, unnormalised like FFTW's ``brfft``: ``dest = N *
    numpy.fft.irfft(src, n=N)``.  The imaginary parts of bins 0 and N/2 are ignored and
    ``src`` is left unmodified."""
    return _rfft(dest, src, False)


_R2R_KINDS = {"REDFT10": _lib.PA_REDFT10, "REDFT01": _lib.PA_REDFT01,
              "RODFT10": _lib.PA_RODFT10, "RODFT01": _lib.PA_RODFT01}


def _same_geometry(a: Pencil, b: Pencil) -> bool:
    return (a is b or (a.topology is b.topology and a.size_global == b.size_global
                       and a.decomp_dims == b.decomp_dims and a.perm == b.perm))


def r2r_(dest: PencilArray, src: PencilArray, kind: str):
    """Real-to-real 1-d transform along the first memory dimension (not decomposed), FFTW's
    unnormalised definitions: ``kind`` is ``"REDFT10"`` (DCT-II, ``scipy.fft.dct(x, 2)``),
    ``"REDFT01"`` (DCT-III), ``"RODFT10"`` (DST-II) or ``"RODFT01"`` (DST-III), and
    ``REDFT01(REDFT10(x)) = RODFT01(RODFT10(x)) = 2N x``.  ``src`` and ``dest``: float64, or
    float32 (single precision), with the same pencil geometry and extra dims; ``dest is src``
    transforms in place.  N is a power of two in 16..2048."""
    if kind not in _R2R_KINDS:
        raise ArgumentError(_lib.PA_EINVAL, f"kind must be one of {sorted(_R2R_KINDS)}: got {kind!r}")
    flags = {torch.float64: 0, torch.float32: _lib.PA_FFT_F32}
    if src.dtype != dest.dtype or src.dtype not in flags:
        raise ArgumentError(_lib.PA_EINVAL, "r2r_ takes two float64 or two float32 arrays: got "
                            f"{dest.dtype} and {src.dtype}")
    if not _same_geometry(src.pencil, dest.pencil):
        raise ArgumentError(_lib.PA_EINVAL, "r2r_: the arrays must have the same pencil geometry")
    if src.extra_dims != dest.extra_dims:
        raise ArgumentError(_lib.PA_EINVAL, "incompatible extra dimensions of PencilArrays: "
                            f"{src.extra_dims} != {dest.extra_dims}")
    ex = dest.extra_dims
    check(lib.pa_r2r(dest.pencil._h, len(ex), i64arr(ex), _R2R_KINDS[kind], flags[src.dtype],
                     C.c_void_p(src.data_ptr() or None), C.c_void_p(dest.data_ptr() or None),
                     _stream_ptr()))
    return dest


def transpose_host_(t: Transposition, host_src: torch.Tensor, host_dst: torch.Tensor):
    """``transpose!`` on HOST arrays through ``pa_transpose_host``: upload, kernels and
    download pipelined inside the library; returns when ``host_dst`` is valid.  Pin the
    tensors (``pin_memory()``) for full PCIe bandwidth."""
    _stream_ptr()
    n_in, n_out = t.plan.info.length_in * t.Ai.elsize, t.plan.info.length_out * t.Ao.elsize
    if host_src.numel() * host_src.element_size() != n_in or \
            host_dst.numel() * host_dst.element_size() != n_out or \
            host_src.is_cuda or host_dst.is_cuda or \
            not host_src.is_contiguous() or not host_dst.is_contiguous():
        raise _lib.DimensionMismatch(_lib.PA_EDIM, "host arrays must be dense CPU tensors of the "
                                     "local array sizes")
    check(lib.pa_transpose_host(t.plan.h, t.Pi.topology.comm.handle,
                                C.c_void_p(host_src.data_ptr() if n_in else None),
                                C.c_void_p(host_dst.data_ptr() if n_out else None), 0))
    return host_dst


class HostChain:
    """A sequence of transpositions applied to host arrays (``pa_host_chain_*``): what a
    PencilFFTs-style plan over ``Array``-backed pencils does around its transposes.

        chain = HostChain([t_xy, t_yz, t_zy, t_yx])
        k = chain.submit(hin, hout)      # asynchronous, double-buffered on the device
        chain.wait(k)                    # hout valid

    Only the pencils / methods of the transpositions are used; the device buffers belong
    to the chain (for one-sided methods their windows are registered here, collectively).
    """

    def __init__(self, transpositions):
        ts = list(transpositions)
        self.ts = ts
        n = len(ts)
        arr = (C.c_void_p * n)(*[t.plan.h.value for t in ts])
        comm = ts[0].Pi.topology.comm
        h = C.c_void_p()
        _stream_ptr()
        check(lib.pa_host_chain_create(n, arr, comm.handle, C.byref(h)))
        self.h = h
        for slot in range(4):
            probe = C.c_void_p()
            check(lib.pa_host_chain_buffer(h, slot, 0, C.byref(probe), None))
            if not probe.value:
                break  # the chain has fewer staging sets (tunable "host_slots")
            for i, t in enumerate(ts):
                info = t.plan.info
                if info.dim == 0 or info.nproc == 1 or comm.handle is None:
                    continue
                if info.method in (_lib.PA_PEER_PUT, _lib.PA_PEER_GET):
                    which = (1 - i % 2) if info.method == _lib.PA_PEER_PUT else (i % 2)
                    p = C.c_void_p()
                    check(lib.pa_host_chain_buffer(h, slot, which, C.byref(p), None))
                    _register_window_ptr(t.plan, p.value, comm)
                else:
                    _register_arenas(t.plan, t.Po, comm)

    def submit(self, host_src: torch.Tensor, host_dst: torch.Tensor) -> int:
        k = C.c_int64()
        check(lib.pa_host_chain_submit(self.h, C.c_void_p(host_src.data_ptr()),
                                       C.c_void_p(host_dst.data_ptr()), C.byref(k)))
        return k.value

    def wait(self, ticket: int = -1):
        check(lib.pa_host_chain_wait(self.h, ticket))

    def time_begin(self):
        check(lib.pa_host_chain_time_begin(self.h))

    def time_end(self) -> float:
        ms = C.c_float()
        check(lib.pa_host_chain_time_end(self.h, C.byref(ms)))
        return ms.value

    def __del__(self):
        try:
            lib.pa_host_chain_destroy(self.h)
        except Exception:
            pass
