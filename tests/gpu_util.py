"""GPU-side helpers for the `-m gpu` parity tests (all calls go through the C ABI)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200._lib import lib, check, BlockDesc, i64arr

TORCH_OF = {1: torch.uint8, 2: torch.int16, 4: torch.float32, 8: torch.float64,
            16: torch.complex128}


def dev_bytes(a: np.ndarray) -> torch.Tensor:
    """Upload a NumPy array as raw bytes (bit patterns preserved, NaNs included)."""
    raw = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    return torch.from_numpy(raw.copy()).cuda()


def host_bytes(t: torch.Tensor) -> np.ndarray:
    return t.contiguous().view(torch.uint8).reshape(-1).cpu().numpy()


def stream_ptr():
    check(lib.pa_set_device(torch.cuda.current_device()))
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t: torch.Tensor, byte_offset: int = 0):
    return C.c_void_p(t.data_ptr() + byte_offset)


# ---- ordering checks: hold a stream, then produce the input behind the hold --------------
HOLD_MS = 50.0
_hold_cycles = None


def hold_cycles() -> int:
    """Cycles of `torch.cuda._sleep` that spin for about HOLD_MS, calibrated once with CUDA
    events (the SM clock is not assumed); never more than 1e8 (0.1 s at 1 GHz)."""
    global _hold_cycles
    if _hold_cycles is None:
        torch.cuda._sleep(1000)  # (the first launch loads the kernel)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 1 << 22
        a.record()
        torch.cuda._sleep(n)
        b.record()
        b.synchronize()
        ms = max(a.elapsed_time(b), 1e-3)
        _hold_cycles = min(int(n * HOLD_MS / ms), 100_000_000)
    return _hold_cycles


def timing_event() -> torch.cuda.Event:
    """A timing event recorded on the current stream."""
    ev = torch.cuda.Event(enable_timing=True)
    ev.record()
    return ev


def hold() -> torch.cuda.Event:
    """One bounded spin (about HOLD_MS) on the current stream; returns the event `held`,
    recorded right after it.  Work enqueued on this stream afterwards runs only once the spin
    is over, so a library call that is not ordered behind the caller's stream reads whatever
    the input held before, and `held.query()` is still False when a call that does not
    synchronise the host returns."""
    torch.cuda._sleep(hold_cycles())
    return timing_event()


def box_copy(extent, sstr, dstr, elsize, src: torch.Tensor, dst: torch.Tensor, src_off=0,
             dst_off=0):
    d = BlockDesc()
    check(lib.pa_box_copy(len(extent), i64arr(extent), i64arr(sstr), i64arr(dstr), elsize,
                          ptr(src, src_off * elsize), ptr(dst, dst_off * elsize), stream_ptr(),
                          C.byref(d)))
    return d


def np_box_copy(extent, sstr, dstr, elsize, src: np.ndarray, dst: np.ndarray, src_off=0, dst_off=0):
    """NumPy evaluation of the same strided copy on raw bytes (uint8 arrays)."""
    if any(e == 0 for e in extent):
        return
    dt = np.dtype((np.void, elsize))
    s = src.view(dt)
    d = dst.view(dt)
    sv = np.lib.stride_tricks.as_strided(s[src_off:], shape=extent,
                                         strides=[x * elsize for x in sstr], writeable=False)
    dv = np.lib.stride_tricks.as_strided(d[dst_off:], shape=extent,
                                         strides=[x * elsize for x in dstr])
    dv[...] = sv


def emulate_transpose_gpu(plans, srcs, dsts, fused_self=False):
    """pack -> (device-to-device) exchange -> unpack for all emulated ranks on
    ONE GPU, using pa_pack / pa_unpack / pa_copy_self.  srcs/dsts: uint8 tensors.
    Returns (send_bufs, recv_bufs) as uint8 tensors."""
    n = len(plans)
    sends = [torch.zeros(max(1, p.info.send_bytes), dtype=torch.uint8, device="cuda") for p in plans]
    recvs = [torch.zeros(max(1, p.info.recv_bytes), dtype=torch.uint8, device="cuda") for p in plans]
    st = stream_ptr()
    if plans[0].info.dim == 0:
        for r in range(n):
            check(lib.pa_permute_local(plans[r].h, ptr(srcs[r]), ptr(dsts[r]), None, st))
        return sends, recvs
    nproc = plans[0].info.nproc
    for r in range(n):
        for p in range(1, nproc + 1):
            peer = plans[r].peer(p)
            if peer.is_self and fused_self:
                continue
            check(lib.pa_pack(plans[r].h, p, ptr(srcs[r]),
                              ptr(recvs[r] if peer.is_self else sends[r]), st))
    for r in range(n):
        me = plans[r].peer(plans[r].info.self_index).world_rank
        for p in range(1, nproc + 1):
            peer = plans[r].peer(p)
            if peer.is_self:
                continue
            q = peer.world_rank
            back = [plans[q].peer(pp) for pp in range(1, nproc + 1)]
            back = [b for b in back if b.world_rank == me][0]
            assert back.recv_count == peer.send_count
            recvs[q][back.recv_offset:back.recv_offset + back.recv_count] = \
                sends[r][peer.send_offset:peer.send_offset + peer.send_count]
    for r in range(n):
        for p in range(1, nproc + 1):
            peer = plans[r].peer(p)
            if peer.is_self and fused_self:
                check(lib.pa_copy_self(plans[r].h, ptr(srcs[r]), ptr(dsts[r]), st))
            else:
                check(lib.pa_unpack(plans[r].h, p, ptr(recvs[r]), ptr(dsts[r]), st))
    return sends, recvs
