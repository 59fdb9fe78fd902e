#!/usr/bin/env python
"""NVLink bandwidth of the box-copy kernels with one side in PEER memory.

One process, two GPUs (peer access enabled by torch): the same `pa_box_copy`
kernels the PeerPut / PeerGet paths launch, with src or dst on the other GPU,
timed with CUDA events -- against `cudaMemcpyPeerAsync` (torch `copy_`) as the
yardstick.  Needs >= 2 GPUs:  python profiles/nvlink_microbench.py
"""
import ctypes as C
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pencilarrays_b200 as pa  # noqa: E402
from pencilarrays_b200._lib import lib, check, i64arr, BlockDesc  # noqa: E402

N = 1 << 30  # bytes per transfer


def launch(ext, ss, ds, es, src, dst, dev):
    with torch.cuda.device(dev):
        check(lib.pa_set_device(dev))
        st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        d = BlockDesc()
        check(lib.pa_box_copy(len(ext), i64arr(ext), i64arr(ss), i64arr(ds), es,
                              C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr()), st, C.byref(d)))
        return d.kernel_class


def timeit(fns, devs, reps=10):
    for f in fns:
        f()
    for d in devs:
        torch.cuda.synchronize(d)
    evs = []
    for d in devs:
        with torch.cuda.device(d):
            evs.append((torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
    for (a, _), d in zip(evs, devs):
        with torch.cuda.device(d):
            a.record()
    for _ in range(reps):
        for f in fns:
            f()
    for (_, b), d in zip(evs, devs):
        with torch.cuda.device(d):
            b.record()
    for d in devs:
        torch.cuda.synchronize(d)
    return max(a.elapsed_time(b) for a, b in evs) / reps


def main():
    assert torch.cuda.device_count() >= 2
    a0 = torch.empty(N, dtype=torch.uint8, device="cuda:0").random_()
    b0 = torch.empty(N, dtype=torch.uint8, device="cuda:0")
    a1 = torch.empty(N, dtype=torch.uint8, device="cuda:1").random_()
    b1 = torch.empty(N, dtype=torch.uint8, device="cuda:1")
    b1.copy_(a0)
    b0.copy_(a1)  # enables peer access both ways
    torch.cuda.synchronize(0)
    torch.cuda.synchronize(1)
    rows = []

    def rec(name, ms, nbytes=N):
        rows.append((name, ms, nbytes / ms / 1e6))
        print(f"{name:64s} {ms:8.3f} ms  {nbytes/ms/1e6:8.1f} GB/s", flush=True)

    def memcpy01():
        with torch.cuda.device(0):
            b1.copy_(a0, non_blocking=True)

    def memcpy10():
        with torch.cuda.device(1):
            b0.copy_(a1, non_blocking=True)

    rec("cudaMemcpyPeer 0->1", timeit([memcpy01], [0]))
    rec("cudaMemcpyPeer both directions (per direction)", timeit([memcpy01, memcpy10], [0, 1]))
    nel = N // 16
    rec("k_rows local 0->0 (sanity)", timeit([lambda: launch([nel], [1], [1], 16, a0, b0, 0)], [0]))
    rec("k_rows PUT contiguous (src local, dst peer)", timeit([lambda: launch([nel], [1], [1], 16, a0, b1, 0)], [0]))
    rec("k_rows GET contiguous (src peer, dst local)", timeit([lambda: launch([nel], [1], [1], 16, a1, b0, 0)], [0]))
    rec("k_rows PUT both directions", timeit([lambda: launch([nel], [1], [1], 16, a0, b1, 0),
                                            lambda: launch([nel], [1], [1], 16, a1, b0, 1)], [0, 1]))
    rec("k_rows GET both directions", timeit([lambda: launch([nel], [1], [1], 16, a1, b0, 0),
                                            lambda: launch([nel], [1], [1], 16, a0, b1, 1)], [0, 1]))
    # pack-like: 4 KiB runs out of 16 KiB rows (cfg4 x->y pack shape) into a contiguous peer buffer
    big0 = torch.empty(4 * N, dtype=torch.uint8, device="cuda:0")
    big1 = torch.empty(4 * N, dtype=torch.uint8, device="cuda:1")
    e, s_, d_ = [256, 256 * 1024], [1, 1024], [1, 256]
    rec("k_rows PUT 4KiB runs (strided src local -> dense peer)", timeit([lambda: launch(e, s_, d_, 16, big0, b1, 0)], [0]))
    rec("k_rows GET 4KiB runs (strided src peer -> dense local)", timeit([lambda: launch(e, s_, d_, 16, big1, b0, 0)], [0]))
    # transposes (2,1,3): (256,256,1024) c128 -> (256,256,1024) with dims 0,1 swapped
    e, s_, d_ = [256, 256, 1024], [1, 256, 65536], [256, 1, 65536]
    rec("k_transpose_vec<16> local (sanity)", timeit([lambda: launch(e, s_, d_, 16, a0, b0, 0)], [0]))
    rec("k_transpose_vec<16> PUT (dst peer, 512 B runs)", timeit([lambda: launch(e, s_, d_, 16, a0, b1, 0)], [0]))
    rec("k_transpose_vec<16> GET (src peer, 512 B runs)", timeit([lambda: launch(e, s_, d_, 16, a1, b0, 0)], [0]))
    rec("k_transpose_vec<16> PUT both directions", timeit([lambda: launch(e, s_, d_, 16, a0, b1, 0),
                                                          lambda: launch(e, s_, d_, 16, a1, b0, 1)], [0, 1]))
    rec("k_transpose_vec<16> GET both directions", timeit([lambda: launch(e, s_, d_, 16, a1, b0, 0),
                                                          lambda: launch(e, s_, d_, 16, a0, b1, 1)], [0, 1]))
    # ---- grid cap sweep: how many CTAs does an NVLink-bound kernel need? ----
    def cap(n):
        check(lib.pa_set_tunable(b"box_copy_ctas", n))

    for c in (33, 66, 132, 264, 528, 1056, 0):  # multiples of the 132 SMs
        cap(c)
        rec(f"k_transpose_vec<16> PUT grid cap {c}", timeit([lambda: launch(e, s_, d_, 16, a0, b1, 0)], [0]))
        rec(f"k_transpose_vec<16> GET grid cap {c}", timeit([lambda: launch(e, s_, d_, 16, a1, b0, 0)], [0]))
        rec(f"k_rows PUT contiguous grid cap {c}", timeit([lambda: launch([nel], [1], [1], 16, a0, b1, 0)], [0]))
    cap(0)
    # ---- remote kernel (high-priority stream, capped) beside a local transpose (low priority) ----
    import time
    hi = torch.cuda.Stream(device=0, priority=-1)
    lo = torch.cuda.Stream(device=0, priority=0)
    c0 = torch.empty(N, dtype=torch.uint8, device="cuda:0")
    for c in (0, 132, 264, 528):
        def both():
            with torch.cuda.stream(lo):
                cap(0)
                launch(e, s_, d_, 16, a0, c0, 0)     # local K3-like transpose: 2 GiB of HBM traffic
            with torch.cuda.stream(hi):
                cap(c)
                launch(e, s_, d_, 16, a0, b1, 0)     # put of 1 GiB
        both()
        torch.cuda.synchronize(0)
        t0 = time.perf_counter()
        for _ in range(10):
            both()
            torch.cuda.synchronize(0)
        ms = (time.perf_counter() - t0) * 100
        rec(f"local transpose (lo prio) || PUT (hi prio, cap {c}) wall", ms)
    cap(0)
    # ---- TMA bulk-copy pipeline (k_rows_bulk, tunable bulk_rows) ----
    check(lib.pa_set_tunable(b"bulk_rows", 1))
    e4, s4, d4 = [256, 256 * 1024], [1, 1024], [1, 256]
    for c in (132, 264, 396, 528, 792):
        cap(c)
        rec(f"k_rows_bulk local contiguous, {c} CTAs", timeit([lambda: launch([nel], [1], [1], 16, a0, b0, 0)], [0]))
        rec(f"k_rows_bulk PUT contiguous, {c} CTAs", timeit([lambda: launch([nel], [1], [1], 16, a0, b1, 0)], [0]))
        rec(f"k_rows_bulk GET contiguous, {c} CTAs", timeit([lambda: launch([nel], [1], [1], 16, a1, b0, 0)], [0]))
        rec(f"k_rows_bulk PUT 4KiB runs, {c} CTAs", timeit([lambda: launch(e4, s4, d4, 16, big0, b1, 0)], [0]))
        rec(f"k_rows_bulk PUT both directions, {c} CTAs",
            timeit([lambda: launch([nel], [1], [1], 16, a0, b1, 0), lambda: launch([nel], [1], [1], 16, a1, b0, 1)], [0, 1]))
    cap(0)
    check(lib.pa_set_tunable(b"bulk_rows", 0))
    # f32 transposes (cfg5-like)
    e, s_, d_ = [512, 512, 1024], [1, 512, 262144], [512, 1, 262144]
    rec("k_transpose_vec<4> PUT", timeit([lambda: launch(e, s_, d_, 4, a0, b1, 0)], [0]))
    rec("k_transpose_vec<4> GET", timeit([lambda: launch(e, s_, d_, 4, a1, b0, 0)], [0]))


if __name__ == "__main__":
    main()
