#!/usr/bin/env python
"""Tile-shape / tile-order sweep of the fused permute kernel (K3) over the shapes
bench.py reports: BASELINE configs[1] (256^3 Float64), the 512^3 ComplexF64 chain
and the r2c-shaped (odd leading extent) grids.  One GPU, CUDA events around
back-to-back launches over rotating buffers (everything >> L2).

  python profiles/prof_shapes.py [--json out.json]
"""
import argparse
import itertools
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pencilarrays_b200 as pa  # noqa: E402

PEAK = 3350.0  # H100 SXM data-sheet HBM3 bandwidth (GB/s) unless MEASURED_PEAKS.json says otherwise
try:
    PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass

SHAPES = [
    ("256^3 f64", (256, 256, 256), torch.float64, 8, 6),
    ("512^3 c128", (512, 512, 512), torch.complex128, 16, 1),
    ("(513,512,512) c64", (513, 512, 512), torch.complex64, 8, 1),
    ("(1025,512,256) f32", (1025, 512, 256), torch.float32, 4, 2),
    ("(1025,511,129) f64", (1025, 511, 129), torch.float64, 8, 2),
]
PERMS = [((2, 1, 3), (3, 2, 1)), ((2, 3, 1), (3, 1, 2))]


def timed(fn, reps=4):
    for _ in range(2):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    rows = []
    for (name, dims, dt, es, nrot), (py_, pz_) in itertools.product(SHAPES, PERMS):
        px = pa.Pencil(topo, dims, (2, 3))
        py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(*py_))
        pz = pa.Pencil(py, decomp_dims=(1, 2), permute=pa.Permutation(*pz_))
        sets = []
        for _ in range(nrot):
            ux, uy, uz = (pa.PencilArray.undef(dt, p) for p in (px, py, pz))
            ux.data.view(torch.uint8).random_()
            uy.data.view(torch.uint8).random_()
            sets.append((ux, uy, uz))
        legs = {"x->y": [pa.Transposition(s[1], s[0]) for s in sets],
                "y->z": [pa.Transposition(s[2], s[1]) for s in sets],
                "z->y": [pa.Transposition(s[1], s[2]) for s in sets],
                "y->x": [pa.Transposition(s[0], s[1]) for s in sets]}
        nb = 2 * sets[0][0].data.numel() * es
        for leg, ts in legs.items():
            best = None
            combos = [(16, 0), (16, 1), (32, 0), (32, 1), (0, -1)]  # last: the library's own choice
            for tbq, yf in combos:
                if es == 4 and tbq == 32:
                    continue
                pa.set_tunable("transpose_tbq", tbq)
                pa.set_tunable("transpose_y_fastest", yf)

                def run():
                    for t in ts:
                        pa.transpose_(t)
                ms = timed(run) / len(ts)
                r = dict(shape=name, perms=f"{py_}->{pz_}", leg=leg, tbq=tbq, y_fastest=yf,
                         ms=round(ms, 4), GBps=round(nb / ms / 1e6, 1), frac=round(nb / ms / 1e6 / PEAK, 3))
                rows.append(r)
                if best is None or r["GBps"] > best["GBps"]:
                    best = r
            print(f"{name:20s} {py_}->{pz_} {leg}: " + "  ".join(
                ("auto" if r['y_fastest'] < 0 else f"tbq{r['tbq']}/yf{r['y_fastest']}") + f"={r['frac']:.3f}"
                for r in rows[-(3 if es == 4 else 5):]),
                flush=True)
        pa.set_tunable("transpose_tbq", 0)
        pa.set_tunable("transpose_y_fastest", -1)
        del sets, legs
        torch.cuda.empty_cache()
    if args.json:
        json.dump(rows, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
