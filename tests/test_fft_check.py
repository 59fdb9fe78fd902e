"""`pa_plan_fft_check` (CPU): whether `transpose_(t, fft=...)` can fuse the FFT into the unpack.

pa_transpose asks this before it enqueues anything, so the answer must be the same on every
rank of a grid line: if one rank refused while its peers went ahead with the exchange, the
peers would wait on flags that never come.  Every configuration of the suite (and a seeded set
of power-of-two ones, where the answer is often "yes") is planned for every emulated rank, with
16-byte elements, and the ranks of each line must agree."""
import math
import random

import pytest

import pencilarrays_b200 as pa
from pencilarrays_b200._lib import lib
from pencilarrays_b200.transpositions import _Plan
from util import CASES, build_chain
from test_random_configs import RANDOM_CASES


def pow2_case(rng: random.Random, idx: int):
    """Grids of up to 8 ranks per line, line lengths around the kernel's limits."""
    N = rng.choice([3, 3, 4])
    M = rng.randint(1, 2)
    grid = tuple(rng.choice([1, 2, 3, 5, 6, 8, 9]) for _ in range(M))
    while math.prod(grid) > 24:
        grid = tuple(max(1, g // 2) for g in grid)
    dims = tuple(rng.choice([2, 3, 8, 16, 48, 64, 1024, 2048]) for _ in range(N))
    extra = tuple(rng.choice([2, 3]) for _ in range(rng.choice([0, 1])))
    perms = [None, (2, 1, 3), (3, 2, 1), (2, 3, 1), (3, 1, 2), (1, 3, 2)] if N == 3 else \
        [None, (2, 1, 3, 4), (4, 3, 2, 1), (3, 4, 1, 2)]
    decomp = tuple(rng.sample(range(1, N + 1), M))
    chain = [(decomp, rng.choice(perms))]
    for _ in range(2):
        d = list(chain[-1][0])
        i = rng.randrange(M)
        free = [x for x in range(1, N + 1) if x not in d]
        if free:
            d[i] = rng.choice(free)
        chain.append((tuple(d), rng.choice(perms)))
    return dict(name=f"pow2_{idx}", grid=grid, dims=dims, extra=extra, it=16, chain=chain)


RNG = random.Random(20261015)
POW2_CASES = [pow2_case(RNG, i) for i in range(40)]
ALL = CASES + RANDOM_CASES + POW2_CASES


def answers(case):
    """Per step: [(world ranks of the line, {world rank: status})]."""
    ranks, steps = build_chain(case)
    out = []
    for k in range(1, len(steps)):
        per_rank, lines = {}, {}
        for r in range(len(ranks)):
            plan = _Plan(steps[k - 1][r][0], steps[k][r][0], case["extra"], 16, pa.PointToPoint())
            per_rank[r] = lib.pa_plan_fft_check(plan.h)
            info = plan.info
            line = tuple(sorted(plan.peer(n).world_rank for n in range(1, info.nproc + 1))) \
                if info.dim else (r,)
            lines.setdefault(line, set()).add(r)
        out.append((per_rank, lines))
    return out


@pytest.mark.parametrize("case", ALL, ids=[c["name"] for c in ALL])
def test_fft_check_is_uniform_over_each_grid_line(case):
    for k, (per_rank, lines) in enumerate(answers(case), start=1):
        for line, members in lines.items():
            assert members == set(line), (case["name"], k, line, members)
            got = {per_rank[r] for r in line}
            assert len(got) == 1, (case["name"], k, {r: per_rank[r] for r in line})
            assert got <= {pa._lib.PA_OK, pa._lib.PA_EINVAL}


def test_fft_check_agrees_with_the_fused_transposes_the_suite_runs():
    """The multi-rank fused transposes of the suite: c128_pow2_* are accepted on every step,
    c128_fft_perms (lines of 12 and 10 points) refused on every rank."""
    by_name = {c["name"]: c for c in CASES}
    for name in ("c128_pow2_2x2", "c128_pow2_2x1"):
        for per_rank, _ in answers(by_name[name]):
            assert set(per_rank.values()) == {pa._lib.PA_OK}, name
    for per_rank, _ in answers(by_name["c128_fft_perms"]):
        assert set(per_rank.values()) == {pa._lib.PA_EINVAL}
    # the seeded power-of-two set exercises both answers
    seen = {s for c in POW2_CASES for per_rank, _ in answers(c) for s in per_rank.values()}
    assert seen == {pa._lib.PA_OK, pa._lib.PA_EINVAL}


def line_plans(nproc, L, other=(4, 3), extra=()):
    """x-pencil decomposed along x over `nproc` ranks -> y-pencil with x local and contiguous:
    the fused unpack gathers the x lines of L points from `nproc` blocks."""
    out = []
    for r in range(nproc):
        topo = pa.MPITopology(pa.Comm(r, nproc), (nproc,))
        pa_ = pa.Pencil(topo, (L,) + other, (1,), permute=pa.Permutation(2, 1, 3))
        pb = pa.Pencil(pa_, decomp_dims=(2,), permute=pa.NoPermutation())
        out.append(_Plan(pa_, pb, extra, 16, pa.PointToPoint()))
    return out


@pytest.mark.parametrize("nproc,L,ok,why", [
    (3, 64, True, None), (5, 8, True, None), (6, 1024, True, None), (8, 8, True, None),
    (3, 48, False, "power of two"), (1, 2048, False, "power of two"), (2, 2048, False, "power of two"),
    (9, 16, False, "more than 8 blocks"),
])
def test_fft_check_verdicts_and_reasons(nproc, L, ok, why):
    plans = line_plans(nproc, L, other=(nproc + 1, 3))
    for p in plans:
        st = lib.pa_plan_fft_check(p.h)
        assert st == (pa._lib.PA_OK if ok else pa._lib.PA_EINVAL), (nproc, L)
        if why:
            assert why in lib.pa_last_error().decode()
        # cached: the same answer (and reason) again
        assert lib.pa_plan_fft_check(p.h) == st


def test_fft_check_refuses_other_element_sizes_and_null():
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px = pa.Pencil(topo, (16, 8, 4), (2, 3))
    py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    assert lib.pa_plan_fft_check(_Plan(px, py, (), 16, pa.PointToPoint()).h) == pa._lib.PA_OK  # 8-point y lines
    assert lib.pa_plan_fft_check(_Plan(px, py, (), 8, pa.PointToPoint()).h) == pa._lib.PA_EINVAL
    assert "16-byte" in lib.pa_last_error().decode()
    assert lib.pa_plan_fft_check(None) == pa._lib.PA_EINVAL
