"""The warp-wide lower bound of the edge kernels (csrc/common.cuh: spk_lower_bound_warp) restated lane by lane in numpy and
checked against numpy.searchsorted: the kernels split the CSR rows of a CTA's four groups with it (edge-balanced ranges), so
an off-by-one would drop or duplicate receiver rows.  The CUDA function itself is exercised by every edge-kernel test on the
GPU; this test pins the ALGORITHM (probe positions, narrowing, final round) including the cases the GPU tests rarely hit:
targets below the first / above the last entry, runs of equal row pointers (edge-free rows), n <= 32, n not a multiple of 33."""
import numpy as np
import pytest


def lower_bound_warp(ptr: np.ndarray, n: int, target: int) -> int:
    """first r in [0, n] with ptr[r] >= target (ptr[n] is never read), 32 lanes per round"""
    lanes = np.arange(32)
    lo, hi = 0, n
    rounds = 0
    while hi - lo > 32:
        span = hi - lo
        p = lo + ((lanes + 1) * span) // 33
        assert np.all(np.diff(p) > 0) and p[0] > lo and p[-1] < hi          # strictly increasing, inside (lo, hi)
        ge = ptr[p] >= target
        f = int(np.argmax(ge)) if ge.any() else 32
        new_hi = hi if f == 32 else lo + ((f + 1) * span) // 33
        if f > 0:
            lo = lo + (f * span) // 33 + 1
        hi = new_hi
        rounds += 1
        assert rounds < 8
    p = lo + lanes
    ge = np.where(p < hi, ptr[np.minimum(p, max(n - 1, 0))] >= target, True)
    f = int(np.argmax(ge)) if ge.any() else 32
    return min(lo + f, hi)


def serial(ptr, n, target):
    lo, hi = 0, n
    while lo < hi:
        mid = (lo + hi) >> 1
        if ptr[mid] < target:
            lo = mid + 1
        else:
            hi = mid
    return lo


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 34, 65, 1000, 5376, 8192, 35937, 262144])
def test_warp_lower_bound_matches_searchsorted(n):
    rng = np.random.default_rng(n)
    for trial in range(6):
        deg = rng.integers(0, 4 if trial % 2 else 60, size=n)
        if trial == 2:
            deg[rng.random(n) < 0.7] = 0                                       # long runs of edge-free rows
        ptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
        E = int(ptr[-1])
        targets = list(rng.integers(-3, E + 4, size=40)) + [0, E, E + 1, -1]
        nb = 528                                                                # 132 CTAs x 4 groups
        targets += [(E * b) // nb for b in range(0, nb + 1, 37)]
        for t in targets:
            want = min(int(np.searchsorted(ptr[:n], t, side="left")), n)
            assert serial(ptr, n, int(t)) == want
            assert lower_bound_warp(ptr, n, int(t)) == want, (n, trial, t)


def test_group_ranges_cover_every_row_once():
    """the four group ranges of all 132 CTAs tile [0, n) without gaps or overlap (what the kernels rely on)"""
    rng = np.random.default_rng(5)
    n = 5376
    ptr = np.concatenate([[0], np.cumsum(rng.integers(0, 30, size=n))]).astype(np.int64)
    E, nb = int(ptr[-1]), 132 * 4
    b = [0 if k <= 0 else (n if k >= nb else lower_bound_warp(ptr, n, (E * k) // nb)) for k in range(nb + 1)]
    assert b[0] == 0 and b[-1] == n and all(x <= y for x, y in zip(b, b[1:]))
