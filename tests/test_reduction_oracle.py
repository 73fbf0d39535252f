"""CPU checks of tests/reduction_oracle.py: the layouts have the shape their names claim, and the fp64 restatements and
the block-effect helper agree with np.add.reduceat."""
import numpy as np
import pytest

import reduction_oracle as RO


@pytest.mark.parametrize("T", [8, 128, 256])
def test_layouts_are_what_they_claim(T):
    F = RO.SEG_FIN_T
    g = RO.layout("giant", T)
    ptr, nb = RO.seg_ptr(g), RO.n_blocks(g, T)
    assert nb[1] > 2 * F and ptr[1] % T != 0 and nb.max() == nb[1]

    a = RO.layout("aligned", T)
    ptr, nb = RO.seg_ptr(a), RO.n_blocks(a, T)
    assert ptr[1] % T == 0 and nb[1] == F + 1 and a[1] == (F + 1) * T
    assert ptr[3] % T == T - 1                                  # the third system ends one item before a boundary

    e = RO.layout("empties", T)
    ptr, nb = RO.seg_ptr(e), RO.n_blocks(e, T)
    assert e[0] == e[1] == 0 and e[-1] == 0 and e[-2] == 1 and e[-3] == 0
    zero = np.flatnonzero(e == 0)
    assert np.any(np.convolve(e == 0, np.ones(300), "valid") == 300)   # a run of 300 empties
    assert nb.max() > F and e[np.argmax(nb) - 1] == 0 and len(zero) >= 304

    m = RO.layout("many", T)
    assert len(m) > 65_535 and set(np.unique(m)) == {0, 1, 2, 3} and m[-1] == 0
    assert not RO.layout("none", T).any() and len(RO.layout("none", T)) == 3


def test_restatements_match_reduceat():
    rng = np.random.default_rng(0)
    counts = np.array([3, 1, 7, 2, 9])                          # reduceat cannot express empty segments
    t = rng.normal(size=(counts.sum(), 4))
    ptr = RO.seg_ptr(counts)
    ref = np.add.reduceat(t, ptr[:-1], axis=0)
    np.testing.assert_allclose(RO.seg_sum(t, counts), ref, rtol=1e-14, atol=1e-14)
    np.testing.assert_allclose(RO.seg_sum(t[:, 0], counts), ref[:, 0], rtol=1e-14, atol=1e-14)
    b = RO.bound(t, counts)
    assert b.shape == ref.shape
    np.testing.assert_allclose(b, 4 * (counts[:, None] + 20) * 2.0 ** -53 * np.add.reduceat(np.abs(t), ptr[:-1]))
    # empty systems sum to exact zeros
    c0 = np.array([0, 2, 0, 0, 3, 0])
    s = RO.seg_sum(rng.normal(size=(5, 2)), c0)
    assert (s[[0, 2, 3, 5]] == 0).all() and (s[[1, 4]] != 0).all()


def test_smallest_block_effect():
    T = 8
    counts = RO.layout("giant", T)
    rng = np.random.default_rng(1)
    t = rng.normal(size=(counts.sum(), 2))
    eff = RO.smallest_block_effect(counts, T, t)
    assert np.isinf(eff[[0, 2]]).all() and np.isfinite(eff[1]).all()
    a, b = RO.seg_ptr(counts)[1:3]
    cuts = np.r_[a, np.arange((a // T + 1) * T, b, T)]
    assert len(cuts) == RO.n_blocks(counts, T)[1]
    np.testing.assert_array_equal(eff[1], np.abs(np.add.reduceat(t[a:b], cuts - a)).min(0))
    # the bound of this data sees any one block dropped
    assert (eff[1] > 10 * RO.bound(t, counts)[1]).all()
