"""CPU: the neighbour-list oracle (oracle/nl_oracle.py) beyond the reference fixtures -- positions any number of cells
away, zero rows on non-periodic axes, and the exact coordination of perfect crystals (tests/nl_cases.py)."""
import numpy as np
import pytest

import nl_cases as C
from oracle import nl_oracle as NL


def _keys(ii, jj, ss):
    return {(i, j, *s) for i, j, s in zip(ii.tolist(), jj.tolist(), np.asarray(ss).tolist())}


@pytest.mark.parametrize("name", ["skewed", "thin_axis", "coarsened_3", "slab_zero", "wire_finite", "one_atom"])
def test_lattice_translation_maps_image_vectors(name):
    """Moving atom i by k_i lattice vectors maps every listed (i, j, S) to (i, j, S + k_i - k_j) and nothing else."""
    R, cell, pbc, rc = C.random_cases()[name]
    k = np.random.default_rng(3).integers(-20, 21, (R.shape[0], 3)) * pbc
    ii, jj, ss, off = NL.neighbor_list(R, cell, pbc, rc)
    assert ii.size > 0
    mi, mj, ms, _ = NL.neighbor_list(R + k @ cell, cell, pbc, rc)
    assert _keys(mi, mj, ms) == _keys(ii, jj, ss + k[ii] - k[jj])


@pytest.mark.parametrize("zero,finite", C.ZERO_FINITE_PAIRS)
def test_zero_non_periodic_rows_give_the_same_list(zero, finite):
    cases = C.random_cases()
    a, b = NL.neighbor_list(*cases[zero]), NL.neighbor_list(*cases[finite])
    assert a[0].size > 0
    for x, y in zip(a[:3], b[:3]):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("variant", C.VARIANTS)
@pytest.mark.parametrize("name", list(C.CRYSTALS))
def test_crystal_coordination(name, variant):
    """Every atom has exactly K neighbours at the shell radii, in fp64 and for the fp32-rounded crystal (no band)."""
    R, cell, pbc, rc = C.crystal(name, variant)
    K = C.coordination(name)
    ii, jj, ss, off = NL.neighbor_list(R, cell, pbc, rc)
    assert np.array_equal(np.bincount(ii, minlength=R.shape[0]), np.full(R.shape[0], K))
    d = np.linalg.norm(R[jj] - R[ii] + off, axis=1)
    assert np.abs(d[:, None] - C.shell_radii(name)[None]).min(axis=1).max() < 1e-9
    definite, band = NL.band_neighbor_list(R.astype(np.float32), cell.astype(np.float32), pbc, rc)
    assert not band and definite == _keys(ii, jj, ss)


def test_band_separates_pairs_at_the_cutoff():
    """A pair at exactly the cutoff lands in the band, pairs 1e-3 inside and outside do not."""
    cell = np.eye(3, dtype=np.float32) * 20
    R = np.array([[1, 1, 1], [5, 1, 1], [1, 4.999, 1], [1, 1, 5.001]], dtype=np.float32)
    definite, band = NL.band_neighbor_list(R, cell, np.ones(3, bool), 4.0)
    assert band == {(0, 1, 0, 0, 0), (1, 0, 0, 0, 0)}
    assert definite == {(0, 2, 0, 0, 0), (2, 0, 0, 0, 0)}
