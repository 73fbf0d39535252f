"""GPU neighbour list (csrc/neighbors.cu) on the cells where a linked-cell search goes wrong: perfect crystals whose
coordination is exact, cells thinner than the cutoff and heavily skewed, atoms on bin boundaries and just below
fractional 0, positions many cells away, coarsened grids, bins of more than 32 atoms, and sheets and wires whose
non-periodic cell rows are zero (tests/nl_cases.py).  Pair sets are judged against the fp64 oracle with its fp32 band
(oracle/nl_oracle.band_neighbor_list); order, padding and batching are checked bit for bit."""
import numpy as np
import pytest
import torch

import nl_cases as C
from oracle import nl_oracle as NL

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _f32(case):
    R, cell, pbc, rc = case
    return np.asarray(R, np.float32).reshape(-1, 3), np.asarray(cell, np.float32), np.asarray(pbc, bool), rc


def _call(systems, cutoff, capacity=None, pad=False):
    """One device call on the collated fp32 systems [(R, cell, pbc)] -> numpy idx_i, idx_j, offsets, shifts, n_pairs."""
    from schnetpack_b200.neighbors import neighbor_list

    R = np.concatenate([s[0] for s in systems]).astype(np.float32).reshape(-1, 3)
    cells = np.stack([s[1] for s in systems]).astype(np.float32)
    pbcs = np.stack([s[2] for s in systems])
    n_atoms = [s[0].shape[0] for s in systems]
    out = neighbor_list(torch.as_tensor(R, device=DEV), torch.as_tensor(cells, device=DEV),
                        torch.as_tensor(pbcs, device=DEV), torch.as_tensor(n_atoms, device=DEV), cutoff,
                        capacity=capacity, pad=pad, return_shifts=True)
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in out)


def _keys(ii, jj, sh):
    return [(i, j, *s) for i, j, s in zip(ii.tolist(), jj.tolist(), sh.tolist())]


def _check_list(case, out):
    """Flag clear, rows sorted, no duplicates, (i, j, S) <=> (j, i, -S); returns the set of (i, j, Sx, Sy, Sz)."""
    ii, jj, off, sh, n_pairs = out
    assert n_pairs[1] == 0 and n_pairs[0] == ii.shape[0]
    assert (np.diff(ii) >= 0).all()
    keys = _keys(ii, jj, sh)
    got = set(keys)
    assert len(got) == len(keys), "duplicate entries"
    assert got == {(j, i, -a, -b, -c) for i, j, a, b, c in got}
    assert not (~case[2][None, :] & (sh != 0)).any(), "image shift on a non-periodic axis"
    return got


@pytest.mark.parametrize("variant", C.VARIANTS)
@pytest.mark.parametrize("name", list(C.CRYSTALS))
def test_crystal_coordination_is_exact(name, variant):
    """Every atom has exactly K neighbours, each at a shell radius; the cutoff lies between shells, so there is no band."""
    R, cell, pbc, rc = case = _f32(C.crystal(name, variant))
    out = _call([case], rc)
    got = _check_list(case, out)
    ii, jj, _, sh, _ = out
    assert np.array_equal(np.bincount(ii, minlength=R.shape[0]), np.full(R.shape[0], C.coordination(name)))
    R64, cell64 = R.astype(np.float64), cell.astype(np.float64)
    d = np.linalg.norm(R64[jj] - R64[ii] + sh @ cell64, axis=1)
    delta = NL.band_width(R64, cell64, ii, jj, sh, rc)
    assert (np.abs(d[:, None] - C.shell_radii(name)[None]).min(axis=1) <= delta).all()
    definite, band = NL.band_neighbor_list(R, cell, pbc, rc)
    assert not band and got == definite


@pytest.mark.parametrize("name", list(C.random_cases()))
def test_random_structures_against_the_fp64_band(name):
    """Every definite pair is listed and nothing outside the band is; the band stays a small fraction of the list."""
    case = _f32(C.random_cases()[name])
    got = _check_list(case, _call([case], case[3]))
    definite, band = NL.band_neighbor_list(*case)
    assert definite and len(band) <= 0.01 * len(definite), (len(definite), len(band))
    assert not definite - got, sorted(definite - got)[:8]
    assert not got - definite - band, sorted(got - definite - band)[:8]


@pytest.mark.parametrize("zero,finite", C.ZERO_FINITE_PAIRS)
def test_zero_and_finite_non_periodic_rows_give_identical_lists(zero, finite):
    """Binning depends on the periodic rows only: same pairs, same order, same offsets."""
    cases = C.random_cases()
    a = _call([_f32(cases[zero])], cases[zero][3])
    b = _call([_f32(cases[finite])], cases[finite][3])
    assert a[0].shape[0] > 0
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def _batch_systems():
    """Every structure above once, with empty systems between them."""
    empty = (np.zeros((0, 3), np.float32), np.eye(3, dtype=np.float32) * 10, np.ones(3, bool))
    systems = [empty]
    for case in list(C.random_cases().values()) + [C.crystal(n, "primitive") for n in C.CRYSTALS] + \
            [C.crystal("fcc", "shifted"), C.crystal("graphene", "rotated")]:
        systems += [_f32(case)[:3]] + ([empty] if len(systems) % 3 == 0 else [])
    return systems + [empty]


def test_collated_batch_equals_per_system_calls_bit_for_bit():
    rc = 5.0
    systems = _batch_systems()
    whole = _call(systems, rc)
    assert whole[4][1] == 0
    parts, start = [[], [], [], []], 0
    for s in systems:
        ii, jj, off, sh, _ = _call([s], rc)
        for p, x in zip(parts, (ii + start, jj + start, off, sh)):
            p.append(x)
        start += s[0].shape[0]
    for p, x in zip(parts, whole[:4]):
        y = np.concatenate(p)
        assert x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8))
    again = _call(systems, rc)
    for x, y in zip(whole, again):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))


def test_fixed_capacity_padding_overflow_and_count_only():
    rc = 5.0
    cases = C.random_cases()
    systems = [_f32(cases[n])[:3] for n in ("skewed", "coarsened_3", "one_atom", "slab_zero", "wire_zero")]
    N = sum(s[0].shape[0] for s in systems)
    ii, jj, off, sh, n_pairs = _call(systems, rc)
    T = ii.shape[0]
    assert n_pairs.tolist() == [T, 0] and T > 0
    # pads: row i is followed by floor((i+1)P/N) - floor(iP/N) self pairs (i, i, (2rc, 0, 0), S = 0)
    P = 37
    pads = (np.arange(1, N + 1) * P) // N - (np.arange(N) * P) // N
    rows = np.searchsorted(ii, np.arange(N + 1))
    want = [[], [], [], []]
    for i in range(N):
        a, b = rows[i], rows[i + 1]
        for w, x in zip(want, (ii[a:b], jj[a:b], off[a:b], sh[a:b])):
            w.append(x)
        k = pads[i]
        want[0].append(np.full(k, i, np.int64))
        want[1].append(np.full(k, i, np.int64))
        want[2].append(np.tile(np.array([2 * rc, 0, 0], np.float32), (k, 1)))
        want[3].append(np.zeros((k, 3), np.int32))
    padded = _call(systems, rc, capacity=T + P, pad=True)
    assert padded[4].tolist() == [T, 0]
    for w, x in zip(want, padded[:4]):
        assert np.array_equal(np.concatenate(w).view(np.uint8), x.view(np.uint8))
    # capacity == total: the exact list, no flag; one short: flag set and the exact list's prefix, with or without pad
    full = _call(systems, rc, capacity=T, pad=True)
    assert full[4].tolist() == [T, 0]
    for x, y in zip(full[:4], (ii, jj, off, sh)):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))
    for pad in (True, False):
        short = _call(systems, rc, capacity=T - 1, pad=pad)
        assert short[4].tolist() == [T, 1]
        for x, y in zip(short[:4], (ii, jj, off, sh)):
            assert np.array_equal(x.view(np.uint8), y[:T - 1].view(np.uint8))
    # capacity 0 only counts
    assert _call(systems, rc, capacity=0)[4].tolist() == [T, 1]
