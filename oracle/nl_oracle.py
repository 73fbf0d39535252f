"""ORACLE -- test infrastructure, NOT product code: CPU restatement (numpy, float64) of the reference's neighbour-list
semantics for the "next" row f1 of SURVEY.md section 8.

The reference's own torch implementation is ``transform/neighborlist.py:428-553`` (``TorchNeighborList``); its ASE /
matscipy / vesin front ends (``:213-286``) return the same SET of pairs.  Contract restated here:

  * a pair (i, j, S) is listed iff  | R[j] - R[i] + S @ cell | < cutoff  (strict, ``:500-501``), for integer image
    vectors S with |S_a| <= ceil(cutoff * |row a of inverse(cell).T|) on periodic axes and S_a = 0 elsewhere
    (``_get_shifts`` ``:515-553``), excluding (i == j, S == 0); self-image pairs i == j with S != 0 are listed;
  * the list is symmetric ((j, i, -S) is listed with (i, j, S), ``:444-456``), ordered by idx_i (``:450``);
  * offsets = S @ cell (``:457``).

Beyond the reference class (whose ASE / matscipy front ends accept both): positions may lie outside the cell, any number
of cells away, and the rows of non-periodic axes may be zero (a sheet or a wire built with ``vacuum=None``).
``band_neighbor_list`` classifies the pairs of fp32 inputs by the fp32 rounding of the distance test.

Parity pin: ``tests/golden/make_golden_nl.py`` runs the UNMODIFIED reference class and stores its output in canonical
(i, j, S) order under ``tests/golden/nl_*.npz``; ``tests/test_oracle_golden.py`` holds this oracle to those fixtures.
"""
from __future__ import annotations

import numpy as np


def canonical(idx_i, idx_j, shifts):
    """Sort a pair list by (i, j, Sx, Sy, Sz) -- the comparison order of the reference's tests
    (tests/data/test_transforms.py:53-104 sort both lists before comparing)."""
    idx_i, idx_j, shifts = np.asarray(idx_i), np.asarray(idx_j), np.asarray(shifts).reshape(-1, 3)
    order = np.lexsort((shifts[:, 2], shifts[:, 1], shifts[:, 0], idx_j, idx_i))
    return idx_i[order], idx_j[order], shifts[order]


def complete_cell(cell, pbc):
    """The cell with every non-periodic row replaced by an orthonormal completion of the periodic rows (the unit normal
    of two periodic rows; two unit vectors orthogonal to one periodic row and to each other).  Heights, fractional
    coordinates and wraps along the periodic axes then depend on the periodic rows only, and a sheet or a wire whose
    non-periodic rows are zero gets an invertible cell.  Without a periodic axis the cell is returned unchanged."""
    c = np.array(cell, dtype=np.float64).reshape(3, 3)
    pbc = np.asarray(pbc).astype(bool).reshape(3)
    per, non = np.flatnonzero(pbc), np.flatnonzero(~pbc)
    if per.size == 2:
        n = np.cross(c[per[0]], c[per[1]])
        c[non[0]] = n / np.linalg.norm(n)
    elif per.size == 1:
        p = c[per[0]] / np.linalg.norm(c[per[0]])
        u = np.cross(p, np.eye(3)[np.argmin(np.abs(p))])      # the coordinate axis least aligned with p
        u /= np.linalg.norm(u)
        c[non[0]], c[non[1]] = u, np.cross(p, u)
    return c


def image_reach(cell, pbc, cutoff):
    """transform/neighborlist.py:529-535 -- images needed per axis for positions inside the (completed) cell."""
    cell = complete_cell(cell, pbc)
    pbc = np.asarray(pbc).astype(bool).reshape(3)
    if not pbc.any():
        return np.zeros(3, dtype=np.int64)
    inv_len = np.linalg.norm(np.linalg.inv(cell).T, axis=1)
    return np.where(pbc, np.ceil(cutoff * inv_len).astype(np.int64), 0)


def wraps(positions, cell, pbc):
    """k [n,3] (int64): R - k @ cell lies inside the completed cell along every periodic axis (k = 0 elsewhere)."""
    R = np.asarray(positions, dtype=np.float64).reshape(-1, 3)
    pbc = np.asarray(pbc).astype(bool).reshape(3)
    if not pbc.any():
        return np.zeros((R.shape[0], 3), dtype=np.int64)
    frac = R @ np.linalg.inv(complete_cell(cell, pbc))
    return np.where(pbc[None, :], np.floor(frac), 0.0).astype(np.int64)


def _pairs_within(R, cell, pbc, rmax):
    """Every (i, j, S) with |R[j] - R[i] + S @ cell| < rmax in fp64, (i == j, S == 0) excluded, for positions anywhere:
    the image search runs on the positions wrapped into the cell and maps each S back by the wrap difference, so
    (i, j, S') of the wrapped positions is (i, j, S' + k_i - k_j) of the given ones.  Returns i, j, S, distance."""
    R = np.asarray(R, dtype=np.float64).reshape(-1, 3)
    cell = np.asarray(cell, dtype=np.float64).reshape(3, 3)
    n = R.shape[0]
    reach = image_reach(cell, pbc, rmax)
    k = wraps(R, cell, pbc)
    dk = k[:, None, :] - k[None, :, :]                                                      # [i, j]: k_i - k_j
    out_i, out_j, out_s, out_d = [], [], [], []
    for sx in range(-reach[0], reach[0] + 1):
        for sy in range(-reach[1], reach[1] + 1):
            for sz in range(-reach[2], reach[2] + 1):
                S = np.array([sx, sy, sz], dtype=np.int64)
                if k.any():
                    Sij = S + dk
                    off = (Sij.astype(np.float64).reshape(-1, 3) @ cell).reshape(n, n, 3)
                else:
                    Sij = np.broadcast_to(S, (n, n, 3))
                    off = (S.astype(np.float64) @ cell)[None, None, :]
                d = np.linalg.norm(R[None, :, :] + off - R[:, None, :], axis=-1)            # [i, j]
                mask = d < rmax
                mask &= ~(np.eye(n, dtype=bool) & ~Sij.any(axis=-1))
                ii, jj = np.nonzero(mask)
                out_i.append(ii)
                out_j.append(jj)
                out_s.append(Sij[ii, jj])
                out_d.append(d[ii, jj])
    if not out_i:
        return (np.zeros(0, dtype=np.int64),) * 2 + (np.zeros((0, 3), dtype=np.int64), np.zeros(0))
    return (np.concatenate(out_i).astype(np.int64), np.concatenate(out_j).astype(np.int64),
            np.concatenate(out_s).reshape(-1, 3).astype(np.int64), np.concatenate(out_d))


def neighbor_list(positions, cell, pbc, cutoff):
    """One structure.  Returns idx_i, idx_j (int64), shifts S [E,3] (int64) in canonical order and offsets = S @ cell.
    Positions may lie anywhere, and non-periodic rows of the cell may be zero."""
    cell = np.asarray(cell, dtype=np.float64).reshape(3, 3)
    ii, jj, ss, _ = _pairs_within(positions, cell, pbc, cutoff)
    ii, jj, ss = canonical(ii, jj, ss)
    return ii, jj, ss, ss.astype(np.float64) @ cell


# fp32 rounding band.  The device list decides | R[j] - R[i] + S @ cell | < cutoff in fp32 on the fp32 inputs; the
# binning only picks which cells are visited, and its cells are wider than the cutoff, so it drops no pair at the
# coordinates tested here.  What can differ from fp64 is the distance test itself.  Per component, S @ cell costs at
# most 3u sum_a |S_a| |cell_a,x|, R[j] - R[i] costs u (|R_i,x| + |R_j,x|), the final sum u |r_x| <= u rc; the squared
# norm and the fp32 cutoff**2 add about 2u rc on the distance.  Summing components bounds the error of the distance by
# u (||R_i||_1 + ||R_j||_1 + 3 sum_a |S_a| ||cell_a||_1 + 5 rc); BAND_UNITS doubles that.
U32 = 2.0 ** -24
BAND_UNITS = 2.0


def band_width(R, cell, idx_i, idx_j, shifts, cutoff):
    """delta of each pair (i, j, S): the largest difference between the fp32 and the exact distance, see above."""
    R = np.asarray(R, dtype=np.float64).reshape(-1, 3)
    l1 = np.abs(np.asarray(cell, dtype=np.float64).reshape(3, 3)).sum(axis=1)
    s = np.abs(np.asarray(shifts, dtype=np.float64).reshape(-1, 3))
    r1 = np.abs(R).sum(axis=1)
    return BAND_UNITS * U32 * (r1[idx_i] + r1[idx_j] + 3.0 * (s @ l1) + 5.0 * cutoff)


def band_neighbor_list(positions, cell, pbc, cutoff):
    """The pairs an fp32 list of the fp32 ``positions`` and ``cell`` must and may contain, each as (i, j, Sx, Sy, Sz):
    ``definite`` with d64 < cutoff - delta (must be listed) and ``band`` with |d64 - cutoff| <= delta (may be listed),
    d64 being the fp64 distance of the given inputs and delta = band_width(...)."""
    R = np.asarray(positions, dtype=np.float64).reshape(-1, 3)
    cell = np.asarray(cell, dtype=np.float64).reshape(3, 3)
    k = wraps(R, cell, pbc)
    # search radius: cutoff + the largest delta any pair can have (|S_a| <= reach_a + the spread of the wraps)
    smax = image_reach(cell, pbc, cutoff * 1.01) + (k.max(axis=0) - k.min(axis=0) if R.shape[0] else 0)
    dmax = BAND_UNITS * U32 * (2 * np.abs(R).sum(axis=1).max(initial=0.0) + 3.0 * smax @ np.abs(cell).sum(axis=1)
                               + 5.0 * cutoff)
    assert dmax < 0.01 * cutoff
    ii, jj, ss, d = _pairs_within(R, cell, pbc, cutoff + dmax)
    delta = band_width(R, cell, ii, jj, ss, cutoff)
    keys = np.concatenate([ii[:, None], jj[:, None], ss], axis=1).tolist()
    definite = {tuple(t) for t, m in zip(keys, d < cutoff - delta) if m}
    band = {tuple(t) for t, m in zip(keys, np.abs(d - cutoff) <= delta) if m}
    return definite, band


def batch_neighbor_list(positions, cells, pbcs, n_atoms, cutoff):
    """Collated batch (data/loader.py:35-46: indices of system b are shifted by the atoms before it)."""
    out_i, out_j, out_s, out_o = [], [], [], []
    start = 0
    for b, na in enumerate(np.asarray(n_atoms).tolist()):
        ii, jj, ss, oo = neighbor_list(np.asarray(positions)[start:start + na], np.asarray(cells).reshape(-1, 3, 3)[b],
                                       np.asarray(pbcs).reshape(-1, 3)[b], cutoff)
        out_i.append(ii + start)
        out_j.append(jj + start)
        out_s.append(ss)
        out_o.append(oo)
        start += na
    return (np.concatenate(out_i), np.concatenate(out_j), np.concatenate(out_s).reshape(-1, 3),
            np.concatenate(out_o).reshape(-1, 3))
