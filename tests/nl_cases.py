"""Structures for the neighbour-list tests (tests/test_nl_oracle.py on the CPU, tests/test_cuda_neighbor_cells.py on the
GPU): perfect crystals whose coordination is known exactly, and random structures at the edges of the cell-list search
of csrc/neighbors.cu.  Every structure is (R [n,3], cell [3,3], pbc [3], cutoff), in fp64; the tests round it to fp32."""
from __future__ import annotations

import itertools

import numpy as np

from oracle import nl_oracle as NL

# name: primitive cell, basis in fractional coordinates of it, pbc, cutoff, conventional cell as integer combinations of
# the primitive rows, supercell multiples of the conventional cell, and the shells inside the cutoff (radius, count) --
# each cutoff lies between two shells, far from both, so the coordination is exact in fp32.
_S2, _S3 = np.sqrt(2.0), np.sqrt(3.0)
CRYSTALS = {
    "fcc": dict(a=4.05, prim=0.5 * np.array([[0, 1, 1], [1, 0, 1], [1, 1, 0]], float), basis=[[0, 0, 0]],
                pbc=[True] * 3, cutoff=5.0, conv=[[-1, 1, 1], [1, -1, 1], [1, 1, -1]], sup=(5, 5, 5),
                shells=[(1 / _S2, 12), (1.0, 6), (np.sqrt(1.5), 24)]),
    "bcc": dict(a=3.3, prim=0.5 * np.array([[-1, 1, 1], [1, -1, 1], [1, 1, -1]], float), basis=[[0, 0, 0]],
                pbc=[True] * 3, cutoff=5.0, conv=[[0, 1, 1], [1, 0, 1], [1, 1, 0]], sup=(6, 6, 6),
                shells=[(_S3 / 2, 8), (1.0, 6), (_S2, 12)]),
    "diamond": dict(a=5.43, prim=0.5 * np.array([[0, 1, 1], [1, 0, 1], [1, 1, 0]], float),
                    basis=[[0, 0, 0], [0.25, 0.25, 0.25]], pbc=[True] * 3, cutoff=5.0,
                    conv=[[-1, 1, 1], [1, -1, 1], [1, 1, -1]], sup=(3, 3, 3),
                    shells=[(_S3 / 4, 4), (1 / _S2, 12), (np.sqrt(11) / 4, 12)]),
    # a sheet as ase.build.graphene(vacuum=None) builds it: the third row is zero
    "graphene": dict(a=2.46, prim=np.array([[1, 0, 0], [0.5, _S3 / 2, 0], [0, 0, 0]]),
                     basis=[[0, 0, 0], [1 / 3, 1 / 3, 0]], pbc=[True, True, False], cutoff=3.0,
                     conv=[[1, 0, 0], [-1, 2, 0], [0, 0, 1]], sup=(4, 3, 1),
                     shells=[(1 / _S3, 3), (1.0, 6), (2 / _S3, 3)]),
}
VARIANTS = ["conventional", "supercell", "primitive", "rotated", "left_handed", "shifted"]


def coordination(name):
    return sum(m for _, m in CRYSTALS[name]["shells"])


def shell_radii(name):
    c = CRYSTALS[name]
    return np.array([r * c["a"] for r, _ in c["shells"]])


def _build(c, M):
    """The crystal in the cell M @ primitive (M integer): every lattice site whose fractional coordinates in the new
    cell lie in [0, 1) along the periodic axes."""
    prim = c["a"] * c["prim"]
    M = np.asarray(M, dtype=np.int64)
    cell = M @ prim
    pbc = np.asarray(c["pbc"])
    inv = np.linalg.inv(NL.complete_cell(cell, pbc))
    span = np.abs(M).sum(axis=0)
    rng = [range(-s, s + 1) if p else range(1) for s, p in zip(span, pbc)]
    sites = np.array(list(itertools.product(*rng)), dtype=np.float64)
    R = (sites[:, None, :] + np.asarray(c["basis"], float)[None]).reshape(-1, 3) @ prim
    f = np.round(R @ inv, 9)
    R = R[np.all(~pbc[None] | ((f >= 0) & (f < 1)), axis=1)]
    assert R.shape[0] == round(abs(np.linalg.det(M))) * len(c["basis"]), R.shape
    return R, cell


def crystal(name, variant):
    """(R, cell, pbc, cutoff) of a perfect crystal.  conventional: thinner than the cutoff (several images per axis,
    self images); supercell: at least three bins per periodic axis, atoms on the bin boundaries; primitive: heights far
    below the cutoff; rotated: the primitive cell under a random rotation; left_handed: conventional with two rows
    swapped; shifted: the supercell moved by -1e-7 of its periodic rows, so atoms sit just below fractional 0."""
    c = CRYSTALS[name]
    pbc = np.asarray(c["pbc"])
    conv = np.asarray(c["conv"])
    if variant in ("primitive", "rotated"):
        R, cell = _build(c, np.eye(3, dtype=np.int64))
    elif variant in ("supercell", "shifted"):
        R, cell = _build(c, np.diag(c["sup"]) @ conv)
    else:
        R, cell = _build(c, conv)
    if variant == "rotated":
        q, r = np.linalg.qr(np.random.default_rng(sum(map(ord, name))).normal(size=(3, 3)))
        q = q * np.sign(np.diag(r))
        if np.linalg.det(q) < 0:
            q[:, 0] = -q[:, 0]
        R, cell = R @ q.T, cell @ q.T
    elif variant == "left_handed":
        cell = cell[[1, 0, 2]]
    elif variant == "shifted":
        R = R - 1e-7 * (pbc[:, None] * cell).sum(axis=0)
    return R, cell, pbc, c["cutoff"]


def random_cases():
    """Random structures at the edges of the search, as {name: (R, cell, pbc, cutoff)}."""
    rng = np.random.default_rng(20261017)
    out = {}
    # heights far below the edge lengths: one height 2.4 < rc, reach > 1 and a single bin on that axis
    tri = np.array([[8.0, 0.0, 0.0], [7.0, 3.5, 0.0], [6.0, 1.5, 2.4]])
    out["skewed"] = (rng.uniform(0, 1, (40, 3)) @ tri, tri, np.ones(3, bool), 4.0)
    thin = np.diag([2.0, 14.0, 14.0])
    out["thin_axis"] = (rng.uniform(0, 1, (60, 3)) @ thin, thin, np.ones(3, bool), 5.0)
    # fewer atoms than cells: the grid is coarsened; the first two atoms are neighbours only across the boundary
    box = np.eye(3) * 60.0
    out["coarsened_3"] = (np.array([[0.4, 30.0, 30.0], [59.1, 30.6, 29.5], [31.0, 12.0, 47.0]]), box, np.ones(3, bool), 5.0)
    out["coarsened_2"] = (np.array([[20.0, 0.2, 59.7], [20.5, 59.3, 0.9]]), box, np.ones(3, bool), 5.0)
    # more than 32 atoms per bin: 2 x 2 x 2 bins of 12 Å hold about 100 atoms each
    out["dense"] = (rng.uniform(0, 12.0, (800, 3)), np.eye(3) * 12.0, np.ones(3, bool), 5.0)
    # every atom moved by its own random lattice vector in [-20, 20]^3
    cell = np.array([[9.0, 0.0, 0.0], [2.5, 8.0, 0.0], [-1.5, 2.0, 7.5]])
    k = rng.integers(-20, 21, (70, 3))
    out["unwrapped"] = (rng.uniform(0, 1, (70, 3)) @ cell + k @ cell, cell, np.ones(3, bool), 4.0)
    # a slab and a wire, with zero and with finite (tilted) non-periodic rows, atoms far outside the finite rows
    slab = np.array([[11.0, 0.0, 0.0], [2.0, 12.5, 0.0], [0.0, 0.0, 0.0]])
    R = rng.uniform(0, 1, (80, 3)) @ slab + rng.uniform(-6, 6, (80, 1)) * [[0.0, 0.0, 1.0]]
    out["slab_zero"] = (R, slab, np.array([True, True, False]), 5.0)
    out["slab_finite"] = (R, slab + [[0, 0, 0], [0, 0, 0], [1.0, -2.0, 3.0]], np.array([True, True, False]), 5.0)
    wire = np.array([[0.0, 0.0, 0.0], [0.0, 0.0, 0.0], [0.3, -0.2, 4.1]])
    R = rng.normal(size=(30, 3)) * [2.5, 2.5, 0.0] + rng.uniform(0, 1, (30, 1)) * wire[2]
    out["wire_zero"] = (R, wire, np.array([False, False, True]), 5.0)
    out["wire_finite"] = (R, wire + [[3.0, 0.5, 0.0], [-1.0, 2.0, 0.5], [0, 0, 0]], np.array([False, False, True]), 5.0)
    one = np.array([[3.1, 0.0, 0.0], [1.2, 2.9, 0.0], [0.4, -0.7, 3.3]])
    out["one_atom"] = (np.array([[0.7, -0.3, 1.9]]), one, np.ones(3, bool), 5.0)
    return out


ZERO_FINITE_PAIRS = [("slab_zero", "slab_finite"), ("wire_zero", "wire_finite")]
