"""Generate golden neighbour-list fixtures from the UNMODIFIED reference ``TorchNeighborList``
(/root/reference/src/schnetpack/transform/neighborlist.py:428-553), imported through the stub-package loader.
Run in the build container only:  python tests/golden/make_golden_nl.py   ->  tests/golden/nl_*.npz
Stored: positions, cell, pbc, cutoff and the reference's pair list in canonical (i, j, S) order (S recovered from the
returned offsets = S @ cell)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_loader as _ref_loader  # noqa: E402

from oracle import nl_oracle as NL  # noqa: E402


def cases():
    rng = np.random.default_rng(20260922)
    out = {}
    # molecule, no periodicity (the reference skips the shift construction when pbc is all False)
    out["molecule"] = dict(R=rng.normal(size=(21, 3)) * 2.0, cell=np.zeros((3, 3)), pbc=[False] * 3, cutoff=5.0)
    # cubic box larger than 3 cutoffs (cell-list regime)
    L = 16.5
    out["cubic"] = dict(R=rng.uniform(-3.0, L + 3.0, size=(160, 3)), cell=np.eye(3) * L, pbc=[True] * 3, cutoff=5.0)
    # small box: several images per axis, self-image pairs
    out["small_box"] = dict(R=rng.uniform(0, 3.1, size=(7, 3)), cell=np.eye(3) * 3.1, pbc=[True] * 3, cutoff=5.0)
    # triclinic cell
    tri = np.array([[9.0, 0.0, 0.0], [2.5, 8.0, 0.0], [-1.5, 2.0, 7.5]])
    out["triclinic"] = dict(R=rng.uniform(0, 1, size=(60, 3)) @ tri + rng.normal(size=(60, 3)), cell=tri, pbc=[True] * 3,
                            cutoff=4.0)
    # slab: periodic in x, y only
    slab = np.diag([11.0, 12.5, 30.0])
    out["slab"] = dict(R=rng.uniform(0, 1, size=(80, 3)) @ np.diag([11.0, 12.5, 9.0]), cell=slab,
                       pbc=[True, True, False], cutoff=5.0)
    # primitive fcc cell: one atom, 60 degree angles, every height a / sqrt(3) far below the cutoff
    fcc = 4.05 / 2 * np.array([[0.0, 1.0, 1.0], [1.0, 0.0, 1.0], [1.0, 1.0, 0.0]])
    out["fcc_primitive"] = dict(R=np.array([[0.3, -0.2, 0.1]]), cell=fcc, pbc=[True] * 3, cutoff=5.0)
    # strongly skewed triclinic cell: edges of 8-10 A, one height of 2.4 A below the cutoff
    skew = np.array([[8.0, 0.0, 0.0], [7.0, 3.5, 0.0], [6.0, 1.5, 2.4]])
    out["skewed"] = dict(R=rng.uniform(0, 1, size=(30, 3)) @ skew, cell=skew, pbc=[True] * 3, cutoff=4.0)
    return out


def main():
    spk = _ref_loader.load()
    nl = spk.transform.TorchNeighborList(cutoff=1.0)
    for name, c in cases().items():
        R = torch.tensor(np.asarray(c["R"]), dtype=torch.float64)
        cell = torch.tensor(np.asarray(c["cell"]), dtype=torch.float64)
        pbc = torch.tensor(c["pbc"])
        Z = torch.ones(R.shape[0], dtype=torch.long)
        ii, jj, off = nl._build_neighbor_list(Z, R, cell, pbc, float(c["cutoff"]))
        ii, jj, off = ii.numpy(), jj.numpy(), off.numpy()
        if pbc.any():
            S = np.rint(off @ np.linalg.inv(cell.numpy())).astype(np.int64)
            assert np.abs(S @ cell.numpy() - off).max() < 1e-9
        else:
            S = np.zeros((ii.shape[0], 3), dtype=np.int64)
        ci, cj, cs = NL.canonical(ii, jj, S)
        np.savez_compressed(os.path.join(HERE, f"nl_{name}.npz"), positions=np.asarray(c["R"]), cell=np.asarray(c["cell"]),
                            pbc=np.asarray(c["pbc"]), cutoff=np.float64(c["cutoff"]), idx_i=ci, idx_j=cj, shifts=cs)
        oi, oj, os_, _ = NL.neighbor_list(c["R"], c["cell"], c["pbc"], c["cutoff"])
        same = oi.shape == ci.shape and (oi == ci).all() and (oj == cj).all() and (os_ == cs).all()
        print(f"{name}: {ci.shape[0]} pairs from the reference; oracle identical: {same}")


if __name__ == "__main__":
    main()
