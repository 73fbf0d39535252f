"""Generate tests/golden/phonons_cscl.npz: force constants of the UNMODIFIED reference (oracle/ref_loader) in fp64 for the
phonon method of schnetpack_b200.phonons.

The crystal is a 2-atom CsCl-type primitive cell (cubic, a = 2.9 A, Z = 6 at the origin and Z = 8 near the centre) and its
3 x 3 x 3 supercell (54 atoms, 8.7 A), built as tests/phonon_oracle.py builds it (atom l n + b = x_b + n_l . cell in
fp64, rounded to fp32).  A seeded PaiNN model (32 features, 2 interactions, cutoff 4 A, below half the supercell) is
evaluated by the reference's ``Response("energy", ["forces", "hessian"])`` on the supercell: ref64:hessian [54^2, 3, 3]
is its analytic Hessian and ref64:force_constants [2 * 54, 3, 3] the rows of the two primitive atoms.  ASE-style
finite differences at h = 0.01 A, nfree = 2, displace the primitive atoms only: the displaced coordinate is rounded to
fp32 as the device does, the reference's fp64 forces are taken at the fp32 positions with the neighbour list rebuilt,
and fd2:steps [6, 2] / fd2:forces [6, 2, 54, 3] keep the realised steps and the forces.

The second atom sits off the cube centre: at the symmetric site PaiNN's vector features vanish, and the regularised norm
sqrt(|v|^2 + epsilon) then curves on a 1e-4 A scale, far below any finite-difference step.

Run from the repository root:  python tests/golden/make_golden_phonons.py
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import phonon_oracle as O  # noqa: E402
from oracle import ref_loader as rl  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402

H = 0.01
A = 2.9
SUPERCELL = np.array([3, 3, 3])
MASSES = np.array([12.011, 15.999])


def _inputs(R, cell, z, cutoff):
    ii, jj, ss = S.periodic_cell_list(R.astype(np.float64), float(cell[0, 0]), cutoff)
    n = R.shape[0]
    return {S.Z: z, S.R: R, S.cell: cell[None].astype(np.float32), S.pbc: np.ones((1, 3), dtype=bool),
            S.idx_m: np.zeros(n, dtype=np.int64), S.n_atoms: np.array([n]), S.idx_i: ii, S.idx_j: jj,
            S.offsets: (ss * cell[0, 0]).astype(np.float32)}


def _x(inputs):
    return {k: (torch.as_tensor(v).double() if np.asarray(v).dtype.kind == "f" else torch.as_tensor(v))
            for k, v in inputs.items()}


def main():
    torch.set_grad_enabled(True)
    spec = S.model_spec("painn", n_atom_basis=32, n_interactions=2, cutoff=4.0)
    params = S.init_params(spec, 7)
    model = rl.build_from_spec(spec, params, torch.float64)
    spk = rl.load()
    resp = spk.model.NeuralNetworkPotential(
        model.representation, input_modules=list(model.input_modules),
        output_modules=[model.output_modules[0], spk.atomistic.Response("energy", ["forces", "hessian"])],
        postprocessors=[], do_postprocessing=False).double().eval()
    pos = np.array([[0.0, 0.0, 0.0], [A / 2 + 0.13, A / 2 - 0.07, A / 2 + 0.21]], dtype=np.float32)
    cell = (A * np.eye(3)).astype(np.float32)
    z = np.array([6, 8], dtype=np.int64)
    lattice, _ = O.translations(SUPERCELL)
    sp, sc = O.supercell(pos, cell, SUPERCELL, lattice)
    zs = np.tile(z, lattice.shape[0])
    n, n_super = 2, sp.shape[0]
    out = resp(_x(_inputs(sp, sc, zs, spec["cutoff"])))
    hess = out["hessian"].detach().numpy()
    steps, forces = np.zeros((3 * n, 2)), np.zeros((3 * n, 2, n_super, 3))
    for d in range(3 * n):
        for s, o in enumerate((-1.0, 1.0)):
            R = sp.copy()
            R[d // 3, d % 3] = np.float32(sp[d // 3, d % 3]) + np.float32(o * H)
            steps[d, s] = float(R[d // 3, d % 3]) - float(sp[d // 3, d % 3])
            forces[d, s] = model(_x(_inputs(R, sc, zs, spec["cutoff"])))["forces"].detach().numpy()
    prim = {S.Z: z, S.R: pos, S.cell: cell[None], S.pbc: np.ones((1, 3), dtype=bool), S.idx_m: np.zeros(n, np.int64),
            S.n_atoms: np.array([n])}
    blob = {"spec_json": np.array(json.dumps(spec)), "H": np.array(H), "supercell": SUPERCELL, "masses": MASSES,
            "super_positions": sp, "super_cell": sc, "ref64:hessian": hess,
            "ref64:force_constants": O.fc_from_hessian(hess, n, n_super), "fd2:steps": steps, "fd2:forces": forces}
    blob.update({"in:" + k: v for k, v in prim.items()})
    blob.update({"param:" + k: np.asarray(v) for k, v in params.items()})
    path = os.path.join(HERE, "phonons_cscl.npz")
    np.savez_compressed(path, **blob)
    print(f"phonons_cscl: {n_super} supercell atoms -> {os.path.getsize(path) / 1e3:.0f} kB")


if __name__ == "__main__":
    main()
