"""Generate tests/golden/md_system.npz: the reference's own motion removal and wrapping (md/system.py:258-315,652-684),
initializers (md/initial_conditions.py) and basic simulation hooks (md/simulation_hooks/basic_hooks.py) applied to a
reference ``System`` in fp64.

The System holds three molecules of 3, 9 and 20 atoms, with R = 1 and R = 4 replicas.  Every molecule has a cell: a
triclinic box (pbc T, T, T), a slab (T, T, F) and a skewed box (T, T, T), and its atoms sit several cells away from the
origin on both sides.  The replicas of R = 4 differ by small displacements, and no atom sits near a cell face, so
wrapping every replica on its own (the reference) and wrapping by centroids (the device) agree there.

The modules are loaded with the stubs of make_golden_md_thermostats.py.  ``torch.randn_like`` inside
md/initial_conditions.py is replaced by a recorder that returns seeded normals and stores them, so that the oracle can
be fed the same draws.  ``MaxwellBoltzmannInit`` with one temperature per molecule is run too; the reference raises
there (``expand_atoms`` indexes a 1-D tensor with two indices), and the fixture records that it does.

Run from the repository root:  python tests/golden/make_golden_md_system.py
"""
import importlib
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden_md_thermostats import load_reference_md  # noqa: E402
from schnetpack_b200.md import KB_MD  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "md_system.npz")
N_ATOMS = [3, 9, 20]
PBC = np.array([[True, True, True], [True, True, False], [True, True, True]])
CELLS = np.array([[[6.0, 0.0, 0.0], [1.5, 5.5, 0.0], [0.8, -1.1, 7.0]],
                  [[8.0, 0.0, 0.0], [0.0, 7.0, 0.0], [0.0, 0.0, 30.0]],
                  [[9.0, 0.5, 0.0], [-2.0, 8.5, 0.3], [1.0, 1.5, 10.0]]])
INITIALIZERS = {
    "mb_default": ("MaxwellBoltzmannInit", 300.0, {}),
    "mb_all": ("MaxwellBoltzmannInit", 300.0, dict(remove_rotation=True, wrap_positions=True)),
    "mb_none": ("MaxwellBoltzmannInit", 250.0, dict(remove_center_of_mass=False, remove_translation=False)),
    "mb_rot_origin": ("MaxwellBoltzmannInit", 300.0, dict(remove_center_of_mass=False, remove_translation=False,
                                                          remove_rotation=True)),
    "uni_default": ("UniformInit", 300.0, {}),
    "uni_all": ("UniformInit", [200.0, 300.0, 450.0], dict(remove_rotation=True, wrap_positions=True)),
    "uni_wrap_rot": ("UniformInit", 350.0, dict(remove_center_of_mass=False, remove_rotation=True,
                                                wrap_positions=True)),
}


def inputs(n_replicas, seed=11):
    rng = np.random.default_rng(seed + n_replicas)
    n = sum(N_ATOMS)
    masses = rng.choice([1.008, 12.011, 15.999, 32.06], size=n)
    idx = np.repeat(np.arange(len(N_ATOMS)), N_ATOMS)
    frac = rng.uniform(0.15, 0.85, size=(n, 3))
    frac[:, :2] += rng.integers(-3, 4, size=(n, 2))                     # several cells away, both sides
    frac[:, 2] += np.where(PBC[idx, 2], rng.integers(-3, 4, size=n), 0)
    x = np.einsum("nj,nji->ni", frac, CELLS[idx])
    x = x[None] + 0.02 * rng.normal(size=(n_replicas, n, 3)) * (n_replicas > 1)
    p = rng.normal(size=(n_replicas, n, 3)) * np.sqrt(masses * KB_MD * 300.0)[None, :, None]
    return masses, x, p


def make_system(system_mod, masses, x, p):
    s = system_mod.System()
    R, n = x.shape[:2]
    M = len(N_ATOMS)
    s.n_replicas, s.n_molecules, s.total_n_atoms = R, M, n
    s.n_atoms = torch.tensor(N_ATOMS, dtype=torch.long)
    s.index_m = torch.repeat_interleave(torch.arange(M), torch.tensor(N_ATOMS))
    s.atom_types = torch.ones(n, dtype=torch.long)
    s.masses = torch.tensor(masses, dtype=torch.float64).reshape(1, n, 1)
    s.positions = torch.tensor(x, dtype=torch.float64).clone()
    s.momenta = torch.tensor(p, dtype=torch.float64).clone()
    s.forces = torch.zeros(R, n, 3, dtype=torch.float64)
    s.energy = torch.zeros(R, M, 1, dtype=torch.float64)
    s.cells = torch.tensor(CELLS, dtype=torch.float64)[None].repeat(R, 1, 1, 1)
    s.stress = torch.zeros(R, M, 3, 3, dtype=torch.float64)
    s.pbc = torch.tensor(PBC)[None]
    s._dd_dummy = torch.zeros(1, dtype=torch.float64)
    return s


class _RecordedNormals:
    def __init__(self, seed):
        self.gen = torch.Generator().manual_seed(seed)
        self.draws = []

    def __call__(self, like):
        z = torch.randn(like.shape, generator=self.gen, dtype=torch.float64)
        self.draws.append(z.numpy().copy())
        return z


def main():
    _, system_mod = load_reference_md()
    md = sys.modules["schnetpack.md"]
    md.System = system_mod.System
    ic = importlib.import_module("schnetpack.md.initial_conditions")
    hooks = importlib.import_module("schnetpack.md.simulation_hooks.basic_hooks")
    out = {"n_atoms": np.array(N_ATOMS), "cells": CELLS, "pbc": PBC, "kB": KB_MD}
    for R in (1, 4):
        masses, x, p = inputs(R)
        key = f"r{R}"
        out[f"{key}:masses"], out[f"{key}:positions"], out[f"{key}:momenta"] = masses, x, p
        for k, (name, (cls, temp, kw)) in enumerate(INITIALIZERS.items()):
            s = make_system(system_mod, masses, x, p)
            rec = _RecordedNormals(seed=100 * R + k)
            torch.randn_like = rec                      # the name md/initial_conditions.py calls
            try:
                getattr(ic, cls)(temp, **kw).initialize_system(s)
            finally:
                torch.randn_like = _TORCH_RANDN_LIKE
            assert len(rec.draws) == 1
            out[f"{key}:{name}:normals"] = rec.draws[0]
            out[f"{key}:{name}:positions"] = s.positions.numpy().copy()
            out[f"{key}:{name}:momenta"] = s.momenta.numpy().copy()
        s = make_system(system_mod, masses, x, p)
        torch.randn_like = _RecordedNormals(0)
        try:
            ic.MaxwellBoltzmannInit([200.0, 300.0, 450.0]).initialize_system(s)
            out[f"{key}:mb_per_system_raises"] = np.array(False)
        except (IndexError, RuntimeError):
            out[f"{key}:mb_per_system_raises"] = np.array(True)
        finally:
            torch.randn_like = _TORCH_RANDN_LIKE
        for name, hook in (("com_rot", hooks.RemoveCOMMotion(1, True)), ("com", hooks.RemoveCOMMotion(1, False)),
                           ("wrap", hooks.WrapPositions(1))):
            s = make_system(system_mod, masses, x, p)
            hook.on_step_finalize(SimpleNamespace(step=0, system=s))
            out[f"{key}:hook_{name}:positions"] = s.positions.numpy().copy()
            out[f"{key}:hook_{name}:momenta"] = s.momenta.numpy().copy()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays")


_TORCH_RANDN_LIKE = torch.randn_like

if __name__ == "__main__":
    main()
