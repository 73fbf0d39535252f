"""Generate tests/golden/md_barostats.npz: the reference's own NHCBarostatIsotropic and NHCBarostatAnisotropic
(md/simulation_hooks/barostats.py:162-927) driving a reference ``System`` (md/system.py) of three periodic boxes of 5, 12
and 27 atoms (the last one triclinic), in fp64.

Stubs as in make_golden_md_thermostats.py (ASE-free ``schnetpack.units`` with kB, fs and, new here, bar; omegaconf), plus
one shim: the anisotropic barostat calls ``torch.symeig``, which current torch has removed.  It is replaced by
``torch.linalg.eigh(A, UPLO="U")`` -- what symeig(eigenvectors=True, upper=True) computed (ascending eigenvalues, the upper
triangle read).

Units are exact binary fractions (kB = 2^-7, fs = 2^-10, bar = 2^-12, T = 300 K, tau = 128 fs, dt = 2^-7), so the
reference's float32 parameter buffers hold exactly the values the fp64 kernels use.  Each case runs on_simulation_start and
then N_STEPS of on_step_begin -> propagate_half_step -> propagate_main_step -> forces / stress from seeded arrays ->
propagate_half_step -> on_step_end, which is NPTVelocityVerlet.half_step / main_step (md/integrators.py:249-263) inside the
step of md/simulator.py:124-150.  Stored: the inputs, and per case positions, momenta, cells, chain and barostat state.

Run from the repository root:  python tests/golden/make_golden_md_barostats.py
"""
import importlib
import os
import sys
import types
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "md_barostats.npz")
UNITS = dict(kB=2.0 ** -7, fs=2.0 ** -10, bar=2.0 ** -12)
N_ATOMS = [5, 12, 27]
T_BATH, TAU_FS, P_BAR, DT = 300.0, 128.0, 40.0, 2.0 ** -7
N_STEPS = 6
CASES = {"iso_o3": dict(anisotropic=False, massive=False, integration_order=3),
         "iso_massive_o7": dict(anisotropic=False, massive=True, integration_order=7),
         "aniso_o7": dict(anisotropic=True, massive=False, integration_order=7),
         "aniso_massive_o3": dict(anisotropic=True, massive=True, integration_order=3, chain_length=3, multi_step=2)}


def _stub(name, path=None, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    if path:
        m.__path__ = [path]
    sys.modules[name] = m
    return m


def load_reference_barostats():
    spk = ref_loader.load()
    ref = ref_loader.REF
    _stub("omegaconf", DictConfig=dict, open_dict=None, OmegaConf=None)
    spk.units = _stub("schnetpack.units", unit2internal=lambda u: 1.0, **UNITS)
    md = _stub("schnetpack.md", ref + "/md")
    spk.md = md
    md.utils = importlib.import_module("schnetpack.md.utils")
    hooks = _stub("schnetpack.md.simulation_hooks", ref + "/md/simulation_hooks")
    hooks.SimulationHook = importlib.import_module("schnetpack.md.simulation_hooks.basic_hooks").SimulationHook
    baro = importlib.import_module("schnetpack.md.simulation_hooks.barostats")
    system = importlib.import_module("schnetpack.md.system")
    return baro, system


def _symeig(a, eigenvectors=True, upper=True):
    """torch.symeig(eigenvectors=True) as it was before its removal (torch 1.9 deprecation)"""
    return torch.linalg.eigh(a, UPLO="U" if upper else "L")


def inputs(seed=11):
    rng = np.random.default_rng(seed)
    n = sum(N_ATOMS)
    masses = rng.choice([1.0, 12.0, 16.0], size=n)
    momenta = rng.normal(size=(n, 3)) * np.sqrt(masses * UNITS["kB"] * 300.0)[:, None]
    cells = []
    for k, na in enumerate(N_ATOMS):
        edge = (na / 0.05) ** (1.0 / 3.0)                      # ~0.05 atoms per unit volume
        c = np.diag([edge, edge * 1.1, edge * 0.9])
        if k == 2:                                            # triclinic
            c[1, 0], c[2, 0], c[2, 1] = 0.3 * edge, -0.2 * edge, 0.25 * edge
        cells.append(c)
    cells = np.stack(cells)
    frac = rng.uniform(size=(n, 3))
    idx = np.repeat(np.arange(len(N_ATOMS)), N_ATOMS)
    positions = np.einsum("na,nab->nb", frac, cells[idx])
    # seeded forces and stresses for every evaluation (stress symmetric up to a small asymmetric part)
    forces = rng.normal(size=(N_STEPS, n, 3)) * 2.0
    stress = rng.normal(size=(N_STEPS, len(N_ATOMS), 3, 3)) * 0.02
    stress = 0.5 * (stress + stress.transpose(0, 1, 3, 2)) + 1e-4 * rng.normal(size=stress.shape)
    stress0 = 0.01 * np.eye(3)[None].repeat(len(N_ATOMS), 0)
    return masses, momenta, positions, cells, forces, stress, stress0


def make_system(system_mod, masses, momenta, positions, cells, stress0):
    s = system_mod.System()
    n = sum(N_ATOMS)
    M = len(N_ATOMS)
    s.n_replicas, s.n_molecules, s.total_n_atoms = 1, M, n
    s.n_atoms = torch.tensor(N_ATOMS, dtype=torch.long)
    s.index_m = torch.repeat_interleave(torch.arange(M), torch.tensor(N_ATOMS))
    s.atom_types = torch.ones(n, dtype=torch.long)
    s.masses = torch.tensor(masses, dtype=torch.float64).reshape(1, n, 1)
    s.positions = torch.tensor(positions, dtype=torch.float64).reshape(1, n, 3)
    s.momenta = torch.tensor(momenta, dtype=torch.float64).reshape(1, n, 3)
    s.forces = torch.zeros(1, n, 3, dtype=torch.float64)
    s.energy = torch.zeros(1, M, 1, dtype=torch.float64)
    s.cells = torch.tensor(cells, dtype=torch.float64).reshape(1, M, 3, 3)
    s.stress = torch.tensor(stress0, dtype=torch.float64).reshape(1, M, 3, 3)
    s.pbc = torch.ones(1, M, 3, dtype=torch.bool)
    s._dd_dummy = torch.zeros(1, dtype=torch.float64)
    return s


def run(hook, s, forces, stress):
    sim = SimpleNamespace(system=s, integrator=SimpleNamespace(time_step=DT), device=torch.device("cpu"),
                          dtype=torch.float64)
    hook.on_simulation_start(sim)
    for k in range(N_STEPS):
        hook.on_step_begin(sim)
        hook.propagate_half_step(s)                               # NPTVelocityVerlet.half_step
        hook.propagate_main_step(s)                               # NPTVelocityVerlet._main_step
        s.forces = torch.tensor(forces[k]).reshape(s.forces.shape)
        s.stress = torch.tensor(stress[k]).reshape(s.stress.shape)
        hook.propagate_half_step(s)
        hook.on_step_end(sim)


def main():
    baro, system_mod = load_reference_barostats()
    torch.symeig = _symeig
    masses, momenta, positions, cells, forces, stress, stress0 = inputs()
    out = {"n_atoms": np.array(N_ATOMS), "masses": masses, "momenta": momenta, "positions": positions, "cells": cells,
           "forces": forces, "stress": stress, "stress0": stress0, "time_step": DT, "temperature_bath": T_BATH,
           "time_constant_fs": TAU_FS, "target_pressure_bar": P_BAR, **UNITS}
    for name, kw in CASES.items():
        kw = dict(kw)
        cls = baro.NHCBarostatAnisotropic if kw.pop("anisotropic") else baro.NHCBarostatIsotropic
        hook = cls(P_BAR, T_BATH, TAU_FS, time_constant_cell=0.5 * TAU_FS, time_constant_barostat=2.0 * TAU_FS, **kw)
        s = make_system(system_mod, masses, momenta, positions, cells, stress0)
        run(hook, s, forces, stress)
        L = int(hook.chain_length)
        out[name + ":positions"] = s.positions[0].numpy().copy()
        out[name + ":momenta"] = s.momenta[0].numpy().copy()
        out[name + ":cells"] = s.cells[0].numpy().copy()
        for k in ("t_velocities", "t_forces", "t_masses", "t_velocities_cell", "t_forces_cell", "t_masses_cell"):
            out[name + ":" + k] = getattr(hook, k).numpy().reshape(-1, L)
        M = len(N_ATOMS)
        for k in ("b_velocities_cell", "b_forces_cell"):
            out[name + ":" + k] = getattr(hook, k).numpy().reshape(M, -1)
        out[name + ":b_masses_cell"] = hook.b_masses_cell.numpy().reshape(-1)
        moved = np.abs(out[name + ":cells"] - cells).max() / np.abs(cells).max()
        print(name, "relative cell change", moved)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays")


if __name__ == "__main__":
    main()
