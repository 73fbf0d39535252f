"""Generate tests/golden/md_rpmd_npt.npz: the reference's own ring-polymer NPT -- PILEBarostat
(md/simulation_hooks/barostats_rpmd.py) with the NPTRingPolymer integrator (md/integrators.py:266-305), alone and next to
each ring-polymer thermostat of md/simulation_hooks/thermostats_rpmd.py -- driving a reference ``System`` (md/system.py) of
three periodic molecules of 1, 3 and 9 atoms, each in its own cell (the third triclinic), with P = 1, 4, 5 and 8 beads, in
fp64.

The stubs are those of make_golden_md_rpmd.py, with ``bar`` added to the ``schnetpack.units`` stub.  Units stay exact binary
fractions: kB = 2^-7, fs = 2^-10, hbar = 2^-4, bar = 2^-4, time = 1, so the float32 buffers of the barostat (target pressure,
temperature, time constant, frequency, kB T, cell masses) hold their values exactly.  Forces come from a seeded harmonic
tether per atom, F = -k (x - x0), on every bead; the cell's time constant of 1024 fs keeps the volume change of six steps
at 1-6 %; each bead system's stress is the tether virial over its volume,
sum_a k (x_a - x0_a) (x) x_a / V, recomputed after every force evaluation.  Every ``torch.randn_like`` draw is recorded:
thermostat draws are [P, N, 3], barostat draws [n_molecules].

Each case runs on_simulation_start and N_STEPS of md/simulator.py:124-150 with the hooks [thermostat, barostat]:
on_step_begin in that order, half_step, main_step, forces + stress, half_step, on_step_end in reverse order.  Stored per
P: the inputs; per case: bead positions, momenta, cells, cell momenta and the recorded noise.

Run from the repository root:  python tests/golden/make_golden_md_rpmd_npt.py
"""
import importlib
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden_md_rpmd as G  # noqa: E402

OUT = os.path.join(HERE, "md_rpmd_npt.npz")
BAR = 2.0 ** -4
N_ATOMS = G.N_ATOMS
BEADS = [1, 4, 5, 8]
T_RP, T_BATH, TAU_FS, DT_FS = 300.0, 300.0, 64.0, 1.0
P_TARGET_BAR, T_CELL, TAU_CELL_FS = 1000.0, 300.0, 1024.0
N_STEPS = 6
CASES = {"none": None, **{k: v for k, v in G.CASES.items() if k != "nve"}}


def cells():
    """one cell per molecule: two orthorhombic, one triclinic"""
    return np.stack([np.diag([1.5, 1.75, 2.0]), np.diag([1.25, 1.25, 1.5]),
                     np.array([[2.0, 0.0, 0.0], [0.5, 1.75, 0.0], [0.25, -0.375, 1.5]])])


def tether(system, x0, k):
    """forces [P, N, 3] and the stress [P, M, 3, 3] of every bead system: sum_a k (x - x0) (x) x / V"""
    x = system.positions
    f = -k * (x - x0)
    w = (-f)[..., :, None] * x[..., None, :]                             # [P, N, 3, 3]
    vir = system.sum_atoms(w.reshape(*w.shape[:2], 9)).reshape(x.shape[0], -1, 3, 3)
    return f, vir / system.volume[..., None]


def main():
    th, system_mod, integrators, nmt = G.load_reference_rpmd()
    sys.modules["schnetpack.units"].bar = BAR
    baro_mod = importlib.import_module("schnetpack.md.simulation_hooks.barostats_rpmd")
    recorded = []
    randn_like = torch.randn_like

    def recording_randn_like(x, *a, **kw):
        z = randn_like(x, *a, **kw)
        recorded.append(z.detach().clone())
        return z

    torch.randn_like = recording_randn_like
    torch.manual_seed(11)
    c0 = cells()
    out = {"n_atoms": np.array(N_ATOMS), "beads": np.array(BEADS), "temperature": T_RP, "temperature_bath": T_BATH,
           "time_constant_fs": TAU_FS, "time_step_fs": DT_FS, "n_steps": N_STEPS, "target_pressure_bar": P_TARGET_BAR,
           "temperature_cell": T_CELL, "time_constant_cell_fs": TAU_CELL_FS, "cells": c0, "bar": BAR, **G.UNITS}
    M = len(N_ATOMS)
    for P in BEADS:
        masses, x0, k_tether, x, p = G.inputs(P)
        pre = f"P{P}:"
        out.update({pre + "masses": masses, pre + "x0": x0, pre + "k_tether": k_tether, pre + "positions": x,
                    pre + "momenta": p})
        for name, spec in CASES.items():
            baro = baro_mod.PILEBarostat(P_TARGET_BAR, T_CELL, TAU_CELL_FS)
            integ = integrators.NPTRingPolymer(DT_FS, P, T_RP, baro)
            s = G.make_system(system_mod, nmt, masses, x, p)
            s.cells = torch.tensor(np.repeat(c0[None], P, axis=0), dtype=torch.float64)
            s.pbc = torch.ones(P, M, 3, dtype=torch.bool)
            x0t, kt = torch.tensor(x0)[None], torch.tensor(k_tether)[None, :, None]
            thermo = None if spec is None else getattr(th, spec[0])(**spec[1])
            hooks = [h for h in (thermo, baro) if h is not None]
            sim = SimpleNamespace(system=s, integrator=integ, device=torch.device("cpu"), dtype=torch.float64)
            for h in hooks:
                h.on_simulation_start(sim)
            recorded.clear()
            s.forces, s.stress = tether(s, x0t, kt)
            for _ in range(N_STEPS):
                for h in hooks:
                    h.on_step_begin(sim)
                integ.half_step(s)
                integ.main_step(s)
                s.forces, s.stress = tether(s, x0t, kt)
                integ.half_step(s)
                for h in reversed(hooks):
                    h.on_step_end(sim)
            key = pre + name + ":"
            out[key + "positions"] = s.positions.numpy().copy()
            out[key + "momenta"] = s.momenta.numpy().copy()
            out[key + "cells"] = s.cells.numpy().copy()
            out[key + "cell_momenta"] = baro.cell_momenta.numpy().copy()
            out[key + "baro_noise"] = torch.stack([z for z in recorded if z.dim() == 1]).numpy()
            thermo_noise = [z for z in recorded if z.dim() == 3]
            if thermo_noise:
                out[key + "noise"] = torch.stack(thermo_noise).numpy()
            if pre + "cell_mass" not in out:
                out[pre + "cell_mass"] = baro.mass.numpy().copy()
                out[pre + "c2"] = baro.c2.numpy().copy()
            assert np.isfinite(out[key + "momenta"]).all(), key
            dv = np.abs(np.linalg.det(out[key + "cells"][0]) / np.linalg.det(c0) - 1.0).max()
            print(key, "moved", float(np.abs(out[key + "positions"] - x).max()), "volume", float(dv))
    torch.randn_like = randn_like
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays")


if __name__ == "__main__":
    main()
