"""Generate tests/golden/md_rpmd.npz: the reference's own ring-polymer MD -- RingPolymer (md/integrators.py:113-229),
NormalModeTransformer (md/utils/normal_model_transformation.py), PILELocalThermostat, PILEGlobalThermostat, TRPMDThermostat
and NHCRingPolymerThermostat local and global (md/simulation_hooks/thermostats_rpmd.py) -- driving a reference ``System``
(md/system.py) of three molecules of 1, 3 and 9 atoms with P = 1, 4, 5 and 8 beads, in fp64.

Stubs as in make_golden_md_barostats.py (``schnetpack.units`` with kB and fs, plus hbar, time and convert_units, which the
integrator reads; omegaconf), and an ``ase.units`` stub with fs (ASE is not needed otherwise).  Units are exact binary
fractions: kB = 2^-7, fs = 2^-10, hbar = 2^-4, time = 1, so dt = 1 fs = 2^-10 and omega_P = 37.5 P; at P = 8 the highest
normal-mode frequency gives omega dt = 0.59.  Forces come from a seeded harmonic tether per atom, F = -k (x - x0), evaluated
on every bead.  The thermostats' ``torch.randn_like`` draws are recorded, so the oracle can replay the same noise.

Each case runs on_simulation_start and N_STEPS of: on_step_begin, half_step, main_step, forces, half_step, on_step_end
(md/simulator.py:124-150).  Stored per P: C, omega_k and the propagator; per case: bead positions, momenta, the recorded noise
and, for NHC, the chain state.

Run from the repository root:  python tests/golden/make_golden_md_rpmd.py
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

OUT = os.path.join(ROOT, "tests", "golden", "md_rpmd.npz")
UNITS = dict(kB=2.0 ** -7, fs=2.0 ** -10, hbar=2.0 ** -4)
N_ATOMS = [1, 3, 9]
BEADS = [1, 4, 5, 8]
T_RP, T_BATH, TAU_FS, DT_FS = 300.0, 300.0, 64.0, 1.0
N_STEPS = 6
CASES = {"nve": None,
         "pile_l": ("PILELocalThermostat", dict(temperature_bath=T_BATH, time_constant=TAU_FS)),
         "pile_g": ("PILEGlobalThermostat", dict(temperature_bath=T_BATH, time_constant=TAU_FS)),
         "trpmd": ("TRPMDThermostat", dict(temperature_bath=T_BATH, damping_factor=0.5)),
         "nhc_local": ("NHCRingPolymerThermostat", dict(temperature_bath=T_BATH, time_constant=TAU_FS, local=True)),
         "nhc_global": ("NHCRingPolymerThermostat", dict(temperature_bath=T_BATH, time_constant=TAU_FS, local=False,
                                                         chain_length=4, integration_order=5))}


def _stub(name, path=None, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    if path:
        m.__path__ = [path]
    sys.modules[name] = m
    return m


def load_reference_rpmd():
    spk = ref_loader.load()
    ref = ref_loader.REF
    _stub("omegaconf", DictConfig=dict, open_dict=None, OmegaConf=None)
    ase = sys.modules.get("ase") or _stub("ase", Atoms=object)
    ase.units = _stub("ase.units", fs=UNITS["fs"])
    spk.units = _stub("schnetpack.units", unit2internal=lambda u: 1.0, time=1.0, convert_units=lambda a, b: a / b,
                      **UNITS)
    md = _stub("schnetpack.md", ref + "/md")
    spk.md = md
    md.utils = importlib.import_module("schnetpack.md.utils")
    hooks = _stub("schnetpack.md.simulation_hooks", ref + "/md/simulation_hooks")
    hooks.SimulationHook = importlib.import_module("schnetpack.md.simulation_hooks.basic_hooks").SimulationHook
    th = importlib.import_module("schnetpack.md.simulation_hooks.thermostats_rpmd")
    hooks.BarostatHook = importlib.import_module("schnetpack.md.simulation_hooks.barostats").BarostatHook
    system = importlib.import_module("schnetpack.md.system")
    md.System = system.System
    integrators = importlib.import_module("schnetpack.md.integrators")
    nmt = importlib.import_module("schnetpack.md.utils.normal_model_transformation")
    return th, system, integrators, nmt


def inputs(P, seed=19):
    rng = np.random.default_rng(seed + P)
    n = sum(N_ATOMS)
    masses = rng.choice([1.0, 2.0, 12.0, 16.0], size=n)
    x0 = rng.normal(size=(n, 3)) * 0.2
    k_tether = rng.uniform(0.5, 2.0, size=n) * 1e3
    x = x0[None] + rng.normal(size=(P, n, 3)) * 0.01
    p = rng.normal(size=(P, n, 3)) * np.sqrt(masses * UNITS["kB"] * 300.0 * P)[None, :, None]
    return masses, x0, k_tether, x, p


def make_system(system_mod, nmt, masses, x, p):
    P, n = x.shape[0], x.shape[1]
    s = system_mod.System()
    M = len(N_ATOMS)
    s.n_replicas, s.n_molecules, s.total_n_atoms = P, M, n
    s.nm_transform = nmt.NormalModeTransformer(P)
    s.n_atoms = torch.tensor(N_ATOMS, dtype=torch.long)
    s.index_m = torch.repeat_interleave(torch.arange(M), torch.tensor(N_ATOMS))
    s.atom_types = torch.ones(n, dtype=torch.long)
    s.masses = torch.tensor(masses, dtype=torch.float64).reshape(1, n, 1)
    s.positions = torch.tensor(x, dtype=torch.float64)
    s.momenta = torch.tensor(p, dtype=torch.float64)
    s.forces = torch.zeros(P, n, 3, dtype=torch.float64)
    s.energy = torch.zeros(P, M, 1, dtype=torch.float64)
    s.cells = torch.zeros(P, M, 3, 3, dtype=torch.float64)
    s.stress = torch.zeros(P, M, 3, 3, dtype=torch.float64)
    s.pbc = torch.zeros(P, M, 3, dtype=torch.bool)
    s._dd_dummy = torch.zeros(1, dtype=torch.float64)
    return s


def main():
    th, system_mod, integrators, nmt = load_reference_rpmd()
    recorded = []
    randn_like = torch.randn_like

    def recording_randn_like(x, *a, **kw):
        z = randn_like(x, *a, **kw)
        recorded.append(z.detach().clone())
        return z

    torch.randn_like = recording_randn_like
    torch.manual_seed(7)
    out = {"n_atoms": np.array(N_ATOMS), "beads": np.array(BEADS), "temperature": T_RP, "temperature_bath": T_BATH,
           "time_constant_fs": TAU_FS, "time_step_fs": DT_FS, "n_steps": N_STEPS, **UNITS}
    for P in BEADS:
        masses, x0, k_tether, x, p = inputs(P)
        pre = f"P{P}:"
        out.update({pre + "masses": masses, pre + "x0": x0, pre + "k_tether": k_tether, pre + "positions": x,
                    pre + "momenta": p, pre + "c_transform": nmt.NormalModeTransformer(P).c_transform.numpy()})
        for name, spec in CASES.items():
            integ = integrators.RingPolymer(DT_FS, P, T_RP)
            if name == "nve":
                out[pre + "omega_normal"] = integ.omega_normal.numpy().copy()
                out[pre + "propagator"] = integ.propagator[..., 0, 0].numpy().copy()
            s = make_system(system_mod, nmt, masses, x, p)
            x0t, kt = torch.tensor(x0)[None], torch.tensor(k_tether)[None, :, None]
            hook = None if spec is None else getattr(th, spec[0])(**spec[1])
            sim = SimpleNamespace(system=s, integrator=integ, device=torch.device("cpu"), dtype=torch.float64)
            if hook is not None:
                hook.on_simulation_start(sim)
            recorded.clear()
            s.forces = -kt * (s.positions - x0t)
            for _ in range(N_STEPS):
                if hook is not None:
                    hook.on_step_begin(sim)
                integ.half_step(s)
                integ.main_step(s)
                s.forces = -kt * (s.positions - x0t)
                integ.half_step(s)
                if hook is not None:
                    hook.on_step_end(sim)
            key = pre + name + ":"
            out[key + "positions"] = s.positions.numpy().copy()
            out[key + "momenta"] = s.momenta.numpy().copy()
            if recorded:
                out[key + "noise"] = torch.stack(recorded).numpy()
            if name.startswith("nhc"):
                L = int(hook.chain_length)
                for k in ("velocities", "forces", "masses"):
                    out[key + k] = getattr(hook, k).numpy().reshape(-1, L)
            assert np.isfinite(out[key + "momenta"]).all(), key
            print(key, "moved", float(np.abs(out[key + "positions"] - x).max()))
    torch.randn_like = randn_like
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays")


if __name__ == "__main__":
    main()
