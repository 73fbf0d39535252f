"""Generate tests/golden/md_thermostats.npz: the reference's own BerendsenThermostat, NHCThermostat and LangevinThermostat
(md/simulation_hooks/thermostats.py) applied to a reference ``System`` (md/system.py) that holds four molecules of 1, 3, 9
and 20 atoms, in fp64.

The reference's ``schnetpack.md`` needs ASE, omegaconf and the full ``schnetpack.units`` at import time; those modules are
stubbed here (the thermostats only read ``units.kB`` and ``units.fs``, which are the CODATA-2014 values restated in
``schnetpack_b200.md``).  ``System.load_molecules`` needs ASE Atoms, so the System's buffers are filled directly.

  * Berendsen and NHC (non-massive with Yoshida-Suzuki orders 3 and 5, massive with orders 3 and 7): momenta and chain
    state after N_APPLY applications (on_step_begin / on_step_end alternately, no dynamics in between);
  * Langevin: c1, c2 and thermostat_factor (its noise is torch.randn, which the device replaces by Philox).

Run from the repository root:  python tests/golden/make_golden_md_thermostats.py
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
from schnetpack_b200.md import FS_MD, KB_MD  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "md_thermostats.npz")
N_ATOMS = [1, 3, 9, 20]
DT = 0.5 * FS_MD
T_BATH = 300.0
TAU_FS = 100.0
N_APPLY = 8
NHC_CASES = {"nhc_o3": dict(massive=False, integration_order=3), "nhc_o5": dict(massive=False, integration_order=5),
             "nhc_massive_o3": dict(massive=True, integration_order=3),
             "nhc_massive_o7": dict(massive=True, integration_order=7, chain_length=4, multi_step=3)}


def _stub(name, path=None, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    if path:
        m.__path__ = [path]
    sys.modules[name] = m
    return m


def load_reference_md():
    spk = ref_loader.load()
    ref = ref_loader.REF
    _stub("omegaconf", DictConfig=dict, open_dict=None, OmegaConf=None)
    spk.units = _stub("schnetpack.units", kB=KB_MD, fs=FS_MD, unit2internal=lambda u: 1.0)
    md = _stub("schnetpack.md", ref + "/md")
    spk.md = md
    md.utils = importlib.import_module("schnetpack.md.utils")
    md.simulation_hooks = _stub("schnetpack.md.simulation_hooks", ref + "/md/simulation_hooks")
    th = importlib.import_module("schnetpack.md.simulation_hooks.thermostats")
    system = importlib.import_module("schnetpack.md.system")
    return th, system


def inputs(seed=5):
    rng = np.random.default_rng(seed)
    n = sum(N_ATOMS)
    masses = rng.choice([1.008, 12.011, 15.999, 32.06], size=n)
    # momenta around 150 .. 600 K per system, so the thermostats pull both ways
    t_sys = np.repeat(rng.uniform(150.0, 600.0, len(N_ATOMS)), N_ATOMS)
    momenta = rng.normal(size=(n, 3)) * np.sqrt(masses * KB_MD * t_sys)[:, None]
    return masses, momenta


def make_system(system_mod, masses, momenta):
    s = system_mod.System()
    n = sum(N_ATOMS)
    s.n_replicas, s.n_molecules, s.total_n_atoms = 1, len(N_ATOMS), n
    s.n_atoms = torch.tensor(N_ATOMS, dtype=torch.long)
    s.index_m = torch.repeat_interleave(torch.arange(len(N_ATOMS)), torch.tensor(N_ATOMS))
    s.atom_types = torch.ones(n, dtype=torch.long)
    s.masses = torch.tensor(masses, dtype=torch.float64).reshape(1, n, 1)
    s.positions = torch.zeros(1, n, 3, dtype=torch.float64)
    s.momenta = torch.tensor(momenta, dtype=torch.float64).reshape(1, n, 3)
    s.forces = torch.zeros(1, n, 3, dtype=torch.float64)
    s.energy = torch.zeros(1, len(N_ATOMS), 1, dtype=torch.float64)
    s.cells = torch.zeros(1, len(N_ATOMS), 3, 3, dtype=torch.float64)
    s.stress = torch.zeros(1, len(N_ATOMS), 3, 3, dtype=torch.float64)
    s.pbc = torch.zeros(1, len(N_ATOMS), 3, dtype=torch.bool)
    s._dd_dummy = torch.zeros(1, dtype=torch.float64)
    return s


def run(hook, system):
    sim = SimpleNamespace(system=system, integrator=SimpleNamespace(time_step=DT), device=torch.device("cpu"),
                          dtype=torch.float64)
    hook.on_simulation_start(sim)
    for k in range(N_APPLY):
        (hook.on_step_begin if k % 2 == 0 else hook.on_step_end)(sim)
    return system.momenta[0].numpy().copy()


def main():
    th, system_mod = load_reference_md()
    masses, momenta = inputs()
    out = {"n_atoms": np.array(N_ATOMS), "masses": masses, "momenta": momenta, "time_step": DT, "temperature_bath": T_BATH,
           "time_constant_fs": TAU_FS, "kB": KB_MD, "fs": FS_MD, "n_apply": N_APPLY}
    s = make_system(system_mod, masses, momenta)
    out["temperature"] = s.temperature.reshape(-1).numpy()
    out["berendsen:momenta"] = run(th.BerendsenThermostat(T_BATH, TAU_FS), s)
    for name, kw in NHC_CASES.items():
        hook = th.NHCThermostat(T_BATH, TAU_FS, **kw)
        s = make_system(system_mod, masses, momenta)
        out[name + ":momenta"] = run(hook, s)
        out[name + ":velocities"] = hook.velocities.numpy().reshape(-1, int(hook.chain_length))
        out[name + ":forces"] = hook.forces.numpy().reshape(-1, int(hook.chain_length))
        out[name + ":masses"] = hook.masses.numpy().reshape(-1, int(hook.chain_length))
    hook = th.LangevinThermostat(T_BATH, TAU_FS)
    s = make_system(system_mod, masses, momenta)
    hook.on_simulation_start(SimpleNamespace(system=s, integrator=SimpleNamespace(time_step=DT),
                                             device=torch.device("cpu"), dtype=torch.float64))
    out["langevin:c1"] = hook.c1.reshape(-1).numpy()
    out["langevin:c2"] = hook.c2.reshape(-1).numpy()
    out["langevin:thermostat_factor"] = hook.thermostat_factor.reshape(-1).numpy()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, sorted(out))


if __name__ == "__main__":
    main()
