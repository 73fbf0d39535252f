"""Generate tests/golden/md_gle.npz and the gle4md-format matrix files tests/golden/gle_*.txt: the reference's own
GLEThermostat (md/simulation_hooks/thermostats.py:527-730), RPMDGLEThermostat and PIGLETThermostat
(thermostats_rpmd.py:237-370), with their matrix parser (md/utils/thermostat_utils.py:64-178), driving the fp64 reference
``System`` of make_golden_md_rpmd.py (three molecules of 1, 3 and 9 atoms, harmonic tether per atom).

No published gle4md file is at hand, so the matrices are synthetic but valid GLEs: A = S + K with S symmetric positive
definite and K antisymmetric (positive-stable and, for K != 0, non-normal), and a non-canonical C solves the Lyapunov
equation A C + C A^T = B B^T for a random full-rank B.  Files:
  * gle_sym.txt          D = 3, symmetric A in femtoseconds^-1, no C;
  * gle_nonnormal.txt    D = 5, non-normal A in picoseconds^-1, no C (canonical: C = kB T I);
  * gle_quantum.txt      D = 5, non-normal A in femtoseconds^-1, C in K, hotter than the bath on p;
  * gle_piglet_p4.txt    P = 4 blocks of D = 4, A in atomic time units^-1, C in eV.

Units are the exact binary fractions of make_golden_md_rpmd.py (kB = 2^-7, fs = 2^-10, hbar = 2^-4); the
``schnetpack.units`` stub converts the gle4md units with the CODATA-2014 constants (eV and Hartree through kelvin, the
atomic unit of time through fs), as ``schnetpack_b200.md.load_gle_matrices`` does.  The thermostats' ``torch.randn`` (the
free-particle-limit start) and ``torch.randn_like`` draws are recorded, so the oracle can replay the same noise.

Run from the repository root:  python tests/golden/make_golden_md_gle.py
"""
import importlib
import os
import sys
import types
from types import SimpleNamespace

import numpy as np
import scipy.linalg as SL
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden_md_rpmd as MR  # noqa: E402
from gle_oracle import write_gle_file  # noqa: E402
from oracle import ref_loader  # noqa: E402

OUT = os.path.join(HERE, "md_gle.npz")
UNITS = MR.UNITS
# CODATA 2014: k_B, e, Hartree energy in J, atomic unit of time in s
K_B, E_CHARGE, HARTREE, AUT = 1.38064852e-23, 1.6021766208e-19, 4.359744650e-18, 2.418884326509e-17
INTERNAL = {"fs": UNITS["fs"], "s": 1e15 * UNITS["fs"], "aut": AUT * 1e15 * UNITS["fs"],
            "eV": E_CHARGE / K_B * UNITS["kB"], "Ha": HARTREE / K_B * UNITS["kB"]}
T_BATH, DT_FS, N_STEPS = 300.0, 1.0, 6
FILES = {"sym": "gle_sym.txt", "nonnormal": "gle_nonnormal.txt", "quantum": "gle_quantum.txt",
         "piglet": "gle_piglet_p4.txt"}
# (case, file, thermostat class, P, keywords)
CASES = [("gle_sym", "sym", "GLEThermostat", 1, {}),
         ("gle_nonnormal", "nonnormal", "GLEThermostat", 1, {}),
         ("gle_quantum", "quantum", "GLEThermostat", 1, {}),
         ("gle_zero_start", "nonnormal", "GLEThermostat", 1, dict(free_particle_limit=False)),
         ("rpmd_gle_nonnormal", "nonnormal", "RPMDGLEThermostat", 4, {}),
         ("rpmd_gle_quantum", "quantum", "RPMDGLEThermostat", 5, {}),
         ("piglet", "piglet", "PIGLETThermostat", 4, {})]


def synthetic_a(rng, D, scale, antisym=1.0):
    """S + K: S symmetric with eigenvalues in scale x [0.2, 3], K antisymmetric of size ~ scale x antisym"""
    Q, _ = np.linalg.qr(rng.normal(size=(D, D)))
    S = Q @ np.diag(scale * rng.uniform(0.2, 3.0, D)) @ Q.T
    K = rng.normal(size=(D, D)) * scale * antisym
    return 0.5 * (S + S.T) + 0.5 * (K - K.T)


def lyapunov_c(rng, A, c00):
    """C with A C + C A^T = B B^T for a random full-rank B, scaled to C[0, 0] = c00"""
    D = A.shape[0]
    B = rng.normal(size=(D, D))
    C = SL.solve_continuous_lyapunov(A, B @ B.T)
    C = 0.5 * (C + C.T)
    return C * (c00 / C[0, 0])


def write_files():
    rng = np.random.default_rng(2024)
    kT_eV = T_BATH * K_B / E_CHARGE
    write_gle_file(os.path.join(HERE, FILES["sym"]), synthetic_a(rng, 3, 0.1, antisym=0.0)[None])
    write_gle_file(os.path.join(HERE, FILES["nonnormal"]), 1e3 * synthetic_a(rng, 5, 0.1)[None], a_unit="picoseconds^-1")
    A = synthetic_a(rng, 5, 0.1)
    write_gle_file(os.path.join(HERE, FILES["quantum"]), A[None], lyapunov_c(rng, A, 1.4 * T_BATH)[None])
    As, Cs = [], []
    for k in range(4):
        A = synthetic_a(rng, 4, 0.1)
        As.append(A * AUT * 1e15)                                  # fs^-1 -> atomic time units^-1
        Cs.append(lyapunov_c(rng, A, 4 * kT_eV * (1.0 + 0.3 * k)))
    write_gle_file(os.path.join(HERE, FILES["piglet"]), np.stack(As), np.stack(Cs), a_unit="atomic time units^-1",
                   c_unit="eV")


def _stub(name, path=None, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    if path:
        m.__path__ = [path]
    sys.modules[name] = m
    return m


def load_reference_gle():
    spk = ref_loader.load()
    ref = ref_loader.REF
    _stub("omegaconf", DictConfig=dict, open_dict=None, OmegaConf=None)
    ase = sys.modules.get("ase") or _stub("ase", Atoms=object)
    ase.units = _stub("ase.units", fs=UNITS["fs"])
    spk.units = _stub("schnetpack.units", unit2internal=lambda u: INTERNAL.get(u, 1.0), time=1.0,
                      convert_units=lambda a, b: a / b, **UNITS)
    md = _stub("schnetpack.md", ref + "/md")
    spk.md = md
    md.utils = importlib.import_module("schnetpack.md.utils")
    hooks = _stub("schnetpack.md.simulation_hooks", ref + "/md/simulation_hooks")
    hooks.SimulationHook = importlib.import_module("schnetpack.md.simulation_hooks.basic_hooks").SimulationHook
    th = importlib.import_module("schnetpack.md.simulation_hooks.thermostats")
    th_rp = importlib.import_module("schnetpack.md.simulation_hooks.thermostats_rpmd")
    hooks.BarostatHook = importlib.import_module("schnetpack.md.simulation_hooks.barostats").BarostatHook
    system = importlib.import_module("schnetpack.md.system")
    md.System = system.System
    integrators = importlib.import_module("schnetpack.md.integrators")
    nmt = importlib.import_module("schnetpack.md.utils.normal_model_transformation")
    return th, th_rp, system, integrators, nmt, md.utils


def main():
    write_files()
    th, th_rp, system_mod, integrators, nmt, utils = load_reference_gle()
    recorded = []
    randn, randn_like = torch.randn, torch.randn_like

    def recording(fn):
        def draw(*a, **kw):
            z = fn(*a, **kw)
            recorded.append(z.detach().clone())
            return z
        return draw

    torch.randn, torch.randn_like = recording(randn), recording(randn_like)
    torch.manual_seed(11)
    out = {"n_atoms": np.array(MR.N_ATOMS), "temperature_bath": T_BATH, "time_step_fs": DT_FS, "n_steps": N_STEPS,
           **UNITS}
    for key, fname in FILES.items():
        a, c = utils.load_gle_matrices(os.path.join(HERE, fname))
        out[f"file:{key}:A"] = a
        if c is not None:
            out[f"file:{key}:C"] = c
    for name, fkey, cls, P, kw in CASES:
        masses, x0, k_tether, x, p = MR.inputs(P, seed=29)
        pre = name + ":"
        out.update({pre + "P": P, pre + "file": fkey, pre + "masses": masses, pre + "x0": x0, pre + "k_tether": k_tether,
                    pre + "positions": x, pre + "momenta": p})
        mod = th if cls == "GLEThermostat" else th_rp
        integ = integrators.VelocityVerlet(DT_FS) if P == 1 and cls == "GLEThermostat" else \
            integrators.RingPolymer(DT_FS, P, T_BATH)
        s = MR.make_system(system_mod, nmt, masses, x, p)
        hook = getattr(mod, cls)(temperature_bath=T_BATH, gle_file=os.path.join(HERE, FILES[fkey]), **kw)
        sim = SimpleNamespace(system=s, integrator=integ, device=torch.device("cpu"), dtype=torch.float64)
        recorded.clear()
        hook.on_simulation_start(sim)
        out[pre + "c1"] = hook.c1.numpy().copy()
        out[pre + "c2"] = hook.c2.numpy().copy()
        x0t, kt = torch.tensor(x0)[None], torch.tensor(k_tether)[None, :, None]
        s.forces = -kt * (s.positions - x0t)
        for _ in range(N_STEPS):
            hook.on_step_begin(sim)
            integ.half_step(s)
            integ.main_step(s)
            s.forces = -kt * (s.positions - x0t)
            integ.half_step(s)
            hook.on_step_end(sim)
        out[pre + "out_positions"] = s.positions.numpy().copy()
        out[pre + "out_momenta"] = s.momenta.numpy().copy()
        out[pre + "state"] = hook.thermostat_momenta.numpy().copy()
        out[pre + "noise"] = torch.stack(recorded).numpy()
        out[pre + "initial_draw"] = int(bool(kw.get("free_particle_limit", True)))
        assert np.isfinite(out[pre + "out_momenta"]).all(), name
        print(name, "draws", len(recorded), "moved p", float(np.abs(out[pre + "out_momenta"] - p).max()))
    torch.randn, torch.randn_like = randn, randn_like
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays")


if __name__ == "__main__":
    main()
