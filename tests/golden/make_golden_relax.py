"""Generate tests/golden/relax_lbfgs.npz: the reference's own ASEBatchwiseLBFGS (interfaces/batchwise_optimization.py,
unmodified) relaxing batches of 6-atom Morse clusters, step by step.

The module imports ASE and two schnetpack modules at load time; they are stubbed here (the optimizer only needs ASE's
``Atoms`` container and ``Dynamics``' ``nsteps`` / ``max_steps`` bookkeeping).  The calculator is an analytic Morse
potential whose forces are rounded to float32-exact values, so the reference runs in fp64 on exactly the inputs the
device will see as float32 forces.  Per case and step the file holds the positions before and after the step, the forces,
the step direction ``p`` (after masking and capping), the newest ``rho`` per system and the converged mask.

Cases:
  * wrap:  memory = 4 over 40 steps, so the history ring wraps many times;
  * early: one configuration starts next to its minimum and converges early while the others continue;
  * fixed: a fixed_atoms_mask (atoms 0 and 7);
  * cap:   maxstep = 0.05 with damping = 0.7, so most steps are capped.

Run from the repository root:  python tests/golden/make_golden_relax.py
"""
import importlib.util
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "relax_lbfgs.npz")
N_ATOMS = 6
MORSE_D, MORSE_A, MORSE_R0 = 1.0, 1.5, 1.3


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


class Atoms:
    def __init__(self, positions=None, numbers=None):
        self.positions = np.array(positions, dtype=np.float64)
        self.numbers = np.array(numbers)
        self.pbc = np.zeros(3, dtype=bool)
        self.cell = np.zeros((3, 3))

    def get_positions(self):
        return self.positions.copy()

    def get_atomic_numbers(self):
        return self.numbers.copy()

    def __len__(self):
        return len(self.positions)


class Dynamics:
    def __init__(self, atoms, logfile=None, trajectory=None, append_trajectory=False, master=None):
        self.atoms = atoms
        self.logfile = None
        self.nsteps = 0
        self.max_steps = 100000000


def load_reference_lbfgs():
    _stub("ase", Atoms=Atoms)
    _stub("ase.optimize")
    _stub("ase.optimize.optimize", Dynamics=Dynamics)
    _stub("ase.parallel", world=types.SimpleNamespace(rank=0), barrier=lambda: None)
    _stub("ase.io", write=lambda *a, **k: None)
    _stub("schnetpack")
    _stub("schnetpack.units", convert_units=lambda a, b: 1.0)
    _stub("schnetpack.interfaces")
    _stub("schnetpack.interfaces.ase_interface", AtomsConverter=object)
    path = os.path.join(ref_loader.REF, "interfaces", "batchwise_optimization.py")
    spec = importlib.util.spec_from_file_location("schnetpack.interfaces.batchwise_optimization", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def morse_forces(r):
    """forces of one cluster, fp64 rounded to float32-exact values"""
    d = r[:, None, :] - r[None, :, :]
    dist = np.sqrt((d ** 2).sum(-1))
    np.fill_diagonal(dist, 1.0)
    e = np.exp(-MORSE_A * (dist - MORSE_R0))
    dE = 2.0 * MORSE_D * MORSE_A * (1.0 - e) * e                 # dE/d dist
    np.fill_diagonal(dE, 0.0)
    f = -(dE / dist)[:, :, None] * d
    return f.sum(1).astype(np.float32).astype(np.float64)


class MorseCalculator:
    def get_forces(self, atoms, fixed_atoms_mask=None):
        f = np.concatenate([morse_forces(a.get_positions()) for a in atoms])
        if fixed_atoms_mask is not None:
            f[fixed_atoms_mask] = 0.0
        return f


def start(rng, n_configs, noise):
    base = MORSE_R0 / np.sqrt(2.0) * np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1.0]])
    return [base + rng.normal(scale=noise[c], size=base.shape) for c in range(n_configs)]


CASES = {
    "wrap": dict(noise=[0.25, 0.3, 0.2], memory=4, maxstep=0.2, damping=1.0, alpha=70.0, fmax=1e-4, steps=40),
    "early": dict(noise=[0.01, 0.3, 0.25], memory=10, maxstep=0.2, damping=1.0, alpha=20.0, fmax=1e-3, steps=60),
    "fixed": dict(noise=[0.25, 0.2], memory=5, maxstep=0.2, damping=1.0, alpha=30.0, fmax=1e-4, steps=40,
                  fixed=[0, 7]),
    "cap": dict(noise=[0.3, 0.35], memory=6, maxstep=0.05, damping=0.7, alpha=10.0, fmax=1e-4, steps=30),
}


def run_case(mod, rng, c):
    configs = start(rng, len(c["noise"]), c["noise"])
    atoms = [Atoms(positions=r, numbers=np.full(N_ATOMS, 18)) for r in configs]
    calc = MorseCalculator()
    n = N_ATOMS * len(atoms)
    fixed = c.get("fixed")
    opt = mod.ASEBatchwiseLBFGS(calculator=calc, atoms=atoms, logfile=None, maxstep=c["maxstep"], memory=c["memory"],
                                damping=c["damping"], alpha=c["alpha"], fixed_atoms_mask=fixed)
    rec = {k: [] for k in ("pos_before", "forces", "p", "rho", "converged", "pos_after")}
    pos = lambda: np.concatenate([a.get_positions() for a in opt.atoms])  # noqa: E731
    gen = opt.irun(fmax=c["fmax"], steps=c["steps"])
    next(gen)                                                   # initial forces
    before, f = pos(), calc.get_forces(opt.atoms, fixed)
    converged = None
    for converged in gen:
        if opt.nsteps == len(rec["p"]):                          # the final yield: no step was taken
            break
        q = -f.reshape(len(atoms), -1, 3)
        rec["pos_before"].append(before)
        rec["forces"].append(f)
        rec["converged"].append((q ** 2).sum(-1).max(-1) < c["fmax"] ** 2)
        rec["p"].append(opt.p.reshape(n, 3).copy())
        rec["rho"].append(np.array([r[0, 0] for r in opt.rho[-1]]) if opt.rho else np.ones(len(atoms)))
        before, f = pos(), calc.get_forces(opt.atoms, fixed)
        rec["pos_after"].append(before)
    mask = np.zeros(n, dtype=bool)
    if fixed is not None:
        mask[fixed] = True
    out = {k: np.array(v) for k, v in rec.items()}
    out.update(memory=c["memory"], maxstep=c["maxstep"], damping=c["damping"], alpha=c["alpha"], fmax=c["fmax"],
               fixed=mask, n_atoms=np.full(len(atoms), N_ATOMS), nsteps=opt.nsteps, all_converged=bool(converged),
               final_forces=f)
    return out


def main():
    mod = load_reference_lbfgs()
    rng = np.random.default_rng(7)
    data = {}
    for name, c in CASES.items():
        out = run_case(mod, rng, c)
        print(name, "steps", out["nsteps"], "converged", out["all_converged"],
              "per-step converged", out["converged"].sum(0))
        data.update({f"{name}:{k}": v for k, v in out.items()})
    np.savez_compressed(OUT, **data)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
