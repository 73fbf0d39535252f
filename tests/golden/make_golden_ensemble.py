"""Generate tests/golden/ensemble_batch.npz: the reference's own ensemble statistics on the predictions of a mixed ensemble.

Members: three PaiNN models (seeds 1, 2, 3) and one SchNet model (seed 4), the reference's NeuralNetworkPotential built by
``oracle.ref_loader.build_from_spec`` and run in fp64.  Batch: aspirin x 3, a periodic 216-atom box and a single atom.

Reference code run here, unmodified, loaded from its files:
  * EnsembleCalculator._accumulate_results (md/calculators/ensemble_calculator.py) on the members' outputs;
  * NNEnsemble (interfaces/batchwise_optimization.py) on the batch;
  * AbsoluteUncertainty / RelativeUncertainty (interfaces/ase_interface.py) one structure at a time, for several weight
    sets, on the members' energies and forces and on a seeded [K, B, 3, 3] stress stack.
These modules import ASE and half of the package at load time; the missing modules are stubs whose attributes are
placeholder classes (a PEP 562 module ``__getattr__``), and ``MDCalculator`` is ``object``.

Run from the repository root:  python tests/golden/make_golden_ensemble.py
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ensemble_batch.npz")
MEMBERS = [("painn", 1), ("painn", 2), ("painn", 3), ("schnet", 4)]
WEIGHTS = [(0.0, 1.0, 0.0), (1.0, 1.0, 0.0), (1.0, 2.0, 0.5), (1.0, 0.0, 0.0), (0.0, 0.0, 1.0), (0.3, 0.0, 0.7)]


def member_spec(kind):
    return S.model_spec(kind, n_atom_basis=32, n_interactions=2)


def batch():
    """aspirin x 3, a periodic 216-atom box and one atom, collated in that order"""
    parts = [S.aspirin_batch(3, seed=1), S.periodic_box(216, seed=2),
             S._collate([S._open_system(np.array([8]), np.zeros((1, 3)), 5.0)])]
    out, base, n_sys = {}, 0, 0
    for p in parts:
        n = p[S.Z].shape[0]
        q = dict(p)
        q[S.idx_i], q[S.idx_j] = p[S.idx_i] + base, p[S.idx_j] + base
        q[S.idx_m] = p[S.idx_m] + n_sys
        q[S.cell] = p[S.cell].reshape(-1, 3, 3)
        q[S.pbc] = p[S.pbc].reshape(-1)
        for k, v in q.items():
            out.setdefault(k, []).append(v)
        base += n
        n_sys += p[S.n_atoms].shape[0]
    return {k: np.concatenate(v) for k, v in out.items()}


class _Placeholders(types.ModuleType):
    def __getattr__(self, name):                 # PEP 562: any name the module imports is a placeholder class
        if name.startswith("__"):
            raise AttributeError(name)
        return type(name, (), {})


def _stub(name, path=None, **attrs):
    m = sys.modules.get(name)
    if m is None or not isinstance(m, _Placeholders):
        m = _Placeholders(name)
        if name in sys.modules:                  # keep what ref_loader registered (e.g. schnetpack.properties)
            m.__dict__.update({k: v for k, v in sys.modules[name].__dict__.items() if not k.startswith("__")})
        sys.modules[name] = m
    m.__dict__.update(attrs)
    if path:
        m.__path__ = [path]
    return m


def load_reference_ensemble():
    ref = ref_loader.REF
    for n in ["ase", "ase.constraints", "ase.calculators", "ase.calculators.calculator", "ase.io", "ase.io.trajectory",
              "ase.md", "ase.md.velocitydistribution", "ase.optimize", "ase.optimize.optimize", "ase.vibrations",
              "ase.parallel", "schnetpack.data", "schnetpack.data.loader", "schnetpack.transform",
              "schnetpack.units", "schnetpack.md", "schnetpack.md.utils", "schnetpack.interfaces"]:
        _stub(n)
    _stub("ase.calculators.calculator", all_changes=[])
    _stub("schnetpack.md.calculators", MDCalculator=object)

    def load(name, rel):
        spec = importlib.util.spec_from_file_location(name, os.path.join(ref, rel))
        m = importlib.util.module_from_spec(spec)
        sys.modules[name] = m
        spec.loader.exec_module(m)
        return m

    ai = load("schnetpack.interfaces.ase_interface", "interfaces/ase_interface.py")
    sys.modules["schnetpack.interfaces"].ase_interface = ai
    ec = load("schnetpack.md.calculators.ensemble_calculator", "md/calculators/ensemble_calculator.py")
    bo = load("schnetpack.interfaces.batchwise_optimization", "interfaces/batchwise_optimization.py")
    return ec.EnsembleCalculator, bo.NNEnsemble, ai.AbsoluteUncertainty, ai.RelativeUncertainty


def main():
    data = batch()
    models = [ref_loader.build_from_spec(member_spec(kind), S.init_params(member_spec(kind), seed=seed),
                                         dtype=torch.float64) for kind, seed in MEMBERS]
    preds = [ref_loader.evaluate(m, data, dtype=torch.float64) for m in models]
    EnsembleCalculator, NNEnsemble, Absolute, Relative = load_reference_ensemble()

    acc = EnsembleCalculator._accumulate_results([{k: p[k] for k in ("energy", "forces")} for p in preds])
    x = {k: torch.as_tensor(v) for k, v in data.items()}
    x = {k: (v.to(torch.float64) if v.is_floating_point() else v) for k, v in x.items()}
    means, stds = NNEnsemble(torch.nn.ModuleList(models), ["energy", "forces"])(x)

    K = len(models)
    energy = np.stack([p["energy"].numpy() for p in preds])                    # [K, B]
    forces = np.stack([p["forces"].numpy() for p in preds])                    # [K, N, 3]
    n_atoms = data[S.n_atoms]
    B = n_atoms.shape[0]
    stress = np.random.default_rng(7).normal(size=(K, B, 3, 3)) * np.array([1.0, 0.1, 3.0])[None, None, :, None]
    ptr = np.concatenate([[0], np.cumsum(n_atoms)])
    unc = np.zeros((2, len(WEIGHTS), B))
    for r, cls in enumerate((Absolute, Relative)):
        for w, (we, wf, ws) in enumerate(WEIGHTS):
            fn = cls(energy_weight=we, force_weight=wf, stress_weight=ws)
            for b in range(B):                   # the ASE calculator's view: one structure at a time
                pred = {"energy": [energy[k, b] for k in range(K)],
                        "forces": [forces[k, ptr[b]:ptr[b + 1]] for k in range(K)],
                        "stress": [stress[k, b] for k in range(K)]}
                unc[r, w, b] = fn(pred)
    out = {"members_json": json.dumps([[member_spec(kind), seed] for kind, seed in MEMBERS]),
           "weights": np.array(WEIGHTS), "pred:energy": energy, "pred:forces": forces, "pred:stress": stress,
           "acc:energy": acc["energy"].numpy(), "acc:energy_var": acc["energy_var"].numpy(),
           "acc:forces": acc["forces"].numpy(), "acc:forces_var": acc["forces_var"].numpy(),
           "nn:mean:energy": means["energy"].detach().numpy(), "nn:std:energy": stds["energy"].detach().numpy(),
           "nn:mean:forces": means["forces"].detach().numpy(), "nn:std:forces": stds["forces"].detach().numpy(),
           "unc:absolute": unc[0], "unc:relative": unc[1]}
    out.update({"in:" + k: v for k, v in data.items()})
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, {k: v.shape for k, v in out.items() if hasattr(v, "shape")})


if __name__ == "__main__":
    main()
