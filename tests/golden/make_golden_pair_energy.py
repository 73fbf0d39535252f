"""Fixtures tests/golden/pair_energy_{a,b,c,d}.npz from the UNMODIFIED reference modules
(atomistic/nuclear_repulsion.py, atomistic/electrostatic.py, atomistic/distances.py, atomistic/aggregation.py,
nn/cutoff.py) on top of the reference hot path that ``oracle.ref_loader.load()`` imports.  ``ase.units`` is stubbed with
the CODATA-2014 unit table (as make_golden_md_gle.py stubs units), so ``schnetpack.units.convert_units`` computes what it
computes with ASE installed.

Cases (model layouts in tests/pair_energy_oracle.py):
  a  PhysNet-style aspirin x3 with total_charge (1, -1, 0): PaiNN, DipoleMoment(return_charges, correct_charges), Atomwise,
     ZBL with CosineCutoff, DampedCoulombPotential + cutoff on the long-range list, FilterShortRange, Aggregation, Forces
  b  plain Coulomb with use_neighbors_lr=False and ZBL without a cutoff
  c  periodic box (48 atoms) with a cutoff Coulomb term and stress (Strain + calc_stress)
  d  the gated (use_vector_representation) charge head
Each file holds the batch, the weights under their state_dict keys ("w/<key>"), and fp64 and fp32 outputs: energy, the
three energy terms, forces, charges, dipole (stress for c), plus the fp64 pair-term energies and forces at the fp64
model's charges held fixed.

Run: python tests/golden/make_golden_pair_energy.py   (needs the reference tree)"""
import importlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_loader as rl  # noqa: E402
from schnetpack_b200 import units as U  # noqa: E402

import pair_energy_oracle as PO  # noqa: E402


def load_reference_pair_modules():
    """Import the reference's units, nuclear_repulsion, electrostatic and aggregation modules (additive to
    ``ref_loader.load()``, whose imports are unchanged)."""
    spk = rl.load()
    ase = sys.modules["ase"]
    units = types.ModuleType("ase.units")
    units.__dict__.update({k: v for k, v in U._UNITS.items()})

    class Units(dict):
        def __getattr__(self, name):
            return self[name]

    units.Units = Units
    ase.units = units
    sys.modules["ase.units"] = units
    spk.units = importlib.import_module("schnetpack.units")
    ato = spk.atomistic
    for n in ("nuclear_repulsion", "electrostatic", "aggregation"):
        m = importlib.import_module("schnetpack.atomistic." + n)
        for k in getattr(m, "__all__", []):
            setattr(ato, k, getattr(m, k))
    ato.FilterShortRange = sys.modules["schnetpack.atomistic.distances"].FilterShortRange
    return spk


def reference_mods(spk):
    a, n = spk.atomistic, spk.nn
    return types.SimpleNamespace(
        PaiNN=spk.representation.PaiNN, GaussianRBF=n.GaussianRBF, CosineCutoff=n.CosineCutoff,
        SwitchFunction=n.SwitchFunction, PairwiseDistances=a.PairwiseDistances, Strain=a.Strain,
        FilterShortRange=a.FilterShortRange, DipoleMoment=a.DipoleMoment, Atomwise=a.Atomwise,
        ZBLRepulsionEnergy=a.ZBLRepulsionEnergy, EnergyCoulomb=a.EnergyCoulomb, CoulombPotential=a.CoulombPotential,
        DampedCoulombPotential=a.DampedCoulombPotential, Aggregation=a.Aggregation, Forces=a.Forces,
        NeuralNetworkPotential=spk.model.NeuralNetworkPotential)


def evaluate(model, batch, dtype):
    x = {k: (torch.as_tensor(v).to(dtype) if np.asarray(v).dtype.kind == "f" else torch.as_tensor(v))
         for k, v in batch.items()}
    out = dict(model(x))
    out.update({k: v for k, v in x.items() if k not in out})   # terms that are no model output stay in the batch dict
    keys = ["energy", "e_nn", "e_zbl", "e_coul", "forces", "partial_charges", "dipole_moment"]
    if "stress" in out:
        keys.append("stress")
    return {k: out[k].detach().double().numpy() for k in keys}


def main():
    spk = load_reference_pair_modules()
    mods = reference_mods(spk)
    for case in PO.CASES:
        torch.manual_seed(100 + ord(case))
        model = PO.build_case(mods, case)
        with torch.no_grad():                      # visible biases, so that no weight is a trivial zero
            for name, p in model.named_parameters():
                if name.endswith("bias"):
                    p.uniform_(-0.1, 0.1)
        model.eval()
        batch = PO.case_batch(case)
        out64 = evaluate(model.double(), batch, torch.float64)
        sd = {k: v.detach().numpy() for k, v in model.state_dict().items()}
        out32 = evaluate(model.float(), batch, torch.float32)
        e_z, e_c, f_pair = PO.pair_terms_fixed_q(case, batch, sd, out64["partial_charges"])
        blob = {f"in/{k}": np.asarray(v) for k, v in batch.items()}
        blob.update({f"w/{k}": v for k, v in sd.items()})
        blob.update({f"fp64/{k}": v for k, v in out64.items()})
        blob.update({f"fp32/{k}": v for k, v in out32.items()})
        blob.update({"pair/e_zbl": e_z.numpy(), "pair/e_coul": e_c.numpy(), "pair/forces": f_pair.numpy()})
        path = os.path.join(HERE, f"pair_energy_{case}.npz")
        np.savez_compressed(path, **blob)
        print(case, path, {k: float(np.abs(v).max()) for k, v in out64.items()})


if __name__ == "__main__":
    main()
