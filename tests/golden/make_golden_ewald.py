"""Fixtures tests/golden/ewald_{e1,e2}.npz from the UNMODIFIED reference modules (atomistic/electrostatic.py
EnergyEwald, atomistic/distances.py, atomistic/aggregation.py, nn/cutoff.py) on top of the reference hot path, loaded as
make_golden_pair_energy.py loads them.

Cases (model layouts in tests/ewald_oracle.py):
  e1  48-atom water box: PaiNN, DipoleMoment(return_charges, correct_charges), Atomwise, EnergyEwald with a
      SwitchFunction screen on the long-range list, FilterShortRange, Aggregation, Forces with stress
  e2  three triclinic cells of different sizes and atom counts, one of them with total charge 1: EnergyEwald without a
      screen on the standard list, Forces with stress
Each file holds the batch, the weights under their state_dict keys ("w/<key>"), and fp64 and fp32 outputs: energy, the
two energy terms, forces, charges, dipole and stress, the fp64 Ewald energy and forces at the fp64 model's charges held
fixed, and the fp64 weight gradients of a force loss in train() mode ("grad/<parameter name>").

Run: python tests/golden/make_golden_ewald.py   (needs the reference tree)"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import ewald_oracle as EO  # noqa: E402
from make_golden_pair_energy import load_reference_pair_modules  # noqa: E402


def reference_mods(spk):
    a, n = spk.atomistic, spk.nn
    return types.SimpleNamespace(
        PaiNN=spk.representation.PaiNN, GaussianRBF=n.GaussianRBF, CosineCutoff=n.CosineCutoff,
        SwitchFunction=n.SwitchFunction, PairwiseDistances=a.PairwiseDistances, Strain=a.Strain,
        FilterShortRange=a.FilterShortRange, DipoleMoment=a.DipoleMoment, Atomwise=a.Atomwise,
        EnergyEwald=a.EnergyEwald, Aggregation=a.Aggregation, Forces=a.Forces,
        NeuralNetworkPotential=spk.model.NeuralNetworkPotential)


def evaluate(model, batch, dtype):
    x = {k: (torch.as_tensor(v).to(dtype) if np.asarray(v).dtype.kind == "f" else torch.as_tensor(v))
         for k, v in batch.items()}
    out = dict(model(x))
    out.update({k: v for k, v in x.items() if k not in out})
    keys = ["energy", "e_nn", "e_ewald", "forces", "partial_charges", "dipole_moment", "stress"]
    return {k: out[k].detach().double().numpy() for k in keys}


def force_loss_weight_grads(model, batch):
    """fp64 gradients of FORCE_LOSS with respect to every weight, in train() mode (Forces differentiates with
    create_graph), so the force term's double backward is part of them."""
    model.train()
    x = {k: (torch.as_tensor(v).to(torch.float64) if np.asarray(v).dtype.kind == "f" else torch.as_tensor(v))
         for k, v in batch.items()}
    out = model(x)
    params = [(k, p) for k, p in model.named_parameters() if p.requires_grad]
    g = torch.autograd.grad(EO.force_loss(out), [p for _, p in params], allow_unused=True)
    return {k: v.detach().numpy() for (k, _), v in zip(params, g) if v is not None}


def main():
    spk = load_reference_pair_modules()
    mods = reference_mods(spk)
    for case in EO.CASES:
        torch.manual_seed(200 + int(case[1:]))
        model = EO.build_case(mods, case)
        with torch.no_grad():                      # visible biases, so that no weight is a trivial zero
            for name, p in model.named_parameters():
                if name.endswith("bias"):
                    p.uniform_(-0.1, 0.1)
        model.eval()
        batch = EO.case_batch(case)
        out64 = evaluate(model.double(), batch, torch.float64)
        grads = force_loss_weight_grads(model, batch)
        model.eval()
        sd = {k: v.detach().numpy() for k, v in model.state_dict().items()}
        out32 = evaluate(model.float(), batch, torch.float32)
        e_ew, f_ew = EO.ewald_fixed_q(case, batch, out64["partial_charges"])
        blob = {f"in/{k}": np.asarray(v) for k, v in batch.items()}
        blob.update({f"w/{k}": v for k, v in sd.items()})
        blob.update({f"fp64/{k}": v for k, v in out64.items()})
        blob.update({f"fp32/{k}": v for k, v in out32.items()})
        blob.update({"ewald/energy": e_ew.numpy(), "ewald/forces": f_ew.numpy()})
        blob.update({f"grad/{k}": v for k, v in grads.items()})
        path = os.path.join(HERE, f"ewald_{case}.npz")
        np.savez_compressed(path, **blob)
        print(case, path, {k: float(np.abs(v).max()) for k, v in out64.items()})


if __name__ == "__main__":
    main()
