"""CPU: the fp64 pair-energy restatement (tests/pair_energy_oracle.py), the unit conversion and the ATen training
formulas of the pair terms, held to the fixtures the unmodified reference produced (tests/golden/pair_energy_*.npz)."""
import os
import types

import numpy as np
import pytest
import torch

import pair_energy_oracle as PO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_case(case):
    z = np.load(os.path.join(GOLDEN, f"pair_energy_{case}.npz"))
    batch = {k[3:]: z[k] for k in z.files if k.startswith("in/")}
    weights = {k[2:]: z[k] for k in z.files if k.startswith("w/")}
    ref = {k: z[k] for k in z.files if not (k.startswith("in/") or k.startswith("w/"))}
    return batch, weights, ref


def package_mods():
    from schnetpack_b200 import atomistic as A
    from schnetpack_b200 import nn as snn
    from schnetpack_b200 import representation as Rp
    from schnetpack_b200.model import NeuralNetworkPotential

    return types.SimpleNamespace(
        PaiNN=Rp.PaiNN, GaussianRBF=snn.GaussianRBF, CosineCutoff=snn.CosineCutoff, SwitchFunction=snn.SwitchFunction,
        PairwiseDistances=A.PairwiseDistances, Strain=A.Strain, FilterShortRange=A.FilterShortRange,
        DipoleMoment=A.DipoleMoment, Atomwise=A.Atomwise, ZBLRepulsionEnergy=A.ZBLRepulsionEnergy,
        EnergyCoulomb=A.EnergyCoulomb, CoulombPotential=A.CoulombPotential,
        DampedCoulombPotential=A.DampedCoulombPotential, Aggregation=A.Aggregation, Forces=A.Forces,
        NeuralNetworkPotential=NeuralNetworkPotential)


def package_model(case, weights, dtype):
    model = PO.build_case(package_mods(), case)
    sd = model.state_dict()
    assert set(sd) == set(weights), set(sd) ^ set(weights)          # identical state_dict keys
    model.load_state_dict({k: torch.as_tensor(v).to(sd[k].dtype) for k, v in weights.items()})
    return model.to(dtype)


def torch_batch(batch, dtype, device="cpu"):
    return {k: (torch.as_tensor(v).to(dtype) if np.asarray(v).dtype.kind == "f" else torch.as_tensor(v)).to(device)
            for k, v in batch.items()}


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("case", PO.CASES)
def test_oracle_pair_energies_match_reference_fixtures(case):
    batch, w, ref = load_case(case)
    L = PO.LAYOUT[case]
    R = torch.as_tensor(batch["_positions"], dtype=torch.float64)
    ii, jj = torch.as_tensor(batch["_idx_i"]), torch.as_tensor(batch["_idx_j"])
    r = PO.rij(R, ii, jj, torch.as_tensor(batch["_offsets"], dtype=torch.float64))
    n_sys = len(batch["_n_atoms"])
    zp = [w[f"output_modules.2.{k}"] for k in ("a_pow", "a_div", "coefficients", "exponents")]
    e_z = PO.zbl_energy(batch["_atomic_numbers"], r, ii, jj, batch["_idx_m"], n_sys, zp, float(w["output_modules.2.ke"]),
                        cutoff=L["zbl_cut"], d_max=L["src"])
    shift = float(np.asarray(w["output_modules.3.shift"]).reshape(-1)[0]) if L["coul_cut"] is not None else None
    e_c = PO.coulomb_energy(torch.as_tensor(ref["fp64/partial_charges"]).reshape(-1), r, ii, jj, batch["_idx_m"], n_sys,
                            float(w["output_modules.3.ke"][0]), damped=L["damped"], cutoff=L["coul_cut"], shift=shift,
                            d_max=None if L["lr"] else L["src"])
    assert rel(e_z.numpy(), ref["fp64/e_zbl"]) <= 1e-11
    assert rel(e_c.numpy(), ref["fp64/e_coul"]) <= 1e-11
    assert float(w["output_modules.2.ke"]) == pytest.approx(PO.KE_KCAL_ANG, rel=1e-6)   # stored in fp32 by the reference


@pytest.mark.parametrize("case", PO.CASES)
def test_aten_training_path_matches_reference_fixtures(case):
    """train() mode runs the ATen formulas of functional_torch (FilterShortRange compacts exactly, as the reference)."""
    batch, w, ref = load_case(case)
    model = package_model(case, w, torch.float64)
    model.train()
    x = torch_batch(batch, torch.float64)
    out = dict(model(x))
    out.update({k: v for k, v in x.items() if k not in out})
    for k in ("energy", "e_zbl", "e_coul", "forces", "partial_charges", "dipole_moment") + (
            ("stress",) if PO.LAYOUT[case]["stress"] else ()):
        assert rel(out[k].detach().numpy(), ref["fp64/" + k]) <= 1e-10, k


def test_convert_units_known_values():
    from schnetpack_b200.units import convert_units

    assert convert_units("Ha", "kcal/mol") == pytest.approx(627.509474, rel=1e-9)
    assert convert_units("Ha", "kcal / mol") == convert_units("Ha", "kcal/mol")
    # ASE derives Bohr from the CODATA-2014 constants (0.52917721056...); CODATA's own value is 0.52917721067
    assert convert_units("Bohr", "Ang") == pytest.approx(0.52917721067, rel=1e-9)
    assert convert_units("Ha", "eV") == pytest.approx(27.21138602, rel=1e-9)
    assert convert_units("kcal/mol", "kJ/mol") == pytest.approx(4.184, rel=1e-15)
    assert convert_units("nm", "Angstrom") == 10.0
    assert convert_units(2.0, 4.0) == 0.5
    with pytest.raises(Warning, match="Ampere"):
        convert_units("A", "nm")


def test_short_range_cutoff_below_representation_cutoff_raises():
    from schnetpack_b200 import atomistic as A
    from schnetpack_b200 import nn as snn
    from schnetpack_b200 import representation as Rp
    from schnetpack_b200.model import NeuralNetworkPotential

    rep = Rp.PaiNN(16, 1, snn.GaussianRBF(5, 5.0), snn.CosineCutoff(5.0))
    with pytest.raises(ValueError, match="short_range_cutoff"):
        NeuralNetworkPotential(rep, [A.PairwiseDistances(), A.FilterShortRange(4.0)], [A.Atomwise(16, output_key="e")])


def test_scripting_a_pair_term_raises():
    from schnetpack_b200 import script

    _, w, _ = load_case("b")
    model = package_model("b", w, torch.float32).eval()
    with pytest.raises(NotImplementedError, match="DipoleMoment|ZBLRepulsionEnergy|EnergyCoulomb"):
        script.to_scriptable(model)
