"""CPU: the fp64 Ewald restatement (tests/ewald_oracle.py) against the fixtures the unmodified reference produced
(tests/golden/ewald_*.npz), its analytic reverse against autograd and finite differences, Madelung constants, the ATen
training formula and ``convert_model`` on a live reference EnergyEwald."""
import math
import os
import types

import numpy as np
import pytest
import torch

import ewald_oracle as EO

from oracle import nl_oracle
from oracle import ref_loader as rl

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
needs_ref = pytest.mark.skipif(not rl.available(), reason="reference modules absent (neither /root/reference nor oracle/_ref)")


def load_case(case):
    z = np.load(os.path.join(GOLDEN, f"ewald_{case}.npz"))
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
        DipoleMoment=A.DipoleMoment, Atomwise=A.Atomwise, EnergyEwald=A.EnergyEwald, Aggregation=A.Aggregation,
        Forces=A.Forces, NeuralNetworkPotential=NeuralNetworkPotential)


def package_model(case, weights, dtype):
    model = EO.build_case(package_mods(), case)
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


def _parts(batch):
    R = torch.as_tensor(batch["_positions"], dtype=torch.float64)
    ii, jj = torch.as_tensor(batch["_idx_i"]), torch.as_tensor(batch["_idx_j"])
    off = torch.as_tensor(batch["_offsets"], dtype=torch.float64)
    cell = torch.as_tensor(batch["_cell"], dtype=torch.float64).reshape(-1, 3, 3)
    return R, ii, jj, off, cell, torch.as_tensor(batch["_idx_m"]), len(batch["_n_atoms"])


@pytest.mark.parametrize("case", EO.CASES)
def test_oracle_matches_reference_fixtures(case):
    batch, w, ref = load_case(case)
    L = EO.LAYOUT[case]
    R, ii, jj, off, cell, idx_m, B = _parts(batch)
    q = torch.as_tensor(ref["fp64/partial_charges"]).reshape(-1)
    alpha, ke = float(w["output_modules.2.alpha"][0]), float(w["output_modules.2.ke"][0])
    assert alpha == EO.buffer_value(L["alpha"]) and ke == EO.buffer_value(EO.KE)
    e = EO.real_space(q, EO.PO.rij(R, ii, jj, off), ii, jj, idx_m, B, alpha, ke, screen=L["screen"])
    e = e + EO.reciprocal_self(q, R, cell, idx_m, B, alpha, EO.kvecs(L["k_max"]), ke)
    assert rel(e.numpy(), ref["fp64/e_ewald"]) <= 1e-11
    assert np.array_equal(w["output_modules.2.kvecs"], EO.kvecs(L["k_max"]).float().numpy())


def _random_system(seed=3):
    """Three triclinic systems (9, 1 and 14 atoms) and a trailing empty one, positions up to a few cells outside."""
    sizes = (9, 1, 14, 0)
    cell = torch.tensor(EO.E2_CELLS + ([[5.0, 0, 0], [0, 5.0, 0], [0, 0, 5.0]],), dtype=torch.float64)
    g = torch.Generator().manual_seed(seed)
    idx_m = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
    frac = 3.0 * torch.rand((sum(sizes), 3), generator=g, dtype=torch.float64) - 1.0
    R = torch.einsum("na,nab->nb", frac, cell[idx_m])
    B = len(sizes)
    q = torch.randn(R.shape[0], generator=g, dtype=torch.float64)
    g_E = torch.randn(B, generator=g, dtype=torch.float64)
    return R, q, cell, idx_m, B, g_E


def test_analytic_reverse_matches_autograd_and_finite_differences():
    R, q, cell, idx_m, B, g_E = _random_system()
    alpha, kv = 0.3, EO.kvecs(3)
    Rg, qg, cg = R.clone().requires_grad_(), q.clone().requires_grad_(), cell.clone().requires_grad_()
    e = EO.reciprocal_self(qg, Rg, cg, idx_m, B, alpha, kv, EO.KE)
    gR_a, gq_a, gc_a = torch.autograd.grad((g_E * e).sum(), (Rg, qg, cg))
    gR, gq, gc, W = EO.reciprocal_reverse(q, R, cell, idx_m, B, alpha, kv, EO.KE, g_E)
    assert rel(gR, gR_a) < 1e-12 and rel(gq, gq_a) < 1e-12 and rel(gc, gc_a) < 1e-12
    # the virial is the strain derivative of the Strain module (positions and cell scaled by 1 + strain)
    eps = torch.zeros(B, 3, 3, dtype=torch.float64, requires_grad=True)
    et = eps.transpose(1, 2)
    e = EO.reciprocal_self(q, R + torch.einsum("na,nab->nb", R, et[idx_m]), cell + cell @ et, idx_m, B, alpha, kv, EO.KE)
    (W_a,) = torch.autograd.grad((g_E * e).sum(), eps)
    assert rel(W, W_a) < 1e-12
    assert torch.allclose(W, W.transpose(1, 2), rtol=0, atol=1e-12 * float(W.abs().max()))
    # central differences of a few entries
    h = 1e-6

    def f(R_, q_, c_):
        return float((g_E * EO.reciprocal_self(q_, R_, c_, idx_m, B, alpha, kv, EO.KE)).sum())

    for a in (0, 11, 23):
        for c in range(3):
            Rp, Rm = R.clone(), R.clone()
            Rp[a, c] += h
            Rm[a, c] -= h
            assert (f(Rp, q, cell) - f(Rm, q, cell)) / (2 * h) == pytest.approx(float(gR[a, c]), rel=1e-6, abs=1e-6)
        qp, qm = q.clone(), q.clone()
        qp[a] += h
        qm[a] -= h
        assert (f(R, qp, cell) - f(R, qm, cell)) / (2 * h) == pytest.approx(float(gq[a]), rel=1e-6, abs=1e-6)
    for m in (0, 2):
        for b, c in ((0, 0), (1, 0), (2, 1)):
            cp, cm = cell.clone(), cell.clone()
            cp[m, b, c] += h
            cm[m, b, c] -= h
            assert (f(R, q, cp) - f(R, q, cm)) / (2 * h) == pytest.approx(float(gc[m, b, c]), rel=1e-6, abs=1e-6)


def _crystal_energy(frac, charges, a, alpha, k_max, cutoff):
    cell = np.eye(3) * a
    R = np.asarray(frac, np.float64) @ cell
    ii, jj, _, off = nl_oracle.neighbor_list(R, cell, np.ones(3, bool), cutoff)
    Rt = torch.as_tensor(R)
    q = torch.as_tensor(charges, dtype=torch.float64)
    ii, jj = torch.as_tensor(ii), torch.as_tensor(jj)
    r = EO.PO.rij(Rt, ii, jj, torch.as_tensor(off))
    idx_m = torch.zeros(len(charges), dtype=torch.int64)
    e = EO.real_space(q, r, ii, jj, idx_m, 1, alpha, 1.0)
    e = e + EO.reciprocal_self(q, Rt, torch.as_tensor(cell)[None], idx_m, 1, alpha, EO.kvecs(k_max), 1.0)
    return float(e[0])


def test_madelung_constants():
    """Independent of the reference: rock salt (nearest-neighbour distance 1) and CsCl at converged alpha, k_max."""
    fcc = np.array([[0, 0, 0], [0, .5, .5], [.5, 0, .5], [.5, .5, 0]])
    nacl = np.concatenate([fcc, fcc + np.array([.5, 0, 0])])
    e = _crystal_energy(nacl, [1.0] * 4 + [-1.0] * 4, 2.0, 2.25, 6, 4.0)
    assert -e / 4 == pytest.approx(1.747565, abs=1e-6)
    e = _crystal_energy([[0, 0, 0], [.5, .5, .5]], [1.0, -1.0], 1.0, 4.0, 4, 4.0)
    assert -e * math.sqrt(3) / 2 == pytest.approx(1.762675, abs=1e-6)


def test_energy_invariant_under_lattice_translation_of_one_atom():
    """Moving atom a by a lattice vector L (and its list offsets by -L / +L, so that every r_ij is kept) changes
    nothing: the phases of the reciprocal term see the raw position."""
    batch, _, ref = load_case("e2")
    L = EO.LAYOUT["e2"]
    q = torch.as_tensor(ref["fp64/partial_charges"]).reshape(-1)
    R, ii, jj, off, cell, idx_m, B = _parts(batch)

    def energy(R, off):
        e = EO.real_space(q, EO.PO.rij(R, ii, jj, off), ii, jj, idx_m, B, L["alpha"], EO.KE)
        return (e + EO.reciprocal_self(q, R, cell, idx_m, B, L["alpha"], EO.kvecs(L["k_max"]), EO.KE)).numpy()

    a = 25                                                          # an atom of system 1
    shift = 2 * cell[1, 1] - 3 * cell[1, 0] + cell[1, 2]
    R2, off2 = R.clone(), off.clone()
    R2[a] += shift
    off2[ii == a] += shift
    off2[jj == a] -= shift
    assert rel(energy(R2, off2), energy(R, off)) < 1e-12


@pytest.mark.parametrize("case", EO.CASES)
def test_aten_training_path_matches_reference_fixtures(case):
    """train() mode runs the ATen formula of functional_torch (FilterShortRange compacts exactly, as the reference)."""
    batch, w, ref = load_case(case)
    model = package_model(case, w, torch.float64)
    model.train()
    x = torch_batch(batch, torch.float64)
    out = dict(model(x))
    out.update({k: v for k, v in x.items() if k not in out})
    for k in ("energy", "e_ewald", "forces", "partial_charges", "dipole_moment", "stress"):
        assert rel(out[k].detach().numpy(), ref["fp64/" + k]) <= 1e-10, k


@pytest.mark.parametrize("case", EO.CASES)
def test_aten_training_path_weight_gradients_of_a_force_loss_match_reference(case):
    """The weight gradients of a force loss in train() mode (Forces with create_graph, so the double backward through the
    Ewald term and the charges) match those the unmodified reference computed in fp64."""
    batch, w, ref = load_case(case)
    model = package_model(case, w, torch.float64)
    model.train()
    out = model(torch_batch(batch, torch.float64))
    params = dict(model.named_parameters())
    names = sorted(k[5:] for k in ref if k.startswith("grad/"))
    assert any(n.startswith("output_modules.0.") for n in names)            # the charge head
    grads = torch.autograd.grad(EO.force_loss(out), [params[n] for n in names])
    for n, g in zip(names, grads):
        assert rel(g.numpy(), ref["grad/" + n]) <= 1e-9, n


def test_aten_training_path_raises_for_a_zero_volume_cell():
    from schnetpack_b200.atomistic import EnergyEwaldError

    batch, w, _ = load_case("e2")
    model = package_model("e2", w, torch.float64)
    model.train()
    x = torch_batch(batch, torch.float64)
    x["_cell"] = x["_cell"].clone()
    x["_cell"][1] = 1e-3 * torch.eye(3, dtype=torch.float64)           # invertible, but of (close to) zero volume
    with pytest.raises(EnergyEwaldError, match="no volume"):
        model(x)


def test_ewald_screening_other_than_switch_function_raises():
    from schnetpack_b200 import atomistic as A
    from schnetpack_b200 import nn as snn

    m = A.EnergyEwald(0.2, 2, "kcal/mol", "Ang", "e", screening_fn=snn.CosineCutoff(3.0))
    with pytest.raises(NotImplementedError, match="SwitchFunction"):
        m._screen()


@needs_ref
def test_convert_model_swaps_a_live_reference_ewald_and_keeps_state_dict():
    import sys

    sys.path.insert(0, GOLDEN)
    from make_golden_ewald import reference_mods
    from make_golden_pair_energy import load_reference_pair_modules

    from schnetpack_b200 import atomistic as A
    from schnetpack_b200.model import convert_model

    spk = load_reference_pair_modules()
    torch.manual_seed(0)
    ref = EO.build_case(reference_mods(spk), "e1")
    new = convert_model(ref)
    ew = [m for m in new.output_modules if type(m).__name__ == "EnergyEwald"]
    assert len(ew) == 1 and isinstance(ew[0], A.EnergyEwald)
    assert type(ew[0].screening_fn).__module__.startswith("schnetpack_b200")
    sd_ref, sd_new = ref.state_dict(), new.state_dict()
    assert set(sd_ref) == set(sd_new)
    for k in ("output_modules.2.ke", "output_modules.2.alpha", "output_modules.2.kvecs"):
        assert torch.equal(sd_ref[k].float(), sd_new[k])
    assert [m.differentiable_charges for m in new.output_modules if hasattr(m, "differentiable_charges")] == [True]
