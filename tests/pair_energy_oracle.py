"""fp64 restatement of the pair energies (atomistic/nuclear_repulsion.py:70-108, atomistic/electrostatic.py:14-152,
nn/cutoff.py:14-33,107-158) and the model layouts of the pair-energy fixtures (tests/golden/pair_energy_*.npz).

``build_case(mods, case)`` assembles a case from a namespace of module classes.  The reference's classes and this
package's have the same constructor signatures and ``state_dict`` keys, so the fixture generator builds the reference
model with it and the GPU tests build the CUDA model with it, then load the stored weights."""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np
import torch

KE_KCAL_ANG = 627.5094738898777 * 0.5291772105638411      # Ha * Bohr in kcal/mol * Angstrom (CODATA 2014, as ASE)

CASES = ("a", "b", "c", "d")


def _softplus(x):
    return torch.nn.functional.softplus(x)


def zbl_energy(Z, r_ij, idx_i, idx_j, idx_m, n_sys, params, ke, cutoff=None, d_max=None):
    """Per-system ZBL energy; params = (a_pow, a_div, coefficients, exponents) raw (softplus applied here)."""
    a_pow, a_div, coef, expo = (torch.as_tensor(p, dtype=torch.float64) for p in params)
    Zd = torch.as_tensor(Z).double()
    d = torch.linalg.norm(r_ij, dim=1)
    a = Zd ** _softplus(a_pow)
    a_ij = (a[idx_i] + a[idx_j]) * _softplus(a_div)
    c = _softplus(coef)
    c = c / torch.clamp(c.abs().sum(), min=1e-12)
    screen = (c[None, :] * torch.exp(-a_ij[:, None] * _softplus(expo)[None, :] * d[:, None])).sum(1)
    e = Zd[idx_i] * Zd[idx_j] / d * screen
    if cutoff is not None:
        e = e * 0.5 * (torch.cos(math.pi * d / cutoff) + 1.0) * (d < cutoff).double()
    if d_max is not None:
        e = torch.where(d <= d_max, e, torch.zeros_like(e))
    return 0.5 * ke * torch.zeros(n_sys, dtype=torch.float64).index_add(0, torch.as_tensor(idx_m)[idx_i], e)


def switch(d, on, off):
    x = (d - on) / (off - on)

    def comp(y):
        return torch.where(y <= 0, torch.zeros_like(y), torch.exp(-1.0 / torch.where(y <= 0, torch.ones_like(y), y)))

    fp, fm = comp(x), comp(1 - x)
    return torch.where(x <= 0, torch.ones_like(x), torch.where(x >= 1, torch.zeros_like(x), fm / (fp + fm)))


def coulomb_potential(d, damped=None):
    """1/d, or with damped = (switch_on, switch_off) the damped form."""
    if damped is None:
        return 1.0 / d
    f = switch(d, *damped)
    return f / torch.sqrt(d ** 2 + 1) + (1 - f) / d


def coulomb_energy(q, r_ij, idx_i, idx_j, idx_m, n_sys, ke, damped=None, cutoff=None, shift=None, d_max=None):
    d = torch.linalg.norm(r_ij, dim=1)
    V = coulomb_potential(d, damped)
    if cutoff is not None:
        if shift is None:
            shift = coulomb_potential(torch.tensor(float(cutoff), dtype=torch.float64), damped)
        V = V + shift ** 2 / V - 2.0 * shift
        V = torch.where(d <= cutoff, V, torch.zeros_like(V))
    if d_max is not None:
        V = torch.where(d <= d_max, V, torch.zeros_like(V))
    e = q[idx_i] * q[idx_j] * V
    return 0.5 * ke * torch.zeros(n_sys, dtype=torch.float64).index_add(0, torch.as_tensor(idx_m)[idx_i], e)


def rij(R, idx_i, idx_j, offsets):
    return R[idx_j] - R[idx_i] + offsets


# ---- model layouts of the fixtures ---------------------------------------------------------------------------------
LAYOUT = {
    # (list cutoff, representation cutoff, short_range_cutoff or None, ZBL cosine cutoff or None,
    #  Coulomb: (damped switch or None, cutoff or None, use_neighbors_lr), gated head, stress)
    "a": dict(list_cutoff=9.0, rep_cutoff=4.0, src=4.5, zbl_cut=4.5, damped=(1.0, 4.0), coul_cut=8.0, lr=True,
              gated=False, stress=False),
    "b": dict(list_cutoff=5.0, rep_cutoff=5.0, src=None, zbl_cut=None, damped=None, coul_cut=None, lr=False,
              gated=False, stress=False),
    "c": dict(list_cutoff=5.0, rep_cutoff=3.0, src=3.0, zbl_cut=3.0, damped=(1.0, 3.0), coul_cut=5.0, lr=True,
              gated=False, stress=True),
    "d": dict(list_cutoff=9.0, rep_cutoff=4.0, src=4.5, zbl_cut=4.5, damped=None, coul_cut=8.0, lr=True,
              gated=True, stress=False),
}
F_BASIS = 32


def build_case(mods: SimpleNamespace, case: str):
    """PairwiseDistances [+ Strain] [+ FilterShortRange] -> PaiNN -> DipoleMoment(return_charges) + Atomwise + ZBL +
    EnergyCoulomb + Aggregation + Forces."""
    L = LAYOUT[case]
    rep = mods.PaiNN(n_atom_basis=F_BASIS, n_interactions=2, radial_basis=mods.GaussianRBF(n_rbf=10, cutoff=L["rep_cutoff"]),
                     cutoff_fn=mods.CosineCutoff(L["rep_cutoff"]))
    ins = ([mods.Strain()] if L["stress"] else []) + [mods.PairwiseDistances()]
    if L["src"] is not None:
        ins.append(mods.FilterShortRange(L["src"]))
    pot = mods.CoulombPotential() if L["damped"] is None else mods.DampedCoulombPotential(mods.SwitchFunction(*L["damped"]))
    outs = [
        mods.DipoleMoment(F_BASIS, return_charges=True, correct_charges=True, use_vector_representation=L["gated"]),
        mods.Atomwise(F_BASIS, output_key="e_nn"),
        mods.ZBLRepulsionEnergy("kcal/mol", "Ang", "e_zbl",
                                cutoff_fn=mods.CosineCutoff(L["zbl_cut"]) if L["zbl_cut"] is not None else None),
        mods.EnergyCoulomb("kcal/mol", "Ang", pot, "e_coul", use_neighbors_lr=L["lr"], cutoff=L["coul_cut"]),
        mods.Aggregation(["e_nn", "e_zbl", "e_coul"], "energy"),
        mods.Forces(calc_forces=True, calc_stress=L["stress"]),
    ]
    return mods.NeuralNetworkPotential(representation=rep, input_modules=ins, output_modules=outs, postprocessors=[],
                                       do_postprocessing=False)


def case_batch(case: str) -> dict:
    """numpy batch of a case (synthetic molecules / box with the list at the case's list cutoff)."""
    from schnetpack_b200 import synthetic as S

    L = LAYOUT[case]
    if case == "c":
        b = S.periodic_box(n_atoms_total=48, density=0.1002, cutoff=L["list_cutoff"], seed=3)
    else:
        b = S.aspirin_batch(3, cutoff=L["list_cutoff"], jitter=0.05, seed=11 + ord(case))
    if case in ("a", "b"):
        b["total_charge"] = np.array([1.0, -1.0, 0.0], dtype=np.float32)
    return b


def pair_terms_fixed_q(case: str, batch: dict, sd: dict, charges):
    """fp64 ZBL and Coulomb energies of a case at the given charges and their -d/dR (charges held fixed)."""
    L = LAYOUT[case]
    R = torch.as_tensor(batch["_positions"], dtype=torch.float64).requires_grad_()
    off = torch.as_tensor(batch["_offsets"], dtype=torch.float64)
    ii, jj = torch.as_tensor(batch["_idx_i"]), torch.as_tensor(batch["_idx_j"])
    idx_m = torch.as_tensor(batch["_idx_m"])
    n_sys = int(len(batch["_n_atoms"]))
    r = rij(R, ii, jj, off)
    zp = [sd[f"output_modules.2.{k}"] for k in ("a_pow", "a_div", "coefficients", "exponents")]
    e_z = zbl_energy(batch["_atomic_numbers"], r, ii, jj, idx_m, n_sys, zp, float(sd["output_modules.2.ke"]),
                     cutoff=L["zbl_cut"], d_max=L["src"])
    shift = float(np.asarray(sd["output_modules.3.shift"]).reshape(-1)[0]) if L["coul_cut"] is not None else None
    e_c = coulomb_energy(torch.as_tensor(charges, dtype=torch.float64).reshape(-1), r, ii, jj, idx_m, n_sys,
                         float(np.asarray(sd["output_modules.3.ke"]).reshape(-1)[0]), damped=L["damped"],
                         cutoff=L["coul_cut"], shift=shift, d_max=None if L["lr"] else L["src"])
    (g,) = torch.autograd.grad((e_z + e_c).sum(), R)
    return e_z.detach(), e_c.detach(), -g
