"""fp64 restatement of the Ewald sum (atomistic/electrostatic.py:155-375) with the analytic reverse of the reciprocal and
self terms (dE/dR, dE/dq, dE/dcell and the reciprocal virial), and the model layouts of the Ewald fixtures
(tests/golden/ewald_*.npz).

``build_case(mods, case)`` assembles a case from a namespace of module classes; the reference's classes and this
package's have the same constructor signatures and ``state_dict`` keys, so the fixture generator builds the reference
model with it and the GPU tests build the CUDA model with it, then load the stored weights."""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np
import torch

import pair_energy_oracle as PO

CASES = ("e1", "e2")
KE = PO.KE_KCAL_ANG


def kvecs(k_max: int) -> torch.Tensor:
    """electrostatic.py:209-224 in fp64: integer triples with 0 < |n|^2 <= k_max^2 + 2 (the full sphere)."""
    kr = torch.arange(0, k_max + 1, dtype=torch.float64)
    kr = torch.cat([kr, -kr[1:]])
    kv = torch.cartesian_prod(kr, kr, kr)
    norm = (kv ** 2).sum(1)
    kv = kv[norm <= k_max ** 2 + 2]
    return kv[(kv ** 2).sum(1) != 0]


def buffer_value(x: float) -> float:
    """A value as the module's fp32 buffer holds it (the reference registers ke and alpha as torch.Tensor([x]))."""
    return float(np.float32(x))


def _seg(x, idx_m, n_sys):
    return torch.zeros((n_sys,) + x.shape[1:], dtype=x.dtype).index_add(0, torch.as_tensor(idx_m), x)


def real_space(q, r_ij, idx_i, idx_j, idx_m, n_sys, alpha, ke, screen=None, d_max=None):
    """electrostatic.py:266-308; ``screen`` = (switch_on, switch_off) of a SwitchFunction, ``d_max`` a distance mask."""
    d = torch.linalg.norm(r_ij, dim=1)
    f = torch.erfc(math.sqrt(alpha) * d) / d
    if screen is not None:
        f = f * (1.0 - PO.switch(d, *screen))
    if d_max is not None:
        f = torch.where(d <= d_max, f, torch.zeros_like(f))
    e = q[idx_i] * q[idx_j] * f
    return 0.5 * ke * _seg(e, torch.as_tensor(idx_m)[idx_i], n_sys)


def reciprocal_self(q, R, cell, idx_m, n_sys, alpha, kv, ke):
    """electrostatic.py:310-375: E_rec - E_self per system."""
    cell = cell.reshape(-1, 3, 3)
    recip = 2.0 * math.pi * torch.linalg.inv(cell).transpose(1, 2)
    V = torch.abs(torch.linalg.det(cell))
    k = torch.matmul(kv[None], recip)                                       # [B,K,3]
    k2 = (k ** 2).sum(2)
    theta = (k[idx_m] * R[:, None, :]).sum(2)                               # [N,K]
    re = _seg(q[:, None] * torch.cos(theta), idx_m, n_sys)
    im = _seg(q[:, None] * torch.sin(theta), idx_m, n_sys)
    e_rec = 2.0 * math.pi / V * ((re ** 2 + im ** 2) * torch.exp(-0.25 * k2 / alpha) / k2).sum(1)
    e_self = math.sqrt(alpha / math.pi) * _seg(q ** 2, idx_m, n_sys)
    return ke * (e_rec - e_self)


def reciprocal_reverse(q, R, cell, idx_m, n_sys, alpha, kv, ke, g_E):
    """The analytic reverse of ``reciprocal_self`` for the upstream g_E [B]: (g_R [N,3], g_q [N], g_cell [B,3,3],
    W_rec [B,3,3]).  With H = h^-1, E_k = ke (2 pi / V) f_k |S_k|^2 and T = sum_k E_k (1/k^2 + 1/(4 alpha)) k (x) k:
      g_R_i  = ke (2 pi / V) g_E sum_k 2 f_k q_i k (Im S cos t_i - Re S sin t_i)
      g_q_i  = g_E ke [(2 pi / V) sum_k 2 f_k (Re S cos t_i + Im S sin t_i) - 2 sqrt(alpha / pi) q_i]
      g_cell = -H^T [sum_i r_i (x) g_R_i - 2 g_E T + g_E E_rec I]       (dk/dh_bc = -H_ab k_c, V dE/dV = -E)
      W_rec  = -g_E (E_rec I - 2 T)                                      (the strain derivative: phases are invariant)"""
    cell = cell.reshape(-1, 3, 3)
    H = torch.linalg.inv(cell)
    V = torch.abs(torch.linalg.det(cell))
    k = torch.matmul(kv[None], 2.0 * math.pi * H.transpose(1, 2))
    k2 = (k ** 2).sum(2)
    f = torch.exp(-0.25 * k2 / alpha) / k2
    theta = (k[idx_m] * R[:, None, :]).sum(2)
    c, s = torch.cos(theta), torch.sin(theta)
    re, im = _seg(q[:, None] * c, idx_m, n_sys), _seg(q[:, None] * s, idx_m, n_sys)
    pre = ke * 2.0 * math.pi / V                                            # [B]
    am = idx_m
    u = 2.0 * f[am] * (im[am] * c - re[am] * s)                             # [N,K]
    g_R = (pre * g_E)[am, None] * q[:, None] * (u[:, :, None] * k[am]).sum(1)
    g_q = g_E[am] * (pre[am] * (2.0 * f[am] * (re[am] * c + im[am] * s)).sum(1) - 2.0 * ke * math.sqrt(alpha / math.pi) * q)
    E_k = pre[:, None] * f * (re ** 2 + im ** 2)                            # [B,K]
    E_rec = E_k.sum(1)
    w = E_k * (1.0 / k2 + 0.25 / alpha)
    T = torch.einsum("bk,bka,bkc->bac", w, k, k)
    I = torch.eye(3, dtype=torch.float64)[None]
    RG = _seg(R[:, :, None] * g_R[:, None, :], idx_m, n_sys)
    M = RG - 2.0 * g_E[:, None, None] * T + (g_E * E_rec)[:, None, None] * I
    g_cell = -torch.matmul(H.transpose(1, 2), M)
    W = -g_E[:, None, None] * (E_rec[:, None, None] * I - 2.0 * T)
    return g_R, g_q, g_cell, W


# ---- model layouts of the fixtures ---------------------------------------------------------------------------------
LAYOUT = {
    # e1: water box, screened real space on the long-range list after FilterShortRange, stress
    "e1": dict(list_cutoff=6.0, rep_cutoff=3.0, src=3.0, screen=(1.0, 3.0), lr=True, alpha=0.12, k_max=4,
               stress=True),
    # e2: three triclinic cells, no screen, standard list, stress
    "e2": dict(list_cutoff=5.0, rep_cutoff=5.0, src=None, screen=None, lr=False, alpha=0.2, k_max=3, stress=True),
}
F_BASIS = 32


def force_loss(out):
    """The loss whose weight gradients the fixtures hold: sum of squared forces plus the energies."""
    return (out["forces"] ** 2).sum() + out["energy"].sum()


def build_case(mods: SimpleNamespace, case: str):
    """Strain + PairwiseDistances [+ FilterShortRange] -> PaiNN -> DipoleMoment(return_charges, correct_charges) +
    Atomwise + EnergyEwald + Aggregation + Forces(stress)."""
    L = LAYOUT[case]
    rep = mods.PaiNN(n_atom_basis=F_BASIS, n_interactions=2, radial_basis=mods.GaussianRBF(n_rbf=10, cutoff=L["rep_cutoff"]),
                     cutoff_fn=mods.CosineCutoff(L["rep_cutoff"]))
    ins = ([mods.Strain()] if L["stress"] else []) + [mods.PairwiseDistances()]
    if L["src"] is not None:
        ins.append(mods.FilterShortRange(L["src"]))
    screen = mods.SwitchFunction(*L["screen"]) if L["screen"] is not None else None
    outs = [
        mods.DipoleMoment(F_BASIS, return_charges=True, correct_charges=True),
        mods.Atomwise(F_BASIS, output_key="e_nn"),
        mods.EnergyEwald(L["alpha"], L["k_max"], "kcal/mol", "Ang", "e_ewald", use_neighbors_lr=L["lr"],
                         screening_fn=screen),
        mods.Aggregation(["e_nn", "e_ewald"], "energy"),
        mods.Forces(calc_forces=True, calc_stress=L["stress"]),
    ]
    return mods.NeuralNetworkPotential(representation=rep, input_modules=ins, output_modules=outs, postprocessors=[],
                                       do_postprocessing=False)


def triclinic_batch(sizes, cells, cutoff, seed, total_charge=None):
    """Random positions (minimum distance 0.9 A) in the given cells, O/H/H atomic numbers, list from the fp64 oracle."""
    from oracle import nl_oracle

    rng = np.random.default_rng(seed)
    pos = []
    for n, h in zip(sizes, cells):
        h = np.asarray(h, np.float64)
        pts = []
        while len(pts) < n:
            p = rng.uniform(0, 1, 3) @ h
            ok = True
            for o in pts:
                d = p - o
                fr = d @ np.linalg.inv(h)
                d = (fr - np.round(fr)) @ h
                if np.linalg.norm(d) < 0.9:
                    ok = False
                    break
            if ok:
                pts.append(p)
        pos.append(np.array(pts))
    R = np.concatenate(pos)
    cells = np.asarray(cells, np.float64)
    n_atoms = np.array(sizes, dtype=np.int64)
    ii, jj, _, off = nl_oracle.batch_neighbor_list(R, cells, np.ones((len(sizes), 3), bool), n_atoms, cutoff)
    out = {
        "_n_atoms": n_atoms, "_idx_m": np.repeat(np.arange(len(sizes)), sizes).astype(np.int64),
        "_atomic_numbers": np.tile(np.array([8, 1, 1], np.int64), R.shape[0] // 3 + 1)[:R.shape[0]],
        "_positions": R.astype(np.float32), "_idx_i": ii.astype(np.int64), "_idx_j": jj.astype(np.int64),
        "_offsets": off.astype(np.float32), "_cell": cells.astype(np.float32), "_pbc": np.ones((len(sizes), 3), bool),
    }
    if total_charge is not None:
        out["total_charge"] = np.asarray(total_charge, np.float32)
    return out


E2_CELLS = ([[7.0, 0.0, 0.0], [1.5, 6.5, 0.0], [0.8, -1.1, 7.2]],
            [[8.5, 0.0, 0.0], [-2.0, 7.8, 0.0], [1.3, 2.1, 8.0]],
            [[6.2, 0.4, 0.0], [2.2, 6.0, 0.5], [-0.6, 1.4, 6.6]])


def case_batch(case: str) -> dict:
    L = LAYOUT[case]
    if case == "e1":
        from schnetpack_b200 import synthetic as S

        return S.periodic_box(n_atoms_total=48, density=0.1002, cutoff=L["list_cutoff"], seed=5)
    return triclinic_batch((21, 30, 15), E2_CELLS, L["list_cutoff"], seed=7, total_charge=(0.0, 1.0, 0.0))


def ewald_fixed_q(case: str, batch: dict, charges):
    """fp64 Ewald energy of a case at the given charges and its -d/dR (charges held fixed)."""
    L = LAYOUT[case]
    R = torch.as_tensor(batch["_positions"], dtype=torch.float64).requires_grad_()
    off = torch.as_tensor(batch["_offsets"], dtype=torch.float64)
    ii, jj = torch.as_tensor(batch["_idx_i"]), torch.as_tensor(batch["_idx_j"])
    idx_m = torch.as_tensor(batch["_idx_m"])
    cell = torch.as_tensor(batch["_cell"], dtype=torch.float64).reshape(-1, 3, 3)
    n_sys = int(len(batch["_n_atoms"]))
    q = torch.as_tensor(charges, dtype=torch.float64).reshape(-1)
    r = PO.rij(R, ii, jj, off)
    alpha, ke = buffer_value(L["alpha"]), buffer_value(KE)
    e = real_space(q, r, ii, jj, idx_m, n_sys, alpha, ke, screen=L["screen"], d_max=None if L["lr"] else L["src"])
    e = e + reciprocal_self(q, R, cell, idx_m, n_sys, alpha, kvecs(L["k_max"]), ke)
    (g,) = torch.autograd.grad(e.sum(), R)
    return e.detach(), -g
