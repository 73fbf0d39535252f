"""TRAINING-MODE path (SURVEY.md section 8 f3): the hot-path math written with differentiable ATen operations.

The CUDA kernels of this package provide the forward pass and first-order gradients with respect to positions / strain --
everything inference, forces and MD need.  Training needs more: gradients with respect to every weight and, for force
losses, a second differentiation through the force computation (``create_graph=self.training``,
/root/reference/src/schnetpack/atomistic/response.py:62-68).  Those are NOT implemented as kernels.  So that the modules
still drop in under ``spktrain`` (``task.py:166-185``), a module that is in ``train()`` mode with trainable parameters under
grad mode evaluates the SAME formulas below with plain torch operations (autograd-complete, any device, reference speed);
``eval()`` mode -- validation, inference, MD, deployment -- always runs the kernels.  The switch is
``schnetpack_b200.nn.use_training_path`` and is exercised by tests/test_training_path.py against the reference's own weight
gradients.  Formulas and line citations as in oracle/spk_oracle.py (which this package never imports).
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F_

from . import properties

Tensor = torch.Tensor


def _act(code_fn, x):
    return x if code_fn is None else code_fn(x)


def ssp(x: Tensor) -> Tensor:
    """nn/activations.py:9-22."""
    return F_.softplus(x) - math.log(2.0)


def _activation(act):
    from . import nn as snn
    from . import ops

    code = snn.activation_code(act)
    return {ops.ACT_NONE: None, ops.ACT_SILU: F_.silu, ops.ACT_SSP: ssp}[code]


def dense(x: Tensor, lin, act=None) -> Tensor:
    """nn/base.py:52-55."""
    y = F_.linear(x, lin.weight, lin.bias)
    return y if act is None else act(y)


def radial(rb, d: Tensor) -> Tensor:
    if type(rb).__name__ == "GaussianRBF":                                   # nn/radial.py:11-15
        coeff = -0.5 / torch.pow(rb.widths, 2)
        return torch.exp(coeff * torch.pow(d[..., None] - rb.offsets, 2))
    ax = d[..., None] * rb.freqs                                             # nn/radial.py:105-110
    norm = torch.where(d == 0, torch.ones_like(d), d)
    return torch.sin(ax) / norm[..., None]


def cutoff(cf, d: Tensor) -> Tensor:
    rc = cf.cutoff
    return 0.5 * (torch.cos(d * math.pi / rc) + 1.0) * (d < rc).to(d.dtype)   # nn/cutoff.py:14-33


def scatter_add(x: Tensor, idx: Tensor, dim_size: int) -> Tensor:
    """nn/scatter.py:26-34."""
    return torch.zeros((dim_size,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device).index_add(0, idx, x)


def pairwise(inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
    R, off = inputs[properties.R], inputs[properties.offsets]                # atomistic/distances.py:14-26
    inputs[properties.Rij] = R[inputs[properties.idx_j]] - R[inputs[properties.idx_i]] + off
    return inputs


def _embed(mod, inputs):
    x = mod.embedding(inputs[properties.Z])
    for e in mod.electronic_embeddings:
        x = x + e(x, inputs)
    return x


def painn(mod, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """representation/painn.py:207-256."""
    r_ij, idx_i, idx_j = inputs[properties.Rij], inputs[properties.idx_i], inputs[properties.idx_j]
    n_atoms = inputs[properties.Z].shape[0]
    F = mod.n_atom_basis
    act = _activation(mod.activation)
    d = torch.norm(r_ij, dim=1, keepdim=True)                                # :227
    u = r_ij / d                                                             # :228
    phi = radial(mod.radial_basis, d)                                        # :229
    fc = cutoff(mod.cutoff_fn, d)                                            # :230
    filters = dense(phi, mod.filter_net) * fc[..., None]                     # :232
    flist = [filters] * mod.n_interactions if mod.share_filters else torch.split(filters, 3 * F, dim=-1)
    q = _embed(mod, inputs)[:, None]                                         # :239-242
    mu = torch.zeros((n_atoms, 3, F), dtype=q.dtype, device=q.device)        # :246
    for it, mx, W in zip(mod.interactions, mod.mixing, flist):
        c = it.interatomic_context_net
        x = dense(dense(q, c[0], act), c[1])                                 # :54
        y = W * x[idx_j]                                                     # :55,:57
        dq, dmuR, dmumu = torch.split(y, F, dim=-1)                          # :59
        dq = scatter_add(dq, idx_i, n_atoms)                                 # :60
        dmu = scatter_add(dmuR * u[..., None] + dmumu * mu[idx_j], idx_i, n_atoms)     # :61-62
        q = q + dq
        mu = mu + dmu
        V, Wm = torch.split(dense(mu, mx.mu_channel_mix), F, dim=-1)         # :103-104
        Vn = torch.sqrt(torch.sum(V ** 2, dim=-2, keepdim=True) + mx.epsilon)  # :105
        m = mx.intraatomic_context_net
        s = dense(dense(torch.cat([q, Vn], dim=-1), m[0], act), m[1])        # :107-108
        dq_i, dmu_i, dqmu_i = torch.split(s, F, dim=-1)
        q = q + dq_i + dqmu_i * torch.sum(V * Wm, dim=1, keepdim=True)       # :113-115
        mu = mu + dmu_i * Wm                                                 # :111,:116
    inputs["scalar_representation"] = q.squeeze(1)
    inputs["vector_representation"] = mu
    return inputs


def schnet(mod, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """representation/schnet.py:147-173."""
    r_ij, idx_i, idx_j = inputs[properties.Rij], inputs[properties.idx_i], inputs[properties.idx_j]
    act = _activation(mod.activation)
    d = torch.norm(r_ij, dim=1)                                              # :156
    f_ij = radial(mod.radial_basis, d)                                       # :157
    rcut = cutoff(mod.cutoff_fn, d)                                          # :158
    x = _embed(mod, inputs)                                                  # :161
    for it in mod.interactions:
        h = dense(x, it.in2f)                                                # :60
        Wij = dense(dense(f_ij, it.filter_network[0], act), it.filter_network[1]) * rcut[:, None]   # :61-62
        m = scatter_add(h[idx_j] * Wij, idx_i, x.shape[0])                   # :65-67
        x = x + dense(dense(m, it.f2out[0], act), it.f2out[1])               # :69, :168
    inputs["scalar_representation"] = x
    return inputs


def so3net(mod, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """representation/so3net.py:103-155 with the nn.so3 modules' own ATen formulas."""
    from .nn import so3

    r_ij, idx_i, idx_j = inputs[properties.Rij], inputs[properties.idx_i], inputs[properties.idx_j]
    d = torch.norm(r_ij, dim=1, keepdim=True)                                # :122
    Y = mod.sphharm(r_ij / d)                                                # :123-125
    phi = radial(mod.radial_basis, d)                                        # :126
    fc = cutoff(mod.cutoff_fn, d)[..., None]                                 # :127
    x = so3.scalar2rsh(_embed(mod, inputs)[:, None], int(mod.lmax))          # :130-136
    for conv, m1, m2, gate, m3 in zip(mod.so3convs, mod.mixings1, mod.mixings2, mod.gatings, mod.mixings3):
        dx = conv(x, phi, Y, fc, idx_i, idx_j)                               # :140
        dx = dx + mod.so3product(dx, m1(dx))                                 # :141-142
        x = x + m3(gate(m2(dx)))                                             # :143-146
    inputs["scalar_representation"] = x[:, 0]
    inputs["multipole_representation"] = x
    if mod.return_vector_representation:
        inputs["vector_representation"] = torch.roll(x[:, 1:4], 1, 1)
    return inputs


def atomwise(mod, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """atomistic/atomwise.py:69-88."""
    act = _activation(mod.activation)
    y = inputs["scalar_representation"]
    n = len(mod.outnet)
    for k, lin in enumerate(mod.outnet):
        y = dense(y, lin, act if k < n - 1 else None)
    if mod.per_atom_output_key is not None:
        inputs[mod.per_atom_output_key] = y
    if mod.aggregation_mode is not None:
        idx_m = inputs[properties.idx_m]
        n_mol = int(inputs[properties.n_atoms].shape[0]) if properties.n_atoms in inputs else int(idx_m[-1]) + 1
        y = scatter_add(y, idx_m, n_mol)
        y = torch.squeeze(y, -1)
        if mod.aggregation_mode == "avg":
            y = y / inputs[properties.n_atoms]
    inputs[mod.output_key] = y
    return inputs


def gated_block(blk, s: Tensor, v: Tensor):
    """nn/equivariant.py:57-71."""
    vmix = F_.linear(v, blk.mix_vectors.weight)
    vV, vW = torch.split(vmix, blk.n_vout, dim=-1)
    ctx = torch.cat([s, torch.norm(vV, dim=-2)], dim=-1)
    x = dense(ctx, blk.scalar_net[0], _activation(blk.scalar_net[0].activation))
    x = dense(x, blk.scalar_net[1])
    s_out, x = torch.split(x, [blk.n_sout, blk.n_vout], dim=-1)
    v_out = x.unsqueeze(-2) * vW
    if blk.sactivation:
        s_out = _act(_activation(blk.sactivation), s_out)
    return s_out, v_out


def _n_sys(inputs: Dict[str, Tensor]) -> int:
    return int(inputs[properties.n_atoms].shape[0])


def dipole_moment(mod, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """atomistic/atomwise.py:172-213."""
    R, idx_m = inputs[properties.R], inputs[properties.idx_m]
    n_sys = _n_sys(inputs)
    s = inputs["scalar_representation"]
    if mod.use_vector_representation:
        v = inputs["vector_representation"]
        for blk in mod.outnet:
            s, v = gated_block(blk, s, v)
        charges, atomic_dipoles = s, v.squeeze(-1)
    else:
        for lin in mod.outnet:
            s = dense(s, lin, _activation(lin.activation))
        charges, atomic_dipoles = s, None
    if mod.correct_charges:
        sum_charge = scatter_add(charges, idx_m, n_sys)
        total = inputs[properties.total_charge][:, None] if properties.total_charge in inputs else torch.zeros_like(sum_charge)
        charges = charges + ((total - sum_charge) / inputs[properties.n_atoms].unsqueeze(-1))[idx_m]
    if mod.return_charges:
        inputs[mod.charges_key] = charges
    y = R * charges
    if atomic_dipoles is not None:
        y = y + atomic_dipoles
    y = scatter_add(y, idx_m, n_sys)
    if mod.predict_magnitude:
        y = torch.norm(y, dim=1, keepdim=False)
    inputs[mod.dipole_key] = y
    return inputs


def polarizability(mod, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """atomistic/atomwise.py:267-293."""
    R = inputs[properties.R]
    s, v = inputs["scalar_representation"], inputs["vector_representation"]
    for blk in mod.outnet:
        s, v = gated_block(blk, s, v)
    alpha = torch.diag_embed(s[..., 0:1].expand(-1, 3))
    mur = v[..., None, 0] * R[..., None, :]
    alpha = alpha + mur + mur.transpose(-2, -1)
    inputs[mod.polarizability_key] = scatter_add(alpha, inputs[properties.idx_m], _n_sys(inputs))
    return inputs


def _norm(r_ij: Tensor) -> Tensor:
    return torch.norm(r_ij, dim=1)


def zbl_repulsion(mod, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """atomistic/nuclear_repulsion.py:70-108."""
    z = inputs[properties.Z]
    d_ij = _norm(inputs[properties.Rij])
    idx_i, idx_j, idx_m = inputs[properties.idx_i], inputs[properties.idx_j], inputs[properties.idx_m]
    a = z ** F_.softplus(mod.a_pow)
    a_ij = (a[idx_i] + a[idx_j]) * F_.softplus(mod.a_div)
    exponents = a_ij[..., None] * F_.softplus(mod.exponents)[None, ...]
    coefficients = F_.normalize(F_.softplus(mod.coefficients)[None, ...], p=1.0, dim=1)
    screening = torch.sum(coefficients * torch.exp(-exponents * d_ij[:, None]), dim=1)
    repulsion = (z[idx_i] * z[idx_j]) / d_ij
    if mod.cutoff_fn is not None:
        repulsion = repulsion * cutoff(mod.cutoff_fn, d_ij)
    y = scatter_add(repulsion * screening, idx_i, z.shape[0])
    y = scatter_add(y, idx_m, _n_sys(inputs))
    inputs[mod.output_key] = 0.5 * mod.ke * y
    return inputs


def energy_coulomb(mod, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """atomistic/electrostatic.py:109-152."""
    q = inputs[mod.charges_key].squeeze(-1)
    if mod.use_neighbors_lr:
        r_ij, idx_i, idx_j = inputs[properties.Rij_lr], inputs[properties.idx_i_lr], inputs[properties.idx_j_lr]
    else:
        r_ij, idx_i, idx_j = inputs[properties.Rij], inputs[properties.idx_i], inputs[properties.idx_j]
    d_ij = _norm(r_ij)
    potential = mod.coulomb_potential(d_ij)
    if mod.cutoff is not None:
        potential = potential + mod.shift ** 2 / potential - 2.0 * mod.shift
        potential = torch.where(d_ij <= mod.cutoff, potential, torch.zeros_like(potential))
    y = scatter_add(q[idx_i] * q[idx_j] * potential, idx_i, q.shape[0])
    y = scatter_add(y, inputs[properties.idx_m], _n_sys(inputs))
    inputs[mod.output_key] = 0.5 * mod.ke * torch.squeeze(y, -1)
    return inputs


def energy_ewald(mod, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """atomistic/electrostatic.py:226-375 with the number of systems from ``_n_atoms``."""
    q = inputs[mod.charges_key].squeeze(-1)
    idx_m = inputs[properties.idx_m]
    if mod.use_neighbors_lr:
        r_ij, idx_i, idx_j = inputs[properties.Rij_lr], inputs[properties.idx_i_lr], inputs[properties.idx_j_lr]
    else:
        r_ij, idx_i, idx_j = inputs[properties.Rij], inputs[properties.idx_i], inputs[properties.idx_j]
    d_ij = _norm(r_ij)
    R, cell = inputs[properties.R], inputs[properties.cell]
    n_sys = _n_sys(inputs)
    f_r = torch.erfc(torch.sqrt(mod.alpha) * d_ij) / d_ij
    if mod.screening_fn is not None:
        f_r = f_r * (1.0 - mod.screening_fn(d_ij))
    y = scatter_add(q[idx_i] * q[idx_j] * f_r, idx_i, q.shape[0])
    y_real = 0.5 * mod.ke * scatter_add(y, idx_m, n_sys).squeeze(-1)
    recip_box = 2.0 * math.pi * torch.linalg.inv(cell).transpose(1, 2)
    v_box = torch.abs(torch.linalg.det(cell))
    if torch.any(torch.isclose(v_box, torch.zeros_like(v_box))):
        from .atomistic.pair_terms import EnergyEwaldError

        raise EnergyEwaldError("Simulation box has no volume.")
    kvecs = torch.matmul(mod.kvecs[None, :, :], recip_box)
    k_squared = torch.sum(kvecs ** 2, dim=2)
    q_gauss = torch.exp(-0.25 * k_squared / mod.alpha)
    kvec_dot_pos = torch.sum(kvecs[idx_m] * R[:, None, :], dim=2)
    q_real = scatter_add(q[:, None] * torch.cos(kvec_dot_pos), idx_m, n_sys)
    q_imag = scatter_add(q[:, None] * torch.sin(kvec_dot_pos), idx_m, n_sys)
    y_ewald = 2.0 * math.pi / v_box * torch.sum((q_real ** 2 + q_imag ** 2) * q_gauss / k_squared, dim=1)
    self_interaction = torch.sqrt(mod.alpha / math.pi) * scatter_add(q ** 2, idx_m, n_sys)
    inputs[mod.output_key] = y_real + mod.ke * (y_ewald - self_interaction)
    return inputs


def filter_short_range(mod, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """atomistic/distances.py:42-57 (exact compaction; a host sync and a data-dependent shape)."""
    idx_i, idx_j, Rij = inputs[properties.idx_i], inputs[properties.idx_j], inputs[properties.Rij]
    cidx = torch.nonzero(_norm(Rij) <= mod.short_range_cutoff).squeeze(-1)
    inputs[properties.Rij_lr] = Rij
    inputs[properties.idx_i_lr] = idx_i
    inputs[properties.idx_j_lr] = idx_j
    inputs[properties.Rij] = Rij[cidx]
    inputs[properties.idx_i] = idx_i[cidx]
    inputs[properties.idx_j] = idx_j[cidx]
    return inputs
