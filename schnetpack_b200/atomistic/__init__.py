"""Mirror of the hot-path output/input modules of ``schnetpack.atomistic`` on the CUDA kernels:
``PairwiseDistances`` (atomistic/distances.py:9-26), ``Atomwise`` (atomistic/atomwise.py:14-88) and ``Forces``
(atomistic/response.py:18-92), and the gated equivariant heads ``DipoleMoment`` / ``Polarizability``
(atomistic/atomwise.py:91-293)."""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Union

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd import grad

from .. import functional as K
from .. import nn as snn
from .. import ops
from .. import properties

__all__ = ["PairwiseDistances", "Atomwise", "Forces", "Strain", "DipoleMoment", "Polarizability", "ZBLRepulsionEnergy",
           "CoulombPotential", "DampedCoulombPotential", "EnergyCoulomb", "EnergyEwald", "EnergyEwaldError", "Aggregation",
           "FilterShortRange", "EnergyPME", "pme_mesh", "use_pme"]


class PairwiseDistances(nn.Module):
    """Rij = R[idx_j] - R[idx_i] + offsets (distances.py:14-26).  The backward assembles dE/dR per atom from the
    receiver- and sender-grouped edge views (deterministic; the reference uses index_put atomics).

    Virial on request: with a caller-owned fp64 ``[n_sys, 3, 3]`` CUDA tensor under ``properties.virial`` the backward also
    writes W[m] = sum_{e in m} dE/dr_e (x) r_e into it (fp64 sums in a fixed order), so that stress = W / V without a strain
    leaf.  This costs one ``spk_segment_ptr`` launch in the forward and the two launches of ``spk_pairwise_virial`` (plus
    its small workspace) in the backward; the buffer is only written when a backward runs, so the evaluation needs grad
    mode and positions that require grad.  Without the key nothing changes.  An ``EnergyEwald`` deposits its reciprocal
    virial, which does not go through r_ij, in the buffer first (its backward always runs before this one, which reads
    r_ij's gradient from it); the pairwise pass then adds to the buffer instead of overwriting it."""

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        virial = inputs.get(properties.virial)
        if self.training and torch.is_grad_enabled():     # training graph: differentiable twice (functional_torch)
            if virial is not None:
                raise ValueError(f"PairwiseDistances: the '{properties.virial}' output is computed by the CUDA kernels "
                                 "only; evaluate the model in eval() mode (or under no trainable parameters) to get it")
            from .. import functional_torch as T

            return T.pairwise(inputs)
        R = inputs[properties.R]
        offsets = inputs[properties.offsets]
        idx_i = inputs[properties.idx_i].long()
        idx_j = inputs[properties.idx_j].long()
        graph = ops.get_graph(inputs[properties.idx_i] if inputs[properties.idx_i].dtype == torch.int64 else idx_i,
                              inputs[properties.idx_j] if inputs[properties.idx_j].dtype == torch.int64 else idx_j,
                              R.shape[0])
        holder = dict(idx_i=idx_i.contiguous(), idx_j=idx_j.contiguous(), graph=graph)
        if virial is not None:
            idx_m = inputs[properties.idx_m]
            off_grad = offsets is not None and offsets.requires_grad
            if not (torch.is_grad_enabled() and (R.requires_grad or off_grad)):
                raise ValueError(f"PairwiseDistances: '{properties.virial}' is filled by the backward pass; evaluate with "
                                 "grad enabled and positions that require grad (a Forces output does both)")
            if (not virial.is_cuda or virial.dtype != torch.float64 or not virial.is_contiguous() or virial.dim() != 3
                    or virial.shape[1:] != (3, 3) or virial.device != R.device):
                raise ValueError(f"PairwiseDistances: '{properties.virial}' must be a contiguous float64 [n_sys, 3, 3] "
                                 f"tensor on {R.device}")
            idx_m = idx_m if idx_m.dtype == torch.int64 else idx_m.long()
            holder.update(virial=virial, sys_ptr=ops.segment_ptr(idx_m.contiguous(), virial.shape[0]))
            inputs[properties.virial_sink] = holder
        inputs[properties.Rij] = K.PairwiseDistancesFunction.apply(R, offsets, holder)
        return inputs


class Atomwise(nn.Module):
    """Atom-wise MLP + per-system sum (atomwise.py:14-88).  The fused kernel path covers the reference default
    ``n_out=1, n_layers=2`` head with ``aggregation_mode in {"sum","avg",None}``."""

    def __init__(self, n_in: int, n_out: int = 1, n_hidden: Optional[Union[int, Sequence[int]]] = None,
                 n_layers: int = 2, activation: Callable = F.silu, aggregation_mode: str = "sum",
                 output_key: str = "y", per_atom_output_key: Optional[str] = None):
        super().__init__()
        self.output_key = output_key
        self.model_outputs = [output_key]
        self.per_atom_output_key = per_atom_output_key
        if self.per_atom_output_key is not None:
            self.model_outputs.append(self.per_atom_output_key)
        self.n_out = n_out
        if aggregation_mode is None and self.per_atom_output_key is None:
            raise ValueError("If `aggregation_mode` is None, `per_atom_output_key` needs to be set,"
                             + " since no accumulated output will be returned!")
        self.outnet = snn.build_mlp(n_in=n_in, n_out=n_out, n_hidden=n_hidden, n_layers=n_layers,
                                    activation=activation)
        self.aggregation_mode = aggregation_mode
        self.activation = activation
        self._pk, self._sig = None, None

    def _pack(self):
        params = list(self.outnet.parameters())
        sig = K.ParamPack.signature(params)
        if self._sig != sig:
            l0, l1 = self.outnet[0], self.outnet[1]
            self._pk = dict(l0=ops.Lin(l0.weight, l0.bias),
                            w1=l1.weight.detach().reshape(-1).contiguous(),
                            b1=l1.bias.detach().contiguous() if l1.bias is not None else None)
            self._sig = sig
        return self._pk

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if snn.use_training_path(self):           # training: differentiable ATen path (functional_torch), SURVEY 8 f3
            from .. import functional_torch as T

            return T.atomwise(self, inputs)
        if self.n_out != 1 or len(self.outnet) != 2:
            raise NotImplementedError("schnetpack_b200.Atomwise: fused head covers n_out=1, n_layers=2")
        q = inputs["scalar_representation"]
        idx_m, n_mol = None, 0
        if self.aggregation_mode is not None:
            idx_m = inputs[properties.idx_m]
            if properties.n_atoms in inputs:      # number of systems without the reference's host sync
                n_mol = int(inputs[properties.n_atoms].shape[0])
            else:                                 # atomwise.py:80 (forces a device->host read)
                n_mol = int(idx_m[-1]) + 1
        y, e = K.AtomwiseFunction.apply(q, dict(pack=self._pack(), idx_m=idx_m, n_mol=n_mol,
                                                act=snn.activation_code(self.activation)))
        if self.per_atom_output_key is not None:
            inputs[self.per_atom_output_key] = y.unsqueeze(-1)
        if self.aggregation_mode is not None:
            if self.aggregation_mode == "avg":
                e = e / inputs[properties.n_atoms]
            inputs[self.output_key] = e
        else:
            inputs[self.output_key] = y.unsqueeze(-1)
        return inputs


class Strain(nn.Module):
    """Adds a zero strain leaf and applies (1 + strain^T) to cell, positions and offsets so that ``Forces(calc_stress=True)``
    can differentiate the energy with respect to it (response.py:434-464).  Plain tensor algebra on the device; the
    derivative reaches the strain through the positions / offsets gradients of ``PairwiseDistances``."""

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        cell = inputs[properties.cell].reshape(-1, 3, 3)
        eps = torch.zeros_like(cell).requires_grad_()
        inputs[properties.strain] = eps
        eps_t = eps.transpose(1, 2)
        inputs[properties.cell] = cell + cell @ eps_t
        per_atom = eps_t[inputs[properties.idx_m]]
        R = inputs[properties.R]
        inputs[properties.R] = R + torch.einsum("na,nab->nb", R, per_atom)
        off = inputs[properties.offsets]
        inputs[properties.offsets] = off + torch.einsum("ea,eab->eb", off, per_atom[inputs[properties.idx_i]])
        return inputs


class Forces(nn.Module):
    """forces = -dE/dR, stress = dE/dstrain / V via autograd over the kernel pipeline (response.py:18-92)."""

    def __init__(self, calc_forces: bool = True, calc_stress: bool = False, energy_key: str = properties.energy,
                 force_key: str = properties.forces, stress_key: str = properties.stress):
        super().__init__()
        self.calc_forces = calc_forces
        self.calc_stress = calc_stress
        self.energy_key = energy_key
        self.force_key = force_key
        self.stress_key = stress_key
        self.model_outputs = []
        if calc_forces:
            self.model_outputs.append(force_key)
        if calc_stress:
            self.model_outputs.append(stress_key)
        self.required_derivatives = []
        if self.calc_forces:
            self.required_derivatives.append(properties.R)
        if self.calc_stress:
            self.required_derivatives.append(properties.strain)

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        Epred = inputs[self.energy_key]
        go: List[Optional[torch.Tensor]] = [torch.ones_like(Epred)]
        grads = grad([Epred], [inputs[prop] for prop in self.required_derivatives], grad_outputs=go,
                     create_graph=self.training)
        if self.calc_forces:
            dEdR = grads[0]
            if dEdR is None:
                dEdR = torch.zeros_like(inputs[properties.R])
            inputs[self.force_key] = -dEdR
        if self.calc_stress:
            stress = grads[-1]
            if stress is None:
                stress = torch.zeros_like(inputs[properties.cell])
            cell = inputs[properties.cell].reshape(-1, 3, 3)
            volume = torch.sum(cell[:, 0, :] * torch.cross(cell[:, 1, :], cell[:, 2, :], dim=1), dim=1,
                               keepdim=True)[:, :, None]
            inputs[self.stress_key] = stress / volume
        return inputs


class _GatedHead(nn.Module):
    """Kernel plumbing shared by DipoleMoment and Polarizability: weight packing, the limits of the tail kernel and the
    per-system index arrays (the number of systems comes from ``_n_atoms``, so there is no host read)."""

    MAX_F = 256     # Fi and gating width of the last block (csrc/equivariant.cu HT_MAXF)

    def _pack(self) -> K.HeadPack:
        params = list(self.outnet.parameters())
        if self._pk.stale(params):
            self._pk.build(self)
            self._pk.mark(params)
        return self._pk

    def _apply(self, fn, *a, **k):  # .to()/.cuda()/.float(): drop the cached kernel-side weights
        self._pk = K.HeadPack()
        return super()._apply(fn, *a, **k)

    def _check_kernel_shape(self):
        for m in self.modules():
            if isinstance(m, snn.Dense):
                snn.activation_code(m.activation)
        if self._vector:
            last = self.outnet[-1]
            if last.n_sin > self.MAX_F or last.n_hidden > self.MAX_F:
                raise NotImplementedError(f"{type(self).__name__}: the last gated block's input width ({last.n_sin}) and "
                                          f"gating width ({last.n_hidden}) must be <= {self.MAX_F} for the CUDA kernels")
            for blk in self.outnet:
                snn.activation_code(blk.sactivation)

    def _holder(self, inputs, kind, correct=False, magnitude=False, want_charges=False):
        if properties.n_atoms not in inputs:
            raise KeyError(f"{type(self).__name__} needs '{properties.n_atoms}' (the number of systems, without a host read)")
        n_sys = int(inputs[properties.n_atoms].shape[0])
        idx_m = inputs[properties.idx_m]
        idx_m = (idx_m if idx_m.dtype == torch.int64 else idx_m.long()).contiguous()
        tq = None
        if correct and properties.total_charge in inputs:
            tq = inputs[properties.total_charge].detach().to(torch.float32).contiguous()
        return dict(pack=self._pack(), kind=kind, idx_m=idx_m, sys_ptr=ops.segment_ptr(idx_m, n_sys), n_sys=n_sys,
                    total_charge=tq, correct=bool(correct), magnitude=bool(magnitude), want_charges=bool(want_charges))


class DipoleMoment(_GatedHead):
    """atomistic/atomwise.py:91-213 -- dipole moments from latent partial charges and, with
    ``use_vector_representation``, atomic dipoles from the vector features.  Output [B, 3] ([B] with
    ``predict_magnitude``), charges [N, 1] with ``return_charges``.

    ``eval()``: the gated blocks / the charge MLP and the per-system assembly run on the kernels of csrc/equivariant.cu
    (fp64 segmented sums, no atomics, no host read), differentiable with respect to positions and the representation
    (dipole derivatives through ``torch.autograd.grad``).  The charges output is differentiable when
    ``differentiable_charges`` is set -- ``NeuralNetworkPotential`` sets it when an ``EnergyCoulomb`` of the model reads
    these charges, so that its energy has the ``dE/dq dq/dR`` force term; otherwise the charges are a plain output and the
    reverse is exactly that of the dipole.
    ``train()`` with trainable parameters under grad mode: the ATen formula of ``functional_torch``."""

    def __init__(self, n_in: int, n_hidden: Optional[Union[int, Sequence[int]]] = None, n_layers: int = 2,
                 activation: Callable = F.silu, predict_magnitude: bool = False, return_charges: bool = False,
                 dipole_key: str = properties.dipole_moment, charges_key: str = properties.partial_charges,
                 correct_charges: bool = True, use_vector_representation: bool = False):
        super().__init__()
        self.dipole_key = dipole_key
        self.charges_key = charges_key
        self.return_charges = return_charges
        self.model_outputs = [dipole_key]
        if self.return_charges:
            self.model_outputs.append(charges_key)
        self.predict_magnitude = predict_magnitude
        self.use_vector_representation = use_vector_representation
        self.correct_charges = correct_charges
        self.differentiable_charges = False
        if use_vector_representation:
            self.outnet = snn.build_gated_equivariant_mlp(n_in=n_in, n_out=1, n_hidden=n_hidden, n_layers=n_layers,
                                                          activation=activation, sactivation=activation)
        else:
            self.outnet = snn.build_mlp(n_in=n_in, n_out=1, n_hidden=n_hidden, n_layers=n_layers, activation=activation)
        self._pk = K.HeadPack()

    @property
    def _vector(self) -> bool:
        return self.use_vector_representation

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if snn.use_training_path(self):
            from .. import functional_torch as T

            return T.dipole_moment(self, inputs)
        self._check_kernel_shape()
        h = self._holder(inputs, ops.HEAD_DIPOLE, self.correct_charges, self.predict_magnitude, self.return_charges)
        h["diff_charges"] = self.return_charges and self.differentiable_charges
        s, R = inputs["scalar_representation"], inputs[properties.R]
        if self.use_vector_representation:
            y, charges = K.GatedHeadFunction.apply(s, inputs["vector_representation"], R, h)
        else:
            y, charges = K.ScalarDipoleFunction.apply(s, R, h)
        if self.return_charges:
            inputs[self.charges_key] = charges.unsqueeze(-1)
        inputs[self.dipole_key] = y
        return inputs


class Polarizability(_GatedHead):
    """atomistic/atomwise.py:216-293 -- rank-factorised polarizability alpha_m = sum alpha_i I + sum (nu_i (x) R_i +
    R_i (x) nu_i), output [B, 3, 3]; needs scalar and vector features.  Kernel and training paths as ``DipoleMoment``."""

    def __init__(self, n_in: int, n_hidden: Optional[Union[int, Sequence[int]]] = None, n_layers: int = 2,
                 activation: Callable = F.silu, polarizability_key: str = properties.polarizability):
        super().__init__()
        self.n_in = n_in
        self.n_layers = n_layers
        self.n_hidden = n_hidden
        self.polarizability_key = polarizability_key
        self.model_outputs = [polarizability_key]
        self.outnet = snn.build_gated_equivariant_mlp(n_in=n_in, n_out=1, n_hidden=n_hidden, n_layers=n_layers,
                                                      activation=activation, sactivation=activation)
        self.requires_dr = False
        self.requires_stress = False
        self._pk = K.HeadPack()

    _vector = True

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if snn.use_training_path(self):
            from .. import functional_torch as T

            return T.polarizability(self, inputs)
        self._check_kernel_shape()
        h = self._holder(inputs, ops.HEAD_POLAR)
        alpha, _ = K.GatedHeadFunction.apply(inputs["scalar_representation"], inputs["vector_representation"],
                                             inputs[properties.R], h)
        inputs[self.polarizability_key] = alpha
        return inputs


from .pair_terms import (Aggregation, CoulombPotential, DampedCoulombPotential, EnergyCoulomb,  # noqa: E402
                         EnergyEwald, EnergyEwaldError, EnergyPME, FilterShortRange, ZBLRepulsionEnergy, pme_mesh,
                         use_pme)
