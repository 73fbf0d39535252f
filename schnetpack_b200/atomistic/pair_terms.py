"""Physics add-ons of PhysNet-style potentials on the kernels of csrc/pair_energy.cu and csrc/ewald.cu: ZBL repulsion
(atomistic/nuclear_repulsion.py:13-108), the Coulomb energy of point charges with its potentials
(atomistic/electrostatic.py:14-152), the Ewald sum of periodic systems (atomistic/electrostatic.py:155-375),
``Aggregation`` (atomistic/aggregation.py) and a capture-safe ``FilterShortRange``
(atomistic/distances.py:29-57).  Constructor signatures, parameters, buffers and ``state_dict`` keys are the
reference's.

``eval()``: every pair term is one ``spk_pair_energy_fwd`` (fp64 per-system sums in a fixed order, no atomics, no host
read: the number of systems comes from ``_n_atoms``) and its reverse gives dE/dr_ij and, for Coulomb, dE/dq -- which
reaches the charge head through the differentiable ``charges`` output of ``DipoleMoment``.  ``train()`` with trainable
parameters under grad mode: the ATen formulas of ``functional_torch``."""
from __future__ import annotations

import contextlib
import math
from typing import Callable, Dict, List, Optional, Union

import torch
import torch.nn as nn

from .. import functional as K
from .. import nn as snn
from .. import ops
from .. import properties
from ..units import convert_units

__all__ = ["ZBLRepulsionEnergy", "CoulombPotential", "DampedCoulombPotential", "EnergyCoulomb", "EnergyEwald", "EnergyPME",
           "pme_mesh", "use_pme",
           "EnergyEwaldError", "Aggregation", "FilterShortRange", "check_padded_pair_terms", "check_ewald_cells", "padded_list_cutoff",
           "check_short_range_cutoff", "link_charges"]


def _softplus_inverse(x: torch.Tensor) -> torch.Tensor:
    """nn/utils.py softplus_inverse: x + log(-expm1(-x))."""
    x = torch.as_tensor(x)
    return x + torch.log(-torch.expm1(-x))


class _HostScalars:
    """Python floats of small buffers (ke, cutoff, shift, switch limits): one host read per change of a buffer (loading a
    state dict), none on the evaluation path."""

    def __init__(self):
        self._key, self._vals = None, None

    def get(self, *bufs: Optional[torch.Tensor]):
        key = tuple((b.data_ptr(), b._version) if b is not None else None for b in bufs)
        if key != self._key:
            self._vals = tuple(float(b.reshape(-1)[0]) if b is not None else None for b in bufs)
            self._key = key
        return self._vals


def _systems(inputs: Dict[str, torch.Tensor], who: str):
    if properties.n_atoms not in inputs:
        raise KeyError(f"{who} needs '{properties.n_atoms}' (the number of systems, without a host read)")
    n_sys = int(inputs[properties.n_atoms].shape[0])
    idx_m = inputs[properties.idx_m]
    idx_m = (idx_m if idx_m.dtype == torch.int64 else idx_m.long()).contiguous()
    return idx_m, n_sys, ops.segment_ptr(idx_m, n_sys)


def _edges(inputs: Dict[str, torch.Tensor], key_r: str, key_i: str, key_j: str, n_atoms: int):
    idx_i, idx_j = inputs[key_i], inputs[key_j]
    idx_i = (idx_i if idx_i.dtype == torch.int64 else idx_i.long()).contiguous()
    idx_j = (idx_j if idx_j.dtype == torch.int64 else idx_j.long()).contiguous()
    return inputs[key_r], idx_i, idx_j, ops.get_graph(idx_i, idx_j, n_atoms)


def _short_range_d_max(inputs: Dict[str, torch.Tensor]) -> Optional[float]:
    src = inputs.get(properties.short_range_cutoff)
    return None if src is None else float(src)


def _cosine_cutoff_radius(cutoff_fn, who: str) -> Optional[float]:
    if cutoff_fn is None:
        return None
    if type(cutoff_fn).__name__ != "CosineCutoff":
        raise NotImplementedError(f"{who}: cutoff {type(cutoff_fn).__name__} has no CUDA kernel (CosineCutoff or None)")
    return cutoff_fn.value() if isinstance(cutoff_fn, snn.CosineCutoff) else float(cutoff_fn.cutoff)


class ZBLRepulsionEnergy(nn.Module):
    """nuclear_repulsion.py:13-108.  The kernel reads the raw parameters from device memory and applies softplus and the
    L1 normalisation there, so a captured graph sees parameter updates.  ``cutoff_fn`` in {None, CosineCutoff}."""

    def __init__(self, energy_unit: Union[str, float], position_unit: Union[str, float], output_key: str,
                 trainable: bool = True, cutoff_fn: Optional[Callable] = None):
        super().__init__()
        energy_units = convert_units("Ha", energy_unit)
        position_units = convert_units("Bohr", position_unit)
        ke = energy_units * position_units
        self.register_buffer("ke", torch.tensor(ke))
        self.cutoff_fn = cutoff_fn
        self.output_key = output_key
        a_div = _softplus_inverse(torch.tensor([1.0 / (position_units * 0.8854)]))
        a_pow = _softplus_inverse(torch.tensor([0.23]))
        exponents = _softplus_inverse(torch.tensor([3.19980, 0.94229, 0.40290, 0.20162]))
        coefficients = _softplus_inverse(torch.tensor([0.18175, 0.50986, 0.28022, 0.02817]))
        self.a_pow = nn.Parameter(a_pow, requires_grad=trainable)
        self.a_div = nn.Parameter(a_div, requires_grad=trainable)
        self.coefficients = nn.Parameter(coefficients, requires_grad=trainable)
        self.exponents = nn.Parameter(exponents, requires_grad=trainable)
        self._host = _HostScalars()

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if snn.use_training_path(self):
            from .. import functional_torch as T

            return T.zbl_repulsion(self, inputs)
        rc = _cosine_cutoff_radius(self.cutoff_fn, "ZBLRepulsionEnergy")
        (ke,) = self._host.get(self.ke)
        Z = inputs[properties.Z]
        Z = (Z if Z.dtype == torch.int64 else Z.long()).contiguous()
        idx_m, n_sys, sys_ptr = _systems(inputs, "ZBLRepulsionEnergy")
        r_ij, idx_i, idx_j, graph = _edges(inputs, properties.Rij, properties.idx_i, properties.idx_j, Z.shape[0])
        params, keep = ops.pair_params(ops.PAIR_ZBL, ke, cutoff=rc, d_max=_short_range_d_max(inputs),
                                       zbl=(self.a_pow, self.a_div, self.coefficients, self.exponents))
        holder = dict(params=params, keep=keep, idx_i=idx_i, idx_j=idx_j, Z=Z, idx_m=idx_m, graph=graph,
                      sys_ptr=sys_ptr, n_sys=n_sys)
        inputs[self.output_key] = K.PairEnergyFunction.apply(r_ij, None, holder)
        return inputs


class CoulombPotential(nn.Module):
    """electrostatic.py:14-23: 1 / d."""

    def forward(self, d_ij: torch.Tensor) -> torch.Tensor:
        return 1.0 / d_ij


class DampedCoulombPotential(nn.Module):
    """electrostatic.py:26-57: f_sw / sqrt(d^2 + 1) + (1 - f_sw) / d with ``switch_fn`` a ``SwitchFunction``."""

    def __init__(self, switch_fn: nn.Module):
        super().__init__()
        self.switch_fn = switch_fn

    def forward(self, d_ij: torch.Tensor) -> torch.Tensor:
        potential = 1.0 / d_ij
        damped = 1.0 / torch.sqrt(d_ij ** 2 + 1)
        f_switch = self.switch_fn(d_ij)
        return f_switch * damped + (1 - f_switch) * potential


class EnergyCoulomb(nn.Module):
    """electrostatic.py:60-152: Coulomb energy of the charges under ``charges_key`` by direct summation over the
    long-range (``use_neighbors_lr``) or the standard neighbour list, shifted to zero at ``cutoff`` when given.  The
    potential is ``CoulombPotential`` or ``DampedCoulombPotential`` with a ``SwitchFunction``."""

    def __init__(self, energy_unit: Union[str, float], position_unit: Union[str, float], coulomb_potential: nn.Module,
                 output_key: str, charges_key: str = properties.partial_charges, use_neighbors_lr: bool = True,
                 cutoff: Optional[float] = None):
        super().__init__()
        ke = convert_units("Ha", energy_unit) * convert_units("Bohr", position_unit)
        self.register_buffer("ke", torch.Tensor([ke]))
        self.coulomb_potential = coulomb_potential
        self.charges_key = charges_key
        self.output_key = output_key
        self.model_outputs = [output_key]
        self.use_neighbors_lr = use_neighbors_lr
        if cutoff is not None:
            cutoff = torch.tensor(cutoff)
            shift = self.coulomb_potential(cutoff).detach()
            self.register_buffer("cutoff", cutoff)
            self.register_buffer("shift", shift)
        else:
            self.cutoff = None
            self.shift = None
        self._host = _HostScalars()

    def _kind(self):
        name = type(self.coulomb_potential).__name__
        if name == "CoulombPotential":
            return ops.PAIR_COULOMB, None
        if name == "DampedCoulombPotential":
            sw = self.coulomb_potential.switch_fn
            if type(sw).__name__ != "SwitchFunction":
                raise NotImplementedError(f"EnergyCoulomb: switch {type(sw).__name__} has no CUDA kernel")
            return ops.PAIR_DAMPED_COULOMB, sw
        raise NotImplementedError(f"EnergyCoulomb: potential {name} has no CUDA kernel "
                                  "(CoulombPotential, DampedCoulombPotential)")

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if self.training and torch.is_grad_enabled():      # no parameters: the charges carry the training graph
            from .. import functional_torch as T

            return T.energy_coulomb(self, inputs)
        kind, sw = self._kind()
        ke, rc, shift, s_on, s_off = self._host.get(self.ke, self.cutoff, self.shift,
                                                    sw.switch_on if sw is not None else None,
                                                    sw.switch_off if sw is not None else None)
        q = inputs[self.charges_key].reshape(-1)
        if q.dtype != torch.float32:
            raise TypeError("EnergyCoulomb: the charges must be float32 on the kernel path")
        idx_m, n_sys, sys_ptr = _systems(inputs, "EnergyCoulomb")
        if self.use_neighbors_lr:
            r_ij, idx_i, idx_j, graph = _edges(inputs, properties.Rij_lr, properties.idx_i_lr, properties.idx_j_lr,
                                               q.shape[0])
            d_max = None
        else:
            r_ij, idx_i, idx_j, graph = _edges(inputs, properties.Rij, properties.idx_i, properties.idx_j, q.shape[0])
            d_max = _short_range_d_max(inputs)
        params, keep = ops.pair_params(kind, ke, cutoff=rc, shift=shift or 0.0, switch_on=s_on or 0.0,
                                       switch_off=s_off or 0.0, d_max=d_max)
        holder = dict(params=params, keep=keep, idx_i=idx_i, idx_j=idx_j, idx_m=idx_m, graph=graph, sys_ptr=sys_ptr,
                      n_sys=n_sys)
        inputs[self.output_key] = K.PairEnergyFunction.apply(r_ij, q, holder)
        return inputs


class EnergyEwaldError(Exception):
    """electrostatic.py:155-156: raised for a system whose cell has zero volume."""


class _EwaldSum(nn.Module):
    """What ``EnergyEwald`` and ``EnergyPME`` share: the buffers ``ke`` and ``alpha``, the keys, the list choice and the
    screen, and the kernel inputs of the real-space and self terms (``_kernel_inputs``)."""

    # the cutoff of the padded neighbour list being evaluated (set by ``padded_list_cutoff``), else None
    list_cutoff: Optional[float] = None

    def __init__(self, alpha: float, energy_unit: Union[str, float], position_unit: Union[str, float], output_key: str,
                 charges_key: str, use_neighbors_lr: bool, screening_fn: Optional[nn.Module]):
        super().__init__()
        ke = convert_units("Ha", energy_unit) * convert_units("Bohr", position_unit)
        self.register_buffer("ke", torch.Tensor([ke]))
        self.charges_key = charges_key
        self.output_key = output_key
        self.model_outputs = [output_key]
        self.use_neighbors_lr = use_neighbors_lr
        self.screening_fn = screening_fn
        self.register_buffer("alpha", torch.Tensor([alpha]))
        self._host = _HostScalars()

    def _screen(self):
        sw = self.screening_fn
        if sw is None:
            return None
        if type(sw).__name__ != "SwitchFunction":
            raise NotImplementedError(f"{type(self).__name__}: screening_fn {type(sw).__name__} has no CUDA kernel "
                                      "(SwitchFunction or None)")
        return sw

    def _kernel_inputs(self, inputs: Dict[str, torch.Tensor]):
        """-> (r_ij, q, cell, holder) of the real-space launch pair and the reciprocal and self terms"""
        who = type(self).__name__
        sw = self._screen()
        ke, alpha, s_on, s_off = self._host.get(self.ke, self.alpha, sw.switch_on if sw is not None else None,
                                                sw.switch_off if sw is not None else None)
        q = inputs[self.charges_key].reshape(-1)
        if q.dtype != torch.float32:
            raise TypeError(f"{who}: the charges must be float32 on the kernel path")
        idx_m, n_sys, sys_ptr = _systems(inputs, who)
        if self.use_neighbors_lr:
            r_ij, idx_i, idx_j, graph = _edges(inputs, properties.Rij_lr, properties.idx_i_lr, properties.idx_j_lr,
                                               q.shape[0])
            d_max = None
        else:
            r_ij, idx_i, idx_j, graph = _edges(inputs, properties.Rij, properties.idx_i, properties.idx_j, q.shape[0])
            d_max = _short_range_d_max(inputs)
        if self.list_cutoff is not None:
            d_max = self.list_cutoff if d_max is None else min(d_max, self.list_cutoff)
        params, keep = ops.pair_params(ops.PAIR_EWALD_REAL, ke, switch_on=s_on or 0.0, switch_off=s_off or 0.0,
                                       d_max=d_max, alpha=alpha)
        holder = dict(params=params, keep=keep, idx_i=idx_i, idx_j=idx_j, idx_m=idx_m, graph=graph, sys_ptr=sys_ptr,
                      n_sys=n_sys, ke=ke, alpha=alpha, sink=inputs.get(properties.virial_sink))
        cell = inputs[properties.cell]
        if cell.dtype != torch.float32 or cell.numel() != 9 * n_sys:
            raise TypeError(f"{who}: the cell must be float32 [{n_sys}, 3, 3] on the kernel path")
        return r_ij, q, cell, holder


class EnergyEwald(_EwaldSum):
    """electrostatic.py:159-375: Coulomb energy of the charges under ``charges_key`` in a periodic box by Ewald summation,
    E = E_real + E_rec - E_self.  The real-space term runs over every pair of the long-range (``use_neighbors_lr``) or the
    standard list, screened by ``1 - screening_fn(d)`` when a ``SwitchFunction`` is given; the reciprocal term over the
    integer triples n of the ``kvecs`` buffer (the full sphere |n|^2 <= k_max^2 + 2, n != 0) with k = 2 pi n h^-T.
    ``alpha`` is the square of the usual splitting parameter.  The cell is inverted, so triclinic cells work.

    ``eval()``: one ``EwaldFunction`` (a pair-energy launch pair for the real space, four launches for the reciprocal and
    self terms, no host read: the number of systems comes from ``_n_atoms``), differentiable with respect to r_ij, the
    positions, the charges and the cell.  A system of zero volume gets a NaN energy there (the check would be a host read);
    ``DeviceMD`` and ``DeviceLBFGS`` check the cells at construction and raise ``EnergyEwaldError`` as the reference does.
    Inside ``padded_list_cutoff(model, cutoff)`` (``DeviceMD`` and ``DeviceLBFGS`` evaluate in it) the real-space term masks
    d > the list cutoff, which drops the padding pairs of a fixed-capacity list and nothing else.  ``train()`` under grad mode: the ATen formulas of
    ``functional_torch``."""

    def __init__(self, alpha: float, k_max: int, energy_unit: Union[str, float], position_unit: Union[str, float],
                 output_key: str, charges_key: str = properties.partial_charges, use_neighbors_lr: bool = True,
                 screening_fn: Optional[nn.Module] = None):
        super().__init__(alpha, energy_unit, position_unit, output_key, charges_key, use_neighbors_lr, screening_fn)
        self.k_max = k_max
        self.register_buffer("kvecs", self._generate_kvecs())

    def _generate_kvecs(self) -> torch.Tensor:
        """electrostatic.py:209-224."""
        krange = torch.arange(0, self.k_max + 1, dtype=self.alpha.dtype)
        krange = torch.cat([krange, -krange[1:]])
        kvecs = torch.cartesian_prod(krange, krange, krange)
        norm = torch.sum(kvecs ** 2, dim=1)
        kvecs = kvecs[norm <= self.k_max ** 2 + 2, :]
        norm = norm[norm <= self.k_max ** 2 + 2]
        return kvecs[norm != 0, :]

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if self.training and torch.is_grad_enabled():      # no parameters: the charges carry the training graph
            from .. import functional_torch as T

            return T.energy_ewald(self, inputs)
        r_ij, q, cell, holder = self._kernel_inputs(inputs)
        kvecs = self.kvecs if self.kvecs.dtype == torch.float32 else self.kvecs.float()
        holder["kvecs"] = kvecs.contiguous()
        inputs[self.output_key] = K.EwaldFunction.apply(r_ij, inputs[properties.R], q, cell, holder)
        return inputs


PME_FFT_PRIMES = (2, 3, 5, 7)


def _fft_friendly(n: int) -> bool:
    for p in PME_FFT_PRIMES:
        while n % p == 0:
            n //= p
    return n == 1


def pme_mesh(cell: torch.Tensor, spacing: float, order: int = 4) -> tuple:
    """The smallest mesh (n1, n2, n3) whose sizes have no prime factor above 7 and give every system of the batch a
    spacing |h_a| / n_a <= ``spacing`` along each lattice vector h_a, and at least ``order`` points per axis."""
    h = torch.as_tensor(cell, dtype=torch.float64).detach().cpu().reshape(-1, 3, 3)
    lengths = torch.linalg.norm(h, dim=2).amax(0)
    out = []
    for length in lengths.tolist():
        n = max(int(order), int(math.ceil(length / float(spacing) - 1e-9)))
        while not _fft_friendly(n):
            n += 1
        out.append(n)
    return tuple(out)


class EnergyPME(_EwaldSum):
    """Coulomb energy of the charges under ``charges_key`` in a periodic box by smooth particle-mesh Ewald (Essmann et
    al., J. Chem. Phys. 103, 8577 (1995)): E = E_real + E_rec - E_self, where E_real and E_self are ``EnergyEwald``'s (the
    same kernels, screen and list handling) and E_rec = ke (2 pi / V) sum_k f_k |b(k)|^2 |Q^(k)|^2 over the mesh
    frequencies k != 0 (a Nyquist frequency of an even axis left out), with Q the B-spline charge mesh of order ``order``
    in fractional coordinates.  The cost is O(N order^3 + M log M) for M mesh points instead of Ewald's O(N K), so PME
    wins on large boxes and Ewald on small ones.  ``mesh`` = (n1, n2, n3) is one mesh for every system of a batch
    (``pme_mesh`` picks one from a spacing); ``order`` in {4, 6, 8}, each axis at least ``order`` points.

    The buffers and keys are ``EnergyEwald``'s without ``kvecs``; ``use_pme`` swaps the modules of a converted model.  No
    background term for non-neutral systems, NaN for a zero-volume cell (the drivers refuse one at construction).  The
    kernel path only: ``train()`` under grad mode raises (train with ``EnergyEwald``)."""

    def __init__(self, alpha: float, mesh, order: int, energy_unit: Union[str, float], position_unit: Union[str, float],
                 output_key: str, charges_key: str = properties.partial_charges, use_neighbors_lr: bool = True,
                 screening_fn: Optional[nn.Module] = None):
        super().__init__(alpha, energy_unit, position_unit, output_key, charges_key, use_neighbors_lr, screening_fn)
        mesh = tuple(int(n) for n in mesh)
        if int(order) not in ops.PME_ORDERS:
            raise ValueError(f"EnergyPME: order {order} is not one of {ops.PME_ORDERS}")
        if len(mesh) != 3 or any(n < int(order) for n in mesh):
            raise ValueError(f"EnergyPME: mesh {mesh} must have 3 axes of at least order = {order} points (an atom's "
                             "support along an axis must be distinct mesh points)")
        self.mesh = mesh
        self.order = int(order)

    def extra_repr(self) -> str:
        return f"mesh={self.mesh}, order={self.order}"

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if self.training and torch.is_grad_enabled():
            raise NotImplementedError("EnergyPME has no training path; train with EnergyEwald and switch with use_pme")
        r_ij, q, cell, holder = self._kernel_inputs(inputs)
        holder["mesh"], holder["order"] = self.mesh, self.order
        inputs[self.output_key] = K.PMEFunction.apply(r_ij, inputs[properties.R], q, cell, holder)
        return inputs


def use_pme(model: nn.Module, mesh, order: int) -> nn.Module:
    """Replace every ``EnergyEwald`` of ``model`` by an ``EnergyPME`` with the same ke, alpha, keys, list choice and
    screen, in place, and return the model: train and convert with Ewald, then run MD or relaxation with PME."""
    for parent in list(model.modules()):
        for name, child in list(parent.named_children()):
            if type(child).__name__ != "EnergyEwald":
                continue
            new = EnergyPME(1.0, mesh, order, 1.0, 1.0, child.output_key, charges_key=child.charges_key,
                            use_neighbors_lr=child.use_neighbors_lr, screening_fn=child.screening_fn)
            new.ke = child.ke.detach().clone()
            new.alpha = child.alpha.detach().clone()
            setattr(parent, name, new.to(child.ke.device).train(child.training))
    return model


class Aggregation(nn.Module):
    """aggregation.py: the sum of several per-system outputs."""

    def __init__(self, keys: List[str], output_key: str = "y"):
        super().__init__()
        self.keys: List[str] = list(keys)
        self.output_key = output_key
        self.model_outputs = [output_key]

    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        inputs[self.output_key] = torch.stack([inputs[key] for key in self.keys]).sum(0)
        return inputs


class FilterShortRange(nn.Module):
    """distances.py:29-57 without the compaction.  The long-range keys (``_Rij_lr``, ``_idx_i_lr``, ``_idx_j_lr``) alias
    the full list (no copy); the short-range keys keep the full list too, and ``short_range_cutoff`` is recorded in the
    batch (``properties.short_range_cutoff``).  Pair terms that read the short list apply it as a distance mask
    d <= short_range_cutoff, and the representation gives exactly zero for edges beyond its own cutoff, which
    ``NeuralNetworkPotential`` checks is at most ``short_range_cutoff``.  So the result is the reference's, without a
    host sync or a data-dependent shape; the price is that the representation iterates over the long-range edges too.

    ``train()`` under grad mode: the reference's exact compaction (``torch.nonzero``)."""

    def __init__(self, short_range_cutoff: float):
        super().__init__()
        self.short_range_cutoff = short_range_cutoff

    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if self.training and torch.is_grad_enabled():
            from .. import functional_torch as T

            return T.filter_short_range(self, inputs)
        inputs[properties.Rij_lr] = inputs[properties.Rij]
        inputs[properties.idx_i_lr] = inputs[properties.idx_i]
        inputs[properties.idx_j_lr] = inputs[properties.idx_j]
        inputs[properties.short_range_cutoff] = torch.tensor(float(self.short_range_cutoff), dtype=torch.float64)
        return inputs


def _representation_cutoff(rep) -> Optional[float]:
    cf = getattr(rep, "cutoff_fn", None)
    if cf is None:
        return None
    return cf.value() if isinstance(cf, snn.CosineCutoff) else float(cf.cutoff)


def check_short_range_cutoff(representation: nn.Module, input_modules) -> None:
    """A ``FilterShortRange`` keeps the full list under the short-range keys; that is exact only when the
    representation's own cutoff removes every edge beyond ``short_range_cutoff``."""
    rc = _representation_cutoff(representation)
    for m in input_modules:
        if type(m).__name__ == "FilterShortRange" and rc is not None and rc > float(m.short_range_cutoff):
            raise ValueError(f"FilterShortRange: the representation's cutoff ({rc}) exceeds short_range_cutoff "
                             f"({m.short_range_cutoff}); the short-range list keeps every edge, so the representation "
                             "would see pairs the reference filters out")


def check_padded_pair_terms(model: nn.Module, list_cutoff: float, who: str) -> None:
    """The padded fixed-capacity neighbour list of the device drivers puts inert self pairs at distance 2 list_cutoff.
    They are inert only for terms that vanish beyond a cutoff no larger than the list's.  ``EnergyEwald`` has no cutoff
    (its real-space term is q_i^2 erfc(sqrt(alpha) d) / d on a padding pair); the drivers evaluate it inside
    ``padded_list_cutoff``, where it masks d > list_cutoff, which is exact because an unpadded list at that cutoff holds
    the same pairs."""
    for m in model.modules():
        name = type(m).__name__
        if name == "ZBLRepulsionEnergy":
            rc = _cosine_cutoff_radius(m.cutoff_fn, who) if m.cutoff_fn is not None else None
            if rc is None:
                raise ValueError(f"{who}: ZBLRepulsionEnergy without cutoff_fn would add the padding pairs of the "
                                 "fixed-capacity neighbour list; give it a CosineCutoff")
            if rc > list_cutoff:
                raise ValueError(f"{who}: ZBLRepulsionEnergy cutoff {rc} exceeds the neighbour-list cutoff {list_cutoff}")
        elif name == "EnergyCoulomb":
            if m.cutoff is None:
                raise ValueError(f"{who}: EnergyCoulomb without a cutoff would add the padding pairs of the "
                                 "fixed-capacity neighbour list; give it a cutoff")
            rc = float(m.cutoff)
            if rc > list_cutoff:
                raise ValueError(f"{who}: EnergyCoulomb cutoff {rc} exceeds the neighbour-list cutoff {list_cutoff}")


@contextlib.contextmanager
def padded_list_cutoff(model: nn.Module, list_cutoff: float):
    """Evaluate ``model`` on a padded fixed-capacity neighbour list of cutoff ``list_cutoff``: every ``EnergyEwald`` or
    ``EnergyPME`` of it
    masks real-space pairs with d > list_cutoff for the duration (the padding self pairs sit at 2 list_cutoff).  A plain
    module attribute, read when the forward is traced, so nothing enters the batch and a captured graph keeps it.  Models
    without either are untouched."""
    mods = [m for m in model.modules() if isinstance(m, _EwaldSum)]
    old = [m.list_cutoff for m in mods]
    for m in mods:
        m.list_cutoff = float(list_cutoff)
    try:
        yield
    finally:
        for m, v in zip(mods, old):
            m.list_cutoff = v


def check_ewald_cells(model: nn.Module, batch: Dict[str, torch.Tensor], who: str) -> None:
    """electrostatic.py:333-336 at the construction of a device driver: raise ``EnergyEwaldError`` when the model has an
    ``EnergyEwald`` or ``EnergyPME`` and a system's cell has (close to) zero volume.  One host read, outside the captured
    step."""
    names = {type(m).__name__ for m in model.modules()} & {"EnergyEwald", "EnergyPME"}
    if not names:
        return
    cell = batch.get(properties.cell)
    if cell is None:
        raise ValueError(f"{who}: {sorted(names)[0]} needs a periodic batch with a '{properties.cell}'")
    v_box = torch.abs(torch.linalg.det(cell.detach().reshape(-1, 3, 3).double()))
    if bool(torch.any(torch.isclose(v_box, torch.zeros_like(v_box)))):
        raise EnergyEwaldError("Simulation box has no volume.")


def link_charges(output_modules) -> None:
    """Make the charges of a ``DipoleMoment`` differentiable when an ``EnergyCoulomb``, ``EnergyEwald`` or ``EnergyPME``
    of the same model reads them (the kernel head returns plain charges otherwise, so models that only output charges are
    unchanged)."""
    keys = {m.charges_key for m in output_modules if type(m).__name__ in ("EnergyCoulomb", "EnergyEwald", "EnergyPME")}
    for m in output_modules:
        if hasattr(m, "differentiable_charges") and m.return_charges and m.charges_key in keys:
            m.differentiable_charges = True
