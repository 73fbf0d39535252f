"""Vibrational analysis on the device: finite-difference Hessians, harmonic frequencies, normal modes and IR / Raman
intensities of every system of a batch (DESIGN.md section 16).

The reference computes the Hessian and the dipole / polarizability derivatives with ``atomistic.Response``: one
``create_graph`` backward pass per Cartesian row (``derivative_from_atomic``, nn/utils.py:65-126), molecule after
molecule.  Its users get frequencies and spectra from ASE's ``Vibrations`` / ``Infrared`` through ``SpkCalculator``, which
displace one coordinate at a time.  ``DeviceVibrations`` evaluates ASE's central differences with first-order forces
only: every displaced copy of every system of the batch is one system of a replica batch, so a few captured steps give
the whole Hessian.  The dipole moments and polarizabilities of the same copies give their derivatives.

Kernels (``csrc/vibrations.cu``): ``spk_vib_displace`` writes the replica positions of a chunk and records the steps
actually taken in fp64; ``spk_vib_assemble`` turns the replica forces into Hessian columns with the Lagrange weights of
those steps; ``spk_vib_finish`` symmetrises and writes the reference's layouts and the mass-weighted blocks.
Eigenvalues, frequencies and intensities are computed in torch fp64, once per ``run``, outside the captured step.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import torch

from . import _lib, ops
from . import properties as P
from .md import _CapturedEvaluation, replicate_batch
from .units import _amu, _e, _hbar, _UNITS

__all__ = ["DeviceVibrations"]

Tensor = torch.Tensor
# replica atoms per chunk when not given: the tape of section 2 for PaiNN 128 x 3 at this size is about 6 GB
DEFAULT_MAX_REPLICA_ATOMS = 262_144
# hbar omega in eV for omega^2 in eV / (Angstrom^2 amu) (ase/vibrations/data.py), and eV per cm^-1
_HBAR_OMEGA = _hbar * 1e10 / math.sqrt(_e * _amu)
_INVCM = _UNITS["invcm"]
_VIB_PROPERTIES = (P.dipole_moment, P.polarizability)


class DeviceVibrations(_CapturedEvaluation):
    """Harmonic vibrational analysis of every system of ``batch`` by ASE's finite differences (``Vibrations`` with
    ``delta`` and ``nfree``; ``Infrared`` for the dipole).  ``batch[_positions]`` is in model units; ``position_conversion``
    and ``energy_conversion`` turn model lengths and energies into Angstrom and eV, ``delta`` is in Angstrom and
    ``masses`` [N] in amu.  ``cutoff`` and ``capacity`` (the pair capacity of ``batch``) size the device neighbour list,
    which is rebuilt on the replica batch in every step.

    Coordinate d = 3 a + k of every system is displaced by -h, +h (``nfree`` = 2) or -2h, -h, +h, +2h (``nfree`` = 4) in
    its own copy of the system.  The copies of ``n_cols`` coordinates form one replica batch of ``n_cols * nfree`` copies
    of ``batch``, evaluated in one captured step; ``run`` replays it ``n_chunks`` times.  ``max_replica_atoms`` bounds
    the replica batch (and so sets ``n_cols``).  ``properties`` (a subset of ``("dipole_moment", "polarizability")``)
    asks for the derivatives of those per-system model outputs from the same evaluations.

    Results after ``run``: ``hessian`` [sum n_m^2, 3, 3] fp64 in model units (energy / length^2) in the layout of the
    reference's ``Response`` (row i n + j, block [a, b] = d2E / dR_ia dR_jb), ``dipole_derivatives`` [N, 3, 3] and
    ``polarizability_derivatives`` [N, 3, 3, 3] (element [i, comp..., dir] = d comp / d R_i,dir, model units), and the
    frequencies, modes and intensities below.  Rigid-body modes are not projected out, as in ASE."""

    def __init__(self, model: torch.nn.Module, batch: Dict[str, Tensor], masses: Tensor, cutoff: float, capacity: int,
                 delta: float = 0.01, nfree: int = 2, position_conversion: float = 1.0, energy_conversion: float = 1.0,
                 properties: Sequence[str] = (), max_replica_atoms: Optional[int] = None, use_graph: bool = True):
        if int(nfree) not in (2, 4):
            raise ValueError(f"DeviceVibrations: nfree must be 2 or 4 (ase/vibrations/vibrations.py), got {nfree}")
        if not float(delta) > 0.0:
            raise ValueError(f"DeviceVibrations: delta must be > 0, got {delta}")
        from .parallel import PartitionedPotential

        if isinstance(model, PartitionedPotential):
            raise NotImplementedError("DeviceVibrations: PartitionedPotential is not supported (one GPU per batch)")
        from .ensemble import members_of

        if members_of(model) is not None:
            raise NotImplementedError("DeviceVibrations: ensembles are not supported; pass a single model")
        properties = list(dict.fromkeys(properties))
        unknown = [p for p in properties if p not in _VIB_PROPERTIES]
        if unknown:
            raise ValueError(f"DeviceVibrations: properties must be a subset of {_VIB_PROPERTIES}, got {unknown}")
        outputs = getattr(model, "model_outputs", None)
        if outputs is not None:
            missing = [p for p in [self.energy_key, self.force_key] + properties if p not in outputs]
            if missing:
                raise ValueError(f"DeviceVibrations: the model does not output {missing} (it outputs {sorted(outputs)})")
        idx_m, n_sys = self._setup(model, batch, cutoff, capacity, use_graph)
        self.required_properties = properties
        self.nfree, self.p_conv, self.e_conv = int(nfree), float(position_conversion), float(energy_conversion)
        self.delta = float(delta)

        base, dev = self.static, batch[P.R].device
        pos = base[P.R]
        if pos.dtype != torch.float32 or not pos.is_contiguous():
            raise ValueError("DeviceVibrations: '_positions' must be a contiguous float32 tensor")
        n = pos.shape[0]
        masses = torch.as_tensor(masses).reshape(-1)
        if masses.shape[0] != n:
            raise ValueError(f"DeviceVibrations: {masses.shape[0]} masses for {n} atoms")
        self.n_atoms, self.n_sys = n, n_sys
        self.masses = masses.to(dev, torch.float64).contiguous()
        self.idx_m = idx_m
        self.sys_ptr = ops.segment_ptr(idx_m, n_sys)
        sizes = (self.sys_ptr[1:] - self.sys_ptr[:-1]).to(torch.int64).cpu()         # one host read, at set-up
        self.sizes = sizes.tolist()
        self.max_atoms = max(self.sizes) if self.sizes else 0
        n_coords = 3 * self.max_atoms
        limit = DEFAULT_MAX_REPLICA_ATOMS if max_replica_atoms is None else int(max_replica_atoms)
        self.n_cols = max(1, min(n_coords, limit // max(1, self.nfree * n)))
        self.n_copies = self.n_cols * self.nfree
        self.n_chunks = -(-n_coords // self.n_cols) if n_coords else 0
        hess_ptr = torch.zeros(n_sys + 1, dtype=torch.int64)
        hess_ptr[1:] = torch.cumsum(9 * sizes * sizes, 0)
        self.hess_ptr = hess_ptr.to(dev)
        n_hess = int(hess_ptr[-1])

        base.setdefault(P.idx_m, idx_m)
        base.setdefault(P.n_atoms, sizes.to(dev))
        self.base_positions = pos
        self.static = replicate_batch(base, self.n_copies, n_sys)
        self.nl.capacity *= self.n_copies                # ``capacity`` is that of ``batch``, once per copy
        f64 = dict(dtype=torch.float64, device=dev)
        self.steps = torch.zeros(self.n_copies, n_sys, **f64)
        self.counter = torch.zeros(2, dtype=torch.int64, device=dev)
        self.h_raw = torch.zeros(n_hess, **f64)
        self.hessian = torch.zeros(n_hess // 9, 3, 3, **f64)
        self.hessian_mw = torch.zeros(n_hess, **f64)
        self.dipole_derivatives = torch.zeros(n, 3, 3, **f64) if P.dipole_moment in properties else None
        self.polarizability_derivatives = (torch.zeros(n, 3, 3, 3, **f64) if P.polarizability in properties
                                           else None)
        self.outputs: Dict[str, Tensor] = {}       # the replica batch's dipoles / polarizabilities, copied per step
        self._eig: Optional[List[tuple]] = None
        self._calculate()                          # shapes of the outputs, buffers of the captured step
        p = ops._p
        self._params = _lib.VibParams(
            p(self.base_positions), p(self.static[P.R]), p(self.steps), p(self.counter), p(self.forces),
            p(self.outputs.get(P.dipole_moment)), p(self.outputs.get(P.polarizability)), p(self.idx_m),
            p(self.sys_ptr), None, p(self.hess_ptr), p(self.masses), p(self.h_raw), p(self.hessian), p(self.hessian_mw),
            p(self.dipole_derivatives), p(self.polarizability_derivatives), n, n_sys, self.n_cols, self.nfree,
            self.max_atoms, self.delta / self.p_conv, self.e_conv / self.p_conv ** 2)

    # ---- the captured step ----------------------------------------------------------------------------------------------
    def _refresh_properties(self, out: Dict[str, Tensor]):
        rows = self.n_copies * self.n_sys
        for p in self.required_properties:
            v = out[p].detach()
            shape = (rows, 3) if p == P.dipole_moment else (rows, 3, 3)
            if tuple(v.shape) != shape:
                raise ValueError(f"DeviceVibrations: '{p}' must be a per-system {list(shape[1:])} output, got shape "
                                 f"{tuple(v.shape)} for {rows} replica systems (a scalar dipole has no derivative "
                                 "layout)")
            if v.dtype != torch.float32 or not v.is_contiguous():
                raise TypeError(f"DeviceVibrations: property '{p}' must be a contiguous float32 model output")
            buf = self.outputs.get(p)
            if buf is None:
                buf = self.outputs[p] = torch.empty(shape, dtype=torch.float32, device=v.device)
            _lib.call("spk_md_property", ops._p(v), v.numel(), 1.0, ops._p(buf), ops._stream())

    def _step(self):
        ops.vib_displace(self._params)
        self._calculate()
        ops.vib_assemble(self._params)

    def _step_state(self) -> Dict[str, object]:
        state = dict(positions=self.static[P.R], steps=self.steps, counter=self.counter, h_raw=self.h_raw,
                     outputs=self.outputs, dipole_derivatives=self.dipole_derivatives,
                     polarizability_derivatives=self.polarizability_derivatives, **self._evaluation_state())
        return {k: v for k, v in state.items() if v is not None}

    def run(self):
        """Evaluate every displaced copy (``n_chunks`` replays of the captured step) and finish the Hessian and the
        derivatives."""
        self.counter.zero_()
        self._run_steps(self.n_chunks)
        ops.vib_finish(self._params)
        self.check_neighbor_list()
        self._eig = None

    # ---- post-processing (torch fp64, outside the graph) ------------------------------------------------------------------
    def _eigensystems(self) -> List[tuple]:
        """per system: (eigenvalues [3n] ascending, eigenvectors [3n, 3n] as columns) of the mass-weighted Hessian in
        eV / (Angstrom^2 amu); systems of one size share one batched eigh"""
        if self._eig is not None:
            return self._eig
        eig: List[Optional[tuple]] = [None] * self.n_sys
        ptr = self.hess_ptr.tolist()
        for size in sorted(set(self.sizes)):
            ids = [m for m in range(self.n_sys) if self.sizes[m] == size]
            if size == 0:
                for m in ids:
                    eig[m] = (self.hessian_mw.new_zeros(0), self.hessian_mw.new_zeros(0, 0))
                continue
            blocks = torch.stack([self.hessian_mw[ptr[m]:ptr[m + 1]].view(3 * size, 3 * size) for m in ids])
            w, v = torch.linalg.eigh(blocks)
            for k, m in enumerate(ids):
                eig[m] = (w[k], v[k])
        self._eig = eig
        return eig

    def frequencies(self) -> Tensor:
        """[3N] harmonic frequencies in cm^-1: system m at 3 sys_ptr[m] .. 3 sys_ptr[m+1], ascending per system.  An
        imaginary frequency (negative eigenvalue) is returned as the negative of its magnitude, where ASE returns a
        complex number."""
        w = torch.cat([e[0] for e in self._eigensystems()])
        return torch.sign(w) * torch.sqrt(torch.abs(w)) * (_HBAR_OMEGA / _INVCM)

    def mode(self, m: int) -> Tensor:
        """[3 n_m, n_m, 3] normal modes of system m: mass-weighted eigenvectors divided by sqrt(mass), in the order of
        ``frequencies`` (ASE's get_mode)"""
        v = self._eigensystems()[m][1]
        lo, hi = self._atoms(m)
        inv_sqrt_m = (1.0 / torch.sqrt(self.masses[lo:hi])).repeat_interleave(3)
        return (v.T * inv_sqrt_m).reshape(3 * (hi - lo), hi - lo, 3)

    def _atoms(self, m: int):
        ptr = self.sys_ptr
        return int(ptr[m]), int(ptr[m + 1])

    def _project(self, deriv: Tensor) -> Tensor:
        """sum_i d y / d x_i L_ik / sqrt(m_i) per mode k of every system: [3N, n_comp] for ``deriv`` [N, n_comp, 3]
        in per-Angstrom units"""
        out = []
        for m in range(self.n_sys):
            lo, hi = self._atoms(m)
            d = deriv[lo:hi].permute(1, 0, 2).reshape(deriv.shape[1], -1) / self.p_conv   # [n_comp, 3n]
            out.append((self.mode(m).reshape(3 * (hi - lo), -1) @ d.T))
        return torch.cat(out)

    def ir_intensities(self) -> Tensor:
        """[3N] IR intensities sum_c (sum_i d mu_c / d x_i L_ik / sqrt(m_i))^2 in (model dipole unit / Angstrom)^2 / amu,
        in the order of ``frequencies`` (ASE's Infrared).  For a dipole in Debye, multiply by 42.255 for km/mol."""
        if self.dipole_derivatives is None:
            raise RuntimeError("DeviceVibrations: ir_intensities needs properties=('dipole_moment', ...)")
        return (self._project(self.dipole_derivatives) ** 2).sum(1)

    def raman_activities(self) -> Tensor:
        """[3N] Raman activities 45 a'^2 + 7 g'^2 of the mode-projected polarizability derivative A' (its symmetric part):
        a' = tr(A') / 3, g'^2 = ((A'xx - A'yy)^2 + (A'yy - A'zz)^2 + (A'zz - A'xx)^2 + 6 (A'xy^2 + A'yz^2 + A'zx^2)) / 2,
        in (model polarizability unit / Angstrom)^2 / amu, in the order of ``frequencies``."""
        if self.polarizability_derivatives is None:
            raise RuntimeError("DeviceVibrations: raman_activities needs properties=('polarizability', ...)")
        a = self._project(self.polarizability_derivatives.reshape(self.n_atoms, 9, 3)).reshape(-1, 3, 3)
        a = 0.5 * (a + a.transpose(1, 2))
        mean = a.diagonal(dim1=1, dim2=2).sum(1) / 3.0
        xx, yy, zz = a[:, 0, 0], a[:, 1, 1], a[:, 2, 2]
        gamma2 = 0.5 * ((xx - yy) ** 2 + (yy - zz) ** 2 + (zz - xx) ** 2
                        + 6.0 * (a[:, 0, 1] ** 2 + a[:, 1, 2] ** 2 + a[:, 2, 0] ** 2))
        return 45.0 * mean ** 2 + 7.0 * gamma2
