"""Batchwise structure relaxation on the device: the L-BFGS of the reference's ``ASEBatchwiseLBFGS``
(interfaces/batchwise_optimization.py:613-917) with one optimizer per system of a collated batch, its state and history
in fp64 on the device, and the whole step -- optimizer, neighbour list, energy + forces, convergence test -- captured
once as a CUDA graph (DESIGN.md section 12).

The reference copies positions and forces to the host on every step and runs the two-loop recursion in numpy.  Here the
step is two kinds of kernels of ``csrc/relax.cu``: ``spk_relax_step`` (history update, two-loop recursion, masking of
converged systems, step capping, position update) and ``spk_relax_converged`` (per-system largest force and the count of
unconverged systems), and ``DeviceLBFGS.run`` reads that count once per ``check_every`` steps.

Systems may differ in size (the reference needs equal atom counts).  The fp64 recursion departs on purpose from the
reference, whose float32 forces keep ``q`` and ``z`` in float32 through numpy's in-place updates.

``DeviceFIRE`` (DESIGN.md section 18) relaxes with ASE's FIRE instead, optionally on the generalized coordinates of ASE's
``UnitCellFilter``, so that periodic systems relax their cells too, under an external pressure.  Its kernels are those of
``csrc/fire.cu``: ``spk_fire_forces`` after every evaluation and ``spk_fire_step``.
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, Optional

import torch

from . import _lib, ops
from . import properties as P
from .md import _CapturedEvaluation, _clone_state, _load_state, _TensorState

__all__ = ["DeviceLBFGS", "LBFGSState", "DeviceFIRE", "FIREState", "UnitCellFilter"]

Tensor = torch.Tensor
DEFAULT_MAX_STEPS = 100_000_000          # ASE's Dynamics default, which the reference's run loop inherits


def _fixed_mask(fixed_atoms_mask, n_atoms: int, dev) -> Optional[Tensor]:
    """uint8 [N] from a boolean mask of length N or a list of atom indices (both index ``f[mask] = 0`` in the
    reference's get_forces)"""
    if fixed_atoms_mask is None:
        return None
    m = torch.as_tensor(fixed_atoms_mask).reshape(-1).cpu()
    if m.dtype == torch.bool:
        if m.numel() != n_atoms:
            raise ValueError(f"fixed_atoms_mask: a boolean mask needs {n_atoms} entries, got {m.numel()}")
        out = m
    else:
        idx = m.to(torch.int64)
        if idx.numel() and (int(idx.min()) < -n_atoms or int(idx.max()) >= n_atoms):
            raise ValueError(f"fixed_atoms_mask: atom index out of range for {n_atoms} atoms")
        out = torch.zeros(n_atoms, dtype=torch.bool)
        out[idx] = True
    return out.to(torch.uint8).to(dev)


class _ConvergenceState(_TensorState):
    """The convergence test's device buffers, which the optimizer kernels keep alike: the step counter pair, the fmax
    target, the largest force, the converged flag and the step count at which it was met per system, and the count of
    unconverged systems.  Subclasses set ``n_atoms`` and define ``tensors()``, every buffer a step writes."""

    def _init_convergence(self, n_sys: int, fmax: float, dev):
        self.counter = torch.zeros(2, dtype=torch.int64, device=dev)
        self.fmax_target = torch.full((1,), float(fmax), dtype=torch.float64, device=dev)
        self.fmax = torch.zeros(n_sys, dtype=torch.float64, device=dev)
        self.converged = torch.zeros(n_sys, dtype=torch.int32, device=dev)
        self.steps_to_converge = torch.full((n_sys,), -1, dtype=torch.int64, device=dev)
        self.n_unconverged = torch.full((1,), n_sys, dtype=torch.int32, device=dev)

    def _convergence_tensors(self) -> Dict[str, Tensor]:
        return {"counter": self.counter, "fmax_target": self.fmax_target, "fmax": self.fmax,
                "converged": self.converged, "steps_to_converge": self.steps_to_converge,
                "n_unconverged": self.n_unconverged}

    def _forces(self, forces: Tensor) -> Tensor:
        f = ops.f32(forces, "forces")
        if f.numel() != 3 * self.n_atoms:
            raise ValueError(f"{type(self).__name__}: forces of {f.numel()} values for {self.n_atoms} atoms")
        return f

    def set_fmax(self, fmax: float):
        self.fmax_target.fill_(float(fmax))

    def _state(self) -> Dict[str, Tensor]:
        return self.tensors()


class LBFGSState(_ConvergenceState):
    """Optimizer state of a batch and the launches of its kernels (the step and the convergence test), given a forces
    tensor.  ``positions`` [N, 3] are the starting positions in optimizer units (model positions x
    ``position_conversion``); forces are model forces, multiplied by ``force_conversion`` in the kernels.  Systems are
    the ``idx_m`` segments.  ``check(forces)`` must run on the forces of the current positions before every ``step``
    with the same forces.  ``model_positions`` (fp32 [N, 3], allocated if not given) receives r / position_conversion
    at every step."""

    def __init__(self, positions: Tensor, idx_m: Tensor, n_sys: int, memory: int = 100, maxstep: float = 0.2,
                 damping: float = 1.0, alpha: float = 70.0, fixed_atoms_mask=None, position_conversion: float = 1.0,
                 force_conversion: float = 1.0, model_positions: Optional[Tensor] = None, fmax: float = 0.05):
        dev = positions.device
        if dev.type != "cuda":
            raise ValueError("LBFGSState needs CUDA tensors (no CPU fallback)")
        if not 1 <= int(memory) <= _lib.RELAX_MAX_MEMORY:
            raise ValueError(f"LBFGSState: memory must be in [1, {_lib.RELAX_MAX_MEMORY}], got {memory}")
        n, n_sys = int(positions.shape[0]), int(n_sys)
        if n_sys < 1:
            raise ValueError("LBFGSState: the batch has no system")
        f64 = dict(dtype=torch.float64, device=dev)
        self.n_atoms, self.n_sys, self.memory = n, n_sys, int(memory)
        self.r = positions.detach().to(**f64).reshape(n, 3).contiguous().clone()
        self.r0 = torch.zeros_like(self.r)
        self.f0 = torch.zeros_like(self.r)
        self.s = torch.zeros(self.memory, n, 3, **f64)
        self.y = torch.zeros_like(self.s)
        self.rho = torch.ones(self.memory, n_sys, **f64)
        self.p = torch.zeros_like(self.r)
        self._init_convergence(n_sys, fmax, dev)
        self.fixed = _fixed_mask(fixed_atoms_mask, n, dev)
        p_conv = float(position_conversion)
        if model_positions is None:
            model_positions = (self.r / p_conv).float()
        self.model_positions = ops.f32(model_positions, "model_positions")
        self.idx_m = idx_m.to(dev, torch.int64).contiguous()
        self.sys_ptr = ops.segment_ptr(self.idx_m, n_sys)
        # size path of every system (one host read, here only): warp systems first, then the cluster systems
        sizes = (self.sys_ptr[1:] - self.sys_ptr[:-1]).cpu()
        small = sizes <= _lib.RELAX_WARP_ATOMS
        self.n_warp = int(small.sum())
        ids = torch.arange(n_sys)
        self.order = torch.cat([ids[small], ids[~small]]).to(dev, torch.int32)
        p = ops._p
        self._params = _lib.LBFGSState(
            p(self.r), p(self.r0), p(self.f0), p(self.s), p(self.y), p(self.rho), p(self.p), p(self.counter),
            p(self.fmax_target), p(self.fmax), p(self.converged), p(self.steps_to_converge), p(self.n_unconverged),
            p(self.fixed), p(self.model_positions), p(self.sys_ptr), p(self.order), n, n_sys, self.n_warp,
            self.memory, float(force_conversion), p_conv, float(maxstep), float(damping), 1.0 / float(alpha))

    def check(self, forces: Tensor):
        """the convergence test of the forces at the current positions (fmax, converged, steps_to_converge and the
        unconverged count, on the device)"""
        _lib.call("spk_relax_converged", ctypes.byref(self._params), ops._p(self._forces(forces)), ops._stream())

    def step(self, forces: Tensor):
        """one L-BFGS step with the forces at the current positions"""
        _lib.call("spk_relax_step", ctypes.byref(self._params), ops._p(self._forces(forces)), ops._stream(),
                  launches=int(self.n_warp > 0) + int(self.n_warp < self.n_sys))

    def tensors(self) -> Dict[str, Tensor]:
        """every buffer the step writes"""
        return {"r": self.r, "r0": self.r0, "f0": self.f0, "s": self.s, "y": self.y, "rho": self.rho, "p": self.p,
                **self._convergence_tensors(), "model_positions": self.model_positions}


class _BatchOptimizer(_CapturedEvaluation):
    """The driver of a batchwise optimizer in the captured step: ``self.opt`` (a ``_ConvergenceState``) holds the
    optimizer state and the convergence buffers.  A driver defines ``_advance()``, its optimizer step, and ``_check()``,
    the force side and convergence test on the current evaluation; one step is ``_advance()``, the evaluation and
    ``_check()``.  Results are in optimizer units."""

    def _check_outputs(self, model, energy_key: str, force_key: str):
        """refuse a model that does not output both keys, and take them as the evaluation's keys"""
        outputs = getattr(model, "model_outputs", None)
        if outputs is not None and (force_key not in outputs or energy_key not in outputs):
            raise ValueError(f"{type(self).__name__}: the model must output '{energy_key}' and '{force_key}' (it outputs "
                             f"{sorted(outputs)})")
        self.energy_key, self.force_key = energy_key, force_key

    def _set_conversions(self, position_conversion: float, energy_conversion: float):
        self.p_conv = float(position_conversion)
        self.e_conv = float(energy_conversion)
        self.f_conv = self.e_conv / self.p_conv

    def _fp32_positions(self) -> Tensor:
        """the model positions ``static[_positions]``, checked to be a contiguous fp32 tensor"""
        mp = self.static[P.R]
        if mp.dtype != torch.float32 or not mp.is_contiguous():
            raise ValueError(f"{type(self).__name__}: '_positions' must be a contiguous float32 tensor")
        return mp

    def _start(self):
        """the step counts and the convergence test of the starting positions"""
        self.iterations = 0                      # steps taken (host mirror of the device counter)
        self.nsteps = 0
        self._calculate()                        # forces of the starting positions (irun, :417)
        self._check()

    def _step(self):
        self._advance()
        self._calculate()
        self._check()

    def _step_state(self) -> Dict[str, object]:
        state = dict(opt=self.opt.tensors(), **self._evaluation_state())
        if self.virial is not None:
            state["virial"] = self.virial
        return state

    def run(self, fmax: float = 0.05, steps: Optional[int] = None, check_every: int = 10) -> bool:
        """Relax until every system's largest force is below ``fmax`` or ``steps`` steps (default: unlimited) were taken
        in this call; returns whether every system converged.  ``nsteps`` is then the step count at which the reference's
        loop would have stopped."""
        if int(check_every) < 1:
            raise ValueError(f"{type(self).__name__}: check_every must be >= 1")
        budget = DEFAULT_MAX_STEPS if not steps else int(steps)
        self.opt.set_fmax(fmax)
        self._check()                            # the convergence test under this fmax
        done = 0
        left = int(self.opt.n_unconverged.item())
        while left and done < budget:
            k = min(int(check_every), budget - done)
            self._run_steps(k)
            done += k
            self.iterations += k
            left = int(self.opt.n_unconverged.item())
        self.check_neighbor_list()
        self.nsteps = int(self.opt.steps_to_converge.max().item()) if left == 0 else self.iterations
        return left == 0

    # ---- results ------------------------------------------------------------------------------------------------------
    @property
    def positions(self) -> Tensor:
        """[N, 3] fp64 positions in optimizer units (Angstrom in the reference)"""
        return self.opt.r

    @property
    def model_positions(self) -> Tensor:
        """[N, 3] fp32 positions the model reads (positions / position_conversion)"""
        return self.static[P.R]

    def get_forces(self) -> Tensor:
        """forces of the current positions [N, 3] fp64 in optimizer units, zero on fixed atoms (get_forces, :182-198)"""
        f = self.forces.double() * self.f_conv
        if self.opt.fixed is not None:
            f = f * (1 - self.opt.fixed.double())[:, None]
        return f

    def get_uncertainty(self) -> Dict[str, Tensor]:
        """Ensemble runs: the unbiased std over the members of the energies [n_sys] and forces [N, 3] at the current
        positions, in optimizer units (BatchwiseEnsembleCalculator.calculate, :329-335)"""
        if self.ensemble is None:
            raise RuntimeError(f"{type(self).__name__}: get_uncertainty needs an ensemble (model=[m1, m2, ...])")
        from .ensemble import ensemble_moments

        e = ensemble_moments(self.stacks[self.energy_key], ddof=1, spread_scale=self.e_conv, var=False, std=True)[2]
        f = ensemble_moments(self.stacks[self.force_key], ddof=1, spread_scale=self.f_conv, var=False, std=True)[2]
        return {"energy_uncertainty": e, "forces_uncertainty": f}

    @property
    def fmax(self) -> Tensor:
        """largest force per system [n_sys] fp64 (the quantity the convergence test compares with ``fmax``)"""
        return self.opt.fmax

    @property
    def converged(self) -> Tensor:
        return self.opt.converged.bool()

    @property
    def steps_to_converge(self) -> Tensor:
        """[n_sys] the step count at which each system met the criterion (-1 while it has not)"""
        return self.opt.steps_to_converge

    def state_dict(self) -> Dict[str, object]:
        """Everything a restart needs to continue bitwise (it replaces the reference's pickle restart file)."""
        return dict(_clone_state(self._step_state()), iterations=self.iterations, nsteps=self.nsteps)

    def load_state_dict(self, state: Dict[str, object]):
        """Copy a ``state_dict`` into the existing buffers (a captured graph stays valid)."""
        _load_state(self._step_state(), state)
        self.iterations = int(state["iterations"])
        self.nsteps = int(state["nsteps"])


class DeviceLBFGS(_BatchOptimizer):
    """Relax every system of ``batch`` with the reference's batchwise L-BFGS (keywords and defaults of
    ASEBatchwiseLBFGS; ``alpha`` gives H0 = 1 / alpha).  ``batch[_positions]`` is in model units;
    ``position_conversion`` and ``energy_conversion`` turn model lengths and energies into the optimizer's units (Angstrom
    and eV in the reference), so ``maxstep`` and ``fmax`` are in those.  ``fixed_atoms_mask`` (boolean mask or atom
    indices) zeroes the forces of atoms that must not move.  ``cutoff`` and ``capacity`` size the device neighbour list,
    which is rebuilt at every step.

    One step is the optimizer kernels, the neighbour list, the model and the convergence test, captured once as a CUDA
    graph (``use_graph``).  ``run`` replays it in chunks of ``check_every`` steps and reads the count of unconverged
    systems once per chunk; steps replayed after every system has converged leave the positions bitwise unchanged.

    ``model`` may be a list (or ``nn.ModuleList``) of at least two members, as the reference's
    BatchwiseEnsembleCalculator (interfaces/batchwise_optimization.py:229-347): the mean forces drive the optimizer
    and its ``fmax`` test, and ``get_uncertainty`` gives the unbiased std over the members."""

    def __init__(self, model: torch.nn.Module, batch: Dict[str, Tensor], cutoff: float, capacity: int,
                 maxstep: float = 0.2, memory: int = 100, damping: float = 1.0, alpha: float = 70.0,
                 fixed_atoms_mask=None, position_conversion: float = 1.0, energy_conversion: float = 1.0,
                 energy_key: str = P.energy, force_key: str = P.forces, use_graph: bool = True):
        if float(maxstep) > 1.0:                                                 # batchwise_optimization.py:711-715
            raise ValueError("You are using a much too large value for the maximum step size: %.1f Angstrom"
                             % float(maxstep))
        self._check_outputs(model, energy_key, force_key)
        idx_m, n_sys = self._setup(model, batch, cutoff, capacity, use_graph)
        self._set_conversions(position_conversion, energy_conversion)
        mp = self._fp32_positions()
        self.opt = LBFGSState(mp.double() * self.p_conv, idx_m, n_sys, memory=memory, maxstep=maxstep,
                              damping=damping, alpha=alpha, fixed_atoms_mask=fixed_atoms_mask,
                              position_conversion=self.p_conv, force_conversion=self.f_conv, model_positions=mp)
        self._start()

    def _advance(self):
        self.opt.step(self.forces)

    def _check(self):
        self.opt.check(self.forces)

    def get_energy(self) -> Tensor:
        """energies of the current positions [n_sys] in optimizer units"""
        return self.energy * self.e_conv


# ---- FIRE and the unit-cell filter -------------------------------------------------------------------------------------
class UnitCellFilter:
    """The settings of ASE's ``UnitCellFilter`` for ``DeviceFIRE``: the cell of every system relaxes with its atoms.
    ``mask``: 6 Voigt components (xx, yy, zz, yz, xz, xy) or a 3 x 3 array multiplied into the cell forces;
    ``cell_factor`` scales the cell coordinates (default: each system's atom count); ``hydrostatic_strain`` keeps the
    cell shape; ``constant_volume`` removes the trace of the cell forces; ``scalar_pressure`` is the external pressure in
    optimizer energy / length^3 (eV / Angstrom^3 in ASE's units; ``units.convert_units("GPa", "eV / Ang / Ang / Ang")``
    gives the factor from GPa)."""

    def __init__(self, mask=None, cell_factor: Optional[float] = None, hydrostatic_strain: bool = False,
                 constant_volume: bool = False, scalar_pressure: float = 0.0):
        if mask is None:
            full = torch.ones(3, 3, dtype=torch.float64)
        else:
            m = torch.as_tensor(mask, dtype=torch.float64).cpu()
            if m.shape == (6,):
                xx, yy, zz, yz, xz, xy = m.tolist()              # ASE's voigt_6_to_full_3x3_stress
                full = torch.tensor([[xx, xy, xz], [xy, yy, yz], [xz, yz, zz]], dtype=torch.float64)
            elif m.shape == (3, 3):
                full = m.clone()
            else:
                raise ValueError(f"UnitCellFilter: mask must have 6 Voigt components or be 3 x 3, got shape "
                                 f"{tuple(m.shape)}")
        if cell_factor is not None and not float(cell_factor) > 0.0:
            raise ValueError(f"UnitCellFilter: cell_factor must be > 0, got {cell_factor}")
        if not math.isfinite(float(scalar_pressure)):
            raise ValueError("UnitCellFilter: scalar_pressure must be finite")
        self.mask = full
        self.cell_factor = None if cell_factor is None else float(cell_factor)
        self.hydrostatic_strain = bool(hydrostatic_strain)
        self.constant_volume = bool(constant_volume)
        self.scalar_pressure = float(scalar_pressure)


FIRE_DEFAULTS = dict(dt=0.1, maxstep=0.2, dtmax=1.0, Nmin=5, finc=1.1, fdec=0.5, astart=0.1, fa=0.99, a=0.1)


def _check_fire_keywords(kw: Dict[str, float]):
    for k in ("dt", "maxstep", "dtmax", "finc", "fdec", "fa"):
        if not float(kw[k]) > 0.0:
            raise ValueError(f"FIRE: {k} must be > 0, got {kw[k]}")
    for k in ("astart", "a"):
        if not 0.0 <= float(kw[k]) <= 1.0:
            raise ValueError(f"FIRE: {k} must be in [0, 1], got {kw[k]}")
    if int(kw["Nmin"]) != kw["Nmin"] or int(kw["Nmin"]) < 0:
        raise ValueError(f"FIRE: Nmin must be a non-negative integer, got {kw['Nmin']}")


class FIREState(_ConvergenceState):
    """FIRE state of a batch and the launches of its kernels, given a forces tensor (and, with ``cell_filter``, the fp64
    model virial [n_sys, 3, 3]).  ``positions`` [N, 3] are the starting positions in optimizer units (model positions x
    ``position_conversion``), ``cell`` [n_sys, 3, 3] the starting cells in the same units (needed with the filter);
    forces are model forces, multiplied by ``force_conversion``, and the virial is multiplied by ``energy_conversion``.
    ``check(forces, virial)`` must run on the forces of the current positions before every ``step``.
    ``model_positions`` (fp32 [N, 3]) and ``model_cell`` (fp32 [n_sys, 3, 3]), allocated if not given, receive the new
    positions and cells / position_conversion at every step.  Keywords are those of ASE's FIRE."""

    def __init__(self, positions: Tensor, idx_m: Tensor, n_sys: int, dt: float = 0.1, maxstep: float = 0.2,
                 dtmax: float = 1.0, Nmin: int = 5, finc: float = 1.1, fdec: float = 0.5, astart: float = 0.1,
                 fa: float = 0.99, a: float = 0.1, fixed_atoms_mask=None, cell: Optional[Tensor] = None,
                 cell_filter: Optional[UnitCellFilter] = None, position_conversion: float = 1.0,
                 force_conversion: float = 1.0, energy_conversion: float = 1.0,
                 model_positions: Optional[Tensor] = None, model_cell: Optional[Tensor] = None, fmax: float = 0.05):
        dev = positions.device
        if dev.type != "cuda":
            raise ValueError("FIREState needs CUDA tensors (no CPU fallback)")
        kw = dict(dt=dt, maxstep=maxstep, dtmax=dtmax, Nmin=Nmin, finc=finc, fdec=fdec, astart=astart, fa=fa, a=a)
        _check_fire_keywords(kw)
        if cell_filter is not None and not isinstance(cell_filter, UnitCellFilter):
            raise TypeError("FIREState: cell_filter must be a UnitCellFilter")
        n, n_sys = int(positions.shape[0]), int(n_sys)
        if n_sys < 1:
            raise ValueError("FIREState: the batch has no system")
        f64 = dict(dtype=torch.float64, device=dev)
        self.n_atoms, self.n_sys, self.filter = n, n_sys, cell_filter
        self.idx_m = idx_m.to(dev, torch.int64).contiguous()
        self.sys_ptr = ops.segment_ptr(self.idx_m, n_sys)
        p_conv = float(position_conversion)
        self.s = positions.detach().to(**f64).reshape(n, 3).contiguous().clone()
        self.r = torch.zeros_like(self.s) if cell_filter is not None else self.s
        self.v = torch.zeros_like(self.s)
        self.g = torch.zeros_like(self.s)
        self.dt = torch.full((n_sys,), float(dt), **f64)
        self.a = torch.full((n_sys,), float(a), **f64)
        self.nsteps = torch.zeros(n_sys, dtype=torch.int64, device=dev)
        self.started = torch.zeros(n_sys, dtype=torch.int32, device=dev)
        self.sums = torch.zeros(n_sys, 3, **f64)
        self.coef = torch.zeros(n_sys, _lib.FIRE_COEF, **f64)
        nbytes = int(_lib.lib().spk_fire_workspace_bytes(n, n_sys))
        self.workspace = torch.zeros(max(nbytes // 8, 1), **f64)
        self._init_convergence(n_sys, fmax, dev)
        self.fixed = _fixed_mask(fixed_atoms_mask, n, dev)
        if model_positions is None:
            model_positions = (self.s / p_conv).float()
        self.model_positions = ops.f32(model_positions, "model_positions")
        self.h = self.hv = self.hg = self.cell0 = self.cell_factor = self.model_cell = None
        mask = [1.0] * 9
        if cell_filter is not None:
            if cell is None:
                raise ValueError("FIREState: a cell filter needs the starting cells")
            self.cell0 = cell.detach().to(**f64).reshape(n_sys, 9).contiguous().clone()
            sizes = (self.sys_ptr[1:] - self.sys_ptr[:-1]).to(torch.float64)
            cf = sizes if cell_filter.cell_factor is None else torch.full_like(sizes, cell_filter.cell_factor)
            if bool((cf <= 0).any()):
                raise ValueError("FIREState: the default cell_factor (the atom count) needs atoms in every system")
            self.cell_factor = cf.contiguous()
            self.h = (torch.eye(3, **f64).reshape(1, 9) * cf[:, None]).contiguous()    # cell_factor F with F = I
            self.hv = torch.zeros_like(self.h)
            self.hg = torch.zeros_like(self.h)
            self.r.copy_(self.s)
            if model_cell is None:
                model_cell = (self.cell0 / p_conv).float()
            self.model_cell = ops.f32(model_cell, "model_cell")
            if self.model_cell.numel() != 9 * n_sys:
                raise ValueError(f"FIREState: model_cell of {self.model_cell.numel()} values for {n_sys} systems")
            mask = cell_filter.mask.reshape(-1).tolist()
        p = ops._p
        self._params = _lib.FIREState(
            p(self.s), p(self.r), p(self.v), p(self.g), p(self.h), p(self.hv), p(self.hg), p(self.cell0),
            p(self.cell_factor), p(self.dt), p(self.a), p(self.nsteps), p(self.started), p(self.sums), p(self.coef),
            p(self.workspace), p(self.counter), p(self.fmax_target), p(self.fmax), p(self.converged),
            p(self.steps_to_converge), p(self.n_unconverged), p(self.fixed), p(self.model_positions),
            p(self.model_cell), p(self.idx_m), p(self.sys_ptr), (ctypes.c_double * 9)(*mask), n, n_sys, int(Nmin),
            int(cell_filter is not None), int(bool(cell_filter and cell_filter.hydrostatic_strain)),
            int(bool(cell_filter and cell_filter.constant_volume)), 0, float(force_conversion),
            float(energy_conversion), p_conv, float(cell_filter.scalar_pressure) if cell_filter else 0.0,
            float(maxstep), float(dtmax), float(finc), float(fdec), float(astart), float(fa))

    def check(self, forces: Tensor, virial: Optional[Tensor] = None):
        """the generalized forces at the current positions and the convergence test (fmax, converged,
        steps_to_converge and the unconverged count, on the device)"""
        f = self._forces(forces)
        w = None
        if self.filter is not None:
            if (virial is None or virial.dtype != torch.float64 or not virial.is_contiguous()
                    or virial.numel() != 9 * self.n_sys or virial.device != f.device):
                raise ValueError("FIREState: a cell filter needs the fp64 contiguous [n_sys, 3, 3] model virial")
            w = virial
        _lib.call("spk_fire_forces", ctypes.byref(self._params), ops._p(f), ops._p(w), ops._stream(),
                  launches=2 + int(self.n_atoms > 0))

    def step(self):
        """one FIRE step with the generalized forces of the last ``check``"""
        _lib.call("spk_fire_step", ctypes.byref(self._params), ops._stream(), launches=1 + int(self.n_atoms > 0))

    def deformation_gradient(self) -> Optional[Tensor]:
        """F [n_sys, 3, 3] fp64 (cell = cell0 F^T), None without a filter"""
        if self.filter is None:
            return None
        return (self.h / self.cell_factor[:, None]).reshape(-1, 3, 3)

    def cell(self) -> Optional[Tensor]:
        """the current cells [n_sys, 3, 3] fp64 in optimizer units, None without a filter"""
        if self.filter is None:
            return None
        return torch.matmul(self.cell0.reshape(-1, 3, 3), self.deformation_gradient().transpose(1, 2))

    def tensors(self) -> Dict[str, Tensor]:
        """every buffer the step and the force side write and a later step reads"""
        out = {"s": self.s, "v": self.v, "g": self.g, "dt": self.dt, "a": self.a, "nsteps": self.nsteps,
               "started": self.started, "sums": self.sums, **self._convergence_tensors(),
               "model_positions": self.model_positions}
        if self.filter is not None:
            out.update(r=self.r, h=self.h, hv=self.hv, hg=self.hg, model_cell=self.model_cell)
        return out


class DeviceFIRE(_BatchOptimizer):
    """Relax every system of ``batch`` with ASE's FIRE (its keywords and defaults; no ``downhill_check``), one optimizer
    per system, with the batch semantics of ``DeviceLBFGS``: a system whose largest (generalized) force is below
    ``fmax`` takes no step and keeps its optimizer state, and systems may differ in size.  ``batch[_positions]`` (and
    ``_cell``) are in model units; ``position_conversion`` and ``energy_conversion`` turn model lengths and energies into
    the optimizer's units, in which ``dt``, ``maxstep``, ``fmax`` and the filter's ``scalar_pressure`` are given.
    ``fixed_atoms_mask`` (boolean mask or atom indices) zeroes the forces of atoms that must not move; under a filter
    they keep their scaled coordinates and so move with the cell.

    ``cell_filter`` (a ``UnitCellFilter``) relaxes the cells too: every system must be periodic on all three axes, the
    model's virial is evaluated at every step, and the neighbour list is rebuilt on the new cell.  It is refused for
    an ensemble, which has no stress.

    One step is the optimizer kernels, the neighbour list, the model and the convergence test, captured once as a CUDA
    graph (``use_graph``).  ``model`` may be a list of at least two members: their mean forces drive a fixed-cell
    relaxation and ``get_uncertainty`` gives the unbiased std over the members, as in ``DeviceLBFGS``.  ``fmax`` is the
    largest generalized force per system (atom rows and, under the filter, cell rows); ``positions`` and ``get_forces``
    are Cartesian."""

    def __init__(self, model: torch.nn.Module, batch: Dict[str, Tensor], cutoff: float, capacity: int,
                 dt: float = 0.1, maxstep: float = 0.2, dtmax: float = 1.0, Nmin: int = 5, finc: float = 1.1,
                 fdec: float = 0.5, astart: float = 0.1, fa: float = 0.99, a: float = 0.1, fixed_atoms_mask=None,
                 cell_filter: Optional[UnitCellFilter] = None, position_conversion: float = 1.0,
                 energy_conversion: float = 1.0, energy_key: str = P.energy, force_key: str = P.forces,
                 use_graph: bool = True):
        _check_fire_keywords(dict(dt=dt, maxstep=maxstep, dtmax=dtmax, Nmin=Nmin, finc=finc, fdec=fdec,
                                  astart=astart, fa=fa, a=a))
        if cell_filter is not None and not isinstance(cell_filter, UnitCellFilter):
            raise TypeError("DeviceFIRE: cell_filter must be a UnitCellFilter")
        self._check_outputs(model, energy_key, force_key)
        idx_m, n_sys = self._setup(model, batch, cutoff, capacity, use_graph)
        if cell_filter is not None and self.ensemble is not None:
            raise NotImplementedError("DeviceFIRE: a cell filter needs the stress, which an ensemble does not have (the "
                                      "reference's EnsembleCalculator._activate_stress raises)")
        self._set_conversions(position_conversion, energy_conversion)
        mp = self._fp32_positions()
        cell = model_cell = None
        if cell_filter is not None:
            model_cell = self._setup_virial(n_sys, "a cell filter")
            cell = model_cell.reshape(n_sys, 3, 3).double() * self.p_conv
            self._check_periodic(n_sys, torch.linalg.det(cell), "a cell filter")
        self.opt = FIREState(mp.double() * self.p_conv, idx_m, n_sys, dt=dt, maxstep=maxstep, dtmax=dtmax, Nmin=Nmin,
                             finc=finc, fdec=fdec, astart=astart, fa=fa, a=a, fixed_atoms_mask=fixed_atoms_mask,
                             cell=cell, cell_filter=cell_filter, position_conversion=self.p_conv,
                             force_conversion=self.f_conv, energy_conversion=self.e_conv, model_positions=mp,
                             model_cell=model_cell)
        self._start()

    def _advance(self):
        self.opt.step()

    def _check(self):
        self.opt.check(self.forces, self.virial)

    # ---- results, in optimizer units ----------------------------------------------------------------------------------
    @property
    def cell(self) -> Optional[Tensor]:
        """[n_sys, 3, 3] fp64 cells (rows = lattice vectors) under a cell filter, else None"""
        return self.opt.cell()

    def get_energy(self) -> Tensor:
        """energies of the current positions [n_sys]"""
        return self.energy * self.e_conv

    def get_stress(self) -> Tensor:
        """stress of the current cells [n_sys, 3, 3] fp64: the symmetric part of W / V (cell filter only)"""
        if self.virial is None:
            raise RuntimeError("DeviceFIRE: the stress is evaluated under a cell filter only")
        w = 0.5 * (self.virial + self.virial.transpose(1, 2)) * self.e_conv
        return w / torch.linalg.det(self.cell).abs()[:, None, None]

    def get_enthalpy(self) -> Tensor:
        """E + p V per system [n_sys] fp64 (the energy without a cell filter)"""
        e = self.get_energy().double()
        if self.opt.filter is None:
            return e
        return e + self.opt.filter.scalar_pressure * torch.linalg.det(self.cell).abs()
