"""Device-resident NVE step (SURVEY.md section 8, "next" rows f1 + f2): the reference's simulation loop
(/root/reference/src/schnetpack/md/simulator.py:93-144 -- half_step, main_step, calculator.calculate, half_step with the
velocity-Verlet integrator of md/integrators.py:59-70,97-110) with NOTHING leaving the GPU between steps:

  * the neighbour list is rebuilt on the device every step (``neighbors.CellListNeighborList`` with a fixed capacity and
    inert padding -- no Verlet skin, no host copy of positions as in md/neighborlist_md.py:129,213-232);
  * momenta / positions are updated by device kernels on static buffers;
  * the whole step (kick, drift, neighbour list, graph views, energy + forces, kick) is captured once as a CUDA graph and
    replayed; the host only counts steps.  ``n_pairs`` (true pair count, overflow flag) stays on the device for the caller
    to poll when it wants to.

Units follow the reference's calculator (md/calculators/base_calculator.py:85-98,120-152): the MD state (positions, momenta,
masses, time step) lives in the caller's MD units; ``position_conversion`` turns MD positions into the model's length unit
before every evaluation and ``energy_conversion`` turns the model's energies into MD energy units, so forces are scaled by
``energy_conversion / position_conversion``.  Both default to 1 (MD units == model units).  The integrator is the
velocity-Verlet of md/integrators.py:59-70,97-110 as one kernel per half step (``spk_md_velocity_verlet``).  No Verlet skin
is kept (md/neighborlist_md.py:55-98 rebuilds when an atom moved more than skin / 2): rebuilding the exact-cutoff list on the
device every step costs less than the bookkeeping (0.22 ms at 8192 atoms) and gives the same forces, since the model's
cutoff function removes every pair beyond the cutoff either way.

Constant-temperature runs (DESIGN.md section 9): ``DeviceMD(..., thermostat=...)`` applies a ``BerendsenThermostat``,
``LangevinThermostat`` or ``NHCThermostat`` (md/simulation_hooks/thermostats.py:149-513) before the first and after the
second half kick, as the reference's ThermostatHook does at on_step_begin / on_step_end (md/simulator.py:127-150), inside the
same captured graph.  Systems are those of the batch (``_idx_m`` / ``_n_atoms``); per-system kinetic energies are fp64 sums
in a fixed order, the chain state of the Nose-Hoover thermostat and the application counter of the Langevin noise live in
device memory, so a replayed step neither syncs with the host nor repeats its noise.

Constant-pressure runs (DESIGN.md section 9): ``DeviceMD(..., barostat=...)`` with an ``NHCBarostatIsotropic`` or
``NHCBarostatAnisotropic`` (md/simulation_hooks/barostats.py:162-927) runs the step of NPTVelocityVerlet
(md/integrators.py:232-263, md/simulator.py:124-150): barostat on_step_begin, half step, main step (positions and cell),
neighbour list on the new cell, energy + forces + virial, half step, on_step_end -- all in the same captured graph.  The
virial W = sum_e dE/dr_e (x) r_e comes out of the backward of ``PairwiseDistances`` (one fp64 kernel with a fixed summation
order); the stress in MD units is W / V * energy_conversion / position_conversion^3 (base_calculator.py:97,218-222) with V
the volume of the model cell.  ``compute_stress=True`` keeps the same virial up to date in NVE / NVT runs.

Ring-polymer MD (DESIGN.md section 9): ``DeviceMD(..., ring_polymer=RingPolymer(...))`` replicates the batch into P beads
(replica-major, as md/calculators/base_calculator.py:154-221 collates them) and runs the RingPolymer step
(md/integrators.py:113-229, md/simulator.py:124-150): thermostat, half kick per bead, normal-mode propagation of the free ring
polymer, neighbour list + energy + forces on all beads, half kick, thermostat -- with the PILE-L / PILE-G / TRPMD and
ring-polymer NHC thermostats of md/simulation_hooks/thermostats_rpmd.py, all in the same captured graph.  With a
``PILEBarostat`` (md/simulation_hooks/barostats_rpmd.py) the step is that of NPTRingPolymer (md/integrators.py:266-305):
the barostat propagates the centroid mode and the cell, the virial of every bead system is kept, and any ring-polymer
thermostat (or none) runs next to it.

Colored-noise runs (DESIGN.md section 9): ``GLEThermostat`` (classical), ``RPMDGLEThermostat`` (one GLE on every normal mode)
and ``PIGLETThermostat`` (one GLE per normal mode) of md/simulation_hooks/thermostats.py:527-730 and thermostats_rpmd.py:
237-370 read gle4md matrix files with ``load_gle_matrices`` and keep D extended momenta per (normal mode, degree of
freedom) in fp64 on the device.  One kernel (``spk_rpmd_gle``) transforms to normal modes, propagates s = c1 s + sqrt(m)
c2 xi and transforms back; the classical thermostat is the same kernel at P = 1.  It uses the propagator of the GLE
papers, where the reference multiplies by the transpose of c1, which samples a wrong distribution for a non-normal drift
matrix.  RPMD-GLE and PIGLET also run next to ``PILEBarostat``.

Initial conditions and basic hooks (DESIGN.md section 19): ``DeviceMD(..., initializer=MaxwellBoltzmannInit(...) or
UniformInit(...))`` sets the starting state as the reference's system.initializer (md/initial_conditions.py) -- centre of
mass, wrapping, momenta from Philox, translation and rotation removal -- and ``hooks=[RemoveCOMMotion(...),
WrapPositions(...)]`` run the reference's basic simulation hooks (md/simulation_hooks/basic_hooks.py) inside the captured
step, gated by a device step counter.  A singular inertia tensor gets its pseudo-inverse, and ring polymers wrap by their
centroids.
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, List, Optional

import torch

from . import _lib, ops
from . import properties as P
from .atomistic.pair_terms import check_ewald_cells, check_padded_pair_terms, padded_list_cutoff
from .neighbors import CellListNeighborList
from .units import _amu, _e, _hbar, _k, _Nav

__all__ = ["DeviceMD", "BerendsenThermostat", "LangevinThermostat", "NHCThermostat", "NHCBarostatIsotropic",
           "NHCBarostatAnisotropic", "RingPolymer", "PILELocalThermostat", "PILEGlobalThermostat", "TRPMDThermostat",
           "NHCRingPolymerThermostat", "PILEBarostat", "GLEThermostat", "RPMDGLEThermostat", "PIGLETThermostat",
           "load_gle_matrices", "MaxwellBoltzmannInit", "UniformInit", "RemoveCOMMotion", "WrapPositions", "KB_MD",
           "FS_MD", "BAR_MD", "HBAR_MD"]

Tensor = torch.Tensor

# ---- MD units of the reference (units.py:10-40): energy kJ/mol, length nm, mass Da; time = nm sqrt(Da / (kJ/mol)).
# From the CODATA-2014 constants of ``units`` (Boltzmann constant, elementary charge, Avogadro constant, atomic mass
# unit, reduced Planck constant), in ASE's frame (eV, Angstrom, amu): kJ/mol = 1e3 / (e N_A) eV, nm = 10 Angstrom,
# fs = 1e-15 s with s = 1e10 sqrt(e / amu).
_MD_ENERGY = 1e3 / _e / _Nav                                    # kJ/mol in eV
_MD_TIME = 10.0 * math.sqrt(1.0 / _MD_ENERGY)                 # units.py:37, in ASE time units
KB_MD = (_k / _e) / _MD_ENERGY                                 # units.py:79: ~0.0083144598 kJ/mol/K
FS_MD = 1e-15 * 1e10 * math.sqrt(_e / _amu) / _MD_TIME         # units.py:59: ~1.0e-3
# units.py:37-40,64-65: 1 bar = 1e5 Pa = 1e5 J/m^3 = 1e5 N_A / 1e30 kJ/mol/nm^3 (~0.0602214)
BAR_MD = 1e5 * _Nav / 1e30
# units.py:80-82: hbar in J s, times ASE's J * s = (1 / e) eV * 1e10 sqrt(e / amu), over energy * time (~0.0635)
HBAR_MD = _hbar / _e * 1e10 * math.sqrt(_e / _amu) / (_MD_ENERGY * _MD_TIME)
# units of gle4md matrix files (thermostat_utils.py:78-86), CODATA 2014: Hartree energy in J, atomic unit of time in s;
# energies go through kelvin (x kB) and times through femtoseconds (x fs), so custom MD units need no further constant
_CODATA_HARTREE, _CODATA_AUT = 4.359744650e-18, 2.418884326509e-17
_EV_K = _e / _k                                                 # 1 eV in K (~11604.5)
_HARTREE_K = _CODATA_HARTREE / _k                               # 1 Hartree in K (~315775)
_AUT_FS = _CODATA_AUT * 1e15                                    # 1 atomic time unit in fs (~0.0241888)


class _Systems:
    """The systems of a collated batch as the thermostat kernels address them: per-atom masses and system index, the
    first atom of every system and the fp64 workspaces of the per-system sums."""

    def __init__(self, masses: Tensor, idx_m: Tensor, n_sys: int):
        self.masses = masses
        self.idx_m = idx_m
        self.n_sys = int(n_sys)
        self.n_atoms = int(masses.shape[0])
        self.sys_ptr = ops.segment_ptr(idx_m, self.n_sys)
        self.n_atoms_sys = (self.sys_ptr[1:] - self.sys_ptr[:-1]).to(torch.float64)
        self._workspaces: Dict[str, Tensor] = {}

    def workspace(self, size_fn: str) -> Tensor:
        """The workspace of the kernels sized by the library's ``size_fn(n_atoms, n_sys)``, allocated on first use (the
        eager warm-up before a capture, so never inside one)."""
        ws = self._workspaces.get(size_fn)
        if ws is None:
            nbytes = int(getattr(_lib.lib(), size_fn)(self.n_atoms, self.n_sys))
            ws = self._workspaces[size_fn] = torch.empty(nbytes, dtype=torch.uint8, device=self.masses.device)
        return ws

    def call(self, name: str, momenta: Tensor, *args, launches: Optional[int] = None):
        ws = self.workspace("spk_md_thermostat_workspace_bytes")
        _lib.call(name, ops._p(momenta), ops._p(self.masses), ops._p(self.idx_m), ops._p(self.sys_ptr), self.n_atoms,
                  self.n_sys, *args, ops._p(ws), ws.numel(), ops._stream(), launches=launches)

    def kinetic_energy_and_temperature(self, momenta: Tensor, kB: float):
        dev = momenta.device
        ke = torch.empty(self.n_sys, dtype=torch.float64, device=dev)
        temp = torch.empty(self.n_sys, dtype=torch.float64, device=dev)
        self.call("spk_md_kinetic_energy", momenta, float(kB), ops._p(ke), ops._p(temp))
        return ke, temp

    def kinetic_energy_tensor(self, momenta: Tensor) -> Tensor:
        """1/2 sum_a p_a p_a^T / m_a per system, [n_sys, 3, 3] fp64 (system.py:389-404)"""
        out = torch.empty(self.n_sys, 3, 3, dtype=torch.float64, device=momenta.device)
        ws = self.workspace("spk_md_barostat_workspace_bytes")
        _lib.call("spk_md_kinetic_energy_tensor", ops._p(momenta), ops._p(self.masses), ops._p(self.idx_m),
                  ops._p(self.sys_ptr), self.n_atoms, self.n_sys, ops._p(out), ops._p(ws), ws.numel(), ops._stream())
        return out


def _batch_layout(static: Dict[str, Tensor]):
    """(idx_m int64, n_sys) of a collated batch: one system when it has no ``_idx_m`` / ``_n_atoms``"""
    idx_m = static.get(P.idx_m)
    if idx_m is None:
        idx_m = torch.zeros(static[P.R].shape[0], dtype=torch.int64, device=static[P.R].device)
    n_sys = static[P.n_atoms].shape[0] if P.n_atoms in static else 1
    return idx_m.to(torch.int64).contiguous(), n_sys


def replicate_batch(static: Dict[str, Tensor], n_copies: int, n_sys: int) -> Dict[str, Tensor]:
    """``n_copies`` replicas of the batch, replica-major as the reference's calculator collates ring-polymer beads
    (md/calculators/base_calculator.py:154-221): ``_idx_m`` + r B, every other tensor repeated along its first axis.
    A ``_cell`` / ``_pbc`` shared by all B systems ([3, 3] or [1, 3, 3] / [3] or [1, 3], which the neighbour list
    broadcasts) is first expanded to one row per system, so the replica batch has one per replica system."""
    out = {}
    for k, v in static.items():
        if k == P.idx_m:
            out[k] = torch.cat([v + r * n_sys for r in range(n_copies)])
            continue
        if k in (P.cell, P.pbc):
            width = 9 if k == P.cell else 3
            rows = v.reshape(-1, width)
            if rows.shape[0] == 1:
                rows = rows.expand(n_sys, width)
            if rows.shape[0] != n_sys:
                raise ValueError(f"'{k}' of shape {tuple(v.shape)} is neither shared nor one per system for {n_sys} "
                                 "systems")
            v = rows.reshape(n_sys, 3, 3) if k == P.cell else rows.reshape(-1) if v.dim() == 1 else rows
        out[k] = torch.cat([v] * n_copies).contiguous()
    return out


def _flatten(state: Dict[str, object]) -> List[Tensor]:
    return [t for v in state.values() for t in (_flatten(v) if isinstance(v, dict) else [v])]


def _clone_state(state: Dict[str, object]) -> Dict[str, object]:
    return {k: _clone_state(v) if isinstance(v, dict) else v.clone() for k, v in state.items()}


def _load_state(dst: Dict[str, object], src: Dict[str, object]):
    """copy the (nested) dict ``src`` into the tensors of ``dst``, key by key"""
    for k, v in dst.items():
        if isinstance(v, dict):
            _load_state(v, src[k])
        else:
            v.copy_(src[k])


class _TensorState:
    """``state_dict`` / ``load_state_dict`` over the device tensors ``_state()`` names (the state a step writes)."""

    def _state(self) -> Dict[str, Tensor]:
        return {}

    def state_dict(self) -> Dict[str, Tensor]:
        return _clone_state(self._state())

    def load_state_dict(self, state: Dict[str, Tensor]):
        _load_state(self._state(), state)


def _bath_temperature(value, who: str, per_system: bool = False):
    """``temperature_bath`` as one float in K, or as a list of floats when it is a sequence or tensor of them, which only
    thermostats with ``per_system`` take"""
    if isinstance(value, (int, float)):
        return float(value)
    temps = torch.as_tensor(value, dtype=torch.float64)
    if temps.dim() == 0:
        return float(temps)
    if not per_system:
        raise ValueError(f"{who}: temperature_bath must be one number; only LangevinThermostat and NHCThermostat take one "
                         "temperature per system")
    if temps.numel() == 0:
        raise ValueError(f"{who}: temperature_bath is an empty sequence")
    return [float(t) for t in temps.reshape(-1).tolist()]


def _one_per_system(temps: List[float], n_sys: int, who: str) -> Tensor:
    """[n_sys] fp64 (host) from one temperature or one per system"""
    if len(temps) not in (1, n_sys):
        raise ValueError(f"{who}: {len(temps)} temperatures for {n_sys} systems; give one temperature or one per system")
    return torch.tensor(temps * (n_sys if len(temps) == 1 else 1), dtype=torch.float64)


def _noise(seed: int, device) -> tuple:
    """(seed, counter) of a Philox noise hook: the seed taken to 64 bits and a fresh device counter laid out as
    advance_counter (md_common.cuh) reads it, [0] = application index, [1] = the kernel's internal ticket (zero between
    calls)"""
    return int(seed) & 0xFFFFFFFFFFFFFFFF, torch.zeros(2, dtype=torch.int64, device=device)


# ---- Nose-Hoover chains -------------------------------------------------------------------------------------------------
_YS_WEIGHTS = {                                                          # md/utils/thermostat_utils.py:18-44
    3: (1.35120719195966, -1.70241438391932, 1.35120719195966),
    5: (0.41449077179438, 0.41449077179438, -0.65796308717750, 0.41449077179438, 0.41449077179438),
    7: (0.78451361047756, 0.23557321335936, -1.17767998417887, 1.31518632068390, -1.17767998417887,
        0.23557321335936, 0.78451361047756),
}


def _check_nhc(chain_length: int, multi_step: int, integration_order: int):
    if integration_order not in _YS_WEIGHTS:
        raise ValueError(f"Order {integration_order:d} not supported for YS integration weights")
    if int(chain_length) < 1 or int(multi_step) < 1:
        raise ValueError("chain_length and multi_step must be >= 1")


def _ys_steps(time_step: float, multi_step: int, integration_order: int):
    """the Yoshida-Suzuki sub-steps dt w_k / multi_step as the kernels' 7-entry array (thermostats.py:339-341)"""
    w = _YS_WEIGHTS[integration_order]
    return (ctypes.c_double * 7)(*([time_step * wk / multi_step for wk in w] + [0.0] * (7 - len(w))))


def _chain_masses(n_chains: int, dof, chain_length: int, kbt, frequency: float, device) -> Tensor:
    """[n_chains, chain_length] fp64 chain masses kB T / omega^2, the first link times the degrees of freedom ``dof`` of
    its chain (a number or an [n_chains] tensor) (thermostats.py:387-396).  ``kbt`` is a number or an [n_chains] tensor;
    a tensor goes through the same fp64 operations, elementwise, so equal values give the same bits."""
    if isinstance(kbt, Tensor):       # true division (torch divides a device tensor by a number via its reciprocal)
        link = torch.from_numpy(kbt.cpu().numpy() / frequency ** 2).to(device)
        masses = link[:, None].repeat(1, chain_length)
    else:
        masses = torch.full((n_chains, chain_length), kbt / frequency ** 2, dtype=torch.float64, device=device)
    masses[:, 0] = dof * kbt / frequency ** 2
    return masses


class _Thermostat(_TensorState):
    """Common part of the device thermostats (ThermostatHook, thermostats.py:41-146): bath temperature in K, time constant
    in fs.  ``kB`` (MD energy per kelvin) and ``fs`` (one femtosecond in MD time) define the caller's MD units; the
    defaults are the reference's (kJ/mol, nm, Da).  ``bind`` sizes the state for a batch, ``apply`` updates the momenta in
    place (enqueue-only, capturable).

    Thermostats with ``takes_per_system`` (Langevin, NHC) also take a sequence or tensor of bath temperatures: one, or one
    per system of the batch, checked by ``bind``, which keeps them as ``temperatures`` (fp64 [n_sys] on the device) and
    ``kb_temperatures`` (kB T_s).  ``temperatures`` is None with one number."""

    takes_per_system = False

    def __init__(self, temperature_bath, time_constant: float, kB: float = KB_MD, fs: float = FS_MD):
        self.temperature_bath = _bath_temperature(temperature_bath, type(self).__name__, self.takes_per_system)
        self.time_constant = float(time_constant) * float(fs)          # thermostats.py:57-59
        self.kB = float(kB)
        self.systems: Optional[_Systems] = None
        self.time_step: Optional[float] = None
        self.temperatures: Optional[Tensor] = None
        self.kb_temperatures: Optional[Tensor] = None

    @property
    def per_system(self) -> bool:
        return isinstance(self.temperature_bath, list)

    def bind(self, systems: _Systems, time_step: float):
        self.systems = systems
        self.time_step = float(time_step)
        if self.per_system:
            t = _one_per_system(self.temperature_bath, systems.n_sys, type(self).__name__)
            if not bool((t >= 0.0).all()):
                raise ValueError(f"{type(self).__name__}: bath temperatures must be >= 0 K, got {t.min().item()}")
            self.temperatures = t.to(systems.masses.device)
            self.kb_temperatures = self.temperatures * self.kB          # the scalar path's kB * T, elementwise
        self._init_state()

    def _init_state(self):
        pass

    def apply(self, momenta: Tensor):
        raise NotImplementedError


class BerendsenThermostat(_Thermostat):
    """Berendsen rescaling (thermostats.py:149-189): p *= sqrt(1 + dt / tau (T_bath / T - 1)) per system.  A system whose
    kinetic energy is zero is left as it is (the reference would divide by T = 0)."""

    def apply(self, momenta: Tensor):
        self.systems.call("spk_md_berendsen", momenta, self.kB, self.time_step / self.time_constant,
                          self.temperature_bath)


class LangevinThermostat(_Thermostat):
    """Langevin thermostat (thermostats.py:192-261): p = c1 p + c2 sqrt(m kB T_bath) xi with c1 = exp(-dt / (2 tau)),
    c2 = sqrt(1 - c1^2).  xi comes from Philox4x32-10 keyed by ``seed`` with the counter (atom, application); the
    application index lives on the device and advances with every application, also inside a replayed graph.
    ``temperature_bath`` may give one temperature per system: T_bath is then that of the atom's system."""

    takes_per_system = True

    def __init__(self, temperature_bath, time_constant: float, seed: int = 0, kB: float = KB_MD,
                 fs: float = FS_MD):
        super().__init__(temperature_bath, time_constant, kB=kB, fs=fs)
        self.seed = seed

    def _init_state(self):
        gamma = 1.0 / self.time_constant                                 # :227-230
        self.c1 = math.exp(-0.5 * self.time_step * gamma)                 # :233
        self.c2 = math.sqrt(1.0 - self.c1 ** 2)                           # :234
        self.seed, self.counter = _noise(self.seed, self.systems.masses.device)

    def apply(self, momenta: Tensor):
        s = self.systems
        if self.per_system:
            _lib.call("spk_md_langevin_per_system", ops._p(momenta), ops._p(s.masses), ops._p(s.idx_m), s.n_atoms,
                      self.c1, self.c2, ops._p(self.kb_temperatures), self.seed, ops._p(self.counter), ops._stream())
            return
        _lib.call("spk_md_langevin", ops._p(momenta), ops._p(s.masses), s.n_atoms, self.c1, self.c2,
                  self.kB * self.temperature_bath, self.seed, ops._p(self.counter), ops._stream())

    def _state(self):
        return {"counter": self.counter}


class NHCThermostat(_Thermostat):
    """Nose-Hoover chain thermostat (thermostats.py:264-513) with the reference's keywords and defaults: one chain per
    system, or per degree of freedom with ``massive``; ``multi_step`` sub-steps of a Yoshida-Suzuki scheme of order
    ``integration_order`` (3, 5 or 7).  The chain state is fp64 on the device.  With one ``temperature_bath`` per system,
    the masses and forces of every chain use kB T_s of its system (of its atom's system with ``massive``)."""

    takes_per_system = True

    def __init__(self, temperature_bath, time_constant: float, chain_length: int = 3, massive: bool = False,
                 multi_step: int = 2, integration_order: int = 3, kB: float = KB_MD, fs: float = FS_MD):
        super().__init__(temperature_bath, time_constant, kB=kB, fs=fs)
        _check_nhc(chain_length, multi_step, integration_order)
        self.chain_length = int(chain_length)
        self.massive = bool(massive)
        self.multi_step = int(multi_step)
        self.integration_order = int(integration_order)
        self.velocities = self.forces = self.masses = None

    def _init_state(self):
        s = self.systems
        dev = s.masses.device
        if self.per_system and not bool((self.temperatures > 0.0).all()):
            raise ValueError("NHCThermostat: bath temperatures must be > 0 K (they set the chain masses)")
        kbt = self.kb_temperatures if self.per_system else self.temperature_bath * self.kB     # :308
        if self.massive:                                                  # :348-359
            dof = torch.ones(3 * s.n_atoms, dtype=torch.float64, device=dev)
            chain_kbt = kbt[s.idx_m].repeat_interleave(3) if self.per_system else kbt
        else:
            dof = 3.0 * s.n_atoms_sys
            chain_kbt = kbt
        self.masses = _chain_masses(dof.shape[0], dof, self.chain_length, chain_kbt, 1.0 / self.time_constant,  # :304
                                    dev)
        self.velocities = torch.zeros_like(self.masses)
        self.forces = torch.zeros_like(self.masses)
        self.params = _lib.NHCParams(self.chain_length, self.multi_step, self.integration_order, int(self.massive),
                                     0.0 if self.per_system else kbt,
                                     _ys_steps(self.time_step, self.multi_step, self.integration_order))

    def apply(self, momenta: Tensor):
        if self.per_system:
            self.systems.call("spk_md_nhc_per_system", momenta, ctypes.byref(self.params), ops._p(self.kb_temperatures),
                              ops._p(self.velocities), ops._p(self.forces), ops._p(self.masses),
                              launches=1 if self.massive else None)
            return
        self.systems.call("spk_md_nhc", momenta, ctypes.byref(self.params), ops._p(self.velocities),
                          ops._p(self.forces), ops._p(self.masses))

    def _state(self):
        return {"velocities": self.velocities, "forces": self.forces}


class _NHCBarostat(_TensorState):
    """Nose-Hoover-chain barostat (barostats.py:162-705) with the reference's keywords and defaults: target pressure in bar,
    bath temperature in K, time constants in fs; ``kB``, ``fs`` and ``bar`` define the caller's MD units (defaults: the
    reference's kJ/mol, nm, Da).  Two chains as in the reference: one on the particles (per system, or per degree of freedom
    with ``massive``) and one on the cell (per system).  It thermostats the particles itself, so ``DeviceMD`` takes no
    separate thermostat with it.  State (chains, cell velocities and forces) is fp64 on the device."""

    anisotropic = False
    ring_polymer = False
    temperature_control = True

    def __init__(self, target_pressure: float, temperature_bath: float, time_constant: float,
                 time_constant_cell: Optional[float] = None, time_constant_barostat: Optional[float] = None,
                 chain_length: int = 4, multi_step: int = 4, integration_order: int = 7, massive: bool = False,
                 kB: float = KB_MD, fs: float = FS_MD, bar: float = BAR_MD):
        _check_nhc(chain_length, multi_step, integration_order)
        self.target_pressure = float(target_pressure) * float(bar)               # :51-53
        self.temperature_bath = _bath_temperature(temperature_bath, type(self).__name__)
        self.time_constant = float(time_constant) * float(fs)
        self.frequency = 1.0 / self.time_constant                               # :209
        self.cell_frequency = self.frequency if time_constant_cell is None else 1.0 / (float(time_constant_cell) * fs)
        self.barostat_frequency = (self.frequency if time_constant_barostat is None
                                   else 1.0 / (float(time_constant_barostat) * fs))
        self.kB = float(kB)
        self.kb_temperature = self.temperature_bath * self.kB                   # :227
        self.chain_length = int(chain_length)
        self.multi_step = int(multi_step)
        self.integration_order = int(integration_order)
        self.massive = bool(massive)
        self.systems: Optional[_Systems] = None

    def bind(self, systems: _Systems, time_step: float):
        """on_simulation_start (:263-383, :760-796): masses and zero state for the systems of a batch."""
        self.systems = s = systems
        self.time_step = float(time_step)
        dev = s.masses.device
        f64 = dict(dtype=torch.float64, device=dev)
        kbt, L = self.kb_temperature, self.chain_length
        dof = 3.0 * s.n_atoms_sys                                                # :285-287
        self.b_masses = (dof + 3.0) * kbt / self.barostat_frequency ** 2         # :318-322
        if self.anisotropic:
            self.b_masses = self.b_masses / 3.0                                  # :771-776
            self.b_velocities = torch.zeros(s.n_sys, 3, 3, **f64)
        else:
            self.b_velocities = torch.zeros(s.n_sys, **f64)
        self.b_forces = torch.zeros_like(self.b_velocities)
        dof_p = torch.ones(3 * s.n_atoms, **f64) if self.massive else dof       # :293-302
        self.t_masses = _chain_masses(dof_p.shape[0], dof_p, L, kbt, self.frequency, dev)       # :343-371
        dof_cell = 6.0 if self.anisotropic else 1.0                              # :328-330, :794-796
        self.t_masses_cell = _chain_masses(s.n_sys, dof_cell, L, kbt, self.cell_frequency, dev)
        self.t_velocities = torch.zeros_like(self.t_masses)
        self.t_forces = torch.zeros_like(self.t_masses)
        self.t_velocities_cell = torch.zeros_like(self.t_masses_cell)
        self.t_forces_cell = torch.zeros_like(self.t_masses_cell)
        p = ops._p
        self.params = _lib.NHCBarostat(
            int(self.anisotropic), int(self.massive), L, self.multi_step, self.integration_order, 0, kbt, self.time_step,
            self.target_pressure, _ys_steps(self.time_step, self.multi_step, self.integration_order),   # :273-281
            p(self.t_velocities), p(self.t_forces), p(self.t_masses), p(self.t_velocities_cell), p(self.t_forces_cell),
            p(self.t_masses_cell), p(self.b_velocities), p(self.b_forces), p(self.b_masses))

    def _call(self, name: str, *args, launches: Optional[int] = None):
        ws = self.systems.workspace("spk_md_barostat_workspace_bytes")
        _lib.call(name, ctypes.byref(self.params), *args, ops._p(ws), ws.numel(), ops._stream(), launches=launches)

    def apply_thermostat(self, momenta: Tensor):
        """_update_thermostat (:408-481): particle and cell chains; scales the momenta and the cell velocities."""
        s = self.systems
        self._call("spk_md_barostat_thermostat", ops._p(momenta), ops._p(s.masses), ops._p(s.idx_m), ops._p(s.sys_ptr),
                   s.n_atoms, s.n_sys, launches=2 if self.massive else 4)   # massive: no kinetic-energy passes

    def kick(self, momenta: Tensor, cell: Tensor, virial: Tensor, virial_scale: float):
        """_update_barostat (:604-631, :822-842) with stress = virial_scale * virial / det(cell)."""
        s = self.systems
        self._call("spk_md_barostat_kick", ops._p(momenta), ops._p(s.masses), ops._p(s.idx_m), ops._p(s.sys_ptr),
                   s.n_atoms, s.n_sys, ops._p(cell), ops._p(virial), float(virial_scale))

    def half_step(self, momenta: Tensor, forces: Tensor, force_conversion: float = 1.0):
        """propagate_half_step (:661-686, :885-926) with forces * force_conversion in MD units."""
        s = self.systems
        self._call("spk_md_barostat_half_step", ops._p(momenta), ops._p(forces), float(force_conversion),
                   ops._p(s.idx_m), ops._p(s.sys_ptr), s.n_atoms, s.n_sys)

    def main_step(self, positions: Tensor, momenta: Tensor, cell: Tensor, model_positions: Optional[Tensor] = None,
                  model_cell: Optional[Tensor] = None, position_conversion: float = 1.0):
        """propagate_main_step (:633-659, :844-883): positions and the MD cell in place, plus their model-unit copies."""
        s = self.systems
        self._call("spk_md_barostat_main_step", ops._p(positions), ops._p(model_positions), ops._p(momenta),
                   ops._p(s.masses), ops._p(s.idx_m), ops._p(s.sys_ptr), s.n_atoms, s.n_sys, ops._p(cell),
                   ops._p(model_cell), float(position_conversion))

    def _state(self) -> Dict[str, Tensor]:
        return {"t_velocities": self.t_velocities, "t_forces": self.t_forces,
                "t_velocities_cell": self.t_velocities_cell, "t_forces_cell": self.t_forces_cell,
                "b_velocities": self.b_velocities, "b_forces": self.b_forces}


class NHCBarostatIsotropic(_NHCBarostat):
    """Isotropic cell fluctuations (barostats.py:162-705): one cell velocity per system; the barostat force uses the
    pressure without its kinetic part, -tr(stress) / 3."""


class NHCBarostatAnisotropic(_NHCBarostat):
    """Full 3x3 cell fluctuations (barostats.py:707-927): the barostat force uses the pressure tensor -stress + 2 K / V with
    the kinetic-energy tensor K; the propagators come from a per-system fp64 Jacobi eigendecomposition of the cell velocity
    (the reference's torch.symeig no longer exists in current torch)."""

    anisotropic = True


# ---- ring-polymer MD ------------------------------------------------------------------------------------------------------
class RingPolymer:
    """Ring-polymer integrator (md/integrators.py:113-229) with the reference's keywords: ``n_beads`` replicas (beads) of
    every molecule at ring-polymer temperature ``temperature`` in K; ``kB`` (MD energy per kelvin) and ``hbar`` (MD energy
    x MD time) define the caller's MD units.  The time step is ``DeviceMD``'s ``time_step``.  The normal-mode matrix C
    (md/utils/normal_model_transformation.py:37-68) and the free ring-polymer propagator (integrators.py:154-202) are built
    on the host in fp64 (the reference builds the propagator in float32)."""

    MAX_BEADS = 64

    def __init__(self, n_beads: int, temperature: float, kB: float = KB_MD, hbar: float = HBAR_MD):
        if int(n_beads) != n_beads or not 1 <= int(n_beads) <= self.MAX_BEADS:
            raise ValueError(f"RingPolymer: n_beads must be an integer in [1, {self.MAX_BEADS}], got {n_beads}")
        if not float(temperature) > 0.0:
            raise ValueError(f"RingPolymer: temperature must be > 0 K, got {temperature}")
        self.n_beads = int(n_beads)
        self.temperature = float(temperature)
        self.kB = float(kB)
        self.hbar = float(hbar)
        self.omega = self.kB * self.n_beads * self.temperature / self.hbar                     # integrators.py:146
        k = torch.arange(self.n_beads, dtype=torch.float64)
        self.omega_normal = 2.0 * self.omega * torch.sin(k * math.pi / self.n_beads)            # :175-179

    def transform_matrix(self) -> Tensor:
        """C [P, P] fp64 (normal_model_transformation.py:37-68): modes = C beads, beads = C^T modes"""
        P = self.n_beads
        n = torch.arange(1, P + 1, dtype=torch.float64)
        c = torch.zeros(P, P, dtype=torch.float64)
        c[0, :] = 1.0
        for k in range(1, P // 2 + 1):
            c[k, :] = math.sqrt(2.0) * torch.cos(2.0 * math.pi * k * n / P)
        for k in range(P // 2 + 1, P):
            c[k, :] = math.sqrt(2.0) * torch.sin(2.0 * math.pi * k * n / P)
        if P % 2 == 0:
            c[P // 2, :] = (-1.0) ** n
        return c / math.sqrt(P)

    def propagator(self, time_step: float) -> Tensor:
        """[P, 2, 2] fp64 (integrators.py:181-200): [[cos, -m-less w sin], [sin / w, cos]] per mode, [0, 1, 0] = dt"""
        w = self.omega_normal
        wdt = w * float(time_step)
        u = torch.zeros(self.n_beads, 2, 2, dtype=torch.float64)
        u[:, 0, 0] = torch.cos(wdt)
        u[:, 1, 1] = torch.cos(wdt)
        u[:, 0, 1] = -torch.sin(wdt) * w
        u[1:, 1, 0] = torch.sin(wdt[1:]) / w[1:]
        u[0, 1, 0] = float(time_step)
        return u

    def bind(self, base: "_Systems", time_step: float):
        """device copies of C and the propagator for the base batch ``base`` (its masses are one copy of every atom)"""
        dev = base.masses.device
        self.base = base
        self.time_step = float(time_step)
        self.c_transform = self.transform_matrix().to(dev)
        self.u = self.propagator(time_step).to(dev)

    def main_step(self, positions: Tensor, momenta: Tensor, model_positions: Optional[Tensor], position_conversion: float):
        """integrators.py:204-229 on the [P, N, 3] bead state, in place"""
        b = self.base
        _lib.call("spk_rpmd_main_step", ops._p(positions), ops._p(momenta), ops._p(model_positions), ops._p(b.masses),
                  b.n_atoms, self.n_beads, ops._p(self.c_transform), ops._p(self.u), float(position_conversion),
                  ops._stream())

    def normal_modes(self, x: Tensor, inverse: bool = False) -> Tensor:
        """beads -> normal modes (or back with ``inverse``) of a [P, N, 3] fp32 tensor, on the device"""
        x = x.contiguous()
        out = torch.empty_like(x)
        _lib.call("spk_rpmd_normal_modes", ops._p(x), ops._p(out), x.numel() // (3 * self.n_beads), self.n_beads,
                  ops._p(self.c_transform), 1 if inverse else 0, ops._stream())
        return out


class _RingPolymerThermostat(_Thermostat):
    """Common part of the ring-polymer thermostats (thermostats_rpmd.py): they act on the normal modes of the bead momenta
    and need the ``RingPolymer`` of the run.  ``systems`` are those of the base batch (one copy of every molecule)."""

    ring_polymer = True

    def bind(self, systems: _Systems, time_step: float, ring_polymer: Optional[RingPolymer] = None):
        if ring_polymer is None:
            raise ValueError(f"{type(self).__name__} is a ring-polymer thermostat: pass DeviceMD(ring_polymer=...)")
        self.rp = ring_polymer
        super().bind(systems, time_step)


class PILELocalThermostat(_RingPolymerThermostat):
    """Local path-integral Langevin thermostat (thermostats_rpmd.py:33-119): in normal-mode space p~_k = c1_k p~_k +
    c2_k sqrt(m kB P T) xi with gamma_k = 2 omega_k (gamma_0 = 1 / tau when ``thermostat_centroid``), all times
    ``damping_factor``, c1 = exp(-dt gamma / 2), c2 = sqrt(1 - c1^2).  xi comes from Philox4x32-10 keyed by ``seed`` with the
    counter (k N + atom, application): mode 0 draws exactly the bits of ``LangevinThermostat`` with the same seed."""

    _global = 0

    def __init__(self, temperature_bath: float, time_constant: float, thermostat_centroid: bool = True,
                 damping_factor: float = 1.0, seed: int = 0, kB: float = KB_MD, fs: float = FS_MD):
        super().__init__(temperature_bath, time_constant, kB=kB, fs=fs)
        self.thermostat_centroid = bool(thermostat_centroid)
        self.damping_factor = float(damping_factor)
        self.seed = seed

    def _init_state(self):
        dev = self.systems.masses.device
        gamma = 2.0 * self.rp.omega_normal.clone()                            # :75
        if self.thermostat_centroid:
            gamma[0] = 1.0 / self.time_constant                               # :78-79
        gamma = gamma * self.damping_factor                                   # :82
        c1 = torch.exp(-0.5 * self.time_step * gamma)                         # :85
        self.c1, self.c2 = c1.to(dev), torch.sqrt(1.0 - c1 ** 2).to(dev)      # :86
        self.kbt_p = self.kB * self.rp.n_beads * self.temperature_bath        # :92-97
        self.seed, self.counter = _noise(self.seed, dev)

    def apply(self, momenta: Tensor):
        s = self.systems
        ws = s.workspace("spk_rpmd_workspace_bytes")
        _lib.call("spk_rpmd_pile", ops._p(momenta), ops._p(s.masses), ops._p(s.idx_m), ops._p(s.sys_ptr), s.n_atoms,
                  s.n_sys, self.rp.n_beads, ops._p(self.rp.c_transform), ops._p(self.c1), ops._p(self.c2), self.kbt_p,
                  self._global, self.seed, ops._p(self.counter), ops._p(ws), ws.numel(), ops._stream(),
                  launches=3 if self._global else 1)

    def _state(self):
        return {"counter": self.counter}


class PILEGlobalThermostat(PILELocalThermostat):
    """Global path-integral Langevin thermostat (thermostats_rpmd.py:122-208): stochastic velocity rescaling of the centroid
    mode of every system, PILE-L on modes 1..P-1.  Per system, K0 = sum_a |p~_0,a|^2 / m_a, factor = K0 / (kB T P),
    cf = (1 - c) / factor with c = c1_0, S = sum |xi_0|^2 over the system's 3 N centroid noises, alpha^2 = c + S cf +
    2 R sqrt(c cf), alpha = sqrt(alpha^2) sign(R + sqrt(c / cf)), p~_0 *= alpha.

    Two deliberate differences from the reference:
      * R is the x-noise of each system's own first atom.  The reference takes the x-noise of the first atom of the whole
        batch, so all molecules of a batch share one R; for a one-system batch the two agree.
      * A system whose centroid kinetic energy is zero keeps its centroid as it is (the reference divides by zero and
        writes NaN there, which happens when a run starts from zero momenta), as ``BerendsenThermostat`` does at T = 0."""

    _global = 1

    def __init__(self, temperature_bath: float, time_constant: float, seed: int = 0, kB: float = KB_MD,
                 fs: float = FS_MD):
        super().__init__(temperature_bath, time_constant, thermostat_centroid=True, damping_factor=1.0, seed=seed, kB=kB,
                         fs=fs)


class TRPMDThermostat(PILELocalThermostat):
    """Thermostatted RPMD (thermostats_rpmd.py:211-234): PILE-L with time_constant = 1 fs, no centroid thermostat (the
    centroid momenta pass through) and friction ``damping_factor`` x 2 omega_k on the other modes."""

    def __init__(self, temperature_bath: float, damping_factor: float, seed: int = 0, kB: float = KB_MD,
                 fs: float = FS_MD):
        super().__init__(temperature_bath, 1.0, thermostat_centroid=False, damping_factor=damping_factor, seed=seed, kB=kB,
                         fs=fs)


class NHCRingPolymerThermostat(_RingPolymerThermostat):
    """Ring-polymer Nose-Hoover chains (thermostats_rpmd.py:373-501): one chain per normal mode and degree of freedom on
    p~, kinetic energy p~^2 / m, chain temperature P kB T, every link of mode k of mass P kB T / omega_k^2 with omega_0
    replaced by 1 / (2 tau).  With ``local=False`` mode 0 of every degree of freedom sees its system's total centroid
    sum |p~_0|^2 / m, with 3 N_s degrees of freedom and its first link 3 N_s times heavier.  The chain state is fp64 on the
    device, [P 3 N, chain_length]."""

    def __init__(self, temperature_bath: float, time_constant: float, local: bool = True, chain_length: int = 3,
                 multi_step: int = 2, integration_order: int = 3, kB: float = KB_MD, fs: float = FS_MD):
        super().__init__(temperature_bath, time_constant, kB=kB, fs=fs)
        _check_nhc(chain_length, multi_step, integration_order)
        self.local = bool(local)
        self.chain_length = int(chain_length)
        self.multi_step = int(multi_step)
        self.integration_order = int(integration_order)
        self.velocities = self.forces = self.masses = None

    def _init_state(self):
        s = self.systems
        dev = s.masses.device
        P, L, n_dof = self.rp.n_beads, self.chain_length, 3 * s.n_atoms
        kbt = self.kB * self.temperature_bath * P                              # :431
        freq = self.rp.omega_normal.clone()
        freq[0] = 0.5 / self.time_constant                                     # :434-436
        masses = (kbt / freq ** 2)[:, None, None].expand(P, n_dof, L).clone()  # :439-445
        if not self.local:                                                     # :449-458
            n_s = s.n_atoms_sys.cpu()[s.idx_m.cpu()]
            masses[0, :, 0] *= (3.0 * n_s).repeat_interleave(3)
        self.masses = masses.reshape(P * n_dof, L).to(dev)
        self.velocities = torch.zeros_like(self.masses)
        self.forces = torch.zeros_like(self.masses)
        self.params = _lib.NHCParams(L, self.multi_step, self.integration_order, 1, kbt,
                                     _ys_steps(self.time_step, self.multi_step, self.integration_order))

    def apply(self, momenta: Tensor):
        s = self.systems
        ws = s.workspace("spk_rpmd_workspace_bytes")
        g = 0 if self.local else 1
        _lib.call("spk_rpmd_nhc", ops._p(momenta), ops._p(s.masses), ops._p(s.idx_m), ops._p(s.sys_ptr), s.n_atoms,
                  s.n_sys, self.rp.n_beads, ops._p(self.rp.c_transform), ctypes.byref(self.params), g,
                  ops._p(self.velocities), ops._p(self.forces), ops._p(self.masses), ops._p(ws), ws.numel(),
                  ops._stream(), launches=3 if g else 1)

    def _state(self):
        return {"velocities": self.velocities, "forces": self.forces}


# ---- generalized-Langevin (colored-noise) thermostats ------------------------------------------------------------------------
GLE_MAX_DIM = 16      # extended momenta per degree of freedom the kernel keeps in registers


def _gle_unit(name: str, kB: float, fs: float) -> Optional[float]:
    """the factor that turns a gle4md unit into MD units (thermostat_utils.py:78-86), or None if the unit is unknown"""
    return {"femtoseconds^-1": 1.0 / fs, "picoseconds^-1": 1e-3 / fs, "seconds^-1": 1e-15 / fs,
            "atomic time units^-1": 1.0 / (_AUT_FS * fs), "K": kB, "eV": _EV_K * kB,
            "atomic energy units": _HARTREE_K * kB}.get(name)


def load_gle_matrices(path: str, kB: float = KB_MD, fs: float = FS_MD):
    """Read a gle4md matrix file in raw format (GLEMatrixParser, thermostat_utils.py:64-178): the drift matrix A between
    ``A MATRIX:`` and ``C MATRIX:``, the covariance C after ``C MATRIX:``, blocks split at ``# Matrix for normal mode``
    comment lines, the unit taken from the ``(...)`` of each header line.  Returns (A [n_blocks, D, D], C [n_blocks, D, D]
    or None) fp64 in the MD units given by ``kB`` (energy per kelvin) and ``fs`` (one femtosecond in MD time).  Raises
    ``ValueError`` for an unknown unit, a file without A, blocks that are not square or do not match, and D > 16."""
    heads = {"A": ("A MATRIX:", "C MATRIX:"), "C": ("C MATRIX:", None)}
    reading = {"A": False, "C": False}
    units: Dict[str, float] = {}
    blocks = {"A": [], "C": []}
    current = {"A": [], "C": []}
    with open(path) as f:
        for line in f:
            line = line.strip()
            if not line:
                continue
            for key, (start, stop) in heads.items():
                if start in line:                                           # thermostat_utils.py:108-112
                    unit = line.split("(")[-1].replace(")", "")
                    factor = _gle_unit(unit, kB, fs)
                    if factor is None:
                        raise ValueError(f"load_gle_matrices: unknown unit {unit!r} in the {key} header of {path}")
                    reading[key], units[key] = True, factor
                elif reading[key]:
                    if line.startswith("#"):                                # :114-121
                        if stop is not None and stop in line:
                            reading[key] = False
                        if "Matrix for normal mode" in line and current[key]:
                            blocks[key].append(current[key])
                            current[key] = []
                    else:
                        try:
                            current[key].append([float(x) for x in line.split()])
                        except ValueError:
                            raise ValueError(f"load_gle_matrices: cannot read the {key} row {line!r} of {path}") from None
    out = {}
    for key in ("A", "C"):
        if current[key]:
            blocks[key].append(current[key])
        if key not in units:
            out[key] = None
            continue
        if not blocks[key]:
            raise ValueError(f"load_gle_matrices: the {key} MATRIX section of {path} has no rows")
        for n, b in enumerate(blocks[key]):
            if any(len(row) != len(b) for row in b):
                raise ValueError(f"load_gle_matrices: {key} block {n} of {path} is not square ({len(b)} rows of "
                                 f"{sorted({len(row) for row in b})} columns)")
        if len({len(b) for b in blocks[key]}) != 1:
            raise ValueError(f"load_gle_matrices: the {key} blocks of {path} differ in size")
        out[key] = torch.tensor(blocks[key], dtype=torch.float64) * units[key]     # :140-145
    A, C = out["A"], out["C"]
    if A is None:
        raise ValueError(f"load_gle_matrices: no 'A MATRIX:' section in {path} (not a gle4md matrix file)")
    if C is not None and C.shape != A.shape:
        raise ValueError(f"load_gle_matrices: A {tuple(A.shape)} and C {tuple(C.shape)} of {path} do not match")
    if A.shape[-1] > GLE_MAX_DIM:
        raise ValueError(f"load_gle_matrices: D = {A.shape[-1]} extended momenta in {path}; at most {GLE_MAX_DIM} "
                         "are supported")
    return A, C


def _gle_propagators(A: Tensor, C: Tensor, time_step: float):
    """_init_single_gle_matrix (thermostats.py:653-657) in fp64 on the host: c1 = exp(-dt/2 A) and c2 the symmetric square
    root of C - c1 C c1^T, from its eigendecomposition.  Eigenvalues that are negative by rounding only are clamped to
    zero; a clearly negative one means C is not a stationary covariance of A, and no GLE has these matrices."""
    c1 = torch.linalg.matrix_exp(-0.5 * float(time_step) * A)
    m = C - c1 @ C @ c1.T
    m = 0.5 * (m + m.T)
    w, v = torch.linalg.eigh(m)
    tol = 1e3 * torch.finfo(torch.float64).eps * float(torch.linalg.matrix_norm(C, 2))
    if float(w.min()) < -tol:
        raise ValueError(f"GLE: C - c1 C c1^T has the eigenvalue {float(w.min()):.3e} < 0; A and C are not a valid "
                         "GLE (C must be a stationary covariance of the drift A)")
    c2 = (v * torch.sqrt(w.clamp_min(0.0))) @ v.T
    return c1, 0.5 * (c2 + c2.T)


class _GLE:
    """State and kernel call shared by the GLE thermostats: D extended momenta per (normal mode, degree of freedom) in fp64
    on the device, [P 3 N, D], row k 3 N + i (P = 1 for the classical thermostat), and the Philox application counter.

    The extended momenta s (s[0] = p, or the normal-mode momentum p~_k) follow s <- c1 s + sqrt(m) c2 xi with c1 =
    exp(-dt/2 A) and c2 = sqrt(C - c1 C c1^T), the propagator of Ceriotti, Bussi, Parrinello (JCTC 6, 1170, 2010).  The
    reference multiplies the row vector s by c1, which is c1^T s: for a non-normal A that chain does not keep C as its
    stationary covariance, so this thermostat departs from it there on purpose (DESIGN.md section 9).  For a symmetric A
    both are the same.  xi comes from Philox4x32-10 keyed by ``seed``: normal d of the draw of element (j P + k) N + a for
    column j; the free-particle-limit start s = xi c2 (no mass factor, thermostats.py:687-701) is application 0."""

    _per_mode = False

    def __init__(self, temperature_bath: float, gle_file: str, free_particle_limit: bool = True, seed: int = 0,
                 kB: float = KB_MD, fs: float = FS_MD):
        super().__init__(temperature_bath, 0.0, kB=kB, fs=fs)          # thermostats.py:557-559
        self.gle_file = str(gle_file)
        self.free_particle_limit = bool(free_particle_limit)
        self.seed = seed
        self.A, self.C = load_gle_matrices(self.gle_file, kB=kB, fs=fs)
        if not self._per_mode and self.A.shape[0] > 1:                    # thermostats.py:603-606
            raise ValueError(f"{type(self).__name__}: more than one A matrix found in {self.gle_file}. Could be PIGLET "
                             "input (PIGLETThermostat).")
        self.state: Optional[Tensor] = None

    def _n_beads(self) -> int:
        return self.rp.n_beads if self.ring_polymer else 1

    def _init_state(self):
        s = self.systems
        dev = s.masses.device
        P = self._n_beads()
        A, C, D = self.A, self.C, int(self.A.shape[-1])
        if self._per_mode and A.shape[0] != P:                            # thermostats_rpmd.py:348-352
            raise ValueError(f"{type(self).__name__}: expected {P} A matrices, one per normal mode, but found "
                             f"{A.shape[0]} in {self.gle_file}")
        if C is None:                                                     # thermostats.py:639-648
            C = torch.eye(D, dtype=torch.float64).expand_as(A) * (self.temperature_bath * self.kB)
            if self.ring_polymer:
                C = C * P
        c1, c2 = zip(*(_gle_propagators(A[b], C[b], self.time_step) for b in range(A.shape[0])))
        self.c1, self.c2 = torch.stack(c1).to(dev), torch.stack(c2).to(dev)
        self.c_transform = self.rp.c_transform if self.ring_polymer else torch.ones(1, 1, dtype=torch.float64,
                                                                                    device=dev)
        self.state = torch.zeros(P * 3 * s.n_atoms, D, dtype=torch.float64, device=dev)
        self.seed, self.counter = _noise(self.seed, dev)
        if self.free_particle_limit:
            self._call(None, 1)

    def _call(self, momenta: Optional[Tensor], initial: int):
        s = self.systems
        _lib.call("spk_rpmd_gle", ops._p(momenta), ops._p(s.masses), s.n_atoms, self._n_beads(),
                  ops._p(self.c_transform), ops._p(self.c1), ops._p(self.c2), int(self.A.shape[-1]),
                  1 if self._per_mode else 0, ops._p(self.state), self.seed, ops._p(self.counter), initial, ops._stream())

    def apply(self, momenta: Tensor):
        self._call(momenta, 0)

    def _state(self):
        return {"state": self.state, "counter": self.counter}


class GLEThermostat(_GLE, _Thermostat):
    """Generalized-Langevin (colored-noise) thermostat (thermostats.py:527-730) with the reference's keywords plus ``seed``,
    ``kB`` and ``fs``: the matrices come from the gle4md file ``gle_file`` (one A block; with no C, C = kB T I), and with
    ``free_particle_limit`` the extended momenta start as xi c2, else at zero.  See ``_GLE`` for the propagator, which is
    that of the GLE papers and not the reference's transpose."""

    ring_polymer = False


class RPMDGLEThermostat(_GLE, _RingPolymerThermostat):
    """GLE thermostat on every normal mode of the bead momenta (thermostats_rpmd.py:237-295): one A for all modes, with
    no C in the file C = P kB T I.  It runs the classical thermostat's kernel on p~_k, so at P = 1 it equals
    ``GLEThermostat`` bitwise.  The reference notes that its version "does not seem to give the proper temperature
    average"; its transposed propagator is the cause for a non-normal A (see ``_GLE``)."""


class PIGLETThermostat(RPMDGLEThermostat):
    """PIGLET (Ceriotti and Manolopoulos 2012; thermostats_rpmd.py:298-370): one GLE per normal mode, block k of the file
    on mode k, so the file needs exactly ``n_beads`` blocks.  Always starts in the free-particle limit."""

    _per_mode = True

    def __init__(self, temperature_bath: float, gle_file: str, seed: int = 0, kB: float = KB_MD, fs: float = FS_MD):
        super().__init__(temperature_bath, gle_file, free_particle_limit=True, seed=seed, kB=kB, fs=fs)


class PILEBarostat(_TensorState):
    """Isotropic barostat of ring-polymer NPT (barostats_rpmd.py:21-208, after i-PI 2.0, Kapil et al. 2019) with the
    reference's keywords: target pressure in bar, bath temperature of the cell in K, time constant in fs; ``kB``, ``fs``
    and ``bar`` define the caller's MD units.  It acts on the centroid mode and the cell only and thermostats the cell
    momentum with a PILE step, so any ring-polymer thermostat (or none) can run next to it.

    One cell momentum p_c per system of mass W = 3 N_s kB T / omega^2 with omega = 1 / tau (:83-85); the cell thermostat
    is p_c = c1 p_c + c2 xi with c1 = exp(-dt / (2 tau)) and c2 = sqrt(P W kB T (1 - c1^2)) (:88-99).  xi comes from
    Philox4x32-10 keyed by ``seed`` with the counter (system, application); the application index lives on the device and
    advances with every application, also inside a replayed graph.  State (p_c, counter) is on the device."""

    ring_polymer = True
    temperature_control = False

    def __init__(self, target_pressure: float, temperature_bath: float, time_constant: float, seed: int = 0,
                 kB: float = KB_MD, fs: float = FS_MD, bar: float = BAR_MD):
        self.target_pressure = float(target_pressure) * float(bar)               # barostats.py:51-53
        self.temperature_bath = _bath_temperature(temperature_bath, type(self).__name__)
        self.time_constant = float(time_constant) * float(fs)
        self.frequency = 1.0 / self.time_constant                               # barostats_rpmd.py:53
        self.kB = float(kB)
        self.kb_temperature = self.temperature_bath * self.kB                   # :56
        self.seed = seed
        self.cell_momenta: Optional[Tensor] = None

    def bind(self, systems: _Systems, time_step: float, ring_polymer: Optional[RingPolymer] = None):
        """_init_barostat (:66-99) for the base batch ``systems`` (one copy of every molecule)."""
        if ring_polymer is None:
            raise ValueError("PILEBarostat is a ring-polymer barostat: pass DeviceMD(ring_polymer=...)")
        self.rp = ring_polymer
        self.systems = s = systems
        self.time_step = float(time_step)
        dev = s.masses.device
        kbt = self.kb_temperature
        self.cell_momenta = torch.zeros(s.n_sys, dtype=torch.float64, device=dev)
        self.cell_mass = 3.0 * s.n_atoms_sys * kbt / self.frequency ** 2                # :83-85
        self.c1 = math.exp(-0.5 * self.frequency * self.time_step)                      # :88-93
        self.c2 = torch.sqrt(ring_polymer.n_beads * self.cell_mass * kbt * (1.0 - self.c1 ** 2))   # :94-99
        self.seed, self.counter = _noise(self.seed, dev)

    def apply_thermostat(self):
        """_update_barostat (:101-110) at on_step_begin and on_step_end"""
        _lib.call("spk_rpmd_barostat_thermostat", ops._p(self.cell_momenta), self.systems.n_sys, self.c1,
                  ops._p(self.c2), self.seed, ops._p(self.counter), ops._stream())

    def half_step(self, momenta: Tensor, forces: Tensor, force_conversion: float, cell: Tensor, virial: Tensor,
                  virial_scale: float):
        """propagate_half_step (:164-205) up to the particle kick, which DeviceMD enqueues next: p_c from the momenta
        before the kick, the forces * force_conversion, and the bead systems' cells and virials"""
        s, rp = self.systems, self.rp
        ws = s.workspace("spk_rpmd_barostat_workspace_bytes")
        _lib.call("spk_rpmd_barostat_half_step", ops._p(momenta), ops._p(forces), float(force_conversion),
                  ops._p(s.masses), ops._p(s.idx_m), ops._p(s.sys_ptr), s.n_atoms, s.n_sys, rp.n_beads,
                  ops._p(rp.c_transform), ops._p(cell), ops._p(virial), float(virial_scale), self.target_pressure,
                  self.kb_temperature, self.time_step, ops._p(self.cell_mass), ops._p(self.cell_momenta),
                  ops._p(ws), ws.numel(), ops._stream())

    def main_step(self, positions: Tensor, momenta: Tensor, model_positions: Optional[Tensor], cell: Tensor,
                  model_cell: Optional[Tensor], position_conversion: float):
        """propagate_main_step (:113-162): centroid mode and cell scaled by the cell momentum, modes k >= 1 free"""
        s, rp = self.systems, self.rp
        ws = s.workspace("spk_rpmd_barostat_workspace_bytes")
        _lib.call("spk_rpmd_barostat_main_step", ops._p(positions), ops._p(momenta), ops._p(model_positions),
                  ops._p(s.masses), ops._p(s.idx_m), s.n_atoms, s.n_sys, rp.n_beads, ops._p(rp.c_transform),
                  ops._p(rp.u), self.time_step, ops._p(self.cell_momenta), ops._p(self.cell_mass), ops._p(cell),
                  ops._p(model_cell), float(position_conversion), ops._p(ws), ws.numel(), ops._stream())

    def _state(self) -> Dict[str, Tensor]:
        return {"cell_momenta": self.cell_momenta, "counter": self.counter}


# ---- initial conditions and basic simulation hooks --------------------------------------------------------------------------
WRAP_EPS = 1e-6          # system.py:652, the buffer of wrap_positions


class _Initializer:
    """Common part of the initializers (md/initial_conditions.py:17-116) with the reference's keywords and defaults plus
    ``seed`` and ``kB`` (MD energy per kelvin).  ``DeviceMD(..., initializer=...)`` applies it once, after ring-polymer
    replication and the binding of the hooks and before the forces at t = 0, in the reference's order: centre of mass,
    wrapping, momenta, translation, rotation.  ``temperature`` in K is one number or one per system of the batch; every
    bead of a ring polymer draws its own momenta.

    Deliberate differences from the reference: the normals come from Philox4x32-10 keyed by ``seed`` with the counter
    (atom, 2^64 - 1), an application index that no thermostat reaches (the reference uses torch.randn); the rotation of a
    single atom or a linear molecule uses the pseudo-inverse of its inertia tensor (``RemoveCOMMotion``); ring polymers
    wrap by their centroids (``WrapPositions``)."""

    uniform = 0

    def __init__(self, temperature, remove_center_of_mass: bool = True, remove_translation: bool = True,
                 remove_rotation: bool = False, wrap_positions: bool = False, seed: int = 0, kB: float = KB_MD):
        name = type(self).__name__
        temps = temperature.tolist() if isinstance(temperature, torch.Tensor) else temperature
        temps = [float(t) for t in (temps if isinstance(temps, (list, tuple)) else [temps])]
        if not temps or not all(t >= 0.0 for t in temps):
            raise ValueError(f"{name}: temperature must be one or more values >= 0 K, got {temperature}")
        self.temperature = temps
        self.remove_center_of_mass = bool(remove_center_of_mass)
        self.remove_translation = bool(remove_translation)
        self.remove_rotation = bool(remove_rotation)
        self.wrap_positions = bool(wrap_positions)
        self.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        self.kB = float(kB)

    def system_temperatures(self, n_sys: int, n_copies: int, device) -> Tensor:
        """[n_copies n_sys] fp64 target temperature of every (bead) system (initial_conditions.py:57-61)"""
        return _one_per_system(self.temperature, n_sys, type(self).__name__).repeat(n_copies).to(device)

    def initialize(self, md: "DeviceMD"):
        """initialize_system (initial_conditions.py:50-75) on the state of ``md``, in place"""
        s = md.systems
        base = md._rp_base if md._rp_base is not None else s
        temps = self.system_temperatures(base.n_sys, md._n_replicas(), md.positions.device)
        if self.remove_center_of_mass:
            md._remove_motion(_lib.MOTION_CENTER_OF_MASS)
        if self.wrap_positions:
            md._wrap_positions()
        ws = s.workspace("spk_md_motion_workspace_bytes")
        _lib.call("spk_md_initial_momenta", ops._p(md.momenta), ops._p(s.masses), ops._p(s.idx_m), ops._p(s.sys_ptr),
                  s.n_atoms, s.n_sys, self.uniform, self.kB, ops._p(temps), self.seed, ops._p(ws), ws.numel(),
                  ops._stream(), launches=4 if self.uniform else 1)
        flags = (_lib.MOTION_TRANSLATION if self.remove_translation else 0) | \
                (_lib.MOTION_ROTATION if self.remove_rotation else 0)
        if flags:
            md._remove_motion(flags)


class MaxwellBoltzmannInit(_Initializer):
    """Momenta from the Maxwell-Boltzmann distribution (initial_conditions.py:138-188): p = sqrt(m kB T_s) xi per atom,
    with T_s the temperature of the atom's system.  (With one temperature per system the reference fails in
    ``expand_atoms``; here each system gets its own width.)"""


class UniformInit(_Initializer):
    """Momenta p = m xi, then every (bead) system rescaled to exactly its temperature (initial_conditions.py:91-135; the
    weight is the mass, not its square root, as in the reference).  A system whose draw has zero kinetic energy (no
    atoms) is left unchanged."""

    uniform = 1


def _check_every(every_n_steps, who: str) -> int:
    if int(every_n_steps) != every_n_steps or int(every_n_steps) < 1:
        raise ValueError(f"{who}: every_n_steps must be an integer >= 1, got {every_n_steps}")
    return int(every_n_steps)


class RemoveCOMMotion:
    """md/simulation_hooks/basic_hooks.py:41-61: on steps s % every_n_steps == 0 (s = 0, 1, ... counted on the device, so
    the first step runs it) move every (bead) system to its centre of mass, remove its mean momentum and, with
    ``remove_rotation``, its rotation about the origin.  Runs after the thermostat and barostat of the step and before the
    recorder, inside the captured step.  The rotation uses the pseudo-inverse of the inertia tensor: eigenvalues at or
    below 1e-10 x the largest give no angular velocity (a single atom, a linear molecule), where the reference's
    torch.inverse fails; where the tensor is regular this is I^-1 L."""

    def __init__(self, every_n_steps: int, remove_rotation: bool):
        self.every_n_steps = _check_every(every_n_steps, "RemoveCOMMotion")
        self.remove_rotation = bool(remove_rotation)

    def apply(self, md: "DeviceMD"):
        flags = _lib.MOTION_CENTER_OF_MASS | _lib.MOTION_TRANSLATION
        md._remove_motion(flags | (_lib.MOTION_ROTATION if self.remove_rotation else 0), self.every_n_steps)


class WrapPositions:
    """md/simulation_hooks/basic_hooks.py:64-78: on steps s % every_n_steps == 0 wrap the atoms back into the cell on its
    periodic axes (system.py:652-684, eps = 1e-6).  The cell is the run's MD cell when it keeps one (barostat or
    ``compute_stress``), else the batch's ``_cell`` / position_conversion.  All beads of a ring-polymer atom move by the
    lattice translation that wraps their centroid (the reference wraps every bead on its own, which tears a ring polymer
    that straddles a face and changes its spring energy)."""

    def __init__(self, every_n_steps: int):
        self.every_n_steps = _check_every(every_n_steps, "WrapPositions")

    def apply(self, md: "DeviceMD"):
        md._wrap_positions(self.every_n_steps)


class _CapturedEvaluation:
    """The force evaluation of a device-resident loop (calculator.calculate) and the capture of one whole step with it:
    neighbour list on the fixed-capacity ``self.nl``, ``self.model`` on ``self.static`` and copies of the outputs into
    ``self.energy`` / ``self.forces``, with the sticky overflow watch ``self.nl_watch``.  ``DeviceMD``,
    ``vibrations.DeviceVibrations`` and the batchwise optimizers of ``relax._BatchOptimizer`` (``relax.DeviceLBFGS``,
    ``relax.DeviceFIRE`` and ``neb.DeviceNEB``) build their steps around it: each defines ``_step()`` and
    ``_step_state()``, the (nested) dict of every tensor the step writes."""

    energy_key = P.energy
    force_key = P.forces
    virial: Optional[Tensor] = None
    required_properties: List[str] = []
    # members of an ensemble run (None: one model); their outputs are stacked into ``self.stacks[key]`` [K, ...]
    ensemble: Optional[List[torch.nn.Module]] = None
    stacks: Dict[str, Tensor] = {}

    def _setup(self, model, batch: Dict[str, Tensor], cutoff: float, capacity: int, use_graph: bool):
        """The set-up every driver shares: checks of the batch and the model, ``self.model`` (``_set_ensemble``),
        ``self.static`` (the batch without its neighbour list), the padded neighbour list of ``capacity`` pairs and the
        empty evaluation buffers.  Returns the batch layout (idx_m, n_sys)."""
        name = type(self).__name__
        if batch[P.R].device.type != "cuda":
            raise ValueError(f"{name} needs a CUDA batch (no CPU fallback)")
        model = self._set_ensemble(model, name)
        check_padded_pair_terms(model, float(cutoff), name)
        check_ewald_cells(model, batch, name)
        self.model = model
        self.use_graph = use_graph
        self.static = {k: v.detach().clone() for k, v in batch.items() if k not in (P.idx_i, P.idx_j, P.offsets)}
        self.nl = CellListNeighborList(cutoff, capacity=int(capacity), pad=True)
        self.energy: Optional[Tensor] = None
        self.forces: Optional[Tensor] = None
        self.n_pairs: Optional[Tensor] = None
        # sticky bookkeeping of the fixed-capacity neighbour list, updated INSIDE the captured step: [0] = largest pair
        # count seen so far, [1] = 1 if any step overflowed ``capacity`` (its list was then truncated)
        self.nl_watch = torch.zeros(2, dtype=torch.int64, device=batch[P.R].device)
        self._graph = None
        return _batch_layout(self.static)

    # ---- one force evaluation on the current positions (calculator.calculate) ---------------------------------------------
    def _calculate(self):
        ops._GRAPH_CACHE.clear()
        x = {k: (v.detach() if v.is_floating_point() else v) for k, v in self.static.items()}
        if self.virial is not None:
            x[P.virial] = self.virial
        x = self.nl(x)
        if self.ensemble is not None:
            return self._calculate_ensemble(x)
        with padded_list_cutoff(self.model, self.nl._cutoff):     # the padding pairs of the fixed-capacity list
            out = self.model(x)
        e, f = out[self.energy_key].detach(), out[self.force_key].detach()
        if self.energy is None:
            self.energy, self.forces, self.n_pairs = e.clone(), f.clone(), x["_n_pairs"].clone()
        else:
            self.energy.copy_(e)
            self.forces.copy_(f)
            self.n_pairs.copy_(x["_n_pairs"])
        torch.maximum(self.nl_watch, x["_n_pairs"], out=self.nl_watch)
        if self.required_properties:
            self._refresh_properties(out)

    def _calculate_ensemble(self, x: Dict[str, Tensor]):
        """EnsembleCalculator.calculate (ensemble_calculator.py:20-35): every member on the same neighbour list (and so on
        the same EdgeGraph of ops._GRAPH_CACHE), each output copied into its slot before the next member reuses its
        buffers, then the statistics over the slots (``_ensemble_statistics``)."""
        keys = [self.energy_key, self.force_key] + [p for p in self.required_properties
                                                     if p not in (self.energy_key, self.force_key)]
        K = len(self.ensemble)
        first = not self.stacks
        for k, member in enumerate(self.ensemble):
            with padded_list_cutoff(member, self.nl._cutoff):
                out = member(dict(x))
            for p in keys:
                v = out[p].detach()
                if first and k == 0:
                    if v.dtype != torch.float32 or not v.is_contiguous():
                        raise TypeError(f"{type(self).__name__}: output '{p}' must be a contiguous float32 tensor")
                    self.stacks[p] = torch.empty((K,) + tuple(v.shape), dtype=torch.float32, device=v.device)
                elif tuple(v.shape) != tuple(self.stacks[p].shape[1:]):
                    raise ValueError(f"{type(self).__name__}: ensemble member {k} predicts '{p}' of shape "
                                     f"{tuple(v.shape)}, member 0 {tuple(self.stacks[p].shape[1:])}")
                self.stacks[p][k].copy_(v)
        if self.energy is None:
            e, f = self.stacks[self.energy_key], self.stacks[self.force_key]
            self.energy = torch.empty(e.shape[1:], dtype=torch.float32, device=e.device)
            self.forces = torch.empty(f.shape[1:], dtype=torch.float32, device=f.device)
            self.n_pairs = x["_n_pairs"].clone()
        else:
            self.n_pairs.copy_(x["_n_pairs"])
        torch.maximum(self.nl_watch, x["_n_pairs"], out=self.nl_watch)
        self._ensemble_statistics()

    def _ensemble_statistics(self):
        """the mean energies and forces that drive the step (BatchwiseEnsembleCalculator.calculate)"""
        from .ensemble import ensemble_forces, ensemble_moments

        ensemble_moments(self.stacks[self.energy_key], var=False, out_mean=self.energy)
        ensemble_forces(self.stacks[self.force_key], var=False, out_mean=self.forces)

    def _set_ensemble(self, model, who: str) -> torch.nn.Module:
        """``model`` as the module the driver keeps: an ``nn.ModuleList`` of the members of an ensemble (``self.ensemble``)
        or the single model"""
        from .ensemble import members_of

        members = members_of(model)
        if members is None:
            return model
        self.ensemble = members
        self.stacks = {}
        for m in members:
            outputs = getattr(m, "model_outputs", None)
            if outputs is not None and (self.energy_key not in outputs or self.force_key not in outputs):
                raise ValueError(f"{who}: every ensemble member must output '{self.energy_key}' and '{self.force_key}' "
                                 f"(one outputs {sorted(outputs)})")
        return torch.nn.ModuleList(members)

    def _evaluation_state(self) -> Dict[str, Tensor]:
        return {"energy": self.energy, "forces": self.forces, "n_pairs": self.n_pairs, "nl_watch": self.nl_watch}

    def _setup_virial(self, n_sys: int, what: str) -> Tensor:
        """The model cell ``static[_cell]`` (checked to be a contiguous fp32 [n_sys, 3, 3] tensor, returned as it is) and
        ``self.virial``, the fp64 [n_sys, 3, 3] model-unit virial that every evaluation then writes."""
        name = type(self).__name__
        if P.cell not in self.static:
            raise ValueError(f"{name}: {what} need a periodic batch with a '_cell'")
        model_cell = self.static[P.cell]
        if model_cell.dtype != torch.float32 or not model_cell.is_contiguous() or model_cell.numel() != 9 * n_sys:
            raise ValueError(f"{name}: '_cell' must be a contiguous float32 [n_sys, 3, 3] tensor")
        self.virial = torch.zeros(n_sys, 3, 3, dtype=torch.float64, device=model_cell.device)
        return model_cell

    def _check_periodic(self, n_sys: int, volume: Tensor, what: str):
        """refuse a batch in which a system is not periodic on all three axes or has zero ``volume`` [n_sys]"""
        name = type(self).__name__
        pbc = self.static.get(P.pbc)
        if pbc is None or not bool(pbc.reshape(-1, 3).all()) or pbc.reshape(-1, 3).shape[0] not in (1, n_sys):
            raise ValueError(f"{name}: {what} needs every system periodic on all three axes (system.py:599-602)")
        if bool((volume == 0.0).any()):
            raise ValueError(f"{name}: {what} needs a non-zero cell volume for every system (system.py:599-602)")

    def _run_steps(self, n: int):
        """``n`` steps: replays of the step, captured on first use, or eager ``_step()`` calls without ``use_graph``."""
        if n > 0 and self.use_graph and self._graph is None:
            self._graph = self._capture_step()
        for _ in range(n):
            if self.use_graph:
                self._graph.replay()
            else:
                self._step()

    def _capture_step(self) -> "torch.cuda.CUDAGraph":
        """Capture ``self._step()`` into a CUDA graph.  The tensors of ``_step_state()`` are restored after the warm-up
        iteration, so that capturing does not advance the run."""
        dev = self.static[P.R].device
        state = _flatten(self._step_state())
        saved = [t.clone() for t in state]
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            self._step()
        torch.cuda.current_stream(dev).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._step()
        for dst, src in zip(state, saved):
            dst.copy_(src)
        return graph

    def check_neighbor_list(self):
        """One host read per ``run``: raise if ANY step since the start overflowed the list capacity (the search then
        dropped pairs and the trajectory is wrong from that step on).  ``peak_pairs`` tells how much head-room is left."""
        peak, over = (int(v) for v in self.nl_watch.tolist())
        self.peak_pairs = peak
        if over:
            name = type(self).__name__
            raise RuntimeError(
                f"{name}: the neighbour list overflowed its capacity of {self.nl.capacity} pairs during the run (peak "
                f"{peak}); the trajectory is invalid from that step on -- re-create {name} with a larger capacity")


class DeviceMD(_CapturedEvaluation):
    def __init__(self, model: torch.nn.Module, batch: Dict[str, Tensor], masses: Tensor, time_step: float, cutoff: float,
                 capacity: int, momenta: Optional[Tensor] = None, use_graph: bool = True,
                 position_conversion: float = 1.0, energy_conversion: float = 1.0,
                 thermostat: Optional[_Thermostat] = None, barostat: Optional[object] = None,
                 compute_stress: bool = False, ring_polymer: Optional[RingPolymer] = None,
                 required_properties: Optional[List[str]] = None,
                 property_conversion: Optional[Dict[str, float]] = None, record_every: int = 1,
                 record_capacity: int = 0, uncertainty_fn: Optional[object] = None, record_velocities: bool = False,
                 initializer: Optional[_Initializer] = None, hooks: Optional[List[object]] = None,
                 stream: Optional[object] = None):
        """``batch[_positions]`` (and ``_cell``) are in MODEL units as everywhere in this package; ``self.positions`` is the
        MD-unit state (= model positions / position_conversion).  ``thermostat`` (None = NVE) is bound to the systems of
        the batch and applied around every step.  ``barostat`` (an NHC barostat, which thermostats the particles itself)
        makes the run NPT: every system must be periodic on all three axes.  ``compute_stress`` keeps the virial (and so
        ``stress`` / ``pressure``) up to date in an NVE / NVT run.

        ``ring_polymer`` (a ``RingPolymer``) makes the run ring-polymer MD: the B-system ``batch`` is replicated into P
        beads, replica-major (P B systems; bead r of system m is system r B + m, positions [P, N, 3] flat as [P N, 3]), all
        beads start at the batch positions, ``momenta`` may be [N, 3] (copied to every bead) or [P, N, 3], and ``capacity``
        is the pair capacity of the whole bead batch.  It takes only the ring-polymer thermostats and, for NPT, the
        ``PILEBarostat`` (next to a ring-polymer thermostat or alone); no NHC barostat and no ``compute_stress``.

        ``required_properties`` (model output keys such as ``dipole_moment`` or ``polarizability``) are kept in
        ``self.properties[name]`` after every evaluation, shaped ``[n_replicas, B, ...]`` (n_replicas = number of beads,
        1 without a ring polymer) and multiplied by ``property_conversion[name]`` (default 1.0), as the reference's
        calculator does (md/calculators/base_calculator.py:50-141).  The conversion is a number: unit strings would need
        ASE's unit tables.  With ``record_capacity`` > 0 the step also appends them to a device-side time series every
        ``record_every`` steps (steps s with s % record_every == 0, counted from the start), written inside the captured
        step; ``recorded(name)`` returns the series, ``drain()`` empties it, and ``run`` refuses a call that would store
        more than ``record_capacity`` records since the last drain.  ``record_velocities`` adds the series
        ``"velocities"`` [record_capacity, n_replicas, N, 3] = momenta / masses in MD units (the FileLogger's
        MoleculeStream with store_velocities), which power spectra need; it needs ``record_capacity`` > 0 and no
        required property of that name.  ``series()`` hands the records since the last drain to ``spectra``.

        ``model`` may be a list (or ``nn.ModuleList``) of at least two members: an ensemble run
        (md/calculators/ensemble_calculator.py).  Every member runs on the step's one neighbour list, the mean energies and
        forces drive the dynamics, and ``self.properties`` holds ``energy``, ``forces`` and every required property as
        the member mean times ``property_conversion[p]`` (default 1.0, for the energy and forces too, as the reference's
        calculator), plus ``{p}_var``: the unbiased variance over the members times the same linear factor
        (ensemble_calculator.py:70-81).  ``uncertainty_fn`` (an ``ensemble.AbsoluteUncertainty`` /
        ``RelativeUncertainty`` on the run's energy and force keys, without a stress weight) adds
        ``properties["uncertainty"]`` [n_replicas, B] of the energies and forces as ``properties`` holds them.  Stress
        and barostats are refused with an ensemble, as in the reference.

        ``initializer`` (a ``MaxwellBoltzmannInit`` or ``UniformInit``) sets the starting state as the reference's
        system.initializer does (md/cli.py:154-157): after ring-polymer replication and the binding of the thermostat and
        barostat, before the forces at t = 0; it replaces ``momenta``, which it refuses next to it.  ``hooks`` (a list of
        ``RemoveCOMMotion`` / ``WrapPositions`` / ``structure.RadialDistribution`` / ``structure.MeanSquaredDisplacement`` /
        ``exchange.ReplicaExchange``) run in the listed order after the step's thermostat or barostat and before the
        recorder, as the reference's simulation hooks at on_step_finalize; they are gated by a device step counter, which
        ``state_dict`` carries with the structure hooks' accumulators and the exchange statistics, so a restarted run keeps
        their phase and continues bitwise.

        ``stream`` (a ``spectra.SpectrumStream``) accumulates the autocorrelations the spectra need inside the step, on
        the steps the recorder would record, before the step counter advances; it works without a recorder, reads the
        properties it needs from ``required_properties``, is carried by ``state_dict`` and untouched by ``drain``."""
        idx_m, n_sys = self._setup(model, batch, cutoff, capacity, use_graph)
        self.hooks = self._check_hooks(hooks, initializer, momenta)
        self._check_ensemble(barostat, compute_stress, uncertainty_fn)
        self.uncertainty_fn = uncertainty_fn
        if barostat is not None and thermostat is not None and getattr(barostat, "temperature_control", True):
            raise ValueError("DeviceMD: the NHC barostats contain their own thermostat (temperature_control = True); "
                             "pass either a thermostat or a barostat")
        self._check_ring_polymer(ring_polymer, thermostat, barostat, compute_stress)
        dev = batch[P.R].device
        self.ring_polymer = ring_polymer
        self.dt = float(time_step)
        self.p_conv = float(position_conversion)
        self.e_conv = float(energy_conversion)
        self.f_conv = self.e_conv / self.p_conv                                   # base_calculator.py:96
        masses = masses.to(dev, torch.float32).reshape(-1).contiguous().clone()
        self._rp_base: Optional[_Systems] = None
        if ring_polymer is not None:
            n = self.static[P.R].shape[0]
            if masses.shape[0] != n:
                raise ValueError(f"DeviceMD: {masses.shape[0]} masses for {n} atoms")
            self._rp_base = b = _Systems(masses, idx_m, n_sys)
            self.static.setdefault(P.idx_m, idx_m)
            self.static.setdefault(P.n_atoms, (b.sys_ptr[1:] - b.sys_ptr[:-1]).to(torch.int64))
            self.static = replicate_batch(self.static, ring_polymer.n_beads, n_sys)
            masses = masses.repeat(ring_polymer.n_beads)
            ring_polymer.bind(b, self.dt)
        self.model_positions = self.static[P.R]                                   # what the model reads
        self.positions = self.model_positions if self.p_conv == 1.0 else self.model_positions / self.p_conv
        # the model-unit copy the position kernels update next to the MD positions (None when the units agree)
        self._mp = self.model_positions if self.model_positions is not self.positions else None
        self.masses = masses
        if momenta is None:
            self.momenta = torch.zeros_like(self.positions)
        elif ring_polymer is None:
            self.momenta = momenta.to(dev, torch.float32).clone()
        else:
            momenta = momenta.to(dev, torch.float32).reshape(-1, 3)
            if momenta.shape[0] == self._rp_base.n_atoms:
                momenta = momenta.repeat(ring_polymer.n_beads, 1)                # [N, 3] -> every bead
            if momenta.shape != self.positions.shape:
                raise ValueError(f"DeviceMD: ring-polymer momenta must be [N, 3] or [P, N, 3], got "
                                 f"{momenta.shape[0]} rows for N = {self._rp_base.n_atoms}, P = {ring_polymer.n_beads}")
            self.momenta = momenta.contiguous().clone()
        self.steps_done = 0
        self._systems: Optional[_Systems] = None
        self.thermostat = thermostat
        if ring_polymer is not None and thermostat is not None:
            thermostat.bind(self._rp_base, self.dt, ring_polymer)                # on_simulation_start
        elif thermostat is not None:
            thermostat.bind(self.systems, self.dt)
        self.barostat = barostat
        self.cell: Optional[Tensor] = None          # MD-unit cell [n_sys, 3, 3] fp64 (the model reads static[_cell])
        self.virial: Optional[Tensor] = None        # model-unit virial [n_sys, 3, 3] fp64, written by every evaluation
        if barostat is not None or compute_stress:
            n_sys = self.systems.n_sys
            self.model_cell = self._setup_virial(n_sys, "stress and NPT")
            self.cell = self.model_cell.reshape(n_sys, 3, 3).double() / self.p_conv
        if barostat is not None:
            self._check_periodic(n_sys, self.volume(), "NPT")
            if ring_polymer is not None:
                barostat.bind(self._rp_base, self.dt, ring_polymer)               # on_simulation_start
            else:
                barostat.bind(self.systems, self.dt)
        self._setup_properties(required_properties, property_conversion, record_every, record_capacity,
                               record_velocities)
        self.stream = self._check_stream(stream)
        self._wrap_cell = None
        if any(isinstance(h, WrapPositions) for h in self.hooks) or getattr(initializer, "wrap_positions", False):
            self._setup_wrap()
        if initializer is not None:
            initializer.initialize(self)        # md/cli.py:154-157
        self._calculate()                       # forces at t = 0 (simulator.py:118)
        for h in self.hooks:                    # the accumulators of the structure hooks
            if hasattr(h, "_bind"):
                h._bind(self)
        if stream is not None:
            base = self._rp_base if self.ring_polymer is not None else self.systems
            stream._bind(self, base.sys_ptr.tolist(), self._n_replicas())

    def _check_stream(self, stream):
        if stream is None:
            return None
        from .spectra import SpectrumStream

        if not isinstance(stream, SpectrumStream):
            raise TypeError(f"DeviceMD: stream must be a spectra.SpectrumStream, got {type(stream).__name__}")
        if stream._md is not None:
            raise ValueError("DeviceMD: this SpectrumStream already belongs to another DeviceMD")
        missing = [p for p in stream.required_properties if p not in self.required_properties]
        if missing:
            raise ValueError(f"DeviceMD: the stream reads {missing}, which are not in required_properties "
                             f"{self.required_properties}")
        return stream

    @staticmethod
    def _check_hooks(hooks, initializer, momenta) -> list:
        if initializer is not None:
            if not isinstance(initializer, _Initializer):
                raise TypeError(f"DeviceMD: initializer must be a MaxwellBoltzmannInit or UniformInit, got "
                                f"{type(initializer).__name__}")
            if momenta is not None:
                raise ValueError("DeviceMD: pass either momenta or an initializer, which draws them")
        from .exchange import ReplicaExchange
        from .structure import MeanSquaredDisplacement, RadialDistribution

        hooks = list(hooks or [])
        for h in hooks:
            if not isinstance(h, (RemoveCOMMotion, WrapPositions, RadialDistribution, MeanSquaredDisplacement,
                                  ReplicaExchange)):
                raise TypeError(f"DeviceMD: hooks take RemoveCOMMotion, WrapPositions, structure.RadialDistribution, "
                                f"structure.MeanSquaredDisplacement and exchange.ReplicaExchange, got "
                                f"{type(h).__name__}")
            if getattr(h, "_md", None) is not None:
                raise ValueError(f"DeviceMD: this {type(h).__name__} already belongs to another DeviceMD")
        return hooks

    # ---- motion removal and wrapping (system.py:258-315,652-684) -------------------------------------------------------
    def _remove_motion(self, flags: int, every: Optional[int] = None):
        """spk_md_remove_motion on every (bead) system; with ``every`` gated by the device step counter"""
        s = self.systems
        ws = s.workspace("spk_md_motion_workspace_bytes")
        _lib.call("spk_md_remove_motion", ops._p(self.positions), ops._p(self._mp), ops._p(self.momenta),
                  ops._p(s.masses), ops._p(s.idx_m), ops._p(s.sys_ptr), s.n_atoms, s.n_sys, int(flags), self.p_conv,
                  ops._p(self._rec_counter if every else None), int(every or 1), ops._p(ws), ws.numel(), ops._stream())

    def _setup_wrap(self):
        """The cell and pbc rows the wrap reads: the MD cell when the run keeps one (it follows the barostat), else the
        batch's ``_cell`` / position_conversion, shared or one per system as the neighbour list takes them."""
        n_sys = self.systems.n_sys
        pbc = self.static.get(P.pbc)
        if self.cell is not None:
            cell = self.cell
        else:
            if P.cell not in self.static:
                raise ValueError("DeviceMD: wrapping positions needs a periodic batch with a '_cell'")
            cell = self.static[P.cell].reshape(-1, 3, 3).to(torch.float64) / self.p_conv
            if cell.shape[0] not in (1, n_sys):
                raise ValueError(f"DeviceMD: '_cell' has {cell.shape[0]} cells for {n_sys} systems")
            cell = cell.contiguous()
        if bool((torch.linalg.det(cell) == 0.0).any()):
            raise ValueError("DeviceMD: wrapping positions needs a non-zero cell volume for every system "
                             "(system.py:662-663)")
        if pbc is None:
            pbc = torch.zeros(1, 3, dtype=torch.uint8, device=cell.device)
        pbc = pbc.reshape(-1, 3).to(torch.uint8).contiguous()
        if pbc.shape[0] not in (1, n_sys):
            raise ValueError(f"DeviceMD: '_pbc' has {pbc.shape[0]} rows for {n_sys} systems")
        self._wrap_cell, self._wrap_pbc = cell, pbc

    def _wrap_positions(self, every: Optional[int] = None):
        """spk_md_wrap_positions on the (bead) positions; ring polymers move by their centroids' translations"""
        base = self._rp_base if self._rp_base is not None else self.systems
        cell, pbc = self._wrap_cell, self._wrap_pbc
        _lib.call("spk_md_wrap_positions", ops._p(self.positions), ops._p(self._mp), ops._p(base.idx_m), base.n_atoms,
                  self._n_replicas(), ops._p(cell), 9 if cell.shape[0] > 1 else 0, ops._p(pbc),
                  3 if pbc.shape[0] > 1 else 0, WRAP_EPS, self.p_conv, ops._p(self._rec_counter if every else None),
                  int(every or 1), ops._stream())

    @property
    def systems(self) -> _Systems:
        if self._systems is None:
            self._systems = _Systems(self.masses, *_batch_layout(self.static))
        return self._systems

    def _check_ensemble(self, barostat, compute_stress: bool, uncertainty_fn):
        if self.ensemble is None:
            if uncertainty_fn is not None:
                raise ValueError("DeviceMD: uncertainty_fn needs an ensemble (model=[m1, m2, ...])")
            return
        if compute_stress or barostat is not None:
            raise NotImplementedError("DeviceMD: stress and constant pressure are not available for ensembles (the "
                                      "reference's EnsembleCalculator._activate_stress raises, "
                                      "md/calculators/ensemble_calculator.py:62-68)")
        if uncertainty_fn is None:
            return
        from .ensemble import Uncertainty

        if not isinstance(uncertainty_fn, Uncertainty):
            raise TypeError(f"DeviceMD: uncertainty_fn must be an AbsoluteUncertainty or RelativeUncertainty, got "
                            f"{type(uncertainty_fn).__name__}")
        if uncertainty_fn.stress_weight > 0:
            raise NotImplementedError("DeviceMD: an ensemble run has no stress, so uncertainty_fn takes no stress_weight")
        keys = (uncertainty_fn.energy_key, uncertainty_fn.force_key)
        if keys != (self.energy_key, self.force_key):
            raise ValueError(f"DeviceMD: uncertainty_fn reads {keys}, the run predicts ('{self.energy_key}', "
                             f"'{self.force_key}')")

    # ---- ring-polymer set-up ------------------------------------------------------------------------------------------------
    @staticmethod
    def _check_ring_polymer(ring_polymer, thermostat, barostat, compute_stress):
        """the combinations the reference refuses (md/cli.py:256-267) or this package does not build"""
        rp_thermostat = getattr(thermostat, "ring_polymer", False)
        rp_barostat = getattr(barostat, "ring_polymer", False)
        if ring_polymer is None:
            if rp_thermostat:
                raise ValueError(f"DeviceMD: {type(thermostat).__name__} is a ring-polymer thermostat; it needs "
                                 "ring_polymer=RingPolymer(...)")
            if rp_barostat:
                raise ValueError(f"DeviceMD: {type(barostat).__name__} is a ring-polymer barostat; it needs "
                                 "ring_polymer=RingPolymer(...)")
            return
        if not isinstance(ring_polymer, RingPolymer):
            raise TypeError("DeviceMD: ring_polymer must be a RingPolymer")
        if thermostat is not None and not rp_thermostat:
            raise ValueError(f"DeviceMD: {type(thermostat).__name__} is a classical thermostat; ring-polymer MD takes "
                             "PILELocalThermostat, PILEGlobalThermostat, TRPMDThermostat, NHCRingPolymerThermostat, "
                             "RPMDGLEThermostat or PIGLETThermostat")
        if barostat is not None and not rp_barostat:
            raise ValueError(f"DeviceMD: {type(barostat).__name__} is not a ring-polymer barostat (md/cli.py:267-275); "
                             "ring-polymer NPT takes PILEBarostat")
        if compute_stress:
            raise ValueError("DeviceMD: compute_stress is not supported for ring-polymer MD")

    # ---- per-step model properties and their device-side time series ------------------------------------------------------
    def _setup_properties(self, required, conversion, every, capacity, velocities=False):
        self.required_properties = list(dict.fromkeys(required or []))
        if velocities and "velocities" in self.required_properties:
            raise ValueError("DeviceMD: record_velocities records the series 'velocities'; a required property of that "
                             "name would share it")
        conversion = dict(conversion or {})
        known = list(self.required_properties)
        if self.ensemble is not None:                # energy and forces are always required (base_calculator.py:65-69)
            known += [p for p in (self.energy_key, self.force_key) if p not in known]
        unknown = sorted(set(conversion) - set(known))
        if unknown:
            raise ValueError(f"DeviceMD: property_conversion names properties that are not required: {unknown}")
        for k, v in conversion.items():
            if isinstance(v, str):
                raise NotImplementedError(f"DeviceMD: property_conversion['{k}'] = {v!r}: give the conversion factor as a "
                                          "number (unit strings need ASE's unit tables)")
        self.property_conversion = {p: float(conversion.get(p, 1.0)) for p in known}
        for model in self.ensemble or [self.model]:
            outputs = getattr(model, "model_outputs", None)
            if outputs is not None:
                missing = [p for p in self.required_properties if p not in outputs]
                if missing:
                    raise ValueError(f"DeviceMD: required properties {missing} are not model outputs "
                                     f"({sorted(outputs)})")
        if int(every) < 1 or int(capacity) < 0:
            raise ValueError("DeviceMD: record_every must be >= 1 and record_capacity >= 0")
        if int(capacity) > 0 and not self.required_properties and self.ensemble is None and not velocities:
            raise ValueError("DeviceMD: record_capacity needs required_properties or record_velocities")
        if velocities and int(capacity) < 1:
            raise ValueError("DeviceMD: record_velocities needs record_capacity > 0")
        self.record_every, self.record_capacity = int(every), int(capacity)
        self.properties: Dict[str, Tensor] = {}
        self._records: Dict[str, Tensor] = {}
        if velocities:
            n_rep = self._n_replicas()
            self._records["velocities"] = torch.zeros(self.record_capacity, n_rep, self.positions.shape[0] // n_rep, 3,
                                                      dtype=torch.float32, device=self.positions.device)
        self._hook_series: Dict[str, Tensor] = {}    # series a hook records from its own buffer (name -> source)
        self._n_records = 0                      # host mirror of the device count: the record count is deterministic
        self._rec_counter = torch.zeros(2, dtype=torch.int64, device=self.positions.device)

    def _n_replicas(self) -> int:
        return self.ring_polymer.n_beads if self.ring_polymer is not None else 1

    def _refresh_properties(self, out: Dict[str, Tensor]):
        """properties[p] = out[p] viewed [n_replicas, B, ...] times the conversion (base_calculator.py:132-137)"""
        for p in self.required_properties:
            v = out[p].detach()
            if v.dtype != torch.float32 or not v.is_contiguous():
                raise TypeError(f"DeviceMD: property '{p}' must be a contiguous float32 model output")
            buf = self.properties.get(p)
            if buf is None:
                buf = torch.empty(v.reshape(self._n_replicas(), -1, *v.shape[1:]).shape, dtype=torch.float32,
                                  device=v.device)
                self.properties[p] = buf
                if self.record_capacity:
                    self._records[p] = torch.zeros((self.record_capacity,) + tuple(buf.shape), dtype=torch.float32,
                                                   device=v.device)
            _lib.call("spk_md_property", ops._p(v), v.numel(), self.property_conversion[p], ops._p(buf), ops._stream())

    def _property_buffer(self, name: str, shape, dtype=torch.float32) -> Tensor:
        """properties[name] of ``shape`` (and its record series), allocated on first use"""
        buf = self.properties.get(name)
        if buf is None:
            buf = torch.empty(shape, dtype=dtype, device=self.positions.device)
            self.properties[name] = buf
            if self.record_capacity:
                self._records[name] = torch.zeros((self.record_capacity,) + tuple(buf.shape), dtype=dtype,
                                                  device=buf.device)
        return buf

    def _ensemble_statistics(self):
        """EnsembleCalculator._accumulate_results (ensemble_calculator.py:38-59) and _update_system (base_calculator.py:
        120-141) with the conversions of _update_required_properties (ensemble_calculator.py:70-81): the mean energies
        and forces drive the step in model units; properties[p] = mean x property_conversion[p] and properties[p_var] =
        unbiased variance x the same factor, for the energy and forces too (default 1.0); with ``uncertainty_fn`` the
        per-system uncertainty of the energies and forces as properties holds them."""
        from .ensemble import ensemble_forces, ensemble_moments, ensemble_workspace

        ek, fk, st, n_rep = self.energy_key, self.force_key, self.stacks, self._n_replicas()
        conv = self.property_conversion
        prop = {}
        for p in conv:
            view = (n_rep, int(st[p].shape[1]) // n_rep) + tuple(st[p].shape[2:])      # [n_replicas, B, ...]
            prop[p] = self._property_buffer(p, view)
            prop[p + "_var"] = self._property_buffer(p + "_var", view)
        s, unc = self.systems, self.uncertainty_fn
        need_terms = unc is not None and unc.force_weight > 0
        if need_terms and not hasattr(self, "_ens_terms"):
            self._ens_terms = torch.empty(s.n_sys, 2, dtype=torch.float64, device=self.positions.device)
            self._ens_ws = ensemble_workspace(s.n_atoms, s.n_sys, self.positions.device)
        ensemble_moments(st[ek], ddof=1, spread_scale=conv[ek], out_mean=self.energy, out_var=prop[ek + "_var"])
        _lib.call("spk_md_property", ops._p(self.energy), self.energy.numel(), conv[ek], ops._p(prop[ek]), ops._stream())
        ensemble_forces(st[fk], s.idx_m, s.sys_ptr, s.n_sys, spread_scale=conv[fk], out_mean=self.forces,
                        out_var=prop[fk + "_var"], terms=need_terms, out_terms=self._ens_terms if need_terms else None,
                        workspace=self._ens_ws if need_terms else None)
        _lib.call("spk_md_property", ops._p(self.forces), self.forces.numel(), conv[fk], ops._p(prop[fk]), ops._stream())
        for p in conv:
            if p not in (ek, fk):
                ensemble_moments(st[p], ddof=1, mean_scale=conv[p], spread_scale=conv[p], out_mean=prop[p],
                                 out_var=prop[p + "_var"])
        if unc is not None:
            out = self._property_buffer("uncertainty", (n_rep, s.n_sys // n_rep))
            unc.combine(st[ek] if unc.energy_weight > 0 else None, self._ens_terms if need_terms else None, s.sys_ptr,
                        None, None, energy_scale=conv[ek], out_f32=out)

    def _record(self):
        if self.stream is not None:              # reads the counter before this step's advance, as the recorder does
            self.stream._push(self)
        if not self.record_capacity:
            if self.hooks or self.stream is not None:    # the step counter: the recorder's, which advances it otherwise
                _lib.call("spk_md_step_advance", ops._p(self._rec_counter), ops._stream())
            return
        for p, rec in self._records.items():
            if p == "velocities":
                _lib.call("spk_md_record_velocities", ops._p(self.momenta), ops._p(self.masses), self.momenta.shape[0],
                          ops._p(self._rec_counter), self.record_every, self.record_capacity, ops._p(rec),
                          ops._stream())
                continue
            buf = self._hook_series[p] if p in self._hook_series else self.properties[p]
            _lib.call("spk_md_record", ops._p(buf), buf.numel(), ops._p(self._rec_counter), self.record_every,
                      self.record_capacity, ops._p(rec), ops._stream())
        _lib.call("spk_md_record_advance", ops._p(self._rec_counter), self.record_every, self.record_capacity,
                  ops._stream())

    def _records_in(self, n_steps: int) -> int:
        k = self.record_every
        return (self.steps_done + n_steps) // k - self.steps_done // k

    def recorded(self, name: str) -> Tensor:
        """The time series of ``name`` since the last ``drain`` in step order, [n_records, n_replicas, B, ...] on the host
        (one device-to-host copy)."""
        if name not in self._records:
            raise KeyError(f"DeviceMD: '{name}' is not recorded (required_properties={self.required_properties}, "
                           f"record_capacity={self.record_capacity})")
        return self._records[name][:self._n_records].cpu()

    def series(self):
        """The records since the last ``drain`` as a ``spectra.RecordedSeries``: device views (no copy) with the record
        time step ``record_every * time_step`` in fs and the systems of one replica."""
        from .spectra import RecordedSeries

        if not self.record_capacity:
            raise RuntimeError("DeviceMD: series() needs a recorder (record_capacity > 0)")
        n = self._n_records
        base = self._rp_base if self.ring_polymer is not None else self.systems
        vel = self._records.get("velocities")
        return RecordedSeries(self.record_every * self.dt / FS_MD, base.sys_ptr, self._n_replicas(),
                              velocities=None if vel is None else vel[:n],
                              properties={p: v[:n] for p, v in self._records.items()
                                          if p != "velocities" and p not in self._hook_series})

    def drain(self) -> Dict[str, Tensor]:
        """Return every recorded series (as ``recorded``) and empty the recorder."""
        out = {p: self.recorded(p) for p in self._records}
        self._rec_counter[1].zero_()
        self._n_records = 0
        return out

    def _verlet(self, drift: bool):
        n = self.positions.shape[0]
        _lib.call("spk_md_velocity_verlet", ops._p(self.momenta), ops._p(self.positions), ops._p(self._mp),
                  ops._p(self.forces),
                  ops._p(self.masses), n, self.dt, self.f_conv, self.p_conv, 1 if drift else 0, ops._stream())

    def _virial_scale(self) -> float:
        # stress_MD = W / V_model * e_conv / p_conv^3 with V_model = V_MD p_conv^3 (base_calculator.py:97,218-222)
        return self.e_conv / self.p_conv ** 6

    def _npt_step(self):
        b = self.barostat
        b.apply_thermostat(self.momenta)                                           # simulator.py:127-128 on_step_begin
        b.kick(self.momenta, self.cell, self.virial, self._virial_scale())
        b.half_step(self.momenta, self.forces, self.f_conv)                        # integrators.py:249-257
        b.main_step(self.positions, self.momenta, self.cell, self._mp, self.model_cell, self.p_conv)   # :259-263
        self._calculate()                                                          # neighbour list on the new cell
        b.half_step(self.momenta, self.forces, self.f_conv)
        b.kick(self.momenta, self.cell, self.virial, self._virial_scale())        # simulator.py:149-150 on_step_end
        b.apply_thermostat(self.momenta)

    def _rpmd_step(self):
        """md/simulator.py:124-150 with the RingPolymer integrator (integrators.py:59-70,204-229): thermostat, half kick on
        every bead, ring-polymer main step, neighbour list + energy + forces on all P B bead systems, half kick,
        thermostat"""
        if self.thermostat is not None:
            self.thermostat.apply(self.momenta)
        self._verlet(False)
        self.ring_polymer.main_step(self.positions, self.momenta, self._mp, self.p_conv)
        self._calculate()
        self._verlet(False)
        if self.thermostat is not None:
            self.thermostat.apply(self.momenta)

    def _rpmd_npt_step(self):
        """md/simulator.py:124-150 with NPTRingPolymer (integrators.py:266-305) and hooks [thermostat, barostat]:
        thermostat, cell PILE, barostat half step + kick, centroid / cell / free-mode propagation, neighbour list on the new
        cells + energy + forces + virial on all P B bead systems, half step + kick, cell PILE, thermostat"""
        b = self.barostat
        if self.thermostat is not None:
            self.thermostat.apply(self.momenta)
        b.apply_thermostat()
        b.half_step(self.momenta, self.forces, self.f_conv, self.cell, self.virial, self._virial_scale())
        self._verlet(False)                                                        # barostats_rpmd.py:207-208
        b.main_step(self.positions, self.momenta, self._mp, self.cell, self.model_cell, self.p_conv)
        self._calculate()
        b.half_step(self.momenta, self.forces, self.f_conv, self.cell, self.virial, self._virial_scale())
        self._verlet(False)
        b.apply_thermostat()
        if self.thermostat is not None:
            self.thermostat.apply(self.momenta)

    def _step(self):
        self._dynamics()
        for hook in self.hooks:                  # simulation hooks at on_step_finalize (md/cli.py:231-314)
            hook.apply(self)
        self._record()

    def _dynamics(self):
        if self.ring_polymer is not None and self.barostat is not None:
            return self._rpmd_npt_step()
        if self.ring_polymer is not None:
            return self._rpmd_step()
        if self.barostat is not None:
            return self._npt_step()
        if self.thermostat is not None:
            self.thermostat.apply(self.momenta)   # simulator.py:127-128 on_step_begin
        self._verlet(True)        # integrators.py:70 half_step + :108 main_step (momenta, then positions with the new momenta)
        self._calculate()         # simulator.py:137
        self._verlet(False)       # simulator.py:144 half_step
        if self.thermostat is not None:
            self.thermostat.apply(self.momenta)   # simulator.py:149-150 on_step_end

    def _step_state(self) -> Dict[str, object]:
        """the MD state, the neighbour-list bookkeeping, the hooks' state, the properties and the records held"""
        state = dict(positions=self.positions, momenta=self.momenta, **self._evaluation_state())
        if self._mp is not None:
            state["model_positions"] = self._mp
        if self.thermostat is not None:
            state["thermostat"] = self.thermostat._state()
        if self.virial is not None:
            state.update(cell=self.cell, model_cell=self.model_cell, virial=self.virial)
        if self.barostat is not None:
            state["barostat"] = self.barostat._state()
        if self.properties:
            state["properties"] = self.properties
        if self.record_capacity:
            state["recorder"] = {"counter": self._rec_counter,
                                 "records": {p: v[:self._n_records] for p, v in self._records.items()}}
        elif self.hooks or self.stream is not None:
            state["step_counter"] = self._rec_counter
        if self.stream is not None:
            state["stream"] = self.stream._state()
        accumulators = {str(k): h._state() for k, h in enumerate(self.hooks) if hasattr(h, "_state")}
        if accumulators:
            state["hooks"] = accumulators
        return state

    def run(self, n_steps: int):
        """Advance ``n_steps`` velocity-Verlet steps; returns (energy, forces) buffers of the last step (device).  With a
        recorder, a call that would store more than ``record_capacity`` records since the last ``drain`` is refused before
        anything is launched."""
        if self.record_capacity:
            new = self._records_in(int(n_steps))
            if self._n_records + new > self.record_capacity:
                raise RuntimeError(f"DeviceMD: run({int(n_steps)}) would store {new} records on top of the "
                                   f"{self._n_records} held, more than record_capacity = {self.record_capacity}; "
                                   "call drain() first")
        self._run_steps(int(n_steps))
        if self.record_capacity:
            self._n_records += self._records_in(int(n_steps))
        self.steps_done += int(n_steps)
        self.check_neighbor_list()
        for h in self.hooks:
            if hasattr(h, "_check"):
                h._check()
        return self.energy, self.forces

    def kinetic_energy(self) -> Tensor:
        return 0.5 * (self.momenta ** 2 / self.masses[:, None]).sum()

    def potential_energy(self) -> Tensor:
        """model energy in MD units (base_calculator.py: property_conversion of the energy key)"""
        return self.energy * self.e_conv

    def temperature(self, kB: Optional[float] = None) -> Tensor:
        """Instantaneous temperature of every system in K (system.py:407-421), fp64 on the device; ``kB`` in MD energy per
        kelvin defaults to the thermostat's, else to the reference's MD units."""
        if kB is None:
            kB = self._kB()
        t = self.systems.kinetic_energy_and_temperature(self.momenta, kB)[1]
        if self.ring_polymer is not None:                                  # per bead and system (system.py:407-421)
            t = t.reshape(self.ring_polymer.n_beads, -1)
        return t

    def _kB(self) -> float:
        hook = self.thermostat if self.thermostat is not None else self.barostat
        if hook is not None:
            return hook.kB
        return self.ring_polymer.kB if self.ring_polymer is not None else KB_MD

    # ---- centroid accessors of ring-polymer runs (system.py:484-565), MD units, on the device -----------------------------
    def _need_rp(self) -> RingPolymer:
        if self.ring_polymer is None:
            raise RuntimeError("DeviceMD: centroid quantities need a ring-polymer run (ring_polymer=RingPolymer(...))")
        return self.ring_polymer

    def centroid_positions(self) -> Tensor:
        """bead average of the positions [N, 3] (system.py:484-495)"""
        rp = self._need_rp()
        return self.positions.reshape(rp.n_beads, -1, 3).mean(0)

    def centroid_momenta(self) -> Tensor:
        """bead average of the momenta [N, 3] (system.py:497-508)"""
        rp = self._need_rp()
        return self.momenta.reshape(rp.n_beads, -1, 3).mean(0)

    def centroid_temperature(self, kB: Optional[float] = None) -> Tensor:
        """2 / (3 N_s kB) * 1/2 sum_a |p_c,a|^2 / m_a per system [B] fp64 (system.py:523-555)"""
        self._need_rp()
        pc = self.centroid_momenta().contiguous()
        return self._rp_base.kinetic_energy_and_temperature(pc, self._kB() if kB is None else kB)[1]

    def centroid_potential_energy(self) -> Tensor:
        """bead average of the potential energy [B] in MD units (system.py:557-565)"""
        rp = self._need_rp()
        return self.potential_energy().reshape(rp.n_beads, -1).mean(0)

    def centroid_pressure(self, tensor: bool = False, kinetic_component: bool = False) -> Tensor:
        """system.py:616-650 for a ring-polymer NPT run: -(bead mean of the stress), its trace / 3 ([B]) or the tensor
        ([B, 3, 3]), optionally plus the kinetic part 2 K_c / (3 V_bar) (2 K_c / V_bar for the tensor) with K_c from the
        bead mean of the momenta and V_bar the bead mean of the volume.  The tensor's kinetic part uses the kinetic-energy
        tensor of the centroid momenta (the reference raises there)."""
        rp = self._need_rp()
        if self.virial is None:
            raise RuntimeError("DeviceMD: the centroid pressure needs a ring-polymer NPT run (barostat=PILEBarostat(...))")
        P_ = rp.n_beads
        return self._pressure(-self.stress.reshape(P_, -1, 3, 3).mean(0), self.volume().reshape(P_, -1).mean(0),
                              self._rp_base, self.centroid_momenta().contiguous(), tensor, kinetic_component)

    def state_dict(self) -> Dict[str, object]:
        """Everything a restarted run needs to continue bitwise: the MD state, the neighbour-list bookkeeping and the
        thermostat state (chain velocities / forces, Langevin application counter)."""
        sd = _clone_state(self._step_state())
        sd["steps_done"] = self.steps_done
        if self.record_capacity:
            sd["recorder"]["n_records"] = self._n_records
        return sd

    def load_state_dict(self, state: Dict[str, object]):
        """Copy a ``state_dict`` into the existing buffers (a captured graph stays valid)."""
        if self.record_capacity:
            n = int(state["recorder"]["n_records"])
            if n > self.record_capacity:
                raise ValueError(f"DeviceMD: the state holds {n} records, more than record_capacity = "
                                 f"{self.record_capacity}")
            self._n_records = n
        _load_state(self._step_state(), state)
        self.steps_done = int(state["steps_done"])

    # ---- cell, stress and pressure (system.py:567-614), MD units, per system, fp64 on the device ----------------------------
    def volume(self) -> Tensor:
        """cell volumes [n_sys] (system.py:567-581)"""
        c = self._need_cell()
        return torch.sum(c[:, 0] * torch.cross(c[:, 1], c[:, 2], dim=1), dim=1)

    def _need_cell(self) -> Tensor:
        if self.cell is None:
            raise RuntimeError("DeviceMD: create it with compute_stress=True or a barostat to track the cell and stress")
        return self.cell

    @property
    def stress(self) -> Tensor:
        """stress of the last evaluation [n_sys, 3, 3] in MD units: W / V_model * energy_conversion /
        position_conversion^3 (base_calculator.py:97,218-222)"""
        v_model = self.volume() * self.p_conv ** 3
        return self.virial / v_model[:, None, None] * (self.e_conv / self.p_conv ** 3)

    def pressure(self, tensor: bool = False, kinetic_component: bool = False) -> Tensor:
        """system.py:583-614: -stress ([n_sys, 3, 3]) or its trace / 3 ([n_sys]), optionally with the kinetic part."""
        return self._pressure(-self.stress, self.volume(), self.systems, self.momenta, tensor, kinetic_component)

    @staticmethod
    def _pressure(p: Tensor, vol: Tensor, systems: _Systems, momenta: Tensor, tensor: bool,
                  kinetic_component: bool) -> Tensor:
        """the pressure tensor ``p`` (-stress) or its trace / 3, optionally plus the kinetic part 2 K / V of ``momenta``
        in ``systems`` (2 K / (3 V) for the trace)"""
        if tensor:
            if kinetic_component:
                p = p + 2.0 * systems.kinetic_energy_tensor(momenta) / vol[:, None, None]
            return p
        p = torch.diagonal(p, dim1=1, dim2=2).sum(-1) / 3.0
        if kinetic_component:
            ke = systems.kinetic_energy_and_temperature(momenta, KB_MD)[0]
            p = p + 2.0 * ke / vol / 3.0
        return p
