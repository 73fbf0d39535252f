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
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, Optional

import torch

from . import _lib, ops
from . import properties as P
from .neighbors import CellListNeighborList

__all__ = ["DeviceMD", "BerendsenThermostat", "LangevinThermostat", "NHCThermostat", "KB_MD", "FS_MD"]

Tensor = torch.Tensor

# ---- MD units of the reference (units.py:10-40): energy kJ/mol, length nm, mass Da; time = nm sqrt(Da / (kJ/mol)).
# Restated from the CODATA-2014 constants that ASE's units module is built on (Boltzmann constant, elementary charge,
# Avogadro constant, atomic mass unit), in ASE's frame (eV, Angstrom, amu): kJ/mol = 1e3 / (e N_A) eV, nm = 10 Angstrom,
# fs = 1e-15 s with s = 1e10 sqrt(e / amu).
_CODATA_K, _CODATA_E, _CODATA_NA, _CODATA_AMU = 1.38064852e-23, 1.6021766208e-19, 6.022140857e23, 1.660539040e-27
_MD_ENERGY = 1e3 / _CODATA_E / _CODATA_NA                      # kJ/mol in eV
_MD_TIME = 10.0 * math.sqrt(1.0 / _MD_ENERGY)                 # units.py:37, in ASE time units
KB_MD = (_CODATA_K / _CODATA_E) / _MD_ENERGY                   # units.py:79: ~0.0083144598 kJ/mol/K
FS_MD = 1e-15 * 1e10 * math.sqrt(_CODATA_E / _CODATA_AMU) / _MD_TIME   # units.py:59: ~1.0e-3


class _Systems:
    """The systems of a collated batch as the thermostat kernels address them: per-atom masses and system index, the
    first atom of every system and the fp64 workspace of the per-system sums (allocated once, outside any capture)."""

    def __init__(self, masses: Tensor, idx_m: Tensor, n_sys: int):
        self.masses = masses
        self.idx_m = idx_m
        self.n_sys = int(n_sys)
        self.n_atoms = int(masses.shape[0])
        self.sys_ptr = ops.segment_ptr(idx_m, self.n_sys)
        self.n_atoms_sys = (self.sys_ptr[1:] - self.sys_ptr[:-1]).to(torch.float64)
        nbytes = int(_lib.lib().spk_md_thermostat_workspace_bytes(self.n_atoms, self.n_sys))
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=masses.device)

    def call(self, name: str, momenta: Tensor, *args):
        _lib.call(name, ops._p(momenta), ops._p(self.masses), ops._p(self.idx_m), ops._p(self.sys_ptr), self.n_atoms,
                  self.n_sys, *args, ops._p(self.ws), self.ws.numel(), ops._stream())

    def kinetic_energy_and_temperature(self, momenta: Tensor, kB: float):
        dev = momenta.device
        ke = torch.empty(self.n_sys, dtype=torch.float64, device=dev)
        temp = torch.empty(self.n_sys, dtype=torch.float64, device=dev)
        self.call("spk_md_kinetic_energy", momenta, float(kB), ops._p(ke), ops._p(temp))
        return ke, temp


class _Thermostat:
    """Common part of the device thermostats (ThermostatHook, thermostats.py:41-146): bath temperature in K, time constant
    in fs.  ``kB`` (MD energy per kelvin) and ``fs`` (one femtosecond in MD time) define the caller's MD units; the
    defaults are the reference's (kJ/mol, nm, Da).  ``bind`` sizes the state for a batch, ``apply`` updates the momenta in
    place (enqueue-only, capturable)."""

    def __init__(self, temperature_bath: float, time_constant: float, kB: float = KB_MD, fs: float = FS_MD):
        self.temperature_bath = float(temperature_bath)
        self.time_constant = float(time_constant) * float(fs)          # thermostats.py:57-59
        self.kB = float(kB)
        self.systems: Optional[_Systems] = None
        self.time_step: Optional[float] = None

    def bind(self, systems: _Systems, time_step: float):
        self.systems = systems
        self.time_step = float(time_step)
        self._init_state()

    def _init_state(self):
        pass

    def apply(self, momenta: Tensor):
        raise NotImplementedError

    def _state(self) -> Dict[str, Tensor]:
        return {}

    def state_dict(self) -> Dict[str, Tensor]:
        return {k: v.clone() for k, v in self._state().items()}

    def load_state_dict(self, state: Dict[str, Tensor]):
        for k, v in self._state().items():
            v.copy_(state[k])


class BerendsenThermostat(_Thermostat):
    """Berendsen rescaling (thermostats.py:149-189): p *= sqrt(1 + dt / tau (T_bath / T - 1)) per system.  A system whose
    kinetic energy is zero is left as it is (the reference would divide by T = 0)."""

    def apply(self, momenta: Tensor):
        self.systems.call("spk_md_berendsen", momenta, self.kB, self.time_step / self.time_constant,
                          self.temperature_bath)


class LangevinThermostat(_Thermostat):
    """Langevin thermostat (thermostats.py:192-261): p = c1 p + c2 sqrt(m kB T_bath) xi with c1 = exp(-dt / (2 tau)),
    c2 = sqrt(1 - c1^2).  xi comes from Philox4x32-10 keyed by ``seed`` with the counter (atom, application); the
    application index lives on the device and advances with every application, also inside a replayed graph."""

    def __init__(self, temperature_bath: float, time_constant: float, seed: int = 0, kB: float = KB_MD,
                 fs: float = FS_MD):
        super().__init__(temperature_bath, time_constant, kB=kB, fs=fs)
        self.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        self.counter: Optional[Tensor] = None

    def _init_state(self):
        gamma = 1.0 / self.time_constant                                 # :227-230
        self.c1 = math.exp(-0.5 * self.time_step * gamma)                 # :233
        self.c2 = math.sqrt(1.0 - self.c1 ** 2)                           # :234
        # [0] = application index, [1] = the kernel's internal ticket (zero between calls)
        self.counter = torch.zeros(2, dtype=torch.int64, device=self.systems.masses.device)

    def apply(self, momenta: Tensor):
        s = self.systems
        _lib.call("spk_md_langevin", ops._p(momenta), ops._p(s.masses), s.n_atoms, self.c1, self.c2,
                  self.kB * self.temperature_bath, self.seed, ops._p(self.counter), ops._stream())

    def _state(self):
        return {"counter": self.counter}


class NHCThermostat(_Thermostat):
    """Nose-Hoover chain thermostat (thermostats.py:264-513) with the reference's keywords and defaults: one chain per
    system, or per degree of freedom with ``massive``; ``multi_step`` sub-steps of a Yoshida-Suzuki scheme of order
    ``integration_order`` (3, 5 or 7).  The chain state is fp64 on the device."""

    YS_WEIGHTS = {                                                       # md/utils/thermostat_utils.py:18-44
        3: (1.35120719195966, -1.70241438391932, 1.35120719195966),
        5: (0.41449077179438, 0.41449077179438, -0.65796308717750, 0.41449077179438, 0.41449077179438),
        7: (0.78451361047756, 0.23557321335936, -1.17767998417887, 1.31518632068390, -1.17767998417887,
            0.23557321335936, 0.78451361047756),
    }

    def __init__(self, temperature_bath: float, time_constant: float, chain_length: int = 3, massive: bool = False,
                 multi_step: int = 2, integration_order: int = 3, kB: float = KB_MD, fs: float = FS_MD):
        super().__init__(temperature_bath, time_constant, kB=kB, fs=fs)
        if integration_order not in self.YS_WEIGHTS:
            raise ValueError(f"Order {integration_order:d} not supported for YS integration weights")
        if int(chain_length) < 1 or int(multi_step) < 1:
            raise ValueError("chain_length and multi_step must be >= 1")
        self.chain_length = int(chain_length)
        self.massive = bool(massive)
        self.multi_step = int(multi_step)
        self.integration_order = int(integration_order)
        self.velocities = self.forces = self.masses = None

    def _init_state(self):
        s = self.systems
        dev = s.masses.device
        kbt = self.temperature_bath * self.kB                             # :308
        freq2 = (1.0 / self.time_constant) ** 2                          # :304
        if self.massive:                                                  # :348-359
            dof = torch.ones(3 * s.n_atoms, dtype=torch.float64, device=dev)
        else:
            dof = 3.0 * s.n_atoms_sys
        L = self.chain_length
        self.masses = torch.full((dof.shape[0], L), kbt / freq2, dtype=torch.float64, device=dev)     # :387-396
        self.masses[:, 0] = dof * kbt / freq2
        self.velocities = torch.zeros_like(self.masses)
        self.forces = torch.zeros_like(self.masses)
        w = self.YS_WEIGHTS[self.integration_order]
        steps = [self.time_step * wk / self.multi_step for wk in w] + [0.0] * (7 - len(w))   # :339-341
        self.params = _lib.NHCParams(L, self.multi_step, self.integration_order, int(self.massive), kbt,
                                     (ctypes.c_double * 7)(*steps))

    def apply(self, momenta: Tensor):
        self.systems.call("spk_md_nhc", momenta, ctypes.byref(self.params), ops._p(self.velocities),
                          ops._p(self.forces), ops._p(self.masses))

    def _state(self):
        return {"velocities": self.velocities, "forces": self.forces}


class DeviceMD:
    def __init__(self, model: torch.nn.Module, batch: Dict[str, Tensor], masses: Tensor, time_step: float, cutoff: float,
                 capacity: int, momenta: Optional[Tensor] = None, use_graph: bool = True,
                 position_conversion: float = 1.0, energy_conversion: float = 1.0,
                 thermostat: Optional[_Thermostat] = None):
        """``batch[_positions]`` (and ``_cell``) are in MODEL units as everywhere in this package; ``self.positions`` is the
        MD-unit state (= model positions / position_conversion).  ``thermostat`` (None = NVE) is bound to the systems of
        the batch and applied around every step."""
        dev = batch[P.R].device
        if dev.type != "cuda":
            raise ValueError("DeviceMD needs a CUDA batch (no CPU fallback)")
        self.model = model
        self.dt = float(time_step)
        self.p_conv = float(position_conversion)
        self.e_conv = float(energy_conversion)
        self.f_conv = self.e_conv / self.p_conv                                   # base_calculator.py:96
        self.static = {k: v.detach().clone() for k, v in batch.items() if k not in (P.idx_i, P.idx_j, P.offsets)}
        self.model_positions = self.static[P.R]                                   # what the model reads
        self.positions = self.model_positions if self.p_conv == 1.0 else self.model_positions / self.p_conv
        self.masses = masses.to(dev, torch.float32).reshape(-1).contiguous().clone()
        self.momenta = torch.zeros_like(self.positions) if momenta is None else momenta.to(dev, torch.float32).clone()
        self.nl = CellListNeighborList(cutoff, capacity=int(capacity), pad=True)
        self.use_graph = use_graph
        self.energy: Optional[Tensor] = None
        self.forces: Optional[Tensor] = None
        self.n_pairs: Optional[Tensor] = None
        # sticky bookkeeping of the fixed-capacity neighbour list, updated INSIDE the captured step: [0] = largest pair
        # count seen so far, [1] = 1 if any step overflowed ``capacity`` (its list was then truncated)
        self.nl_watch = torch.zeros(2, dtype=torch.int64, device=dev)
        self._graph = None
        self._chain_ws = ops.ChainWorkspace()      # dependency counters of the persistent per-atom stages, owned here
        self.steps_done = 0
        self._systems: Optional[_Systems] = None
        self.thermostat = thermostat
        if thermostat is not None:
            thermostat.bind(self.systems, self.dt)                                # on_simulation_start
        self._calculate()                       # forces at t = 0 (simulator.py:118)

    @property
    def systems(self) -> _Systems:
        if self._systems is None:
            n = self.masses.shape[0]
            idx_m = self.static.get(P.idx_m)
            if idx_m is None:
                idx_m = torch.zeros(n, dtype=torch.int64, device=self.masses.device)
            n_sys = self.static[P.n_atoms].shape[0] if P.n_atoms in self.static else 1
            self._systems = _Systems(self.masses, idx_m.to(torch.int64).contiguous(), n_sys)
        return self._systems

    # ---- one force evaluation on the current positions (calculator.calculate) ---------------------------------------------
    def _calculate(self):
        ops._GRAPH_CACHE.clear()
        x = {k: (v.detach() if v.is_floating_point() else v) for k, v in self.static.items()}
        x = self.nl(x)
        out = self.model(x)
        e, f = out["energy"].detach(), out["forces"].detach()
        if self.energy is None:
            self.energy, self.forces, self.n_pairs = e.clone(), f.clone(), x["_n_pairs"].clone()
        else:
            self.energy.copy_(e)
            self.forces.copy_(f)
            self.n_pairs.copy_(x["_n_pairs"])
        torch.maximum(self.nl_watch, x["_n_pairs"], out=self.nl_watch)

    def _verlet(self, drift: bool):
        n = self.positions.shape[0]
        mp = self.model_positions if self.model_positions is not self.positions else None
        _lib.call("spk_md_velocity_verlet", ops._p(self.momenta), ops._p(self.positions), ops._p(mp), ops._p(self.forces),
                  ops._p(self.masses), n, self.dt, self.f_conv, self.p_conv, 1 if drift else 0, ops._stream())

    def _step(self):
        if self.thermostat is not None:
            self.thermostat.apply(self.momenta)   # simulator.py:127-128 on_step_begin
        self._verlet(True)        # integrators.py:70 half_step + :108 main_step (momenta, then positions with the new momenta)
        self._calculate()         # simulator.py:137
        self._verlet(False)       # simulator.py:144 half_step
        if self.thermostat is not None:
            self.thermostat.apply(self.momenta)   # simulator.py:149-150 on_step_end

    def _capture(self):
        dev = self.positions.device
        # capture works on copies of the state so that warm-up iterations do not advance the trajectory
        state = [self.positions, self.momenta, self.forces, self.energy]
        if self.model_positions is not self.positions:
            state.append(self.model_positions)
        if self.thermostat is not None:
            state.extend(self.thermostat._state().values())
        saved = [t.clone() for t in state]
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with self._chain_ws:
            with torch.cuda.stream(side):
                self._step()
            torch.cuda.current_stream(dev).wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                self._step()
        for dst, src in zip(state, saved):
            dst.copy_(src)
        self._graph = graph

    def run(self, n_steps: int):
        """Advance ``n_steps`` velocity-Verlet steps; returns (energy, forces) buffers of the last step (device)."""
        if self.use_graph and self._graph is None:
            self._capture()
        for _ in range(int(n_steps)):
            if self.use_graph:
                self._graph.replay()
            else:
                self._step()
        self.steps_done += int(n_steps)
        self.check_neighbor_list()
        return self.energy, self.forces

    def check_neighbor_list(self):
        """One host read per ``run``: raise if ANY step since the start overflowed the list capacity (the search then
        dropped pairs and the trajectory is wrong from that step on).  ``peak_pairs`` tells how much head-room is left."""
        peak, over = (int(v) for v in self.nl_watch.tolist())
        self.peak_pairs = peak
        if over:
            raise RuntimeError(
                f"DeviceMD: the neighbour list overflowed its capacity of {self.nl.capacity} pairs during the run (peak "
                f"{peak}); the trajectory is invalid from that step on -- re-create DeviceMD with a larger capacity")

    def kinetic_energy(self) -> Tensor:
        return 0.5 * (self.momenta ** 2 / self.masses[:, None]).sum()

    def potential_energy(self) -> Tensor:
        """model energy in MD units (base_calculator.py: property_conversion of the energy key)"""
        return self.energy * self.e_conv

    def temperature(self, kB: Optional[float] = None) -> Tensor:
        """Instantaneous temperature of every system in K (system.py:407-421), fp64 on the device; ``kB`` in MD energy per
        kelvin defaults to the thermostat's, else to the reference's MD units."""
        if kB is None:
            kB = self.thermostat.kB if self.thermostat is not None else KB_MD
        return self.systems.kinetic_energy_and_temperature(self.momenta, kB)[1]

    def state_dict(self) -> Dict[str, object]:
        """Everything a restarted run needs to continue bitwise: the MD state, the neighbour-list bookkeeping and the
        thermostat state (chain velocities / forces, Langevin application counter)."""
        sd = {"positions": self.positions.clone(), "momenta": self.momenta.clone(), "forces": self.forces.clone(),
              "energy": self.energy.clone(), "n_pairs": self.n_pairs.clone(), "nl_watch": self.nl_watch.clone(),
              "steps_done": self.steps_done}
        if self.model_positions is not self.positions:
            sd["model_positions"] = self.model_positions.clone()
        if self.thermostat is not None:
            sd["thermostat"] = self.thermostat.state_dict()
        return sd

    def load_state_dict(self, state: Dict[str, object]):
        """Copy a ``state_dict`` into the existing buffers (a captured graph stays valid)."""
        for k in ("positions", "momenta", "forces", "energy", "n_pairs", "nl_watch"):
            getattr(self, k).copy_(state[k])
        if self.model_positions is not self.positions:
            self.model_positions.copy_(state["model_positions"])
        if self.thermostat is not None:
            self.thermostat.load_state_dict(state["thermostat"])
        self.steps_done = int(state["steps_done"])
