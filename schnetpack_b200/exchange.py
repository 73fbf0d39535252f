"""Temperature replica exchange (parallel tempering, REMD) inside the captured step of ``DeviceMD`` (DESIGN.md section 25).

K copies of every molecule run at a ladder of temperatures T_0 < T_1 < ... < T_K-1 as K G systems of one batch, rung-major:
system k G + g is rung k of group g, the layout ``md.replicate_batch(static, K, G)`` produces.  A per-system
``LangevinThermostat`` or ``NHCThermostat`` holds every system at its rung's temperature, and ``ReplicaExchange`` swaps
configurations between neighbouring rungs with a Metropolis test, so a walker that is stuck in a basin at T_0 can leave it
through the hotter rungs.

::

    batch = md.replicate_batch(static, K, G)                       # K copies of G molecules
    temps = [300.0 * 1.15 ** k for k in range(K) for _ in range(G)]
    remd = ReplicaExchange(n_temperatures=K, every_n_steps=100, seed=1)
    run = DeviceMD(model, batch, masses.repeat(K), dt, cutoff, capacity, thermostat=LangevinThermostat(temps, 100.0),
                   initializer=MaxwellBoltzmannInit(temps), hooks=[RemoveCOMMotion(10, False), remd])
    run.run(100_000)
    remd.acceptance()                                              # [G, K - 1]
    remd.walkers()                                                 # [K, G]: which initial system sits where

Every other hook and the recorder then describe a fixed temperature: rung k's series are the rung-k ensemble.  The
recorded series ``"walker"`` [n_records, K, G] tells which walker each rung held, to follow one walker's trajectory.
"""
from __future__ import annotations

import ctypes
from typing import Dict

import torch

from . import _lib, ops
from . import properties as P
from .md import LangevinThermostat, NHCThermostat, _check_every

Tensor = torch.Tensor

__all__ = ["ReplicaExchange"]


class ReplicaExchange:
    """``DeviceMD`` hook that tries temperature swaps between neighbouring rungs on the steps s % every_n_steps == 0 of the
    device step counter (the first step included), at on_step_finalize in the listed order of ``hooks``.

    Attempt n (a device counter) tries the pairs (k, k + 1) with k = n (mod 2) of every group and accepts one iff
    Delta >= 0 or u < exp(Delta), Delta = (1 / (kB T_k) - 1 / (kB T_k+1)) (U_k - U_k+1) in fp64, U the potential energy in
    MD units from the step's evaluation.  u comes from Philox4x32-10 keyed by ``seed`` with the counter
    (g (K - 1) + k, 2^63 + n), which no thermostat or initializer reaches.  An accepted pair swaps positions, momenta
    (times sqrt(T_new / T_old)), forces, energies and every required property of its two systems; the thermostat state
    stays with the temperature.  The temperatures are the thermostat's per-system ``temperature_bath``.

    ``DeviceMD`` refuses the hook without a per-system Langevin or NHC thermostat, for n_sys not a multiple of K, for a
    ladder that does not increase strictly with k in every group, for groups whose systems differ in atoms (count,
    atomic numbers in order, masses) or in ``_cell`` / ``_pbc``, and next to a barostat, ``compute_stress``, ring
    polymers, a model ensemble, ``structure.MeanSquaredDisplacement`` or a ``spectra.SpectrumStream``."""

    def __init__(self, n_temperatures: int, every_n_steps: int, seed: int = 0):
        if int(n_temperatures) != n_temperatures or int(n_temperatures) < 2:
            raise ValueError(f"ReplicaExchange: n_temperatures must be an integer >= 2, got {n_temperatures}")
        self.n_temperatures = int(n_temperatures)
        self.every_n_steps = _check_every(every_n_steps, "ReplicaExchange")
        self.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        self._md = None

    # ---- set-up by DeviceMD ------------------------------------------------------------------------------------------
    def _refuse_combinations(self, md):
        from .structure import MeanSquaredDisplacement

        if md.ring_polymer is not None:
            raise NotImplementedError("ReplicaExchange: ring-polymer MD (PIMD-REMD) is not supported")
        if md.barostat is not None or md.virial is not None:
            raise NotImplementedError("ReplicaExchange: constant pressure and compute_stress (NPT-REMD, which needs the PV "
                                      "term and swapped cells and virials) are not supported")
        if md.ensemble is not None:
            raise NotImplementedError("ReplicaExchange: model ensembles are not supported")
        if md.stream is not None:
            raise ValueError("ReplicaExchange: a spectra.SpectrumStream cannot run next to the exchange; time "
                             "correlations across swaps have no meaning")
        for h in md.hooks:
            if isinstance(h, MeanSquaredDisplacement):
                raise ValueError("ReplicaExchange: MeanSquaredDisplacement cannot run next to the exchange; "
                                 "displacements across swaps have no meaning")
            if isinstance(h, ReplicaExchange) and h is not self:
                raise ValueError("ReplicaExchange: one exchange hook per run")
        th = md.thermostat
        if not isinstance(th, (LangevinThermostat, NHCThermostat)) or not th.per_system:
            raise ValueError("ReplicaExchange: needs a LangevinThermostat or NHCThermostat with one temperature_bath per "
                             f"system (the ladder), got {type(th).__name__ if th is not None else None}")

    def _check_groups(self, md, K: int, G: int):
        """the ladder increases with k and the systems of every group are copies of one molecule"""
        s = md.systems
        T = md.thermostat.temperatures.cpu().reshape(K, G)
        if not bool((T[1:] > T[:-1]).all()):
            raise ValueError("ReplicaExchange: the bath temperature must increase strictly with the rung k in every "
                             "group (system k G + g is rung k of group g)")
        counts = (s.sys_ptr[1:] - s.sys_ptr[:-1]).cpu().reshape(K, G)
        if not bool((counts == counts[0]).all()):
            raise ValueError("ReplicaExchange: the systems of a group differ in their atom counts")
        for name, v in (("atomic numbers", md.static[P.Z]), ("masses", md.masses)):
            rows = v.reshape(K, -1)
            if not bool((rows == rows[0]).all()):
                raise ValueError(f"ReplicaExchange: the systems of a group differ in their {name}")
        for key, width in ((P.cell, 9), (P.pbc, 3)):
            v = md.static.get(key)
            if v is None:
                continue
            rows = v.reshape(-1, width)
            if rows.shape[0] == s.n_sys:
                rows = rows.reshape(K, G, width)
                if not bool((rows == rows[0]).all()):
                    raise ValueError(f"ReplicaExchange: the systems of a group differ in '{key}'")

    def _buffer_table(self, md):
        """the rows an accepted swap exchanges besides the momenta: positions (and their model-unit copy), forces, energy
        and every required property, per atom or per system"""
        s = md.systems
        bufs = [(md.positions, True, 3), (md.forces, True, 3), (md.energy, False, md.energy.numel() // s.n_sys)]
        if md._mp is not None:
            bufs.append((md._mp, True, 3))
        for name, v in md.properties.items():
            rows = v.shape[1]
            if rows not in (s.n_sys, s.n_atoms):
                raise ValueError(f"ReplicaExchange: property '{name}' has {rows} rows, neither one per system nor one "
                                 "per atom")
            bufs.append((v, rows != s.n_sys, v.numel() // rows))     # one row per system where both counts agree
        limit = _lib.CONSTANTS["SPK_REMD_MAX_BUFFERS"]
        if len(bufs) > limit:
            raise ValueError(f"ReplicaExchange: {len(bufs)} buffers to swap, at most {limit}")
        table = _lib.STRUCTS["spk_remd_buffers_t"]()
        table.n_buffers = len(bufs)
        for i, (t, per_atom, width) in enumerate(bufs):
            if t.dtype != torch.float32 or not t.is_contiguous():
                raise TypeError("ReplicaExchange: every swapped buffer must be a contiguous float32 tensor")
            table.per_atom[i], table.width[i], table.data[i] = int(per_atom), int(width), t.data_ptr()
        return table

    def _bind(self, md):
        if self._md is not None:
            raise ValueError("ReplicaExchange: this hook already belongs to a DeviceMD")
        self._refuse_combinations(md)
        K, n_sys = self.n_temperatures, md.systems.n_sys
        if n_sys % K:
            raise ValueError(f"ReplicaExchange: {n_sys} systems are not K G for K = {K} rungs")
        G = n_sys // K
        self._check_groups(md, K, G)
        self.n_groups = G
        self._table = self._buffer_table(md)
        dev = md.positions.device
        self._walker = torch.arange(n_sys, dtype=torch.int32, device=dev)
        self._attempted = torch.zeros(G, K - 1, dtype=torch.int64, device=dev)
        self._accepted = torch.zeros(G, K - 1, dtype=torch.int64, device=dev)
        self._attempt = torch.zeros(1, dtype=torch.int64, device=dev)
        self._decision = torch.zeros(G, K - 1, dtype=torch.uint8, device=dev)
        if md.record_capacity:
            if "walker" in md.required_properties:
                raise ValueError("ReplicaExchange: records the series 'walker'; a required property of that name would "
                                 "share it")
            md._records["walker"] = torch.zeros(md.record_capacity, K, G, dtype=torch.int32, device=dev)
            md._hook_series["walker"] = self._walker
        self._md = md

    def apply(self, md):
        s, th = md.systems, md.thermostat
        _lib.call("spk_remd_exchange", ops._p(md.energy), md.e_conv, ops._p(th.temperatures), th.kB, ops._p(s.idx_m),
                  ops._p(s.sys_ptr), s.n_atoms, self.n_groups, self.n_temperatures, self.seed, ops._p(md._rec_counter),
                  self.every_n_steps, ops._p(self._attempt), ops._p(self._walker), ops._p(self._attempted),
                  ops._p(self._accepted), ops._p(self._decision), ops._p(md.momenta), ctypes.byref(self._table),
                  ops._stream())

    def _state(self) -> Dict[str, Tensor]:
        return {"walker": self._walker, "attempted": self._attempted, "accepted": self._accepted,
                "attempt": self._attempt}

    # ---- results -----------------------------------------------------------------------------------------------------
    def _need_md(self):
        if self._md is None:
            raise ValueError("ReplicaExchange: the hook is not attached to a run; pass it in DeviceMD(..., hooks=...)")
        return self._md

    def reset(self):
        """zero the attempt and acceptance counts (walkers and the attempt counter keep going)"""
        self._need_md()
        self._attempted.zero_()
        self._accepted.zero_()

    @property
    def attempts(self) -> int:
        """exchange attempts so far (one host read)"""
        self._need_md()
        return int(self._attempt.item())

    def acceptance(self) -> Tensor:
        """accepted / attempted swaps of every neighbouring pair (k, k + 1), [G, K - 1] fp64 on the host (NaN for a pair
        not tried yet)"""
        self._need_md()
        return self._accepted.cpu().double() / self._attempted.cpu().double()

    def walkers(self) -> Tensor:
        """[K, G] int32 on the host: the initial system k' G + g now held by rung k of group g"""
        self._need_md()
        return self._walker.cpu().reshape(self.n_temperatures, self.n_groups)
