"""Test infrastructure, not product code: fp64 restatement of the reference's thermostats (md/simulation_hooks/
thermostats.py:149-513, md/utils/thermostat_utils.py:10-60, md/system.py:374-421) and of the NVT loop around them
(md/simulator.py:118-150), pinned to tests/golden/md_thermostats.npz (made by the reference's own classes), plus a numpy
restatement of Philox4x32-10 + Box-Muller that reproduces the noise of ``schnetpack_b200.md.LangevinThermostat``.

Systems are given flat: masses [N], momenta [N, 3], n_atoms [n_sys] (atoms of a system are contiguous).  Like the reference,
the bath temperature and time constant pass through float32 buffers (thermostats.py:55-59, 304, 308) before being used in
fp64; ``schnetpack_b200.md`` keeps them in fp64, a relative difference of ~1e-8 in the parameters.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import nl_oracle as NL
from oracle import spk_oracle as O

YS_WEIGHTS = {                                                         # thermostat_utils.py:18-44
    3: torch.tensor([1.35120719195966, -1.70241438391932, 1.35120719195966], dtype=torch.float64),
    5: torch.tensor([0.41449077179438, 0.41449077179438, -0.65796308717750, 0.41449077179438, 0.41449077179438],
                    dtype=torch.float64),
    7: torch.tensor([0.78451361047756, 0.23557321335936, -1.17767998417887, 1.31518632068390, -1.17767998417887,
                     0.23557321335936, 0.78451361047756], dtype=torch.float64),
}


# ---- Philox4x32-10 (Salmon et al., SC'11; Random123) and Box-Muller ----------------------------------------------------
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(counter, key):
    """counter [n, 4] uint32, key (k0, k1) -> [n, 4] uint32."""
    c = [np.asarray(counter, dtype=np.uint64)[:, i].copy() for i in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
            k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
    return np.stack(c, axis=1).astype(np.uint32)


def philox_bits(seed: int, app: int, n: int):
    """The draw of elements 0..n-1 at application ``app``: counter (element lo, element hi, app lo, app hi), key = seed."""
    e = np.arange(n, dtype=np.uint64)
    ctr = np.stack([e & _M32, e >> np.uint64(32), np.full(n, app & 0xFFFFFFFF, np.uint64),
                    np.full(n, app >> 32, np.uint64)], axis=1)
    return philox4x32_10(ctr, (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))


def box_muller(x0, x1):
    u0 = (x0.astype(np.float64) + 0.5) * 2.0 ** -32
    u1 = (x1.astype(np.float64) + 0.5) * 2.0 ** -32
    r = np.sqrt(-2.0 * np.log(u0))
    return r * np.cos(2.0 * np.pi * u1), r * np.sin(2.0 * np.pi * u1)


def langevin_normals(seed: int, app: int, n_atoms: int):
    """[n_atoms, 3] standard normals of one Langevin application: normals 0, 1, 2 of each atom's draw."""
    x = philox_bits(seed, app, n_atoms)
    z0, z1 = box_muller(x[:, 0], x[:, 1])
    z2, _ = box_muller(x[:, 2], x[:, 3])
    return np.stack([z0, z1, z2], axis=1)


# ---- thermostats ---------------------------------------------------------------------------------------------------------
class _System:
    """The parts of md/system.py the thermostats read, for one replica."""

    def __init__(self, masses, n_atoms):
        self.n_atoms = torch.as_tensor(np.asarray(n_atoms), dtype=torch.long)
        self.index_m = torch.repeat_interleave(torch.arange(len(self.n_atoms)), self.n_atoms)
        self.masses = torch.as_tensor(np.asarray(masses, dtype=np.float64)).reshape(1, -1, 1)

    def sum_atoms(self, x):                                               # system.py:217-231
        return torch.zeros(x.shape[0], len(self.n_atoms), *x.shape[2:], dtype=x.dtype).index_add(1, self.index_m, x)

    def kinetic_energy(self, p):                                          # system.py:374-386
        return 0.5 * self.sum_atoms(torch.sum(p ** 2, dim=2, keepdim=True) / self.masses)

    def temperature(self, p, kB):                                         # system.py:406-421
        return 2.0 / (3.0 * self.n_atoms[None, :, None] * kB) * self.kinetic_energy(p)


class Thermostat:
    def __init__(self, temperature_bath, time_constant, kB, fs):
        self.temperature_bath = torch.tensor(temperature_bath).double()   # thermostats.py:55-59 (float32 buffers)
        self.time_constant = torch.tensor(time_constant * fs).double()
        self._tb32, self._tau32 = torch.tensor(temperature_bath), torch.tensor(time_constant * fs)
        self.kB = kB

    def init(self, masses, n_atoms, time_step):
        self.system = _System(masses, n_atoms)
        self.time_step = time_step
        self._init()

    def _init(self):
        pass

    def apply(self, p):
        """p [N, 3] fp64 tensor -> new momenta"""
        return self._apply(p[None])[0]


class Berendsen(Thermostat):
    def _apply(self, p):                                                  # thermostats.py:172-189
        T = self.system.temperature(p, self.kB)
        scaling = torch.sqrt(1.0 + self.time_step / self.time_constant * (self.temperature_bath / T - 1))
        return scaling[:, self.system.index_m, ...] * p


class Langevin(Thermostat):
    def __init__(self, temperature_bath, time_constant, kB, fs, seed=0):
        super().__init__(temperature_bath, time_constant, kB, fs)
        self.seed = seed
        self.app = 0

    def _init(self):                                                      # thermostats.py:218-242
        gamma = torch.ones(1, dtype=torch.float64) / self.time_constant
        c1 = torch.exp(-0.5 * self.time_step * gamma)
        c2 = torch.sqrt(1 - c1 ** 2)
        self.c1, self.c2 = c1[:, None, None], c2[:, None, None]
        self.thermostat_factor = torch.sqrt(self.system.masses * self.kB * self.temperature_bath)

    def _apply(self, p):                                                  # thermostats.py:244-261
        noise = torch.as_tensor(langevin_normals(self.seed, self.app, p.shape[1]))[None]
        self.app += 1
        return self.c1 * p + self.thermostat_factor * self.c2 * noise


class NHC(Thermostat):
    def __init__(self, temperature_bath, time_constant, kB, fs, chain_length=3, massive=False, multi_step=2,
                 integration_order=3):
        super().__init__(temperature_bath, time_constant, kB, fs)
        self.chain_length, self.massive = chain_length, massive
        self.multi_step, self.integration_order = multi_step, integration_order
        # float32 buffers while _init_thermostat runs; on_simulation_start converts them to fp64 afterwards
        self._freq32 = 1.0 / self._tau32                                  # :304
        self._kbt32 = self._tb32 * kB                                     # :308
        self.kb_temperature = self._kbt32.double()

    def _init(self):                                                      # :323-396
        self.ts = self.time_step * YS_WEIGHTS[self.integration_order] / self.multi_step
        s = self.system
        n_tot = int(s.n_atoms.sum())
        if self.massive:
            shape = (1, n_tot, 3, self.chain_length)
            self.dof = torch.ones((1, n_tot, 3), dtype=torch.float64)
        else:
            shape = (1, len(s.n_atoms), 1, self.chain_length)
            self.dof = (3 * s.n_atoms[None, :, None]).double()
        self.masses = torch.ones(shape, dtype=torch.float64)
        self.masses[..., 0] = self.dof * self._kbt32 / self._freq32 ** 2
        self.masses[..., 1:] = self._kbt32 / self._freq32 ** 2
        self.velocities = torch.zeros(shape, dtype=torch.float64)
        self.forces = torch.zeros(shape, dtype=torch.float64)

    def _propagate(self, ke):                                             # :398-468
        v, f, M, kbt = self.velocities, self.forces, self.masses, self.kb_temperature
        f[..., 0] = (ke - self.dof * kbt) / M[..., 0]
        scaling = 1.0
        for _ in range(self.multi_step):
            for k in range(self.integration_order):
                h = self.ts[k]
                v[..., -1] += 0.25 * f[..., -1] * h
                for c in range(self.chain_length - 2, -1, -1):
                    coeff = torch.exp(-0.125 * h * v[..., c + 1])
                    v[..., c] = v[..., c] * coeff ** 2 + 0.25 * f[..., c] * coeff * h
                scaling *= torch.exp(-0.5 * h * v[..., 0])
                f[..., 0] = (scaling * scaling * ke - self.dof * kbt) / M[..., 0]
                for c in range(self.chain_length - 1):
                    coeff = torch.exp(-0.125 * h * v[..., c + 1])
                    v[..., c] = v[..., c] * coeff ** 2 + 0.25 * f[..., c] * coeff * h
                    f[..., c + 1] = (M[..., c] * v[..., c] ** 2 - kbt) / M[..., c + 1]
                v[..., -1] += 0.25 * f[..., -1] * h
        return scaling

    def _apply(self, p):                                                  # :470-511
        if self.massive:
            ke = p ** 2 / self.system.masses
        else:
            ke = 2.0 * self.system.kinetic_energy(p)
        scaling = self._propagate(ke)
        if not self.massive:
            scaling = scaling[:, self.system.index_m, ...]
        return p * scaling

    def chain_state(self):
        L = self.chain_length
        return (self.velocities.reshape(-1, L).numpy(), self.forces.reshape(-1, L).numpy(),
                self.masses.reshape(-1, L).numpy())


# ---- the NVT loop ----------------------------------------------------------------------------------------------------------
def nvt_trajectory(spec, params, batch, masses, momenta, time_step, n_steps, thermostat, position_conversion=1.0,
                   energy_conversion=1.0):
    """oracle/md_oracle.py's NVE loop with ``thermostat`` applied before the first and after the second half kick
    (simulator.py:127-150).  ``batch`` holds ONE periodic or open system in model units; returns MD-unit positions,
    momenta, energy and forces after ``n_steps``."""
    f_conv = energy_conversion / position_conversion
    cell = np.asarray(batch["_cell"], dtype=np.float64).reshape(3, 3)
    pbc = np.asarray(batch["_pbc"]).reshape(3)
    x = torch.as_tensor(np.asarray(batch["_positions"], dtype=np.float64)) / position_conversion
    p = torch.as_tensor(np.asarray(momenta, dtype=np.float64)).clone()
    m = torch.as_tensor(np.asarray(masses, dtype=np.float64)).reshape(-1, 1)
    thermostat.init(masses, [x.shape[0]], time_step)                      # on_simulation_start

    def calculate(x_md):
        R = (x_md * position_conversion).numpy()
        ii, jj, ss, off = NL.neighbor_list(R, cell, pbc, spec["cutoff"])
        b = dict(batch)
        b.update({"_positions": R, "_idx_i": ii, "_idx_j": jj, "_offsets": off})
        out = O.energy_forces(spec, params, b, dtype=torch.float64)
        return out["energy"] * energy_conversion, out["forces"] * f_conv

    e, f = calculate(x)
    for _ in range(n_steps):
        p = thermostat.apply(p)                                           # on_step_begin
        p = p + 0.5 * f * time_step
        x = x + time_step * p / m
        e, f = calculate(x)
        p = p + 0.5 * f * time_step
        p = thermostat.apply(p)                                           # on_step_end
    return x.numpy(), p.numpy(), e.numpy(), f.numpy()
