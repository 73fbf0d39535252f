"""Test infrastructure, not product code: fp64 restatement of the reference's Nose-Hoover-chain barostats
(md/simulation_hooks/barostats.py:162-927, md/utils/thermostat_utils.py:181-201, md/system.py:374-614) and of the NPT loop
around them (md/integrators.py:232-263, md/simulator.py:118-150), pinned to tests/golden/md_barostats.npz (made by the
reference's own classes).

Systems are given flat: masses [N], positions / momenta / forces [N, 3], cells and stress [n_sys, 3, 3], n_atoms [n_sys]
(atoms of a system are contiguous).  As in the reference, the bath temperature, time constants, frequencies and target
pressure pass through float32 buffers (barostats.py:51-57,209-227) before being used in fp64.
"""
from __future__ import annotations

import numpy as np
import torch

from nvt_oracle import YS_WEIGHTS
from oracle import nl_oracle as NL
from oracle import spk_oracle as O


def sinh_div(x):
    """StableSinhDiv.f as written: series for x < eps (not |x|), with x where x^2 is meant in its third term"""
    e0 = 1.0
    e2 = e0 / 6.0
    e4 = e2 / 20.0
    e6 = e4 / 42.0
    e8 = e6 / 72.0
    x2 = x * x
    return torch.where(x < 1e-4, (((e8 * x2 + e6) * x2 + e4) * x + e2) * x2 + e0, torch.sinh(x) / x)


def _chain(v, f, M, ke, dof, kbt, ts, multi_step, order):
    """barostats.py:408-481 / thermostats.py:398-468 for a stack of chains [n, L]; returns the momentum scaling [n]"""
    L = v.shape[1]
    f[:, 0] = (ke - dof * kbt) / M[:, 0]
    scaling = torch.ones_like(ke)
    for _ in range(multi_step):
        for k in range(order):
            h = ts[k]
            v[:, -1] += 0.25 * f[:, -1] * h
            for c in range(L - 2, -1, -1):
                coeff = torch.exp(-0.125 * h * v[:, c + 1])
                v[:, c] = v[:, c] * coeff ** 2 + 0.25 * f[:, c] * coeff * h
            scaling = scaling * torch.exp(-0.5 * h * v[:, 0])
            f[:, 0] = (ke * scaling ** 2 - dof * kbt) / M[:, 0]
            for c in range(L - 1):
                coeff = torch.exp(-0.125 * h * v[:, c + 1])
                v[:, c] = v[:, c] * coeff ** 2 + 0.25 * f[:, c] * coeff * h
                f[:, c + 1] = (M[:, c] * v[:, c] ** 2 - kbt) / M[:, c + 1]
            v[:, -1] += 0.25 * f[:, -1] * h
    return scaling


def volume(cells):
    """system.py:567-581"""
    return torch.sum(cells[:, 0] * torch.cross(cells[:, 1], cells[:, 2], dim=1), dim=1)


class NHCBarostat:
    def __init__(self, target_pressure, temperature_bath, time_constant, kB, fs, bar, time_constant_cell=None,
                 time_constant_barostat=None, chain_length=4, multi_step=4, integration_order=7, massive=False,
                 anisotropic=False):
        self.P0 = torch.tensor(target_pressure * bar).double()                    # float32 buffers, :51-57
        tau32 = torch.tensor(time_constant * fs)
        self.freq = 1.0 / tau32                                                     # :209
        self.cell_freq = self.freq if time_constant_cell is None else torch.tensor(1.0 / (time_constant_cell * fs))
        self.baro_freq = (self.freq if time_constant_barostat is None
                          else torch.tensor(1.0 / (time_constant_barostat * fs)))
        self.kbt32 = torch.tensor(temperature_bath) * kB                           # :227
        self.kbt = self.kbt32.double()
        self.L, self.multi_step, self.order = chain_length, multi_step, integration_order
        self.massive, self.anisotropic = massive, anisotropic

    def init(self, masses, n_atoms, time_step):
        """on_simulation_start (:263-383, :760-796)"""
        self.dt = time_step
        self.ts = time_step * YS_WEIGHTS[self.order] / self.multi_step
        n = torch.as_tensor(np.asarray(n_atoms), dtype=torch.long)
        self.n_sys = len(n)
        self.index_m = torch.repeat_interleave(torch.arange(self.n_sys), n)
        self.m = torch.as_tensor(np.asarray(masses, dtype=np.float64)).reshape(-1, 1)
        self.dof = 3.0 * n.double()
        self.b_m = (self.dof + 3) * self.kbt32 / self.baro_freq ** 2
        if self.anisotropic:
            self.b_m = self.b_m / 3.0
            self.b_v = torch.zeros(self.n_sys, 3, 3, dtype=torch.float64)
        else:
            self.b_v = torch.zeros(self.n_sys, dtype=torch.float64)
        self.b_f = torch.zeros_like(self.b_v)
        dof_p = torch.ones(3 * int(n.sum()), dtype=torch.float64) if self.massive else self.dof
        self.t_m = torch.zeros(dof_p.shape[0], self.L, dtype=torch.float64)
        self.t_m[:, 0] = dof_p * self.kbt32 / self.freq ** 2
        self.t_m[:, 1:] = self.kbt32 / self.freq ** 2
        self.dof_p = dof_p
        self.dof_cell = 6.0 if self.anisotropic else 1.0
        self.c_m = torch.zeros(self.n_sys, self.L, dtype=torch.float64)
        self.c_m[:, 0] = torch.tensor(self.dof_cell, dtype=torch.float64) * self.kbt32 / self.cell_freq ** 2
        self.c_m[:, 1:] = self.kbt32 / self.cell_freq ** 2
        self.t_v, self.t_f = torch.zeros_like(self.t_m), torch.zeros_like(self.t_m)
        self.c_v, self.c_f = torch.zeros_like(self.c_m), torch.zeros_like(self.c_m)

    def _sum(self, x):
        return torch.zeros(self.n_sys, *x.shape[1:], dtype=x.dtype).index_add(0, self.index_m, x)

    def ke2(self, p):                                                               # 2 * system.py:374-386
        return 2.0 * (0.5 * self._sum(torch.sum(p ** 2, dim=1, keepdim=True) / self.m)[:, 0])

    def ke_tensor(self, p):                                                         # system.py:389-404
        return 0.5 * self._sum(p[:, :, None] * p[:, None, :] / self.m[:, :, None])

    def thermostat(self, p):
        """_update_thermostat (:408-481)"""
        ke_p = (p ** 2 / self.m).reshape(-1) if self.massive else self.ke2(p)
        ke_c = self.b_m * (torch.sum(self.b_v ** 2, dim=(1, 2)) if self.anisotropic else self.b_v ** 2)
        sp = _chain(self.t_v, self.t_f, self.t_m, ke_p, self.dof_p, self.kbt, self.ts, self.multi_step, self.order)
        sc = _chain(self.c_v, self.c_f, self.c_m, ke_c, self.dof_cell, self.kbt, self.ts, self.multi_step, self.order)
        p = p * (sp.reshape(-1, 3) if self.massive else sp[self.index_m, None])
        self.b_v = self.b_v * (sc[:, None, None] if self.anisotropic else sc)
        return p

    def kick(self, p, cells, stress):
        """_update_barostat (:604-631, :822-842)"""
        V = volume(cells)
        ke2 = self.ke2(p)
        if self.anisotropic:
            pt = -stress + 2 * self.ke_tensor(p) / V[:, None, None]
            eye = torch.eye(3, dtype=torch.float64)[None]
            self.b_f = (V[:, None, None] * (pt - eye * self.P0) + (ke2 / self.dof)[:, None, None] * eye) / \
                self.b_m[:, None, None]
        else:
            P = torch.einsum("bii->b", -stress) / 3.0
            self.b_f = ((1.0 + 3.0 / self.dof) * ke2 + 3.0 * V * (P - self.P0)) / self.b_m
        self.b_v = self.b_v + 0.5 * self.dt * self.b_f

    def _operators(self, main):
        dt = self.dt
        if not self.anisotropic:
            if main:
                x = dt * self.b_v
                a = torch.exp(0.5 * x)
                b = a * sinh_div(0.5 * x)
            else:
                x = 0.25 * dt * self.b_v * (1.0 + 3.0 / self.dof)
                a = torch.exp(-x)
                b = a * sinh_div(x)
            eye = torch.eye(3, dtype=torch.float64)[None]
            return (a ** 2)[:, None, None] * eye, b[:, None, None] * eye
        lam, Q = torch.linalg.eigh(self.b_v, UPLO="U")
        if main:
            x = lam * dt
            ca = torch.exp(0.5 * x)
        else:
            x = (lam + lam.sum(1, keepdim=True) / self.dof[:, None]) * dt * 0.5
            ca = torch.exp(-0.5 * x)
        cb = ca * sinh_div(0.5 * x)
        A = Q @ torch.diag_embed(ca ** 2) @ Q.transpose(1, 2)
        B = Q @ torch.diag_embed(cb) @ Q.transpose(1, 2)
        return A, B

    def half_step(self, p, f):
        """propagate_half_step (:661-686, :885-926); f in MD units"""
        A, B = self._operators(False)
        i = self.index_m
        return torch.einsum("ni,nij->nj", p, A[i]) + 0.5 * self.dt * torch.einsum("ni,nij->nj", f, B[i])

    def main_step(self, x, p, cells):
        """propagate_main_step (:633-659, :844-883) -> (positions, cells)"""
        A, B = self._operators(True)
        i = self.index_m
        x = torch.einsum("ni,nij->nj", x, A[i]) + self.dt * torch.einsum("ni,nij->nj", p / self.m, B[i])
        if self.anisotropic:
            cells = cells @ A
        else:
            cells = cells * torch.exp(self.dt * self.b_v)[:, None, None]
        return x, cells

    def state(self):
        return dict(t_velocities=self.t_v, t_forces=self.t_f, t_masses=self.t_m, t_velocities_cell=self.c_v,
                    t_forces_cell=self.c_f, t_masses_cell=self.c_m, b_velocities_cell=self.b_v.reshape(self.n_sys, -1),
                    b_forces_cell=self.b_f.reshape(self.n_sys, -1), b_masses_cell=self.b_m)


def golden_case(g, name, **kw):
    """Run the golden's protocol for one case with the restatement; returns the barostat, positions, momenta, cells."""
    b = NHCBarostat(float(g["target_pressure_bar"]), float(g["temperature_bath"]), float(g["time_constant_fs"]),
                    float(g["kB"]), float(g["fs"]), float(g["bar"]), time_constant_cell=0.5 * float(g["time_constant_fs"]),
                    time_constant_barostat=2.0 * float(g["time_constant_fs"]), **kw)
    b.init(g["masses"], g["n_atoms"], float(g["time_step"]))
    t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))  # noqa: E731
    x, p, cells, stress = t(g["positions"]), t(g["momenta"]), t(g["cells"]), t(g["stress0"])
    for k in range(g["forces"].shape[0]):
        p = b.thermostat(p)
        b.kick(p, cells, stress)
        p = b.half_step(p, _prev_forces(g, k))
        x, cells = b.main_step(x, p, cells)
        f, stress = t(g["forces"][k]), t(g["stress"][k])
        p = b.half_step(p, f)
        b.kick(p, cells, stress)
        p = b.thermostat(p)
    return b, x, p, cells


def _prev_forces(g, k):
    """forces before evaluation k: zero at the start (System.forces), then those of evaluation k - 1"""
    if k == 0:
        return torch.zeros(g["forces"].shape[1:], dtype=torch.float64)
    return torch.as_tensor(g["forces"][k - 1])


def stress_from_virial(spec, params, batch, cell_model):
    """the fp64 oracle's W = sum_e dE/dr_e (x) r_e per system and W / V on the model cell"""
    x = O.to_torch(batch, torch.float64)
    r_ij = O.pairwise_distances(x["_positions"], x["_idx_i"], x["_idx_j"], x["_offsets"])
    x["_Rij"] = r_ij.detach()
    out = O.energy_forces(spec, params, x, dtype=torch.float64, n_mol=int(x["_idx_m"].max()) + 1)
    g = out["dEdRij"]
    n_sys = int(x["_idx_m"].max()) + 1
    sys_e = x["_idx_m"][x["_idx_i"]]
    W = torch.zeros(n_sys, 3, 3, dtype=torch.float64).index_add(0, sys_e, g[:, :, None] * r_ij.detach()[:, None, :])
    return W, W / volume(torch.as_tensor(np.asarray(cell_model, dtype=np.float64)).reshape(-1, 3, 3))[:, None, None]


def npt_trajectory(spec, params, batch, masses, momenta, time_step, n_steps, barostat, position_conversion=1.0,
                   energy_conversion=1.0):
    """NPT loop of md/simulator.py:124-150 with NPTVelocityVerlet for ONE periodic system in model units, with an exact
    neighbour list on the current cell every step; returns MD-unit positions, momenta, energy, cell after ``n_steps``."""
    f_conv = energy_conversion / position_conversion
    pbc = np.asarray(batch["_pbc"]).reshape(3)
    x = torch.as_tensor(np.asarray(batch["_positions"], dtype=np.float64)) / position_conversion
    cells = torch.as_tensor(np.asarray(batch["_cell"], dtype=np.float64)).reshape(1, 3, 3) / position_conversion
    p = torch.as_tensor(np.asarray(momenta, dtype=np.float64)).clone()
    barostat.init(masses, [x.shape[0]], time_step)

    def calculate(x_md, cells_md):
        R = (x_md * position_conversion).numpy()
        cell = (cells_md[0] * position_conversion).numpy()
        ii, jj, ss, off = NL.neighbor_list(R, cell, pbc, spec["cutoff"])
        b = dict(batch)
        b.update({"_positions": R, "_idx_i": ii, "_idx_j": jj, "_offsets": off, "_cell": cell.reshape(1, 3, 3)})
        out = O.energy_forces(spec, params, b, dtype=torch.float64)
        _, s = stress_from_virial(spec, params, b, cell)
        return (out["energy"] * energy_conversion, out["forces"] * f_conv,
                s * energy_conversion / position_conversion ** 3)

    e, f, stress = calculate(x, cells)
    for _ in range(n_steps):
        p = barostat.thermostat(p)
        barostat.kick(p, cells, stress)
        p = barostat.half_step(p, f)
        x, cells = barostat.main_step(x, p, cells)
        e, f, stress = calculate(x, cells)
        p = barostat.half_step(p, f)
        barostat.kick(p, cells, stress)
        p = barostat.thermostat(p)
    return x.numpy(), p.numpy(), e.numpy(), cells.numpy()
