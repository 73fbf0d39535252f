"""Test infrastructure, not product code: fp64 restatement of the reference's ring-polymer NPT -- PILEBarostat
(md/simulation_hooks/barostats_rpmd.py) with the NPTRingPolymer integrator (md/integrators.py:266-305), the centroid
pressure (md/system.py:616-650) and the step around them (md/simulator.py:124-150 with the hooks [thermostat, barostat]) --
pinned to tests/golden/md_rpmd_npt.npz, which the reference's own classes made.  It builds on rpmd_oracle.py (normal modes,
free propagator, ring-polymer thermostats) and npt_oracle.py (StableSinhDiv, volume) without changing them.

Bead arrays are [P, N, 3] fp64 torch tensors, cells and stress [P, B, 3, 3] (replica-major), masses [N], systems contiguous
with n_atoms [B].  The reference passes the target pressure, temperature and time constant through float32 buffers; the
fixture's binary-fraction units make them exact, so the restatement computes in fp64 throughout, as the device does.
"""
from __future__ import annotations

import math

import numpy as np
import torch

import npt_oracle as NPO
import nvt_oracle as NO
import rpmd_oracle as RO

F64 = torch.float64


def philox_cell_noise(seed):
    """the device's barostat noise: normal 0 of the Philox draw of system s at application ``app``"""
    def draw(app, shape):
        return torch.as_tensor(NO.langevin_normals(seed, app, shape[0])[:, 0])
    return draw


def volumes(cells):
    """[P, B] volumes of [P, B, 3, 3] cells (system.py:567-581)"""
    return NPO.volume(cells.reshape(-1, 3, 3)).reshape(cells.shape[:2])


def centroid_pressure(p, masses, n_atoms, cells, stress, tensor=False, kinetic_component=False):
    """system.py:616-650: [B] or [B, 3, 3].  The tensor's kinetic part is the kinetic-energy tensor of the bead-mean
    momenta over the mean volume (the reference raises there)."""
    s = RO._Systems(masses, n_atoms)
    vol = volumes(cells).mean(0)
    pressure = -stress.mean(0)
    pc = p.mean(0, keepdim=True)
    if tensor:
        if kinetic_component:
            kt = 0.5 * s.sum_atoms((pc[..., :, None] * pc[..., None, :] / s.masses[..., None]).reshape(1, -1, 9))
            pressure = pressure + 2.0 * kt[0].reshape(-1, 3, 3) / vol[:, None, None]
        return pressure
    pressure = torch.einsum("bii->b", pressure) / 3.0
    if kinetic_component:
        ke = 0.5 * s.sum_atoms(torch.sum(pc ** 2, dim=2, keepdim=True) / s.masses)[0, :, 0]
        pressure = pressure + 2.0 * ke / vol / 3.0
    return pressure


class PILEBarostat:
    """barostats_rpmd.py:21-208.  ``noise(app, shape)`` returns the [B] standard normals of cell application ``app``."""

    def __init__(self, target_pressure, temperature_bath, time_constant, kB, fs, bar, noise):
        self.P0 = target_pressure * bar
        self.kbt = temperature_bath * kB                                   # :56
        self.frequency = 1.0 / (time_constant * fs)                         # :53
        self.noise = noise
        self.app = 0

    def init(self, rp: RO.RingPolymer, masses, n_atoms):
        """_init_barostat (:66-99)"""
        self.rp, self.sys = rp, RO._Systems(masses, n_atoms)
        self.masses_np, self.n_atoms_np = np.asarray(masses, dtype=np.float64), np.asarray(n_atoms)
        self.dt = rp.time_step
        n = self.sys.n_atoms.to(F64)
        self.mass = 3.0 * n / self.frequency ** 2 * self.kbt                # :83-85
        self.c1 = math.exp(-0.5 * self.frequency * self.dt)                 # :88-93
        self.c2 = torch.sqrt(rp.n_beads * self.mass * self.kbt * (1.0 - self.c1 ** 2))   # :94-99
        self.cell_momenta = torch.zeros(len(n), dtype=F64)

    def thermostat(self):
        """_update_barostat (:101-110)"""
        z = self.noise(self.app, self.cell_momenta.shape)
        self.app += 1
        self.cell_momenta = self.c1 * self.cell_momenta + self.c2 * z

    def half_step(self, p, f, cells, stress):
        """propagate_half_step (:164-208) -> new bead momenta; f in MD units"""
        rp, s = self.rp, self.sys
        P = rp.n_beads
        pn0 = rp.to_normal(p)[0]
        fn0 = rp.to_normal(f)[0]
        vol = volumes(cells).mean(0)
        pcent = centroid_pressure(p, self.masses_np, self.n_atoms_np, cells, stress, kinetic_component=True)
        c1 = 3.0 * P * (vol * (pcent - self.P0) + self.kbt)
        fbm = fn0 / s.masses[0]
        c2 = s.sum_atoms(torch.sum(fbm * pn0, dim=1)[None, ...])[0]
        c3 = s.sum_atoms(torch.sum(fbm * fn0 / 3.0, dim=1)[None, ...])[0]
        h = 0.5 * self.dt
        self.cell_momenta = self.cell_momenta + (h * c1 + h ** 2 * c2 + h ** 3 * c3)
        return p + 0.5 * f * self.dt

    def main_step(self, x, p, cells):
        """propagate_main_step (:113-162) -> (positions, momenta, cells)"""
        rp, s = self.rp, self.sys
        red = (self.cell_momenta / self.mass)[None, :, None]
        a = torch.exp(-self.dt * red)
        b = NPO.sinh_div(self.dt * red)
        a_at, b_at = s.expand_atoms(a), s.expand_atoms(b)
        xn, pn = rp.to_normal(x).clone(), rp.to_normal(p).clone()
        pn[0:1] = pn[0:1] * a_at
        xn[0:1] = xn[0:1] / a_at + b_at * (pn[0:1] / s.masses[0:1]) * self.dt
        cells = cells / a[..., None]
        u = rp.propagator
        xt, pt = xn.clone(), pn.clone()
        pn[1:] = u[1:, 0, 0] * pt[1:] + u[1:, 0, 1] * xt[1:] * s.masses
        xn[1:] = u[1:, 1, 0] * pt[1:] / s.masses + u[1:, 1, 1] * xt[1:]
        return rp.to_beads(xn), rp.to_beads(pn), cells


def tether(x0, k):
    """the fixture's forces and stress: F = -k (x - x0), stress = sum_a k (x - x0) (x) x / V per bead system"""
    x0, k = torch.as_tensor(np.asarray(x0))[None], torch.as_tensor(np.asarray(k))[None, :, None]

    def calc(x, cells, n_atoms):
        s = RO._Systems(np.ones(x.shape[1]), n_atoms)
        f = -k * (x - x0)
        w = (-f)[..., :, None] * x[..., None, :]
        vir = s.sum_atoms(w.reshape(*w.shape[:2], 9)).reshape(x.shape[0], -1, 3, 3)
        return f, vir / volumes(cells)[..., None, None]
    return calc


def rpmd_npt_trajectory(rp: RO.RingPolymer, x, p, cells, masses, n_atoms, calc, n_steps, barostat: PILEBarostat,
                        thermostat=None):
    """md/simulator.py:124-150 with NPTRingPolymer and hooks [thermostat, barostat].  ``calc(x, cells, n_atoms)`` returns
    (forces [P, N, 3] in MD units, stress [P, B, 3, 3] in MD units).  Returns positions, momenta, cells."""
    m = np.asarray(masses, dtype=np.float64)
    if thermostat is not None:
        thermostat.init(rp, m, n_atoms)
    barostat.init(rp, m, n_atoms)
    x = torch.as_tensor(np.asarray(x, dtype=np.float64)).clone()
    p = torch.as_tensor(np.asarray(p, dtype=np.float64)).clone()
    cells = torch.as_tensor(np.asarray(cells, dtype=np.float64)).clone()
    f, stress = calc(x, cells, n_atoms)
    for _ in range(n_steps):
        if thermostat is not None:
            p = thermostat.apply(p)
        barostat.thermostat()
        p = barostat.half_step(p, f, cells, stress)
        x, p, cells = barostat.main_step(x, p, cells)
        f, stress = calc(x, cells, n_atoms)
        p = barostat.half_step(p, f, cells, stress)
        barostat.thermostat()
        if thermostat is not None:
            p = thermostat.apply(p)
    return x, p, cells
