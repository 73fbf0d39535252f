"""Test infrastructure, not product code: fp64 restatement of the reference's ring-polymer MD -- the RingPolymer integrator
(md/integrators.py:113-229), NormalModeTransformer (md/utils/normal_model_transformation.py:37-101), the PILE-L / PILE-G /
TRPMD and NHC ring-polymer thermostats (md/simulation_hooks/thermostats_rpmd.py:33-234,373-501) and the step around them
(md/simulator.py:124-150) -- pinned to tests/golden/md_rpmd.npz, which the reference's own classes made.

Bead arrays are [P, N, 3] fp64 torch tensors (replica-major, as md/system.py:166-168), masses [N], systems contiguous with
n_atoms [n_sys].  Two switches reproduce the reference where ``schnetpack_b200.md`` deliberately differs; only the pinning
test turns them on:
  * ``reference_float32_propagator``: the reference forms omega_k = 2 omega_P sin(k pi / P) in float32
    (integrators.py:175-179), and with it the propagator, the PILE friction coefficients and the NHC masses;
  * ``shared_centroid_noise``: PILE-G takes R from the x-noise of the first atom of the whole batch
    (thermostats_rpmd.py:181,184) instead of each system's own first atom.
Without ``shared_centroid_noise`` a system with zero centroid kinetic energy keeps its centroid, as on the device.
"""
from __future__ import annotations

import numpy as np
import torch

import nvt_oracle as NO

F64 = torch.float64


def transform_matrix(n_beads: int) -> torch.Tensor:
    """normal_model_transformation.py:37-68"""
    c = np.zeros((n_beads, n_beads))
    n = np.arange(1, n_beads + 1)
    c[0, :] = 1.0
    for k in range(1, n_beads // 2 + 1):
        c[k, :] = np.sqrt(2) * np.cos(2 * np.pi * k * n / n_beads)
    for k in range(n_beads // 2 + 1, n_beads):
        c[k, :] = np.sqrt(2) * np.sin(2 * np.pi * k * n / n_beads)
    if n_beads % 2 == 0:
        c[n_beads // 2, :] = (-1) ** n
    return torch.from_numpy(c / np.sqrt(n_beads))


class _Systems:
    def __init__(self, masses, n_atoms):
        self.n_atoms = torch.as_tensor(np.asarray(n_atoms), dtype=torch.long)
        self.index_m = torch.repeat_interleave(torch.arange(len(self.n_atoms)), self.n_atoms)
        self.first = torch.cumsum(self.n_atoms, 0) - self.n_atoms
        self.masses = torch.as_tensor(np.asarray(masses, dtype=np.float64)).reshape(1, -1, 1)

    def sum_atoms(self, x):                                               # system.py:217-231
        return torch.zeros(x.shape[0], len(self.n_atoms), *x.shape[2:], dtype=x.dtype).index_add(1, self.index_m, x)

    def expand_atoms(self, x):                                            # system.py:245-256
        return x[:, self.index_m, ...]


class RingPolymer:
    """integrators.py:113-229 with the normal-mode transform of normal_model_transformation.py:70-101"""

    def __init__(self, n_beads, temperature, time_step, kB, hbar, reference_float32_propagator=False):
        self.n_beads, self.time_step = n_beads, time_step
        self.f32 = reference_float32_propagator
        self.dtype = torch.float32 if self.f32 else F64
        self.omega = kB * n_beads * temperature / hbar                     # :146
        self.c = transform_matrix(n_beads)
        k = torch.arange(n_beads).to(self.dtype)
        self.omega_normal = 2.0 * self.omega * torch.sin(k * np.pi / n_beads)    # :175-179
        omega_dt = self.omega_normal * time_step                           # :182-184
        cos_dt, sin_dt = torch.cos(omega_dt), torch.sin(omega_dt)
        u = torch.zeros(n_beads, 2, 2, dtype=self.dtype)                   # :187-200
        u[:, 0, 0] = cos_dt
        u[:, 1, 1] = cos_dt
        u[:, 0, 1] = -sin_dt * self.omega_normal
        u[1:, 1, 0] = sin_dt[1:] / self.omega_normal[1:]
        u[0, 1, 0] = time_step
        self.propagator = u[..., None, None]

    def to_normal(self, x):                                               # :70-83
        return torch.mm(self.c, x.reshape(self.n_beads, -1)).view(x.shape)

    def to_beads(self, x):                                                # :85-101
        return torch.mm(self.c.transpose(0, 1), x.reshape(self.n_beads, -1)).view(x.shape)

    def main_step(self, x, p, masses):                                    # :204-229
        m = torch.as_tensor(np.asarray(masses, dtype=np.float64)).reshape(1, -1, 1)
        xn, pn = self.to_normal(x), self.to_normal(p)
        u = self.propagator
        p_new = u[:, 0, 0] * pn + u[:, 0, 1] * xn * m
        x_new = u[:, 1, 0] * pn / m + u[:, 1, 1] * xn
        return self.to_beads(x_new), self.to_beads(p_new)


def philox_noise(seed):
    """the device's PILE noise: normals 0..2 of the Philox draw of element k N + a at application ``app``"""
    def draw(app, shape):
        P, N = shape[0], shape[1]
        return torch.as_tensor(NO.langevin_normals(seed, app, P * N).reshape(P, N, 3))
    return draw


class PILE:
    """PILE-L (thermostats_rpmd.py:33-119), PILE-G (``global_``, :122-208) and TRPMD (:211-234: time_constant = 1,
    thermostat_centroid = False).  ``noise(app, shape)`` returns the [P, N, 3] standard normals of application ``app``."""

    def __init__(self, temperature_bath, time_constant, kB, fs, noise, thermostat_centroid=True, damping_factor=1.0,
                 global_=False, shared_centroid_noise=False):
        self.T, self.tau, self.kB = temperature_bath, time_constant * fs, kB
        self.noise, self.centroid, self.damping = noise, thermostat_centroid, damping_factor
        self.global_, self.shared = global_, shared_centroid_noise
        self.app = 0

    def init(self, rp: RingPolymer, masses, n_atoms):
        self.rp, self.sys = rp, _Systems(masses, n_atoms)
        dt = rp.dtype                                                     # float32 buffers in the reference
        gamma = 2 * rp.omega_normal                                       # :75
        if self.centroid:
            gamma[0] = 1.0 / torch.tensor(self.tau, dtype=dt)             # :78-79
        gamma = gamma * torch.tensor(self.damping, dtype=dt)              # :82
        c1 = torch.exp(-0.5 * rp.time_step * gamma)                       # :85-86
        c2 = torch.sqrt(1 - c1 ** 2)
        self.c1, self.c2 = c1[:, None, None].double(), c2[:, None, None].double()
        self.t_bath = torch.tensor(self.T, dtype=dt)
        self.factor = torch.sqrt(self.sys.masses * self.kB * rp.n_beads * self.t_bath)   # :92-97

    def apply(self, p):
        rp, s = self.rp, self.sys
        momenta = rp.to_normal(p)
        noise = self.noise(self.app, p.shape)
        self.app += 1
        if not self.global_:                                              # :115-119
            return rp.to_beads(self.c1 * momenta + self.factor * self.c2 * noise)
        c1c = self.c1[0][None, ...]                                       # :160-189
        mc, nc = momenta[0][None, ...], noise[0][None, ...]
        ke = s.sum_atoms(torch.sum(mc ** 2 / s.masses, dim=2, keepdim=True))
        kef = ke / (self.t_bath * self.kB * rp.n_beads)
        cf = (1 - c1c) / kef
        if self.shared:
            R = nc[0, 0, 0]
        else:
            R = nc[0, s.first, 0][None, :, None]
        alpha_sq = c1c + s.sum_atoms(torch.sum(nc ** 2, dim=2, keepdim=True)) * cf + 2 * R * torch.sqrt(c1c * cf)
        alpha = torch.sqrt(alpha_sq) * torch.sign(R + torch.sqrt(c1c / cf))
        if not self.shared:
            alpha = torch.where(ke > 0, alpha, torch.ones_like(alpha))
        momenta = momenta.clone()
        momenta[0] = s.expand_atoms(alpha)[0] * momenta[0]
        momenta[1:] = self.c1[1:] * momenta[1:] + self.factor * self.c2[1:] * noise[1:]   # :191-195
        return rp.to_beads(momenta)


class NHCRingPolymer:
    """thermostats_rpmd.py:373-501 on top of the massive NHC of thermostats.py:264-468"""

    def __init__(self, temperature_bath, time_constant, kB, fs, local=True, chain_length=3, multi_step=2,
                 integration_order=3):
        self.T, self.tau, self.kB = temperature_bath, time_constant * fs, kB
        self.local, self.L, self.multi_step, self.order = local, chain_length, multi_step, integration_order

    def init(self, rp: RingPolymer, masses, n_atoms):
        self.rp, self.sys = rp, _Systems(masses, n_atoms)
        dt = rp.dtype
        P, N, L = rp.n_beads, self.sys.masses.shape[1], self.L
        self.ts = rp.time_step * NO.YS_WEIGHTS[self.order] / self.multi_step
        frequency = 1.0 / torch.tensor(self.tau, dtype=dt)                # thermostats.py:304
        kbt = torch.tensor(self.T, dtype=dt) * self.kB                    # :308
        self.kbt = (kbt * P).double()                                     # thermostats_rpmd.py:431
        self.dof = torch.ones(P, N, 3, dtype=F64)
        pf = rp.omega_normal.clone()
        pf[0] = 0.5 * frequency                                           # :434-436
        self.masses = torch.ones(P, N, 3, L, dtype=F64)
        self.masses *= (kbt * P) / pf[:, None, None, None] ** 2           # :439-445
        if not self.local:                                                # :449-458
            af = 3.0 * self.sys.expand_atoms(self.sys.n_atoms[None, :, None])[0]
            self.masses[0, :, :, 0] *= af
            self.dof[0, :, :] *= af
        self.v = torch.zeros(P, N, 3, L, dtype=F64)
        self.f = torch.zeros(P, N, 3, L, dtype=F64)

    def _propagate(self, ke):                                             # thermostats.py:398-468
        v, f, M, kbt, dof = self.v, self.f, self.masses, self.kbt, self.dof
        f[..., 0] = (ke - dof * kbt) / M[..., 0]
        scaling = 1.0
        for _ in range(self.multi_step):
            for k in range(self.order):
                h = self.ts[k]
                v[..., -1] += 0.25 * f[..., -1] * h
                for c in range(self.L - 2, -1, -1):
                    coeff = torch.exp(-0.125 * h * v[..., c + 1])
                    v[..., c] = v[..., c] * coeff ** 2 + 0.25 * f[..., c] * coeff * h
                scaling *= torch.exp(-0.5 * h * v[..., 0])
                f[..., 0] = (scaling * scaling * ke - dof * kbt) / M[..., 0]
                for c in range(self.L - 1):
                    coeff = torch.exp(-0.125 * h * v[..., c + 1])
                    v[..., c] = v[..., c] * coeff ** 2 + 0.25 * f[..., c] * coeff * h
                    f[..., c + 1] = (M[..., c] * v[..., c] ** 2 - kbt) / M[..., c + 1]
                v[..., -1] += 0.25 * f[..., -1] * h
        return scaling

    def apply(self, p):                                                   # thermostats_rpmd.py:465-501
        rp, s = self.rp, self.sys
        momenta = rp.to_normal(p)
        ke = momenta ** 2 / s.masses
        if not self.local:
            kec = s.sum_atoms(torch.sum(ke[0:1], dim=2, keepdim=True))
            ke[0, ...] = s.expand_atoms(kec)[0]
        return rp.to_beads(momenta * self._propagate(ke))

    def chain_state(self):
        L = self.L
        return self.v.reshape(-1, L).numpy(), self.f.reshape(-1, L).numpy(), self.masses.reshape(-1, L).numpy()


def rpmd_trajectory(rp: RingPolymer, x, p, masses, n_atoms, forces, n_steps, thermostat=None):
    """md/simulator.py:124-150 with RingPolymer: thermostat, half kick, main step, forces(x) [P, N, 3] in MD units, half
    kick, thermostat.  Returns bead positions and momenta after ``n_steps``."""
    m = np.asarray(masses, dtype=np.float64)
    if thermostat is not None:
        thermostat.init(rp, m, n_atoms)
    x = torch.as_tensor(np.asarray(x, dtype=np.float64)).clone()
    p = torch.as_tensor(np.asarray(p, dtype=np.float64)).clone()
    f = forces(x)
    for _ in range(n_steps):
        if thermostat is not None:
            p = thermostat.apply(p)
        p = p + 0.5 * f * rp.time_step                                    # integrators.py:59-70
        x, p = rp.main_step(x, p, m)
        f = forces(x)
        p = p + 0.5 * f * rp.time_step
        if thermostat is not None:
            p = thermostat.apply(p)
    return x, p


def drift_and_fluctuation(t, H):
    """Least-squares line H ~ a + b t through a conserved-quantity series: returns the drift |b| (t_end - t_0) over the run
    and the standard deviation of the residuals about the line, a fluctuation measured independently of any trend."""
    t, H = np.asarray(t, dtype=np.float64), np.asarray(H, dtype=np.float64)
    A = np.stack([np.ones_like(t), t - t.mean()], axis=1)
    coef, *_ = np.linalg.lstsq(A, H, rcond=None)
    res = H - A @ coef
    return abs(coef[1]) * (t[-1] - t[0]), float(res.std(ddof=2))


def block_mean(x, n_blocks=20):
    """mean of a time series and its standard error from ``n_blocks`` consecutive block means"""
    x = np.asarray(x, dtype=np.float64)
    x = x[: len(x) // n_blocks * n_blocks]
    blocks = x.reshape(n_blocks, -1, *x.shape[1:]).mean(1)
    return blocks.mean(0), blocks.std(0, ddof=1) / np.sqrt(n_blocks)
