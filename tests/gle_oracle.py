"""Test infrastructure, not product code: fp64 restatement of the reference's generalized-Langevin thermostats --
GLEThermostat (md/simulation_hooks/thermostats.py:527-730), RPMDGLEThermostat and PIGLETThermostat
(thermostats_rpmd.py:237-370) -- pinned to tests/golden/md_gle.npz, which the reference's own classes made.

``convention`` selects the propagator of the extended momenta s (s[0] = p, or the normal-mode momentum p~_k):
  * "reference": the reference's row-vector update s <- s c1 + (xi c2) sqrt(m) (thermostats.py:723-726), i.e. c1^T s;
  * "paper": s <- c1 s + sqrt(m) c2 xi (Ceriotti, Bussi, Parrinello 2010), which ``schnetpack_b200.md`` runs.
Bead arrays are [P, N, 3] fp64 torch tensors as in rpmd_oracle.py; the classical thermostat is P = 1 (C = [[1]]).
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as SL
import torch

import nvt_oracle as NO
import rpmd_oracle as RO


def propagators(A, C, time_step):
    """thermostats.py:653-657: c1 = expm(-dt/2 A), c2 = sqrtm(C - c1 C c1^T)"""
    A, C = np.asarray(A, np.float64), np.asarray(C, np.float64)
    c1 = SL.expm(-0.5 * time_step * A)
    c2 = SL.sqrtm(C - c1 @ C @ c1.T)
    return c1, np.real(c2)


def stationary_covariance(c1, c2, convention):
    """the stationary covariance of the map s <- M s + N xi with unit mass: X = M X M^T + N N^T"""
    M, N = (c1, c2) if convention == "paper" else (c1.T, c2.T)
    return SL.solve_discrete_lyapunov(M, N @ N.T)


def philox_noise(seed):
    """the device's GLE noise of application ``app``: [P, N, 3, D], column j of mode k, atom a, component d = normal d of
    the Philox draw of element (j P + k) N + a"""
    def draw(app, P, N, D):
        z = NO.langevin_normals(seed, app, D * P * N).reshape(D, P, N, 3)
        return np.moveaxis(z, 0, -1)
    return draw


class GLE:
    """GLE (``per_mode=False``; RPMD-GLE when run with P > 1) and PIGLET (``per_mode=True``).  ``A`` [n_blocks, D, D] and
    ``C`` (or None) in MD units.  ``noise(app, P, N, D)`` returns standard normals [P, N, 3, D]; application 0 is the
    free-particle-limit start."""

    def __init__(self, A, C, temperature_bath, kB, noise, convention="paper", free_particle_limit=True,
                 per_mode=False, ring_polymer=True):
        self.A = np.asarray(A, np.float64)
        self.C = None if C is None else np.asarray(C, np.float64)
        self.T, self.kB, self.noise = temperature_bath, kB, noise
        self.convention, self.fpl, self.per_mode, self.ring_polymer = convention, free_particle_limit, per_mode, ring_polymer

    def init(self, rp: RO.RingPolymer, masses, n_atoms):
        P, N, D = rp.n_beads, len(masses), self.A.shape[-1]
        self.P, self.c = P, RO.transform_matrix(P).numpy()
        C = self.C
        if C is None:                                                     # thermostats.py:639-648
            C = np.eye(D)[None].repeat(self.A.shape[0], 0) * self.T * self.kB * (P if self.ring_polymer else 1)
        pairs = [propagators(self.A[b], C[b], rp.time_step) for b in range(self.A.shape[0])]
        c1, c2 = np.stack([q[0] for q in pairs]), np.stack([q[1] for q in pairs])
        self.c1 = c1[:, None, None] if self.per_mode else c1[0]           # [P, 1, 1, D, D] or [D, D]
        self.c2 = c2[:, None, None] if self.per_mode else c2[0]
        self.sqm = np.sqrt(np.asarray(masses, np.float64))[None, :, None, None]
        self.app = 0
        self.s = np.zeros((P, N, 3, D))
        if self.fpl:                                                      # thermostats.py:687-701: xi c2
            self.s = np.einsum("...j,...jc->...c", self._draw(), self.c2)

    def _draw(self):
        xi = np.asarray(self.noise(self.app, *self.s.shape[:2], self.s.shape[-1]), np.float64)
        self.app += 1
        return xi

    def apply(self, p):
        pn = np.einsum("kb,b...->k...", self.c, np.asarray(p, np.float64))
        xi = self._draw()
        s = self.s.copy()
        s[..., 0] = pn                                                    # thermostats.py:720
        if self.convention == "reference":                                # :723-726
            s = np.einsum("...c,...cr->...r", s, self.c1) + np.einsum("...c,...cr->...r", xi, self.c2) * self.sqm
        else:
            s = np.einsum("...rc,...c->...r", self.c1, s) + self.sqm * np.einsum("...rc,...c->...r", self.c2, xi)
        self.s = s
        return torch.as_tensor(np.einsum("kb,k...->b...", self.c, s[..., 0]))


def write_gle_file(path, A, C=None, a_unit="femtoseconds^-1", c_unit="K"):
    """a gle4md raw-format matrix file: A [n_blocks, D, D] (and C) in the given units, one '# Matrix for normal mode k'
    block each when there is more than one"""
    A = np.asarray(A, np.float64)

    def section(title, unit, M):
        lines = [f"# {title} ({unit})"]
        for k, block in enumerate(M):
            if len(M) > 1:
                lines.append(f"# Matrix for normal mode {k}")
            lines += ["  ".join(f"{v: .17e}" for v in row) for row in block]
        return lines

    lines = section("A MATRIX:", a_unit, A)
    if C is not None:
        lines += section("C MATRIX:", c_unit, np.asarray(C, np.float64))
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")
