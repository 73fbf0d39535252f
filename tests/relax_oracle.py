"""fp64 numpy restatement of the reference's batchwise L-BFGS (interfaces/batchwise_optimization.py:613-917), one
optimizer per system, with systems of any size (the reference needs equal atom counts).  It is the checker of
``schnetpack_b200.relax``: tests/test_relax_oracle.py pins it to the reference's own runs (tests/golden/relax_lbfgs.npz)."""
import numpy as np


class LBFGSOracle:
    """``positions`` [N, 3] in optimizer units; systems are the segments ``sys_ptr`` [n_sys + 1]; ``fixed`` a boolean
    [N] mask (or None).  ``step(forces, fmax)`` takes forces in optimizer units (before zeroing the fixed atoms)."""

    def __init__(self, positions, sys_ptr, memory=100, maxstep=0.2, damping=1.0, alpha=70.0, fixed=None):
        self.r = np.array(positions, dtype=np.float64).reshape(-1, 3)
        self.sys_ptr = np.asarray(sys_ptr, dtype=np.int64)
        self.n_sys = len(self.sys_ptr) - 1
        self.memory, self.maxstep, self.damping, self.H0 = int(memory), float(maxstep), float(damping), 1.0 / alpha
        self.fixed = None if fixed is None else np.asarray(fixed, dtype=bool)
        self.iteration = 0
        self.s = [[] for _ in range(self.n_sys)]
        self.y = [[] for _ in range(self.n_sys)]
        self.rho = [[] for _ in range(self.n_sys)]
        self.r0 = self.f0 = None
        self.p = np.zeros_like(self.r)
        self.steps_to_converge = np.full(self.n_sys, -1, dtype=np.int64)

    def forces(self, f):
        f = np.array(f, dtype=np.float64).reshape(-1, 3)
        if self.fixed is not None:
            f[self.fixed] = 0.0                                           # get_forces, :196-197
        return f

    def fmax(self, f):
        f = self.forces(f)
        return np.array([np.sqrt((f[a:b] ** 2).sum(-1).max()) if b > a else 0.0
                         for a, b in zip(self.sys_ptr[:-1], self.sys_ptr[1:])])

    def converged(self, f, fmax):
        """per-system mask of step (:773-781) and the reference's converged() per system; updates steps_to_converge"""
        f = self.forces(f)
        conv = np.array([(f[a:b] ** 2).sum(-1).max() < fmax ** 2 if b > a else True
                         for a, b in zip(self.sys_ptr[:-1], self.sys_ptr[1:])])
        self.steps_to_converge = np.where(conv, np.where(self.steps_to_converge >= 0, self.steps_to_converge,
                                                         self.iteration), -1)
        return conv

    def step(self, f, fmax):
        f = self.forces(f)
        conv = self.converged(f, fmax)
        r = self.r
        for m, (a, b) in enumerate(zip(self.sys_ptr[:-1], self.sys_ptr[1:])):
            s_l, y_l, rho_l = self.s[m], self.y[m], self.rho[m]
            fm = f[a:b].reshape(-1)
            if self.iteration > 0:                                          # update, :886-909
                s0 = r[a:b].reshape(-1) - self.r0[a:b].reshape(-1)
                y0 = self.f0[a:b].reshape(-1) - fm
                ys = float(np.dot(y0, s0))
                s_l.append(s0)
                y_l.append(y0)
                rho_l.append(1.0 / ys if ys > 1e-8 else 1.0)
            if self.iteration > self.memory:
                s_l.pop(0)
                y_l.pop(0)
                rho_l.pop(0)
            loopmax = min(self.memory, self.iteration)
            alpha = np.empty(loopmax)
            q = -fm.copy()
            for i in range(loopmax - 1, -1, -1):                            # :806-817
                alpha[i] = rho_l[i] * np.dot(s_l[i], q)
                q -= alpha[i] * y_l[i]
            z = self.H0 * q
            for i in range(loopmax):
                beta = rho_l[i] * np.dot(y_l[i], z)
                z += s_l[i] * (alpha[i] - beta)
            p = np.zeros_like(z) if conv[m] else -z
            p = p.reshape(-1, 3)
            if b > a:                                                       # determine_step, :865-884
                longest = np.max(np.sqrt((p ** 2).sum(-1)))
                if longest >= self.maxstep:
                    p = p * (self.maxstep / longest)
            self.p[a:b] = p
        self.r0, self.f0 = r.copy(), f.copy()
        self.r = r + self.p * self.damping
        self.iteration += 1
        return self.p

    def newest_rho(self):
        """rho of the newest history entry per system (1.0 before the first entry)"""
        return np.array([lst[-1] if lst else 1.0 for lst in self.rho])
