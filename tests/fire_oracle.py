"""fp64 numpy restatement of ASE's FIRE (without downhill_check) and ASE's UnitCellFilter, one optimizer per system of a
batch, written in ASE's own order of operations.  It is the checker of ``schnetpack_b200.relax.FIREState`` /
``DeviceFIRE``; tests/test_fire_oracle.py pins it by finite differences, a hand-derived trace and physics.

Also here: a periodic shifted-force Morse potential with analytic fp64 energies, forces and virials (the strain
derivative W = dE/d(strain), the convention of the device virial), on a pair list of integer image shifts."""
import numpy as np


# ---- FIRE and the unit-cell filter -------------------------------------------------------------------------------------
def voigt_mask(mask):
    """ASE's voigt_6_to_full_3x3_stress of a 6-component mask (xx, yy, zz, yz, xz, xy); a 3 x 3 mask as it is"""
    if mask is None:
        return np.ones((3, 3))
    m = np.asarray(mask, dtype=np.float64)
    if m.shape == (3, 3):
        return m
    xx, yy, zz, yz, xz, xy = m
    return np.array([[xx, xy, xz], [xy, yy, yz], [xz, yz, zz]])


class FIREOracle:
    """``positions`` [N, 3] in optimizer units; systems are the segments ``sys_ptr``; ``fixed`` a boolean [N] mask or
    None.  With ``cells`` [n_sys, 3, 3] (rows = lattice vectors) every system gets a unit-cell filter with the keywords
    ``mask``, ``cell_factor`` (None: the atom count), ``hydrostatic_strain``, ``constant_volume`` and
    ``scalar_pressure``.  ``step(forces, virials, fmax)`` takes forces [N, 3] and virials [n_sys, 3, 3] in optimizer
    units (the virial: the strain derivative of the energy, as the model's virial times energy_conversion)."""

    def __init__(self, positions, sys_ptr, cells=None, fixed=None, dt=0.1, maxstep=0.2, dtmax=1.0, Nmin=5, finc=1.1,
                 fdec=0.5, astart=0.1, fa=0.99, a=0.1, mask=None, cell_factor=None, hydrostatic_strain=False,
                 constant_volume=False, scalar_pressure=0.0):
        self.sys_ptr = np.asarray(sys_ptr, dtype=np.int64)
        self.n_sys = len(self.sys_ptr) - 1
        self.fixed = None if fixed is None else np.asarray(fixed, dtype=bool)
        self.maxstep, self.dtmax, self.Nmin, self.finc = float(maxstep), float(dtmax), int(Nmin), float(finc)
        self.fdec, self.astart, self.fa = float(fdec), float(astart), float(fa)
        self.filter = cells is not None
        self.mask = voigt_mask(mask)
        self.hydrostatic_strain, self.constant_volume = bool(hydrostatic_strain), bool(constant_volume)
        self.pressure = float(scalar_pressure)
        pos = np.array(positions, dtype=np.float64).reshape(-1, 3)
        self.X, self.cell0, self.cf = [], [], []
        for m, (i0, i1) in enumerate(self._segments()):
            if self.filter:
                cf = float(i1 - i0) if cell_factor is None else float(cell_factor)
                self.cell0.append(np.array(cells[m], dtype=np.float64).reshape(3, 3))
                self.cf.append(cf)
                self.X.append(np.concatenate([pos[i0:i1], cf * np.eye(3)]))     # F = I: s = x
            else:
                self.X.append(pos[i0:i1].copy())
        self.v = [None] * self.n_sys
        self.dt = np.full(self.n_sys, float(dt))
        self.a = np.full(self.n_sys, float(a))
        self.Nsteps = np.zeros(self.n_sys, dtype=np.int64)
        self.iteration = 0
        self.steps_to_converge = np.full(self.n_sys, -1, dtype=np.int64)

    def _segments(self):
        return list(zip(self.sys_ptr[:-1], self.sys_ptr[1:]))

    def _n(self, m):
        return int(self.sys_ptr[m + 1] - self.sys_ptr[m])

    # UnitCellFilter.deform_grad / get_positions / set_positions
    def deform_grad(self, m):
        return self.X[m][self._n(m):] / self.cf[m]

    def cell(self, m):
        return self.cell0[m] @ self.deform_grad(m).T

    @property
    def cells(self):
        return np.stack([self.cell(m) for m in range(self.n_sys)])

    @property
    def positions(self):
        out = []
        for m in range(self.n_sys):
            n = self._n(m)
            out.append(self.X[m][:n] @ self.deform_grad(m).T if self.filter else self.X[m])
        return np.concatenate(out)

    @property
    def scaled(self):
        """the atom rows of the generalized coordinates [N, 3] (the positions without a filter)"""
        return np.concatenate([self.X[m][:self._n(m)] for m in range(self.n_sys)])

    @property
    def velocities(self):
        """atom rows [N, 3] and cell rows [n_sys, 9] of v (zeros before a system's first step)"""
        va, vc = [], []
        for m in range(self.n_sys):
            n = self._n(m)
            v = self.v[m] if self.v[m] is not None else np.zeros_like(self.X[m])
            va.append(v[:n])
            vc.append(v[n:].reshape(-1))
        return np.concatenate(va), (np.stack(vc) if self.filter else None)

    def generalized_forces(self, m, forces, virial):
        """UnitCellFilter.get_forces of system m: atom rows f F, cell rows P(Vir F^-T) / cell_factor"""
        i0, i1 = self.sys_ptr[m], self.sys_ptr[m + 1]
        f = np.array(forces[i0:i1], dtype=np.float64).reshape(-1, 3)
        if self.fixed is not None:
            f[self.fixed[i0:i1]] = 0.0
        if not self.filter:
            return f
        F = self.deform_grad(m)
        volume = abs(np.linalg.det(self.cell(m)))
        stress = 0.5 * (virial[m] + virial[m].T) / volume
        vir = -volume * (stress + np.diag([self.pressure] * 3))
        f = f @ F
        vir = np.linalg.solve(F, vir.T).T
        if self.hydrostatic_strain:
            vir = np.diag([np.trace(vir) / 3.0] * 3)
        vir = vir * self.mask
        if self.constant_volume:
            vtr = np.trace(vir)
            np.fill_diagonal(vir, np.diag(vir) - vtr / 3.0)
        return np.concatenate([f, vir / self.cf[m]])

    def fmax(self, forces, virials=None):
        return np.array([np.sqrt((self.generalized_forces(m, forces, virials) ** 2).sum(-1).max())
                         for m in range(self.n_sys)])

    def converged(self, forces, virials, fmax):
        """per-system convergence test; updates steps_to_converge as the device does"""
        conv = np.array([(self.generalized_forces(m, forces, virials) ** 2).sum(-1).max() < fmax ** 2
                         for m in range(self.n_sys)])
        self.steps_to_converge = np.where(conv, np.where(self.steps_to_converge >= 0, self.steps_to_converge,
                                                         self.iteration), -1)
        return conv

    def fire_step(self, m, f):
        """FIRE.step of system m on the generalized forces f"""
        if self.v[m] is None:
            self.v[m] = np.zeros_like(self.X[m])
        else:
            vf = np.vdot(f, self.v[m])
            if vf > 0.0:
                self.v[m] = (1.0 - self.a[m]) * self.v[m] + self.a[m] * f / np.sqrt(np.vdot(f, f)) * np.sqrt(
                    np.vdot(self.v[m], self.v[m]))
                if self.Nsteps[m] > self.Nmin:
                    self.dt[m] = min(self.dt[m] * self.finc, self.dtmax)
                    self.a[m] *= self.fa
                self.Nsteps[m] += 1
            else:
                self.v[m][:] *= 0.0
                self.a[m] = self.astart
                self.dt[m] *= self.fdec
                self.Nsteps[m] = 0
        self.v[m] += self.dt[m] * f
        dr = self.dt[m] * self.v[m]
        normdr = np.sqrt(np.vdot(dr, dr))
        if normdr > self.maxstep:
            dr = self.maxstep * dr / normdr
        self.X[m] = self.X[m] + dr

    def step(self, forces, virials=None, fmax=0.0):
        """the convergence test, then one step of every unconverged system"""
        conv = self.converged(forces, virials, fmax)
        for m in range(self.n_sys):
            if not conv[m]:
                self.fire_step(m, self.generalized_forces(m, forces, virials))
        self.iteration += 1
        return conv


# ---- periodic shifted-force Morse --------------------------------------------------------------------------------------
def morse_pair(r, D=1.0, alpha=3.0, r0=1.2, rc=2.4):
    """shifted-force Morse phi(r) - phi(rc) - (r - rc) phi'(rc) for r < rc (0 beyond) and its derivative"""
    def phi(x):
        e = np.exp(-alpha * (x - r0))
        return D * (e * e - 2.0 * e), D * (-2.0 * alpha * e * e + 2.0 * alpha * e)

    p, dp = phi(r)
    pc, dpc = phi(rc)
    inside = r < rc
    return np.where(inside, p - pc - (r - rc) * dpc, 0.0), np.where(inside, dp - dpc, 0.0)


def pair_list(x, cell, reach):
    """ordered pairs (i, j, image n) of one system with |x_j + n cell - x_i| < reach, i != j or n != 0, found among all
    images that can be that close (for small systems)"""
    inv = np.linalg.inv(cell)
    widths = 1.0 / np.linalg.norm(inv, axis=0)                 # distances between opposite cell faces
    nmax = np.ceil(reach / widths).astype(int) + 1
    shifts = np.array(np.meshgrid(*[np.arange(-k, k + 1) for k in nmax], indexing="ij")).reshape(3, -1).T
    n = len(x)
    ii, jj = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    ii, jj = ii.reshape(-1), jj.reshape(-1)
    out = []
    for s in shifts:
        d = x[jj] + s @ cell - x[ii]
        keep = (np.linalg.norm(d, axis=1) < reach) & ((ii != jj) | np.any(s != 0))
        if keep.any():
            out.append(np.column_stack([ii[keep], jj[keep], np.tile(s, (int(keep.sum()), 1))]))
    return np.concatenate(out).astype(np.int64) if out else np.zeros((0, 5), dtype=np.int64)


def pair_list_orthorhombic(x, lengths, reach):
    """the same for a large orthorhombic cell with reach < min(lengths) / 2, by a periodic k-d tree"""
    from scipy.spatial import cKDTree

    xs = np.mod(x, lengths)
    ij = cKDTree(xs, boxsize=lengths).query_pairs(reach, output_type="ndarray")
    d = x[ij[:, 1]] - x[ij[:, 0]]
    s = -np.round(d / lengths).astype(np.int64)
    fwd = np.column_stack([ij[:, 0], ij[:, 1], s])
    bwd = np.column_stack([ij[:, 1], ij[:, 0], -s])
    return np.concatenate([fwd, bwd])


def morse(x, cell, pairs, **kw):
    """energy, forces [n, 3] and virial W [3, 3] (dE/d strain) of one system on the pair list ``pairs``"""
    i, j, s = pairs[:, 0], pairs[:, 1], pairs[:, 2:].astype(np.float64)
    d = x[j] + s @ cell - x[i]
    r = np.linalg.norm(d, axis=1)
    e, de = morse_pair(r, **kw)
    u = de[:, None] * d / r[:, None]                    # dE_pair/dd, each ordered pair counted with weight 1/2
    f = np.zeros_like(x)
    np.add.at(f, i, u)
    return 0.5 * e.sum(), f, 0.5 * np.einsum("pa,pb->ab", u, d)


def fcc(a, reps=(1, 1, 1)):
    """fcc crystal of lattice constant a: positions and the (cubic) cell"""
    base = np.array([[0, 0, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [0.5, 0.5, 0]])
    cells = np.array([[i, j, k] for i in range(reps[0]) for j in range(reps[1]) for k in range(reps[2])])
    frac = (base[None] + cells[:, None]).reshape(-1, 3)
    return frac * a, np.diag(np.asarray(reps, dtype=np.float64) * a)
