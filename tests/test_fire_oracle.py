"""CPU: the fp64 FIRE / unit-cell-filter oracle (tests/fire_oracle.py) pinned without any implementation: generalized
forces against central differences of the enthalpy, the FIRE recurrence against a hand-derived trace, and the relaxed
Morse crystal against its lattice sum."""
import numpy as np
import pytest
from scipy.optimize import brentq, minimize_scalar

from fire_oracle import FIREOracle, fcc, morse, pair_list

RC = 2.4


def _strained_crystal(seed=0):
    rng = np.random.default_rng(seed)
    x, cell = fcc(1.7)
    cell0 = cell @ (np.eye(3) + np.array([[0.0, 0.08, -0.05], [0.03, 0.0, 0.06], [0.0, -0.04, 0.0]]))   # triclinic
    x = x @ np.linalg.solve(cell, cell0) + rng.normal(scale=0.05, size=x.shape)
    return x, cell0


def _set_state(o, s, F):
    n = o._n(0)
    o.X[0] = np.concatenate([s, o.cf[0] * F])
    return n


@pytest.mark.parametrize("p", [0.0, 0.07])
def test_generalized_forces_are_minus_the_enthalpy_gradient(p):
    x0, cell0 = _strained_crystal()
    o = FIREOracle(x0, [0, len(x0)], cells=[cell0], scalar_pressure=p)
    F = np.eye(3) + np.array([[0.02, -0.03, 0.01], [0.04, -0.01, 0.02], [-0.02, 0.03, 0.015]])    # not symmetric
    s = x0 + np.random.default_rng(1).normal(scale=0.02, size=x0.shape)
    n = _set_state(o, s, F)
    pairs = pair_list(o.positions, o.cell(0), RC + 1.0)

    def enthalpy(X):
        o.X[0] = X
        e = morse(o.positions, o.cell(0), pairs, rc=RC)[0]
        return e + p * abs(np.linalg.det(o.cell(0)))

    X = o.X[0].copy()
    _, f, W = morse(o.positions, o.cell(0), pairs, rc=RC)
    g = o.generalized_forces(0, f, W[None])
    fd = np.zeros_like(X)
    h = 1e-5
    for k in np.ndindex(*X.shape):
        Xp, Xm = X.copy(), X.copy()
        Xp[k] += h
        Xm[k] -= h
        fd[k] = -(enthalpy(Xp) - enthalpy(Xm)) / (2 * h)
    o.X[0] = X
    assert np.abs(g - fd).max() <= 1e-7 * np.abs(fd).max()
    assert np.abs(g[n:]).max() > 1e-3 * np.abs(g).max()             # the cell rows carry force

    hyd = FIREOracle(x0, [0, n], cells=[cell0], scalar_pressure=p, hydrostatic_strain=True)
    _set_state(hyd, s, F)
    gc = hyd.generalized_forces(0, f, W[None])[n:]
    assert np.count_nonzero(gc - np.diag(np.diag(gc))) == 0 and gc[0, 0] == gc[1, 1] == gc[2, 2] != 0.0
    masked = FIREOracle(x0, [0, n], cells=[cell0], scalar_pressure=p, mask=[1, 0, 1, 0, 1, 1])
    _set_state(masked, s, F)
    gc = masked.generalized_forces(0, f, W[None])[n:]
    assert gc[1, 1] == gc[1, 2] == gc[2, 1] == 0.0 and np.count_nonzero(gc) == 6
    cv = FIREOracle(x0, [0, n], cells=[cell0], scalar_pressure=p, constant_volume=True)
    _set_state(cv, s, F)
    gc = cv.generalized_forces(0, f, W[None])[n:]
    assert abs(np.trace(gc)) <= 1e-14 * np.abs(gc).max()
    np.testing.assert_allclose(gc - np.diag(np.diag(gc)), (g[n:] - np.diag(np.diag(g[n:]))), rtol=1e-14)


def test_fire_trace_on_a_quadratic_bowl():
    """E = k |x|^2 / 2 for one atom on the x axis.  In one dimension v and g are parallel while going downhill, so the
    mixing leaves v unchanged and the step reduces to the scalar recurrence below; its first values are worked out by
    hand.  The trace passes through the Nmin gate, the dtmax clamp, the maxstep cap and a velocity reset."""
    kw = dict(dt=0.1, maxstep=0.2, dtmax=0.15, Nmin=5, finc=1.1, fdec=0.5, astart=0.1, fa=0.99, a=0.1)
    o = FIREOracle([[8.0, 0.0, 0.0]], [0, 1], **kw)
    x, v, dt, a, ns, first = 8.0, 0.0, 0.1, 0.1, 0, True
    events = set()
    for k in range(80):
        g = -0.125 * x
        if not first:
            if v * g > 0:
                if ns > kw["Nmin"]:
                    grown = min(dt * kw["finc"], kw["dtmax"])
                    events.add("clamp" if grown == kw["dtmax"] and dt * kw["finc"] > kw["dtmax"] else "grow")
                    dt, a = grown, a * kw["fa"]
                elif dt == 0.1 and ns == kw["Nmin"]:
                    events.add("gate")
                ns += 1
            else:
                v, a, dt, ns = 0.0, kw["astart"], dt * kw["fdec"], 0
                events.add("reset")
        first = False
        v += dt * g
        dr = dt * v
        if abs(dr) > kw["maxstep"]:
            dr = kw["maxstep"] * np.sign(dr)
            events.add("cap")
        x += dr
        o.step(np.array([[g, 0.0, 0.0]]), None, 0.0)
        assert abs(o.positions[0, 0] - x) <= 1e-13 and o.positions[0, 1] == o.positions[0, 2] == 0.0, k
        assert o.dt[0] == pytest.approx(dt, rel=1e-14) and o.a[0] == pytest.approx(a, rel=1e-14)
        assert o.Nsteps[0] == ns and abs(o.velocities[0][0, 0] - v) <= 1e-13, k
        if k == 0:
            assert x == pytest.approx(7.99, abs=1e-14)                 # g = -1, v = -0.1, dr = -0.01
        if k == 1:
            assert x == pytest.approx(7.9700125, abs=1e-14)            # g = -0.99875, v = -0.199875, dr = -0.0199875
    assert events >= {"gate", "grow", "clamp", "cap", "reset"}, events


def _lattice_energy(a):
    x, cell = fcc(a)
    return morse(x, cell, pair_list(x, cell, RC), rc=RC)[0]


def _relax(o, fmax=1e-9, steps=5000):
    for _ in range(steps):
        x, cell = o.positions, o.cells[0]
        _, f, W = morse(x, cell, pair_list(x, cell, RC), rc=RC)
        if o.step(f, W[None], fmax).all():
            return True
    return False


@pytest.mark.parametrize("p", [0.0, 0.05])
def test_strained_fcc_relaxes_to_the_lattice_sum_minimum(p):
    a0 = minimize_scalar(_lattice_energy, bounds=(1.4, 2.0), method="bounded", options={"xatol": 1e-12}).x
    if p > 0:        # -dE/dV = p with V = a^3: -E'(a) / (3 a^2) = p
        h = 1e-5
        press = lambda a: -(_lattice_energy(a + h) - _lattice_energy(a - h)) / (2 * h) / (3 * a * a) - p   # noqa: E731
        a_p = brentq(press, 0.8 * a0, a0, xtol=1e-13)
    else:
        a_p = a0
    x, cell = fcc(1.05 * a0)
    strain = np.eye(3) + np.array([[0.02, 0.01, 0.0], [0.01, -0.03, 0.02], [0.0, 0.02, 0.01]])
    o = FIREOracle(x @ strain, [0, 4], cells=[cell @ strain], scalar_pressure=p)
    assert _relax(o)
    c = o.cells[0]
    assert abs(abs(np.linalg.det(c)) ** (1 / 3) / a_p - 1.0) <= 1e-6
    np.testing.assert_allclose(c @ c.T, a_p * a_p * np.eye(3), atol=1e-6 * a_p * a_p)


def test_hydrostatic_strain_keeps_the_shape_and_mask_keeps_masked_components():
    x, cell = _strained_crystal(3)
    o = FIREOracle(x, [0, 4], cells=[cell], hydrostatic_strain=True, scalar_pressure=0.02)
    for _ in range(60):
        _relax(o, steps=1)
    F = o.deform_grad(0)
    assert np.count_nonzero(F - np.diag(np.diag(F))) == 0 and F[0, 0] == F[1, 1] == F[2, 2] != 1.0
    np.testing.assert_allclose(o.cells[0], F[0, 0] * cell, rtol=1e-15)
    for mask, fixed in (([1, 1, 1, 0, 0, 0], [(0, 1), (0, 2), (1, 0), (1, 2), (2, 0), (2, 1)]),
                        ([1, 0, 1, 1, 1, 1], [(1, 1)])):
        o = FIREOracle(x, [0, 4], cells=[cell], mask=mask, scalar_pressure=0.02)
        for _ in range(60):
            _relax(o, steps=1)
        F = o.deform_grad(0)
        for i, j in fixed:
            assert F[i, j] == float(i == j), (mask, i, j)
        assert np.abs(F - np.eye(3)).max() > 1e-3
