"""CPU: the NEB oracle (tests/neb_oracle.py) anchored without an implementation -- climbing-image NEB on the Mueller-Brown
surface ends at its published saddle, every tangent branch picks the documented tangent and the five-sum force equals
the plain projection, a band on a flat surface spaces its images evenly -- and ``neb.interpolate`` with and without the
minimum image."""
import numpy as np
import pytest
import torch
from scipy.optimize import minimize, root

from neb_oracle import NEBOracle, muller_brown, neb_forces, neb_forces_projection, tangent_weights
from schnetpack_b200.neb import interpolate

MB_MINIMA = ((-0.558, 1.442, 0.0), (-0.050, 0.467, 0.0))
MB_SADDLE = (-0.822, 0.624)          # the published saddle between these two minima


def _minimum(start):
    r = minimize(lambda q: muller_brown(q)[0], np.asarray(start, dtype=np.float64), jac=lambda q: -muller_brown(q)[1],
                 method="BFGS", options=dict(gtol=1e-10))
    return r.x


def _evaluate(x):
    e, f = zip(*[muller_brown(r)[:2] for r in x])
    return np.array(f), np.array(e)


def test_climbing_image_on_mueller_brown_is_the_saddle():
    a, c = (_minimum(m)[None] for m in MB_MINIMA)
    n = 7
    x = np.concatenate([a + (j / (n + 1)) * (c - a) for j in range(1, n + 1)])
    ends = [[muller_brown(a[0])[0], muller_brown(c[0])[0]]]
    o = NEBOracle(x, a, c, ends, [1], n, k=10.0, climb=True, dt=0.005, dtmax=0.025, maxstep=0.05)
    for _ in range(5000):
        f, e = _evaluate(o.positions)
        if o.step(f, e, fmax=1e-3)[1].all():
            break
    f, e = _evaluate(o.positions)
    top = int(o.forces(f, e)[3][0])
    assert top == int(np.argmax(e)) and 0 < top < n - 1
    ci = o.positions[top]
    assert np.linalg.norm(muller_brown(ci)[1]) < 1e-3                  # the climbing image's own force vanishes
    sol = root(lambda q: -muller_brown(q)[1], ci, jac=lambda q: muller_brown(q)[2])
    assert np.linalg.norm(muller_brown(sol.x)[1]) < 1e-9 and np.abs(sol.x - ci).max() < 1e-4
    w = np.linalg.eigvalsh(muller_brown(sol.x)[2])
    assert (w < 0).sum() == 1 and w[0] < -100.0
    assert np.abs(sol.x[:2] - MB_SADDLE).max() < 1e-3 and abs(sol.x[2]) < 1e-10


def _one_image(vp, v0, vn, dp, dm, rng):
    """a band of one interior image of 4 atoms with the given energies and differences"""
    x = rng.normal(size=(4, 3))
    f = rng.normal(size=(4, 3))
    return x, x - dm, x + dp, f, [vp, vn], [v0]


@pytest.mark.parametrize("climb", [False, True])
def test_tangent_branches_and_the_projection(climb):
    rng = np.random.default_rng(0)
    dp, dm = rng.normal(size=(4, 3)), rng.normal(size=(4, 3))
    a, b, c = np.vdot(dp, dp), np.vdot(dm, dm), np.vdot(dp, dm)
    cases = {  # (V_{i-1}, V_i, V_{i+1}) -> (alpha, beta)
        "up": ((0.0, 1.0, 3.0), (1.0, 0.0)),
        "down": ((3.0, 1.0, 0.0), (0.0, 1.0)),
        "max, next higher": ((0.0, 2.0, 1.5), (2.0, 0.5)),          # dV_max = 2 (to i-1), dV_min = 0.5
        "max, previous higher": ((1.5, 2.0, 0.0), (0.5, 2.0)),
        "min, next higher": ((1.0, 0.0, 3.0), (3.0, 1.0)),
        "min, previous higher": ((3.0, 0.0, 1.0), (1.0, 3.0)),
        "flat": ((0.5, 0.5, 0.5), (1.0 / np.sqrt(a), 1.0 / np.sqrt(b))),
    }
    for name, ((vp, v0, vn), want) in cases.items():
        assert np.allclose(tangent_weights(vp, v0, vn, a, b, c), want, rtol=0, atol=1e-15), name
        x, x0, x1, f, ends, e = _one_image(vp, v0, vn, dp, dm, rng)
        k = 0.7
        got, coef, diag, climbing = neb_forces(x, x0, x1, f, e, [ends], [4], 1, k, climb)
        assert np.allclose(coef[0, :2], want, rtol=0, atol=1e-15), name
        naive = neb_forces_projection(dp, dm, f, want[0], want[1], k, climb)
        assert np.abs(got - naive).max() <= 1e-13 * max(1.0, np.abs(naive).max()), name
        t = (want[0] * dp + want[1] * dm)
        t /= np.linalg.norm(t)
        assert abs(diag[0, 1] - np.vdot(f, t)) <= 1e-13 and int(climbing[0]) == (0 if climb else -1), name
        if climb:        # the parallel force reverses, the perpendicular force stays
            assert abs(np.vdot(got, t) + np.vdot(f, t)) <= 1e-13, name
        else:            # only the spring acts along the tangent
            assert abs(np.vdot(got, t) - k * (np.sqrt(a) - np.sqrt(b))) <= 1e-13, name


def test_climbing_image_ties_go_to_the_lowest_index():
    x = np.zeros((4, 3))
    x[:, 0] = [1.0, 2.0, 3.0, 4.0]
    _, _, diag, climbing = neb_forces(x, np.zeros((1, 3)), np.array([[5.0, 0, 0]]), np.zeros((4, 3)),
                                      [0.0, 2.0, 2.0, 1.0], [[0.0, 0.0]], [1], 4, 1.0, True)
    assert climbing.tolist() == [1] and diag[:, 5].tolist() == [0.0, 1.0, 0.0, 0.0]


def test_flat_surface_spaces_the_images_evenly():
    """V = 0 everywhere: every tangent is the bisector, and the springs alone equalise the spacing along the line"""
    n = 6
    t = np.array([0.05, 0.1, 0.45, 0.5, 0.55, 0.9])
    direction = np.array([1.0, -2.0, 0.5])
    a, c = np.zeros((1, 3)), 3.0 * direction[None]
    x = t[:, None] * c
    o = NEBOracle(x, a, c, [[0.0, 0.0]], [1], n, k=1.0, dt=0.05)
    zero_f, zero_e = np.zeros((n, 3)), np.zeros(n)
    for _ in range(2000):
        if o.step(zero_f, zero_e, fmax=1e-8)[1].all():
            break
    assert o.fire.steps_to_converge[0] >= 0
    steps = np.linalg.norm(np.diff(o.path(0)[:, 0], axis=0), axis=1)
    assert np.abs(steps - np.linalg.norm(c) / (n + 1)).max() < 1e-7
    assert np.abs(np.cross(o.positions, direction)).max() < 1e-12          # still on the line


def _endpoints(x0, x1, cell):
    base = {"_atomic_numbers": torch.tensor([29, 29]), "_n_atoms": torch.tensor([2]),
            "_cell": torch.as_tensor(cell, dtype=torch.float32)[None], "_pbc": torch.ones(1, 3, dtype=torch.bool)}
    return (dict(base, _positions=torch.as_tensor(x0, dtype=torch.float32)),
            dict(base, _positions=torch.as_tensor(x1, dtype=torch.float32)))


@pytest.mark.parametrize("skew", [0.0, 0.3])
def test_interpolate_takes_the_short_path_across_a_periodic_face_with_mic(skew):
    cell = np.array([[4.0, 0.0, 0.0], [skew * 4.0, 4.0, 0.0], [0.0, 0.0, 4.0]])
    x0 = np.array([[0.2, 1.0, 1.0], [2.0, 2.0, 2.0]])
    x1 = np.array([[3.8, 1.0, 1.0], [2.0, 2.0, 2.5]])                       # atom 0 hops -0.4 across the x face
    initial, final = _endpoints(x0, x1, cell)
    n = 3
    short = interpolate(initial, final, n, mic=True)
    long = interpolate(initial, final, n, mic=False)
    for batch in (short, long):
        assert batch["_n_atoms"].tolist() == [2] * n and batch["_idx_m"].tolist() == [0, 0, 1, 1, 2, 2]
        assert batch["_atomic_numbers"].tolist() == [29] * 6 and batch["_cell"].shape == (n, 3, 3)
    xs, xl = short["_positions"].double().numpy(), long["_positions"].double().numpy()
    for j in range(1, n + 1):
        np.testing.assert_allclose(xs[2 * (j - 1)], x0[0] + j / (n + 1) * np.array([-0.4, 0.0, 0.0]), atol=1e-6)
        np.testing.assert_allclose(xl[2 * (j - 1)], x0[0] + j / (n + 1) * np.array([3.6, 0.0, 0.0]), atol=1e-6)
        np.testing.assert_allclose(xs[2 * j - 1], xl[2 * j - 1], atol=1e-6)               # atom 1 does not cross
    with pytest.raises(ValueError, match="n_images"):
        interpolate(initial, final, 0)
    with pytest.raises(ValueError, match="atomic numbers"):
        interpolate(initial, dict(final, _atomic_numbers=torch.tensor([29, 28])), 2)
    with pytest.raises(ValueError, match="cells"):
        interpolate(initial, dict(final, _cell=final["_cell"] * 1.01), 2)
