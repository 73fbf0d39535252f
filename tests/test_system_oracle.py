"""CPU: the fp64 restatement of motion removal, wrapping, the initializers and the basic hooks (tests/system_oracle.py)
against the reference's own classes (tests/golden/md_system.npz, given the recorded normals), and the properties of its
two deliberate extensions: the pseudo-inverse of a singular inertia tensor and the centroid wrap of ring polymers."""
import os

import numpy as np
import pytest

import system_oracle as S

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "md_system.npz")
INITIALIZERS = {
    "mb_default": (False, 300.0, dict()),
    "mb_all": (False, 300.0, dict(remove_rotation_=True, wrap_positions_=True)),
    "mb_none": (False, 250.0, dict(remove_center_of_mass_=False, remove_translation_=False)),
    "mb_rot_origin": (False, 300.0, dict(remove_center_of_mass_=False, remove_translation_=False, remove_rotation_=True)),
    "uni_default": (True, 300.0, dict()),
    "uni_all": (True, [200.0, 300.0, 450.0], dict(remove_rotation_=True, wrap_positions_=True)),
    "uni_wrap_rot": (True, 350.0, dict(remove_center_of_mass_=False, remove_rotation_=True, wrap_positions_=True)),
}


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _close(a, b, tol=1e-12):
    scale = max(1.0, float(np.abs(b).max()))
    assert np.abs(a - b).max() <= tol * scale, np.abs(a - b).max()


@pytest.mark.parametrize("R", [1, 4])
@pytest.mark.parametrize("name", sorted(INITIALIZERS))
def test_initializers_match_reference(golden, R, name):
    g, k = golden, f"r{R}"
    uniform, temp, kw = INITIALIZERS[name]
    x, p = S.initialize(g[f"{k}:positions"], g[f"{k}:{name}:normals"], g[f"{k}:masses"], g["n_atoms"], temp, float(g["kB"]),
                        uniform, cells=g["cells"], pbc=g["pbc"], by_centroid=False, f32_factor=True,
                        **kw)
    _close(x, g[f"{k}:{name}:positions"])
    _close(p, g[f"{k}:{name}:momenta"])


@pytest.mark.parametrize("R", [1, 4])
def test_hooks_match_reference(golden, R):
    g, k = golden, f"r{R}"
    m, n = g[f"{k}:masses"], g["n_atoms"]
    for rot, name in ((True, "com_rot"), (False, "com")):
        x, p = S.remove_com_motion(g[f"{k}:positions"], g[f"{k}:momenta"], m, n, rot)
        _close(x, g[f"{k}:hook_{name}:positions"])
        _close(p, g[f"{k}:hook_{name}:momenta"])
    _close(S.wrap_positions(g[f"{k}:positions"], g["cells"], g["pbc"], n, by_centroid=False),
           g[f"{k}:hook_wrap:positions"])
    # the beads of the fixture do not straddle a face before centring, so the centroid wrap agrees there
    _close(S.wrap_positions(g[f"{k}:positions"], g["cells"], g["pbc"], n), g[f"{k}:hook_wrap:positions"])


def test_reference_maxwell_boltzmann_per_system_raises(golden):
    """the device defines the per-system width because the reference cannot run it"""
    assert bool(golden["r1:mb_per_system_raises"]) and bool(golden["r4:mb_per_system_raises"])


def test_uniform_hits_its_temperatures(golden):
    g = golden
    x, p = S.initialize(g["r4:positions"], g["r4:uni_all:normals"], g["r4:masses"], g["n_atoms"], [200.0, 300.0, 450.0],
                        float(g["kB"]), True, remove_translation_=False)
    t = S.temperature(p, g["r4:masses"], g["n_atoms"], float(g["kB"]))
    assert np.allclose(t, [[200.0, 300.0, 450.0]] * 4, rtol=1e-13)


def test_pinv_equals_inverse_for_regular_inertia():
    rng = np.random.default_rng(3)
    x, p, m = rng.normal(size=(1, 7, 3)), rng.normal(size=(1, 7, 3)), rng.uniform(1, 16, 7)
    inertia, L = S.inertia_and_angular_momentum(x, p, m, [7])
    assert np.allclose(S.pinv_solve(inertia, L), np.linalg.solve(inertia, L[..., None])[..., 0], rtol=1e-12, atol=0)


def test_pinv_linear_molecule_removes_perpendicular_angular_momentum():
    rng = np.random.default_rng(4)
    axis = np.array([1.0, 2.0, -0.5]) / np.linalg.norm([1.0, 2.0, -0.5])
    x = (np.array([-1.2, 0.1, 1.3])[:, None] * axis)[None] + np.array([0.3, -0.2, 0.5])
    m = np.array([16.0, 12.0, 16.0])
    x = S.remove_center_of_mass(x, m, [3])
    p = rng.normal(size=(1, 3, 3))
    L0 = S.inertia_and_angular_momentum(x, p, m, [3])[1][0, 0]
    p2 = S.remove_rotation(x, p, m, [3])
    L = S.inertia_and_angular_momentum(x, p2, m, [3])[1][0, 0]
    assert np.all(np.isfinite(p2))
    assert np.abs(L - np.dot(L, axis) * axis).max() < 1e-12 * np.abs(L0).max()     # perpendicular part removed
    assert abs(np.dot(L, axis) - np.dot(L0, axis)) < 1e-12 * np.abs(L0).max()      # the axial part is untouched (zero)


def test_pinv_single_atom_and_empty_system():
    x, p, m = np.array([[[1.0, 2.0, 3.0]]]), np.array([[[0.3, -0.1, 0.2]]]), np.array([12.0])
    xs = S.remove_center_of_mass(x, m, [1, 0])
    assert np.array_equal(S.remove_rotation(xs, p, m, [1, 0]), p)


def test_centroid_wrap_keeps_springs_and_centroids_in_cell():
    rng = np.random.default_rng(5)
    cells = np.array([[[5.0, 0.0, 0.0], [1.0, 4.5, 0.0], [0.5, 0.5, 6.0]]])
    pbc = np.array([[True, True, True]])
    n, R = 40, 8
    frac = rng.uniform(-3, 4, size=(n, 3))
    frac[:5] = np.round(frac[:5])                       # ring polymers that straddle a face
    base = frac @ cells[0]
    x = base[None] + 0.3 * rng.normal(size=(R, n, 3))
    y = S.wrap_positions(x, cells, pbc, [n])
    springs = lambda z: np.sum((z - np.roll(z, -1, axis=0)) ** 2)      # noqa: E731
    assert abs(springs(y) - springs(x)) < 1e-10 * springs(x)
    f = S.fractional(y.mean(axis=0)[None], cells, [n])
    assert np.all(f >= -S.WRAP_EPS - 1e-12) and np.all(f < 1.0 - S.WRAP_EPS + 1e-12)
    shift = S.fractional(x - y, cells, [n])
    assert np.abs(shift - np.round(shift)).max() < 1e-9


def test_wrap_refuses_zero_volume():
    with pytest.raises(ValueError):
        S.wrap_positions(np.zeros((1, 2, 3)), np.zeros((1, 3, 3)), np.ones((1, 3), bool), [2])
