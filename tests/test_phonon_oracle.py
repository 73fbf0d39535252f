"""CPU: the fp64 restatement of the phonon method (tests/phonon_oracle.py) against closed forms -- chains, simple cubic,
Einstein solid --, the multiplicity weights of the minimum-image table at exact ties and on a skewed cell, the q-point
helpers and the reference-generated fixture (tests/golden/make_golden_phonons.py)."""
import os

import numpy as np
import pytest

import phonon_oracle as O
from schnetpack_b200.phonons import monkhorst_pack, q_path, supercell_translations

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FCC_M = [[-1, 1, 1], [1, -1, 1], [1, 1, -1]]
TOL = 1e-5
CM = O.HBAR_OMEGA_CM


def _run(pos, cell, s, springs, masses, qs, acoustic=False, rounds=0):
    lattice, neg = O.translations(s)
    fc = O.spring_fc(pos, cell, s, lattice, springs)
    fc = O.symmetrize(fc, len(masses), neg, rounds, acoustic)
    img = O.images(pos, cell, s, lattice, TOL)
    return np.array([O.frequencies(O.dynmat(fc, img, np.asarray(masses), q)) for q in qs])


def test_monatomic_chain():
    K, m = 2.0, 3.0
    cell = np.diag([1.0, 8.0, 8.0])
    qs = np.random.default_rng(0).uniform(-0.5, 0.5, (7, 3)) * [1, 0, 0]
    for s in ([4, 1, 1], [5, 1, 1]):
        f = _run(np.zeros((1, 3)), cell, s, [(0, 0, (1, 0, 0), K)], [m], qs)
        want = 2 * np.sqrt(K / m) * np.abs(np.sin(np.pi * qs[:, 0])) * CM
        assert np.allclose(f[:, -1], want, rtol=1e-12, atol=1e-9)
        assert np.allclose(f[:, :2], 0.0, atol=1e-9)


def test_diatomic_chain():
    K, m1, m2 = 1.5, 1.0, 4.0
    cell = np.diag([1.0, 8.0, 8.0])
    pos = np.array([[0.0, 0, 0], [0.5, 0, 0]])
    qs = np.linspace(-0.5, 0.5, 9)[:, None] * [1, 0, 0]
    f = _run(pos, cell, [4, 1, 1], [(0, 1, (0, 0, 0), K), (1, 0, (1, 0, 0), K)], [m1, m2], qs)
    s = 1 / m1 + 1 / m2
    root = np.sqrt(s ** 2 - 4 * np.sin(np.pi * qs[:, 0]) ** 2 / (m1 * m2))
    assert np.allclose(f[:, -1], np.sqrt(K * (s + root)) * CM, rtol=1e-12)                     # optical
    assert np.allclose(f[:, -2], np.sqrt(np.maximum(K * (s - root), 0)) * CM, rtol=1e-9, atol=1e-6)   # acoustic


def test_simple_cubic_nearest_neighbours():
    K, m = 1.0, 2.0
    springs = [(0, 0, e, K) for e in np.eye(3, dtype=int)]
    qs = np.random.default_rng(1).uniform(-0.5, 0.5, (6, 3))
    f = _run(np.zeros((1, 3)), 3.0 * np.eye(3), [4, 4, 4], springs, [m], qs)
    want = np.sort(2 * np.sqrt(K / m) * np.abs(np.sin(np.pi * qs)), axis=1) * CM
    assert np.allclose(f, want, rtol=1e-12, atol=1e-9)


def test_acoustic_sum_rule_zeroes_gamma():
    rng = np.random.default_rng(2)
    lattice, neg = O.translations([3, 3, 3])
    fc = rng.normal(size=(2 * 2 * 27, 3, 3))
    fc = O.symmetrize(fc, 2, neg, 10, True)
    phi = fc.reshape(2, 27, 2, 3, 3)
    assert np.abs(phi.sum(axis=(1, 2))).max() < 1e-12
    raw = O.symmetrize(fc, 2, neg, 0, False)
    assert np.array_equal(raw, fc)


def test_einstein_solid_and_classical_limit():
    w = 300.0                                    # cm^-1, 3 modes, one q
    freq = np.full((1, 3), w)
    T = np.array([0.0, 10.0, 300.0, 1e6])
    zpe, F, S, C, nx, ni = O.thermo(freq, T)
    e = w * O.INVCM
    assert np.isclose(zpe, 1.5 * e) and nx == 0 and ni == 0
    x = e / (O.KB * T[1:])
    assert np.allclose(F[1:], 3 * (e / 2 + O.KB * T[1:] * np.log(1 - np.exp(-x))), rtol=1e-12)
    assert np.allclose(S[1:], 3 * O.KB * (x / np.expm1(x) - np.log(-np.expm1(-x))), rtol=1e-10)
    assert np.allclose(C[1:3], 3 * O.KB * (x[:2] / (2 * np.sinh(x[:2] / 2))) ** 2, rtol=1e-10)
    assert abs(C[-1] / (3 * O.KB) - 1) < 1e-7                    # C_v -> 3 n k_B (1 - x^2 / 12: 1.6e-8 here)
    assert F[0] == zpe and S[0] == 0 and C[0] == 0
    assert O.thermo(np.array([[-5.0, 0.1, w]]), T)[4:] == (2, 1)


def test_multiplicity_weights_at_ties():
    lattice, _ = O.translations([4, 4, 4])
    img = O.images(np.zeros((1, 3)), 2.0 * np.eye(3), [4, 4, 4], lattice, TOL)
    counts = {tuple(n): img[l][0] for l, n in enumerate(lattice)}
    assert counts[(2, 0, 0)] == 2 and counts[(0, 2, 2)] == 4 and counts[(2, 2, 2)] == 8 and counts[(1, 2, 3)] == 2
    assert counts[(1, 1, 1)] == 1 and counts[(0, 0, 0)] == 1
    for cnt, tr in img:                          # every image is the translation modulo the supercell
        assert len(tr) == cnt
        d = (tr - tr[0]) / 4.0
        assert np.array_equal(d, np.round(d))


def test_skewed_cell_against_a_wide_search():
    cell = np.array([[3.0, 0.0, 0.0], [2.7, 1.1, 0.0], [2.5, 0.8, 0.9]])       # strongly sheared
    pos = np.array([[0.0, 0.0, 0.0], [1.3, 0.4, 0.3]])
    s = [[2, 1, 0], [0, 2, 1], [1, 0, 2]]
    lattice, _ = O.translations(s)
    got = O.images(pos, cell, s, lattice, TOL)
    wide = O.images(pos, cell, s, lattice, TOL, search=6)
    for (c1, t1), (c2, t2) in zip(got, wide):
        assert c1 == c2 and sorted(map(tuple, t1)) == sorted(map(tuple, t2))


@pytest.mark.parametrize("s", [[3, 3, 3], [2, 1, 4], FCC_M, [[2, 1, 0], [0, 2, 1], [1, 0, 2]]])
def test_translations_match_the_package(s):
    lat, neg = O.translations(s)
    lat2, neg2 = supercell_translations(s)
    assert sorted(map(tuple, lat)) == sorted(map(tuple, lat2))
    assert not lat2[0].any()
    order = {tuple(n): i for i, n in enumerate(lat)}
    assert all(order[tuple(lat2[neg2[i]])] == neg[order[tuple(n)]] for i, n in enumerate(lat2))


def test_refused_supercells():
    with pytest.raises(ValueError, match="det > 0"):
        supercell_translations([[1, 0, 0], [0, 1, 0], [0, 0, -1]])
    with pytest.raises(ValueError, match="integer"):
        supercell_translations([2.5, 1, 1])
    with pytest.raises(ValueError, match="det > 0"):
        supercell_translations([0, 1, 1])


def test_helpers():
    q = monkhorst_pack([4, 3, 2]).numpy()
    assert q.shape == (24, 3) and np.any(np.all(q == 0, axis=1))
    assert np.all(q >= -0.5) and np.all(q < 0.5)
    qs = monkhorst_pack([2, 2, 2], shifted=True).numpy()
    assert np.allclose(np.abs(qs), 0.25) and not np.any(np.all(qs == 0, axis=1))
    p = q_path([[0, 0, 0], [0.5, 0, 0], [0.5, 0.5, 0]], 5).numpy()
    assert p.shape == (11, 3) and np.array_equal(p[0], [0, 0, 0]) and np.array_equal(p[5], [0.5, 0, 0])
    assert np.array_equal(p[-1], [0.5, 0.5, 0]) and np.allclose(p[1], [0.1, 0, 0])


def test_golden_force_constants():
    """the rows of the reference's analytic supercell Hessian are the stored force constants, and the finite
    differences of the stored reference forces at the realised steps are within the O(h^2) truncation of them"""
    z = np.load(os.path.join(GOLDEN, "phonons_cscl.npz"))
    n = int(z["in:_n_atoms"][0])
    n_super = z["super_positions"].shape[0]
    fc = O.fc_from_hessian(z["ref64:hessian"], n, n_super)
    assert np.array_equal(fc, z["ref64:force_constants"])
    lattice, _ = O.translations(z["supercell"])
    sp, sc = O.supercell(z["in:_positions"], z["in:_cell"][0], z["supercell"], lattice)
    assert np.array_equal(sp, z["super_positions"]) and np.array_equal(sc, z["super_cell"])
    fd = O.fc_from_displaced(z["fd2:steps"], z["fd2:forces"])
    err = np.abs(fd - fc).max() / np.abs(fc).max()
    print(f"golden: |FC_fd - FC_analytic| / max = {err:.2e}")
    assert err <= TRUNC_BOUND


# largest |FC_fd - FC_analytic| / max |FC_analytic| of the fixture at h = 0.01 A, nfree 2: the O(h^2) truncation of a
# random PaiNN model (measured 3.0e-2, the on-site block of the carbon atom)
TRUNC_BOUND = 5e-2
