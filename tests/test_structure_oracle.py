"""CPU: the fp64 oracle of the structural observables (tests/structure_oracle.py) against closed forms."""
import math

import numpy as np

from structure_oracle import (coordination_from_sums, fcc, msd_oracle, rdf_counts, rdf_from_sums, shell_volumes,
                              wrap)


def _single_species(N):
    return np.zeros(N, int), np.array([[0]]), 1


def test_fcc_shells_and_coordination():
    """perfect fcc (a = 4, 3 x 3 x 3 conventional cells, r_max = 6 = half the cell width): delta shells at a / sqrt 2,
    a, a sqrt(3/2) and a sqrt 2 holding 12, 6, 24 and 12 neighbours"""
    a, r_max, n_bins = 4.0, 6.0, 590
    R, cell = fcc(a, 3)
    N = R.shape[0]
    types, slot_of, n_slots = _single_species(N)
    counts, amb = rdf_counts(R, cell, types, slot_of, -1, n_slots, r_max, n_bins)
    assert amb.sum() == 0
    V = abs(np.linalg.det(cell))
    n = coordination_from_sums(counts[None] * V, np.array([V]), np.array([[N]]))[0, 0]
    dr = r_max / n_bins
    radii = [a / math.sqrt(2), a, a * math.sqrt(1.5), a * math.sqrt(2)]
    shells = [12, 6, 24, 12]
    nonzero = np.nonzero(counts[0])[0]
    assert list(nonzero) == [int(r / dr) for r in radii]
    assert [int(counts[0, k]) // N for k in nonzero] == shells
    cumulative = np.cumsum(shells)
    for k, c in zip(nonzero, cumulative):
        assert math.isclose(n[k], c, rel_tol=1e-12)
    g = rdf_from_sums(counts[None] * V, 1, np.array([[N]]), np.array([[N]]), r_max)[0, 0]
    rho = N / V
    for k, z in zip(nonzero, shells):           # the integral of the delta shell: 4 pi rho g r^2 dr = z
        assert math.isclose(rho * g[k] * shell_volumes(r_max, n_bins)[k], z, rel_tol=1e-12)


def test_fcc_species_pairs_and_triclinic_cell():
    """the same crystal in its primitive (triclinic) cell with two sublattices: the pair slots add up to the total and
    r_max beyond half the cell width counts self-images"""
    a = 4.0
    cell = a * np.array([[0.0, 0.5, 0.5], [0.5, 0.0, 0.5], [0.5, 0.5, 0.0]]) * 2        # 2 x 2 x 2 primitive cells
    prim = a * np.array([[0.0, 0.5, 0.5], [0.5, 0.0, 0.5], [0.5, 0.5, 0.0]])
    R = np.array([i * prim[0] + j * prim[1] + k * prim[2] for i in range(2) for j in range(2) for k in range(2)])
    types = np.array([0, 1] * 4)
    slot_of = np.array([[0, 1], [-1, 2]])
    counts, amb = rdf_counts(R, cell, types, slot_of, 3, 4, 6.0, 590)
    assert amb.sum() == 0
    # ordered a-b counted once per direction of the table: aa + 2 ab + bb = total
    assert np.array_equal(counts[0] + 2 * counts[1] + counts[2], counts[3])
    n = coordination_from_sums(counts[None] * 1.0, np.array([1.0]), np.array([[len(R)] * 4]))[0, 3]
    dr = 6.0 / 590
    np.testing.assert_allclose([n[int(a / math.sqrt(2) / dr)], n[int(a / dr)], n[int(a * math.sqrt(1.5) / dr)]],
                               [12, 18, 42], rtol=1e-12)


def test_uniform_random_points_give_one():
    """N uniform points: E[n(k)] = N (N - 1) shell_k / V (minimum image not involved: r_max < L / 2), and the ordered
    count of a bin has variance 2 E (each unordered pair counts twice), so |g - (N - 1) / N| < 5 sqrt(2 / E) per bin"""
    rng = np.random.default_rng(7)
    N, L, r_max, n_bins = 800, 16.0, 6.0, 30
    R = rng.uniform(0.0, L, (N, 3))
    cell = np.eye(3) * L
    types, slot_of, n_slots = _single_species(N)
    counts, _ = rdf_counts(R, cell, types, slot_of, -1, n_slots, r_max, n_bins)
    V = L ** 3
    g = rdf_from_sums(counts[None] * V, 1, np.array([[N]]), np.array([[N]]), r_max)[0, 0]
    E = N * (N - 1) * shell_volumes(r_max, n_bins) / V
    assert np.all(np.abs(g - (N - 1) / N) < 5.0 * np.sqrt(2.0 / E))
    assert abs(g[n_bins // 2:].mean() - (N - 1) / N) < 0.02


def _constant_velocity(wrapped, remove_com):
    rng = np.random.default_rng(3)
    N, L, T = 12, 10.0, 40
    cell = np.array([[L, 0, 0], [1.5, L, 0], [-1.0, 2.0, L]])
    x0 = rng.uniform(0, L, (N, 3))
    v = rng.normal(0, 0.6, (N, 3))          # |v| dt well below half a cell height
    traj = np.stack([x0 + v * t for t in range(T)])
    if wrapped:
        traj = np.stack([wrap(x, cell) for x in traj])
    species = np.array([0, 1, 2] * 4)
    masses = rng.uniform(1, 20, N)
    acc, count, jump = msd_oracle(traj, np.broadcast_to(cell, (T, 1, 3, 3)), np.ones((1, 3), bool), masses, species,
                                  [0, N], 3, 25, 5, remove_com)
    return acc, count, jump, v, species, masses


def test_constant_velocity_msd_is_v2_t2():
    for wrapped in (False, True):
        acc, count, jump, v, species, _ = _constant_velocity(wrapped, remove_com=False)
        assert not jump
        m = acc / count
        t = np.arange(25)
        for s in range(3):
            want = (v[species == s] ** 2).sum() * t ** 2
            np.testing.assert_allclose(m[0, s], want, rtol=1e-10, atol=1e-9)
        # origins at samples 0, 5, ..., 35 in 5 slots, each held for 25 samples: lag 24 is reached by the origins 0, 5,
        # 10 and 15 (at samples 24 to 39), lag 0 by all 8
        assert count[0] == 8 and count[24] == 4


def test_constant_velocity_msd_without_com_drift():
    acc, count, _, v, species, masses = _constant_velocity(True, remove_com=True)
    vc = (masses[:, None] * v).sum(0) / masses.sum()
    t = np.arange(25)
    for s in range(3):
        want = ((v[species == s] - vc) ** 2).sum() * t ** 2
        np.testing.assert_allclose((acc / count)[0, s], want, rtol=1e-10, atol=1e-9)


def test_jump_of_more_than_half_a_cell_is_flagged():
    L = 10.0
    cell = np.eye(3) * L
    traj = np.zeros((3, 2, 3))
    traj[:, 1] = 5.0
    traj[2, 0] = [4.5, 4.5, 4.5]            # |d| = 7.8 > L / 2: its minimum image is still 7.8 long
    _, _, jump = msd_oracle(traj, np.broadcast_to(cell, (3, 1, 3, 3)), np.ones((1, 3), bool), np.ones(2),
                            np.zeros(2, int), [0, 2], 1, 3, 1, False)
    assert jump
