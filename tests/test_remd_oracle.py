"""CPU: the replica-exchange oracle (tests/remd_oracle.py) pinned to closed forms: the Metropolis rule on hand-built pairs,
detailed balance on exact Boltzmann samples of a harmonic well, the acceptance against its integral, and the per-system
thermostats against tests/nvt_oracle.py."""
import math

import numpy as np
import pytest
import torch

import nvt_oracle as NO
import remd_oracle as RO

KB = 0.0083144598


def test_two_rung_delta_and_acceptance():
    T = np.array([300.0, 400.0])
    # the colder rung holds the higher energy: Delta > 0, always accepted
    d = RO.deltas([-10.0, -12.0], T, KB, 2, 1)
    assert d.shape == (1, 1)
    assert d[0, 0] == pytest.approx((1 / (KB * 300) - 1 / (KB * 400)) * 2.0, rel=1e-15) and d[0, 0] > 0
    for seed in range(20):
        assert RO.decide([-10.0, -12.0], T, KB, 2, 1, 0, seed)[1][0, 0]
    # equal energies: Delta = 0, accepted
    assert RO.decide([5.0, 5.0], T, KB, 2, 1, 0, 3)[1][0, 0]
    # the colder rung far lower: exp(Delta) ~ 1e-87, never accepted
    assert not any(RO.decide([-1000.0, 0.0], T, KB, 2, 1, 0, seed)[1][0, 0] for seed in range(20))
    # a moderate Delta < 0: accepted exactly when u < exp(Delta)
    U = [-10.0, -9.0]
    d = RO.deltas(U, T, KB, 2, 1)[0, 0]
    assert d < 0
    for seed in range(50):
        u = RO.uniforms(seed, 0, 1)[0]
        assert RO.decide(U, T, KB, 2, 1, 0, seed)[1][0, 0] == (u < math.exp(d))
    # attempt 1 tries only odd k: with K = 2 no pair
    active, acc = RO.decide([-10.0, -12.0], T, KB, 2, 1, 1, 0)
    assert not active.any() and not acc.any()


def test_even_odd_pairs_walkers_and_statistics():
    K, G = 5, 7
    rng = np.random.default_rng(0)
    T = np.repeat(300.0 * 1.1 ** np.arange(K), G)
    ex = RO.Exchange(K, G, KB, seed=11)
    for n in range(6):
        U = rng.normal(0.0, 2.0, K * G)
        active, acc = RO.decide(U, T, KB, K, G, n, 11)
        assert (active[:, n % 2::2]).all() and not active[:, 1 - n % 2::2].any()
        assert (ex.step(U, T) == acc).all()
        assert sorted(ex.walker.tolist()) == list(range(K * G))                 # a permutation
        assert (ex.walker.reshape(K, G) % G == np.arange(G)).all()              # walkers stay in their group
    assert ex.attempt == 6 and (ex.attempted == 3).all()
    assert 0 < ex.accepted.sum() < ex.attempted.sum()


def test_swap_moves_rows_and_rescales_momenta():
    K, G = 2, 2
    n_atoms = [2, 3, 2, 3]
    sys_ptr = np.concatenate([[0], np.cumsum(n_atoms)])
    T = np.array([300.0, 300.0, 600.0, 600.0])
    rng = np.random.default_rng(1)
    p = rng.normal(size=(10, 3)).astype(np.float32)
    x = rng.normal(size=(10, 3)).astype(np.float32)
    e = rng.normal(size=4).astype(np.float32)
    dec = np.array([[False], [True]])                                        # group 1 swaps systems 1 and 3
    p2, (x2,), (e2,) = RO.swap(dec, K, G, sys_ptr, T, p, [x], [e])
    a, b = np.arange(2, 5), np.arange(7, 10)
    assert (x2[a] == x[b]).all() and (x2[b] == x[a]).all() and (x2[:2] == x[:2]).all()
    assert e2.tolist() == [e[0], e[3], e[2], e[1]]
    assert np.allclose(p2[b], p[a] * math.sqrt(2.0), rtol=1e-7) and np.allclose(p2[a], p[b] / math.sqrt(2.0), rtol=1e-7)
    # the kinetic temperature of the moved configuration follows the rung: K' / K = T_new / T_old
    assert (p2[b].astype(np.float64) ** 2).sum() / (p[a].astype(np.float64) ** 2).sum() == pytest.approx(2.0, rel=1e-6)


def _harmonic_rounds(K, G, d, T, rounds, seed, flip=False):
    """rounds of: fresh exact samples U_k ~ Gamma(d / 2, kB T_k) at every rung, one exchange attempt, the energies each
    rung holds afterwards.  Returns the mean of those energies per rung [K] and the exchange state."""
    rng = np.random.default_rng(seed)
    ex = RO.Exchange(K, G, KB, seed=seed)
    Tk = np.repeat(T, G)
    sums = np.zeros(K)
    for _ in range(rounds):
        U = rng.gamma(d / 2.0, KB * Tk)
        acc = ex.step(-U if flip else U, Tk)
        _, _, (U2,) = RO.swap(acc, K, G, None, Tk, None, per_system=[U])
        sums += U2.reshape(K, G).mean(1)
    return sums / rounds, ex


def test_exchange_keeps_the_boltzmann_energies_of_every_rung():
    """Exchange moves between exact samples of the product of Boltzmann distributions keep it: after every attempt rung k
    still has <U> = d kB T_k / 2.  With the sign of Delta flipped the cold rung heats up, which the test detects."""
    K, G, d, rounds = 4, 4000, 12, 40
    T = 300.0 * 1.2 ** np.arange(K)
    mean, ex = _harmonic_rounds(K, G, d, T, rounds, seed=5)
    expect = d * KB * T / 2.0
    sigma = expect * math.sqrt(2.0 / d) / math.sqrt(G * rounds)            # std of Gamma(d/2) mean over the samples
    assert np.all(np.abs(mean - expect) < 5.0 * sigma), (mean, expect, sigma)
    assert (0.05 < ex.accepted.sum() / ex.attempted.sum() < 0.95)
    bad, _ = _harmonic_rounds(K, G, d, T, rounds, seed=5, flip=True)
    assert abs(bad[0] - expect[0]) > 20.0 * sigma[0]


def test_mean_acceptance_matches_its_integral():
    """P(accept) = E[min(1, exp((beta_0 - beta_1)(U_0 - U_1)))] with U_k ~ Gamma(d/2, kB T_k), integrated with scipy"""
    from scipy import integrate, stats

    d, T = 12, np.array([300.0, 360.0])
    b0, b1 = 1.0 / (KB * T)
    f0, f1 = stats.gamma(d / 2.0, scale=KB * T[0]), stats.gamma(d / 2.0, scale=KB * T[1])
    hi = 20.0 * d * KB * T[1]
    expect = integrate.dblquad(lambda u1, u0: f0.pdf(u0) * f1.pdf(u1) * min(1.0, math.exp((b0 - b1) * (u0 - u1))),
                               0.0, hi, 0.0, hi, epsabs=1e-10)[0]
    G, rounds = 20000, 10
    rng = np.random.default_rng(2)
    ex = RO.Exchange(2, G, KB, seed=9)
    Tk = np.repeat(T, G)
    for _ in range(rounds):
        ex.step(rng.gamma(d / 2.0, KB * Tk), Tk)                              # odd attempts try no pair at K = 2
    n = int(ex.attempted.sum())
    p = ex.accepted.sum() / n
    assert n == G * rounds // 2
    assert abs(p - expect) < 5.0 * math.sqrt(expect * (1 - expect) / n), (p, expect)


def test_per_system_langevin_equals_the_scalar_oracle_at_one_temperature():
    rng = np.random.default_rng(3)
    n_atoms = [3, 1, 5]
    m = rng.uniform(1.0, 16.0, 9)
    p = rng.normal(size=(9, 3))
    c1, c2 = 0.9, math.sqrt(1 - 0.81)
    th = NO.Langevin(250.0, 10.0, KB, 1.0, seed=4)
    th.init(m, n_atoms, 1.0)
    th.c1[:], th.c2[:] = c1, c2
    ref = th.apply(torch.as_tensor(p)).numpy()
    assert np.allclose(RO.langevin_kick(p, m, n_atoms, [250.0] * 3, KB, c1, c2, 4, 0), ref, rtol=1e-12, atol=0)
    hot = RO.langevin_kick(p, m, n_atoms, [250.0, 250.0, 1000.0], KB, c1, c2, 4, 0)
    assert np.array_equal(hot[:4], RO.langevin_kick(p, m, n_atoms, [250.0] * 3, KB, c1, c2, 4, 0)[:4])
    noise = (hot[4:] - c1 * p[4:]) / (ref[4:] - c1 * p[4:])
    assert np.allclose(noise, 2.0, rtol=1e-12)                               # sqrt(1000 / 250)


@pytest.mark.parametrize("massive", [False, True])
def test_per_system_nhc_equals_the_scalar_oracle_at_one_temperature(massive):
    rng = np.random.default_rng(4)
    n_atoms = [4, 2, 6]
    m = rng.uniform(1.0, 16.0, 12)
    p = rng.normal(size=(12, 3))
    a = NO.NHC(300.0, 20.0, KB, 1.0, massive=massive)
    b = RO.NHCPerSystem([300.0] * 3, 20.0, KB, 1.0, massive=massive)
    a.init(m, n_atoms, 0.5)
    b.init(m, n_atoms, 0.5)
    pa, pb = torch.as_tensor(p), p
    for _ in range(4):
        pa, pb = a.apply(pa), b.apply(pb)
    assert np.allclose(pb.numpy(), pa.numpy(), rtol=1e-12, atol=1e-14)
    for x, y in zip(a.chain_state(), b.chain_state()):
        assert np.allclose(x, y, rtol=1e-12, atol=1e-14)
