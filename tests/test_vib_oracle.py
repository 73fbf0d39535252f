"""CPU: the fp64 restatement of the vibrational analysis (tests/vib_oracle.py) against the reference-generated fixtures
(tests/golden/make_golden_vibrations.py), against closed forms for a Morse diatomic, and its chunk bookkeeping."""
import os

import numpy as np
import pytest

import vib_oracle as V

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["vib_ethanol", "vib_heads", "vib_box"]


def _load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    ptr = np.concatenate([[0], np.cumsum(z["in:_n_atoms"])])
    return z, ptr


def _fd(z, ptr, nfree):
    raws = [V.hessian_from_displaced(z[f"fd{nfree}:steps:{m}"], z[f"fd{nfree}:forces:{m}"]) for m in range(len(ptr) - 1)]
    return V.finish(raws, z["masses"], ptr)


@pytest.mark.parametrize("nfree", [2, 4])
@pytest.mark.parametrize("name", CASES)
def test_reproduces_the_stored_finite_differences(name, nfree):
    z, ptr = _load(name)
    h, mw = _fd(z, ptr, nfree)
    fd = z[f"fd{nfree}:hessian"]
    assert h.shape == z["ref64:hessian"].shape == fd.shape
    assert np.abs(h - fd).max() <= 1e-10 * np.abs(fd).max()
    for m, b in enumerate(mw):                                   # the symmetrised blocks are exactly symmetric
        assert np.array_equal(b, b.T), m


# largest |FD - analytic| / max |analytic| at h = 0.01 A (measured: ethanol 1.7e-3 / 1.4e-3, heads 4.6e-3 / 7.7e-3, box
# 1.2e-3 / 1.0e-3 for nfree 2 / 4).  The columns converge as h^2 and h^4 (test_truncation_order); at this h the random
# heads model's O-H terms are anharmonic enough on the +-2h span that the 4-point stencil is not yet the tighter one.
BOUNDS = {"vib_ethanol": 3e-3, "vib_heads": 1.5e-2, "vib_box": 2.5e-3}


@pytest.mark.parametrize("name", CASES)
def test_matches_the_reference_analytic_hessian(name):
    z, ptr = _load(name)
    ref = z["ref64:hessian"]
    err = {nf: np.abs(_fd(z, ptr, nf)[0] - ref).max() / np.abs(ref).max() for nf in (2, 4)}
    assert max(err.values()) <= BOUNDS[name], err
    if name != "vib_heads":
        assert err[4] < err[2], err


def _morse_forces(D, a, r0):
    def forces(pos, ptr):
        f = np.zeros_like(pos)
        for m in range(len(ptr) - 1):
            r = pos[ptr[m]:ptr[m + 1]]
            d = r[:, None, :] - r[None, :, :]
            dist = np.sqrt((d ** 2).sum(-1))
            np.fill_diagonal(dist, 1.0)
            e = np.exp(-a * (dist - r0))
            dE = 2.0 * D * a * (1.0 - e) * e
            np.fill_diagonal(dE, 0.0)
            f[ptr[m]:ptr[m + 1]] = -((dE / dist)[:, :, None] * d).sum(1)
        return f
    return forces


def _replica(fn, ptr):
    n = ptr[-1]
    return lambda pos, C: np.concatenate([fn(pos[c * n:(c + 1) * n], ptr) for c in range(C)])


def test_truncation_order():
    """the scheme's error falls as h^2 (nfree 2) and h^4 (nfree 4) on a stretched Morse diatomic, whose exact second
    derivative is known"""
    D, a, r0 = 0.8, 1.7, 1.25
    base = np.array([[0.0, 0.0, 0.0], [r0 + 0.05, 0.0, 0.0]], dtype=np.float32)
    ptr = np.array([0, 2])
    r = float(base[1, 0]) - float(base[0, 0])
    e = np.exp(-a * (r - r0))
    k_exact = 2.0 * D * a * a * e * (2.0 * e - 1.0)               # d2E/dr2
    fn = _replica(_morse_forces(D, a, r0), ptr)
    errs = {}
    for nfree in (2, 4):
        for h in (0.02, 0.01):
            hess = V.hessian(fn, base, ptr, np.ones(2), h, nfree, 6)[0]
            errs[nfree, h] = abs(hess[0, 0, 0] - k_exact)
    assert 3.5 <= errs[2, 0.02] / errs[2, 0.01] <= 4.5, errs
    assert 12.0 <= errs[4, 0.02] / errs[4, 0.01] <= 20.0, errs
    assert errs[4, 0.01] < errs[2, 0.01]


@pytest.mark.parametrize("nfree,h", [(2, 1e-4), (4, 1e-3)])
def test_morse_stretch_frequency_and_ir_intensity(nfree, h):
    D, a, r0, q = 0.8, 1.7, 1.25, 0.37
    masses = np.array([12.011, 15.999])
    base = np.array([[0.0, 0.0, 0.0], [r0, 0.0, 0.0]], dtype=np.float32)
    ptr = np.array([0, 2])
    fn = _replica(_morse_forces(D, a, r0), ptr)

    def dipole(pos, C):
        p = pos.reshape(C, 2, 3)
        return {"dipole_moment": q * (p[:, 0] - p[:, 1])}

    hess, mw, d = V.hessian(fn, base, ptr, masses, h, nfree, 3, props_fn=dipole)
    mu = masses.prod() / masses.sum()
    freq = V.frequencies(mw)
    expect = V.HBAR_OMEGA_CM * np.sqrt(2.0 * D * a * a / mu)
    assert abs(freq[-1] - expect) <= 1e-6 * expect
    assert np.abs(freq[:-1]).max() <= 1e-3 * expect                    # translations and rotations
    ir = V.ir_intensities(mw, masses, ptr, d["dipole_moment"])
    assert abs(ir[-1] - q * q / mu) <= 1e-6 * q * q / mu
    # sum rule over all 3n modes (they are complete): sum_c,i (d mu_c / d x_i)^2 / m_i = 3 q^2 / mu; the rotations of the
    # dipole carry the rest, the translations nothing
    assert abs(ir.sum() - 3.0 * q * q / mu) <= 1e-6 * q * q / mu


@pytest.mark.parametrize("n_cols", [1, 2, 4, 5, 7, 9, 30])
def test_chunk_bookkeeping_and_layout_independence(n_cols):
    """every (system, coordinate, stencil node) is evaluated exactly once, idle copies are exactly d >= 3 n_m, and the
    Hessian does not depend on the number of coordinates per chunk (9 does not divide 3 n_max = 12 or 30)"""
    sizes = np.array([1, 4, 2, 0, 3])
    ptr = np.concatenate([[0], np.cumsum(sizes)])
    nfree = 2
    n_chunks, table = V.chunk_layout(sizes, n_cols, nfree)
    assert n_chunks == -(-12 // n_cols)
    for m, n in enumerate(sizes):
        seen = table[:, :, m].reshape(-1)
        ds = seen[seen >= 0]
        assert sorted(ds.tolist()) == sorted(list(range(3 * n)) * nfree)
        assert (seen < 0).sum() == n_chunks * n_cols * nfree - 3 * n * nfree
    rng = np.random.default_rng(3)
    base = (rng.normal(size=(ptr[-1], 3)) * 1.2).astype(np.float32)
    masses = rng.uniform(1.0, 16.0, ptr[-1])
    fn = _replica(_morse_forces(0.5, 1.3, 1.4), ptr)
    ref = V.hessian(fn, base, ptr, masses, 0.01, nfree, 30)[0]
    got = V.hessian(fn, base, ptr, masses, 0.01, nfree, n_cols)[0]
    assert np.array_equal(got, ref)
    pos, steps = V.displace(base, ptr, n_chunks - 1, n_cols, nfree, 0.01)
    idle = table[n_chunks - 1] < 0
    assert np.all(steps[idle] == 0.0) and np.all(steps[~idle] != 0.0)


def test_lagrange_weights_reduce_to_ase_for_equal_steps():
    h = 0.01
    np.testing.assert_allclose(V.lagrange_d0(np.array([-h, h])), np.array([-1.0, 1.0]) / (2 * h), rtol=1e-14)
    np.testing.assert_allclose(V.lagrange_d0(np.array([-2 * h, -h, h, 2 * h])),
                               np.array([1.0, -8.0, 8.0, -1.0]) / (12 * h), rtol=1e-12)
