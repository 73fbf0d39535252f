"""CPU checks of the NVT test oracle (tests/nvt_oracle.py): its thermostats against the reference's own, recorded in
tests/golden/md_thermostats.npz, and its Philox4x32-10 against published known-answer vectors."""
import os

import numpy as np
import pytest
import torch

import nvt_oracle as NO

GOLD = os.path.join(os.path.dirname(__file__), "golden", "md_thermostats.npz")
NHC_CASES = {"nhc_o3": dict(massive=False, integration_order=3), "nhc_o5": dict(massive=False, integration_order=5),
             "nhc_massive_o3": dict(massive=True, integration_order=3),
             "nhc_massive_o7": dict(massive=True, integration_order=7, chain_length=4, multi_step=3)}


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def _args(g):
    return float(g["temperature_bath"]), float(g["time_constant_fs"]), float(g["kB"]), float(g["fs"])


def _run(th, g):
    th.init(g["masses"], g["n_atoms"], float(g["time_step"]))
    p = torch.as_tensor(g["momenta"])
    for _ in range(int(g["n_apply"])):
        p = th.apply(p)
    return p.numpy()


def _close(a, b, tol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    assert np.max(np.abs(a - b)) <= tol * max(np.max(np.abs(b)), 1e-300), np.max(np.abs(a - b))


def test_temperature_matches_reference(gold):
    s = NO._System(gold["masses"], gold["n_atoms"])
    T = s.temperature(torch.as_tensor(gold["momenta"])[None], float(gold["kB"])).reshape(-1).numpy()
    _close(T, gold["temperature"])
    assert (T > 10).all()


def test_berendsen_matches_reference(gold):
    p = _run(NO.Berendsen(*_args(gold)), gold)
    _close(p, gold["berendsen:momenta"])
    assert np.abs(p - gold["momenta"]).max() > 1e-3 * np.abs(gold["momenta"]).max()   # it did rescale


@pytest.mark.parametrize("name", sorted(NHC_CASES))
def test_nhc_matches_reference(gold, name):
    th = NO.NHC(*_args(gold), **NHC_CASES[name])
    p = _run(th, gold)
    _close(p, gold[name + ":momenta"])
    v, f, m = th.chain_state()
    _close(v, gold[name + ":velocities"])
    _close(f, gold[name + ":forces"])
    _close(m, gold[name + ":masses"])
    assert np.abs(v).max() > 0


def test_langevin_coefficients_match_reference(gold):
    th = NO.Langevin(*_args(gold), seed=3)
    th.init(gold["masses"], gold["n_atoms"], float(gold["time_step"]))
    _close(th.c1.reshape(-1), gold["langevin:c1"])
    _close(th.c2.reshape(-1), gold["langevin:c2"])
    _close(th.thermostat_factor.reshape(-1), gold["langevin:thermostat_factor"])


@pytest.mark.parametrize("ctr,key,expect", [
    # Random123 kat_vectors, philox4x32_10
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, expect):
    out = NO.philox4x32_10(np.array([ctr], dtype=np.uint32), key)
    assert tuple(int(v) for v in out[0]) == expect


def test_langevin_normals_are_standard_normal():
    z = NO.langevin_normals(seed=11, app=4, n_atoms=200_000).reshape(-1)
    n = z.size
    assert abs(z.mean()) < 5 / np.sqrt(n)
    assert abs(z.var() - 1.0) < 5 * np.sqrt(2.0 / n)
    # different applications and seeds draw independent noise
    z2 = NO.langevin_normals(seed=11, app=5, n_atoms=200_000).reshape(-1)
    z3 = NO.langevin_normals(seed=12, app=4, n_atoms=200_000).reshape(-1)
    assert abs(np.corrcoef(z, z2)[0, 1]) < 5 / np.sqrt(n)
    assert abs(np.corrcoef(z, z3)[0, 1]) < 5 / np.sqrt(n)
