"""CPU checks of the ring-polymer test oracle (tests/rpmd_oracle.py) against the reference's own ring-polymer MD, recorded in
tests/golden/md_rpmd.npz, and host-side checks of ``schnetpack_b200.md``'s ring-polymer set-up that need no device."""
import math
import os

import numpy as np
import pytest
import torch

import rpmd_oracle as RO

GOLD = os.path.join(os.path.dirname(__file__), "golden", "md_rpmd.npz")
BEADS = [1, 4, 5, 8]
THERMOSTATS = ["pile_l", "pile_g", "trpmd", "nhc_local", "nhc_global"]


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def _close(a, b, tol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.max(np.abs(a - b)) <= tol * max(np.max(np.abs(b)), 1e-300), np.max(np.abs(a - b))


def _rp(g, P, f32=True):
    return RO.RingPolymer(P, float(g["temperature"]), float(g["time_step_fs"]) * float(g["fs"]), float(g["kB"]),
                          float(g["hbar"]), reference_float32_propagator=f32)


def _thermostat(g, name, noise):
    T, tau, kB, fs = float(g["temperature_bath"]), float(g["time_constant_fs"]), float(g["kB"]), float(g["fs"])
    if name == "pile_l":
        return RO.PILE(T, tau, kB, fs, noise)
    if name == "pile_g":
        return RO.PILE(T, tau, kB, fs, noise, global_=True, shared_centroid_noise=True)
    if name == "trpmd":
        return RO.PILE(T, 1.0, kB, fs, noise, thermostat_centroid=False, damping_factor=0.5)
    if name == "nhc_local":
        return RO.NHCRingPolymer(T, tau, kB, fs, local=True)
    return RO.NHCRingPolymer(T, tau, kB, fs, local=False, chain_length=4, integration_order=5)


def _run(g, P, name):
    pre = f"P{P}:"
    rp = _rp(g, P)
    x0, k = torch.as_tensor(g[pre + "x0"])[None], torch.as_tensor(g[pre + "k_tether"])[None, :, None]
    noise = None
    if pre + name + ":noise" in g:
        rec = torch.as_tensor(g[pre + name + ":noise"])
        noise = lambda app, shape: rec[app]   # noqa: E731
    th = None if name == "nve" else _thermostat(g, name, noise)
    x, p = RO.rpmd_trajectory(rp, g[pre + "positions"], g[pre + "momenta"], g[pre + "masses"], g["n_atoms"],
                              lambda x: -k * (x - x0), int(g["n_steps"]), th)
    return x, p, th


@pytest.mark.parametrize("P", BEADS)
def test_transform_and_propagator_match_reference(gold, P):
    pre = f"P{P}:"
    _close(RO.transform_matrix(P).numpy(), gold[pre + "c_transform"], 0.0)
    c = gold[pre + "c_transform"]
    _close(c @ c.T, np.eye(P), 1e-14)                                       # C is orthogonal
    rp = _rp(gold, P)
    _close(rp.omega_normal.numpy(), gold[pre + "omega_normal"], 0.0)
    _close(rp.propagator[..., 0, 0].numpy(), gold[pre + "propagator"], 0.0)
    rp64 = _rp(gold, P, f32=False)                                         # the fp64 propagator of the library
    _close(rp64.propagator[..., 0, 0].numpy(), gold[pre + "propagator"], 1e-6)


@pytest.mark.parametrize("name", ["nve"] + THERMOSTATS)
@pytest.mark.parametrize("P", BEADS)
def test_oracle_matches_reference(gold, P, name):
    x, p, th = _run(gold, P, name)
    key = f"P{P}:{name}:"
    _close(x.numpy(), gold[key + "positions"])
    _close(p.numpy(), gold[key + "momenta"])
    assert np.abs(gold[key + "positions"] - gold[f"P{P}:positions"]).max() > 1e-3        # the run moved
    if name.startswith("nhc"):
        v, f, m = th.chain_state()
        _close(v, gold[key + "velocities"])
        _close(f, gold[key + "forces"])
        _close(m, gold[key + "masses"])
        assert np.abs(v).max() > 0


def test_pile_global_per_system_noise_differs_only_by_R(gold):
    """with one R per system the PILE-G update equals the reference's for the first system (whose first atom supplies the
    batch-global R) and differs for the others"""
    P = 4
    pre = f"P{P}:"
    rec = torch.as_tensor(gold[pre + "pile_g:noise"])
    rp = _rp(gold, P)
    out = {}
    for shared in (True, False):
        th = RO.PILE(300.0, 64.0, float(gold["kB"]), float(gold["fs"]), lambda app, shape: rec[app], global_=True,
                     shared_centroid_noise=shared)
        th.init(rp, gold[pre + "masses"], gold["n_atoms"])
        out[shared] = th.apply(torch.as_tensor(gold[pre + "momenta"])).numpy()
    n0 = int(gold["n_atoms"][0])
    _close(out[False][:, :n0], out[True][:, :n0], 1e-14)
    assert np.abs(out[False][:, n0:] - out[True][:, n0:]).max() > 1e-6


def test_hbar_matches_the_reference_formula():
    """units.py:80-82: hbar = ase._hbar * (J * s) / (energy * time) with ASE's CODATA-2014 constants"""
    from schnetpack_b200.md import HBAR_MD

    _hplanck, _e, _amu, _Nav = 6.626070040e-34, 1.6021766208e-19, 1.660539040e-27, 6.022140857e23
    _hbar = _hplanck / (2 * math.pi)
    J, s = 1.0 / _e, 1e10 * math.sqrt(_e / _amu)                            # ASE: eV, Angstrom, amu frame
    kJmol = 1000.0 * J / _Nav
    nm = 10.0
    time = nm * math.sqrt(1.0 / kJmol)                                      # units.py:37 (mass Da = amu)
    ref = _hbar * (J * s) / (kJmol * time)
    assert abs(HBAR_MD - ref) <= 1e-14 * ref
    assert 0.0634 < HBAR_MD < 0.0636


def test_ring_polymer_arguments_are_checked_on_the_host():
    from schnetpack_b200 import md

    for bad in (0, 65, -1, 2.5):
        with pytest.raises(ValueError):
            md.RingPolymer(bad, 300.0)
    for bad in (0.0, -10.0):
        with pytest.raises(ValueError):
            md.RingPolymer(8, bad)
    rp = md.RingPolymer(64, 300.0)
    c = rp.transform_matrix()
    assert torch.allclose(c @ c.T, torch.eye(64, dtype=torch.float64), atol=1e-13)
    assert torch.allclose(c, RO.transform_matrix(64), rtol=0.0, atol=1e-15)
    u = rp.propagator(1e-3)
    assert float(u[0, 1, 0]) == 1e-3 and float(u[0, 0, 1]) == 0.0 and float(u[0, 0, 0]) == 1.0
    w = rp.omega_normal
    assert abs(float(w[1]) - 2.0 * md.KB_MD * 64 * 300.0 / md.HBAR_MD * math.sin(math.pi / 64)) < 1e-9 * float(w[1])


def test_forbidden_combinations_are_refused_on_the_host():
    from schnetpack_b200 import md

    rp = md.RingPolymer(4, 300.0)
    check = md.DeviceMD._check_ring_polymer
    with pytest.raises(ValueError, match="classical thermostat"):
        check(rp, md.LangevinThermostat(300.0, 100.0), None, False)
    with pytest.raises(ValueError, match="ring-polymer thermostat"):
        check(None, md.PILELocalThermostat(300.0, 100.0), None, False)
    with pytest.raises(ValueError, match="barostat"):
        check(rp, None, md.NHCBarostatIsotropic(1.0, 300.0, 100.0), False)
    with pytest.raises(ValueError, match="compute_stress"):
        check(rp, None, None, True)
    for th in (md.PILELocalThermostat(300.0, 100.0), md.PILEGlobalThermostat(300.0, 100.0),
               md.TRPMDThermostat(300.0, 0.5), md.NHCRingPolymerThermostat(300.0, 100.0, local=False), None):
        check(rp, th, None, False)                                          # accepted
    check(None, md.NHCThermostat(300.0, 100.0), None, False)
    with pytest.raises(ValueError):
        md.PILELocalThermostat(300.0, 100.0).bind(None, 1e-3)               # no ring polymer to bind to


def test_drift_check_trips_on_heating_and_passes_stationary_series():
    """the test of a conserved ring-polymer Hamiltonian bounds the fitted drift by 3 residual standard deviations: a
    stationary, correlated series passes; linear or exponential heating of a few fluctuations trips it"""
    rng = np.random.default_rng(0)
    t = np.arange(150.0)
    noise = np.zeros(150)
    for i in range(1, 150):                                                # AR(1), correlation time ~10 samples
        noise[i] = 0.9 * noise[i - 1] + rng.normal()
    sigma = noise.std()
    for series, ok in ((noise, True), (noise + 5.0 * sigma * t / t[-1], False),
                       (noise + 5.0 * sigma * np.expm1(3.0 * t / t[-1]) / np.expm1(3.0), False),
                       (100.0 + noise - 4.0 * sigma * t / t[-1], False)):
        drift, fluct = RO.drift_and_fluctuation(t, series)
        assert (drift < 3.0 * fluct) == ok, (drift, fluct, ok)


def test_shared_cell_and_pbc_are_expanded_per_bead_system():
    """a cell / pbc shared by all systems becomes one row per bead system (the neighbour list broadcasts only one row)"""
    from schnetpack_b200 import md

    B, P = 3, 4
    cell = torch.eye(3)[None] * 7.0
    static = {"_positions": torch.zeros(5, 3), "_idx_m": torch.tensor([0, 0, 1, 2, 2]), "_n_atoms": torch.tensor([2, 1, 2]),
              "_cell": cell, "_pbc": torch.tensor([True, False, True])}
    out = md.replicate_batch(static, P, B)
    assert out["_cell"].shape == (P * B, 3, 3) and torch.equal(out["_cell"], cell.expand(P * B, 3, 3))
    assert out["_pbc"].shape == (3 * P * B,) and torch.equal(out["_pbc"].reshape(-1, 3), static["_pbc"].expand(P * B, 3))
    assert torch.equal(out["_idx_m"][5:10], static["_idx_m"] + B) and out["_positions"].shape == (P * 5, 3)
    per_system = dict(static, _cell=cell.expand(B, 3, 3).clone(), _pbc=static["_pbc"].repeat(B))
    out2 = md.replicate_batch(per_system, P, B)
    for k in out:
        assert torch.equal(out[k], out2[k]), k
    with pytest.raises(ValueError, match="neither shared nor one per system"):
        md.replicate_batch(dict(static, _cell=torch.eye(3).repeat(2, 1, 1)), P, B)
