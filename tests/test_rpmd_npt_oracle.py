"""CPU checks of the ring-polymer NPT test oracle (tests/rpmd_npt_oracle.py) against the reference's own PILEBarostat with
NPTRingPolymer, recorded in tests/golden/md_rpmd_npt.npz, of the Philox restatement of the barostat noise, and host-side
checks of ``schnetpack_b200.md``'s ring-polymer NPT set-up that need no device."""
import os

import numpy as np
import pytest
import torch

import nvt_oracle as NO
import rpmd_npt_oracle as RNO
import rpmd_oracle as RO

GOLD = os.path.join(os.path.dirname(__file__), "golden", "md_rpmd_npt.npz")
BEADS = [1, 4, 5, 8]
CASES = ["none", "pile_l", "pile_g", "trpmd", "nhc_local", "nhc_global"]


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def _close(a, b, tol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.max(np.abs(a - b)) <= tol * max(np.max(np.abs(b)), 1e-300), np.max(np.abs(a - b))


def _thermostat(g, name, noise):
    T, tau, kB, fs = float(g["temperature_bath"]), float(g["time_constant_fs"]), float(g["kB"]), float(g["fs"])
    if name == "none":
        return None
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
    pre, key = f"P{P}:", f"P{P}:{name}:"
    rp = RO.RingPolymer(P, float(g["temperature"]), float(g["time_step_fs"]) * float(g["fs"]), float(g["kB"]),
                        float(g["hbar"]), reference_float32_propagator=True)
    noise = None
    if key + "noise" in g:
        rec = torch.as_tensor(g[key + "noise"])
        noise = lambda app, shape: rec[app]   # noqa: E731
    baro_rec = torch.as_tensor(g[key + "baro_noise"])
    baro = RNO.PILEBarostat(float(g["target_pressure_bar"]), float(g["temperature_cell"]),
                            float(g["time_constant_cell_fs"]), float(g["kB"]), float(g["fs"]), float(g["bar"]),
                            lambda app, shape: baro_rec[app])
    cells = np.repeat(g["cells"][None], P, axis=0)
    x, p, c = RNO.rpmd_npt_trajectory(rp, g[pre + "positions"], g[pre + "momenta"], cells, g[pre + "masses"],
                                      g["n_atoms"], RNO.tether(g[pre + "x0"], g[pre + "k_tether"]), int(g["n_steps"]),
                                      baro, _thermostat(g, name, noise))
    return x, p, c, baro


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("P", BEADS)
def test_oracle_matches_the_reference_pile_barostat(gold, P, name):
    x, p, c, baro = _run(gold, P, name)
    key = f"P{P}:{name}:"
    _close(x.numpy(), gold[key + "positions"])
    _close(p.numpy(), gold[key + "momenta"])
    _close(c.numpy(), gold[key + "cells"])
    _close(baro.cell_momenta.numpy(), gold[key + "cell_momenta"])
    _close(baro.mass.numpy(), gold[f"P{P}:cell_mass"], 1e-15)
    _close(baro.c2.numpy(), gold[f"P{P}:c2"], 1e-15)
    assert gold[key + "baro_noise"].shape == (2 * int(gold["n_steps"]), len(gold["n_atoms"]))
    v0 = np.linalg.det(gold["cells"])
    assert np.abs(np.linalg.det(gold[key + "cells"][0]) / v0 - 1.0).max() > 5e-3          # the cells moved
    for r in range(1, P):                                                                 # every bead copy alike
        assert np.array_equal(gold[key + "cells"][r], gold[key + "cells"][0])


def test_centroid_pressure_at_one_bead_is_the_pressure(gold):
    """at P = 1 the centroid pressure is the reference's compute_pressure of the same state (system.py:583-614)"""
    rng = np.random.default_rng(3)
    n_atoms = gold["n_atoms"]
    n = int(n_atoms.sum())
    m = gold["P1:masses"]
    p = torch.as_tensor(rng.normal(size=(1, n, 3)))
    cells = torch.as_tensor(np.repeat(gold["cells"][None], 1, axis=0))
    stress = torch.as_tensor(rng.normal(size=(1, 3, 3, 3)))
    s = RO._Systems(m, n_atoms)
    vol = RNO.volumes(cells)[0]
    ke = 0.5 * s.sum_atoms(torch.sum(p ** 2, dim=2, keepdim=True) / s.masses)[0, :, 0]
    ref = torch.einsum("bii->b", -stress[0]) / 3.0 + 2.0 * ke / vol / 3.0
    _close(RNO.centroid_pressure(p, m, n_atoms, cells, stress, kinetic_component=True).numpy(), ref.numpy(), 1e-14)
    kt = 0.5 * torch.stack([torch.einsum("ni,nj->ij", p[0, s.index_m == b], p[0, s.index_m == b] /
                                         s.masses[0, s.index_m == b]) for b in range(len(n_atoms))])
    _close(RNO.centroid_pressure(p, m, n_atoms, cells, stress, tensor=True, kinetic_component=True).numpy(),
           (-stress[0] + 2.0 * kt / vol[:, None, None]).numpy(), 1e-14)


def test_barostat_noise_restatement_is_normal_zero_of_the_langevin_draw():
    """system s of cell application ``app`` takes the x-normal of the Philox draw (seed; s, app), the bits that
    LangevinThermostat draws for atom s"""
    noise = RNO.philox_cell_noise(21)
    z = noise(4, (5000,)).numpy()
    assert np.array_equal(z, NO.langevin_normals(21, 4, 5000)[:, 0])
    assert abs(z.mean()) < 5.0 / np.sqrt(z.size) and abs(z.std() - 1.0) < 0.05
    z2 = noise(5, (5000,)).numpy()
    assert abs(np.corrcoef(z, z2)[0, 1]) < 5.0 / np.sqrt(z.size)


def test_pile_barostat_combinations_on_the_host():
    from schnetpack_b200 import md

    rp = md.RingPolymer(4, 300.0)
    check = md.DeviceMD._check_ring_polymer
    baro = md.PILEBarostat(1000.0, 300.0, 500.0)
    assert baro.ring_polymer and not baro.temperature_control
    for th in (md.PILELocalThermostat(300.0, 100.0), md.PILEGlobalThermostat(300.0, 100.0),
               md.TRPMDThermostat(300.0, 0.5), md.NHCRingPolymerThermostat(300.0, 100.0),
               md.NHCRingPolymerThermostat(300.0, 100.0, local=False), None):
        check(rp, th, baro, False)                                          # accepted
    with pytest.raises(ValueError, match="ring-polymer barostat"):
        check(None, None, baro, False)
    for cls in (md.NHCBarostatIsotropic, md.NHCBarostatAnisotropic):
        with pytest.raises(ValueError, match="barostat"):
            check(rp, None, cls(1.0, 300.0, 100.0), False)
    with pytest.raises(ValueError, match="compute_stress"):
        check(rp, None, baro, True)
    with pytest.raises(ValueError, match="classical thermostat"):
        check(rp, md.LangevinThermostat(300.0, 100.0), baro, False)
    with pytest.raises(ValueError):
        baro.bind(None, 1e-3)                                               # no ring polymer to bind to
    sd = md.PILEBarostat(1.0, 300.0, 500.0, bar=2.0)
    assert sd.target_pressure == 2.0 and abs(sd.time_constant - 500.0 * md.FS_MD) < 1e-18
