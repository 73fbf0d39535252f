"""Thermostats of the device MD step (csrc/thermostat.cu, schnetpack_b200.md) against the fp64 oracle tests/nvt_oracle.py,
which is pinned to the reference's own thermostats (tests/test_nvt_oracle.py)."""
import math

import numpy as np
import pytest
import torch

import nvt_oracle as NO
from conftest import load_case, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# Units in which the thermostat parameters are exact binary fractions, so the oracle's float32 parameter buffers (as in
# the reference) and the library's fp64 ones hold the same values: tau = 128 fs = 1/8, kB T = 300/128, dt = tau / 16.
EXACT = dict(kB=2.0 ** -7, fs=2.0 ** -10)
T_EXACT, TAU_EXACT, DT_EXACT = 300.0, 128.0, 2.0 ** -7


def _np(t):
    return t.detach().cpu().numpy()


def _mixed_batch(seed=3):
    """a 1-atom system, small molecules and one 20 000-atom system (79 CTAs of the partial pass), near 300 K"""
    n_atoms = [1, 3, 9, 20_000, 20, 1, 5]
    rng = np.random.default_rng(seed)
    n = sum(n_atoms)
    masses = rng.choice([1.008, 12.011, 15.999], size=n).astype(np.float32)
    t_sys = np.repeat(rng.uniform(100.0, 600.0, len(n_atoms)), n_atoms)
    p = (rng.normal(size=(n, 3)) * np.sqrt(masses * EXACT["kB"] * t_sys)[:, None]).astype(np.float32)
    return n_atoms, masses, p


def _systems(n_atoms, masses):
    from schnetpack_b200.md import _Systems

    idx_m = torch.repeat_interleave(torch.arange(len(n_atoms)), torch.tensor(n_atoms)).to(DEV)
    return _Systems(torch.as_tensor(masses, device=DEV), idx_m, len(n_atoms))


def test_kinetic_energy_is_fp64_and_bitwise_reproducible():
    n_atoms, masses, p = _mixed_batch()
    sy = _systems(n_atoms, masses)
    pt = torch.as_tensor(p, device=DEV)
    ke1, t1 = sy.kinetic_energy_and_temperature(pt, EXACT["kB"])
    ke2, t2 = sy.kinetic_energy_and_temperature(pt, EXACT["kB"])
    torch.cuda.synchronize()
    assert torch.equal(ke1, ke2) and torch.equal(t1, t2)
    ref = NO._System(masses.astype(np.float64), n_atoms)
    p64 = torch.as_tensor(p.astype(np.float64))[None]
    ke_ref = ref.kinetic_energy(p64).reshape(-1).numpy()
    assert rel_err(_np(ke1), ke_ref) < 1e-12
    assert rel_err(_np(t1), 2.0 * ke_ref / (3.0 * np.asarray(n_atoms) * EXACT["kB"])) < 1e-12
    # the reference forms 3 n kB in float32 (system.py:416-420), hence 1e-6 against its formula
    assert rel_err(_np(t1), ref.temperature(p64, EXACT["kB"]).reshape(-1).numpy()) < 1e-6


@pytest.mark.parametrize("kind,kw", [("berendsen", {}), ("nhc", dict(massive=False)),
                                     ("nhc", dict(massive=True)),
                                     ("nhc", dict(massive=False, integration_order=7, chain_length=4, multi_step=1))])
def test_thermostat_kernels_follow_the_oracle(kind, kw):
    from schnetpack_b200 import md

    n_atoms, masses, p = _mixed_batch()
    sy = _systems(n_atoms, masses)
    if kind == "berendsen":
        dev_th, ref_th = md.BerendsenThermostat(T_EXACT, TAU_EXACT, **EXACT), NO.Berendsen(T_EXACT, TAU_EXACT, **EXACT)
    else:
        dev_th = md.NHCThermostat(T_EXACT, TAU_EXACT, **kw, **EXACT)
        ref_th = NO.NHC(T_EXACT, TAU_EXACT, EXACT["kB"], EXACT["fs"], **kw)
    dev_th.bind(sy, DT_EXACT)
    ref_th.init(masses.astype(np.float64), n_atoms, DT_EXACT)
    pt = torch.as_tensor(p, device=DEV)
    pr = torch.as_tensor(p.astype(np.float64))
    for _ in range(6):
        dev_th.apply(pt)
        pr = ref_th.apply(pr)
    torch.cuda.synchronize()
    assert rel_err(_np(pt), pr.numpy()) < 1e-6
    assert np.abs(pr.numpy() - p).max() > 1e-2 * np.abs(p).max()        # the thermostat acted
    if kind == "nhc":
        v, f, m = ref_th.chain_state()
        assert rel_err(_np(dev_th.masses), m) < 1e-12
        assert rel_err(_np(dev_th.velocities), v) < 1e-6
        assert rel_err(_np(dev_th.forces), f) < 1e-6


def _philox_device(seed, app, n):
    from schnetpack_b200 import _lib, ops

    ctr = torch.tensor([app, 0], dtype=torch.int64, device=DEV)
    out = torch.empty(n, 4, dtype=torch.int32, device=DEV)
    _lib.call("spk_philox4x32_10", seed, ops._p(ctr), n, ops._p(out), ops._stream())
    torch.cuda.synchronize()
    return _np(out).view(np.uint32)


def test_philox_bits_equal_the_numpy_restatement():
    for seed, app in ((0, 0), (0x1234_5678_9ABC_DEF0, 7), (2 ** 64 - 1, 2 ** 33 + 5)):
        assert (_philox_device(seed, app, 100_003) == NO.philox_bits(seed, app, 100_003)).all()


def _langevin_unit(n, seed, counter):
    """p = 0, m = 1, kB T = 1, c1 = 0, c2 = 1: the kernel writes its standard normals into p"""
    from schnetpack_b200 import _lib, ops

    p = torch.zeros(n, 3, device=DEV)
    m = torch.ones(n, device=DEV)
    _lib.call("spk_md_langevin", ops._p(p), ops._p(m), n, 0.0, 1.0, 1.0, seed, ops._p(counter), ops._stream())
    return p


def test_langevin_noise_is_standard_normal_and_matches_the_restatement():
    from scipy import stats

    n, seed = 400_000, 2024                                                   # 1.2e6 degrees of freedom
    counter = torch.tensor([3, 0], dtype=torch.int64, device=DEV)
    z = _langevin_unit(n, seed, counter)
    torch.cuda.synchronize()
    assert counter.tolist() == [4, 0]                                         # advanced once, ticket back to 0
    z = _np(z).astype(np.float64)
    assert np.abs(z - NO.langevin_normals(seed, 3, n)).max() < 1e-6
    x = z.reshape(-1)
    N = x.size
    assert abs(x.mean()) < 5.0 / math.sqrt(N)
    assert abs(x.var() - 1.0) < 5.0 * math.sqrt(2.0 / N)
    assert stats.kstest(x, "norm").pvalue > 1e-3


def test_langevin_graph_replays_draw_fresh_noise():
    n, seed = 200_000, 5
    counter = torch.zeros(2, dtype=torch.int64, device=DEV)
    p = torch.zeros(n, 3, device=DEV)
    m = torch.ones(n, device=DEV)
    from schnetpack_b200 import _lib, ops

    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        p.zero_()
        _lib.call("spk_md_langevin", ops._p(p), ops._p(m), n, 0.0, 1.0, 1.0, seed, ops._p(counter), ops._stream())
    draws = []
    for _ in range(3):
        g.replay()
        torch.cuda.synchronize()
        draws.append(_np(p).astype(np.float64))
    assert counter.tolist() == [3, 0]
    for k, z in enumerate(draws):
        assert np.abs(z - NO.langevin_normals(seed, k, n)).max() < 1e-6
    c = np.corrcoef(draws[0].reshape(-1), draws[1].reshape(-1))[0, 1]
    assert abs(c) < 5.0 / math.sqrt(3 * n), c


# ---- DeviceMD with thermostats --------------------------------------------------------------------------------------------
THERMOSTATS = {
    "berendsen": (lambda md: md.BerendsenThermostat(5.0, 20.0), lambda: NO.Berendsen(5.0, 20.0, *_units())),
    "langevin": (lambda md: md.LangevinThermostat(5.0, 20.0, seed=17), lambda: NO.Langevin(5.0, 20.0, *_units(), seed=17)),
    "nhc": (lambda md: md.NHCThermostat(5.0, 20.0), lambda: NO.NHC(5.0, 20.0, *_units())),
    "nhc_massive": (lambda md: md.NHCThermostat(5.0, 20.0, massive=True, integration_order=5),
                    lambda: NO.NHC(5.0, 20.0, *_units(), massive=True, integration_order=5)),
}


def _units():
    from schnetpack_b200.md import FS_MD, KB_MD

    return KB_MD, FS_MD


def _box_md(thermostat, p_conv=1.0, e_conv=1.0, use_graph=True):
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.md import DeviceMD
    from schnetpack_b200.model import batch_to_device, from_spec

    spec = S.model_spec("painn", n_atom_basis=128, n_interactions=2)
    data = S.periodic_box(150, seed=9)
    params = S.init_params(spec, seed=8)
    dev = torch.device(DEV)
    model = from_spec(spec, params, dev)
    N = data["_positions"].shape[0]
    masses = np.where(data["_atomic_numbers"] == 8, 16.0, 1.0)
    p0 = np.random.default_rng(2).normal(0, 0.05, (N, 3))
    md = DeviceMD(model, batch_to_device(data, dev), torch.as_tensor(masses), time_step=1e-3, cutoff=spec["cutoff"],
                  capacity=int(data["_idx_i"].shape[0] * 1.5), momenta=torch.as_tensor(p0), use_graph=use_graph,
                  position_conversion=p_conv, energy_conversion=e_conv, thermostat=thermostat)
    return md, (spec, params, data, masses, p0)


@pytest.mark.parametrize("name", sorted(THERMOSTATS))
@pytest.mark.parametrize("p_conv,e_conv", [(1.0, 1.0), (10.0, 0.5)])
def test_device_md_follows_the_reference_nvt_loop(name, p_conv, e_conv):
    """12 steps of the 150-atom periodic box with each thermostat against nvt_trajectory (same cases and tolerances as the
    NVE test in test_cuda_neighbors.py); the Langevin oracle regenerates the device's normals."""
    from schnetpack_b200 import md as M

    make_dev, make_ref = THERMOSTATS[name]
    md, (spec, params, data, masses, p0) = _box_md(make_dev(M), p_conv, e_conv)
    n_steps = 12
    md.run(n_steps)
    torch.cuda.synchronize()
    x_ref, p_ref, e_ref, f_ref = NO.nvt_trajectory(spec, params, data, masses, p0, 1e-3, n_steps, make_ref(), p_conv,
                                                   e_conv)
    assert rel_err(_np(md.positions), x_ref) < 1e-6
    assert rel_err(_np(md.momenta), p_ref) < 1e-4
    assert rel_err(_np(md.potential_energy()), e_ref) < 1e-5
    assert rel_err(_np(md.forces) * (e_conv / p_conv), f_ref) < 1e-4
    # the thermostat changed the trajectory: NVE from the same start ends elsewhere
    from oracle import md_oracle as MO

    _, p_nve, _, _ = MO.nve_trajectory(spec, params, data, masses, p0, 1e-3, n_steps, p_conv, e_conv)
    assert rel_err(p_nve, p_ref) > 1e-3


@pytest.mark.parametrize("name", sorted(THERMOSTATS))
def test_graph_replay_equals_eager_and_restart_is_bitwise(name):
    from schnetpack_b200 import md as M

    make_dev = THERMOSTATS[name][0]
    runs = {}
    for use_graph in (True, False):
        md, _ = _box_md(make_dev(M), use_graph=use_graph)
        md.run(10)
        torch.cuda.synchronize()
        runs[use_graph] = (_np(md.positions), _np(md.momenta), md.thermostat.state_dict())
    assert rel_err(runs[True][0], runs[False][0]) < 1e-6
    assert rel_err(runs[True][1], runs[False][1]) < 1e-5
    if name == "langevin":
        assert runs[True][2]["counter"].tolist() == runs[False][2]["counter"].tolist() == [20, 0]

    # one run of 8 steps against 4 + save + restore into a fresh DeviceMD + 4 (both graph replays)
    a, _ = _box_md(make_dev(M))
    a.run(4)
    saved = a.state_dict()
    a.run(4)
    b, _ = _box_md(make_dev(M))
    b.load_state_dict(saved)
    b.run(4)
    torch.cuda.synchronize()
    assert b.steps_done == a.steps_done == 8
    assert torch.equal(a.positions, b.positions) and torch.equal(a.momenta, b.momenta)
    assert torch.equal(a.forces, b.forces) and torch.equal(a.energy, b.energy)
    for k, v in a.thermostat.state_dict().items():
        assert torch.equal(v, b.thermostat.state_dict()[k]), k


# ---- physics: a batch of ethanol molecules brought to 300 K from rest -------------------------------------------------------
MASS = {1: 1.008, 6: 12.011, 8: 15.999}


def _ethanol_batch(copies):
    spec, params, inputs, _, _ = load_case("painn_md_ethanol_trained")
    n_mol = inputs["_n_atoms"].shape[0]
    n = inputs["_positions"].shape[0]
    b = {"_positions": np.tile(inputs["_positions"], (copies, 1)),
         "_atomic_numbers": np.tile(inputs["_atomic_numbers"], copies),
         "_n_atoms": np.tile(inputs["_n_atoms"], copies),
         "_idx_m": (np.tile(inputs["_idx_m"], copies) + np.repeat(np.arange(copies) * n_mol, n)).astype(np.int64),
         "_cell": np.tile(inputs["_cell"], (copies, 1, 1)),
         "_pbc": np.tile(inputs["_pbc"].reshape(n_mol, 3), (copies, 1)).reshape(-1)}
    return spec, params, b


@pytest.mark.parametrize("name", ["langevin", "nhc"])
def test_thermostat_brings_ethanol_batch_to_300K(name):
    """256 ethanol molecules (trained PaiNN, kcal/mol and Angstrom; MD in kJ/mol, nm, Da) start at rest.  The batch
    temperature over N = 2304 atoms fluctuates by sigma = 300 K * sqrt(2 / (3 N)) = 5.1 K at equilibrium.  With dt = 0.5 fs
    and tau = 50 fs, 6000 steps (3 ps = 60 tau) are run and the mean of the second half (sampled every 10 steps) must lie
    within 5 sigma of 300 K."""
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params, b = _ethanol_batch(128)
    dev = torch.device(DEV)
    model = from_spec(spec, params, dev)
    masses = torch.tensor([MASS[int(z)] for z in b["_atomic_numbers"]])
    th = M.LangevinThermostat(300.0, 50.0, seed=1) if name == "langevin" else M.NHCThermostat(300.0, 50.0)
    n_atoms = masses.shape[0]
    assert b["_n_atoms"].shape[0] == 256 and n_atoms == 2304
    md = M.DeviceMD(model, batch_to_device(b, dev), masses, time_step=0.5 * M.FS_MD, cutoff=spec["cutoff"],
                    capacity=int(b["_n_atoms"].shape[0] * 9 * 8 * 1.5), position_conversion=10.0, energy_conversion=4.184,
                    thermostat=th)
    assert float(md.temperature().max()) == 0.0
    md.run(3000)
    samples = []
    for _ in range(300):
        md.run(10)
        t = md.temperature()                                           # per molecule; all have 9 atoms
        samples.append(float(t.mean()))
    sigma = 300.0 * math.sqrt(2.0 / (3.0 * n_atoms))
    mean = float(np.mean(samples))
    assert abs(mean - 300.0) < 5.0 * sigma, (mean, sigma)
    assert np.isfinite(_np(md.positions)).all()
