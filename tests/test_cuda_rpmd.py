"""Ring-polymer MD on the device (csrc/rpmd.cu, schnetpack_b200.md.RingPolymer and the ring-polymer thermostats) against the
fp64 oracle tests/rpmd_oracle.py, which is pinned to the reference's own ring-polymer MD (tests/test_rpmd_oracle.py)."""
import math

import numpy as np
import pytest
import torch

import nvt_oracle as NO
import rpmd_oracle as RO
from conftest import load_case, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# exact binary-fraction units, as in the golden fixture: omega_P = 37.5 P; dt = 2^-12 keeps omega_max dt = 0.59 at P = 32
EXACT = dict(kB=2.0 ** -7, fs=2.0 ** -10)
HBAR_EXACT = 2.0 ** -4
T_EXACT, TAU_EXACT, DT_EXACT = 300.0, 64.0, 2.0 ** -12


def _np(t):
    return t.detach().cpu().numpy()


def _mixed_batch(P, seed=3, n_atoms=(1, 3, 9, 20_000, 20, 1, 5)):
    """by default a 1-atom system, small molecules and one 20 000-atom system, with bead positions and momenta near 300 K.
    Positions stay near the origin: the fp32 state resolves them to ~1e-8 there, which the stiff high modes (omega_k m up
    to 4e4) turn into momentum errors"""
    n_atoms = [int(n) for n in n_atoms]
    rng = np.random.default_rng(seed + P)
    n = sum(n_atoms)
    masses = rng.choice([1.0, 12.0, 16.0], size=n).astype(np.float32)
    x = (0.1 * rng.normal(size=(n, 3))[None] + 0.01 * rng.normal(size=(P, n, 3))).astype(np.float32)
    p = (rng.normal(size=(P, n, 3)) * np.sqrt(masses * EXACT["kB"] * 300.0 * P)[None, :, None]).astype(np.float32)
    return n_atoms, masses, x, p


def _bind(P, n_atoms, masses):
    from schnetpack_b200 import md

    idx_m = torch.repeat_interleave(torch.arange(len(n_atoms)), torch.tensor(n_atoms)).to(DEV)
    base = md._Systems(torch.as_tensor(masses, device=DEV), idx_m, len(n_atoms))
    rp = md.RingPolymer(P, T_EXACT, kB=EXACT["kB"], hbar=HBAR_EXACT)
    rp.bind(base, DT_EXACT)
    return base, rp


def _rp_oracle(P):
    return RO.RingPolymer(P, T_EXACT, DT_EXACT, EXACT["kB"], HBAR_EXACT)


# ---- 1. the normal-mode transform ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [1, 2, 3, 4, 5, 8, 16, 31, 64])
def test_normal_modes_match_numpy_and_round_trip(P):
    from schnetpack_b200 import md

    rng = np.random.default_rng(P)
    x = rng.normal(size=(P, 1001, 3)).astype(np.float32)
    rp = md.RingPolymer(P, 300.0)
    rp.c_transform = rp.transform_matrix().to(DEV)
    xt = torch.as_tensor(x, device=DEV)
    modes = rp.normal_modes(xt)
    back = rp.normal_modes(modes, inverse=True)
    torch.cuda.synchronize()
    c = RO.transform_matrix(P).numpy()
    ref = (c @ x.reshape(P, -1).astype(np.float64)).reshape(x.shape)
    assert rel_err(_np(modes), ref) < 1e-6
    assert rel_err(_np(back), x) < 1e-6


@pytest.mark.parametrize("P", [0, 65])
def test_normal_modes_refuse_bead_counts_out_of_range(P):
    from schnetpack_b200 import _lib, ops

    x = torch.zeros(max(P, 1), 10, 3, device=DEV)
    c = torch.zeros(max(P, 1), max(P, 1), dtype=torch.float64, device=DEV)
    with pytest.raises(ValueError):
        _lib.call("spk_rpmd_normal_modes", ops._p(x), ops._p(x), 10, P, ops._p(c), 0, ops._stream())


# ---- 2. kernels against the oracle ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [1, 5, 8, 32])
def test_main_step_follows_the_oracle(P):
    n_atoms, masses, x, p = _mixed_batch(P)
    base, rp = _bind(P, n_atoms, masses)
    xt, pt = torch.as_tensor(x, device=DEV), torch.as_tensor(p, device=DEV)
    model_x = torch.empty_like(xt)
    for _ in range(3):
        rp.main_step(xt, pt, model_x, 10.0)
    torch.cuda.synchronize()
    ro = _rp_oracle(P)
    xr, pr = torch.as_tensor(x, dtype=torch.float64), torch.as_tensor(p, dtype=torch.float64)
    for _ in range(3):
        xr, pr = ro.main_step(xr, pr, masses.astype(np.float64))
    assert rel_err(_np(xt), xr.numpy()) < 1e-6
    assert rel_err(_np(pt), pr.numpy()) < 1e-5
    assert torch.equal(model_x, xt * 10.0)
    assert np.abs(xr.numpy() - x).max() > 1e-3                                # the ring polymer moved


def _thermostats(md, seed=11):
    T, tau = T_EXACT, TAU_EXACT
    return {
        "pile_l": (md.PILELocalThermostat(T, tau, seed=seed, **EXACT),
                   RO.PILE(T, tau, *EXACT.values(), RO.philox_noise(seed))),
        "pile_g": (md.PILEGlobalThermostat(T, tau, seed=seed, **EXACT),
                   RO.PILE(T, tau, *EXACT.values(), RO.philox_noise(seed), global_=True)),
        "trpmd": (md.TRPMDThermostat(T, 0.5, seed=seed, **EXACT),
                  RO.PILE(T, 1.0, *EXACT.values(), RO.philox_noise(seed), thermostat_centroid=False, damping_factor=0.5)),
        "nhc_local": (md.NHCRingPolymerThermostat(T, tau, **EXACT), RO.NHCRingPolymer(T, tau, *EXACT.values())),
        "nhc_global": (md.NHCRingPolymerThermostat(T, tau, local=False, chain_length=4, integration_order=5, **EXACT),
                       RO.NHCRingPolymer(T, tau, *EXACT.values(), local=False, chain_length=4, integration_order=5)),
    }


@pytest.mark.parametrize("name", ["pile_l", "pile_g", "trpmd", "nhc_local", "nhc_global"])
@pytest.mark.parametrize("P", [1, 5, 8, 32])
def test_thermostat_kernels_follow_the_oracle(P, name):
    from schnetpack_b200 import md

    n_atoms, masses, x, p = _mixed_batch(P)
    base, rp = _bind(P, n_atoms, masses)
    ro = _rp_oracle(P)

    def run(p, n_apply):
        dev_th, ref_th = _thermostats(md)[name]
        dev_th.bind(base, DT_EXACT, rp)
        ref_th.init(ro, masses.astype(np.float64), n_atoms)
        pt = torch.as_tensor(p, device=DEV).reshape(-1, 3)
        pr = torch.as_tensor(p, dtype=torch.float64)
        for _ in range(n_apply):
            dev_th.apply(pt)
            pr = ref_th.apply(pr)
        torch.cuda.synchronize()
        got = _np(pt).reshape(p.shape)
        assert np.isfinite(got).all()
        assert rel_err(got, pr.numpy()) < 1e-5
        return got, pr.numpy(), dev_th, ref_th

    got, ref, dev_th, ref_th = run(p, 4)
    acted = np.abs(ref - p).max() / np.abs(p).max()
    if name == "trpmd" and P == 1:
        assert acted == 0.0                                                    # TRPMD leaves a single bead alone
    else:
        assert acted > (1e-6 if name.startswith("nhc") else 1e-2)              # the thermostat acted
    if name.startswith("pile"):
        assert dev_th.counter.tolist() == [4, 0]
    if name == "trpmd":                                                        # the centroid passes through
        assert rel_err(got.mean(0), p.mean(0)) < 1e-6
    if name == "pile_g":
        # a system whose centroid is at rest keeps it (the reference would write NaN); one application, since the fp32
        # round trip leaves a centroid of rounding size that the next application rescales like any other
        zero = slice(sum(n_atoms[:5]), sum(n_atoms[:6]))
        p0 = p.copy()
        p0[:, zero] = 0.0
        got0, _, _, _ = run(p0, 1)
        assert np.abs(got0[:, zero].mean(0)).max() < 1e-6 * np.abs(p).max()
    if name.startswith("nhc"):
        v, f, m = ref_th.chain_state()
        assert rel_err(_np(dev_th.masses), m) < 1e-12
        assert rel_err(_np(dev_th.velocities), v) < 1e-6
        assert rel_err(_np(dev_th.forces), f) < 1e-6


# ---- 3. noise ---------------------------------------------------------------------------------------------------------------
def test_pile_noise_bits_equal_the_restatement_and_replays_draw_fresh_noise():
    """c1 = 0, c2 = 1, m = 1, P kB T = 1 and p = 0: the kernel writes C^T xi into the beads"""
    from schnetpack_b200 import _lib, md, ops

    P, n, seed = 8, 50_000, 123
    rp = md.RingPolymer(P, 300.0)
    rp.c_transform = rp.transform_matrix().to(DEV)
    p = torch.zeros(P * n, 3, device=DEV)
    m = torch.ones(n, device=DEV)
    c1 = torch.zeros(P, dtype=torch.float64, device=DEV)
    c2 = torch.ones(P, dtype=torch.float64, device=DEV)
    counter = torch.tensor([5, 0], dtype=torch.int64, device=DEV)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        p.zero_()
        _lib.call("spk_rpmd_pile", ops._p(p), ops._p(m), None, None, n, 1, P, ops._p(rp.c_transform), ops._p(c1),
                  ops._p(c2), 1.0, 0, seed, ops._p(counter), None, 0, ops._stream())
    c = RO.transform_matrix(P).numpy()
    draws = []
    for k in range(3):
        g.replay()
        torch.cuda.synchronize()
        xi = (c @ _np(p).astype(np.float64).reshape(P, -1)).reshape(P, n, 3)
        assert np.abs(xi - NO.langevin_normals(seed, 5 + k, P * n).reshape(P, n, 3)).max() < 1e-5
        draws.append(xi)
    assert counter.tolist() == [8, 0]
    corr = np.corrcoef(draws[0].reshape(-1), draws[1].reshape(-1))[0, 1]
    assert abs(corr) < 5.0 / math.sqrt(draws[0].size)
    # mode 0 draws exactly the Langevin thermostat's normals
    assert np.abs(draws[0][0] - NO.langevin_normals(seed, 5, n)).max() < 1e-5


# ---- 4-6. DeviceMD trajectories -------------------------------------------------------------------------------------------
def _box_case():
    from schnetpack_b200 import synthetic as S

    spec = S.model_spec("painn", n_atom_basis=128, n_interactions=2)
    data = S.periodic_box(150, seed=9)
    params = S.init_params(spec, seed=8)
    masses = np.where(data["_atomic_numbers"] == 8, 16.0, 1.0)
    return spec, params, data, masses, 1e-3


MASS = {1: 1.008, 6: 12.011, 8: 15.999}


def _ethanol_case():
    spec, params, inputs, _, _ = load_case("painn_md_ethanol_trained")
    data = {k: inputs[k] for k in ("_positions", "_atomic_numbers", "_n_atoms", "_idx_m", "_cell", "_pbc")}
    masses = np.array([MASS[int(z)] for z in data["_atomic_numbers"]])
    return spec, params, data, masses, 0.25e-3


def _device_md(case, P, thermostat, p_conv=1.0, e_conv=1.0, use_graph=True, momenta=None, cap_per_atom=80):
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params, data, masses, dt = case
    N = data["_positions"].shape[0]
    if momenta is None:                                           # every bead at 300 K P (system.py:407-421)
        momenta = np.random.default_rng(2).normal(size=(P, N, 3)) * np.sqrt(masses * M.KB_MD * 300.0 * P)[None, :, None]
    model = from_spec(spec, params, torch.device(DEV))
    rp = None if P is None else M.RingPolymer(P, 300.0)
    md = M.DeviceMD(model, batch_to_device(data, torch.device(DEV)), torch.as_tensor(masses), time_step=dt,
                    cutoff=spec["cutoff"], capacity=int(N * (P or 1) * cap_per_atom), momenta=torch.as_tensor(momenta),
                    use_graph=use_graph, position_conversion=p_conv, energy_conversion=e_conv, thermostat=thermostat,
                    ring_polymer=rp)
    return md, momenta


def _oracle_forces(case, p_conv, e_conv):
    """forces [P, N, 3] (MD units) on every bead of every system from the fp64 model oracle"""
    from oracle import nl_oracle as NL
    from oracle import spk_oracle as O

    spec, params, data, _, _ = case
    n_atoms = np.asarray(data["_n_atoms"])
    starts = np.concatenate([[0], np.cumsum(n_atoms)])
    cells = np.asarray(data["_cell"], dtype=np.float64).reshape(-1, 3, 3)
    pbcs = np.asarray(data["_pbc"]).reshape(-1, 3)

    def forces(x_md):
        f = torch.zeros_like(x_md)
        for r in range(x_md.shape[0]):
            for m in range(len(n_atoms)):
                a0, a1 = starts[m], starts[m + 1]
                R = (x_md[r, a0:a1] * p_conv).numpy()
                cell, pbc = cells[m if cells.shape[0] > 1 else 0], pbcs[m if pbcs.shape[0] > 1 else 0]
                ii, jj, _, off = NL.neighbor_list(R, cell, pbc, spec["cutoff"])
                b = {"_positions": R, "_atomic_numbers": data["_atomic_numbers"][a0:a1],
                     "_n_atoms": np.array([a1 - a0]), "_idx_m": np.zeros(a1 - a0, dtype=np.int64),
                     "_cell": cell[None], "_pbc": pbc, "_idx_i": ii, "_idx_j": jj, "_offsets": off}
                f[r, a0:a1] = O.energy_forces(spec, params, b, dtype=torch.float64)["forces"] * (e_conv / p_conv)
        return f

    return forces


TRAJ_THERMOSTATS = ["none", "pile_l", "pile_g", "trpmd", "nhc_local", "nhc_global"]


def _traj_thermostat(name, seed=17):
    from schnetpack_b200 import md as M
    from schnetpack_b200.md import FS_MD, KB_MD

    u = (KB_MD, FS_MD)
    return {"none": (None, None),
            "pile_l": (M.PILELocalThermostat(300.0, 20.0, seed=seed), RO.PILE(300.0, 20.0, *u, RO.philox_noise(seed))),
            "pile_g": (M.PILEGlobalThermostat(300.0, 20.0, seed=seed),
                       RO.PILE(300.0, 20.0, *u, RO.philox_noise(seed), global_=True)),
            "trpmd": (M.TRPMDThermostat(300.0, 0.5, seed=seed),
                      RO.PILE(300.0, 1.0, *u, RO.philox_noise(seed), thermostat_centroid=False, damping_factor=0.5)),
            "nhc_local": (M.NHCRingPolymerThermostat(300.0, 20.0), RO.NHCRingPolymer(300.0, 20.0, *u)),
            "nhc_global": (M.NHCRingPolymerThermostat(300.0, 20.0, local=False),
                           RO.NHCRingPolymer(300.0, 20.0, *u, local=False))}[name]


@pytest.mark.parametrize("name", TRAJ_THERMOSTATS)
@pytest.mark.parametrize("system,P,p_conv,e_conv", [("box", 4, 10.0, 0.5), ("ethanol", 5, 1.0, 1.0),
                                                    ("ethanol", 5, 10.0, 4.184)])
def test_device_md_follows_the_oracle_rpmd_loop(name, system, P, p_conv, e_conv):
    """12 RPMD steps from 300 K bead momenta of the 150-atom periodic box (P = 4) and of the two trained ethanol molecules
    (P = 5; in model units, and in MD units kJ/mol, nm, Da against the model's kcal/mol and Angstrom) against
    rpmd_trajectory with the oracle's forces.  Momenta to 2e-4: the thermal bead momenta excite the stiff high modes, whose
    springs turn the fp32 rounding of positions and forces into momentum errors of ~1e-4 over 12 steps"""
    from schnetpack_b200.md import HBAR_MD, KB_MD

    case = _box_case() if system == "box" else _ethanol_case()
    dev_th, ref_th = _traj_thermostat(name)
    md, p0 = _device_md(case, P, dev_th, p_conv, e_conv)
    n_steps = 12
    md.run(n_steps)
    torch.cuda.synchronize()
    _, _, data, masses, dt = case
    x0 = np.repeat(np.asarray(data["_positions"], dtype=np.float64)[None] / p_conv, P, axis=0)
    ro = RO.RingPolymer(P, 300.0, dt, KB_MD, HBAR_MD)
    xr, pr = RO.rpmd_trajectory(ro, x0, p0, masses, data["_n_atoms"], _oracle_forces(case, p_conv, e_conv), n_steps,
                                ref_th)
    assert rel_err(_np(md.positions).reshape(P, -1, 3), xr.numpy()) < 1e-6
    assert rel_err(_np(md.momenta).reshape(P, -1, 3), pr.numpy()) < 2e-4
    assert md.energy.shape[0] == P * len(data["_n_atoms"])


def test_one_bead_reproduces_nve_and_pile_reproduces_langevin():
    from schnetpack_b200 import md as M

    case = _box_case()
    N = case[2]["_positions"].shape[0]
    p0 = np.random.default_rng(4).normal(0, 0.05, (N, 3)) * np.sqrt(case[3])[:, None]
    for classical, ring in ((None, None), (M.LangevinThermostat(300.0, 20.0, seed=9),
                                           M.PILELocalThermostat(300.0, 20.0, seed=9))):
        a, _ = _device_md(case, None, classical, momenta=p0)
        b, _ = _device_md(case, 1, ring, momenta=p0)
        a.run(12)
        b.run(12)
        torch.cuda.synchronize()
        ex, ep = rel_err(_np(b.positions), _np(a.positions)), rel_err(_np(b.momenta), _np(a.momenta))
        print(f"P = 1 against {'NVE' if classical is None else 'Langevin'}: positions {ex:.2e}, momenta {ep:.2e}")
        assert ex <= 1e-6 and ep <= 1e-6, (ex, ep)
        assert b.temperature().shape == (1, 1)


def test_shared_cell_gives_the_per_system_cell_trajectory():
    """two copies of the periodic box with ONE shared cell / pbc ([1, 3, 3] / [3], which the neighbour list broadcasts)
    follow bitwise the trajectory of the same batch with one cell per system: the bead batch expands the shared cell to
    one row per bead system instead of handing the neighbour list P rows for P B systems"""
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params, data, masses, dt = _box_case()
    n = data["_positions"].shape[0]
    two = {"_positions": np.tile(data["_positions"], (2, 1)), "_atomic_numbers": np.tile(data["_atomic_numbers"], 2),
           "_n_atoms": np.array([n, n]), "_idx_m": np.repeat(np.arange(2), n), "_cell": data["_cell"].reshape(1, 3, 3),
           "_pbc": data["_pbc"].reshape(3)}
    per_system = dict(two, _cell=np.tile(two["_cell"], (2, 1, 1)), _pbc=np.tile(two["_pbc"], 2))
    model = from_spec(spec, params, torch.device(DEV))
    p0 = np.random.default_rng(6).normal(size=(2, 2 * n, 3)) * np.sqrt(np.tile(masses, 2) * M.KB_MD * 600.0)[None, :, None]
    runs = []
    for batch in (two, per_system):
        md = M.DeviceMD(model, batch_to_device(batch, torch.device(DEV)), torch.as_tensor(np.tile(masses, 2)), dt,
                        spec["cutoff"], capacity=2 * 2 * n * 80, momenta=torch.as_tensor(p0),
                        ring_polymer=M.RingPolymer(2, 300.0))
        assert md.static["_cell"].shape == (4, 3, 3)
        md.run(3)
        torch.cuda.synchronize()
        runs.append((md.positions.clone(), md.momenta.clone(), md.energy.clone()))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("name", ["pile_g", "nhc_global"])
def test_graph_replay_equals_eager_and_restart_is_bitwise(name):
    case = _box_case()
    runs = {}
    for use_graph in (True, False):
        md, _ = _device_md(case, 4, _traj_thermostat(name)[0], use_graph=use_graph)
        md.run(10)
        torch.cuda.synchronize()
        runs[use_graph] = (_np(md.positions), _np(md.momenta), md.thermostat.state_dict())
    assert rel_err(runs[True][0], runs[False][0]) < 1e-6
    assert rel_err(runs[True][1], runs[False][1]) < 1e-5
    if name == "pile_g":
        assert runs[True][2]["counter"].tolist() == runs[False][2]["counter"].tolist() == [20, 0]

    a, _ = _device_md(case, 4, _traj_thermostat(name)[0])
    a.run(4)
    saved = a.state_dict()
    a.run(4)
    b, _ = _device_md(case, 4, _traj_thermostat(name)[0])
    b.load_state_dict(saved)
    b.run(4)
    torch.cuda.synchronize()
    assert b.steps_done == a.steps_done == 8
    assert torch.equal(a.positions, b.positions) and torch.equal(a.momenta, b.momenta)
    assert torch.equal(a.forces, b.forces) and torch.equal(a.energy, b.energy)
    for k, v in a.thermostat.state_dict().items():
        assert torch.equal(v, b.thermostat.state_dict()[k]), k


# ---- 7. physics: the free ring polymer --------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["pile_l", "pile_g"])
def test_free_ring_polymer_samples_the_exact_normal_mode_distribution(name):
    """512 non-interacting atoms (the last Atomwise layer is zero, so E = F = 0 while the whole kernel path runs) at 300 K
    with P = 8.  Exact for any P: <p~_k^2> = m P kB T for every mode and <x~_k^2> = P kB T / (m omega_k^2) for k >= 1.
    dt = 1 fs, tau = 20 fs; 1000 steps of equilibration, then 4000 steps sampled every 10.  Every mode's mean (over the
    3 N degrees of freedom, in units of its expectation) must be within 5 standard errors of 1, from 20 block means."""
    from schnetpack_b200 import md as M
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, from_spec

    N, T, P, mass, p_conv = 512, 300.0, 8, 12.0, 10.0
    L = 2.0
    rng = np.random.default_rng(5)
    batch = {"_positions": (rng.uniform(0.0, L, (N, 3)) * p_conv).astype(np.float32),
             "_atomic_numbers": np.full(N, 6, dtype=np.int64), "_n_atoms": np.array([N], dtype=np.int64),
             "_idx_m": np.zeros(N, dtype=np.int64), "_cell": (L * p_conv * np.eye(3, dtype=np.float32))[None],
             "_pbc": np.ones(3, dtype=bool)}
    spec = S.model_spec("painn", n_atom_basis=128, n_interactions=1)
    dev = torch.device(DEV)
    model = from_spec(spec, S.init_params(spec, seed=3), dev)
    last = model.output_modules[0].outnet[1]
    with torch.no_grad():
        last.weight.zero_()
        last.bias.zero_()
    th = M.PILELocalThermostat(T, 20.0, seed=3) if name == "pile_l" else M.PILEGlobalThermostat(T, 20.0, seed=3)
    rp = M.RingPolymer(P, T)
    p0 = rng.normal(size=(N, 3)) * math.sqrt(mass * M.KB_MD * T)     # PILE-G keeps a centroid at rest at rest
    md = M.DeviceMD(model, batch_to_device(batch, dev), torch.full((N,), mass), time_step=1.0 * M.FS_MD,
                    cutoff=spec["cutoff"], capacity=P * N * 80, momenta=torch.as_tensor(p0), position_conversion=p_conv,
                    thermostat=th, ring_polymer=rp)
    md.run(1000)
    pk, xk = [], []
    for _ in range(400):
        md.run(10)
        pn = rp.normal_modes(md.momenta.reshape(P, N, 3))
        xn = rp.normal_modes(md.positions.reshape(P, N, 3))
        pk.append(_np((pn.double() ** 2).mean(dim=(1, 2))))
        xk.append(_np((xn.double() ** 2).mean(dim=(1, 2))))
    assert float(md.forces.abs().max()) == 0.0
    kbt = M.KB_MD * T
    p_exp = mass * P * kbt
    w = rp.omega_normal.numpy()
    x_exp = P * kbt / (mass * w[1:] ** 2)
    mp, sp = RO.block_mean(np.asarray(pk) / p_exp)
    mx, sx = RO.block_mean(np.asarray(xk)[:, 1:] / x_exp)
    assert (np.abs(mp - 1.0) < 5.0 * sp).all() and (sp < 0.05).all(), (mp, sp)
    assert (np.abs(mx - 1.0) < 5.0 * sx).all() and (sx < 0.05).all(), (mx, sx)


# ---- 8. physics: trained ethanol ----------------------------------------------------------------------------------------------
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


def test_trained_ethanol_conserves_the_ring_polymer_hamiltonian_and_pile_reaches_300K():
    """32 trained ethanol molecules, P = 8, with the MD in the model's units (kcal/mol, Angstrom, Da; kB, fs and hbar
    restated from the package's kJ/mol, nm, Da constants), so that position_conversion = energy_conversion = 1.

    NVE from 300 K momenta, dt = 0.25 fs, 3000 steps sampled every 20: the ring-polymer Hamiltonian sum_b [p_b^2 / 2m +
    V(x_b)] + sum_b 1/2 m omega_P^2 |x_b - x_b+1|^2 is fitted with a line; the drift of that line over the run must stay
    below 3 standard deviations of the residuals about it (the fluctuation, measured apart from any trend;
    test_rpmd_oracle.py shows that this check trips on linear or exponential heating of a few fluctuations).

    PILE-L at 300 K (tau = 20 fs, dt = 0.5 fs) from rest: after 2000 steps, 4000 more are sampled every 10.  The mean
    centroid temperature must lie within 5 standard errors of 300 K and the mean bead temperature within 5 standard errors
    of P 300 K, both errors from 20 block means and each below 1 % of its target (so the bound is at most 5 %)."""
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params, b = _ethanol_batch(16)
    dev = torch.device(DEV)
    model = from_spec(spec, params, dev)
    masses = torch.tensor([MASS[int(z)] for z in b["_atomic_numbers"]])
    N, P, T = masses.shape[0], 8, 300.0
    kcal, angstrom = 4.184, 0.1                                     # in kJ/mol and nm
    t_unit = angstrom / math.sqrt(kcal)                             # Angstrom sqrt(Da / (kcal/mol)) in MD time units
    kB, fs, hbar = M.KB_MD / kcal, M.FS_MD / t_unit, M.HBAR_MD / (kcal * t_unit)
    p0 = np.random.default_rng(1).normal(size=(P, N, 3)) * np.sqrt(masses.numpy() * kB * T * P)[None, :, None]
    kw = dict(cutoff=spec["cutoff"], capacity=P * N * 12)

    rp = M.RingPolymer(P, T, kB=kB, hbar=hbar)
    md = M.DeviceMD(model, batch_to_device(b, dev), masses, time_step=0.25 * fs, momenta=torch.as_tensor(p0),
                    ring_polymer=rp, **kw)
    m = md.masses.reshape(P, N, 1).double()
    w2 = rp.omega ** 2

    def hamiltonian():
        x = md.positions.reshape(P, N, 3).double()
        p = md.momenta.reshape(P, N, 3).double()
        spring = 0.5 * (m * w2 * (x - torch.roll(x, -1, 0)) ** 2).sum()
        return float((p ** 2 / (2 * m)).sum() + md.potential_energy().double().sum() + spring)

    t, H = [], []
    for _ in range(150):
        md.run(20)
        t.append(md.steps_done * 0.25)
        H.append(hamiltonian())
    assert np.isfinite(H).all()
    drift, fluct = RO.drift_and_fluctuation(t, H)
    ke = 0.5 * 3 * N * P * kB * T * P                                        # bead kinetic energy at P 300 K
    print(f"ring-polymer Hamiltonian: drift {drift:.3e}, fluctuation {fluct:.3e}, kinetic energy {ke:.3e} kcal/mol")
    assert fluct < 1e-3 * ke, (fluct, ke)                                      # dt is small: H is nearly constant
    assert drift < 3.0 * fluct, (drift, fluct)

    th = M.PILELocalThermostat(T, 20.0, seed=4, kB=kB, fs=fs)
    md = M.DeviceMD(model, batch_to_device(b, dev), masses, time_step=0.5 * fs, thermostat=th,
                    ring_polymer=M.RingPolymer(P, T, kB=kB, hbar=hbar), **kw)
    md.run(2000)
    tc, tb = [], []
    for _ in range(400):
        md.run(10)
        tc.append(float(md.centroid_temperature().mean()))
        tb.append(float(md.temperature().mean()))
    assert md.temperature().shape == (P, b["_n_atoms"].shape[0])
    assert md.centroid_positions().shape == (N, 3) and md.centroid_potential_energy().shape == (b["_n_atoms"].shape[0],)
    mc, sc = RO.block_mean(tc)
    mb, sb = RO.block_mean(tb)
    print(f"PILE-L: centroid {mc:.1f} +- {sc:.1f} K, beads {mb:.1f} +- {sb:.1f} K (P T = {P * T:.0f} K)")
    assert sc < 0.01 * T and sb < 0.01 * P * T, (sc, sb)
    assert abs(mc - T) < 5.0 * sc, (mc, sc)
    assert abs(mb - P * T) < 5.0 * sb, (mb, sb)


# ---- 9. refusals --------------------------------------------------------------------------------------------------------------
def test_device_md_refuses_forbidden_combinations():
    from schnetpack_b200 import md as M

    case = _box_case()
    with pytest.raises(ValueError, match="classical thermostat"):
        _device_md(case, 2, M.LangevinThermostat(300.0, 20.0))
    with pytest.raises(ValueError, match="ring-polymer thermostat"):
        _device_md(case, None, M.PILELocalThermostat(300.0, 20.0), momenta=np.zeros((150, 3)))
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params, data, masses, dt = case
    model = from_spec(spec, params, torch.device(DEV))
    batch = batch_to_device(data, torch.device(DEV))
    with pytest.raises(ValueError, match="barostat"):
        M.DeviceMD(model, batch, torch.as_tensor(masses), dt, spec["cutoff"], 10**6, ring_polymer=M.RingPolymer(2, 300.0),
                   barostat=M.NHCBarostatIsotropic(1.0, 300.0, 100.0))
    with pytest.raises(ValueError, match="compute_stress"):
        M.DeviceMD(model, batch, torch.as_tensor(masses), dt, spec["cutoff"], 10**6, ring_polymer=M.RingPolymer(2, 300.0),
                   compute_stress=True)
    with pytest.raises(RuntimeError, match="ring-polymer run"):
        _device_md(case, None, None, momenta=np.zeros((150, 3)))[0].centroid_positions()
