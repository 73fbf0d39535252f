"""Ring-polymer NPT on the device (the PILE barostat kernels of csrc/rpmd.cu, schnetpack_b200.md.PILEBarostat and the
NPTRingPolymer step of DeviceMD) against the fp64 oracle tests/rpmd_npt_oracle.py, which is pinned to the reference's own
PILEBarostat (tests/test_rpmd_npt_oracle.py)."""
import math

import numpy as np
import pytest
import torch

import npt_oracle as NPO
import nvt_oracle as NO
import rpmd_npt_oracle as RNO
import rpmd_oracle as RO
from conftest import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# exact binary-fraction units as in tests/test_cuda_rpmd.py, plus bar = 2^-4
EXACT = dict(kB=2.0 ** -7, fs=2.0 ** -10)
HBAR_EXACT, BAR_EXACT = 2.0 ** -4, 2.0 ** -4
T_EXACT, DT_EXACT = 300.0, 2.0 ** -12


def _np(t):
    return t.detach().cpu().numpy()


# ---- 1. kernels against the oracle ----------------------------------------------------------------------------------------
def _mixed_batch(P, seed=3, n_atoms=(1, 20_000, 3, 9)):
    """by default a 1-atom system next to a 20 000-atom one and small molecules, with bead state near 300 K, forces, cells
    (the third one triclinic) and virials of every bead system"""
    n_atoms = [int(n) for n in n_atoms]
    B = len(n_atoms)
    rng = np.random.default_rng(seed + P)
    n = sum(n_atoms)
    masses = rng.choice([1.0, 12.0, 16.0], size=n).astype(np.float32)
    x = (0.1 * rng.normal(size=(n, 3))[None] + 0.01 * rng.normal(size=(P, n, 3))).astype(np.float32)
    p = (rng.normal(size=(P, n, 3)) * np.sqrt(masses * EXACT["kB"] * 300.0 * P)[None, :, None]).astype(np.float32)
    f = (rng.normal(size=(P, n, 3)) * 10.0).astype(np.float32)
    cells = np.stack([np.diag(rng.uniform(2.0, 4.0, 3)) for _ in range(B)])
    cells[2] += np.array([[0.0, 0.0, 0.0], [0.5, 0.0, 0.0], [0.25, -0.375, 0.0]])
    cells = np.repeat(cells[None], P, axis=0)                                          # [P, B, 3, 3]
    virial = rng.normal(size=(P, B, 3, 3)) * 20.0
    return n_atoms, masses, x, p, f, cells, virial


def _bind(P, n_atoms, masses, seed=5, tau=64.0):
    from schnetpack_b200 import md

    idx_m = torch.repeat_interleave(torch.arange(len(n_atoms)), torch.tensor(n_atoms)).to(DEV)
    base = md._Systems(torch.as_tensor(masses, device=DEV), idx_m, len(n_atoms))
    rp = md.RingPolymer(P, T_EXACT, kB=EXACT["kB"], hbar=HBAR_EXACT)
    rp.bind(base, DT_EXACT)
    baro = md.PILEBarostat(1000.0, T_EXACT, tau, seed=seed, bar=BAR_EXACT, **EXACT)
    baro.bind(base, DT_EXACT, rp)
    return base, rp, baro


@pytest.mark.parametrize("P", [1, 5, 8, 32])
def test_barostat_kernels_follow_the_oracle(P):
    """two rounds of cell PILE, half step (p_c only: the particle kick is spk_md_velocity_verlet) and main step; each round
    starts the oracle from the device's state, so p_c and the cells are held to 1e-9 and the fp32 bead state to its
    rounding.  All P bead copies of a cell stay bitwise equal and the model cell is the MD cell * position_conversion."""
    barostat_follows_the_oracle(P, _mixed_batch(P))


def barostat_follows_the_oracle(P, batch):
    """the checks of test_barostat_kernels_follow_the_oracle on ``batch`` (as _mixed_batch returns it)"""
    n_atoms, masses, x, p, f, cells, virial = batch
    B = len(n_atoms)
    base, rp, baro = _bind(P, n_atoms, masses)
    f_conv, v_scale, p_conv = 0.5, 0.25, 10.0
    xt, pt, ft = (torch.as_tensor(a, device=DEV).reshape(-1, 3) for a in (x, p, f))
    model_x = torch.empty_like(xt)
    cell = torch.as_tensor(cells.reshape(P * B, 3, 3), device=DEV).contiguous()
    model_cell = torch.empty(P * B, 3, 3, dtype=torch.float32, device=DEV)
    vir = torch.as_tensor(virial.reshape(P * B, 3, 3), device=DEV).contiguous()
    baro.cell_momenta.copy_(torch.as_tensor(np.random.default_rng(P).normal(size=B) * 0.05, device=DEV))
    ref = RNO.PILEBarostat(1000.0, T_EXACT, 64.0, EXACT["kB"], EXACT["fs"], BAR_EXACT, RNO.philox_cell_noise(5))
    ro = RO.RingPolymer(P, T_EXACT, DT_EXACT, EXACT["kB"], HBAR_EXACT)
    ref.init(ro, masses.astype(np.float64), n_atoms)
    f64 = torch.as_tensor(f, dtype=torch.float64) * f_conv
    for k in range(2):
        ref.app = k
        xr = torch.as_tensor(_np(xt).reshape(P, -1, 3), dtype=torch.float64)
        pr = torch.as_tensor(_np(pt).reshape(P, -1, 3), dtype=torch.float64)
        cr = torch.as_tensor(_np(cell).reshape(P, B, 3, 3))
        ref.cell_momenta = torch.as_tensor(_np(baro.cell_momenta))
        baro.apply_thermostat()
        baro.half_step(pt, ft, f_conv, cell, vir, v_scale)
        baro.main_step(xt, pt, model_x, cell, model_cell, p_conv)
        torch.cuda.synchronize()
        ref.thermostat()
        ref.half_step(pr, f64, cr, v_scale * torch.as_tensor(virial) / RNO.volumes(cr)[..., None, None])
        xr, pr, cr = ref.main_step(xr, pr, cr)
        assert rel_err(_np(baro.cell_momenta), ref.cell_momenta.numpy()) < 1e-9, k
        assert rel_err(_np(cell).reshape(P, B, 3, 3), cr.numpy()) < 1e-9, k
        assert rel_err(_np(xt).reshape(P, -1, 3), xr.numpy()) < 1e-6, k
        assert rel_err(_np(pt).reshape(P, -1, 3), pr.numpy()) < 1e-5, k
        assert torch.equal(model_x, xt * p_conv)
        c = cell.reshape(P, B, 9)
        for r in range(1, P):
            assert torch.equal(c[r], c[0])
        assert torch.equal(model_cell, (cell * p_conv).float())
    assert baro.counter.tolist() == [2, 0]
    dv = np.abs(np.linalg.det(_np(cell).reshape(P, B, 3, 3)) / np.linalg.det(cells) - 1.0)
    assert dv.max() > 1e-6                                                                  # the cells moved


def test_barostat_noise_bits_equal_the_restatement_and_replays_draw_fresh_noise():
    """c1 = 0, c2 = 1: the kernel writes xi into p_c"""
    from schnetpack_b200 import _lib, ops

    n, seed = 20_000, 77
    pc = torch.zeros(n, dtype=torch.float64, device=DEV)
    c2 = torch.ones(n, dtype=torch.float64, device=DEV)
    counter = torch.tensor([3, 0], dtype=torch.int64, device=DEV)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _lib.call("spk_rpmd_barostat_thermostat", ops._p(pc), n, 0.0, ops._p(c2), seed, ops._p(counter), ops._stream())
    draws = []
    for k in range(3):
        g.replay()
        torch.cuda.synchronize()
        z = _np(pc)
        assert np.abs(z - NO.langevin_normals(seed, 3 + k, n)[:, 0]).max() < 1e-12
        draws.append(z)
    assert counter.tolist() == [6, 0]
    assert abs(np.corrcoef(draws[0], draws[1])[0, 1]) < 5.0 / math.sqrt(n)


# ---- 2. DeviceMD against the oracle's NPT-RPMD loop -----------------------------------------------------------------------
def _box_case():
    from schnetpack_b200 import synthetic as S

    spec = S.model_spec("painn", n_atom_basis=128, n_interactions=2)
    data = S.periodic_box(150, seed=9)
    params = S.init_params(spec, seed=8)
    masses = np.where(data["_atomic_numbers"] == 8, 16.0, 1.0)
    return spec, params, data, masses, 1e-3


def _device_md(case, P, thermostat, barostat, p_conv=1.0, e_conv=1.0, use_graph=True):
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params, data, masses, dt = case
    N = data["_positions"].shape[0]
    momenta = np.random.default_rng(2).normal(size=(P, N, 3)) * np.sqrt(masses * M.KB_MD * 300.0 * P)[None, :, None]
    model = from_spec(spec, params, torch.device(DEV))
    md = M.DeviceMD(model, batch_to_device(data, torch.device(DEV)), torch.as_tensor(masses), time_step=dt,
                    cutoff=spec["cutoff"], capacity=int(N * P * 80), momenta=torch.as_tensor(momenta),
                    use_graph=use_graph, position_conversion=p_conv, energy_conversion=e_conv, thermostat=thermostat,
                    barostat=barostat, ring_polymer=M.RingPolymer(P, 300.0))
    return md, momenta


def _oracle_calc(case, p_conv, e_conv):
    """forces [P, N, 3] and stress [P, B, 3, 3] in MD units of every bead system from the fp64 model oracle, with an exact
    neighbour list on the bead system's current cell"""
    from oracle import nl_oracle as NL
    from oracle import spk_oracle as O

    spec, params, data, _, _ = case
    pbc = np.asarray(data["_pbc"]).reshape(3)

    def calc(x_md, cells_md, n_atoms):
        assert len(n_atoms) == 1
        f = torch.zeros_like(x_md)
        stress = torch.zeros(x_md.shape[0], 1, 3, 3, dtype=torch.float64)
        for r in range(x_md.shape[0]):
            R = (x_md[r] * p_conv).numpy()
            cell = (cells_md[r, 0] * p_conv).numpy()
            ii, jj, _, off = NL.neighbor_list(R, cell, pbc, spec["cutoff"])
            b = dict(data)
            b.update({"_positions": R, "_idx_i": ii, "_idx_j": jj, "_offsets": off, "_cell": cell.reshape(1, 3, 3)})
            f[r] = O.energy_forces(spec, params, b, dtype=torch.float64)["forces"] * (e_conv / p_conv)
            _, s = NPO.stress_from_virial(spec, params, b, cell)
            stress[r] = s * e_conv / p_conv ** 3
        return f, stress

    return calc


TRAJ_THERMOSTATS = ["none", "pile_l", "pile_g", "trpmd", "nhc_local", "nhc_global"]
TAU_CELL = 100.0


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


def _baro(seed=23, target_bar=1000.0, tau=TAU_CELL):
    from schnetpack_b200 import md as M

    return M.PILEBarostat(target_bar, 300.0, tau, seed=seed)


# (p_conv, e_conv, target pressure in bar, cell time constant in fs).  With p_conv = 1 the box's Angstrom coordinates
# are read as nm: a 1500 nm^3 box of 150 atoms, whose pressure is a few bar, so it is run at 0 bar with a heavier cell
UNIT_SYSTEMS = [(1.0, 1.0, 0.0, 1000.0), (10.0, 0.5, 1000.0, TAU_CELL)]


@pytest.mark.parametrize("name", TRAJ_THERMOSTATS)
@pytest.mark.parametrize("p_conv,e_conv,target_bar,tau", UNIT_SYSTEMS)
def test_device_md_follows_the_oracle_npt_rpmd_loop(name, p_conv, e_conv, target_bar, tau):
    """12 NPT-RPMD steps of the 150-atom periodic PaiNN box at P = 4 from 300 K bead momenta against rpmd_npt_trajectory
    with the oracle's forces and virials; tolerances of the NPT and RPMD trajectory tests"""
    from schnetpack_b200.md import BAR_MD, FS_MD, HBAR_MD, KB_MD

    P = 4
    case = _box_case()
    dev_th, ref_th = _traj_thermostat(name)
    md, p0 = _device_md(case, P, dev_th, _baro(target_bar=target_bar, tau=tau), p_conv, e_conv)
    n_steps = 12
    md.run(n_steps)
    torch.cuda.synchronize()
    _, _, data, masses, dt = case
    x0 = np.repeat(np.asarray(data["_positions"], dtype=np.float64)[None] / p_conv, P, axis=0)
    c0 = np.asarray(data["_cell"], dtype=np.float64).reshape(1, 1, 3, 3).repeat(P, axis=0) / p_conv
    ro = RO.RingPolymer(P, 300.0, dt, KB_MD, HBAR_MD)
    ref_b = RNO.PILEBarostat(target_bar, 300.0, tau, KB_MD, FS_MD, BAR_MD, RNO.philox_cell_noise(23))
    xr, pr, cr = RNO.rpmd_npt_trajectory(ro, x0, p0, c0, masses, data["_n_atoms"], _oracle_calc(case, p_conv, e_conv),
                                         n_steps, ref_b, ref_th)
    dv = abs(float(md.volume()[0]) / float(np.linalg.det(c0[0, 0])) - 1.0)
    errs = [rel_err(_np(md.positions).reshape(P, -1, 3), xr.numpy()), rel_err(_np(md.momenta).reshape(P, -1, 3), pr.numpy()),
            rel_err(_np(md.cell).reshape(P, 1, 3, 3), cr.numpy()),
            rel_err(_np(md.barostat.cell_momenta), ref_b.cell_momenta.numpy())]
    print(f"{name} p_conv={p_conv}: relative volume change over {n_steps} steps {dv:.2e}; errors {errs}")
    # the chains scale every (mode, dof) by exp(-h v) with v driven by p~^2 / m, which turns the fp32 rounding of the
    # forces (20x larger in MD units at p_conv = 1) into bead-momentum errors up to 1.0e-3 over 12 steps, while the cell
    # and p_c stay within 1e-11 and 1e-7 of the oracle
    p_tol = 2e-3 if name.startswith("nhc") else 2e-4
    assert errs[0] < 1e-6 and errs[1] < p_tol and errs[2] < 1e-6 and errs[3] < 1e-4, errs
    assert dv > 5e-6                                                                  # the cell moved
    for r in range(1, P):
        assert torch.equal(md.cell[r], md.cell[0])


def test_graph_replay_equals_eager_and_restart_is_bitwise():
    from schnetpack_b200 import md as M

    case = _box_case()
    runs = {}
    for use_graph in (True, False):
        md, _ = _device_md(case, 4, M.PILELocalThermostat(300.0, 20.0, seed=3), _baro(), 10.0, 0.5, use_graph=use_graph)
        md.run(10)
        torch.cuda.synchronize()
        runs[use_graph] = (_np(md.positions), _np(md.momenta), _np(md.cell), md.barostat.state_dict())
    assert rel_err(runs[True][0], runs[False][0]) < 1e-6
    assert rel_err(runs[True][1], runs[False][1]) < 1e-5
    assert rel_err(runs[True][2], runs[False][2]) < 1e-9
    assert runs[True][3]["counter"].tolist() == runs[False][3]["counter"].tolist() == [20, 0]

    def make():
        return _device_md(case, 4, M.PILELocalThermostat(300.0, 20.0, seed=3), _baro(), 10.0, 0.5)[0]

    a = make()
    a.run(4)
    saved = a.state_dict()
    a.run(4)
    b = make()
    b.load_state_dict(saved)
    b.run(4)
    torch.cuda.synchronize()
    assert b.steps_done == a.steps_done == 8
    for k in ("positions", "momenta", "forces", "energy", "cell", "model_cell", "virial"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    for k, v in a.barostat.state_dict().items():
        assert torch.equal(v, b.barostat.state_dict()[k]), k
    assert a.barostat.counter.tolist() == [16, 0]


def test_centroid_pressure_at_one_bead_is_the_pressure():
    case = _box_case()
    md, _ = _device_md(case, 1, None, _baro())
    md.run(3)
    torch.cuda.synchronize()
    for kw in (dict(), dict(kinetic_component=True), dict(tensor=True), dict(tensor=True, kinetic_component=True)):
        a, b = md.centroid_pressure(**kw), md.pressure(**kw)
        assert a.shape == b.shape == ((1, 3, 3) if kw.get("tensor") else (1,)), kw
        assert rel_err(_np(a), _np(b)) < 1e-12, kw


def test_centroid_pressure_follows_the_oracle_and_needs_npt():
    P = 4
    case = _box_case()
    md, _ = _device_md(case, P, None, _baro(), 10.0, 0.5)
    md.run(2)
    torch.cuda.synchronize()
    _, _, data, masses, _ = case
    p = torch.as_tensor(_np(md.momenta).reshape(P, -1, 3), dtype=torch.float64)
    cells = torch.as_tensor(_np(md.cell).reshape(P, 1, 3, 3))
    stress = torch.as_tensor(_np(md.stress).reshape(P, 1, 3, 3))
    for kw in (dict(), dict(kinetic_component=True), dict(tensor=True, kinetic_component=True)):
        ref = RNO.centroid_pressure(p, masses, data["_n_atoms"], cells, stress, **kw)
        assert rel_err(_np(md.centroid_pressure(**kw)), ref.numpy()) < 1e-5, kw
    nvt, _ = _device_md(case, P, None, None)
    with pytest.raises(RuntimeError, match="ring-polymer NPT"):
        nvt.centroid_pressure()


def test_device_md_refuses_what_ring_polymer_npt_cannot_run():
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device, from_spec

    case = _box_case()
    spec, params, data, masses, dt = case
    model = from_spec(spec, params, torch.device(DEV))
    dev = torch.device(DEV)
    kw = dict(time_step=dt, cutoff=spec["cutoff"], capacity=10 ** 6)
    with pytest.raises(ValueError, match="ring-polymer barostat"):
        M.DeviceMD(model, batch_to_device(data, dev), torch.as_tensor(masses), barostat=_baro(), **kw)
    open_axis = dict(data, _pbc=np.array([True, True, False]))
    with pytest.raises(ValueError, match="periodic"):
        M.DeviceMD(model, batch_to_device(open_axis, dev), torch.as_tensor(masses), barostat=_baro(),
                   ring_polymer=M.RingPolymer(4, 300.0), **kw)
    flat = dict(data, _cell=np.asarray(data["_cell"]) * np.array([1.0, 1.0, 0.0], dtype=np.float32)[:, None])
    with pytest.raises(ValueError, match="volume"):
        M.DeviceMD(model, batch_to_device(flat, dev), torch.as_tensor(masses), barostat=_baro(),
                   ring_polymer=M.RingPolymer(4, 300.0), **kw)
    with pytest.raises(ValueError, match="compute_stress"):
        M.DeviceMD(model, batch_to_device(data, dev), torch.as_tensor(masses), barostat=_baro(),
                   ring_polymer=M.RingPolymer(4, 300.0), compute_stress=True, **kw)


# ---- 3. physics: the ideal gas ----------------------------------------------------------------------------------------------
def test_ideal_gas_samples_the_isobaric_volume():
    """1000 non-interacting atoms of mass 40 at P = 4 (the last Atomwise layer is zero, so E, F and W are exactly 0 while
    the whole kernel path still runs) with PILE-L at 300 K and the PILE barostat at 400 bar.  The scheme samples
    P(V) ~ V^N exp(-P0 V / kT) (DESIGN.md section 9), so <V> = (N + 1) kT / P0 = 103.6 nm^3 with sigma_V / <V> =
    1 / sqrt(N + 1) = 3.2 % per sample.  dt = 2 fs, tau = 100 fs for the centroid and the cell; 20 000 steps of
    equilibration from <V>, then 60 000 steps sampled every 20.  The mean volume must lie within 1 % of <V>, with a
    standard error from 20 block means of at most a third of that, and the mean centroid temperature within 5 sigma of
    the bath.  About a minute on an H100."""
    from schnetpack_b200 import md as M
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, from_spec

    N, P, T, P_bar, mass, p_conv = 1000, 4, 300.0, 400.0, 40.0, 10.0
    v_exp = (N + 1) * M.KB_MD * T / (P_bar * M.BAR_MD)                      # nm^3
    L = v_exp ** (1.0 / 3.0)
    rng = np.random.default_rng(7)
    batch = {"_positions": (rng.uniform(0.0, L, (N, 3)) * p_conv).astype(np.float32),
             "_atomic_numbers": np.full(N, 8, dtype=np.int64), "_n_atoms": np.array([N], dtype=np.int64),
             "_idx_m": np.zeros(N, dtype=np.int64), "_cell": (L * p_conv * np.eye(3, dtype=np.float32))[None],
             "_pbc": np.ones(3, dtype=bool)}
    spec = S.model_spec("painn", n_atom_basis=128, n_interactions=1)
    dev = torch.device(DEV)
    model = from_spec(spec, S.init_params(spec, seed=3), dev)
    last = model.output_modules[0].outnet[1]
    with torch.no_grad():
        last.weight.zero_()
        last.bias.zero_()
    p0 = rng.normal(size=(P, N, 3)) * math.sqrt(mass * M.KB_MD * T * P)
    md = M.DeviceMD(model, batch_to_device(batch, dev), torch.full((N,), mass), time_step=2.0 * M.FS_MD,
                    cutoff=spec["cutoff"], capacity=16 * N * P, momenta=torch.as_tensor(p0), position_conversion=p_conv,
                    thermostat=M.PILELocalThermostat(T, 100.0, seed=1), barostat=M.PILEBarostat(P_bar, T, 100.0, seed=2),
                    ring_polymer=M.RingPolymer(P, T))
    md.run(20_000)
    vols, temps = [], []
    for _ in range(3000):
        md.run(20)
        vols.append(float(md.volume()[0]))
        temps.append(float(md.centroid_temperature()[0]))
    assert float(md.forces.abs().max()) == 0.0 and float(md.virial.abs().max()) == 0.0
    assert torch.equal(md.cell[1:], md.cell[:1].expand(P - 1, 3, 3))
    vols = np.asarray(vols)
    mean = vols.mean()
    se = vols.reshape(20, -1).mean(1).std(ddof=1) / math.sqrt(20)
    print(f"ideal gas: <V> = {mean:.3f} nm^3 +- {se:.3f} against {v_exp:.3f}; <T_c> = {np.mean(temps):.1f} K")
    assert se <= 0.01 * v_exp / 3.0, (se, v_exp)
    assert abs(mean / v_exp - 1.0) < 0.01, (mean, v_exp, se)
    sigma_t = T * math.sqrt(2.0 / (3.0 * N))
    assert abs(np.mean(temps) - T) < 5.0 * sigma_t, (np.mean(temps), sigma_t)
