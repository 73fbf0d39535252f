"""Virial kernel and NHC barostats of the device MD step (csrc/geometry.cu, csrc/barostat.cu, schnetpack_b200.md) against
the reference stress fixture and the fp64 restatement tests/npt_oracle.py, which is pinned to the reference's own barostats
(tests/test_npt_oracle.py)."""
import json

import numpy as np
import pytest
import torch

import npt_oracle as NPO
from conftest import GOLDEN, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _np(t):
    return t.detach().cpu().numpy()


# ---- virial ---------------------------------------------------------------------------------------------------------------
def _stress_box():
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, from_spec

    z = np.load(f"{GOLDEN}/painn_box_stress.npz")
    spec = json.loads(str(z["spec_json"]))
    params = S.init_params(spec, int(z["seed"]))
    batch = {k[3:]: z[k] for k in z.files if k.startswith("in:")}
    spec_plain = dict(spec, stress=False)
    model = from_spec(spec_plain, params, torch.device(DEV))
    return z, spec_plain, params, model, batch_to_device(batch, torch.device(DEV))


def _eval(model, x, virial=None):
    x = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in x.items()}
    if virial is not None:
        x["_virial"] = virial
    out = model(x)
    return out["energy"].detach(), out["forces"].detach()


def test_virial_matches_reference_stress_and_is_bitwise_reproducible():
    z, _, _, model, x = _stress_box()
    e0, f0 = _eval(model, x)
    W1 = torch.full((1, 3, 3), float("nan"), dtype=torch.float64, device=DEV)
    e1, f1 = _eval(model, x, W1)
    W2 = torch.empty_like(W1)
    _eval(model, x, W2)
    torch.cuda.synchronize()
    assert torch.equal(e0, e1) and torch.equal(f0, f1)          # asking for the virial changes nothing else
    assert torch.equal(W1, W2)
    cell = z["in:_cell"].reshape(3, 3).astype(np.float64)
    stress = _np(W1) / abs(np.linalg.det(cell))
    assert rel_err(stress, z["ref64:stress"]) < 1e-5

    # graph replay equals the eager call
    W3 = torch.zeros_like(W1)
    xs = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in x.items()}
    _eval(model, xs, W3)                                        # warm-up outside the capture (graph views, packs)
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _eval(model, xs, W3)
    torch.cuda.current_stream().wait_stream(side)
    with torch.cuda.graph(g):
        _eval(model, xs, W3)
    W3.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(W3, W1)


def test_virial_with_padded_list_and_strain_path():
    from schnetpack_b200.model import from_spec
    from schnetpack_b200.neighbors import CellListNeighborList

    z, spec, params, model, x = _stress_box()
    W = torch.zeros(1, 3, 3, dtype=torch.float64, device=DEV)
    _eval(model, x, W)
    # the same box through the padded device neighbour list (padding pairs at 2 cutoff add nothing)
    nl = CellListNeighborList(spec["cutoff"], capacity=int(x["_idx_i"].shape[0] * 1.5), pad=True)
    xp = {k: v for k, v in x.items() if k not in ("_idx_i", "_idx_j", "_offsets")}
    xp = nl(xp)
    Wp = torch.zeros_like(W)
    _eval(model, xp, Wp)
    # this package's Strain + Forces(calc_stress=True) path
    ms = from_spec(dict(spec, stress=True), params, torch.device(DEV))
    out = ms({k: (v.clone() if torch.is_tensor(v) else v) for k, v in x.items()})
    torch.cuda.synchronize()
    V = abs(np.linalg.det(z["in:_cell"].reshape(3, 3).astype(np.float64)))
    # not 1e-12: the padded list holds the real pairs in another order, so the model's fp32 neighbour sums -- and with them
    # the edge gradients g_e -- round differently; the padding pairs themselves add exact zeros
    assert rel_err(_np(Wp), _np(W)) < 1e-5
    assert rel_err(_np(W) / V, _np(out["stress"]).reshape(1, 3, 3)) < 1e-5


# ---- barostat kernels on the golden protocol ------------------------------------------------------------------------------
CASES = {"iso_o3": dict(anisotropic=False, massive=False, integration_order=3),
         "iso_massive_o7": dict(anisotropic=False, massive=True, integration_order=7),
         "aniso_o7": dict(anisotropic=True, massive=False, integration_order=7),
         "aniso_massive_o3": dict(anisotropic=True, massive=True, integration_order=3, chain_length=3, multi_step=2)}


@pytest.mark.parametrize("name", sorted(CASES))
def test_barostat_kernels_follow_the_oracle(name):
    from schnetpack_b200 import md as M

    g = dict(np.load(f"{GOLDEN}/md_barostats.npz"))
    kw = dict(CASES[name])
    cls = M.NHCBarostatAnisotropic if kw.pop("anisotropic") else M.NHCBarostatIsotropic
    tau = float(g["time_constant_fs"])
    b = cls(float(g["target_pressure_bar"]), float(g["temperature_bath"]), tau, time_constant_cell=0.5 * tau,
            time_constant_barostat=2.0 * tau, kB=float(g["kB"]), fs=float(g["fs"]), bar=float(g["bar"]), **kw)
    n_atoms = [int(n) for n in g["n_atoms"]]
    idx_m = torch.repeat_interleave(torch.arange(len(n_atoms)), torch.tensor(n_atoms)).to(DEV)
    sy = M._Systems(torch.as_tensor(g["masses"], dtype=torch.float32, device=DEV), idx_m, len(n_atoms))
    b.bind(sy, float(g["time_step"]))
    f32 = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float32, device=DEV).contiguous()  # noqa: E731
    x, p = f32(g["positions"]), f32(g["momenta"])
    cell = torch.as_tensor(g["cells"], dtype=torch.float64, device=DEV).contiguous()
    forces = torch.zeros_like(x)
    stress = torch.as_tensor(g["stress0"], dtype=torch.float64, device=DEV)

    def kick():
        vir = (stress * torch.linalg.det(cell)[:, None, None]).contiguous()   # stress = virial / V
        b.kick(p, cell, vir, 1.0)

    for k in range(g["forces"].shape[0]):
        b.apply_thermostat(p)
        kick()
        b.half_step(p, forces)
        b.main_step(x, p, cell)
        forces = f32(g["forces"][k])
        stress = torch.as_tensor(g["stress"][k], dtype=torch.float64, device=DEV)
        b.half_step(p, forces)
        kick()
        b.apply_thermostat(p)
    torch.cuda.synchronize()
    assert rel_err(_np(x), g[name + ":positions"]) < 1e-6
    assert rel_err(_np(p), g[name + ":momenta"]) < 1e-6
    assert rel_err(_np(cell), g[name + ":cells"]) < 1e-6
    for k in ("t_masses", "t_masses_cell", "b_masses_cell"):
        dev = {"t_masses": b.t_masses, "t_masses_cell": b.t_masses_cell, "b_masses_cell": b.b_masses}[k]
        assert rel_err(_np(dev).reshape(g[name + ":" + k].shape), g[name + ":" + k]) < 1e-12, k
    # the chain and cell state is fp64 on the device but is driven by fp32 momenta and positions, so it follows the fp64
    # golden to the fp32 level rather than to 1e-12
    for k, dev in (("t_velocities", b.t_velocities), ("t_forces", b.t_forces), ("t_velocities_cell", b.t_velocities_cell),
                   ("t_forces_cell", b.t_forces_cell), ("b_velocities_cell", b.b_velocities),
                   ("b_forces_cell", b.b_forces)):
        assert rel_err(_np(dev).reshape(g[name + ":" + k].shape), g[name + ":" + k]) < 1e-5, k


def test_kinetic_energy_tensor():
    from schnetpack_b200 import md as M

    n_atoms = [1, 3, 20_000, 7]
    rng = np.random.default_rng(1)
    n = sum(n_atoms)
    m = rng.choice([1.0, 12.0, 16.0], size=n).astype(np.float32)
    p = rng.normal(size=(n, 3)).astype(np.float32)
    idx_m = torch.repeat_interleave(torch.arange(len(n_atoms)), torch.tensor(n_atoms)).to(DEV)
    sy = M._Systems(torch.as_tensor(m, device=DEV), idx_m, len(n_atoms))
    pt = torch.as_tensor(p, device=DEV)
    K1, K2 = sy.kinetic_energy_tensor(pt), sy.kinetic_energy_tensor(pt)
    torch.cuda.synchronize()
    assert torch.equal(K1, K2)
    p64, m64 = p.astype(np.float64), m.astype(np.float64)
    ref = np.stack([0.5 * np.einsum("na,nb->ab", p64[s:e], p64[s:e] / m64[s:e, None])
                    for s, e in zip(np.cumsum([0] + n_atoms[:-1]), np.cumsum(n_atoms))])
    assert rel_err(_np(K1), ref) < 1e-12


# ---- DeviceMD NPT ---------------------------------------------------------------------------------------------------------
def _units():
    from schnetpack_b200.md import BAR_MD, FS_MD, KB_MD

    return KB_MD, FS_MD, BAR_MD


BARO_KW = dict(time_constant_barostat=1000.0, integration_order=3, multi_step=2)


def _box_md(barostat=None, thermostat=None, p_conv=1.0, e_conv=1.0, use_graph=True, compute_stress=False):
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
                  position_conversion=p_conv, energy_conversion=e_conv, thermostat=thermostat, barostat=barostat,
                  compute_stress=compute_stress)
    return md, (spec, params, data, masses, p0)


@pytest.mark.parametrize("aniso", [False, True])
@pytest.mark.parametrize("massive", [False, True])
@pytest.mark.parametrize("p_conv,e_conv", [(1.0, 1.0), (10.0, 0.5)])
def test_device_md_follows_the_reference_npt_loop(aniso, massive, p_conv, e_conv):
    from schnetpack_b200 import md as M

    cls = M.NHCBarostatAnisotropic if aniso else M.NHCBarostatIsotropic
    md, (spec, params, data, masses, p0) = _box_md(cls(0.0, 5.0, 20.0, massive=massive, **BARO_KW), p_conv=p_conv,
                                                   e_conv=e_conv)
    n_steps = 12
    md.run(n_steps)
    torch.cuda.synchronize()
    ref = NPO.NHCBarostat(0.0, 5.0, 20.0, *_units(), massive=massive, anisotropic=aniso, **BARO_KW)
    x_ref, p_ref, e_ref, c_ref = NPO.npt_trajectory(spec, params, data, masses, p0, 1e-3, n_steps, ref, p_conv, e_conv)
    assert rel_err(_np(md.positions), x_ref) < 1e-6
    assert rel_err(_np(md.momenta), p_ref) < 1e-4
    assert rel_err(_np(md.potential_energy()), e_ref) < 1e-5
    assert rel_err(_np(md.cell), c_ref) < 1e-6
    v0 = abs(np.linalg.det(np.asarray(data["_cell"], dtype=np.float64).reshape(3, 3))) / p_conv ** 3
    assert abs(float(md.volume()[0]) / v0 - 1.0) > 5e-6                      # the cell moved, well above its tolerance
    if not aniso and not massive and p_conv == 1.0:                           # NVT-NHC from the same start ends elsewhere
        nvt, _ = _box_md(thermostat=M.NHCThermostat(5.0, 20.0))
        nvt.run(n_steps)
        assert rel_err(_np(nvt.positions), x_ref) > 1e-5


@pytest.mark.parametrize("aniso", [False, True])
def test_npt_graph_replay_equals_eager_and_restart_is_bitwise(aniso):
    from schnetpack_b200 import md as M

    cls = M.NHCBarostatAnisotropic if aniso else M.NHCBarostatIsotropic
    make = lambda: cls(0.0, 5.0, 20.0, massive=aniso, **BARO_KW)  # noqa: E731
    runs = {}
    for use_graph in (True, False):
        md, _ = _box_md(make(), use_graph=use_graph)
        md.run(10)
        torch.cuda.synchronize()
        runs[use_graph] = (_np(md.positions), _np(md.cell))
    assert rel_err(runs[True][0], runs[False][0]) < 1e-6
    assert rel_err(runs[True][1], runs[False][1]) < 1e-9

    a, _ = _box_md(make())
    a.run(4)
    saved = a.state_dict()
    a.run(4)
    b, _ = _box_md(make())
    b.load_state_dict(saved)
    b.run(4)
    torch.cuda.synchronize()
    for k in ("positions", "momenta", "forces", "energy", "cell", "model_cell", "virial"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    for k, v in a.barostat.state_dict().items():
        assert torch.equal(v, b.barostat.state_dict()[k]), k


def test_nvt_with_compute_stress_tracks_the_virial():
    from schnetpack_b200 import md as M

    md, (spec, params, data, _, _) = _box_md(thermostat=M.NHCThermostat(5.0, 20.0), compute_stress=True)
    ref, _ = _box_md(thermostat=M.NHCThermostat(5.0, 20.0))
    md.run(5)
    ref.run(5)
    torch.cuda.synchronize()
    assert torch.equal(md.positions, ref.positions)                            # stress on request changes nothing else
    x = {k: v for k, v in data.items()}
    x["_positions"] = _np(md.positions)
    nl = NPO.NL.neighbor_list(x["_positions"], np.asarray(data["_cell"]).reshape(3, 3), np.asarray(data["_pbc"]),
                              spec["cutoff"])
    x.update(_idx_i=nl[0], _idx_j=nl[1], _offsets=nl[3])
    _, s_ref = NPO.stress_from_virial(spec, params, x, np.asarray(data["_cell"]).reshape(3, 3))
    assert rel_err(_np(md.stress), s_ref.numpy()) < 1e-4
    assert md.pressure().shape == (1,) and md.pressure(tensor=True, kinetic_component=True).shape == (1, 3, 3)


def test_npt_and_virial_refuse_what_they_cannot_compute():
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device

    md, (spec, params, data, masses, _) = _box_md()
    kw = dict(time_step=1e-3, cutoff=spec["cutoff"], capacity=int(data["_idx_i"].shape[0] * 1.5))
    baro = lambda: M.NHCBarostatIsotropic(1.0, 5.0, 20.0)  # noqa: E731
    dev = torch.device(DEV)
    with pytest.raises(ValueError, match="own thermostat"):
        M.DeviceMD(md.model, batch_to_device(data, dev), torch.as_tensor(masses), thermostat=M.NHCThermostat(5.0, 20.0),
                   barostat=baro(), **kw)
    open_axis = dict(data, _pbc=np.array([True, True, False]))
    with pytest.raises(ValueError, match="periodic"):
        M.DeviceMD(md.model, batch_to_device(open_axis, dev), torch.as_tensor(masses), barostat=baro(), **kw)
    flat = dict(data, _cell=np.asarray(data["_cell"]) * np.array([1.0, 1.0, 0.0], dtype=np.float32)[:, None])
    with pytest.raises(ValueError, match="volume"):
        M.DeviceMD(md.model, batch_to_device(flat, dev), torch.as_tensor(masses), barostat=baro(), **kw)
    # the virial comes from the kernels' backward: the training path and a grad-free evaluation refuse the key
    x = batch_to_device(data, dev)
    W = torch.zeros(1, 3, 3, dtype=torch.float64, device=DEV)
    md.model.train()
    try:
        with pytest.raises(ValueError, match="eval"):
            md.model(dict(x, _virial=W))
    finally:
        md.model.eval()
    from schnetpack_b200.atomistic import PairwiseDistances

    with torch.no_grad(), pytest.raises(ValueError, match="backward"):
        PairwiseDistances().eval()(dict(x, _virial=W))


def _collate(parts):
    """concatenate single-system batches into one batch of len(parts) systems"""
    out, off = {}, 0
    for k in ("_positions", "_atomic_numbers", "_offsets"):
        out[k] = np.concatenate([p[k] for p in parts])
    out["_idx_i"] = np.concatenate([p["_idx_i"] + o for p, o in zip(parts, np.cumsum([0] + [len(p["_atomic_numbers"])
                                                                                          for p in parts[:-1]]))])
    out["_idx_j"] = np.concatenate([p["_idx_j"] + o for p, o in zip(parts, np.cumsum([0] + [len(p["_atomic_numbers"])
                                                                                          for p in parts[:-1]]))])
    n = [len(p["_atomic_numbers"]) for p in parts]
    out["_n_atoms"] = np.array(n, dtype=np.int64)
    out["_idx_m"] = np.repeat(np.arange(len(parts)), n).astype(np.int64)
    out["_cell"] = np.concatenate([np.asarray(p["_cell"], dtype=np.float32).reshape(1, 3, 3) for p in parts])
    out["_pbc"] = np.concatenate([np.asarray(p["_pbc"]).reshape(3) for p in parts])
    return out


def test_virial_per_system_on_a_mixed_batch():
    """Boxes of 128, 150 (7856 edges, 31 CTAs of the partial pass) and 216 atoms and a 1-atom system without any edge,
    in one launch: W_m / V_m equals this package's Strain path for every system, the empty system gets exact zeros, and
    two calls are bitwise equal."""
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, from_spec

    lone = {"_positions": np.array([[1.0, 2.0, 3.0]], dtype=np.float32), "_atomic_numbers": np.array([8]),
            "_offsets": np.zeros((0, 3), dtype=np.float32), "_idx_i": np.zeros(0, dtype=np.int64),
            "_idx_j": np.zeros(0, dtype=np.int64), "_cell": 30.0 * np.eye(3, dtype=np.float32),
            "_pbc": np.ones(3, dtype=bool)}
    parts = [S.periodic_box(128, seed=4), lone, S.periodic_box(150, seed=9), S.periodic_box(216, seed=5)]
    batch = _collate(parts)
    spec = S.model_spec("painn", n_atom_basis=128, n_interactions=2)
    params = S.init_params(spec, seed=8)
    dev = torch.device(DEV)
    model = from_spec(spec, params, dev)
    x = batch_to_device(batch, dev)
    W1 = torch.full((4, 3, 3), float("nan"), dtype=torch.float64, device=DEV)
    W2 = torch.full_like(W1, float("nan"))
    _eval(model, x, W1)
    _eval(model, x, W2)
    ms = from_spec(dict(spec, stress=True), params, dev)
    out = ms({k: v.clone() for k, v in x.items()})
    torch.cuda.synchronize()
    assert torch.equal(W1, W2)
    assert torch.equal(W1[1], torch.zeros(3, 3, dtype=torch.float64, device=DEV))
    V = np.abs(np.linalg.det(batch["_cell"].astype(np.float64)))
    stress = _np(out["stress"]).reshape(4, 3, 3)
    for m in (0, 2, 3):
        assert rel_err(_np(W1[m]) / V[m], stress[m]) < 1e-5, m
        assert np.abs(_np(W1[m])).max() > 0.0
    assert np.abs(stress[1]).max() == 0.0


def test_ideal_gas_samples_the_isobaric_volume():
    """2000 non-interacting atoms (the last Atomwise layer is zero, so E, F and W are exactly 0 while the whole kernel path
    still runs) under the isotropic barostat at 300 K and 400 bar.  MTK samples P(V) ~ V^N exp(-PV / kT), so <V> =
    (N + 1) kT / P = 207.2 nm^3, with sigma_V / <V> = 1 / sqrt(N + 1) = 2.2 % per sample.  dt = 2 fs, tau = 100 fs,
    tau_barostat = 200 fs; 100 000 steps (200 ps, ~1000 barostat time constants).  The second half is sampled every 20 steps;
    its mean volume must lie within 1 % of <V>, with a standard error from 20 block means of at most a third of that, and
    the mean temperature within 5 sigma of the bath."""
    import math

    from schnetpack_b200 import md as M
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, from_spec

    N, T, P_bar, mass, p_conv = 2000, 300.0, 400.0, 40.0, 10.0
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
    p0 = rng.normal(size=(N, 3)) * math.sqrt(mass * M.KB_MD * T)
    baro = M.NHCBarostatIsotropic(P_bar, T, 100.0, time_constant_barostat=200.0)
    md = M.DeviceMD(model, batch_to_device(batch, dev), torch.full((N,), mass), time_step=2.0 * M.FS_MD,
                    cutoff=spec["cutoff"], capacity=16 * N, momenta=torch.as_tensor(p0), position_conversion=p_conv,
                    barostat=baro)
    md.run(50_000)
    vols, temps = [], []
    for _ in range(2500):
        md.run(20)
        vols.append(float(md.volume()[0]))
        temps.append(float(md.temperature()[0]))
    assert float(md.forces.abs().max()) == 0.0 and float(md.virial.abs().max()) == 0.0
    vols = np.asarray(vols)
    mean = vols.mean()
    se = vols.reshape(20, -1).mean(1).std(ddof=1) / math.sqrt(20)
    assert se <= 0.01 * v_exp / 3.0, (se, v_exp)
    assert abs(mean / v_exp - 1.0) < 0.01, (mean, v_exp, se)
    sigma_t = T * math.sqrt(2.0 / (3.0 * N))
    assert abs(np.mean(temps) - T) < 5.0 * sigma_t, (np.mean(temps), sigma_t)
