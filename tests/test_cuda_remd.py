"""GPU: per-system bath temperatures of the Langevin and NHC thermostats and temperature replica exchange in DeviceMD
(csrc/thermostat.cu, csrc/exchange.cu, schnetpack_b200.exchange) against the scalar thermostats and the fp64 oracle
tests/remd_oracle.py."""
import ctypes
import math

import numpy as np
import pytest
import torch

import remd_oracle as RO
from conftest import load_case, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MASS = {1: 1.008, 6: 12.011, 7: 14.007, 8: 15.999, 9: 18.998}
K, G = 4, 3
LADDER = [300.0 * 1.1 ** k for k in range(K)]


def _np(t):
    return t.detach().cpu().numpy()


def _mixed(K=K, seed=0):
    """K rung-major copies of G = 3 QM9-like molecules of 18, 21 and 22 atoms"""
    from schnetpack_b200 import md as M
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device

    data = S.qm9like_batch(G, seed=seed)
    assert len(set(data[S.n_atoms].tolist())) == G
    b = {k: v for k, v in batch_to_device(data, torch.device(DEV)).items() if k not in (S.idx_i, S.idx_j, S.offsets)}
    b = M.replicate_batch(b, K, G)
    masses = torch.tensor([MASS[int(z)] for z in b[S.Z].tolist()], dtype=torch.float32)
    return b, masses


def _model(seed=3):
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import from_spec

    spec = S.model_spec("painn", n_atom_basis=32, n_interactions=2)
    return spec, from_spec(spec, S.init_params(spec, seed=seed), torch.device(DEV))


def _temps(K=K):
    return [t for t in LADDER[:K] for _ in range(G)]


def _run(thermostat, hooks=(), batch=None, masses=None, model=None, **kw):
    from schnetpack_b200 import md as M

    spec, m = _model() if model is None else model
    b, ms = _mixed() if batch is None else (batch, masses)
    kw.setdefault("initializer", M.MaxwellBoltzmannInit(300.0, seed=2))
    return M.DeviceMD(m, b, ms, time_step=0.5 * M.FS_MD, cutoff=spec["cutoff"], capacity=32 * ms.shape[0],
                      thermostat=thermostat, hooks=list(hooks), **kw)


# ---- per-system thermostats -----------------------------------------------------------------------------------------------
SCALAR_OR_PER_SYSTEM = {
    "langevin": lambda M, T: M.LangevinThermostat(T, 20.0, seed=5),
    "nhc": lambda M, T: M.NHCThermostat(T, 20.0),
    "nhc_massive": lambda M, T: M.NHCThermostat(T, 20.0, massive=True, integration_order=5),
}


@pytest.mark.parametrize("name", sorted(SCALAR_OR_PER_SYSTEM))
def test_per_system_thermostat_at_one_temperature_is_bitwise_the_scalar_one(name):
    """300 steps of the 12-system PaiNN batch: one temperature per system, all equal, against one number"""
    from schnetpack_b200 import md as M

    make = SCALAR_OR_PER_SYSTEM[name]
    runs = []
    for T in (310.0, [310.0] * (K * G)):
        md = _run(make(M, T))
        assert md.thermostat.per_system == isinstance(T, list)
        md.run(300)
        torch.cuda.synchronize()
        runs.append(md)
    a, b = runs
    assert torch.equal(a.positions, b.positions) and torch.equal(a.momenta, b.momenta)
    assert torch.equal(a.forces, b.forces) and torch.equal(a.energy, b.energy)
    for k, v in a.thermostat.state_dict().items():
        assert torch.equal(v, b.thermostat.state_dict()[k]), k
    if name.startswith("nhc"):
        assert torch.equal(a.thermostat.masses, b.thermostat.masses)
    assert np.isfinite(_np(a.positions)).all()


# units in which kB T is an exact binary fraction for integer T (as tests/test_cuda_thermostats.py)
EXACT = dict(kB=2.0 ** -7, fs=2.0 ** -10)
TAU, DT = 128.0, 2.0 ** -7


def _thermostat_batch(seed=3):
    n_atoms = [1, 3, 9, 2000, 20, 5]
    temps = [120.0, 250.0, 300.0, 410.0, 600.0, 900.0]
    rng = np.random.default_rng(seed)
    n = sum(n_atoms)
    masses = rng.choice([1.008, 12.011, 15.999], size=n).astype(np.float32)
    t_sys = np.repeat(rng.uniform(100.0, 600.0, len(n_atoms)), n_atoms)
    p = (rng.normal(size=(n, 3)) * np.sqrt(masses * EXACT["kB"] * t_sys)[:, None]).astype(np.float32)
    from schnetpack_b200.md import _Systems

    idx_m = torch.repeat_interleave(torch.arange(len(n_atoms)), torch.tensor(n_atoms)).to(DEV)
    return n_atoms, temps, masses, p, _Systems(torch.as_tensor(masses, device=DEV), idx_m, len(n_atoms))


@pytest.mark.parametrize("kind,kw", [("langevin", {}), ("nhc", dict(massive=False)), ("nhc", dict(massive=True))])
def test_per_system_thermostats_follow_the_oracle(kind, kw):
    from schnetpack_b200 import md

    n_atoms, temps, masses, p, sy = _thermostat_batch()
    if kind == "langevin":
        dev_th = md.LangevinThermostat(temps, TAU, seed=7, **EXACT)
    else:
        dev_th = md.NHCThermostat(torch.tensor(temps), TAU, **kw, **EXACT)
        ref_th = RO.NHCPerSystem(temps, TAU, EXACT["kB"], EXACT["fs"], **kw)
        ref_th.init(masses.astype(np.float64), n_atoms, DT)
    dev_th.bind(sy, DT)
    assert _np(dev_th.temperatures).tolist() == temps
    pt = torch.as_tensor(p, device=DEV)
    pr = p.astype(np.float64)
    for app in range(6):
        dev_th.apply(pt)
        if kind == "langevin":
            pr = RO.langevin_kick(pr, masses, n_atoms, temps, EXACT["kB"], dev_th.c1, dev_th.c2, 7, app)
        else:
            pr = ref_th.apply(pr).numpy()
    torch.cuda.synchronize()
    assert rel_err(_np(pt), pr) < 1e-6
    assert np.abs(pr - p).max() > 1e-2 * np.abs(p).max()
    if kind == "nhc":
        v, f, m = ref_th.chain_state()
        assert rel_err(_np(dev_th.masses), m) < 1e-12
        assert rel_err(_np(dev_th.velocities), v) < 1e-6
        assert rel_err(_np(dev_th.forces), f) < 1e-6


# ---- the exchange kernel through the C ABI --------------------------------------------------------------------------------
def test_exchange_kernel_matches_the_oracle_and_keeps_boltzmann_energies():
    """G = 100 000 groups of K = 4 rungs on host-made energies: decisions, walkers, statistics and swapped energies equal
    the oracle exactly; on fresh exact samples of a harmonic well every rung keeps <U> = d kB T_k / 2."""
    from schnetpack_b200 import _lib, ops

    K4, GG, d, kB, e_conv, seed = 4, 100_000, 12, 0.0083144598, 0.5, 0xC0FFEE
    T = np.repeat(300.0 * 1.2 ** np.arange(K4), GG)
    dev = torch.device(DEV)
    energy = torch.empty(K4 * GG, dtype=torch.float32, device=dev)
    temperature = torch.as_tensor(T, device=dev)
    walker = torch.arange(K4 * GG, dtype=torch.int32, device=dev)
    attempted = torch.zeros(GG, K4 - 1, dtype=torch.int64, device=dev)
    accepted = torch.zeros_like(attempted)
    attempt = torch.zeros(1, dtype=torch.int64, device=dev)
    decision = torch.zeros(GG, K4 - 1, dtype=torch.uint8, device=dev)
    table = _lib.STRUCTS["spk_remd_buffers_t"]()
    table.n_buffers, table.per_atom[0], table.width[0], table.data[0] = 1, 0, 1, energy.data_ptr()
    ex = RO.Exchange(K4, GG, kB, seed)
    rng = np.random.default_rng(4)
    sums = np.zeros(K4)
    rounds = 40
    for r in range(rounds):
        e32 = (rng.gamma(d / 2.0, kB * T) / e_conv).astype(np.float32)
        energy.copy_(torch.as_tensor(e32))
        _lib.call("spk_remd_exchange", ops._p(energy), e_conv, ops._p(temperature), kB, None, None, 0, GG, K4, seed,
                  None, 1, ops._p(attempt), ops._p(walker), ops._p(attempted), ops._p(accepted), ops._p(decision), None,
                  ctypes.byref(table), ops._stream())
        U = e32.astype(np.float64) * e_conv
        acc = ex.step(U, T)
        _, _, (e_ref,) = RO.swap(acc, K4, GG, None, T, None, per_system=[e32])
        if r < 6:
            assert np.array_equal(_np(decision).astype(bool), acc), r
            assert np.array_equal(_np(walker), ex.walker)
            assert np.array_equal(_np(attempted), ex.attempted) and np.array_equal(_np(accepted), ex.accepted)
            assert np.array_equal(_np(energy), e_ref)
            assert int(attempt.item()) == r + 1
        sums += _np(energy).astype(np.float64).reshape(K4, GG).mean(1) * e_conv
    assert np.array_equal(_np(walker), ex.walker) and np.array_equal(_np(accepted), ex.accepted)
    expect = d * kB * 300.0 * 1.2 ** np.arange(K4) / 2.0
    sigma = expect * math.sqrt(2.0 / d) / math.sqrt(GG * rounds)
    assert np.all(np.abs(sums / rounds - expect) < 5.0 * sigma), (sums / rounds, expect)
    p = ex.accepted / np.maximum(ex.attempted, 1)
    assert 0.05 < p.mean() < 0.95


# ---- ReplicaExchange in DeviceMD ------------------------------------------------------------------------------------------
def _snapshot(md, remd):
    return dict(x=_np(md.positions), mp=_np(md._mp), p=_np(md.momenta), f=_np(md.forces), e=_np(md.energy),
                pe=_np(md.properties["energy"]).reshape(-1), pf=_np(md.properties["forces"]).reshape(-1, 3),
                step=int(md._rec_counter[0].item()), walker=_np(remd._walker), attempted=_np(remd._attempted),
                accepted=_np(remd._accepted), attempt=int(remd._attempt.item()), decision=_np(remd._decision))


def _within_ulp(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return bool(np.all(np.abs(a.astype(np.float64) - b) <= np.spacing(np.maximum(np.abs(a), np.abs(b)))))


def test_exchange_in_device_md_follows_the_oracle():
    """Eager steps with an exchange every 2 steps; the state just before and after the hook is compared with the
    oracle's attempt on the state before.  Copies are bitwise, rescaled momenta within one ulp; after a step with swaps
    the forces equal a fresh evaluation at the swapped positions."""
    from schnetpack_b200 import md as M
    from schnetpack_b200.exchange import ReplicaExchange
    from schnetpack_b200.neighbors import CellListNeighborList

    every, e_conv, seed = 2, 0.5, 3
    remd = ReplicaExchange(K, every, seed=seed)
    md = _run(M.LangevinThermostat(_temps(), 20.0, seed=1), hooks=[remd], use_graph=False, position_conversion=2.0,
              energy_conversion=e_conv, required_properties=["energy", "forces"], property_conversion={"energy": 2.0},
              initializer=M.MaxwellBoltzmannInit(_temps(), seed=2))
    assert md._mp is not None
    T = _np(md.thermostat.temperatures)
    sys_ptr = _np(md.systems.sys_ptr)
    pre, post = [], []
    orig = remd.apply

    def spy(run):
        pre.append(_snapshot(run, remd))
        orig(run)
        post.append(_snapshot(run, remd))

    remd.apply = spy
    swaps, fresh_checked = 0, False
    for _ in range(16):
        md.run(1)
        a, b = pre[-1], post[-1]
        if a["step"] % every:
            for key in ("x", "mp", "p", "f", "e", "pe", "pf", "walker", "attempted", "accepted"):
                assert np.array_equal(a[key], b[key]), key
            assert b["attempt"] == a["attempt"]
            continue
        ex = RO.Exchange(K, G, md.thermostat.kB, seed)
        ex.walker, ex.attempted, ex.accepted, ex.attempt = (a["walker"].astype(np.int64), a["attempted"].copy(),
                                                            a["accepted"].copy(), a["attempt"])
        acc = ex.step(a["e"].astype(np.float64) * e_conv, T)
        p, (x, mp, f, pf), (e, pe) = RO.swap(acc, K, G, sys_ptr, T, a["p"], [a["x"], a["mp"], a["f"], a["pf"]],
                                             [a["e"], a["pe"]])
        assert np.array_equal(b["decision"].astype(bool), acc)
        for key, ref in (("x", x), ("mp", mp), ("f", f), ("pf", pf), ("e", e), ("pe", pe)):
            assert np.array_equal(b[key], ref), key
        assert _within_ulp(b["p"], p)
        assert np.array_equal(b["walker"], ex.walker) and b["attempt"] == ex.attempt
        assert np.array_equal(b["attempted"], ex.attempted) and np.array_equal(b["accepted"], ex.accepted)
        swaps += int(acc.sum())
        if acc.any() and not fresh_checked:
            x_in = {k: (v.detach().clone() if v.is_floating_point() else v) for k, v in md.static.items()}
            x_in["_positions"] = md.model_positions.clone()
            nl = CellListNeighborList(md.nl._cutoff, capacity=md.nl.capacity, pad=True)
            out = md.model(nl(x_in))
            assert rel_err(_np(md.forces), _np(out["forces"])) < 1e-6
            assert rel_err(_np(md.energy), _np(out["energy"])) < 1e-6
            fresh_checked = True
    assert swaps > 0 and fresh_checked
    assert remd.attempts == 8
    assert np.array_equal(_np(remd.walkers()).reshape(-1), post[-1]["walker"])


def _recorded_run(use_graph=True):
    from schnetpack_b200 import md as M
    from schnetpack_b200.exchange import ReplicaExchange

    remd = ReplicaExchange(K, 3, seed=9)
    md = _run(M.LangevinThermostat(_temps(), 20.0, seed=4), hooks=[M.RemoveCOMMotion(5, False), remd],
              use_graph=use_graph, required_properties=["energy"], record_capacity=64,
              initializer=M.MaxwellBoltzmannInit(_temps(), seed=2))
    return md, remd


def test_graph_replay_equals_eager_and_restart_is_bitwise():
    runs = {}
    for use_graph in (True, False):
        md, remd = _recorded_run(use_graph)
        md.run(30)
        torch.cuda.synchronize()
        runs[use_graph] = (md, remd)
    (g, rg), (e, re_) = runs[True], runs[False]
    assert torch.equal(g.positions, e.positions) and torch.equal(g.momenta, e.momenta)
    assert torch.equal(g.energy, e.energy) and torch.equal(g.forces, e.forces)
    for k, v in rg._state().items():
        assert torch.equal(v, re_._state()[k]), k
    assert torch.equal(g.recorded("walker"), e.recorded("walker"))
    assert rg.attempts == 10 and int(rg._accepted.sum()) > 0

    a, ra = _recorded_run()
    a.run(15)
    saved = a.state_dict()
    a.run(15)
    b, rb = _recorded_run()
    b.load_state_dict(saved)
    b.run(15)
    torch.cuda.synchronize()
    assert torch.equal(a.positions, b.positions) and torch.equal(a.momenta, b.momenta)
    assert torch.equal(a.forces, b.forces) and torch.equal(a.energy, b.energy)
    for k, v in ra._state().items():
        assert torch.equal(v, rb._state()[k]), k
    assert torch.equal(a.recorded("walker"), b.recorded("walker"))
    assert torch.equal(a.recorded("walker"), g.recorded("walker"))          # 30 steps in one go
    walkers = a.recorded("walker")
    assert walkers.shape == (30, K, G) and torch.equal(walkers[-1], ra.walkers())
    assert (walkers.sort(1).values == torch.arange(K * G).reshape(K, G)).all()   # a permutation inside every group
    # drain empties the recorder and leaves the exchange alone; reset zeroes the statistics only
    before = {k: v.clone() for k, v in ra._state().items()}
    a.drain()
    for k, v in ra._state().items():
        assert torch.equal(v, before[k]), k
    ra.reset()
    assert int(ra._attempted.sum()) == 0 and torch.equal(ra._walker, before["walker"])
    assert torch.isnan(ra.acceptance()).all()


MASS_ETHANOL = {1: 1.008, 6: 12.011, 8: 15.999}


def test_exchange_samples_every_rung_at_its_temperature():
    """8 trained-PaiNN ethanol molecules at 4 rungs (300 K x 1.15^k), Langevin with tau = 50 fs, dt = 0.5 fs, exchanges
    every 20 steps: 4000 steps of equilibration, then 16 000 steps sampled every 20.  A rung's kinetic temperature over
    8 molecules of 9 atoms fluctuates by 0.27 T / sqrt(8) per sample; with ~160 decorrelated samples (one per 50 fs) its
    mean lies within 2 % of T at 3 sigma, so 4 % is asked."""
    from schnetpack_b200 import md as M
    from schnetpack_b200.exchange import ReplicaExchange
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params, inputs, _, _ = load_case("painn_md_ethanol_trained")
    n_mol = inputs["_n_atoms"].shape[0]
    copies = 8 // n_mol
    n = inputs["_positions"].shape[0]
    base = {"_positions": np.tile(inputs["_positions"], (copies, 1)),
            "_atomic_numbers": np.tile(inputs["_atomic_numbers"], copies),
            "_n_atoms": np.tile(inputs["_n_atoms"], copies),
            "_idx_m": (np.tile(inputs["_idx_m"], copies) + np.repeat(np.arange(copies) * n_mol, n)).astype(np.int64),
            "_cell": np.tile(inputs["_cell"], (copies, 1, 1)),
            "_pbc": np.tile(inputs["_pbc"].reshape(n_mol, 3), (copies, 1)).reshape(-1)}
    GE = copies * n_mol
    dev = torch.device(DEV)
    b = M.replicate_batch(batch_to_device(base, dev), K, GE)
    masses = torch.tensor([MASS_ETHANOL[int(z)] for z in b["_atomic_numbers"].tolist()])
    ladder = [300.0 * 1.15 ** k for k in range(K)]
    temps = [t for t in ladder for _ in range(GE)]
    remd = ReplicaExchange(K, 20, seed=11)
    md = M.DeviceMD(from_spec(spec, params, dev), b, masses, time_step=0.5 * M.FS_MD, cutoff=spec["cutoff"],
                    capacity=K * GE * 9 * 8 * 2, position_conversion=10.0, energy_conversion=4.184,
                    thermostat=M.LangevinThermostat(temps, 50.0, seed=1), hooks=[remd],
                    initializer=M.MaxwellBoltzmannInit(temps, seed=3))
    md.run(4000)
    remd.reset()
    t_sum, u_sum, n_samples = torch.zeros(K, dtype=torch.float64, device=dev), torch.zeros(K, dtype=torch.float64,
                                                                                            device=dev), 800
    for _ in range(n_samples):
        md.run(20)
        t_sum += md.temperature().reshape(K, GE).mean(1)
        u_sum += md.potential_energy().double().reshape(K, GE).mean(1)
    t_mean = _np(t_sum) / n_samples
    u_mean = _np(u_sum) / n_samples
    assert np.all(np.abs(t_mean / np.array(ladder) - 1.0) < 0.04), t_mean
    assert np.all(np.diff(u_mean) > 0.0), u_mean
    acc = _np(remd.acceptance())
    assert acc.shape == (GE, K - 1) and np.all((acc > 0.0) & (acc < 1.0)), acc
    assert np.isfinite(_np(md.positions)).all()


# ---- refusals -------------------------------------------------------------------------------------------------------------
def _refusal_case(name):
    from schnetpack_b200 import md as M
    from schnetpack_b200 import spectra as SP
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.exchange import ReplicaExchange
    from schnetpack_b200.model import batch_to_device
    from schnetpack_b200.structure import MeanSquaredDisplacement

    b, masses = _mixed()
    lang = M.LangevinThermostat(_temps(), 20.0)
    kw = dict(thermostat=lang, hooks=[ReplicaExchange(K, 5)])
    if name == "n_sys":
        kw["hooks"] = [ReplicaExchange(5, 5)]
    elif name == "no_thermostat":
        kw["thermostat"] = None
    elif name == "scalar":
        kw["thermostat"] = M.LangevinThermostat(300.0, 20.0)
    elif name == "berendsen":
        kw["thermostat"] = M.BerendsenThermostat(300.0, 20.0)
    elif name == "ladder":
        kw["thermostat"] = M.NHCThermostat(_temps()[::-1], 20.0)
    elif name == "atom_counts":
        data = S.qm9like_batch(K * G, seed=0)
        b = {k: v for k, v in batch_to_device(data, torch.device(DEV)).items()
             if k not in (S.idx_i, S.idx_j, S.offsets)}
        masses = torch.tensor([MASS[int(z)] for z in b[S.Z].tolist()], dtype=torch.float32)
    elif name == "atomic_numbers":
        b[S.Z] = b[S.Z].clone()
        b[S.Z][-1] = 9 if int(b[S.Z][-1]) != 9 else 8
    elif name == "masses":
        masses = masses.clone()
        masses[-2] += 1.0
    elif name == "cell":
        b[S.cell] = b[S.cell].clone()
        b[S.cell][G + 1] = torch.eye(3, device=DEV) * 50.0
    elif name == "pbc":
        b[S.cell] = (torch.eye(3, device=DEV) * 60.0).expand(K * G, 3, 3).contiguous()
        b[S.pbc] = b[S.pbc].clone()
        b[S.pbc][3 * (G + 1)] = True
    elif name == "compute_stress":
        kw["compute_stress"] = True
    elif name == "ring_polymer":
        kw.update(thermostat=None, ring_polymer=M.RingPolymer(2, 300.0))
    elif name == "ensemble":
        kw["model"] = (_model()[0], [_model(3)[1], _model(4)[1]])
    elif name == "msd":
        kw["hooks"] = [MeanSquaredDisplacement(10), ReplicaExchange(K, 5)]
    elif name == "stream":
        kw["stream"] = SP.SpectrumStream("power", resolution=64)
    elif name == "two_hooks":
        kw["hooks"] = [ReplicaExchange(K, 5), ReplicaExchange(K, 7)]
    return b, masses, kw


REFUSALS = {"n_sys": "not K G", "no_thermostat": "needs a LangevinThermostat", "scalar": "needs a LangevinThermostat",
            "berendsen": "needs a LangevinThermostat", "ladder": "increase strictly", "atom_counts": "atom counts",
            "atomic_numbers": "atomic numbers", "masses": "masses", "cell": "_cell", "pbc": "_pbc",
            "compute_stress": "NPT-REMD", "ring_polymer": "ring-polymer", "ensemble": "ensembles",
            "msd": "MeanSquaredDisplacement", "stream": "SpectrumStream", "two_hooks": "one exchange hook"}


@pytest.mark.parametrize("name", sorted(REFUSALS))
def test_device_md_refuses_what_replica_exchange_does_not_support(name):
    b, masses, kw = _refusal_case(name)
    model = kw.pop("model", None)
    thermostat, hooks = kw.pop("thermostat"), kw.pop("hooks")
    with pytest.raises((ValueError, NotImplementedError), match=REFUSALS[name]):
        _run(thermostat, hooks, batch=b, masses=masses, model=model, **kw)
