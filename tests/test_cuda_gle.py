"""GLE, RPMD-GLE and PIGLET thermostats on the device (csrc/rpmd.cu ``spk_rpmd_gle``, schnetpack_b200.md) against the fp64
oracle tests/gle_oracle.py with the propagator of the GLE papers ("paper"); the oracle's "reference" convention is pinned to
the reference's own classes in tests/test_gle_oracle.py."""
import math
import os

import numpy as np
import pytest
import scipy.linalg as SL
import torch

import gle_oracle as GO
import rpmd_oracle as RO
import test_cuda_rpmd as TR
from conftest import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EXACT, HBAR_EXACT, T_EXACT, DT_EXACT = TR.EXACT, TR.HBAR_EXACT, TR.T_EXACT, TR.DT_EXACT
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _np(t):
    return t.detach().cpu().numpy()


def _synthetic_a(rng, D, scale):
    """S + K in fs^-1: S symmetric positive definite, K antisymmetric -- positive-stable and non-normal"""
    Q, _ = np.linalg.qr(rng.normal(size=(D, D)))
    S = Q @ np.diag(scale * rng.uniform(0.2, 3.0, D)) @ Q.T
    K = rng.normal(size=(D, D)) * scale
    return 0.5 * (S + S.T) + 0.5 * (K - K.T)


def _gle_file(path, D, n_blocks, seed, scale=1.0, with_c=True, c00=None, same=False):
    """a gle4md file of n_blocks synthetic GLEs (A in fs^-1, C in K solving A C + C A^T = B B^T); ``same``: every block
    is the first one"""
    rng = np.random.default_rng(seed)
    As, Cs = [], []
    for k in range(n_blocks):
        if same and k:
            As.append(As[0])
            Cs.append(Cs[0])
            continue
        A = _synthetic_a(rng, D, scale)
        B = rng.normal(size=(D, D))
        C = SL.solve_continuous_lyapunov(A, B @ B.T)
        C = 0.5 * (C + C.T)
        As.append(A)
        Cs.append(C * ((c00 or T_EXACT * (1.0 + 0.2 * k)) / C[0, 0]))
    GO.write_gle_file(path, np.stack(As), np.stack(Cs) if with_c else None)
    return str(path)


def _thermostat(md, path, P, seed=11, kind=None):
    if kind == "classical":
        return md.GLEThermostat(T_EXACT, path, seed=seed, **EXACT)
    if kind == "piglet":
        return md.PIGLETThermostat(T_EXACT, path, seed=seed, **EXACT)
    return md.RPMDGLEThermostat(T_EXACT, path, seed=seed, **EXACT)


def _oracle(md, path, per_mode, seed=11):
    A, C = md.load_gle_matrices(path, **EXACT)
    return GO.GLE(A.numpy(), None if C is None else C.numpy(), T_EXACT, EXACT["kB"], GO.philox_noise(seed),
                  convention="paper", per_mode=per_mode)


def _small_mixed_batch(P, seed=3):
    """the mixed batch of test_cuda_rpmd.py with its large system cut to 3000 atoms (the oracle holds [P, N, 3, D])"""
    n_atoms = [1, 3, 9, 3000, 20, 1, 5]
    rng = np.random.default_rng(seed + P)
    n = sum(n_atoms)
    masses = rng.choice([1.0, 12.0, 16.0], size=n).astype(np.float32)
    p = (rng.normal(size=(P, n, 3)) * np.sqrt(masses * EXACT["kB"] * 300.0 * P)[None, :, None]).astype(np.float32)
    return n_atoms, masses, p


# ---- 1. kernel against the oracle ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("per_mode", [False, True])
@pytest.mark.parametrize("P", [1, 4, 5, 8, 32])
@pytest.mark.parametrize("D", [2, 5, 9, 16])
def test_gle_kernel_follows_the_oracle(tmp_path, D, P, per_mode):
    from schnetpack_b200 import md

    path = _gle_file(tmp_path / "g.txt", D, P if per_mode else 1, seed=D * 100 + P)
    n_atoms, masses, p = _small_mixed_batch(P)
    base, rp = TR._bind(P, n_atoms, masses)
    th = _thermostat(md, path, P, kind="piglet" if per_mode else None)
    th.bind(base, DT_EXACT, rp)
    ref = _oracle(md, path, per_mode)
    ref.init(TR._rp_oracle(P), masses.astype(np.float64), n_atoms)
    torch.cuda.synchronize()
    assert rel_err(_np(th.state).reshape(ref.s.shape), ref.s) < 1e-12          # the free-particle-limit start
    pt = torch.as_tensor(p, device=DEV).reshape(-1, 3)
    pr = torch.as_tensor(p, dtype=torch.float64)
    for _ in range(3):
        th.apply(pt)
        pr = ref.apply(pr)
    torch.cuda.synchronize()
    got = _np(pt).reshape(p.shape)
    assert np.isfinite(got).all()
    assert rel_err(got, pr.numpy()) < 1e-5
    assert rel_err(_np(th.state).reshape(ref.s.shape), ref.s) < 1e-5
    assert np.abs(pr.numpy() - p).max() > 1e-2 * np.abs(p).max()                # the thermostat acted
    assert th.counter.tolist() == [4, 0]


# ---- 2. noise, graph replay, restarts --------------------------------------------------------------------------------------
def test_graph_replays_draw_fresh_noise_and_equal_the_eager_loop(tmp_path):
    from schnetpack_b200 import md

    P, D = 8, 5
    path = _gle_file(tmp_path / "g.txt", D, 1, seed=1)
    n_atoms, masses, p = _small_mixed_batch(P)
    base, rp = TR._bind(P, n_atoms, masses)
    runs = []
    for use_graph in (True, False):
        th = _thermostat(md, path, P)
        th.bind(base, DT_EXACT, rp)
        pt = torch.as_tensor(p, device=DEV).reshape(-1, 3)
        if use_graph:
            g = torch.cuda.CUDAGraph()
            saved = th.state_dict()
            p_saved = pt.clone()
            with torch.cuda.graph(g):
                th.apply(pt)
            th.load_state_dict(saved)                 # capture does not run the kernel; keep the start anyway
            pt.copy_(p_saved)
            for _ in range(3):
                g.replay()
        else:
            for _ in range(3):
                th.apply(pt)
        torch.cuda.synchronize()
        runs.append((pt.clone(), th.state.clone(), th.counter.tolist()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    assert runs[0][2] == runs[1][2] == [4, 0]
    ref = _oracle(md, path, False)
    ref.init(TR._rp_oracle(P), masses.astype(np.float64), n_atoms)
    pr = torch.as_tensor(p, dtype=torch.float64)
    for _ in range(3):
        pr = ref.apply(pr)
    assert rel_err(_np(runs[0][0]).reshape(p.shape), pr.numpy()) < 1e-5       # applications 1, 2, 3: fresh noise


def test_device_md_graph_equals_eager_and_restart_is_bitwise():
    from schnetpack_b200 import md as M

    path = os.path.join(GOLDEN, "gle_nonnormal.txt")
    case = TR._box_case()
    runs = {}
    for use_graph in (True, False):
        dmd, _ = TR._device_md(case, 4, M.RPMDGLEThermostat(300.0, path, seed=5), use_graph=use_graph)
        dmd.run(10)
        torch.cuda.synchronize()
        runs[use_graph] = (_np(dmd.positions), _np(dmd.momenta), dmd.thermostat.state_dict())
    assert rel_err(runs[True][0], runs[False][0]) < 1e-6
    assert rel_err(runs[True][1], runs[False][1]) < 1e-5
    assert runs[True][2]["counter"].tolist() == runs[False][2]["counter"].tolist() == [21, 0]

    a, _ = TR._device_md(case, 4, M.RPMDGLEThermostat(300.0, path, seed=5))
    a.run(4)
    saved = a.state_dict()
    a.run(4)
    b, _ = TR._device_md(case, 4, M.RPMDGLEThermostat(300.0, path, seed=5))
    b.load_state_dict(saved)
    b.run(4)
    torch.cuda.synchronize()
    assert torch.equal(a.positions, b.positions) and torch.equal(a.momenta, b.momenta)
    assert torch.equal(a.forces, b.forces) and torch.equal(a.energy, b.energy)
    for k, v in a.thermostat.state_dict().items():
        assert torch.equal(v, b.thermostat.state_dict()[k]), k


# ---- 3. invariants ------------------------------------------------------------------------------------------------------------
def test_classical_gle_equals_rpmd_gle_at_one_bead_bitwise(tmp_path):
    from schnetpack_b200 import md

    path = _gle_file(tmp_path / "g.txt", 9, 1, seed=4)
    n_atoms, masses, p = _small_mixed_batch(1)
    base, rp = TR._bind(1, n_atoms, masses)
    out = []
    for kind in ("classical", None):
        th = _thermostat(md, path, 1, kind=kind)
        if kind == "classical":
            th.bind(base, DT_EXACT)
        else:
            th.bind(base, DT_EXACT, rp)
        pt = torch.as_tensor(p, device=DEV).reshape(-1, 3)
        for _ in range(5):
            th.apply(pt)
        torch.cuda.synchronize()
        out.append((pt, th.state))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


@pytest.mark.parametrize("P", [4, 8])
def test_piglet_with_identical_blocks_equals_rpmd_gle_bitwise(tmp_path, P):
    from schnetpack_b200 import md

    one = _gle_file(tmp_path / "one.txt", 5, 1, seed=7)
    same = _gle_file(tmp_path / "same.txt", 5, P, seed=7, same=True)
    n_atoms, masses, p = _small_mixed_batch(P)
    base, rp = TR._bind(P, n_atoms, masses)
    out = []
    for path, kind in ((one, None), (same, "piglet")):
        th = _thermostat(md, path, P, kind=kind)
        th.bind(base, DT_EXACT, rp)
        pt = torch.as_tensor(p, device=DEV).reshape(-1, 3)
        for _ in range(5):
            th.apply(pt)
        torch.cuda.synchronize()
        out.append((pt, th.state))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


# ---- 4. physics: the Ornstein-Uhlenbeck process of the non-canonical GLE ----------------------------------------------------
def test_thermostat_only_run_samples_m_c_and_not_the_reference_covariance():
    """70 000 free atoms (210 000 degrees of freedom) of mass 2 under the non-canonical fixture gle_quantum.txt alone: after
    4000 applications (2000 fs), 20 snapshots 400 applications apart.  Every entry of the sample covariance of (p, s)
    must lie within 5 standard errors (from the 20 snapshot means) of m C; the stationary <p^2> of the reference's
    transposed propagator must lie more than 10 standard errors away."""
    from schnetpack_b200 import md

    N, mass = 70_000, 2.0
    th = md.GLEThermostat(300.0, os.path.join(GOLDEN, "gle_quantum.txt"), seed=3)
    idx_m = torch.zeros(N, dtype=torch.int64, device=DEV)
    systems = md._Systems(torch.full((N,), mass, device=DEV), idx_m, 1)
    th.bind(systems, 1.0 * md.FS_MD)
    p = torch.zeros(N, 3, device=DEV)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(200):
            th.apply(p)
    for _ in range(20):
        g.replay()
    covs = []
    for _ in range(20):
        g.replay()
        g.replay()
        s = th.state.double()
        covs.append(_np(s.T @ s / s.shape[0] / mass))
    covs = np.asarray(covs)
    mean, se = covs.mean(0), covs.std(0, ddof=1) / math.sqrt(len(covs))
    C = _np(th.C[0])
    z = np.abs(mean - C) / se
    c1, c2 = _np(th.c1[0]), _np(th.c2[0])
    ref00 = GO.stationary_covariance(c1, c2, "reference")[0, 0]
    print(f"GLE OU: <p^2>/m = {mean[0, 0]:.6g} +- {se[0, 0]:.2g}, C00 = {C[0, 0]:.6g}, max |z| = {z.max():.2f}; "
          f"reference map predicts {ref00:.6g} ({abs(ref00 - C[0, 0]) / se[0, 0]:.0f} standard errors away)")
    assert (z < 5.0).all(), z
    assert abs(ref00 - C[0, 0]) > 10.0 * se[0, 0]


# ---- 5. physics: trained ethanol ------------------------------------------------------------------------------------------------
def _ethanol_units():
    from schnetpack_b200 import md as M

    kcal, angstrom = 4.184, 0.1
    t_unit = angstrom / math.sqrt(kcal)
    return M.KB_MD / kcal, M.FS_MD / t_unit, M.HBAR_MD / (kcal * t_unit)


def test_trained_ethanol_nvt_with_canonical_gle_reaches_300K():
    """256 trained ethanol molecules (2304 atoms) in the model's units, the canonical non-normal fixture gle_nonnormal.txt
    at 300 K, dt = 0.5 fs from rest: after 2000 steps, 4000 more sampled every 10; the mean temperature must lie within 5
    standard errors (20 block means, below 1 % of 300 K) of 300 K"""
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params, b = TR._ethanol_batch(128)
    dev = torch.device(DEV)
    model = from_spec(spec, params, dev)
    masses = torch.tensor([TR.MASS[int(z)] for z in b["_atomic_numbers"]])
    kB, fs, _ = _ethanol_units()
    th = M.GLEThermostat(300.0, os.path.join(GOLDEN, "gle_nonnormal.txt"), seed=4, kB=kB, fs=fs)
    dmd = M.DeviceMD(model, batch_to_device(b, dev), masses, time_step=0.5 * fs, cutoff=spec["cutoff"],
                     capacity=masses.shape[0] * 12, thermostat=th)
    dmd.run(2000)
    temps = []
    for _ in range(400):
        dmd.run(10)
        temps.append(float(dmd.temperature().mean()))
    m, s = RO.block_mean(temps)
    print(f"GLE NVT ethanol: {m:.1f} +- {s:.1f} K")
    assert s < 0.01 * 300.0, s
    assert abs(m - 300.0) < 5.0 * s, (m, s)


def test_trained_ethanol_piglet_reaches_the_centroid_and_bead_temperatures(tmp_path):
    """the same batch at P = 8 with PIGLET, one canonical block per normal mode (A in fs^-1, no C, so C = P kB T I): after
    2000 steps of 0.5 fs, 4000 more sampled every 10.  The centroid temperature must lie within 5 standard errors of
    300 K and the bead temperature within 5 standard errors of P 300 K, each error below 1 % of its target"""
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device, from_spec

    P, T = 8, 300.0
    path = _gle_file(tmp_path / "piglet8.txt", 4, P, seed=8, scale=0.1, with_c=False)
    spec, params, b = TR._ethanol_batch(16)
    dev = torch.device(DEV)
    model = from_spec(spec, params, dev)
    masses = torch.tensor([TR.MASS[int(z)] for z in b["_atomic_numbers"]])
    kB, fs, hbar = _ethanol_units()
    th = M.PIGLETThermostat(T, path, seed=6, kB=kB, fs=fs)
    dmd = M.DeviceMD(model, batch_to_device(b, dev), masses, time_step=0.5 * fs, cutoff=spec["cutoff"],
                     capacity=P * masses.shape[0] * 12, thermostat=th, ring_polymer=M.RingPolymer(P, T, kB=kB, hbar=hbar))
    dmd.run(2000)
    tc, tb = [], []
    for _ in range(400):
        dmd.run(10)
        tc.append(float(dmd.centroid_temperature().mean()))
        tb.append(float(dmd.temperature().mean()))
    mc, sc = RO.block_mean(tc)
    mb, sb = RO.block_mean(tb)
    print(f"PIGLET ethanol: centroid {mc:.1f} +- {sc:.1f} K, beads {mb:.1f} +- {sb:.1f} K (P T = {P * T:.0f} K)")
    assert sc < 0.01 * T and sb < 0.01 * P * T, (sc, sb)
    assert abs(mc - T) < 5.0 * sc, (mc, sc)
    assert abs(mb - P * T) < 5.0 * sb, (mb, sb)


# ---- 6. refusals and the barostat -------------------------------------------------------------------------------------------
def test_argument_errors():
    from schnetpack_b200 import _lib, ops
    from schnetpack_b200 import md as M

    piglet = os.path.join(GOLDEN, "gle_piglet_p4.txt")
    nonnormal = os.path.join(GOLDEN, "gle_nonnormal.txt")
    n_atoms, masses, _ = _small_mixed_batch(8)
    base, rp = TR._bind(8, n_atoms, masses)
    with pytest.raises(ValueError, match="expected 8 A matrices"):
        M.PIGLETThermostat(300.0, piglet).bind(base, DT_EXACT, rp)
    with pytest.raises(ValueError, match="ring-polymer thermostat"):
        M.RPMDGLEThermostat(300.0, nonnormal).bind(base, DT_EXACT)
    case = TR._box_case()
    with pytest.raises(ValueError, match="classical thermostat"):
        TR._device_md(case, 2, M.GLEThermostat(300.0, nonnormal))
    with pytest.raises(ValueError, match="ring-polymer thermostat"):
        TR._device_md(case, None, M.PIGLETThermostat(300.0, piglet), momenta=np.zeros((150, 3)))
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params, data, m, dt = case
    model = from_spec(spec, params, torch.device(DEV))
    with pytest.raises(ValueError, match="own thermostat"):
        M.DeviceMD(model, batch_to_device(data, torch.device(DEV)), torch.as_tensor(m), dt, spec["cutoff"], 10**6,
                   thermostat=M.GLEThermostat(300.0, nonnormal), barostat=M.NHCBarostatIsotropic(1.0, 300.0, 100.0))
    p = torch.zeros(10, 3, device=DEV)
    mm = torch.ones(10, device=DEV)
    c = torch.ones(1, 1, dtype=torch.float64, device=DEV)
    mats = torch.zeros(17, 17, dtype=torch.float64, device=DEV)
    state = torch.zeros(30, 17, dtype=torch.float64, device=DEV)
    counter = torch.zeros(2, dtype=torch.int64, device=DEV)
    for D in (0, 17):
        with pytest.raises(ValueError):
            _lib.call("spk_rpmd_gle", ops._p(p), ops._p(mm), 10, 1, ops._p(c), ops._p(mats), ops._p(mats), D, 0,
                      ops._p(state), 0, ops._p(counter), 0, ops._stream())
    with pytest.raises(ValueError):                                  # no state
        _lib.call("spk_rpmd_gle", ops._p(p), ops._p(mm), 10, 1, ops._p(c), ops._p(mats), ops._p(mats), 4, 0, None, 0,
                  ops._p(counter), 0, ops._stream())


def test_rpmd_gle_runs_next_to_the_pile_barostat():
    """the periodic PaiNN box at P = 4 in MD units (p_conv = 10, e_conv = 0.5; a 1.5 nm^3 box) at 1000 bar, as the
    NPT-RPMD trajectory tests run it"""
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params, data, masses, dt = TR._box_case()
    P, N = 4, data["_positions"].shape[0]
    p0 = np.random.default_rng(2).normal(size=(P, N, 3)) * np.sqrt(masses * M.KB_MD * 300.0 * P)[None, :, None]
    dmd = M.DeviceMD(from_spec(spec, params, torch.device(DEV)), batch_to_device(data, torch.device(DEV)),
                     torch.as_tensor(masses), time_step=dt, cutoff=spec["cutoff"], capacity=N * P * 80,
                     position_conversion=10.0, energy_conversion=0.5,
                     momenta=torch.as_tensor(p0), thermostat=M.RPMDGLEThermostat(300.0, os.path.join(
                         GOLDEN, "gle_nonnormal.txt"), seed=3),
                     barostat=M.PILEBarostat(1000.0, 300.0, 100.0, seed=2), ring_polymer=M.RingPolymer(P, 300.0))
    v0 = dmd.volume().clone()
    dmd.run(20)
    torch.cuda.synchronize()
    assert torch.isfinite(dmd.momenta).all() and torch.isfinite(dmd.positions).all()
    assert dmd.thermostat.counter.tolist() == [41, 0]
    assert dmd.barostat.counter.tolist() == [40, 0]
    assert not torch.equal(dmd.volume(), v0)
