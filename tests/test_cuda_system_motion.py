"""Motion removal, wrapping, initial momenta and the basic simulation hooks on the device (csrc/system_motion.cu,
schnetpack_b200.md) against the fp64 oracle tests/system_oracle.py, which is pinned to the reference's own classes
(tests/test_system_oracle.py)."""
import math

import numpy as np
import pytest
import torch

import nvt_oracle as NO
import system_oracle as SO
from conftest import load_case, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DRAW_APP = 2 ** 64 - 1          # SPK_MOTION_DRAW_APPLICATION
F32 = 2.0 ** -24


def _np(t):
    return t.detach().cpu().numpy()


# ---- the kernels on a ragged batch ------------------------------------------------------------------------------------------
def _ragged(seed=1):
    """an empty system, 1 atom, a linear triatomic, water, 9 atoms and a 20 000-atom box whose centre of mass lies 10^3
    length units from the origin; momenta near 300 K in the reference's MD units"""
    rng = np.random.default_rng(seed)
    n_atoms = [0, 1, 3, 3, 9, 20_000]
    axis = np.array([0.3, -0.8, 0.52]) / np.linalg.norm([0.3, -0.8, 0.52])
    parts = [np.array([[0.4, -1.0, 2.0]]),
             np.array([1.0, 1.0, 1.0]) + np.array([-0.116, 0.0, 0.116])[:, None] * axis,
             np.array([[0.0, 0.0, 0.0], [0.0757, 0.0586, 0.0], [-0.0757, 0.0586, 0.0]]) + 0.3,
             rng.normal(size=(9, 3)) * 0.15 - 2.0,
             rng.uniform(0.0, 6.0, size=(20_000, 3)) + np.array([600.0, -500.0, 600.0])]
    x = np.concatenate(parts).astype(np.float32)
    masses = rng.choice([1.008, 12.011, 15.999], size=x.shape[0]).astype(np.float32)
    p = (rng.normal(size=x.shape) * np.sqrt(masses * 0.0083144598 * 300.0)[:, None]).astype(np.float32)
    return n_atoms, masses, x, p


def _systems(n_atoms, masses):
    from schnetpack_b200.md import _Systems

    idx_m = torch.repeat_interleave(torch.arange(len(n_atoms)), torch.tensor(n_atoms)).to(DEV)
    return _Systems(torch.as_tensor(masses, device=DEV), idx_m, len(n_atoms))


def _remove(sy, x, p, flags, mx=None, p_conv=1.0, step=None, every=1):
    from schnetpack_b200 import _lib, ops

    ws = sy.workspace("spk_md_motion_workspace_bytes")
    _lib.call("spk_md_remove_motion", ops._p(x), ops._p(mx), ops._p(p), ops._p(sy.masses), ops._p(sy.idx_m),
              ops._p(sy.sys_ptr), sy.n_atoms, sy.n_sys, flags, p_conv, ops._p(step), every, ops._p(ws), ws.numel(),
              ops._stream())


def _replicas(n_atoms, masses, x, p, P, seed=2):
    """P bead copies of the batch as P P-fold systems, each bead displaced and with its own momenta"""
    rng = np.random.default_rng(seed)
    xs = np.concatenate([x + (0.01 * k) * rng.normal(size=x.shape).astype(np.float32) for k in range(P)])
    ps = np.concatenate([p * (1.0 + 0.1 * k) for k in range(P)]).astype(np.float32)
    return n_atoms * P, np.tile(masses, P), xs, ps


@pytest.mark.parametrize("P", [1, 4, 8])
@pytest.mark.parametrize("rotation", [False, True])
def test_motion_removal_follows_the_oracle(P, rotation):
    from schnetpack_b200 import _lib

    n_atoms, masses, x, p = _replicas(*_ragged(), P)
    sy = _systems(n_atoms, masses)
    flags = _lib.MOTION_CENTER_OF_MASS | _lib.MOTION_TRANSLATION | (_lib.MOTION_ROTATION if rotation else 0)
    xt, pt = torch.as_tensor(x, device=DEV), torch.as_tensor(p, device=DEV)
    mx = xt * 10.0
    _remove(sy, xt, pt, flags, mx=mx, p_conv=10.0)
    torch.cuda.synchronize()
    x64, p64, m64 = x.astype(np.float64)[None], p.astype(np.float64)[None], masses.astype(np.float64)
    x_ref, p_ref = SO.remove_com_motion(x64, p64, m64, n_atoms, rotation)
    assert rel_err(_np(xt), x_ref[0]) < 1e-6
    assert rel_err(_np(pt), p_ref[0]) < 1e-5
    assert torch.equal(mx, xt * 10.0)
    # what is left is the fp32 rounding of the written momenta, |sum p| <= 2 eps32 sum |p| and |L| <= 8 eps32 sum |x| |p|
    # per system, plus the fp64 rounding of the removal, which cancels terms of the size of the input momenta p_in
    # (a planar molecule has no z-momentum left after the removals)
    xo, po = _np(xt).astype(np.float64)[None], _np(pt).astype(np.float64)[None]
    sp = SO.sum_atoms(po, n_atoms)[0]
    fp64 = 1e-12 * SO.sum_atoms(np.abs(p64), n_atoms)[0]
    assert np.all(np.abs(sp) <= 2 * F32 * SO.sum_atoms(np.abs(po), n_atoms)[0] + fp64 + 1e-300)
    if rotation:
        L = SO.inertia_and_angular_momentum(xo, po, m64, n_atoms)[1][0]
        xn = np.linalg.norm(xo, axis=2)
        bound = (8 * F32 * SO.sum_atoms((xn * np.linalg.norm(po, axis=2))[..., None], n_atoms)[0]
                 + 1e-12 * SO.sum_atoms((xn * np.linalg.norm(p64, axis=2))[..., None], n_atoms)[0])
        linear = np.arange(len(n_atoms)) % 6 == 2
        assert np.all(np.abs(L[~linear]) <= bound[~linear] + 1e-300)
        # the linear molecule keeps the angular momentum along its axis (the pseudo-inverse drops that direction);
        # the perpendicular part is gone
        a0 = int(np.cumsum([0] + n_atoms)[2])
        axis = xo[0, a0 + 2] - xo[0, a0]
        axis /= np.linalg.norm(axis)
        perp = L[linear] - (L[linear] @ axis)[:, None] * axis[None]
        assert np.all(np.abs(perp) <= bound[linear] + 1e-300)
    # repeated calls are bitwise equal
    xt2, pt2 = torch.as_tensor(x, device=DEV), torch.as_tensor(p, device=DEV)
    _remove(sy, xt2, pt2, flags, mx=xt2 * 10.0, p_conv=10.0)
    assert torch.equal(xt2, xt) and torch.equal(pt2, pt)


def test_rotation_about_origin_without_centering():
    from schnetpack_b200 import _lib

    n_atoms, masses, x, p = _ragged(4)
    sy = _systems(n_atoms, masses)
    xt, pt = torch.as_tensor(x, device=DEV), torch.as_tensor(p, device=DEV)
    _remove(sy, xt, pt, _lib.MOTION_ROTATION)
    p_ref = SO.remove_rotation(x.astype(np.float64)[None], p.astype(np.float64)[None], masses.astype(np.float64), n_atoms)
    assert torch.equal(xt, torch.as_tensor(x, device=DEV))
    assert rel_err(_np(pt), p_ref[0]) < 1e-5


@pytest.mark.parametrize("P", [1, 4, 8])
def test_wrap_follows_the_oracle(P):
    from schnetpack_b200 import _lib, ops

    rng = np.random.default_rng(P)
    cells = np.array([[[6.0, 0.0, 0.0], [1.5, 5.5, 0.0], [0.8, -1.1, 7.0]],
                      [[8.0, 0.0, 0.0], [0.0, 7.0, 0.0], [0.0, 0.0, 30.0]]])
    pbc = np.array([[1, 1, 1], [1, 1, 0]], dtype=np.uint8)
    n_atoms = [5000, 3000]
    idx = SO.system_index(n_atoms)
    frac = rng.uniform(-3.0, 4.0, size=(sum(n_atoms), 3))
    base = np.einsum("nj,nji->ni", frac, cells[idx])
    x = (base[None] + 0.05 * rng.normal(size=(P, base.shape[0], 3))).astype(np.float32)
    xt = torch.as_tensor(x.reshape(-1, 3), device=DEV)
    mx = xt * 2.0
    cell_t = torch.as_tensor(cells, device=DEV)
    pbc_t = torch.as_tensor(pbc, device=DEV)
    idx_t = torch.as_tensor(idx, device=DEV)
    _lib.call("spk_md_wrap_positions", ops._p(xt), ops._p(mx), ops._p(idx_t), base.shape[0], P, ops._p(cell_t), 9,
              ops._p(pbc_t), 3, SO.WRAP_EPS, 2.0, None, 1, ops._stream())
    torch.cuda.synchronize()
    y_ref = SO.wrap_positions(x.astype(np.float64), cells, pbc.astype(bool), n_atoms)
    y = _np(xt).reshape(P, -1, 3)
    assert rel_err(y, y_ref) < 1e-6
    assert torch.equal(mx, xt * 2.0)
    shift = SO.fractional(x.astype(np.float64) - y, cells, n_atoms)
    assert np.abs(shift - np.round(shift)).max() < 1e-4
    fc = SO.fractional(y.astype(np.float64).mean(axis=0)[None], cells, n_atoms)[0]
    per = pbc.astype(bool)[idx]
    assert np.all(fc[per] >= -SO.WRAP_EPS - 1e-5) and np.all(fc[per] < 1.0 - SO.WRAP_EPS + 1e-5)
    springs = lambda z: np.sum((z - np.roll(z, -1, axis=0)) ** 2, axis=(0, 2))     # noqa: E731
    assert np.allclose(springs(y.astype(np.float64)), springs(x.astype(np.float64)), rtol=1e-3, atol=1e-6)


# ---- initial momenta -------------------------------------------------------------------------------------------------------
def _draw(n, seed, uniform=0, masses=None, temps=None, n_sys=1, kB=1.0):
    from schnetpack_b200 import _lib, ops

    sizes = [n // n_sys] * n_sys
    sizes[-1] += n - sum(sizes)
    sy = _systems(sizes, np.ones(n, np.float32) if masses is None else masses)
    t = torch.as_tensor(np.ones(n_sys) if temps is None else temps, dtype=torch.float64, device=DEV)
    p = torch.zeros(n, 3, device=DEV)
    ws = sy.workspace("spk_md_motion_workspace_bytes")
    _lib.call("spk_md_initial_momenta", ops._p(p), ops._p(sy.masses), ops._p(sy.idx_m), ops._p(sy.sys_ptr), n, n_sys,
              uniform, kB, ops._p(t), seed, ops._p(ws), ws.numel(), ops._stream())
    torch.cuda.synchronize()
    return _np(p).astype(np.float64), sizes


def test_maxwell_boltzmann_normals_are_philox_and_normal():
    from scipy import stats

    from schnetpack_b200 import _lib, ops

    seed, n = 0xC0FFEE, 1_000_000 // 3 + 1
    ctr = torch.tensor([-1, 0], dtype=torch.int64, device=DEV)                    # application 2^64 - 1
    bits = torch.empty(n, 4, dtype=torch.int32, device=DEV)
    _lib.call("spk_philox4x32_10", seed, ops._p(ctr), n, ops._p(bits), ops._stream())
    assert (_np(bits).view(np.uint32) == NO.philox_bits(seed, DRAW_APP, n)).all()
    z, _ = _draw(n, seed)                                                         # m = 1, kB T = 1: p = xi
    ref = NO.langevin_normals(seed, DRAW_APP, n)
    # p = float(xi): equal to the restated normals rounded to fp32, up to one fp32 ulp where the fp64 transcendentals differ
    assert np.abs(z - ref.astype(np.float32)).max() <= 2.0 ** -23 * np.abs(ref).max()
    assert np.mean(z == ref.astype(np.float32)) > 0.999
    x = z.reshape(-1)
    N = x.size
    assert N >= 1_000_000
    assert abs(x.mean()) < 5.0 / math.sqrt(N)
    assert abs(x.var() - 1.0) < 5.0 * math.sqrt(2.0 / N)
    assert stats.kstest(x, "norm").pvalue > 1e-3


def test_initial_momenta_are_uncorrelated_with_the_first_langevin_application():
    seed, n = 7, 200_000
    z, _ = _draw(n, seed)
    lang = NO.langevin_normals(seed, 0, n)
    c = np.corrcoef(z.reshape(-1), lang.reshape(-1))[0, 1]
    assert abs(c) < 5.0 / math.sqrt(3 * n), c


def test_widths_and_uniform_rescale_follow_the_oracle():
    seed, n = 3, 3000
    rng = np.random.default_rng(0)
    masses = rng.choice([1.008, 12.011, 15.999], size=n).astype(np.float32)
    temps = np.array([100.0, 300.0, 0.0, 450.0])
    kB = 0.0083144598
    z = NO.langevin_normals(seed, DRAW_APP, n)[None]
    for uniform in (0, 1):
        p, sizes = _draw(n, seed, uniform, masses, temps, n_sys=4, kB=kB)
        ref = SO.draw_momenta(z, masses.astype(np.float64), sizes, temps, kB, bool(uniform))[0]
        assert rel_err(p, ref) < 1e-5
        if uniform:
            t = SO.temperature(p[None], masses.astype(np.float64), sizes, kB)[0]
            assert np.allclose(t, temps, rtol=1e-5)


# ---- DeviceMD with an initializer and hooks --------------------------------------------------------------------------------
def _box_md(p_conv=1.0, e_conv=1.0, n=150, capacity_factor=1.5, scatter=False, **kw):
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.md import DeviceMD
    from schnetpack_b200.model import batch_to_device, from_spec

    spec = S.model_spec("painn", n_atom_basis=64, n_interactions=2)
    data = S.periodic_box(n, seed=9)
    if scatter:             # every atom some lattice vectors away, on both sides
        shift = np.random.default_rng(1).integers(-3, 4, size=(n, 3)).astype(np.float32)
        data["_positions"] = (data["_positions"] + shift @ data["_cell"].reshape(3, 3)).astype(np.float32)
    params = S.init_params(spec, seed=8)
    model = from_spec(spec, params, torch.device(DEV))
    masses = np.where(data["_atomic_numbers"] == 8, 16.0, 1.0)
    md = DeviceMD(model, batch_to_device(data, torch.device(DEV)), torch.as_tensor(masses), time_step=1e-3,
                  cutoff=spec["cutoff"], capacity=int(data["_idx_i"].shape[0] * capacity_factor), position_conversion=p_conv,
                  energy_conversion=e_conv, **kw)
    return md, spec, params, data, masses


@pytest.mark.parametrize("p_conv,e_conv", [(1.0, 1.0), (10.0, 0.5)])
def test_device_md_with_initializer_follows_the_nve_oracle(p_conv, e_conv):
    from oracle import md_oracle as MO
    from schnetpack_b200.md import MaxwellBoltzmannInit

    kB, T, seed = 0.0025 / 300.0, 300.0, 11
    init = MaxwellBoltzmannInit(T, remove_rotation=True, wrap_positions=True, seed=seed, kB=kB)
    md, spec, params, data, masses = _box_md(p_conv, e_conv, initializer=init)
    x_md = np.asarray(data["_positions"], dtype=np.float64)[None] / p_conv
    cell = np.asarray(data["_cell"], dtype=np.float64).reshape(1, 3, 3) / p_conv
    n = x_md.shape[1]
    x0, p0 = SO.initialize(x_md, NO.langevin_normals(seed, DRAW_APP, n)[None], masses.astype(np.float64), [n], T, kB,
                           False, remove_rotation_=True, wrap_positions_=True, cells=cell,
                           pbc=np.asarray(data["_pbc"]).reshape(1, 3))
    torch.cuda.synchronize()
    assert rel_err(_np(md.positions), x0[0]) < 1e-6
    assert rel_err(_np(md.momenta), p0[0]) < 1e-5
    md.run(12)
    torch.cuda.synchronize()
    start = dict(data)
    start["_positions"] = x0[0] * p_conv
    x_ref, p_ref, e_ref, _ = MO.nve_trajectory(spec, params, start, masses, p0[0], 1e-3, 12, p_conv, e_conv)
    assert rel_err(_np(md.positions), x_ref) < 1e-6
    assert rel_err(_np(md.momenta), p_ref) < 1e-4
    assert rel_err(_np(md.potential_energy()), e_ref) < 1e-5


MASS = {1: 1.008, 6: 12.011, 8: 15.999}


def _initial_temperature_moments(x, m, n_atoms, T):
    """Mean and standard deviation of the batch temperature 2 K / (3 N kB) after p ~ N(0, m kB T), the (unweighted)
    translation removal and the rotation removal, which are linear in p: K = 1/2 p^T B p with B = A^T W A, W = 1/m, so
    E K = 1/2 tr(B C) and Var K = 1/2 tr((B C)^2) with C = kB T diag(m) (in units where kB = 1)."""
    mean = var = 0.0
    a0 = 0
    for n in n_atoms:
        xs, ms = x[None, a0:a0 + n], m[a0:a0 + n]
        basis = np.eye(3 * n).reshape(3 * n, n, 3)
        cols = [SO.remove_rotation(xs, SO.remove_translation(b[None], [n]), ms, [n])[0].reshape(-1) for b in basis]
        A = np.stack(cols, axis=1)
        w = np.repeat(1.0 / ms, 3)
        BC = (A.T * w) @ A * (T * np.repeat(ms, 3))[None, :]
        mean += 0.5 * np.trace(BC)
        var += 0.5 * np.trace(BC @ BC)
        a0 += n
    scale = 2.0 / (3.0 * sum(n_atoms))
    return scale * mean, scale * math.sqrt(var)


def test_trained_ethanol_conserves_momentum_and_angular_momentum():
    """256 ethanol molecules (trained PaiNN; MD in kJ/mol, nm, Da) start from MaxwellBoltzmannInit(300, rotation removed).
    The model is invariant, so every molecule's total and angular momentum stay at their initial values, which are fp32
    rounding: |sum p| <= 2 eps32 sum |p| per step, accumulated over 1000 steps as a random walk (x 4 sqrt(1000)), and
    likewise for L with the bound 8 eps32 sum |x| |p|.  The initial temperature of the N = 2304 atoms must lie within
    5 sigma of its expectation after the removals (``_initial_temperature_moments``)."""
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params, inputs, _, _ = load_case("painn_md_ethanol_trained")
    n_mol, n1 = inputs["_n_atoms"].shape[0], inputs["_positions"].shape[0]
    copies = 256 // n_mol
    b = {"_positions": np.tile(inputs["_positions"], (copies, 1)),
         "_atomic_numbers": np.tile(inputs["_atomic_numbers"], copies),
         "_n_atoms": np.tile(inputs["_n_atoms"], copies),
         "_idx_m": (np.tile(inputs["_idx_m"], copies) + np.repeat(np.arange(copies) * n_mol, n1)).astype(np.int64),
         "_cell": np.tile(inputs["_cell"], (copies, 1, 1)),
         "_pbc": np.tile(inputs["_pbc"].reshape(n_mol, 3), (copies, 1)).reshape(-1)}
    dev = torch.device(DEV)
    masses = torch.tensor([MASS[int(z)] for z in b["_atomic_numbers"]])
    md = M.DeviceMD(from_spec(spec, params, dev), batch_to_device(b, dev), masses, time_step=0.5 * M.FS_MD,
                    cutoff=spec["cutoff"], capacity=int(b["_n_atoms"].shape[0] * 9 * 8 * 1.5), position_conversion=10.0,
                    energy_conversion=4.184, initializer=M.MaxwellBoltzmannInit(300.0, remove_rotation=True, seed=5))
    n_atoms = b["_n_atoms"].tolist()
    assert len(n_atoms) == 256
    N = sum(n_atoms)
    m64 = masses.numpy().astype(np.float64)
    t0 = float(md.temperature().mean())
    expect, sigma = _initial_temperature_moments(_np(md.positions).astype(np.float64), m64, n_atoms, 300.0)
    assert abs(t0 - expect) < 5 * sigma, (t0, expect, sigma)

    def drift():
        x, p = _np(md.positions).astype(np.float64)[None], _np(md.momenta).astype(np.float64)[None]
        sp = np.abs(SO.sum_atoms(p, n_atoms)[0])
        L = np.abs(SO.inertia_and_angular_momentum(x - SO.center_of_mass(x, m64, n_atoms)[:, SO.system_index(n_atoms)],
                                                   p, m64, n_atoms)[1][0])
        scale_p = SO.sum_atoms(np.abs(p), n_atoms)[0]
        scale_l = SO.sum_atoms((np.linalg.norm(x, axis=2) * np.linalg.norm(p, axis=2))[..., None], n_atoms)[0]
        return sp / scale_p, L / scale_l

    sp0, l0 = drift()
    assert sp0.max() <= 2 * F32 and l0.max() <= 8 * F32
    md.run(1000)
    sp, lm = drift()
    walk = 4.0 * math.sqrt(1000.0)
    assert sp.max() <= 2 * F32 * walk, sp.max()
    assert lm.max() <= 8 * F32 * walk, lm.max()


def _ethanol_free_md(hooks, record=False, **kw):
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params, inputs, _, _ = load_case("painn_md_ethanol_trained")
    dev = torch.device(DEV)
    masses = torch.tensor([MASS[int(z)] for z in inputs["_atomic_numbers"]])
    extra = dict(record_velocities=True, record_capacity=16) if record else {}
    return M.DeviceMD(from_spec(spec, params, dev), batch_to_device(inputs, dev), masses, time_step=0.5 * M.FS_MD,
                      cutoff=spec["cutoff"], capacity=int(inputs["_n_atoms"].shape[0] * 9 * 8 * 1.5),
                      position_conversion=10.0, energy_conversion=4.184, hooks=hooks, **extra, **kw)


def test_remove_com_motion_hook_gates_and_runs_before_the_recorder():
    from schnetpack_b200 import md as M

    md = _ethanol_free_md([M.RemoveCOMMotion(5, True)], record=True, use_graph=True,
                          thermostat=M.LangevinThermostat(300.0, 20.0, seed=3),
                          initializer=M.UniformInit(300.0, remove_translation=False))
    n_atoms = md.systems.n_atoms_sys.to(torch.int64).tolist()
    sums = []
    for _ in range(10):
        md.run(1)
        sums.append(np.abs(SO.sum_atoms(_np(md.momenta).astype(np.float64)[None], n_atoms)[0]).max())
    scale = float(md.momenta.abs().max()) * max(n_atoms)
    for s, v in enumerate(sums):                         # steps 0 and 5 run the hook
        assert (v < 64 * F32 * scale) == (s % 5 == 0), (s, v, scale)
    vel = md.recorded("velocities").numpy().astype(np.float64)        # [10, 1, N, 3]
    pm = vel[:, 0] * md.masses.cpu().numpy()[None, :, None]
    rec_sums = [np.abs(SO.sum_atoms(pm[k][None], n_atoms)[0]).max() for k in (0, 5)]
    assert max(rec_sums) < 64 * F32 * scale                              # the recorder saw the hooked momenta


def test_wrap_hook_only_moves_by_lattice_vectors():
    from schnetpack_b200 import md as M

    def run(hooks):
        md, _, _, data, _ = _box_md(1.0, 1.0, n=300, hooks=hooks, scatter=True,
                                    momenta=torch.as_tensor(np.random.default_rng(4).normal(0, 0.05, (300, 3))))
        md.run(12)
        torch.cuda.synchronize()
        return md, data

    a, data = run([M.WrapPositions(1)])
    b, _ = run(None)
    cell = np.asarray(data["_cell"], dtype=np.float64).reshape(1, 3, 3)
    n = [a.positions.shape[0]]
    xa, xb = _np(a.positions).astype(np.float64)[None], _np(b.positions).astype(np.float64)[None]
    d = SO.fractional(xb - xa, cell, n)
    assert np.abs(d - np.round(d)).max() < 1e-4
    assert np.abs(np.round(d)).max() >= 1                                # something was wrapped
    assert rel_err(_np(a.momenta), _np(b.momenta)) < 1e-4
    f = SO.fractional(xa, cell, n)
    assert np.all(f >= -SO.WRAP_EPS - 1e-6) and np.all(f < 1.0 - SO.WRAP_EPS + 1e-6)


def test_wrap_with_isotropic_npt_uses_the_current_cell():
    from schnetpack_b200 import md as M

    baro = M.NHCBarostatIsotropic(1.0, 300.0, 50.0, kB=0.0025 / 300.0)
    md, *_ = _box_md(1.0, 1.0, n=300, capacity_factor=3.0, barostat=baro, hooks=[M.WrapPositions(1)], scatter=True,
                     momenta=torch.as_tensor(np.random.default_rng(4).normal(0, 0.05, (300, 3))))
    v0 = float(md.volume()[0])
    md.run(20)
    torch.cuda.synchronize()
    cell = md.cell.cpu().numpy()
    assert abs(float(md.volume()[0]) - v0) > 1e-6 * v0                   # the cell moved
    f = SO.fractional(_np(md.positions).astype(np.float64)[None], cell, [md.positions.shape[0]])
    assert np.all(f >= -SO.WRAP_EPS - 1e-5) and np.all(f < 1.0 - SO.WRAP_EPS + 1e-5)


def test_wrap_keeps_the_ring_polymer_springs():
    """One RPMD step of a 4-bead box from MaxwellBoltzmannInit (which centres it, so many atoms leave the cell), with and
    without WrapPositions(1): the wrapped beads differ from the free ones by lattice vectors, the bead separations (and
    so the spring energy) are those of the free run, and every centroid lies in the cell."""
    from schnetpack_b200 import md as M

    P, kB = 4, 0.0025 / 300.0

    def run(hooks):
        md, _, _, data, _ = _box_md(1.0, 1.0, n=150, capacity_factor=1.5 * P,
                                    ring_polymer=M.RingPolymer(P, 300.0, kB=kB, hbar=0.05),
                                    hooks=hooks, initializer=M.MaxwellBoltzmannInit(300.0, seed=2, kB=kB))
        md.run(1)
        torch.cuda.synchronize()
        return _np(md.positions).astype(np.float64).reshape(P, -1, 3), data

    x1, data = run([M.WrapPositions(1)])
    x2, _ = run(None)
    cell = np.asarray(data["_cell"], dtype=np.float64).reshape(1, 3, 3)
    n = [x1.shape[1]]
    d = SO.fractional(x2 - x1, cell, n)
    assert np.abs(d - np.round(d)).max() < 1e-4 and np.abs(np.round(d)).max() >= 1
    assert np.all(np.round(d) == np.round(d)[:1])                           # every bead of an atom moved alike
    sep = lambda z: z - np.roll(z, -1, axis=0)                               # noqa: E731
    assert np.abs(sep(x1) - sep(x2)).max() < 1e-5
    springs = lambda z: np.sum(sep(z) ** 2)                                  # noqa: E731
    assert abs(springs(x1) - springs(x2)) <= 1e-3 * springs(x2)
    fc = SO.fractional(x1.mean(axis=0)[None], cell, n)
    assert np.all(fc >= -SO.WRAP_EPS - 1e-5) and np.all(fc < 1.0 - SO.WRAP_EPS + 1e-5)


def _box_hooked(use_graph=True, hooks=None, **kw):
    from schnetpack_b200 import md as M

    kB = 0.0025 / 300.0
    return _box_md(1.0, 1.0, n=300, use_graph=use_graph, hooks=hooks,
                   thermostat=M.LangevinThermostat(300.0, 20.0, seed=9, kB=kB),
                   initializer=M.MaxwellBoltzmannInit(300.0, seed=4, kB=kB), **kw)[0]


def test_replay_equals_eager_and_restart_keeps_the_hook_phase():
    from schnetpack_b200 import md as M

    hooks = lambda: [M.RemoveCOMMotion(3, True), M.WrapPositions(3)]       # noqa: E731
    g, e = _box_hooked(True, hooks()), _box_hooked(False, hooks())
    g.run(8)
    e.run(8)
    assert torch.equal(g.positions, e.positions) and torch.equal(g.momenta, e.momenta)
    a = _box_hooked(True, hooks())
    a.run(4)
    sd = a.state_dict()
    assert int(sd["step_counter"][0]) == 4
    b = _box_hooked(True, hooks())
    b.load_state_dict(sd)
    b.run(4)
    assert torch.equal(b.positions, g.positions) and torch.equal(b.momenta, g.momenta)


def test_without_the_new_keywords_the_step_launches_as_before():
    from schnetpack_b200 import _lib
    from schnetpack_b200 import md as M

    plain = _box_md(use_graph=False)[0]
    hooked = _box_md(use_graph=False, hooks=[M.RemoveCOMMotion(2, True), M.WrapPositions(1)])[0]
    init = _box_md(use_graph=False, initializer=M.UniformInit(300.0, remove_rotation=True, wrap_positions=True))[0]
    counts = []
    for md in (plain, hooked, init):
        c0 = _lib.launch_count
        md.run(1)
        counts.append(_lib.launch_count - c0)
    assert counts[1] == counts[0] + 3 + 1 + 1                # removal, wrap, step counter
    assert counts[2] == counts[0]


def test_refusals():
    from schnetpack_b200 import md as M

    for bad in (0, -1, 1.5):
        with pytest.raises(ValueError, match="every_n_steps"):
            M.RemoveCOMMotion(bad, True)
        with pytest.raises(ValueError, match="every_n_steps"):
            M.WrapPositions(bad)
    with pytest.raises(TypeError, match="hooks"):
        _ethanol_free_md([M.LangevinThermostat(300.0, 20.0)])
    with pytest.raises(ValueError, match="temperatures"):
        _ethanol_free_md(None, initializer=M.MaxwellBoltzmannInit([300.0, 200.0, 100.0, 50.0, 10.0, 1.0, 2.0]))
    with pytest.raises(ValueError, match="momenta"):
        _ethanol_free_md(None, initializer=M.UniformInit(300.0), momenta=torch.zeros(9, 3))
    with pytest.raises(ValueError, match="temperature"):
        M.UniformInit(-1.0)
    md, _, _, data, masses = _box_md()
    zero = {k: v for k, v in data.items()}
    zero["_cell"] = np.zeros_like(data["_cell"])
    from schnetpack_b200.md import DeviceMD
    from schnetpack_b200.model import batch_to_device

    with pytest.raises(ValueError, match="volume"):
        DeviceMD(md.model, batch_to_device(zero, torch.device(DEV)), torch.as_tensor(masses), time_step=1e-3,
                 cutoff=5.0, capacity=10_000, hooks=[M.WrapPositions(1)])
    cpu = {k: torch.as_tensor(v) for k, v in data.items()}
    with pytest.raises(ValueError, match="CUDA"):
        DeviceMD(md.model, cpu, torch.as_tensor(masses), time_step=1e-3, cutoff=5.0, capacity=10_000,
                 initializer=M.UniformInit(300.0))
