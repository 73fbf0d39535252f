"""GPU checks of the device FIRE and unit-cell filter (schnetpack_b200.relax, csrc/fire.cu): the kernels against the fp64
oracle on a ragged batch fed analytic Morse forces and virials, DeviceFIRE with PaiNN against host-driven oracle loops,
the bitwise invariants of the captured step, and the refusals."""
import numpy as np
import pytest
import torch

from conftest import load_case
from fire_oracle import FIREOracle, fcc, morse, pair_list, pair_list_orthorhombic
from schnetpack_b200 import properties as P
from schnetpack_b200.model import batch_to_device, from_spec
from schnetpack_b200.neighbors import CellListNeighborList
from schnetpack_b200.relax import DeviceFIRE, FIREState, UnitCellFilter

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
MORSE = dict(rc=2.2)
REACH = 2.6


def _np(t):
    return t.detach().double().cpu().numpy()


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


# ---- the optimizer kernels alone, fed Morse forces and virials ---------------------------------------------------------
def _ragged_crystals():
    """1 atom, 21 atoms (fcc with vacancies), 300 atoms and 20 000 atoms (an fcc block spanning 79 CTAs); triclinic cells
    except the largest, each with its fixed pair list"""
    rng = np.random.default_rng(4)
    shear = np.eye(3) + np.array([[0.0, 0.05, -0.03], [0.02, 0.0, 0.04], [0.0, -0.03, 0.0]])
    systems = [(np.zeros((1, 3)), 1.25 * np.eye(3) @ shear)]
    x, cell = fcc(1.62, (3, 2, 1))
    systems.append((np.delete(x, [2, 9, 17], axis=0) @ shear, cell @ shear))
    x, cell = fcc(1.62, (5, 5, 3))
    systems.append((x @ shear, cell @ shear))
    systems.append(fcc(1.62, (10, 10, 50)))
    out = []
    for k, (x, cell) in enumerate(systems):
        x = x + rng.normal(scale=0.04, size=x.shape) * (k > 0)
        pairs = pair_list_orthorhombic(x, np.diag(cell), REACH) if len(x) > 1000 else pair_list(x, cell, REACH)
        out.append((x, cell, pairs))
    return out


def _morse_batch(systems, x, cells, ptr):
    f, W = np.zeros_like(x), np.zeros((len(systems), 3, 3))
    for m, (_, _, pairs) in enumerate(systems):
        _, f[ptr[m]:ptr[m + 1]], W[m] = morse(x[ptr[m]:ptr[m + 1]], cells[m], pairs, **MORSE)
    return f.astype(np.float32), W


FILTERS = {"fixed_cell": None, "filter": dict(scalar_pressure=0.3), "hydrostatic": dict(hydrostatic_strain=True),
           "mask": dict(mask=[1, 1, 0, 1, 0, 1], scalar_pressure=0.1), "constant_volume": dict(constant_volume=True)}


@pytest.mark.parametrize("name", list(FILTERS))
def test_state_follows_the_oracle_on_a_ragged_batch(name):
    systems = _ragged_crystals()
    sizes = [len(s[0]) for s in systems]
    ptr = np.concatenate([[0], np.cumsum(sizes)])
    x0 = np.concatenate([s[0] for s in systems])
    cells0 = np.stack([s[1] for s in systems])
    fixed = np.zeros(len(x0), dtype=bool)
    fixed[[3, 30, 5000, 20000]] = True
    kw = dict(dt=0.05, maxstep=0.1, dtmax=0.2, Nmin=3)
    fkw = FILTERS[name]
    o = FIREOracle(x0, ptr, cells=None if fkw is None else cells0, fixed=fixed, **kw, **(fkw or {}))
    idx_m = torch.repeat_interleave(torch.arange(len(sizes)), torch.as_tensor(sizes)).to(DEV)
    st = FIREState(torch.as_tensor(x0, device=DEV), idx_m, len(sizes), fixed_atoms_mask=fixed, fmax=1e-12,
                   cell=None if fkw is None else torch.as_tensor(cells0, device=DEV),
                   cell_filter=None if fkw is None else UnitCellFilter(**fkw), **kw)
    resets = 0
    for k in range(60):
        cells = o.cells if fkw is not None else cells0
        f, W = _morse_batch(systems, o.positions, cells, ptr)
        st.check(torch.as_tensor(f, device=DEV), torch.as_tensor(W, device=DEV) if fkw is not None else None)
        st.step()
        before = o.Nsteps.copy()
        fmax = o.fmax(f.astype(np.float64), W)                 # of the generalized forces the step used
        o.step(f.astype(np.float64), W, 1e-12)
        resets += int(((o.Nsteps == 0) & (before > 0)).sum())
        assert _rel(_np(st.r), o.positions) <= 1e-10, k
    va, vc = o.velocities
    assert _rel(_np(st.v), va) <= 1e-10
    assert _rel(_np(st.dt), o.dt) <= 1e-12 and _rel(_np(st.a), o.a) <= 1e-12
    assert st.nsteps.cpu().tolist() == o.Nsteps.tolist()
    np.testing.assert_allclose(_np(st.fmax), fmax, rtol=1e-9)
    assert resets > 0
    if fkw is not None:
        assert _rel(_np(st.cell()), o.cells) <= 1e-10 and _rel(_np(st.hv), vc) <= 1e-10
        assert _rel(_np(st.s), o.scaled) <= 1e-10
        assert np.array_equal(_np(st.s)[fixed], x0[fixed])                                   # fixed atoms keep s
        assert torch.equal(st.model_cell.reshape(-1, 3, 3), st.cell().float())
        assert np.abs(_np(st.cell()) - cells0).max() > 1e-3
    else:
        assert np.array_equal(_np(st.r)[fixed], x0[fixed])                                   # fixed atoms stay put
    assert torch.equal(st.model_positions, st.r.float())


# ---- DeviceFIRE with PaiNN on periodic boxes ---------------------------------------------------------------------------
def _box(seed=9, n=150):
    from schnetpack_b200 import synthetic as S

    spec = S.model_spec("painn", n_atom_basis=128, n_interactions=2)
    data = S.periodic_box(n, seed=seed)
    params = S.init_params(spec, seed=8)
    return spec, from_spec(spec, params, DEV), data


def _box_fire(model, data, spec, **kw):
    return DeviceFIRE(model, batch_to_device(data, DEV), cutoff=spec["cutoff"],
                      capacity=int(data["_idx_i"].shape[0] * 2), **kw)


class _EagerModel:
    """the same CUDA model evaluated eagerly at given positions and cell (its own neighbour list), with the virial"""

    def __init__(self, model, data, spec, p_conv=1.0):
        self.model, self.p_conv = model, p_conv
        self.batch = {k: v for k, v in batch_to_device(data, DEV).items() if k not in (P.idx_i, P.idx_j, P.offsets)}
        self.nl = CellListNeighborList(spec["cutoff"], capacity=int(data["_idx_i"].shape[0] * 2), pad=True)

    def __call__(self, r, cell=None):
        x = dict(self.batch)
        x[P.R] = torch.as_tensor(r / self.p_conv, dtype=torch.float64, device=DEV).float()
        if cell is not None:
            x[P.cell] = torch.as_tensor(cell / self.p_conv, dtype=torch.float64, device=DEV).float().reshape(
                self.batch[P.cell].shape)
        n_sys = x[P.n_atoms].shape[0]
        x[P.virial] = torch.zeros(n_sys, 3, 3, dtype=torch.float64, device=DEV)
        out = self.model(self.nl(x))
        return (out["forces"].detach().double().cpu().numpy(), out["energy"].detach().double().cpu().numpy(),
                x[P.virial].cpu().numpy())


@pytest.mark.parametrize("p_conv,e_conv", [(1.0, 1.0), (0.5, 2.0)])
def test_cell_filter_follows_the_host_driven_oracle(p_conv, e_conv):
    spec, model, data = _box()
    filt = dict(scalar_pressure=0.02)
    dev = _box_fire(model, data, spec, cell_filter=UnitCellFilter(**filt), position_conversion=p_conv,
                    energy_conversion=e_conv, maxstep=0.05)
    ev = _EagerModel(model, data, spec, p_conv)
    x0 = data["_positions"].astype(np.float64) * p_conv
    cell0 = np.asarray(data["_cell"], dtype=np.float64).reshape(1, 3, 3) * p_conv
    o = FIREOracle(x0, [0, len(x0)], cells=cell0, maxstep=0.05, **filt)
    traj = []
    for _ in range(8):
        dev.run(fmax=1e-9, steps=1)
        traj.append((dev.positions.cpu().numpy().copy(), dev.cell.cpu().numpy().copy()))
    f_conv = e_conv / p_conv
    for k in range(8):
        f, _, W = ev(o.positions, o.cells)
        o.step(f * f_conv, W * e_conv, 1e-9)
        assert np.abs(traj[k][0] - o.positions).max() <= 1e-4 * p_conv, k
        assert _rel(traj[k][1], o.cells) <= 1e-6, k
    assert np.abs(o.cells - cell0).max() > 1e-4
    f, e, W = ev(o.positions, o.cells)
    assert _rel(_np(dev.get_energy()), e * e_conv) <= 1e-5
    vol = abs(np.linalg.det(o.cells[0]))
    assert _rel(_np(dev.get_stress()), 0.5 * (W + W.transpose(0, 2, 1)) * e_conv / vol) <= 1e-4
    assert _rel(_np(dev.get_enthalpy()), e * e_conv + 0.02 * vol) <= 1e-5


def test_converged_cell_satisfies_the_stress_bound():
    """Three strained fcc Morse cells under pressure relax on the device until every generalized force is below fmax.
    The cell rows then bound the stress: every row of V (sigma + p I) F^-T / cell_factor is shorter than fmax."""
    fmax, p = 1e-4, 0.05
    strains = [np.eye(3) + e for e in (np.diag([0.04, -0.02, 0.03]), np.array([[0.0, 0.03, 0.0], [0.03, 0.05, 0.0],
                                                                                [0.0, 0.0, -0.04]]),
                                       0.02 * np.ones((3, 3)))]
    crystals = [fcc(1.62) for _ in strains]
    x0 = np.concatenate([x @ e for (x, _), e in zip(crystals, strains)])
    cells0 = np.stack([c @ e for (_, c), e in zip(crystals, strains)])
    idx_m = torch.arange(3).repeat_interleave(4).to(DEV)
    st = FIREState(torch.as_tensor(x0, device=DEV), idx_m, 3, cell=torch.as_tensor(cells0, device=DEV),
                   cell_filter=UnitCellFilter(scalar_pressure=p), fmax=fmax)
    for _ in range(4000):
        r, cells = _np(st.r), _np(st.cell())
        f, W = np.zeros_like(r), np.zeros((3, 3, 3))
        for m in range(3):
            xm = r[4 * m:4 * m + 4]
            _, f[4 * m:4 * m + 4], W[m] = morse(xm, cells[m], pair_list(xm, cells[m], 2.4))
        st.check(torch.as_tensor(f, dtype=torch.float32, device=DEV), torch.as_tensor(W, device=DEV))
        if int(st.n_unconverged.item()) == 0:
            break
        st.step()
    assert int(st.n_unconverged.item()) == 0 and (_np(st.fmax) < fmax).all()
    F = _np(st.deformation_gradient())
    for m in range(3):
        vol = abs(np.linalg.det(cells[m]))
        sigma = 0.5 * (W[m] + W[m].T) / vol
        rows = np.linalg.solve(F[m], (-vol * (sigma + p * np.eye(3))).T).T / 4.0
        assert np.linalg.norm(rows, axis=1).max() < fmax, m
        assert np.abs(sigma + p * np.eye(3)).max() < 4.0 * fmax * np.abs(F[m]).max() * 3 / vol, m
    assert np.abs(F - np.eye(3)).max() > 1e-2


def test_graph_replay_equals_eager_and_restart_is_bitwise_with_a_filter():
    spec, model, data = _box()
    kw = dict(cell_filter=UnitCellFilter(scalar_pressure=0.02), maxstep=0.05)
    a = _box_fire(model, data, spec, use_graph=True, **kw)
    b = _box_fire(model, data, spec, use_graph=False, **kw)
    a.run(fmax=1e-9, steps=14, check_every=4)
    b.run(fmax=1e-9, steps=14, check_every=4)
    for k, v in a.opt.tensors().items():
        assert torch.equal(v, b.opt.tensors()[k]), k
    assert torch.equal(a.energy, b.energy) and torch.equal(a.virial, b.virial)
    first = _box_fire(model, data, spec, **kw)
    first.run(fmax=1e-9, steps=9)
    sd = first.state_dict()
    second = _box_fire(model, data, spec, **kw)
    second.load_state_dict(sd)
    second.run(fmax=1e-9, steps=5)
    assert second.iterations == a.iterations == 14
    for k, v in a.opt.tensors().items():
        assert torch.equal(v, second.opt.tensors()[k]), k
    assert torch.equal(second.model_positions, a.model_positions) and torch.equal(second.static[P.cell],
                                                                                  a.static[P.cell])


def test_fixed_atoms_keep_their_scaled_coordinates_under_the_filter():
    spec, model, data = _box()
    fixed = [0, 7, 100]
    r = _box_fire(model, data, spec, cell_filter=UnitCellFilter(scalar_pressure=0.05), fixed_atoms_mask=fixed)
    s0 = r.opt.s.clone()
    r.run(fmax=1e-9, steps=20)
    assert torch.equal(r.opt.s[fixed], s0[fixed]) and not torch.equal(r.opt.s, s0)
    F = r.opt.deformation_gradient()[0]
    torch.testing.assert_close(r.positions[fixed], s0[fixed] @ F.T, rtol=1e-14, atol=1e-14)


# ---- fixed-cell FIRE with the trained PaiNN ethanol model -------------------------------------------------------------
FMAX = 0.05          # kcal/mol/Angstrom: the model's units


def _ethanol(noise=0.08, seed=0):
    spec, params, inputs, _, _ = load_case("painn_md_ethanol_trained")
    rng = np.random.default_rng(seed)
    inputs = dict(inputs)
    inputs["_positions"] = (inputs["_positions"] + rng.normal(scale=noise, size=inputs["_positions"].shape)).astype(
        np.float32)
    return spec, params, from_spec(spec, params, DEV), inputs


def _relaxer(model, inputs, spec, **kw):
    return DeviceFIRE(model, batch_to_device(inputs, DEV), cutoff=spec["cutoff"], capacity=18 * 18, **kw)


def test_ethanol_converges_and_follows_the_oracle():
    spec, _, model, inputs = _ethanol()
    dev = _relaxer(model, inputs, spec)
    ev = _EagerModel(model, inputs, spec)
    o = FIREOracle(inputs["_positions"].astype(np.float64), [0, 9, 18])
    traj = []
    for _ in range(10):
        dev.run(fmax=FMAX, steps=1)
        traj.append(dev.positions.cpu().numpy().copy())
    for k in range(10):
        o.step(ev(o.positions)[0], None, FMAX)
        assert np.abs(traj[k] - o.positions).max() <= 1e-5, k
    assert dev.run(fmax=FMAX, steps=2000)
    assert (dev.fmax.cpu().numpy() < FMAX).all() and dev.nsteps == int(dev.steps_to_converge.max())
    f = ev(dev.positions.cpu().numpy())[0]
    assert np.sqrt((f ** 2).sum(-1)).max() < FMAX * 1.01


def test_converged_system_is_frozen_and_fixed_atoms_stay():
    spec, _, model, inputs = _ethanol(noise=0.0)
    relaxed = _relaxer(model, inputs, spec)
    relaxed.run(fmax=0.005, steps=3000)
    pos = relaxed.model_positions.cpu().numpy().copy()
    rng = np.random.default_rng(5)
    pos[:9] += rng.normal(scale=0.002, size=(9, 3))
    pos[9:] += rng.normal(scale=0.15, size=(9, 3))
    inputs = dict(inputs, _positions=pos.astype(np.float32))
    dev = _relaxer(model, inputs, spec, fixed_atoms_mask=[12])
    start = dev.positions.clone()
    frozen = 0
    for _ in range(1000):
        before = dev.positions.clone()
        state = {k: v.clone() for k, v in dev.opt.tensors().items()}
        done = dev.run(fmax=FMAX, steps=1)
        m0 = 0 <= int(dev.steps_to_converge[0]) < dev.iterations
        if m0:
            frozen += 1
            assert torch.equal(dev.positions[:9], before[:9])
            for k in ("dt", "a", "nsteps"):
                assert torch.equal(dev.opt.tensors()[k][0], state[k][0]), k
            assert torch.equal(dev.opt.v[:9], state["v"][:9])
        if done:
            break
    assert done and frozen > 0
    assert torch.equal(dev.positions[12], start[12])


def test_system_in_a_batch_matches_it_alone():
    spec, _, model, inputs = _ethanol()
    batch = _relaxer(model, inputs, spec)
    one = {"_n_atoms": inputs["_n_atoms"][:1], "_idx_m": inputs["_idx_m"][:9],
           "_atomic_numbers": inputs["_atomic_numbers"][:9], "_positions": inputs["_positions"][:9],
           "_cell": inputs["_cell"][:1], "_pbc": inputs["_pbc"][:3]}
    alone = _relaxer(model, one, spec)
    batch.run(fmax=1e-6, steps=12)
    alone.run(fmax=1e-6, steps=12)
    assert float((batch.positions[:9] - alone.positions).abs().max()) <= 1e-6


def test_ensemble_follows_the_oracle_fed_the_mean_forces():
    spec, params, model, inputs = _ethanol()
    other = from_spec(spec, {k: v * (1.0 + 0.02 * np.random.default_rng(1).standard_normal(v.shape)).astype(v.dtype)
                             if v.dtype.kind == "f" else v for k, v in params.items()}, DEV)
    dev = _relaxer([model, other], inputs, spec)
    evs = [_EagerModel(m, inputs, spec) for m in (model, other)]
    o = FIREOracle(inputs["_positions"].astype(np.float64), [0, 9, 18])
    traj = []
    for _ in range(6):
        dev.run(fmax=1e-6, steps=1)
        traj.append(dev.positions.cpu().numpy().copy())
    for k in range(6):
        f = np.mean([ev(o.positions)[0] for ev in evs], axis=0)
        o.step(f, None, 1e-6)
        assert np.abs(traj[k] - o.positions).max() <= 1e-5, k
    u = dev.get_uncertainty()
    assert u["forces_uncertainty"].shape == (18, 3) and float(u["energy_uncertainty"].abs().max()) > 0.0


# ---- refusals ----------------------------------------------------------------------------------------------------------
def test_refusals():
    spec, params, model, inputs = _ethanol()
    cpu = {k: torch.as_tensor(v) for k, v in inputs.items()}
    with pytest.raises(ValueError, match="CUDA"):
        DeviceFIRE(model, cpu, cutoff=spec["cutoff"], capacity=400)
    for bad in (dict(dt=0.0), dict(maxstep=-1.0), dict(Nmin=-1), dict(a=1.5), dict(fdec=0.0)):
        with pytest.raises(ValueError, match="FIRE"):
            _relaxer(model, inputs, spec, **bad)
    with pytest.raises(ValueError, match="mask"):
        UnitCellFilter(mask=[1, 1, 1])
    with pytest.raises(ValueError, match="cell_factor"):
        UnitCellFilter(cell_factor=0.0)
    with pytest.raises(ValueError, match="forces"):
        _relaxer(from_spec(dict(spec, forces=False), params, DEV), inputs, spec)
    with pytest.raises(NotImplementedError, match="ensemble"):
        _relaxer([model, model], inputs, spec, cell_filter=UnitCellFilter())
    with pytest.raises(ValueError, match="periodic"):                   # ethanol in a non-periodic batch
        _relaxer(model, inputs, spec, cell_filter=UnitCellFilter())
    bspec, bmodel, data = _box()
    flat = dict(data, _cell=np.asarray(data["_cell"]) * np.array([1.0, 1.0, 0.0], dtype=np.float32)[:, None])
    with pytest.raises(ValueError, match="volume"):
        _box_fire(bmodel, flat, bspec, cell_filter=UnitCellFilter())
    with pytest.raises(ValueError, match="CUDA"):
        FIREState(torch.zeros(3, 3), torch.zeros(3, dtype=torch.int64), 1)
    small = DeviceFIRE(model, batch_to_device(inputs, DEV), cutoff=spec["cutoff"], capacity=20)
    with pytest.raises(RuntimeError, match="overflowed"):
        small.run(fmax=1e-6, steps=3)
