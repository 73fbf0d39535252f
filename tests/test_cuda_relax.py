"""GPU checks of the device L-BFGS (schnetpack_b200.relax): the optimizer kernels against the reference's recorded runs
and the fp64 oracle (both size paths, ragged batches), DeviceLBFGS with the trained PaiNN ethanol model against a
host-driven oracle loop, the bitwise invariants of the captured step, and the refusals."""
import numpy as np
import pytest
import torch

from conftest import load_case
from relax_oracle import LBFGSOracle
from schnetpack_b200 import properties as P
from schnetpack_b200.model import batch_to_device, from_spec
from schnetpack_b200.neighbors import CellListNeighborList
from schnetpack_b200.relax import DeviceLBFGS, LBFGSState
from test_relax_oracle import CASES, load

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


# ---- the optimizer kernels alone ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_state_reproduces_reference_run(name):
    c = load(name)
    n_atoms = c["n_atoms"]
    idx_m = torch.repeat_interleave(torch.arange(len(n_atoms)), torch.as_tensor(n_atoms)).to(DEV)
    st = LBFGSState(torch.as_tensor(c["pos_before"][0], device=DEV), idx_m, len(n_atoms), memory=int(c["memory"]),
                    maxstep=float(c["maxstep"]), damping=float(c["damping"]), alpha=float(c["alpha"]),
                    fixed_atoms_mask=c["fixed"], fmax=float(c["fmax"]))
    for k in range(c["p"].shape[0]):
        f = torch.as_tensor(c["forces"][k], dtype=torch.float32, device=DEV)
        assert np.array_equal(f.double().cpu().numpy(), c["forces"][k])          # the recorded forces are fp32-exact
        st.check(f)
        st.step(f)
        assert np.array_equal(st.converged.cpu().numpy().astype(bool), c["converged"][k]), k
        assert _rel(st.p.cpu(), c["p"][k]) <= 1e-10 or np.abs(c["p"][k]).max() == 0.0, k
        assert _rel(st.r.cpu(), c["pos_after"][k]) <= 1e-10, k
        if k > 0:
            slot = (k - 1) % int(c["memory"])
            assert _rel(st.rho[slot].cpu(), c["rho"][k]) <= 1e-10, k
    assert torch.equal(st.model_positions, st.r.float())


def test_mixed_ragged_batch_matches_oracle_on_both_paths():
    """1 atom, small molecules (warp per system), 300 atoms and about 20 000 atoms (a cluster each), 30 steps with a
    wrapping history, synthetic fp32 forces from a field that differs per atom."""
    sizes = [1, 21, 9, 300, 13, 20000, 2]
    ptr = np.concatenate([[0], np.cumsum(sizes)])
    rng = np.random.default_rng(11)
    n = int(ptr[-1])
    r = rng.normal(scale=3.0, size=(n, 3))
    centre = r + rng.normal(scale=0.4, size=(n, 3))
    stiff = rng.uniform(0.5, 3.0, size=(n, 1))
    fixed = np.zeros(n, dtype=bool)
    fixed[[5, 400, 9000]] = True

    def forces(x):
        return (-(x - centre) * stiff + 0.2 * np.sin(2.0 * x)).astype(np.float32)

    idx_m = torch.repeat_interleave(torch.arange(len(sizes)), torch.as_tensor(sizes)).to(DEV)
    kw = dict(memory=7, maxstep=0.15, damping=0.9, alpha=4.0)
    st = LBFGSState(torch.as_tensor(r, device=DEV), idx_m, len(sizes), fixed_atoms_mask=fixed, fmax=1e-9, **kw)
    assert st.n_warp == 5 and st.order.tolist()[5:] == [3, 5]
    o = LBFGSOracle(r, ptr, fixed=fixed, **kw)
    for k in range(30):
        f = forces(o.r)
        ft = torch.as_tensor(f, device=DEV)
        st.check(ft)
        st.step(ft)
        o.step(f.astype(np.float64), 1e-9)
        assert _rel(st.r.cpu(), o.r) <= 1e-9, k
        assert _rel(st.p.cpu(), o.p) <= 1e-9, k
    np.testing.assert_allclose(st.fmax.cpu().numpy(), o.fmax(forces(o.r0)), rtol=1e-12)
    assert np.array_equal(st.r.cpu().numpy()[fixed], r[fixed])


# ---- DeviceLBFGS with the trained PaiNN ethanol model ------------------------------------------------------------------
FMAX = 0.02          # kcal/mol/Angstrom: the model's units


def _ethanol(noise=0.08, seed=0):
    spec, params, inputs, _, _ = load_case("painn_md_ethanol_trained")
    rng = np.random.default_rng(seed)
    inputs = dict(inputs)
    inputs["_positions"] = (inputs["_positions"] + rng.normal(scale=noise, size=inputs["_positions"].shape)).astype(
        np.float32)
    model = from_spec(spec, params, DEV)
    return spec, model, inputs


def _relaxer(model, inputs, spec, **kw):
    return DeviceLBFGS(model, batch_to_device(inputs, DEV), cutoff=spec["cutoff"], capacity=18 * 18, **kw)


class _EagerForces:
    """the same CUDA model evaluated eagerly at given positions (its own neighbour list)"""

    def __init__(self, model, inputs, spec):
        self.model = model
        self.batch = {k: v for k, v in batch_to_device(inputs, DEV).items() if k not in (P.idx_i, P.idx_j, P.offsets)}
        self.nl = CellListNeighborList(spec["cutoff"], capacity=18 * 18, pad=True)

    def __call__(self, r):
        x = dict(self.batch)
        x[P.R] = torch.as_tensor(r, dtype=torch.float64, device=DEV).float()
        out = self.model(self.nl(x))
        return out["forces"].detach().double().cpu().numpy(), out["energy"].detach().double().cpu().numpy()


def test_ethanol_matches_host_driven_oracle_and_reconverges_in_zero_steps():
    spec, model, inputs = _ethanol()
    dev = _relaxer(model, inputs, spec)
    ev = _EagerForces(model, inputs, spec)
    o = LBFGSOracle(inputs["_positions"].astype(np.float64), [0, 9, 18])
    traj = []
    for _ in range(10):
        dev.run(fmax=FMAX, steps=1)
        traj.append(dev.positions.cpu().numpy().copy())
    for k in range(10):
        f, _ = ev(o.r)
        o.converged(f, FMAX)
        o.step(f, FMAX)
        assert np.abs(traj[k] - o.r).max() <= 1e-5, k
    ok = dev.run(fmax=FMAX, steps=400)
    for _ in range(400):
        f, e_o = ev(o.r)
        if o.converged(f, FMAX).all():
            break
        o.step(f, FMAX)
    assert ok and o.converged(ev(o.r)[0], FMAX).all()
    e_dev = dev.get_energy().double().cpu().numpy()
    assert _rel(e_dev, ev(o.r)[1]) <= 1e-5
    assert dev.nsteps == int(dev.steps_to_converge.max()) and (dev.fmax.cpu().numpy() < FMAX).all()
    again = DeviceLBFGS(model, dict(batch_to_device(inputs, DEV), _positions=dev.model_positions.clone()),
                        cutoff=spec["cutoff"], capacity=18 * 18)
    assert again.run(fmax=FMAX) and again.nsteps == 0 and again.iterations == 0


def test_graph_replay_equals_eager():
    spec, model, inputs = _ethanol()
    a = _relaxer(model, inputs, spec, use_graph=True)
    b = _relaxer(model, inputs, spec, use_graph=False)
    a.run(fmax=1e-6, steps=15, check_every=4)
    b.run(fmax=1e-6, steps=15, check_every=4)
    assert torch.equal(a.positions, b.positions) and torch.equal(a.model_positions, b.model_positions)
    assert torch.equal(a.energy, b.energy) and torch.equal(a.forces, b.forces)
    assert torch.equal(a.opt.s, b.opt.s) and torch.equal(a.opt.rho, b.opt.rho)


def test_restart_is_bitwise():
    spec, model, inputs = _ethanol()
    ref = _relaxer(model, inputs, spec, memory=6)
    ref.run(fmax=1e-6, steps=20)
    first = _relaxer(model, inputs, spec, memory=6)
    first.run(fmax=1e-6, steps=11)
    sd = first.state_dict()
    second = _relaxer(model, inputs, spec, memory=6)
    second.load_state_dict(sd)
    second.run(fmax=1e-6, steps=9)
    assert second.iterations == ref.iterations == 20
    for k, v in ref.opt.tensors().items():
        assert torch.equal(v, second.opt.tensors()[k]), k
    assert torch.equal(second.energy, ref.energy) and torch.equal(second.forces, ref.forces)


def test_fixed_atoms_never_move():
    spec, model, inputs = _ethanol()
    for mask in ([0, 10, 17], np.isin(np.arange(18), [3, 4])):
        r = _relaxer(model, inputs, spec, fixed_atoms_mask=mask)
        start = r.positions.clone()
        r.run(fmax=FMAX, steps=60)
        fixed = r.opt.fixed.bool()
        assert torch.equal(r.positions[fixed], start[fixed]) and not torch.equal(r.positions, start)
        assert float(r.get_forces()[fixed].abs().max()) == 0.0


def test_converged_system_is_frozen_and_steps_match_the_oracle():
    """molecule 0 starts much closer to its minimum than molecule 1, so it converges first and must stay put while the
    other one continues"""
    spec, model, inputs = _ethanol(noise=0.0)
    relaxed = _relaxer(model, inputs, spec)
    relaxed.run(fmax=0.002, steps=1000)
    inputs = dict(inputs)
    pos = relaxed.model_positions.cpu().numpy().copy()
    rng = np.random.default_rng(5)
    pos[:9] += rng.normal(scale=0.002, size=(9, 3))
    pos[9:] += rng.normal(scale=0.15, size=(9, 3))
    inputs["_positions"] = pos.astype(np.float32)
    dev = _relaxer(model, inputs, spec)
    ev = _EagerForces(model, inputs, spec)
    o = LBFGSOracle(inputs["_positions"].astype(np.float64), [0, 9, 18])
    frozen_steps = 0
    done = False
    for k in range(500):
        before = dev.positions.clone()
        done = dev.run(fmax=FMAX, steps=1)
        f, _ = ev(o.r)
        if not o.converged(f, FMAX).all():
            o.step(f, FMAX)
        for m, sl in enumerate((slice(0, 9), slice(9, 18))):
            if 0 <= int(dev.steps_to_converge[m]) < dev.iterations:      # converged before this step
                frozen_steps += 1
                assert torch.equal(dev.positions[sl], before[sl]), (k, m)
        if done:
            break
    assert done and bool(dev.converged.all()) and frozen_steps > 0
    o.converged(ev(o.r)[0], FMAX)
    assert dev.steps_to_converge.cpu().tolist() == o.steps_to_converge.tolist()
    assert int(dev.steps_to_converge.min()) < int(dev.steps_to_converge.max()) == dev.nsteps


def test_system_in_a_batch_matches_it_alone():
    spec, model, inputs = _ethanol()
    batch = _relaxer(model, inputs, spec)
    one = {"_n_atoms": inputs["_n_atoms"][:1], "_idx_m": inputs["_idx_m"][:9],
           "_atomic_numbers": inputs["_atomic_numbers"][:9], "_positions": inputs["_positions"][:9],
           "_cell": inputs["_cell"][:1], "_pbc": inputs["_pbc"][:3]}
    alone = _relaxer(model, one, spec)
    batch.run(fmax=1e-6, steps=12)
    alone.run(fmax=1e-6, steps=12)
    assert float((batch.positions[:9] - alone.positions).abs().max()) <= 1e-6


def test_periodic_box_rebuilds_the_neighbour_list_every_step():
    spec, params, inputs, _, _ = load_case("painn_box_216")
    model = from_spec(spec, params, DEV)
    cap = int(inputs["_idx_i"].shape[0] * 1.5)
    r = DeviceLBFGS(model, batch_to_device(inputs, DEV), cutoff=spec["cutoff"], capacity=cap, maxstep=0.05)
    start = r.model_positions.clone()
    r.run(fmax=1e-6, steps=25, check_every=5)
    assert r.peak_pairs <= cap and r.iterations == 25
    assert not torch.equal(r.model_positions, start)
    # the forces of the last step are those of a fresh evaluation at the final positions
    x = {k: v for k, v in batch_to_device(inputs, DEV).items() if k not in (P.idx_i, P.idx_j, P.offsets)}
    x[P.R] = r.model_positions.clone()
    out = model(CellListNeighborList(spec["cutoff"], capacity=cap, pad=True)(x))
    assert _rel(r.forces.cpu(), out["forces"].detach().cpu()) <= 1e-5


# ---- refusals ----------------------------------------------------------------------------------------------------------
def test_refusals():
    spec, model, inputs = _ethanol()
    cpu = {k: torch.as_tensor(v) for k, v in inputs.items()}
    cpu[P.R] = cpu[P.R].float()
    with pytest.raises(ValueError, match="CUDA"):
        DeviceLBFGS(model, cpu, cutoff=spec["cutoff"], capacity=400)
    with pytest.raises(ValueError, match="maximum step size"):
        _relaxer(model, inputs, spec, maxstep=1.5)
    spec_nf = dict(spec, forces=False)
    _, params, _, _, _ = load_case("painn_md_ethanol_trained")
    with pytest.raises(ValueError, match="forces"):
        _relaxer(from_spec(spec_nf, params, DEV), inputs, spec)
    small = DeviceLBFGS(model, batch_to_device(inputs, DEV), cutoff=spec["cutoff"], capacity=20)
    with pytest.raises(RuntimeError, match="overflowed"):
        small.run(fmax=FMAX, steps=3)
