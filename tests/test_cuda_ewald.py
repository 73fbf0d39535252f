"""H100: Ewald summation on csrc/pair_energy.cu (real space) and csrc/ewald.cu (reciprocal and self terms), with forces
through the differentiable charges of DipoleMoment, the cell gradient and the NPT virial, against the fp64 fixtures of
the unmodified reference (tests/golden/ewald_*.npz) and the fp64 restatement of tests/ewald_oracle.py."""
import contextlib

import numpy as np
import pytest
import torch

import ewald_oracle as EO
from test_ewald_oracle import load_case, package_model, rel, torch_batch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = 1e-5
KEYS = ["energy", "e_nn", "e_ewald", "forces", "partial_charges", "dipole_moment", "stress"]


def _run(model, x):
    out = dict(model(x))
    out.update({k: v for k, v in x.items() if k not in out})
    return out


@contextlib.contextmanager
def _layout(case, **kw):
    old = EO.LAYOUT[case]
    EO.LAYOUT[case] = dict(old, **kw)
    try:
        yield
    finally:
        EO.LAYOUT[case] = old


@pytest.fixture(scope="module", params=EO.CASES)
def case(request):
    batch, w, ref = load_case(request.param)
    model = package_model(request.param, w, torch.float32).to(DEV).eval()
    return request.param, batch, w, model, ref


def test_fixtures_match_reference(case):
    name, batch, _, model, ref = case
    out = _run(model, torch_batch(batch, torch.float32, DEV))
    for k in KEYS:
        assert rel(out[k].detach().cpu().numpy(), ref["fp64/" + k]) <= TOL, (name, k)


def test_fixed_charges_match_oracle_and_the_charge_path_matters(case):
    """At the fp64 model's charges held fixed the Ewald energy, its forces and dE/dq match the oracle; with the charge
    path cut (plain charges, as a passed-through EnergyEwald would get) the model forces are wrong."""
    name, batch, w, model, ref = case
    L = EO.LAYOUT[name]
    ew = model.output_modules[2]
    x = torch_batch(batch, torch.float32, DEV)
    x["_positions"].requires_grad_()
    for m in model.input_modules:
        x = m(x)
    q = torch.as_tensor(ref["fp64/partial_charges"], dtype=torch.float32).reshape(-1).to(DEV).requires_grad_()
    x[ew.charges_key] = q
    e = ew(x)[ew.output_key]
    gR, gq = torch.autograd.grad(e.sum(), [x["_positions"], q])
    assert rel(e.detach().cpu().numpy(), ref["ewald/energy"]) <= TOL
    assert rel(-gR.cpu().numpy(), ref["ewald/forces"]) <= TOL
    R, ii, jj, off = (torch.as_tensor(batch[k]) for k in ("_positions", "_idx_i", "_idx_j", "_offsets"))
    q64 = torch.as_tensor(ref["fp64/partial_charges"]).reshape(-1).requires_grad_()
    R64, cell64 = R.double(), torch.as_tensor(batch["_cell"]).double()
    idx_m, B = torch.as_tensor(batch["_idx_m"]), len(batch["_n_atoms"])
    alpha, ke = EO.buffer_value(L["alpha"]), EO.buffer_value(EO.KE)
    e64 = EO.real_space(q64, EO.PO.rij(R64, ii, jj, off.double()), ii, jj, idx_m, B, alpha, ke, screen=L["screen"])
    e64 = e64 + EO.reciprocal_self(q64, R64, cell64, idx_m, B, alpha, EO.kvecs(L["k_max"]), ke)
    (gq64,) = torch.autograd.grad(e64.sum(), q64)
    assert rel(gq.cpu().numpy(), gq64.numpy()) <= TOL
    cut = package_model(name, w, torch.float32).to(DEV).eval()
    cut.output_modules[0].differentiable_charges = False
    f_cut = _run(cut, torch_batch(batch, torch.float32, DEV))["forces"].detach().cpu().numpy()
    assert rel(f_cut, ref["fp64/forces"]) > 100 * TOL


def _adversarial(k_max, screen, seed=0):
    """Mixed triclinic cells, a one-atom system, a 300-atom system (more than a CTA stages), a trailing empty system,
    shuffled edges and positions moved several cells out (offsets moved with them, so every r_ij is kept)."""
    cells = list(EO.E2_CELLS) + [[[15.0, 0, 0], [0.5, 14.0, 0], [0.0, 1.0, 14.5]]]
    b = EO.triclinic_batch((20, 1, 12, 300), cells, 4.0, seed)
    rng = np.random.default_rng(seed)
    R = b["_positions"].astype(np.float64)
    cell = b["_cell"].astype(np.float64)
    sh = rng.integers(-4, 5, (R.shape[0], 3)).astype(np.float64)
    L = np.einsum("na,nab->nb", sh, cell[b["_idx_m"]])
    R = R + L
    off = b["_offsets"].astype(np.float64) + L[b["_idx_i"]] - L[b["_idx_j"]]
    perm = rng.permutation(b["_idx_i"].shape[0])
    b.update(_positions=R.astype(np.float32), _offsets=off[perm].astype(np.float32), _idx_i=b["_idx_i"][perm],
             _idx_j=b["_idx_j"][perm])
    b["_n_atoms"] = np.append(b["_n_atoms"], 0)
    b["_cell"] = np.concatenate([b["_cell"], np.eye(3, dtype=np.float32)[None] * 5.0])
    q = rng.normal(0, 0.6, R.shape[0]).astype(np.float32)
    return b, q


@pytest.mark.parametrize("k_max,screen", [(1, None), (7, None), (4, (1.0, 3.0))])
def test_adversarial_batches_match_oracle(k_max, screen):
    from schnetpack_b200 import atomistic as A
    from schnetpack_b200 import nn as snn

    alpha = 0.25
    b, q = _adversarial(k_max, screen)
    ew = A.EnergyEwald(alpha, k_max, "kcal/mol", "Ang", "e", use_neighbors_lr=False,
                       screening_fn=snn.SwitchFunction(*screen) if screen else None).to(DEV).eval()
    assert ew.kvecs.shape[0] > 128 or k_max == 1

    def inputs(dtype, dev):
        x = torch_batch(b, dtype, dev)
        for k in ("_positions", "_cell"):
            x[k].requires_grad_()
        x["partial_charges"] = torch.as_tensor(q).to(dtype).to(dev).requires_grad_()
        x["_Rij"] = x["_positions"][x["_idx_j"]] - x["_positions"][x["_idx_i"]] + x["_offsets"]
        return x

    x = inputs(torch.float32, DEV)
    e = ew(x)["e"]
    w = torch.linspace(0.5, 1.5, e.shape[0], device=DEV)
    g = torch.autograd.grad((w * e).sum(), [x["_positions"], x["partial_charges"], x["_cell"]])
    x64 = inputs(torch.float64, "cpu")
    B = len(b["_n_atoms"])
    a64, ke64 = EO.buffer_value(alpha), EO.buffer_value(EO.KE)
    e64 = EO.real_space(x64["partial_charges"], x64["_Rij"], x64["_idx_i"], x64["_idx_j"], x64["_idx_m"], B, a64, ke64,
                        screen=screen)
    e64 = e64 + EO.reciprocal_self(x64["partial_charges"], x64["_positions"], x64["_cell"], x64["_idx_m"], B, a64,
                                   EO.kvecs(k_max), ke64)
    g64 = torch.autograd.grad((w.cpu().double() * e64).sum(), [x64["_positions"], x64["partial_charges"], x64["_cell"]])
    assert rel(e.detach().cpu().numpy(), e64.detach().numpy()) <= TOL
    assert float(e[-1].detach()) == 0.0                                                  # the empty system
    for name, a, r in zip(("dE/dR", "dE/dq", "dE/dcell"), g, g64):
        assert rel(a.cpu().numpy(), r.numpy()) <= TOL, name
    # a second run is bitwise equal
    x2 = inputs(torch.float32, DEV)
    e2 = ew(x2)["e"]
    g2 = torch.autograd.grad((w * e2).sum(), [x2["_positions"], x2["partial_charges"], x2["_cell"]])
    assert torch.equal(e, e2) and all(torch.equal(a, c) for a, c in zip(g, g2))


def test_second_run_is_bitwise_equal_and_graph_replay_takes_new_positions_and_cell():
    from schnetpack_b200.model import GraphedPotential

    batch, w, _ = load_case("e2")
    model = package_model("e2", w, torch.float32).to(DEV).eval()
    o1 = {k: v.detach().clone() for k, v in model(torch_batch(batch, torch.float32, DEV)).items()}
    o2 = model(torch_batch(batch, torch.float32, DEV))
    for k in o1:
        assert torch.equal(o1[k], o2[k].detach()), k
    gp = GraphedPotential(model)
    gp(torch_batch(batch, torch.float32, DEV))
    b2 = dict(batch)
    s = np.float32(1.02)
    rng = np.random.default_rng(1)
    b2["_positions"] = batch["_positions"] * s + rng.normal(0, 0.01, batch["_positions"].shape).astype(np.float32)
    b2["_cell"], b2["_offsets"] = batch["_cell"] * s, batch["_offsets"] * s
    rep = {k: v.clone() for k, v in gp(torch_batch(b2, torch.float32, DEV)).items()}
    eager = model(torch_batch(b2, torch.float32, DEV))
    assert not torch.equal(rep["energy"], o1["energy"])
    for k in ("energy", "forces", "stress"):
        assert rel(rep[k].cpu().numpy(), eager[k].detach().cpu().numpy()) <= 1e-6, k


def _md_model(w):
    with _layout("e1", stress=False):
        return package_model("e1", w, torch.float32).to(DEV).eval()


def _masses(batch):
    return torch.as_tensor(np.where(batch["_atomic_numbers"] == 1, 1.008, 15.999), dtype=torch.float32)


def test_device_md_nve_conserves_energy_on_a_charged_periodic_box():
    """0.5 ps of NVE (2000 steps of 0.25 fs) on the charged e1 box under the captured step."""
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device

    batch, w, _ = load_case("e1")
    model = _md_model(w)
    n = batch["_positions"].shape[0]
    masses = _masses(batch)
    rng = np.random.default_rng(0)
    mom = torch.as_tensor(rng.normal(0, 0.05, (n, 3)), dtype=torch.float32) * masses[:, None]
    md = M.DeviceMD(model, batch_to_device(batch, DEV), masses, time_step=0.25 * M.FS_MD, cutoff=6.0,
                    capacity=n * 256, momenta=mom)
    totals, pots, kins = [], [], []
    for _ in range(40):
        md.run(50)
        pot, kin = float(md.potential_energy().sum()), float(md.kinetic_energy())
        totals.append(pot + kin)
        pots.append(pot)
        kins.append(kin)
    md.check_neighbor_list()
    drift = max(abs(t - totals[0]) for t in totals)
    swing = max(pots) - min(pots)
    print(f"NVE Ewald box, 2000 x 0.25 fs: max |E - E0| {drift:.3e}, potential swing {swing:.3e}, "
          f"mean kinetic {np.mean(kins):.3e}, ratio to swing {drift / swing:.3e}")
    assert swing > 0.0
    # bound: the total energy stays within 1 % of the potential energy's swing over the 0.5 ps (measured on an H100:
    # 0.41 %, 0.61 kcal/mol against a swing of 149 kcal/mol; the run is bitwise reproducible on one GPU)
    assert drift <= 0.01 * swing, (drift, swing)


def test_device_md_keeps_fp32_forces_of_a_model_that_casts_its_inputs():
    """convert_model sets cast_inputs on a model that arrives in fp64 (every floating input that is not fp32 is cast,
    and the outputs are cast back to that dtype).  The drivers add nothing floating to the batch, so the forces the step
    integrates stay fp32 and equal the reference's."""
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device

    batch, w, ref = load_case("e1")
    model = _md_model(w)
    model.cast_inputs = True
    n = batch["_positions"].shape[0]
    md = M.DeviceMD(model, batch_to_device(batch, DEV), _masses(batch), time_step=0.25 * M.FS_MD, cutoff=6.0,
                    capacity=n * 256)
    assert md.forces.dtype == torch.float32 and md.energy.dtype == torch.float32
    assert rel(md.forces.cpu().numpy(), ref["fp64/forces"]) <= TOL
    assert rel(md.energy.cpu().numpy(), ref["fp64/energy"]) <= TOL
    md.run(5)
    assert md.forces.dtype == torch.float32 and bool(torch.isfinite(md.forces).all())


def test_device_md_virial_matches_strain_stress_and_zero_volume_is_refused():
    from schnetpack_b200 import md as M
    from schnetpack_b200 import relax as RX
    from schnetpack_b200.atomistic import EnergyEwaldError
    from schnetpack_b200.model import batch_to_device

    batch, w, _ = load_case("e1")
    n = batch["_positions"].shape[0]
    md = M.DeviceMD(_md_model(w), batch_to_device(batch, DEV), _masses(batch), time_step=0.02 * M.FS_MD, cutoff=6.0,
                    capacity=n * 256, compute_stress=True)
    strain = package_model("e1", w, torch.float32).to(DEV).eval()
    ref = strain(torch_batch(batch, torch.float32, DEV))["stress"].detach()
    assert rel(md.stress.cpu().numpy(), ref.double().cpu().numpy()) <= TOL
    bad = dict(batch)
    bad["_cell"] = np.zeros_like(batch["_cell"])
    with pytest.raises(EnergyEwaldError):
        M.DeviceMD(_md_model(w), batch_to_device(bad, DEV), _masses(batch), time_step=0.02 * M.FS_MD, cutoff=6.0,
                   capacity=n * 256)
    with pytest.raises(EnergyEwaldError):
        RX.DeviceLBFGS(_md_model(w), batch_to_device(bad, DEV), cutoff=6.0, capacity=n * 256)
