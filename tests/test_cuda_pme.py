"""H100: smooth particle-mesh Ewald on csrc/pme.cu against the fp64 restatement of tests/pme_oracle.py at the same mesh
and order, against the converged fp64 Ewald sum of the fixtures (tests/golden/ewald_*.npz) under ``use_pme``, and in the
captured device drivers."""
import numpy as np
import pytest
import torch

import ewald_oracle as EO
import pme_oracle as PM
from test_cuda_ewald import _adversarial, _masses, _run
from test_ewald_oracle import load_case, package_model, rel, torch_batch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = 1e-5
KEYS = ["energy", "forces", "partial_charges", "dipole_moment", "stress"]


def _pme_model(case, w, stress=True):
    from schnetpack_b200.atomistic import pme_mesh, use_pme

    with _layout_stress(case, stress):
        model = package_model(case, w, torch.float32).to(DEV).eval()
    batch, _, _ = load_case(case)
    order, spacing = PM.FIXTURE_PARAMS
    return use_pme(model, pme_mesh(batch["_cell"], spacing, order), order)


class _layout_stress:
    def __init__(self, case, stress):
        self.case, self.stress = case, stress

    def __enter__(self):
        self.old = EO.LAYOUT[self.case]
        EO.LAYOUT[self.case] = dict(self.old, stress=self.stress)

    def __exit__(self, *a):
        EO.LAYOUT[self.case] = self.old


def _max_bin(b, mesh, order):
    """the most atoms in one spreading bin: (system, 8^3-point brick of the first support point) as csrc/pme.cu bins"""
    R = b["_positions"].astype(np.float64)
    H = np.linalg.inv(b["_cell"].astype(np.float64))[b["_idx_m"]]
    s = np.einsum("nb,nbc->nc", R, H)
    s -= np.floor(s)
    n = np.array(mesh)
    base = (np.floor(s * n).astype(np.int64) - (order - 1)) % n
    keys = np.concatenate([b["_idx_m"][:, None], base // 8], 1)
    return int(np.unique(keys, axis=0, return_counts=True)[1].max())


@pytest.mark.parametrize("order,mesh,screen", [(4, (45, 48, 50), None), (6, (20, 18, 16), (1.0, 3.0)),
                                               (8, (16, 15, 14), None), (6, (8, 9, 10), None)])
def test_adversarial_batches_match_oracle(order, mesh, screen):
    """Mixed triclinic and skewed cells, a one-atom system, a 300-atom system, a trailing empty system, positions several
    cells out and shuffled edges: E, dE/dR, dE/dq and dE/dcell against the oracle at the same mesh and order, and a
    second run bitwise equal.  The coarse 8 x 9 x 10 mesh puts more atoms in a bin than a spreading CTA stages at once
    (64), next to one-point last bricks."""
    from schnetpack_b200 import atomistic as A
    from schnetpack_b200 import nn as snn

    alpha = 0.25
    b, q = _adversarial(4, screen)
    if mesh == (8, 9, 10):
        assert _max_bin(b, mesh, order) > 64
    mod = A.EnergyPME(alpha, mesh, order, "kcal/mol", "Ang", "e", use_neighbors_lr=False,
                      screening_fn=snn.SwitchFunction(*screen) if screen else None).to(DEV).eval()

    def inputs(dtype, dev):
        x = torch_batch(b, dtype, dev)
        for k in ("_positions", "_cell"):
            x[k].requires_grad_()
        x["partial_charges"] = torch.as_tensor(q).to(dtype).to(dev).requires_grad_()
        x["_Rij"] = x["_positions"][x["_idx_j"]] - x["_positions"][x["_idx_i"]] + x["_offsets"]
        return x

    x = inputs(torch.float32, DEV)
    e = mod(x)["e"]
    w = torch.linspace(0.5, 1.5, e.shape[0], device=DEV)
    g = torch.autograd.grad((w * e).sum(), [x["_positions"], x["partial_charges"], x["_cell"]])
    x64 = inputs(torch.float64, "cpu")
    B = len(b["_n_atoms"])
    a64, ke64 = EO.buffer_value(alpha), EO.buffer_value(EO.KE)
    e64 = EO.real_space(x64["partial_charges"], x64["_Rij"], x64["_idx_i"], x64["_idx_j"], x64["_idx_m"], B, a64, ke64,
                        screen=screen)
    e64 = e64 + PM.energy(x64["partial_charges"], x64["_positions"], x64["_cell"], x64["_idx_m"], B, mesh, order, a64,
                          ke64)
    g64 = torch.autograd.grad((w.cpu().double() * e64).sum(), [x64["_positions"], x64["partial_charges"], x64["_cell"]])
    assert rel(e.detach().cpu().numpy(), e64.detach().numpy()) <= TOL
    assert float(e[-1].detach()) == 0.0                                                  # the empty system
    for name, a, r in zip(("dE/dR", "dE/dq", "dE/dcell"), g, g64):
        assert rel(a.cpu().numpy(), r.numpy()) <= TOL, name
    x2 = inputs(torch.float32, DEV)
    e2 = mod(x2)["e"]
    g2 = torch.autograd.grad((w * e2).sum(), [x2["_positions"], x2["partial_charges"], x2["_cell"]])
    assert torch.equal(e, e2) and all(torch.equal(a, c) for a, c in zip(g, g2))


def test_cfg4_box_matches_ewald_kernels_beyond_convergence():
    """On the cfg4 water box (8192 atoms, L = 43.4 A, alpha = 0.46 A^-2) the PME reciprocal and self terms at the
    recorded order and spacing agree with the Ewald kernels at k_max = 45, far past the 1e-5 point (k_max 40 and 45
    agree to 1e-6), within 1e-5 in energy, forces, dE/dq and dE/dcell."""
    from schnetpack_b200 import atomistic as A
    from schnetpack_b200 import ops
    from schnetpack_b200 import synthetic as S

    b = S.periodic_box(n_atoms_total=8192, cutoff=5.0, seed=0, build_list=False)
    R = torch.as_tensor(b[S.R], device=DEV)
    cell = torch.as_tensor(b[S.cell], device=DEV).reshape(1, 3, 3).contiguous()
    q = torch.as_tensor(np.where(b[S.Z] == 8, -0.8476, 0.4238), dtype=torch.float32, device=DEV)
    idx_m = torch.zeros(R.shape[0], dtype=torch.int64, device=DEV)
    sys_ptr = ops.segment_ptr(idx_m, 1)
    alpha, g_E = 0.46, torch.ones(1, device=DEV)

    def ewald(k_max):
        kv = A.EnergyEwald(alpha, k_max, 1.0, 1.0, "e").kvecs.to(DEV).contiguous()
        e, ws = ops.ewald_fwd(R, q, cell, kv, idx_m, sys_ptr, 1, EO.KE, alpha)
        g_q = torch.zeros_like(q)
        g_R, g_c = ops.ewald_bwd(R, q, cell, kv, idx_m, sys_ptr, 1, EO.KE, alpha, g_E, ws, True, g_q, True)
        return [t.double().cpu() for t in (e, g_R, g_q, g_c)]

    order, spacing = next(iter(PM.ACCURACY.items()))
    mesh = A.pme_mesh(cell, spacing, order)
    e, conv, ws = ops.pme_fwd(R, q, cell, idx_m, sys_ptr, 1, mesh, order, EO.KE, alpha)
    g_q = torch.zeros_like(q)
    g_R, g_c = ops.pme_bwd(R, q, idx_m, sys_ptr, 1, mesh, order, EO.KE, alpha, g_E, conv, ws, True, g_q, True)
    pme = [t.double().cpu() for t in (e, g_R, g_q, g_c)]
    e45, e40, e32 = ewald(45), ewald(40), ewald(32)
    names = ("energy", "dE/dR", "dE/dq", "dE/dcell")
    err = {n: rel(a.numpy(), r.numpy()) for n, a, r in zip(names, pme, e45)}
    trunc40 = {n: rel(a.numpy(), r.numpy()) for n, a, r in zip(names, e40, e45)}
    trunc32 = {n: rel(a.numpy(), r.numpy()) for n, a, r in zip(names, e32, e45)}
    print(f"cfg4 mesh {mesh}: PME vs Ewald k_max 45 {err}; k_max 40 vs 45 {trunc40}; k_max 32 vs 45 {trunc32}")
    assert max(trunc40.values()) <= 1e-6
    for n in names:
        assert err[n] <= TOL, (n, err[n])


@pytest.fixture(scope="module", params=EO.CASES)
def case(request):
    batch, w, ref = load_case(request.param)
    return request.param, batch, w, _pme_model(request.param, w), ref


def test_fixture_models_under_pme_match_converged_ewald(case):
    """At the recorded accuracy parameters PME gives the energy, forces, charges, dipole and stress of the same model
    with a converged Ewald sum (k_max = 10; the e2 fixture's own k_max = 3 truncates at about 5e-5) to 1e-5; the
    converged Ewald model itself matches the fp64 fixture of e1, whose k_max = 4 is converged at alpha = 0.12."""
    name, batch, w, model, ref = case
    out = _run(model, torch_batch(batch, torch.float32, DEV))
    conv = package_model(name, w, torch.float32).to(DEV).eval()
    ew = conv.output_modules[2]
    ew.k_max = 10
    ew.kvecs = ew._generate_kvecs().to(DEV)
    conv_out = _run(conv, torch_batch(batch, torch.float32, DEV))
    for k in KEYS:
        err = rel(out[k].detach().cpu().numpy(), conv_out[k].detach().cpu().numpy())
        print(f"{name} {k}: {err:.2e} (fixture k_max: {rel(out[k].detach().cpu().numpy(), ref['fp64/' + k]):.2e})")
        assert err <= TOL, (name, k)
        if name == "e1":
            assert rel(conv_out[k].detach().cpu().numpy(), ref["fp64/" + k]) <= TOL, k


def test_graph_replay_with_new_positions_and_cell_equals_eager():
    """The captured step (cuFFT plans made in the eager warm-up) replays bitwise what an eager call computes."""
    from schnetpack_b200.model import GraphedPotential

    batch, w, _ = load_case("e2")
    model = _pme_model("e2", w)
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
        assert torch.equal(rep[k], eager[k].detach()), k


def test_device_md_nve_conserves_energy_with_pme():
    """0.5 ps of NVE (2000 steps of 0.25 fs) on the charged e1 box with PME under the captured step."""
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device

    batch, w, _ = load_case("e1")
    model = _pme_model("e1", w, stress=False)
    n = batch["_positions"].shape[0]
    masses = _masses(batch)
    rng = np.random.default_rng(0)
    mom = torch.as_tensor(rng.normal(0, 0.05, (n, 3)), dtype=torch.float32) * masses[:, None]
    md = M.DeviceMD(model, batch_to_device(batch, DEV), masses, time_step=0.25 * M.FS_MD, cutoff=6.0,
                    capacity=n * 256, momenta=mom)
    totals, pots = [], []
    for _ in range(40):
        md.run(50)
        pot, kin = float(md.potential_energy().sum()), float(md.kinetic_energy())
        totals.append(pot + kin)
        pots.append(pot)
    md.check_neighbor_list()
    drift = max(abs(t - totals[0]) for t in totals)
    swing = max(pots) - min(pots)
    print(f"NVE PME box, 2000 x 0.25 fs: max |E - E0| {drift:.3e}, potential swing {swing:.3e}, "
          f"ratio {drift / swing:.3e}")
    assert swing > 0.0
    assert drift <= 0.01 * swing, (drift, swing)


def test_device_md_virial_matches_strain_stress_and_zero_volume_is_refused():
    from schnetpack_b200 import md as M
    from schnetpack_b200 import relax as RX
    from schnetpack_b200.atomistic import EnergyEwaldError
    from schnetpack_b200.model import batch_to_device

    batch, w, _ = load_case("e1")
    n = batch["_positions"].shape[0]
    md = M.DeviceMD(_pme_model("e1", w, stress=False), batch_to_device(batch, DEV), _masses(batch),
                    time_step=0.02 * M.FS_MD, cutoff=6.0, capacity=n * 256, compute_stress=True)
    ref = _pme_model("e1", w)(torch_batch(batch, torch.float32, DEV))["stress"].detach()
    assert rel(md.stress.cpu().numpy(), ref.double().cpu().numpy()) <= TOL
    bad = dict(batch)
    bad["_cell"] = np.zeros_like(batch["_cell"])
    with pytest.raises(EnergyEwaldError):
        M.DeviceMD(_pme_model("e1", w, stress=False), batch_to_device(bad, DEV), _masses(batch),
                   time_step=0.02 * M.FS_MD, cutoff=6.0, capacity=n * 256)
    with pytest.raises(EnergyEwaldError):
        RX.DeviceLBFGS(_pme_model("e1", w, stress=False), batch_to_device(bad, DEV), cutoff=6.0, capacity=n * 256)


def test_captured_npt_and_fire_with_cell_filter_run_with_pme():
    from schnetpack_b200 import md as M
    from schnetpack_b200 import relax as RX
    from schnetpack_b200.model import batch_to_device

    batch, w, _ = load_case("e1")
    n = batch["_positions"].shape[0]
    baro = M.NHCBarostatIsotropic(1.0, 300.0, 100.0, time_constant_barostat=1000.0, integration_order=3, multi_step=2,
                                  kB=M.KB_MD, fs=M.FS_MD)
    md = M.DeviceMD(_pme_model("e1", w, stress=False), batch_to_device(batch, DEV), _masses(batch),
                    time_step=0.25 * M.FS_MD, cutoff=6.0, capacity=n * 256, barostat=baro)
    md.run(100)
    assert bool(torch.isfinite(md.forces).all()) and bool(torch.isfinite(md.potential_energy()).all())
    fire = RX.DeviceFIRE(_pme_model("e1", w, stress=False), batch_to_device(batch, DEV), cutoff=6.0, capacity=n * 256,
                         cell_filter=RX.UnitCellFilter(scalar_pressure=0.0))
    fire.run(fmax=1e-9, steps=50)
    assert bool(torch.isfinite(fire.energy).all())
