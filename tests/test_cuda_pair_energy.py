"""H100: ZBL repulsion and Coulomb energies on csrc/pair_energy.cu, with forces through the differentiable charges of
DipoleMoment, against the fp64 fixtures of the unmodified reference (tests/golden/pair_energy_*.npz) and the fp64
restatement of tests/pair_energy_oracle.py."""
import numpy as np
import pytest
import torch

import pair_energy_oracle as PO
from test_pair_energy_oracle import load_case, package_model, rel, torch_batch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = 1e-5


def _run(model, x):
    out = dict(model(x))
    out.update({k: v for k, v in x.items() if k not in out})
    return out


@pytest.fixture(scope="module", params=PO.CASES)
def case(request):
    batch, w, ref = load_case(request.param)
    model = package_model(request.param, w, torch.float32).to(DEV).eval()
    return request.param, batch, model, ref


def test_fixtures_match_reference(case):
    name, batch, model, ref = case
    out = _run(model, torch_batch(batch, torch.float32, DEV))
    keys = ["energy", "e_nn", "e_zbl", "e_coul", "forces", "partial_charges", "dipole_moment"]
    if PO.LAYOUT[name]["stress"]:
        keys.append("stress")
    for k in keys:
        assert rel(out[k].detach().cpu().numpy(), ref["fp64/" + k]) <= TOL, (name, k)


def test_charge_path_carries_the_force_term(case):
    """The forces minus those of the pair terms at fixed charges is dE/dq dq/dR (plus the network's own forces): the
    full model matches the reference only because the charge path is there, and the charge term is not small."""
    name, batch, model, ref = case
    x = torch_batch(batch, torch.float32, DEV)
    f = _run(model, x)["forces"].detach().cpu().numpy()
    assert rel(f, ref["fp64/forces"]) <= TOL
    # the same model with the charges cut off from the graph (fixed-charge Coulomb forces)
    for m in model.output_modules:
        if type(m).__name__ == "DipoleMoment":
            m.register_forward_hook(lambda mod, inp, out: out.__setitem__(mod.charges_key, out[mod.charges_key].detach()))
    try:
        out = _run(model, torch_batch(batch, torch.float32, DEV))
        f_fixed = out["forces"].detach().cpu().numpy()
        x = torch_batch(batch, torch.float32, DEV)
        x["_positions"].requires_grad_()
        out = _run(model, x)
        g_pair = torch.autograd.grad(out["e_zbl"].sum() + out["e_coul"].sum(), x["_positions"])[0]
    finally:
        for m in model.output_modules:
            m._forward_hooks.clear()
    q_term = ref["fp64/forces"] - f_fixed
    assert np.abs(q_term).max() > 1e2 * TOL * np.abs(ref["fp64/forces"]).max(), name   # the term matters
    if PO.LAYOUT[name]["stress"]:
        return      # Strain rewrites the positions: the pair terms differentiate the strained copy
    # at fixed charges the pair terms' forces are the fp64 oracle's at the same charges
    q = torch.as_tensor(out["partial_charges"].detach().double().cpu().numpy())
    _, _, f_oracle = PO.pair_terms_fixed_q(name, batch, ref_weights(name), q)
    assert rel(-g_pair.cpu().numpy(), f_oracle.numpy()) <= TOL


def ref_weights(name):
    return load_case(name)[1]


def test_convert_model_path_matches():
    """The reference-built model goes through convert_model where the reference is importable (test_reference_live's
    loader); here the package's own swap of the pair modules is checked on the fixture weights."""
    from schnetpack_b200.model import convert_model

    batch, w, ref = load_case("a")
    src = package_model("a", w, torch.float32)
    conv = convert_model(src).to(DEV)
    out = _run(conv, torch_batch(batch, torch.float32, DEV))
    for k in ("energy", "forces", "partial_charges"):
        assert rel(out[k].detach().cpu().numpy(), ref["fp64/" + k]) <= TOL, k


# ---- adversarial batches against the fp64 oracle ------------------------------------------------------------------
def _adversarial(seed=0):
    """Systems: a 260-atom cluster with all pairs (67k slots: its partials span > 128 CTAs of the partial pass), a small
    molecule with one isolated atom, a periodic box of 4 atoms whose list holds self-image pairs, and a trailing empty
    system.  Edges shuffled (unsorted idx_i)."""
    rng = np.random.default_rng(seed)
    pos, Z, ii, jj, off, nat = [], [], [], [], [], []
    base = 0
    # cluster: distances spread over 0.6 .. 12 A
    n = 260
    p = rng.uniform(0.0, 9.0, (n, 3))
    a, b = np.where(~np.eye(n, dtype=bool))
    pos.append(p); Z.append(rng.integers(1, 9, n)); ii.append(a + base); jj.append(b + base)
    off.append(np.zeros((a.size, 3))); nat.append(n); base += n
    # molecule with an isolated atom (index 3)
    p = np.array([[0, 0, 0], [1.1, 0, 0], [0, 2.3, 0], [40.0, 40.0, 40.0], [0, 0, 3.9]], dtype=np.float64)
    a = np.array([0, 1, 0, 2, 1, 2, 0, 4]); b = np.array([1, 0, 2, 0, 2, 1, 4, 0])
    pos.append(p); Z.append(np.array([6, 1, 8, 1, 7])); ii.append(a + base); jj.append(b + base)
    off.append(np.zeros((a.size, 3))); nat.append(5); base += 5
    # small periodic box (L = 3.2) with self-image pairs and their periodic images
    L = 3.2
    p = rng.uniform(0, L, (4, 3))
    a, b, o = [], [], []
    for i in range(4):
        for j in range(4):
            for s in [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, 0, -1), (0, 0, 0)]:
                if i == j and s == (0, 0, 0):
                    continue
                a.append(i); b.append(j); o.append(np.array(s) * L)
    pos.append(p); Z.append(np.array([8, 1, 1, 3])); ii.append(np.array(a) + base); jj.append(np.array(b) + base)
    off.append(np.array(o)); nat.append(4); base += 4
    nat.append(0)                                                           # trailing empty system
    P, I, J, O = np.concatenate(pos), np.concatenate(ii), np.concatenate(jj), np.concatenate(off)
    d = np.linalg.norm(P[J] - P[I] + O, axis=1)
    keep = np.ones(d.size, dtype=bool)            # distances on both sides of every bound of TERMS, none on one
    for bnd in BOUNDS:
        keep &= np.abs(d - bnd) > 1e-3
    ii, jj, off = [I[keep]], [J[keep]], [O[keep]]
    perm = rng.permutation(int(keep.sum()))
    batch = {
        "_positions": np.concatenate(pos).astype(np.float32),
        "_atomic_numbers": np.concatenate(Z).astype(np.int64),
        "_idx_i": np.concatenate(ii).astype(np.int64)[perm],
        "_idx_j": np.concatenate(jj).astype(np.int64)[perm],
        "_offsets": np.concatenate(off).astype(np.float32)[perm],
        "_n_atoms": np.array(nat, dtype=np.int64),
        "_idx_m": np.repeat(np.arange(len(nat)), nat).astype(np.int64),
    }
    q = rng.normal(0, 0.4, base).astype(np.float32)
    return batch, q


BOUNDS = (1.0, 1.5, 3.0, 3.5, 4.0, 5.0, 7.5)


def _not_on_a_boundary(batch, bounds):
    R, o = batch["_positions"].astype(np.float64), batch["_offsets"].astype(np.float64)
    d = np.linalg.norm(R[batch["_idx_j"]] - R[batch["_idx_i"]] + o, axis=1)
    return all(np.abs(d - b).min() > 1e-4 for b in bounds)


TERMS = [
    ("zbl", dict(cut=None, d_max=None)),
    ("zbl", dict(cut=4.0, d_max=3.5)),
    ("coulomb", dict(damped=None, cut=None, d_max=None)),
    ("coulomb", dict(damped=(1.0, 4.0), cut=7.5, d_max=None)),
    ("coulomb", dict(damped=(1.5, 3.0), cut=None, d_max=5.0)),
]


def _module(kind, kw):
    from schnetpack_b200 import atomistic as A
    from schnetpack_b200 import nn as snn

    if kind == "zbl":
        return A.ZBLRepulsionEnergy("kcal/mol", "Ang", "e",
                                    cutoff_fn=snn.CosineCutoff(kw["cut"]) if kw["cut"] is not None else None)
    pot = A.CoulombPotential() if kw["damped"] is None else A.DampedCoulombPotential(snn.SwitchFunction(*kw["damped"]))
    return A.EnergyCoulomb("kcal/mol", "Ang", pot, "e", use_neighbors_lr=False, cutoff=kw["cut"])


def _evaluate_term(mod, batch, q, kw):
    from schnetpack_b200 import atomistic as A

    x = torch_batch(batch, torch.float32, DEV)
    x["_positions"].requires_grad_()
    x = A.PairwiseDistances()(x)
    if kw.get("d_max") is not None:
        x["_short_range_cutoff"] = torch.tensor(float(kw["d_max"]), dtype=torch.float64)
    qt = torch.as_tensor(q, device=DEV).requires_grad_()
    x["partial_charges"] = qt[:, None]
    e = mod(x)["e"]
    g_R, g_q = torch.autograd.grad(e.sum(), [x["_positions"], qt], allow_unused=True)
    return e.detach(), g_R, (g_q if g_q is not None else torch.zeros_like(qt))


def _oracle_term(kind, kw, mod, batch, q):
    R = torch.as_tensor(batch["_positions"], dtype=torch.float64).requires_grad_()
    qd = torch.as_tensor(q, dtype=torch.float64).requires_grad_()
    ii, jj = torch.as_tensor(batch["_idx_i"]), torch.as_tensor(batch["_idx_j"])
    r = PO.rij(R, ii, jj, torch.as_tensor(batch["_offsets"], dtype=torch.float64))
    n_sys = len(batch["_n_atoms"])
    if kind == "zbl":
        params = [getattr(mod, k).detach().double() for k in ("a_pow", "a_div", "coefficients", "exponents")]
        e = PO.zbl_energy(batch["_atomic_numbers"], r, ii, jj, batch["_idx_m"], n_sys, params, float(mod.ke),
                          cutoff=kw["cut"], d_max=kw["d_max"])
    else:
        shift = float(mod.shift) if mod.shift is not None else None
        e = PO.coulomb_energy(qd, r, ii, jj, batch["_idx_m"], n_sys, float(mod.ke[0]), damped=kw["damped"],
                              cutoff=kw["cut"], shift=shift, d_max=kw["d_max"])
    g_R, g_q = torch.autograd.grad(e.sum(), [R, qd], allow_unused=True)
    return e.detach(), g_R, (g_q if g_q is not None else torch.zeros_like(qd))


@pytest.mark.parametrize("kind,kw", TERMS)
def test_adversarial_batches_match_fp64_oracle(kind, kw):
    batch, q = _adversarial()
    bounds = [v for v in (kw.get("cut"), kw.get("d_max")) + tuple(kw.get("damped") or ()) if v is not None]
    assert _not_on_a_boundary(batch, bounds)
    mod = _module(kind, kw).to(DEV).eval()
    e, g_R, g_q = _evaluate_term(mod, batch, q, kw)
    e0, g_R0, g_q0 = _oracle_term(kind, kw, mod.cpu(), batch, q)
    assert e.shape == (4,) and float(e[-1]) == 0.0                     # the trailing empty system
    assert rel(e.cpu().numpy(), e0.numpy()) <= TOL
    assert rel(g_R.cpu().numpy(), g_R0.numpy()) <= TOL
    if kind == "coulomb":
        assert rel(g_q.cpu().numpy(), g_q0.numpy()) <= TOL
    # determinism: a second evaluation is bitwise the same
    mod = mod.to(DEV)
    e2, g_R2, g_q2 = _evaluate_term(mod, batch, q, kw)
    assert torch.equal(e, e2) and torch.equal(g_R, g_R2) and torch.equal(g_q, g_q2)


def test_charges_are_differentiable_only_under_a_coulomb_term(case):
    name, batch, model, _ = case
    assert model.output_modules[0].differentiable_charges
    out = _run(model, torch_batch(batch, torch.float32, DEV))
    assert out["partial_charges"].requires_grad


def test_two_runs_are_bitwise_equal(case):
    name, batch, model, _ = case
    o1 = _run(model, torch_batch(batch, torch.float32, DEV))
    o2 = _run(model, torch_batch(batch, torch.float32, DEV))
    for k in ("energy", "forces", "partial_charges"):
        assert torch.equal(o1[k], o2[k]), k


def test_graph_replay_with_new_positions_and_zbl_parameters():
    from schnetpack_b200.model import GraphedPotential

    batch, w, _ = load_case("a")
    model = package_model("a", w, torch.float32).to(DEV).eval()
    gp = GraphedPotential(model)
    x = torch_batch(batch, torch.float32, DEV)
    gp(x)
    rng = np.random.default_rng(5)
    batch2 = dict(batch)
    batch2["_positions"] = (batch["_positions"] + rng.normal(0, 0.02, batch["_positions"].shape)).astype(np.float32)
    zbl = model.output_modules[2]
    with torch.no_grad():
        zbl.a_pow.add_(0.05)
        zbl.exponents.mul_(1.1)
    replay = {k: v.clone() for k, v in gp(torch_batch(batch2, torch.float32, DEV)).items()}
    eager = model(torch_batch(batch2, torch.float32, DEV))
    for k in ("energy", "forces", "partial_charges"):
        assert rel(replay[k].cpu().numpy(), eager[k].detach().cpu().numpy()) <= 1e-6, k


def test_device_md_nve_conserves_energy_and_refuses_uncut_coulomb():
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device

    batch, w, _ = load_case("a")
    model = package_model("a", w, torch.float32).to(DEV).eval()
    data = dict(batch)
    n = batch["_positions"].shape[0]
    masses = torch.as_tensor(np.where(batch["_atomic_numbers"] == 1, 1.008, 12.0), dtype=torch.float32)
    rng = np.random.default_rng(0)
    mom = torch.as_tensor(rng.normal(0, 0.05, (n, 3)), dtype=torch.float32) * masses[:, None]
    md = M.DeviceMD(model, batch_to_device(data, DEV), masses, time_step=0.02 * M.FS_MD, cutoff=9.0, capacity=n * 64,
                    momenta=mom)
    totals, pots = [], []
    for _ in range(20):
        md.run(5)
        pot = float(md.potential_energy().sum())
        totals.append(pot + float(md.kinetic_energy()))
        pots.append(pot)
    drift = max(abs(t - totals[0]) for t in totals)
    swing = max(pots) - min(pots)
    assert swing > 0.0
    # bound: the total energy moves by less than 2 % of the potential energy's swing over the 100 steps
    assert drift <= 0.02 * swing, (drift, swing)
    # a Coulomb term without a cutoff would sum the padding pairs of the fixed-capacity list
    mb = package_model("a", w, torch.float32).to(DEV).eval()
    mb.output_modules[3].cutoff = None
    with pytest.raises(ValueError, match="EnergyCoulomb without a cutoff"):
        M.DeviceMD(mb, batch_to_device(data, DEV), masses, time_step=0.02 * M.FS_MD, cutoff=9.0, capacity=n * 64)


def test_dipole_gradients_unchanged_without_a_charge_gradient():
    """Differentiable charges with nothing downstream of them run the same reverse as return_charges=False."""
    from schnetpack_b200 import atomistic as A
    from schnetpack_b200 import synthetic as S

    data = S.aspirin_batch(4, seed=2)
    torch.manual_seed(0)
    for gated in (False, True):
        heads = [A.DipoleMoment(32, return_charges=rc, use_vector_representation=gated) for rc in (False, True)]
        heads[1].load_state_dict(heads[0].state_dict())
        heads[1].differentiable_charges = True
        res = []
        for h in heads:
            h = h.to(DEV).eval()
            x = torch_batch(data, torch.float32, DEV)
            s = torch.randn(x["_positions"].shape[0], 32, generator=torch.Generator().manual_seed(1)).to(DEV)
            V = torch.randn(x["_positions"].shape[0], 3, 32, generator=torch.Generator().manual_seed(2)).to(DEV)
            s.requires_grad_(); V.requires_grad_(); x["_positions"].requires_grad_()
            x["scalar_representation"], x["vector_representation"] = s, V
            y = h(x)["dipole_moment"]
            g = torch.autograd.grad((y * torch.arange(1.0, 4.0, device=DEV)).sum(), [s, x["_positions"]] +
                                    ([V] if gated else []))
            res.append((y.detach(),) + tuple(g))
        for a, b in zip(*res):
            assert torch.equal(a, b)
