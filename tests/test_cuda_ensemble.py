"""GPU checks of the model ensembles: the kernels of csrc/ensemble.cu against the fp64 oracle (tests/ensemble_oracle.py) on
adversarial layouts, NNEnsemble against the reference's own statistics (tests/golden/ensemble_batch.npz), and the ensemble
modes of DeviceMD and DeviceLBFGS against the members evaluated one by one."""
import json
import os

import numpy as np
import pytest
import torch

import ensemble_oracle as EO
import heads_oracle as HO
from conftest import GOLDEN, rel_err
from schnetpack_b200 import ensemble as E
from schnetpack_b200 import md as M
from schnetpack_b200 import ops
from schnetpack_b200 import synthetic as S
from schnetpack_b200.model import GraphedPotential, batch_to_device, from_spec
from schnetpack_b200.neighbors import CellListNeighborList
from schnetpack_b200.relax import DeviceLBFGS, LBFGSState

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
F32 = 2.0 ** -24


# ---- kernels against the fp64 oracle ---------------------------------------------------------------------------------------
def _layout(K, seed, identical=False):
    rng = np.random.default_rng(seed)
    n_atoms = np.array([300, 1, 0, 129, 0, 5, 1000, 128, 1])          # systems across CTAs of 128, one atom, empty
    N, B = int(n_atoms.sum()), n_atoms.shape[0]
    f = rng.normal(size=(1 if identical else K, N, 3)) * rng.uniform(0.1, 10.0, size=(1, N, 1))
    f = np.broadcast_to(f, (K, N, 3)).astype(np.float32)
    e = (1e4 + 1e-3 * rng.normal(size=(1 if identical else K, B)))  # mean 1e4, spread 1e-3
    e = np.broadcast_to(e, (K, B)).astype(np.float32)
    s = np.broadcast_to(rng.normal(size=(1 if identical else K, B, 3, 3)), (K, B, 3, 3)).astype(np.float32)
    return n_atoms, f, e, s


def _dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).to(DEV)


def _assert_bound(got, ref, rel, absolute=0.0):
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape
    err = np.abs(got - ref)
    bound = rel * np.abs(ref) + absolute
    assert np.all(err <= bound), float(np.max(err - bound))


@pytest.mark.parametrize("identical", [False, True])
@pytest.mark.parametrize("K", [2, 3, 8])
def test_kernels_match_oracle(K, identical):
    n_atoms, f, e, s = _layout(K, seed=K, identical=identical)
    B = n_atoms.shape[0]
    idx_m = _dev(np.repeat(np.arange(B), n_atoms))
    sys_ptr = ops.segment_ptr(idx_m, B)
    fd, ed, sd = _dev(f), _dev(e), _dev(s)
    f64, e64, s64 = f.astype(np.float64), e.astype(np.float64), s.astype(np.float64)

    runs = []
    for _ in range(2):
        out = {}
        out["e_mean"], out["e_var"], out["e_std"] = E.ensemble_moments(ed, ddof=1, std=True)
        out["e_mean0"], out["e_var0"], _ = E.ensemble_moments(ed, ddof=0, mean_scale=2.0, spread_scale=3.0)
        out["f_mean"], out["f_var"], out["terms"] = E.ensemble_forces(fd, idx_m, sys_ptr, B, terms=True)
        for cls in (E.AbsoluteUncertainty, E.RelativeUncertainty):
            fn = cls(energy_weight=1.0, force_weight=2.0, stress_weight=0.5)
            out[cls.__name__] = fn({"energy": ed, "forces": fd, "stress": sd}, idx_m, B)
        runs.append({k: v.cpu() for k, v in out.items()})
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k                 # bitwise reproducible
    r = {k: v.numpy() for k, v in runs[0].items()}

    _assert_bound(r["e_mean"], e64.mean(0), F32)
    _assert_bound(r["e_var"], e64.var(0, ddof=1), 2 * F32, 1e-30)
    _assert_bound(r["e_std"], e64.std(0, ddof=1), 2 * F32, 1e-30)
    _assert_bound(r["e_mean0"], 2.0 * e64.mean(0), F32)
    _assert_bound(r["e_var0"], 3.0 * e64.var(0), 2 * F32, 1e-30)
    _assert_bound(r["f_mean"], f64.mean(0), F32, 1e-30)
    _assert_bound(r["f_var"], f64.var(0, ddof=1), 2 * F32, 1e-30)
    _assert_bound(r["terms"], EO.force_terms(f64, n_atoms), 1e-12, 1e-300)
    assert r["terms"][2].tolist() == [0.0, 0.0] and r["terms"][4].tolist() == [0.0, 0.0]     # empty systems
    for name, relative in (("AbsoluteUncertainty", False), ("RelativeUncertainty", True)):
        ref = EO.batched_uncertainty(e64, f64, n_atoms, s64, (1.0, 2.0, 0.5), relative)
        _assert_bound(r[name], ref, 1e-12, 1e-300)
        assert np.all(np.isfinite(r[name]))
    if identical:
        assert not r["e_var"].any() and not r["f_var"].any() and not r["terms"].any()
        assert not r["RelativeUncertainty"].any()


def test_two_pass_keeps_a_small_spread_next_to_a_large_mean():
    x = np.float32(1e4) + np.array([[0.0], [1e-3], [-1e-3], [2e-3]], dtype=np.float32)     # fp32-exact offsets of 1e4
    _, var, _ = E.ensemble_moments(_dev(x), ddof=1)
    ref = x.astype(np.float64).var(0, ddof=1)
    _assert_bound(var.cpu().numpy(), ref, 2 * F32)


def test_refusals_of_the_kernels():
    x = torch.zeros(1, 4, device=DEV)
    with pytest.raises(ValueError):
        E.ensemble_moments(x, ddof=1)                                  # K = 1 has no unbiased variance
    with pytest.raises(ValueError, match="total_weight"):
        E.AbsoluteUncertainty(force_weight=0.0)


def test_malformed_inputs_are_refused_on_the_host():
    n_atoms, f, e, _ = _layout(3, seed=0)
    B = n_atoms.shape[0]
    idx_m = _dev(np.repeat(np.arange(B), n_atoms))
    sys_ptr = ops.segment_ptr(idx_m, B)
    fd, ed = _dev(f), _dev(e)
    with pytest.raises(ValueError, match=r"\[K, N, 3\]"):
        E.ensemble_forces(fd.reshape(3, -1), idx_m, sys_ptr, B, terms=True)
    with pytest.raises(ValueError, match="idx_m"):
        E.ensemble_forces(fd, idx_m[:-1].contiguous(), sys_ptr, B, terms=True)
    with pytest.raises(ValueError, match="out_mean"):
        E.ensemble_moments(ed, out_mean=torch.empty(B - 1, device=DEV))
    with pytest.raises(ValueError, match="workspace"):
        E.ensemble_forces(fd, idx_m, sys_ptr, B, terms=True, workspace=torch.empty(8, dtype=torch.uint8, device=DEV))
    fn = E.AbsoluteUncertainty(energy_weight=1.0)
    with pytest.raises(ValueError, match="member counts"):
        fn({"energy": ed[:2].contiguous(), "forces": fd}, idx_m, B)
    with pytest.raises(ValueError, match="sorted"):
        fn({"energy": ed, "forces": fd}, idx_m.flip(0).contiguous(), B)
    with pytest.raises(ValueError, match="entries"):
        fn({"energy": ed, "forces": fd}, idx_m[1:].contiguous(), B)


# ---- NNEnsemble against the reference's NNEnsemble ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(GOLDEN, "ensemble_batch.npz"))
    members = [from_spec(spec, S.init_params(spec, seed=seed), DEV) for spec, seed in json.loads(str(z["members_json"]))]
    inputs = {k[3:]: z[k] for k in z.files if k.startswith("in:")}
    return z, members, inputs


def test_nn_ensemble_matches_reference(golden):
    z, members, inputs = golden
    ens = E.NNEnsemble(members, ["energy", "forces"])
    means, stds = ens(batch_to_device(inputs, DEV))
    for k in ("energy", "forces"):
        assert rel_err(means[k].cpu(), z["nn:mean:" + k]) < 1e-5, k
        assert rel_err(stds[k].cpu(), z["nn:std:" + k]) < 1e-5, k
    graphed = GraphedPotential(ens)
    g_means, g_stds = graphed(batch_to_device(inputs, DEV))
    g_means, g_stds = graphed(batch_to_device(inputs, DEV))        # a replay
    for k in ("energy", "forces"):
        assert rel_err(g_means[k].cpu(), means[k].cpu()) < 1e-6 and rel_err(g_stds[k].cpu(), stds[k].cpu()) < 1e-6


def test_uncertainty_of_reference_predictions_matches_ase(golden):
    z, _, inputs = golden
    idx_m = _dev(inputs["_idx_m"])
    B = inputs["_n_atoms"].shape[0]
    pred = {"energy": _dev(z["pred:energy"].astype(np.float32)), "forces": _dev(z["pred:forces"].astype(np.float32)),
            "stress": _dev(z["pred:stress"].astype(np.float32))}
    for relative, cls in ((False, E.AbsoluteUncertainty), (True, E.RelativeUncertainty)):
        ref = z["unc:relative" if relative else "unc:absolute"]
        for w, (we, wf, ws) in enumerate(z["weights"]):
            u = cls(energy_weight=we, force_weight=wf, stress_weight=ws)(pred, idx_m, B).cpu().numpy()
            assert rel_err(u, ref[w]) < 1e-5, (relative, w)


# ---- DeviceMD and DeviceLBFGS --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def md_setup():
    spec = S.model_spec("painn", n_atom_basis=32, n_interactions=2)
    members = [from_spec(spec, S.init_params(spec, seed=s), DEV) for s in (1, 2, 3)]
    data = HO._centered(S.aspirin_batch(3, seed=2))
    masses = torch.as_tensor([HO.MASSES[int(z)] for z in data[S.Z]], dtype=torch.float32)
    rng = np.random.default_rng(0)
    momenta = torch.as_tensor(rng.normal(size=(masses.shape[0], 3)) * np.sqrt(masses.numpy() * M.KB_MD * 300.0)[:, None],
                              dtype=torch.float32)
    return spec, members, data, masses, momenta


def _md(md_setup, use_graph=True, capacity=12, model=None, **kw):
    spec, members, data, masses, momenta = md_setup
    kw.setdefault("uncertainty_fn", E.AbsoluteUncertainty(energy_weight=1.0, force_weight=1.0))
    kw.setdefault("property_conversion", {"energy": 3.0})
    return M.DeviceMD(members if model is None else model, batch_to_device(data, DEV), masses, time_step=0.5 * M.FS_MD,
                      cutoff=spec["cutoff"], capacity=int(data[S.Z].shape[0]) * 160, momenta=momenta,
                      use_graph=use_graph, record_capacity=capacity, energy_conversion=2.0, **kw)


def _members_at(drv, positions):
    """every member on its own, with a neighbour list of its own -> stacked fp64 energies [K, B] and forces [K, N, 3]"""
    es, fs = [], []
    for m in drv.ensemble:
        x = {k: (v.detach().clone() if v.is_floating_point() else v) for k, v in drv.static.items()}
        x[S.R] = positions.clone()
        nl = CellListNeighborList(drv.nl._cutoff, capacity=drv.nl.capacity, pad=True)
        out = m(nl(x))
        es.append(out["energy"].detach().double().cpu().numpy())
        fs.append(out["forces"].detach().double().cpu().numpy())
    return np.stack(es), np.stack(fs)


def test_device_md_matches_members_evaluated_separately(md_setup):
    """energy_conversion = 2 acts on the dynamics only; properties follow property_conversion (energy x 3, forces x 1)
    as the reference's calculator does, and the uncertainty is that of the properties' energies and forces"""
    md = _md(md_setup)
    pos, forces = [], []
    for _ in range(12):
        md.run(1)
        pos.append(md.model_positions.clone())
        forces.append(md.forces.clone())
    rec = md.drain()
    assert set(rec) == {"energy", "energy_var", "forces", "forces_var", "uncertainty"}
    n_atoms = md_setup[2][S.n_atoms]
    for s in range(12):
        e, f = _members_at(md, pos[s])
        assert rel_err(forces[s].cpu(), f.mean(0)) < 1e-5, s
        assert rel_err(rec["energy"][s][0], 3.0 * e.mean(0)) < 1e-5, s
        assert rel_err(rec["energy_var"][s][0], 3.0 * e.var(0, ddof=1)) < 1e-5, s
        assert rel_err(rec["forces"][s][0], f.mean(0)) < 1e-5, s
        assert rel_err(rec["forces_var"][s][0], f.var(0, ddof=1)) < 1e-5, s
        u = EO.batched_uncertainty(3.0 * e, f, n_atoms, weights=(1.0, 1.0, 0.0))
        assert rel_err(rec["uncertainty"][s][0], u) < 1e-5, s


def test_device_md_graph_equals_eager(md_setup):
    a, b = _md(md_setup, use_graph=True), _md(md_setup, use_graph=False)
    a.run(6)
    b.run(6)
    ra, rb = a.drain(), b.drain()
    for k in ra:
        assert torch.equal(ra[k], rb[k]), k
    assert torch.equal(a.positions, b.positions) and torch.equal(a.forces, b.forces)


def test_device_md_ring_polymer_shapes(md_setup):
    md = _md(md_setup, ring_polymer=M.RingPolymer(4, 300.0), capacity=3)
    md.run(3)
    n = int(md_setup[2][S.Z].shape[0])
    assert md.properties["uncertainty"].shape == (4, 3) and md.properties["energy_var"].shape == (4, 3)
    assert md.properties["forces_var"].shape == (4, n, 3)
    assert md.recorded("uncertainty").shape == (3, 4, 3) and torch.isfinite(md.recorded("uncertainty")).all()


class _Reshaped(torch.nn.Module):
    def __init__(self, m):
        super().__init__()
        self.m = m

    def forward(self, x):
        out = dict(self.m(x))
        out["energy"] = out["energy"].reshape(-1, 1)
        return out


def test_device_md_refusals(md_setup):
    spec, members, data, *_ = md_setup
    with pytest.raises(NotImplementedError, match="ensemble_calculator.py:62-68"):
        _md(md_setup, compute_stress=True)
    with pytest.raises(NotImplementedError, match="ensemble_calculator.py:62-68"):
        _md(md_setup, barostat=M.NHCBarostatIsotropic(1.0, 300.0, 100.0))
    with pytest.raises(ValueError, match="at least two"):
        _md(md_setup, model=[members[0]])
    with pytest.raises(ValueError, match="shape"):
        _md(md_setup, model=[members[0], _Reshaped(members[1])])
    with pytest.raises(ValueError, match="uncertainty_fn needs an ensemble"):
        _md(md_setup, model=members[0], capacity=0, property_conversion=None)
    with pytest.raises(TypeError, match="uncertainty_fn"):
        _md(md_setup, uncertainty_fn=lambda *a: None)
    with pytest.raises(ValueError, match="uncertainty_fn reads"):
        _md(md_setup, uncertainty_fn=E.AbsoluteUncertainty(energy_key="free_energy", energy_weight=1.0))
    with pytest.raises(ValueError, match="not required"):
        _md(md_setup, property_conversion={"dipole_moment": 2.0})


def test_device_md_default_conversions_are_one(md_setup):
    md = _md(md_setup, property_conversion=None, capacity=0)
    e, f = _members_at(md, md.model_positions)
    assert rel_err(md.properties["energy"][0].cpu(), e.mean(0)) < 1e-5
    assert rel_err(md.properties["forces_var"][0].cpu(), f.var(0, ddof=1)) < 1e-5


def test_device_lbfgs_follows_the_oracle_mean_forces(md_setup):
    spec, members, data, *_ = md_setup
    batch = batch_to_device(data, DEV)
    dev = DeviceLBFGS(members, batch, cutoff=spec["cutoff"], capacity=int(data[S.Z].shape[0]) * 160)

    idx_m = batch[S.idx_m]
    mp = batch[S.R].clone()
    opt = LBFGSState(mp.double(), idx_m, 3, model_positions=mp)

    def mean_forces():
        return torch.as_tensor(_members_at(dev, opt.model_positions)[1].mean(0), dtype=torch.float32, device=DEV)

    f = mean_forces()
    opt.check(f)
    opt.set_fmax(0.05)
    opt.check(f)
    for _ in range(4):
        opt.step(f)
        f = mean_forces()
        opt.check(f)
    dev.run(fmax=0.05, steps=4, check_every=4)
    assert rel_err(dev.positions.cpu(), opt.r.cpu()) < 1e-6
    assert rel_err(dev.forces.cpu(), f.cpu()) < 1e-5
    e, fm = _members_at(dev, dev.model_positions)
    unc = dev.get_uncertainty()
    assert rel_err(unc["energy_uncertainty"].cpu(), e.std(0, ddof=1)) < 1e-5
    assert rel_err(unc["forces_uncertainty"].cpu(), fm.std(0, ddof=1)) < 1e-5
