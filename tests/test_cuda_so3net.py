"""GPU: SO3net on the kernels of csrc/so3net.cu against the reference (golden fixtures and the live modules), robustness
(neighbour order, degenerate batches, rotations, finite differences, bitwise repeatability) and integration (graph replay,
stress through Strain and the virial buffer, DeviceMD NVE and NPT)."""
import math

import numpy as np
import pytest
import torch

from conftest import load_case, rel_err
from oracle import ref_loader as rl
import so3net_oracle as SO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = ["so3net_ethanol_l1", "so3net_aspirin_b4", "so3net_lmax3", "so3net_bessel_shared", "so3net_box_216"]


def _np(t):
    return t.detach().double().cpu().numpy()


def _model(spec, params, **kw):
    from schnetpack_b200.model import from_spec

    return from_spec(dict(spec, **kw), params, torch.device(DEV))


def _run(model, data):
    from schnetpack_b200.model import batch_to_device

    x = batch_to_device(data, torch.device(DEV))
    out = model(x)
    return out, x


@pytest.mark.parametrize("name", CASES)
def test_golden(name):
    spec, params, inputs, _, ref64 = load_case(name)
    model = _model(spec, params)
    out, x = _run(model, inputs)
    torch.cuda.synchronize()
    assert rel_err(_np(out["energy"]), ref64["energy"]) < 1e-5
    assert rel_err(_np(out["forces"]), ref64["forces"]) < 1e-5
    assert rel_err(_np(x["scalar_representation"]), ref64["scalar_representation"]) < 1e-5
    assert rel_err(_np(x["multipole_representation"]), ref64["multipole_representation"]) < 1e-5
    if "vector_representation" in ref64:
        assert rel_err(_np(x["vector_representation"]), ref64["vector_representation"]) < 1e-5


@pytest.mark.skipif(not rl.available(), reason="reference modules absent")
@pytest.mark.parametrize("lmax", [0, 1, 2, 3])
@pytest.mark.parametrize("F", [36, 64, 128])
def test_live_reference_on_the_gpu_then_convert_model(lmax, F):
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import convert_model

    spec = S.model_spec("so3net", n_atom_basis=F, n_interactions=2, lmax=lmax, n_rbf=32 if lmax == 3 else 20)
    params = S.init_params(spec, seed=40 + lmax)
    data = S.aspirin_batch(3, seed=lmax)
    ref = SO.build_reference(spec, params, torch.float32, torch.device(DEV))
    r = SO.evaluate(ref, data, torch.float32, torch.device(DEV))
    mine = convert_model(ref.to("cpu")).to(DEV)
    out, x = _run(mine, data)
    torch.cuda.synchronize()
    for k, v in (("energy", out["energy"]), ("forces", out["forces"]),
                 ("scalar_representation", x["scalar_representation"]),
                 ("multipole_representation", x["multipole_representation"])):
        assert rel_err(_np(v), _np(r[k])) < 1e-5, k


def _base(lmax=2, F=64, seed=5):
    from schnetpack_b200 import synthetic as S

    spec = dict(S.model_spec("so3net", n_atom_basis=F, n_interactions=2, lmax=lmax), return_vector_representation=True)
    return spec, S.init_params(spec, seed=seed)


def test_unsorted_neighbor_list_and_bitwise_repeat():
    from schnetpack_b200 import synthetic as S

    spec, params = _base()
    model = _model(spec, params)
    data = S.aspirin_batch(4, seed=2)
    o1, _ = _run(model, data)
    o2, _ = _run(model, data)
    torch.cuda.synchronize()
    assert torch.equal(o1["energy"], o2["energy"]) and torch.equal(o1["forces"], o2["forces"])
    perm = np.random.default_rng(0).permutation(data["_idx_i"].shape[0])
    shuffled = dict(data, _idx_i=data["_idx_i"][perm], _idx_j=data["_idx_j"][perm], _offsets=data["_offsets"][perm])
    o3, _ = _run(model, shuffled)
    assert rel_err(_np(o3["energy"]), _np(o1["energy"])) < 1e-6
    assert rel_err(_np(o3["forces"]), _np(o1["forces"])) < 1e-6


def test_degenerate_batches_are_finite():
    from schnetpack_b200 import synthetic as S

    spec, params = _base()
    model = _model(spec, params)
    lone = S.ethanol_batch(1)
    lone = {k: v for k, v in lone.items()}
    one_atom = dict(lone, _atomic_numbers=lone["_atomic_numbers"][:1], _positions=lone["_positions"][:1],
                    _idx_m=lone["_idx_m"][:1], _n_atoms=np.array([1]), _idx_i=np.zeros(0, np.int64),
                    _idx_j=np.zeros(0, np.int64), _offsets=np.zeros((0, 3), np.float32))
    far = S.ethanol_batch(1, cutoff=0.1)                   # a system without edges
    mixed = S._collate([{k: v for k, v in S._open_system(S.ETHANOL_Z[:1], S.ETHANOL_R[:1], 5.0).items()},
                        S._open_system(S.ETHANOL_Z, S.ETHANOL_R * 10.0, 5.0),
                        S._open_system(S.ASPIRIN_Z, S.ASPIRIN_R, 5.0)])
    for data in (one_atom, far, mixed):
        out, _ = _run(model, data)
        torch.cuda.synchronize()
        assert torch.isfinite(out["energy"]).all() and torch.isfinite(out["forces"]).all()
    ref = SO.energy_forces(dict(spec), params, mixed, dtype=torch.float64)
    out, _ = _run(model, mixed)
    assert rel_err(_np(out["energy"]), ref["energy"].numpy()) < 1e-5
    assert rel_err(_np(out["forces"]), ref["forces"].numpy()) < 1e-5


def test_rotation_equivariance():
    from scipy.spatial.transform import Rotation

    from schnetpack_b200 import synthetic as S

    spec, params = _base(lmax=3, F=32)
    model = _model(spec, params)
    data = S.aspirin_batch(2, seed=3)
    Rm = Rotation.from_rotvec([0.3, -1.1, 0.7]).as_matrix()
    rot = dict(data, _positions=(data["_positions"].astype(np.float64) @ Rm.T).astype(np.float32))
    o1, x1 = _run(model, data)
    o2, x2 = _run(model, rot)
    torch.cuda.synchronize()
    assert rel_err(_np(o2["energy"]), _np(o1["energy"])) < 1e-5
    assert rel_err(_np(o2["forces"]), _np(o1["forces"]) @ Rm.T) < 1e-5
    v1, v2 = _np(x1["vector_representation"]), _np(x2["vector_representation"])
    assert rel_err(v2, np.einsum("ab,nbf->naf", Rm, v1)) < 1e-4


def test_forces_match_finite_differences():
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device

    spec, params = _base(lmax=2, F=32)
    model = _model(spec, params)
    data = S.ethanol_batch(1)
    out, _ = _run(model, data)
    f = _np(out["forces"])
    x = batch_to_device(data, torch.device(DEV))
    h = 1e-2
    fd = np.zeros_like(f)
    for a in range(f.shape[0]):
        for k in range(3):
            e = []
            for sgn in (1.0, -1.0):
                xx = {kk: v.clone() for kk, v in x.items()}
                xx["_positions"][a, k] += sgn * h
                e.append(float(model(xx)["energy"].detach().double().sum()))
            fd[a, k] = -(e[0] - e[1]) / (2 * h)
    assert rel_err(fd, f) < 2e-3


def test_graphed_potential_replay_equals_eager():
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import GraphedPotential

    spec, params = _base()
    model = _model(spec, params)
    data = S.aspirin_batch(8, seed=6)
    eager, _ = _run(model, data)
    gp = GraphedPotential(model)
    from schnetpack_b200.model import batch_to_device

    out = gp(batch_to_device(data, torch.device(DEV)))
    out = gp.replay()
    torch.cuda.synchronize()
    assert torch.equal(out["energy"], eager["energy"]) and torch.equal(out["forces"], eager["forces"])


def test_stress_through_strain_and_virial():
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device

    spec, params, inputs, _, _ = load_case("so3net_box_216")
    ref = SO.energy_forces(spec, params, inputs, dtype=torch.float64, stress=True)
    model = _model(spec, params, stress=True)
    out, _ = _run(model, inputs)
    torch.cuda.synchronize()
    assert rel_err(_np(out["stress"]), ref["stress"].numpy()) < 1e-5
    plain = _model(spec, params)
    x = batch_to_device(inputs, torch.device(DEV))
    W = torch.zeros((1, 3, 3), dtype=torch.float64, device=DEV)
    x["_virial"] = W
    plain(x)
    torch.cuda.synchronize()
    cell = inputs["_cell"].reshape(3, 3).astype(np.float64)
    assert rel_err(_np(W) / abs(np.linalg.det(cell)), ref["stress"].numpy()) < 1e-5
    assert S is not None


def _box(F=64):
    from schnetpack_b200 import synthetic as S

    spec = S.model_spec("so3net", n_atom_basis=F, n_interactions=2, lmax=2)
    data = S.periodic_box(150, seed=9)
    params = S.init_params(spec, seed=8)
    masses = np.where(data["_atomic_numbers"] == 8, 16.0, 1.0)
    p0 = np.random.default_rng(2).normal(0, 0.05, (data["_positions"].shape[0], 3))
    return spec, data, params, masses, p0


def test_device_md_nve_follows_the_oracle():
    from schnetpack_b200.md import DeviceMD
    from schnetpack_b200.model import batch_to_device

    spec, data, params, masses, p0 = _box()
    model = _model(spec, params)
    md = DeviceMD(model, batch_to_device(data, torch.device(DEV)), torch.as_tensor(masses), time_step=1e-3,
                  cutoff=spec["cutoff"], capacity=int(data["_idx_i"].shape[0] * 1.5), momenta=torch.as_tensor(p0))
    md.run(12)
    torch.cuda.synchronize()
    x_ref, p_ref, e_ref, f_ref = SO.nve_trajectory(spec, params, data, masses, p0, 1e-3, 12)
    assert rel_err(_np(md.positions), x_ref) < 1e-6
    assert rel_err(_np(md.momenta), p_ref) < 1e-4
    assert rel_err(_np(md.potential_energy()), e_ref) < 1e-5
    assert rel_err(_np(md.forces), f_ref) < 1e-4


def test_device_md_npt_moves_the_cell():
    from schnetpack_b200 import md as M
    from schnetpack_b200.model import batch_to_device

    spec, data, params, masses, p0 = _box()
    model = _model(spec, params)
    md = M.DeviceMD(model, batch_to_device(data, torch.device(DEV)), torch.as_tensor(masses), time_step=0.5 * M.FS_MD,
                    cutoff=spec["cutoff"], capacity=int(data["_idx_i"].shape[0] * 2), momenta=torch.as_tensor(p0),
                    barostat=M.NHCBarostatIsotropic(1.0, 300.0, 100.0))
    v0 = float(md.volume()[0])
    md.run(50)
    torch.cuda.synchronize()
    assert float(md.volume()[0]) != v0 and math.isfinite(float(md.volume()[0]))
    assert torch.isfinite(md.potential_energy()).all() and torch.isfinite(md.forces).all()
