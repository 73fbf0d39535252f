"""GPU: the CUDA path (through the module API -> C ABI -> sm_90a kernels) against
  (1) the committed golden fixtures produced by the UNMODIFIED reference (tests/golden/*.npz), and
  (2) the oracle (oracle/spk_oracle.py, fp64) on seeded inputs of the named configurations.

Tolerance (BASELINE.json north_star): energies / forces within 1e-5 relative fp32, measured as
max|x - x_ref| / max|x_ref| against the fp64 reference; the fp32 reference's own error against fp64 is printed
alongside for scale.
"""
import numpy as np
import pytest
import torch

from conftest import MODEL_CASES, load_case, rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-5


def _run_cuda(spec, params, inputs):
    import schnetpack_b200 as sb
    from schnetpack_b200.model import batch_to_device, from_spec

    dev = torch.device("cuda:0")
    model = from_spec(spec, params, dev)
    x = batch_to_device(inputs, dev)
    if "_Rij" in x:  # padded neighbour list: call representation + head directly on the given r_ij
        x["_Rij"].requires_grad_(bool(spec.get("forces", True)))
        x = model.representation(x)
        x = model.output_modules[0](x)
        res = {"energy": x["energy"]}
    else:
        res = model(x)
    out = {k: v.detach().cpu().numpy() for k, v in res.items()}
    out["scalar_representation"] = x["scalar_representation"].detach().cpu().numpy()
    if "vector_representation" in x:
        out["vector_representation"] = x["vector_representation"].detach().cpu().numpy()
    return out


@pytest.mark.parametrize("name", MODEL_CASES)
def test_golden_parity(name):
    spec, params, inputs, ref32, ref64 = load_case(name)
    out = _run_cuda(spec, params, inputs)
    errs = {}
    for k in ("energy", "forces", "scalar_representation", "vector_representation"):
        if k in ref64 and k in out:
            errs[k] = (rel_err(out[k], ref64[k]), rel_err(ref32[k], ref64[k]))
    print(name, {k: f"cuda {a:.2e} / ref-fp32 {b:.2e}" for k, (a, b) in errs.items()})
    for k, (a, b) in errs.items():
        assert a < TOL, f"{name}:{k} rel err {a:.3e} (reference fp32 itself: {b:.3e})"


def _oracle_vs_cuda(cfg, **kw):
    from oracle import spk_oracle as O
    from schnetpack_b200 import synthetic as S

    spec, inputs = S.make_config(cfg, **kw)
    params = S.init_params(spec, seed=7)
    out = _run_cuda(spec, params, inputs)
    ref = O.energy_forces(spec, params, inputs, dtype=torch.float64)
    e = rel_err(out["energy"], ref["energy"].numpy())
    print(cfg, "energy rel err", e)
    assert e < TOL
    if spec.get("forces", True) and "forces" in ref:
        f = rel_err(out["forces"], ref["forces"].numpy())
        print(cfg, "forces rel err", f)
        assert f < TOL
    return out, ref


def test_cfg1_ethanol_schnet():
    _oracle_vs_cuda("cfg1")


def test_cfg2_aspirin_painn_b32():
    # same generator as the benchmark workload, 32 molecules so that the fp64 oracle finishes in seconds
    _oracle_vs_cuda("cfg2", batch=32)


def test_cfg3_qm9_schnet_padded_b64():
    _oracle_vs_cuda("cfg3", batch=64)


def test_cfg4_box_painn_1000():
    _oracle_vs_cuda("cfg4", n_atoms_total=1000)


@pytest.mark.parametrize("batch", [8, 20])   # 2.4k edges: streaming edge kernels; 6.1k edges: tensor-core edge kernels
def test_unsorted_neighbor_list_matches_sorted(batch):
    """idx_i is not guaranteed sorted (vesin / LAMMPS order): a random permutation of the edge list must give the same
    energy and forces (graph build falls back to a stable grouping)."""
    from schnetpack_b200 import synthetic as S

    spec, inputs = S.make_config("cfg2", batch=batch)
    params = S.init_params(spec, seed=3)
    a = _run_cuda(spec, params, inputs)
    rng = np.random.default_rng(0)
    perm = rng.permutation(inputs["_idx_i"].shape[0])
    shuf = dict(inputs)
    for k in ("_idx_i", "_idx_j", "_offsets"):
        shuf[k] = inputs[k][perm]
    b = _run_cuda(spec, params, shuf)
    assert rel_err(b["energy"], a["energy"]) < 2e-6
    assert rel_err(b["forces"], a["forces"]) < 2e-6


def test_empty_and_ragged_inputs():
    """single atoms (no edges), an isolated atom inside a batch and a system with zero neighbours inside the cutoff."""
    from oracle import spk_oracle as O
    from schnetpack_b200 import synthetic as S

    for kind in ("painn", "schnet"):
        spec = S.model_spec(kind)
        params = S.init_params(spec, seed=5)
        # batch: ethanol + a lone atom + a far-apart pair (no edges)
        a = S.ethanol_batch(1)
        n0 = a["_atomic_numbers"].shape[0]
        inputs = {
            "_atomic_numbers": np.concatenate([a["_atomic_numbers"], [8, 1, 1]]),
            "_positions": np.concatenate([a["_positions"], [[50, 0, 0], [80, 0, 0], [95, 0, 0]]]).astype(np.float32),
            "_idx_i": a["_idx_i"], "_idx_j": a["_idx_j"], "_offsets": a["_offsets"],
            "_idx_m": np.concatenate([a["_idx_m"], [1, 2, 2]]),
            "_n_atoms": np.array([n0, 1, 2]),
            "_cell": np.zeros((3, 3, 3), dtype=np.float32), "_pbc": np.zeros(9, dtype=bool),
        }
        out = _run_cuda(spec, params, inputs)
        ref = O.energy_forces(spec, params, inputs, dtype=torch.float64)
        assert rel_err(out["energy"], ref["energy"].numpy()) < TOL
        assert rel_err(out["forces"], ref["forces"].numpy()) < TOL
        assert np.all(out["forces"][n0:] == 0.0)
        # a batch with no edges at all
        lone = {k: v for k, v in inputs.items()}
        lone["_idx_i"] = np.zeros(0, dtype=np.int64)
        lone["_idx_j"] = np.zeros(0, dtype=np.int64)
        lone["_offsets"] = np.zeros((0, 3), dtype=np.float32)
        out = _run_cuda(spec, params, lone)
        ref = O.energy_forces(spec, params, lone, dtype=torch.float64)
        assert rel_err(out["energy"], ref["energy"].numpy()) < TOL
        assert np.all(out["forces"] == 0.0)


def test_energy_translation_rotation_invariance_full_size():
    """Size-independent property at the FULL benchmark size (cfg2, batch 256): energy invariant under a rigid rotation
    + translation of every molecule, forces co-rotate (equivariance of the PaiNN vector channel)."""
    from schnetpack_b200 import synthetic as S

    spec, inputs = S.make_config("cfg2")
    params = S.init_params(spec, seed=9)
    a = _run_cuda(spec, params, inputs)
    rng = np.random.default_rng(1)
    A = rng.normal(size=(3, 3))
    Q, _ = np.linalg.qr(A)
    if np.linalg.det(Q) < 0:
        Q[:, 0] *= -1
    rot = dict(inputs)
    rot["_positions"] = (inputs["_positions"].astype(np.float64) @ Q.T + np.array([1.5, -2.0, 0.7])).astype(np.float32)
    b = _run_cuda(spec, params, rot)
    assert rel_err(b["energy"], a["energy"]) < 5e-6
    assert rel_err(b["forces"], a["forces"] @ Q.T) < 5e-5   # positions re-rounded to fp32 after rotation
    # Newton's third law: net force on every molecule vanishes
    net = np.add.reduceat(a["forces"], np.arange(0, a["forces"].shape[0], 21), axis=0)
    assert np.abs(net).max() / np.abs(a["forces"]).max() < 1e-5


def test_finite_difference_forces():
    """forces are the derivative of the energy the same kernels produce (central differences in fp32, loose tol)."""
    from schnetpack_b200 import synthetic as S

    spec, inputs = S.make_config("cfg2", batch=2)
    params = S.init_params(spec, seed=2)
    base = _run_cuda(spec, params, inputs)
    h = 1e-2
    for (atom, comp) in ((0, 0), (7, 1), (30, 2)):
        ep = dict(inputs); em = dict(inputs)
        rp = inputs["_positions"].copy(); rm = inputs["_positions"].copy()
        rp[atom, comp] += h; rm[atom, comp] -= h
        ep["_positions"] = rp; em["_positions"] = rm
        fd = -(_run_cuda(spec, params, ep)["energy"].sum() - _run_cuda(spec, params, em)["energy"].sum()) / (2 * h)
        assert abs(fd - base["forces"][atom, comp]) < 2e-2 * max(1.0, abs(base["forces"][atom, comp]))


def test_cuda_graph_replay_matches_eager_and_tracks_new_inputs():
    """GraphedPotential: replayed results equal the eager ones, and a replay with NEW positions / a re-ordered neighbour
    list (same shapes) gives the results of those new inputs (the CSR build is part of the captured graph)."""
    from oracle import spk_oracle as O
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import GraphedPotential, batch_to_device, from_spec

    dev = torch.device("cuda:0")
    spec, a = S.make_config("cfg2", batch=6)
    params = S.init_params(spec, seed=4)
    model = from_spec(spec, params, dev)
    gp = GraphedPotential(model)
    xa = batch_to_device(a, dev)
    out1 = {k: v.clone() for k, v in gp(xa).items()}
    eager = model(batch_to_device(a, dev))
    assert rel_err(out1["energy"].cpu().numpy(), eager["energy"].detach().cpu().numpy()) < 1e-6
    assert rel_err(out1["forces"].cpu().numpy(), eager["forces"].detach().cpu().numpy()) < 1e-6
    # second batch: same shapes, different geometry and a permuted (unsorted) edge list
    _, b = S.make_config("cfg2", batch=6)
    rng = np.random.default_rng(5)
    b = dict(b)
    b["_positions"] = (a["_positions"] + rng.normal(0, 0.02, a["_positions"].shape)).astype(np.float32)
    perm = rng.permutation(a["_idx_i"].shape[0])
    for k in ("_idx_i", "_idx_j", "_offsets"):
        b[k] = a[k][perm]
    out2 = {k: v.clone() for k, v in gp(batch_to_device(b, dev)).items()}
    ref = O.energy_forces(spec, params, b, dtype=torch.float64)
    assert rel_err(out2["energy"].cpu().numpy(), ref["energy"].numpy()) < TOL
    assert rel_err(out2["forces"].cpu().numpy(), ref["forces"].numpy()) < TOL
    assert len(gp._cache) == 1


def test_stress_through_strain_module_matches_reference():
    """Optional part of row a14: ``Strain`` -> ``PairwiseDistances`` -> PaiNN -> ``Atomwise`` -> ``Forces(calc_stress=True)``
    on the CUDA path == the unmodified reference (fixture painn_box_stress, fp64) within 1e-5 relative."""
    import torch

    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params, inputs, _, ref64 = load_case("painn_box_stress")
    dev = torch.device("cuda:0")
    model = from_spec(spec, params, dev)
    out = model(batch_to_device(inputs, dev))
    torch.cuda.synchronize()
    for k in ("energy", "forces", "stress"):
        err = rel_err(out[k].detach().cpu().numpy(), ref64[k])
        assert err < 1e-5, (k, err)
