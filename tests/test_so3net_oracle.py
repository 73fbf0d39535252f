"""CPU checks of SO3net: the package's Clebsch-Gordan tables and harmonics against the reference's, the fp64 oracle
against the golden fixtures, the training path's gradients against the reference, module trees / state_dict keys,
conversion, the shipped config and the TorchScript refusal."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_case
from oracle import ref_loader as rl
from schnetpack_b200 import synthetic as S
from schnetpack_b200.nn import so3

import so3net_oracle as SO

needs_ref = pytest.mark.skipif(not rl.available(), reason="reference modules absent")
CASES = ["so3net_ethanol_l1", "so3net_aspirin_b4", "so3net_lmax3", "so3net_bessel_shared", "so3net_box_216"]
TABLES = np.load(os.path.join(GOLDEN, "so3net_tables.npz"))


@pytest.mark.parametrize("lmax,nnz", [(0, 1), (1, 10), (2, 83), (3, 353)])
def test_cg_table_matches_reference_fixture(lmax, nnz):
    cg, i1, i2, io = so3.sparse_clebsch_gordan(lmax)
    assert cg.shape[0] == nnz and cg.dtype == torch.float32
    for k, v in (("idx_in_1", i1), ("idx_in_2", i2), ("idx_out", io)):
        assert np.array_equal(v.numpy(), TABLES[f"cg{lmax}:{k}"]), k
    assert float(np.abs(cg.numpy() - TABLES[f"cg{lmax}:values"]).max()) <= 1e-7


@needs_ref
@pytest.mark.parametrize("lmax", [0, 1, 2, 3])
def test_cg_table_and_buffers_match_live_reference(lmax):
    spk = rl.load()
    import schnetpack.nn.so3 as R

    ref, mine = R.SO3Convolution(lmax, 8, 5), so3.SO3Convolution(lmax, 8, 5)
    for k in ("idx_in_1", "idx_in_2", "idx_out", "Widx"):
        assert torch.equal(getattr(ref, k), getattr(mine, k)), k
    assert float((ref.clebsch_gordan - mine.clebsch_gordan).abs().max()) <= 1e-7
    rs, ms = R.RealSphericalHarmonics(lmax), so3.RealSphericalHarmonics(lmax)
    assert dict((k, v.shape) for k, v in rs.named_buffers()) == dict((k, v.shape) for k, v in ms.named_buffers())
    assert spk is not None


@pytest.mark.parametrize("lmax", [0, 1, 2, 3])
def test_harmonics_match_reference_fixture(lmax):
    u = torch.as_tensor(TABLES["dirs"])
    mine = so3.RealSphericalHarmonics(lmax).double()(u).numpy()
    assert np.abs(mine - TABLES[f"Y{lmax}"]).max() <= 1e-12
    assert np.abs(SO.real_sph_harm(u, lmax).numpy() - TABLES[f"Y{lmax}"]).max() <= 1e-12


def test_kernel_table_header_is_generated():
    path = os.path.join(os.path.dirname(so3.__file__), "..", "csrc", "so3_tables.cuh")
    assert open(path).read() == so3.cuda_tables_source() + "\n"


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_golden(name):
    spec, params, inputs, _, ref64 = load_case(name)
    out = SO.energy_forces(spec, params, inputs, dtype=torch.float64)
    for k in ("energy", "forces", "scalar_representation", "multipole_representation"):
        err = float(np.abs(out[k].numpy() - ref64[k]).max() / np.abs(ref64[k]).max())
        assert err <= 1e-10, (k, err)
    if "vector_representation" in ref64:
        assert np.abs(out["vector_representation"].numpy() - ref64["vector_representation"]).max() <= 1e-10


def _pair(lmax, shared):
    from schnetpack_b200.model import from_spec

    spec = S.model_spec("so3net", n_atom_basis=16, n_interactions=2, lmax=lmax, shared_interactions=shared)
    params = S.init_params(spec, seed=13)
    mine = from_spec(spec, params).double()
    ref = SO.build_reference(spec, params, torch.float64)
    # the reference rounds its (non-persistent) CG table through a complex64 einsum, 1 ulp off the exact fp32 values:
    # give both models the same constants so that the formulas are compared at fp64 precision
    rr, mr = ref.representation, mine.representation
    for a, b in [(rr.so3product, mr.so3product)] + list(zip(rr.so3convs, mr.so3convs)):
        b.clebsch_gordan.copy_(a.clebsch_gordan)
    data = S.aspirin_batch(2, seed=4)
    x = {k: (torch.as_tensor(v).double() if np.asarray(v).dtype.kind == "f" else torch.as_tensor(v)) for k, v in data.items()}
    return mine, ref, x


@needs_ref
@pytest.mark.parametrize("lmax,shared", [(1, False), (2, True), (3, False)])
def test_training_path_weight_gradients_match_reference(lmax, shared):
    mine, ref, x = _pair(lmax, shared)
    mine.train()
    ref.train()
    grads = []
    for model in (mine, ref):
        out = model({k: v.clone() for k, v in x.items()})
        loss = (out["energy"] ** 2).sum() + (out["forces"] ** 2).sum()      # create_graph: the double backward
        model.zero_grad()
        loss.backward()
        grads.append({k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None})
    assert set(grads[0]) == set(grads[1]) and len(grads[0]) >= 10
    for k in grads[1]:
        a, b = grads[0][k], grads[1][k]
        assert float((a - b).abs().max()) <= 1e-10 * max(1.0, float(b.abs().max())), k


@needs_ref
@pytest.mark.parametrize("lmax,shared", [(1, False), (2, False), (3, False), (2, True)])
def test_state_dict_keys_and_dtypes_match_reference(lmax, shared):
    spk = rl.load()
    from schnetpack_b200 import nn as snn
    from schnetpack_b200.representation import SO3net

    ref = spk.representation.SO3net(16, 3, lmax, spk.nn.GaussianRBF(20, 5.0), spk.nn.CosineCutoff(5.0),
                                     shared_interactions=shared)
    mine = SO3net(16, 3, lmax, snn.GaussianRBF(20, 5.0), snn.CosineCutoff(5.0), shared_interactions=shared)
    a = {k: (tuple(v.shape), v.dtype) for k, v in mine.state_dict().items()}
    b = {k: (tuple(v.shape), v.dtype) for k, v in ref.state_dict().items()}
    assert a == b
    assert b["so3convs.0.Widx"][1] == torch.int64
    mine.load_state_dict(ref.state_dict(), strict=True)
    assert [type(m).__name__ for m in mine.modules()] == [type(m).__name__ for m in ref.modules()]


@needs_ref
def test_convert_model_of_reference_so3net():
    from schnetpack_b200 import representation
    from schnetpack_b200.model import convert_model

    spec = S.model_spec("so3net", n_atom_basis=16, n_interactions=2, lmax=2, shared_interactions=True)
    ref = SO.build_reference(spec, S.init_params(spec, 3))
    new = convert_model(ref)
    rep = new.representation
    assert isinstance(rep, representation.SO3net) and rep.lmax == 2 and rep.so3convs[0] is rep.so3convs[1]
    for k, v in ref.representation.state_dict().items():
        assert torch.equal(rep.state_dict()[k], v), k


def test_config_instantiates():
    from test_configs import CFG, _instantiate, _load

    import schnetpack_b200 as sb

    d = _load(os.path.join(CFG, "representation", "so3net_b200.yaml"), os.path.join(CFG, "representation"))
    rep = _instantiate(d, {"globals.cutoff": 5.0})
    assert isinstance(rep, sb.representation.SO3net) and rep.lmax == 2 and rep.n_atom_basis == 128
    assert len(rep.so3convs) == 3 and rep.radial_basis.n_rbf == 20 and not rep.return_vector_representation
    ref_cfg = os.path.join(rl.REF or "", "configs", "model", "representation", "so3net.yaml")
    if os.path.exists(ref_cfg):                        # the reference tree ships its configs; the vendored copy does not
        import yaml

        ref = yaml.safe_load(open(ref_cfg))
        assert set(ref) == set(yaml.safe_load(open(os.path.join(CFG, "representation", "so3net_b200.yaml"))))


def test_to_scriptable_refuses_so3net():
    from schnetpack_b200.model import from_spec
    from schnetpack_b200.script import to_scriptable

    spec = S.model_spec("so3net", n_atom_basis=16, n_interactions=1, lmax=1)
    with pytest.raises(NotImplementedError, match="SO3net"):
        to_scriptable(from_spec(spec, S.init_params(spec, 0)))


def test_eval_mode_refuses_shapes_outside_the_kernels():
    from schnetpack_b200 import nn as snn
    from schnetpack_b200.representation import SO3net

    mod = SO3net(16, 1, 4, snn.GaussianRBF(20, 5.0), snn.CosineCutoff(5.0)).eval()
    x = {k: torch.as_tensor(v) for k, v in S.ethanol_batch(1).items()}
    x["_Rij"] = (x["_positions"][x["_idx_j"]] - x["_positions"][x["_idx_i"]]).float()
    with pytest.raises(NotImplementedError, match="lmax <= 3"):
        mod(x)
