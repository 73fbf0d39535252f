"""CPU checks of the DipoleMoment / Polarizability heads: the fp64 restatement (tests/heads_oracle.py) against the
reference-generated fixtures, module trees and state_dict keys against the reference, the training path's weight
gradients against the live reference, conversion and the TorchScript refusal."""
import numpy as np
import pytest
import torch

from conftest import load_case
from oracle import ref_loader as rl
from schnetpack_b200 import atomistic as A
from schnetpack_b200 import nn as snn
from schnetpack_b200 import synthetic as S

import heads_oracle as HO

needs_ref = pytest.mark.skipif(not rl.available(), reason="reference modules absent")


@pytest.mark.parametrize("name", list(HO.CASES))
def test_oracle_matches_golden(name):
    spec, params, inputs, _, ref64 = load_case(name)
    heads = HO.CASES[name]["heads"]
    out = HO.evaluate(spec, params, inputs, heads)
    keys = HO.head_keys(heads) + ["d:" + h["key"] for h in heads]
    for k in keys:
        err = float(np.abs(out[k] - ref64[k]).max() / max(np.abs(ref64[k]).max(), 1e-30))
        assert err <= 1e-10, (k, err)
    assert np.all(np.isfinite(ref64["d:" + heads[0]["key"]]))


def test_isolated_case_has_atoms_without_neighbours():
    _, _, inputs, _, ref64 = load_case("heads_painn_isolated")
    n_nbh = np.bincount(inputs[S.idx_i], minlength=inputs[S.Z].shape[0])
    assert (n_nbh == 0).sum() == 2                       # the 1-atom system and the far atom
    assert ref64["dipole_moment"][1] == 0.0              # |q R| at R = 0 with no atomic dipole


def _ref_head(cfg, n_in=32):
    spk = rl.load()
    return HO._ref_head(spk, cfg, n_in)


def _mine(cfg, n_in=32):
    act = torch.nn.functional.silu if cfg["act"] == "silu" else snn.shifted_softplus
    if cfg["kind"] == "dipole":
        return A.DipoleMoment(n_in, n_hidden=cfg["n_hidden"], n_layers=cfg["n_layers"], activation=act,
                              predict_magnitude=cfg["magnitude"], return_charges=cfg["charges"], dipole_key=cfg["key"],
                              charges_key=cfg["charges_key"], correct_charges=cfg["correct"],
                              use_vector_representation=cfg["vector"])
    return A.Polarizability(n_in, n_hidden=cfg["n_hidden"], n_layers=cfg["n_layers"], activation=act,
                            polarizability_key=cfg["key"])


HEAD_VARIANTS = [HO.dip(), HO.dip(n_layers=3, n_hidden=24), HO.dip(vector=False, n_layers=1), HO.pol(),
                 HO.pol(n_layers=1), HO.pol(n_layers=3, act="ssp")]


@needs_ref
@pytest.mark.parametrize("cfg", HEAD_VARIANTS, ids=lambda c: f"{c['kind']}-{c['n_layers']}-{c.get('vector', True)}")
def test_module_tree_and_state_dict_keys_match_reference(cfg):
    ref, mine = _ref_head(cfg), _mine(cfg)
    assert {k: v.shape for k, v in ref.state_dict().items()} == {k: v.shape for k, v in mine.state_dict().items()}
    assert ref.model_outputs == mine.model_outputs
    mine.load_state_dict(ref.state_dict())


@needs_ref
def test_gated_block_standalone_matches_reference():
    spk = rl.load()
    torch.manual_seed(3)
    ref = spk.nn.GatedEquivariantBlock(16, 16, 8, 8, 12, activation=torch.nn.functional.silu,
                                       sactivation=torch.nn.functional.silu).double()
    mine = snn.GatedEquivariantBlock(16, 16, 8, 8, 12, activation=torch.nn.functional.silu,
                                     sactivation=torch.nn.functional.silu).double()
    mine.load_state_dict(ref.state_dict())
    s, v = torch.randn(5, 16, dtype=torch.float64), torch.randn(5, 3, 16, dtype=torch.float64)
    v[2] = 0.0
    for a, b in zip(ref((s, v)), mine((s, v))):
        assert float((a - b).abs().max()) == 0.0
    net_r = spk.nn.build_gated_equivariant_mlp(32, 1, n_layers=3)
    net_m = snn.build_gated_equivariant_mlp(32, 1, n_layers=3)
    assert [k for k in net_r.state_dict()] == [k for k in net_m.state_dict()]


def _pair(kind, heads):
    from schnetpack_b200.model import NeuralNetworkPotential, from_spec

    spec = S.model_spec(kind, n_atom_basis=32, n_interactions=2)
    params = S.init_params(spec, seed=13)
    ref = HO.build_reference(spec, params, heads, torch.float64)
    base = from_spec(spec, params)
    mods = list(base.output_modules) + [_mine(h) for h in heads]
    mine = NeuralNetworkPotential(base.representation, list(base.input_modules), mods, postprocessors=[],
                                  do_postprocessing=False).double()
    mine.load_state_dict(ref.state_dict())
    x = HO._to(HO._centered(HO._mixed_batch(4)), torch.float64)
    x["total_charge"] = torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64)
    return mine, ref, x


@needs_ref
@pytest.mark.parametrize("kind,heads", [("painn", [HO.dip(charges=True), HO.pol()]),
                                        ("painn", [HO.dip(magnitude=True, correct=False, n_layers=3), HO.pol(n_layers=1)]),
                                        ("schnet", [HO.dip(vector=False, n_layers=3, act="ssp")])],
                         ids=["painn-vector", "painn-magnitude", "schnet-scalar"])
def test_training_mode_weight_gradients_match_reference(kind, heads):
    mine, ref, x = _pair(kind, heads)
    mine.train()
    ref.train()
    grads = []
    for model in (mine, ref):
        out = model({k: v.clone() for k, v in x.items()})
        loss = (out["energy"] ** 2).sum() + (out["forces"] ** 2).sum()
        for h in heads:
            loss = loss + (out[h["key"]] ** 2).sum()
        model.zero_grad()
        loss.backward()
        grads.append({k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None})
    assert set(grads[0]) == set(grads[1])
    assert any(k.startswith("output_modules.2.") for k in grads[1])
    for k in grads[1]:
        a, b = grads[0][k], grads[1][k]
        assert float((a - b).abs().max()) <= 1e-10 * max(1.0, float(b.abs().max())), k


@needs_ref
def test_convert_model_swaps_the_heads_and_script_refuses_them():
    from schnetpack_b200.model import convert_model
    from schnetpack_b200.script import to_scriptable

    spec = S.model_spec("painn", n_atom_basis=32, n_interactions=2)
    heads = [HO.dip(n_hidden=16, charges=True, magnitude=True), HO.pol(n_layers=3, act="ssp"),
             HO.dip(vector=False, key="d2", charges_key="c2", n_layers=1)]
    ref = HO.build_reference(spec, S.init_params(spec, 5), heads, torch.float32)
    new = convert_model(ref)
    kinds = [type(m) for m in new.output_modules][2:]
    assert kinds == [A.DipoleMoment, A.Polarizability, A.DipoleMoment]
    ref_sd = ref.state_dict()
    for k, v in new.state_dict().items():
        assert torch.equal(v, ref_sd[k]), k
    assert new.output_modules[2].predict_magnitude and new.output_modules[2].return_charges
    with pytest.raises(NotImplementedError, match="DipoleMoment"):
        to_scriptable(new)


def test_eval_mode_has_no_cpu_fallback():
    head = _mine(HO.pol()).eval()
    x = {"scalar_representation": torch.randn(4, 32), "vector_representation": torch.randn(4, 3, 32),
         "_positions": torch.randn(4, 3), "_idx_m": torch.tensor([0, 0, 1, 1]), "_n_atoms": torch.tensor([2, 2])}
    with pytest.raises(RuntimeError, match="CUDA"):
        head(x)
