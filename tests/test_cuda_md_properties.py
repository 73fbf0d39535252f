"""GPU checks of the per-step model properties of DeviceMD (required_properties / property_conversion, reference
md/calculators/base_calculator.py:50-141) and of the device-side recorder (record_every, record_capacity, recorded,
drain, state_dict) with the DipoleMoment / Polarizability heads."""
import numpy as np
import pytest
import torch

from schnetpack_b200 import atomistic as A
from schnetpack_b200 import md as M
from schnetpack_b200 import synthetic as S
from schnetpack_b200.model import NeuralNetworkPotential, batch_to_device, from_spec
from schnetpack_b200.neighbors import CellListNeighborList

import heads_oracle as HO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KEYS = ["dipole_moment", "polarizability"]


@pytest.fixture(scope="module")
def setup():
    spec = S.model_spec("painn", n_atom_basis=32, n_interactions=2)
    base = from_spec(spec, S.init_params(spec, seed=3))
    torch.manual_seed(1)
    heads = [A.DipoleMoment(32, use_vector_representation=True), A.Polarizability(32)]
    model = NeuralNetworkPotential(base.representation, list(base.input_modules), list(base.output_modules) + heads,
                                   postprocessors=[], do_postprocessing=False).to(DEV).eval()
    plain = from_spec(spec, S.init_params(spec, seed=3), DEV)
    data = HO._centered(S.aspirin_batch(3, seed=2))
    masses = torch.as_tensor([HO.MASSES[int(z)] for z in data[S.Z]], dtype=torch.float32)
    rng = np.random.default_rng(0)
    momenta = torch.as_tensor(rng.normal(size=(masses.shape[0], 3)) * np.sqrt(masses.numpy() * M.KB_MD * 300.0)[:, None],
                              dtype=torch.float32)
    return spec, model, plain, data, masses, momenta


def _md(setup, props=KEYS, every=1, capacity=16, use_graph=True, model=None, **kw):
    spec, m, _, data, masses, momenta = setup
    return M.DeviceMD(model if model is not None else m, batch_to_device(data, DEV), masses, time_step=0.5 * M.FS_MD,
                      cutoff=spec["cutoff"], capacity=int(data[S.Z].shape[0]) * 160, momenta=momenta, use_graph=use_graph,
                      required_properties=props, record_every=every, record_capacity=capacity, **kw)


def _evaluate(md, positions):
    x = {k: (v.detach().clone() if v.is_floating_point() else v) for k, v in md.static.items()}
    x[S.R] = positions.clone()
    nl = CellListNeighborList(md.nl._cutoff, capacity=md.nl.capacity, pad=True)     # not the one inside the step
    out = md.model(nl(x))
    return {k: out[k].detach() for k in KEYS}


def test_recorded_series_equals_model_evaluations(setup):
    md = _md(setup, capacity=12, property_conversion={"dipole_moment": 2.0})
    assert md.properties["dipole_moment"].shape == (1, 3, 3) and md.properties["polarizability"].shape == (1, 3, 3, 3)
    pos, props = [], []
    for _ in range(12):
        md.run(1)
        pos.append(md.model_positions.clone())
        props.append({k: md.properties[k].clone() for k in KEYS})
    rec = {k: md.recorded(k) for k in KEYS}
    assert rec["dipole_moment"].shape == (12, 1, 3, 3) and rec["polarizability"].shape == (12, 1, 3, 3, 3)
    for s in range(12):
        ref = _evaluate(md, pos[s])
        for k in KEYS:
            assert torch.equal(rec[k][s], props[s][k].cpu())
            conv = 2.0 if k == "dipole_moment" else 1.0
            r = (ref[k] * conv).cpu()
            assert float((rec[k][s][0] - r).abs().max()) <= 1e-6 * float(r.abs().max()), (k, s)
    with pytest.raises(RuntimeError, match="record_capacity"):
        md.run(1)
    out = md.drain()
    assert torch.equal(out["dipole_moment"], rec["dipole_moment"]) and md.recorded("dipole_moment").shape[0] == 0
    md.run(2)
    assert md.recorded("polarizability").shape[0] == 2


def test_graph_equals_eager(setup):
    a, b = _md(setup, use_graph=True), _md(setup, use_graph=False)
    a.run(6)
    b.run(6)
    for k in KEYS:
        assert torch.equal(a.recorded(k), b.recorded(k)), k
    assert torch.equal(a.positions, b.positions) and torch.equal(a.energy, b.energy)


def test_restart_is_bitwise(setup):
    ref = _md(setup)
    ref.run(8)
    first = _md(setup)
    first.run(4)
    sd = first.state_dict()
    second = _md(setup)
    second.load_state_dict(sd)
    second.run(4)
    for k in KEYS:
        assert torch.equal(second.recorded(k), ref.recorded(k)), k
        assert torch.equal(second.properties[k], ref.properties[k]), k
    assert torch.equal(second.positions, ref.positions) and torch.equal(second.momenta, ref.momenta)


def test_record_every_three(setup):
    every1, every3 = _md(setup), _md(setup, every=3)
    every1.run(10)
    every3.run(10)
    for k in KEYS:
        r3 = every3.recorded(k)
        assert r3.shape[0] == 3
        assert torch.equal(r3, every1.recorded(k)[[2, 5, 8]]), k


def test_ring_polymer_records(setup):
    md = _md(setup, ring_polymer=M.RingPolymer(4, 300.0), capacity=5)
    md.run(5)
    rec = md.recorded("dipole_moment")
    assert rec.shape == (5, 4, 3, 3) and md.recorded("polarizability").shape == (5, 4, 3, 3, 3)
    assert md.properties["dipole_moment"].shape == (4, 3, 3)
    assert torch.isfinite(rec).all() and torch.equal(rec[-1], md.properties["dipole_moment"].cpu())


def test_run_refuses_an_overflowing_call_before_launching(setup):
    md = _md(setup, capacity=2)
    p0, m0 = md.positions.clone(), md.momenta.clone()
    with pytest.raises(RuntimeError, match="record_capacity"):
        md.run(3)
    assert md._graph is None and md.steps_done == 0
    assert torch.equal(md.positions, p0) and torch.equal(md.momenta, m0)
    md3 = _md(setup, capacity=2, every=3)
    md3.run(8)                                             # records at steps 3 and 6 only
    assert md3.recorded("dipole_moment").shape[0] == 2


def test_without_required_properties_the_step_is_unchanged(setup):
    _, model, plain, *_ = setup
    a = _md(setup, props=None, capacity=0, model=plain)
    b = _md(setup, model=model)
    c = _md(setup, props=None, capacity=0, model=model)
    for md in (a, b, c):
        md.run(5)
    for md in (b, c):
        assert torch.equal(md.energy, a.energy) and torch.equal(md.forces, a.forces)
        assert torch.equal(md.positions, a.positions)
    assert c.properties == {} and c.required_properties == []


def test_argument_checks(setup):
    with pytest.raises(ValueError, match="not model outputs"):
        _md(setup, props=["dipole_moment", "nope"])
    with pytest.raises(NotImplementedError, match="number"):
        _md(setup, property_conversion={"dipole_moment": "Debye"})
    with pytest.raises(ValueError, match="needs required_properties"):
        _md(setup, props=None, capacity=4)
