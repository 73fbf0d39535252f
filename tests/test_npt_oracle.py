"""CPU: the fp64 barostat restatement tests/npt_oracle.py against the reference's own barostats (tests/golden/
md_barostats.npz, made by tests/golden/make_golden_md_barostats.py), and the oracle's virial formula against the reference
stress of tests/golden/painn_box_stress.npz."""
import json

import numpy as np
import pytest
import torch

import npt_oracle as NPO
from conftest import GOLDEN, rel_err

CASES = {"iso_o3": dict(anisotropic=False, massive=False, integration_order=3),
         "iso_massive_o7": dict(anisotropic=False, massive=True, integration_order=7),
         "aniso_o7": dict(anisotropic=True, massive=False, integration_order=7),
         "aniso_massive_o3": dict(anisotropic=True, massive=True, integration_order=3, chain_length=3, multi_step=2)}


def _golden():
    return dict(np.load(f"{GOLDEN}/md_barostats.npz"))


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_matches_the_reference_barostats(name):
    g = _golden()
    b, x, p, cells = NPO.golden_case(g, name, **CASES[name])
    assert rel_err(x.numpy(), g[name + ":positions"]) < 1e-12
    assert rel_err(p.numpy(), g[name + ":momenta"]) < 1e-12
    assert rel_err(cells.numpy(), g[name + ":cells"]) < 1e-12
    for k, v in b.state().items():
        assert rel_err(v.numpy().reshape(g[name + ":" + k].shape), g[name + ":" + k]) < 1e-12, k
    assert np.abs(g[name + ":cells"] - g["cells"]).max() > 1e-3 * np.abs(g["cells"]).max()      # the cell moved


def test_sinh_div_keeps_the_reference_quirks():
    x = torch.tensor([-3.0, -1e-3, 0.0, 5e-5, 2e-4, 1.0], dtype=torch.float64)
    y = NPO.sinh_div(x)
    # x < eps takes the series, including every negative x; its odd powers past x^2 (x^3 / 120, ...) stand where
    # x^4 / 120, ... are meant
    e = 1.0 + x ** 2 / 6.0 + x ** 3 / 120.0 + x ** 5 / 5040.0 + x ** 7 / 362880.0
    assert torch.allclose(y[:4], e[:4], rtol=1e-14, atol=0)
    assert torch.allclose(y[4:], torch.sinh(x[4:]) / x[4:], rtol=1e-15, atol=0)


def test_virial_over_volume_is_the_reference_stress():
    z = np.load(f"{GOLDEN}/painn_box_stress.npz")
    spec = json.loads(str(z["spec_json"]))
    from schnetpack_b200 import synthetic as S

    params = S.init_params(spec, int(z["seed"]))
    batch = {k[3:]: z[k] for k in z.files if k.startswith("in:")}
    cell = batch["_cell"].reshape(-1, 3, 3)
    _, stress = NPO.stress_from_virial(spec, params, batch, cell)
    assert rel_err(stress.numpy(), z["ref64:stress"]) < 1e-11
