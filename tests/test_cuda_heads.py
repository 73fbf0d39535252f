"""GPU checks of the DipoleMoment / Polarizability kernels (csrc/equivariant.cu): parity with the reference-generated fp64
fixtures (outputs, charges and the derivatives d(head)/dR), finite differences, shape coverage against the ATen
formula, and at the cfg2 size (aspirin x 256, PaiNN 128 x 3) equivariance, determinism, graph capture and unchanged
energies / forces."""
import numpy as np
import pytest
import torch

from conftest import load_case, rel_err
from oracle import ref_loader as rl
from schnetpack_b200 import atomistic as A
from schnetpack_b200 import functional_torch as T
from schnetpack_b200 import nn as snn
from schnetpack_b200 import synthetic as S
from schnetpack_b200.model import GraphedPotential, NeuralNetworkPotential, batch_to_device, from_spec

import heads_oracle as HO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _head(cfg, n_in):
    act = torch.nn.functional.silu if cfg["act"] == "silu" else snn.shifted_softplus
    if cfg["kind"] == "dipole":
        return A.DipoleMoment(n_in, n_hidden=cfg["n_hidden"], n_layers=cfg["n_layers"], activation=act,
                              predict_magnitude=cfg["magnitude"], return_charges=cfg["charges"], dipole_key=cfg["key"],
                              charges_key=cfg["charges_key"], correct_charges=cfg["correct"],
                              use_vector_representation=cfg["vector"])
    return A.Polarizability(n_in, n_hidden=cfg["n_hidden"], n_layers=cfg["n_layers"], activation=act,
                            polarizability_key=cfg["key"])


def _models(spec, params, heads, full_params=None):
    """(model with [Atomwise, Forces, heads...], model with the same modules and [heads...] only)"""
    base = from_spec(spec, params)
    hs = [_head(h, spec["n_atom_basis"]) for h in heads]
    full = NeuralNetworkPotential(base.representation, list(base.input_modules), list(base.output_modules) + hs,
                                  postprocessors=[], do_postprocessing=False)
    if full_params is not None:
        sd = full.state_dict()
        full.load_state_dict({k: torch.as_tensor(np.asarray(full_params[k])).to(sd[k].dtype) for k in sd})
    full = full.to(DEV).eval()
    only = NeuralNetworkPotential(full.representation, list(full.input_modules), hs, postprocessors=[],
                                  do_postprocessing=False).eval()
    return full, only


def _derivs(only, batch, heads):
    x = batch_to_device(batch, DEV)
    x[S.R].requires_grad_(True)
    out = only(dict(x))
    return {h["key"]: HO._jac(out[h["key"]], x[S.R]).cpu().numpy() for h in heads}


@pytest.mark.parametrize("name", list(HO.CASES))
def test_heads_match_fp64_fixtures(name):
    spec, params, inputs, _, ref64 = load_case(name)
    heads = HO.CASES[name]["heads"]
    full, only = _models(spec, params, heads, params)
    out = full(batch_to_device(inputs, DEV))
    for h in heads:
        got, ref = out[h["key"]].detach().cpu().numpy(), ref64[h["key"]]
        if h["kind"] == "dipole" and not h["magnitude"] and "translated" in name:
            # in fp32, sum_i q'_i R_i cancels at |R| ~ 35 A: the reference's own fp32 result is accurate to the scale of
            # max_m sum_i |q'_i| |R_i|, so the dipole is judged against that scale
            scale = np.zeros(ref.shape[0])
            np.add.at(scale, inputs[S.idx_m], np.abs(ref64[h["charges_key"]][:, 0]) *
                      np.linalg.norm(inputs[S.R].astype(np.float64), axis=1))
            assert np.abs(got - ref).max() / scale.max() <= 1e-5, h["key"]
        else:
            assert rel_err(got, ref) <= 1e-5, (h["key"], rel_err(got, ref))
        if h["kind"] == "dipole" and h["charges"]:
            assert out[h["charges_key"]].shape == (inputs[S.Z].shape[0], 1)
            assert rel_err(out[h["charges_key"]].cpu().numpy(), ref64[h["charges_key"]]) <= 1e-5
    d = _derivs(only, inputs, heads)
    for h in heads:
        assert np.all(np.isfinite(d[h["key"]]))
        assert rel_err(d[h["key"]], ref64["d:" + h["key"]]) <= 1e-5, (h["key"], rel_err(d[h["key"]], ref64["d:" + h["key"]]))


def test_dipole_derivatives_agree_with_finite_differences():
    spec, params, inputs, _, _ = load_case("heads_painn_centered")
    heads = HO.CASES["heads_painn_centered"]["heads"]
    full, only = _models(spec, params, heads, params)
    d = _derivs(only, inputs, heads)["dipole_moment"]
    base = batch_to_device(inputs, DEV)
    R64 = base[S.R].double()
    h = 1e-2
    for atom, comp in ((0, 0), (7, 2), (30, 1), (50, 0)):
        ys = []
        for sgn in (1, -1):
            x = dict(base)
            Rp = R64.clone()
            Rp[atom, comp] += sgn * h
            x[S.R] = Rp.float()
            with torch.no_grad():
                ys.append(only(x)["dipole_moment"].double().sum(0).cpu().numpy())
        fd = (ys[0] - ys[1]) / (2 * h)
        assert np.abs(fd - d[:, atom, comp]).max() <= 2e-3 * max(1.0, np.abs(d).max()), (atom, comp)


@pytest.mark.parametrize("F", [32, 64, 128, 256])
@pytest.mark.parametrize("n_layers,n_hidden", [(1, None), (2, None), (3, None), (2, 48)])
def test_kernels_match_aten_formula(F, n_layers, n_hidden):
    torch.manual_seed(F + n_layers)
    N, B = 300, 7
    idx_m = torch.sort(torch.randint(0, B, (N,)))[0]
    idx_m[idx_m == 3] = 4                                            # system 3 is empty
    n_atoms = torch.bincount(idx_m, minlength=B)
    s = torch.randn(N, F, device=DEV)
    V = torch.randn(N, 3, F, device=DEV)
    V[5] = 0.0                                                       # ||V|| = 0 in every block
    R = torch.randn(N, 3, device=DEV) * 3
    base = {"scalar_representation": s, "vector_representation": V, S.R: R, S.idx_m: idx_m.to(DEV),
            S.n_atoms: n_atoms.to(DEV), "total_charge": torch.randn(B, device=DEV)}
    for cfg in (HO.dip(n_layers=n_layers, n_hidden=n_hidden, charges=True), HO.pol(n_layers=n_layers, n_hidden=n_hidden),
                HO.dip(vector=False, n_layers=n_layers, n_hidden=n_hidden, magnitude=True, act="ssp")):
        head = _head(cfg, F).to(DEV).eval()
        outs = []
        for kind in ("kernel", "aten"):
            x = {k: (v.clone().double() if kind == "aten" and v.is_floating_point() else v.clone())
                 for k, v in base.items()}
            for k in ("scalar_representation", "vector_representation", S.R):
                x[k].requires_grad_(True)
            if kind == "aten":
                y = (T.dipole_moment if cfg["kind"] == "dipole" else T.polarizability)(head.double(), dict(x))
                head.float()
            else:
                y = head(dict(x))
            out = y[cfg["key"]]
            w = torch.randn(out.shape, generator=torch.Generator().manual_seed(1)).to(DEV, out.dtype)
            g = torch.autograd.grad((out * w).sum(), [x["scalar_representation"], x["vector_representation"], x[S.R]],
                                    allow_unused=True)
            res = [out] + [gg if gg is not None else torch.zeros_like(v) for gg, v in
                           zip(g, (x["scalar_representation"], x["vector_representation"], x[S.R]))]
            if cfg.get("charges"):
                res.append(y[cfg["charges_key"]])
            outs.append([r.detach().double().cpu().numpy() for r in res])
            assert torch.all(out.reshape(B, -1)[3] == 0)              # the empty system: exact zeros
        for i, (a, b) in enumerate(zip(*outs)):
            assert rel_err(a, b) <= 1e-5, (cfg["kind"], i, rel_err(a, b))


def test_shape_limits_raise():
    head = _head(HO.pol(n_layers=1), 512).to(DEV).eval()
    x = {"scalar_representation": torch.randn(4, 512, device=DEV), "vector_representation": torch.randn(4, 3, 512, device=DEV),
         S.R: torch.randn(4, 3, device=DEV), S.idx_m: torch.tensor([0, 0, 1, 1], device=DEV),
         S.n_atoms: torch.tensor([2, 2], device=DEV)}
    with pytest.raises(NotImplementedError, match="256"):
        head(x)


@pytest.fixture(scope="module")
def cfg2():
    spec, data = S.make_config("cfg2")
    params = S.init_params(spec, seed=1)
    heads = [HO.dip(charges=True), HO.pol()]
    torch.manual_seed(0)
    full, only = _models(spec, params, heads)
    plain = from_spec(spec, params, DEV)
    return spec, data, full, plain


def test_cfg2_equivariance_determinism_and_unchanged_energy(cfg2):
    spec, data, full, plain = cfg2
    x = batch_to_device(data, DEV)
    a, b = full(dict(x)), full(dict(x))
    for k in a:
        assert torch.equal(a[k], b[k]), k
    p = plain(dict(x))
    assert torch.equal(a["energy"], p["energy"]) and torch.equal(a["forces"], p["forces"])
    Q = torch.linalg.qr(torch.randn(3, 3, generator=torch.Generator().manual_seed(5), dtype=torch.float64))[0]
    xr = dict(x)
    xr[S.R] = (x[S.R].double() @ Q.T.to(DEV)).float()
    r = full(xr)
    Qd = Q.to(DEV)
    mu, mur = a["dipole_moment"].detach().double(), r["dipole_moment"].detach().double()
    al, alr = a["polarizability"].detach().double(), r["polarizability"].detach().double()
    assert rel_err((mu @ Qd.T).cpu(), mur.cpu()) <= 1e-4
    assert rel_err((Qd @ al @ Qd.T).cpu(), alr.cpu()) <= 1e-4


def test_cfg2_graph_replay_equals_eager(cfg2):
    spec, data, full, _ = cfg2
    x = batch_to_device(data, DEV)
    eager = full(dict(x))
    gp = GraphedPotential(full)
    out = gp(batch_to_device(data, DEV))
    out = gp(batch_to_device(data, DEV))
    for k in eager:
        assert torch.equal(out[k], eager[k]), k


@pytest.mark.skipif(not rl.available(), reason="reference modules absent")
def test_convert_model_reproduces_the_reference_on_gpu():
    from schnetpack_b200.model import convert_model

    spec, params, inputs, _, _ = load_case("heads_painn_centered")
    heads = [HO.dip(n_hidden=16, charges=True), HO.pol(n_layers=3, act="ssp")]
    ref = HO.build_reference(spec, params, heads, torch.float32).to(DEV)
    new = convert_model(ref).to(DEV)
    r = ref({k: v.to(DEV) for k, v in HO._to(inputs, torch.float32).items()})
    m = new(batch_to_device(inputs, DEV))
    for k in ("dipole_moment", "partial_charges", "polarizability", "energy", "forces"):
        assert rel_err(m[k].detach().cpu().numpy(), r[k].detach().cpu().numpy()) <= 1e-5, k
