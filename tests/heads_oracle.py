"""ORACLE -- test infrastructure, NOT product code: the DipoleMoment / Polarizability heads for
tests/test_heads_oracle.py, tests/test_cuda_heads.py and tests/golden/make_golden_heads.py.

* ``CASES`` / ``case_inputs``: the fixture cases -- representation spec, batch and head configurations.
* ``build_reference`` / ``run_reference``: the UNMODIFIED reference model [PairwiseDistances] -> rep -> [Atomwise, Forces,
  heads...] through oracle/ref_loader.py, with the outputs and the derivatives d(head output)/dR.
* ``evaluate``: fp64 restatement of atomistic/atomwise.py:172-213, 267-293 with nn/equivariant.py:57-71 inlined, on the
  representations of oracle/spk_oracle.py / tests/so3net_oracle.py, with the same derivatives.
Nothing under ``schnetpack_b200/`` imports this module.
"""
from __future__ import annotations

from typing import Dict, List

import numpy as np
import torch
import torch.nn.functional as F_

from oracle import spk_oracle as O
from schnetpack_b200 import synthetic as S

import so3net_oracle as SO

Tensor = torch.Tensor
MASSES = {1: 1.008, 6: 12.011, 7: 14.007, 8: 15.999}


def _centered(batch):
    """positions minus each system's centre of mass (the SubtractCenterOfMass transform of the qm9_dipole config)"""
    b = dict(batch)
    R = b[S.R].astype(np.float64)
    m = np.array([MASSES[int(z)] for z in b[S.Z]])
    for s in range(b[S.n_atoms].shape[0]):
        sel = b[S.idx_m] == s
        R[sel] -= (m[sel, None] * R[sel]).sum(0) / m[sel].sum()
    b[S.R] = R.astype(np.float32)
    return b


def _isolated_batch():
    """ethanol, a 1-atom system, and ethanol with one extra atom 12 A away (no neighbours)"""
    eth = S._open_system(S.ETHANOL_Z, S.ETHANOL_R.copy(), 5.0)
    one = S._open_system(np.array([8]), np.zeros((1, 3)), 5.0)
    z = np.concatenate([S.ETHANOL_Z, [7]])
    pos = np.concatenate([S.ETHANOL_R + 0.03, [[12.0, 0.5, -0.3]]])
    far = S._open_system(z, pos, 5.0)
    return S._collate([eth, one, far])


def _mixed_batch(seed):
    a = S.aspirin_batch(2, seed=seed)
    e = S.ethanol_batch(1)
    sys = []
    for b in (a, e):
        for s in range(b[S.n_atoms].shape[0]):
            sel = b[S.idx_m] == s
            off = np.flatnonzero(sel)[0]
            es = np.isin(b[S.idx_i], np.flatnonzero(sel))
            sys.append({S.Z: b[S.Z][sel], S.R: b[S.R][sel], S.idx_i: b[S.idx_i][es] - off, S.idx_j: b[S.idx_j][es] - off,
                        S.offsets: b[S.offsets][es], S.cell: np.zeros((3, 3)), S.pbc: np.zeros(3, dtype=bool)})
    return S._collate(sys)


def dip(**kw):
    d = dict(kind="dipole", n_layers=2, n_hidden=None, act="silu", vector=True, magnitude=False, correct=True,
             charges=False, key="dipole_moment", charges_key="partial_charges")
    d.update(kw)
    return d


def pol(**kw):
    d = dict(kind="polar", n_layers=2, n_hidden=None, act="silu", key="polarizability")
    d.update(kw)
    return d


def _painn():
    return S.model_spec("painn", n_atom_basis=32, n_interactions=2)


CASES = {
    "heads_painn_centered": dict(spec=_painn, batch=lambda: _centered(_mixed_batch(1)), total_charge=[0.0, 1.0, -1.0],
                                 heads=[dip(charges=True), pol()]),
    "heads_painn_translated": dict(spec=_painn, batch=lambda: _translated(_centered(_mixed_batch(1))), total_charge=None,
                                   heads=[dip(charges=True), pol()]),
    "heads_painn_isolated": dict(spec=_painn, batch=_isolated_batch, total_charge=None,
                                 heads=[dip(magnitude=True, correct=False, n_layers=3, act="ssp"),
                                        pol(n_layers=3, act="ssp")]),
    "heads_so3net": dict(spec=lambda: dict(S.model_spec("so3net", n_atom_basis=32, n_interactions=2, lmax=2),
                                           return_vector_representation=True),
                         batch=lambda: _centered(_mixed_batch(2)), total_charge=None,
                         heads=[dip(n_hidden=16, charges=True), pol(n_layers=1)]),
    "heads_schnet": dict(spec=lambda: S.model_spec("schnet", n_atom_basis=32, n_interactions=2),
                         batch=lambda: _centered(_mixed_batch(3)), total_charge=[0.0, 0.0, 1.0],
                         heads=[dip(vector=False, n_layers=3, act="ssp", charges=True),
                                dip(vector=False, n_layers=1, magnitude=True, key="dipole_magnitude",
                                    charges_key="charges_b")]),
}
REP_SEED, HEAD_SEED = 41, 42


def _translated(b):
    b = dict(b)
    b[S.R] = (b[S.R] + np.array([20.0, 20.0, 20.0], dtype=np.float32)).astype(np.float32)
    return b


def case_inputs(name):
    c = CASES[name]
    x = c["batch"]()
    if c["total_charge"] is not None:
        x["total_charge"] = np.asarray(c["total_charge"], dtype=np.float32)
    return c["spec"](), x, c["heads"]


# --------------------------------------------------------------------------------------------------------- reference
def _ref_head(spk, cfg, n_in):
    act = F_.silu if cfg["act"] == "silu" else spk.nn.shifted_softplus
    if cfg["kind"] == "dipole":
        return spk.atomistic.DipoleMoment(n_in, n_hidden=cfg["n_hidden"], n_layers=cfg["n_layers"], activation=act,
                                          predict_magnitude=cfg["magnitude"], return_charges=cfg["charges"],
                                          dipole_key=cfg["key"], charges_key=cfg["charges_key"],
                                          correct_charges=cfg["correct"],
                                          use_vector_representation=cfg["vector"])
    return spk.atomistic.Polarizability(n_in, n_hidden=cfg["n_hidden"], n_layers=cfg["n_layers"], activation=act,
                                        polarizability_key=cfg["key"])


def build_reference(spec, params, heads: List[dict], dtype=torch.float64, head_params=None):
    """NeuralNetworkPotential([PairwiseDistances], rep, [Atomwise, Forces, heads...]) of the reference.  Head weights:
    ``head_params`` (flat reference keys) or the reference's own initialisation under torch.manual_seed(HEAD_SEED)."""
    from oracle import ref_loader as rl

    spk = rl.load()
    base = SO.build_reference(spec, params, torch.float32) if spec["kind"] == "so3net" else \
        rl.build_from_spec(spec, params, torch.float32)
    torch.manual_seed(HEAD_SEED)
    outs = list(base.output_modules) + [_ref_head(spk, h, spec["n_atom_basis"]) for h in heads]
    model = spk.model.NeuralNetworkPotential(base.representation, input_modules=list(base.input_modules),
                                             output_modules=outs, postprocessors=[], do_postprocessing=False)
    if head_params is not None:
        sd = model.state_dict()
        model.load_state_dict({k: torch.as_tensor(np.asarray(head_params[k])).to(sd[k].dtype) for k in sd})
    return model.to(dtype).eval()


def _jac(y: Tensor, R: Tensor) -> Tensor:
    """[n_comp, N, 3]: d(sum over systems of component c)/dR"""
    flat = y.reshape(y.shape[0], -1)
    rows = []
    for c in range(flat.shape[1]):
        (g,) = torch.autograd.grad(flat[:, c].sum(), R, retain_graph=True, allow_unused=True)
        rows.append(torch.zeros_like(R) if g is None else g)
    return torch.stack(rows).detach()


def _to(inputs, dtype):
    return {k: (torch.as_tensor(v).to(dtype) if np.asarray(v).dtype.kind == "f" else torch.as_tensor(v))
            for k, v in inputs.items()}


def run_reference(model, inputs: dict, heads: List[dict], dtype=torch.float64) -> Dict[str, np.ndarray]:
    x = _to(inputs, dtype)
    res = model(dict(x))
    out = {k: v.detach().numpy() for k, v in res.items()}
    # derivatives: a second evaluation without Forces (its backward frees the graph the heads share)
    y = dict(x)
    y[S.R] = y[S.R].clone().requires_grad_(True)
    for m in model.input_modules:
        y = m(y)
    y = model.representation(y)
    for m in list(model.output_modules)[2:]:
        y = m(y)
    for h in heads:
        out["d:" + h["key"]] = _jac(y[h["key"]], y[S.R]).numpy()
    return out


# --------------------------------------------------------------------------------------------------------- restatement
def _act(name):
    return F_.silu if name == "silu" else O.shifted_softplus


def _gated(p, pre, s, v, n_blocks, act):
    """nn/equivariant.py:57-71 for every block of nn/blocks.py:79-156 (scalar activation on all but the last)"""
    for b in range(n_blocks):
        k = f"{pre}outnet.{b}."
        vmix = torch.einsum("ndk,ck->ndc", v, p[k + "mix_vectors.weight"])
        n_out = vmix.shape[-1] // 2
        vV, vW = vmix[..., :n_out], vmix[..., n_out:]
        ctx = torch.cat([s, torch.linalg.vector_norm(vV, dim=1)], dim=-1)       # zero gradient at ||V|| = 0
        x = O.dense(ctx, p[k + "scalar_net.0.weight"], p[k + "scalar_net.0.bias"], _act(act))
        x = O.dense(x, p[k + "scalar_net.1.weight"], p[k + "scalar_net.1.bias"])
        s, x = x[:, :n_out], x[:, n_out:]
        v = x[:, None, :] * vW
        if b < n_blocks - 1:
            s = _act(act)(s)
    return s, v


def _head(p, pre, cfg, q, mu, R, x, n_sys):
    idx_m = x[S.idx_m]
    if cfg["kind"] == "dipole":
        if cfg["vector"]:
            charges, v = _gated(p, pre, q, mu, cfg["n_layers"], cfg["act"])
            atomic = v[..., 0]
        else:
            h = q
            for layer in range(cfg["n_layers"]):
                k = f"{pre}outnet.{layer}."
                h = O.dense(h, p[k + "weight"], p[k + "bias"], _act(cfg["act"]) if layer < cfg["n_layers"] - 1 else None)
            charges, atomic = h, None
        if cfg["correct"]:                                                       # atomwise.py:187-197
            ssum = O.scatter_add(charges, idx_m, n_sys)
            tq = x["total_charge"][:, None] if "total_charge" in x else torch.zeros_like(ssum)
            charges = charges + ((tq - ssum) / x[S.n_atoms].to(ssum.dtype)[:, None])[idx_m]
        y = R * charges
        if atomic is not None:
            y = y + atomic
        y = O.scatter_add(y, idx_m, n_sys)
        if cfg["magnitude"]:
            y = torch.linalg.vector_norm(y, dim=1)
        return y, charges
    s, v = _gated(p, pre, q, mu, cfg["n_layers"], cfg["act"])                 # atomwise.py:273-290
    alpha = s[:, 0, None, None] * torch.eye(3, dtype=R.dtype)
    mur = v[:, :, 0, None] * R[:, None, :]
    return O.scatter_add(alpha + mur + mur.transpose(1, 2), idx_m, n_sys), None


def evaluate(spec, params, inputs: dict, heads: List[dict], dtype=torch.float64) -> Dict[str, np.ndarray]:
    p = O.to_torch(params, dtype)
    x = _to(inputs, dtype)
    n_sys = int(x[S.n_atoms].shape[0])
    R = x[S.R].clone().requires_grad_(True)
    r_ij = O.pairwise_distances(R, x[S.idx_i], x[S.idx_j], x[S.offsets])
    args = (spec, p, x[S.Z], r_ij, x[S.idx_i], x[S.idx_j])
    mu = None
    if spec["kind"] == "painn":
        q, mu = O.painn_representation(*args)
    elif spec["kind"] == "so3net":
        q, mp = SO.so3net_representation(*args)
        mu = torch.roll(mp[:, 1:4], 1, 1)
    else:
        q = O.schnet_representation(*args)
    out = {}
    for i, cfg in enumerate(heads):
        y, charges = _head(p, f"output_modules.{2 + i}.", cfg, q, mu, R, x, n_sys)
        out[cfg["key"]] = y.detach().numpy()
        if cfg["kind"] == "dipole" and cfg["charges"]:
            out[cfg["charges_key"]] = charges.detach().numpy()
        out["d:" + cfg["key"]] = _jac(y, R).numpy()
    return out


def head_keys(heads: List[dict]) -> List[str]:
    keys = []
    for h in heads:
        keys.append(h["key"])
        if h["kind"] == "dipole" and h["charges"]:
            keys.append(h["charges_key"])
    return keys

