"""ORACLE -- test infrastructure, NOT product code: SO3net for the checks of tests/test_so3net_oracle.py,
tests/test_cuda_so3net.py, tests/golden/make_golden_so3net.py and ``__graft_entry__.smoke()``.

* ``so3net_representation`` / ``energy_forces``: CPU restatement (plain torch, fp32 or fp64) of the reference's
  representation/so3net.py:103-155 with nn/so3.py:101-334 inlined, over a flat weight dictionary with the reference
  ``state_dict`` keys, on the primitives of oracle/spk_oracle.py.  Like the reference, it keeps fp32 constants in an fp64
  run: the Clebsch-Gordan table is the reference's own (tests/golden/so3net_tables.npz) and the harmonic coefficients and
  sqrt(1/2) are rounded to fp32, which pins it to the fp64 golden fixtures at 1e-10.
* ``nve_trajectory``: the NVE loop of oracle/md_oracle.py (same cited lines) with this energy / force engine.
* ``build_reference`` / ``evaluate``: the UNMODIFIED reference SO3net model through oracle/ref_loader.py.
Nothing under ``schnetpack_b200/`` imports this module.
"""
from __future__ import annotations

import math
import os
import re
from typing import Dict, Tuple

import numpy as np
import torch

from oracle import nl_oracle as NL
from oracle import spk_oracle as O

Tensor = torch.Tensor
HERE = os.path.dirname(os.path.abspath(__file__))
SHARED = r"\.(so3convs|mixings1|mixings2|mixings3|gatings)\.\d+\."
_TABLES = None


def so3_tables(lmax: int):
    """The reference's sparse real-basis CG table (values in fp32 as it stores them, idx_in_1, idx_in_2, idx_out)."""
    global _TABLES
    if _TABLES is None:
        _TABLES = dict(np.load(os.path.join(HERE, "golden", "so3net_tables.npz")))
    return tuple(torch.as_tensor(_TABLES[f"cg{lmax}:{k}"]) for k in ("values", "idx_in_1", "idx_in_2", "idx_out"))


def real_sph_harm(u: Tensor, lmax: int) -> Tensor:
    """nn/so3.py:101-149 -- Y_lm(u) = sqrt((2l+1)/(2 pi)) Pi_l^|m|(z) T_m(x, y), T_m = Re (x+iy)^m (m > 0), Im (x+iy)^|m|
    (m < 0), sqrt(1/2) (m = 0); Pi coefficients and sqrt(1/2) rounded to fp32 as the reference's buffers are."""
    x, y, z = u[:, 0], u[:, 1], u[:, 2]
    f = math.factorial

    def r32(v):
        return float(torch.tensor(v, dtype=torch.float32))

    re_, im_ = [torch.ones_like(x)], [torch.zeros_like(x)]
    for _ in range(lmax):
        re_, im_ = re_ + [x * re_[-1] - y * im_[-1]], im_ + [x * im_[-1] + y * re_[-1]]
    cols = []
    for l in range(lmax + 1):
        for m in range(-l, l + 1):
            am = abs(m)
            P = torch.zeros_like(z)
            for k in range((l - am) // 2 + 1):
                c = (math.sqrt(f(l - am) / f(l + am)) * (-1.0) ** k * 2.0 ** (-l) * math.comb(l, k)
                     * math.comb(2 * l - 2 * k, l) * f(l - 2 * k) / f(l - 2 * k - am))
                P = P + r32(c) * z ** (l - 2 * k - am)
            T = re_[am] if m > 0 else (im_[am] if m < 0 else r32(math.sqrt(0.5)))
            cols.append(math.sqrt((2 * l + 1) / (2 * math.pi)) * P * T)
    return torch.stack(cols, dim=1)


def so3net_representation(spec: dict, p: Dict[str, Tensor], Z: Tensor, r_ij: Tensor, idx_i: Tensor,
                          idx_j: Tensor) -> Tuple[Tensor, Tensor]:
    """representation/so3net.py:103-155 with SO3Convolution / SO3TensorProduct / SO3ParametricGatedNonlinearity
    (nn/so3.py:200-334) inlined.  Returns (scalar [N,F], multipoles [N,S,F])."""
    n, Fd, L = Z.shape[0], spec["n_atom_basis"], spec["lmax"]
    S = (L + 1) ** 2
    cg, i1, i2, io = so3_tables(L)
    cg = cg.to(r_ij.dtype)
    lidx = torch.tensor([l for l in range(L + 1) for _ in range(2 * l + 1)])
    d = torch.linalg.norm(r_ij, dim=1, keepdim=True)                     # :122
    Y = real_sph_harm(r_ij / d, L)                                       # :123-125
    phi = O.radial_basis(spec, p, d)                                     # :126  [E,1,R]
    fcut = O.cosine_cutoff(d, spec["cutoff"])[..., None]                 # :127  [E,1,1]

    def scatter_s(v):                                                    # nn/so3.py:217, :303-305
        return torch.zeros((v.shape[0], S, Fd), dtype=v.dtype).index_add(1, io, v)

    x = torch.zeros((n, S, Fd), dtype=r_ij.dtype)
    x[:, 0] = p["representation.embedding.weight"][Z]                    # :130-136
    for t in range(spec["n_interactions"]):
        tt = 0 if spec["shared_interactions"] else t
        c = f"representation.so3convs.{tt}.filternet."
        W = (O.dense(phi, p[c + "weight"], p[c + "bias"]) * fcut).reshape(-1, L + 1, Fd)[:, lidx[i1]]   # so3.py:266-269
        v = W * Y[:, i1, None] * cg[None, :, None] * x[idx_j][:, i2]    # so3.py:294-302
        dx = O.scatter_add(scatter_s(v), idx_i, n)                       # so3.py:303-306
        ddx = O.dense(dx, p[f"representation.mixings1.{tt}.weight"])     # :141
        dx = dx + scatter_s(dx[:, i1] * ddx[:, i2] * cg[None, :, None])  # :142, so3.py:214-218
        dx = O.dense(dx, p[f"representation.mixings2.{tt}.weight"])      # :143
        g = f"representation.gatings.{tt}.scaling."
        h = O.dense(dx[:, 0], p[g + "weight"], p[g + "bias"]).reshape(-1, L + 1, Fd)[:, lidx]            # so3.py:330-332
        dx = dx * torch.sigmoid(h)                                                                        # so3.py:333
        x = x + O.dense(dx, p[f"representation.mixings3.{tt}.weight"])  # :145-146
    return x[:, 0], x


def energy_forces(spec: dict, params: dict, inputs: dict, dtype=torch.float64, stress: bool = False):
    """model/base.py:174-190 for [(Strain), PairwiseDistances] -> SO3net -> [Atomwise, Forces]; forces = -dE/dR
    (atomistic/response.py:59-90).  Returns energy, forces, (stress), scalar / multipole / vector representations."""
    p = O.to_torch(params, dtype)
    x = O.to_torch(inputs, dtype)
    Z, idx_i, idx_j, idx_m = x["_atomic_numbers"], x["_idx_i"], x["_idx_j"], x["_idx_m"]
    n_mol = int(x["_n_atoms"].shape[0]) if "_n_atoms" in x else int(idx_m[-1]) + 1
    if stress:
        x["_positions"] = x["_positions"].clone().requires_grad_(True)
        x["_cell"] = x["_cell"].reshape(-1, 3, 3)
        strain, cell_s, R, off = O.apply_strain(x)
    else:
        R, off = x["_positions"].clone().requires_grad_(True), x["_offsets"]
    q, mp = so3net_representation(spec, p, Z, O.pairwise_distances(R, idx_i, idx_j, off), idx_i, idx_j)
    e = O.atomwise(p, q, idx_m, n_mol)
    out = {"energy": e.detach(), "scalar_representation": q.detach(), "multipole_representation": mp.detach(),
           "vector_representation": torch.roll(mp[:, 1:4], 1, 1).detach()}
    if stress:
        g, gs = torch.autograd.grad([e], [R, strain], grad_outputs=[torch.ones_like(e)])
        vol = torch.sum(cell_s[:, 0] * torch.cross(cell_s[:, 1], cell_s[:, 2], dim=1), dim=1)[:, None, None]
        out["stress"] = (gs / vol).detach()
    else:
        (g,) = torch.autograd.grad([e], [R], grad_outputs=[torch.ones_like(e)])
    out["forces"] = -g.detach()
    return out


def nve_trajectory(spec, params, batch, masses, momenta, time_step, n_steps):
    """oracle/md_oracle.py's velocity-Verlet loop (md/simulator.py:118-144, md/integrators.py:59-110, unit conversions 1)
    for ONE system, exact neighbour list per step (oracle/nl_oracle.py)."""
    cell = np.asarray(batch["_cell"], dtype=np.float64).reshape(3, 3)
    pbc = np.asarray(batch["_pbc"]).reshape(3)
    x = torch.as_tensor(np.asarray(batch["_positions"], dtype=np.float64))
    p = torch.as_tensor(np.asarray(momenta, dtype=np.float64)).clone()
    m = torch.as_tensor(np.asarray(masses, dtype=np.float64)).reshape(-1, 1)

    def calculate(xx):
        ii, jj, _, off = NL.neighbor_list(xx.numpy(), cell, pbc, spec["cutoff"])
        out = energy_forces(spec, params, dict(batch, _positions=xx.numpy(), _idx_i=ii, _idx_j=jj, _offsets=off))
        return out["energy"], out["forces"]

    e, f = calculate(x)
    for _ in range(n_steps):
        p = p + 0.5 * f * time_step
        x = x + time_step * p / m
        e, f = calculate(x)
        p = p + 0.5 * f * time_step
    return x.numpy(), p.numpy(), e.numpy(), f.numpy()


def build_reference(spec: dict, params: dict, dtype=None, device=None):
    """The reference's own NeuralNetworkPotential([PairwiseDistances], SO3net, [Atomwise, Forces]) for an
    ``S.model_spec("so3net", ...)`` dictionary, loaded with a flat weight dictionary (reference ``state_dict`` keys)."""
    from oracle import ref_loader as rl

    spk = rl.load()
    nn_ = spk.nn
    rbf = (nn_.GaussianRBF(n_rbf=spec["n_rbf"], cutoff=spec["cutoff"]) if spec["rbf"] == "gaussian"
           else nn_.BesselRBF(n_rbf=spec["n_rbf"], cutoff=spec["cutoff"]))
    rep = spk.representation.SO3net(spec["n_atom_basis"], spec["n_interactions"], spec["lmax"], rbf,
                                    nn_.CosineCutoff(spec["cutoff"]), shared_interactions=spec["shared_interactions"],
                                    return_vector_representation=bool(spec.get("return_vector_representation")))
    model = spk.model.NeuralNetworkPotential(
        rep, input_modules=[spk.atomistic.PairwiseDistances()],
        output_modules=[spk.atomistic.Atomwise(n_in=spec["n_atom_basis"], output_key="energy"),
                        spk.atomistic.Forces(energy_key="energy", force_key="forces")],
        postprocessors=[], do_postprocessing=False)
    sd = model.state_dict()
    new = {}
    for k in sd:
        kk = k if k in params or not spec["shared_interactions"] else re.sub(SHARED, r".\1.0.", k)
        new[k] = torch.as_tensor(params[kk]).to(sd[k].dtype)
    model.load_state_dict(new)
    if dtype is not None:
        model = model.to(dtype)
    if device is not None:
        model = model.to(device)
    return model.eval()


def evaluate(model, inputs: dict, dtype=None, device=None):
    """Run a reference model on a numpy batch -> dict of detached tensors incl. the representations."""
    x = {}
    for k, v in inputs.items():
        t = torch.as_tensor(v)
        if t.is_floating_point() and dtype is not None:
            t = t.to(dtype)
        x[k] = t.to(device) if device is not None else t
    res = model(x)
    out = {k: v.detach() for k, v in res.items()}
    for k in ("scalar_representation", "multipole_representation", "vector_representation"):
        if k in x:
            out[k] = x[k].detach()
    return out
