"""Generate tests/golden/vib_*.npz: Hessians and dipole / polarizability derivatives of the UNMODIFIED reference
(oracle/ref_loader) in fp64, for the vibrational analysis of schnetpack_b200.vibrations.

Each file holds the model (spec_json, param:*), the inputs (in:*), the masses, the reference's analytic Hessian from
``Response("energy", ["forces", "hessian"])`` (ref64:hessian, [sum n^2, 3, 3]) and, for headed models, the autograd
derivatives of the head outputs in the layout of ``derivative_from_molecular`` (ref64:dipole_derivatives [N, 3, 3],
ref64:polarizability_derivatives [N, 3, 3, 3]).  It also holds ASE-style finite differences at the tests' step H, for
nfree = 2 and 4 (fd{nfree}:hessian): the displaced coordinate x + o h is rounded to fp32 as the device does, the
reference's fp64 forces are taken at the fp32 positions, and the derivative at 0 of the polynomial through the realised
steps (fd{nfree}:steps:{m} [3n, nfree]; forces fd{nfree}:forces:{m} [3n, nfree, n, 3]) is formed here by solving the
scaled Vandermonde system, independently of tests/vib_oracle.py.

Cases:
  * vib_ethanol: the trained PaiNN ethanol model (painn_md_ethanol_trained, whose file keeps the weights), both
    molecules relaxed in fp64 (L-BFGS, then Newton steps with the analytic Hessian) to a largest force of ~1e-13
    kcal/mol/A; the inputs are those positions rounded to fp32 (largest force there ~2e-4 kcal/mol/A), and every
    Hessian of the file is taken at the fp32 positions;
  * vib_heads: a PaiNN model with a DipoleMoment and a Polarizability head (the reference's own head initialisation) on
    ethanol, a 1-atom system and a 10-atom system with an isolated atom;
  * vib_box: a periodic cubic cell of 24 atoms whose neighbour list crosses the cell boundary; its finite differences
    rebuild the neighbour list at every displaced geometry, as the device does.

Run from the repository root:  python tests/golden/make_golden_vibrations.py
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import heads_oracle as HO  # noqa: E402
from oracle import ref_loader as rl  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402

H = 0.01                                         # Angstrom: ASE's default step, the step the tests use
MASS = {1: 1.008, 6: 12.011, 7: 14.007, 8: 15.999}


def _load(name):
    z = np.load(os.path.join(HERE, name + ".npz"))
    spec = json.loads(str(z["spec_json"]))
    inputs = {k[3:]: z[k] for k in z.files if k.startswith("in:")}
    params = {k[6:]: z[k] for k in z.files if k.startswith("param:")}
    return spec, params, inputs


def _x(inputs, R=None):
    x = {k: (torch.as_tensor(v).double() if np.asarray(v).dtype.kind == "f" else torch.as_tensor(v))
         for k, v in inputs.items()}
    if R is not None:
        x[S.R] = torch.as_tensor(R, dtype=torch.float64)
    return x


def _response_model(model):
    spk = rl.load()
    resp = spk.atomistic.Response("energy", ["forces", "hessian"])
    return spk.model.NeuralNetworkPotential(model.representation, input_modules=list(model.input_modules),
                                            output_modules=[model.output_modules[0], resp], postprocessors=[],
                                            do_postprocessing=False).double().eval()


def _forces(model, inputs, R):
    out = model(_x(inputs, R))
    return out["energy"].detach().numpy(), out["forces"].detach().numpy()


def _relax(model, resp, inputs):
    from scipy.optimize import minimize

    R = inputs[S.R].astype(np.float64)
    fun = lambda r: (float(_forces(model, inputs, r.reshape(-1, 3))[0].sum()),  # noqa: E731
                     -_forces(model, inputs, r.reshape(-1, 3))[1].reshape(-1))
    R = minimize(fun, R.reshape(-1), jac=True, method="L-BFGS-B", options=dict(gtol=1e-9, maxiter=5000)).x.reshape(-1, 3)
    ptr = np.concatenate([[0], np.cumsum(inputs[S.n_atoms])])
    for _ in range(4):                           # Newton steps per molecule (pseudo-inverse over the 6 rigid modes)
        out = resp(_x(inputs, R))
        f, hb = out["forces"].detach().numpy(), out["hessian"].detach().numpy()
        off = 0
        for m in range(len(ptr) - 1):
            n = ptr[m + 1] - ptr[m]
            h = hb[off:off + n * n].reshape(n, n, 3, 3).transpose(0, 2, 1, 3).reshape(3 * n, 3 * n)
            R[ptr[m]:ptr[m + 1]] += (np.linalg.pinv(h, rcond=1e-8) @ f[ptr[m]:ptr[m + 1]].reshape(-1)).reshape(n, 3)
            off += n * n
    return R


def _derivative_d0(steps, values):
    """p'(0) of the polynomial through (steps, values), from the Vandermonde system in t / H"""
    u = steps / H
    V = np.vander(u, len(u), increasing=True)
    coef = np.linalg.solve(V, values.reshape(len(u), -1))
    return coef[1] / H


def _relisted(inputs, R, cutoff):
    """the periodic cell's inputs with the neighbour list of positions R (pairs enter and leave the cutoff as atoms move)"""
    box_len = float(inputs[S.cell][0, 0, 0])
    ii, jj, ss = S.periodic_cell_list(R, box_len, cutoff)
    return dict(inputs, **{S.idx_i: ii, S.idx_j: jj, S.offsets: (ss * box_len).astype(np.float32)})


def _finite_differences(model, inputs, R32, nfree, props=(), cutoff=None):
    ptr = np.concatenate([[0], np.cumsum(inputs[S.n_atoms])])
    mult = {2: [-1.0, 1.0], 4: [-2.0, -1.0, 1.0, 2.0]}[nfree]
    blocks, out, dprops = [], {}, {p: np.zeros((R32.shape[0], 3 if p == "dipole_moment" else 9, 3)) for p in props}
    for m in range(len(ptr) - 1):
        lo, hi = ptr[m], ptr[m + 1]
        n = hi - lo
        steps, forces = np.zeros((3 * n, nfree)), np.zeros((3 * n, nfree, n, 3))
        vals = {p: np.zeros((3 * n, nfree, 3 if p == "dipole_moment" else 9)) for p in props}
        for d in range(3 * n):
            a, k = lo + d // 3, d % 3
            for s, o in enumerate(mult):
                R = R32.copy()
                R[a, k] = np.float32(R32[a, k]) + np.float32(o * H)
                steps[d, s] = float(R[a, k]) - float(R32[a, k])
                x = _relisted(inputs, R.astype(np.float64), cutoff) if cutoff else inputs
                res = model(_x(x, R.astype(np.float64)))
                forces[d, s] = res["forces"].detach().numpy()[lo:hi]
                for p in props:
                    vals[p][d, s] = res[p].detach().numpy()[m].reshape(-1)
        raw = np.stack([-_derivative_d0(steps[d], forces[d]) for d in range(3 * n)], axis=1)
        h = 0.5 * (raw + raw.T)
        blocks.append(h.reshape(n, 3, n, 3).transpose(0, 2, 1, 3).reshape(n * n, 3, 3))
        out[f"fd{nfree}:steps:{m}"] = steps
        out[f"fd{nfree}:forces:{m}"] = forces
        for p in props:
            for d in range(3 * n):
                dprops[p][lo + d // 3, :, d % 3] = _derivative_d0(steps[d], vals[p][d])
    out[f"fd{nfree}:hessian"] = np.concatenate(blocks)
    for p, v in dprops.items():
        key = "dipole_derivatives" if p == "dipole_moment" else "polarizability_derivatives"
        out[f"fd{nfree}:{key}"] = v if p == "dipole_moment" else v.reshape(-1, 3, 3, 3)
    return out


def _save(name, spec, params, inputs, extra):
    blob = {"spec_json": np.array(json.dumps(spec)), "seed": np.array(0), "H": np.array(H)}
    blob.update({"in:" + k: v for k, v in inputs.items()})
    blob.update({"param:" + k: np.asarray(v) for k, v in params.items()})
    blob.update(extra)
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **blob)
    print(f"{name}: N={inputs[S.Z].shape[0]} -> {os.path.getsize(path) / 1e3:.0f} kB")


def ethanol():
    spec, params, inputs = _load("painn_md_ethanol_trained")
    model = rl.build_from_spec(spec, params, torch.float64)
    resp = _response_model(model)
    R = _relax(model, resp, inputs)
    inputs = dict(inputs, **{S.R: R.astype(np.float32)})
    R32 = inputs[S.R]
    f64 = _forces(model, inputs, R)[1]
    f32pos = _forces(model, inputs, R32.astype(np.float64))[1]
    print(f"ethanol: max |F| at the fp64 minimum {np.abs(f64).max():.2e}, at its fp32 rounding {np.abs(f32pos).max():.2e}"
          " kcal/mol/A")
    out = resp(_x(inputs, R32.astype(np.float64)))
    extra = {"relaxed_positions": R, "masses": np.array([MASS[int(z)] for z in inputs[S.Z]]),
             "ref64:hessian": out["hessian"].detach().numpy(), "ref64:forces": out["forces"].detach().numpy()}
    for nfree in (2, 4):
        extra.update(_finite_differences(model, inputs, R32, nfree))
    _save("vib_ethanol", spec, {}, inputs, extra)          # weights: painn_md_ethanol_trained.npz


def heads():
    spec = HO._painn()
    heads_cfg = [HO.dip(), HO.pol()]
    inputs = HO._isolated_batch()
    params = S.init_params(spec, HO.REP_SEED)
    flat = {k: v.detach().numpy() for k, v in HO.build_reference(spec, params, heads_cfg, torch.float32)
            .state_dict().items()}
    model = HO.build_reference(spec, params, heads_cfg, torch.float64, head_params=flat)
    ref = HO.run_reference(model, inputs, heads_cfg, torch.float64)
    resp = _response_model(model)
    out = resp(_x(inputs))
    N = inputs[S.Z].shape[0]
    extra = {"masses": np.array([MASS[int(z)] for z in inputs[S.Z]]),
             "ref64:hessian": out["hessian"].detach().numpy(),
             "ref64:dipole_moment": ref["dipole_moment"], "ref64:polarizability": ref["polarizability"],
             "ref64:dipole_derivatives": ref["d:dipole_moment"].transpose(1, 0, 2),
             "ref64:polarizability_derivatives": ref["d:polarizability"].reshape(3, 3, N, 3).transpose(2, 0, 1, 3)}
    for nfree in (2, 4):
        extra.update(_finite_differences(model, inputs, inputs[S.R], nfree, props=("dipole_moment", "polarizability")))
    _save("vib_heads", spec, flat, inputs, extra)


def box():
    spec = S.model_spec("painn", n_atom_basis=32, n_interactions=2)
    inputs = S.periodic_box(24, cutoff=spec["cutoff"], seed=3)
    params = S.init_params(spec, 5)
    model = rl.build_from_spec(spec, params, torch.float64)
    resp = _response_model(model)
    out = resp(_x(inputs))
    box_len = float(inputs[S.cell][0, 0, 0])
    print(f"box: L = {box_len:.2f} A, {inputs[S.idx_i].shape[0]} pairs, "
          f"{int((np.abs(inputs[S.offsets]).sum(1) > 0).sum())} across the boundary")
    extra = {"masses": np.array([MASS[int(z)] for z in inputs[S.Z]]),
             "ref64:hessian": out["hessian"].detach().numpy()}
    for nfree in (2, 4):
        extra.update(_finite_differences(model, inputs, inputs[S.R], nfree, cutoff=spec["cutoff"]))
    _save("vib_box", spec, params, inputs, extra)


if __name__ == "__main__":
    torch.set_grad_enabled(True)
    ethanol()
    heads()
    box()
