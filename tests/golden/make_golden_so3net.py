"""Regenerate the SO3net fixtures tests/golden/so3net_*.npz from the UNMODIFIED reference (oracle/ref_loader via
tests/so3net_oracle.py):

- ``so3net_tables.npz``: the reference's sparse Clebsch-Gordan tables (SO3TensorProduct buffers) for lmax 0..3 and its
  RealSphericalHarmonics on a fixed set of unit vectors (fp64 evaluation of the fp32 coefficient buffers);
- one file per model case with the same layout as make_golden.py (spec, weight seed, inputs, fp32 and fp64 results),
  plus the multipole representation of the fp64 run.

Run from the repository root:  python tests/golden/make_golden_so3net.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from make_golden import save_case  # noqa: E402

import so3net_oracle as SO  # noqa: E402
from oracle import ref_loader as rl  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402


def tables(spk):
    import schnetpack.nn.so3 as so3

    rng = np.random.default_rng(7)
    u = rng.normal(size=(64, 3))
    u = np.concatenate([u / np.linalg.norm(u, axis=1, keepdims=True), np.eye(3), -np.eye(3)])
    blob = {"dirs": u}
    for L in range(4):
        tp = so3.SO3TensorProduct(L)
        for k in ("idx_in_1", "idx_in_2", "idx_out"):
            blob[f"cg{L}:{k}"] = getattr(tp, k).numpy()
        blob[f"cg{L}:values"] = tp.clebsch_gordan.numpy()
        blob[f"Y{L}"] = so3.RealSphericalHarmonics(L).double()(torch.as_tensor(u)).numpy()
    np.savez_compressed(os.path.join(HERE, "so3net_tables.npz"), **blob)


def case(name, spec, inputs, seed):
    params = S.init_params(spec, seed)
    outs = {}
    for tag, dt in (("32", torch.float32), ("64", torch.float64)):
        model = SO.build_reference(spec, params, dt)
        r = SO.evaluate(model, inputs, dt)
        outs[tag] = {k: v.numpy() for k, v in r.items() if k != "multipole_representation" or tag == "64"}
    save_case(name, spec, seed, inputs, outs["32"], outs["64"])


def main():
    torch.set_grad_enabled(True)
    spk = rl.load()
    tables(spk)
    so3 = lambda **kw: S.model_spec("so3net", **kw)     # noqa: E731
    case("so3net_ethanol_l1", dict(so3(lmax=1), return_vector_representation=True), S.ethanol_batch(1), 31)
    case("so3net_aspirin_b4", so3(n_atom_basis=64, lmax=2), S.aspirin_batch(4, seed=1), 32)
    case("so3net_lmax3", so3(n_atom_basis=32, lmax=3), S.ethanol_batch(2, jitter=0.05, seed=3), 33)
    case("so3net_bessel_shared", so3(n_atom_basis=32, lmax=2, rbf="bessel", shared_interactions=True),
         S.aspirin_batch(2, seed=5), 34)
    case("so3net_box_216", so3(n_atom_basis=32, lmax=2), S.periodic_box(216, seed=4), 35)


if __name__ == "__main__":
    main()
