#!/usr/bin/env python
"""Cost of the device vibrational analysis (one JSON line).

    python tools/bench_vibrations.py [--reps 3] [--warmup 1]

For cfg2 (MD17 aspirin x 256: 256 systems of 21 atoms), PaiNN F=128 T=3, nfree = 2, this times with CUDA events:
  * whole ``DeviceVibrations.run`` calls (every chunk plus the finish kernel) -> Hessians per second, with the default
    ``max_replica_atoms`` and with one large enough for a single chunk;
  * one replay of the captured step against one ``GraphedPotential`` replay of the same replica batch and neighbour
    list, so the displacement and assembly kernels and the neighbour list show as the difference;
  * the reference's eager ``Response(hessian)`` (oracle/ref_loader) on the same GPU for a few molecules, per molecule.
The GPU name and its power limit are reported with the numbers.  Nothing is written to the repository.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_relax import gpu_info, time_ms  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.model import GraphedPotential, batch_to_device, from_spec  # noqa: E402
from schnetpack_b200.vibrations import DeviceVibrations  # noqa: E402

MASS = {1: 1.008, 6: 12.011, 7: 14.007, 8: 15.999}


def bench_driver(model, spec, data, dev, reps, warmup, max_replica_atoms):
    resident = batch_to_device(data, dev)
    B, E = int(data[S.n_atoms].shape[0]), int(data[S.idx_i].shape[0])
    masses = torch.tensor([MASS[int(z)] for z in data[S.Z]])
    vib = DeviceVibrations(model, resident, masses, cutoff=spec["cutoff"], capacity=int(E * 1.3),
                           max_replica_atoms=max_replica_atoms)
    for _ in range(warmup):
        vib.run()
    torch.cuda.synchronize()
    run_ms = time_ms(lambda k: [vib.run() for _ in range(k)], reps)
    out = {"max_replica_atoms": max_replica_atoms, "replica_atoms": vib.n_copies * vib.n_atoms,
           "coords_per_chunk": vib.n_cols, "chunks": vib.n_chunks, "run_ms": run_ms,
           "hessians_per_s": B / (run_ms * 1e-3), "peak_pairs": vib.peak_pairs}
    step_ms = time_ms(lambda k: [vib._graph.replay() for _ in range(k)], 5 * reps)
    x = vib.nl(dict(vib.static))
    x = {k: v for k, v in x.items() if k != "_n_pairs"}
    gp = GraphedPotential(model)
    for _ in range(2):
        gp(x)
    torch.cuda.synchronize()
    eval_ms = time_ms(lambda k: [gp(x) for _ in range(k)], 5 * reps)
    out.update(captured_step_ms=step_ms, evaluation_ms=eval_ms, step_minus_evaluation_ms=step_ms - eval_ms)
    del vib, gp, x
    torch.cuda.empty_cache()
    return out


def bench_reference(spec, params, dev, n_mol):
    from oracle import ref_loader as rl

    spk = rl.load()
    base = rl.build_from_spec(spec, params, torch.float32, dev)
    resp = spk.atomistic.Response("energy", ["forces", "hessian"])
    model = spk.model.NeuralNetworkPotential(base.representation, input_modules=list(base.input_modules),
                                             output_modules=[base.output_modules[0], resp], postprocessors=[],
                                             do_postprocessing=False).to(dev).eval()
    data = S.aspirin_batch(n_mol)
    x = {k: torch.as_tensor(v).to(dev) for k, v in data.items()}
    model(dict(x))
    torch.cuda.synchronize()
    ms = time_ms(lambda k: [model(dict(x)) for _ in range(k)], 2)
    return {"molecules": n_mol, "ms_per_molecule": ms / n_mol, "hessians_per_s": n_mol / (ms * 1e-3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vibrations.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.set_grad_enabled(True)
    spec, data = S.make_config("cfg2")
    params = S.init_params(spec, seed=0)
    model = from_spec(spec, params, dev)
    result = {"gpu": gpu_info(dev), "config": "cfg2: aspirin x 256, PaiNN 128 x 3, nfree 2, delta 0.01"}
    result["default_chunks"] = bench_driver(model, spec, data, dev, args.reps, args.warmup, None)
    result["one_chunk"] = bench_driver(model, spec, data, dev, args.reps, args.warmup, 1 << 20)
    result["reference_response"] = bench_reference(spec, params, dev, 4)
    result["speedup_vs_reference"] = (result["one_chunk"]["hessians_per_s"]
                                      / result["reference_response"]["hessians_per_s"])
    print(json.dumps(result))


if __name__ == "__main__":
    main()
