#!/usr/bin/env python
"""Cost of the structure hooks in the captured DeviceMD step (one JSON line).

    python tools/bench_structure.py [--reps 2] [--rounds 3] [--steps 100] [--sizes 3000 24000]

Times with CUDA events, after warm-up, the captured NVT (Langevin) step of ``synthetic.periodic_box`` (PaiNN 128 x 3,
cutoff 5) without hooks, with ``RadialDistribution(r_max=8, n_bins=400)``, with ``MeanSquaredDisplacement(n_lags=2000,
origin_every=50)`` and with both, each at every_n_steps 1 and 10.  The variants alternate for ``--rounds`` rounds of
``--steps`` steps (a multiple of 10, so every timed call samples alike); the overheads are per step against the step
without hooks, with the spread of the rounds.  The GPU name and its power limit are reported with the numbers.  Nothing
is written to the repository.
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
from schnetpack_b200 import md as M  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.model import batch_to_device, from_spec  # noqa: E402
from schnetpack_b200.structure import MeanSquaredDisplacement, RadialDistribution  # noqa: E402

R_MAX, N_BINS, N_LAGS, ORIGIN_EVERY = 8.0, 400, 2000, 50


def hooks_of(kind, every):
    rdf = lambda: RadialDistribution(R_MAX, N_BINS, every_n_steps=every)                                 # noqa: E731
    msd = lambda: MeanSquaredDisplacement(N_LAGS, every_n_steps=every, origin_every=ORIGIN_EVERY)        # noqa: E731
    return {"none": [], "rdf": [rdf()], "msd": [msd()], "both": [rdf(), msd()]}[kind]


def make_md(n, dev, hooks):
    spec = S.model_spec("painn", n_atom_basis=128, n_interactions=3)
    data = S.periodic_box(n, seed=0, build_list=False)
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    z = data[S.Z]
    masses = torch.where(torch.as_tensor(z) == 8, 16.0, 1.0)
    kB = 0.0025 / 300.0
    return M.DeviceMD(model, batch_to_device(data, dev), masses, time_step=1e-3, cutoff=spec["cutoff"],
                      capacity=int(n * 70), hooks=hooks, thermostat=M.LangevinThermostat(300.0, 20.0, seed=1, kB=kB),
                      initializer=M.MaxwellBoltzmannInit(300.0, seed=2, kB=kB))


def size_cost(n, dev, reps, rounds, steps):
    variants = [("none", 1)] + [(k, e) for e in (1, 10) for k in ("rdf", "msd", "both")]
    mds = {}
    for kind, every in variants:
        mds[(kind, every)] = make_md(n, dev, hooks_of(kind, every))
        mds[(kind, every)].run(steps)
    torch.cuda.synchronize()
    times = {v: [] for v in variants}
    for _ in range(rounds):
        for v in variants:
            times[v].append(time_ms(lambda k: mds[v].run(k * steps), reps) / steps)
    base = times[("none", 1)]
    out = {"atoms": n, "step_ms": base}
    for kind, every in variants[1:]:
        t = times[(kind, every)]
        out[f"{kind}_every{every}"] = {
            "step_ms": t, "overhead_us": [(a - b) * 1e3 for a, b in zip(t, base)],
            "overhead_percent": [100.0 * (a - b) / b for a, b in zip(t, base)]}
    for md in mds.values():
        md.check_neighbor_list()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--sizes", type=int, nargs="+", default=[3000, 24000])
    args = ap.parse_args()
    if args.steps % 10:
        raise SystemExit("--steps must be a multiple of 10")
    if not torch.cuda.is_available():
        raise SystemExit("bench_structure.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    result = {"gpu": gpu_info(dev), "r_max": R_MAX, "n_bins": N_BINS, "n_lags": N_LAGS, "origin_every": ORIGIN_EVERY,
              "model": "painn 128x3", "sizes": []}
    for n in args.sizes:
        result["sizes"].append(size_cost(n, dev, args.reps, args.rounds, args.steps))
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
