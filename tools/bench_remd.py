#!/usr/bin/env python
"""Cost of temperature replica exchange and of per-system bath temperatures in the captured DeviceMD step (one JSON line).

    python tools/bench_remd.py [--reps 2] [--rounds 3] [--steps 100] [--groups 143]

The batch is K = 8 rungs of ``--groups`` aspirin molecules (21 atoms; 143 groups make 24 024 atoms, the size of
tools/bench_structure.py), open systems, PaiNN 128 x 3 with cutoff 5, Langevin NVT with dt = 0.5 fs and tau = 100 fs.
Times with CUDA events, after warm-up, the captured step of four variants, alternated for ``--rounds`` rounds of
``--steps`` steps (a multiple of 100, so every timed call attempts alike):
  * ``scalar``: one bath temperature (300 K) for all systems, no hook;
  * ``per_system``: the ladder 300 K x 1.1^k as per-system bath temperatures, no hook;
  * ``remd_every10`` / ``remd_every100``: the same with ``ReplicaExchange`` every 10 / 100 steps.
The overheads are per step, of ``per_system`` against ``scalar`` and of the exchange variants against ``per_system``,
with the spread of the rounds.  The GPU name and its power limit are reported with the numbers.  Nothing is written to
the repository.
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
from schnetpack_b200.exchange import ReplicaExchange  # noqa: E402
from schnetpack_b200.model import batch_to_device, from_spec  # noqa: E402

K = 8
MASS = {1: 1.008, 6: 12.011, 8: 15.999}


def make_md(groups, dev, variant):
    spec = S.model_spec("painn", n_atom_basis=128, n_interactions=3)
    data = S.aspirin_batch(groups, seed=0)
    base = {k: v for k, v in batch_to_device(data, dev).items() if k not in (S.idx_i, S.idx_j, S.offsets)}
    batch = M.replicate_batch(base, K, groups)
    masses = torch.tensor([MASS[int(z)] for z in batch[S.Z].tolist()])
    temps = 300.0 if variant == "scalar" else [300.0 * 1.1 ** k for k in range(K) for _ in range(groups)]
    hooks = [ReplicaExchange(K, int(variant[len("remd_every"):]), seed=1)] if variant.startswith("remd") else []
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    return M.DeviceMD(model, batch, masses, time_step=0.5 * M.FS_MD, cutoff=spec["cutoff"],
                      capacity=int(masses.shape[0] * 24), thermostat=M.LangevinThermostat(temps, 100.0, seed=1),
                      initializer=M.MaxwellBoltzmannInit(temps, seed=2), hooks=hooks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--groups", type=int, default=143)
    args = ap.parse_args()
    if args.steps % 100:
        raise SystemExit("--steps must be a multiple of 100")
    if not torch.cuda.is_available():
        raise SystemExit("bench_remd.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    variants = ["scalar", "per_system", "remd_every10", "remd_every100"]
    mds = {}
    for v in variants:
        mds[v] = make_md(args.groups, dev, v)
        mds[v].run(args.steps)
    torch.cuda.synchronize()
    times = {v: [] for v in variants}
    for _ in range(args.rounds):
        for v in variants:
            times[v].append(time_ms(lambda k: mds[v].run(k * args.steps), args.reps) / args.steps)
    out = {"gpu": gpu_info(dev), "model": "painn 128x3", "rungs": K, "groups": args.groups,
           "atoms": int(mds["scalar"].positions.shape[0]), "steps_per_call": args.steps}
    for v, ref in (("scalar", None), ("per_system", "scalar"), ("remd_every10", "per_system"),
                   ("remd_every100", "per_system")):
        t = times[v]
        out[v] = {"step_ms": t}
        if ref is not None:
            b = times[ref]
            out[v]["overhead_us"] = [(x - y) * 1e3 for x, y in zip(t, b)]
            out[v]["overhead_percent"] = [100.0 * (x - y) / y for x, y in zip(t, b)]
    remd = mds["remd_every10"].hooks[0]
    out["remd_every10"]["attempts"] = remd.attempts
    out["remd_every10"]["mean_acceptance"] = float(remd.acceptance().nanmean())
    for md in mds.values():
        md.check_neighbor_list()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
