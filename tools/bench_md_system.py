#!/usr/bin/env python
"""Cost of the basic simulation hooks in the captured MD step (one JSON line).

    python tools/bench_md_system.py [--configs cfg2,cfg4] [--steps 50] [--warmup 5]

For each configuration this times, with CUDA events around graph replays:
  * the NVE ``DeviceMD`` step against NVE + ``RemoveCOMMotion(1, True)`` + ``WrapPositions(1)``, alternated three times
    in one process (wrapping only where every cell has a volume; molecules in vacuum get the removal alone);
  * each hook alone: 100 applications captured into one graph and replayed;
  * a step with both hooks gated to every_n_steps = 100 (99 of 100 steps skip them on the device).
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

from bench_md_thermostats import gpu_info, time_ms  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.md import DeviceMD, RemoveCOMMotion, WrapPositions  # noqa: E402
from schnetpack_b200.model import batch_to_device, from_spec  # noqa: E402


def graph_of(fn, dev, n=100):
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream(dev).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    g.replay()
    torch.cuda.synchronize()
    return g


def bench(config, steps, warmup, dev):
    spec, data = S.make_config(config)
    if S.Rij in data:
        raise SystemExit(f"{config}: DeviceMD needs a batch without precomputed neighbour vectors")
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    resident = batch_to_device(data, dev)
    N, E = int(data[S.Z].shape[0]), int(data[S.idx_i].shape[0])
    masses = torch.ones(N, device=dev)
    periodic = S.cell in data and bool((torch.linalg.det(torch.as_tensor(data[S.cell]).reshape(-1, 3, 3).double())
                                        != 0).all())

    def hooks(every):
        return [RemoveCOMMotion(every, True)] + ([WrapPositions(every)] if periodic else [])

    def make(h):
        md = DeviceMD(model, resident, masses, time_step=1e-4, cutoff=spec["cutoff"], capacity=int(E * 1.15), hooks=h)
        md.run(warmup)
        torch.cuda.synchronize()
        return md

    runs = {"nve": make(None), "hooks": make(hooks(1)), "gated_100": make(hooks(100))}
    times = {k: [] for k in runs}
    for _ in range(3):
        for k, md in runs.items():
            times[k].append(time_ms(md.run, steps))
    out = {"atoms": N, "systems": int(data[S.n_atoms].shape[0]), "wrap": periodic,
           "ms_per_step": {k: v for k, v in times.items()}}
    md = runs["hooks"]
    for h in md.hooks:
        g = graph_of(lambda: h.apply(md), dev)
        out[f"{type(h).__name__}_us"] = 1e3 * time_ms(lambda reps: [g.replay() for _ in range(reps)], 5) / 100
    nve = min(times["nve"])
    out["hooks_share_of_step"] = (min(times["hooks"]) - nve) / nve
    out["gated_share_of_step"] = (min(times["gated_100"]) - nve) / nve
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="cfg2,cfg4")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_md_system.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    result = {"gpu": gpu_info(dev)}
    for c in args.configs.split(","):
        result[c] = bench(c, args.steps, args.warmup, dev)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
