#!/usr/bin/env python
"""Cost of ring-polymer MD in the captured DeviceMD step (one JSON line).

    python tools/bench_md_rpmd.py [--steps 50] [--warmup 5]

With CUDA events around graph replays this times:
  * an MD17 aspirin batch (B = 16, PaiNN 128x3 as cfg2) at P = 1, 4, 8, 16, 32 beads: the RPMD step with PILE-L (300 K,
    100 fs) against the NVE step of the same P B-system bead batch;
  * one MD17 ethanol molecule (PaiNN 128x3) at P = 32, the launch-bound case;
  * the ring-polymer kernels alone (main step and PILE-L, P = 32 on the aspirin batch): 100 applications captured into
    one graph and replayed.
The GPU name, its power limit and its maximum SM clock are reported with the numbers.  Nothing is written to the repository.
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
from schnetpack_b200.md import DeviceMD, PILELocalThermostat, RingPolymer  # noqa: E402
from schnetpack_b200.model import batch_to_device, from_spec  # noqa: E402


def _strip(data):
    return {k: v for k, v in data.items() if k not in (S.idx_i, S.idx_j, S.offsets)}


def graphed_us(fn, dev):
    """one call of ``fn`` in us: 100 calls captured into one graph, warmed up on a side stream, replayed 5 times"""
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream(dev).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(100):
            fn()
    g.replay()
    torch.cuda.synchronize()
    return 1e3 * time_ms(lambda reps: [g.replay() for _ in range(reps)], 5) / 100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_md_rpmd.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    spec = S.model_spec("painn", n_interactions=3)
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    result = {"model": "painn 128x3", "gpu": gpu_info(dev), "cases": []}
    cases = [("aspirin", 16, P) for P in (1, 4, 8, 16, 32)] + [("ethanol", 1, 32)]
    for mol, B, P in cases:
        data = _strip(S.aspirin_batch(batch=B) if mol == "aspirin" else S.ethanol_batch(batch=1))
        resident = batch_to_device(data, dev)
        N = int(data[S.Z].shape[0])
        masses = torch.ones(N, device=dev)

        def make(th, rp):
            return DeviceMD(model, resident, masses, time_step=1e-4, cutoff=spec["cutoff"], capacity=P * N * 24,
                            thermostat=th, ring_polymer=rp)

        row = {"molecule": mol, "systems": B, "beads": P, "bead_atoms": P * N}
        for name, th in (("nve", None), ("rpmd_pile_l", PILELocalThermostat(300.0, 100.0, seed=1))):
            md = make(th, RingPolymer(P, 300.0))
            if name == "nve":                    # the same P B-system bead batch without the ring polymer
                md.ring_polymer = None
            md.run(args.warmup)
            torch.cuda.synchronize()
            row[name + "_ms_per_step"] = time_ms(md.run, args.steps)
            if name != "nve" and mol == "aspirin" and P == 32:
                rp, x, p = md.ring_polymer, md.positions.clone(), md.momenta.clone()
                row["main_step_us"] = graphed_us(lambda: rp.main_step(x, p, None, 1.0), dev)
                row["pile_l_us"] = graphed_us(lambda: th.apply(p), dev)
            del md
        row["rpmd_over_nve"] = row["rpmd_pile_l_ms_per_step"] / row["nve_ms_per_step"]
        result["cases"].append(row)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
