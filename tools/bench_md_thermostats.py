#!/usr/bin/env python
"""Cost of the device thermostats in the captured MD step (one JSON line).

    python tools/bench_md_thermostats.py [--config cfg2] [--steps 50] [--warmup 5]

For the workload of ``bench.py`` (default cfg2: MD17 aspirin x 256, PaiNN F=128 T=3) this times, with CUDA events around
graph replays:
  * the ``DeviceMD`` step without a thermostat (NVE) and with ``LangevinThermostat`` / ``NHCThermostat`` (300 K, 100 fs);
  * each thermostat alone: 100 applications (50 steps' worth, two per step) captured into one graph and replayed.
The GPU name and its power limit are reported with the numbers.  Nothing is written to the repository.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.md import DeviceMD, LangevinThermostat, NHCThermostat  # noqa: E402
from schnetpack_b200.model import batch_to_device, from_spec  # noqa: E402


def gpu_info(dev):
    info = {"name": torch.cuda.get_device_name(dev)}
    try:
        out = subprocess.run(["nvidia-smi", f"--id={dev.index}", "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout
        pl, mx = (v.strip() for v in out.strip().split(","))
        info.update(power_limit_w=float(pl), sm_max_mhz=float(mx))
    except Exception:
        info.update(power_limit_w=None, sm_max_mhz=None)
    return info


def time_ms(fn, reps):
    s, e = torch.cuda.Event(True), torch.cuda.Event(True)
    s.record()
    fn(reps)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2", choices=sorted(S.CONFIGS))
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_md_thermostats.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    spec, data = S.make_config(args.config)
    if S.cell not in data or S.Rij in data:
        raise SystemExit(f"{args.config}: DeviceMD needs a batch with cells and no precomputed neighbour vectors")
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    resident = batch_to_device(data, dev)
    N, E = int(data[S.Z].shape[0]), int(data[S.idx_i].shape[0])
    masses = torch.ones(N, device=dev)

    def make(th):
        return DeviceMD(model, resident, masses, time_step=1e-4, cutoff=spec["cutoff"], capacity=int(E * 1.15),
                        thermostat=th)

    md = make(None)
    md.run(args.warmup)
    torch.cuda.synchronize()
    result = {"config": args.config, "atoms": N, "systems": int(data[S.n_atoms].shape[0]),
              "nve_ms_per_step": time_ms(md.run, args.steps), "gpu": gpu_info(dev)}
    del md
    for name, th in (("langevin", LangevinThermostat(300.0, 100.0, seed=1)), ("nhc", NHCThermostat(300.0, 100.0))):
        md = make(th)
        md.run(args.warmup)
        torch.cuda.synchronize()
        step_ms = time_ms(md.run, args.steps)
        # the thermostat alone, 100 applications in one graph (warmed up on a side stream as capture requires)
        p = md.momenta.clone()
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            th.apply(p)
        torch.cuda.current_stream(dev).wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(100):
                th.apply(p)
        g.replay()
        torch.cuda.synchronize()
        th_us = 1e3 * time_ms(lambda reps: [g.replay() for _ in range(reps)], 5) / 50   # one replay = 50 steps
        result[name] = {"ms_per_step": step_ms, "thermostat_us_per_step": th_us,
                        "thermostat_share_of_step": th_us * 1e-3 / step_ms}
        del md, g
    print(json.dumps(result))


if __name__ == "__main__":
    main()
