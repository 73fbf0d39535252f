#!/usr/bin/env python
"""Cost of constant-pressure MD in the captured MD step (one JSON line).

    python tools/bench_md_barostats.py [--config cfg4] [--steps 50] [--warmup 5] [--rounds 3]

For a periodic workload of ``bench.py`` (default cfg4: 8192-atom water-like box, PaiNN) this times, with CUDA events around
graph replays, one ``DeviceMD`` step in each mode -- NVE, NVT with ``NHCThermostat``, NPT with ``NHCBarostatIsotropic`` and
with ``NHCBarostatAnisotropic`` -- alternating the modes ``--rounds`` times in one process so that clock drift hits all of
them alike, and the per-system virial kernel alone (100 calls on the workload's edge list captured into one graph).  The
GPU name, its power limit and the SM clock are reported with the numbers.  Nothing is written to the repository.
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
from schnetpack_b200 import ops  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.md import DeviceMD, NHCBarostatAnisotropic, NHCBarostatIsotropic, NHCThermostat  # noqa: E402
from schnetpack_b200.model import batch_to_device, from_spec  # noqa: E402

MODES = {
    "nve": lambda: {},
    "nvt_nhc": lambda: {"thermostat": NHCThermostat(300.0, 100.0)},
    "npt_iso": lambda: {"barostat": NHCBarostatIsotropic(1.0, 300.0, 100.0, time_constant_barostat=1000.0)},
    "npt_aniso": lambda: {"barostat": NHCBarostatAnisotropic(1.0, 300.0, 100.0, time_constant_barostat=1000.0)},
}


def sm_clock_mhz(dev):
    try:
        import pynvml

        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(dev.index)
        return float(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM))
    except Exception:
        return None


def virial_us(resident, dev):
    """spk_pairwise_virial alone on the workload's edge list: 100 calls in one graph"""
    idx_i, idx_j = resident[S.idx_i], resident[S.idx_j]
    N, E = int(resident[S.Z].shape[0]), int(idx_i.shape[0])
    n_sys = int(resident[S.n_atoms].shape[0])
    graph = ops.get_graph(idx_i, idx_j, N)
    sys_ptr = ops.segment_ptr(resident[S.idx_m], n_sys)
    gen = torch.Generator(device=dev).manual_seed(0)
    g_rij = torch.randn(E, 3, device=dev, generator=gen)
    r_ij = torch.randn(E, 3, device=dev, generator=gen)
    W = torch.empty(n_sys, 3, 3, dtype=torch.float64, device=dev)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        ops.pairwise_virial(g_rij, r_ij, graph, sys_ptr, W)
    torch.cuda.current_stream(dev).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(100):
            ops.pairwise_virial(g_rij, r_ij, graph, sys_ptr, W)
    g.replay()
    torch.cuda.synchronize()
    return 1e3 * time_ms(lambda reps: [g.replay() for _ in range(reps)], 5) / 100, E


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg4", choices=sorted(S.CONFIGS))
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_md_barostats.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    spec, data = S.make_config(args.config)
    if S.cell not in data or S.Rij in data:
        raise SystemExit(f"{args.config}: DeviceMD needs a batch with cells and no precomputed neighbour vectors")
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    resident = batch_to_device(data, dev)
    N, E = int(data[S.Z].shape[0]), int(data[S.idx_i].shape[0])
    masses = torch.ones(N, device=dev)
    runs = {}
    for name, kw in MODES.items():
        runs[name] = DeviceMD(model, resident, masses, time_step=1e-4, cutoff=spec["cutoff"], capacity=int(E * 1.15),
                              **kw())
        runs[name].run(args.warmup)
    torch.cuda.synchronize()
    times = {name: [] for name in MODES}
    clocks = []
    for _ in range(args.rounds):
        for name, md in runs.items():
            times[name].append(time_ms(md.run, args.steps))
            clocks.append(sm_clock_mhz(dev))
    vir, n_edges = virial_us(resident, dev)
    result = {"config": args.config, "atoms": N, "edges": n_edges, "systems": int(data[S.n_atoms].shape[0]),
              "steps": args.steps, "rounds": args.rounds,
              "ms_per_step": {k: [round(v, 4) for v in t] for k, t in times.items()},
              "virial_us_per_call": round(vir, 2), "sm_mhz_samples": clocks, "gpu": gpu_info(dev)}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
