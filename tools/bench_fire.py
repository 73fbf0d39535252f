#!/usr/bin/env python
"""Cost of the device FIRE relaxation (one JSON line).

    python tools/bench_fire.py [--steps 50] [--warmup 5]

For cfg2 (MD17 aspirin x 256: 256 systems of 21 atoms, fixed cells) and cfg4 (one 8192-atom box, with the unit-cell
filter, so every step also evaluates the virial and rebuilds the neighbour list on the new cell), PaiNN F=128 T=3, this
times with CUDA events:
  * the captured ``DeviceFIRE`` step (optimizer, neighbour list, energy + forces (+ virial), convergence test);
  * the evaluation alone (``GraphedPotential`` replay of the same batch, without the virial);
  * the optimizer kernels alone: force side + step captured ``--steps`` times into one graph and replayed;
  * the captured ``DeviceLBFGS`` step on the same batch (fixed cell).
The GPU name and its power limit are read in the same call and reported with the numbers.  Nothing is written to the
repository.
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
from schnetpack_b200.relax import DeviceFIRE, DeviceLBFGS, FIREState, UnitCellFilter  # noqa: E402


def bench_config(cfg, dev, steps, warmup, with_filter):
    spec, data = S.make_config(cfg)
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    resident = batch_to_device(data, dev)
    N, E, B = int(data[S.Z].shape[0]), int(data[S.idx_i].shape[0]), int(data[S.n_atoms].shape[0])
    out = {"atoms": N, "systems": B, "cell_filter": with_filter}
    filt = UnitCellFilter(scalar_pressure=1e-3) if with_filter else None

    fire = DeviceFIRE(model, resident, cutoff=spec["cutoff"], capacity=int(E * 1.3), maxstep=0.01, cell_filter=filt)
    fire.run(fmax=0.0, steps=warmup)                       # fmax = 0: no system converges, every step does full work
    torch.cuda.synchronize()
    out["step_ms"] = time_ms(lambda k: fire.run(fmax=0.0, steps=k, check_every=k), steps)
    del fire

    gp = GraphedPotential(model)
    for _ in range(warmup):
        gp(resident)
    torch.cuda.synchronize()
    out["evaluation_ms"] = time_ms(lambda k: [gp(resident) for _ in range(k)], steps)
    del gp

    # the optimizer kernels alone, forces (and virial) fixed
    g = torch.Generator(device=dev).manual_seed(0)
    forces = torch.randn(N, 3, device=dev, generator=g)
    virial = torch.randn(B, 3, 3, device=dev, generator=g, dtype=torch.float64) if with_filter else None
    cell = resident[S.cell].reshape(B, 3, 3).double() if with_filter else None
    st = FIREState(resident[S.R].double(), resident[S.idx_m], B, maxstep=0.01, fmax=0.0, cell=cell, cell_filter=filt)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        st.check(forces, virial)
        st.step()
    torch.cuda.current_stream(dev).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(steps):
            st.check(forces, virial)
            st.step()
    graph.replay()
    torch.cuda.synchronize()
    out["optimizer_us"] = 1e3 * time_ms(lambda k: [graph.replay() for _ in range(k)], 5) / steps
    out["optimizer_share_of_step"] = out["optimizer_us"] * 1e-3 / out["step_ms"]
    del st, graph

    lbfgs = DeviceLBFGS(model, resident, cutoff=spec["cutoff"], capacity=int(E * 1.3), maxstep=0.01)
    lbfgs.run(fmax=0.0, steps=warmup)
    torch.cuda.synchronize()
    out["lbfgs_step_ms"] = time_ms(lambda k: lbfgs.run(fmax=0.0, steps=k, check_every=k), steps)
    del lbfgs
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fire.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    result = {"gpu": gpu_info(dev)}
    for cfg, with_filter in (("cfg2", False), ("cfg4", True)):
        result[cfg] = bench_config(cfg, dev, args.steps, args.warmup, with_filter)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
