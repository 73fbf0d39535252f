#!/usr/bin/env python
"""Cost of the device climbing-image NEB (one JSON line).

    python tools/bench_neb.py [--steps 50] [--warmup 5]

Workload: 32 bands of 7 interior images of the cfg2 aspirin molecule (21 atoms; 224 images, 4 704 atoms), PaiNN 128 x 3
from ``synthetic``; the final endpoints are the initial ones displaced by 0.1 Angstrom at random.  Timed with CUDA events:
  * the captured ``DeviceNEB`` step (FIRE step, neighbour list, energy + forces, NEB forces, FIRE force side);
  * the evaluation alone (``GraphedPotential`` replay of the same image batch and neighbour list);
  * the three NEB kernels alone, captured 100 times into one graph and replayed;
  * one band per ``DeviceNEB`` (7 images each), the 32 drivers stepped one after another -- what batching the bands saves.
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
from schnetpack_b200.neb import DeviceNEB, NEBState, interpolate  # noqa: E402
from schnetpack_b200.neighbors import CellListNeighborList  # noqa: E402

BANDS, IMAGES, KERNEL_REPS = 32, 7, 100


def endpoints(data, dev):
    keep = {k: v for k, v in batch_to_device(data, dev).items() if k not in (S.idx_i, S.idx_j, S.offsets)}
    g = torch.Generator(device=dev).manual_seed(0)
    final = dict(keep, **{S.R: keep[S.R] + 0.1 * torch.randn(keep[S.R].shape, device=dev, generator=g)})
    return keep, final


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_neb.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    spec, _ = S.make_config("cfg2")
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    data = S.aspirin_batch(BANDS)
    pairs = int(data[S.idx_i].shape[0]) // BANDS                     # pairs per molecule
    initial, final = endpoints(data, dev)
    cap = int(1.3 * pairs * BANDS)
    out = {"gpu": gpu_info(dev), "bands": BANDS, "images_per_band": IMAGES,
           "atoms": int(initial[S.R].shape[0]) * IMAGES, "steps": args.steps}

    neb = DeviceNEB(model, initial, final, cutoff=spec["cutoff"], capacity=cap, n_images=IMAGES, climb=True,
                    maxstep=0.01)
    neb.run(fmax=0.0, steps=args.warmup)                  # fmax = 0: no band converges, every step does full work
    torch.cuda.synchronize()
    out["step_ms"] = time_ms(lambda k: neb.run(fmax=0.0, steps=k, check_every=k), args.steps)
    forces, energies = neb.forces.clone(), neb.energy.clone()
    del neb

    images = interpolate(initial, final, IMAGES)
    nl = CellListNeighborList(spec["cutoff"], capacity=cap * IMAGES, pad=True)
    resident = nl(images)
    gp = GraphedPotential(model)
    for _ in range(args.warmup):
        gp(resident)
    torch.cuda.synchronize()
    out["evaluation_ms"] = time_ms(lambda k: [gp(resident) for _ in range(k)], args.steps)
    del gp

    # the NEB kernels alone, forces and energies fixed
    sizes = [int(s) for s in initial[S.n_atoms].tolist()]
    ends = torch.zeros(BANDS, 2, dtype=torch.float64, device=dev)
    st = NEBState(images[S.R].double().contiguous(), initial[S.R].double(), final[S.R].double(), ends, sizes, IMAGES,
                  climb=True)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        st.forces(forces, energies)
    torch.cuda.current_stream(dev).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(KERNEL_REPS):
            st.forces(forces, energies)
    graph.replay()
    torch.cuda.synchronize()
    out["neb_kernels_us"] = 1e3 * time_ms(lambda k: [graph.replay() for _ in range(k)], 5) / KERNEL_REPS
    out["neb_kernels_share_of_step"] = out["neb_kernels_us"] * 1e-3 / out["step_ms"]
    del st, graph

    # one band per driver, stepped one after another
    ptr = [0]
    for s in sizes:
        ptr.append(ptr[-1] + s)
    singles = []
    for b in range(BANDS):
        one = lambda x: {S.R: x[S.R][ptr[b]:ptr[b + 1]], S.Z: x[S.Z][ptr[b]:ptr[b + 1]],  # noqa: E731
                         S.n_atoms: x[S.n_atoms][b:b + 1],
                         S.idx_m: torch.zeros(sizes[b], dtype=torch.int64, device=dev)}
        drv = DeviceNEB(model, one(initial), one(final), cutoff=spec["cutoff"], capacity=int(1.3 * pairs) + 64,
                        n_images=IMAGES, climb=True, maxstep=0.01)
        drv.run(fmax=0.0, steps=args.warmup)
        singles.append(drv)
    torch.cuda.synchronize()
    out["one_band_per_driver_ms"] = time_ms(
        lambda k: [d.run(fmax=0.0, steps=k, check_every=k) for d in singles], args.steps)
    out["batching_speedup"] = out["one_band_per_driver_ms"] / out["step_ms"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
