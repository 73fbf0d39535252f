#!/usr/bin/env python
"""Cost of ring-polymer NPT in the captured DeviceMD step (one JSON line).

    python tools/bench_md_rpmd_npt.py [--steps 20] [--warmup 3] [--repeats 3]

With CUDA events around graph replays this times a batch of two periodic water-density boxes of 1536 atoms each (PaiNN
128x3 as cfg4) at P = 8 and P = 32 beads: NVT-RPMD with PILE-L (300 K, 100 fs) against NPT-RPMD with PILE-L and the PILE
barostat (1 bar, 300 K, 500 fs), alternated ``--repeats`` times in one process.  The NPT step adds the per-bead-system
virial to every force evaluation and the barostat kernels.  The barostat kernels are also timed alone at P = 32: 100
applications of each captured into one graph and replayed.  The GPU name, its power limit and its maximum SM clock are
reported with the numbers.  Nothing is written to the repository.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_md_rpmd import graphed_us  # noqa: E402
from bench_md_thermostats import gpu_info, time_ms  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.md import DeviceMD, PILEBarostat, PILELocalThermostat, RingPolymer  # noqa: E402
from schnetpack_b200.model import batch_to_device, from_spec  # noqa: E402

BOX_ATOMS, N_BOXES = 1536, 2


def boxes():
    parts = [S.periodic_box(BOX_ATOMS, seed=s, build_list=False) for s in range(N_BOXES)]
    n = [len(p[S.Z]) for p in parts]
    return {S.R: np.concatenate([p[S.R] for p in parts]), S.Z: np.concatenate([p[S.Z] for p in parts]),
            "_n_atoms": np.array(n, dtype=np.int64), "_idx_m": np.repeat(np.arange(len(parts)), n).astype(np.int64),
            "_cell": np.concatenate([np.asarray(p["_cell"], dtype=np.float32).reshape(1, 3, 3) for p in parts]),
            "_pbc": np.concatenate([np.asarray(p["_pbc"]).reshape(3) for p in parts])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_md_rpmd_npt.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    spec = S.model_spec("painn", n_interactions=3)
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    data = boxes()
    resident = batch_to_device(data, dev)
    N = int(data[S.Z].shape[0])
    masses = torch.where(torch.as_tensor(data[S.Z]) == 8, 16.0, 1.0).to(dev)
    result = {"model": "painn 128x3", "systems": N_BOXES, "atoms_per_system": BOX_ATOMS, "gpu": gpu_info(dev),
              "cases": []}
    for P in (8, 32):
        mds = {}
        for name in ("nvt", "npt"):
            baro = PILEBarostat(1.0, 300.0, 500.0, seed=2) if name == "npt" else None
            mds[name] = DeviceMD(model, resident, masses, time_step=5e-4, cutoff=spec["cutoff"], capacity=P * N * 64,
                                 thermostat=PILELocalThermostat(300.0, 100.0, seed=1), barostat=baro,
                                 ring_polymer=RingPolymer(P, 300.0))
            mds[name].run(args.warmup)
        torch.cuda.synchronize()
        row = {"beads": P, "bead_atoms": P * N, "nvt_ms_per_step": [], "npt_ms_per_step": []}
        for _ in range(args.repeats):
            for name in ("nvt", "npt"):
                row[name + "_ms_per_step"].append(time_ms(mds[name].run, args.steps))
        row["npt_over_nvt"] = [b / a for a, b in zip(row["nvt_ms_per_step"], row["npt_ms_per_step"])]
        if P == 32:
            md = mds["npt"]
            b = md.barostat
            x, p, cell = md.positions.clone(), md.momenta.clone(), md.cell.clone()
            mcell = md.model_cell.clone()
            row["barostat_thermostat_us"] = graphed_us(b.apply_thermostat, dev)
            row["barostat_half_step_us"] = graphed_us(
                lambda: b.half_step(p, md.forces, md.f_conv, cell, md.virial, md._virial_scale()), dev)
            b.cell_momenta.zero_()                     # the timed main steps then leave the cell as it is
            row["barostat_main_step_us"] = graphed_us(lambda: b.main_step(x, p, None, cell, mcell, 1.0), dev)
            row["rpmd_main_step_us"] = graphed_us(lambda: md.ring_polymer.main_step(x, p, None, 1.0), dev)
        result["cases"].append(row)
        del mds
    print(json.dumps(result))


if __name__ == "__main__":
    main()
