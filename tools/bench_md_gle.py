#!/usr/bin/env python
"""Cost of the GLE thermostats in the captured DeviceMD step (one JSON line).

    python tools/bench_md_gle.py [--steps 50] [--warmup 5]

With CUDA events around graph replays this times:
  * the cfg2 workload (MD17 aspirin x 256, PaiNN 128x3) NVT step with ``LangevinThermostat`` (300 K, 100 fs) against
    ``GLEThermostat`` with D = 5, 9 and 16 extended momenta;
  * an aspirin batch (B = 16) at P = 8 beads: the RPMD step with PILE-L against ``RPMDGLEThermostat`` and
    ``PIGLETThermostat`` (D = 5);
  * the GLE kernel alone on the cfg2 batch at each D: 100 applications captured into one graph and replayed.
The matrices are synthetic canonical GLEs (A = S + K, S symmetric positive definite, K antisymmetric, in fs^-1), written to
a temporary directory.  The GPU name, its power limit and its maximum SM clock are reported with the numbers.  Nothing is
written to the repository.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_md_rpmd import graphed_us  # noqa: E402
from bench_md_thermostats import gpu_info, time_ms  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.md import (DeviceMD, GLEThermostat, LangevinThermostat, PIGLETThermostat,  # noqa: E402
                                PILELocalThermostat, RingPolymer, RPMDGLEThermostat)
from schnetpack_b200.model import batch_to_device, from_spec  # noqa: E402


def write_gle(path, D, n_blocks, seed=0):
    """n_blocks canonical GLE drift matrices of size D in a gle4md-format file (no C: C = kB T I)"""
    rng = np.random.default_rng(seed)
    lines = ["# A MATRIX: (femtoseconds^-1)"]
    for k in range(n_blocks):
        q, _ = np.linalg.qr(rng.normal(size=(D, D)))
        s = q @ np.diag(0.1 * rng.uniform(0.2, 3.0, D)) @ q.T
        a = rng.normal(size=(D, D)) * 0.1
        A = 0.5 * (s + s.T) + 0.5 * (a - a.T)
        if n_blocks > 1:
            lines.append(f"# Matrix for normal mode {k}")
        lines += [" ".join(f"{v:.17e}" for v in row) for row in A]
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")
    return path


def step_ms(md, args):
    md.run(args.warmup)
    torch.cuda.synchronize()
    return time_ms(md.run, args.steps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_md_gle.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    tmp = tempfile.TemporaryDirectory()
    result = {"gpu": gpu_info(dev)}

    spec, data = S.make_config("cfg2")
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    resident = batch_to_device(data, dev)
    N, E = int(data[S.Z].shape[0]), int(data[S.idx_i].shape[0])
    masses = torch.ones(N, device=dev)

    def make(th):
        return DeviceMD(model, resident, masses, time_step=1e-4, cutoff=spec["cutoff"], capacity=int(E * 1.15),
                        thermostat=th)

    nvt = {"config": "cfg2", "atoms": N}
    md = make(LangevinThermostat(300.0, 100.0, seed=1))
    nvt["langevin_ms_per_step"] = step_ms(md, args)
    del md
    for D in (5, 9, 16):
        th = GLEThermostat(300.0, write_gle(os.path.join(tmp.name, f"gle{D}.txt"), D, 1), seed=1)
        md = make(th)
        nvt[f"gle_d{D}_ms_per_step"] = step_ms(md, args)
        nvt[f"gle_d{D}_over_langevin"] = nvt[f"gle_d{D}_ms_per_step"] / nvt["langevin_ms_per_step"]
        p = md.momenta.clone()
        nvt[f"gle_d{D}_kernel_us"] = graphed_us(lambda: th.apply(p), dev)
        del md
    result["nvt"] = nvt

    P, B = 8, 16
    adata = {k: v for k, v in S.aspirin_batch(batch=B).items() if k not in (S.idx_i, S.idx_j, S.offsets)}
    aresident = batch_to_device(adata, dev)
    NA = int(adata[S.Z].shape[0])
    amasses = torch.ones(NA, device=dev)
    rpmd = {"molecule": "aspirin", "systems": B, "beads": P, "bead_atoms": P * NA}
    for name, th in (("pile_l", PILELocalThermostat(300.0, 100.0, seed=1)),
                     ("rpmd_gle_d5", RPMDGLEThermostat(300.0, write_gle(os.path.join(tmp.name, "r5.txt"), 5, 1), seed=1)),
                     ("piglet_d5", PIGLETThermostat(300.0, write_gle(os.path.join(tmp.name, "p5.txt"), 5, P), seed=1))):
        md = DeviceMD(model, aresident, amasses, time_step=1e-4, cutoff=spec["cutoff"], capacity=P * NA * 24,
                      thermostat=th, ring_polymer=RingPolymer(P, 300.0))
        rpmd[name + "_ms_per_step"] = step_ms(md, args)
        del md
    for name in ("rpmd_gle_d5", "piglet_d5"):
        rpmd[name + "_over_pile_l"] = rpmd[name + "_ms_per_step"] / rpmd["pile_l_ms_per_step"]
    result["rpmd"] = rpmd
    tmp.cleanup()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
