#!/usr/bin/env python
"""Cost of an ensemble MD step (one JSON line).

    python tools/bench_ensemble.py [--steps 50] [--warmup 5]

For cfg2 (MD17 aspirin x 256) and cfg4 (one 8192-atom box), PaiNN F=128 T=3, this times with CUDA events:
  * the captured ``DeviceMD`` step with K = 1 (one model), 2 and 4 members (with an ``AbsoluteUncertainty``);
  * one member's evaluation alone (``GraphedPotential`` replay) on the padded fixed-capacity neighbour list the step
    evaluates (same capacity, so the same padding pairs), so that K member evaluations plus one neighbour list can be
    set against the ensemble step; and, for comparison, on the batch's exact list;
  * the statistics kernels alone for K = 4 (moments of the energies, force statistics with per-system terms, the
    uncertainty), captured ``--steps`` times into one graph and replayed.
The claim to check: an ensemble step costs about K member evaluations plus one neighbour list, the statistics a small
share.  The GPU name and its power limit are reported with the numbers.  Nothing is written to the repository.
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

from schnetpack_b200 import ensemble as E  # noqa: E402
from schnetpack_b200 import md as M  # noqa: E402
from schnetpack_b200 import ops  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.model import GraphedPotential, batch_to_device, from_spec  # noqa: E402
from schnetpack_b200.neighbors import CellListNeighborList  # noqa: E402


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


def bench_config(cfg, dev, steps, warmup):
    spec, data = S.make_config(cfg)
    members = [from_spec(spec, S.init_params(spec, seed=k), dev) for k in range(4)]
    resident = batch_to_device(data, dev)
    N, E_, B = int(data[S.Z].shape[0]), int(data[S.idx_i].shape[0]), int(data[S.n_atoms].shape[0])
    out = {"atoms": N, "systems": B}
    masses = torch.full((N,), 12.0)
    for K in (1, 2, 4):
        model = members[0] if K == 1 else members[:K]
        unc = None if K == 1 else E.AbsoluteUncertainty(energy_weight=1.0, force_weight=1.0)
        md = M.DeviceMD(model, resident, masses, time_step=0.5 * M.FS_MD, cutoff=spec["cutoff"],
                        capacity=int(E_ * 1.3), uncertainty_fn=unc)
        md.run(warmup)
        torch.cuda.synchronize()
        out[f"step_ms_k{K}"] = time_ms(lambda k: md.run(k), steps)
        del md
    nl = CellListNeighborList(spec["cutoff"], capacity=int(E_ * 1.3), pad=True)
    padded = nl({k: v for k, v in resident.items() if k not in (S.idx_i, S.idx_j, S.offsets)})
    for name, batch in (("member_evaluation_ms", padded), ("member_evaluation_exact_list_ms", resident)):
        gp = GraphedPotential(members[0])
        for _ in range(warmup):
            gp(batch)
        torch.cuda.synchronize()
        out[name] = time_ms(lambda k: [gp.replay() for _ in range(k)], steps)
        del gp

    K = 4
    g = torch.Generator(device=dev).manual_seed(0)
    energies = torch.randn(K, B, device=dev, generator=g)
    forces = torch.randn(K, N, 3, device=dev, generator=g)
    idx_m = resident[S.idx_m]
    sys_ptr = ops.segment_ptr(idx_m, B)
    mean_e, var_e = torch.empty(B, device=dev), torch.empty(B, device=dev)
    mean_f, var_f = torch.empty(N, 3, device=dev), torch.empty(N, 3, device=dev)
    terms = torch.empty(B, 2, dtype=torch.float64, device=dev)
    ws = E.ensemble_workspace(N, B, dev)
    u = torch.empty(B, device=dev)
    fn = E.AbsoluteUncertainty(energy_weight=1.0, force_weight=1.0)

    def stats():
        E.ensemble_moments(energies, out_mean=mean_e, out_var=var_e)
        E.ensemble_forces(forces, idx_m, sys_ptr, B, out_mean=mean_f, out_var=var_f, terms=True, out_terms=terms,
                          workspace=ws)
        fn.combine(energies, terms, sys_ptr, None, None, out_f32=u)

    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        stats()
    torch.cuda.current_stream(dev).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(steps):
            stats()
    graph.replay()
    torch.cuda.synchronize()
    out["statistics_us_k4"] = 1e3 * time_ms(lambda k: [graph.replay() for _ in range(k)], 5) / steps
    out["statistics_share_of_step_k4"] = out["statistics_us_k4"] * 1e-3 / out["step_ms_k4"]
    for K in (2, 4):
        out[f"step_over_k_evaluations_k{K}"] = out[f"step_ms_k{K}"] / (K * out["member_evaluation_ms"])
    del graph
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ensemble.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    result = {"model": "painn F=128 T=3", "gpu": gpu_info(dev)}
    for cfg in ("cfg2", "cfg4"):
        result[cfg] = bench_config(cfg, dev, args.steps, args.warmup)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
