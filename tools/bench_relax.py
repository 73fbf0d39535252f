#!/usr/bin/env python
"""Cost of the device L-BFGS relaxation (one JSON line).

    python tools/bench_relax.py [--steps 50] [--warmup 5]

For cfg2 (MD17 aspirin x 256: 256 systems of 21 atoms, the warp-per-system path) and cfg4 (one 8192-atom box, the
cluster-per-system path), PaiNN F=128 T=3, this times with CUDA events:
  * the captured ``DeviceLBFGS`` step (optimizer, neighbour list, energy + forces, convergence test);
  * the evaluation alone (``GraphedPotential`` replay of the same batch);
  * the optimizer kernels alone with a full 100-entry history: step + convergence test captured ``--steps`` times into
    one graph and replayed;
  * the same two-loop recursion written with torch operations (eager, batched over the equal-size systems).
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
from schnetpack_b200.model import GraphedPotential, batch_to_device, from_spec  # noqa: E402
from schnetpack_b200.relax import DeviceLBFGS, LBFGSState  # noqa: E402

MEMORY = 100


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


def torch_two_loop(S_, Y_, rho, f, h0):
    """the reference's recursion with torch operations, systems batched: S_, Y_ [L, B, d], rho [L, B], f [B, d]"""
    q = -f
    alpha = [None] * S_.shape[0]
    for i in range(S_.shape[0] - 1, -1, -1):
        alpha[i] = rho[i] * (S_[i] * q).sum(-1)
        q = q - alpha[i][:, None] * Y_[i]
    z = h0 * q
    for i in range(S_.shape[0]):
        b = rho[i] * (Y_[i] * z).sum(-1)
        z = z + S_[i] * (alpha[i] - b)[:, None]
    return -z


def bench_config(cfg, dev, steps, warmup):
    spec, data = S.make_config(cfg)
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    resident = batch_to_device(data, dev)
    N, E, B = int(data[S.Z].shape[0]), int(data[S.idx_i].shape[0]), int(data[S.n_atoms].shape[0])
    out = {"atoms": N, "systems": B}

    relax = DeviceLBFGS(model, resident, cutoff=spec["cutoff"], capacity=int(E * 1.3), memory=MEMORY, maxstep=0.01)
    relax.run(fmax=0.0, steps=warmup)                      # fmax = 0: no system converges, every step does full work
    torch.cuda.synchronize()
    out["step_ms"] = time_ms(lambda k: relax.run(fmax=0.0, steps=k, check_every=k), steps)
    del relax

    gp = GraphedPotential(model)
    for _ in range(warmup):
        gp(resident)
    torch.cuda.synchronize()
    out["evaluation_ms"] = time_ms(lambda k: [gp(resident) for _ in range(k)], steps)
    del gp

    # the optimizer alone, history full (MEMORY + 1 steps taken), forces fixed
    g = torch.Generator(device=dev).manual_seed(0)
    forces = torch.randn(N, 3, device=dev, generator=g)
    st = LBFGSState(resident[S.R].double(), resident[S.idx_m], B, memory=MEMORY, maxstep=0.01, fmax=0.0)
    for _ in range(MEMORY + 1):
        st.check(forces)
        st.step(forces)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        st.step(forces)
        st.check(forces)
    torch.cuda.current_stream(dev).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(steps):
            st.step(forces)
            st.check(forces)
    graph.replay()
    torch.cuda.synchronize()
    out["optimizer_us"] = 1e3 * time_ms(lambda k: [graph.replay() for _ in range(k)], 5) / steps
    out["optimizer_share_of_step"] = out["optimizer_us"] * 1e-3 / out["step_ms"]
    # HBM traffic of the two loops: s and y read twice each
    out["two_loop_bytes"] = 4 * MEMORY * 3 * N * 8

    d = 3 * N // B
    S_ = st.s.reshape(MEMORY, B, d)
    Y_ = st.y.reshape(MEMORY, B, d)
    f64 = forces.double().reshape(B, d)
    rho = st.rho
    for _ in range(2):
        torch_two_loop(S_, Y_, rho, f64, 1.0 / 70.0)
    torch.cuda.synchronize()
    out["torch_two_loop_us"] = 1e3 * time_ms(lambda k: [torch_two_loop(S_, Y_, rho, f64, 1.0 / 70.0)
                                                         for _ in range(k)], 5)
    del st, graph
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_relax.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    result = {"memory": MEMORY, "gpu": gpu_info(dev)}
    for cfg in ("cfg2", "cfg4"):
        result[cfg] = bench_config(cfg, dev, args.steps, args.warmup)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
