#!/usr/bin/env python
"""Cost of the streaming spectra in the captured DeviceMD step (one JSON line).

    python tools/bench_spectra_stream.py [--reps 4] [--rounds 2] [--steps 128]

Times with CUDA events, after warm-up:
  * the captured step of (a) cfg2 (aspirin x 256, PaiNN 128 x 3 with dipole and polarizability heads) with an IR and
    Raman stream and (b) cfg4 (8192-atom water box, PaiNN 128 x 3) with a power-spectrum stream, both at L = 4096, each
    against the same step without the stream, alternating for ``--rounds`` rounds (``--steps``, a multiple of the block
    of 64 samples, per timed call); the per-step cost of the stream is reported with the spread of the rounds;
  * the block update alone (the push with the counter on the last sample of a block, minus the push on a sample that
    completes no block), and its achieved fp64 rate against 2 F L flops per sample;
  * the finalisation (spk_spectrum_stream_finalise) and a whole compute_spectrum from the stream;
  * the stream's state bytes against what the stored path needs for 200 000 records (the fp32 records plus the
    normalised fp64 series compute_spectrum builds).
The GPU name and its power limit are reported with the numbers.  Nothing is written to the repository.
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

from bench_relax import gpu_info, time_ms  # noqa: E402
from schnetpack_b200 import _lib, ops  # noqa: E402
from schnetpack_b200 import atomistic as A  # noqa: E402
from schnetpack_b200 import md as M  # noqa: E402
from schnetpack_b200 import spectra as SP  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.model import NeuralNetworkPotential, batch_to_device, from_spec  # noqa: E402

L, BLOCK, STORED_RECORDS = 4096, 64, 200_000
KEYS = ["dipole_moment", "polarizability"]


def make_md(cfg, dev, stream, heads):
    spec, data = S.make_config(cfg)
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    if heads:
        torch.manual_seed(0)
        heads = [A.DipoleMoment(128, use_vector_representation=True), A.Polarizability(128)]
        model = NeuralNetworkPotential(model.representation, list(model.input_modules),
                                       list(model.output_modules) + heads, postprocessors=[],
                                       do_postprocessing=False).to(dev).eval()
    resident = batch_to_device(data, dev)
    N, E = int(data[S.Z].shape[0]), int(data[S.idx_i].shape[0])
    return M.DeviceMD(model, resident, torch.ones(N), time_step=1e-4, cutoff=spec["cutoff"], capacity=int(E * 1.15),
                      required_properties=KEYS if heads else None, stream=stream)


def step_cost(cfg, dev, kinds, heads, reps, rounds, steps):
    mds = {}
    for flag in (False, True):
        mds[flag] = make_md(cfg, dev, SP.SpectrumStream(kinds, resolution=L) if flag else None, heads)
        mds[flag].run(2 * steps)
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for _ in range(rounds):
        for flag in (False, True):
            times[flag].append(time_ms(lambda k: mds[flag].run(k * steps), reps) / steps)
    cost = [(w - wo) * 1e3 for w, wo in zip(times[True], times[False])]
    out = {"without_ms": times[False], "with_ms": times[True], "stream_us_per_step": cost,
           "stream_percent_of_step": [100 * c * 1e-3 / wo for c, wo in zip(cost, times[False])]}
    stream = mds[True].stream
    F = sum(int(g["index"].shape[0]) for g in stream._groups.values())
    out["fields"] = F
    out["state_bytes"] = sum(int(g["state"].numel()) * 8 for g in stream._groups.values())
    # finalisation and a whole spectrum from the stream
    spec = SP.PowerSpectrum(stream, resolution=L) if "power" in kinds else SP.IRSpectrum(stream, resolution=L)
    group = stream._groups["velocities" if "power" in kinds else "dipole_moment"]
    mols = list(range(stream.n_systems))
    spec.compute_spectrum(None)
    torch.cuda.synchronize()
    out["finalise_ms"] = time_ms(lambda k: [stream._autocorrelation(spec, mols) for _ in range(k)], 3)
    out["compute_spectrum_ms"] = time_ms(lambda k: [spec.compute_spectrum(None) for _ in range(k)], 3)
    out["finalised_fields"] = int(group["index"].shape[0])
    return out, mds[True]


def block_update_rate(md, reps):
    """the block update alone on the run's own stream groups: push on sample u = 63 (a block ends) minus u = 62"""
    stream = md.stream
    flops = 0
    counter = torch.zeros(2, dtype=torch.int64, device=md.positions.device)
    saved = {k: v.clone() for k, v in stream._state().items()}

    def push(c, k):
        counter[0] = c
        for _ in range(k):
            stream._push(_Fake(md, counter))

    for g in stream._groups.values():
        flops += 2.0 * int(g["index"].shape[0]) * L * BLOCK
    off = 2 if all(g["derivative"] for g in stream._groups.values()) else 0
    push(BLOCK - 1 + off, 2)
    torch.cuda.synchronize()
    t_block = time_ms(lambda k: push(BLOCK - 1 + off, k), reps)
    t_none = time_ms(lambda k: push(BLOCK - 2 + off, k), reps)
    for k, v in stream._state().items():
        v.copy_(saved[k])
    dt = t_block - t_none
    return {"block_ms": dt, "push_ms": t_none, "fp64_tflops": flops / dt * 1e-9, "flops_per_block": flops}


class _Fake:
    """the DeviceMD attributes the push reads, with a private step counter"""

    def __init__(self, md, counter):
        self.momenta, self.masses, self.properties, self.record_every = md.momenta, md.masses, md.properties, 1
        self._rec_counter = counter


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_spectra_stream.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    result = {"gpu": gpu_info(dev), "lags": L, "block": BLOCK}
    ir, md = step_cost("cfg2", dev, ["ir", "raman"], True, args.reps, args.rounds, args.steps)
    ir["block_update"] = block_update_rate(md, 20)
    B = md.stream.n_systems
    ir["stored_bytes_200k_records"] = STORED_RECORDS * B * (3 + 9) * 4 + (STORED_RECORDS - 2) * B * (3 + 2) * 8
    result["cfg2_ir_raman"] = ir
    del md
    torch.cuda.empty_cache()
    power, md = step_cost("cfg4", dev, ["power"], False, args.reps, args.rounds, args.steps)
    power["block_update"] = block_update_rate(md, 5)
    N = md.positions.shape[0]
    power["stored_bytes_200k_records"] = STORED_RECORDS * N * 3 * 4 + STORED_RECORDS * N * 3 * 8
    result["cfg4_power"] = power
    print(json.dumps(result))


if __name__ == "__main__":
    main()
