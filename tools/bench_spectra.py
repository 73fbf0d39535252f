#!/usr/bin/env python
"""Cost of the device vibrational spectra and of the velocity recorder (one JSON line).

    python tools/bench_spectra.py [--reps 5] [--warmup 2] [--steps 200]

Times with CUDA events, after warm-up:
  * IR spectra of 256 molecules from T = 20 000 dipole records at resolution 4096 (one batched compute_spectrum), and
    the autocorrelation kernel alone;
  * the power spectrum of a 216-atom system from T = 20 000 velocity records at resolution 4096, and its
    autocorrelation alone;
  * the reference's numpy FFT route (per-field fft_autocorrelation, then |dt FFT| of the mirrored lags) on the host for
    the same inputs, in fp64;
  * one replay of the captured DeviceMD step for cfg2 (aspirin x 256, PaiNN 128 x 3), without and with
    record_velocities.
The achieved fp64 rate of the autocorrelation counts 2 n L F flops (n points, L lags, F fields; the 4th MMA field of
3-field channels is not counted).  The GPU name and its power limit are reported with the numbers.  Nothing is written
to the repository.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_relax import gpu_info, time_ms  # noqa: E402
from schnetpack_b200 import md as M  # noqa: E402
from schnetpack_b200 import spectra as SP  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.model import batch_to_device, from_spec  # noqa: E402

T_RECORDS, RESOLUTION, DT_FS = 20000, 4096, 0.5


def records(rng, shape, dev):
    """cosines at vibrational frequencies plus noise, fp32 [T, ...]"""
    t = np.arange(T_RECORDS)[:, None] * DT_FS * 1e-15
    n = int(np.prod(shape))
    nu = rng.uniform(500, 3500, size=(1, n)) * 100 * SP._C
    x = np.cos(2 * np.pi * nu * t + rng.uniform(0, 6.3, size=(1, n))) + 0.05 * rng.normal(size=(T_RECORDS, n))
    return torch.as_tensor(x.reshape((T_RECORDS,) + shape).astype(np.float32)).to(dev)


def host_fft_route(x, derivative, channels, dt_fs, resolution):
    """the reference's algorithm in numpy fp64: fields x [T, F] -> spectra of the channels (lists of fields)"""
    x = x.astype(np.float64)
    if derivative:
        x = (x[2:] - x[:-2]) / (2 * dt_fs)
    n = x.shape[0]
    x = (x - x.mean(0)) / x.std(0)
    f = np.fft.rfft(x, n=2 * n, axis=0)
    acf = np.fft.irfft(f * np.conj(f), n=2 * n, axis=0)[: n - 1] / n
    L = min(resolution, n - 1)
    window = SP.cosine_sq_window(L)
    out = []
    for ch in channels:
        a = acf[:L, ch].sum(1) * window
        padded = np.zeros(4 * L)
        padded[:L] = a
        out.append(np.abs(dt_fs * np.fft.fft(np.hstack((padded[::-1], padded)))[: 4 * L]))
    return out


def bench_spectrum(spec, n_fields, n_points, reps, warmup):
    for _ in range(warmup):
        spec.compute_spectrum(None)
    torch.cuda.synchronize()
    total = time_ms(lambda k: [spec.compute_spectrum(None) for _ in range(k)], reps)
    # the autocorrelation kernel alone, on normalised series of the same shape
    B = len(spec._series().sys_ptr) - 1
    per = n_fields // B
    dev = torch.device("cuda", 0)
    z = torch.randn(n_fields, n_points, dtype=torch.float64, device=dev)
    ch = torch.arange(0, n_fields + 1, per, dtype=torch.int64, device=dev)
    w = torch.ones(n_fields, dtype=torch.float64, device=dev)
    L = min(RESOLUTION, n_points - 1)
    for _ in range(warmup):
        SP.autocorrelation(z, ch, w, L)
    torch.cuda.synchronize()
    acf = time_ms(lambda k: [SP.autocorrelation(z, ch, w, L) for _ in range(k)], reps)
    flops = 2.0 * n_points * L * n_fields
    return {"compute_spectrum_ms": total, "autocorrelation_ms": acf, "autocorrelation_fp64_tflops": flops / acf * 1e-9,
            "n_points": n_points, "lags": L, "fields": n_fields}


def bench_record(reps, warmup, steps):
    dev = torch.device("cuda", 0)
    spec, data = S.make_config("cfg2")
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    resident = batch_to_device(data, dev)
    N, E = int(data[S.Z].shape[0]), int(data[S.idx_i].shape[0])
    out = {}
    for flag in (False, True):
        md = M.DeviceMD(model, resident, torch.ones(N), time_step=1e-4, cutoff=spec["cutoff"], capacity=int(E * 1.15),
                        record_capacity=(warmup + reps) * steps + steps if flag else 0, record_velocities=flag)
        md.run(warmup * steps)
        torch.cuda.synchronize()
        out["with_velocities_ms" if flag else "without_ms"] = time_ms(lambda k: md.run(k * steps), reps) / steps
        del md
        torch.cuda.empty_cache()
    out["velocity_record_us_per_step"] = (out["with_velocities_ms"] - out["without_ms"]) * 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--steps", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_spectra.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(0)
    result = {"gpu": gpu_info(dev), "records": T_RECORDS, "resolution": RESOLUTION}

    dip = records(rng, (1, 256, 3), dev)
    ir = SP.IRSpectrum(SP.RecordedSeries(DT_FS, list(range(257)), 1, properties={"dipole_moment": dip}),
                       resolution=RESOLUTION)
    result["ir_256_molecules"] = bench_spectrum(ir, 768, T_RECORDS - 2, args.reps, args.warmup)
    vel = records(rng, (1, 216, 3), dev)
    power = SP.PowerSpectrum(SP.RecordedSeries(DT_FS, [0, 216], 1, velocities=vel), resolution=RESOLUTION)
    result["power_216_atoms"] = bench_spectrum(power, 648, T_RECORDS, args.reps, args.warmup)

    x = dip.reshape(T_RECORDS, -1).cpu().numpy()
    t0 = time.perf_counter()
    host_fft_route(x, True, [list(range(3 * m, 3 * m + 3)) for m in range(256)], DT_FS, RESOLUTION)
    result["ir_256_molecules"]["host_numpy_ms"] = (time.perf_counter() - t0) * 1e3
    x = vel.reshape(T_RECORDS, -1).cpu().numpy()
    t0 = time.perf_counter()
    host_fft_route(x, False, [list(range(648))], DT_FS, RESOLUTION)
    result["power_216_atoms"]["host_numpy_ms"] = (time.perf_counter() - t0) * 1e3
    for k in ("ir_256_molecules", "power_216_atoms"):
        result[k]["speedup_vs_host"] = result[k]["host_numpy_ms"] / result[k]["compute_spectrum_ms"]

    result["record_velocities_cfg2"] = bench_record(args.reps, args.warmup, args.steps)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
