#!/usr/bin/env python
"""Cost of the device phonons (one JSON line).

    python tools/bench_phonons.py [--reps 3] [--warmup 1] [--mesh 24]

For 16 two-atom CsCl-type crystals (a = 3.0 A, the second atom jittered per crystal), PaiNN F=128 T=3 (cutoff 5 A),
a 4 x 4 x 4 supercell (2 048 supercell atoms in all), nfree = 2, this times with CUDA events:
  * whole ``DevicePhonons.run`` calls (displaced supercells, force constants with 10 sum-rule rounds, image table);
  * ``DeviceVibrations.run`` on the same supercells (every supercell atom displaced), for comparison;
  * on a mesh^3 Monkhorst-Pack mesh: the dynamical matrices (``spk_ph_dynmat``), the batched ``eigvalsh``, the DOS on
    2 000 grid points and the thermodynamics at 100 temperatures, each alone.
The GPU name and its power limit are read in the same call.  Nothing is written to the repository.
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
from schnetpack_b200 import ops  # noqa: E402
from schnetpack_b200 import properties as P  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.model import from_spec  # noqa: E402
from schnetpack_b200.phonons import _KB, _INVCM, DevicePhonons, monkhorst_pack  # noqa: E402
from schnetpack_b200.vibrations import DeviceVibrations  # noqa: E402

B, A, SUPERCELL = 16, 3.0, [4, 4, 4]


def crystals(dev):
    rng = np.random.default_rng(0)
    pos = np.zeros((2 * B, 3), dtype=np.float32)
    pos[1::2] = A / 2 + rng.uniform(-0.15, 0.15, (B, 3))
    return {P.Z: torch.tensor([6, 8] * B, device=dev), P.R: torch.tensor(pos, device=dev),
            P.cell: torch.tensor(np.tile(A * np.eye(3, dtype=np.float32), (B, 1, 1)), device=dev),
            P.pbc: torch.ones(B, 3, dtype=torch.bool, device=dev),
            P.idx_m: torch.arange(B, device=dev).repeat_interleave(2), P.n_atoms: torch.full((B,), 2, device=dev)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--mesh", type=int, default=24)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_phonons.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.set_grad_enabled(True)
    spec = S.model_spec("painn", n_atom_basis=128, n_interactions=3, cutoff=5.0)
    model = from_spec(spec, S.init_params(spec, seed=0), dev)
    masses = torch.tensor([12.011, 15.999] * B)
    result = {"gpu": gpu_info(dev), "config": f"{B} x CsCl-type (2 atoms), PaiNN 128 x 3, supercell 4x4x4, nfree 2, "
                                              f"mesh {args.mesh}^3"}
    ph = DevicePhonons(model, crystals(dev), masses, SUPERCELL, cutoff=5.0, capacity=2 * 64 * B * 64)
    for _ in range(args.warmup):
        ph.run()
    result["phonons"] = {"run_ms": time_ms(lambda k: [ph.run() for _ in range(k)], args.reps),
                         "replica_atoms": ph.static[P.R].shape[0],
                         "chunks": ph.n_chunks, "peak_pairs": ph.peak_pairs}
    sb = ph.supercell_batch
    n_super = sb[P.R].shape[0]
    vib = DeviceVibrations(model, sb, torch.tensor([12.011, 15.999] * (n_super // 2)), cutoff=5.0,
                           capacity=2 * 64 * B * 64)
    vib.run()
    torch.cuda.synchronize()
    result["vibrations_same_supercells"] = {"run_ms": time_ms(lambda k: [vib.run() for _ in range(k)], 1),
                                            "chunks": vib.n_chunks}
    del vib
    torch.cuda.empty_cache()
    result["speedup_vs_vibrations"] = result["vibrations_same_supercells"]["run_ms"] / result["phonons"]["run_ms"]

    q = monkhorst_pack([args.mesh] * 3).to(dev)
    chunks = list(ph._chunks(q))                          # warm-up
    dyn_ms = time_ms(lambda k: [list(ph._chunks(q)) for _ in range(k)], args.reps)
    d = torch.stack([ph._blocks(chunks[0], m) for m in range(B)], 1)
    if not bool(torch.isfinite(torch.view_as_real(d)).all()):
        raise SystemExit("bench_phonons.py: non-finite dynamical matrices")
    torch.linalg.eigvalsh(0.5 * (d + d.transpose(-1, -2).conj()))
    eig_ms = time_ms(lambda k: [torch.linalg.eigvalsh(0.5 * (d + d.transpose(-1, -2).conj())) for _ in range(k)],
                     args.reps) * len(chunks)
    freq = ph.frequencies(q).contiguous()
    grid = torch.linspace(-100.0, float(freq.max()) + 100.0, 2000, dtype=torch.float64, device=dev)
    ops.ph_dos(freq, ph.prim_ptr, grid, 5.0)
    dos_ms = time_ms(lambda k: [ops.ph_dos(freq, ph.prim_ptr, grid, 5.0) for _ in range(k)], args.reps)
    temps = torch.linspace(0.0, 2000.0, 100, dtype=torch.float64)
    counts = (q.shape[0] * 6 * torch.ones(B, dtype=torch.int64)).repeat(100)
    seg_ptr = torch.zeros(counts.shape[0] + 1, dtype=torch.int32)
    seg_ptr[1:] = torch.cumsum(counts, 0)
    n_items = int(counts.sum())
    targs = (freq, ph.prim_ptr, temps.to(dev), seg_ptr.to(dev), n_items, 1.0, _INVCM, _KB)
    ops.ph_thermo(*targs)
    thermo_ms = time_ms(lambda k: [ops.ph_thermo(*targs) for _ in range(k)], args.reps)
    result["mesh"] = {"q_points": q.shape[0], "dynmat_chunks": len(chunks), "dynmat_ms": dyn_ms, "eigh_ms": eig_ms,
                      "dos_ms_2000_points": dos_ms, "thermo_ms_100_temperatures": thermo_ms,
                      "frequencies_total_ms": time_ms(lambda k: [ph.frequencies(q) for _ in range(k)], 1)}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
