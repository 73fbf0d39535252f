"""Cost of the Ewald sum on one GPU: the reciprocal forward and reverse kernels alone (spk_ewald_fwd / spk_ewald_bwd, CUDA
events) with their complex-term rate N K / time, at the cfg4 box (8192 atoms) and at a batch of 64 boxes of 128 atoms,
each with alpha and k_max chosen for about 1e-5 truncation error at rc = 5 A (alpha rc^2 = 11.5, k_max = ceil(k_c L /
2 pi) with k_c^2 = 4 alpha 11.5); and the graphed energy + forces step of cfg4 (PaiNN 128 x 3) with charges, with and
without EnergyEwald on the same model (variants alternated in one session, every shape warmed up first).

    python tools/bench_ewald.py [--reps 20]

Prints one JSON object.  The GPU name, its power limit and SM clocks are read in the same run.  Nothing is written to the
repository.
"""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_so3net import gpu_info, time_ms  # noqa: E402

from schnetpack_b200 import atomistic as A  # noqa: E402
from schnetpack_b200 import ops  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.model import GraphedPotential, NeuralNetworkPotential, batch_to_device, from_spec  # noqa: E402

RC = 5.0
ALPHA = 11.5 / RC ** 2


def k_max_for(box):
    return int(math.ceil(math.sqrt(4 * ALPHA * 11.5) * box / (2 * math.pi)))


def boxes(n_boxes, n_per_box, seed):
    parts = [S.periodic_box(n_atoms_total=n_per_box, cutoff=RC, seed=seed + b, build_list=False) for b in range(n_boxes)]
    R = np.concatenate([p[S.R] for p in parts])
    return dict(R=R, cell=np.concatenate([p[S.cell] for p in parts]), n=np.array([n_per_box] * n_boxes),
                box=float(parts[0][S.cell][0, 0, 0]))


def kernel_times(b, reps, dev):
    R = torch.as_tensor(b["R"], device=dev)
    N, B = R.shape[0], len(b["n"])
    idx_m = torch.repeat_interleave(torch.arange(B, device=dev), torch.as_tensor(b["n"], device=dev))
    sys_ptr = ops.segment_ptr(idx_m, B)
    cell = torch.as_tensor(b["cell"], device=dev).contiguous()
    kmax = k_max_for(b["box"])
    kv = A.EnergyEwald(ALPHA, kmax, 1.0, 1.0, "e").kvecs.to(dev).contiguous()
    q = (0.3 * torch.randn(N, device=dev, generator=torch.Generator(dev).manual_seed(0))).contiguous()
    g_E = torch.ones(B, device=dev)
    g_q = torch.zeros(N, device=dev)
    _, ws = ops.ewald_fwd(R, q, cell, kv, idx_m, sys_ptr, B, 1.0, ALPHA)

    def fwd():
        ops.ewald_fwd(R, q, cell, kv, idx_m, sys_ptr, B, 1.0, ALPHA)

    def bwd():
        ops.ewald_bwd(R, q, cell, kv, idx_m, sys_ptr, B, 1.0, ALPHA, g_E, ws, True, g_q, True)

    for fn in (fwd, bwd):
        fn()
    torch.cuda.synchronize()
    t = {"fwd": [], "bwd": []}
    for _ in range(3):
        t["fwd"].append(time_ms(fwd, reps))
        t["bwd"].append(time_ms(bwd, reps))
    K = int(kv.shape[0])
    fwd_ms, bwd_ms = min(t["fwd"]), min(t["bwd"])
    return dict(n_atoms=N, n_sys=B, box=b["box"], alpha=ALPHA, k_max=kmax, K=K, fwd_ms=fwd_ms, bwd_ms=bwd_ms,
                fwd_gterms_per_s=N * K / fwd_ms * 1e-6, bwd_gterms_per_s=N * K / bwd_ms * 1e-6, all_ms=t)


def with_charges(base, ewald):
    old = base.output_modules[0]
    e_nn = A.Atomwise(old.outnet[0].in_features, output_key="e_nn")
    e_nn.load_state_dict(old.state_dict())
    outs = [A.DipoleMoment(128, return_charges=True), e_nn]
    keys = ["e_nn"]
    if ewald:
        outs.append(A.EnergyEwald(ALPHA, k_max_for(43.4), "kcal/mol", "Ang", "e_ewald", use_neighbors_lr=False))
        keys.append("e_ewald")
    outs += [A.Aggregation(keys, "energy"), A.Forces()]
    return NeuralNetworkPotential(base.representation, list(base.input_modules), outs, postprocessors=[],
                                  do_postprocessing=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    res = dict(gpu=gpu_info(dev))
    res["reciprocal_kernels"] = {"cfg4_box_8192": kernel_times(boxes(1, 8192, 0), a.reps, dev),
                                 "64_boxes_of_128": kernel_times(boxes(64, 128, 10), a.reps, dev)}
    spec, data = S.make_config("cfg4")
    base = from_spec(spec, S.init_params(spec, seed=1), dev)
    torch.manual_seed(0)
    heads = with_charges(base, False).to(dev).eval()
    torch.manual_seed(0)
    full = with_charges(base, True).to(dev).eval()
    gps = {"painn+charges": GraphedPotential(heads), "painn+charges+ewald": GraphedPotential(full)}
    for gp in gps.values():
        gp(batch_to_device(data, dev))
    steps = {k: [] for k in gps}
    for _ in range(3):                                     # alternate the variants
        for k, gp in gps.items():
            steps[k].append(time_ms(gp.replay, a.reps))
    res["graphed_step"] = dict(n_atoms=int(data[S.Z].shape[0]), n_edges=int(data[S.idx_i].shape[0]),
                               K=int(full.output_modules[2].kvecs.shape[0]),
                               step_ms={k: min(v) for k, v in steps.items()}, step_ms_all=steps)
    res["gpu_after"] = gpu_info(dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
