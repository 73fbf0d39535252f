"""Cost of smooth particle-mesh Ewald on one GPU against the Ewald sum at matched accuracy (alpha = 0.46 A^-2 as in
tools/bench_ewald.py; Ewald k_max for about 1e-5 truncation, PME at the order and spacing of tests/pme_oracle.py
ACCURACY, which reach 1e-5 against the converged Ewald sum):

1. the reciprocal term alone, forward (spread, rfftn, influence) and reverse (irfftn, gather), against spk_ewald_fwd /
   spk_ewald_bwd, on the cfg4 box (8192 atoms) and on 64 boxes of 128 atoms;
2. the graphed cfg4 E+F step of bench_ewald's charged PaiNN 128 x 3 model with no long-range term, with EnergyEwald and
   with EnergyPME (variants alternated in one session, every shape and cuFFT plan warmed up first, best of three);
   and how far the two, and Ewald at that k_max, are from the same model with Ewald at k_max 45 (past convergence);
3. the cfg5 box (262 144 atoms) E+F with EnergyPME next to the same model without it.  Ewald is not run there.

    python tools/bench_pme.py [--reps 20] [--no-cfg5]

Prints one JSON object.  The GPU name, its power limit and SM clocks are read in the same run.  Nothing is written to the
repository.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_ewald import ALPHA, boxes, k_max_for, kernel_times, with_charges  # noqa: E402
from bench_so3net import gpu_info, time_ms  # noqa: E402

import pme_oracle  # noqa: E402
from schnetpack_b200 import atomistic as A  # noqa: E402
from schnetpack_b200 import ops  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.model import GraphedPotential, batch_to_device, from_spec  # noqa: E402

ORDER, SPACING = next(iter(pme_oracle.ACCURACY.items()))


def pme_callables(b, dev):
    """-> (mesh, forward, reverse) of the PME reciprocal term on boxes ``b``, both warmed up"""
    R = torch.as_tensor(b["R"], device=dev)
    N, B = R.shape[0], len(b["n"])
    idx_m = torch.repeat_interleave(torch.arange(B, device=dev), torch.as_tensor(b["n"], device=dev))
    sys_ptr = ops.segment_ptr(idx_m, B)
    cell = torch.as_tensor(b["cell"], device=dev).contiguous()
    mesh = A.pme_mesh(cell, SPACING, ORDER)
    q = (0.3 * torch.randn(N, device=dev, generator=torch.Generator(dev).manual_seed(0))).contiguous()
    g_E = torch.ones(B, device=dev)
    g_q = torch.zeros(N, device=dev)
    _, conv, ws = ops.pme_fwd(R, q, cell, idx_m, sys_ptr, B, mesh, ORDER, 1.0, ALPHA)

    def fwd():
        ops.pme_fwd(R, q, cell, idx_m, sys_ptr, B, mesh, ORDER, 1.0, ALPHA)

    def bwd():
        ops.pme_bwd(R, q, idx_m, sys_ptr, B, mesh, ORDER, 1.0, ALPHA, g_E, conv, ws, True, g_q, True)

    for fn in (fwd, bwd):
        fn()
    torch.cuda.synchronize()
    return mesh, fwd, bwd


def reciprocal(b, reps, dev):
    mesh, fwd, bwd = pme_callables(b, dev)
    t = {"pme_fwd": [], "pme_bwd": []}
    ew = None
    for _ in range(3):                                     # alternate PME and Ewald
        t["pme_fwd"].append(time_ms(fwd, reps))
        t["pme_bwd"].append(time_ms(bwd, reps))
        e = kernel_times(b, reps, dev)
        ew = e if ew is None or e["fwd_ms"] + e["bwd_ms"] < ew["fwd_ms"] + ew["bwd_ms"] else ew
    return dict(n_atoms=int(b["R"].shape[0]), n_sys=len(b["n"]), box=b["box"], order=ORDER, spacing=SPACING,
                mesh=list(mesh), pme_fwd_ms=min(t["pme_fwd"]), pme_bwd_ms=min(t["pme_bwd"]),
                ewald_k_max=ew["k_max"], ewald_K=ew["K"], ewald_fwd_ms=ew["fwd_ms"], ewald_bwd_ms=ew["bwd_ms"],
                pme_all_ms=t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--no-cfg5", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    res = dict(gpu=gpu_info(dev))
    res["reciprocal"] = {"cfg4_box_8192": reciprocal(boxes(1, 8192, 0), a.reps, dev),
                         "64_boxes_of_128": reciprocal(boxes(64, 128, 10), a.reps, dev)}
    spec, data = S.make_config("cfg4")
    base = from_spec(spec, S.init_params(spec, seed=1), dev)
    mesh = A.pme_mesh(torch.as_tensor(data[S.cell]), SPACING, ORDER)
    models = {}
    for name, ewald in (("painn+charges", False), ("painn+charges+ewald", True), ("painn+charges+pme", True)):
        torch.manual_seed(0)
        m = with_charges(base, ewald).to(dev).eval()
        models[name] = A.use_pme(m, mesh, ORDER) if name.endswith("pme") else m
    gps = {k: GraphedPotential(m) for k, m in models.items()}
    outs = {k: {o: v.detach().clone() for o, v in gp(batch_to_device(data, dev)).items()} for k, gp in gps.items()}
    steps = {k: [] for k in gps}
    for _ in range(3):                                     # alternate the variants
        for k, gp in gps.items():
            steps[k].append(time_ms(gp.replay, a.reps))
    # the same model with the Ewald sum far past convergence (k_max 45), evaluated once, not timed
    ew45 = models["painn+charges+ewald"]
    ewm = ew45.output_modules[2]
    ewm.k_max = 45
    ewm.kvecs = ewm._generate_kvecs().to(dev)
    outs["painn+charges+ewald45"] = {o: v.detach().clone() for o, v in ew45(batch_to_device(data, dev)).items()}

    def agree(a, b):
        return {k: float((outs[a][k] - outs[b][k]).abs().max() / outs[b][k].abs().max())
                for k in ("energy", "e_ewald", "forces") if k in outs[a] and k in outs[b]}

    res["graphed_cfg4_step"] = dict(
        n_atoms=int(data[S.Z].shape[0]), mesh=list(mesh), order=ORDER, step_ms={k: min(v) for k, v in steps.items()},
        step_ms_all=steps, ewald_k_max=k_max_for(43.4),
        pme_vs_ewald=agree("painn+charges+pme", "painn+charges+ewald"),
        pme_vs_ewald45=agree("painn+charges+pme", "painn+charges+ewald45"),
        ewald_vs_ewald45=agree("painn+charges+ewald", "painn+charges+ewald45"))
    del gps, models, outs, ew45
    torch.cuda.empty_cache()
    if not a.no_cfg5:
        spec, data = S.make_config("cfg5")
        base = from_spec(spec, S.init_params(spec, seed=1), dev)
        mesh = A.pme_mesh(torch.as_tensor(data[S.cell]), SPACING, ORDER)
        torch.manual_seed(0)
        plain = with_charges(base, False).to(dev).eval()
        torch.manual_seed(0)
        pme = A.use_pme(with_charges(base, True).to(dev).eval(), mesh, ORDER)
        x = batch_to_device(data, dev)
        runs = {"painn+charges": lambda: plain(dict(x)), "painn+charges+pme": lambda: pme(dict(x))}
        for fn in runs.values():
            fn()
        torch.cuda.synchronize()
        t = {k: [] for k in runs}
        for _ in range(3):
            for k, fn in runs.items():
                t[k].append(time_ms(fn, 3))
        res["cfg5_eager_e_f"] = dict(n_atoms=int(data[S.Z].shape[0]), mesh=list(mesh), order=ORDER,
                                     ms={k: min(v) for k, v in t.items()}, ms_all=t,
                                     max_memory_gb=torch.cuda.max_memory_allocated(dev) / 2 ** 30)
    res["gpu_after"] = gpu_info(dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
