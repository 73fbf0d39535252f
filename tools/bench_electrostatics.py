"""Cost of the PhysNet-style add-ons at cfg2 (aspirin x 256, PaiNN 128 x 3) on one GPU: the graphed energy + forces step
with and without DipoleMoment(return_charges) + ZBL (CosineCutoff) + damped Coulomb (shifted at the cutoff) + Aggregation
(CUDA events, variants alternated in one session), and the pair kernels alone (forward and reverse of each term on fixed
distances and charges, 100 calls captured in one graph).

    python tools/bench_electrostatics.py [--reps 50]

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

from bench_so3net import gpu_info, graphed_ms, time_ms  # noqa: E402

from schnetpack_b200 import atomistic as A  # noqa: E402
from schnetpack_b200 import nn as snn  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.model import GraphedPotential, NeuralNetworkPotential, batch_to_device, from_spec  # noqa: E402


def with_pair_terms(base, cutoff):
    old = base.output_modules[0]
    e_nn = A.Atomwise(old.outnet[0].in_features, output_key="e_nn")
    e_nn.load_state_dict(old.state_dict())
    outs = [A.DipoleMoment(128, return_charges=True), e_nn,
            A.ZBLRepulsionEnergy("kcal/mol", "Ang", "e_zbl", cutoff_fn=snn.CosineCutoff(cutoff)),
            A.EnergyCoulomb("kcal/mol", "Ang", A.DampedCoulombPotential(snn.SwitchFunction(1.0, cutoff - 1.0)), "e_coul",
                            use_neighbors_lr=False, cutoff=cutoff),
            A.Aggregation(["e_nn", "e_zbl", "e_coul"], "energy"), A.Forces()]
    return NeuralNetworkPotential(base.representation, list(base.input_modules), outs, postprocessors=[],
                                  do_postprocessing=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    info = gpu_info(dev)
    spec, data = S.make_config("cfg2")
    base = from_spec(spec, S.init_params(spec, seed=1), dev)
    torch.manual_seed(0)
    full = with_pair_terms(base, spec["cutoff"]).to(dev).eval()
    gps = {"painn": GraphedPotential(base), "painn+charges+zbl+coulomb": GraphedPotential(full)}
    for gp in gps.values():
        gp(batch_to_device(data, dev))
    steps = {k: [] for k in gps}
    for _ in range(3):                                     # alternate the variants
        for k, gp in gps.items():
            steps[k].append(time_ms(gp.replay, a.reps))
    res = dict(gpu=info, n_atoms=int(data[S.Z].shape[0]), n_edges=int(data[S.idx_i].shape[0]),
               step_ms={k: min(v) for k, v in steps.items()}, step_ms_all=steps)

    # the pair kernels alone on fixed distances and charges
    x = batch_to_device(data, dev)
    R = x[S.R].detach().requires_grad_(True)
    q = (0.1 * torch.randn(R.shape[0], 1, device=dev)).requires_grad_(True)
    zbl, coul = full.output_modules[2], full.output_modules[3]

    def term(mod, key, want_q):
        def run():
            y = dict(x, _positions=R, partial_charges=q)
            y = A.PairwiseDistances()(y)
            e = mod(y)[key]
            torch.autograd.grad(e.sum(), [R, q] if want_q else [R])
        return run

    def pairwise_only():
        y = A.PairwiseDistances()(dict(x, _positions=R))
        torch.autograd.grad(y[S.Rij].sum(), [R])

    pw = graphed_ms(pairwise_only)
    res["pair_kernels_ms"] = {
        "pairwise_distances_fwd_bwd": pw,
        "zbl_fwd_bwd_incl_distances": graphed_ms(term(zbl, "e_zbl", False)),
        "damped_coulomb_fwd_bwd_incl_distances": graphed_ms(term(coul, "e_coul", True)),
    }
    res["gpu_after"] = gpu_info(dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
