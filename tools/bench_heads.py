"""DipoleMoment / Polarizability timing on one GPU at cfg2 (aspirin x 256, PaiNN 128 x 3): the graphed energy + forces step
with and without each head (CUDA events, steps alternated), the head kernels alone (forward and reverse of the head on
fixed representations, 100 calls captured in one graph), the reference heads run eagerly on the same GPU on top of
this package's representation, and the NVE DeviceMD step without heads, with both heads, and with both heads recorded
every step.

    python tools/bench_heads.py [--reps 50]

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
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_so3net import gpu_info, graphed_ms, time_ms  # noqa: E402

from schnetpack_b200 import atomistic as A  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.model import GraphedPotential, NeuralNetworkPotential, batch_to_device, from_spec  # noqa: E402


def with_heads(base, heads):
    return NeuralNetworkPotential(base.representation, list(base.input_modules), list(base.output_modules) + heads,
                                  postprocessors=[], do_postprocessing=False).eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    info = gpu_info(dev)
    spec, data = S.make_config("cfg2")
    base = from_spec(spec, S.init_params(spec, seed=1), dev)
    torch.manual_seed(0)
    dip = A.DipoleMoment(128, use_vector_representation=True).to(dev)
    dip_s = A.DipoleMoment(128).to(dev)
    pol = A.Polarizability(128).to(dev)
    variants = {"none": [], "dipole_vector": [dip], "dipole_scalar": [dip_s], "polarizability": [pol],
                "dipole_vector+polarizability": [dip, pol]}
    gps = {}
    for k, hs in variants.items():
        gps[k] = GraphedPotential(with_heads(base, hs))
        gps[k](batch_to_device(data, dev))
    steps = {k: [] for k in variants}
    for _ in range(3):                                     # alternate the variants
        for k, gp in gps.items():
            steps[k].append(time_ms(gp.replay, a.reps))
    res = dict(gpu=info, n_atoms=int(data[S.Z].shape[0]), step_ms={k: min(v) for k, v in steps.items()},
               step_ms_all=steps)
    # the heads alone on fixed representations (forward + reverse with respect to s, V and R)
    x = batch_to_device(data, dev)
    rep_out = base.representation(base.input_modules[0](dict(x)))
    s = rep_out["scalar_representation"].detach().requires_grad_(True)
    V = rep_out["vector_representation"].detach().requires_grad_(True)
    R = x[S.R].detach().requires_grad_(True)
    fixed = {S.idx_m: x[S.idx_m], S.n_atoms: x[S.n_atoms]}

    def head_fb(h, key):
        def run():
            y = h(dict(fixed, scalar_representation=s, vector_representation=V, _positions=R))[key]
            torch.autograd.grad(y.sum(), [s, V, R], allow_unused=True)
        return run

    def head_f(h, key):
        def run():
            with torch.no_grad():
                h(dict(fixed, scalar_representation=s, vector_representation=V, _positions=R))
        return run

    res["head_alone_ms"] = {
        "dipole_vector_fwd": graphed_ms(head_f(dip, "dipole_moment")),
        "dipole_vector_fwd_bwd": graphed_ms(head_fb(dip, "dipole_moment")),
        "polarizability_fwd": graphed_ms(head_f(pol, "polarizability")),
        "polarizability_fwd_bwd": graphed_ms(head_fb(pol, "polarizability")),
        "dipole_scalar_fwd_bwd": graphed_ms(head_fb(dip_s, "dipole_moment")),
    }
    from oracle import ref_loader as rl

    if rl.available():
        spk = rl.load()
        torch.manual_seed(0)
        rd = spk.atomistic.DipoleMoment(128, use_vector_representation=True).to(dev)
        rp = spk.atomistic.Polarizability(128).to(dev)
        rd.load_state_dict(dip.state_dict())
        rp.load_state_dict(pol.state_dict())
        res["reference_heads_eager_ms"] = {"dipole_vector_fwd_bwd": time_ms(head_fb(rd, "dipole_moment"), a.reps),
                                           "polarizability_fwd_bwd": time_ms(head_fb(rp, "polarizability"), a.reps)}
        full = with_heads(base, [rd, rp])
        res["reference_heads_on_package_rep_step_ms"] = time_ms(lambda: full(batch_to_device(data, dev)), 10)
    from schnetpack_b200.md import DeviceMD

    N, E = int(data[S.Z].shape[0]), int(data[S.idx_i].shape[0])
    masses = torch.ones(N, device=dev)
    both = with_heads(base, [dip, pol])
    mds = {"no_heads": DeviceMD(base, x, masses, time_step=1e-4, cutoff=spec["cutoff"], capacity=int(E * 1.15)),
           "heads": DeviceMD(both, x, masses, time_step=1e-4, cutoff=spec["cutoff"], capacity=int(E * 1.15)),
           "heads_recorded": DeviceMD(both, x, masses, time_step=1e-4, cutoff=spec["cutoff"], capacity=int(E * 1.15),
                                      required_properties=["dipole_moment", "polarizability"], record_every=1,
                                      record_capacity=10 * (a.reps + 5))}
    for md in mds.values():
        md.run(5)
    md_ms = {k: [] for k in mds}
    for _ in range(3):
        for k, md in mds.items():
            md_ms[k].append(time_ms(lambda: md.run(a.reps), 1) / a.reps)
    res["device_md_nve_ms_per_step"] = {k: min(v) for k, v in md_ms.items()}
    res["device_md_nve_ms_all"] = md_ms
    res["gpu_after"] = gpu_info(dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
