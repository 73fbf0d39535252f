"""SO3net E+F timing on one GPU: graphed model step (CUDA events), the edge forward / reverse kernels alone (100 launches
captured in one graph), the reference modules run eagerly on the same GPU, an lmax sweep and the 8192-atom periodic box.

    python tools/bench_so3net.py [--reps 50]

Prints one JSON object.  The GPU name, its power limit and SM clocks are read in the same run.  Nothing is written to the
repository.  Traffic / FLOP estimates of the edge kernels come from the shapes (see ``edge_model``).
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from schnetpack_b200 import ops  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402
from schnetpack_b200.model import GraphedPotential, batch_to_device, from_spec  # noqa: E402
from schnetpack_b200.nn import so3  # noqa: E402


def gpu_info(dev):
    info = {"name": torch.cuda.get_device_name(dev)}
    try:
        out = subprocess.run(["nvidia-smi", f"--id={dev.index}", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout
        pl, sm, mx = (v.strip() for v in out.strip().split(","))
        info.update(power_limit_w=float(pl), sm_mhz=float(sm), sm_max_mhz=float(mx))
    except Exception:
        info.update(power_limit_w=None, sm_mhz=None, sm_max_mhz=None)
    return info


def time_ms(fn, reps):
    s, e = torch.cuda.Event(True), torch.cuda.Event(True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def graphed_ms(fn, n=100):
    """mean time of one ``fn`` call with ``n`` calls captured in one CUDA graph"""
    fn()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    g.replay()
    torch.cuda.synchronize()
    return time_ms(g.replay, 5) / n


def edge_model(N, E, F, L, n_rbf):
    """bytes / FLOPs of one edge forward: per edge the sender row (S F floats, from L2 when it is reused), the phi/geo
    records, 2 FLOPs per CG term and channel plus the filter (2 (L+1) n_rbf per channel); output S F floats per atom."""
    S_ = (L + 1) ** 2
    nnz = so3.sparse_clebsch_gordan(L)[0].shape[0]
    flops = E * F * (2 * nnz + 2 * (L + 1) * n_rbf + 2 * S_)
    gather = E * S_ * F * 4
    dram = N * S_ * F * 4 * 2 + E * (ops.kp(n_rbf) + 8) * 4
    return dict(flops=flops, gather_bytes=gather, dram_bytes=dram)


def case(dev, data, lmax, reps, with_ref=False):
    spec = S.model_spec("so3net", n_atom_basis=128, n_interactions=3, lmax=lmax)
    params = S.init_params(spec, seed=1)
    model = from_spec(spec, params, dev)
    x = batch_to_device(data, dev)
    gp = GraphedPotential(model)
    gp(x)
    step = time_ms(gp.replay, reps)
    # the edge kernels alone, on the graph / records of this batch
    rep = model.representation
    pk = rep._pack()
    xin = {k: v.clone() for k, v in x.items()}
    xin["_positions"].requires_grad_(True)
    r_ij = (xin["_positions"][xin["_idx_j"]] - xin["_positions"][xin["_idx_i"]] + xin["_offsets"]).detach().contiguous()
    N = x["_atomic_numbers"].shape[0]
    graph = ops.get_graph(x["_idx_i"], x["_idx_j"], N)
    phi, dphi, geo = ops.edge_geometry(r_ij, graph, rep._rbf_kind, rep._n_rbf, rep._rbf_p0, rep._rbf_p1,
                                       rep._cutoff_value, True)
    F, S_ = 128, (lmax + 1) ** 2
    feat = torch.randn((N, S_, F), device=dev)
    g_rij = torch.zeros((graph.n_edges, 3), device=dev)
    b = pk.blocks[1]
    fwd = graphed_ms(lambda: ops.so3_conv_fwd(feat, phi, geo, graph, b["wf"], b["bf"], lmax, F, rep._n_rbf))
    bwd = graphed_ms(lambda: ops.so3_conv_bwd(feat, feat, phi, dphi, geo, graph, b["wf"], b["bf"], lmax, F, rep._n_rbf,
                                              feat, g_rij, accumulate=False))
    out = dict(lmax=lmax, n_atoms=int(N), n_edges=int(graph.n_edges), step_ms=step, edge_fwd_ms=fwd, edge_bwd_ms=bwd,
               edge_fwd_model=edge_model(N, graph.n_edges, F, lmax, rep._n_rbf))
    if with_ref:
        import so3net_oracle as SO
        from oracle import ref_loader as rl

        if rl.available():
            ref = SO.build_reference(spec, params, torch.float32, dev)
            try:
                out["reference_eager_ms"] = time_ms(lambda: SO.evaluate(ref, data, torch.float32, dev), max(2, reps // 10))
            except torch.cuda.OutOfMemoryError:
                out["reference_eager_ms"] = "out of memory"
            del ref
            torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    info = gpu_info(dev)
    cfg2 = S.aspirin_batch(256)
    res = dict(gpu=info, cfg2=[case(dev, cfg2, 2, a.reps, with_ref=True), case(dev, cfg2, 1, a.reps),
                               case(dev, cfg2, 3, a.reps)],
               cfg4=case(dev, S.periodic_box(8192), 2, a.reps))
    res["gpu_after"] = gpu_info(dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
