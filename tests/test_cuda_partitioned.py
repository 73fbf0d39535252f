"""GPU: ONE periodic system evaluated by several ranks with the CUDA engine (SURVEY.md section 8e, cfg5 path):
``parallel.partition_graph`` + ``parallel.PartitionedPotential`` (per-block kernel pipelines, HaloExchange of ghost rows in
front of every edge kernel, reverse halo in the backward sweep) must reproduce the single-device CUDA evaluation and the fp64
reference of the same box -- the parity oracle for multi-GPU, since the reference itself has no multi-device path.

* ``test_two_ranks_one_gpu``: two processes share cuda:0 and exchange over gloo (rows staged through the host); runs on the
  single-GPU box the driver tests on, and exercises every line of the partitioned CUDA engine except the NCCL transport.
* ``test_ranks_over_nccl``: one process per GPU over NCCL point-to-point (skipped below 2 GPUs).
"""
import os
import socket
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, backend, n_atoms, out_path):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    if backend == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    from schnetpack_b200 import parallel as P
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, from_spec

    spec = S.model_spec("painn", n_atom_basis=128, n_interactions=3)
    params = S.init_params(spec, seed=11)
    box = S.periodic_box(n_atoms, seed=12)
    model = from_spec(spec, params, dev)
    owner = P.slab_owners(box["_positions"], world)
    plan = P.partition_graph(owner, box["_idx_i"], box["_idx_j"], rank, world)
    engine = P.PartitionedPotential(model, box, plan, dev)
    for _ in range(2):                                  # twice: cached plan tensors, graph views, weight packs
        energy, f_own = engine()
    torch.cuda.synchronize()
    # gather the owned force blocks on rank 0 (test plumbing)
    parts = [None] * world
    dist.all_gather_object(parts, (plan.owned, f_own.cpu().numpy()))
    if rank == 0:
        forces = np.zeros((n_atoms, 3), dtype=np.float32)
        for own, f in parts:
            forces[own] = f
        single = model(batch_to_device(box, dev))       # the same box on ONE device through the monolithic pipeline
        np.savez(out_path, e=energy.cpu().numpy(), f=forces, e1=single["energy"].detach().cpu().numpy(),
                 f1=single["forces"].detach().cpu().numpy(), ghosts=np.array([plan.n_ghost]))
    dist.barrier()
    dist.destroy_process_group()


def _check(out, n_atoms):
    from conftest import rel_err
    from oracle import spk_oracle as O
    from schnetpack_b200 import synthetic as S

    z = np.load(out)
    assert int(z["ghosts"][0]) > 0
    # vs the single-device CUDA evaluation of the same box (same kernels, different summation grouping of nothing: each
    # edge is computed once by exactly one rank, so only the graph partition differs)
    assert rel_err(z["e"], z["e1"]) < 2e-6
    assert rel_err(z["f"], z["f1"]) < 5e-6
    spec = S.model_spec("painn", n_atom_basis=128, n_interactions=3)
    ref = O.energy_forces(spec, S.init_params(spec, seed=11), S.periodic_box(n_atoms, seed=12), dtype=torch.float64)
    assert rel_err(z["e"], ref["energy"].numpy()) < 1e-5
    assert rel_err(z["f"], ref["forces"].numpy()) < 1e-5


@pytest.mark.timeout(600)
@pytest.mark.parametrize("world", [2, 3])
def test_two_ranks_one_gpu(tmp_path, world):
    import torch.multiprocessing as mp

    out = str(tmp_path / "res.npz")
    n_atoms = 1200                                      # ~62 k edges: tensor-core edge kernels on every rank
    mp.spawn(_worker, args=(world, _free_port(), "gloo", n_atoms, out), nprocs=world, join=True)
    _check(out, n_atoms)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("transport", ["peer", "nccl"])
def test_ranks_over_nccl(tmp_path, transport, monkeypatch):
    """one process per GPU: halo over NVLink peer memory (default: hand-written pull kernels over symmetric memory) and over
    NCCL point-to-point (SPK_B200_HALO=nccl)"""
    import torch.multiprocessing as mp

    monkeypatch.setenv("SPK_B200_HALO", transport)
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs >= 2 GPUs (NCCL cannot put two ranks on one device))")
    out = str(tmp_path / "res.npz")
    n_atoms = 3000
    mp.spawn(_worker, args=(world, _free_port(), "nccl", n_atoms, out), nprocs=world, join=True)
    _check(out, n_atoms)


def test_model_on_second_device_without_set_device():
    """A model moved to cuda:1 while cuda:0 stays the current device: streams, launch caches and the >48 KB shared-memory
    opt-ins follow the tensors' device (ops.device_of, per-device caches in the library)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    sys.path.insert(0, ROOT)
    from conftest import rel_err
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, data = S.make_config("cfg2", batch=24)
    params = S.init_params(spec, seed=3)
    torch.cuda.set_device(0)
    outs = []
    for d in ("cuda:0", "cuda:1"):
        model = from_spec(spec, params, torch.device(d))
        out = model(batch_to_device(data, torch.device(d)))
        torch.cuda.synchronize(torch.device(d))
        outs.append({k: v.detach().cpu().numpy() for k, v in out.items()})
    assert torch.cuda.current_device() == 0
    assert rel_err(outs[1]["energy"], outs[0]["energy"]) < 1e-6 and rel_err(outs[1]["forces"], outs[0]["forces"]) < 1e-6
