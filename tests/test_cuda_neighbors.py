"""GPU neighbour list (csrc/neighbors.cu, SURVEY.md section 8 row f1) against the pinned oracle (oracle/nl_oracle.py ==
reference TorchNeighborList on tests/golden/nl_*.npz): bit-exact pair sets and image vectors after the canonical sort."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err  # noqa: F401

from oracle import nl_oracle as NL

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _np(t):
    return t.detach().cpu().numpy()


def _gpu_nl(R, cell, pbc, n_atoms, cutoff, **kw):
    from schnetpack_b200.neighbors import neighbor_list

    out = neighbor_list(torch.as_tensor(np.asarray(R), dtype=torch.float32, device=DEV),
                        None if cell is None else torch.as_tensor(np.asarray(cell), dtype=torch.float32, device=DEV),
                        None if pbc is None else torch.as_tensor(np.asarray(pbc), device=DEV),
                        torch.as_tensor(np.asarray(n_atoms), device=DEV), cutoff, return_shifts=True, **kw)
    torch.cuda.synchronize()
    return out


def _same_set(out, ref, n=None):
    ii, jj, off, sh, n_pairs = out
    n = int(n_pairs[0]) if n is None else n
    gi, gj, gs = NL.canonical(ii[:n].cpu().numpy(), jj[:n].cpu().numpy(), sh[:n].cpu().numpy().astype(np.int64))
    ri, rj, rs, roff = ref
    assert gi.shape == ri.shape, (gi.shape, ri.shape)
    assert (gi == ri).all() and (gj == rj).all() and (gs == rs).all()
    return n


@pytest.mark.parametrize("name", ["molecule", "cubic", "small_box", "triclinic", "slab", "fcc_primitive", "skewed"])
def test_neighbor_list_matches_reference_fixture(name):
    d = np.load(os.path.join(GOLD, f"nl_{name}.npz"))
    R = d["positions"].astype(np.float32)
    out = _gpu_nl(R, d["cell"][None], d["pbc"][None], [R.shape[0]], float(d["cutoff"]))
    assert int(out[-1][1]) == 0
    n = _same_set(out, (d["idx_i"], d["idx_j"], d["shifts"], None))
    ii, jj, off, sh, _ = out
    # rows sorted by receiver, offsets = S @ cell, every listed pair inside the cutoff as the model computes r_ij
    assert (ii[1:] >= ii[:-1]).all()
    cell = torch.as_tensor(d["cell"], dtype=torch.float32, device=DEV)
    assert torch.allclose(off, sh.float() @ cell, atol=1e-5)
    Rt = torch.as_tensor(R, device=DEV)
    assert ((Rt[jj] - Rt[ii] + off).norm(dim=1) < float(d["cutoff"])).all()
    assert n == d["idx_i"].shape[0]


def test_neighbor_list_collated_batch_mixed_systems():
    """molecules, an empty system, a single atom, a periodic box and a slab in ONE collated batch."""
    rng = np.random.default_rng(5)
    sys_R, cells, pbcs = [], [], []
    for na in (21, 0, 1, 9):
        sys_R.append(rng.normal(size=(na, 3)) * 1.8)
        cells.append(np.zeros((3, 3)))
        pbcs.append([False] * 3)
    L = 17.0
    sys_R.append(rng.uniform(-2, L + 2, size=(300, 3)))
    cells.append(np.eye(3) * L)
    pbcs.append([True] * 3)
    sys_R.append(rng.uniform(0, 1, size=(120, 3)) @ np.diag([12.0, 11.0, 8.0]))
    cells.append(np.diag([12.0, 11.0, 40.0]))
    pbcs.append([True, True, False])
    R = np.concatenate(sys_R).astype(np.float32)
    n_atoms = [r.shape[0] for r in sys_R]
    ref = NL.batch_neighbor_list(R.astype(np.float64), np.stack(cells), np.array(pbcs), n_atoms, 5.0)
    out = _gpu_nl(R, np.stack(cells), np.array(pbcs), n_atoms, 5.0)
    _same_set(out, ref)


def test_neighbor_list_matches_generator_of_cfg4_and_feeds_the_model():
    """The list the benchmark generator builds on the host (synthetic.periodic_box) == the device list, and the model gives
    the same energy and forces with either (edge order differs: the graph build regroups)."""
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, from_spec
    from schnetpack_b200.neighbors import CellListNeighborList

    spec, data = S.make_config("cfg4", n_atoms_total=1500)
    params = S.init_params(spec, seed=2)
    model = from_spec(spec, params, torch.device(DEV))
    a = model(batch_to_device(data, torch.device(DEV)))
    x = batch_to_device(data, torch.device(DEV))
    for k in ("_idx_i", "_idx_j", "_offsets"):
        x.pop(k)
    x = CellListNeighborList(spec["cutoff"])(x)
    assert x["_idx_i"].shape[0] == data["_idx_i"].shape[0]
    b = model(x)
    torch.cuda.synchronize()
    from conftest import rel_err

    assert rel_err(_np(b["energy"]), _np(a["energy"])) < 2e-6
    assert rel_err(_np(b["forces"]), _np(a["forces"])) < 2e-6


def test_neighbor_list_fixed_capacity_padding_is_inert():
    """capacity + pad: no host read; the padded tail lies outside the cutoff and changes neither energy nor forces."""
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, from_spec
    from schnetpack_b200.neighbors import CellListNeighborList
    from conftest import rel_err

    spec, data = S.make_config("cfg2", batch=24)
    params = S.init_params(spec, seed=4)
    model = from_spec(spec, params, torch.device(DEV))
    x = batch_to_device(data, torch.device(DEV))
    x["_cell"] = torch.zeros((24, 3, 3), device=DEV)
    x["_pbc"] = torch.zeros((24, 3), dtype=torch.bool, device=DEV)
    a = model(dict(x))
    E = data["_idx_i"].shape[0]
    y = {k: v for k, v in x.items() if k not in ("_idx_i", "_idx_j", "_offsets")}
    y = CellListNeighborList(spec["cutoff"], capacity=E + 500, pad=True)(y)
    assert y["_idx_i"].shape[0] == E + 500 and int(y["_n_pairs"][0]) == E and int(y["_n_pairs"][1]) == 0
    b = model(y)
    torch.cuda.synchronize()
    assert rel_err(_np(b["energy"]), _np(a["energy"])) < 2e-6
    assert rel_err(_np(b["forces"]), _np(a["forces"])) < 2e-6
    # overflow is reported, not silently truncated
    z = {k: v for k, v in x.items() if k not in ("_idx_i", "_idx_j", "_offsets")}
    z = CellListNeighborList(spec["cutoff"], capacity=E - 10)(z)
    assert int(z["_n_pairs"][0]) == E and int(z["_n_pairs"][1]) == 1


def test_device_md_graph_replay_matches_eager_loop_and_conserves_energy():
    """schnetpack_b200.md.DeviceMD (velocity Verlet + device neighbour list + model, one CUDA graph per step) follows the
    same trajectory as the eager loop, never reads the device, and conserves total energy at a small time step."""
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.md import DeviceMD
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, data = S.make_config("cfg4", n_atoms_total=600)
    params = S.init_params(spec, seed=6)
    dev = torch.device(DEV)
    model = from_spec(spec, params, dev)
    x = batch_to_device(data, dev)
    N = data["_positions"].shape[0]
    masses = torch.where(torch.as_tensor(data["_atomic_numbers"]) == 8, 16.0, 1.0)
    torch.manual_seed(0)
    p0 = torch.randn(N, 3) * 0.05
    cap = int(data["_idx_i"].shape[0] * 1.3)
    runs = {}
    for use_graph in (True, False):
        md = DeviceMD(model, x, masses, time_step=2e-3, cutoff=spec["cutoff"], capacity=cap, momenta=p0, use_graph=use_graph)
        e0 = float(md.energy.sum() + md.kinetic_energy())
        md.run(40)
        torch.cuda.synchronize()
        runs[use_graph] = (_np(md.positions), float(md.energy.sum() + md.kinetic_energy()), e0, _np(md.n_pairs))
    assert np.abs(runs[True][0] - runs[False][0]).max() < 1e-4
    assert runs[True][3][1] == 0 and runs[True][3][0] > 0          # no overflow, pairs found
    moved = np.abs(runs[True][0] - data["_positions"]).max()
    assert moved > 1e-3                                             # the trajectory actually advanced
    for g in (True, False):
        assert abs(runs[g][1] - runs[g][2]) < 2e-3 * max(1.0, abs(runs[g][2])), runs[g]


@pytest.mark.parametrize("p_conv,e_conv", [(1.0, 1.0), (10.0, 0.5)])
def test_device_md_follows_the_reference_nve_loop(p_conv, e_conv):
    """DeviceMD (integrator kernel spk_md_velocity_verlet, device neighbour list, CUDA model, unit conversions) against
    oracle/md_oracle.py -- the reference's simulator / VelocityVerlet / calculator arithmetic restated in fp64 with the pinned
    energy-force oracle and an exact neighbour list per step -- over 12 steps of a 150-atom periodic box, with MD units that
    differ from the model's (positions x 1/10, energies x 1/2) in the second case."""
    from oracle import md_oracle as MO
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.md import DeviceMD
    from schnetpack_b200.model import batch_to_device, from_spec

    spec = S.model_spec("painn", n_atom_basis=128, n_interactions=2)
    data = S.periodic_box(150, seed=9)
    params = S.init_params(spec, seed=8)
    dev = torch.device(DEV)
    model = from_spec(spec, params, dev)
    N = data["_positions"].shape[0]
    masses = np.where(data["_atomic_numbers"] == 8, 16.0, 1.0)
    rng = np.random.default_rng(2)
    p0 = rng.normal(0, 0.05, (N, 3))
    dt, n_steps = 1e-3, 12
    md = DeviceMD(model, batch_to_device(data, dev), torch.as_tensor(masses), time_step=dt, cutoff=spec["cutoff"],
                  capacity=int(data["_idx_i"].shape[0] * 1.5), momenta=torch.as_tensor(p0), position_conversion=p_conv,
                  energy_conversion=e_conv)
    md.run(n_steps)
    torch.cuda.synchronize()
    x_ref, p_ref, e_ref, f_ref = MO.nve_trajectory(spec, params, data, masses, p0, dt, n_steps, p_conv, e_conv)
    assert rel_err(_np(md.positions), x_ref) < 1e-6
    assert rel_err(_np(md.momenta), p_ref) < 1e-4
    assert rel_err(_np(md.potential_energy()), e_ref) < 1e-5
    assert rel_err(_np(md.forces) * (e_conv / p_conv), f_ref) < 1e-4
    assert md.peak_pairs > 0
