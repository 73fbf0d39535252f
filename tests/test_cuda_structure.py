"""Radial distribution functions and mean-squared displacements accumulated inside the captured DeviceMD step
(csrc/structure.cu, schnetpack_b200.structure) against the fp64 oracle tests/structure_oracle.py, fed with the positions
and cells of the same run read on the host after every step.

Tolerances: pair counts are integers and must match the oracle exactly except for pairs within EDGE_RTOL (relative) of
a bin edge, whose fp32 distance may fall on either side; the MSD unwraps the same fp32 positions in fp64 on both sides,
so only the summation order differs (rtol 1e-9)."""
import numpy as np
import pytest
import torch

import structure_oracle as SO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KB = 0.0025 / 300.0
SHEAR = np.array([[1.0, 0.0, 0.0], [0.22, 1.0, 0.0], [-0.15, 0.18, 1.0]])      # rows: a, b, c of the triclinic cell


def _np(t):
    return t.detach().cpu().numpy().astype(np.float64)


def _box(n=150, seed=9, triclinic=True, pbc=True, scatter=False):
    """a periodic box of O, H and C atoms (synthetic.periodic_box with every fifth atom made carbon), sheared into a
    triclinic cell; ``scatter`` moves every atom by a few lattice vectors"""
    from schnetpack_b200 import synthetic as S

    data = S.periodic_box(n, seed=seed, build_list=False)
    cell = data["_cell"].reshape(3, 3).astype(np.float64)
    if triclinic:
        new = SHEAR @ cell
        data["_positions"] = (data["_positions"].astype(np.float64) @ np.linalg.inv(cell) @ new).astype(np.float32)
        data["_cell"] = new[None].astype(np.float32)
    if scatter:
        shift = np.random.default_rng(1).integers(-2, 3, size=(n, 3)).astype(np.float64)
        data["_positions"] = (data["_positions"] + shift @ data["_cell"].reshape(3, 3)).astype(np.float32)
    data["_atomic_numbers"] = data["_atomic_numbers"].copy()
    data["_atomic_numbers"][::5] = 6
    if not pbc:
        data["_pbc"] = np.zeros(3, dtype=bool)
    return data


def _md(hooks, data=None, use_graph=True, momenta_seed=4, speed=1.0, **kw):
    from schnetpack_b200 import md as M
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, from_spec

    data = _box() if data is None else data
    spec = S.model_spec("painn", n_atom_basis=64, n_interactions=2)
    model = from_spec(spec, S.init_params(spec, seed=8), torch.device(DEV))
    z = data["_atomic_numbers"]
    masses = np.where(z == 8, 16.0, np.where(z == 6, 12.0, 1.0))
    n = z.shape[0]
    P = kw["ring_polymer"].n_beads if "ring_polymer" in kw else 1
    if "initializer" not in kw:
        kw["momenta"] = torch.as_tensor(np.random.default_rng(momenta_seed).normal(0, speed, (n, 3)) * masses[:, None])
    return M.DeviceMD(model, batch_to_device(data, torch.device(DEV)), torch.as_tensor(masses), time_step=1e-3,
                      cutoff=spec["cutoff"], capacity=n * 120 * P, use_graph=use_graph, hooks=hooks, **kw)


def _tables(rdf):
    T = len(rdf.species)
    slot_of = np.full((T, T), -1)
    total = -1
    for k, (a, b) in enumerate(rdf.pairs):
        if (a, b) == (0, 0):
            total = k
        else:
            slot_of[rdf.species.index(a), rdf.species.index(b)] = k
    return slot_of, total


def _trace(md, n_steps, every):
    """step one at a time; the model positions, model cells, MD cells and MD positions after every sampled step"""
    frames = []
    for s in range(n_steps):
        md.run(1)
        if s % every == 0:
            torch.cuda.synchronize()
            frames.append(dict(R=_np(md.model_positions), cell=_np(md.static["_cell"]).reshape(-1, 3, 3),
                               md_cell=None if md.cell is None else _np(md.cell), x=_np(md.positions)))
    return frames


def _rdf_reference(rdf, frames, n_atoms, n_beads=1):
    """sum over frames and beads of V counts and of V amb, per system of the batch (one system here)"""
    slot_of, total = _tables(rdf)
    types = np.array([rdf.species.index(int(z)) for z in rdf._md.static["_atomic_numbers"][:n_atoms].tolist()])
    acc = np.zeros((len(rdf.pairs), rdf.n_bins))
    amb = np.zeros_like(acc)
    vol = 0.0
    for f in frames:
        for r in range(n_beads):
            R = f["R"][r * n_atoms:(r + 1) * n_atoms]
            cell = f["cell"][r if f["cell"].shape[0] > 1 else 0]
            V = abs(np.linalg.det(f["md_cell"][r])) if f["md_cell"] is not None else abs(np.linalg.det(cell))
            c, a = SO.rdf_counts(R, cell, types, slot_of, total, len(rdf.pairs), rdf.r_max, rdf.n_bins)
            acc += V * c
            amb += V * a
            vol += V
    return acc, amb, vol


def _check_rdf(rdf, frames, n_atoms, n_beads=1):
    acc, amb, vol = _rdf_reference(rdf, frames, n_atoms, n_beads)
    got = _np(rdf._acc)[0]
    assert rdf.frames == len(frames)
    assert np.all(np.abs(got - acc) <= amb + 1e-9 * np.abs(acc)), np.abs(got - acc - amb).max()
    assert got.sum() > 0 and amb.sum() <= 1e-2 * acc.sum()         # 2e-5 x (bin index) of the pairs lie near an edge
    assert np.isclose(_np(rdf._volume)[0], vol, rtol=1e-12)
    na, nb = rdf._na.numpy()[0], rdf._nb.numpy()[0]
    r, g = rdf.result()
    ref = SO.rdf_from_sums(acc, len(frames) * n_beads, na, nb, rdf.r_max)
    tol = SO.rdf_from_sums(amb, len(frames) * n_beads, na, nb, rdf.r_max) + 1e-9 * np.abs(ref)
    assert np.all(np.abs(g[0].numpy() - ref) <= tol)
    n = rdf.coordination()[0].numpy()
    assert np.allclose(n, SO.coordination_from_sums(acc[None], np.array([vol]), na[None])[0], rtol=1e-9,
                       atol=SO.coordination_from_sums(amb[None], np.array([vol]), na[None])[0].max() + 1e-12)


def _check_msd(msd, frames, masses, species, cells, pbc, n_beads=1):
    N = species.shape[0]
    traj = np.stack([f["x"].reshape(n_beads, N, 3).mean(0) for f in frames])
    acc, count, jump = SO.msd_oracle(traj, cells, pbc, masses, species, [0, N], len(msd.species), msd.n_lags,
                                     msd.origin_every, msd.remove_com)
    assert not jump and int(msd._meta[1]) == 0
    assert msd.samples == len(frames)
    assert np.array_equal(msd._count.cpu().numpy(), count)
    np.testing.assert_allclose(_np(msd._acc), acc, rtol=1e-9, atol=1e-12 * max(acc.max(), 1.0))
    t, m = msd.result()
    live = count > 0
    np.testing.assert_allclose(m.numpy()[..., live], (acc / np.maximum(count, 1))[..., live]
                               / np.array([[(species == s).sum() for s in range(len(msd.species))]])[..., None],
                               rtol=1e-9, atol=1e-12)
    from schnetpack_b200.md import FS_MD

    np.testing.assert_allclose(t.numpy(), np.arange(msd.n_lags) * msd.every_n_steps * msd._md.dt / FS_MD, rtol=1e-12)


def _z(md, n):
    return md.static["_atomic_numbers"][:n].cpu().numpy()


def test_triclinic_box_several_species_sparse_sampling():
    """NVT (Langevin) in a triclinic box of three species: RDF every 3 steps at r_max beyond half the cell width
    (self-images counted), MSD every 2 steps with origins every 3 samples"""
    from schnetpack_b200 import md as M
    from schnetpack_b200.structure import MeanSquaredDisplacement, RadialDistribution

    rdf = RadialDistribution(r_max=7.5, n_bins=150, every_n_steps=3)
    msd = MeanSquaredDisplacement(n_lags=7, every_n_steps=2, origin_every=3)
    md = _md([rdf, msd], thermostat=M.LangevinThermostat(300.0, 20.0, seed=9, kB=KB))
    cell = md.static["_cell"].reshape(3, 3).cpu().numpy()
    assert 7.5 > 0.5 * SO.heights(cell.astype(np.float64)).min()
    assert rdf.pairs == [(1, 1), (1, 6), (1, 8), (6, 6), (6, 8), (8, 8), (0, 0)]
    frames = _trace(md, 13, 1)
    _check_rdf(rdf, frames[::3], md.positions.shape[0])
    N = md.positions.shape[0]
    z = _z(md, N)
    species = np.array([msd.species.index(int(v)) for v in z])
    masses = md.masses.cpu().numpy().astype(np.float64)
    cells = np.broadcast_to(cell.astype(np.float64), (len(frames[::2]), 1, 3, 3))
    _check_msd(msd, frames[::2], masses, species, cells, np.ones((1, 3), bool))


def test_npt_volume_enters_frame_by_frame():
    from schnetpack_b200 import md as M
    from schnetpack_b200.structure import MeanSquaredDisplacement, RadialDistribution

    rdf = RadialDistribution(r_max=6.0, n_bins=60, every_n_steps=2)
    msd = MeanSquaredDisplacement(n_lags=5, every_n_steps=2, origin_every=2)
    baro = M.NHCBarostatIsotropic(1.0, 300.0, 50.0, kB=KB)
    md = _md([rdf, msd], data=_box(n=300, triclinic=False), barostat=baro)
    v0 = float(md.volume()[0])
    frames = _trace(md, 12, 2)
    assert abs(float(md.volume()[0]) - v0) > 1e-6 * v0
    _check_rdf(rdf, frames, md.positions.shape[0])
    N = md.positions.shape[0]
    species = np.array([msd.species.index(int(v)) for v in _z(md, N)])
    cells = np.stack([f["md_cell"] for f in frames])
    _check_msd(msd, frames, md.masses.cpu().numpy().astype(np.float64), species, cells, np.ones((1, 3), bool))


def test_ring_polymer_bead_averaged_rdf_and_centroid_msd():
    from schnetpack_b200 import md as M
    from schnetpack_b200.structure import MeanSquaredDisplacement, RadialDistribution

    P = 3
    rdf = RadialDistribution(r_max=6.0, n_bins=60, every_n_steps=2, pairs=[(8, 1), (0, 0)])
    msd = MeanSquaredDisplacement(n_lags=6, every_n_steps=1, origin_every=2)
    md = _md([rdf, msd], ring_polymer=M.RingPolymer(P, 300.0, kB=KB, hbar=0.05),
             thermostat=M.PILELocalThermostat(300.0, 20.0, seed=3, kB=KB),
             initializer=M.MaxwellBoltzmannInit(300.0, seed=2, kB=KB))
    N = md.positions.shape[0] // P
    frames = _trace(md, 9, 1)
    _check_rdf(rdf, frames[::2], N, n_beads=P)
    species = np.array([msd.species.index(int(v)) for v in _z(md, N)])
    cell = md.static["_cell"].reshape(-1, 3, 3)[0].cpu().numpy().astype(np.float64)
    cells = np.broadcast_to(cell, (len(frames), 1, 3, 3))
    _check_msd(msd, frames, md.masses[:N].cpu().numpy().astype(np.float64), species, cells, np.ones((1, 3), bool),
               n_beads=P)


def test_wrapping_does_not_change_the_msd():
    """atoms scattered a few cells away, with and without WrapPositions(1) (which moves them back at once): the MSDs
    agree within the fp32 round-off of the positions, delta = 64 eps32 max|x| per atom, |dm| <= 2 sqrt(m) delta + delta^2"""
    from schnetpack_b200 import md as M
    from schnetpack_b200.structure import MeanSquaredDisplacement

    def run(wrap):
        msd = MeanSquaredDisplacement(n_lags=10, every_n_steps=1, origin_every=2, remove_com=False)
        md = _md(([M.WrapPositions(1)] if wrap else []) + [msd], data=_box(scatter=True), momenta_seed=6, speed=3.0)
        md.run(20)
        torch.cuda.synchronize()
        return msd, md

    (a, ma), (b, mb) = run(True), run(False)
    assert np.abs(_np(ma.positions) - _np(mb.positions)).max() > 1.0          # something was wrapped
    _, m_wrapped = a.result()
    _, m_free = b.result()
    m = m_free.numpy()
    assert np.nanmax(m) > 1e-3
    delta = 64 * 2.0 ** -24 * np.abs(_np(mb.positions)).max()
    live = np.isfinite(m)
    assert np.all(np.abs(m_wrapped.numpy() - m)[live] <= (2 * np.sqrt(m) * delta + delta ** 2)[live])


def _accumulators(md):
    return {k: v.clone() for k, v in _flat(md._step_state()["hooks"]).items()}


def _flat(d, prefix=""):
    out = {}
    for k, v in d.items():
        if isinstance(v, dict):
            out.update(_flat(v, prefix + k + "."))
        else:
            out[prefix + k] = v
    return out


def _hooks():
    from schnetpack_b200 import md as M
    from schnetpack_b200.structure import MeanSquaredDisplacement, RadialDistribution

    return [M.WrapPositions(2), RadialDistribution(7.0, 70, every_n_steps=2),
            MeanSquaredDisplacement(8, every_n_steps=1, origin_every=3)]


def _nvt(use_graph=True):
    from schnetpack_b200 import md as M

    return _md(_hooks(), use_graph=use_graph, thermostat=M.LangevinThermostat(300.0, 20.0, seed=9, kB=KB),
               initializer=M.MaxwellBoltzmannInit(300.0, seed=4, kB=KB))


def test_replay_equals_eager_and_runs_repeat_bitwise():
    g, e, g2 = _nvt(True), _nvt(False), _nvt(True)
    for md in (g, e, g2):
        md.run(7)
        md.run(6)
    torch.cuda.synchronize()
    A, B, C = _accumulators(g), _accumulators(e), _accumulators(g2)
    for k in A:
        assert torch.equal(A[k], B[k]), k
        assert torch.equal(A[k], C[k]), k
    assert float(A["1.acc"].sum()) > 0 and float(A["2.acc"].sum()) > 0


def test_restart_continues_bitwise():
    a = _nvt()
    a.run(9)
    sd = a.state_dict()
    a.run(8)
    b = _nvt()
    b.load_state_dict(sd)
    b.run(8)
    torch.cuda.synchronize()
    A, B = _accumulators(a), _accumulators(b)
    for k in A:
        assert torch.equal(A[k], B[k]), k
    # drain leaves the accumulators alone; reset zeroes them
    b.drain()
    assert torch.equal(_accumulators(b)["1.acc"], A["1.acc"])
    b.hooks[1].reset()
    b.hooks[2].reset()
    assert all(float(v.abs().sum()) == 0 for k, v in _accumulators(b).items())


def test_rdf_refuses_open_systems():
    from schnetpack_b200.structure import MeanSquaredDisplacement, RadialDistribution

    data = _box(pbc=False)
    with pytest.raises(ValueError, match="periodic"):
        _md([RadialDistribution(6.0, 60)], data=data)
    msd = MeanSquaredDisplacement(4, every_n_steps=1)            # the MSD works on open systems
    md = _md([msd], data=_box(pbc=False))
    md.run(5)
    t, m = msd.result()
    assert torch.isfinite(m).all() and float(m[..., 1:].min()) > 0


def test_jump_of_more_than_half_a_cell_is_reported():
    from schnetpack_b200.structure import MeanSquaredDisplacement

    msd = MeanSquaredDisplacement(4, every_n_steps=1)
    md = _md([msd], data=_box(triclinic=False))
    md.run(2)
    cell = md.static["_cell"].reshape(3, 3)
    with torch.no_grad():
        md.positions[0] += 0.45 * cell.sum(0)                  # minimum image 0.78 L long: more than L / 2
    with pytest.raises(RuntimeError, match="half the shortest cell height"):
        md.run(1)
