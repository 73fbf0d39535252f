"""GPU checks of the device phonons (schnetpack_b200.phonons, csrc/phonons.cu): force constants against the fixture's fp64
finite differences and analytic Hessian (tests/golden/make_golden_phonons.py), the commensurate identity with
DeviceVibrations on the same supercells, dynamical matrices, DOS and thermodynamics against tests/phonon_oracle.py, the
acoustic sum rule, invariance under translation and rotation, ragged batches, the bitwise invariants of the chunked
captured step, and the refusals."""
import json
import os

import numpy as np
import pytest
import torch

import phonon_oracle as O
from schnetpack_b200 import properties as P
from schnetpack_b200.model import from_spec
from schnetpack_b200.phonons import DevicePhonons, monkhorst_pack
from schnetpack_b200.vibrations import DeviceVibrations

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FCC_M = [[-1, 1, 1], [1, -1, 1], [1, 1, -1]]
# fp32 force noise over the step, as in DeviceVibrations (DESIGN.md section 16): relative to the largest element
NOISE_BOUND = 5e-5
TRUNC_BOUND = 5e-2                 # tests/test_phonon_oracle.py


def _golden():
    z = np.load(os.path.join(GOLDEN, "phonons_cscl.npz"))
    spec = json.loads(str(z["spec_json"]))
    params = {k[6:]: z[k] for k in z.files if k.startswith("param:")}
    return z, spec, from_spec(spec, params, DEV)


def _crystal(pos, cell, z):
    n = len(z)
    return {P.Z: torch.tensor(z, device=DEV), P.R: torch.tensor(np.asarray(pos, np.float32), device=DEV),
            P.cell: torch.tensor(np.asarray(cell, np.float32)[None], device=DEV),
            P.pbc: torch.ones(1, 3, dtype=torch.bool, device=DEV), P.idx_m: torch.zeros(n, dtype=torch.int64, device=DEV),
            P.n_atoms: torch.tensor([n], device=DEV)}


def _collate(*crystals):
    out = {}
    for m, c in enumerate(crystals):
        c = dict(c, **{P.idx_m: c[P.idx_m] + m})
        for k, v in c.items():
            out.setdefault(k, []).append(v)
    return {k: torch.cat(v) for k, v in out.items()}


def _cscl(z):
    return _crystal(z["in:_positions"], z["in:_cell"][0], [6, 8])


def _fcc():
    a = 3.9
    cell = 0.5 * a * np.array([[0.0, 1, 1], [1, 0, 1], [1, 1, 0]])
    return _crystal([[0.0, 0, 0], [0.27 * a, 0.22 * a, 0.31 * a]], cell, [6, 8])


def _ph(model, batch, supercell, masses=None, **kw):
    n = batch[P.R].shape[0]
    masses = masses if masses is not None else torch.tensor([12.011, 15.999] * (n // 2) + [12.011] * (n % 2))
    L = abs(round(float(np.linalg.det(np.diag(supercell) if np.ndim(supercell) == 1 else np.asarray(supercell)))))
    ph = DevicePhonons(model, batch, masses, supercell, cutoff=4.0, capacity=n * L * 128, **kw)
    ph.run()
    return ph


def _rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return float(np.abs(a - b).max() / np.abs(b).max())


def test_force_constants_against_fixture():
    z, spec, model = _golden()
    ph = _ph(model, _cscl(z), [3, 3, 3], symmetrize=0, acoustic=False)
    assert np.array_equal(ph.supercell_batch[P.R].cpu().numpy(), z["super_positions"])
    got = ph.force_constants.cpu().numpy()
    noise = _rel(got, O.fc_from_displaced(z["fd2:steps"], z["fd2:forces"]))
    trunc = _rel(got, z["ref64:force_constants"])
    print(f"cscl: |FC - FC_fd| / max = {noise:.3e}, |FC - FC_analytic| / max = {trunc:.3e}")
    assert noise <= NOISE_BOUND and trunc <= TRUNC_BOUND


@pytest.mark.parametrize("case", ["cscl_333", "fcc_nondiagonal"])
def test_commensurate_identity_with_device_vibrations(case):
    z, spec, model = _golden()
    batch, s = (_cscl(z), [3, 3, 3]) if case == "cscl_333" else (_fcc(), FCC_M)
    ph = _ph(model, batch, s, symmetrize=0, acoustic=False)
    sb = ph.supercell_batch
    n_super = sb[P.R].shape[0]
    masses = torch.tensor([12.011, 15.999] * (n_super // 2))
    vib = DeviceVibrations(model, sb, masses, cutoff=4.0, capacity=n_super * 128)
    vib.run()
    w_vib = np.sort(np.linalg.eigvalsh(vib.hessian_mw.view(3 * n_super, 3 * n_super).cpu().numpy()))
    M = np.asarray(O.supercell_matrix(s))
    g, _ = O.translations(M.T)                   # q = M^-1 g: M q integer, one q per class of g modulo M Z^3
    q = np.array([np.linalg.solve(M.astype(float), v) for v in g.astype(float)])
    q = q - np.floor(q + 0.5)
    D = torch.cat(ph.dynamical_matrices(q)).cpu().numpy()
    w_ph = np.sort(np.concatenate([np.linalg.eigvalsh(0.5 * (d + d.conj().T)) for d in D]))
    err = np.abs(w_ph - w_vib).max() / np.abs(w_vib).max()
    print(f"{case}: L = {len(q)}, |eig(D(q)) - eig(H_super)| / max = {err:.3e}")
    assert err <= NOISE_BOUND


def _oracle_dynmat(ph, m, q):
    lo, hi = int(ph.prim_ptr[m]), int(ph.prim_ptr[m + 1])
    n, L = hi - lo, ph.n_cells
    rows = slice(int(ph.fc_ptr[m]), int(ph.fc_ptr[m + 1]))
    img = O.images(ph.positions64[lo:hi].cpu().numpy(), ph.cell64[m].cpu().numpy(), ph.supercell,
                   ph.lattice.cpu().numpy(), 1e-5)
    cnt = ph.img_count[rows].cpu().numpy()
    assert np.array_equal(cnt, [c for c, _ in img])
    fc = ph.force_constants[rows].cpu().numpy()
    return np.array([O.dynmat(fc, img, ph.masses[lo:hi].cpu().numpy(), qq) for qq in q]), n, L


@pytest.mark.parametrize("case", ["cscl_333", "cscl_222_ties", "fcc_nondiagonal", "skewed"])
def test_dynamical_matrices_against_oracle(case):
    z, spec, model = _golden()
    if case == "skewed":
        cell = np.array([[2.9, 0.0, 0.0], [2.2, 2.1, 0.0], [1.7, 0.9, 2.4]])
        batch, s = _crystal([[0.0, 0, 0], [1.9, 1.0, 1.1]], cell, [6, 8]), [[2, 1, 0], [0, 2, 1], [1, 0, 2]]
    elif case == "fcc_nondiagonal":
        batch, s = _fcc(), FCC_M
    else:
        batch, s = _cscl(z), [3, 3, 3] if case == "cscl_333" else [2, 2, 2]
    ph = _ph(model, batch, s, acoustic=False)      # one symmetrisation: Phi exactly symmetric, so D(q) is Hermitian
    q = np.random.default_rng(3).uniform(-0.5, 0.5, (5, 3))
    want, n, L = _oracle_dynmat(ph, 0, q)
    got = ph.dynamical_matrices(q)[0].cpu().numpy()
    err = _rel(got, want)
    herm = np.abs(got - got.conj().transpose(0, 2, 1)).max() / np.abs(got).max()
    print(f"{case}: L = {L}, ties {int((ph.img_count > 1).sum())}, |D - D_oracle| / max = {err:.2e}, "
          f"|D - D^H| / max = {herm:.2e}")
    if case == "cscl_222_ties":
        assert int(ph.img_count.max()) == 8
    assert err <= 1e-12 and herm <= 1e-12


def test_acoustic_sum_rule_at_gamma():
    """the fixture crystal is not at a minimum of the random model (it has two imaginary optical modes at Gamma), so the
    acoustic modes are the three of smallest |omega|"""
    z, spec, model = _golden()
    f_asr = _ph(model, _cscl(z), [3, 3, 3]).frequencies([0, 0, 0]).cpu().numpy()[0]
    f_raw = _ph(model, _cscl(z), [3, 3, 3], symmetrize=0, acoustic=False).frequencies([0, 0, 0]).cpu().numpy()[0]
    a_asr, a_raw = np.sort(np.abs(f_asr))[:3], np.sort(np.abs(f_raw))[:3]
    print(f"Gamma: all modes {f_asr}; acoustic |omega| with the sum rule {a_asr}, raw {a_raw} cm^-1")
    assert a_asr.max() <= ACOUSTIC_BOUND and a_raw.max() <= RAW_ACOUSTIC_BOUND
    assert a_asr.max() < a_raw.max()
    assert np.all(np.diff(f_asr) >= 0)


# |omega| of the three acoustic modes at Gamma, cm^-1 (DESIGN.md section 23; the fp64 oracle on the fixture's reference
# finite differences gives 0.36 with the sum rule and 0.95 without)
ACOUSTIC_BOUND = 1.0
RAW_ACOUSTIC_BOUND = 5.0


def _rotation():
    a, b = 0.7, -0.4
    rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    rx = np.array([[1, 0, 0], [0, np.cos(b), -np.sin(b)], [0, np.sin(b), np.cos(b)]])
    return rz @ rx


def test_translation_and_rotation_invariance():
    z, spec, model = _golden()
    pos, cell = z["in:_positions"].astype(np.float64), z["in:_cell"][0].astype(np.float64)
    q = np.random.default_rng(4).uniform(-0.5, 0.5, (6, 3))
    base = _ph(model, _crystal(pos, cell, [6, 8]), [3, 3, 3]).frequencies(q).cpu().numpy()
    R = _rotation()
    moved = _ph(model, _crystal(pos + [0.37, -0.21, 0.55], cell, [6, 8]), [3, 3, 3]).frequencies(q).cpu().numpy()
    turned = _ph(model, _crystal(pos @ R.T, cell @ R.T, [6, 8]), [3, 3, 3]).frequencies(q).cpu().numpy()
    e1, e2 = np.abs(moved - base).max(), np.abs(turned - base).max()
    print(f"translation {e1:.3e}, rotation {e2:.3e} cm^-1 (largest {np.abs(base).max():.1f})")
    assert e1 <= TRANSLATION_BOUND and e2 <= ROTATION_BOUND * np.abs(base).max()


# A translation changes only the fp32 rounding of the positions, so the frequencies move by the force noise (cm^-1).  A
# rotation also turns the directions of the finite differences, so they move by the O(h^2) truncation, which is 3e-2 of
# the force constants for this off-equilibrium crystal and half of that in frequency: relative to the largest |omega|.
TRANSLATION_BOUND = 0.05
ROTATION_BOUND = 0.5 * TRUNC_BOUND


def test_ragged_batch_equals_separate_runs():
    z, spec, model = _golden()
    one = _crystal([[0.0, 0.0, 0.0]], 2.6 * np.eye(3), [6])
    two = _cscl(z)
    both = _ph(model, _collate(two, one), [3, 3, 3], masses=torch.tensor([12.011, 15.999, 12.011]))
    a = _ph(model, two, [3, 3, 3])
    b = _ph(model, one, [3, 3, 3], masses=torch.tensor([12.011]))
    fc = both.force_constants.cpu().numpy()
    na = a.force_constants.shape[0]
    ea, eb = _rel(fc[:na], a.force_constants.cpu().numpy()), _rel(fc[na:], b.force_constants.cpu().numpy())
    q = np.random.default_rng(5).uniform(-0.5, 0.5, (4, 3))
    f = both.frequencies(q).cpu().numpy()
    ef = max(np.abs(f[:, :6] - a.frequencies(q).cpu().numpy()).max(), np.abs(f[:, 6:] - b.frequencies(q).cpu().numpy()).max())
    print(f"ragged: force constants {ea:.2e} / {eb:.2e}, frequencies {ef:.2e} cm^-1")
    assert ea <= 1e-6 and eb <= 1e-6 and ef <= 1e-3


def test_bitwise_chunks_graph_and_repeat():
    z, spec, model = _golden()
    one = _ph(model, _cscl(z), [3, 3, 3])
    chunked = _ph(model, _cscl(z), [3, 3, 3], max_replica_atoms=2 * 54)
    eager = _ph(model, _cscl(z), [3, 3, 3], max_replica_atoms=2 * 54, use_graph=False)
    assert one.n_chunks == 1 and chunked.n_chunks == 6
    assert torch.equal(one.force_constants, chunked.force_constants)
    assert torch.equal(chunked.force_constants, eager.force_constants)
    fc = one.force_constants.clone()
    one.run()
    assert torch.equal(fc, one.force_constants)
    q = monkhorst_pack([3, 3, 3])
    assert torch.equal(one.frequencies(q), chunked.frequencies(q))


def test_dos_and_thermodynamics_against_oracle():
    z, spec, model = _golden()
    ph = _ph(model, _collate(_cscl(z), _fcc()), [3, 3, 3])
    mesh = [6, 6, 6]
    freq = ph.frequencies(monkhorst_pack(mesh)).cpu().numpy()
    grid = np.linspace(freq.min() - 100.0, freq.max() + 100.0, 4001)        # imaginary modes included
    g = ph.dos(mesh, grid, 8.0).cpu().numpy()
    T = np.array([0.0, 5.0, 77.0, 300.0, 1500.0])
    th = {k: v.cpu().numpy() for k, v in ph.thermodynamics(mesh, T).items()}
    for m in range(2):
        fm = freq[:, 6 * m:6 * (m + 1)]
        want = O.dos(fm, grid, 8.0)
        assert _rel(g[m], want) <= 1e-12
        integral = np.trapezoid(g[m], grid)
        zpe, F, S, C, nx, ni = O.thermo(fm, T)
        print(f"system {m}: int g = {integral:.6f}, zpe {zpe:.6f} eV, excluded {nx}, imaginary {ni}")
        assert abs(integral - 6.0) <= 1e-6
        assert abs(th["zero_point_energy"][m] - zpe) <= 1e-12 * abs(zpe)
        for key, ref in (("free_energy", F), ("entropy", S), ("heat_capacity", C)):
            assert np.abs(th[key][:, m] - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1e-30), key
        assert th["n_excluded"][m] == nx and th["n_imaginary"][m] == ni


def test_refusals():
    z, spec, model = _golden()
    c = _cscl(z)
    masses = torch.tensor([12.011, 15.999])
    kw = dict(cutoff=4.0, capacity=10000)
    with pytest.raises(ValueError, match="periodic"):
        DevicePhonons(model, dict(c, **{P.pbc: torch.tensor([[True, True, False]], device=DEV)}), masses, [3, 3, 3], **kw)
    with pytest.raises(ValueError, match="det > 0"):
        DevicePhonons(model, c, masses, [[0, 1, 0], [1, 0, 0], [0, 0, 1]], **kw)
    with pytest.raises(ValueError, match="integer"):
        DevicePhonons(model, c, masses, [2, 2.5, 2], **kw)
    with pytest.raises(ValueError, match="masses"):
        DevicePhonons(model, c, masses[:1], [3, 3, 3], **kw)
    with pytest.raises(NotImplementedError, match="ensembles"):
        DevicePhonons([model, model], c, masses, [3, 3, 3], **kw)
    from schnetpack_b200.parallel import PartitionedPotential

    with pytest.raises(NotImplementedError, match="PartitionedPotential"):
        DevicePhonons(PartitionedPotential.__new__(PartitionedPotential), c, masses, [3, 3, 3], **kw)
