"""GPU checks of the climbing-image NEB (schnetpack_b200.neb, csrc/neb.cu): the kernels against the fp64 oracle of
tests/neb_oracle.py on ragged batches of bands fed analytic Morse forces, a vacancy hop across a periodic face, DeviceNEB
with the trained PaiNN ethanol model against a host-driven oracle, the methyl rotation of ethanol as a real saddle checked
by the device vibrational analysis, the bitwise invariants of the captured step, ensembles and the refusals."""
import numpy as np
import pytest
import torch

from conftest import load_case
from fire_oracle import fcc, morse, pair_list, pair_list_orthorhombic
from neb_oracle import NEBOracle, neb_forces
from schnetpack_b200 import properties as P
from schnetpack_b200.model import from_spec
from schnetpack_b200.neb import DeviceNEB, NEBState, interpolate
from schnetpack_b200.neighbors import CellListNeighborList
from schnetpack_b200.relax import DeviceFIRE, FIREState

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
MORSE = dict(rc=2.2)
REACH = 2.6


def _np(t):
    return t.detach().double().cpu().numpy()


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


# ---- the kernels alone, fed Morse forces -------------------------------------------------------------------------------
class _MorseBands:
    """Periodic Morse bands: 1 atom (translation-invariant, so every energy is equal and every tangent is the bisector),
    13 atoms (fcc with vacancies), 300 atoms and, with ``big``, 20 400 atoms (images that straddle CTAs of 256 atoms).
    Each image gets its own pair list, built at its starting positions with a skin (REACH > rc)."""

    def __init__(self, n_images, big, seed=3):
        rng = np.random.default_rng(seed)
        shear = np.eye(3) + np.array([[0.0, 0.05, -0.03], [0.02, 0.0, 0.04], [0.0, -0.03, 0.0]])
        systems = [(np.zeros((1, 3)), 1.25 * np.eye(3) @ shear)]
        x, cell = fcc(1.62, (2, 2, 1))
        systems.append((np.delete(x, [2, 9, 14], axis=0) @ shear, cell @ shear))
        x, cell = fcc(1.62, (5, 5, 3))
        systems.append((x @ shear, cell @ shear))
        if big:
            systems.append(fcc(1.62, (10, 10, 51)))
        self.n, self.sizes, self.cells = n_images, [len(s[0]) for s in systems], [s[1] for s in systems]
        x0, x1 = [], []
        for k, (x, _) in enumerate(systems):
            if k == 0:
                x0.append(x)
                x1.append(x + np.array([[0.3, 0.1, 0.2]]))
                continue
            x0.append(x + rng.normal(scale=0.05, size=x.shape))
            x1.append(x + rng.normal(scale=0.05, size=x.shape))
        self.x0, self.x1 = np.concatenate(x0), np.concatenate(x1)
        self.eptr = np.concatenate([[0], np.cumsum(self.sizes)])
        # interior images, band-major, image-major
        rows = []
        for b in range(len(self.sizes)):
            a0, a1 = x0[b], x1[b]
            rows += [a0 + (j / (n_images + 1)) * (a1 - a0) for j in range(1, n_images + 1)]
        self.x = np.concatenate(rows)
        self.pairs = [self._pairs(b, img) for b in range(len(self.sizes)) for img in self._images(self.x, b)]
        self.end_pairs = [(self._pairs(b, x0[b]), self._pairs(b, x1[b])) for b in range(len(self.sizes))]
        self.end_energies = np.array([[morse(x0[b], self.cells[b], p0, **MORSE)[0],
                                       morse(x1[b], self.cells[b], p1, **MORSE)[0]]
                                      for b, (p0, p1) in enumerate(self.end_pairs)])
        # the 1-atom band's energy does not depend on where the atom is; pin it so that rounding cannot break the tie
        self.end_energies[0] = float(np.float32(self.end_energies[0, 0]))

    def _pairs(self, b, x):
        cell = self.cells[b]
        return pair_list_orthorhombic(x, np.diag(cell), REACH) if len(x) > 1000 else pair_list(x, cell, REACH)

    def _images(self, x, b):
        p0 = self.n * self.eptr[b]
        return [x[p0 + j * self.sizes[b]:p0 + (j + 1) * self.sizes[b]] for j in range(self.n)]

    def evaluate(self, x):
        """fp32 forces [N, 3] and energies [n_img] of the interior images x"""
        f, e, k = np.zeros_like(x), [], 0
        for b in range(len(self.sizes)):
            p0 = self.n * self.eptr[b]
            for j, xi in enumerate(self._images(x, b)):
                ei, fi, _ = morse(xi, self.cells[b], self.pairs[k], **MORSE)
                f[p0 + j * self.sizes[b]:p0 + (j + 1) * self.sizes[b]] = fi
                e.append(ei)
                k += 1
        f[:self.n], e[:self.n] = 0.0, [self.end_energies[0, 0]] * self.n          # the 1-atom band: flat
        return f.astype(np.float32), np.array(e, dtype=np.float32)

    def fixed(self):
        m = np.zeros(len(self.x), dtype=bool)
        p = self.n * self.eptr
        m[[p[1] + 2, p[2] + 5, p[3] - 7]] = True        # in the 13- and 300-atom bands
        if len(self.sizes) > 3:
            m[p[3] + 20_100] = True
        return m

    def states(self, k=0.5, climb=False, fixed=None, **fire):
        st = FIREState(torch.as_tensor(self.x, device=DEV), self._band_index(), len(self.sizes), fmax=1e-12, **fire)
        neb = NEBState(st.r, torch.as_tensor(self.x0, device=DEV), torch.as_tensor(self.x1, device=DEV),
                       torch.as_tensor(self.end_energies, device=DEV), self.sizes, self.n, k=k, climb=climb,
                       fixed_atoms_mask=fixed)
        return st, neb

    def _band_index(self):
        return torch.repeat_interleave(torch.arange(len(self.sizes)), torch.as_tensor(self.sizes) * self.n).to(DEV)


def _branch(coef):
    """tangent branch of every image: 0 up, 1 down, 2 extremum, 3 bisector"""
    a, b = coef[:, 0], coef[:, 1]
    out = np.full(len(a), 2)
    out[(a == 1.0) & (b == 0.0)] = 0
    out[(a == 0.0) & (b == 1.0)] = 1
    return out


def _check_kernels(bands, neb, x, f, e, k, climb, fixed):
    """one spk_neb_forces call against the oracle at the same positions, forces and energies.  Each quantity is compared
    on the scale of the terms that enter it (|F| |D|, k |D|), since its own value may be a small difference of them."""
    out = _np(neb.forces(torch.as_tensor(f, device=DEV), torch.as_tensor(e, device=DEV)))
    f64 = f.astype(np.float64)
    f64[fixed] = 0.0
    want, coef, diag, climbing = neb_forces(x, bands.x0, bands.x1, f64, e.astype(np.float64), bands.end_energies,
                                            bands.sizes, bands.n, k, climb, fixed)
    img = np.repeat(np.arange(len(coef)), np.repeat(bands.sizes, bands.n))
    fn = np.sqrt(np.bincount(img, weights=(f64 ** 2).sum(1), minlength=len(coef)))
    alpha, beta, dp, dm, tn = coef[:, 0], coef[:, 1], diag[:, 3], diag[:, 4], diag[:, 0]
    tau_scale = alpha * dp + beta * dm
    got_c, got_d = _np(neb.coef), _np(neb.diag)
    assert _rel(got_c[:, :2], coef[:, :2]) <= 1e-12
    gamma_scale = np.where(tn > 0, fn * tau_scale / np.maximum(tn, 1e-300) ** 2 + k * (dp + dm) / np.maximum(tn, 1e-300),
                           0.0)
    assert np.all(np.abs(got_c[:, 2] - coef[:, 2]) <= 1e-12 * gamma_scale + 1e-300)
    scales = [tau_scale, fn, k * (dp + dm), dp, dm]
    for c, scale in enumerate(scales):
        assert np.all(np.abs(got_d[:, c] - diag[:, c]) <= 1e-12 * scale + 1e-300), c
    assert np.array_equal(got_d[:, 5], diag[:, 5])
    assert neb.climbing.cpu().tolist() == climbing.tolist()
    atom_scale = (fn + k * (dp + dm))[img][:, None]
    assert np.all(np.abs(out - want) <= 2.0 ** -24 * np.abs(want) + 1e-12 * atom_scale)
    assert np.all(out[fixed] == 0.0)
    return coef


@pytest.mark.parametrize("n_images", [1, 3, 7])
def test_kernels_follow_the_oracle_on_ragged_bands(n_images):
    """the NEB kernels against the oracle on bands of 1, 13, 300 and 20 400 atoms with fixed atoms, climb off and on"""
    bands = _MorseBands(n_images, big=True)
    fixed = bands.fixed()
    branches = set()
    for climb in (False, True):
        st, neb = bands.states(climb=climb, fixed=fixed)
        x = _np(st.r)
        f, e = bands.evaluate(x)
        coef = _check_kernels(bands, neb, x, f, e, 0.5, climb, fixed)
        branches |= set(_branch(coef).tolist())
        # a step later, from moved positions
        st.check(neb.neb_forces)
        st.step()
        x = _np(st.r)
        f, e = bands.evaluate(x)
        _check_kernels(bands, neb, x, f, e, 0.5, climb, fixed)
    flat = np.arange(n_images)                                   # the 1-atom band's images: the bisector
    assert np.all(np.isclose(coef[flat, 0], 1.0 / np.linalg.norm(bands.x1[0] - bands.x0[0]) * (n_images + 1)))
    assert {2} <= branches


@pytest.mark.parametrize("n_images", [1, 3, 7])
def test_state_follows_the_oracle_for_60_steps(n_images):
    """NEBState + FIREState against NEBOracle for 60 steps (bands of 1, 13 and 300 atoms, fixed atoms, climbing turned
    on after 30 steps); every tangent branch is met on the way"""
    bands = _MorseBands(n_images, big=False)
    fixed = bands.fixed()
    kw = dict(dt=0.05, maxstep=0.1, dtmax=0.2, Nmin=3)
    st, neb = bands.states(fixed=fixed, **kw)
    o = NEBOracle(bands.x, bands.x0, bands.x1, bands.end_energies, bands.sizes, n_images, k=0.5, fixed=fixed, **kw)
    branches = set()
    for step in range(60):
        if step == 30:
            neb.set_climb(True)
            o.climb = True
        f, e = bands.evaluate(o.positions)
        fneb = neb.forces(torch.as_tensor(f, device=DEV), torch.as_tensor(e, device=DEV))
        st.check(fneb)
        st.step()
        branches |= set(_branch(_np(neb.coef)).tolist())
        o.step(f.astype(np.float64), e.astype(np.float64), 1e-12)
        assert _rel(_np(st.r), o.positions) <= 1e-9, step
    assert np.array_equal(_np(st.r)[fixed], bands.x[fixed])
    assert int(neb.climbing[1]) >= 0 and torch.equal(st.model_positions, st.r.float())
    if n_images >= 3:
        assert branches == {0, 1, 2}, branches


# ---- a vacancy hop across the periodic face -----------------------------------------------------------------------------
def _relaxed(x, cell, fmax=1e-10):
    from scipy.optimize import minimize

    def fun(q):
        y = q.reshape(-1, 3)
        e, f, _ = morse(y, cell, pair_list(y, cell, REACH), **MORSE)
        return e, -f.reshape(-1)

    r = minimize(fun, x.reshape(-1), jac=True, method="BFGS", options=dict(gtol=fmax, maxiter=10_000))
    return r.x.reshape(-1, 3)


def test_vacancy_hop_across_the_periodic_face():
    """fcc Morse crystal (2 x 2 x 2 cells, 31 atoms): the atom at the origin's face neighbour hops into the vacancy
    across the periodic face.  The two relaxed endpoints are mirror images, so the barrier is symmetric and the saddle
    puts the hopping atom at the midpoint of the two sites."""
    x, cell = fcc(1.62, (2, 2, 2))
    hop = int(np.argmin(np.linalg.norm(x - np.array([2.43, 2.43, 0.0]), axis=1))) - 1
    x_init = np.delete(x, 0, axis=0)                            # the vacancy at the origin
    x_final = x_init.copy()
    x_final[hop] = x[0]                                          # stored wrapped: only mic finds the short path
    a, b = _relaxed(x_init, cell), _relaxed(x_final, cell)
    mk = lambda y: {"_positions": torch.as_tensor(y, dtype=torch.float32, device=DEV),  # noqa: E731
                    "_atomic_numbers": torch.full((len(y),), 29, device=DEV), "_n_atoms": torch.tensor([len(y)]),
                    "_cell": torch.as_tensor(cell, dtype=torch.float32, device=DEV)[None],
                    "_pbc": torch.ones(1, 3, dtype=torch.bool, device=DEV)}
    n = 5
    images = interpolate(mk(a), mk(b), n, mic=True)
    L = cell[0, 0]
    x0, x1 = a, a + (b - a) - np.round((b - a) / L) * L          # the minimum image of every difference (cubic cell)
    d = x1[hop] - x0[hop]
    assert np.linalg.norm(d) < 1.3                               # the short path: one nearest-neighbour distance
    ends = [[morse(y, cell, pair_list(y, cell, REACH), **MORSE)[0] for y in (x0, x1)]]
    xi = images["_positions"].double().cpu().numpy()
    idx = torch.zeros(len(xi), dtype=torch.int64, device=DEV)
    st = FIREState(torch.as_tensor(xi, device=DEV), idx, 1, fmax=1e-4, maxstep=0.05)
    neb = NEBState(st.r, torch.as_tensor(x0, device=DEV), torch.as_tensor(x1, device=DEV),
                   torch.as_tensor(ends, device=DEV), [len(a)], n, k=1.0, climb=True)
    for _ in range(3000):
        x = _np(st.r)
        f, e = np.zeros_like(x), np.zeros(n)
        for j in range(n):
            y = x[j * len(a):(j + 1) * len(a)]
            e[j], f[j * len(a):(j + 1) * len(a)], _ = morse(y, cell, pair_list(y, cell, REACH), **MORSE)
        st.check(neb.forces(torch.as_tensor(f, dtype=torch.float32, device=DEV),
                            torch.as_tensor(e, dtype=torch.float32, device=DEV)))
        if int(st.n_unconverged.item()) == 0:
            break
        st.step()
    assert int(st.n_unconverged.item()) == 0
    top = int(neb.climbing[0])
    assert top == n // 2
    ci = _np(st.r)[top * len(a):(top + 1) * len(a)]
    assert np.abs(ci[hop] - (x0[hop] + 0.5 * d)).max() < 1e-3
    forward, backward = e[top] - ends[0][0], e[top] - ends[0][1]
    assert forward > 0.05 and abs(forward - backward) <= 1e-9 * forward


# ---- DeviceNEB with the trained PaiNN ethanol model ----------------------------------------------------------------------
def _ethanol():
    spec, params, inputs, _, _ = load_case("painn_md_ethanol_trained")
    return spec, params, from_spec(spec, params, DEV), inputs


def _molecules(inputs, shift_seed=None, scale=0.25):
    """the fixture's two molecules as an endpoint batch (optionally displaced at random)"""
    x = inputs["_positions"].astype(np.float64)
    if shift_seed is not None:
        x = x + np.random.default_rng(shift_seed).normal(scale=scale, size=x.shape)
    return {k: torch.as_tensor(v).to(DEV) for k, v in inputs.items() if k not in (P.idx_i, P.idx_j, P.offsets)} | {
        P.R: torch.as_tensor(x, dtype=torch.float32, device=DEV)}


def _one(batch, m):
    """system m of a 9-atom-per-system batch"""
    return {P.R: batch[P.R][9 * m:9 * m + 9], P.Z: batch[P.Z][9 * m:9 * m + 9], P.n_atoms: batch[P.n_atoms][m:m + 1],
            P.idx_m: torch.zeros(9, dtype=torch.int64, device=DEV), P.cell: batch[P.cell][m:m + 1],
            P.pbc: batch[P.pbc].reshape(-1, 3)[m:m + 1]}


def _neb(model, initial, final, spec, **kw):
    return DeviceNEB(model, initial, final, cutoff=spec["cutoff"], capacity=18 * 18, **kw)


class _EagerImages:
    """eager model evaluation of interior images (the batch layout of ``template``) at given positions"""

    def __init__(self, model, template, spec, p_conv=1.0):
        self.model, self.p_conv = model, p_conv
        self.batch = dict(template)
        n = int(template[P.R].shape[0])
        self.nl = CellListNeighborList(spec["cutoff"], capacity=n * n, pad=True)

    def __call__(self, r):
        x = dict(self.batch)
        x[P.R] = torch.as_tensor(r / self.p_conv, dtype=torch.float64, device=DEV).float()
        out = self.model(self.nl(x))
        return out["forces"].detach().double().cpu().numpy(), out["energy"].detach().double().cpu().numpy()


@pytest.mark.parametrize("p_conv,e_conv", [(1.0, 1.0), (0.5, 2.0)])
def test_device_neb_follows_the_host_driven_oracle(p_conv, e_conv):
    spec, _, model, inputs = _ethanol()
    initial, final = _molecules(inputs), _molecules(inputs, shift_seed=1)
    n = 3
    dev = _neb(model, initial, final, spec, n_images=n, k=0.5 * e_conv / p_conv ** 2, climb=True, maxstep=0.05 * p_conv,
               position_conversion=p_conv, energy_conversion=e_conv)
    images = interpolate(initial, final, n)
    ev = _EagerImages(model, images, spec, p_conv)
    ends = _EagerImages(model, interpolate(initial, final, 2), spec)        # (initial, final) of each band
    _, e_ends = ends(torch.cat([initial[P.R][:9], final[P.R][:9], initial[P.R][9:], final[P.R][9:]]).double().cpu()
                     .numpy())
    assert _rel(_np(dev.neb.end_energies).reshape(-1), e_ends * e_conv) <= 1e-6
    x0 = images[P.R].double().cpu().numpy() * p_conv
    o = NEBOracle(x0, _np(dev.neb.initial), _np(dev.neb.final), _np(dev.neb.end_energies), [9, 9], n,
                  k=0.5 * e_conv / p_conv ** 2, climb=True, maxstep=0.05 * p_conv)
    traj = []
    for _ in range(8):
        dev.run(fmax=1e-9, steps=1)
        traj.append(_np(dev.positions).copy())
    for k in range(8):
        f, e = ev(o.positions)
        o.step(f * e_conv / p_conv, e * e_conv, 1e-9)
        assert np.abs(traj[k] - o.positions).max() <= 1e-4 * p_conv, k
    assert np.abs(traj[-1] - x0).max() > 1e-2 * p_conv
    f, e = ev(o.positions)
    assert _rel(_np(dev.get_energies())[:, 1:-1].reshape(-1), e * e_conv) <= 1e-5
    assert dev.climbing_image.cpu().tolist() == o.forces(f * e_conv / p_conv, e * e_conv)[3].tolist()
    # the results' shapes and definitions
    path = dev.path()
    assert len(path) == 2 and path[0].shape == (n + 2, 9, 3)
    assert torch.equal(path[1][1:-1].reshape(-1, 3), dev.positions[27:])
    s = _np(dev.reaction_coordinate())
    assert s.shape == (2, n + 2) and np.all(np.diff(s, axis=1) > 0) and np.all(s[:, 0] == 0)
    fwd, bwd = (_np(t) for t in dev.barriers())
    energies = _np(dev.get_energies())
    np.testing.assert_allclose(fwd, energies[:, 1:-1].max(1) - energies[:, 0], rtol=1e-12)
    np.testing.assert_allclose(bwd, energies[:, 1:-1].max(1) - energies[:, -1], rtol=1e-12)
    assert dev.tangent_forces().shape == (2, n) and dev.get_forces().shape == (6 * 9, 3)


def _relaxed_ethanol(model, inputs, spec):
    """molecule 0 of the fixture relaxed by DeviceFIRE (the model's kcal/mol and Angstrom)"""
    one = _one(_molecules(inputs), 0)
    fire = DeviceFIRE(model, one, cutoff=spec["cutoff"], capacity=81)
    assert fire.run(fmax=0.01, steps=5000)
    return fire.positions.cpu().numpy()


def _rotate(x, atoms, axis_from, axis_to, angle):
    """x with ``atoms`` rotated rigidly by ``angle`` about the axis through x[axis_from], x[axis_to]"""
    from scipy.spatial.transform import Rotation

    u = x[axis_to] - x[axis_from]
    rot = Rotation.from_rotvec(angle * u / np.linalg.norm(u))
    y = x.copy()
    y[atoms] = rot.apply(x[atoms] - x[axis_from]) + x[axis_from]
    return y


def test_ethanol_methyl_rotation_is_a_first_order_saddle():
    """Methyl rotation of ethanol (atoms: 0 methyl C, 1 CH2 C, 2-4 methyl H): the relaxed molecule and the same positions
    with the methyl hydrogens relabelled cyclically are equivalent minima; rigid rotations of the methyl group are the
    starting images.  CI-NEB converges, the barriers are equal, and the Hessian at the climbing image has one clearly
    negative eigenvalue."""
    from schnetpack_b200.units import convert_units
    from schnetpack_b200.vibrations import DeviceVibrations

    spec, _, model, inputs = _ethanol()
    x = _relaxed_ethanol(model, inputs, spec)
    final = x.copy()
    final[[2, 3, 4]] = x[[3, 4, 2]]
    u = x[1] - x[0]
    u /= np.linalg.norm(u)
    p, q = x[2] - x[0], x[3] - x[0]
    p, q = p - (p @ u) * u, q - (q @ u) * u
    angle = np.arctan2(np.cross(p, q) @ u, p @ q)               # the rotation that takes H 2 to H 3's position
    n = 5
    images = np.concatenate([_rotate(x, [2, 3, 4], 0, 1, angle * j / (n + 1)) for j in range(1, n + 1)])
    base = _one(_molecules(inputs), 0)
    mk = lambda y: dict(base, _positions=torch.as_tensor(y, dtype=torch.float32, device=DEV))  # noqa: E731
    img_batch = interpolate(mk(x), mk(final), n) | {P.R: torch.as_tensor(images, dtype=torch.float32, device=DEV)}
    dev = _neb(model, mk(x), mk(final), spec, n_images=n, images=img_batch, k=1.0, climb=True, maxstep=0.05)
    assert abs(float(dev.neb.end_energies[0, 0] - dev.neb.end_energies[0, 1])) < 1e-3
    # measured on an H100 80GB HBM3: converged after 829 steps to fmax 0.02 kcal/mol/Angstrom, barriers 2.96211 /
    # 2.96210 kcal/mol; the budget is about 2.4 times that
    converged = dev.run(fmax=0.02, steps=2000)
    fwd, bwd = (float(t) for t in dev.barriers())
    print(f"methyl rotation: converged {converged} after {dev.nsteps} steps, fmax {float(dev.fmax[0]):.4f}, "
          f"barriers {fwd:.5f} / {bwd:.5f} kcal/mol, climbing image {int(dev.climbing_image[0])}")
    assert converged
    assert fwd > 0.5 and abs(fwd - bwd) <= 1e-3
    top = int(dev.climbing_image[0])
    ci = dev.positions[9 * top:9 * top + 9].float()
    z = np.load(__import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "vib_ethanol.npz"))
    vib = DeviceVibrations(model, dict(base, _positions=ci), torch.as_tensor(z["masses"][:9]), cutoff=spec["cutoff"],
                           capacity=81, energy_conversion=convert_units("kcal/mol", "eV"))
    vib.run()
    freq = vib.frequencies().cpu().numpy()
    print(f"methyl rotation saddle: frequencies {np.round(freq[:8], 1)} cm^-1")
    # measured: -245.5 cm^-1, then the rigid-body modes (-12.8 .. 0.8 cm^-1) and the real modes from 291 cm^-1 on
    assert freq[0] < -150.0 and np.all(freq[1:] > -40.0)


def test_two_bands_in_one_batch_match_each_band_alone():
    spec, _, model, inputs = _ethanol()
    initial, final = _molecules(inputs), _molecules(inputs, shift_seed=2)
    both = _neb(model, initial, final, spec, n_images=3, climb=True)
    both.run(fmax=1e-9, steps=20)
    worst = 0.0
    for m in range(2):
        alone = _neb(model, _one(initial, m), _one(final, m), spec, n_images=3, climb=True)
        alone.run(fmax=1e-9, steps=20)
        worst = max(worst, float((both.positions[27 * m:27 * m + 27] - alone.positions).abs().max()))
    print(f"two bands vs each alone after 20 steps: {worst:.2e} Angstrom")
    # measured 0 on an H100 80GB HBM3 (each image's and each band's sums happened to run in the same order in both
    # layouts); the bound leaves room for fp32 model noise if a layout changes that order
    assert worst <= 1e-5


def test_graph_replay_restart_and_climb_toggling_are_bitwise():
    spec, _, model, inputs = _ethanol()
    initial, final = _molecules(inputs), _molecules(inputs, shift_seed=3)
    a = _neb(model, initial, final, spec, n_images=3, use_graph=True)
    b = _neb(model, initial, final, spec, n_images=3, use_graph=False)
    for drv in (a, b):
        drv.run(fmax=1e-9, steps=10, check_every=4)
    graph = a._graph
    assert int(a.opt.nsteps.max()) > 0 and int(a.climbing_image.max()) == -1
    for drv in (a, b):
        drv.run(fmax=1e-9, steps=1, climb=True)
    assert a._graph is graph                                           # no recapture
    for drv in (a, b):                                                 # one step after a reset: a fresh FIRE's first
        assert torch.equal(drv.opt.nsteps, torch.zeros_like(drv.opt.nsteps))
        assert torch.all(drv.opt.dt == 0.1) and torch.all(drv.opt.a == 0.1)
        assert bool((drv.climbing_image >= 0).all())
    for drv in (a, b):
        drv.run(fmax=1e-9, steps=6, check_every=4)
    for key in ("opt", "neb"):
        for k, v in getattr(a, key).tensors().items():
            assert torch.equal(v, getattr(b, key).tensors()[k]), (key, k)
    assert torch.equal(a.energy, b.energy) and torch.equal(a.forces, b.forces)

    first = _neb(model, initial, final, spec, n_images=3, climb=True)
    first.run(fmax=1e-9, steps=5)
    sd = first.state_dict()
    first.run(fmax=1e-9, steps=7)
    second = _neb(model, initial, final, spec, n_images=3)
    second.load_state_dict(sd)
    assert second.climb
    second.run(fmax=1e-9, steps=7)
    assert second.iterations == first.iterations == 12
    for key in ("opt", "neb"):
        for k, v in getattr(first, key).tensors().items():
            assert torch.equal(v, getattr(second, key).tensors()[k]), (key, k)


def test_ensemble_follows_the_oracle_fed_the_mean():
    spec, params, model, inputs = _ethanol()
    other = from_spec(spec, {k: v * (1.0 + 0.02 * np.random.default_rng(1).standard_normal(v.shape)).astype(v.dtype)
                             if v.dtype.kind == "f" else v for k, v in params.items()}, DEV)
    initial, final = _molecules(inputs), _molecules(inputs, shift_seed=4)
    n = 3
    dev = _neb([model, other], initial, final, spec, n_images=n, climb=True)
    images = interpolate(initial, final, n)
    evs = [_EagerImages(m, images, spec) for m in (model, other)]
    o = NEBOracle(images[P.R].double().cpu().numpy(), _np(dev.neb.initial), _np(dev.neb.final),
                  _np(dev.neb.end_energies), [9, 9], n, climb=True)
    traj = []
    for _ in range(6):
        dev.run(fmax=1e-9, steps=1)
        traj.append(_np(dev.positions).copy())
    for k in range(6):
        f, e = (np.mean(v, axis=0) for v in zip(*[ev(o.positions) for ev in evs]))
        o.step(f, e, 1e-9)
        assert np.abs(traj[k] - o.positions).max() <= 1e-4, k
    u = dev.get_uncertainty()
    assert u["energy_uncertainty"].shape == (2 * n,) and u["forces_uncertainty"].shape == (2 * n * 9, 3)
    assert float(u["energy_uncertainty"].abs().max()) > 0.0


def test_refusals():
    from schnetpack_b200.parallel import PartitionedPotential

    spec, params, model, inputs = _ethanol()
    initial, final = _molecules(inputs), _molecules(inputs, shift_seed=5)
    with pytest.raises(ValueError, match="n_images"):
        _neb(model, initial, final, spec, n_images=0)
    with pytest.raises(ValueError, match="spring"):
        _neb(model, initial, final, spec, k=0.0)
    with pytest.raises(ValueError, match="systems"):
        _neb(model, initial, _one(final, 0), spec)
    with pytest.raises(ValueError, match="atom counts"):
        _neb(model, initial, dict(final, _n_atoms=torch.tensor([8, 10], device=DEV)), spec)
    swapped = dict(final, _atomic_numbers=final[P.Z].flip(0))
    with pytest.raises(ValueError, match="atomic numbers"):
        _neb(model, initial, swapped, spec)
    with pytest.raises(ValueError, match="cells"):
        _neb(model, initial, dict(final, _cell=final[P.cell] + 1.0), spec)
    with pytest.raises(ValueError, match="pbc"):
        _neb(model, initial, dict(final, _pbc=~final[P.pbc]), spec)
    images = interpolate(initial, final, 3)
    with pytest.raises(ValueError, match="images"):
        _neb(model, initial, final, spec, n_images=2, images=images)
    with pytest.raises(ValueError, match="atomic numbers"):
        _neb(model, initial, final, spec, n_images=3, images=dict(images, _atomic_numbers=images[P.Z].flip(0)))
    with pytest.raises(ValueError, match="FIRE"):
        _neb(model, initial, final, spec, dt=0.0)
    with pytest.raises(ValueError, match="CUDA"):
        _neb(model, {k: v.cpu() for k, v in initial.items()}, final, spec)
    with pytest.raises(NotImplementedError, match="PartitionedPotential"):
        _neb(PartitionedPotential.__new__(PartitionedPotential), initial, final, spec)
    with pytest.raises(ValueError, match="spring"):
        NEBState(torch.zeros(9, 3, dtype=torch.float64, device=DEV), torch.zeros(9, 3), torch.zeros(9, 3),
                 torch.zeros(1, 2), [9], 1, k=-1.0)
    with pytest.raises(ValueError, match="CUDA"):
        NEBState(torch.zeros(9, 3, dtype=torch.float64), torch.zeros(9, 3), torch.zeros(9, 3), torch.zeros(1, 2), [9], 1)
