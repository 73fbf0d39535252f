"""Test infrastructure, not product code: fp64 numpy restatement of the reference's motion removal and wrapping
(md/system.py:258-315,652-684), its initializers (md/initial_conditions.py:50-188) and its two basic simulation hooks
(md/simulation_hooks/basic_hooks.py:41-78), pinned to tests/golden/md_system.npz (made by the reference's own classes).

States are [R, N, 3] (R replicas / beads, N atoms); masses [N]; n_atoms [M] (atoms of a system are contiguous); cells
[R, M, 3, 3] with the lattice vectors as rows, pbc [M, 3].  The normals of an initializer are passed in ([R, N, 3]), so
the oracle reproduces the reference given its recorded draws, and the device given ``nvt_oracle.langevin_normals``.

Where the reference is undefined the oracle states what the device does: the inertia tensor is inverted through its
eigenvalues, dropping those at or below PINV_RTOL x the largest (single atoms, linear molecules, empty systems), and the
beads of a ring polymer move by the lattice translation that wraps their centroid.  For a regular tensor and R = 1 both are
the reference's operations.
"""
from __future__ import annotations

import numpy as np

PINV_RTOL = 1e-10        # SPK_MOTION_PINV_RTOL
WRAP_EPS = 1e-6          # system.py:652


def system_index(n_atoms) -> np.ndarray:
    return np.repeat(np.arange(len(n_atoms)), np.asarray(n_atoms, dtype=np.int64))


def sum_atoms(x: np.ndarray, n_atoms) -> np.ndarray:
    """[R, N, ...] -> [R, M, ...] per-system sums (system.py:217-231)"""
    idx = system_index(n_atoms)
    out = np.zeros((x.shape[0], len(n_atoms)) + x.shape[2:], dtype=np.float64)
    for r in range(x.shape[0]):
        np.add.at(out[r], idx, x[r])
    return out


def center_of_mass(x, m, n_atoms):
    msum = sum_atoms(np.broadcast_to(m[None, :], x.shape[:2]).astype(np.float64), n_atoms)
    mx = sum_atoms(x * m[None, :, None], n_atoms)
    return np.divide(mx, msum[..., None], out=np.zeros_like(mx), where=msum[..., None] > 0)


def remove_center_of_mass(x, m, n_atoms):
    """x -= sum m x / sum m per (replica, system) (system.py:258-276)"""
    return x - center_of_mass(x, m, n_atoms)[:, system_index(n_atoms)]


def remove_translation(p, n_atoms):
    """p -= the unweighted mean of p over the system's atoms (system.py:278-283)"""
    n = np.asarray(n_atoms, dtype=np.float64)
    mean = np.divide(sum_atoms(p, n_atoms), n[None, :, None], out=np.zeros((p.shape[0], len(n_atoms), 3)),
                     where=n[None, :, None] > 0)
    return p - mean[:, system_index(n_atoms)]


def inertia_and_angular_momentum(x, p, m, n_atoms):
    """I = sum m (|x|^2 1 - x x^T) and L = sum x x p about the origin, [R, M, 3, 3] and [R, M, 3] (system.py:291-305)"""
    r2 = np.sum(x * x, axis=2)
    per_atom = r2[..., None, None] * np.eye(3) - x[..., :, None] * x[..., None, :]
    inertia = sum_atoms(per_atom * m[None, :, None, None], n_atoms)
    return inertia, sum_atoms(np.cross(x, p), n_atoms)


def pinv_solve(inertia, L, rtol: float = PINV_RTOL):
    """w = I^+ L with the eigenvalues <= rtol x the largest dropped; I^-1 L for a regular I"""
    w, v = np.linalg.eigh(inertia)
    lmax = w.max(axis=-1, keepdims=True)
    keep = w > rtol * lmax
    coef = np.einsum("...ke,...k->...e", v, L)
    coef = np.divide(coef, w, out=np.zeros_like(coef), where=keep)
    return np.einsum("...ke,...e->...k", v, coef)


def remove_rotation(x, p, m, n_atoms, rtol: float = PINV_RTOL):
    """p -= m (w x x) with w = I^+ L, about the origin (system.py:285-315)"""
    inertia, L = inertia_and_angular_momentum(x, p, m, n_atoms)
    omega = pinv_solve(inertia, L, rtol)
    return p - np.cross(omega[:, system_index(n_atoms)], x) * m[None, :, None]


def wrap_positions(x, cells, pbc, n_atoms, eps: float = WRAP_EPS, by_centroid: bool = True):
    """system.py:652-684 by centroids: every bead of an atom moves by -floor(f_c + eps) C on the periodic axes, f_c the
    fractional coordinates of the bead centroid in the cell of bead 0.  For R = 1, f <- ((f + eps) mod 1) - eps.
    ``by_centroid=False`` wraps every bead on its own, as the reference does."""
    cells = np.asarray(cells, dtype=np.float64)
    if cells.ndim == 3:
        cells = cells[None]
    if np.any(np.linalg.det(cells) == 0.0):
        raise ValueError("zero-volume cell")
    idx = system_index(n_atoms)
    cell_a = cells[0][idx]                                                    # [N, 3, 3]
    xc = x.mean(axis=0, keepdims=True) if by_centroid else x
    frac_c = np.einsum("rnj,nji->rni", xc, np.linalg.inv(cell_a))
    shift = np.floor(frac_c + eps) * np.asarray(pbc, dtype=bool)[idx][None]
    return x - np.einsum("rnj,nji->rni", shift, cell_a)


def fractional(x, cells, n_atoms):
    cells = np.asarray(cells, dtype=np.float64)
    if cells.ndim == 3:
        cells = cells[None]
    idx = system_index(n_atoms)
    inv = np.linalg.inv(cells)[:, idx] if cells.shape[0] == x.shape[0] else np.linalg.inv(cells[0])[idx][None]
    return np.einsum("rnj,rnji->rni", x, inv)


def temperature(p, m, n_atoms, kB, f32_factor: bool = False):
    """2 / (3 n_s kB) * 1/2 sum p^2 / m per (replica, system) (system.py:374-421).  ``f32_factor``: the factor
    2 / (3 n_s kB) rounded as the reference computes it, in float32 (an int64 tensor times Python floats); a relative
    difference of ~1e-8 that the device, which keeps it in fp64, does not repeat."""
    n = np.asarray(n_atoms, dtype=np.float64)
    ke = 0.5 * sum_atoms(np.sum(p * p, axis=2) / m[None, :], n_atoms)
    with np.errstate(divide="ignore"):
        if f32_factor:
            f32 = np.float32
            factor = (f32(2.0) / ((f32(3.0) * n.astype(f32)) * f32(kB))).astype(np.float64)
        else:
            factor = 2.0 / (3.0 * n * kB)
    return np.where(n[None] > 0, factor[None] * ke, 0.0)


def draw_momenta(normals, m, n_atoms, temperatures, kB, uniform: bool, f32_factor: bool = False):
    """UniformInit._setup_momenta (initial_conditions.py:119-135) or MaxwellBoltzmannInit._setup_momenta (:169-188) given
    the normals; one temperature or one per system (the Maxwell-Boltzmann width is then the atom's system's)"""
    t = np.broadcast_to(np.asarray(temperatures, dtype=np.float64).reshape(-1), (len(n_atoms),))
    if uniform:
        p = normals * m[None, :, None]
        cur = temperature(p, m, n_atoms, kB, f32_factor)
        scale = np.divide(t[None], cur, out=np.ones_like(cur), where=cur > 0)
        return p * np.sqrt(scale)[:, system_index(n_atoms), None]
    return normals * np.sqrt(m * kB * t[system_index(n_atoms)])[None, :, None]


def initialize(x, normals, m, n_atoms, temperatures, kB, uniform: bool, remove_center_of_mass_=True,
               remove_translation_=True, remove_rotation_=False, wrap_positions_=False, cells=None, pbc=None,
               by_centroid: bool = True, f32_factor: bool = False):
    """Initializer.initialize_system (initial_conditions.py:50-75): centre of mass, wrap, momenta, translation, rotation"""
    if remove_center_of_mass_:
        x = remove_center_of_mass(x, m, n_atoms)
    if wrap_positions_:
        x = wrap_positions(x, cells, pbc, n_atoms, by_centroid=by_centroid)
    p = draw_momenta(normals, m, n_atoms, temperatures, kB, uniform, f32_factor)
    if remove_translation_:
        p = remove_translation(p, n_atoms)
    if remove_rotation_:
        p = remove_rotation(x, p, m, n_atoms)
    return x, p


def remove_com_motion(x, p, m, n_atoms, rotation: bool):
    """RemoveCOMMotion.on_step_finalize (basic_hooks.py:55-61)"""
    x = remove_center_of_mass(x, m, n_atoms)
    p = remove_translation(p, n_atoms)
    if rotation:
        p = remove_rotation(x, p, m, n_atoms)
    return x, p
