"""fp64 numpy restatement of the climbing-image nudged elastic band: the improved tangent of Henkelman & Jonsson, J. Chem.
Phys. 113, 9978 (2000), and the climbing image of Henkelman, Uberuaga & Jonsson, J. Chem. Phys. 113, 9901 (2000), in the
form DESIGN.md section 21 defines (with the bisector where the paper's tangent is zero), relaxed by ``FIREOracle`` of
tests/fire_oracle.py with every band as one of its systems.  It is the checker of ``schnetpack_b200.neb.NEBState`` /
``DeviceNEB``.

ASE, whose ``NEB`` object users know, is not installed where these tests run, so the oracle cannot be pinned to it
directly.  tests/test_neb_oracle.py anchors it instead: climbing-image NEB on the Mueller-Brown surface ends at the
published saddle, where the analytic Hessian has exactly one negative eigenvalue; every tangent branch picks the
documented tangent; the five-sum form of the force equals the plain projection; and a band on a flat surface spaces its
images evenly.

Also here: the Mueller-Brown surface (K. Mueller & L. D. Brown, Theor. Chim. Acta 53, 75 (1979)) embedded as one atom
with a harmonic z, with its analytic gradient and Hessian."""
import numpy as np

from fire_oracle import FIREOracle


# ---- the NEB force -------------------------------------------------------------------------------------------------------
def tangent_weights(vp, v0, vn, a, b, c):
    """(alpha, beta) of tau = alpha D+ + beta D- for energies V_{i-1}, V_i, V_{i+1} and the sums a = D+.D+, b = D-.D-,
    c = D+.D-; the bisector (1 / |D+|, 1 / |D-|) when the improved tangent is zero"""
    if vn > v0 > vp:
        alpha, beta = 1.0, 0.0
    elif vn < v0 < vp:
        alpha, beta = 0.0, 1.0
    else:
        dmax, dmin = max(abs(vn - v0), abs(vp - v0)), min(abs(vn - v0), abs(vp - v0))
        alpha, beta = (dmax, dmin) if vn > vp else (dmin, dmax)
    if alpha * alpha * a + 2.0 * alpha * beta * c + beta * beta * b == 0.0:
        alpha = 1.0 / np.sqrt(a) if a > 0.0 else 0.0
        beta = 1.0 / np.sqrt(b) if b > 0.0 else 0.0
    return alpha, beta


def climbing_images(energies, n_bands, n_images, climb):
    """[n_bands] interior index of the highest interior image (ties: the lowest index), -1 without climbing"""
    e = np.asarray(energies, dtype=np.float64).reshape(n_bands, n_images)
    return np.argmax(e, axis=1).astype(np.int64) if climb else np.full(n_bands, -1, dtype=np.int64)


def neb_forces(x, initial, final, forces, energies, end_energies, sizes, n_images, k, climb, fixed=None):
    """NEB forces of the interior images x [N, 3] (band-major, image-major) of bands with ``sizes`` atoms per image,
    endpoint rows ``initial`` / ``final`` [sum sizes, 3], forces [N, 3] and energies [n_bands * n_images] of the interior
    images and ``end_energies`` [n_bands, 2], all in optimizer units.  Returns (F_NEB [N, 3], coef [n_img, 3] =
    (alpha, beta, gamma), diag [n_img, 6] = (|tau|, F.tau^, spring term, |D+|, |D-|, climbing), climbing [n_bands])."""
    x, f = np.asarray(x, dtype=np.float64), np.array(forces, dtype=np.float64)
    if fixed is not None:
        f[np.asarray(fixed, dtype=bool)] = 0.0
    n_bands = len(sizes)
    energies = np.asarray(energies, dtype=np.float64)
    climbing = climbing_images(energies, n_bands, n_images, climb)
    out = np.zeros_like(x)
    coef = np.zeros((n_bands * n_images, 3))
    diag = np.zeros((n_bands * n_images, 6))
    p, e0 = 0, 0
    for band, size in enumerate(sizes):
        images = [initial[e0:e0 + size]] + [x[p + j * size:p + (j + 1) * size] for j in range(n_images)] + \
                 [final[e0:e0 + size]]
        v = [end_energies[band][0]] + list(energies[band * n_images:(band + 1) * n_images]) + [end_energies[band][1]]
        for i in range(n_images):
            img = band * n_images + i
            rows = slice(p + i * size, p + (i + 1) * size)
            dp, dm, fi = images[i + 2] - images[i + 1], images[i + 1] - images[i], f[rows]
            a, b, c = np.vdot(dp, dp), np.vdot(dm, dm), np.vdot(dp, dm)
            d, e = np.vdot(fi, dp), np.vdot(fi, dm)
            alpha, beta = tangent_weights(v[i], v[i + 1], v[i + 2], a, b, c)
            tau2 = alpha * alpha * a + 2.0 * alpha * beta * c + beta * beta * b
            tn, ftau = np.sqrt(tau2), alpha * d + beta * e
            is_climbing = climbing[band] == i
            spring = 0.0 if is_climbing else k * (np.sqrt(a) - np.sqrt(b))
            gamma = 0.0 if tau2 == 0.0 else (-2.0 * ftau / tau2 if is_climbing else -ftau / tau2 + spring / tn)
            out[rows] = fi + gamma * (alpha * dp + beta * dm)
            coef[img] = alpha, beta, gamma
            diag[img] = tn, (ftau / tn if tau2 > 0.0 else 0.0), spring, np.sqrt(a), np.sqrt(b), float(is_climbing)
        p += n_images * size
        e0 += size
    if fixed is not None:
        out[np.asarray(fixed, dtype=bool)] = 0.0
    return out, coef, diag, climbing


def neb_forces_projection(dp, dm, f, alpha, beta, k, climbing):
    """the same force of one image written as the papers do: F - (F.t) t + k (|D+| - |D-|) t, or F - 2 (F.t) t for the
    climbing image, with t the unit tangent"""
    tau = alpha * dp + beta * dm
    t = tau / np.linalg.norm(tau)
    if climbing:
        return f - 2.0 * np.vdot(f, t) * t
    return f - np.vdot(f, t) * t + k * (np.linalg.norm(dp) - np.linalg.norm(dm)) * t


class NEBOracle:
    """Bands of interior images x [N, 3] relaxed by ``FIREOracle`` with band segments as its systems.  ``step(forces,
    energies, fmax)`` takes the forces [N, 3] and energies [n_img] of the current interior images in optimizer units,
    rounds the NEB forces to fp32 (as the device hands them to FIRE) and takes one FIRE step of every unconverged band."""

    def __init__(self, x, initial, final, end_energies, sizes, n_images, k=0.1, climb=False, fixed=None, **fire):
        self.initial = np.asarray(initial, dtype=np.float64)
        self.final = np.asarray(final, dtype=np.float64)
        self.end_energies = np.asarray(end_energies, dtype=np.float64).reshape(-1, 2)
        self.sizes, self.n_images, self.k, self.climb = list(sizes), int(n_images), float(k), bool(climb)
        self.fixed = fixed
        self.band_ptr = np.concatenate([[0], np.cumsum(np.asarray(self.sizes) * self.n_images)])
        self.fire = FIREOracle(x, self.band_ptr, **fire)

    @property
    def positions(self):
        return self.fire.positions

    def forces(self, forces, energies):
        return neb_forces(self.positions, self.initial, self.final, forces, energies, self.end_energies, self.sizes,
                          self.n_images, self.k, self.climb, self.fixed)

    def step(self, forces, energies, fmax=0.0):
        """one step; returns (F_NEB rounded to fp32, the per-band converged flags before the step)"""
        fneb = self.forces(forces, energies)[0].astype(np.float32).astype(np.float64)
        return fneb, self.fire.step(fneb, None, fmax)

    def fmax(self, forces, energies):
        fneb = self.forces(forces, energies)[0].astype(np.float32).astype(np.float64)
        return self.fire.fmax(fneb)

    def path(self, band):
        """[n + 2, A, 3] images of one band, endpoints included"""
        size, e0 = self.sizes[band], int(np.sum(self.sizes[:band]))
        x = self.positions[self.band_ptr[band]:self.band_ptr[band + 1]].reshape(self.n_images, size, 3)
        return np.concatenate([self.initial[None, e0:e0 + size], x, self.final[None, e0:e0 + size]])


# ---- the Mueller-Brown surface -------------------------------------------------------------------------------------------
MB_A = np.array([-200.0, -100.0, -170.0, 15.0])
MB_a = np.array([-1.0, -1.0, -6.5, 0.7])
MB_b = np.array([0.0, 0.0, 11.0, 0.6])
MB_c = np.array([-10.0, -10.0, -6.5, 0.7])
MB_X = np.array([1.0, 0.0, -0.5, -1.0])
MB_Y = np.array([0.0, 0.5, 1.5, 1.0])
MB_KZ = 50.0                       # the harmonic z that makes the surface one atom


def muller_brown(r):
    """energy, force [3] and Hessian [3, 3] of one atom at r = (x, y, z): V = MB(x, y) + KZ z^2 / 2"""
    x, y, z = r
    dx, dy = x - MB_X, y - MB_Y
    t = MB_A * np.exp(MB_a * dx * dx + MB_b * dx * dy + MB_c * dy * dy)
    gx = 2.0 * MB_a * dx + MB_b * dy
    gy = MB_b * dx + 2.0 * MB_c * dy
    e = t.sum() + 0.5 * MB_KZ * z * z
    grad = np.array([(t * gx).sum(), (t * gy).sum(), MB_KZ * z])
    h = np.zeros((3, 3))
    h[0, 0] = (t * (gx * gx + 2.0 * MB_a)).sum()
    h[1, 1] = (t * (gy * gy + 2.0 * MB_c)).sum()
    h[0, 1] = h[1, 0] = (t * (gx * gy + MB_b)).sum()
    h[2, 2] = MB_KZ
    return e, -grad, h
