"""ORACLE -- test infrastructure, NOT product code: an fp64 numpy restatement of schnetpack_b200.phonons and
csrc/phonons.cu for tests/test_phonon_oracle.py and tests/test_cuda_phonons.py.

* ``translations``: the L = det M primitive translations of a supercell (zero first) and the index of -n mod M.
* ``supercell``: fp32 supercell positions (x_b + n . cell in fp64, then rounded) and the fp64 supercell cell.
* ``fc_from_displaced``: force constants from displaced forces at the realised steps; ``fc_from_hessian``: the rows of
  the primitive atoms of a supercell Hessian in the reference's Response layout.
* ``symmetrize``: ASE's Phonons.read rounds (pair symmetrisation, acoustic sum rule).
* ``images``: the minimum-image table; ``dynmat``: D(q); ``frequencies``; ``dos``; ``thermo``.
* ``spring_fc``: force constants of central springs, for closed forms.
Nothing under ``schnetpack_b200/`` imports this module.
"""
from __future__ import annotations

import itertools
import math

import numpy as np

import vib_oracle as V
from schnetpack_b200.units import _UNITS

HBAR_OMEGA_CM = V.HBAR_OMEGA_CM
INVCM = _UNITS["invcm"]
KB = _UNITS["kB"]
MAX_IMAGES = 8


def supercell_matrix(s) -> np.ndarray:
    m = np.asarray(s, dtype=np.int64)
    return np.diag(m) if m.shape == (3,) else m


def translations(s):
    """(lattice [L, 3], neg [L]) from fractional coordinates n M^-1 (fp64 solve, rounded), zero first"""
    M = supercell_matrix(s)
    L = int(round(np.linalg.det(M)))
    Minv = np.linalg.inv(M.astype(np.float64))
    r = int(np.abs(M).sum())
    cand = np.array(list(itertools.product(range(-r, r + 1), repeat=3)))
    f = cand @ Minv
    keep = np.all((f > -1e-9) & (f < 1 - 1e-9), axis=1)
    lattice = cand[keep]
    lattice = lattice[np.argsort(np.any(lattice != 0, axis=1), kind="stable")]
    assert lattice.shape[0] == L

    def same(a, b):
        d = (a - b) @ Minv
        return np.allclose(d, np.round(d), atol=1e-9)

    neg = np.array([next(i for i, n2 in enumerate(lattice) if same(-n, n2)) for n in lattice])
    return lattice, neg


def supercell(pos32, cell32, s, lattice):
    """positions fp32 [n L, 3] (atom l n + b), supercell fp64 [3, 3]"""
    A = cell32.astype(np.float64)
    x = pos32.astype(np.float64)
    lat = lattice.astype(np.float64)
    t = lat[:, 0:1] * A[0] + lat[:, 1:2] * A[1] + lat[:, 2:3] * A[2]
    return (x[None] + t[:, None]).reshape(-1, 3).astype(np.float32), supercell_matrix(s).astype(np.float64) @ A


def fc_from_displaced(steps, forces):
    """steps [3n, nfree] realised, forces [3n, nfree, n L, 3] -> raw force constants [n n L, 3, 3]"""
    n3 = steps.shape[0]
    rows = np.stack([-np.tensordot(V.lagrange_d0(steps[d]), forces[d], axes=(0, 0)) for d in range(n3)])   # [3n, nL, 3]
    n = n3 // 3
    return rows.reshape(n, 3, -1, 3).transpose(0, 2, 1, 3).reshape(-1, 3, 3)


def fc_from_hessian(h, n, n_super):
    """Response-layout Hessian [n_super^2, 3, 3] -> the rows of atoms 0..n-1: [n n_super, 3, 3]"""
    return h.reshape(n_super, n_super, 3, 3)[:n].reshape(-1, 3, 3).copy()


def symmetrize(fc, n, neg, rounds, acoustic):
    L = len(neg)
    phi = fc.reshape(n, L, n, 3, 3).copy()
    rounds = rounds if acoustic else min(rounds, 1)
    for _ in range(rounds):
        partner = phi[:, neg].transpose(2, 1, 0, 4, 3)          # [a, l, b] <- phi[b, neg l, a]^T
        phi = 0.5 * (phi + partner)
        if acoustic:
            s = phi.sum(axis=(1, 2))
            for a in range(n):
                phi[a, 0, a] -= s[a]
    return phi.reshape(-1, 3, 3)


def images(pos64, cell64, s, lattice, tol, search=None):
    """-> list over rows (a, l, b) of (count, [k, 3] primitive translations) of the closest images within tol"""
    M = supercell_matrix(s)
    C = M.astype(np.float64) @ cell64
    Cinv = np.linalg.inv(C)
    n = pos64.shape[0]
    vol = abs(np.linalg.det(C))
    h = np.array([vol / np.linalg.norm(np.cross(C[(i + 1) % 3], C[(i + 2) % 3])) for i in range(3)])
    out = []
    for a in range(n):
        for l, nl in enumerate(lattice):
            for b in range(n):
                r0 = pos64[b] + nl @ cell64 - pos64[a]
                g = np.rint(r0 @ Cinv)
                r0 = r0 - g @ C
                length = np.linalg.norm(r0)
                K = (np.floor((length + tol) / h + 0.5).astype(int) if search is None else np.full(3, search))
                S = np.array(list(itertools.product(*[range(-k, k + 1) for k in K])))
                d = np.linalg.norm(r0[None] + S @ C, axis=1)
                sel = S[d <= d.min() + tol]
                out.append((len(sel), nl[None] + (sel - g) @ M))
    return out


def dynmat(fc, img, masses, q, mw=1.0):
    """D(q) [3n, 3n] complex for one system"""
    n = len(masses)
    L = fc.shape[0] // (n * n)
    phi = fc.reshape(n, L, n, 3, 3)
    D = np.zeros((n, 3, n, 3), dtype=np.complex128)
    for a in range(n):
        for l in range(L):
            for b in range(n):
                cnt, tr = img[(a * L + l) * n + b]
                ph = np.exp(2j * np.pi * (tr @ q)).sum() / cnt
                D[a, :, b, :] += phi[a, l, b] * ph
    D *= mw / np.sqrt(np.outer(masses, masses))[:, None, :, None]
    return D.reshape(3 * n, 3 * n)


def frequencies(D):
    w = np.linalg.eigvalsh(0.5 * (D + D.conj().T))
    return np.sign(w) * np.sqrt(np.abs(w)) * HBAR_OMEGA_CM


def dos(freq, grid, width):
    """freq [Q, 3n] -> g [G], states per cm^-1 per cell"""
    u = (grid[:, None, None] - freq[None]) / width
    return np.exp(-0.5 * u ** 2).sum(axis=(1, 2)) / (width * math.sqrt(2 * math.pi) * freq.shape[0])


def thermo(freq, temperatures, min_freq=1.0):
    """freq [Q, 3n] cm^-1 -> (zpe, F [T], S [T], Cv [T], n_excluded, n_imaginary) per cell, textbook forms"""
    w = freq.reshape(-1)
    keep = w >= min_freq
    e = w[keep] * INVCM
    nq = freq.shape[0]
    zpe = 0.5 * e.sum() / nq
    F, S, C = [], [], []
    for T in temperatures:
        if T == 0:
            F.append(zpe), S.append(0.0), C.append(0.0)
            continue
        x = e / (KB * T)
        F.append(zpe + KB * T * np.log(1 - np.exp(-x)).sum() / nq)
        S.append(KB * (x / (np.exp(x) - 1) - np.log(1 - np.exp(-x))).sum() / nq)
        C.append(KB * (x ** 2 * np.exp(x) / (np.exp(x) - 1) ** 2).sum() / nq)
    return zpe, np.array(F), np.array(S), np.array(C), int((~keep).sum()), int((w < 0).sum())


def spring_fc(pos, cell, s, lattice, springs):
    """force constants [n n L, 3, 3] of central springs (a, b, n_vec, K): atom a of cell 0 to atom b of cell n_vec"""
    M = supercell_matrix(s)
    Minv = np.linalg.inv(M.astype(np.float64))
    n, L = pos.shape[0], lattice.shape[0]
    phi = np.zeros((n, L, n, 3, 3))

    def index(t):
        for i, nl in enumerate(lattice):
            d = (np.asarray(t) - nl) @ Minv
            if np.allclose(d, np.round(d)):
                return i
        raise AssertionError(t)

    for a, b, t, k in springs:
        for (i, j, tt) in ((a, b, np.asarray(t)), (b, a, -np.asarray(t))):
            r = pos[j] + tt @ cell - pos[i]
            e = r / np.linalg.norm(r)
            blk = -k * np.outer(e, e)
            phi[i, index(tt), j] += blk
            phi[i, 0, i] -= blk
    return phi.reshape(-1, 3, 3)
