"""ORACLE -- test infrastructure, NOT product code: an fp64 numpy restatement of schnetpack_b200.vibrations and
csrc/vibrations.cu for tests/test_vib_oracle.py and tests/test_cuda_vibrations.py.

* ``chunk_layout``: the chunk / copy / idle bookkeeping of the replica batch.
* ``displace``: the fp32 replica positions and the realised fp64 steps of one chunk.
* ``lagrange_d0``: the weights of the derivative at 0 through the realised nodes.
* ``hessian``: the whole scheme on a force function of the replica batch -> the Response layout and the mass-weighted
  blocks; ``hessian_from_displaced``: the same from recorded displaced forces of one system.
* ``frequencies`` / ``modes`` / ``ir_intensities`` / ``raman_activities``: ASE's conventions (ase/vibrations), with an
  imaginary frequency returned as a negative number.
Nothing under ``schnetpack_b200/`` imports this module.
"""
from __future__ import annotations

import math

import numpy as np

from schnetpack_b200.units import _UNITS, _amu, _e, _hbar

HBAR_OMEGA_CM = _hbar * 1e10 / math.sqrt(_e * _amu) / _UNITS["invcm"]     # cm^-1 per sqrt(eV / (A^2 amu))


def stencil(nfree: int) -> np.ndarray:
    """offsets in units of h, in copy order (ASE's displacements)"""
    return {2: np.array([-1.0, 1.0]), 4: np.array([-2.0, -1.0, 1.0, 2.0])}[nfree]


def n_columns(sizes, n_atoms: int, nfree: int, max_replica_atoms: int) -> int:
    return max(1, min(3 * max(sizes), max_replica_atoms // max(1, nfree * n_atoms)))


def chunk_layout(sizes, n_cols: int, nfree: int):
    """-> (n_chunks, table): table[chunk][copy][m] = displaced coordinate d of system m in that copy, or -1 (idle)"""
    n_coords = 3 * max(sizes)
    n_chunks = -(-n_coords // n_cols)
    table = np.full((n_chunks, n_cols * nfree, len(sizes)), -1, dtype=np.int64)
    for k in range(n_chunks):
        for c in range(n_cols * nfree):
            d = k * n_cols + c // nfree
            for m, n in enumerate(sizes):
                if d < 3 * n:
                    table[k, c, m] = d
    return n_chunks, table


def displace(base32: np.ndarray, sys_ptr, chunk: int, n_cols: int, nfree: int, delta: float):
    """-> (replica positions fp32 [C N, 3], realised steps fp64 [C, B])"""
    sizes = np.diff(sys_ptr)
    n_chunks, table = chunk_layout(sizes, n_cols, nfree)
    C, N, B = n_cols * nfree, base32.shape[0], len(sizes)
    pos = np.tile(base32.astype(np.float32), (C, 1, 1))
    steps = np.zeros((C, B))
    off = stencil(nfree)
    for c in range(C):
        o = np.float32(off[c % nfree] * delta)
        for m in range(B):
            d = table[chunk, c, m]
            if d < 0:
                continue
            a, k = sys_ptr[m] + d // 3, d % 3
            x = np.float32(base32[a, k])
            pos[c, a, k] = x + o
            steps[c, m] = float(pos[c, a, k]) - float(x)
    return pos.reshape(C * N, 3), steps


def lagrange_d0(t: np.ndarray) -> np.ndarray:
    """weights w with sum_s w_s y_s = p'(0) for the polynomial p through (t_s, y_s)"""
    k = len(t)
    w = np.zeros(k)
    for s in range(k):
        num = 0.0
        for q in range(k):
            if q != s:
                num += np.prod([-t[r] for r in range(k) if r not in (s, q)])
        w[s] = num / np.prod([t[s] - t[r] for r in range(k) if r != s])
    return w


def finish(raw_blocks, masses, sys_ptr, mw_scale: float = 1.0):
    """raw [3n, 3n] per system (row r, column d = -dF_r/dx_d) -> (Response layout [sum n^2, 3, 3], mass-weighted
    blocks): symmetrised, row i n + j, block [a, b] = H[3i + a, 3j + b]"""
    out, mw = [], []
    for m, raw in enumerate(raw_blocks):
        n = raw.shape[0] // 3
        h = 0.5 * (raw + raw.T)
        out.append(h.reshape(n, 3, n, 3).transpose(0, 2, 1, 3).reshape(n * n, 3, 3))
        sm = np.repeat(np.sqrt(masses[sys_ptr[m]:sys_ptr[m + 1]]), 3)
        mw.append(h * mw_scale / np.outer(sm, sm))
    return np.concatenate(out) if out else np.zeros((0, 3, 3)), mw


def hessian(force_fn, base32, sys_ptr, masses, delta, nfree, n_cols, props_fn=None):
    """The whole scheme: ``force_fn(pos [C N, 3] fp64, C)`` -> forces [C N, 3]; ``props_fn(pos, C)`` -> dict of
    per-system outputs [C B, ...].  Returns (hessian [sum n^2, 3, 3], mass-weighted blocks, derivatives {key: [N, ..., 3]})"""
    sizes = np.diff(sys_ptr)
    N, B = base32.shape[0], len(sizes)
    n_chunks, table = chunk_layout(sizes, n_cols, nfree)
    raw = [np.zeros((3 * n, 3 * n)) for n in sizes]
    derivs = {}
    for k in range(n_chunks):
        pos, steps = displace(base32, sys_ptr, k, n_cols, nfree, delta)
        C = n_cols * nfree
        f = force_fn(pos.astype(np.float64), C).reshape(C, N, 3)
        props = props_fn(pos.astype(np.float64), C) if props_fn else {}
        for dl in range(n_cols):
            cs = [dl * nfree + s for s in range(nfree)]
            for m in range(B):
                d = table[k, cs[0], m]
                if d < 0:
                    continue
                w = lagrange_d0(steps[cs, m])
                lo, hi = sys_ptr[m], sys_ptr[m + 1]
                raw[m][:, d] = -np.einsum("s,snk->nk", w, f[cs, lo:hi]).reshape(-1)
                for key, v in props.items():
                    v = v.reshape(C, B, -1)
                    dv = derivs.setdefault(key, np.zeros((N, v.shape[-1], 3)))
                    dv[lo + d // 3, :, d % 3] = np.einsum("s,sc->c", w, v[cs, m])
    h, mw = finish(raw, masses, sys_ptr)
    return h, mw, derivs


def hessian_from_displaced(steps, forces):
    """one system: ``steps`` [3n, nfree] realised steps of coordinate d, ``forces`` [3n, nfree, n, 3] -> raw [3n, 3n]"""
    n3 = steps.shape[0]
    raw = np.zeros((n3, n3))
    for d in range(n3):
        raw[:, d] = -np.einsum("s,snk->nk", lagrange_d0(steps[d]), forces[d]).reshape(-1)
    return raw


# ---- ASE's post-processing ---------------------------------------------------------------------------------------------
def eigensystem(mw_block):
    return np.linalg.eigh(mw_block)


def frequencies(mw_blocks) -> np.ndarray:
    """[3N] cm^-1, ascending per system; imaginary as negative"""
    w = np.concatenate([np.linalg.eigvalsh(b) for b in mw_blocks]) if mw_blocks else np.zeros(0)
    return np.sign(w) * np.sqrt(np.abs(w)) * HBAR_OMEGA_CM


def modes(mw_block, masses_m) -> np.ndarray:
    """[3n, n, 3]: eigenvectors / sqrt(m) (ASE's get_mode)"""
    _, v = np.linalg.eigh(mw_block)
    n = len(masses_m)
    return (v.T / np.repeat(np.sqrt(masses_m), 3)).reshape(3 * n, n, 3)


def _project(mode, deriv):
    """mode [3n, n, 3], deriv [n, n_comp, 3] -> [3n, n_comp]"""
    return np.einsum("kid,icd->kc", mode, deriv)


def ir_intensities(mw_blocks, masses, sys_ptr, dipole_deriv) -> np.ndarray:
    out = []
    for m, b in enumerate(mw_blocks):
        lo, hi = sys_ptr[m], sys_ptr[m + 1]
        out.append((_project(modes(b, masses[lo:hi]), dipole_deriv[lo:hi]) ** 2).sum(1))
    return np.concatenate(out)


def raman_activities(mw_blocks, masses, sys_ptr, polar_deriv) -> np.ndarray:
    out = []
    for m, b in enumerate(mw_blocks):
        lo, hi = sys_ptr[m], sys_ptr[m + 1]
        a = _project(modes(b, masses[lo:hi]), polar_deriv[lo:hi].reshape(hi - lo, 9, 3)).reshape(-1, 3, 3)
        a = 0.5 * (a + a.transpose(0, 2, 1))
        mean = np.trace(a, axis1=1, axis2=2) / 3.0
        xx, yy, zz = a[:, 0, 0], a[:, 1, 1], a[:, 2, 2]
        g2 = 0.5 * ((xx - yy) ** 2 + (yy - zz) ** 2 + (zz - xx) ** 2
                    + 6.0 * (a[:, 0, 1] ** 2 + a[:, 1, 2] ** 2 + a[:, 2, 0] ** 2))
        out.append(45.0 * mean ** 2 + 7.0 * g2)
    return np.concatenate(out)
