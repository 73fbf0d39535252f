"""SO(3) building blocks of SO3net -- drop-ins for ``schnetpack.nn.so3`` (RealSphericalHarmonics, SO3TensorProduct,
SO3Convolution, SO3ParametricGatedNonlinearity, SO3GatedNonlinearity, scalar2rsh).

Constructors, buffers and parameter names follow the reference, so module trees and ``state_dict`` keys are identical
(``SO3Convolution.Widx`` is the one persistent buffer).  Called on their own the modules evaluate differentiable ATen
formulas on any device; ``SO3net.forward`` runs the fused kernels of ``csrc/so3net.cu`` instead.

The real-basis Clebsch-Gordan table is computed here without sympy: Racah's closed form in fp64 for the complex basis,
the complex-to-real change of basis, the parity mask (l1 + l2 + l3 even), then fp32 rounding.  Its sparse form lists the
nonzeros row-major over (s1, s2, s_out) -- the order ``torch.nonzero`` returns -- with s = l^2 + l + m.
``cuda_tables_source`` writes the same table and the spherical-harmonic polynomials as the C++ header the kernels include
(``csrc/so3_tables.cuh``); a test keeps that header equal to this generator's output.
"""
from __future__ import annotations

import math
from functools import lru_cache
from typing import Tuple

import numpy as np
import torch
import torch.nn as nn

from . import Dense

__all__ = ["RealSphericalHarmonics", "SO3TensorProduct", "SO3Convolution", "SO3GatedNonlinearity",
           "SO3ParametricGatedNonlinearity", "scalar2rsh", "sh_indices", "clebsch_gordan_rsh", "sparse_clebsch_gordan",
           "KERNEL_LMAX", "cuda_tables_source"]

KERNEL_LMAX = 3          # highest angular momentum the CUDA kernels are compiled for


@lru_cache(maxsize=16)
def sh_indices(lmax: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """(l, m) of every combined index s = l^2 + l + m, s < (lmax + 1)^2."""
    ls = [l for l in range(lmax + 1) for _ in range(2 * l + 1)]
    ms = [m for l in range(lmax + 1) for m in range(-l, l + 1)]
    return torch.tensor(ls, dtype=torch.int64), torch.tensor(ms, dtype=torch.int64)


def _cg_complex(l1: int, m1: int, l2: int, m2: int, l3: int, m3: int) -> float:
    """<l1 m1; l2 m2 | l3 m3> (Condon-Shortley phase) from Racah's closed form, fp64."""
    if m1 + m2 != m3 or not abs(l1 - l2) <= l3 <= l1 + l2 or abs(m1) > l1 or abs(m2) > l2 or abs(m3) > l3:
        return 0.0
    f = math.factorial
    num = (2 * l3 + 1) * f(l3 + l1 - l2) * f(l3 - l1 + l2) * f(l1 + l2 - l3)
    num *= f(l3 + m3) * f(l3 - m3) * f(l1 - m1) * f(l1 + m1) * f(l2 - m2) * f(l2 + m2)
    den = f(l1 + l2 + l3 + 1)
    s = 0.0
    for k in range(0, l1 + l2 - l3 + 1):
        args = (k, l1 + l2 - l3 - k, l1 - m1 - k, l2 + m2 - k, l3 - l2 + m1 + k, l3 - l1 - m2 + k)
        if min(args) < 0:
            continue
        d = 1
        for a in args:
            d *= f(a)
        s += (-1.0) ** k / d
    return math.sqrt(num / den) * s


def _complex_to_real(lmax: int) -> np.ndarray:
    """U[s_real, s_complex]: real harmonics as combinations of the complex ones (block diagonal in l)."""
    lidx, midx = (t.numpy() for t in sh_indices(lmax))
    n = lidx.shape[0]
    U = np.zeros((n, n), dtype=np.complex128)
    r = 1.0 / math.sqrt(2.0)
    for a in range(n):
        l, m = lidx[a], midx[a]
        off = l * l + l
        if m == 0:
            U[a, off] = 1.0
        elif m > 0:
            U[a, off + m] = (-1.0) ** m * r
            U[a, off - m] = r
        else:
            U[a, off - m] = -1j * (-1.0) ** (-m) * r
            U[a, off + m] = 1j * r
    return U


@lru_cache(maxsize=16)
def clebsch_gordan_rsh(lmax: int) -> np.ndarray:
    """Dense real-basis table C[s1, s2, s_out] (fp64, exact zeros), outputs truncated at lmax, parity-invariant."""
    lidx, midx = (t.numpy() for t in sh_indices(lmax))
    n = lidx.shape[0]
    cg = np.zeros((n, n, n), dtype=np.complex128)
    for a in range(n):
        for b in range(n):
            for c in range(n):
                cg[a, b, c] = _cg_complex(int(lidx[a]), int(midx[a]), int(lidx[b]), int(midx[b]), int(lidx[c]),
                                          int(midx[c]))
    U = _complex_to_real(lmax)
    real = np.einsum("ijk,mi,nj,ok->mno", cg, U, U, U.conj())
    parity = (lidx[:, None, None] + lidx[None, :, None] + lidx[None, None, :]) % 2 == 0
    out = np.where(parity, real.real, 0.0)
    out[np.abs(out) < 1e-12] = 0.0          # rounding residue of the change of basis: the exact value is zero
    return out


@lru_cache(maxsize=16)
def sparse_clebsch_gordan(lmax: int):
    """(values fp32, idx_in_1, idx_in_2, idx_out) of the nonzeros, row-major over (s1, s2, s_out)."""
    dense = torch.from_numpy(clebsch_gordan_rsh(lmax)).to(torch.float32)
    idx = torch.nonzero(dense)
    i1, i2, io = idx[:, 0].contiguous(), idx[:, 1].contiguous(), idx[:, 2].contiguous()
    return dense[i1, i2, io].contiguous(), i1, i2, io


def _ylm_coefficients(lmax: int):
    """Coefficient buffers of RealSphericalHarmonics (fp64): Y_lm = sqrt((2l+1)/(2 pi)) Pi_l^|m|(z) T_m(x, y) with
    T_m = Re (x + iy)^m for m > 0, Im (x + iy)^|m| for m < 0, sqrt(1/2) for m = 0, and
    Pi_l^m(z) = sum_k cPi[l, m, k] z^zpow[l, m, k];  (x + iy)^m = sum_p (cAm + i cBm)[m-1, p] x^p y^(m-p)."""
    L = lmax
    cAm = np.zeros((L, L + 1))
    cBm = np.zeros((L, L + 1))
    powers = np.zeros((L, L + 1, 2))
    for m in range(1, L + 1):
        for p in range(m + 1):
            c = math.comb(m, p)
            q = (m - p) % 4                           # i^(m-p)
            cAm[m - 1, p] = c * (1.0, 0.0, -1.0, 0.0)[q]
            cBm[m - 1, p] = c * (0.0, 1.0, 0.0, -1.0)[q]
            powers[m - 1, p] = (p, m - p)
    K = L // 2 + 1
    cPi = np.zeros((L + 1, L + 1, K))
    zpow = np.zeros((L + 1, L + 1, K))
    f = math.factorial
    for l in range(L + 1):
        for m in range(l + 1):
            for k in range((l - m) // 2 + 1):
                cPi[l, m, k] = (math.sqrt(f(l - m) / f(l + m)) * (-1.0) ** k * 2.0 ** (-l) * math.comb(l, k)
                                * math.comb(2 * l - 2 * k, l) * f(l - 2 * k) / f(l - 2 * k - m))
                zpow[l, m, k] = l - 2 * k - m
    return [torch.from_numpy(a) for a in (powers, zpow, cAm, cBm, cPi)]


class RealSphericalHarmonics(nn.Module):
    """Real spherical harmonics of unit vectors [E, 3] -> [E, (lmax+1)^2], ordered (l, m = -l..l)."""

    def __init__(self, lmax: int, dtype_str: str = "float32"):
        super().__init__()
        self.lmax = lmax
        dtype = getattr(torch, dtype_str)
        powers, zpow, cAm, cBm, cPi = _ylm_coefficients(lmax)
        self.register_buffer("powers", powers.to(dtype=dtype), False)
        self.register_buffer("zpow", zpow.to(dtype=dtype), False)
        self.register_buffer("cAm", cAm.to(dtype=dtype), False)
        self.register_buffer("cBm", cBm.to(dtype=dtype), False)
        self.register_buffer("cPi", cPi.to(dtype=dtype), False)
        self.lidx, self.midx = sh_indices(lmax)
        self.register_buffer("flidx", self.lidx.to(dtype=dtype), False)

    def forward(self, directions: torch.Tensor) -> torch.Tensor:
        L = self.lmax
        x, y, z = directions[:, 0], directions[:, 1], directions[:, 2]

        def pows(v):
            out = [torch.ones_like(v)]
            for _ in range(L):
                out.append(out[-1] * v)
            return torch.stack(out, dim=1)                                   # [E, L+1]

        xp, yp, zp = pows(x), pows(y), pows(z)
        pw = self.powers.long()
        mono = xp[:, pw[..., 0]] * yp[:, pw[..., 1]]                          # [E, L, L+1]
        A = (mono * self.cAm).sum(-1)                                        # Re (x+iy)^m, m = 1..L
        B = (mono * self.cBm).sum(-1)                                        # Im (x+iy)^m
        half = torch.full((x.shape[0], 1), math.sqrt(0.5), dtype=torch.float32, device=x.device).to(A.dtype)
        T = torch.cat([torch.flip(B, (1,)), half, A], dim=1)[:, self.midx.to(x.device) + L]
        Pi = (zp[:, self.zpow.long()] * self.cPi).sum(-1)                    # [E, L+1, L+1]
        Pi = Pi[:, self.lidx.to(x.device), self.midx.to(x.device).abs()]
        return torch.sqrt((2 * self.flidx + 1) / (2 * math.pi)) * Pi * T


def scalar2rsh(x: torch.Tensor, lmax: int) -> torch.Tensor:
    """[N, 1, F] -> [N, (lmax+1)^2, F], zero above l = 0."""
    pad = torch.zeros((x.shape[0], (lmax + 1) ** 2 - 1, x.shape[2]), device=x.device, dtype=x.dtype)
    return torch.cat([x, pad], dim=1)


def _scatter_dim1(v: torch.Tensor, idx: torch.Tensor, n: int) -> torch.Tensor:
    out = torch.zeros((v.shape[0], n) + tuple(v.shape[2:]), dtype=v.dtype, device=v.device)
    return out.index_add(1, idx, v)


class _CGBuffers(nn.Module):
    def _register_cg(self, lmax: int):
        cg, i1, i2, io = sparse_clebsch_gordan(lmax)
        self.register_buffer("idx_in_1", i1.clone(), persistent=False)
        self.register_buffer("idx_in_2", i2.clone(), persistent=False)
        self.register_buffer("idx_out", io.clone(), persistent=False)
        self.register_buffer("clebsch_gordan", cg.clone(), persistent=False)


class SO3TensorProduct(_CGBuffers):
    """y[n, s, f] = sum_{s1, s2} C[s1, s2, s] x1[n, s1, f] x2[n, s2, f]."""

    def __init__(self, lmax: int):
        super().__init__()
        self.lmax = lmax
        self._register_cg(lmax)

    def forward(self, x1: torch.Tensor, x2: torch.Tensor) -> torch.Tensor:
        y = x1[:, self.idx_in_1, :] * x2[:, self.idx_in_2, :] * self.clebsch_gordan[None, :, None]
        return _scatter_dim1(y, self.idx_out, (self.lmax + 1) ** 2)


class SO3Convolution(_CGBuffers):
    """y[i, s, f] = sum_{j, s1, s2} C[s1, s2, s] W[l(s1), f](d_ij) Y[s1](r_ij) x[j, s2, f] with the radial filter
    W[l, f] = fcut(d) * filternet(phi(d))[l * F + f].  ``dir_ij`` receives the harmonics Y_ij, as in the reference."""

    def __init__(self, lmax: int, n_atom_basis: int, n_radial: int):
        super().__init__()
        self.lmax = lmax
        self.n_atom_basis = n_atom_basis
        self.n_radial = n_radial
        self._register_cg(lmax)
        self.filternet = Dense(n_radial, n_atom_basis * (lmax + 1), activation=None)
        lidx, _ = sh_indices(lmax)
        self.register_buffer("Widx", lidx[self.idx_in_1])

    def _compute_radial_filter(self, radial_ij: torch.Tensor, cutoff_ij: torch.Tensor) -> torch.Tensor:
        from .. import functional_torch as T

        W = T.dense(radial_ij, self.filternet) * cutoff_ij
        return W.reshape(-1, self.lmax + 1, self.n_atom_basis)[:, self.Widx]

    def forward(self, x, radial_ij, dir_ij, cutoff_ij, idx_i, idx_j):
        xj = x[idx_j[:, None], self.idx_in_2[None, :], :]
        W = self._compute_radial_filter(radial_ij, cutoff_ij)
        v = W * dir_ij[:, self.idx_in_1, None] * self.clebsch_gordan[None, :, None] * xj
        yij = _scatter_dim1(v, self.idx_out, (self.lmax + 1) ** 2)
        return torch.zeros((x.shape[0],) + tuple(yij.shape[1:]), dtype=yij.dtype, device=yij.device).index_add(
            0, idx_i, yij)


class SO3ParametricGatedNonlinearity(nn.Module):
    """y[n, s, f] = x[n, s, f] * sigmoid(scaling(x[n, 0, :])[l(s) * F + f])."""

    def __init__(self, n_in: int, lmax: int):
        super().__init__()
        self.lmax = lmax
        self.n_in = n_in
        self.lidx, _ = sh_indices(lmax)
        self.scaling = nn.Linear(n_in, n_in * (lmax + 1))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        h = self.scaling(x[:, 0, :]).reshape(-1, self.lmax + 1, self.n_in)
        return x * torch.sigmoid(h[:, self.lidx.to(h.device)])


class SO3GatedNonlinearity(nn.Module):
    """y[n, s, f] = x[n, s, f] * sigmoid(x[n, 0, f])."""

    def __init__(self, lmax: int):
        super().__init__()
        self.lmax = lmax
        self.lidx, _ = sh_indices(lmax)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return x * torch.sigmoid(x[:, 0, :])[:, None, :]


# ----------------------------------------------------------------------------------------------- kernel tables
def _f32(v: float) -> str:
    s = "%.9e" % float(np.float32(v))
    return s + "f"


def cuda_tables_source() -> str:
    """Text of ``csrc/so3_tables.cuh``: for every lmax <= KERNEL_LMAX the CG nonzeros (in the sparse order above) and
    the harmonics as Y_s = poly_s(z) * T_m(x, y), poly_s holding sqrt((2l+1)/(2 pi)) (and sqrt(1/2) at m = 0)."""
    out = ["// Generated by schnetpack_b200.nn.so3.cuda_tables_source() -- do not edit; tests/test_so3net_oracle.py",
           "// keeps this file equal to the generator's output.",
           "#pragma once", "", "template <int L> struct So3Tab;", ""]
    for L in range(KERNEL_LMAX + 1):
        cg, i1, i2, io = sparse_clebsch_gordan(L)
        _, zpow, _, _, cPi = _ylm_coefficients(L)
        lidx, midx = sh_indices(L)
        out.append(f"template <> struct So3Tab<{L}> {{")
        out.append(f"    static constexpr int S = {(L + 1) ** 2};")
        out.append(f"    static constexpr int NNZ = {cg.shape[0]};")
        out.append("    // op(s1, s2, s_out, C)")
        out.append("    template <class Op> __device__ __forceinline__ static void cg(Op&& op) {")
        for n in range(cg.shape[0]):
            out.append(f"        op({int(i1[n])}, {int(i2[n])}, {int(io[n])}, {_f32(float(cg[n]))});")
        out.append("    }")
        out.append("    // op(s, m, c0, c1, c2, c3): Y_s = (c0 + c1 z + c2 z^2 + c3 z^3) * T_m(x, y)")
        out.append("    template <class Op> __device__ __forceinline__ static void sh(Op&& op) {")
        for s in range(lidx.shape[0]):
            l, m = int(lidx[s]), int(midx[s])
            am = abs(m)
            c = [0.0] * 4
            for k in range(zpow.shape[2]):
                if float(cPi[l, am, k]) != 0.0:
                    c[int(zpow[l, am, k])] += float(cPi[l, am, k])
            norm = math.sqrt((2 * l + 1) / (2 * math.pi)) * (math.sqrt(0.5) if m == 0 else 1.0)
            out.append(f"        op({s}, {m}, " + ", ".join(_f32(v * norm) for v in c) + ");")
        out.append("    }")
        out.append("};")
        out.append("")
    return "\n".join(out)
