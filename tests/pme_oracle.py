"""fp64 torch restatement of smooth particle-mesh Ewald (Essmann et al., J. Chem. Phys. 103, 8577 (1995)) in the
conventions of csrc/pme.cu, with the analytic reverse of the reciprocal and self terms.

The charge mesh is Q_m(x) = sum_i q_i prod_a M_p(u_ia - x_a mod n_a), u_ia = n_a s_ia, s_i = r_i H mod 1, with M_p the
cardinal B-spline from its two-term recursion (independent of the kernels' weight recursion), and
E_rec = sum_{j != 0} theta_j |Q^(j)|^2, theta_j = ke (2 pi / V) f_k |b(j)|^2, over the signed mesh frequencies j with
the Nyquist index of an even axis left out.  ``energy`` is differentiable by autograd in R, q and the cell, so the tests
can check the analytic reverse (``reverse``) against it."""
from __future__ import annotations

import math

import torch


def bspline(t: torch.Tensor, p: int) -> torch.Tensor:
    """M_p(t), zero outside (0, p): M_2(t) = 1 - |t - 1|, M_p(t) = (t M_{p-1}(t) + (p - t) M_{p-1}(t - 1)) / (p - 1)."""
    if p == 2:
        return torch.clamp(1.0 - torch.abs(t - 1.0), min=0.0)
    return (t * bspline(t, p - 1) + (p - t) * bspline(t - 1.0, p - 1)) / (p - 1)


def bspline_d(t: torch.Tensor, p: int) -> torch.Tensor:
    """dM_p/dt = M_{p-1}(t) - M_{p-1}(t - 1)."""
    return bspline(t, p - 1) - bspline(t - 1.0, p - 1)


def moduli(n: int, p: int) -> torch.Tensor:
    """|sum_{l < p-1} M_p(l + 1) e^{2 pi i j l / n}|^2 for j = 0 .. n-1 (|b_j|^2 is its inverse)."""
    l = torch.arange(p - 1, dtype=torch.float64)
    c = bspline(l + 1.0, p)
    j = torch.arange(n, dtype=torch.float64)
    ph = 2.0 * math.pi * torch.outer(j, l) / n
    return (c * torch.cos(ph)).sum(1) ** 2 + (c * torch.sin(ph)).sum(1) ** 2


def _support(s: torch.Tensor, n: int, p: int):
    """mesh indices [N, p] and offsets t = u - x in (0, p) [N, p] of the support along one axis"""
    u = s * n
    fl = torch.floor(u)
    l = torch.arange(p, dtype=torch.float64)
    idx = (fl.long()[:, None] - (p - 1) + torch.arange(p)[None]) % n
    t = (u - fl)[:, None] + (p - 1) - l[None]
    return idx, t


def _frequencies(cell: torch.Tensor, mesh, p: int, alpha: float, ke: float):
    """theta [B, n1, n2, n3 // 2 + 1], k [B, ..., 3] and the half-spectrum weights w (1 or 2)"""
    n1, n2, n3 = mesh
    H = torch.linalg.inv(cell)
    V = torch.abs(torch.linalg.det(cell))

    def signed(n, half=False):
        j = torch.arange(n // 2 + 1 if half else n)
        return torch.where(2 * j < n, j, j - n) if not half else j

    j1, j2, j3 = signed(n1), signed(n2), signed(n3, True)
    J = torch.stack(torch.meshgrid(j1, j2, j3, indexing="ij"), -1).to(torch.float64)     # [n1, n2, h3, 3]
    k = 2.0 * math.pi * torch.einsum("bac,xyzc->bxyza", H, J)
    k2 = (k ** 2).sum(-1)
    b = (moduli(n1, p)[:, None, None] * moduli(n2, p)[None, :, None] * moduli(n3, p)[None, None, : n3 // 2 + 1])
    nyq = torch.zeros((n1, n2, n3 // 2 + 1), dtype=torch.bool)
    if n1 % 2 == 0:
        nyq[n1 // 2] = True
    if n2 % 2 == 0:
        nyq[:, n2 // 2] = True
    if n3 % 2 == 0:
        nyq[:, :, n3 // 2] = True
    nyq[0, 0, 0] = True
    k2s = torch.where(nyq, torch.ones_like(k2), k2)
    theta = ke * 2.0 * math.pi / V[:, None, None, None] * torch.exp(-0.25 * k2s / alpha) / k2s / b
    theta = torch.where(nyq, torch.zeros_like(theta), theta)
    w = torch.full((n3 // 2 + 1,), 2.0, dtype=torch.float64)
    w[0] = 1.0
    return theta, k, k2s, w


def charge_mesh(q, R, cell, idx_m, n_sys, mesh, p):
    cell = cell.reshape(-1, 3, 3)
    H = torch.linalg.inv(cell)
    s = torch.einsum("nb,nbc->nc", R, H[idx_m])
    s = s - torch.floor(s)
    sup = [_support(s[:, a], mesh[a], p) for a in range(3)]
    w = [bspline(t, p) for _, t in sup]
    W = q[:, None, None, None] * w[0][:, :, None, None] * w[1][:, None, :, None] * w[2][:, None, None, :]
    i1, i2, i3 = (x[0] for x in sup)
    N = R.shape[0]
    ii = [torch.as_tensor(idx_m)[:, None, None, None].expand(N, p, p, p), i1[:, :, None, None].expand(N, p, p, p),
          i2[:, None, :, None].expand(N, p, p, p), i3[:, None, None, :].expand(N, p, p, p)]
    Q = torch.zeros((n_sys,) + tuple(mesh), dtype=torch.float64)
    return Q.index_put(tuple(x.reshape(-1) for x in ii), W.reshape(-1), accumulate=True), s, sup


def energy(q, R, cell, idx_m, n_sys, mesh, p, alpha, ke):
    """E_rec - E_self per system [B] (autograd-differentiable in q, R and cell)"""
    cell = cell.reshape(-1, 3, 3)
    Q, _, _ = charge_mesh(q, R, cell, idx_m, n_sys, mesh, p)
    theta, _, _, w = _frequencies(cell, mesh, p, alpha, ke)
    F = torch.fft.rfftn(Q, dim=(1, 2, 3))
    e_rec = (w * theta * (F.real ** 2 + F.imag ** 2)).sum((1, 2, 3))
    e_self = ke * math.sqrt(alpha / math.pi) * torch.zeros(n_sys, dtype=torch.float64).index_add(
        0, torch.as_tensor(idx_m), q ** 2)
    return e_rec - e_self


def reverse(q, R, cell, idx_m, n_sys, mesh, p, alpha, ke, g_E):
    """The analytic reverse of ``energy`` for the upstream g_E [B]: (g_R [N,3], g_q [N], g_cell [B,3,3], W [B,3,3]).
    phi = dE_rec/dQ = irfftn(2 M theta Q^) (M mesh points); with phi_i and grad_u phi_i gathered over the support:
      g_R_i  = g_E q_i H grad_s phi_i,   g_q_i = g_E (phi_i - 2 ke sqrt(alpha / pi) q_i)
      g_cell = -H^T [sum_i r_i (x) g_R_i - 2 g_E T + g_E E_rec I],   W = -g_E (E_rec I - 2 T)
    with T = sum_j E_j (1/k^2 + 1/(4 alpha)) k (x) k, as in the Ewald sum (E_rec depends on the cell through s, k, V)."""
    with torch.no_grad():
        cell = cell.reshape(-1, 3, 3)
        idx_m = torch.as_tensor(idx_m)
        H = torch.linalg.inv(cell)
        Q, s, sup = charge_mesh(q, R, cell, idx_m, n_sys, mesh, p)
        theta, k, k2, w = _frequencies(cell, mesh, p, alpha, ke)
        F = torch.fft.rfftn(Q, dim=(1, 2, 3))
        M = mesh[0] * mesh[1] * mesh[2]
        phi = torch.fft.irfftn(2.0 * M * theta * F, s=tuple(mesh), dim=(1, 2, 3))
        (i1, t1), (i2, t2), (i3, t3) = sup
        vals = phi[idx_m[:, None, None, None], i1[:, :, None, None], i2[:, None, :, None], i3[:, None, None, :]]
        w1, w2, w3 = bspline(t1, p), bspline(t2, p), bspline(t3, p)
        d1, d2, d3 = bspline_d(t1, p), bspline_d(t2, p), bspline_d(t3, p)
        phi_i = torch.einsum("nabc,na,nb,nc->n", vals, w1, w2, w3)
        gu = torch.stack([torch.einsum("nabc,na,nb,nc->n", vals, d1, w2, w3),
                          torch.einsum("nabc,na,nb,nc->n", vals, w1, d2, w3),
                          torch.einsum("nabc,na,nb,nc->n", vals, w1, w2, d3)], 1)
        gs = gu * torch.tensor(mesh, dtype=torch.float64)
        gE = g_E[idx_m]
        g_R = (gE * q)[:, None] * torch.einsum("nbc,nc->nb", H[idx_m], gs)
        g_q = gE * (phi_i - 2.0 * ke * math.sqrt(alpha / math.pi) * q)
        Ej = w * theta * (F.real ** 2 + F.imag ** 2)
        E_rec = Ej.sum((1, 2, 3))
        T = torch.einsum("bxyz,bxyza,bxyzc->bac", Ej * (1.0 / k2 + 0.25 / alpha), k, k)
        I = torch.eye(3, dtype=torch.float64)[None]
        RG = torch.zeros((n_sys, 3, 3), dtype=torch.float64).index_add(0, idx_m, R[:, :, None] * g_R[:, None, :])
        Mt = RG - 2.0 * g_E[:, None, None] * T + (g_E * E_rec)[:, None, None] * I
        g_cell = -torch.matmul(H.transpose(1, 2), Mt)
        W = -g_E[:, None, None] * (E_rec[:, None, None] * I - 2.0 * T)
    return g_R, g_q, g_cell, W


def ewald_reciprocal_chunked(q, R, cell, alpha, ke, k_max, chunk=4096):
    """E_rec - E_self of one system by the Ewald sum over |n|^2 <= k_max^2 + 2, with -dE/dR, dE/dq and dE/dcell, in
    k-chunks so a box of a few thousand atoms fits in memory (the reference sum and reverse of tests/ewald_oracle.py,
    restated chunked)."""
    import ewald_oracle as EO

    cell = cell.reshape(3, 3)
    H = torch.linalg.inv(cell)
    kv = EO.kvecs(k_max)
    k_all = torch.matmul(kv, 2.0 * math.pi * H.T)
    V = float(torch.abs(torch.linalg.det(cell)))
    pre = ke * 2.0 * math.pi / V
    e = 0.0
    f = torch.zeros_like(R)
    gq = torch.zeros_like(q)
    T = torch.zeros((3, 3), dtype=torch.float64)
    for c0 in range(0, k_all.shape[0], chunk):
        k = k_all[c0:c0 + chunk]
        k2 = (k ** 2).sum(1)
        fk = torch.exp(-0.25 * k2 / alpha) / k2
        th = R @ k.T                                                          # [N, K]
        c, s = torch.cos(th), torch.sin(th)
        re, im = q @ c, q @ s
        ek = fk * (re ** 2 + im ** 2)
        e += float(ek.sum())
        T += torch.einsum("k,ka,kc->ac", ek * (1.0 / k2 + 0.25 / alpha), k, k)
        u = 2.0 * fk * (im[None] * c - re[None] * s)                          # [N, K]
        f -= q[:, None] * (u @ k)
        gq += (2.0 * fk * (re[None] * c + im[None] * s)).sum(1)
    f, T, e_rec = pre * f, pre * T, pre * e
    M = R.T @ (-f) - 2.0 * T + e_rec * torch.eye(3, dtype=torch.float64)     # g_R = -f
    g_cell = -H.T @ M
    e_self = ke * math.sqrt(alpha / math.pi) * float((q ** 2).sum())
    return e_rec - e_self, f, pre * gq - 2.0 * ke * math.sqrt(alpha / math.pi) * q, g_cell


# (order, spacing in A) that reach max|d|/max|ref| <= 1e-5 in the reciprocal energy, forces, dE/dq and dE/dcell against
# the converged Ewald sum on a 1536-atom water box (L = 24.84 A, alpha = 0.46 A^-2; tests/test_pme_oracle.py measures
# it).  Order 6 at 0.4 A and order 4 at 0.4 A do not reach it (forces 1.5e-5 and 1.1e-3).
ACCURACY = {8: 0.5}
FIXTURE_PARAMS = (8, 0.5)          # order, spacing used for the e1 / e2 fixture models (alpha 0.12 and 0.2)
