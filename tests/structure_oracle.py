"""fp64 numpy restatement of the structural observables of schnetpack_b200.structure (DESIGN.md section 24).

RDF: the ordered pairs (i, j, S) with |R_j - R_i + S cell| < r_max, (i, i, 0) excluded and self-images included, found by
explicit enumeration of the image shifts S (any triclinic cell, positions anywhere), binned at floor(d n_bins / r_max)
per species-pair slot.  MSD: a stored trajectory unwrapped sample by sample (fractional displacement wrapped to
[-1/2, 1/2) in the current cell), time origins every ``origin_every`` samples in a ring of ceil(n_lags / origin_every)
slots, optional removal of the mass-weighted centre-of-mass shift."""
import math

import numpy as np

EDGE_RTOL = 1e-5        # pairs this close (relative) to a bin edge may fall on either side in fp32


def heights(cell):
    """distances between opposite faces of the cell [3, 3] (rows = lattice vectors)"""
    inv = np.linalg.inv(cell)
    return 1.0 / np.linalg.norm(inv, axis=0)


def rdf_counts(R, cell, types, slot_of, total_slot, n_slots, r_max, n_bins):
    """Integer pair counts [n_slots, n_bins] of one frame and the counts of the pairs within EDGE_RTOL of an edge of
    their bin (the same shape).  R [N, 3], cell [3, 3], types [N] (species indices), slot_of [T, T] (-1: none)."""
    R = np.asarray(R, np.float64)
    cell = np.asarray(cell, np.float64)
    N = R.shape[0]
    f = R @ np.linalg.inv(cell)
    df = f[None, :, :] - f[:, None, :]                                  # f_j - f_i  [N, N, 3]
    reach = np.ceil(r_max / heights(cell) + np.abs(df).reshape(-1, 3).max(0)).astype(int) + 1
    dr = r_max / n_bins
    counts = np.zeros((n_slots, n_bins), np.int64)
    amb = np.zeros((n_slots, n_bins), np.int64)
    slot = slot_of[types[:, None], types[None, :]]                     # [N, N]
    eye = np.eye(N, dtype=bool)
    for s0 in range(-reach[0], reach[0] + 1):
        for s1 in range(-reach[1], reach[1] + 1):
            for s2 in range(-reach[2], reach[2] + 1):
                S = np.array([s0, s1, s2], np.float64)
                d = np.linalg.norm((df + S) @ cell, axis=-1)
                hit = d < r_max
                if s0 == 0 and s1 == 0 and s2 == 0:
                    hit &= ~eye
                if not hit.any():
                    continue
                dd, sl = d[hit], slot[hit]
                k = np.minimum(np.floor(dd / dr).astype(int), n_bins - 1)
                x = dd / dr
                near = (np.abs(x - np.round(x)) <= EDGE_RTOL * np.maximum(x, 1.0)) | (dd > r_max * (1 - EDGE_RTOL))
                for target, sel in ((sl, sl >= 0), (np.full_like(sl, total_slot), np.full(sl.shape, total_slot >= 0))):
                    np.add.at(counts, (target[sel], k[sel]), 1)
                    np.add.at(amb, (target[sel & near], k[sel & near]), 1)
    return counts, amb


def shell_volumes(r_max, n_bins):
    e = np.linspace(0.0, r_max, n_bins + 1)
    return 4.0 * math.pi / 3.0 * (e[1:] ** 3 - e[:-1] ** 3)


def rdf_from_sums(acc, n_frames, na, nb, r_max):
    """g [.., n_slots, n_bins] from acc = sum over frames of V counts, n_frames frames (times beads), na / nb [.., n_slots]"""
    n_bins = acc.shape[-1]
    return acc / (n_frames * (np.asarray(na) * np.asarray(nb))[..., None] * shell_volumes(r_max, n_bins))


def coordination_from_sums(acc, volume_sum, na):
    """running coordination numbers: cumsum(acc) / (N_a sum V)"""
    return np.cumsum(acc, -1) / (np.asarray(na)[..., None] * np.asarray(volume_sum)[..., None, None])


def fcc(a, n):
    """positions of an n x n x n supercell of the conventional fcc cell of edge a, and its cell"""
    basis = np.array([[0, 0, 0], [0.5, 0.5, 0], [0.5, 0, 0.5], [0, 0.5, 0.5]])
    g = np.array([[i, j, k] for i in range(n) for j in range(n) for k in range(n)], np.float64)
    R = ((g[:, None, :] + basis[None]) * a).reshape(-1, 3)
    return R, np.eye(3) * a * n


def msd_oracle(traj, cells, pbc, masses, species, sys_ptr, n_species, n_lags, origin_every, remove_com):
    """acc [B, n_species, n_lags], count [n_lags], jump flag of the trajectory traj [T, N, 3] (positions as sampled,
    possibly wrapped), cells [T, B, 3, 3] or None (open systems), pbc [B, 3] bool."""
    traj = np.asarray(traj, np.float64)
    T, N, _ = traj.shape
    B = len(sys_ptr) - 1
    sys_of = np.repeat(np.arange(B), np.diff(sys_ptr))
    masses = np.asarray(masses, np.float64)
    K = -(-n_lags // origin_every)
    acc = np.zeros((B, n_species, n_lags))
    count = np.zeros(n_lags, np.int64)
    origins = np.zeros((K, N, 3))
    origin_com = np.zeros((K, B, 3))
    origin_sample = np.full(K, -1)
    jump = False

    def com(u):
        out = np.zeros((B, 3))
        for b in range(B):
            sl = slice(sys_ptr[b], sys_ptr[b + 1])
            m = masses[sl]
            out[b] = (m[:, None] * u[sl]).sum(0) / m.sum() if m.sum() > 0 else 0.0
        return out

    u = traj[0].copy()
    last = traj[0].copy()
    for n in range(T):
        x = traj[n]
        if n > 0:
            d = x - last
            if cells is not None:
                for b in range(B):
                    if not np.any(pbc[b]):
                        continue
                    sl = slice(sys_ptr[b], sys_ptr[b + 1])
                    C = cells[n][b]
                    f = d[sl] @ np.linalg.inv(C)
                    f[:, pbc[b]] -= np.floor(f[:, pbc[b]] + 0.5)
                    d[sl] = f @ C
                    h = heights(C)[pbc[b]].min()
                    jump |= bool((np.linalg.norm(d[sl], axis=1) > 0.5 * h).any())
            u = u + d
            last = x.copy()
        c = com(u)
        if n % origin_every == 0:
            o = (n // origin_every) % K
            origins[o], origin_com[o], origin_sample[o] = u, c, n
        for o in range(K):
            if origin_sample[o] < 0 or n - origin_sample[o] >= n_lags:
                continue
            lag = n - origin_sample[o]
            disp = u - origins[o]
            if remove_com:
                disp = disp - (c - origin_com[o])[sys_of]
            r2 = (disp ** 2).sum(1)
            for b in range(B):
                for s in range(n_species):
                    sel = (sys_of == b) & (species == s)
                    acc[b, s, lag] += r2[sel].sum()
            count[lag] += 1
    return acc, count, jump


def wrap(R, cell):
    """positions wrapped into the cell on all three axes"""
    f = R @ np.linalg.inv(cell)
    return (f - np.floor(f)) @ cell
