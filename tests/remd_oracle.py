"""Test infrastructure, not product code: an fp64 numpy restatement of one temperature replica-exchange attempt of
``schnetpack_b200.exchange.ReplicaExchange`` (csrc/exchange.cu) and of the per-system Langevin kick and Nose-Hoover chain of
``md.LangevinThermostat`` / ``md.NHCThermostat`` with one bath temperature per system, built on tests/nvt_oracle.py.

Layout: K G systems, rung-major (system k G + g is rung k of group g); a pair index is g (K - 1) + k.
"""
from __future__ import annotations

import numpy as np
import torch

import nvt_oracle as NO

REMD_APPLICATION = 2 ** 63          # Philox application index of attempt n: 2^63 + n


def uniforms(seed: int, n: int, n_pairs: int) -> np.ndarray:
    """u = (x + 1/2) 2^-32 of every pair of attempt n, x = word 0 of the draw (pair, 2^63 + n)"""
    x = NO.philox_bits(seed, REMD_APPLICATION + n, n_pairs)[:, 0]
    return (x.astype(np.float64) + 0.5) * 2.0 ** -32


def deltas(U, T, kB: float, K: int, G: int) -> np.ndarray:
    """[G, K - 1] Delta = (1 / (kB T_k) - 1 / (kB T_k+1)) (U_k - U_k+1) of every neighbouring pair, U and T [K G] fp64"""
    U, T = np.asarray(U, np.float64).reshape(K, G), np.asarray(T, np.float64).reshape(K, G)
    beta = 1.0 / (kB * T)
    return ((beta[:-1] - beta[1:]) * (U[:-1] - U[1:])).T


def decide(U, T, kB: float, K: int, G: int, n: int, seed: int):
    """(active, accepted) [G, K - 1] bool of attempt n: pairs (k, k + 1) with k = n (mod 2), accepted iff Delta >= 0 or
    u < exp(Delta)"""
    d = deltas(U, T, kB, K, G)
    active = np.broadcast_to((np.arange(K - 1) % 2) == (n % 2), d.shape)
    u = uniforms(seed, n, G * (K - 1)).reshape(G, K - 1)
    with np.errstate(over="ignore"):
        acc = active & ((d >= 0.0) | (u < np.exp(d)))
    return active, acc


def pairs(decision, G: int):
    """(lower, upper) system indices of the pairs set in ``decision`` [G, K - 1]; the pairs of one attempt are disjoint"""
    g, k = np.nonzero(decision)
    return k * G + g, (k + 1) * G + g


class Exchange:
    """the state of ``ReplicaExchange``: walker [K G], attempted / accepted [G, K - 1], the attempt counter"""

    def __init__(self, K: int, G: int, kB: float, seed: int):
        self.K, self.G, self.kB, self.seed = K, G, kB, seed
        self.walker = np.arange(K * G, dtype=np.int64)
        self.attempted = np.zeros((G, K - 1), np.int64)
        self.accepted = np.zeros((G, K - 1), np.int64)
        self.attempt = 0

    def step(self, U, T):
        """one attempt on the potential energies U [K G] (MD units); returns the decisions [G, K - 1]"""
        K, G = self.K, self.G
        active, acc = decide(U, T, self.kB, K, G, self.attempt, self.seed)
        self.attempted += active
        self.accepted += acc
        lo, hi = pairs(acc, G)
        self.walker[lo], self.walker[hi] = self.walker[hi], self.walker[lo].copy()
        self.attempt += 1
        return acc


def swap(decision, K: int, G: int, sys_ptr, T, momenta, per_atom=(), per_system=()):
    """The configuration swap of the pairs ``decision`` [G, K - 1] on copies of the arrays: momenta [N, 3] fp32 (or None)
    rescaled by sqrt(T_new / T_old) in fp64 and rounded once; every per-atom [N, ...] and per-system [K G, ...] array
    copied.  Returns (momenta, [per_atom], [per_system])."""
    p = None if momenta is None else np.array(momenta, dtype=np.float32)
    pa = [np.array(a) for a in per_atom]
    ps = [np.array(a) for a in per_system]
    T = np.asarray(T, np.float64)
    los, his = pairs(decision, G)
    for x in ps:
        x[los], x[his] = x[his], x[los].copy()
    for lo, hi in zip(los, his) if p is not None or pa else ():
        a = np.arange(sys_ptr[lo], sys_ptr[lo + 1])
        b = np.arange(sys_ptr[hi], sys_ptr[hi + 1])
        if p is not None:
            p_lo, p_hi = p[a].astype(np.float64), p[b].astype(np.float64)
            p[a] = (p_hi * np.sqrt(T[lo] / T[hi])).astype(np.float32)
            p[b] = (p_lo * np.sqrt(T[hi] / T[lo])).astype(np.float32)
        for x in pa:
            x[a], x[b] = x[b].copy(), x[a].copy()
    return p, pa, ps


# ---- per-system thermostats ------------------------------------------------------------------------------------------------
def langevin_kick(p, masses, n_atoms, T_sys, kB: float, c1: float, c2: float, seed: int, app: int):
    """p = c1 p + c2 sqrt(m kB T_s) xi with T_s of the atom's system; xi the normals of ``NO.langevin_normals``"""
    p = np.asarray(p, np.float64)
    z = NO.langevin_normals(seed, app, p.shape[0])
    kbt = np.repeat(kB * np.asarray(T_sys, np.float64), n_atoms)
    return c1 * p + np.sqrt(np.asarray(masses, np.float64) * kbt)[:, None] * c2 * z


class NHCPerSystem:
    """One ``nvt_oracle.NHC`` per system at its own bath temperature; systems are independent, so each advances its slice"""

    def __init__(self, T_sys, time_constant, kB, fs, **kw):
        self.chains = [NO.NHC(float(t), time_constant, kB, fs, **kw) for t in T_sys]

    def init(self, masses, n_atoms, time_step):
        self.ptr = np.concatenate([[0], np.cumsum(n_atoms)])
        for s, th in enumerate(self.chains):
            th.init(np.asarray(masses)[self.ptr[s]:self.ptr[s + 1]], [n_atoms[s]], time_step)

    def apply(self, p):
        p = torch.as_tensor(np.asarray(p, np.float64))
        return torch.cat([th.apply(p[self.ptr[s]:self.ptr[s + 1]]) for s, th in enumerate(self.chains)])

    def chain_state(self):
        return tuple(np.concatenate(x) for x in zip(*(th.chain_state() for th in self.chains)))
