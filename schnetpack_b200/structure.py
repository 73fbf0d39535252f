"""Radial distribution functions and mean-squared displacements of a ``DeviceMD`` run, accumulated inside its captured
step (DESIGN.md section 24).

Both classes are simulation hooks: pass them in ``DeviceMD(..., hooks=[...])``.  They sample the steps
s % every_n_steps == 0 of the device step counter (the first step included), keep fixed-size fp64 accumulators on the
device, send nothing to the host between steps and are carried by ``DeviceMD.state_dict`` (``drain()`` does not touch
them; ``reset()`` zeroes them).

::

    rdf = RadialDistribution(r_max=8.0, n_bins=400, every_n_steps=10)
    msd = MeanSquaredDisplacement(n_lags=2000, every_n_steps=5, origin_every=50)
    md = DeviceMD(model, batch, masses, dt, cutoff, capacity, thermostat=..., hooks=[WrapPositions(10), rdf, msd])
    md.run(200_000)
    r, g = rdf.result()                       # [n_bins], [B, n_pairs, n_bins]
    t, m = msd.result()                       # fs, [B, n_species, n_lags]
    D = msd.diffusion_coefficient(500.0, 5000.0)
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib, ops
from . import properties as P
from .md import FS_MD, _check_every

Tensor = torch.Tensor

__all__ = ["RadialDistribution", "MeanSquaredDisplacement"]

MSD_MAX_SPECIES = 8          # the widest per-species partial pass of csrc/structure.cu


def _species(z: Tensor) -> Tuple[List[int], Tensor]:
    """(sorted atomic numbers present, per-atom species index int32)"""
    zs = sorted(int(v) for v in torch.unique(z.cpu()))
    lut = {v: k for k, v in enumerate(zs)}
    idx = torch.tensor([lut[int(v)] for v in z.cpu().tolist()], dtype=torch.int32)
    return zs, idx


def _counts(species: Tensor, sys_ptr: List[int], n_species: int) -> Tensor:
    """[B, n_species] fp64 number of atoms of every species in every system"""
    out = torch.zeros(len(sys_ptr) - 1, n_species, dtype=torch.float64)
    for b in range(len(sys_ptr) - 1):
        out[b] = torch.bincount(species[sys_ptr[b]:sys_ptr[b + 1]].long(), minlength=n_species).double()
    return out


class RadialDistribution:
    """g_ab(r) per species pair and system, in model length units.

    Pairs are those of the neighbour list at cutoff ``r_max``: ordered (i, j, S) with |R_j - R_i + S cell| < r_max,
    (i = j, S = 0) excluded and self-images included, so ``r_max`` may exceed half the cell width.  Bin k covers
    [k dr, (k + 1) dr), dr = r_max / n_bins, and

        g_ab(r_k) = < V n_ab(k) > / (N_a N_b 4 pi / 3 (r_{k+1}^3 - r_k^3))

    with n_ab(k) the ordered pairs with Z_i = a, Z_j = b in bin k (for a != b one direction only), V the frame's
    volume (the run's MD cell when it keeps one, so NPT volumes enter frame by frame; else the batch cell) and the
    average over sampled frames.  The normalisation uses N_a N_b also for like pairs, so an ideal gas of N_a atoms gives
    g_aa -> (N_a - 1) / N_a away from the self-image shells.  ``pairs=None`` takes every unordered species pair present
    in the batch plus the total (all atoms, listed as (0, 0)); a list of (Z_a, Z_b) takes those pairs ((0, 0) for the
    total).  Ring-polymer runs fold the beads of each system together (the bead-averaged, quantum g(r)).  Every system
    must be periodic on all three axes."""

    def __init__(self, r_max: float, n_bins: int, every_n_steps: int = 1,
                 pairs: Optional[Sequence[Tuple[int, int]]] = None):
        if not float(r_max) > 0.0:
            raise ValueError(f"RadialDistribution: r_max must be positive, got {r_max}")
        if int(n_bins) != n_bins or int(n_bins) < 1:
            raise ValueError(f"RadialDistribution: n_bins must be an integer >= 1, got {n_bins}")
        self.r_max = float(r_max)
        self.n_bins = int(n_bins)
        self.every_n_steps = _check_every(every_n_steps, "RadialDistribution")
        self.requested = None if pairs is None else [(int(a), int(b)) for a, b in pairs]
        if self.requested is not None and not self.requested:
            raise ValueError("RadialDistribution: pairs must be None or a non-empty list of (Z_a, Z_b)")
        self._md = None

    # ---- set-up by DeviceMD ------------------------------------------------------------------------------------------
    def _bind(self, md):
        if self._md is not None:
            raise ValueError("RadialDistribution: this hook already belongs to a DeviceMD")
        s = md.systems
        base = md._rp_base if md._rp_base is not None else s
        n_sys, B, dev = s.n_sys, base.n_sys, md.positions.device
        static = md.static
        if P.cell not in static:
            raise ValueError("DeviceMD: RadialDistribution needs a periodic batch with a '_cell'")
        cell = static[P.cell].reshape(-1, 3, 3)
        vcell, vscale = (md.cell, md.p_conv ** 3) if md.cell is not None else (cell.to(torch.float64).contiguous(), 1.0)
        md._check_periodic(n_sys, torch.linalg.det(vcell), "RadialDistribution")
        if cell.shape[0] not in (1, n_sys):
            raise ValueError(f"DeviceMD: '_cell' has {cell.shape[0]} cells for {n_sys} systems")
        # the fp32 cell the grid reads: the live model cell when there is one per system (it follows a barostat)
        self._cell = cell if cell.shape[0] == n_sys and cell.is_contiguous() else cell.expand(n_sys, 3, 3).contiguous()
        self._pbc = static[P.pbc].reshape(-1, 3).to(torch.uint8).expand(n_sys, 3).contiguous()
        self._vcell, self._vstride, self._vscale = vcell, 9 if vcell.shape[0] > 1 else 0, float(vscale)
        z = static[P.Z][:base.n_atoms]
        zs, species = _species(z)
        T = len(zs)
        if self.requested is None:
            pairs = [(zs[a], zs[b]) for a in range(T) for b in range(a, T)] + [(0, 0)]
        else:
            pairs = list(dict.fromkeys(self.requested))
            for a, b in pairs:
                if (a, b) != (0, 0) and (a not in zs or b not in zs):
                    raise ValueError(f"RadialDistribution: pair ({a}, {b}) names a species not in the batch ({zs})")
        slot_of = torch.full((T, T), -1, dtype=torch.int32)
        total = -1
        for k, (a, b) in enumerate(pairs):
            if (a, b) == (0, 0):
                total = k
            else:
                slot_of[zs.index(a), zs.index(b)] = k
        self.pairs = pairs
        self.species = zs
        n_rep = n_sys // B
        self._type = species.repeat(n_rep).to(dev)
        self._slot_of = slot_of.reshape(-1).to(dev)
        self._total, self._n_types, self._n_out = total, T, B
        # N_a N_b per (system, pair): the total pair counts all N atoms on both sides
        sys_ptr = base.sys_ptr.tolist()
        n_of = _counts(species, sys_ptr, T)
        n_tot = n_of.sum(1)
        na = torch.stack([n_tot if (a, b) == (0, 0) else n_of[:, zs.index(a)] for a, b in pairs], 1)
        nb = torch.stack([n_tot if (a, b) == (0, 0) else n_of[:, zs.index(b)] for a, b in pairs], 1)
        self._na, self._nb = na, nb
        self._n_replicas = n_rep
        self._acc = torch.zeros(B, len(pairs), self.n_bins, dtype=torch.float64, device=dev)
        self._volume = torch.zeros(B, dtype=torch.float64, device=dev)
        self._frames = torch.zeros(1, dtype=torch.int64, device=dev)
        nbytes = int(_lib.lib().spk_rdf_workspace_bytes(s.n_atoms, n_sys, len(pairs), self.n_bins))
        self._ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)     # the count region must start at zero
        self._md = md

    def apply(self, md):
        s = md.systems
        R = md.model_positions
        _lib.call("spk_rdf_accumulate", ops._p(R), ops._p(self._cell), ops._p(self._pbc), ops._p(s.sys_ptr), s.n_atoms,
                  s.n_sys, ops._p(self._type), self._n_types, ops._p(self._slot_of), self._total, len(self.pairs),
                  self.r_max, self.n_bins, ops._p(self._vcell), self._vstride, self._vscale, self._n_out,
                  ops._p(md._rec_counter), self.every_n_steps, ops._p(self._acc), ops._p(self._volume),
                  ops._p(self._frames), ops._p(self._ws), self._ws.numel(), ops._stream(),
                  launches=None if s.n_atoms else 2)

    def _state(self) -> Dict[str, Tensor]:
        return {"acc": self._acc, "volume": self._volume, "frames": self._frames}

    # ---- results -----------------------------------------------------------------------------------------------------
    def _need_md(self):
        if self._md is None:
            raise ValueError("RadialDistribution: the hook is not attached to a run; pass it in DeviceMD(..., hooks=...)")
        return self._md

    def reset(self):
        """zero the accumulators (the next sampled step starts a new average)"""
        self._need_md()
        for t in self._state().values():
            t.zero_()

    @property
    def frames(self) -> int:
        """sampled frames so far (one host read)"""
        self._need_md()
        return int(self._frames.item())

    def bin_edges(self) -> Tensor:
        return torch.linspace(0.0, self.r_max, self.n_bins + 1, dtype=torch.float64)

    def result(self, average: bool = False) -> Tuple[Tensor, Tensor]:
        """(r, g): bin centres [n_bins] and g(r) [B, n_pairs, n_bins] fp64 on the host for the pairs ``self.pairs``;
        ``average`` takes the mean over the systems, [n_pairs, n_bins]."""
        frames = self.frames
        if frames < 1:
            raise ValueError("RadialDistribution: no frame has been sampled yet")
        e = self.bin_edges()
        shell = 4.0 * math.pi / 3.0 * (e[1:] ** 3 - e[:-1] ** 3)
        g = self._acc.cpu() / (frames * self._n_replicas * (self._na * self._nb)[:, :, None] * shell)
        r = 0.5 * (e[1:] + e[:-1])
        return r, (g.mean(0) if average else g)

    def coordination(self, average: bool = False) -> Tensor:
        """running coordination numbers n_ab(r_{k+1}) = 4 pi rho_b int_0^r_{k+1} g_ab r^2 dr with rho_b = N_b / <V>:
        the mean number of b atoms within r_{k+1} of an a atom, [B, n_pairs, n_bins] (or the mean over systems)"""
        if self.frames < 1:
            raise ValueError("RadialDistribution: no frame has been sampled yet")
        n = torch.cumsum(self._acc.cpu(), -1) / (self._na[:, :, None] * self._volume.cpu()[:, None, None])
        return n.mean(0) if average else n


class MeanSquaredDisplacement:
    """MSD(t) per species and system in MD length units^2, and self-diffusion coefficients from it.

    Every sampled step (s % every_n_steps == 0) each atom (ring polymers: its centroid) moves its fp64 unwrapped
    position u by the displacement since the last sample, with the fractional components of the periodic axes wrapped to
    [-1/2, 1/2) in the current cell, so ``WrapPositions`` and barostat rescaling do not enter.  A displacement longer
    than half the shortest cell height cannot be unwrapped; it sets a device flag that ``DeviceMD.run`` turns into an
    error.  Every ``origin_every`` samples u is stored as a time origin in a ring of ceil(n_lags / origin_every) slots;
    each sample adds |u - u_o - (com - com_o)|^2 (the mass-weighted centre-of-mass shift of the system only with
    ``remove_com``) for every held origin into the sum of lag = sample - origin sample, per system and species, with a
    count per lag.  MSD = sum / (count N_species).  Open and periodic systems, at most 8 species."""

    def __init__(self, n_lags: int, every_n_steps: int = 1, origin_every: int = 1, remove_com: bool = True):
        if int(n_lags) != n_lags or int(n_lags) < 1:
            raise ValueError(f"MeanSquaredDisplacement: n_lags must be an integer >= 1, got {n_lags}")
        if int(origin_every) != origin_every or int(origin_every) < 1:
            raise ValueError(f"MeanSquaredDisplacement: origin_every must be an integer >= 1, got {origin_every}")
        self.n_lags = int(n_lags)
        self.every_n_steps = _check_every(every_n_steps, "MeanSquaredDisplacement")
        self.origin_every = int(origin_every)
        self.n_slots = -(-self.n_lags // self.origin_every)
        self.remove_com = bool(remove_com)
        self._md = None

    def _bind(self, md):
        if self._md is not None:
            raise ValueError("MeanSquaredDisplacement: this hook already belongs to a DeviceMD")
        base = md._rp_base if md._rp_base is not None else md.systems
        N, B, dev = base.n_atoms, base.n_sys, md.positions.device
        zs, species = _species(md.static[P.Z][:N])
        if len(zs) > MSD_MAX_SPECIES:
            raise NotImplementedError(f"MeanSquaredDisplacement: {len(zs)} species, at most {MSD_MAX_SPECIES}")
        self.species = zs
        self._species = species.to(dev)
        self._n_of = _counts(species, base.sys_ptr.tolist(), len(zs))
        self._base = base
        # the cell of the unwrapping: the MD cell when the run keeps one (it follows the barostat), else the batch cell
        pbc = md.static.get(P.pbc)
        self._cell = self._pbc = None
        if pbc is not None and bool(pbc.any()):
            if md.cell is not None:
                cell = md.cell
            else:
                cell = (md.static[P.cell].reshape(-1, 3, 3).to(torch.float64) / md.p_conv).contiguous()
            self._cell, self._pbc = cell, pbc.reshape(-1, 3).to(torch.uint8).contiguous()
        K, L, S = self.n_slots, self.n_lags, len(zs)
        self._track = torch.zeros(N, 6, dtype=torch.float64, device=dev)
        self._origins = torch.zeros(K, N, 3, dtype=torch.float64, device=dev)
        self._origin_com = torch.zeros(K, B, 3, dtype=torch.float64, device=dev)
        self._acc = torch.zeros(B, S, L, dtype=torch.float64, device=dev)
        self._count = torch.zeros(L, dtype=torch.int64, device=dev)
        self._meta = torch.zeros(2, dtype=torch.int64, device=dev)
        nbytes = int(_lib.lib().spk_msd_workspace_bytes(N, B, S, K))
        self._ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        self.dt_fs = self.every_n_steps * md.dt / FS_MD
        self._md = md

    def apply(self, md):
        b, cell, pbc = self._base, self._cell, self._pbc
        _lib.call("spk_msd_accumulate", ops._p(md.positions), b.n_atoms, md._n_replicas(), ops._p(b.masses),
                  ops._p(b.idx_m), ops._p(b.sys_ptr), b.n_sys, ops._p(self._species), len(self.species), ops._p(cell),
                  0 if cell is None or cell.shape[0] == 1 else 9, ops._p(pbc), 0 if pbc is None or pbc.shape[0] == 1 else 3,
                  1 if self.remove_com else 0, self.n_lags, self.origin_every, self.n_slots, ops._p(md._rec_counter),
                  self.every_n_steps, ops._p(self._track), ops._p(self._origins), ops._p(self._origin_com),
                  ops._p(self._acc), ops._p(self._count), ops._p(self._meta), ops._p(self._ws), self._ws.numel(),
                  ops._stream(), launches=7 if self.remove_com else 5)

    def _state(self) -> Dict[str, Tensor]:
        return {"track": self._track, "origins": self._origins, "origin_com": self._origin_com, "acc": self._acc,
                "count": self._count, "meta": self._meta}

    def _check(self):
        """one host read per run: raise if an atom moved more than half a cell height between two samples"""
        if int(self._meta[1].item()):
            raise RuntimeError(
                "MeanSquaredDisplacement: an atom moved more than half the shortest cell height between two samples; "
                "its displacement cannot be unwrapped and the MSD is invalid from that sample on -- sample more often "
                "(smaller every_n_steps)")

    # ---- results -----------------------------------------------------------------------------------------------------
    def _need_md(self):
        if self._md is None:
            raise ValueError("MeanSquaredDisplacement: the hook is not attached to a run; pass it in "
                             "DeviceMD(..., hooks=...)")
        return self._md

    def reset(self):
        """zero the accumulators and the unwrapped positions (the next sampled step is sample 0 again)"""
        self._need_md()
        for t in self._state().values():
            t.zero_()

    @property
    def samples(self) -> int:
        self._need_md()
        return int(self._meta[0].item())

    def result(self) -> Tuple[Tensor, Tensor]:
        """(t, msd): lag times in fs [n_lags] and MSD [B, n_species, n_lags] fp64 on the host (NaN where no origin has
        reached the lag yet or the system has no atom of the species), species ``self.species``"""
        self._need_md()
        t = torch.arange(self.n_lags, dtype=torch.float64) * self.dt_fs
        count = self._count.cpu().double()
        m = self._acc.cpu() / (count * self._n_of[:, :, None])
        return t, m

    def diffusion_coefficient(self, t_min_fs: float, t_max_fs: float) -> Tensor:
        """Self-diffusion coefficients [B, n_species]: the least-squares slope of MSD(t) over the lags with
        t_min_fs <= t <= t_max_fs, divided by 6, in MD length units^2 per fs"""
        t, m = self.result()
        sel = (t >= float(t_min_fs)) & (t <= float(t_max_fs)) & (self._count.cpu() > 0)
        if int(sel.sum()) < 2:
            raise ValueError(f"MeanSquaredDisplacement: fewer than two sampled lags in [{t_min_fs}, {t_max_fs}] fs")
        t, m = t[sel], m[..., sel]
        tc = t - t.mean()
        slope = ((m - m.mean(-1, keepdim=True)) * tc).sum(-1) / (tc * tc).sum()
        return slope / 6.0
