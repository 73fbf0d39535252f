"""Phonons of crystals on the device: force constants from displaced supercells, dynamical matrices at any wave vector,
phonon frequencies and modes, densities of states and harmonic thermodynamics (DESIGN.md section 23).

The reference's users get phonons from ASE's ``Phonons`` through ``SpkCalculator``, one displaced supercell at a time.
``DevicePhonons`` builds the supercell of every primitive cell of a batch and displaces only the atoms of the primitive
cell at translation 0, with the replica batch, the captured step and the kernels of ``DeviceVibrations``
(``csrc/vibrations.cu`` with a per-system count of displaced atoms): 3 n displaced coordinates per system instead of
the 3 n L of a whole-supercell Hessian.  From the force constants, ``csrc/phonons.cu`` symmetrises and applies the
acoustic sum rule, builds the minimum-image table of the supercell and forms the dynamical matrix at any q, the density
of states and the thermodynamics.  Eigensystems are ``torch.linalg.eigh`` in fp64, outside the graph.
"""
from __future__ import annotations

import itertools
from ctypes import c_int32
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib, ops
from . import properties as P
from .md import _CapturedEvaluation, _batch_layout, replicate_batch
from .units import _UNITS
from .vibrations import _HBAR_OMEGA, _INVCM, DEFAULT_MAX_REPLICA_ATOMS

__all__ = ["DevicePhonons", "monkhorst_pack", "q_path", "supercell_translations"]

Tensor = torch.Tensor
# two images of an atom pair are tied when their distances differ by less than this (Angstrom)
TIE_TOLERANCE = 1e-5
# largest dynamical-matrix chunk of one ``spk_ph_dynmat`` call: q-points are processed in chunks of at most this many bytes
DYNMAT_BYTES = 1 << 28
# and of at most this many matrices: the batched eigensolver rejects batches of 32 768 6x6 complex matrices (cusolver,
# torch 2.11 on an H100) and takes 4 096
EIGH_MATRICES = 1 << 12
_KB = _UNITS["kB"]


def _supercell_matrix(supercell) -> np.ndarray:
    m = np.asarray(supercell, dtype=np.float64)
    if m.shape == (3,):
        m = np.diag(m)
    if m.shape != (3, 3):
        raise ValueError(f"DevicePhonons: supercell must be 3 integers or an integer 3x3 matrix, got shape {m.shape}")
    if not np.array_equal(m, np.round(m)):
        raise ValueError(f"DevicePhonons: the supercell matrix must be integer, got {m.tolist()}")
    m = np.round(m).astype(np.int64)
    det = int(round(np.linalg.det(m)))
    if det <= 0:
        raise ValueError(f"DevicePhonons: the supercell matrix must have det > 0, got det = {det}")
    return m


def supercell_translations(supercell) -> tuple:
    """(lattice [L, 3] int64, neg [L] int64) for the supercell matrix M (rows of the supercell = M . cell, L = det M):
    the L primitive translations n with n M^-1 in [0, 1)^3, the zero translation first, and the index of -n modulo
    the supercell.  Exact integer arithmetic: n M^-1 = n adj(M) / det."""
    M = _supercell_matrix(supercell)
    det = int(round(np.linalg.det(M)))
    adj = np.round(np.linalg.inv(M) * det).astype(np.int64)
    assert np.array_equal(M @ adj, det * np.eye(3, dtype=np.int64))
    lo, hi = np.minimum(M, 0).sum(0), np.maximum(M, 0).sum(0)
    box = np.array(list(itertools.product(*[range(int(a), int(b) + 1) for a, b in zip(lo, hi)])), dtype=np.int64)
    f = box @ adj
    lattice = box[np.all((f >= 0) & (f < det), axis=1)]
    lattice = lattice[np.argsort(np.any(lattice != 0, axis=1), kind="stable")]     # zero first
    assert lattice.shape[0] == det and not lattice[0].any()

    def key(n):
        g = (n @ adj) % det
        return tuple(((g @ M) // det).tolist())

    index = {key(n): i for i, n in enumerate(lattice)}
    neg = np.array([index[key(-n)] for n in lattice], dtype=np.int64)
    return lattice, neg


def monkhorst_pack(mesh: Sequence[int], shifted: bool = False) -> Tensor:
    """[n1 n2 n3, 3] fp64 q-points (i_k + s / 2) / n_k, s = 1 if ``shifted`` else 0, in reduced reciprocal coordinates
    wrapped to [-1/2, 1/2).  The unshifted mesh contains Gamma."""
    mesh = [int(n) for n in mesh]
    if len(mesh) != 3 or min(mesh) < 1:
        raise ValueError(f"monkhorst_pack: mesh must be 3 positive integers, got {mesh}")
    idx = torch.stack(torch.meshgrid(*[torch.arange(n, dtype=torch.float64) for n in mesh], indexing="ij"), -1)
    q = (idx.reshape(-1, 3) + (0.5 if shifted else 0.0)) / torch.tensor(mesh, dtype=torch.float64)
    return q - torch.floor(q + 0.5)


def q_path(corners, n_per_segment: int) -> Tensor:
    """[(K - 1) n + 1, 3] fp64 q-points along the K ``corners`` (reduced reciprocal coordinates): n points per segment,
    linearly interpolated from its start, and the last corner"""
    c = torch.as_tensor(np.asarray(corners, dtype=np.float64))
    n = int(n_per_segment)
    if c.dim() != 2 or c.shape[1] != 3 or c.shape[0] < 2 or n < 1:
        raise ValueError("q_path: corners must be [K >= 2, 3] and n_per_segment >= 1")
    t = torch.arange(n, dtype=torch.float64)[:, None] / n
    seg = [c[k] + t * (c[k + 1] - c[k]) for k in range(c.shape[0] - 1)]
    return torch.cat(seg + [c[-1:]])


def _as_q(q) -> Tensor:
    q = torch.as_tensor(q, dtype=torch.float64)
    if q.dim() == 1:
        q = q[None]
    if q.dim() != 2 or q.shape[1] != 3:
        raise ValueError(f"DevicePhonons: q must be [Q, 3] reduced coordinates, got shape {tuple(q.shape)}")
    return q


class DevicePhonons(_CapturedEvaluation):
    """Phonons of every crystal of ``batch`` (B primitive cells, ragged sizes allowed, periodic on all three axes) by
    ASE's finite-difference supercell method.  ``supercell`` is one integer matrix M (3 ints for a diagonal one), det M
    > 0, applied to every system: the supercell's rows are M . cell and it holds L = det M primitive cells, supercell atom
    j = l n + b being primitive atom b translated by ``lattice[l]`` (``supercell_translations``).  ``masses`` [N] are the
    primitive atoms' masses in amu; ``delta`` is in Angstrom; ``position_conversion`` / ``energy_conversion`` turn model
    lengths and energies into Angstrom and eV.  ``cutoff`` and ``capacity`` (the pair capacity of the supercell batch)
    size the device neighbour list, which is rebuilt on the replica batch in every step.

    Only the n atoms of the primitive cell at translation 0 are displaced (``nfree`` = 2 or 4 as in DeviceVibrations);
    ``max_replica_atoms`` bounds the replica batch and so the coordinates per chunk; ``run`` replays the captured step
    once per chunk.  Then ``symmetrize`` rounds (ASE's Phonons.read) each symmetrise the force constants and, with
    ``acoustic``, restore the acoustic sum rule; ``symmetrize=0, acoustic=False`` keeps the raw finite differences.

    Results after ``run``: ``force_constants`` [sum_m n_m n_m L, 3, 3] fp64 in model units (row a n L + j, block
    [alpha, beta] = d2E / dR_{a alpha} dR_{j beta}), and ``dynamical_matrices``, ``frequencies``, ``mode``, ``dos`` and
    ``thermodynamics`` at any q in reduced coordinates of each system's reciprocal primitive lattice."""

    def __init__(self, model: torch.nn.Module, batch: Dict[str, Tensor], masses: Tensor, supercell, cutoff: float,
                 capacity: int, delta: float = 0.01, nfree: int = 2, position_conversion: float = 1.0,
                 energy_conversion: float = 1.0, max_replica_atoms: Optional[int] = None, acoustic: bool = True,
                 symmetrize: int = 10, use_graph: bool = True):
        if int(nfree) not in (2, 4):
            raise ValueError(f"DevicePhonons: nfree must be 2 or 4 (ase/vibrations/vibrations.py), got {nfree}")
        if not float(delta) > 0.0:
            raise ValueError(f"DevicePhonons: delta must be > 0, got {delta}")
        if int(symmetrize) < 0:
            raise ValueError(f"DevicePhonons: symmetrize must be >= 0, got {symmetrize}")
        from .parallel import PartitionedPotential

        if isinstance(model, PartitionedPotential):
            raise NotImplementedError("DevicePhonons: PartitionedPotential is not supported (one GPU per batch)")
        from .ensemble import members_of

        if members_of(model) is not None:
            raise NotImplementedError("DevicePhonons: ensembles are not supported; pass a single model")
        outputs = getattr(model, "model_outputs", None)
        if outputs is not None:
            missing = [p for p in (self.energy_key, self.force_key) if p not in outputs]
            if missing:
                raise ValueError(f"DevicePhonons: the model does not output {missing} (it outputs {sorted(outputs)})")
        M = _supercell_matrix(supercell)
        pos = batch[P.R]
        if pos.device.type != "cuda":
            raise ValueError("DevicePhonons needs a CUDA batch (no CPU fallback)")
        if pos.dtype != torch.float32 or not pos.is_contiguous():
            raise ValueError("DevicePhonons: '_positions' must be a contiguous float32 tensor")
        dev = pos.device
        idx_m, n_sys = _batch_layout(batch)
        n = pos.shape[0]
        masses = torch.as_tensor(masses).reshape(-1)
        if masses.shape[0] != n:
            raise ValueError(f"DevicePhonons: {masses.shape[0]} masses for {n} atoms")
        if P.cell not in batch or P.pbc not in batch:
            raise ValueError("DevicePhonons: the batch needs '_cell' and '_pbc' (crystals periodic on all three axes)")
        pbc = batch[P.pbc].reshape(-1, 3).expand(n_sys, 3).cpu()
        if not bool(pbc.all()):
            bad = [m for m in range(n_sys) if not bool(pbc[m].all())]
            raise ValueError(f"DevicePhonons: systems {bad} are not periodic on all three axes")
        cell32 = batch[P.cell].reshape(-1, 3, 3).expand(n_sys, 3, 3).to(torch.float32).cpu()

        self.nfree, self.p_conv, self.e_conv = int(nfree), float(position_conversion), float(energy_conversion)
        self.delta, self.acoustic, self.symmetrize = float(delta), bool(acoustic), int(symmetrize)
        self.supercell = M
        lattice, neg = supercell_translations(M)
        L = lattice.shape[0]
        self.n_cells = L
        prim_ptr = ops.segment_ptr(idx_m, n_sys)
        sizes = (prim_ptr[1:] - prim_ptr[:-1]).to(torch.int64).cpu()                 # one host read, at set-up
        if int(sizes.min()) < 1:
            raise ValueError("DevicePhonons: every system needs at least one atom")
        self.sizes = sizes.tolist()
        self.n_atoms, self.n_sys, self.max_atoms = n, n_sys, max(self.sizes)

        # the supercells, in fp64 on the host: atom l n + b = x_b + lattice[l] . cell, then rounded to fp32
        x64 = pos.detach().cpu().to(torch.float64)
        A64 = cell32.to(torch.float64)
        lat = torch.as_tensor(lattice, dtype=torch.float64)
        Mt = torch.as_tensor(M, dtype=torch.float64)
        ptr = [0] + torch.cumsum(sizes, 0).tolist()
        z = batch[P.Z].cpu()
        sc_pos, sc_z = [], []
        for m in range(n_sys):
            A = A64[m]
            t = lat[:, 0:1] * A[0] + lat[:, 1:2] * A[1] + lat[:, 2:3] * A[2]             # [L, 3]
            sc_pos.append((x64[ptr[m]:ptr[m + 1]][None] + t[:, None]).reshape(-1, 3))
            sc_z.append(z[ptr[m]:ptr[m + 1]].repeat(L))
        super_cell64 = torch.matmul(Mt, A64).contiguous()
        sc_sizes = sizes * L
        super_batch = {
            P.Z: torch.cat(sc_z).to(dev), P.R: torch.cat(sc_pos).to(torch.float32).to(dev),
            P.cell: super_cell64.to(torch.float32).to(dev), P.pbc: torch.ones(n_sys, 3, dtype=torch.bool, device=dev),
            P.idx_m: torch.repeat_interleave(torch.arange(n_sys), sc_sizes).to(dev), P.n_atoms: sc_sizes.to(dev)}
        self.supercell_batch = {k: v.clone() for k, v in super_batch.items()}

        self.sc_idx_m, _ = self._setup(model, super_batch, cutoff, capacity, use_graph)
        base = self.static
        n_super = base[P.R].shape[0]
        n_coords = 3 * self.max_atoms
        limit = DEFAULT_MAX_REPLICA_ATOMS if max_replica_atoms is None else int(max_replica_atoms)
        self.n_cols = max(1, min(n_coords, limit // max(1, self.nfree * n_super)))
        self.n_copies = self.n_cols * self.nfree
        self.n_chunks = -(-n_coords // self.n_cols)
        fc_rows = sizes * sizes * L
        fc_ptr = torch.zeros(n_sys + 1, dtype=torch.int64)
        fc_ptr[1:] = torch.cumsum(fc_rows, 0)
        self.n_rows = int(fc_ptr[-1])
        dyn_ptr = torch.zeros(n_sys + 1, dtype=torch.int64)
        dyn_ptr[1:] = torch.cumsum(9 * sizes * sizes, 0)
        self._dyn_ptr_host = dyn_ptr.tolist()
        self.dyn_ptr = dyn_ptr.to(dev)

        self.base_positions = base[P.R]
        self.static = replicate_batch(base, self.n_copies, n_sys)
        self.nl.capacity *= self.n_copies                # ``capacity`` is that of the supercell batch, once per copy
        f64 = dict(dtype=torch.float64, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        self.steps = torch.zeros(self.n_copies, n_sys, **f64)
        self.counter = torch.zeros(2, dtype=torch.int64, device=dev)
        self.h_raw = torch.zeros(9 * self.n_rows, **f64)
        self.force_constants = torch.zeros(self.n_rows, 3, 3, **f64)
        self._work = torch.zeros(self.n_rows, 3, 3, **f64)
        self.img_count = torch.zeros(self.n_rows, **i32)
        self.img_lattice = torch.zeros(self.n_rows, _lib.PH_MAX_IMAGES, 3, **i32)
        self.masses = masses.to(dev, torch.float64).contiguous()
        self.prim_ptr = prim_ptr
        self.sc_ptr = ops.segment_ptr(self.sc_idx_m, n_sys)
        self.fc_ptr = fc_ptr.to(dev)
        self._hraw_ptr = (9 * fc_ptr).to(dev)      # the finite differences of system m start at 9 fc_ptr[m]
        self.n_displaced = sizes.to(dev)
        self.lattice = torch.as_tensor(lattice).to(**i32)
        self.neg = torch.as_tensor(neg).to(**i32)
        # the kernels read these by raw pointer: row-major, whatever strides the host operations returned
        self.positions64 = x64.contiguous().to(dev)
        self.cell64 = A64.contiguous().to(dev)
        self.super_cell64 = super_cell64.to(dev)
        self.super_inv = torch.linalg.inv(super_cell64).contiguous().to(dev)
        # plane spacings of the supercell: volume / |c_i x c_j|
        vol = torch.det(super_cell64).abs()
        c = super_cell64
        cross = torch.stack([torch.linalg.cross(c[:, 1], c[:, 2]), torch.linalg.cross(c[:, 2], c[:, 0]),
                             torch.linalg.cross(c[:, 0], c[:, 1])], 1)
        self.heights = (vol[:, None] / cross.norm(dim=2)).contiguous().to(dev)
        self._freq_cache: Optional[tuple] = None
        self._calculate()                          # shapes of the outputs, buffers of the captured step
        p = ops._p
        self._params = _lib.VibParams(
            p(self.base_positions), p(self.static[P.R]), p(self.steps), p(self.counter), p(self.forces), None, None,
            p(self.sc_idx_m), p(self.sc_ptr), p(self.n_displaced), p(self._hraw_ptr), None, p(self.h_raw), None, None, None,
            None, n_super, n_sys, self.n_cols, self.nfree, self.max_atoms * L, self.delta / self.p_conv,
            self.e_conv / self.p_conv ** 2)
        self._ph = _lib.PhononParams(
            p(self.h_raw), p(self.force_constants), p(self._work), p(self.prim_ptr), p(self.fc_ptr), p(self.lattice),
            p(self.neg), p(self.positions64), p(self.cell64), p(self.super_cell64), p(self.super_inv), p(self.heights),
            p(self.masses), p(self.img_count), p(self.img_lattice), (c_int32 * 9)(*M.reshape(-1).tolist()), n_sys, n, self.n_rows, L,
            self.max_atoms, self.symmetrize, int(self.acoustic), 0, TIE_TOLERANCE / self.p_conv,
            self.e_conv / self.p_conv ** 2)

    # ---- the captured step ----------------------------------------------------------------------------------------------
    def _step(self):
        ops.vib_displace(self._params)
        self._calculate()
        ops.vib_assemble(self._params)

    def _step_state(self) -> Dict[str, object]:
        return dict(positions=self.static[P.R], steps=self.steps, counter=self.counter, h_raw=self.h_raw,
                    **self._evaluation_state())

    def run(self):
        """Evaluate every displaced supercell (``n_chunks`` replays of the captured step), then form the force constants
        and the minimum-image table."""
        self.counter.zero_()
        self._run_steps(self.n_chunks)
        rounds = self.symmetrize if self.acoustic else min(self.symmetrize, 1)
        ops.ph_force_constants(self._ph, rounds)
        ops.ph_images(self._ph)
        self.check_neighbor_list()
        most = int(self.img_count.max())
        if most > _lib.PH_MAX_IMAGES:
            raise RuntimeError(f"DevicePhonons: an atom pair has {most} equidistant supercell images, more than the "
                               f"{_lib.PH_MAX_IMAGES} the table holds")
        self._freq_cache = None

    # ---- dynamical matrices and eigensystems (outside the graph) --------------------------------------------------------
    def _chunks(self, q: Tensor):
        per_q = 16 * self._dyn_ptr_host[-1]
        step = max(1, min(DYNMAT_BYTES // per_q, EIGH_MATRICES // self.n_sys))
        for lo in range(0, q.shape[0], step):
            yield ops.ph_dynmat(self._ph, q[lo:lo + step], self.dyn_ptr, self._dyn_ptr_host[-1])

    def _blocks(self, dyn: Tensor, m: int) -> Tensor:
        n3 = 3 * self.sizes[m]
        return dyn[:, self._dyn_ptr_host[m]:self._dyn_ptr_host[m + 1]].view(-1, n3, n3)

    def dynamical_matrices(self, q) -> List[Tensor]:
        """per system m: [Q, 3 n_m, 3 n_m] complex128 mass-weighted dynamical matrices D(q) in eV / (Angstrom^2 amu)"""
        q = _as_q(q).to(self.dyn_ptr.device)
        chunks = list(self._chunks(q))
        return [torch.cat([self._blocks(d, m) for d in chunks]) for m in range(self.n_sys)]

    def _eigh(self, q: Tensor, vectors: bool):
        """eigenvalues [Q, 3 N] (system m at 3 prim_ptr[m]) of (D + D^H) / 2, and per system the eigenvectors when asked;
        systems of one size share one batched eigh"""
        vals, vecs = [], [[] for _ in range(self.n_sys)]
        for dyn in self._chunks(q):
            w = torch.empty(dyn.shape[0], 3 * self.n_atoms, dtype=torch.float64, device=dyn.device)
            for size in sorted(set(self.sizes)):
                ids = [m for m in range(self.n_sys) if self.sizes[m] == size]
                d = torch.stack([self._blocks(dyn, m) for m in ids], 1)
                d = 0.5 * (d + d.transpose(-1, -2).conj())
                if vectors:
                    e, v = torch.linalg.eigh(d)
                    for k, m in enumerate(ids):
                        vecs[m].append(v[:, k])
                else:
                    e = torch.linalg.eigvalsh(d)
                ptr = [3 * sum(self.sizes[:m]) for m in ids]
                for k, m in enumerate(ids):
                    w[:, ptr[k]:ptr[k] + 3 * size] = e[:, k]
            vals.append(w)
        return torch.cat(vals), ([torch.cat(v) for v in vecs] if vectors else None)

    def frequencies(self, q) -> Tensor:
        """[Q, 3 N] phonon frequencies in cm^-1 at q [Q, 3]: system m at columns 3 prim_ptr[m] .. 3 prim_ptr[m+1],
        ascending per (q, system); an imaginary frequency is returned as the negative of its magnitude"""
        w, _ = self._eigh(_as_q(q).to(self.dyn_ptr.device), False)
        return torch.sign(w) * torch.sqrt(torch.abs(w)) * (_HBAR_OMEGA / _INVCM)

    def mode(self, q, m: int) -> Tensor:
        """[3 n_m, n_m, 3] complex normal modes of system m at one q: mass-weighted eigenvectors divided by sqrt(mass), in
        the order of ``frequencies``"""
        q = _as_q(q)
        if q.shape[0] != 1:
            raise ValueError("DevicePhonons.mode: one q-point at a time")
        _, vecs = self._eigh(q.to(self.dyn_ptr.device), True)
        v = vecs[m][0]
        lo, hi = int(self.prim_ptr[m]), int(self.prim_ptr[m + 1])
        inv_sqrt_m = (1.0 / torch.sqrt(self.masses[lo:hi])).repeat_interleave(3)
        return (v.T * inv_sqrt_m).reshape(3 * (hi - lo), hi - lo, 3)

    def _mesh_frequencies(self, mesh) -> Tensor:
        key = tuple(int(x) for x in mesh)
        if self._freq_cache is None or self._freq_cache[0] != key:
            self._freq_cache = (key, self.frequencies(monkhorst_pack(key)).contiguous())
        return self._freq_cache[1]

    def dos(self, mesh: Sequence[int], grid, width: float) -> Tensor:
        """[B, G] phonon density of states per primitive cell, in states per cm^-1, on ``grid`` [G] (cm^-1): the
        frequencies of the Gamma-centred ``mesh`` broadened by Gaussians of standard deviation ``width`` (cm^-1).  Each
        system's g integrates to 3 n_m over a grid that covers its spectrum."""
        if not float(width) > 0.0:
            raise ValueError(f"DevicePhonons.dos: width must be > 0, got {width}")
        freq = self._mesh_frequencies(mesh)
        grid = torch.as_tensor(grid, dtype=torch.float64).reshape(-1).to(freq.device).contiguous()
        return ops.ph_dos(freq, self.prim_ptr, grid, float(width))

    def thermodynamics(self, mesh: Sequence[int], temperatures, min_frequency: float = 1.0) -> Dict[str, Tensor]:
        """Harmonic thermodynamics per primitive cell of every system from the frequencies of the Gamma-centred ``mesh``
        at ``temperatures`` [T] (K): ``zero_point_energy`` [B] (eV), ``free_energy`` [T, B] (eV), ``entropy`` and
        ``heat_capacity`` [T, B] (eV/K), all averages over the mesh.  Modes below ``min_frequency`` (cm^-1) -- the
        acoustic modes at Gamma, and imaginary modes -- are left out; ``n_excluded`` [B] counts them over the mesh and
        ``n_imaginary`` [B] the imaginary ones among them."""
        freq = self._mesh_frequencies(mesh)
        temps = torch.as_tensor(temperatures, dtype=torch.float64).reshape(-1)
        if temps.numel() < 1 or bool((temps < 0).any()):
            raise ValueError("DevicePhonons.thermodynamics: temperatures must be >= 0 K")
        n_q, n_t = freq.shape[0], temps.shape[0]
        counts = (n_q * 3 * torch.as_tensor(self.sizes, dtype=torch.int64)).repeat(n_t)
        n_items = int(counts.sum())
        if n_items >= 2 ** 31:
            raise ValueError(f"DevicePhonons.thermodynamics: {n_items} (temperature, mode) items exceed int32 indexing")
        seg_ptr = torch.zeros(counts.shape[0] + 1, dtype=torch.int32)
        seg_ptr[1:] = torch.cumsum(counts, 0)
        out = ops.ph_thermo(freq, self.prim_ptr, temps.to(freq.device), seg_ptr.to(freq.device), n_items,
                            float(min_frequency), _INVCM, _KB).view(n_t, self.n_sys, -1)
        return {"zero_point_energy": out[0, :, 0], "free_energy": out[:, :, 1], "entropy": out[:, :, 2],
                "heat_capacity": out[:, :, 3], "n_excluded": out[0, :, 4].round().to(torch.int64),
                "n_imaginary": out[0, :, 5].round().to(torch.int64)}
