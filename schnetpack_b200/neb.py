"""Minimum-energy paths on the device: the climbing-image nudged elastic band (NEB) with the improved tangent of
Henkelman & Jonsson, J. Chem. Phys. 113, 9978 (2000), and the climbing image of Henkelman, Uberuaga & Jonsson,
J. Chem. Phys. 113, 9901 (2000), relaxed by ASE's FIRE (DESIGN.md section 21).

Every system of ``initial`` / ``final`` is the pair of endpoints of one band.  The interior images of all bands form one
collated batch (band-major, image-major, one model system per image), so one evaluation serves every image of every band.
The NEB projection is three kernels of ``csrc/neb.cu`` (``spk_neb_forces``); the NEB forces then drive the FIRE kernels
of ``csrc/fire.cu`` with the band as FIRE's system, so that the |dr| cap and the fmax test run over all moving
coordinates of a band, as ASE's optimizer does on an ``NEB`` object.  The whole step -- FIRE step, neighbour list,
model, NEB forces, FIRE force side and convergence test -- is captured once as a CUDA graph.
"""
from __future__ import annotations

import ctypes
import itertools
from typing import Dict, List, Optional, Tuple

import torch

from . import _lib, ops
from . import properties as P
from .md import _TensorState
from .relax import FIREState, _BatchOptimizer, _check_fire_keywords, _fixed_mask

__all__ = ["DeviceNEB", "NEBState", "interpolate"]

Tensor = torch.Tensor
_NEIGHBOR_KEYS = (P.idx_i, P.idx_j, P.offsets)
_BATCH_KEYS = (P.R, P.Z, P.idx_m, P.n_atoms, P.cell, P.pbc)


# ---- bands of a collated batch -----------------------------------------------------------------------------------------
class _Systems:
    """The systems of a collated batch as bands or images see them: atom counts, atomic numbers, positions and one cell
    and pbc row per system (None for a batch without them)."""

    def __init__(self, batch: Dict[str, Tensor], what: str):
        unknown = [k for k in batch if k not in _BATCH_KEYS + _NEIGHBOR_KEYS]
        if unknown:
            raise ValueError(f"{what}: the batch has inputs a band cannot carry: {unknown}")
        self.positions = batch[P.R]
        self.Z = batch[P.Z].reshape(-1)
        n = int(self.positions.shape[0])
        if P.n_atoms in batch:
            self.sizes = [int(s) for s in batch[P.n_atoms].reshape(-1).tolist()]
        else:
            self.sizes = [n]
        if sum(self.sizes) != n:
            raise ValueError(f"{what}: '_n_atoms' adds up to {sum(self.sizes)}, the batch has {n} atoms")
        self.n_sys = len(self.sizes)
        self.cell = self._rows(batch.get(P.cell), 9, what)
        self.pbc = self._rows(batch.get(P.pbc), 3, what)

    def _rows(self, v: Optional[Tensor], width: int, what: str) -> Optional[Tensor]:
        if v is None:
            return None
        rows = v.reshape(-1, width)
        if rows.shape[0] == 1:
            rows = rows.expand(self.n_sys, width)
        if rows.shape[0] != self.n_sys:
            raise ValueError(f"{what}: a '_cell' / '_pbc' of shape {tuple(v.shape)} for {self.n_sys} systems")
        return rows

    def ptr(self) -> List[int]:
        return [0] + list(itertools.accumulate(self.sizes))


def _check_same(ref: _Systems, other: _Systems, what: str, per_band: int = 1):
    """refuse ``other`` unless its systems, ``per_band`` per system of ``ref``, have ref's atom counts, atomic numbers,
    cells and pbc"""
    if other.n_sys != ref.n_sys * per_band:
        raise ValueError(f"{what}: {other.n_sys} systems for {ref.n_sys} bands of {per_band} images")
    if other.sizes != [s for s in ref.sizes for _ in range(per_band)]:
        raise ValueError(f"{what}: the atom counts differ from the initial endpoints'")
    rz = torch.cat([ref.Z[p0:p1].repeat(per_band) for p0, p1 in zip(ref.ptr()[:-1], ref.ptr()[1:])])
    if not torch.equal(other.Z.to(rz.device, rz.dtype), rz):
        raise ValueError(f"{what}: the atomic numbers differ from the initial endpoints'")
    for name, a, b in (("cells", ref.cell, other.cell), ("pbc", ref.pbc, other.pbc)):
        if (a is None) != (b is None):
            raise ValueError(f"{what}: the {name} differ from the initial endpoints'")
        if a is not None and not torch.equal(b.to(a.device, a.dtype), a.repeat_interleave(per_band, 0)):
            raise ValueError(f"{what}: the {name} differ from the initial endpoints'")


def _differences(initial: _Systems, final: _Systems, mic: bool) -> Tensor:
    """final - initial per atom [M, 3] fp64; with ``mic`` each band's difference is its minimum image in the band's cell
    (on its periodic axes): the fractional difference is rounded, then the shortest of the 27 neighbouring images is
    taken, which covers skewed cells"""
    d = final.positions.double() - initial.positions.double()
    if not mic or initial.cell is None or initial.pbc is None:
        return d
    out = d.clone()
    for b, (p0, p1) in enumerate(zip(initial.ptr()[:-1], initial.ptr()[1:])):
        pbc = initial.pbc[b].to(torch.bool).cpu()
        if not bool(pbc.any()) or p1 == p0:
            continue
        cell = initial.cell[b].reshape(3, 3).double().to(d.device)
        if float(torch.linalg.det(cell)) == 0.0:
            raise ValueError("interpolate: mic needs a non-singular cell for every periodic band")
        mask = pbc.to(d.device, torch.float64)
        frac = torch.linalg.solve(cell.T, d[p0:p1].T).T                   # d = frac @ cell
        frac = frac - torch.round(frac) * mask
        shifts = torch.tensor(list(itertools.product((-1, 0, 1), repeat=3)), dtype=torch.float64, device=d.device)
        shifts = torch.unique(shifts * mask, dim=0)
        cand = (frac[:, None, :] + shifts[None]) @ cell                     # [A, S, 3]
        best = torch.argmin((cand * cand).sum(-1), dim=1)
        out[p0:p1] = cand[torch.arange(p1 - p0, device=d.device), best]
    return out


def _collate(bands: _Systems, positions: Tensor, per_band: int) -> Dict[str, Tensor]:
    """the collated batch of ``per_band`` systems per band, band-major, with the band's atoms, cell and pbc;
    ``positions`` [per_band * M, 3] in that order"""
    dev = positions.device
    sizes = torch.tensor([s for s in bands.sizes for _ in range(per_band)], dtype=torch.int64, device=dev)
    ptr = bands.ptr()
    out = {P.R: positions.contiguous(),
           P.Z: torch.cat([bands.Z[p0:p1].repeat(per_band) for p0, p1 in zip(ptr[:-1], ptr[1:])]).to(dev),
           P.n_atoms: sizes,
           P.idx_m: torch.repeat_interleave(torch.arange(len(sizes), device=dev), sizes)}
    if bands.cell is not None:
        out[P.cell] = bands.cell.reshape(-1, 3, 3).repeat_interleave(per_band, 0).contiguous().to(dev)
    if bands.pbc is not None:
        out[P.pbc] = bands.pbc.repeat_interleave(per_band, 0).contiguous().to(dev)
    return out


def _band_rows(bands: _Systems, rows: List[Tensor]) -> Tensor:
    """band-major concatenation of per-band blocks: block j of band b is rows[j][band b's atoms]"""
    ptr = bands.ptr()
    return torch.cat([r[p0:p1] for p0, p1 in zip(ptr[:-1], ptr[1:]) for r in rows])


def interpolate(initial: Dict[str, Tensor], final: Dict[str, Tensor], n_images: int, mic: bool = False
                ) -> Dict[str, Tensor]:
    """The ``n_images`` linear interior images R_0 + j / (n + 1) (R_{n+1} - R_0), j = 1 .. n, of every band, as one
    collated batch (band-major, image-major, one system per image; ``_positions`` fp32 in the endpoints' units).  Each
    system of ``initial`` / ``final`` is one band, with the same atoms in the same order, cell and pbc.  With ``mic`` the
    endpoint difference is first mapped to its minimum image in the band's cell, so a hop across a periodic face takes the
    short path (the path then ends at R_0 + the mapped difference, an image of R_{n+1})."""
    n = int(n_images)
    if n < 1:
        raise ValueError(f"interpolate: n_images must be >= 1, got {n_images}")
    a, b = _Systems(initial, "interpolate"), _Systems(final, "interpolate")
    _check_same(a, b, "interpolate: final endpoints")
    x0 = a.positions.double()
    d = _differences(a, b, mic)
    rows = [x0 + (j / (n + 1)) * d for j in range(1, n + 1)]
    return _collate(a, _band_rows(a, rows).to(a.positions.dtype), n)


# ---- the NEB forces ------------------------------------------------------------------------------------------------------
class NEBState(_TensorState):
    """The NEB projection of a batch of bands and the launches of its kernels, given model forces and energies.
    ``positions`` [N, 3] fp64 are the interior images in optimizer units (band-major, image-major: FIRE's ``r``, read in
    place), ``initial`` / ``final`` [M, 3] fp64 the endpoint rows of every band (M = sum of ``band_sizes``, the atoms per
    image of each band) and ``end_energies`` [n_bands, 2] their energies, all in optimizer units.  ``forces`` are model
    forces, multiplied by ``force_conversion``, and ``energies`` [n_bands * n_images] model energies, multiplied by
    ``energy_conversion``.  ``fixed_atoms_mask`` (over the N interior atoms) zeroes forces.  ``forces(f, e)`` returns the
    fp32 NEB forces [N, 3] in optimizer units (``neb_forces``), to hand to ``FIREState.check`` with force_conversion 1;
    ``coef`` [n_img, 3] = (alpha, beta, gamma), ``diag`` [n_img, 6] = (|tau|, F.tau^, spring term, |D+|, |D-|, climbing)
    and ``climbing`` [n_bands] (the climbing image's interior index, -1 without climbing) are written with it."""

    def __init__(self, positions: Tensor, initial: Tensor, final: Tensor, end_energies: Tensor, band_sizes: List[int],
                 n_images: int, k: float = 0.1, climb: bool = False, fixed_atoms_mask=None,
                 force_conversion: float = 1.0, energy_conversion: float = 1.0):
        dev = positions.device
        if dev.type != "cuda":
            raise ValueError("NEBState needs CUDA tensors (no CPU fallback)")
        n, sizes = int(n_images), [int(s) for s in band_sizes]
        if n < 1:
            raise ValueError(f"NEB: n_images must be >= 1, got {n_images}")
        if not float(k) > 0.0:
            raise ValueError(f"NEB: the spring constant k must be > 0, got {k}")
        if not sizes or min(sizes) < 1:
            raise ValueError("NEB: every band needs at least one atom")
        if positions.dtype != torch.float64 or not positions.is_contiguous():
            raise ValueError("NEBState: positions must be a contiguous fp64 tensor")
        n_atoms, n_bands, m = int(positions.shape[0]), len(sizes), sum(sizes)
        if n_atoms != n * m:
            raise ValueError(f"NEBState: {n_atoms} interior atoms for {n} images of bands of {m} atoms in all")
        f64 = dict(dtype=torch.float64, device=dev)
        self.n_atoms, self.n_images, self.n_bands, self.band_sizes = n_atoms, n, n_bands, sizes
        self.r = positions
        self.initial = initial.detach().to(**f64).reshape(m, 3).contiguous().clone()
        self.final = final.detach().to(**f64).reshape(m, 3).contiguous().clone()
        self.end_energies = end_energies.detach().to(**f64).reshape(n_bands, 2).contiguous().clone()
        self.climb = torch.full((1,), int(bool(climb)), dtype=torch.int32, device=dev)
        self.fixed = _fixed_mask(fixed_atoms_mask, n_atoms, dev)
        img_sizes = torch.tensor([s for s in sizes for _ in range(n)], dtype=torch.int64)
        self.idx_img = torch.repeat_interleave(torch.arange(n * n_bands), img_sizes).to(dev)
        self.img_ptr = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(img_sizes, 0)]).to(dev, torch.int32)
        self.band_ptr = self.img_ptr[::n].contiguous()
        self.coef = torch.zeros(n * n_bands, _lib.NEB_COEF, **f64)
        self.diag = torch.zeros(n * n_bands, _lib.NEB_DIAG, **f64)
        self.climbing = torch.full((n_bands,), -1, dtype=torch.int32, device=dev)
        self.neb_forces = torch.zeros(n_atoms, 3, dtype=torch.float32, device=dev)
        nbytes = int(_lib.lib().spk_neb_workspace_bytes(n_atoms, n * n_bands))
        self.workspace = torch.zeros(max(nbytes // 8, 1), **f64)
        p = ops._p
        self._params = _lib.NEBState(
            p(self.r), p(self.initial), p(self.final), p(self.end_energies), p(self.climb), p(self.fixed),
            p(self.idx_img), p(self.img_ptr), p(self.band_ptr), p(self.coef), p(self.diag), p(self.climbing),
            p(self.neb_forces), p(self.workspace), n_atoms, n, n_bands, float(k), float(force_conversion),
            float(energy_conversion))

    def forces(self, forces: Tensor, energies: Tensor) -> Tensor:
        """the NEB forces [N, 3] fp32 of the current positions (and coef, diag, climbing)"""
        f, e = ops.f32(forces, "forces"), ops.f32(energies, "energies")
        if f.numel() != 3 * self.n_atoms:
            raise ValueError(f"NEBState: forces of {f.numel()} values for {self.n_atoms} atoms")
        if e.numel() != self.n_images * self.n_bands:
            raise ValueError(f"NEBState: {e.numel()} energies for {self.n_images * self.n_bands} interior images")
        _lib.call("spk_neb_forces", ctypes.byref(self._params), ops._p(f), ops._p(e), ops._stream())
        return self.neb_forces

    def set_climb(self, climb: bool):
        self.climb.fill_(int(bool(climb)))

    def tensors(self) -> Dict[str, Tensor]:
        """every buffer the kernels write, and the climb flag they read"""
        return {"climb": self.climb, "coef": self.coef, "diag": self.diag, "climbing": self.climbing,
                "neb_forces": self.neb_forces}

    def _state(self) -> Dict[str, Tensor]:
        return self.tensors()


# ---- the captured NEB relaxation -----------------------------------------------------------------------------------------
class DeviceNEB(_BatchOptimizer):
    """Climbing-image NEB between the systems of ``initial`` and ``final`` (collated batches in model units, one band per
    system; the endpoints of a band have the same atoms in the same order, the same cell and pbc), relaxed by ASE's FIRE
    (its keywords and defaults) with each band as one optimizer.  The ``n_images`` interior images of every band are the
    linear interpolation (``interpolate``, with ``mic``) or ``images``, a collated batch of n_bands * n_images images in
    the order of ``interpolate``.  ``k`` is the spring constant in optimizer energy / length^2; ``climb`` turns the
    climbing image on.  ``position_conversion`` and ``energy_conversion`` turn model lengths and energies into the
    optimizer's units, in which ``dt``, ``maxstep``, ``k`` and ``fmax`` are given.  ``fixed_atoms_mask`` (boolean mask or
    indices over the atoms of ``initial``) fixes those atoms in every image of their band.  ``capacity`` is the pair
    capacity of ``initial``: the evaluated batch gets ``n_images`` times that, the endpoint batch twice that.

    The endpoints are evaluated once, at set-up, by the same evaluation path (the member mean for an ensemble).  One step
    is the FIRE step, the neighbour list, the model on the interior images, the NEB forces and FIRE's force side and
    convergence test, captured once as a CUDA graph (``use_graph``).  A band converges when the largest NEB force on its
    moving atoms is below ``fmax``; converged bands take no step.  ``model`` may be a list of at least two members, as in
    ``DeviceFIRE``.  Results are per band (``fmax``: the largest NEB force, ``converged``, ``steps_to_converge``) or
    cover the interior images (``positions``, band-major and image-major; ``get_forces``: the NEB forces;
    ``get_uncertainty``: their energies and forces)."""

    def __init__(self, model: torch.nn.Module, initial: Dict[str, Tensor], final: Dict[str, Tensor], cutoff: float,
                 capacity: int, n_images: int = 5, images: Optional[Dict[str, Tensor]] = None, k: float = 0.1,
                 climb: bool = False, mic: bool = False, fixed_atoms_mask=None, dt: float = 0.1, maxstep: float = 0.2,
                 dtmax: float = 1.0, Nmin: int = 5, finc: float = 1.1, fdec: float = 0.5, astart: float = 0.1,
                 fa: float = 0.99, a: float = 0.1, position_conversion: float = 1.0, energy_conversion: float = 1.0,
                 energy_key: str = P.energy, force_key: str = P.forces, use_graph: bool = True):
        from .parallel import PartitionedPotential

        if isinstance(model, PartitionedPotential):
            raise NotImplementedError("DeviceNEB: PartitionedPotential is not supported (one GPU per batch)")
        if int(n_images) != n_images or int(n_images) < 1:
            raise ValueError(f"DeviceNEB: n_images must be an integer >= 1, got {n_images}")
        if not float(k) > 0.0:
            raise ValueError(f"DeviceNEB: the spring constant k must be > 0, got {k}")
        self.fire_keywords = dict(dt=dt, maxstep=maxstep, dtmax=dtmax, Nmin=Nmin, finc=finc, fdec=fdec, astart=astart,
                                  fa=fa, a=a)
        _check_fire_keywords(self.fire_keywords)
        self._check_outputs(model, energy_key, force_key)
        if initial[P.R].device.type != "cuda":
            raise ValueError("DeviceNEB needs CUDA batches (no CPU fallback)")
        n = self.n_images = int(n_images)
        self._set_conversions(position_conversion, energy_conversion)
        ends = [_Systems(initial, "DeviceNEB: initial"), _Systems(final, "DeviceNEB: final")]
        self.bands = bands = ends[0]
        _check_same(bands, ends[1], "DeviceNEB: final endpoints")
        if min(bands.sizes) < 1:
            raise ValueError("DeviceNEB: every band needs at least one atom")
        for s in ends:
            if s.positions.dtype != torch.float32:
                raise ValueError("DeviceNEB: '_positions' must be float32 (model units)")
        self.n_bands, self.band_sizes = bands.n_sys, list(bands.sizes)
        m = sum(self.band_sizes)
        x0 = bands.positions.double()
        x1 = x0 + _differences(bands, ends[1], mic)
        if images is None:
            images = interpolate(initial, final, n, mic=mic)
        else:
            _check_same(bands, _Systems(images, "DeviceNEB: images"), "DeviceNEB: images", per_band=n)
            images = {k_: v for k_, v in images.items() if k_ not in _NEIGHBOR_KEYS}

        # the endpoints, evaluated once by the evaluation path of the run (band b: systems 2b, 2b + 1)
        self._setup(model, _collate(bands, _band_rows(bands, [x0, x1]).float(), 2), cutoff, 2 * int(capacity), False)
        self._calculate()
        self.check_neighbor_list()
        end_energies = self.energy.double().reshape(self.n_bands, 2) * self.e_conv

        idx_m, n_sys = self._setup(model, images, cutoff, n * int(capacity), use_graph)
        mp = self.static[P.R]
        if mp.dtype != torch.float32 or not mp.is_contiguous():
            raise ValueError("DeviceNEB: '_positions' of the images must be a contiguous float32 tensor")
        fixed = _fixed_mask(fixed_atoms_mask, m, mp.device)
        if fixed is not None:
            fixed = _band_rows(bands, [fixed] * n)
        band_of_atom = torch.repeat_interleave(torch.arange(self.n_bands, device=mp.device),
                                               torch.tensor(self.band_sizes, device=mp.device) * n)
        self.opt = FIREState(mp.double() * self.p_conv, band_of_atom, self.n_bands, fixed_atoms_mask=fixed,
                             position_conversion=self.p_conv, force_conversion=1.0, model_positions=mp,
                             **self.fire_keywords)
        self.neb = NEBState(self.opt.r, x0 * self.p_conv, x1 * self.p_conv, end_energies, self.band_sizes, n, k=k,
                            climb=climb, fixed_atoms_mask=fixed, force_conversion=self.f_conv,
                            energy_conversion=self.e_conv)
        self.climb = bool(climb)
        self._start()

    def _advance(self):
        self.opt.step()

    def _check(self):
        self.opt.check(self.neb.forces(self.forces, self.energy))

    def _step_state(self) -> Dict[str, object]:
        return dict(super()._step_state(), neb=self.neb.tensors())

    def _reset_fire(self):
        """the state of a new FIRE optimizer for every band (v = 0, dt, a, Nsteps), in place"""
        o = self.opt
        o.v.zero_()
        o.dt.fill_(float(self.fire_keywords["dt"]))
        o.a.fill_(float(self.fire_keywords["a"]))
        o.nsteps.zero_()
        o.started.zero_()

    def run(self, fmax: float = 0.05, steps: Optional[int] = None, check_every: int = 10,
            climb: Optional[bool] = None) -> bool:
        """Relax until every band's largest NEB force is below ``fmax`` or ``steps`` steps (default: unlimited) were taken
        in this call; returns whether every band converged.  ``climb`` turns the climbing image on or off first; when that
        changes it, every band's FIRE state is reset, as a new optimizer would start (the captured step stays valid)."""
        if int(check_every) < 1:                 # refused before the climb flag changes
            raise ValueError("DeviceNEB: check_every must be >= 1")
        if climb is not None and bool(climb) != self.climb:
            self.climb = bool(climb)
            self.neb.set_climb(self.climb)
            self._reset_fire()
        return super().run(fmax, steps, check_every)

    # ---- results, in optimizer units ------------------------------------------------------------------------------------
    def path(self) -> List[Tensor]:
        """per band, [n_images + 2, A_b, 3] fp64: the endpoints and the interior images"""
        out, p, e = [], 0, 0
        for size in self.band_sizes:
            inner = self.opt.r[p:p + self.n_images * size].reshape(self.n_images, size, 3)
            out.append(torch.cat([self.neb.initial[e:e + size][None], inner, self.neb.final[e:e + size][None]]))
            p += self.n_images * size
            e += size
        return out

    def get_energies(self) -> Tensor:
        """[n_bands, n_images + 2] fp64 energies of every image of every band, endpoints included"""
        inner = self.energy.double().reshape(self.n_bands, self.n_images) * self.e_conv
        ends = self.neb.end_energies
        return torch.cat([ends[:, :1], inner, ends[:, 1:]], dim=1)

    def barriers(self) -> Tuple[Tensor, Tensor]:
        """(forward, backward) [n_bands] fp64: the highest interior energy minus the initial / final energy"""
        e = self.get_energies()
        top = e[:, 1:-1].max(dim=1).values
        return top - e[:, 0], top - e[:, -1]

    def reaction_coordinate(self) -> Tensor:
        """[n_bands, n_images + 2] fp64 cumulative distance along each band (|R_j - R_{j-1}| over all its coordinates)"""
        out = []
        for x in self.path():
            step = (x[1:] - x[:-1]).reshape(self.n_images + 1, -1).norm(dim=1)
            out.append(torch.cat([step.new_zeros(1), torch.cumsum(step, 0)]))
        return torch.stack(out)

    def tangent_forces(self) -> Tensor:
        """[n_bands, n_images] fp64 F . tau^ of every interior image (the model force along the unit tangent; minus the
        slope dE/ds of the energy profile), at the current positions"""
        return self.neb.diag[:, 1].reshape(self.n_bands, self.n_images).clone()

    @property
    def climbing_image(self) -> Tensor:
        """[n_bands] int32 the interior index (0 .. n_images - 1, image index - 1) of each band's climbing image, -1
        without climbing"""
        return self.neb.climbing

    def get_forces(self) -> Tensor:
        """the NEB forces [N, 3] fp64 of the current positions (0 on fixed atoms)"""
        return self.neb.neb_forces.double()

    def state_dict(self) -> Dict[str, object]:
        return dict(super().state_dict(), climb_on=self.climb)

    def load_state_dict(self, state: Dict[str, object]):
        super().load_state_dict(state)
        self.climb = bool(state["climb_on"])
