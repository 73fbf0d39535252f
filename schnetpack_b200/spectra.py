"""Vibrational spectra from the series ``DeviceMD`` records (md/data/spectra.py: PowerSpectrum, IRSpectrum,
RamanSpectrum; DESIGN.md section 17).

The reference reads an HDF5 file, takes the centroid over the replicas, differentiates dipoles and polarizabilities by
central differences, normalises every field, autocorrelates it through a zero-padded FFT, combines the fields into
channels, windows the first ``resolution`` lags and takes |dt FFT| of the zero-padded, mirrored result.  Here the same
numbers come from three fp64 kernels on the device records (csrc/spectra.cu): the series preparation, the lag-window
autocorrelation (direct, on the fp64 tensor cores) and the spectral transform (its DCT-II form).  Results are fp64
device tensors.  ``molecule_idx=None`` computes every system of the batch in the same launches, with a leading B axis on
the intensities; each row is bitwise equal to the call for that index.

A ``SpectrumStream`` passed as ``DeviceMD(..., stream=...)`` accumulates the first ``resolution`` lags of every field's
autocorrelation inside the captured step, so spectra of runs of any length need no stored series (DESIGN.md section 20);
the spectrum classes take it as their ``data``.

Raman intensities use the reference's cross-section exactly as written, with ``hbar2icm`` and ``kB`` in the MD unit
system (units.py:79-88); DESIGN.md section 17 notes what that factor evaluates to.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from . import _lib, ops
from . import properties as P
from .md import FS_MD as _FS_MD
from .md import HBAR_MD, KB_MD
from .units import _UNITS

__all__ = ["RecordedSeries", "SpectrumStream", "PowerSpectrum", "IRSpectrum", "RamanSpectrum", "cosine_sq_window",
           "HBAR2ICM"]

Tensor = torch.Tensor

_C = _UNITS["_c"]                                           # ase.units._c, m/s
HBAR2ICM = HBAR_MD * 100.0 * _C * _UNITS["_aut"]            # units.py:88, in MD units
RAMAN_FACTOR = 4.160440e-18                                 # md/data/spectra.py:478


def cosine_sq_window(n_points: int) -> np.ndarray:
    """cos(pi i / (n - 1) / 2)^2 for i < n (md/data/spectra.py:24-35)"""
    points = np.arange(n_points)
    return np.cos(np.pi * points / (n_points - 1) / 2) ** 2


class RecordedSeries:
    """Records of a ``DeviceMD`` run in the layout its recorder writes: ``velocities`` [T, n_replicas, N, 3] and
    ``properties[name]`` [T, n_replicas, B, ...] (fp32), with the record time step ``dt_fs`` in fs and ``sys_ptr``
    [B + 1], the first atom of every system of one replica.  ``DeviceMD.series()`` builds one from device views; build
    one from tensors to feed drained or stored records back (they are moved to ``device``, default: where they are)."""

    def __init__(self, dt_fs: float, sys_ptr, n_replicas: int, velocities: Optional[Tensor] = None,
                 properties: Optional[Dict[str, Tensor]] = None, device=None):
        self.dt_fs = float(dt_fs)
        self.n_replicas = int(n_replicas)
        ptr = torch.as_tensor(sys_ptr).reshape(-1)
        self.sys_ptr = [int(v) for v in ptr.tolist()]
        if not (self.dt_fs > 0.0) or self.n_replicas < 1 or len(self.sys_ptr) < 2:
            raise ValueError("RecordedSeries: needs dt_fs > 0, n_replicas >= 1 and sys_ptr with at least two entries")
        if any(b < a for a, b in zip(self.sys_ptr, self.sys_ptr[1:])) or self.sys_ptr[0] != 0:
            raise ValueError("RecordedSeries: sys_ptr must start at 0 and be non-decreasing")

        def _take(v):
            v = torch.as_tensor(v)
            return (v if device is None else v.to(device)).to(torch.float32).contiguous()

        self.velocities = None if velocities is None else _take(velocities)
        if self.velocities is not None and tuple(self.velocities.shape[1:]) != (self.n_replicas, self.sys_ptr[-1], 3):
            raise ValueError(f"RecordedSeries: velocities must be [T, {self.n_replicas}, {self.sys_ptr[-1]}, 3], got "
                             f"{tuple(self.velocities.shape)}")
        self.properties = {k: _take(v) for k, v in (properties or {}).items()}

    @property
    def n_systems(self) -> int:
        return len(self.sys_ptr) - 1


Window = Optional[Callable[[int], np.ndarray]]


class VibrationalSpectrum:
    """Base of the spectra (md/data/spectra.py:58-230): ``compute_spectrum(molecule_idx)`` then ``get_spectrum()``."""

    derivative = True
    averaged = False

    def __init__(self, data, resolution: int = 4096, window: Window = cosine_sq_window):
        stream = isinstance(data, SpectrumStream)
        if not hasattr(data, "series") and not isinstance(data, RecordedSeries) and not stream:
            raise TypeError(f"{type(self).__name__}: data must be a DeviceMD or a RecordedSeries (or the "
                            "SpectrumStream of a DeviceMD)")
        if int(resolution) < 1:
            raise ValueError(f"{type(self).__name__}: resolution must be positive, got {resolution}")
        if stream and int(resolution) > data.resolution:
            raise ValueError(f"{type(self).__name__}: resolution {int(resolution)} is above the stream's "
                             f"{data.resolution} lags")
        self.data = data
        self.resolution = int(resolution)
        self.window = window
        self.timestep = data.dt_fs if stream else self._series().dt_fs
        self.res = 0.5 / self.timestep / (_C / 1e13) / (4 * self.resolution)      # spectral resolution, cm^-1
        self.frequencies: List[Tensor] = []
        self.intensities: List[Tensor] = []

    def _series(self) -> RecordedSeries:
        return self.data if isinstance(self.data, RecordedSeries) else self.data.series()

    # ---- what the subclasses define -------------------------------------------------------------------------------------
    def _records(self, s: RecordedSeries) -> Tensor:
        raise NotImplementedError

    stream_kind = ""

    @staticmethod
    def _table(sys_ptr: List[int], m: int, averaged: bool):
        """(index rows [F_m, 3], coefficient rows [F_m, 3], channels [(first field, weights)]) of molecule m"""
        raise NotImplementedError

    def _fields(self, s: RecordedSeries, m: int):
        return self._table(s.sys_ptr, m, self.averaged)

    def _process_spectrum(self, intensities: List[Tensor], frequencies: Tensor) -> List[Tensor]:
        return intensities

    # ---- the computation -------------------------------------------------------------------------------------------------
    def compute_spectrum(self, molecule_idx: Optional[int] = 0):
        """Spectra of system ``molecule_idx`` of the batch, or of every system (``None``, leading B axis)."""
        s = self.data if isinstance(self.data, SpectrumStream) else self._series()
        B = s.n_systems
        if molecule_idx is None:
            mols = list(range(B))
        else:
            if isinstance(molecule_idx, bool) or not isinstance(molecule_idx, (int, np.integer)):
                raise TypeError(f"{type(self).__name__}: molecule_idx must be an int or None")
            m = int(molecule_idx)
            if not -B <= m < B:
                raise IndexError(f"{type(self).__name__}: molecule_idx {m} out of range for {B} systems")
            mols = [m % B]
        if isinstance(s, SpectrumStream):
            acf, n_out = s._autocorrelation(self, mols)
            return self._finish(acf, mols, n_out, molecule_idx is not None)
        rec = self._records(s)
        if rec.device.type != "cuda":
            raise ValueError(f"{type(self).__name__}: the records must be on a CUDA device (no CPU fallback)")
        T = int(rec.shape[0])
        n = T - 2 if self.derivative else T
        if n < 3:
            raise ValueError(f"{type(self).__name__}: {T} records give {n} points, fewer than the 3 that 2 lags need "
                             f"(need at least {5 if self.derivative else 3} records)")
        L = min(self.resolution, n - 1)
        index, coef, ch_ptr, weight = [], [], [0], []
        n_out = None
        for m in mols:
            idx_m, coef_m, channels = self._fields(s, m)
            base = len(index)
            index += idx_m
            coef += coef_m
            for first, w in channels:
                ch_ptr.append(base + first + len(w))
                weight += list(w)
            n_out = len(channels)
        dev = rec.device
        F, C = len(index), len(ch_ptr) - 1
        assert len(weight) == F and ch_ptr[-1] == F
        index_t = torch.tensor(index, dtype=torch.int64).to(dev)
        coef_t = torch.tensor(coef, dtype=torch.float64).to(dev)
        ch_t = torch.tensor(ch_ptr, dtype=torch.int64).to(dev)
        w_t = torch.tensor(weight, dtype=torch.float64).to(dev)
        z = torch.empty(F, n, dtype=torch.float64, device=dev)
        mean = torch.empty(F, dtype=torch.float64, device=dev)
        std = torch.empty(F, dtype=torch.float64, device=dev)
        stride = rec[0, 0].numel()
        with torch.cuda.device(dev):
            _lib.call("spk_spectrum_series", ops._p(rec), T, s.n_replicas, stride, ops._p(index_t), ops._p(coef_t), F,
                      1 if self.derivative else 0, self.timestep, ops._p(z), ops._p(mean), ops._p(std), ops._stream())
            acf = autocorrelation(z, ch_t, w_t, L)
        self._finish(acf, mols, n_out, molecule_idx is not None)

    def _finish(self, acf: Tensor, mols: List[int], n_out: int, single: bool):
        """the windowed transform of the channel autocorrelations acf [len(mols) n_out, L] and ``_process_spectrum``;
        ``single`` drops the leading axis of one molecule"""
        dev, L = acf.device, int(acf.shape[1])
        with torch.cuda.device(dev):
            win = None
            if self.window is not None:
                win = torch.as_tensor(np.asarray(self.window(L), dtype=np.float64)).reshape(-1).to(dev)
                if win.numel() != L:
                    raise ValueError(f"{type(self).__name__}: the window gave {win.numel()} points for {L} lags")
            spec = transform(acf, win, self.timestep)
        self.autocorrelation = acf.reshape(len(mols), n_out, L)
        spec = spec.reshape(len(mols), n_out, 4 * L)
        frequencies = np.arange(8 * L // 2) / (8 * L * self.timestep)       # numpy divides as the reference does
        frequencies = torch.as_tensor(frequencies / (_C / 1e13)).to(dev)
        intensities = [spec[:, j] for j in range(n_out)]
        intensities = self._process_spectrum(intensities, frequencies)
        if single:
            intensities = [v[0] for v in intensities]
        self.frequencies = [frequencies] * len(intensities)
        self.intensities = intensities

    def get_spectrum(self) -> Union[Tuple[Tensor, Tensor], List[Tuple[Tensor, Tensor]]]:
        """(frequencies in cm^-1, intensities) of every computed spectrum; the tuple itself when there is one"""
        spectrum = list(zip(self.frequencies, self.intensities))
        return spectrum[0] if len(spectrum) == 1 else spectrum


class PowerSpectrum(VibrationalSpectrum):
    """Vibrational density of states from the recorded velocities (``DeviceMD(..., record_velocities=True)``):
    the autocorrelations of every velocity component, summed over xyz and averaged over the atoms."""

    derivative = False
    stream_kind = "power"

    def __init__(self, data, resolution: int = 4096, window: Window = cosine_sq_window):
        super().__init__(data, resolution=resolution, window=window)

    def _records(self, s):
        if s.velocities is None:
            raise KeyError("PowerSpectrum: velocities are not recorded (create DeviceMD with record_velocities=True)")
        return s.velocities

    def _fields(self, s, m):
        if s.sys_ptr[m + 1] == s.sys_ptr[m]:
            raise ValueError(f"PowerSpectrum: system {m} has no atoms")
        return self._table(s.sys_ptr, m, False)

    @staticmethod
    def _table(sys_ptr, m, averaged):
        a0, a1 = sys_ptr[m], sys_ptr[m + 1]
        idx = [[3 * a + k, -1, -1] for a in range(a0, a1) for k in range(3)]
        coef = [[1.0, 0.0, 0.0]] * len(idx)
        return idx, coef, [(0, [1.0 / max(a1 - a0, 1)] * len(idx))]


class IRSpectrum(VibrationalSpectrum):
    """Infrared spectrum from the recorded dipole moments: autocorrelations of the central-difference derivative,
    summed over xyz."""

    def __init__(self, data, resolution: int = 4096, dipole_moment_handle: str = P.dipole_moment,
                 window: Window = cosine_sq_window):
        self.dipole_moment_handle = dipole_moment_handle
        super().__init__(data, resolution=resolution, window=window)

    def _records(self, s):
        return _property(s, self.dipole_moment_handle, (3,), "IRSpectrum")

    stream_kind = "ir"

    def _handle(self) -> str:
        return self.dipole_moment_handle

    @staticmethod
    def _table(sys_ptr, m, averaged):
        return [[3 * m + k, -1, -1] for k in range(3)], [[1.0, 0.0, 0.0]] * 3, [(0, [1.0, 1.0, 1.0])]


class RamanSpectrum(VibrationalSpectrum):
    """Raman spectrum from the recorded polarizabilities: isotropic and anisotropic channels of the central-difference
    derivative (xx and xy; rotationally averaged with ``averaged=True``), times the reference's cross-section.  With
    ``averaged`` the spectra are the parallel and orthogonal polarisations."""

    def __init__(self, data, incident_frequency: float, temperature: float,
                 polarizability_handle: str = P.polarizability, resolution: int = 4096, averaged: bool = False,
                 window: Window = cosine_sq_window):
        if not float(temperature) > 0.0:
            raise ValueError(f"RamanSpectrum: temperature must be positive, got {temperature}")
        self.incident_frequency = float(incident_frequency)
        self.temperature = float(temperature)
        self.averaged = bool(averaged)
        self.polarizability_handle = polarizability_handle
        super().__init__(data, resolution=resolution, window=window)

    def _records(self, s):
        return _property(s, self.polarizability_handle, (3, 3), "RamanSpectrum")

    @property
    def stream_kind(self) -> str:
        return "raman_averaged" if self.averaged else "raman"

    def _handle(self) -> str:
        return self.polarizability_handle

    @staticmethod
    def _table(sys_ptr, m, averaged):
        o = 9 * m
        xx, xy, xz, yy, yz, zz = o, o + 1, o + 2, o + 4, o + 5, o + 8
        if not averaged:
            return [[xx, -1, -1], [xy, -1, -1]], [[1.0, 0.0, 0.0]] * 2, [(0, [1.0]), (1, [1.0])]
        third = 1.0 / 3.0
        idx = [[xx, yy, zz], [xx, yy, -1], [yy, zz, -1], [zz, xx, -1], [xy, -1, -1], [xz, -1, -1], [yz, -1, -1]]
        coef = [[third] * 3, [1.0, -1.0, 0.0], [1.0, -1.0, 0.0], [1.0, -1.0, 0.0]] + [[1.0, 0.0, 0.0]] * 3
        return idx, coef, [(0, [1.0]), (1, [0.5, 0.5, 0.5, 3.0, 3.0, 3.0])]

    def _process_spectrum(self, intensities, frequencies):
        """md/data/spectra.py:462-485, as the reference writes it"""
        cross_section = ((self.incident_frequency - frequencies) ** 4 / frequencies
                         / (1 - torch.exp(-(HBAR2ICM * frequencies) / (KB_MD * self.temperature))))
        cross_section[0] = 0
        out = []
        for v in intensities:
            v = v * cross_section * RAMAN_FACTOR
            v[..., 0] = 0.0
            out.append(v)
        if self.averaged:
            iso, aniso = out
            out = [iso + 4 / 45 * aniso, aniso / 15]
        return out


_STREAM_KINDS = {"power": (PowerSpectrum, False), "ir": (IRSpectrum, False), "raman": (RamanSpectrum, False),
                 "raman_averaged": (RamanSpectrum, True)}


class SpectrumStream:
    """Autocorrelations of a ``DeviceMD`` run accumulated inside its captured step, for spectra of runs of any
    length (DESIGN.md section 20).  ``kinds`` are any of ``"power"``, ``"ir"``, ``"raman"`` and
    ``"raman_averaged"``; the stream samples the steps the recorder would record (``record_every``), forms every
    field of every system of the batch from the live state (velocities = momenta / masses, the dipole moments and
    polarizabilities of ``required_properties``; ring-polymer runs: the centroid) and keeps the first ``resolution``
    lags, in memory that does not grow with the run.  Pass it as ``DeviceMD(..., stream=...)`` (``record_capacity``
    may be 0) and then as the ``data`` of ``PowerSpectrum`` / ``IRSpectrum`` / ``RamanSpectrum`` with a resolution
    up to the stream's.  ``drain()`` does not touch it; ``DeviceMD.state_dict`` carries it."""

    def __init__(self, kinds, resolution: int = 4096, dipole_moment_handle: str = P.dipole_moment,
                 polarizability_handle: str = P.polarizability):
        kinds = [kinds] if isinstance(kinds, str) else list(kinds)
        unknown = [k for k in kinds if k not in _STREAM_KINDS]
        if not kinds or unknown:
            raise ValueError(f"SpectrumStream: kinds must be a non-empty choice of {sorted(_STREAM_KINDS)}, got "
                             f"{kinds}")
        if int(resolution) < 1:
            raise ValueError(f"SpectrumStream: resolution must be positive, got {resolution}")
        self.kinds = list(dict.fromkeys(kinds))
        self.resolution = int(resolution)
        self.dipole_moment_handle = dipole_moment_handle
        self.polarizability_handle = polarizability_handle
        self._md = None

    def _source(self, kind: str) -> str:
        return {"power": "velocities", "ir": self.dipole_moment_handle}.get(kind, self.polarizability_handle)

    @property
    def required_properties(self) -> List[str]:
        """the model outputs the stream reads (they must be among the run's required_properties)"""
        return list(dict.fromkeys(self._source(k) for k in self.kinds if k != "power"))

    # ---- set-up by DeviceMD ------------------------------------------------------------------------------------------
    def _bind(self, md, sys_ptr: List[int], n_replicas: int):
        """Build the field tables (the spectrum classes' ``_table``) of every system for every kind, one group per
        source, and allocate the zeroed state.  Called by ``DeviceMD`` once its properties exist."""
        if self._md is not None:
            raise ValueError("SpectrumStream: this stream already belongs to a DeviceMD")
        self.sys_ptr = [int(v) for v in sys_ptr]
        self.n_replicas = int(n_replicas)
        B = len(self.sys_ptr) - 1
        self._groups: Dict[str, dict] = {}
        self._rows: Dict[Tuple[str, int], int] = {}              # (kind, m) -> first stream row of its fields
        dev = md.positions.device
        for kind in self.kinds:
            cls, averaged = _STREAM_KINDS[kind]
            src = self._source(kind)
            if src != "velocities":
                shape = (3,) if kind == "ir" else (3, 3)
                want = (self.n_replicas, B) + shape
                got = tuple(md.properties[src].shape)
                if got != want:
                    raise ValueError(f"SpectrumStream: '{src}' must be [{', '.join(map(str, want))}], got {list(got)}")
            g = self._groups.setdefault(src, dict(derivative=cls.derivative, index=[], coef=[]))
            for m in range(B):
                idx, coef, _ = cls._table(self.sys_ptr, m, averaged)
                self._rows[(kind, m)] = len(g["index"])
                g["index"] += idx
                g["coef"] += coef
        for src, g in self._groups.items():
            F = len(g["index"])
            g["index"] = torch.tensor(g["index"], dtype=torch.int64).reshape(F, 3).to(dev)
            g["coef"] = torch.tensor(g["coef"], dtype=torch.float64).reshape(F, 3).to(dev)
            nbytes = int(_lib.lib().spk_spectrum_stream_state_bytes(F, self.resolution))
            g["state"] = torch.zeros(max(nbytes // 8, 1), dtype=torch.float64, device=dev)
        self._md = md

    def _state(self) -> Dict[str, Tensor]:
        return {src: g["state"] for src, g in self._groups.items()}

    def _push(self, md):
        """one sample of every group, gated on the device by the recorder's step counter (inside the captured step)"""
        for src, g in self._groups.items():
            if src == "velocities":
                source, masses, stride = md.momenta, md.masses, md.momenta.numel() // self.n_replicas
            else:
                source, masses = md.properties[src], None
                stride = source.numel() // self.n_replicas
            _lib.call("spk_spectrum_stream_push", ops._p(source), ops._p(masses), self.n_replicas, stride,
                      ops._p(g["index"]), ops._p(g["coef"]), int(g["index"].shape[0]), 1 if g["derivative"] else 0,
                      self.dt_fs, ops._p(md._rec_counter), md.record_every, self.resolution, ops._p(g["state"]),
                      ops._stream())

    # ---- what the spectra read ---------------------------------------------------------------------------------------
    def _need_md(self):
        if self._md is None:
            raise ValueError("SpectrumStream: the stream is not attached to a run; pass it as "
                             "DeviceMD(..., stream=...)")
        return self._md

    @property
    def dt_fs(self) -> float:
        """the sample time step ``record_every * time_step`` in fs"""
        md = self._need_md()
        return md.record_every * md.dt / _FS_MD

    @property
    def n_systems(self) -> int:
        self._need_md()
        return len(self.sys_ptr) - 1

    @property
    def frames(self) -> int:
        """samples taken so far (the records the recorder would have stored since the start)"""
        md = self._need_md()
        return md.steps_done // md.record_every

    def _autocorrelation(self, spec: VibrationalSpectrum, mols: List[int]) -> Tuple[Tensor, int]:
        """the channel autocorrelations [len(mols) C, L] of ``spec`` for the systems ``mols`` from the stream"""
        who = type(spec).__name__
        kind = spec.stream_kind
        if kind not in self.kinds:
            raise KeyError(f"{who}: the '{kind}' spectrum is not streamed (the stream has kinds {self.kinds})")
        if kind != "power" and spec._handle() != self._source(kind):
            raise KeyError(f"{who}: '{spec._handle()}' is not streamed (the stream reads '{self._source(kind)}')")
        g = self._groups[self._source(kind)]
        T = self.frames
        n = T - 2 if spec.derivative else T
        if n < 3:
            raise ValueError(f"{who}: {T} records give {n} points, fewer than the 3 that 2 lags need "
                             f"(need at least {5 if spec.derivative else 3} records)")
        L = min(spec.resolution, n - 1)
        rows, ch_ptr, weight = [], [0], []
        n_out = None
        for m in mols:
            idx_m, _, channels = spec._fields(self, m)
            base = len(rows)
            first_row = self._rows[(kind, m)]
            rows += range(first_row, first_row + len(idx_m))
            for first, w in channels:
                ch_ptr.append(base + first + len(w))
                weight += list(w)
            n_out = len(channels)
        dev = g["state"].device
        C = len(ch_ptr) - 1
        rows_t = torch.tensor(rows, dtype=torch.int64).to(dev)
        ch_t = torch.tensor(ch_ptr, dtype=torch.int64).to(dev)
        w_t = torch.tensor(weight, dtype=torch.float64).to(dev)
        acf = torch.empty(C, L, dtype=torch.float64, device=dev)
        ws = torch.empty(max(int(_lib.lib().spk_spectrum_stream_finalise_workspace_bytes(len(rows), L)), 8),
                         dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _lib.call("spk_spectrum_stream_finalise", ops._p(g["state"]), int(g["index"].shape[0]), self.resolution, n,
                      ops._p(rows_t), len(rows), ops._p(ch_t), ops._p(w_t), C, L, ops._p(acf), ops._p(ws), ws.numel(),
                      ops._stream())
        return acf, n_out


def _property(s: RecordedSeries, name: str, shape, who: str) -> Tensor:
    v = s.properties.get(name)
    if v is None:
        raise KeyError(f"{who}: '{name}' is not recorded (recorded: {sorted(s.properties)}); add it to "
                       "required_properties with record_capacity > 0")
    want = (s.n_replicas, s.n_systems) + tuple(shape)
    if tuple(v.shape[1:]) != want:
        raise ValueError(f"{who}: '{name}' records must be [T, {', '.join(map(str, want))}], got {tuple(v.shape)}")
    return v


def _workspace(n_channels: int, n: int, L: int, dev) -> Tensor:
    nbytes = int(_lib.lib().spk_spectrum_workspace_bytes(n_channels, n, L))
    return torch.empty(max(nbytes, 8), dtype=torch.uint8, device=dev)


def autocorrelation(z: Tensor, ch_ptr: Tensor, weight: Tensor, n_lags: int) -> Tensor:
    """acf [C, n_lags] = (1/n) sum_{f in channel c} w_f sum_t z_f[t] z_f[t + k] of normalised series z [F, n] fp64"""
    F, n = z.shape
    C = int(ch_ptr.numel()) - 1
    out = torch.empty(C, n_lags, dtype=torch.float64, device=z.device)
    ws = _workspace(C, n, n_lags, z.device)
    _lib.call("spk_spectrum_autocorrelation", ops._p(z), n, ops._p(ch_ptr), ops._p(weight), C, n_lags, ops._p(out),
              ops._p(ws), ws.numel(), ops._stream())
    return out


def transform(acf: Tensor, window: Optional[Tensor], dt_fs: float) -> Tensor:
    """intensities [C, 4L] = |dt FFT| of the windowed, zero-padded, mirrored acf [C, L] (its DCT-II form)"""
    C, L = acf.shape
    out = torch.empty(C, 4 * L, dtype=torch.float64, device=acf.device)
    ws = _workspace(0, 1, L, acf.device)
    _lib.call("spk_spectrum_transform", ops._p(acf), C, L, ops._p(window), float(dt_fs), ops._p(out), ops._p(ws),
              ws.numel(), ops._stream())
    return out
