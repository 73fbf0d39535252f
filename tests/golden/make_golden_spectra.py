"""Generate tests/golden/spectra_*.npz: power, IR and Raman spectra of the UNMODIFIED reference md/data/spectra.py.

The reference module is imported through oracle/ref_loader with three stubs: ``ase.units`` (``_c``), ``schnetpack.units``
(``fs``, ``kB``, ``hbar2icm`` from this package's restated unit table) and ``schnetpack.md.data`` (``HDF5Loader`` is only
an annotation there).  A stub loader serves fp64 copies of fp32 records, with the centroid (mean over replicas) the
reference's HDF5Loader takes for ``replica_idx=None``, so the reference runs in fp64 on exactly the device's inputs.

Each file holds the records (rec:velocities [T, P, N, 3], rec:dipole_moment [T, P, B, 3], rec:polarizability
[T, P, B, 3, 3]), sys_ptr, n_replicas, dt_fs and a JSON list of runs; run r of system m stores
``r{r}:m{m}:freq``, ``r{r}:m{m}:I{j}`` (the reference's intensities) and ``r{r}:m{m}:acf`` (``_compute_autocorrelations``
of the reference's data, flattened to [F, n - 1]; spectra_long keeps its first min(resolution, n - 1) lags).

Cases:
  * spectra_power: three ragged systems (3, 1 and 4 atoms), P = 4 replicas, at resolutions above and below n - 1;
  * spectra_ir: two systems, P = 1, resolution above and below n - 1;
  * spectra_raman: two systems, P = 2, averaged and not;
  * spectra_short: the shortest series (T = 3 for power, T = 5 for IR and Raman);
  * spectra_zero: a zero-variance field (an atom at rest along x, a constant dipole component): NaN channels;
  * spectra_long: T = 5200 records (three time chunks of the device autocorrelation), one atom and one dipole, P = 2;
    power at resolution 5120 and IR at 1024 (both placements of the transform's cosine table), acf stored for the used
    lags only.  It has its own generator, so it is made alone without rewriting the others.

Run from the repository root:  python tests/golden/make_golden_spectra.py [case ...]  (default: every case)
"""
import importlib
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_loader as rl  # noqa: E402
from schnetpack_b200.md import FS_MD, KB_MD  # noqa: E402
from schnetpack_b200.spectra import HBAR2ICM  # noqa: E402

C_LIGHT = 299792458.0
INCIDENT, TEMPERATURE = 19455.25, 300.0
DT_FS = 0.5


def load_spectra():
    spk = rl.load()
    ase = sys.modules["ase"]
    ase.units = types.ModuleType("ase.units")
    ase.units._c = C_LIGHT
    sys.modules["ase.units"] = ase.units
    units = types.ModuleType("schnetpack.units")
    units.fs, units.kB, units.hbar2icm = FS_MD, KB_MD, HBAR2ICM
    saved = sys.modules.get("schnetpack.units"), getattr(spk, "units", None)
    sys.modules["schnetpack.units"] = units
    spk.units = units
    rl._stubpkg("schnetpack.md", rl.REF + "/md")
    rl._stubpkg("schnetpack.md.data", rl.REF + "/md/data", HDF5Loader=object)
    mod = importlib.import_module("schnetpack.md.data.spectra")
    if saved[0] is not None:
        sys.modules["schnetpack.units"] = saved[0]
    if saved[1] is not None:
        spk.units = saved[1]
    return mod


class StubLoader:
    """The parts of md/data/hdf5_data.py the spectra read: time_step and the centroid of fp64 copies of the records"""

    def __init__(self, records, sys_ptr, dt_fs):
        self.records = {k: v.astype(np.float64) for k, v in records.items()}
        self.sys_ptr = sys_ptr
        self.time_step = dt_fs * FS_MD

    def get_property(self, name, atomistic, mol_idx=0, replica_idx=None):
        sel = slice(self.sys_ptr[mol_idx], self.sys_ptr[mol_idx + 1]) if atomistic else mol_idx
        return np.mean(self.records[name][:, :, sel, ...], axis=1)

    def get_velocities(self, mol_idx=0, replica_idx=None):
        return self.get_property("velocities", True, mol_idx=mol_idx)


def signal(rng, T, shape, dt_fs, n_modes=4):
    """sums of damped-free cosines at vibrational frequencies (500-3500 cm^-1) plus noise, fp32"""
    t = np.arange(T) * dt_fs * 1e-15
    out = np.zeros((T,) + shape)
    flat = out.reshape(T, -1)
    for j in range(flat.shape[1]):
        for _ in range(n_modes):
            nu = rng.uniform(500, 3500) * 100 * C_LIGHT
            flat[:, j] += rng.normal() * np.cos(2 * np.pi * nu * t + rng.uniform(0, 2 * np.pi))
        flat[:, j] += 0.05 * rng.normal(size=T) + rng.normal()
    return out.astype(np.float32)


def run_case(mod, name, records, sys_ptr, n_replicas, runs, acf_lags=False):
    """``acf_lags``: store only the lags the spectrum uses, acf[:, :min(resolution, n - 1)], not all n - 1"""
    loader = StubLoader(records, sys_ptr, DT_FS)
    out = {f"rec:{k}": v for k, v in records.items()}
    out.update(sys_ptr=np.asarray(sys_ptr, np.int64), n_replicas=np.int64(n_replicas), dt_fs=np.float64(DT_FS))
    for r, run in enumerate(runs):
        kind, res = run["kind"], run["resolution"]
        if kind == "power":
            spec = mod.PowerSpectrum(loader, resolution=res)
        elif kind == "ir":
            spec = mod.IRSpectrum(loader, resolution=res)
        else:
            spec = mod.RamanSpectrum(loader, INCIDENT, TEMPERATURE, resolution=res, averaged=run["averaged"])
        for m in range(len(sys_ptr) - 1):
            with np.errstate(invalid="ignore", divide="ignore"):
                data = spec._get_data(m)
                acf = spec._compute_autocorrelations(data.copy())
                spec.compute_spectrum(m)
            acf = acf.reshape(-1, acf.shape[-1])
            out[f"r{r}:m{m}:acf"] = acf[:, :res] if acf_lags else acf
            out[f"r{r}:m{m}:freq"] = np.asarray(spec.frequencies[0])
            for j, v in enumerate(spec.intensities):
                out[f"r{r}:m{m}:I{j}"] = np.asarray(v)
    out["runs"] = np.array(json.dumps(runs))
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print("wrote", name, {k: v.shape for k, v in out.items() if k.startswith("rec:")})


def long_case(mod):
    """one atom and one dipole, P = 2, T = 5200 records (three time chunks of the device autocorrelation): power at
    resolution 5120 (the transform's cosine table in global memory) and IR at 1024 (in shared memory).  The records
    sit on a 2^-10 grid (far finer than their 0.05 noise) and only the used lags are stored, so the file stays small."""
    rng = np.random.default_rng(11)
    T = 5200

    def grid(x):
        return (np.round(x.astype(np.float64) * 1024.0) / 1024.0).astype(np.float32)

    records = {"velocities": grid(signal(rng, T, (2, 1, 3), DT_FS)),
               "dipole_moment": grid(signal(rng, T, (2, 1, 3), DT_FS))}
    run_case(mod, "spectra_long", records, [0, 1], 2,
             [dict(kind="power", resolution=5120), dict(kind="ir", resolution=1024)], acf_lags=True)


def main(names=None):
    mod = load_spectra()
    if names:
        assert set(names) <= {"spectra_long"}, "only spectra_long is made alone; the others share one generator"
        long_case(mod)
        return
    rng = np.random.default_rng(7)
    # power: ragged systems, one of them a single atom, 4 replicas
    sys_ptr = [0, 3, 4, 8]
    vel = signal(rng, 600, (4, 8, 3), DT_FS)
    run_case(mod, "spectra_power", {"velocities": vel}, sys_ptr, 4,
             [dict(kind="power", resolution=4096), dict(kind="power", resolution=100)])
    # IR: resolution above and below n - 1
    dip = signal(rng, 700, (1, 2, 3), DT_FS)
    run_case(mod, "spectra_ir", {"dipole_moment": dip}, [0, 2, 5], 1,
             [dict(kind="ir", resolution=4096), dict(kind="ir", resolution=128)])
    # Raman: averaged and not, 2 replicas
    pol = signal(rng, 500, (2, 2, 3, 3), DT_FS)
    pol = 0.5 * (pol + pol.transpose(0, 1, 2, 4, 3))
    run_case(mod, "spectra_raman", {"polarizability": pol}, [0, 3, 4], 2,
             [dict(kind="raman", resolution=4096, averaged=False), dict(kind="raman", resolution=4096, averaged=True),
              dict(kind="raman", resolution=64, averaged=True)])
    # shortest series: n = 3 points, 2 lags
    run_case(mod, "spectra_short", {"velocities": signal(rng, 3, (2, 2, 3), DT_FS),
                                    "dipole_moment": signal(rng, 5, (2, 1, 3), DT_FS),
                                    "polarizability": signal(rng, 5, (2, 1, 3, 3), DT_FS)}, [0, 2], 2,
             [dict(kind="power", resolution=4096), dict(kind="ir", resolution=4096),
              dict(kind="raman", resolution=4096, averaged=False), dict(kind="raman", resolution=4096, averaged=True)])
    # zero variance: atom 1 at rest along x in every replica, dipole z of system 0 constant, polarizability xy of
    # system 1 constant (the averaged Raman's xy field of that system)
    vel = signal(rng, 200, (1, 3, 3), DT_FS)
    vel[:, :, 1, 0] = 0.0
    dip = signal(rng, 200, (1, 2, 3), DT_FS)
    dip[:, :, 0, 2] = 0.75
    pol = signal(rng, 200, (1, 2, 3, 3), DT_FS)
    pol[:, :, 1, 0, 1] = 1.25
    run_case(mod, "spectra_zero", {"velocities": vel, "dipole_moment": dip, "polarizability": pol}, [0, 2, 3], 1,
             [dict(kind="power", resolution=4096), dict(kind="ir", resolution=4096),
              dict(kind="raman", resolution=4096, averaged=False), dict(kind="raman", resolution=4096, averaged=True)])
    long_case(mod)


if __name__ == "__main__":
    main(sys.argv[1:])
