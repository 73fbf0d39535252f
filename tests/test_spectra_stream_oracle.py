"""CPU checks of tests/spectra_stream_oracle.py: the streaming algebra fed the reference's record fixtures one frame at
a time reproduces their per-field autocorrelations and intensities, agrees with the direct normalised autocorrelation on
awkward series, and gives bitwise-identical accumulators however the samples are chunked; and the library exports the
streaming entry points."""
import ctypes

import numpy as np
import pytest

import spectra_oracle as SO
import spectra_stream_oracle as SS
from schnetpack_b200.md import KB_MD
from schnetpack_b200.spectra import HBAR2ICM

TOL = 1e-12


@pytest.mark.parametrize("name", ["spectra_ir", "spectra_power", "spectra_short", "spectra_zero", "spectra_raman"])
def test_stream_matches_reference_fixtures(name):
    z, cases = SO.golden(name)
    sys_ptr, P, dt = list(z["sys_ptr"]), int(z["n_replicas"]), float(z["dt_fs"])
    for r, run, m in cases:
        kind, averaged = run["kind"], run.get("averaged", False)
        idx, coef, channels = SO.fields(kind, sys_ptr, m, averaged)
        x = SS.fields_of(z["rec:" + SO.PROP[kind]], idx, coef, kind != "power", dt)
        n = x.shape[0]
        st = SS.Stream(len(idx), n - 1)
        st.extend(x)
        acf = st.acf(n - 1)
        key = f"r{r}:m{m}"
        assert SO.rel_err(acf, z[key + ":acf"]) <= TOL, (key, SO.rel_err(acf, z[key + ":acf"]))
        L = min(run["resolution"], n - 1)
        freq, ints, _ = SS.spectrum_from_acf(kind, acf, channels, L, dt, averaged=averaged, incident_frequency=19455.25,
                                             temperature=300.0, hbar2icm=HBAR2ICM, kB=KB_MD)
        assert np.array_equal(freq, z[key + ":freq"]), key
        for j, v in enumerate(ints):
            err = SO.rel_err(v, z[f"{key}:I{j}"])
            assert err <= TOL, (key, j, err)


def _direct(x, n_lags):
    """the direct normalised autocorrelation in extended precision: in fp64 the field at 1e4 with std 1e-2 loses ~1e-10
    in its mean before centring, while the shifted stream does not"""
    x = np.asarray(x, np.longdouble)
    with np.errstate(invalid="ignore", divide="ignore"):
        zz = (x - x.mean(axis=0)) / x.std(axis=0)
    return SO.direct_acf(zz.T, n_lags).astype(np.float64)


@pytest.mark.parametrize("n, L", [(200, 50), (333, 64), (130, 300), (3, 8), (3, 2), (64, 63), (129, 128), (1000, 97)])
def test_stream_equals_direct_acf(n, L):
    rng = np.random.default_rng(n * 1000 + L)
    x = np.stack([rng.normal(size=n).cumsum() + np.sin(np.arange(n) * 0.3),      # drifting
                  np.full(n, 0.75),                                             # constant: NaN
                  1e4 + 1e-2 * rng.normal(size=n),                              # offset 1e4, std 1e-2
                  rng.normal(size=n)], axis=1)
    st = SS.Stream(4, L)
    st.extend(x)
    n_out = min(L, n - 1)
    got, ref = st.acf(n_out), _direct(x, n_out)
    assert np.isnan(got[1]).all() and np.isnan(ref[1]).all()
    assert SO.rel_err(got, ref) <= TOL, SO.rel_err(got, ref)
    for f in (0, 2, 3):                                                         # each field on its own scale
        assert SO.rel_err(got[f], ref[f]) <= TOL, (f, SO.rel_err(got[f], ref[f]))


def test_stream_derivative_fields_equal_direct():
    rng = np.random.default_rng(7)
    T, P, dt = 300, 4, 0.5
    rec = (rng.normal(size=(T, P, 2, 9)).cumsum(axis=0) * 0.1 + 3.0).astype(np.float32)   # polarizabilities, 2 systems
    sys_ptr = [0, 1, 2]
    for kind, averaged, res in (("raman", True, 100), ("raman", False, 400), ("ir", False, 50)):
        recs = rec[..., :3] if kind == "ir" else rec
        for m in range(2):
            idx, coef, channels = SO.fields(kind, sys_ptr, m, averaged)
            x = SS.fields_of(recs, idx, coef, True, dt)
            n = x.shape[0]
            assert n == T - 2
            st = SS.Stream(len(idx), res)
            st.extend(x)
            n_out = min(res, n - 1)
            z = SO.series(recs, idx, coef, True, dt)
            ref = SO.direct_acf(z, n_out)
            assert SO.rel_err(st.acf(n_out), ref) <= TOL, (kind, averaged, m)


def test_chunking_gives_bitwise_identical_accumulators():
    rng = np.random.default_rng(11)
    x = rng.normal(size=(517, 5)) + 2.0
    one = SS.Stream(5, 80)
    for row in x:
        one.extend(row)
    for trial in range(4):
        st = SS.Stream(5, 80)
        cuts = np.sort(rng.choice(np.arange(1, 517), size=trial * 5 + 1, replace=False))
        for part in np.split(x, cuts):
            st.extend(part)
        a, b = one.state(), st.state()
        for k in a:
            assert np.array_equal(a[k], b[k]), (trial, k)
        assert np.array_equal(one.acf(80), st.acf(80))


def test_stream_entry_points_exported_and_bound():
    from schnetpack_b200 import _lib, build

    h = ctypes.CDLL(build.build())
    names = ("spk_spectrum_stream_state_bytes", "spk_spectrum_stream_finalise_workspace_bytes",
             "spk_spectrum_stream_push", "spk_spectrum_stream_finalise")
    for name in names:
        assert hasattr(h, name), name
        assert name in _lib.SIGNATURES, name
    assert _lib.LAUNCHES["spk_spectrum_stream_push"] == 2 and _lib.LAUNCHES["spk_spectrum_stream_finalise"] == 2
    lib = _lib.lib()
    assert lib.spk_spectrum_stream_state_bytes(10, 100) == 8 * 10 * (3 * 100 + SS.BLOCK + 8)
    assert lib.spk_spectrum_stream_state_bytes(24576, 4096) == 8 * 24576 * (3 * 4096 + SS.BLOCK + 8)
    assert lib.spk_spectrum_stream_finalise_workspace_bytes(7, 33) == 8 * 7 * 33
    assert lib.spk_spectrum_stream_state_bytes(1, 0) == 0
