"""CPU checks of tests/spectra_oracle.py: the reference's spectra (fixtures of the unmodified md/data/spectra.py), the
direct-lag autocorrelation against the FFT one, a pure cosine and the NaN channels of zero-variance fields."""
import numpy as np
import pytest

import spectra_oracle as SO
from schnetpack_b200.md import KB_MD
from schnetpack_b200.spectra import HBAR2ICM


def _oracle(z, run, m):
    kind = run["kind"]
    return SO.spectrum(kind, z["rec:" + SO.PROP[kind]], list(z["sys_ptr"]), int(z["n_replicas"]), float(z["dt_fs"]), m,
                       resolution=run["resolution"], averaged=run.get("averaged", False), incident_frequency=19455.25,
                       temperature=300.0, hbar2icm=HBAR2ICM, kB=KB_MD)


@pytest.mark.parametrize("name", SO.GOLDEN)
def test_oracle_matches_reference_fixtures(name):
    z, cases = SO.golden(name)
    for r, run, m in cases:
        freq, ints, acf, _ = _oracle(z, run, m)
        key = f"r{r}:m{m}"
        assert np.array_equal(freq, z[key + ":freq"]), key
        ref = z[key + ":acf"]                     # every lag, or the lags the spectrum uses (spectra_long)
        assert ref.shape[1] in (acf.shape[1], min(run["resolution"], acf.shape[1])), key
        assert SO.rel_err(acf[:, :ref.shape[1]], ref) <= 1e-12, key
        for j, v in enumerate(ints):
            assert SO.rel_err(v, z[f"{key}:I{j}"]) <= 1e-12, (key, j, SO.rel_err(v, z[f"{key}:I{j}"]))


def test_direct_autocorrelation_equals_fft():
    rng = np.random.default_rng(3)
    for n in (3, 4, 17, 250, 1001):
        x = rng.normal(size=n).cumsum() + np.sin(np.arange(n) * 0.3)
        z = ((x - x.mean()) / x.std())[None]
        direct = SO.direct_acf(z, n - 1)[0]
        fft = SO.fft_autocorrelation(x, n - 2)
        assert np.abs(direct - fft).max() <= 1e-13, n


def test_dct_equals_mirrored_fft():
    rng = np.random.default_rng(4)
    for L in (2, 5, 64, 300):
        a = rng.normal(size=L)
        padded = np.zeros(4 * L)
        padded[:L] = a
        mirrored = np.hstack((np.flipud(padded), padded))
        ref = np.abs(0.5 * np.fft.fft(mirrored, n=8 * L)[: 4 * L])
        assert np.abs(SO.dct_spectrum(a, None, 0.5) - ref).max() <= 1e-12 * np.abs(ref).max(), L


def test_fft_routes_equal_direct_forms():
    """the long-series routes of spectrum(): fft_acf against direct_acf over several FFT lengths (n = 4097 pads to
    8194) and fft_spectrum against the DCT-II with and without the window"""
    rng = np.random.default_rng(5)
    for n, L in ((3, 2), (64, 63), (4097, 300)):
        x = rng.normal(size=(3, n)).cumsum(axis=1) + np.sin(np.arange(n) * 0.3)
        z = (x - x.mean(axis=1, keepdims=True)) / x.std(axis=1, keepdims=True)
        direct = SO.direct_acf(z, L)
        assert np.abs(SO.fft_acf(z, L) - direct).max() <= 1e-13 * np.abs(direct).max(), n
    for L in (2, 3, 257, 700):
        a = rng.normal(size=(2, L))
        for win in (None, SO.cosine_sq_window(L)):
            ref = np.stack([SO.dct_spectrum(v, win, 0.5) for v in a])
            assert SO.rel_err(SO.fft_spectrum(a, win, 0.5), ref) <= 1e-12, L


def test_cosine_series_peaks_in_its_bin():
    dt, T, L = 0.5, 4000, 512
    freq = SO.frequencies(L, dt)
    target = 120                                              # bin of the test frequency
    nu = freq[target] * 100 * SO.C_LIGHT                      # cm^-1 -> Hz
    t = np.arange(T) * dt * 1e-15
    rec = np.cos(2 * np.pi * nu * t)[:, None, None] * np.ones((1, 1, 3))
    rec[:, 0, 1] *= 0.5
    rec[:, 0, 2] *= 0.25
    f, ints, _, _ = SO.spectrum("ir", rec.astype(np.float64), [0, 1], 1, dt, 0, resolution=L)
    assert np.argmax(ints[0]) == target


def test_nan_channels_match_reference():
    z, cases = SO.golden("spectra_zero")
    seen = 0
    for r, run, m in cases:
        _, ints, _, _ = _oracle(z, run, m)
        for j, v in enumerate(ints):
            ref = z[f"r{r}:m{m}:I{j}"]
            assert np.array_equal(np.isnan(v), np.isnan(ref))
            seen += int(np.isnan(ref[1:]).all())
    assert seen == 5        # power and IR of system 0, the Raman channels of system 1 with xy (bin 0 is set to 0)
