"""fp64 numpy restatement of md/data/spectra.py in the form of csrc/spectra.cu: centroid, central difference and field
combinations, per-field normalisation, the autocorrelation as direct lag sums with channel weights, and the spectrum as
the DCT-II of the windowed lags.  ``fft_autocorrelation`` restates the reference's FFT route for the identity test.

The direct forms cost n^2 and (4L) L; above DIRECT_MAX (series of a few thousand points) ``spectrum`` takes the
zero-padded FFT routes instead (``fft_acf``, ``fft_spectrum``), which the CPU tests check against the direct forms."""
import numpy as np

C_LIGHT = 299792458.0                     # ase.units._c
RAMAN_FACTOR = 4.160440e-18
DIRECT_MAX = 10 ** 7                      # largest n (n - 1) and 4 L^2 evaluated directly


def cosine_sq_window(n):
    i = np.arange(n)
    return np.cos(np.pi * i / (n - 1) / 2) ** 2


def fields(kind, sys_ptr, m, averaged=False):
    """(index [F, 3] with -1 = unused, coef [F, 3], channels [(first, weights)]) of system m, as spectra.py builds them"""
    if kind == "power":
        a0, a1 = sys_ptr[m], sys_ptr[m + 1]
        idx = [[3 * a + k, -1, -1] for a in range(a0, a1) for k in range(3)]
        return idx, [[1.0, 0, 0]] * len(idx), [(0, [1.0 / (a1 - a0)] * len(idx))]
    if kind == "ir":
        return [[3 * m + k, -1, -1] for k in range(3)], [[1.0, 0, 0]] * 3, [(0, [1.0] * 3)]
    o = 9 * m
    xx, xy, xz, yy, yz, zz = o, o + 1, o + 2, o + 4, o + 5, o + 8
    if not averaged:
        return [[xx, -1, -1], [xy, -1, -1]], [[1.0, 0, 0]] * 2, [(0, [1.0]), (1, [1.0])]
    idx = [[xx, yy, zz], [xx, yy, -1], [yy, zz, -1], [zz, xx, -1], [xy, -1, -1], [xz, -1, -1], [yz, -1, -1]]
    coef = [[1 / 3] * 3, [1.0, -1.0, 0], [1.0, -1.0, 0], [1.0, -1.0, 0]] + [[1.0, 0, 0]] * 3
    return idx, coef, [(0, [1.0]), (1, [0.5, 0.5, 0.5, 3.0, 3.0, 3.0])]


def combine(records, index, coef, derivative, dt_fs):
    """records [T, P, S] -> the fields x [F, n] before normalisation (fp64)"""
    T, P = records.shape[:2]
    c = records.reshape(T, P, -1).astype(np.float64).mean(axis=1)
    d = (c[2:] - c[:-2]) / (2 * dt_fs) if derivative else c
    x = np.zeros((len(index), d.shape[0]))
    for f, (ii, cc) in enumerate(zip(index, coef)):
        for i, w in zip(ii, cc):
            if i >= 0:
                x[f] += w * d[:, i]
    return x


def series(records, index, coef, derivative, dt_fs):
    """records [T, P, S] -> normalised fields z [F, n] (fp64)"""
    x = combine(records, index, coef, derivative, dt_fs)
    with np.errstate(invalid="ignore", divide="ignore"):
        return (x - x.mean(axis=1, keepdims=True)) / x.std(axis=1, keepdims=True)


def direct_acf(z, n_lags):
    """C[f, k] = (1/n) sum_{t < n-k} z_f[t] z_f[t+k], k < n_lags"""
    n = z.shape[1]
    return np.stack([np.einsum("ft,ft->f", z[:, : n - k], z[:, k:]) / n for k in range(n_lags)], axis=1)


def fft_acf(z, n_lags):
    """direct_acf through the FFT of z zero-padded to 2n (no circular wrap), k < n_lags <= n"""
    n = z.shape[1]
    f = np.fft.rfft(z, n=2 * n, axis=1)
    return np.fft.irfft(f.real ** 2 + f.imag ** 2, n=2 * n, axis=1)[:, :n_lags] / n


def fft_spectrum(a, window, dt_fs):
    """dct_spectrum by the reference's route: |dt FFT| of a [..., L] zero-padded to 4L and mirrored to 8L"""
    L = a.shape[-1]
    if window is not None:
        a = a * window
    padded = np.zeros(a.shape[:-1] + (4 * L,))
    padded[..., :L] = a
    mirrored = np.concatenate((padded[..., ::-1], padded), axis=-1)
    return 2 * dt_fs * np.abs(0.5 * np.fft.fft(mirrored, n=8 * L, axis=-1)[..., : 4 * L])


def fft_autocorrelation(x, n_lags):
    """the reference's fft_autocorrelation (md/data/spectra.py:38-55): n_lags + 1 lags"""
    x = (x - np.mean(x)) / np.std(x)
    n = x.shape[0]
    f = np.fft.fft(x, n=2 * n)
    return np.real(np.fft.ifft(f * np.conjugate(f))[:n] / n)[: n_lags + 1]


def dct_spectrum(a, window, dt_fs):
    """|dt FFT| of the zero-padded, mirrored a [L] as 2 dt |sum_i a_i cos(pi m (2i+1) / (8L))|, m < 4L"""
    L = a.shape[-1]
    if window is not None:
        a = a * window
    m = np.arange(4 * L)[:, None]
    i = np.arange(L)[None, :]
    r = (m * (2 * i + 1)) % (16 * L)
    return 2 * dt_fs * np.abs(np.cos(np.pi * r / (8 * L)) @ a)


def frequencies(L, dt_fs):
    f = np.arange(4 * L) / (8 * L * dt_fs)
    return f / (C_LIGHT / 1e13)


def spectrum(kind, records, sys_ptr, n_replicas, dt_fs, m, resolution=4096, averaged=False, incident_frequency=None,
             temperature=None, hbar2icm=None, kB=None, window=cosine_sq_window):
    """(frequencies, [intensities], per-field acf [F, n-1], channel acf [C, L]) of system m"""
    derivative = kind != "power"
    idx, coef, channels = fields(kind, sys_ptr, m, averaged)
    T = records.shape[0]
    z = series(records.reshape(T, n_replicas, -1), idx, coef, derivative, dt_fs)
    n = z.shape[1]
    acf_fields = direct_acf(z, n - 1) if n * (n - 1) <= DIRECT_MAX else fft_acf(z, n - 1)
    L = min(resolution, n - 1)
    chans = []
    for first, w in channels:
        chans.append(sum(wf * acf_fields[first + j] for j, wf in enumerate(w))[:L])
    chans = np.stack(chans)
    win = window(L) if window is not None else None
    transform = dct_spectrum if 4 * L * L <= DIRECT_MAX else fft_spectrum
    out = [transform(a, win, dt_fs) for a in chans]
    freq = frequencies(L, dt_fs)
    if kind == "raman":
        with np.errstate(invalid="ignore", divide="ignore"):
            cs = (incident_frequency - freq) ** 4 / freq / (1 - np.exp(-(hbar2icm * freq) / (kB * temperature)))
        cs[0] = 0
        out = [v * cs * RAMAN_FACTOR for v in out]
        for v in out:
            v[0] = 0.0
        if averaged:
            out = [out[0] + 4 / 45 * out[1], out[1] / 15]
    return freq, out, acf_fields, chans


PROP = {"power": "velocities", "ir": "dipole_moment", "raman": "polarizability"}
GOLDEN = ("spectra_power", "spectra_ir", "spectra_raman", "spectra_short", "spectra_zero", "spectra_long")


def golden(name):
    """the fixture's arrays and its runs: [(r, run, m)] for every run r and system m"""
    import json
    import os

    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name + ".npz"))
    runs = json.loads(str(z["runs"]))
    B = len(z["sys_ptr"]) - 1
    return z, [(r, run, m) for r, run in enumerate(runs) for m in range(B)]


def rel_err(x, ref):
    """max-norm relative error over the finite entries; inf when the NaN masks differ"""
    x, ref = np.asarray(x, np.float64), np.asarray(ref, np.float64)
    if x.shape != ref.shape or not np.array_equal(np.isnan(x), np.isnan(ref)):
        return np.inf
    ok = ~np.isnan(ref)
    if not ok.any():
        return 0.0
    return float(np.abs(x[ok] - ref[ok]).max() / max(np.abs(ref[ok]).max(), 1e-300))
