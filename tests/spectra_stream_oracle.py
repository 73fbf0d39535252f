"""fp64 numpy restatement of the streaming autocorrelation of csrc/spectra.cu (DESIGN.md section 20): per field the
shifted values y = x - x[0], the band sums S[k] = sum_{t < n-k} y[t] y[t+k] added in fixed blocks of BLOCK samples, the
running sum Y, the first L values and a ring of the last L + BLOCK values; ``acf`` applies the mean correction to give
the normalised autocorrelation of spectra_oracle.direct_acf.  ``fields_of`` forms the fields of a record series frame by
frame (centroid over the replicas, central difference lagging two frames) as the device push does."""
import numpy as np

import spectra_oracle as SO

BLOCK = 64                                # SPK_SPECTRUM_STREAM_BLOCK


class Stream:
    def __init__(self, n_fields, n_lags, block=BLOCK):
        self.F, self.L, self.block = int(n_fields), int(n_lags), int(block)
        self.R = self.L + self.block
        self.S = np.zeros((self.F, self.L))
        self.head = np.zeros((self.F, self.L))
        self.ring = np.zeros((self.F, self.R))
        self.Y = np.zeros(self.F)
        self.shift = np.zeros(self.F)
        self.n = 0

    def _y(self, t):
        return self.ring[:, t % self.R]

    def _band(self, b0, b1, n_lags):
        """sum_{b0 <= u < b1} y[u] y[u - k] for k < n_lags (u - k >= 0), in sample order"""
        acc = np.zeros((self.F, n_lags))
        for u in range(b0, b1):
            k = np.arange(min(u + 1, n_lags))
            acc[:, k] += self._y(u)[:, None] * self.ring[:, (u - k) % self.R]
        return acc

    def extend(self, xs):
        """push the samples xs [m, F] in order; a block's band is added to S when its last sample arrives"""
        for x in np.atleast_2d(np.asarray(xs, np.float64)):
            u = self.n
            if u == 0:
                self.shift = x.copy()
            y = x - self.shift
            self.ring[:, u % self.R] = y
            if u < self.L:
                self.head[:, u] = y
            self.Y = self.Y + y
            self.n = u + 1
            if self.n % self.block == 0:
                self.S += self._band(self.n - self.block, self.n, self.L)

    def state(self):
        return dict(S=self.S, head=self.head, ring=self.ring, Y=self.Y, shift=self.shift, n=self.n)

    def acf(self, n_out):
        """C [F, n_out] = (1/n) sum_{t < n-k} (x[t] - mean)(x[t+k] - mean) / var, n_out <= min(L, n - 1)"""
        n = self.n
        assert 1 <= n_out <= min(self.L, n - 1)
        S = self.S[:, :n_out] + self._band(n - n % self.block, n, n_out)
        H = np.concatenate([np.zeros((self.F, 1)), np.cumsum(self.head[:, :n_out - 1], axis=1)], axis=1)
        last = np.stack([self._y(n - 1 - k) for k in range(n_out - 1)], axis=1) if n_out > 1 else np.zeros((self.F, 0))
        tail = np.concatenate([np.zeros((self.F, 1)), np.cumsum(last, axis=1)], axis=1)
        m = self.Y / n
        var = S[:, 0] / n - m * m
        k = np.arange(n_out)
        with np.errstate(invalid="ignore", divide="ignore"):
            return (S - m[:, None] * (2 * self.Y[:, None] - H - tail) + (n - k) * (m * m)[:, None]) / (n * var)[:, None]


def fields_of(records, index, coef, derivative, dt_fs):
    """the field values [n, F] of records [T, P, S], one frame at a time as the device push forms them"""
    T, P = records.shape[:2]
    flat = records.reshape(T, P, -1)
    hist, out = [], []
    for t in range(T):
        c = flat[t].astype(np.float64).sum(axis=0) / P
        hist.append(c)
        if derivative:
            if t < 2:
                continue
            d = (c - hist[t - 2]) / (2 * dt_fs)
        else:
            d = c
        x = np.zeros(len(index))
        for f, (ii, cc) in enumerate(zip(index, coef)):
            for i, w in zip(ii, cc):
                if i >= 0:
                    x[f] += w * d[i]
        out.append(x)
    return np.array(out).reshape(-1, len(index))


def spectrum_from_acf(kind, acf_fields, channels, L, dt_fs, averaged=False, incident_frequency=None, temperature=None,
                      hbar2icm=None, kB=None, window=SO.cosine_sq_window):
    """(frequencies, [intensities], channel acf [C, L]) from the per-field acf, as spectra_oracle.spectrum finishes"""
    chans = np.stack([sum(wf * acf_fields[first + j, :L] for j, wf in enumerate(w)) for first, w in channels])
    win = window(L) if window is not None else None
    out = [SO.dct_spectrum(a, win, dt_fs) for a in chans]
    freq = SO.frequencies(L, dt_fs)
    if kind == "raman":
        with np.errstate(invalid="ignore", divide="ignore"):
            cs = (incident_frequency - freq) ** 4 / freq / (1 - np.exp(-(hbar2icm * freq) / (kB * temperature)))
        cs[0] = 0
        out = [v * cs * SO.RAMAN_FACTOR for v in out]
        for v in out:
            v[0] = 0.0
        if averaged:
            out = [out[0] + 4 / 45 * out[1], out[1] / 15]
    return freq, out, chans
