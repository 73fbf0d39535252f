"""GPU checks of the spectra kernels (csrc/spectra.cu) at the lengths MD runs give, against fp64 oracles that do not share
the kernels' tiling: the stored-series autocorrelation over many time chunks and lag blocks, the transform on both
sides of its shared-memory cosine table and with a partial channel group, the series preparation at T = 20 000, the
stream's push / block update / finalise driven directly (lag-tile switches, a ring that wraps many times, grids with
more items than CTAs), and one end-to-end headed PaiNN run long enough for all of it.

Every case prints what it reached (n, L, n_chunks, n_xb, the transform's table placement, the block-update items
against its CTAs) and its largest error, so a run with -s shows which paths ran."""
from ctypes import c_void_p

import numpy as np
import pytest
import torch
from scipy.signal import lfilter

import spectra_oracle as SO
from schnetpack_b200 import _lib, ops
from schnetpack_b200 import atomistic as A
from schnetpack_b200 import md as M
from schnetpack_b200 import spectra as SP
from schnetpack_b200 import synthetic as S
from schnetpack_b200.model import NeuralNetworkPotential, batch_to_device, from_spec

import heads_oracle as HO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = 1e-10
CHUNK = 2048                    # SPK_SPECTRUM_CHUNK: time rows per CTA of the autocorrelation
LAG_BLOCK = 256                 # lags per CTA column block (8 AC_TPC)
TABLE_MAX = 160 * 1024          # the transform stages its cosine table in shared memory up to this many bytes
BLOCK = 64                      # SPK_SPECTRUM_STREAM_BLOCK


def n_chunks(n):
    return -(-n // CHUNK)


def n_xb(L):
    return -(-(-(-(L + 15) // 8)) // 32)


def staged(L):
    return (4 * L + 1) * 8 <= TABLE_MAX


def _t(a, dtype=torch.float64):
    return torch.as_tensor(np.asarray(a), dtype=dtype).to(DEV)


def _fields(rng, F, n, offset=0.0):
    """F fp64 series of AR(1) noise plus a sinusoid (the acf stays large at long lags), rows [F, n]"""
    out = np.empty((F, n))
    t = np.arange(n)
    for f in range(F):
        phi = rng.uniform(0.5, 0.995)
        x = lfilter([1.0], [1.0, -phi], rng.normal(size=n))
        x = x / x.std() + 2.0 * np.sin(rng.uniform(0.002, 0.3) * t + rng.uniform(0, 2 * np.pi))
        out[f] = x + offset * x.std()
    return out


def _normalised(x):
    return (x - x.mean(axis=1, keepdims=True)) / x.std(axis=1, keepdims=True)


def _acf_oracle(z, n_lags):
    """per-field acf [F, n_lags] of z [F, n], fp64: direct sums while small, the zero-padded FFT beyond"""
    F, n = z.shape
    return SO.direct_acf(z, n_lags) if n * n_lags * F <= 10 ** 8 else SO.fft_acf(z, n_lags)


def _channels(acf_fields, ch_ptr, weight):
    return np.stack([np.asarray(weight[a:b]) @ acf_fields[a:b] for a, b in zip(ch_ptr[:-1], ch_ptr[1:])])


def _channel_errs(got, ref):
    return [SO.rel_err(g, r) for g, r in zip(got, ref)]


# ---- stored-series autocorrelation ------------------------------------------------------------------------------------
# (n, L): one chunk, an exact chunk, one row into a second chunk, three chunks and 17 rows, production length; L at the
# n_xb steps (241/242, 497/498), inside the two-block lags 240..263 of the reduce, at n - 1 and at 4096/4097
SHAPES = [(3, 1), (3, 2), (17, 1), (17, 15), (17, 16),
          (2047, 16), (2047, 257), (2047, 2046),
          (2048, 17), (2048, 241), (2048, 2047),
          (2049, 1), (2049, 2), (2049, 242), (2049, 263), (2049, 2048),
          (4097, 15), (4097, 240), (4097, 497), (4097, 4096),
          (6161, 2), (6161, 16), (6161, 256), (6161, 498), (6161, 4097), (6161, 6160),
          (20000, 1), (20000, 2), (20000, 15), (20000, 17), (20000, 241), (20000, 242), (20000, 248), (20000, 257),
          (20000, 264), (20000, 497), (20000, 498), (20000, 4096), (20000, 4097), (20000, 19999)]

# fields per channel (4 + 3 pads the fourth DMMA field, 7 = averaged Raman) and the sign pattern of their weights
COUNTS = [1, 2, 3, 4, 5, 7, 9]
SIGNS = ["pos", "neg", "zero", "mixed"]


def _layout(rng, C):
    """ch_ptr [C + 1] and weights of C channels cycling through COUNTS and SIGNS"""
    ch_ptr, weight = [0], []
    for c in range(C):
        k, sign = COUNTS[c % len(COUNTS)], SIGNS[(c // len(COUNTS) + c) % len(SIGNS)]
        w = rng.uniform(0.25, 2.0, size=k)
        if sign == "neg":
            w = -w
        elif sign == "zero":
            w[0] = 0.0
        elif sign == "mixed":
            w[::2] *= -1.0
            w[0] = 3.0 * w.size                     # keeps the channel's acf[0] away from a cancellation
        weight += w.tolist()
        ch_ptr.append(len(weight))
    return ch_ptr, weight


def _acf(z, ch_ptr, weight, L):
    return SP.autocorrelation(z, _t(ch_ptr, torch.int64), _t(weight), L)


def _check_acf(n, L, C, seed):
    rng = np.random.default_rng(seed)
    ch_ptr, weight = _layout(rng, C)
    zh = _normalised(_fields(rng, ch_ptr[-1], n, offset=rng.uniform(-5, 5)))
    z = _t(zh)
    got = _acf(z, ch_ptr, weight, L)
    ref = _channels(_acf_oracle(zh, L), ch_ptr, weight)
    errs = _channel_errs(got.cpu().numpy(), ref)
    print(f"acf n={n} L={L} C={C} F={ch_ptr[-1]} n_chunks={n_chunks(n)} n_xb={n_xb(L)} max_err={max(errs):.2e}")
    assert max(errs) <= TOL, (n, L, C, errs)
    return z, ch_ptr, weight, got


@pytest.mark.parametrize("shape", SHAPES, ids=[f"n{n}-L{L}" for n, L in SHAPES])
def test_autocorrelation_shapes(shape):
    n, L = shape
    _check_acf(n, L, 3, seed=n * 31 + L)


# (n, L, channels): 1, 9 and 17 channels on multi-chunk series, and one launch of 300 channels
LAYOUTS = [(20000, 4096, 1), (6161, 498, 9), (20000, 263, 17), (4097, 1100, 17), (2049, 300, 300)]


def _bitwise_properties(z, ch_ptr, weight, L, got, rng):
    """each channel alone equals its row, a second launch equals the first, and a channel permutation permutes rows"""
    C = len(ch_ptr) - 1
    again = _acf(z, ch_ptr, weight, L)
    assert torch.equal(again, got)
    for c in sorted({0, C // 2, C - 1}):
        a, b = ch_ptr[c], ch_ptr[c + 1]
        alone = _acf(z[a:b].contiguous(), [0, b - a], weight[a:b], L)
        assert torch.equal(alone[0], got[c]), c
    perm = rng.permutation(C)
    rows, p_ptr, p_w = [], [0], []
    for c in perm:
        a, b = ch_ptr[c], ch_ptr[c + 1]
        rows += range(a, b)
        p_w += weight[a:b]
        p_ptr.append(len(rows))
    permuted = _acf(z[torch.as_tensor(rows, device=DEV)].contiguous(), p_ptr, p_w, L)
    assert torch.equal(permuted, got[torch.as_tensor(perm, device=DEV)])


@pytest.mark.parametrize("layout", LAYOUTS, ids=[f"n{n}-L{L}-C{C}" for n, L, C in LAYOUTS])
def test_autocorrelation_channel_layouts(layout):
    n, L, C = layout
    z, ch_ptr, weight, got = _check_acf(n, L, C, seed=C)
    _bitwise_properties(z, ch_ptr, weight, L, got, np.random.default_rng(C + 1))


# ---- transform --------------------------------------------------------------------------------------------------------
TRANSFORM_L = [1, 2, 3, 255, 256, 257, 4096, 5119, 5120, 8192]


def _direct_dct(a, window, dt_fs, rows=512):
    """2 dt |sum_i a_i cos(pi m (2i+1) / (8L))| for a [C, L], the cosine matrix built rows bins at a time"""
    C, L = a.shape
    aw = a * window if window is not None else a
    out = np.empty((C, 4 * L))
    i = np.arange(L)[None, :]
    for m0 in range(0, 4 * L, rows):
        m = np.arange(m0, min(m0 + rows, 4 * L))[:, None]
        out[:, m0:m0 + m.shape[0]] = (np.cos(np.pi * ((m * (2 * i + 1)) % (16 * L)) / (8 * L)) @ aw.T).T
    return 2 * dt_fs * np.abs(out)


@pytest.mark.parametrize("L", TRANSFORM_L)
def test_transform_shapes(L):
    rng = np.random.default_rng(L)
    k = np.arange(L)
    acf = np.stack([np.exp(-k / rng.uniform(5, 2 * L + 5)) * np.cos(rng.uniform(0.01, 1.0) * k)
                    + 0.05 * rng.normal(size=L) for _ in range(17)])
    a = _t(acf)
    dt = 0.5
    for win_np in [None] + ([SP.cosine_sq_window(L)] if L > 1 else []):      # the window needs two points
        win = None if win_np is None else _t(win_np)
        ref = SO.fft_spectrum(acf, win_np, dt)
        full = None
        for C in (17, 1, 8, 9):
            got = SP.transform(a[:C].contiguous(), win, dt)
            errs = _channel_errs(got.cpu().numpy(), ref[:C])
            print(f"transform L={L} C={C} window={win_np is not None} stage={int(staged(L))} max_err={max(errs):.2e}")
            assert max(errs) <= TOL, (L, C, errs)
            if full is None:
                full = got
            else:
                assert torch.equal(got, full[:C]), (L, C)       # a channel's bins do not depend on its group
        if L in (5119, 5120) and win_np is not None:                # about 4 s of host cosines each
            direct = _direct_dct(acf[:9], win_np, dt)
            err = max(_channel_errs(full[:9].cpu().numpy(), direct))
            print(f"transform L={L} direct DCT max_err={err:.2e}")
            assert err <= TOL, (L, err)
    assert staged(5119) and not staged(5120)


# ---- series -----------------------------------------------------------------------------------------------------------
def _series_table():
    """fields over two polarizability-like systems (stride 18): Raman combinations, -1 in every slot, single components"""
    idx, coef = [], []
    for m in range(2):
        i, c, _ = SP.RamanSpectrum._table([0, 1, 2], m, True)
        idx += i
        coef += c
    idx += [[-1, 5, -1], [3, -1, 16], [-1, -1, 17], [9, 10, 11]]
    coef += [[0.0, 2.5, 0.0], [1.0, 0.0, -0.75], [0.0, 0.0, 1.0], [0.5, -1.5, 0.25]]
    return idx, coef


@pytest.mark.parametrize("P", [1, 8, 32])
def test_series_long(P):
    rng = np.random.default_rng(P)
    T, stride, dt = 20000, 18, 0.5
    x = _fields(rng, stride * P, T, offset=3.0).reshape(P, stride, T).transpose(2, 0, 1)
    rec_np = np.ascontiguousarray(x).astype(np.float32)
    rec = _t(rec_np, torch.float32)
    idx, coef = _series_table()
    idx_t, coef_t = _t(idx, torch.int64), _t(coef)      # held: a freed argument's memory is reused before the launch
    F = len(idx)
    for derivative in (0, 1):
        n = T - 2 if derivative else T
        z = torch.empty(F, n, dtype=torch.float64, device=DEV)
        mean = torch.empty(F, dtype=torch.float64, device=DEV)
        std = torch.empty(F, dtype=torch.float64, device=DEV)
        _lib.call("spk_spectrum_series", ops._p(rec), T, P, stride, ops._p(idx_t), ops._p(coef_t), F, derivative, dt,
                  ops._p(z), ops._p(mean), ops._p(std), ops._stream())
        xr = SO.combine(rec_np, idx, coef, derivative, dt)
        zr = SO.series(rec_np, idx, coef, derivative, dt)
        m_ref, s_ref = xr.mean(axis=1), xr.std(axis=1)
        z_err = max(SO.rel_err(a, b) for a, b in zip(z.cpu().numpy(), zr))
        # a mean is a sum of values of size std: its error is measured on that scale (a derivative's mean is ~0)
        m_err = float((np.abs(mean.cpu().numpy() - m_ref) / (np.abs(m_ref) + s_ref)).max())
        s_err = float((np.abs(std.cpu().numpy() - s_ref) / s_ref).max())
        print(f"series T={T} P={P} F={F} derivative={derivative} z_err={z_err:.2e} mean_err={m_err:.2e} "
              f"std_err={s_err:.2e}")
        assert max(z_err, m_err, s_err) <= 1e-12, (P, derivative, z_err, m_err, s_err)


# ---- stream -----------------------------------------------------------------------------------------------------------
class DirectStream:
    """one stream state driven through spk_spectrum_stream_push with per-frame source views [P, stride] and per-step
    counters, as the captured MD step drives it"""

    def __init__(self, frames, index, coef, L, every, derivative, dt=0.5):
        self.frames, self.P, self.stride = frames, int(frames.shape[1]), int(frames.shape[2])
        self.index, self.coef = _t(index, torch.int64), _t(coef)
        self.F, self.L, self.every, self.derivative, self.dt = len(index), L, every, derivative, dt
        nbytes = int(_lib.lib().spk_spectrum_stream_state_bytes(self.F, L))
        self.state = torch.zeros(nbytes // 8, dtype=torch.float64, device=DEV)
        self.steps = torch.arange(int(frames.shape[0]) * every, dtype=torch.int64, device=DEV)
        self.step = 0

    def frames_done(self):
        return self.step // self.every

    def advance(self, n_frames):
        """run steps until n_frames frames are sampled; a step reads source frame step // every"""
        lib = _lib.lib()
        fb = self.frames.element_size() * self.P * self.stride
        f0, s0 = self.frames.data_ptr(), self.steps.data_ptr()
        args = (self.P, self.stride, ops._p(self.index), ops._p(self.coef), self.F, self.derivative, self.dt)
        while self.frames_done() < n_frames:
            s = self.step
            rc = lib.spk_spectrum_stream_push(c_void_p(f0 + (s // self.every) * fb), None, *args, c_void_p(s0 + 8 * s),
                                              self.every, self.L, ops._p(self.state), ops._stream())
            _lib.check(rc, "spk_spectrum_stream_push")
            self.step += 1

    def samples(self):
        return self.frames_done() - (2 if self.derivative else 0)

    def finalise(self, fields, ch_ptr, weight, Lo):
        n = self.samples()
        C = len(ch_ptr) - 1
        acf = torch.empty(C, Lo, dtype=torch.float64, device=DEV)
        ws = torch.empty(max(int(_lib.lib().spk_spectrum_stream_finalise_workspace_bytes(len(fields), Lo)), 8),
                         dtype=torch.uint8, device=DEV)
        sel, ch, w = _t(fields, torch.int64), _t(ch_ptr, torch.int64), _t(weight)
        _lib.call("spk_spectrum_stream_finalise", ops._p(self.state), self.F, self.L, n, ops._p(sel), len(fields),
                  ops._p(ch), ops._p(w), C, Lo, ops._p(acf), ops._p(ws), ws.numel(), ops._stream())
        return acf

    def rows(self, f):
        """(S, head, ring, scalars) of field f"""
        F, L = self.F, self.L
        R = L + BLOCK
        st = self.state
        return (st[f * L:(f + 1) * L], st[F * L + f * L:F * L + (f + 1) * L],
                st[2 * F * L + f * R:2 * F * L + (f + 1) * R], st[F * (2 * L + R) + 8 * f:F * (2 * L + R) + 8 * (f + 1)])


def _stream_source(rng, n_frames, P, stride):
    """fp32 frames [n_frames, P, stride] with |mean| / std up to about 5 per component"""
    x = _fields(rng, P * stride, n_frames, offset=rng.uniform(-4, 4))
    return np.ascontiguousarray(x.reshape(P, stride, n_frames).transpose(2, 0, 1)).astype(np.float32)


def _stream_table(rng, F, stride):
    idx, coef = [], []
    for f in range(F):
        k = 1 + f % 3
        comp = rng.choice(stride, size=k, replace=False).tolist() + [-1] * (3 - k)
        perm = rng.permutation(3)
        idx.append([comp[j] for j in perm])
        coef.append([float(rng.uniform(0.5, 1.5) * (1 if rng.random() < 0.7 else -1)) if comp[j] >= 0 else 0.0
                     for j in perm])
    return idx, coef


def _stream_oracle(frames_np, idx, coef, derivative, dt, n, Lo):
    used = frames_np[: n + (2 if derivative else 0)]
    return _acf_oracle(SO.series(used, idx, coef, derivative, dt), Lo)


def _stream_items(F, L):
    """(field, lag tile) items of the block update: tiles of 1024 lags above L = 512, 512 above 256, else one"""
    Q = 4 if L > 512 else 2 if L > 256 else 1
    T = 256 if Q > 1 else -(-L // 32) * 32
    return F * -(-L // (T * Q))


STREAM_L = [32, 33, 256, 257, 512, 513, 1024, 1025, 4096, 4097]
COMBOS = [(every, derivative, P) for every in (1, 3) for derivative in (0, 1) for P in (1, 4)]
STREAM_CASES = [(L,) + COMBOS[(2 * i + j) % len(COMBOS)] for i, L in enumerate(STREAM_L) for j in range(2)]


@pytest.mark.parametrize("case", STREAM_CASES, ids=[f"L{L}-every{e}-d{d}-P{P}" for L, e, d, P in STREAM_CASES])
def test_stream_direct(case):
    L, every, derivative, P = case
    rng = np.random.default_rng(L * 8 + every * 4 + derivative * 2 + P)
    R = L + BLOCK
    # sample counts: fewer than L, L + 1, not a multiple of the block, a ring wrapped more than three times
    checkpoints = sorted({max(3, L // 2 + 1), L + 1, L + 2 * BLOCK + 37, 3 * R + L // 3 + 45})
    F, stride = 6, 7
    extra = 2 if derivative else 0
    frames_np = _stream_source(rng, checkpoints[-1] + extra, P, stride)
    idx, coef = _stream_table(rng, F, stride)
    st = DirectStream(_t(frames_np, torch.float32), idx, coef, L, every, derivative)
    fields, ch_ptr, weight = [4, 0, 2, 5], [0, 1, 3, 4], [1.0, 0.5, -2.0, 0.75]      # a non-contiguous selection
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    for n in checkpoints:
        st.advance(n + extra)
        assert st.samples() == n
        outs = sorted({1, min(L, n - 1, 200), min(L, n - 1, 2 * LAG_BLOCK + 45), min(L, n - 1)})
        ref_fields = _stream_oracle(frames_np, idx, coef, derivative, 0.5, n, outs[-1])
        for Lo in outs:
            got = st.finalise(fields, ch_ptr, weight, Lo).cpu().numpy()
            ref = _channels(ref_fields[fields, :Lo], ch_ptr, weight)
            err = max(_channel_errs(got, ref))
            print(f"stream L={L} every={every} derivative={derivative} P={P} n={n} Lo={Lo} wraps={n / R:.2f} "
                  f"items={_stream_items(F, L)} ctas={min(_stream_items(F, L), 8 * sms)} max_err={err:.2e}")
            assert err <= TOL, (case, n, Lo, err)


# (F, L, samples): more (field, lag-tile) items than the 8 CTAs per SM of the block update
BIG_STREAMS = [(300, 4096, 4200), (1100, 64, 500)]


@pytest.mark.parametrize("big", BIG_STREAMS, ids=[f"F{F}-L{L}" for F, L, _ in BIG_STREAMS])
def test_stream_grid_stride(big):
    F, L, n = big
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    items = _stream_items(F, L)
    assert items > 8 * sms, (items, sms)
    rng = np.random.default_rng(F)
    P, stride = 2, 96
    frames_np = _stream_source(rng, n, P, stride)
    frames = _t(frames_np, torch.float32)
    idx, coef = _stream_table(rng, F, stride)
    st = DirectStream(frames, idx, coef, L, 1, 0)
    st.advance(n)
    # the first field, the first field whose items are second items of a CTA (item >= grid) and the last field
    tiles = items // F
    watch = [0, -(-8 * sms // tiles), F - 1]
    assert watch[1] < F - 1
    small = DirectStream(frames, [idx[f] for f in watch], [coef[f] for f in watch], L, 1, 0)
    small.advance(n)
    for j, f in enumerate(watch):
        for name, a, b in zip(("S", "head", "ring", "scalars"), st.rows(f), small.rows(j)):
            assert torch.equal(a, b), (F, L, f, name)
    fields = list(range(F - 1, -1, -7))
    ch_ptr = [0, len(fields) // 2, len(fields)]
    weight = [1.0 / len(fields)] * len(fields)
    Lo = min(L, n - 1)
    got = st.finalise(fields, ch_ptr, weight, Lo).cpu().numpy()
    ref = _channels(_stream_oracle(frames_np, idx, coef, 0, 0.5, n, Lo)[fields], ch_ptr, weight)
    err = max(_channel_errs(got, ref))
    print(f"stream F={F} L={L} n={n} items={items} ctas={8 * sms} watched={watch} max_err={err:.2e}")
    assert err <= TOL, (F, L, err)


# ---- end to end -------------------------------------------------------------------------------------------------------
def test_end_to_end_production_length():
    """headed PaiNN aspirin x 3, NVE, 6200 steps recorded at every step and streamed at resolution 6000: power, IR,
    Raman and averaged Raman at 4096 (staged table) and 6000 (global table) from the records and from the stream, both
    against the fp64 oracle of the host records (four time chunks, 17 and 25 lag blocks)"""
    spec = S.model_spec("painn", n_atom_basis=32, n_interactions=2)
    base = from_spec(spec, S.init_params(spec, seed=3))
    torch.manual_seed(1)
    heads = [A.DipoleMoment(32, use_vector_representation=True), A.Polarizability(32)]
    model = NeuralNetworkPotential(base.representation, list(base.input_modules), list(base.output_modules) + heads,
                                   postprocessors=[], do_postprocessing=False).to(DEV).eval()
    data = HO._centered(S.aspirin_batch(3, seed=2))
    masses = torch.as_tensor([HO.MASSES[int(z)] for z in data[S.Z]], dtype=torch.float32)
    rng = np.random.default_rng(0)
    width = np.sqrt(masses.numpy() * M.KB_MD * 300.0)[:, None]
    momenta = torch.as_tensor(rng.normal(size=(masses.shape[0], 3)) * width, dtype=torch.float32)
    steps, res = 6200, 6000
    stream = SP.SpectrumStream(["power", "ir", "raman", "raman_averaged"], resolution=res)
    md = M.DeviceMD(model, batch_to_device(data, DEV), masses, time_step=0.5 * M.FS_MD, cutoff=spec["cutoff"],
                    capacity=int(data[S.Z].shape[0]) * 160, momenta=momenta,
                    required_properties=["dipole_moment", "polarizability"], record_capacity=steps,
                    record_velocities=True, stream=stream)
    md.run(steps)
    host = {k: md.recorded(k).numpy() for k in ("velocities", "dipole_moment", "polarizability")}
    s = md.series()

    def spectra(data_, kind, resolution, averaged):
        if kind == "power":
            return SP.PowerSpectrum(data_, resolution=resolution)
        if kind == "ir":
            return SP.IRSpectrum(data_, resolution=resolution)
        return SP.RamanSpectrum(data_, 19455.25, 300.0, resolution=resolution, averaged=averaged)

    for kind, averaged in (("power", False), ("ir", False), ("raman", False), ("raman", True)):
        for resolution in (4096, res):
            oracle = [SO.spectrum(kind, host[SO.PROP[kind]], s.sys_ptr, 1, s.dt_fs, m, resolution=resolution,
                                  averaged=averaged, incident_frequency=19455.25, temperature=300.0,
                                  hbar2icm=SP.HBAR2ICM, kB=M.KB_MD) for m in range(3)]
            for data_ in (md, stream):
                sp = spectra(data_, kind, resolution, averaged)
                sp.compute_spectrum(None)
                worst = 0.0
                for m, (freq, ints, _, chans) in enumerate(oracle):
                    worst = max(worst, SO.rel_err(sp.autocorrelation[m].cpu().numpy(), chans))
                    for j, v in enumerate(ints):
                        worst = max(worst, SO.rel_err(sp.intensities[j][m].cpu().numpy(), v))
                    assert np.array_equal(sp.frequencies[0].cpu().numpy(), freq)
                n = steps - (0 if kind == "power" else 2)
                L = min(resolution, n - 1)
                print(f"end-to-end {kind}{' averaged' if averaged else ''} from "
                      f"{'stream' if data_ is stream else 'records'} n={n} L={L} n_chunks={n_chunks(n)} "
                      f"n_xb={n_xb(L)} stage={int(staged(L))} max_err={worst:.2e}")
                assert worst <= TOL, (kind, averaged, resolution, data_ is stream, worst)
