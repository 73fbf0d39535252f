"""GPU checks of the streaming spectra (spk_spectrum_stream_*, spectra.SpectrumStream, DeviceMD(stream=...)): the
power, IR and Raman spectra of a headed PaiNN run from the stream equal those of the stored records (NVE, NVT and
4-bead RPMD), the stream's state does not depend on how the run is split or restarted, a drain does not touch it, it
runs without a recorder, and every refusal."""
import numpy as np
import pytest
import torch

import spectra_oracle as SO
import spectra_stream_oracle as SS
from schnetpack_b200 import atomistic as A
from schnetpack_b200 import md as M
from schnetpack_b200 import spectra as SP
from schnetpack_b200 import synthetic as S
from schnetpack_b200.model import NeuralNetworkPotential, batch_to_device, from_spec

import heads_oracle as HO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KEYS = ["dipole_moment", "polarizability"]
KINDS = ["power", "ir", "raman", "raman_averaged"]
TOL = 1e-10


@pytest.fixture(scope="module")
def setup():
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
    return spec, model, data, masses, momenta


def _md(setup, stream, props=KEYS, capacity=0, **kw):
    spec, m, data, masses, momenta = setup
    n_beads = kw["ring_polymer"].n_beads if "ring_polymer" in kw else 1
    return M.DeviceMD(m, batch_to_device(data, DEV), masses, time_step=0.5 * M.FS_MD, cutoff=spec["cutoff"],
                      capacity=int(data[S.Z].shape[0]) * 160 * n_beads, momenta=momenta, required_properties=props,
                      record_capacity=capacity, record_velocities=capacity > 0, stream=stream, **kw)


def _specs(data, res):
    return [SP.PowerSpectrum(data, resolution=res), SP.IRSpectrum(data, resolution=res),
            SP.RamanSpectrum(data, 19455.25, 300.0, resolution=res),
            SP.RamanSpectrum(data, 19455.25, 300.0, resolution=res, averaged=True)]


def _compare(got_data, ref_data, res, mols=(0, 2, None)):
    for got, ref in zip(_specs(got_data, res), _specs(ref_data, res)):
        for m in mols:
            got.compute_spectrum(m)
            ref.compute_spectrum(m)
            what = (type(got).__name__, getattr(got, "averaged", False), res, m)
            assert SO.rel_err(got.autocorrelation.cpu().numpy(), ref.autocorrelation.cpu().numpy()) <= TOL, what
            assert len(got.intensities) == len(ref.intensities)
            for a, b in zip(got.intensities, ref.intensities):
                assert a.shape == b.shape and a.dtype == torch.float64, what
                err = SO.rel_err(a.cpu().numpy(), b.cpu().numpy())
                assert err <= TOL, (what, err)
            assert torch.equal(got.frequencies[0], ref.frequencies[0])


def _same_state(a, b):
    sa, sb = a._state(), b._state()
    return sa.keys() == sb.keys() and all(torch.equal(sa[k], sb[k]) for k in sa)


# stream lag windows against run lengths: L above n (the stream holds the whole series), L = 1100 over 1300 samples (the
# ring wraps, the head stops filling, two lag tiles of 1024 meet data) and L = 64 over 301 samples (a one-warp tile; the
# ring wraps several times); each with the spectrum resolutions compared
WINDOWS = [(301, 4096, (4096, 100)), (1300, 1100, (1100, 1030)), (301, 64, (64, 20))]


@pytest.mark.parametrize("window", WINDOWS, ids=["L4096-n301", "L1100-n1300", "L64-n301"])
@pytest.mark.parametrize("ensemble", ["nve", "nvt", "rpmd"])
def test_stream_equals_stored_series(setup, ensemble, window):
    steps, L, resolutions = window
    kw = {}
    if ensemble == "nvt":
        kw["thermostat"] = M.LangevinThermostat(300.0, 50.0, seed=1)
    if ensemble == "rpmd":
        kw["ring_polymer"] = M.RingPolymer(4, 300.0)
    stream = SP.SpectrumStream(KINDS, resolution=L)
    md = _md(setup, stream, capacity=steps, **kw)
    md.run(steps)
    assert stream.frames == steps and stream.n_replicas == (4 if ensemble == "rpmd" else 1)
    for res in resolutions:
        _compare(stream, md, res)
    if ensemble == "nve":
        _check_accumulators(stream, md)


def _check_accumulators(stream, md):
    """the device state of every group (S, head, ring, Y, shift) against the numpy stream fed the recorded frames"""
    s = md.series()
    for src, g in stream._groups.items():
        F, L = int(g["index"].shape[0]), stream.resolution
        R = L + SS.BLOCK
        st = g["state"].cpu().numpy()
        dev = dict(S=st[:F * L].reshape(F, L), head=st[F * L:2 * F * L].reshape(F, L),
                   ring=st[2 * F * L:F * (2 * L + R)].reshape(F, R), scal=st[F * (2 * L + R):F * (2 * L + R + 8)])
        rec = (s.velocities if src == "velocities" else s.properties[src]).cpu().numpy()
        x = SS.fields_of(rec, g["index"].cpu().tolist(), g["coef"].cpu().tolist(), g["derivative"], s.dt_fs)
        ref = SS.Stream(F, L)
        ref.extend(x)
        assert ref.n == x.shape[0]
        scal = dev["scal"].reshape(F, 8)
        pairs = (("S", dev["S"], ref.S), ("head", dev["head"], ref.head), ("ring", dev["ring"], ref.ring),
                 ("Y", scal[:, 0], ref.Y), ("shift", scal[:, 1], ref.shift))
        for name, got, want in pairs:
            scale = np.maximum(np.abs(want).max(axis=-1, keepdims=True), 1e-300)
            err = float((np.abs(got - want) / scale).max())
            assert err <= 1e-12, (src, name, err)


# (stream lags, steps of each run() call): the restart point and the split points fall inside blocks
SPLITS = [(64, (37, 150, 213)), (1100, (37, 700, 563))]


@pytest.mark.parametrize("split", SPLITS, ids=["L64", "L1100"])
def test_split_restart_and_no_recorder_are_bitwise(setup, split):
    L, parts = split
    total = sum(parts)
    whole = SP.SpectrumStream(KINDS, resolution=L)
    md = _md(setup, whole)                                      # record_capacity = 0
    md.run(total)
    assert total > L + 2 * SS.BLOCK
    split_stream = SP.SpectrumStream(KINDS, resolution=L)
    md2 = _md(setup, split_stream, capacity=total)
    md2.run(parts[0])
    sd = md2.state_dict()
    for n in parts[1:]:
        md2.run(n)
    assert _same_state(whole, split_stream)
    resumed = SP.SpectrumStream(KINDS, resolution=L)
    md3 = _md(setup, resumed, capacity=total)
    md3.load_state_dict(sd)
    md3.run(total - parts[0])
    assert _same_state(whole, resumed)
    for a, b in zip(_specs(whole, L), _specs(resumed, L)):
        a.compute_spectrum(None)
        b.compute_spectrum(None)
        assert all(torch.equal(torch.nan_to_num(x), torch.nan_to_num(y)) for x, y in zip(a.intensities, b.intensities))
    _compare(split_stream, md2, L, mols=(None,))               # and the no-recorder run matches the records


# (stream lags, record capacity, steps between drains) at record_every = 2
DRAINS = [(64, 150, (300, 150, 90)), (1100, 500, (1000, 900, 500)), (4096, 80, (130, 150, 40))]


@pytest.mark.parametrize("drain", DRAINS, ids=["L64", "L1100", "L4096"])
def test_drain_leaves_the_stream(setup, drain):
    L, capacity, parts = drain
    stream = SP.SpectrumStream(KINDS, resolution=L)
    md = _md(setup, stream, capacity=capacity, record_every=2)
    drained = []
    for n in parts:
        md.run(n)
        drained.append(md.drain())
    frames = sum(parts) // 2
    assert stream.frames == frames and stream.dt_fs == pytest.approx(1.0)
    rec = {k: torch.cat([p[k] for p in drained]) for k in drained[0]}
    vel = rec.pop("velocities")
    assert vel.shape[0] == frames
    base = md.systems
    joined = SP.RecordedSeries(stream.dt_fs, base.sys_ptr, 1, velocities=vel, properties=rec, device=DEV)
    _compare(stream, joined, L)


def test_refusals(setup):
    with pytest.raises(ValueError, match="kinds"):
        SP.SpectrumStream(["bogus"])
    with pytest.raises(ValueError, match="resolution must be positive"):
        SP.SpectrumStream("ir", resolution=0)
    with pytest.raises(ValueError, match="not attached"):
        SP.IRSpectrum(SP.SpectrumStream("ir"))
    with pytest.raises(ValueError, match="not in required_properties"):
        _md(setup, SP.SpectrumStream(["raman"]), props=["dipole_moment"])
    with pytest.raises(TypeError, match="SpectrumStream"):
        _md(setup, object())
    stream = SP.SpectrumStream(["ir"], resolution=64)
    md = _md(setup, stream)
    with pytest.raises(ValueError, match="already belongs"):
        _md(setup, stream)
    md.run(4)
    with pytest.raises(ValueError, match="above the stream's"):
        SP.IRSpectrum(stream, resolution=65)
    with pytest.raises(ValueError, match="fewer than the 3"):
        SP.IRSpectrum(stream, resolution=64).compute_spectrum(0)
    md.run(10)
    with pytest.raises(KeyError, match="not streamed"):
        SP.PowerSpectrum(stream, resolution=64).compute_spectrum(0)
    with pytest.raises(KeyError, match="not streamed"):
        SP.RamanSpectrum(stream, 19455.25, 300.0, resolution=64).compute_spectrum(0)
    with pytest.raises(KeyError, match="not streamed"):
        SP.IRSpectrum(stream, resolution=64, dipole_moment_handle="other").compute_spectrum(0)
    with pytest.raises(IndexError, match="out of range"):
        SP.IRSpectrum(stream, resolution=64).compute_spectrum(3)
    spec = SP.IRSpectrum(stream, resolution=64)
    spec.compute_spectrum(1)
    assert spec.intensities[0].shape == (4 * 11,)              # n = 12 points, L = 11 lags
