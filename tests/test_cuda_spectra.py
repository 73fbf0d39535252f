"""GPU checks of the vibrational spectra (csrc/spectra.cu, schnetpack_b200/spectra.py) and of the velocity recorder of
DeviceMD: the kernels against the reference's fixtures, determinism, batched == per-index, every refusal, and
end-to-end spectra of headed PaiNN runs (plain and ring-polymer) against the fp64 oracle on the host copies."""
import numpy as np
import pytest
import torch

import spectra_oracle as SO
from schnetpack_b200 import atomistic as A
from schnetpack_b200 import md as M
from schnetpack_b200 import synthetic as S
from schnetpack_b200 import spectra as SP
from schnetpack_b200.model import NeuralNetworkPotential, batch_to_device, from_spec

import heads_oracle as HO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KEYS = ["dipole_moment", "polarizability"]
TOL = 1e-10


def _series(z, device=DEV):
    recs = {k[4:]: torch.as_tensor(z[k]) for k in z.files if k.startswith("rec:")}
    vel = recs.pop("velocities", None)
    return SP.RecordedSeries(float(z["dt_fs"]), z["sys_ptr"], int(z["n_replicas"]), velocities=vel, properties=recs,
                             device=device)


def _spectrum(data, run):
    kind, res = run["kind"], run["resolution"]
    if kind == "power":
        return SP.PowerSpectrum(data, resolution=res)
    if kind == "ir":
        return SP.IRSpectrum(data, resolution=res)
    return SP.RamanSpectrum(data, 19455.25, 300.0, resolution=res, averaged=run["averaged"])


def _oracle(rec, sys_ptr, n_rep, dt, run, m):
    return SO.spectrum(run["kind"], rec, sys_ptr, n_rep, dt, m, resolution=run["resolution"],
                       averaged=run.get("averaged", False), incident_frequency=19455.25, temperature=300.0,
                       hbar2icm=SP.HBAR2ICM, kB=M.KB_MD)


@pytest.mark.parametrize("name", SO.GOLDEN)
def test_kernels_match_reference_fixtures(name):
    z, cases = SO.golden(name)
    data = _series(z)
    for r, run, m in cases:
        spec = _spectrum(data, run)
        spec.compute_spectrum(m)
        out = spec.get_spectrum()
        out = out if isinstance(out, list) else [out]
        key = f"r{r}:m{m}"
        _, _, _, chans = _oracle(z["rec:" + SO.PROP[run["kind"]]], list(z["sys_ptr"]), int(z["n_replicas"]),
                                 float(z["dt_fs"]), run, m)
        assert SO.rel_err(spec.autocorrelation[0].cpu().numpy(), chans) <= TOL, key
        for j, (f, v) in enumerate(out):
            assert f.dtype == torch.float64 and v.dtype == torch.float64 and v.device.type == "cuda"
            assert np.array_equal(f.cpu().numpy(), z[key + ":freq"]), key
            err = SO.rel_err(v.cpu().numpy(), z[f"{key}:I{j}"])
            assert err <= TOL, (key, j, err)


@pytest.mark.parametrize("name", SO.GOLDEN)
def test_repeat_and_batched_are_bitwise(name):
    z, cases = SO.golden(name)
    data = _series(z)
    B = len(z["sys_ptr"]) - 1
    for r, run, _ in cases[::B]:
        spec = _spectrum(data, run)
        spec.compute_spectrum(None)
        batched = [v.clone() for v in spec.intensities]
        spec.compute_spectrum(None)
        assert all(_same(a, b) for a, b in zip(batched, spec.intensities)), r
        for m in range(B):
            spec.compute_spectrum(m)
            for j, v in enumerate(spec.intensities):
                assert _same(batched[j][m], v), (r, m, j)


def _same(a, b):
    """bitwise equal, NaN positions included"""
    return torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(torch.nan_to_num(a), torch.nan_to_num(b))


def test_refusals():
    z, _ = SO.golden("spectra_ir")
    data = _series(z)
    with pytest.raises(KeyError, match="velocities are not recorded"):
        SP.PowerSpectrum(data).compute_spectrum(0)
    with pytest.raises(KeyError, match="not recorded"):
        SP.RamanSpectrum(data, 19455.25, 300.0).compute_spectrum(0)
    with pytest.raises(IndexError, match="out of range"):
        SP.IRSpectrum(data).compute_spectrum(2)
    with pytest.raises(TypeError, match="molecule_idx"):
        SP.IRSpectrum(data).compute_spectrum(0.5)
    with pytest.raises(ValueError, match="temperature"):
        SP.RamanSpectrum(data, 19455.25, 0.0)
    with pytest.raises(ValueError, match="resolution"):
        SP.IRSpectrum(data, resolution=0)
    with pytest.raises(TypeError, match="DeviceMD or a RecordedSeries"):
        SP.IRSpectrum(z)
    short = SP.RecordedSeries(0.5, [0, 1], 1, properties={"dipole_moment": torch.ones(4, 1, 1, 3, device=DEV)})
    with pytest.raises(ValueError, match="fewer than the 3"):
        SP.IRSpectrum(short).compute_spectrum(0)
    short = SP.RecordedSeries(0.5, [0, 1], 1, velocities=torch.ones(2, 1, 1, 3, device=DEV))
    with pytest.raises(ValueError, match="fewer than the 3"):
        SP.PowerSpectrum(short).compute_spectrum(0)
    with pytest.raises(ValueError, match="velocities must be"):
        SP.RecordedSeries(0.5, [0, 2], 1, velocities=torch.ones(5, 1, 1, 3, device=DEV))
    bad = SP.RecordedSeries(0.5, [0, 1], 1, properties={"dipole_moment": torch.ones(9, 1, 1, 4, device=DEV)})
    with pytest.raises(ValueError, match="records must be"):
        SP.IRSpectrum(bad).compute_spectrum(0)


# ---- the velocity recorder and end-to-end spectra ---------------------------------------------------------------------
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
    momenta = torch.as_tensor(rng.normal(size=(masses.shape[0], 3)) * np.sqrt(masses.numpy() * M.KB_MD * 300.0)[:, None],
                              dtype=torch.float32)
    return spec, model, data, masses, momenta


def _md(setup, props=KEYS, capacity=16, use_graph=True, **kw):
    spec, m, data, masses, momenta = setup
    return M.DeviceMD(m, batch_to_device(data, DEV), masses, time_step=0.5 * M.FS_MD, cutoff=spec["cutoff"],
                      capacity=int(data[S.Z].shape[0]) * 160 * (kw["ring_polymer"].n_beads if "ring_polymer" in kw
                                                                else 1),
                      momenta=momenta, use_graph=use_graph, required_properties=props, record_capacity=capacity, **kw)


def test_recorder_refusals(setup):
    with pytest.raises(ValueError, match="share it"):
        _md(setup, props=KEYS + ["velocities"], record_velocities=True)
    with pytest.raises(ValueError, match="record_capacity > 0"):
        _md(setup, capacity=0, record_velocities=True)
    md = _md(setup, props=None, capacity=4, record_velocities=True)         # velocities alone are enough
    md.run(4)
    assert md.recorded("velocities").shape == (4, 1, 63, 3)
    with pytest.raises(RuntimeError, match="record_capacity"):
        md.run(1)


def test_velocities_equal_momenta_over_masses(setup):
    md = _md(setup, capacity=6, use_graph=False, record_velocities=True, record_every=2)
    expect = []
    for s in range(12):
        md.run(1)
        if (s + 1) % 2 == 0:
            expect.append((md.momenta / md.masses[:, None]).cpu())
    rec = md.recorded("velocities")
    assert rec.shape == (6, 1, 63, 3)
    for s, v in enumerate(expect):
        assert torch.equal(rec[s, 0], v), s
    graph = _md(setup, capacity=6, record_velocities=True, record_every=2)
    graph.run(12)
    assert torch.equal(graph.recorded("velocities"), rec)
    assert torch.equal(graph.recorded("dipole_moment"), md.recorded("dipole_moment"))
    out = graph.drain()
    assert torch.equal(out["velocities"], rec) and graph.recorded("velocities").shape[0] == 0
    assert graph.series().velocities.shape == (0, 1, 63, 3)


def test_rpmd_layout_and_restart(setup):
    rp = M.RingPolymer(4, 300.0)
    md = _md(setup, capacity=10, record_velocities=True, ring_polymer=rp)
    md.run(3)
    sd = md.state_dict()
    md.run(5)
    ref = md.recorded("velocities")
    assert ref.shape == (8, 4, 63, 3)
    v = (md.momenta / md.masses[:, None]).reshape(4, 63, 3).cpu()
    assert torch.equal(ref[-1], v)
    md2 = _md(setup, capacity=10, record_velocities=True, ring_polymer=M.RingPolymer(4, 300.0))
    md2.load_state_dict(sd)
    md2.run(5)
    assert torch.equal(md2.recorded("velocities"), ref)
    assert torch.equal(md2.recorded("polarizability"), md.recorded("polarizability"))
    s = md.series()
    assert s.n_replicas == 4 and s.sys_ptr == [0, 21, 42, 63] and s.velocities.shape == (8, 4, 63, 3)
    assert s.velocities.data_ptr() == md._records["velocities"].data_ptr()             # a view, no copy
    assert s.dt_fs == pytest.approx(0.5)


@pytest.mark.parametrize("n_beads", [1, 4])
def test_end_to_end_spectra_equal_oracle(setup, n_beads):
    kw = dict(ring_polymer=M.RingPolymer(n_beads, 300.0)) if n_beads > 1 else {}
    steps = 300
    md = _md(setup, capacity=steps, record_velocities=True, **kw)
    md.run(steps)
    host = {k: md.recorded(k).numpy() for k in KEYS + ["velocities"]}
    s = md.series()
    runs = [dict(kind="power", resolution=4096), dict(kind="power", resolution=128), dict(kind="ir", resolution=4096),
            dict(kind="raman", resolution=4096, averaged=False), dict(kind="raman", resolution=100, averaged=True)]
    for run in runs:
        spec = _spectrum(md, run)
        spec.compute_spectrum(None)
        for m in range(3):
            freq, ints, _, _ = _oracle(host[SO.PROP[run["kind"]]], s.sys_ptr, n_beads, s.dt_fs, run, m)
            for j, v in enumerate(ints):
                got = spec.intensities[j][m].cpu().numpy()
                err = SO.rel_err(got, v)
                assert err <= TOL, (run, m, j, err)
            assert np.array_equal(spec.frequencies[0].cpu().numpy(), freq)
