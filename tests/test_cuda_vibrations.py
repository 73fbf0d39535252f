"""GPU checks of the device vibrational analysis (schnetpack_b200.vibrations, csrc/vibrations.cu): Hessians against the
reference's analytic Hessians and the fp64 finite differences of the fixtures (tests/golden/make_golden_vibrations.py),
dipole / polarizability derivatives against the heads, frequencies and intensities against tests/vib_oracle.py, the
bitwise invariants of the chunked captured step, relaxation followed by vibration, and the refusals."""
import numpy as np
import pytest
import torch

import vib_oracle as V
from conftest import load_case
from schnetpack_b200 import properties as P
from schnetpack_b200.model import NeuralNetworkPotential, batch_to_device, from_spec
from schnetpack_b200.relax import DeviceLBFGS
from schnetpack_b200.vibrations import DeviceVibrations
from test_cuda_heads import _head
from test_vib_oracle import GOLDEN

import heads_oracle as HO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
H = 0.01


def _fixture(name):
    z = np.load(f"{GOLDEN}/{name}.npz")
    import json

    spec = json.loads(str(z["spec_json"]))
    inputs = {k[3:]: z[k] for k in z.files if k.startswith("in:")}
    params = {k[6:]: z[k] for k in z.files if k.startswith("param:")}
    return z, spec, params, inputs


def _heads_model(spec, params, heads):
    base = from_spec(spec, params)
    hs = [_head(h, spec["n_atom_basis"]) for h in heads]
    full = NeuralNetworkPotential(base.representation, list(base.input_modules), list(base.output_modules) + hs,
                                  postprocessors=[], do_postprocessing=False)
    sd = full.state_dict()
    full.load_state_dict({k: torch.as_tensor(np.asarray(params[k])).to(sd[k].dtype) for k in sd})
    return full.to(DEV).eval()


def _ethanol():
    z, _, _, inputs = _fixture("vib_ethanol")
    spec, params, _, _, _ = load_case("painn_md_ethanol_trained")
    return z, spec, from_spec(spec, params, DEV), inputs


def _vib(model, inputs, spec, masses, **kw):
    n = inputs[P.Z].shape[0]
    cap = max(n * n, 2 * inputs[P.idx_i].shape[0])
    return DeviceVibrations(model, batch_to_device(inputs, DEV), torch.as_tensor(masses), cutoff=spec["cutoff"],
                            capacity=cap, **kw)


def _max_rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / np.abs(b).max())


# Hessian parity.  The kernel Hessian differs from the fp64 finite differences of the fixture at the same h and realised
# steps only by the fp32 force noise of the model, divided by the step: err <= eps_F * (sum_s |w_s|) with sum |w| = 1 / h
# (nfree 2) and 1.5 / h (nfree 4).  Measured on an H100 (700 W) for nfree 2 / 4: ethanol 3.8e-6 / 5.5e-6, heads
# 3.7e-6 / 5.0e-6, box 9.3e-6 / 1.3e-5; the bounds keep a margin of about 4x.
NOISE_BOUND = {"vib_ethanol": 2.5e-5, "vib_heads": 2.5e-5, "vib_box": 5e-5}
TRUNC_BOUND = {"vib_ethanol": 3e-3, "vib_heads": 1.5e-2, "vib_box": 2.5e-3}     # as tests/test_vib_oracle.py


def _hessian_case(name, nfree):
    z, spec, params, inputs = _fixture(name)
    if name == "vib_ethanol":
        z, spec, model, inputs = _ethanol()
    elif name == "vib_heads":
        model = _heads_model(spec, params, [HO.dip(), HO.pol()])
    else:
        model = from_spec(spec, params, DEV)
    v = _vib(model, inputs, spec, z["masses"], delta=H, nfree=nfree)
    v.run()
    return z, v


@pytest.mark.parametrize("nfree", [2, 4])
@pytest.mark.parametrize("name", ["vib_ethanol", "vib_heads", "vib_box"])
def test_hessian_matches_finite_differences_and_reference(name, nfree):
    z, v = _hessian_case(name, nfree)
    got = v.hessian.cpu().numpy()
    noise = _max_rel(got, z[f"fd{nfree}:hessian"])
    trunc = _max_rel(got, z["ref64:hessian"])
    print(f"{name} nfree={nfree}: |H - H_fd| / max|H_fd| = {noise:.3e}, |H - H_ref| / max|H_ref| = {trunc:.3e}, "
          f"chunks {v.n_chunks}")
    assert noise <= NOISE_BOUND[name]
    assert trunc <= TRUNC_BOUND[name]
    assert torch.equal(v.hessian, v.hessian.transpose(1, 2)[_swap_index(v)])


def _swap_index(v):
    """row i n + j of every system -> row j n + i (the symmetrised Hessian is exactly symmetric)"""
    idx, off = [], 0
    for n in v.sizes:
        k = torch.arange(n * n)
        idx.append(off + (k % n) * n + k // n)
        off += n * n
    return torch.cat(idx).to(DEV)


def test_ethanol_frequencies():
    """frequencies of the relaxed trained ethanol model (kcal/mol, Angstrom) against the oracle's frequencies of the
    fixture's fp64 finite-difference Hessian at the same h (the difference is force noise) and of the reference's
    analytic Hessian (the difference adds the truncation error)"""
    from schnetpack_b200.units import convert_units

    z, spec, model, inputs = _ethanol()
    conv = convert_units("kcal/mol", "eV")
    v = _vib(model, inputs, spec, z["masses"], delta=H, energy_conversion=conv)
    v.run()
    freq = v.frequencies().cpu().numpy()
    ptr = np.array([0, 9, 18])
    fd = V.frequencies(V.finish([_block(z["fd2:hessian"], ptr, m) for m in range(2)], z["masses"], ptr, conv)[1])
    ref = V.frequencies(V.finish([_block(z["ref64:hessian"], ptr, m) for m in range(2)], z["masses"], ptr, conv)[1])
    for m in range(2):
        f, o, r = (x[27 * m:27 * (m + 1)] for x in (freq, fd, ref))
        print(f"ethanol {m}: rigid-body modes {np.round(f[:6], 2)}; largest |nu - nu_fd| above them "
              f"{np.abs(f[6:] - o[6:]).max():.4f} cm^-1, |nu - nu_analytic| {np.abs(f[6:] - r[6:]).max():.3f} cm^-1")
        assert np.all(np.diff(f) >= 0)
        assert np.abs(f[:6]).max() <= 40.0, f[:6]                   # rigid-body modes of a relaxed molecule
        assert np.all(f[6:] > 100.0), f[6:]
        assert np.abs(f[6:] - o[6:]).max() <= 0.05              # measured 0.0044 cm^-1 on an H100
        assert np.abs(f[6:] - r[6:]).max() <= 5.0               # measured 4.42 cm^-1: the O(h^2) truncation


def _block(hb, ptr, m):
    n = ptr[m + 1] - ptr[m]
    off = int(sum((ptr[k + 1] - ptr[k]) ** 2 for k in range(m)))
    return hb[off:off + n * n].reshape(n, n, 3, 3).transpose(0, 2, 1, 3).reshape(3 * n, 3 * n)


def test_head_derivatives_and_intensities():
    z, spec, params, inputs = _fixture("vib_heads")
    model = _heads_model(spec, params, [HO.dip(), HO.pol()])
    v = _vib(model, inputs, spec, z["masses"], delta=H, nfree=4, properties=(P.dipole_moment, P.polarizability))
    v.run()
    dd, pd = v.dipole_derivatives.cpu().numpy(), v.polarizability_derivatives.cpu().numpy()
    for key, got in (("dipole_derivatives", dd), ("polarizability_derivatives", pd)):
        noise = _max_rel(got, z["fd4:" + key])
        trunc = _max_rel(got, z["ref64:" + key])
        print(f"{key}: vs fd {noise:.3e}, vs analytic {trunc:.3e}")
        assert noise <= 2e-4 and trunc <= 1e-3
    # the existing head fixture: d(dipole)/dR of heads_painn_centered, as [comp, N, 3].  Its jittered aspirins have pairs
    # near the 5 A cutoff, unlike the molecules above; measured on an H100: 1.1e-2 for the dipole (nfree 4, h = 0.01)
    spec_c, params_c, inputs_c, _, ref_c = load_case("heads_painn_centered")
    heads_c = HO.CASES["heads_painn_centered"]["heads"]
    mc = _heads_model(spec_c, params_c, heads_c)
    vc = _vib(mc, inputs_c, spec_c, np.ones(inputs_c[P.Z].shape[0]), delta=H, nfree=4,
              properties=(P.dipole_moment, P.polarizability))
    vc.run()
    N = inputs_c[P.Z].shape[0]
    err_d = _max_rel(vc.dipole_derivatives.cpu().numpy(), ref_c["d:dipole_moment"].transpose(1, 0, 2))
    err_p = _max_rel(vc.polarizability_derivatives.cpu().numpy(),
                     ref_c["d:polarizability"].reshape(3, 3, N, 3).transpose(2, 0, 1, 3))
    print(f"heads_painn_centered: dipole derivatives {err_d:.3e}, polarizability derivatives {err_p:.3e}")
    assert err_d <= 3e-2 and err_p <= 3e-2
    # intensities: the oracle's post-processing of the same Hessian and derivatives
    ptr = np.concatenate([[0], np.cumsum(inputs[P.n_atoms])])
    mw = [_block(v.hessian.cpu().numpy(), ptr, m) / np.sqrt(np.outer(*(2 * [np.repeat(z["masses"][ptr[m]:ptr[m + 1]], 3)])))
          for m in range(len(ptr) - 1)]
    np.testing.assert_allclose(v.frequencies().cpu().numpy(), V.frequencies(mw), rtol=1e-9, atol=1e-6)
    ir, ra = v.ir_intensities().cpu().numpy(), v.raman_activities().cpu().numpy()
    ir_o, ra_o = V.ir_intensities(mw, z["masses"], ptr, dd), V.raman_activities(mw, z["masses"], ptr, pd)
    # modes of (near-)degenerate eigenvalues are any basis of their space: compare the sums over such groups
    for got, ref in ((ir, ir_o), (ra, ra_o)):
        assert abs(got.sum() - ref.sum()) <= 1e-9 * abs(ref).sum()
        freq = V.frequencies(mw)
        clear = np.ones(len(freq), dtype=bool)
        clear[1:] &= np.abs(np.diff(freq)) > 1.0
        clear[:-1] &= np.abs(np.diff(freq)) > 1.0
        np.testing.assert_allclose(got[clear], ref[clear], rtol=1e-6, atol=1e-9 * abs(ref).max())


def test_graph_eager_repeat_and_chunking_are_bitwise():
    """use_graph equals eager, a second run equals the first, and a run forced into several chunks with idle copies on a
    ragged batch with a 1-atom system equals a one-chunk run"""
    z, spec, params, inputs = _fixture("vib_heads")
    model = _heads_model(spec, params, [HO.dip(), HO.pol()])
    kw = dict(delta=H, properties=(P.dipole_moment, P.polarizability))
    one = _vib(model, inputs, spec, z["masses"], **kw)
    assert one.n_chunks == 1
    one.run()
    first = [t.clone() for t in (one.hessian, one.dipole_derivatives, one.polarizability_derivatives)]
    one.run()
    again = (one.hessian, one.dipole_derivatives, one.polarizability_derivatives)
    assert all(torch.equal(a, b) for a, b in zip(first, again))
    eager = _vib(model, inputs, spec, z["masses"], use_graph=False, **kw)
    eager.run()
    assert all(torch.equal(a, b) for a, b in zip(first, (eager.hessian, eager.dipole_derivatives,
                                                         eager.polarizability_derivatives)))
    n = inputs[P.Z].shape[0]
    chunked = _vib(model, inputs, spec, z["masses"], max_replica_atoms=7 * 2 * n, **kw)
    assert chunked.n_cols == 7 and chunked.n_chunks == 5           # 30 coordinates: the last chunk has idle copies
    chunked.run()
    # the model's forces here do not depend on the batch layout, so five chunks give the one-chunk result bitwise
    assert all(torch.equal(a, b) for a, b in zip(first, (chunked.hessian, chunked.dipole_derivatives,
                                                         chunked.polarizability_derivatives)))


def test_relax_then_vibrate():
    z, spec, model, inputs = _ethanol()
    rng = np.random.default_rng(2)
    start = dict(inputs)
    start[P.R] = (inputs[P.R] + rng.normal(scale=0.05, size=inputs[P.R].shape)).astype(np.float32)
    relax = DeviceLBFGS(model, batch_to_device(start, DEV), cutoff=spec["cutoff"], capacity=18 * 18)
    assert relax.run(fmax=1e-3, steps=2000)
    from schnetpack_b200.units import convert_units

    batch = dict(batch_to_device(start, DEV), _positions=relax.model_positions.clone())
    v = DeviceVibrations(model, batch, torch.as_tensor(z["masses"]), cutoff=spec["cutoff"], capacity=18 * 18,
                         energy_conversion=convert_units("kcal/mol", "eV"))
    v.run()
    freq = v.frequencies().cpu().numpy()
    for m in range(2):
        f = freq[27 * m:27 * (m + 1)]
        order = np.argsort(np.abs(f))
        assert np.abs(f[order[:6]]).max() <= 40.0, f
        assert np.all(f[order[6:]] > 100.0), f


def test_refusals():
    z, spec, model, inputs = _ethanol()
    cpu = {k: torch.as_tensor(v) for k, v in inputs.items()}
    masses = z["masses"]
    with pytest.raises(ValueError, match="CUDA"):
        DeviceVibrations(model, cpu, torch.as_tensor(masses), cutoff=5.0, capacity=400)
    with pytest.raises(ValueError, match="nfree"):
        _vib(model, inputs, spec, masses, nfree=3)
    with pytest.raises(ValueError, match="delta"):
        _vib(model, inputs, spec, masses, delta=0.0)
    with pytest.raises(ValueError, match="masses"):
        _vib(model, inputs, spec, masses[:-1])
    with pytest.raises(ValueError, match="dipole_moment"):
        _vib(model, inputs, spec, masses, properties=(P.dipole_moment,))
    with pytest.raises(NotImplementedError, match="ensemble"):
        _vib([model, model], inputs, spec, masses)
    spec_i, params_i, inputs_i, _, _ = load_case("heads_painn_isolated")
    mi = _heads_model(spec_i, params_i, HO.CASES["heads_painn_isolated"]["heads"])
    with pytest.raises(ValueError, match="scalar dipole"):
        _vib(mi, inputs_i, spec_i, np.ones(inputs_i[P.Z].shape[0]), properties=(P.dipole_moment,))
    from schnetpack_b200.parallel import PartitionedPotential

    pp = PartitionedPotential.__new__(PartitionedPotential)
    with pytest.raises(NotImplementedError, match="PartitionedPotential"):
        _vib(pp, inputs, spec, masses)
