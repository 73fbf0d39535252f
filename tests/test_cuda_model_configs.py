"""PaiNN and SchNet end to end against the fp64 oracle at every supported shape and kernel path.

The configurations below are chosen by the branch of the Python glue (functional.py) or of the kernel dispatch each one
reaches: the streaming edge kernels at every warp count (F = 32 ... 256) and both radial-basis templates (NRB = 20, 32),
the tensor-core PaiNN edge kernels up to their n_rbf limit and their refusal past it, the fused SchNet forward against
the materialised-filter path, n_filters != n_atom_basis, dense shapes the tensor-core kernel hands to the fp32 kernel,
shared filters / shared interactions, and one and four interaction blocks.

Every configuration runs on two legs, with a recorder on the C ABI proving which entry points each leg reached:
  tc         the shipped kernel switches, with the edge-count thresholds of the tensor-core paths at 0 so that these
             small batches take the path large batches take;
  cuda-core  the streaming edge kernels, the materialised SchNet filter and the fp32 dense kernel.

Errors are measured per system: for each output, max |x - x64| over the system's rows divided by max |x64| over the same
rows.  The bound for system m is max(1e-5, C * e32(m)), with e32(m) the same error of the fp32 oracle on the CPU, i.e.
the reference's own arithmetic, so an error confined to one small system cannot hide under the batch's largest force.

The CPU part pins the fp64 oracle itself to the reference modules at the same configurations, and the refusal tests
check that shapes without a kernel are refused before the first launch.
"""
import json

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import ref_loader as rl
from oracle import spk_oracle as O
from schnetpack_b200 import synthetic as S

needs_ref = pytest.mark.skipif(not rl.available(), reason="reference modules absent (neither /root/reference nor oracle/_ref)")
DEV = "cuda:0"
C = 4.0          # allowed ratio of a kernel's per-system error to the fp32 reference arithmetic's
FLOOR = 1e-5     # bound below which fp32 rounding of the inputs alone can reach
CUTOFF = 5.0

# id -> (model_spec arguments, expectations): edge_tc = the PaiNN edge kernels run on the tensor cores on the tc leg;
# fused = the energy-only SchNet forward runs the fused kernel on the tc leg; dense_fallback = some dense layer has a
# shape the tensor-core kernel does not take (K or N not a multiple of 4), so the fp32 kernel runs it on the tc leg too
CONFIGS = {
    "P1": (dict(kind="painn", n_atom_basis=32, n_rbf=20), {}),                                 # NW = 1, NRB = 20
    "P2": (dict(kind="painn", n_atom_basis=64, n_rbf=21), {}),                                 # first NRB = 32 case
    "P3": (dict(kind="painn", n_atom_basis=128, n_rbf=23, rbf="bessel"), dict(edge_tc=True)),  # TC limit: K = 24
    "P4": (dict(kind="painn", n_atom_basis=128, n_rbf=32), {}),                                # TC refuses: streaming
    "P9": (dict(kind="painn", n_atom_basis=128, n_rbf=24, n_interactions=2), {}),              # first n_rbf TC refuses
    "P5": (dict(kind="painn", n_atom_basis=256, n_rbf=20, n_interactions=4), {}),              # NW = 8, dense N = 768
    "P6": (dict(kind="painn", n_atom_basis=128, n_rbf=20, shared_filters=True, n_interactions=2),
           dict(edge_tc=True)),                                                                # one filter pack for all t
    "P7": (dict(kind="painn", n_atom_basis=128, n_rbf=13, n_interactions=1), dict(edge_tc=True)),   # mu = None only
    "P8": (dict(kind="painn", n_atom_basis=64, n_rbf=32, rbf="bessel", shared_interactions=True, shared_filters=True),
           {}),                                                                                # shared blocks, NRB = 32
    "S1": (dict(kind="schnet", n_atom_basis=128, n_rbf=20), dict(fused=True)),
    "S2": (dict(kind="schnet", n_atom_basis=128, n_rbf=31, rbf="bessel"), dict(fused=True, dense_fallback=True)),
    "S3": (dict(kind="schnet", n_atom_basis=128, n_rbf=32), {}),                               # fused refused
    "S4": (dict(kind="schnet", n_atom_basis=100, n_filters=128, n_rbf=20), dict(dense_fallback=True)),  # head hidden 50
    "S5": (dict(kind="schnet", n_atom_basis=128, n_filters=64, n_rbf=20), {}),
    "S6": (dict(kind="schnet", n_atom_basis=256, n_rbf=20, n_interactions=4), {}),             # k_cfconv_*<8>
    "S7": (dict(kind="schnet", n_atom_basis=32, n_rbf=13, shared_interactions=True), dict(dense_fallback=True)),
}
INPUTS = ("aspirin", "qm9_padded", "box", "ragged")
LEGS = ("tc", "cuda-core")


def _model(cid):
    kw, _ = CONFIGS[cid]
    spec = S.model_spec(**kw)
    return spec, S.init_params(spec, seed=100 + list(CONFIGS).index(cid))


def _ragged():
    """ethanol, a lone atom and a pair too far apart to be neighbours; returns (batch, index of the first edgeless atom)"""
    a = S.ethanol_batch(1)
    n0 = a[S.Z].shape[0]
    return {
        S.Z: np.concatenate([a[S.Z], [8, 1, 1]]),
        S.R: np.concatenate([a[S.R], [[50, 0, 0], [80, 0, 0], [95, 0, 0]]]).astype(np.float32),
        S.idx_i: a[S.idx_i], S.idx_j: a[S.idx_j], S.offsets: a[S.offsets],
        S.idx_m: np.concatenate([a[S.idx_m], [1, 2, 2]]),
        S.n_atoms: np.array([n0, 1, 2]),
        S.cell: np.zeros((3, 3, 3), dtype=np.float32), S.pbc: np.zeros(9, dtype=bool),
    }, n0


def _qm9_padded():
    """padded QM9-like batch: the generator's padding slots sit at exactly the cutoff; every other one is turned into a
    self pair of its receiver at twice the cutoff, the padding of the fixed-capacity device neighbour lists"""
    d = S.qm9like_batch(3, padded=True, seed=12)
    pad = np.nonzero(np.all(d[S.Rij] == np.array([CUTOFF, 0, 0], np.float32), axis=1))[0][::2]
    d[S.idx_j][pad] = d[S.idx_i][pad]
    d[S.Rij][pad] = np.array([2 * CUTOFF, 0, 0], np.float32)
    return d


_INPUTS = {}


def _input(name):
    if name not in _INPUTS:
        _INPUTS[name] = {"aspirin": lambda: S.aspirin_batch(3, seed=11), "qm9_padded": _qm9_padded,
                         "box": lambda: S.periodic_box(300, seed=13), "ragged": lambda: _ragged()[0]}[name]()
    return _INPUTS[name]


_ORACLE = {}


def _oracle(cid, name):
    """(fp64, fp32) oracle outputs as float64 numpy arrays, once per (configuration, input)"""
    key = (cid, name)
    if key not in _ORACLE:
        spec, params = _model(cid)
        res = []
        for dt in (torch.float64, torch.float32):
            r = O.energy_forces(spec, params, _input(name), dtype=dt, stress=(name == "box"))
            res.append({k: v.double().numpy() for k, v in r.items()})
        _ORACLE[key] = tuple(res)
    return _ORACLE[key]


def _groups(data):
    """output -> system index of each leading row (energies and stresses are one row per system)"""
    m = data[S.idx_m]
    n_sys = int(m.max()) + 1
    sys_rows = np.arange(n_sys)
    return n_sys, {"energy": sys_rows, "stress": sys_rows, "forces": m, "scalar_representation": m,
                   "vector_representation": m, "dEdRij": m[data[S.idx_i]]}


def per_system_error(x, ref, rows, n_sys):
    """max |x - ref| / max |ref| over the rows of each system; 0 where both vanish, inf where only ref does"""
    d = np.abs(x - ref).reshape(len(rows), -1).max(axis=1, initial=0.0)
    a = np.abs(ref).reshape(len(rows), -1).max(axis=1, initial=0.0)
    num, den = np.zeros(n_sys), np.zeros(n_sys)
    np.maximum.at(num, rows, d)
    np.maximum.at(den, rows, a)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(num == 0.0, 0.0, num / den)


def _check(label, out, ref64, ref32, data, stats):
    n_sys, groups = _groups(data)
    for k in out:
        if k not in ref64:
            continue
        err = per_system_error(out[k], ref64[k], groups[k], n_sys)
        e32 = per_system_error(ref32[k], ref64[k], groups[k], n_sys)
        bound = np.maximum(FLOOR, C * e32)
        bad = np.nonzero(~(err <= bound))[0]
        assert bad.size == 0, (f"{label} {k}: systems {bad.tolist()} error {err[bad].tolist()} > bound "
                               f"{bound[bad].tolist()} (fp32 reference {e32[bad].tolist()})")
        stats["worst_err"] = max(stats["worst_err"], float(err.max()))
        stats["worst_of_bound"] = max(stats["worst_of_bound"], float((err / bound).max()))
        scaled = C * e32 > FLOOR                       # systems whose bound is set by e32 rather than by the floor
        if scaled.any():
            stats["worst_ratio"] = max(stats["worst_ratio"], float((err[scaled] / e32[scaled]).max()))


def _run(model, data, forces=True):
    """model on the device -> float64 numpy outputs; a batch with ``_Rij`` (padded list) gives dE/dr_ij instead of
    forces, like the reference with the list handed over directly"""
    from schnetpack_b200.model import batch_to_device

    x = batch_to_device(data, torch.device(DEV))
    if S.Rij in x:
        rij = x[S.Rij].requires_grad_(forces)
        x = model.output_modules[0](model.representation(x))
        out = {"energy": x["energy"]}
        if forces:
            (out["dEdRij"],) = torch.autograd.grad(x["energy"].sum(), rij)
    else:
        out = dict(model(x))
    out["scalar_representation"] = x["scalar_representation"]
    if "vector_representation" in x:
        out["vector_representation"] = x["vector_representation"]
    torch.cuda.synchronize()
    return {k: v.detach().double().cpu().numpy() for k, v in out.items()}


@pytest.fixture
def lib_calls(monkeypatch):
    """names of the C-ABI entry points called (calls pass through to the library)"""
    from schnetpack_b200 import _lib

    seen = []
    real = _lib.call

    def record(name, *args, **kw):
        seen.append(name)
        return real(name, *args, **kw)

    monkeypatch.setattr(_lib, "call", record)
    return seen


def _set_leg(monkeypatch, leg):
    from schnetpack_b200 import ops

    if leg == "tc":
        switches = dict(EDGE_IMPL="tc", CFCONV_IMPL="tc", DENSE_IMPL="tc", EDGE_TC_MIN_EDGES=0, CFCONV_TC_MIN_EDGES=0)
    else:
        switches = dict(EDGE_IMPL="ldg", CFCONV_IMPL="mat", DENSE_IMPL="ffma")
    for k, v in switches.items():
        monkeypatch.setattr(ops, k, v)


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("leg", LEGS)
@pytest.mark.parametrize("cid", list(CONFIGS))
def test_model_against_fp64_per_system(cid, leg, monkeypatch, lib_calls):
    """Energy, forces (dE/dr_ij on the padded list), representations and, on the box, stress through ``Strain``, per
    system within max(1e-5, 4 e32).  SchNet also runs energy-only, the evaluation the fused forward serves.  Worst
    per-system error and worst ratio to e32 measured on an H100 (SXM, 700 W) are listed with the change that added
    this test; a line per configuration and leg is printed under ``-s``."""
    from schnetpack_b200.model import from_spec

    _set_leg(monkeypatch, leg)            # before the models are built: DENSE_IMPL is read when Lin packs its weights
    spec, params = _model(cid)
    _, expect = CONFIGS[cid]
    dev = torch.device(DEV)
    model = from_spec(spec, params, dev)
    stress_model = from_spec(dict(spec, stress=True), params, dev)
    energy_model = from_spec(dict(spec, forces=False), params, dev) if spec["kind"] == "schnet" else None
    stats = dict(worst_err=0.0, worst_ratio=0.0, worst_of_bound=0.0)
    seen, seen_energy_only = set(), set()
    for name in INPUTS:
        data = _input(name)
        ref64, ref32 = _oracle(cid, name)
        lib_calls.clear()
        out = _run(stress_model if name == "box" else model, data)
        seen.update(lib_calls)
        _check(f"{cid}/{leg}/{name}", out, ref64, ref32, data, stats)
        if name == "ragged":
            assert np.all(out["forces"][_ragged()[1]:] == 0.0), "edgeless atoms must get exactly zero force"
        if energy_model is not None:
            lib_calls.clear()
            out = _run(energy_model, data, forces=False)
            seen_energy_only.update(lib_calls)
            _check(f"{cid}/{leg}/{name}/energy-only", out, ref64, ref32, data, stats)
    print("MODEL_CONFIG", json.dumps(dict(config=cid, leg=leg, **stats)))

    tc = leg == "tc"
    if tc:
        assert "spk_dense_tc" in seen
        if expect.get("dense_fallback"):
            assert "spk_dense" in seen
    else:
        assert "spk_dense" in seen and "spk_dense_tc" not in seen and "spk_tc_pack_weight" not in seen
    if spec["kind"] == "painn":
        edge_tc = tc and expect.get("edge_tc", False)
        on, off = ("spk_painn_edge_fwd_tc", "spk_painn_edge_bwd_tc"), ("spk_painn_edge_fwd", "spk_painn_edge_bwd")
        if not edge_tc:
            on, off = off, on
        assert all(n in seen for n in on) and not any(n in seen for n in off), sorted(seen)
    else:
        assert {"spk_cfconv_fwd", "spk_cfconv_bwd"} <= seen and "spk_schnet_cfconv_fwd_tc" not in seen
        on, off = "spk_schnet_cfconv_fwd_tc", "spk_cfconv_fwd"
        if not (tc and expect.get("fused", False)):
            on, off = off, on
        assert on in seen_energy_only and off not in seen_energy_only, sorted(seen_energy_only)


def _supported_model_matches_fp64():
    from schnetpack_b200.model import batch_to_device, from_spec

    spec, params = _model("P1")
    data = S.aspirin_batch(2, seed=3)
    out = from_spec(spec, params, torch.device(DEV))(batch_to_device(data, torch.device(DEV)))
    ref = O.energy_forces(spec, params, data, dtype=torch.float64)
    for k in ("energy", "forces"):
        assert rel_err(out[k].detach().cpu().numpy(), ref[k].numpy()) < 1e-5, k


@pytest.mark.gpu
@pytest.mark.parametrize("kind,kw,match", [
    ("painn", dict(n_atom_basis=48), "n_atom_basis = 48"), ("painn", dict(n_atom_basis=96), "n_atom_basis = 96"),
    ("painn", dict(n_atom_basis=512), "n_atom_basis = 512"), ("painn", dict(n_rbf=33), "n_rbf = 33"),
    ("schnet", dict(n_filters=48), "n_filters = 48"), ("schnet", dict(n_filters=96), "n_filters = 96"),
    ("schnet", dict(n_rbf=33), "n_rbf = 33")])
def test_unsupported_shapes_refused_before_any_launch(kind, kw, match, lib_calls):
    """A shape without a kernel raises NotImplementedError naming it before the representation launches anything (a
    refusal half way through would leave a CUDA-graph capture half recorded); a supported model still runs after it."""
    from schnetpack_b200.model import batch_to_device, from_spec

    spec = S.model_spec(kind, n_interactions=2, **kw)
    model = from_spec(spec, S.init_params(spec, seed=1), torch.device(DEV))
    x = model.initialize_derivatives(batch_to_device(S.aspirin_batch(2), torch.device(DEV)))
    for m in model.input_modules:
        x = m(x)
    assert x[S.Rij].requires_grad
    lib_calls.clear()
    with pytest.raises(NotImplementedError, match=match):
        model.representation(x)
    assert lib_calls == []
    _supported_model_matches_fp64()


@pytest.mark.gpu
def test_schnet_energy_only_beyond_32_radial_functions():
    """Energy-only SchNet with n_rbf = 33 has no radial reverse to run and takes the materialised-filter path."""
    from schnetpack_b200.model import batch_to_device, from_spec

    spec = S.model_spec("schnet", n_interactions=2, n_rbf=33, forces=False)
    params = S.init_params(spec, seed=2)
    data = S.aspirin_batch(2, seed=4)
    out = from_spec(spec, params, torch.device(DEV))(batch_to_device(data, torch.device(DEV)))
    ref = O.energy_forces(spec, params, data, dtype=torch.float64)
    assert rel_err(out["energy"].detach().cpu().numpy(), ref["energy"].numpy()) < 1e-5


# ------------------------------------------------------------------------------------------------------------ CPU
@needs_ref
@pytest.mark.parametrize("cid", list(CONFIGS))
def test_oracle_matches_reference_at_config(cid):
    """The fp64 oracle against the reference modules themselves at each configuration (n_filters != n_atom_basis and
    shared_filters alone included), on molecules and on the ragged batch."""
    spec, params = _model(cid)
    ref_model = rl.build_from_spec(spec, params, torch.float64)
    for data in (S.aspirin_batch(2, seed=21), _ragged()[0]):
        ref = rl.evaluate(ref_model, data, torch.float64)
        o = O.energy_forces(spec, params, data, dtype=torch.float64)
        assert rel_err(o["energy"].numpy(), ref["energy"].numpy()) < 1e-12
        for k in ("forces", "scalar_representation", "vector_representation"):
            if k in ref:
                assert rel_err(o[k].numpy(), ref[k].numpy()) < 1e-10, k


def test_per_system_error_isolates_systems():
    """The metric: one system's error is measured against that system's own scale, and a vanishing reference admits
    only an exact zero."""
    ref = np.array([[100.0], [1.0], [0.0]])
    rows = np.array([0, 1, 2])
    x = ref + np.array([[0.0], [1e-3], [0.0]])
    assert np.allclose(per_system_error(x, ref, rows, 3), [0.0, 1e-3, 0.0])
    assert per_system_error(ref + 1e-30, ref, rows, 3)[2] == np.inf
    # a batch-wide max-norm would report 1e-5 for the same error
    assert rel_err(x, ref) == pytest.approx(1e-5)
