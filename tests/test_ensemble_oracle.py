"""CPU checks of the fp64 ensemble oracle (tests/ensemble_oracle.py) against the reference's own ensemble statistics
(tests/golden/ensemble_batch.npz, written by tests/golden/make_golden_ensemble.py)."""
import os

import numpy as np
import pytest

import ensemble_oracle as EO
from conftest import GOLDEN


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "ensemble_batch.npz"))


def _close(a, b, tol=1e-12):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape
    assert np.all(np.abs(a - b) <= tol * np.maximum(np.abs(b), 1.0)), float(np.max(np.abs(a - b)))


def test_accumulate_equals_ensemble_calculator(golden):
    acc = EO.accumulate({"energy": golden["pred:energy"], "forces": golden["pred:forces"]})
    for k in ("energy", "energy_var", "forces", "forces_var"):
        _close(acc[k], golden["acc:" + k])


def test_nn_ensemble_equals_reference(golden):
    means, stds = EO.nn_ensemble({"energy": golden["pred:energy"], "forces": golden["pred:forces"]})
    for k in ("energy", "forces"):
        _close(means[k], golden["nn:mean:" + k])
        _close(stds[k], golden["nn:std:" + k])


@pytest.mark.parametrize("relative", [False, True])
def test_batched_uncertainty_equals_ase_uncertainties(golden, relative):
    ref = golden["unc:relative" if relative else "unc:absolute"]
    for w, weights in enumerate(golden["weights"]):
        u = EO.batched_uncertainty(golden["pred:energy"], golden["pred:forces"], golden["in:_n_atoms"],
                                   golden["pred:stress"], tuple(weights), relative)
        _close(u, ref[w])


def test_force_terms_restate_the_force_uncertainty(golden):
    n_atoms = golden["in:_n_atoms"]
    t = EO.force_terms(golden["pred:forces"], n_atoms)
    _close(t[:, 0] / n_atoms, golden["unc:absolute"][0])
    _close(t[:, 1] / n_atoms, golden["unc:relative"][0])


def test_zero_total_weight_raises():
    with pytest.raises(ValueError, match="total_weight cannot be zero"):
        EO.normalised_weights(0.0, 0.0, 0.0)


def test_empty_system_has_zero_force_term():
    f = np.random.default_rng(0).normal(size=(3, 4, 3))
    u = EO.batched_uncertainty(None, f, np.array([4, 0]), weights=(0.0, 1.0, 0.0))
    assert u[1] == 0.0 and u[0] > 0.0
