"""CPU: the fp64 L-BFGS oracle (tests/relax_oracle.py) reproduces the reference's ASEBatchwiseLBFGS runs recorded in
tests/golden/relax_lbfgs.npz step by step, and treats every system of a ragged batch as if it were alone."""
import os

import numpy as np
import pytest

from relax_oracle import LBFGSOracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "relax_lbfgs.npz")
CASES = ["wrap", "early", "fixed", "cap"]


def load(name):
    z = np.load(GOLDEN)
    return {k.split(":", 1)[1]: z[k] for k in z.files if k.startswith(name + ":")}


def oracle_for(c):
    ptr = np.concatenate([[0], np.cumsum(c["n_atoms"])])
    return LBFGSOracle(c["pos_before"][0], ptr, memory=int(c["memory"]), maxstep=float(c["maxstep"]),
                       damping=float(c["damping"]), alpha=float(c["alpha"]), fixed=c["fixed"])


def rel(a, b):
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_reference_steps(name):
    c = load(name)
    o = oracle_for(c)
    fmax = float(c["fmax"])
    for k in range(c["p"].shape[0]):
        assert rel(o.r, c["pos_before"][k]) <= 1e-12, k
        conv = o.converged(c["forces"][k], fmax)
        assert np.array_equal(conv, c["converged"][k]), k
        o.step(c["forces"][k], fmax)
        assert np.max(np.abs(o.p - c["p"][k])) <= 1e-12 * max(np.max(np.abs(c["p"][k])), 1e-300) or \
            np.array_equal(o.p, c["p"][k]), k
        assert rel(o.newest_rho(), c["rho"][k]) <= 1e-12, k
        assert rel(o.r, c["pos_after"][k]) <= 1e-12, k
    # the reference's step count: the first step count at which every system met the criterion
    final = o.converged(c["final_forces"], fmax)
    if bool(c["all_converged"]):
        assert final.all() and int(o.steps_to_converge.max()) == int(c["nsteps"])
    else:
        assert not final.all() and int(c["nsteps"]) == c["p"].shape[0]


def test_cases_cover_what_they_claim():
    wrap, early, fixed, cap = (load(n) for n in CASES)
    assert wrap["p"].shape[0] > 2 * int(wrap["memory"])                       # the history ring wraps
    conv = early["converged"]
    assert conv[:, 0].any() and not conv[:, 2].any()                           # one converges while others continue
    first = int(np.argmax(conv[:, 0]))
    assert np.array_equal(early["pos_after"][first:, :6], early["pos_before"][first:, :6])   # and is frozen
    mask = fixed["fixed"]
    assert mask.sum() == 2 and np.array_equal(fixed["pos_after"][:, mask], fixed["pos_before"][:, mask])
    longest = np.sqrt((cap["p"] ** 2).sum(-1)).reshape(cap["p"].shape[0], -1, 6).max(-1)
    assert (np.abs(longest - float(cap["maxstep"])) < 1e-12).sum() >= 5 and float(cap["damping"]) < 1.0


def test_ragged_batch_equals_systems_alone():
    rng = np.random.default_rng(3)
    sizes = [1, 5, 3]
    ptr = np.concatenate([[0], np.cumsum(sizes)])
    r = rng.normal(size=(ptr[-1], 3))
    batch = LBFGSOracle(r, ptr, memory=3, maxstep=0.1, alpha=5.0)
    alone = [LBFGSOracle(r[a:b], [0, b - a], memory=3, maxstep=0.1, alpha=5.0) for a, b in zip(ptr[:-1], ptr[1:])]
    for _ in range(8):
        f = -(batch.r - 0.3 * np.sin(batch.r))                                # a smooth field, different per system
        batch.step(f, 1e-6)
        for m, (a, b) in enumerate(zip(ptr[:-1], ptr[1:])):
            alone[m].step(f[a:b], 1e-6)
            np.testing.assert_array_equal(batch.r[a:b], alone[m].r)
