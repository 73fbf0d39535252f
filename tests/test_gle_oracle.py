"""CPU checks of the GLE test oracle (tests/gle_oracle.py) against the reference's own GLE, RPMD-GLE and PIGLET
thermostats, recorded in tests/golden/md_gle.npz, and host-side checks of ``schnetpack_b200.md``'s GLE set-up (matrix
files, units, propagators) that need no device."""
import os

import numpy as np
import pytest
import torch

import gle_oracle as GO
import rpmd_oracle as RO

HERE = os.path.dirname(__file__)
GOLD = os.path.join(HERE, "golden", "md_gle.npz")
FILES = {"sym": "gle_sym.txt", "nonnormal": "gle_nonnormal.txt", "quantum": "gle_quantum.txt",
         "piglet": "gle_piglet_p4.txt"}
CASES = ["gle_sym", "gle_nonnormal", "gle_quantum", "gle_zero_start", "rpmd_gle_nonnormal", "rpmd_gle_quantum", "piglet"]


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def _close(a, b, tol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.max(np.abs(a - b)) <= tol * max(np.max(np.abs(b)), 1e-300), np.max(np.abs(a - b))


def _path(key):
    return os.path.join(HERE, "golden", FILES[key])


def _matrices(g, fkey):
    return g[f"file:{fkey}:A"], (g[f"file:{fkey}:C"] if f"file:{fkey}:C" in g else None)


def _dt(g):
    return float(g["time_step_fs"]) * float(g["fs"])


def _c_default(g, A, P):
    return np.eye(A.shape[-1])[None].repeat(A.shape[0], 0) * float(g["temperature_bath"]) * float(g["kB"]) * P


@pytest.mark.parametrize("case", CASES)
def test_oracle_reference_convention_matches_reference(gold, case):
    g, pre = gold, case + ":"
    P, fkey = int(g[pre + "P"]), str(g[pre + "file"])
    A, C = _matrices(g, fkey)
    rec = g[pre + "noise"]
    th = GO.GLE(A, C, float(g["temperature_bath"]), float(g["kB"]), lambda app, *shape: rec[app],
                convention="reference", free_particle_limit=bool(g[pre + "initial_draw"]), per_mode=case == "piglet",
                ring_polymer=not case.startswith("gle_"))
    rp = RO.RingPolymer(P, float(g["temperature_bath"]), _dt(g), float(g["kB"]), float(g["hbar"]),
                        reference_float32_propagator=P > 1)
    x0, k = torch.as_tensor(g[pre + "x0"])[None], torch.as_tensor(g[pre + "k_tether"])[None, :, None]
    x, p = RO.rpmd_trajectory(rp, g[pre + "positions"], g[pre + "momenta"], g[pre + "masses"], g["n_atoms"],
                              lambda x: -k * (x - x0), int(g["n_steps"]), th)
    _close(x.numpy(), g[pre + "out_positions"])
    _close(p.numpy(), g[pre + "out_momenta"])
    _close(th.s, g[pre + "state"])
    assert th.app == rec.shape[0]                                         # every recorded draw was used
    assert np.abs(g[pre + "out_momenta"] - g[pre + "momenta"]).max() > 1.0   # the thermostat acted


@pytest.mark.parametrize("case", ["gle_sym", "gle_quantum", "rpmd_gle_nonnormal", "piglet"])
def test_library_propagators_match_reference(gold, case):
    """c1 = matrix_exp(-dt/2 A) and c2 = the eigh square root of C - c1 C c1^T against the reference's expm / sqrtm"""
    from schnetpack_b200 import md

    g, pre = gold, case + ":"
    P = int(g[pre + "P"])
    A, C = _matrices(g, str(g[pre + "file"]))
    if C is None:
        C = _c_default(g, A, P)
    ref1, ref2 = g[pre + "c1"].reshape(A.shape), g[pre + "c2"].reshape(A.shape)
    for b in range(A.shape[0]):
        c1, c2 = md._gle_propagators(torch.as_tensor(A[b]), torch.as_tensor(C[b]), _dt(g))
        _close(c1.numpy(), ref1[b], 1e-13)
        _close(c2.numpy(), ref2[b], 1e-10)
        _close(c2.numpy(), c2.numpy().T, 0.0)                           # symmetric by construction


@pytest.mark.parametrize("key", list(FILES))
def test_load_gle_matrices_parses_as_the_reference(gold, key):
    from schnetpack_b200 import md

    A, C = md.load_gle_matrices(_path(key), kB=float(gold["kB"]), fs=float(gold["fs"]))
    ra, rc = _matrices(gold, key)
    assert A.dtype == torch.float64
    _close(A.numpy(), ra, 1e-15)
    if rc is None:
        assert C is None
    else:
        _close(C.numpy(), rc, 1e-15)
    assert A.shape[0] == (4 if key == "piglet" else 1)


def test_unit_constants_are_codata_2014():
    from schnetpack_b200 import md

    assert md._CODATA_HARTREE == 4.359744650e-18          # J
    assert md._CODATA_AUT == 2.418884326509e-17           # s
    # the tabulated relationships, to within their relative standard uncertainty of ~6e-7
    assert abs(md._EV_K / 1.16045221e4 - 1) < 1e-7        # eV / k_B in K
    assert abs(md._HARTREE_K / 3.1577513e5 - 1) < 1e-7    # E_h / k_B in K
    assert abs(md._HARTREE_K / md._EV_K / 27.21138602 - 1) < 1e-9   # E_h in eV
    # the MD units of the reference: a Hartree is 2625.4996 kJ/mol, an atomic time unit 2.418884e-5 ps
    kB, fs = md.KB_MD, md.FS_MD
    assert abs(md._gle_unit("atomic energy units", kB, fs) / 2625.499638 - 1) < 1e-8
    assert abs(md._gle_unit("eV", kB, fs) / 96.4853329 - 1) < 1e-8
    assert abs(1.0 / md._gle_unit("atomic time units^-1", kB, fs) / (md._AUT_FS * fs) - 1) < 1e-15
    assert abs(md._gle_unit("picoseconds^-1", kB, fs) * 1e3 / md._gle_unit("femtoseconds^-1", kB, fs) - 1) < 1e-15


def _write(tmp_path, text):
    p = tmp_path / "m.txt"
    p.write_text(text)
    return str(p)


@pytest.mark.parametrize("text,match", [
    ("# A MATRIX: (furlongs^-1)\n1 0\n0 1\n", "unknown unit 'furlongs"),
    ("# C MATRIX: (K)\n1 0\n0 1\n", "no 'A MATRIX:'"),
    ("# A MATRIX: (femtoseconds^-1)\n1 0\n0 1 2\n", "not square"),
    ("# A MATRIX: (femtoseconds^-1)\n1 0\n0 1\n# C MATRIX: (K)\n1 0 0\n0 1 0\n0 0 1\n", "do not match"),
    ("# A MATRIX: (femtoseconds^-1)\n# Matrix for normal mode 0\n1 0\n0 1\n# Matrix for normal mode 1\n1\n",
     "differ in size"),
    ("# A MATRIX: (femtoseconds^-1)\n" + "\n".join(" ".join("1" if i == j else "0" for j in range(17))
                                                   for i in range(17)) + "\n", "at most 16"),
])
def test_load_gle_matrices_refuses_bad_files(tmp_path, text, match):
    from schnetpack_b200 import md

    with pytest.raises(ValueError, match=match):
        md.load_gle_matrices(_write(tmp_path, text))


def test_classical_gle_refuses_piglet_input_and_invalid_matrices():
    from schnetpack_b200 import md

    with pytest.raises(ValueError, match="Could be PIGLET input"):
        md.GLEThermostat(300.0, _path("piglet"))
    with pytest.raises(ValueError, match="Could be PIGLET input"):
        md.RPMDGLEThermostat(300.0, _path("piglet"))
    A = torch.tensor([[1.0, 10.0], [0.0, 1.0]], dtype=torch.float64)   # positive-stable, but A + A^T is indefinite
    with pytest.raises(ValueError, match="not a valid GLE"):
        md._gle_propagators(A, torch.eye(2, dtype=torch.float64), 0.1)


@pytest.mark.parametrize("key", ["sym", "nonnormal", "quantum", "piglet"])
def test_paper_map_keeps_C_and_the_reference_map_does_not(key):
    """discrete Lyapunov solve of the unit-mass chain: s <- c1 s + c2 xi has the stationary covariance C exactly, the
    reference's s <- c1^T s + c2 xi only for a symmetric A"""
    from schnetpack_b200 import md

    kB, fs = md.KB_MD, md.FS_MD
    A, C = md.load_gle_matrices(_path(key), kB=kB, fs=fs)
    if C is None:
        C = torch.eye(A.shape[-1], dtype=torch.float64).expand_as(A) * 300.0 * kB
    for b in range(A.shape[0]):
        c1, c2 = (t.numpy() for t in md._gle_propagators(A[b], C[b], 1.0 * fs))
        cb = C[b].numpy()
        paper = GO.stationary_covariance(c1, c2, "paper")
        ref = GO.stationary_covariance(c1, c2, "reference")
        _close(paper, cb, 1e-10)
        off = abs(ref[0, 0] / cb[0, 0] - 1.0)
        if key == "sym":
            assert off < 1e-10
        else:
            assert off > 0.01, off                                        # <p^2> is off by more than 1 %
