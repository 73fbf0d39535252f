"""The PaiNN reverse edge kernel on the tensor cores (k_painn_edge_bwd_tc, csrc/painn_tc.cu), where every consumer warp owns
its own edge-balanced sender range and 2 edges of each 16-edge chunk.

CPU: both instantiations fit the 168 registers of a 384-thread CTA without spilling.
GPU, against the fp64 restatement of tests/edge_oracle.py at the suite's 1e-5 relative tolerance: neighbour lists whose
warp ranges are mostly empty, a hub sender that fills many chunks and the range of many warps, edge counts that are not
a multiple of the 16-edge chunk, n_rbf % 4 != 0, unsorted idx_i, with and without mu; the three reverse launches of a
cfg2-sized step (accumulate 0, 1, 1 into a g_rij buffer that holds other values first); and bitwise repeatability."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from edge_oracle import _painn_layer_ref, rel
from schnetpack_b200 import build, ops

DEV = "cuda:0"
RC = 5.0
F = 128
TOL = 1e-5
REG_CAP = 168                     # 65536 registers / 384 threads, in the 8-register allocation granule


# ------------------------------------------------------------------------------------------------ CPU: registers
def test_bwd_tc_fits_its_registers(tmp_path):
    src = os.path.join(build.CSRC, "painn_tc.cu")
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-Xptxas=-v", "-c", src, "-o", str(tmp_path / "painn_tc.o")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    found = 0
    for block in out.stdout.split("Compiling entry function")[1:]:
        if "k_painn_edge_bwd_tc" not in block.splitlines()[0]:
            continue
        found += 1
        spills = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
        regs = re.search(r"Used (\d+) registers", block)
        assert spills and regs, block
        assert (int(spills.group(1)), int(spills.group(2))) == (0, 0), block
        assert int(regs.group(1)) <= REG_CAP, block
    assert found == 2, out.stdout                 # HAS_MU true and false


# ------------------------------------------------------------------------------------------------ GPU helpers
def _sparse_senders(rng):
    """Just above EDGE_TC_MIN_EDGES (E % 16 == 5) over 20 000 atoms, of which 250 send: most of the ~1000 warp ranges hold
    no edge, and the ones that do cross long runs of edge-free senders."""
    n, E = 20000, ops.EDGE_TC_MIN_EDGES + 5
    senders = rng.choice(n, 250, replace=False)
    return n, rng.integers(0, n, E), rng.choice(senders, E)


def _hub_sender(rng):
    """One sender with 3000 of 9007 edges (E % 16 == 15): ~1500 chunks of one warp, the edge share of ~350 warps."""
    n, E, hub = 3000, 9007, 1234
    jj = rng.integers(0, n, E)
    jj[rng.choice(E, 3000, replace=False)] = hub
    return n, rng.integers(0, n, E), jj


def _edges(name, order):
    rng = np.random.default_rng({"sparse_senders": 3, "hub_sender": 4}[name])
    n, ii, jj = {"sparse_senders": _sparse_senders, "hub_sender": _hub_sender}[name](rng)
    E = ii.shape[0]
    v = rng.normal(size=(E, 3))
    v *= (rng.uniform(0.5, 0.99 * RC, E) / np.linalg.norm(v, axis=1))[:, None]
    o = np.lexsort((jj, ii)) if order == "sorted" else rng.permutation(E)
    assert E % 16 != 0 and (order == "sorted") == bool((np.diff(ii[o]) >= 0).all())
    return n, torch.as_tensor(ii[o], device=DEV), torch.as_tensor(jj[o], device=DEV), \
        torch.as_tensor(v[o], dtype=torch.float32, device=DEV)


def _gauss(n_rbf):
    p0 = torch.linspace(0, RC, n_rbf, device=DEV)
    return p0, torch.full((n_rbf,), float(p0[1] - p0[0]), device=DEV)


class _Tc:
    """The tensor-core edge path whatever SPK_B200_EDGE says."""

    def __enter__(self):
        self.saved = ops.EDGE_IMPL
        ops.EDGE_IMPL = "tc"

    def __exit__(self, *exc):
        ops.EDGE_IMPL = self.saved


def _layer(N, n_rbf, has_mu, gen):
    """Inputs of one interaction: x, mu (or None), g_q, g_mu, wf, bf."""
    x = torch.randn(N, 3 * F, device=DEV, generator=gen)
    mu = torch.randn(N, 3, F, device=DEV, generator=gen) if has_mu else None
    g_q, g_mu = torch.randn(N, F, device=DEV, generator=gen), torch.randn(N, 3, F, device=DEV, generator=gen)
    wf = torch.randn(3 * F, n_rbf, device=DEV, generator=gen) * 0.3
    bf = torch.randn(3 * F, device=DEV, generator=gen) * 0.3
    return x, mu, g_q, g_mu, wf, bf


def _reference(x, mu, g_q, g_mu, wf, bf, r, ti, tj, p0, p1):
    """fp64 (g_x, g_mu_in, g_rij) of one interaction (painn.py:55-65 through autograd)."""
    N = x.shape[0]
    x64, r64 = x.double().requires_grad_(), r.double().requires_grad_()
    mu64 = (mu.double() if mu is not None else torch.zeros(N, 3, F, device=DEV, dtype=torch.float64)).requires_grad_()
    qr, mur = _painn_layer_ref(x64, mu64, torch.zeros(N, F, device=DEV, dtype=torch.float64), r64, ti, tj,
                               wf.double(), bf.double(), RC, p0.double(), p1.double())
    return torch.autograd.grad((qr * g_q.double()).sum() + (mur * g_mu.double()).sum(), [x64, mu64, r64])


def _check(g_x, g_mu_in, g_rij, ref, has_mu, seed=None):
    gx_r, gmu_r, gr_r = ref
    if has_mu:
        assert rel(g_x, gx_r) < TOL, rel(g_x, gx_r)
        assert rel(g_mu_in, gmu_r) < TOL, rel(g_mu_in, gmu_r)
    else:
        assert rel(g_x[:, :2 * F], gx_r[:, :2 * F]) < TOL, rel(g_x[:, :2 * F], gx_r[:, :2 * F])
        assert float(g_x[:, 2 * F:].abs().max()) == 0.0 and g_mu_in is None
    want = gr_r + (seed.double() if seed is not None else 0.0)
    assert rel(g_rij, want) < TOL, rel(g_rij, want)


# ------------------------------------------------------------------------------------------------ GPU: partitions
@pytest.mark.gpu
@pytest.mark.parametrize("order", ["sorted", "shuffled"])
@pytest.mark.parametrize("n_rbf", [20, 23])
@pytest.mark.parametrize("name", ["sparse_senders", "hub_sender"])
def test_bwd_tc_partitions(name, n_rbf, order):
    N, ti, tj, r = _edges(name, order)
    E = ti.shape[0]
    g = ops.EdgeGraph(ti, tj, N)
    p0, p1 = _gauss(n_rbf)
    phi, dphi, geo = ops.edge_geometry(r, g, ops.RBF_GAUSSIAN, n_rbf, p0, p1, RC, True)
    gen = torch.Generator(device=DEV).manual_seed(n_rbf)
    with _Tc():
        assert ops.edge_tc_ok(F, n_rbf, E)
        for has_mu in (True, False):
            x, mu, g_q, g_mu, wf, bf = _layer(N, n_rbf, has_mu, gen)
            wpk = ops.painn_pack_filter(wf, bf, F, n_rbf)
            ref = _reference(x, mu, g_q, g_mu, wf, bf, r, ti, tj, p0, p1)
            for acc in (False, True):
                seed = torch.randn(E, 3, device=DEV, generator=gen) * float(ref[2].abs().max())
                g_rij = seed.clone() if acc else torch.full((E, 3), 7.0, device=DEV)
                g_x, g_mu_in = ops.painn_edge_bwd(x, mu, g_q, g_mu, phi, dphi, geo, g, wf, bf, F, n_rbf, g_rij, acc,
                                                  wf_packed=wpk)
                _check(g_x, g_mu_in, g_rij, ref, has_mu, seed if acc else None)


# ------------------------------------------------------------------------------------------------ GPU: cfg2 size
def _cfg2():
    from schnetpack_b200 import synthetic as S

    b = S.aspirin_batch(256)
    ti, tj = torch.as_tensor(b["_idx_i"], device=DEV), torch.as_tensor(b["_idx_j"], device=DEV)
    R = torch.as_tensor(b["_positions"], device=DEV)
    r = (R[tj] - R[ti] + torch.as_tensor(b["_offsets"], device=DEV)).contiguous()
    N = R.shape[0]
    assert (N, ti.shape[0]) == (5376, 77816)
    return N, ti, tj, r, ops.EdgeGraph(ti, tj, N)


@pytest.mark.gpu
def test_bwd_tc_three_interactions_accumulate():
    """The reverse sweep of a PaiNN 128 x 3 step: interaction 3, 2, 1 into one g_rij buffer, accumulate 0, 1, 1; the
    buffer holds other values before the first launch, which must overwrite them."""
    N, ti, tj, r, g = _cfg2()
    n_rbf = 20
    p0, p1 = _gauss(n_rbf)
    phi, dphi, geo = ops.edge_geometry(r, g, ops.RBF_GAUSSIAN, n_rbf, p0, p1, RC, True)
    gen = torch.Generator(device=DEV).manual_seed(31)
    g_rij = torch.randn(ti.shape[0], 3, device=DEV, generator=gen) * 100.0
    want = None
    with _Tc():
        assert ops.edge_tc_ok(F, n_rbf, ti.shape[0])
        for t, has_mu in enumerate((True, True, False)):      # the first interaction sees mu == 0
            x, mu, g_q, g_mu, wf, bf = _layer(N, n_rbf, has_mu, gen)
            ref = _reference(x, mu, g_q, g_mu, wf, bf, r, ti, tj, p0, p1)
            want = ref[2] if want is None else want + ref[2]
            g_x, g_mu_in = ops.painn_edge_bwd(x, mu, g_q, g_mu, phi, dphi, geo, g, wf, bf, F, n_rbf, g_rij, t > 0,
                                              wf_packed=ops.painn_pack_filter(wf, bf, F, n_rbf))
            _check(g_x, g_mu_in, g_rij, (ref[0], ref[1], want), has_mu)


@pytest.mark.gpu
def test_bwd_tc_repeats_bitwise():
    N, ti, tj, r, g = _cfg2()
    n_rbf = 20
    p0, p1 = _gauss(n_rbf)
    phi, dphi, geo = ops.edge_geometry(r, g, ops.RBF_GAUSSIAN, n_rbf, p0, p1, RC, True)
    gen = torch.Generator(device=DEV).manual_seed(37)
    x, mu, g_q, g_mu, wf, bf = _layer(N, n_rbf, True, gen)
    wpk = ops.painn_pack_filter(wf, bf, F, n_rbf)
    seed = torch.randn(ti.shape[0], 3, device=DEV, generator=gen)
    with _Tc():
        outs = []
        for _ in range(2):
            g_rij = seed.clone()
            outs.append((*ops.painn_edge_bwd(x, mu, g_q, g_mu, phi, dphi, geo, g, wf, bf, F, n_rbf, g_rij, True,
                                             wf_packed=wpk), g_rij))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
