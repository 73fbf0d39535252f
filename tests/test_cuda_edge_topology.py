"""GPU: every edge kernel against an fp64 torch restatement on neighbour lists built to break the edge-balanced row
ranges (spk_block_row_begin / _warp in csrc/common.cuh) and the row-boundary walks inside them: a hub row that spans many
CTA shares, runs of edge-free rows, row degrees on and around the chunk sizes, self images and repeated pairs of a small
periodic box, a single edge, and the hub graph cut at the edge counts where the dispatchers switch kernels -- each in
sorted, permuted and reversed edge order.

Tolerances are those of tests/test_cuda_kernels.py for the same operation.  A hub row is a long fp32 sum, so its error is
judged against the row's fp64 sum of |terms| (bound HUB_TOL); every hub check also shows that this bound would see one
edge dropped from the row.  On ``hub`` and ``empty_runs`` every kernel is called twice and must repeat bit for bit."""
import functools
import math

import numpy as np
import pytest
import torch

from edge_oracle import _check_graph, _painn_layer_ref, rel, so3_conv_ref
from schnetpack_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RC = 5.0
HUB_TOL = 2e-5
CHUNK_DEGREES = (1, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33)
SIZED = {"hub_tc_min-1": ops.EDGE_TC_MIN_EDGES - 1, "hub_tc_min": ops.EDGE_TC_MIN_EDGES,
         "hub_cfconv_min": ops.CFCONV_TC_MIN_EDGES}
TOPOLOGIES = ["hub", "empty_runs", "chunk_edges", "chunk_edges_odd", "self_images", "single_edge", *SIZED]
ORDERS = ["sorted", "permuted", "reversed"]
DETERMINISM = ("hub", "empty_runs")

topo = pytest.mark.parametrize("order", ORDERS)
names = pytest.mark.parametrize("name", TOPOLOGIES)


# ------------------------------------------------------------------------------------------------ graph generators
def _hub_edges(rng):
    """640 atoms, ~8 k edges: atom 37 receives and sends 1500 (about 25 CTA shares on 132 SMs), atom 637 (in the last
    rows) 300 each, the rest a random background."""
    n, hub, hub2 = 640, 37, 637
    rest = np.setdiff1d(np.arange(n), [hub, hub2])
    bg = 8000 - 3600
    bi = rng.integers(0, rest.shape[0], bg)
    ii = [np.full(1500, hub), rng.choice(rest, 1500), np.full(300, hub2), rng.choice(rest, 300), rest[bi]]
    jj = [rng.choice(rest, 1500), np.full(1500, hub), rng.choice(rest, 300), np.full(300, hub2),
          rest[(bi + rng.integers(1, rest.shape[0], bg)) % rest.shape[0]]]
    return n, np.concatenate(ii), np.concatenate(jj), (hub, hub2)


def _empty_runs_edges(rng):
    """4000 atoms, edges only among rows 6..149 and 250..399: edge-free runs at the start, 100 in the middle and 3600 at
    the end, as receivers and as senders; a few active rows draw degree 0 as well."""
    act = np.r_[6:150, 250:400]
    deg = rng.integers(0, 41, act.shape[0])
    ii = np.repeat(act, deg)
    return 4000, ii, rng.choice(act, ii.shape[0]), ()


def _chunk_edges(rng, odd):
    """Row degrees from CHUNK_DEGREES (on, one below and one above the chunk sizes 4 / 8 / 16 / 32), then rows of
    degree 1 up to E = 128 k (+ 1 for ``odd``)."""
    deg = np.concatenate([np.concatenate([CHUNK_DEGREES, rng.permutation(CHUNK_DEGREES)]) for _ in range(6)])
    E = int(deg.sum())
    target = (E // 128 + 1) * 128 + int(odd)
    deg = np.concatenate([deg, np.ones(target - E, dtype=deg.dtype)])
    n = deg.shape[0]
    ii = np.repeat(np.arange(n), deg)
    return n, ii, rng.integers(0, n, ii.shape[0]), ()


def _place(rng, n, ii, jj, special):
    """Positions on a 1/64 grid and offsets such that r_ij = R[j] - R[i] + offset has |r_ij| in [0.5, RC); with
    ``special`` three edges get grid-exact vectors (exact in fp32): two at the cutoff, one beyond it (fc == 0)."""
    pos = rng.integers(0, 1024, (n, 3)) / 64.0
    E = ii.shape[0]
    v = rng.normal(size=(E, 3))
    v *= (rng.uniform(0.5, 0.99 * RC, E) / np.linalg.norm(v, axis=1))[:, None]
    if special:
        v[rng.choice(E, 3, replace=False)] = [[RC, 0.0, 0.0], [0.0, 0.0, -RC], [3.5, 4.0, 0.0]]
    return pos.astype(np.float32), (v - (pos[jj] - pos[ii])).astype(np.float32)


def _self_images():
    """10 atoms in a 4.6 A periodic box (cutoff 5): every atom sees its own images and most pairs appear with several
    offsets; two more self edges sit exactly at the cutoff and beyond it."""
    from schnetpack_b200 import synthetic as S

    b = S.periodic_box(10, density=10 / 4.6 ** 3, cutoff=RC, seed=7)
    ii = np.concatenate([b["_idx_i"], [3, 3]])
    jj = np.concatenate([b["_idx_j"], [3, 3]])
    off = np.concatenate([b["_offsets"], [[RC, 0.0, 0.0], [0.0, 3.0, 4.5]]]).astype(np.float32)
    assert bool(((b["_idx_i"] == b["_idx_j"]) & np.abs(b["_offsets"]).any(1)).any())
    o = np.lexsort((jj, ii))
    return b["_positions"], ii[o], jj[o], off[o], 10


@functools.lru_cache(maxsize=None)
def topology(name, order="sorted"):
    """-> (positions [n,3] f32, idx_i, idx_j, offsets [E,3] f32, n_atoms, hub rows); the same edges in every order."""
    rng = np.random.default_rng(TOPOLOGIES.index(name) + 11)
    hubs = ()
    if name == "self_images":
        pos, ii, jj, off, n = _self_images()
    else:
        if name.startswith("hub"):
            n, ii, jj, hubs = _hub_edges(np.random.default_rng(11))
        elif name == "empty_runs":
            n, ii, jj, hubs = _empty_runs_edges(rng)
        elif name.startswith("chunk_edges"):
            n, ii, jj, hubs = _chunk_edges(rng, name.endswith("odd"))
        else:
            n, ii, jj = 5, np.array([2]), np.array([3])
        o = np.lexsort((jj, ii))
        ii, jj = ii[o], jj[o]
        if name in SIZED:                       # the hub graph cut after its first E edges (hub row 37 stays whole)
            ii, jj, hubs = ii[:SIZED[name]], jj[:SIZED[name]], hubs[:1]
        pos, off = _place(rng, n, ii, jj, special=ii.shape[0] > 1)
    E = ii.shape[0]
    perm = {"sorted": np.arange(E), "permuted": np.random.default_rng(5).permutation(E),
            "reversed": np.arange(E)[::-1].copy()}[order]
    return pos, ii[perm].astype(np.int64), jj[perm].astype(np.int64), off[perm], n, hubs


def test_topologies_are_what_they_claim():
    """CPU-side facts the kernel tests rely on (checked on the generated lists, not assumed)."""
    for name in TOPOLOGIES:
        pos, ii, jj, off, n, hubs = topology(name)
        r = pos[jj].astype(np.float64) - pos[ii] + off
        d = np.linalg.norm(r, axis=1)
        assert d.min() >= 0.5 - 1e-5 and (d < RC).sum() >= ii.shape[0] - 3, name
        deg = np.bincount(ii, minlength=n)
        if name == "hub":
            assert 7900 <= ii.shape[0] <= 8100 and deg[37] == 1500 and np.bincount(jj, minlength=n)[37] == 1500
            assert deg[37] > 20 * ii.shape[0] / 132
        if name == "empty_runs":
            assert deg[:6].sum() == 0 and deg[150:250].sum() == 0 and deg[400:].sum() == 0 and deg.sum() > 3000
        if name.startswith("chunk_edges"):
            assert set(deg.tolist()) <= set(CHUNK_DEGREES) and ii.shape[0] % 128 == int(name.endswith("odd"))
        if name == "self_images":
            assert (ii == jj).sum() > 10
            pairs = np.stack([ii, jj], 1)
            assert np.unique(pairs, axis=0).shape[0] < pairs.shape[0]
        if name in SIZED:
            assert ii.shape[0] == SIZED[name] and deg[37] == 1500
        if name != "single_edge":
            assert (d >= RC).sum() >= 2 and (d == RC).sum() >= 1
    assert topology("single_edge")[1].shape[0] == 1


# ------------------------------------------------------------------------------------------------ helpers
def _case(name, order):
    pos, ii, jj, off, n, hubs = topology(name, order)
    R = torch.as_tensor(pos, device=DEV)
    ti, tj = torch.as_tensor(ii, device=DEV), torch.as_tensor(jj, device=DEV)
    o = torch.as_tensor(off, device=DEV)
    r = ops.pairwise_fwd(R, ti, tj, o)
    assert torch.equal(r, R[tj] - R[ti] + o)
    g = ops.EdgeGraph(ti, tj, n)
    E = ii.shape[0]
    eid = g.slot_eid[:E].long()
    return dict(ii=ii, jj=jj, n=n, E=E, hubs=hubs, ti=ti, tj=tj, r=r, g=g, eid=eid, si=ti[eid], sj=tj[eid],
                det=name in DETERMINISM)


def _run(det, fn):
    """fn() -> tuple of tensors; on the determinism topologies a second call must give bitwise the same tensors."""
    out = fn()
    if det:
        again = fn()
        for a, b in zip(out, again):
            if a is not None:
                assert torch.equal(a, b)
    return out


def _hub_err(got, ref, absterm, h):
    return float((got[h].double() - ref[h].double()).abs().max() / absterm[h].double().abs().max())


def _check(got, ref, tol, hubs=(), absterm=None):
    """rel(got, ref) < tol over the rows that are not hubs; a hub row's max error over its fp64 sum of |terms| < HUB_TOL."""
    got, ref = got.double(), ref.double()
    if not hubs:
        assert rel(got, ref) < tol, rel(got, ref)
        return
    rest = torch.ones(ref.shape[0], dtype=torch.bool, device=ref.device)
    rest[list(hubs)] = False
    assert rel(got[rest], ref[rest]) < tol, rel(got[rest], ref[rest])
    for h in hubs:
        assert _hub_err(got, ref, absterm, h) < HUB_TOL, (h, _hub_err(got, ref, absterm, h))


def _sees_one_edge(ref, ref_dropped, absterm, h):
    """The hub bound is at least ten times finer than the change of one hub-row edge dropped from the reference."""
    assert _hub_err(ref_dropped, ref, absterm, h) >= 10 * HUB_TOL, _hub_err(ref_dropped, ref, absterm, h)


def _hub_edge(c, role, size=None):
    """An edge of hub 0's receiver row (role 'i') or sender row (role 'j'): the first with a large filter (d < 2.5), or
    the one with the largest ``size`` [E] where the terms carry no filter."""
    idx = c["ti"] if role == "i" else c["tj"]
    if size is not None:
        return int(torch.where(idx == c["hubs"][0], size, -1.0).argmax())
    d = c["r"].norm(dim=1)
    return int(torch.nonzero((idx == c["hubs"][0]) & (d < 2.5))[0])


def _without(E, e, device):
    keep = torch.ones(E, dtype=torch.bool, device=device)
    keep[e] = False
    return torch.nonzero(keep)[:, 0]


def _gauss(n_rbf):
    p0 = torch.linspace(0, RC, n_rbf, device=DEV)
    return p0, torch.full((n_rbf,), float(p0[1] - p0[0]), device=DEV)


def _gauss_ref(d, p0, p1):
    return torch.exp(-0.5 / p1.double() ** 2 * (d - p0.double()) ** 2)


def _fc_ref(d):
    return 0.5 * (torch.cos(d * math.pi / RC) + 1) * (d < RC)


# ------------------------------------------------------------------------------------------------ graph structure
@names
@topo
def test_graph_structure(name, order):
    c = _case(name, order)
    ii, jj, n, E = c["ii"], c["jj"], c["n"], c["E"]
    info = c["g"].validate()
    assert info["sorted"] == bool((np.diff(ii) >= 0).all())
    assert info["max_in_degree"] == np.bincount(ii, minlength=n).max()
    assert info["max_out_degree"] == np.bincount(jj, minlength=n).max()
    _check_graph(c["g"], ii, jj, n)
    # the active-edge view (|r_ij| < cutoff) drops exactly the edges at and beyond the cutoff
    ga = ops.EdgeGraph(c["ti"], c["tj"], n, r_ij=c["r"], cutoff=RC)
    act = (c["r"].double().norm(dim=1) < RC).cpu().numpy()
    n_act = int(ga.rowptr[-1])
    cnt = np.bincount(ii[act], minlength=n)
    assert n_act == int(act.sum())
    np.testing.assert_array_equal(ga.rowptr.cpu().numpy(), np.concatenate([[0], np.cumsum(cnt)]))
    se = ga.slot_eid[:n_act].cpu().numpy()
    np.testing.assert_array_equal(np.sort(se), np.nonzero(act)[0])
    np.testing.assert_array_equal(ii[se], np.repeat(np.arange(n), cnt))
    np.testing.assert_array_equal(ga.slot_j[:n_act].cpu().numpy(), jj[se])


# ------------------------------------------------------------------------------------------------ geometry
@names
@topo
@pytest.mark.parametrize("kind,n_rbf", [("gaussian", 18), ("bessel", 18), ("gaussian", 38)])   # two zero pad columns
def test_edge_geometry(name, order, kind, n_rbf):
    from schnetpack_b200 import nn as snn

    c = _case(name, order)
    mod = (snn.GaussianRBF(n_rbf, RC) if kind == "gaussian" else snn.BesselRBF(n_rbf, RC)).to(DEV)
    p0, p1 = mod.kernel_params()
    phi, dphi, geo = _run(c["det"], lambda: ops.edge_geometry(c["r"], c["g"], mod.kind, n_rbf, p0, p1, RC, True))
    r64 = c["r"][c["eid"]].double().requires_grad_()            # slot order
    d = r64.norm(dim=1)
    if kind == "gaussian":
        ref = _gauss_ref(d[:, None], p0, p1)
    else:
        ref = torch.sin(d[:, None] * p0.double()) / d[:, None]
    fc = _fc_ref(d)
    assert rel(phi[:, :n_rbf], ref) < 2e-6
    assert float(phi[:, n_rbf:].abs().max()) == 0.0 and float(dphi[:, n_rbf:].abs().max()) == 0.0
    assert rel(geo[:, 3], d) < 1e-6 and rel(geo[:, :3], r64 / d[:, None]) < 1e-6 and rel(geo[:, 6], 1 / d) < 1e-6
    assert (geo[:, 4] - fc).abs().max() < 2e-7
    assert bool((geo[:, 4][d >= RC] == 0).all()) and bool((geo[:, 5][d >= RC] == 0).all())
    dref = torch.stack([torch.autograd.grad(ref[:, k].sum(), r64, retain_graph=True)[0] for k in range(n_rbf)], 1)
    assert rel(dphi[:, :n_rbf, None].double() * geo[:, None, :3].double(), dref) < 5e-6
    dfc = torch.autograd.grad(fc.sum(), r64)[0]
    assert (geo[:, 5:6].double() * geo[:, :3].double() - dfc).abs().max() < 1e-6


# ------------------------------------------------------------------------------------------------ PaiNN
def _painn_filter(r64, wf, bf, p0, p1):
    d = r64.norm(dim=1, keepdim=True)
    return (_gauss_ref(d, p0, p1) @ wf.double().t() + bf.double()) * _fc_ref(d), r64 / d


def _painn_msg(x, mu, W, u, ii, jj, n, F):
    """The edge sums of one PaiNN interaction (painn.py:55-65) given the filter W [E,3F] and directions u [E,3]."""
    dq, dmuR, dmumu = (W * x[jj]).split(F, dim=-1)
    dmu = dmuR[:, None, :] * u[:, :, None] + dmumu[:, None, :] * mu[jj]
    return (torch.zeros((n, F), dtype=x.dtype, device=x.device).index_add(0, ii, dq),
            torch.zeros((n, 3, F), dtype=x.dtype, device=x.device).index_add(0, ii, dmu))


def _painn_abs(x, mu, g_q, g_mu, W, u, ii, jj, n, F):
    """fp64 sums of |terms| of the forward outputs and of the input gradients."""
    xa, ma = x.double().abs().requires_grad_(), mu.double().abs().requires_grad_()
    qa, mua = _painn_msg(xa, ma, W.abs(), u.abs(), ii, jj, n, F)
    gxa, gma = torch.autograd.grad((qa * g_q.double().abs()).sum() + (mua * g_mu.double().abs()).sum(), [xa, ma])
    return qa.detach(), mua.detach(), gxa, gma


@names
@topo
@pytest.mark.parametrize("impl", ["ldg", "tc"])
def test_painn_edge(name, order, impl):
    """spk_painn_edge_{fwd,bwd} (streaming, csrc/painn.cu) and _tc (wgmma filter, csrc/painn_tc.cu) with and without mu,
    accumulate False and True."""
    c = _case(name, order)
    ti, tj, N, E, hubs = c["ti"], c["tj"], c["n"], c["E"], c["hubs"]
    torch.manual_seed(2)
    F, n_rbf = 128, 20
    p0, p1 = _gauss(n_rbf)
    x, q = torch.randn(N, 3 * F, device=DEV), torch.randn(N, F, device=DEV)
    wf, bf = torch.randn(3 * F, n_rbf, device=DEV) * 0.3, torch.randn(3 * F, device=DEV) * 0.3
    g_q, g_mu = torch.randn(N, F, device=DEV), torch.randn(N, 3, F, device=DEV)
    phi, dphi, geo = ops.edge_geometry(c["r"], c["g"], ops.RBF_GAUSSIAN, n_rbf, p0, p1, RC, True)
    wpk = ops.painn_pack_filter(wf, bf, F, n_rbf) if impl == "tc" else None
    r64 = c["r"].double().requires_grad_()
    W, u = _painn_filter(r64.detach(), wf, bf, p0, p1)
    refargs = (wf.double(), bf.double(), RC, p0.double(), p1.double())
    saved = ops.EDGE_IMPL, ops.EDGE_TC_MIN_EDGES
    ops.EDGE_IMPL, ops.EDGE_TC_MIN_EDGES = impl, 1
    try:
        assert ops.edge_tc_ok(F, n_rbf, E) == (impl == "tc")
        for has_mu in (True, False):
            mu = torch.randn(N, 3, F, device=DEV) if has_mu else None
            x64, q64 = x.double().requires_grad_(), q.double()
            mu64 = (mu.double() if has_mu else torch.zeros(N, 3, F, device=DEV, dtype=torch.float64)).requires_grad_()
            qr, mur = _painn_layer_ref(x64, mu64, q64, r64, ti, tj, *refargs)
            qa, mua, gxa, gma = _painn_abs(x, mu64.detach(), g_q, g_mu, W, u, ti, tj, N, F)
            qa, mua, gma = qa + q64.abs(), mua + mu64.detach().abs(), gma + g_mu.double().abs()
            qo, muo = _run(c["det"], lambda: ops.painn_edge_fwd(x, mu, q, phi, geo, c["g"], wf, bf, F, n_rbf,
                                                                 wf_packed=wpk))
            _check(qo, qr, 3e-6, hubs, qa)
            _check(muo, mur, 3e-6, hubs, mua)
            gx_r, gmu_r, gr_r = torch.autograd.grad((qr * g_q.double()).sum() + (mur * g_mu.double()).sum(),
                                                    [x64, mu64, r64])
            for acc in (False, True):
                seed = torch.randn(E, 3, device=DEV) * float(gr_r.abs().max())

                def bwd():
                    g_rij = seed.clone() if acc else torch.full((E, 3), 7.0, device=DEV)
                    return (*ops.painn_edge_bwd(x, mu, g_q, g_mu, phi, dphi, geo, c["g"], wf, bf, F, n_rbf, g_rij, acc,
                                                wf_packed=wpk), g_rij)

                g_x, g_mu_in, g_rij = _run(c["det"], bwd)
                if has_mu:
                    _check(g_x, gx_r, 5e-6, hubs, gxa)
                    _check(g_mu_in, gmu_r, 5e-6, hubs, gma)
                else:
                    _check(g_x[:, :2 * F], gx_r[:, :2 * F], 5e-6, hubs, gxa)
                    assert float(g_x[:, 2 * F:].abs().max()) == 0.0
                assert rel(g_rij, gr_r + (seed.double() if acc else 0.0)) < 1e-5
            if hubs and has_mu:
                h = hubs[0]
                k = _without(E, _hub_edge(c, "i"), DEV)
                qd, _ = _painn_layer_ref(x64, mu64, q64, r64[k], ti[k], tj[k], *refargs)
                _sees_one_edge(qr, qd, qa, h)
                k = _without(E, _hub_edge(c, "j"), DEV)
                qd, mud = _painn_layer_ref(x64, mu64, q64, r64[k], ti[k], tj[k], *refargs)
                gxd = torch.autograd.grad((qd * g_q.double()).sum() + (mud * g_mu.double()).sum(), x64)[0]
                _sees_one_edge(gx_r, gxd, gxa, h)
    finally:
        ops.EDGE_IMPL, ops.EDGE_TC_MIN_EDGES = saved


@names
@topo
def test_painn_edge_wij(name, order):
    """spk_painn_edge_wij_{fwd,bwd}: materialised filter and directions in the caller's edge order."""
    c = _case(name, order)
    ti, tj, N, E, hubs = c["ti"], c["tj"], c["n"], c["E"], c["hubs"]
    torch.manual_seed(5)
    F = 64
    x, mu, q = torch.randn(N, 3 * F, device=DEV), torch.randn(N, 3, F, device=DEV), torch.randn(N, F, device=DEV)
    W, u = torch.randn(E, 3 * F, device=DEV), torch.randn(E, 3, device=DEV)
    g_q, g_mu = torch.randn(N, F, device=DEV), torch.randn(N, 3, F, device=DEV)
    qo, muo = _run(c["det"], lambda: ops.painn_edge_wij_fwd(x, mu, q, W, u, c["g"], F))
    x64, mu64, W64, u64 = (t.double().requires_grad_() for t in (x, mu, W, u))

    def ref(k):
        dq, dmu = _painn_msg(x64, mu64, W64[k], u64[k], ti[k], tj[k], N, F)
        return q.double() + dq, mu64 + dmu

    qr, mur = ref(slice(None))
    qa, mua, gxa, gma = _painn_abs(x, mu, g_q, g_mu, W.double(), u.double(), ti, tj, N, F)
    _check(qo, qr, 2e-6, hubs, qa + q.double().abs())
    _check(muo, mur, 2e-6, hubs, mua + mu.double().abs())
    gx_r, gmu_r, gW_r, gu_r = torch.autograd.grad((qr * g_q.double()).sum() + (mur * g_mu.double()).sum(),
                                                  [x64, mu64, W64, u64])
    g_x, g_mu_in, g_W, g_u = _run(c["det"], lambda: ops.painn_edge_wij_bwd(x, mu, g_q, g_mu, W, u, c["g"], F))
    _check(g_x, gx_r, 3e-6, hubs, gxa)
    _check(g_mu_in, gmu_r, 3e-6, hubs, gma + g_mu.double().abs())
    assert rel(g_W, gW_r) < 3e-6 and rel(g_u, gu_r) < 5e-6
    if hubs:
        qd, _ = ref(_without(E, _hub_edge(c, "i"), DEV))
        _sees_one_edge(qr, qd, qa, hubs[0])
        qd, mud = ref(_without(E, _hub_edge(c, "j"), DEV))
        gxd = torch.autograd.grad((qd * g_q.double()).sum() + (mud * g_mu.double()).sum(), x64)[0]
        _sees_one_edge(gx_r, gxd, gxa, hubs[0])


# ------------------------------------------------------------------------------------------------ SchNet
@names
@topo
def test_cfconv_and_radial_bwd(name, order):
    """spk_cfconv_{fwd,bwd} (filter and geometry in slot order) and spk_radial_bwd (scattered to the edge order)."""
    c = _case(name, order)
    si, sj, N, E, hubs = c["si"], c["sj"], c["n"], c["E"], c["hubs"]
    torch.manual_seed(6)
    F, n_rbf = 128, 20
    p0, p1 = _gauss(n_rbf)
    phi, dphi, geo = ops.edge_geometry(c["r"], c["g"], ops.RBF_GAUSSIAN, n_rbf, p0, p1, RC, True)
    h, w_raw, g_m = torch.randn(N, F, device=DEV), torch.randn(E, F, device=DEV), torch.randn(N, F, device=DEV)
    (m,) = _run(c["det"], lambda: (ops.cfconv_fwd(h, w_raw, geo, c["g"], F),))
    h64, w64 = h.double().requires_grad_(), w_raw.double().requires_grad_()
    fc64 = geo[:, 4].double().requires_grad_()

    def ref(k):
        return torch.zeros(N, F, device=DEV, dtype=torch.float64).index_add(0, si[k], h64[sj[k]] * w64[k] * fc64[k, None])

    m_ref = ref(slice(None))
    ha = h.double().abs().requires_grad_()
    m_abs = torch.zeros(N, F, device=DEV, dtype=torch.float64).index_add(0, si, ha[sj] * (w64 * fc64[:, None]).abs())
    gh_abs = torch.autograd.grad((m_abs * g_m.double().abs()).sum(), ha)[0]
    _check(m, m_ref, 2e-6, hubs, m_abs.detach())
    gh_r, gw_r, gfc_r = torch.autograd.grad((m_ref * g_m.double()).sum(), [h64, w64, fc64])
    g_h, g_wraw, g_fc = _run(c["det"], lambda: ops.cfconv_bwd(h, w_raw, geo, g_m, c["g"], F))
    _check(g_h, gh_r, 3e-6, hubs, gh_abs)
    assert rel(g_wraw, gw_r) < 3e-6 and rel(g_fc, gfc_r) < 3e-6
    if hubs:
        slot_of = torch.empty_like(c["eid"])
        slot_of[c["eid"]] = torch.arange(E, device=DEV)
        md = ref(_without(E, slot_of[_hub_edge(c, "i")], DEV))
        _sees_one_edge(m_ref, md, m_abs.detach(), hubs[0])
        md = ref(_without(E, slot_of[_hub_edge(c, "j")], DEV))
        ghd = torch.autograd.grad((md * g_m.double()).sum(), h64)[0]
        _sees_one_edge(gh_r, ghd, gh_abs, hubs[0])
    # radial_bwd: chain through phi(d) and fc(d); g_rij lands in the caller's edge order
    g_phi = torch.randn(E, ops.kp(n_rbf), device=DEV)
    r64 = c["r"][c["eid"]].double().requires_grad_()
    d = r64.norm(dim=1)
    gr_ref = torch.autograd.grad((_gauss_ref(d[:, None], p0, p1) * g_phi[:, :n_rbf].double()).sum()
                                 + (_fc_ref(d) * g_fc.double()).sum(), r64)[0]
    for acc in (False, True):
        seed = torch.randn(E, 3, device=DEV)

        def radial():
            g_rij = seed.clone() if acc else torch.full((E, 3), 7.0, device=DEV)
            return (ops.radial_bwd(g_phi, g_fc, dphi, geo, c["g"], n_rbf, g_rij, accumulate=acc),)

        (g_rij,) = _run(c["det"], radial)
        assert rel(g_rij[c["eid"]], gr_ref + (seed[c["eid"]].double() if acc else 0.0)) < 1e-5


@names
@topo
def test_schnet_cfconv_fwd_tc(name, order):
    """csrc/schnet_tc.cu on the active-edge graph (edges at and beyond the cutoff are not in it)."""
    c = _case(name, order)
    ti, tj, N, hubs = c["ti"], c["tj"], c["n"], c["hubs"]
    torch.manual_seed(9)
    F, n_rbf = 128, 20
    p0, p1 = _gauss(n_rbf)
    r = c["r"]
    ga = ops.EdgeGraph(ti, tj, N, r_ij=r, cutoff=RC)
    phi, _, geo = ops.edge_geometry(r, ga, ops.RBF_GAUSSIAN, n_rbf, p0, p1, RC, False, active_only=True)
    w0, b0 = torch.randn(F, n_rbf, device=DEV) * 0.3, torch.randn(F, device=DEV) * 0.3
    w1, b1 = torch.randn(F, F, device=DEV) * 0.1, torch.randn(F, device=DEV) * 0.1
    h = torch.randn(N, F, device=DEV)
    pk = ops.schnet_pack_filter(w0, b0, w1, n_rbf)
    (m,) = _run(c["det"], lambda: (ops.schnet_cfconv_fwd_tc(h, phi, geo, ga, pk, b1, ops.ACT_SSP, n_rbf),))
    d64 = r.double().norm(dim=1)
    hid = torch.nn.functional.softplus(_gauss_ref(d64[:, None], p0, p1) @ w0.double().t() + b0.double()) - math.log(2.0)
    W = (hid @ w1.double().t() + b1.double()) * _fc_ref(d64)[:, None]

    def ref(k):
        return torch.zeros(N, F, device=DEV, dtype=torch.float64).index_add(0, ti[k], h.double()[tj[k]] * W[k])

    m_ref = ref(slice(None))
    m_abs = torch.zeros(N, F, device=DEV, dtype=torch.float64).index_add(0, ti, (h.double()[tj] * W).abs())
    _check(m, m_ref, 3e-6, hubs, m_abs)
    if hubs:
        _sees_one_edge(m_ref, ref(_without(c["E"], _hub_edge(c, "i"), DEV)), m_abs, hubs[0])


# ------------------------------------------------------------------------------------------------ SO3net
@names
@topo
def test_so3_conv(name, order):
    """spk_so3_conv_{fwd,bwd} at lmax 2 (n_rbf 20: filter weights in registers)."""
    c = _case(name, order)
    ti, tj, N, E, hubs = c["ti"], c["tj"], c["n"], c["E"], c["hubs"]
    torch.manual_seed(12)
    L, F, n_rbf = 2, 64, 20
    S = (L + 1) ** 2
    p0, p1 = _gauss(n_rbf)
    phi, dphi, geo = ops.edge_geometry(c["r"], c["g"], ops.RBF_GAUSSIAN, n_rbf, p0, p1, RC, True)
    x = torch.randn(N, S, F, device=DEV)
    wf, bf = torch.randn((L + 1) * F, n_rbf, device=DEV) * 0.3, torch.randn((L + 1) * F, device=DEV) * 0.3
    g_y, g_res = torch.randn(N, S, F, device=DEV), torch.randn(N, S, F, device=DEV)
    (y,) = _run(c["det"], lambda: (ops.so3_conv_fwd(x, phi, geo, c["g"], wf, bf, L, F, n_rbf),))
    x64, r64 = x.double().requires_grad_(), c["r"].double().requires_grad_()
    wf64, bf64 = wf.double(), bf.double()

    def radial(d):
        return _gauss_ref(d, p0, p1)

    def ref(k):
        return so3_conv_ref(x64, r64[k], ti[k], tj[k], wf64, bf64, L, RC, radial)

    y_ref = ref(slice(None))
    xa = x.double().abs().requires_grad_()
    y_abs = so3_conv_ref(xa, r64.detach(), ti, tj, wf64, bf64, L, RC, radial, absolute=True)
    gx_abs = torch.autograd.grad((y_abs * g_y.double().abs()).sum(), xa)[0] + g_res.double().abs()
    _check(y, y_ref, 3e-6, hubs, y_abs.detach())
    gx_r, gr_r = torch.autograd.grad((y_ref * g_y.double()).sum(), [x64, r64])
    for acc in (False, True):
        seed = torch.randn(E, 3, device=DEV) * float(gr_r.abs().max())

        def bwd():
            g_rij = seed.clone() if acc else torch.full((E, 3), 7.0, device=DEV)
            return ops.so3_conv_bwd(x, g_y, phi, dphi, geo, c["g"], wf, bf, L, F, n_rbf, g_res, g_rij, acc), g_rij

        g_x, g_rij = _run(c["det"], bwd)
        _check(g_x, gx_r + g_res.double(), 5e-6, hubs, gx_abs)
        assert rel(g_rij, gr_r + (seed.double() if acc else 0.0)) < 1e-5
    if hubs:
        _sees_one_edge(y_ref, ref(_without(E, _hub_edge(c, "i"), DEV)), y_abs.detach(), hubs[0])
        yd = ref(_without(E, _hub_edge(c, "j"), DEV))
        gxd = torch.autograd.grad((yd * g_y.double()).sum(), x64)[0] + g_res.double()
        _sees_one_edge(gx_r + g_res.double(), gxd, gx_abs, hubs[0])


# ------------------------------------------------------------------------------------------------ pairwise / virial / scatter
@names
@topo
def test_pairwise_bwd(name, order):
    c = _case(name, order)
    ti, tj, N, E, hubs = c["ti"], c["tj"], c["n"], c["E"], c["hubs"]
    torch.manual_seed(8)
    gr = torch.randn(E, 3, device=DEV)

    def ref(k):
        return (torch.zeros(N, 3, device=DEV, dtype=torch.float64).index_add(0, tj[k], gr[k].double())
                .index_add(0, ti[k], -gr[k].double()))

    g_ref = ref(slice(None))
    g_abs = (torch.zeros(N, 3, device=DEV, dtype=torch.float64).index_add(0, tj, gr.double().abs())
             .index_add(0, ti, gr.double().abs()))
    for sign in (1.0, -1.0):
        (gR,) = _run(c["det"], lambda: (ops.pairwise_bwd(gr, c["g"], sign),))
        _check(gR, sign * g_ref, 2e-6, hubs, g_abs)
    if hubs:
        _sees_one_edge(g_ref, ref(_without(E, _hub_edge(c, "i", gr.abs().max(1)[0]), DEV)), g_abs, hubs[0])


def _systems(ii, n):
    """Contiguous atom ranges: one system without atoms, and a system of edge-free atoms wherever the list has a run
    of them; the rest split in three."""
    deg = np.bincount(ii, minlength=n)
    cuts = {0, n, n // 3, (2 * n) // 3}
    free = np.nonzero(deg == 0)[0]
    if free.shape[0]:
        a = int(free[0])
        b = a
        while b < n and deg[b] == 0:
            b += 1
        cuts |= {a, b}
    ptr = sorted(cuts)
    ptr.insert(ptr.index(n // 3), n // 3)                     # n // 3 twice: a system without atoms
    return np.array(ptr, dtype=np.int32)


@names
@topo
def test_pairwise_virial(name, order):
    """Per-system virial (fp64, deterministic segmented sums) with an empty system and, where the list has edge-free
    atoms, a system without edges."""
    c = _case(name, order)
    ii, n, E = c["ii"], c["n"], c["E"]
    torch.manual_seed(10)
    gr = torch.randn(E, 3, device=DEV)
    ptr = _systems(ii, n)
    n_sys = ptr.shape[0] - 1
    sys_ptr = torch.as_tensor(ptr, device=DEV)

    def run():
        W = torch.full((n_sys, 3, 3), 3.0, dtype=torch.float64, device=DEV)
        ops.pairwise_virial(gr, c["r"], c["g"], sys_ptr, W)
        return (W,)

    (W,) = _run(c["det"], run)
    sys_of_atom = torch.as_tensor(np.searchsorted(ptr, np.arange(n), side="right") - 1, device=DEV)
    ref = torch.zeros(n_sys, 3, 3, dtype=torch.float64, device=DEV).index_add(
        0, sys_of_atom[c["ti"]], gr.double()[:, :, None] * c["r"].double()[:, None, :])
    assert rel(W, ref) < 1e-12
    n_edges_sys = np.bincount(np.searchsorted(ptr, ii, side="right") - 1, minlength=n_sys)
    assert (np.diff(ptr) == 0).any()
    for m in np.nonzero(n_edges_sys == 0)[0]:
        assert float(W[m].abs().max()) == 0.0
    if name in ("empty_runs", "single_edge"):
        assert ((np.diff(ptr) > 0) & (n_edges_sys == 0)).any()


@names
@topo
def test_scatter_add(name, order):
    """nn.scatter_add (spk_segment_sum over the receiver grouping)."""
    from schnetpack_b200 import nn as snn

    c = _case(name, order)
    ti, N, E, hubs = c["ti"], c["n"], c["E"], c["hubs"]
    torch.manual_seed(11)
    x = torch.randn(E, 7, device=DEV)
    (s,) = _run(c["det"], lambda: (snn.scatter_add(x, ti, N),))

    def ref(k):
        return torch.zeros(N, 7, dtype=torch.float64, device=DEV).index_add(0, ti[k], x[k].double())

    s_ref = ref(slice(None))
    s_abs = torch.zeros(N, 7, dtype=torch.float64, device=DEV).index_add(0, ti, x.double().abs())
    _check(s, s_ref, 2e-6, hubs, s_abs)
    if hubs:
        _sees_one_edge(s_ref, ref(_without(E, _hub_edge(c, "i", x.abs().max(1)[0]), DEV)), s_abs, hubs[0])
