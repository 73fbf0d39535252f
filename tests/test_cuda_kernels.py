"""GPU: per-kernel numerics -- every C-ABI entry point against a plain torch restatement of the same op on the same
seeded inputs (fp64 torch on the device as truth; tolerance 1e-5 relative unless stated), plus bit-exactness of the
integer graph structure against numpy."""
import math

import numpy as np
import pytest
import torch

from edge_oracle import _check_graph, _painn_layer_ref

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def rel(a, b):
    a = a.double()
    b = b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _graph_inputs(seed=0, batch=6):
    from schnetpack_b200 import synthetic as S

    b = S.aspirin_batch(batch, seed=seed)
    return b, torch.as_tensor(b["_idx_i"], device=DEV), torch.as_tensor(b["_idx_j"], device=DEV), b["_atomic_numbers"].shape[0]


def test_graph_build_sorted_and_unsorted_bit_exact():
    from schnetpack_b200 import ops

    b, ti, tj, n = _graph_inputs()
    g = ops.EdgeGraph(ti, tj, n)
    info = g.validate()
    assert info["sorted"]
    _check_graph(g, b["_idx_i"], b["_idx_j"], n)
    perm = np.random.default_rng(0).permutation(b["_idx_i"].shape[0])
    pi, pj = b["_idx_i"][perm], b["_idx_j"][perm]
    g2 = ops.EdgeGraph(torch.as_tensor(pi, device=DEV), torch.as_tensor(pj, device=DEV), n)
    assert not g2.validate()["sorted"]
    _check_graph(g2, pi, pj, n)
    # out-of-range index is reported, not dereferenced
    bad = torch.as_tensor(pi, device=DEV).clone()
    bad[5] = n + 3
    with pytest.raises(IndexError):
        ops.EdgeGraph(bad, torch.as_tensor(pj, device=DEV), n).validate()
    # no edges
    g3 = ops.EdgeGraph(torch.zeros(0, dtype=torch.int64, device=DEV), torch.zeros(0, dtype=torch.int64, device=DEV), 5)
    assert g3.rowptr.tolist() == [0] * 6 and g3.sptr.tolist() == [0] * 6


def test_graph_build_large_periodic():
    from schnetpack_b200 import ops
    from schnetpack_b200 import synthetic as S

    b = S.periodic_box(4096, seed=1)
    n = 4096
    g = ops.EdgeGraph(torch.as_tensor(b["_idx_i"], device=DEV), torch.as_tensor(b["_idx_j"], device=DEV), n)
    g.validate()
    _check_graph(g, b["_idx_i"], b["_idx_j"], n)


def test_segment_ptr():
    from schnetpack_b200 import ops

    idx_m = torch.tensor([0, 0, 0, 2, 2, 5], device=DEV)
    assert ops.segment_ptr(idx_m, 7).tolist() == [0, 3, 3, 5, 5, 5, 6, 6]


@pytest.mark.parametrize("kind", ["gaussian", "bessel"])
def test_edge_geometry_and_primitives(kind, primitives):
    from schnetpack_b200 import nn as snn
    from schnetpack_b200 import ops

    torch.manual_seed(0)
    E, n_rbf, rc = 4097, 20, 5.0
    r = torch.randn(E, 3, device=DEV) * 2.0
    r[0] = torch.tensor([rc, 0.0, 0.0])          # exactly at the cutoff -> fc == 0 exactly
    r[1] = torch.tensor([6.0, 1.0, 0.0])         # beyond
    if kind == "gaussian":
        mod = snn.GaussianRBF(n_rbf, rc).to(DEV)
    else:
        mod = snn.BesselRBF(n_rbf, rc).to(DEV)
    p0, p1 = mod.kernel_params()
    phi, dphi, geo = ops.edge_geometry(r, None, mod.kind, n_rbf, p0, p1, rc, True)
    r64 = r.double().requires_grad_()
    d = r64.norm(dim=1)
    if kind == "gaussian":
        ref = torch.exp(-0.5 / p1.double() ** 2 * (d[:, None] - p0.double()) ** 2)
    else:
        ref = torch.sin(d[:, None] * p0.double()) / d[:, None]
    fc = 0.5 * (torch.cos(d * math.pi / rc) + 1) * (d < rc)
    assert rel(phi[:, :n_rbf], ref) < 2e-6
    assert rel(geo[:, 3], d) < 1e-6 and rel(geo[:, :3], r64 / d[:, None]) < 1e-6
    assert (geo[:, 4] - fc).abs().max() < 2e-7 and geo[0, 4] == 0.0 and geo[1, 4] == 0.0
    dref = torch.stack([torch.autograd.grad(ref[:, k].sum(), r64, retain_graph=True)[0] for k in range(n_rbf)], 1)
    # d phi / d r = dphi * u
    got = dphi[:, :n_rbf, None].double() * geo[:, None, :3].double()
    assert rel(got, dref) < 5e-6
    dfc = torch.autograd.grad(fc.sum(), r64)[0]
    assert (geo[:, 5:6].double() * geo[:, :3].double() - dfc).abs().max() < 1e-6
    # module-level primitives against the reference's own known-answer vectors (tests/nn/test_radial.py etc.)
    z = primitives
    g6 = snn.GaussianRBF(n_rbf=6, cutoff=5.0).to(DEV)
    np.testing.assert_allclose(g6(torch.as_tensor(z["rbf1_in"], device=DEV)).cpu().numpy(), z["rbf1_ref"], rtol=2e-6)
    cut = snn.CosineCutoff(1.8).to(DEV)
    np.testing.assert_allclose(cut(torch.as_tensor(z["cut_in"], device=DEV)).cpu().numpy(), z["cut_ref"], rtol=1e-6,
                               atol=1e-7)
    np.testing.assert_allclose(cut(3.5 * torch.as_tensor(z["cut_in"], device=DEV)).cpu().numpy(), z["cut_ref35"],
                               rtol=1e-5, atol=2e-7)
    np.testing.assert_allclose(snn.shifted_softplus(torch.as_tensor(z["ssp_in"], device=DEV)).cpu().numpy(),
                               z["ssp_ref"], rtol=1e-6, atol=1e-7)
    bes = snn.BesselRBF(8, 5.0).to(DEV)
    np.testing.assert_allclose(bes(torch.as_tensor(z["bessel_in"], device=DEV)).cpu().numpy(), z["bessel_ref"],
                               rtol=1e-5, atol=2e-6)
    xs, idx = torch.as_tensor(z["scatter_in"], device=DEV), torch.as_tensor(z["scatter_idx"], device=DEV)
    np.testing.assert_allclose(snn.scatter_add(xs, idx, 5).cpu().numpy(), z["scatter_ref"])


@pytest.mark.parametrize("M,K,N", [(5376, 128, 384), (1000, 256, 128), (333, 20, 128), (77, 384, 128), (130, 64, 1),
                                    (4100, 128, 20)])
def test_dense(M, K, N):
    from schnetpack_b200 import ops

    torch.manual_seed(1)
    A = torch.randn(M, K, device=DEV)
    B = torch.randn(K, N, device=DEV) / math.sqrt(K)
    bias = torch.randn(N, device=DEV)
    add = torch.randn(M, N, device=DEV)
    pre_in = torch.randn(M, K, device=DEV)
    ref_lin = A.double() @ B.double() + bias.double()
    for act, f in ((ops.ACT_NONE, lambda v: v), (ops.ACT_SILU, torch.nn.functional.silu),
                   (ops.ACT_SSP, lambda v: torch.nn.functional.softplus(v) - math.log(2.0))):
        Y, pre = ops.dense(A, B, bias, act, addend=add, save_pre=True)
        assert rel(pre, ref_lin) < 2e-6
        assert rel(Y, f(ref_lin) + add.double()) < 2e-6
        # backward prologue: (A .* act'(pre_in)) @ B
        p64 = pre_in.double().requires_grad_()
        dact = torch.autograd.grad(f(p64).sum(), p64)[0]
        Y2 = ops.dense(A, B, a_pre=pre_in, a_act=act)
        assert rel(Y2, (A.double() * dact) @ B.double()) < 3e-6


@pytest.mark.parametrize("M,K,N,lda", [(5376, 128, 384, None), (1000, 256, 128, None), (333, 20, 128, 20),
                                        (4100, 128, 20, None), (16128, 128, 256, None), (130, 128, 64, None),
                                        (77, 384, 128, None), (2000, 20, 128, 24), (5, 64, 128, None)])
def test_dense_tcgen05_3xtf32(M, K, N, lda):
    """wgmma tensor-core layer with 3xTF32 compensation must be fp32-grade (the reference GEMMs are true fp32)."""
    from schnetpack_b200 import ops

    torch.manual_seed(3)
    lda = lda or K
    Afull = torch.randn(M, lda, device=DEV)
    A = Afull[:, :K]
    W = torch.randn(N, K, device=DEV) / math.sqrt(K)
    bias = torch.randn(N, device=DEV)
    add = torch.randn(M, N, device=DEV)
    pre_in = torch.randn(M, lda, device=DEV)
    w_hi, w_lo = ops.split_tf32(W)
    assert torch.equal(w_hi + w_lo, W) and int((w_hi.view(torch.int32) & 0x1FFF).abs().max()) == 0
    wp = ops.tc_pack_weight(W)
    ref_lin = A.double() @ W.double().t() + bias.double()
    for act, f in ((ops.ACT_NONE, lambda v: v), (ops.ACT_SILU, torch.nn.functional.silu),
                   (ops.ACT_SSP, lambda v: torch.nn.functional.softplus(v) - math.log(2.0))):
        Y, pre = ops.dense_tc(Afull, wp, N, bias, act, addend=add, save_pre=True, k=K)
        assert rel(pre, ref_lin) < 3e-6, rel(pre, ref_lin)
        assert rel(Y, f(ref_lin) + add.double()) < 3e-6
        p64 = pre_in[:, :K].double().requires_grad_()
        dact = torch.autograd.grad(f(p64).sum(), p64)[0]
        Y2 = ops.dense_tc(Afull, wp, N, a_pre=pre_in, a_act=act, k=K)
        assert rel(Y2, (A.double() * dact) @ W.double().t()) < 5e-6
    # padded output buffer (ldy > N)
    out = torch.full((M, N + 4), -1.0, device=DEV)
    ops.dense_tc(Afull, wp, N, bias, k=K, out=out)
    assert rel(out[:, :N], ref_lin) < 3e-6 and bool((out[:, N:] == -1.0).all())


@pytest.mark.parametrize("F,n_rbf,has_mu", [(128, 20, True), (128, 20, False), (64, 16, True), (256, 32, True)])
def test_painn_edge_fwd_bwd(F, n_rbf, has_mu):
    from schnetpack_b200 import ops

    b, ti, tj, N = _graph_inputs(seed=3, batch=5)
    g = ops.EdgeGraph(ti, tj, N)
    torch.manual_seed(2)
    rc = 5.0
    R = torch.as_tensor(b["_positions"], device=DEV)
    r = (R[tj] - R[ti]).contiguous()
    p0 = torch.linspace(0, rc, n_rbf, device=DEV)
    p1 = torch.full((n_rbf,), float(p0[1] - p0[0]), device=DEV)
    x = torch.randn(N, 3 * F, device=DEV)
    mu = torch.randn(N, 3, F, device=DEV) if has_mu else None
    q = torch.randn(N, F, device=DEV)
    wf = torch.randn(3 * F, n_rbf, device=DEV) * 0.3
    bf = torch.randn(3 * F, device=DEV) * 0.3
    phi, dphi, geo = ops.edge_geometry(r, g, ops.RBF_GAUSSIAN, n_rbf, p0, p1, rc, True)
    qo, muo = ops.painn_edge_fwd(x, mu, q, phi, geo, g, wf, bf, F, n_rbf)
    # fp64 reference + autograd
    x64, q64, r64 = x.double().requires_grad_(), q.double(), r.double().requires_grad_()
    mu64 = (mu.double() if has_mu else torch.zeros(N, 3, F, device=DEV, dtype=torch.float64)).requires_grad_()
    qr, mur = _painn_layer_ref(x64, mu64, q64, r64, ti, tj, wf.double(), bf.double(), rc, p0.double(), p1.double())
    assert rel(qo, qr) < 3e-6 and rel(muo, mur) < 3e-6
    g_q = torch.randn(N, F, device=DEV)
    g_mu = torch.randn(N, 3, F, device=DEV)
    gx_r, gmu_r, gr_r = torch.autograd.grad((qr * g_q.double()).sum() + (mur * g_mu.double()).sum(), [x64, mu64, r64])
    g_rij = torch.full((r.shape[0], 3), 7.0, device=DEV)
    g_x, g_mu_in = ops.painn_edge_bwd(x, mu, g_q, g_mu, phi, dphi, geo, g, wf, bf, F, n_rbf, g_rij, accumulate=False)
    if has_mu:
        assert rel(g_x, gx_r) < 5e-6
        assert rel(g_mu_in, gmu_r) < 5e-6
    else:
        assert rel(g_x[:, : 2 * F], gx_r[:, : 2 * F]) < 5e-6 and float(g_x[:, 2 * F:].abs().max()) == 0.0
    assert rel(g_rij, gr_r) < 1e-5
    # accumulate=True adds on top
    g_x2, _ = ops.painn_edge_bwd(x, mu, g_q, g_mu, phi, dphi, geo, g, wf, bf, F, n_rbf, g_rij, accumulate=True)
    assert rel(g_rij, 2 * gr_r) < 1e-5


def test_painn_mixing_glue():
    from schnetpack_b200 import ops

    torch.manual_seed(4)
    N, F, eps = 301, 128, 1e-8
    q = torch.randn(N, F, device=DEV)
    mu = torch.randn(N, 3, F, device=DEV)
    VW = torch.randn(N, 3, 2 * F, device=DEV)
    s = torch.randn(N, 3 * F, device=DEV)
    q64, mu64, VW64, s64 = [t.double().requires_grad_() for t in (q, mu, VW, s)]
    V, W = VW64.split(F, dim=-1)
    n = torch.sqrt((V ** 2).sum(1) + eps)
    ctx_ref = torch.cat([q64, n], -1)
    assert rel(ops.painn_mix_ctx(q, VW, F, eps), ctx_ref) < 1e-6
    s1, s2, s3 = s64.split(F, dim=-1)
    qo_ref = q64 + s1 + s3 * (V * W).sum(1)
    muo_ref = mu64 + s2[:, None, :] * W
    qo, muo = ops.painn_mix_update(q, mu, s, VW, F)
    assert rel(qo, qo_ref) < 1e-6 and rel(muo, muo_ref) < 1e-6
    g_q = torch.randn(N, F, device=DEV)
    g_mu = torch.randn(N, 3, F, device=DEV)
    gs_ref, gVW_ref = torch.autograd.grad((qo_ref * g_q.double()).sum() + (muo_ref * g_mu.double()).sum(), [s64, VW64],
                                          retain_graph=True)
    g_s, g_VW = ops.painn_mix_update_bwd(g_q, g_mu, s, VW, F)
    assert rel(g_s, gs_ref) < 2e-6 and rel(g_VW, gVW_ref) < 2e-6
    g_ctx = torch.randn(N, 2 * F, device=DEV)
    gq_ref, gVW2_ref = torch.autograd.grad((ctx_ref * g_ctx.double()).sum(), [q64, VW64])
    g_VW2 = g_VW.clone()
    g_q_out = ops.painn_mix_ctx_bwd(g_ctx, g_q, VW, g_VW2, F, eps)
    assert rel(g_q_out, g_q.double() + gq_ref) < 2e-6
    assert rel(g_VW2, gVW_ref + gVW2_ref) < 2e-6


def test_cfconv_and_radial_bwd():
    from schnetpack_b200 import ops

    b, ti, tj, N = _graph_inputs(seed=5, batch=4)
    g = ops.EdgeGraph(ti, tj, N)
    torch.manual_seed(6)
    F, n_rbf, rc = 128, 20, 5.0
    R = torch.as_tensor(b["_positions"], device=DEV)
    r = (R[tj] - R[ti]).contiguous()
    E = r.shape[0]
    p0 = torch.linspace(0, rc, n_rbf, device=DEV)
    p1 = torch.full((n_rbf,), float(p0[1] - p0[0]), device=DEV)
    phi, dphi, geo = ops.edge_geometry(r, g, ops.RBF_GAUSSIAN, n_rbf, p0, p1, rc, True)
    h = torch.randn(N, F, device=DEV)
    w_raw = torch.randn(E, F, device=DEV)
    m = ops.cfconv_fwd(h, w_raw, geo, g, F)
    h64, w64 = h.double().requires_grad_(), w_raw.double().requires_grad_()
    fc64 = geo[:, 4].double().requires_grad_()
    m_ref = torch.zeros(N, F, device=DEV, dtype=torch.float64).index_add(0, ti, h64[tj] * w64 * fc64[:, None])
    assert rel(m, m_ref) < 2e-6
    g_m = torch.randn(N, F, device=DEV)
    gh_r, gw_r, gfc_r = torch.autograd.grad((m_ref * g_m.double()).sum(), [h64, w64, fc64])
    g_h, g_wraw, g_fc = ops.cfconv_bwd(h, w_raw, geo, g_m, g, F)
    assert rel(g_h, gh_r) < 3e-6 and rel(g_wraw, gw_r) < 3e-6 and rel(g_fc, gfc_r) < 3e-6
    # radial_bwd: chain through phi(d) and fc(d)
    g_phi = torch.randn(E, ops.kp(n_rbf), device=DEV)
    r64 = r.double().requires_grad_()
    d = r64.norm(dim=1)
    phi_ref = torch.exp(-0.5 / p1.double() ** 2 * (d[:, None] - p0.double()) ** 2)
    fc_ref = 0.5 * (torch.cos(d * math.pi / rc) + 1) * (d < rc)
    gr_ref = torch.autograd.grad((phi_ref * g_phi[:, :n_rbf].double()).sum() + (fc_ref * g_fc.double()).sum(), r64)[0]
    g_rij = torch.zeros(E, 3, device=DEV)
    ops.radial_bwd(g_phi, g_fc, dphi, geo, g, n_rbf, g_rij, accumulate=False)
    assert rel(g_rij, gr_ref) < 1e-5


def test_atomwise_and_pairwise():
    from schnetpack_b200 import ops

    torch.manual_seed(8)
    b, ti, tj, N = _graph_inputs(seed=7, batch=5)
    g = ops.EdgeGraph(ti, tj, N)
    H = 64
    hid = torch.randn(N, H, device=DEV)
    w1 = torch.randn(H, device=DEV)
    b1 = torch.randn(1, device=DEV)
    idx_m = torch.as_tensor(b["_idx_m"], device=DEV)
    mol_ptr = ops.segment_ptr(idx_m, 5)
    y, e = ops.atomwise_out(hid, w1, b1, mol_ptr, 5)
    y_ref = hid.double() @ w1.double() + b1.double()
    e_ref = torch.zeros(5, device=DEV, dtype=torch.float64).index_add(0, idx_m, y_ref)
    assert rel(y, y_ref) < 2e-6 and rel(e, e_ref) < 2e-6
    g_e = torch.randn(5, device=DEV)
    g_hid = ops.atomwise_out_bwd(g_e, idx_m, w1, N, H)
    assert rel(g_hid, g_e[idx_m][:, None].double() * w1[None].double()) < 1e-6
    R = torch.as_tensor(b["_positions"], device=DEV)
    off = torch.randn(ti.shape[0], 3, device=DEV)
    rij = ops.pairwise_fwd(R, ti, tj, off)
    assert torch.equal(rij, R[tj] - R[ti] + off)
    gr = torch.randn(ti.shape[0], 3, device=DEV)
    gR = ops.pairwise_bwd(gr, g, 1.0)
    ref = torch.zeros(N, 3, device=DEV, dtype=torch.float64).index_add(0, tj, gr.double()).index_add(0, ti, -gr.double())
    assert rel(gR, ref) < 2e-6


@pytest.mark.parametrize("impl", ["tc", "ffma"])
def test_lin_saved_derivative_backward(impl):
    """Lin.fwd(save_deriv=True) stores act'(pre) (SPK_SAVE_DERIV); Lin.bwd(a_act=ACT_GIVEN) multiplies by it: together they
    are the input gradient of act(x W^T + b)."""
    from schnetpack_b200 import ops

    old = ops.DENSE_IMPL
    ops.DENSE_IMPL = impl
    try:
        torch.manual_seed(5)
        M, K, N = 700, 128, 256
        X = torch.randn(M, K, device=DEV)
        W = torch.randn(N, K, device=DEV) / math.sqrt(K)
        b = torch.randn(N, device=DEV)
        G = torch.randn(M, N, device=DEV)
        lin = ops.Lin(W, b)
        for act, f in ((ops.ACT_SILU, torch.nn.functional.silu),
                       (ops.ACT_SSP, lambda v: torch.nn.functional.softplus(v) - math.log(2.0))):
            Y, d = lin.fwd(X, act, save_deriv=True)
            x64 = X.double().requires_grad_()
            pre = x64 @ W.double().t() + b.double()
            y64 = f(pre)
            assert rel(Y, y64) < 3e-6
            dref = torch.autograd.grad(y64.sum(), pre, retain_graph=True)[0]
            assert rel(d, dref) < 3e-6
            gx_ref = torch.autograd.grad((y64 * G.double()).sum(), x64)[0]
            gx = lin.bwd(G, a_pre=d, a_act=ops.ACT_GIVEN)
            assert rel(gx, gx_ref) < 5e-6
    finally:
        ops.DENSE_IMPL = old


@pytest.mark.parametrize("gen,n_rbf", [("aspirin", 20), ("qm9like", 20), ("aspirin", 13), ("periodic", 20)])
def test_painn_edge_tensor_core_filter_matches_streaming(gen, n_rbf):
    """csrc/painn_tc.cu (filter on wgmma) == csrc/painn.cu (filter on the CUDA cores) to fp32 rounding,
    forward and reverse, with and without mu, on ragged row lengths, tail chunks and an n_rbf that is not a multiple of 4."""
    from schnetpack_b200 import ops
    from schnetpack_b200 import synthetic as S

    if gen == "aspirin":
        b = S.aspirin_batch(37, seed=21)
    elif gen == "qm9like":
        b = S.qm9like_batch(64, seed=22)
    else:
        b = S.periodic_box(600, seed=23)
    ti, tj = torch.as_tensor(b["_idx_i"], device=DEV), torch.as_tensor(b["_idx_j"], device=DEV)
    N = b["_atomic_numbers"].shape[0]
    g = ops.EdgeGraph(ti, tj, N)
    torch.manual_seed(31)
    F, rc = 128, 5.0
    R = torch.as_tensor(b["_positions"], device=DEV)
    off = torch.as_tensor(b["_offsets"], device=DEV) if "_offsets" in b else 0.0
    r = (R[tj] - R[ti] + off).contiguous()
    p0 = torch.linspace(0, rc, n_rbf, device=DEV)
    p1 = torch.full((n_rbf,), float(p0[1] - p0[0]), device=DEV)
    phi, dphi, geo = ops.edge_geometry(r, g, ops.RBF_GAUSSIAN, n_rbf, p0, p1, rc, True)
    x = torch.randn(N, 3 * F, device=DEV)
    q = torch.randn(N, F, device=DEV)
    wf = torch.randn(3 * F, n_rbf, device=DEV) * 0.3
    bf = torch.randn(3 * F, device=DEV) * 0.3
    g_q = torch.randn(N, F, device=DEV)
    g_mu = torch.randn(N, 3, F, device=DEV)
    E = ti.shape[0]
    wpk = ops.painn_pack_filter(wf, bf, F, n_rbf)
    saved = ops.EDGE_IMPL, ops.EDGE_TC_MIN_EDGES
    try:
        for mu in (torch.randn(N, 3, F, device=DEV), None):
            ops.EDGE_IMPL = "ldg"
            q_ref, mu_ref = ops.painn_edge_fwd(x, mu, q, phi, geo, g, wf, bf, F, n_rbf)
            ops.EDGE_IMPL, ops.EDGE_TC_MIN_EDGES = "tc", 1
            q_tc, mu_tc = ops.painn_edge_fwd(x, mu, q, phi, geo, g, wf, bf, F, n_rbf, wf_packed=wpk)
            torch.cuda.synchronize()
            assert rel(q_tc, q_ref.double()) < 2e-6, (gen, mu is None, rel(q_tc, q_ref.double()))
            assert rel(mu_tc, mu_ref.double()) < 2e-6, (gen, mu is None, rel(mu_tc, mu_ref.double()))
            for acc in (False, True):
                seed = torch.randn(E, 3, device=DEV)
                ops.EDGE_IMPL = "ldg"
                gr_ref = seed.clone()
                gx_ref, gm_ref = ops.painn_edge_bwd(x, mu, g_q, g_mu, phi, dphi, geo, g, wf, bf, F, n_rbf, gr_ref, acc)
                ops.EDGE_IMPL = "tc"
                gr_tc = seed.clone()
                gx_tc, gm_tc = ops.painn_edge_bwd(x, mu, g_q, g_mu, phi, dphi, geo, g, wf, bf, F, n_rbf, gr_tc, acc,
                                                  wf_packed=wpk)
                torch.cuda.synchronize()
                assert rel(gx_tc, gx_ref.double()) < 2e-6, (gen, mu is None, acc, rel(gx_tc, gx_ref.double()))
                assert rel(gr_tc, gr_ref.double()) < 3e-6, (gen, mu is None, acc, rel(gr_tc, gr_ref.double()))
                if mu is not None:
                    assert rel(gm_tc, gm_ref.double()) < 2e-6, (gen, acc, rel(gm_tc, gm_ref.double()))
    finally:
        ops.EDGE_IMPL, ops.EDGE_TC_MIN_EDGES = saved


@pytest.mark.parametrize("has_mu", [True, False])
def test_painn_edge_tc_kernels_vs_fp64_restatement(has_mu):
    """Tensor-core edge kernels (forward and reverse) held DIRECTLY against a torch fp64 restatement of painn.py:55-65 +
    :232-236 with autograd (not only against the streaming kernels), on a graph large enough for every persistent CTA to
    own several chunks (aspirin x 40: 12 k edges) and on a periodic box."""
    from schnetpack_b200 import ops
    from schnetpack_b200 import synthetic as S

    saved = ops.EDGE_IMPL, ops.EDGE_TC_MIN_EDGES
    ops.EDGE_IMPL, ops.EDGE_TC_MIN_EDGES = "tc", 1
    try:
        for b in (S.aspirin_batch(40, seed=5), S.periodic_box(700, seed=6)):
            ti, tj = torch.as_tensor(b["_idx_i"], device=DEV), torch.as_tensor(b["_idx_j"], device=DEV)
            N = b["_atomic_numbers"].shape[0]
            g = ops.EdgeGraph(ti, tj, N)
            torch.manual_seed(41)
            F, n_rbf, rc = 128, 20, 5.0
            R = torch.as_tensor(b["_positions"], device=DEV)
            r = (R[tj] - R[ti] + torch.as_tensor(b["_offsets"], device=DEV)).contiguous()
            p0 = torch.linspace(0, rc, n_rbf, device=DEV)
            p1 = torch.full((n_rbf,), float(p0[1] - p0[0]), device=DEV)
            x = torch.randn(N, 3 * F, device=DEV)
            mu = torch.randn(N, 3, F, device=DEV) if has_mu else None
            q = torch.randn(N, F, device=DEV)
            wf = torch.randn(3 * F, n_rbf, device=DEV) * 0.3
            bf = torch.randn(3 * F, device=DEV) * 0.3
            wpk = ops.painn_pack_filter(wf, bf, F, n_rbf)
            assert ops.edge_tc_ok(F, n_rbf, g.n_edges)
            phi, dphi, geo = ops.edge_geometry(r, g, ops.RBF_GAUSSIAN, n_rbf, p0, p1, rc, True)
            qo, muo = ops.painn_edge_fwd(x, mu, q, phi, geo, g, wf, bf, F, n_rbf, wf_packed=wpk)
            x64, q64, r64 = x.double().requires_grad_(), q.double(), r.double().requires_grad_()
            mu64 = (mu.double() if has_mu else torch.zeros(N, 3, F, device=DEV, dtype=torch.float64)).requires_grad_()
            qr, mur = _painn_layer_ref(x64, mu64, q64, r64, ti, tj, wf.double(), bf.double(), rc, p0.double(), p1.double())
            assert rel(qo, qr) < 3e-6 and rel(muo, mur) < 3e-6
            g_q = torch.randn(N, F, device=DEV)
            g_mu = torch.randn(N, 3, F, device=DEV)
            gx_r, gmu_r, gr_r = torch.autograd.grad((qr * g_q.double()).sum() + (mur * g_mu.double()).sum(),
                                                    [x64, mu64, r64])
            g_rij = torch.zeros((r.shape[0], 3), device=DEV)
            g_x, g_mu_in = ops.painn_edge_bwd(x, mu, g_q, g_mu, phi, dphi, geo, g, wf, bf, F, n_rbf, g_rij, False,
                                              wf_packed=wpk)
            if has_mu:
                assert rel(g_x, gx_r) < 5e-6 and rel(g_mu_in, gmu_r + g_mu.double() * 0) < 5e-6
            else:
                assert rel(g_x[:, : 2 * F], gx_r[:, : 2 * F]) < 5e-6
            assert rel(g_rij, gr_r) < 1e-5
    finally:
        ops.EDGE_IMPL, ops.EDGE_TC_MIN_EDGES = saved


def test_painn_edge_wij_block_kernels():
    """spk_painn_edge_wij_{fwd,bwd} (materialised filter, block-level API) vs a torch fp64 restatement of painn.py:55-65 with
    autograd, on an UNSORTED edge list (Wij / dir_ij stay in the caller's order)."""
    from schnetpack_b200 import ops
    from schnetpack_b200 import synthetic as S

    b = S.aspirin_batch(6, seed=8)
    rng = np.random.default_rng(3)
    perm = rng.permutation(b["_idx_i"].shape[0])
    ti = torch.as_tensor(b["_idx_i"][perm], device=DEV)
    tj = torch.as_tensor(b["_idx_j"][perm], device=DEV)
    N, E, F = b["_atomic_numbers"].shape[0], perm.shape[0], 64
    g = ops.EdgeGraph(ti, tj, N)
    torch.manual_seed(5)
    x, mu, q = torch.randn(N, 3 * F, device=DEV), torch.randn(N, 3, F, device=DEV), torch.randn(N, F, device=DEV)
    W, u = torch.randn(E, 3 * F, device=DEV), torch.randn(E, 3, device=DEV)
    qo, muo = ops.painn_edge_wij_fwd(x, mu, q, W, u, g, F)
    x64, mu64, W64, u64 = (t.double().requires_grad_() for t in (x, mu, W, u))
    y = W64 * x64[tj]
    dq, dmuR, dmumu = y.split(F, dim=-1)
    qr = q.double() + torch.zeros(N, F, device=DEV, dtype=torch.float64).index_add(0, ti, dq)
    dmu = dmuR[:, None, :] * u64[:, :, None] + dmumu[:, None, :] * mu64[tj]
    mur = mu64 + torch.zeros(N, 3, F, device=DEV, dtype=torch.float64).index_add(0, ti, dmu)
    assert rel(qo, qr) < 2e-6 and rel(muo, mur) < 2e-6
    g_q, g_mu = torch.randn(N, F, device=DEV), torch.randn(N, 3, F, device=DEV)
    gx_r, gmu_r, gW_r, gu_r = torch.autograd.grad((qr * g_q.double()).sum() + (mur * g_mu.double()).sum(),
                                                  [x64, mu64, W64, u64])
    g_x, g_mu_in, g_W, g_u = ops.painn_edge_wij_bwd(x, mu, g_q, g_mu, W, u, g, F)
    assert rel(g_x, gx_r) < 3e-6 and rel(g_mu_in, gmu_r) < 3e-6 and rel(g_W, gW_r) < 3e-6 and rel(g_u, gu_r) < 5e-6


def test_bad_neighbor_indices_raise_and_never_gather_out_of_bounds():
    """Reference: index_select raises IndexError on a bad index.  Here the first build of a new list raises on the host, and
    the kernels -- which cannot raise -- treat the list as an EMPTY graph (row pointers zeroed) and poison the distances of
    the bad edges with NaN instead of reading out of bounds."""
    from schnetpack_b200 import ops

    b, ti, tj, N = _graph_inputs(seed=1, batch=2)
    bad_j = tj.clone()
    bad_j[5] = N + 1000
    with pytest.raises(IndexError):
        ops.EdgeGraph(ti, bad_j, N)
    old = ops.VALIDATE_INDICES
    ops.VALIDATE_INDICES = False
    try:
        g = ops.EdgeGraph(ti, bad_j, N)
        assert int(g.status[1]) == 1
        assert int(g.rowptr.abs().max()) == 0 and int(g.sptr.abs().max()) == 0
        R = torch.as_tensor(b["_positions"], device=DEV)
        rij = ops.pairwise_fwd(R, ti, bad_j, None)
        assert bool(torch.isnan(rij[5]).all()) and not bool(torch.isnan(rij[:5]).any())
    finally:
        ops.VALIDATE_INDICES = old
    Z = torch.tensor([1, 6, 250, -1], device=DEV)
    out = ops.embedding(torch.randn(100, 32, device=DEV), Z)
    assert not bool(torch.isnan(out[:2]).any()) and bool(torch.isnan(out[2:]).all())


@pytest.mark.parametrize("case", ["qm9", "qm9_padded", "box", "bessel18"])
def test_schnet_fused_forward_block_vs_fp64(case):
    """csrc/schnet_tc.cu (filter network on wgmma inside the edge kernel, CSR over the active edges only) against a torch
    fp64 restatement of schnet.py:56-67 for one block, incl. a padded neighbour list (padding slots at d == cutoff are
    dropped by spk_graph_build_active), a periodic box, and n_rbf % 4 != 0 with the Bessel basis."""
    from schnetpack_b200 import ops
    from schnetpack_b200 import synthetic as S

    torch.manual_seed(9)
    F, rc = 128, 5.0
    n_rbf = 18 if case == "bessel18" else 20
    if case == "box":
        b = S.periodic_box(500, seed=4)
    else:
        b = S.qm9like_batch(48, seed=5, padded=(case == "qm9_padded"))
    ti, tj = torch.as_tensor(b["_idx_i"], device=DEV), torch.as_tensor(b["_idx_j"], device=DEV)
    N = b["_atomic_numbers"].shape[0]
    if "_Rij" in b:
        r = torch.as_tensor(b["_Rij"], device=DEV)
    else:
        R = torch.as_tensor(b["_positions"], device=DEV)
        r = (R[tj] - R[ti] + torch.as_tensor(b["_offsets"], device=DEV)).contiguous()
    if case == "bessel18":
        kind, p0, p1 = ops.RBF_BESSEL, (torch.arange(1, n_rbf + 1, device=DEV) * math.pi / rc).float(), None
    else:
        kind, p0 = ops.RBF_GAUSSIAN, torch.linspace(0, rc, n_rbf, device=DEV)
        p1 = torch.full((n_rbf,), float(p0[1] - p0[0]), device=DEV)
    g = ops.EdgeGraph(ti, tj, N, r_ij=r, cutoff=rc)
    d64 = r.double().norm(dim=1)
    n_act = int(g.rowptr[-1])
    assert n_act == int((r.norm(dim=1) < rc).sum()) and (case != "qm9_padded" or n_act < ti.shape[0])
    phi, _, geo = ops.edge_geometry(r, g, kind, n_rbf, p0, p1, rc, False, active_only=True)
    w0, b0 = torch.randn(F, n_rbf, device=DEV) * 0.3, torch.randn(F, device=DEV) * 0.3
    w1, b1 = torch.randn(F, F, device=DEV) * 0.1, torch.randn(F, device=DEV) * 0.1
    h = torch.randn(N, F, device=DEV)
    m = ops.schnet_cfconv_fwd_tc(h, phi, geo, g, ops.schnet_pack_filter(w0, b0, w1, n_rbf), b1, ops.ACT_SSP, n_rbf)
    if kind == ops.RBF_GAUSSIAN:
        f = torch.exp(-0.5 / p1.double() ** 2 * (d64[:, None] - p0.double()) ** 2)
    else:
        f = torch.sin(d64[:, None] * p0.double()) / d64[:, None]
    fc = 0.5 * (torch.cos(d64 * math.pi / rc) + 1) * (d64 < rc)
    hid = torch.nn.functional.softplus(f @ w0.double().t() + b0.double()) - math.log(2.0)
    W = (hid @ w1.double().t() + b1.double()) * fc[:, None]
    ref = torch.zeros(N, F, device=DEV, dtype=torch.float64).index_add(0, ti, h.double()[tj] * W)
    assert rel(m, ref) < 3e-6, rel(m, ref)
