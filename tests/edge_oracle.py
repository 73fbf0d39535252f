"""fp64 restatements shared by the per-kernel GPU tests of the edge kernels (tests/test_cuda_kernels.py,
tests/test_cuda_edge_topology.py): the integer graph structure checked against numpy, and one PaiNN interaction
(painn.py:55-65 + :232-236) in plain torch."""
import math

import numpy as np
import torch


def rel(a, b):
    """max |a - b| / max |b| in fp64 (the suite's relative error)."""
    a = a.detach().double()
    b = b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _check_graph(g, ii, jj, n):
    ii = np.asarray(ii)
    jj = np.asarray(jj)
    E = ii.shape[0]
    rowptr = g.rowptr.cpu().numpy()
    sptr = g.sptr.cpu().numpy()
    slot_j = g.slot_j.cpu().numpy()[:E]
    slot_eid = g.slot_eid.cpu().numpy()[:E]
    pos_slot = g.pos_slot.cpu().numpy()[:E]
    pos_i = g.pos_i.cpu().numpy()[:E]
    # CSR: stable grouping by receiver
    order = np.argsort(ii, kind="stable")
    np.testing.assert_array_equal(rowptr, np.concatenate([[0], np.cumsum(np.bincount(ii, minlength=n))]))
    np.testing.assert_array_equal(slot_eid, order)
    np.testing.assert_array_equal(slot_j, jj[order])
    # sender grouping: stable by slot
    sj = jj[order]
    order2 = np.argsort(sj, kind="stable")
    np.testing.assert_array_equal(sptr, np.concatenate([[0], np.cumsum(np.bincount(jj, minlength=n))]))
    np.testing.assert_array_equal(pos_slot, order2)
    np.testing.assert_array_equal(pos_i, ii[order][order2])


def _painn_layer_ref(x, mu, q, r, ii, jj, wf, bf, rc, p0, p1):
    d = r.norm(dim=1, keepdim=True)
    u = r / d
    phi = torch.exp(-0.5 / p1 ** 2 * (d - p0) ** 2)
    fc = 0.5 * (torch.cos(d * math.pi / rc) + 1) * (d < rc)
    W = (phi @ wf.t() + bf) * fc
    F = q.shape[1]
    y = W * x[jj]
    dq, dmuR, dmumu = y.split(F, dim=-1)
    N = q.shape[0]
    qo = q + torch.zeros_like(q).index_add(0, ii, dq)
    dmu = dmuR[:, None, :] * u[:, :, None] + dmumu[:, None, :] * mu[jj]
    muo = mu + torch.zeros_like(mu).index_add(0, ii, dmu)
    return qo, muo


def so3_conv_ref(x, r, ii, jj, wf, bf, lmax, rc, radial, absolute=False):
    """SO3Convolution (so3net_oracle.py:88-90) in the dtype of ``x``: y[i] = sum over the edges (i <- j) of
    C[s1, s2, s] W[l(s1)](d) Y[s1](u) x[j, s2] with W = fc(d) (radial(d) wf^T + bf).  ``absolute``: every factor
    replaced by its magnitude, so that the sum is the sum of |terms| of each output."""
    from so3net_oracle import real_sph_harm, so3_tables

    cg, i1, i2, io = (t.to(x.device) for t in so3_tables(lmax))
    cg = cg.to(x.dtype)
    n, F = x.shape[0], x.shape[2]
    S = (lmax + 1) ** 2
    lidx = torch.tensor([l for l in range(lmax + 1) for _ in range(2 * l + 1)], device=x.device)
    d = r.norm(dim=1, keepdim=True)
    Y = real_sph_harm(r / d, lmax)
    fc = 0.5 * (torch.cos(d * math.pi / rc) + 1) * (d < rc)
    W = ((radial(d) @ wf.t() + bf) * fc).reshape(-1, lmax + 1, F)[:, lidx[i1]]
    if absolute:
        W, Y, cg = W.abs(), Y.abs(), cg.abs()
    v = W * Y[:, i1, None] * cg[None, :, None] * x[jj][:, i2]
    y_e = torch.zeros((r.shape[0], S, F), dtype=x.dtype, device=x.device).index_add(1, io, v)
    return torch.zeros((n, S, F), dtype=x.dtype, device=x.device).index_add(0, ii, y_e)
