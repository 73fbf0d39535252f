"""GPU: every SO3net kernel of csrc/so3net.cu on its own, against fp64 torch restatements of the reference operations
(so3net_oracle.py:88-97 with autograd), over all compiled variants: the convolution's filter weights in registers for
n_rbf <= 20 (NRB = 20) and for n_rbf <= 32 below lmax 3 (NRB = 32), read through L1 otherwise (NRB = 0), at lmax 0..3,
with partially active warps (F % 32 != 0); the per-atom tensor product, gate and l = 0 packing at lmax 0..3; the
shapes the kernels refuse; and whole SO3net models in configurations the golden fixtures do not cover."""
import math

import numpy as np
import pytest
import torch

from conftest import rel_err
from edge_oracle import rel, so3_conv_ref
import so3net_oracle as SO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RC = 5.0
LMAXES = [0, 1, 2, 3]
N_RBFS = [13, 20, 27, 32, 40]
FS = [4, 36, 128, 256]


def _variant(lmax, n_rbf):
    """The convolution template spk_so3_conv_{fwd,bwd} dispatches to (SO3_DISPATCH_L_NRB in csrc/so3net.cu)."""
    if n_rbf <= 20:
        return 20
    if n_rbf <= 32 and lmax < 3:
        return 32
    return 0


def _conv_cases():
    """lmax x n_rbf, each with one F of FS (every F appears at every lmax), on a molecule batch and a periodic box."""
    return [(lmax, n_rbf, FS[(lmax + k) % len(FS)], graph) for lmax in LMAXES for k, n_rbf in enumerate(N_RBFS)
            for graph in ("aspirin", "box")]


def test_conv_cases_reach_every_variant():
    seen = {(_variant(lmax, n_rbf), lmax) for lmax, n_rbf, _, _ in _conv_cases()}
    assert seen == {(20, l) for l in LMAXES} | {(32, l) for l in (0, 1, 2)} | {(0, l) for l in LMAXES}
    assert {F for lmax, _, F, _ in _conv_cases() if lmax == 3} == set(FS)
    assert {n_rbf for lmax, n_rbf, _, _ in _conv_cases() if _variant(lmax, n_rbf) == 0 and lmax == 3} == {27, 32, 40}


def _graph(kind):
    from schnetpack_b200 import ops
    from schnetpack_b200 import synthetic as S

    b = S.aspirin_batch(2, seed=1) if kind == "aspirin" else S.periodic_box(40, seed=3)
    R = torch.as_tensor(b["_positions"], device=DEV)
    ti, tj = torch.as_tensor(b["_idx_i"], device=DEV), torch.as_tensor(b["_idx_j"], device=DEV)
    r = (R[tj] - R[ti] + torch.as_tensor(b["_offsets"], device=DEV)).contiguous()
    N = b["_atomic_numbers"].shape[0]
    return ti, tj, r, N, ops.EdgeGraph(ti, tj, N)


@pytest.mark.parametrize("lmax,n_rbf,F,graph", _conv_cases())
def test_so3_conv(lmax, n_rbf, F, graph):
    """spk_so3_conv_fwd / _bwd: forward, dE/dx (with and without the residual g_res, or not wanted) and dE/dr_ij
    (written or accumulated)."""
    from schnetpack_b200 import ops

    ti, tj, r, N, g = _graph(graph)
    E = r.shape[0]
    S = (lmax + 1) ** 2
    torch.manual_seed(100 * lmax + n_rbf)
    p0 = torch.linspace(0, RC, n_rbf, device=DEV)
    p1 = torch.full((n_rbf,), float(p0[1] - p0[0]), device=DEV)
    phi, dphi, geo = ops.edge_geometry(r, g, ops.RBF_GAUSSIAN, n_rbf, p0, p1, RC, True)
    x = torch.randn(N, S, F, device=DEV)
    wf = torch.randn((lmax + 1) * F, n_rbf, device=DEV) * (1.0 / math.sqrt(n_rbf))
    bf = torch.randn((lmax + 1) * F, device=DEV) * 0.3
    g_y, g_res = torch.randn(N, S, F, device=DEV), torch.randn(N, S, F, device=DEV)

    def radial(d):
        return torch.exp(-0.5 / p1.double() ** 2 * (d - p0.double()) ** 2)

    x64, r64 = x.double().requires_grad_(), r.double().requires_grad_()
    y_ref = so3_conv_ref(x64, r64, ti, tj, wf.double(), bf.double(), lmax, RC, radial)
    y = ops.so3_conv_fwd(x, phi, geo, g, wf, bf, lmax, F, n_rbf)
    assert rel(y, y_ref) < 3e-6, rel(y, y_ref)
    gx_r, gr_r = torch.autograd.grad((y_ref * g_y.double()).sum(), [x64, r64])
    for res, acc, need_gx in ((g_res, False, True), (None, True, True), (g_res, True, False)):
        seed = torch.randn(E, 3, device=DEV) * float(gr_r.abs().max())
        g_rij = seed.clone() if acc else torch.full((E, 3), 7.0, device=DEV)
        g_x = ops.so3_conv_bwd(x, g_y, phi, dphi, geo, g, wf, bf, lmax, F, n_rbf, res, g_rij, acc, need_gx=need_gx)
        if need_gx:
            want = gx_r + (res.double() if res is not None else 0.0)
            assert rel(g_x, want) < 5e-6, rel(g_x, want)
        else:
            assert g_x is None
        want = gr_r + (seed.double() if acc else 0.0)
        assert rel(g_rij, want) < 1e-5, rel(g_rij, want)


# ------------------------------------------------------------------------------------------------ per-atom kernels
def _tp_ref(u, v, lmax):
    cg, i1, i2, io = (t.to(u.device) for t in SO.so3_tables(lmax))
    t = u[:, i1] * v[:, i2] * cg.to(u.dtype)[None, :, None]
    return u + torch.zeros_like(u).index_add(1, io, t)


@pytest.mark.parametrize("lmax", LMAXES)
@pytest.mark.parametrize("F", [4, 36, 256])
def test_so3_atom_kernels(lmax, F):
    """spk_so3_tp_{fwd,bwd} (dx + CG(dx, ddx)), spk_so3_gate_{fwd,bwd} (x * sigmoid(h[l(s)]), dE/dx row 0 returned
    apart), spk_so3_put_l0 and spk_so3_take_l0; N * F is not a multiple of the 256-thread block below F = 256."""
    from schnetpack_b200 import ops

    torch.manual_seed(7 * lmax + F)
    N, S = 37, (lmax + 1) ** 2
    assert F == 256 or (N * F) % 256 != 0
    lidx = torch.tensor([l for l in range(lmax + 1) for _ in range(2 * l + 1)], device=DEV)
    dx, ddx, g = (torch.randn(N, S, F, device=DEV) for _ in range(3))
    u64, v64 = dx.double().requires_grad_(), ddx.double().requires_grad_()
    tp_ref = _tp_ref(u64, v64, lmax)
    assert rel(ops.so3_tp_fwd(dx, ddx, lmax, F), tp_ref) < 2e-6
    gu_r, gv_r = torch.autograd.grad((tp_ref * g.double()).sum(), [u64, v64])
    g_dx, g_ddx = ops.so3_tp_bwd(g, dx, ddx, lmax, F)
    assert rel(g_dx, gu_r) < 2e-6 and rel(g_ddx, gv_r) < 2e-6
    # gate
    x = torch.randn(N, S, F, device=DEV)
    h = torch.randn(N, (lmax + 1) * F, device=DEV) * 2.0
    x64, h64 = x.double().requires_grad_(), h.double().requires_grad_()
    y_ref = x64 * torch.sigmoid(h64.view(N, lmax + 1, F)[:, lidx])
    assert rel(ops.so3_gate_fwd(x, h, lmax, F), y_ref) < 2e-6
    gx_r, gh_r = torch.autograd.grad((y_ref * g.double()).sum(), [x64, h64])
    g_x, g_x0, g_h = ops.so3_gate_bwd(g, x, h, lmax, F)
    assert rel(g_x0, gx_r[:, 0]) < 2e-6
    if lmax > 0:
        assert rel(g_x[:, 1:], gx_r[:, 1:]) < 2e-6
    assert rel(g_h, gh_r) < 2e-6
    # l = 0 packing
    src, v = torch.randn(N, S, F, device=DEV), torch.randn(N, F, device=DEV)
    for a, b in ((src, v), (None, v), (src, None)):
        want = (a.clone() if a is not None else torch.zeros(N, S, F, device=DEV))
        if b is not None:
            want[:, 0] += b
        assert torch.equal(ops.so3_put_l0(a, b, N, lmax, F, DEV), want)
    assert torch.equal(ops.so3_take_l0(src, lmax, F), src[:, 0])


@pytest.mark.parametrize("lmax,F", [(2, 30), (2, 260), (4, 32)])
def test_unsupported_shapes_raise(lmax, F):
    """Shapes outside so3_shape_ok (F a multiple of 4 up to 256, lmax <= 3) are refused before any launch."""
    from schnetpack_b200 import ops

    ti, tj, r, N, g = _graph("aspirin")
    n_rbf, S = 20, (lmax + 1) ** 2
    p0 = torch.linspace(0, RC, n_rbf, device=DEV)
    p1 = torch.full((n_rbf,), float(p0[1] - p0[0]), device=DEV)
    phi, dphi, geo = ops.edge_geometry(r, g, ops.RBF_GAUSSIAN, n_rbf, p0, p1, RC, True)
    x = torch.zeros(N, S, F, device=DEV)
    h = torch.zeros(N, (lmax + 1) * F, device=DEV)
    wf, bf = torch.zeros((lmax + 1) * F, n_rbf, device=DEV), torch.zeros((lmax + 1) * F, device=DEV)
    g_rij = torch.zeros(r.shape[0], 3, device=DEV)
    calls = [lambda: ops.so3_conv_fwd(x, phi, geo, g, wf, bf, lmax, F, n_rbf),
             lambda: ops.so3_conv_bwd(x, x, phi, dphi, geo, g, wf, bf, lmax, F, n_rbf, None, g_rij, False),
             lambda: ops.so3_tp_fwd(x, x, lmax, F), lambda: ops.so3_tp_bwd(x, x, x, lmax, F),
             lambda: ops.so3_gate_fwd(x, h, lmax, F), lambda: ops.so3_gate_bwd(x, x, h, lmax, F),
             lambda: ops.so3_put_l0(x, None, N, lmax, F, DEV), lambda: ops.so3_take_l0(x, lmax, F)]
    for call in calls:
        with pytest.raises(NotImplementedError, match="SPK_ERR_UNSUPPORTED"):
            call()
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("lmax,F,n_rbf,rbf", [(0, 36, 20, "gaussian"), (2, 64, 32, "gaussian"), (3, 32, 32, "gaussian"),
                                              (1, 64, 40, "bessel")])
def test_model_against_fp64_oracle(lmax, F, n_rbf, rbf):
    """from_spec SO3net (energy, forces, scalar and multipole representations) against so3net_oracle.energy_forces in
    fp64, on a molecule batch and a periodic box."""
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, from_spec

    spec = S.model_spec("so3net", n_atom_basis=F, n_interactions=2, lmax=lmax, n_rbf=n_rbf, rbf=rbf)
    params = S.init_params(spec, seed=60 + lmax)
    model = from_spec(spec, params, torch.device(DEV))
    for data in (S.aspirin_batch(3, seed=lmax), S.periodic_box(60, seed=lmax)):
        x = batch_to_device(data, torch.device(DEV))
        out = model(x)
        torch.cuda.synchronize()
        ref = SO.energy_forces(spec, params, data, dtype=torch.float64)
        for k, v in (("energy", out["energy"]), ("forces", out["forces"]),
                     ("scalar_representation", x["scalar_representation"]),
                     ("multipole_representation", x["multipole_representation"])):
            assert rel_err(v.detach().double().cpu().numpy(), ref[k].numpy()) < 1e-5, k
    assert np.isfinite(ref["energy"].numpy()).all()
