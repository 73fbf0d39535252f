"""Kernel pipelines of the hot path (forward and reverse sweeps) and their ``torch.autograd.Function`` wrappers.

The pipelines call only the C-ABI kernels of ``ops``; autograd is used as plumbing so that the reference's own
``Forces`` logic (``torch.autograd.grad(E, R)``, /root/reference/src/schnetpack/atomistic/response.py:59-76) works
unchanged on top of them.  First-order gradients w.r.t. ``_Rij`` / ``_positions`` (forces, stress through
``_offsets``) are implemented; weight gradients / double backward (training, SURVEY.md §8 f3) are not -- the modules
refuse to run in training mode instead of silently returning wrong gradients.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import ops
from .ops import ACT_NONE, ACT_SILU, ACT_SSP

Tensor = torch.Tensor


def _c(t: Tensor) -> Tensor:
    return t.detach().contiguous()


def _ct(t: Tensor) -> Tensor:
    return t.detach().t().contiguous()


class ParamPack:
    """Device-resident, kernel-ready copies of a module's weights (W and W^T), rebuilt when any parameter changes."""

    def __init__(self):
        self._sig = None

    @staticmethod
    def signature(tensors: List[Tensor]):
        return tuple((t.data_ptr(), t._version, t.device, t.dtype) for t in tensors)

    def stale(self, tensors: List[Tensor]) -> bool:
        return self._sig != self.signature(tensors)

    def mark(self, tensors: List[Tensor]):
        self._sig = self.signature(tensors)


ACT_CODES = {"silu": ACT_SILU, "ssp": ACT_SSP, None: ACT_NONE, "none": ACT_NONE}


# =====================================================================================================================
# PaiNN  (representation/painn.py:207-256)
# =====================================================================================================================
class PaiNNPack(ParamPack):
    def build(self, mod):
        F, T = mod.n_atom_basis, mod.n_interactions
        self.F, self.T = F, T
        self.eps = float(mod.mixing[0].epsilon)
        fw, fb = _c(mod.filter_net.weight), _c(mod.filter_net.bias)
        self.wf, self.bf = [], []
        for t in range(T):
            if mod.share_filters:
                self.wf.append(fw)
                self.bf.append(fb)
            else:
                self.wf.append(fw[t * 3 * F:(t + 1) * 3 * F].contiguous())
                self.bf.append(fb[t * 3 * F:(t + 1) * 3 * F].contiguous())
        self.wfp = [None] * T                                  # tensor-core operand tiles of (wf, bf), built on first use
        self.blocks = []
        for t in range(T):
            it, mx = mod.interactions[t], mod.mixing[t]
            c0, c1 = it.interatomic_context_net[0], it.interatomic_context_net[1]
            m0, m1 = mx.intraatomic_context_net[0], mx.intraatomic_context_net[1]
            self.blocks.append(dict(
                c0=ops.Lin(c0.weight, c0.bias), c1=ops.Lin(c1.weight, c1.bias),
                mix=ops.Lin(mx.mu_channel_mix.weight), m0=ops.Lin(m0.weight, m0.bias), m1=ops.Lin(m1.weight, m1.bias),
            ))


def _packed_filter(pk: "PaiNNPack", t: int, n_rbf: int, n_edges: int):
    if not ops.edge_tc_ok(pk.F, n_rbf, n_edges):
        return None
    if pk.wfp[t] is None:
        pk.wfp[t] = ops.painn_pack_filter(pk.wf[t], pk.bf[t], pk.F, n_rbf)
    return pk.wfp[t]


# ---- per-block pipelines (pure functions over detached fp32 CUDA tensors) -------------------------------------------
def painn_context_fwd(b, q: Tensor, act: int):
    """x = interatomic_context_net(q) [N,3F] (painn.py:54) and the saved act'(pre) of its first layer."""
    a, hpre = b["c0"].fwd(q, act, save_deriv=True)
    return b["c1"].fwd(a), hpre


def painn_context_bwd(b, g_x: Tensor, hpre: Tensor, addend: Optional[Tensor] = None) -> Tensor:
    """dE/dq through the context net (+ ``addend``, the residual stream's gradient)."""
    g_a = b["c1"].bwd(g_x)                                                                   # [N,3F]x[3F,F]
    return b["c0"].bwd(g_a, a_pre=hpre, a_act=ops.ACT_GIVEN, addend=addend)                  # [N,F]x[F,F]


def painn_mixing_fwd(b, q1: Tensor, mu1: Tensor, F: int, eps: float, act: int):
    """PaiNNMixing.forward (painn.py:103-116): returns q2, mu2 and the tape (VW, act'(cpre), s)."""
    N = q1.shape[0]
    VW = b["mix"].fwd(mu1.view(3 * N, F))                                                    # :103  [3N,2F]
    ctx = ops.painn_mix_ctx(q1, VW, F, eps)                                                  # :104-107
    c, cpre = b["m0"].fwd(ctx, act, save_deriv=True)                                         # :108
    s = b["m1"].fwd(c)
    q2, mu2 = ops.painn_mix_update(q1, mu1, s, VW, F)                                        # :110-116
    return q2, mu2, (VW, cpre, s)


def painn_mixing_bwd(b, g_q: Tensor, g_mu: Tensor, tape, F: int, eps: float):
    """(dE/dq2, dE/dmu2) -> (dE/dq1, dE/dmu1)."""
    VW, cpre, s = tape
    N = g_q.shape[0]
    g_s, g_VW = ops.painn_mix_update_bwd(g_q, g_mu, s, VW, F)
    g_c = b["m1"].bwd(g_s)                                                                   # [N,3F]x[3F,F]
    g_ctx = b["m0"].bwd(g_c, a_pre=cpre, a_act=ops.ACT_GIVEN)                                # [N,F]x[F,2F]
    g_q1 = ops.painn_mix_ctx_bwd(g_ctx, g_q, VW, g_VW, F, eps)
    g_mu1 = b["mix"].bwd(g_VW.view(3 * N, 2 * F), addend=g_mu.view(3 * N, F)).view(N, 3, F)
    return g_q1, g_mu1


def painn_forward(pk: PaiNNPack, q0: Tensor, r_ij: Tensor, graph: ops.EdgeGraph, rbf_kind: int, n_rbf: int,
                  rbf_p0: Tensor, rbf_p1: Optional[Tensor], cutoff: float, act: int, need_grad: bool):
    """Returns q [N,F], mu [N,3,F] and the tape needed by painn_backward."""
    F = pk.F
    phi, dphi, geo = ops.edge_geometry(r_ij, graph, rbf_kind, n_rbf, rbf_p0, rbf_p1, cutoff, need_grad)
    q, mu = q0, None
    tape = []
    for t in range(pk.T):
        b = pk.blocks[t]
        x, hpre = painn_context_fwd(b, q, act)                                               # painn.py:54
        q1, mu1 = ops.painn_edge_fwd(x, mu, q, phi, geo, graph, pk.wf[t], pk.bf[t], F, n_rbf,   # :55-65
                                     wf_packed=_packed_filter(pk, t, n_rbf, graph.n_edges))
        q2, mu2, mtape = painn_mixing_fwd(b, q1, mu1, F, pk.eps, act)                        # :103-116
        if need_grad:
            tape.append((hpre, x, mu, mtape))
        q, mu = q2, mu2
    return q, mu, (phi, dphi, geo, tape)


def painn_backward(pk: PaiNNPack, saved, graph: ops.EdgeGraph, n_rbf: int, act: int, g_q: Tensor,
                   g_mu: Optional[Tensor], n_edges_total: int) -> Tensor:
    """dE/dr_ij [E,3] (in the caller's edge order) from dE/dq [N,F], dE/dmu [N,3,F]."""
    F = pk.F
    phi, dphi, geo, tape = saved
    N = g_q.shape[0]
    dev = g_q.device
    g_rij = torch.empty((n_edges_total, 3), dtype=torch.float32, device=dev)
    if g_mu is None:
        g_mu = torch.zeros((N, 3, F), dtype=torch.float32, device=dev)
    for t in reversed(range(pk.T)):
        b = pk.blocks[t]
        hpre, x, mu_in, mtape = tape[t]
        g_q1, g_mu1 = painn_mixing_bwd(b, g_q, g_mu, mtape, F, pk.eps)                       # painn.py:103-116 reversed
        g_x, g_mu0 = ops.painn_edge_bwd(x, mu_in, g_q1, g_mu1, phi, dphi, geo, graph, pk.wf[t], pk.bf[t], F, n_rbf,
                                        g_rij, accumulate=(t != pk.T - 1),                   # :54-65 reversed
                                        wf_packed=_packed_filter(pk, t, n_rbf, graph.n_edges))
        if t == 0:
            break   # dE/dq0 would only reach the (position-independent) embedding: the first context net is not reversed
        g_q = painn_context_bwd(b, g_x, hpre, addend=g_q1)
        g_mu = g_mu0
    return g_rij


class PaiNNFunction(torch.autograd.Function):
    """(q0 [N,F], r_ij [E,3]) -> (q, mu); backward gives dE/dr_ij (q0 = embedding output is treated as constant)."""

    @staticmethod
    def forward(ctx, r_ij, q0, holder):
        mod, graph = holder["module"], holder["graph"]
        pk = mod._pack()
        need = r_ij.requires_grad
        with ops.device_of(r_ij, q0):
            q, mu, saved = painn_forward(pk, q0, r_ij.detach(), graph, mod._rbf_kind, mod._n_rbf, mod._rbf_p0,
                                         mod._rbf_p1, mod._cutoff_value, mod._act, need)
        ctx.holder = dict(pk=pk, saved=saved, graph=graph, n_rbf=mod._n_rbf, act=mod._act, E=r_ij.shape[0])
        ctx.set_materialize_grads(False)
        return q, mu

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_q, g_mu):
        h = ctx.holder
        some = g_q if g_q is not None else g_mu
        with ops.device_of(some):
            g_q = g_q.contiguous() if g_q is not None else None
            if g_q is None:
                g_q = torch.zeros((h["graph"].n_atoms, h["pk"].F), dtype=torch.float32, device=g_mu.device)
            g_mu = g_mu.contiguous() if g_mu is not None else None
            g_rij = painn_backward(h["pk"], h["saved"], h["graph"], h["n_rbf"], h["act"], g_q, g_mu, h["E"])
        return g_rij, None, None


# ---- block-level autograd functions ---------------------------------------------------------------------------------
# The same kernels, exposed per block: the reference's block API (PaiNNInteraction.forward / PaiNNMixing.forward,
# painn.py:31-67,92-117) and the spatially decomposed evaluation of ONE large system (parallel.py: a halo exchange of ghost
# rows sits between the context net and the edge kernel of every block) are compositions of these.
class EdgeGeometry:
    """Per-evaluation radial basis / cutoff / unit-vector records of an edge list (shared by all interaction blocks)."""

    def __init__(self, mod, r_ij: Tensor, graph: ops.EdgeGraph, need_grad: bool = True):
        self.graph, self.n_rbf, self.E = graph, mod._n_rbf, r_ij.shape[0]
        with ops.device_of(r_ij):
            self.phi, self.dphi, self.geo = ops.edge_geometry(r_ij.detach().contiguous(), graph, mod._rbf_kind, mod._n_rbf,
                                                              mod._rbf_p0, mod._rbf_p1, mod._cutoff_value, need_grad)


class PaiNNContextFunction(torch.autograd.Function):
    """q [N,F] -> x = interatomic_context_net(q) [N,3F]."""

    @staticmethod
    def forward(ctx, q, blk, act):
        with ops.device_of(q):
            x, hpre = painn_context_fwd(blk, q.detach().contiguous(), act)
        ctx.blk, ctx.hpre = blk, hpre
        return x

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_x):
        with ops.device_of(g_x):
            return painn_context_bwd(ctx.blk, g_x.contiguous(), ctx.hpre), None, None


class PaiNNEdgeFunction(torch.autograd.Function):
    """(x [N,3F], mu [N,3,F] | None, q [R,F], r_ij [E,3]) -> (q + dq, mu + dmu) [R rows] with the filter evaluated in-kernel
    from the shared ``EdgeGeometry``; backward returns dE/dx, dE/dmu, dE/dq and this block's contribution to dE/dr_ij.
    R = number of receiver rows: N, or -- on a partition whose sender tables carry ghost rows after the owned atoms -- the
    owned count (edges only arrive at owned atoms, so the kernels need not walk the ghost rows)."""

    @staticmethod
    def forward(ctx, x, mu, q, r_ij, geom, pk, t):
        g = geom.graph
        xd = x.detach().contiguous()
        mud = mu.detach().contiguous() if mu is not None else None
        n_rows = int(q.shape[0])
        with ops.device_of(xd):
            q1, mu1 = ops.painn_edge_fwd(xd, mud, q.detach().contiguous(), geom.phi, geom.geo, g, pk.wf[t], pk.bf[t], pk.F,
                                         geom.n_rbf, wf_packed=_packed_filter(pk, t, geom.n_rbf, g.n_edges), n_rows=n_rows)
        ctx.n_rows = n_rows
        ctx.h = (xd, mud, geom, pk, t)
        ctx.set_materialize_grads(False)
        return q1, mu1

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_q1, g_mu1):
        xd, mud, geom, pk, t = ctx.h
        g = geom.graph
        N, F = g.n_atoms, pk.F
        dev = xd.device
        R = ctx.n_rows
        with ops.device_of(xd):
            g_q1 = g_q1.contiguous() if g_q1 is not None else torch.zeros((R, F), dtype=torch.float32, device=dev)
            g_mu1 = g_mu1.contiguous() if g_mu1 is not None else torch.zeros((R, 3, F), dtype=torch.float32, device=dev)
            g_qk, g_muk = g_q1, g_mu1
            if R < N:      # the reverse kernel walks SENDER rows (ghosts included) and adds dE/dmu_out row-wise: pad with zeros
                g_qk = torch.cat([g_q1, g_q1.new_zeros((N - R, F))], dim=0)
                g_muk = torch.cat([g_mu1, g_mu1.new_zeros((N - R, 3, F))], dim=0)
            g_rij = torch.empty((geom.E, 3), dtype=torch.float32, device=dev)
            g_x, g_mu0 = ops.painn_edge_bwd(xd, mud, g_qk, g_muk, geom.phi, geom.dphi, geom.geo, g, pk.wf[t], pk.bf[t], F,
                                            geom.n_rbf, g_rij, accumulate=False,
                                            wf_packed=_packed_filter(pk, t, geom.n_rbf, g.n_edges))
        return g_x, g_mu0, g_q1, g_rij, None, None, None


class PaiNNEdgeWijFunction(torch.autograd.Function):
    """Interaction with a caller-supplied filter (painn.py:55-65): (x, mu, q, Wij [E,3F], dir_ij [E,3]) -> (q', mu')."""

    @staticmethod
    def forward(ctx, x, mu, q, Wij, dir_ij, graph, F):
        t = [v.detach().contiguous() for v in (x, mu, q, Wij, dir_ij)]
        with ops.device_of(*t):
            q1, mu1 = ops.painn_edge_wij_fwd(t[0], t[1], t[2], t[3], t[4], graph, F)
        ctx.h = (t[0], t[1], t[3], t[4], graph, F)
        ctx.set_materialize_grads(False)
        return q1, mu1

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_q1, g_mu1):
        x, mu, Wij, dir_ij, graph, F = ctx.h
        N, dev = graph.n_atoms, x.device
        with ops.device_of(x):
            g_q1 = g_q1.contiguous() if g_q1 is not None else torch.zeros((N, F), dtype=torch.float32, device=dev)
            g_mu1 = g_mu1.contiguous() if g_mu1 is not None else torch.zeros((N, 3, F), dtype=torch.float32, device=dev)
            g_x, g_mu0, g_W, g_dir = ops.painn_edge_wij_bwd(x, mu, g_q1, g_mu1, Wij, dir_ij, graph, F)
        return g_x, g_mu0, g_q1, g_W, g_dir, None, None


class PaiNNMixingFunction(torch.autograd.Function):
    """PaiNNMixing.forward (painn.py:92-117): (q [N,F], mu [N,3,F]) -> (q', mu')."""

    @staticmethod
    def forward(ctx, q, mu, blk, F, eps, act):
        with ops.device_of(q, mu):
            q2, mu2, tape = painn_mixing_fwd(blk, q.detach().contiguous(), mu.detach().contiguous(), F, eps, act)
        ctx.h = (blk, tape, F, eps)
        ctx.set_materialize_grads(False)
        return q2, mu2

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_q, g_mu):
        blk, tape, F, eps = ctx.h
        N, dev = tape[2].shape[0], tape[2].device
        with ops.device_of(tape[2]):
            g_q = g_q.contiguous() if g_q is not None else torch.zeros((N, F), dtype=torch.float32, device=dev)
            g_mu = g_mu.contiguous() if g_mu is not None else torch.zeros((N, 3, F), dtype=torch.float32, device=dev)
            g_q1, g_mu1 = painn_mixing_bwd(blk, g_q, g_mu, tape, F, eps)
        return g_q1, g_mu1, None, None, None, None


# =====================================================================================================================
# SO3net  (representation/so3net.py:103-155)
# =====================================================================================================================
class SO3netPack(ParamPack):
    def build(self, mod):
        self.F, self.T, self.L = mod.n_atom_basis, mod.n_interactions, mod.lmax
        self.blocks = []
        for t in range(self.T):
            conv, gate = mod.so3convs[t], mod.gatings[t]
            self.blocks.append(dict(
                wf=_c(conv.filternet.weight), bf=_c(conv.filternet.bias), m1=ops.Lin(mod.mixings1[t].weight),
                m2=ops.Lin(mod.mixings2[t].weight), m3=ops.Lin(mod.mixings3[t].weight),
                sc=ops.Lin(gate.scaling.weight, gate.scaling.bias)))


def so3net_forward(pk: SO3netPack, x0: Tensor, r_ij: Tensor, graph: ops.EdgeGraph, rbf_kind: int, n_rbf: int,
                   rbf_p0: Tensor, rbf_p1: Optional[Tensor], cutoff: float, need_grad: bool):
    """Returns the multipole features x [N,S,F] and the tape needed by so3net_backward."""
    F, L = pk.F, pk.L
    N, S = x0.shape[0], (pk.L + 1) ** 2
    phi, dphi, geo = ops.edge_geometry(r_ij, graph, rbf_kind, n_rbf, rbf_p0, rbf_p1, cutoff, need_grad)
    x = ops.so3_put_l0(None, x0, N, L, F, x0.device)                                          # scalar2rsh (:136)
    tape = []
    for b in pk.blocks:
        dx = ops.so3_conv_fwd(x, phi, geo, graph, b["wf"], b["bf"], L, F, n_rbf)              # :140
        ddx = b["m1"].fwd(dx.view(N * S, F)).view(N, S, F)                                    # :141
        tp = ops.so3_tp_fwd(dx, ddx, L, F)                                                    # :142
        m2 = b["m2"].fwd(tp.view(N * S, F)).view(N, S, F)                                     # :143
        h = b["sc"].fwd(m2.view(N, S * F), k=F)                                               # :144, so3.py:330-332
        g = ops.so3_gate_fwd(m2, h, L, F)                                                     # so3.py:333
        x_new = b["m3"].fwd(g.view(N * S, F), addend=x.view(N * S, F)).view(N, S, F)          # :145-146
        if need_grad:
            tape.append((x, dx, ddx, m2, h))
        x = x_new
    return x, (phi, dphi, geo, tape)


def so3net_backward(pk: SO3netPack, saved, graph: ops.EdgeGraph, n_rbf: int, g_x: Tensor, n_edges_total: int) -> Tensor:
    """dE/dr_ij [E,3] (in the caller's edge order) from dE/dx [N,S,F]."""
    F, L = pk.F, pk.L
    phi, dphi, geo, tape = saved
    N, S = g_x.shape[0], (L + 1) ** 2
    g_rij = torch.empty((n_edges_total, 3), dtype=torch.float32, device=g_x.device)
    for t in reversed(range(pk.T)):
        b = pk.blocks[t]
        x, dx, ddx, m2, h = tape[t]
        g_g = b["m3"].bwd(g_x.view(N * S, F)).view(N, S, F)
        g_m2, g_m2_row0, g_h = ops.so3_gate_bwd(g_g, m2, h, L, F)
        b["sc"].bwd(g_h, addend=g_m2_row0, out=g_m2.view(N, S * F))                          # row 0 += scaling^T g_h
        g_tp = b["m2"].bwd(g_m2.view(N * S, F)).view(N, S, F)
        g_dx, g_ddx = ops.so3_tp_bwd(g_tp, dx, ddx, L, F)
        g_dx = b["m1"].bwd(g_ddx.view(N * S, F), addend=g_dx.view(N * S, F)).view(N, S, F)
        # dE/dx_in = residual + convolution reverse; block 0's would only reach the (position-independent) embedding
        g_x = ops.so3_conv_bwd(x, g_dx, phi, dphi, geo, graph, b["wf"], b["bf"], L, F, n_rbf, g_x, g_rij,
                               accumulate=(t != pk.T - 1), need_gx=(t > 0))
    return g_rij


class SO3netFunction(torch.autograd.Function):
    """(r_ij [E,3], x0 [N,F]) -> (scalar rows [N,F], multipoles [N,S,F]); the scalar rows are returned contiguous so that
    the Atomwise gradient arrives without a copy.  Backward gives dE/dr_ij (x0 = embedding output is treated as constant)."""

    @staticmethod
    def forward(ctx, r_ij, x0, holder):
        mod, graph = holder["module"], holder["graph"]
        pk = mod._pack()
        need = r_ij.requires_grad
        with ops.device_of(r_ij, x0):
            x, saved = so3net_forward(pk, x0, r_ij.detach(), graph, mod._rbf_kind, mod._n_rbf, mod._rbf_p0, mod._rbf_p1,
                                      mod._cutoff_value, need)
            q = ops.so3_take_l0(x, pk.L, pk.F)
        ctx.holder = dict(pk=pk, saved=saved, graph=graph, n_rbf=mod._n_rbf, E=r_ij.shape[0], N=x0.shape[0])
        ctx.set_materialize_grads(False)
        return q, x

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_q, g_x):
        h = ctx.holder
        pk = h["pk"]
        some = g_q if g_q is not None else g_x
        with ops.device_of(some):
            g = ops.so3_put_l0(g_x.contiguous() if g_x is not None else None,
                               g_q.contiguous() if g_q is not None else None, h["N"], pk.L, pk.F, some.device)
            g_rij = so3net_backward(pk, h["saved"], h["graph"], h["n_rbf"], g, h["E"])
        return g_rij, None, None


# =====================================================================================================================
# SchNet  (representation/schnet.py:147-173)
# =====================================================================================================================
class SchNetPack(ParamPack):
    def build(self, mod):
        self.F, self.T, self.NF = mod.n_atom_basis, len(mod.interactions), mod.n_filters
        self.blocks = []
        for it in mod.interactions:
            f0, f1 = it.filter_network[0], it.filter_network[1]
            o0, o1 = it.f2out[0], it.f2out[1]
            self.blocks.append(dict(
                in2f=ops.Lin(it.in2f.weight), f0=ops.Lin(f0.weight, f0.bias), f1=ops.Lin(f1.weight, f1.bias),
                o0=ops.Lin(o0.weight, o0.bias), o1=ops.Lin(o1.weight, o1.bias), fpk=None,
            ))


def _schnet_filter_packed(b, n_rbf: int):
    if b["fpk"] is None:      # tensor-core operand tiles of the block's filter network, built on first use
        b["fpk"] = ops.schnet_pack_filter(b["f0"].w, b["f0"].b, b["f1"].w, n_rbf)
    return b["fpk"]


def schnet_forward_fused(pk: SchNetPack, x0: Tensor, r_ij: Tensor, idx_i: Tensor, idx_j: Tensor, rbf_kind: int, n_rbf: int,
                         rbf_p0, rbf_p1, cutoff: float, act: int) -> Tensor:
    """Inference forward (no tape) with ONE fused edge kernel per interaction block (filter network on the tensor cores inside it,
    csrc/schnet_tc.cu) over the ACTIVE edges only (d < cutoff: padding slots of a padded neighbour list are dropped when the
    receiver CSR is built).  schnet.py:56-70,160-171."""
    N = x0.shape[0]
    graph = ops.EdgeGraph(idx_i, idx_j, N, r_ij=r_ij, cutoff=cutoff)
    phi, _, geo = ops.edge_geometry(r_ij, graph, rbf_kind, n_rbf, rbf_p0, rbf_p1, cutoff, False, active_only=True)
    x = x0
    h = pk.blocks[0]["in2f"].fwd(x)                                                          # schnet.py:60
    for t in range(pk.T):
        b = pk.blocks[t]
        m = ops.schnet_cfconv_fwd_tc(h, phi, geo, graph, _schnet_filter_packed(b, n_rbf), b["f1"].b, act, n_rbf)   # :61-67
        v0 = b["o0"].fwd(m, act)
        x = b["o1"].fwd(v0, addend=x)
        if t + 1 < pk.T:
            h = pk.blocks[t + 1]["in2f"].fwd(x)
    return x


def schnet_forward(pk: SchNetPack, x0: Tensor, r_ij: Tensor, graph: ops.EdgeGraph, rbf_kind: int, n_rbf: int,
                   rbf_p0, rbf_p1, cutoff: float, act: int, need_grad: bool):
    NF = pk.NF
    phi, dphi, geo = ops.edge_geometry(r_ij, graph, rbf_kind, n_rbf, rbf_p0, rbf_p1, cutoff, need_grad)
    x = x0
    tape = []
    for t in range(pk.T):
        b = pk.blocks[t]
        h = b["in2f"].fwd(x)                                                                 # schnet.py:60
        w0, w0pre = b["f0"].fwd(phi, act, save_deriv=True, k=n_rbf)                            # :61 (phi is [E,KP])
        w_raw = b["f1"].fwd(w0)                                                              # [E,NF]
        m = ops.cfconv_fwd(h, w_raw, geo, graph, NF)                                         # :62-67
        v0, v0pre = b["o0"].fwd(m, act, save_deriv=True)                                       # :69
        x_new = b["o1"].fwd(v0, addend=x)                                                    # :69 + :168 residual
        if need_grad:
            tape.append((h, w0pre, w_raw, v0pre))
        x = x_new
    return x, (phi, dphi, geo, tape)


def schnet_backward(pk: SchNetPack, saved, graph: ops.EdgeGraph, n_rbf: int, act: int, g_x: Tensor,
                    n_edges_total: int) -> Tensor:
    NF = pk.NF
    phi, dphi, geo, tape = saved
    dev = g_x.device
    g_rij = torch.empty((n_edges_total, 3), dtype=torch.float32, device=dev)
    KP = ops.kp(n_rbf)
    for t in reversed(range(pk.T)):
        b = pk.blocks[t]
        h, w0pre, w_raw, v0pre = tape[t]
        g_v0 = b["o1"].bwd(g_x)                                                              # [N,F]x[F,F]
        g_m = b["o0"].bwd(g_v0, a_pre=v0pre, a_act=ops.ACT_GIVEN)                                      # [N,F]x[F,NF]
        g_h, g_wraw, g_fc = ops.cfconv_bwd(h, w_raw, geo, g_m, graph, NF)
        g_w0 = b["f1"].bwd(g_wraw)                                                           # [E,NF]x[NF,NF]
        E = g_w0.shape[0]
        g_phi = torch.empty((E, KP), dtype=torch.float32, device=dev)
        b["f0"].bwd(g_w0, a_pre=w0pre, a_act=ops.ACT_GIVEN, out=g_phi)                                 # [E,NF]x[NF,n_rbf]
        ops.radial_bwd(g_phi, g_fc, dphi, geo, graph, n_rbf, g_rij, accumulate=(t != pk.T - 1))
        if t == 0:
            break   # the gradient w.r.t. the embedding output is not needed for forces
        g_x = b["in2f"].bwd(g_h, addend=g_x)                                                 # + residual
    return g_rij


class SchNetFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, r_ij, x0, holder):
        mod, graph = holder["module"], holder["graph"]
        pk = mod._pack()
        need = r_ij.requires_grad
        with ops.device_of(r_ij, x0):
            if graph is None:
                x = schnet_forward_fused(pk, x0, r_ij.detach(), holder["idx_i"], holder["idx_j"], mod._rbf_kind, mod._n_rbf,
                                         mod._rbf_p0, mod._rbf_p1, mod._cutoff_value, mod._act)
                saved = None
            else:
                x, saved = schnet_forward(pk, x0, r_ij.detach(), graph, mod._rbf_kind, mod._n_rbf, mod._rbf_p0,
                                          mod._rbf_p1, mod._cutoff_value, mod._act, need)
        ctx.holder = dict(pk=pk, saved=saved, graph=graph, n_rbf=mod._n_rbf, act=mod._act, E=r_ij.shape[0])
        return x

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_x):
        h = ctx.holder
        with ops.device_of(g_x):
            g_rij = schnet_backward(h["pk"], h["saved"], h["graph"], h["n_rbf"], h["act"], g_x.contiguous(), h["E"])
        return g_rij, None, None


class CFConvFunction(torch.autograd.Function):
    """Continuous-filter convolution of the block-level API (schnet.py:62-67): (h [N,F], Wij [E,F], rcut [E]) ->
    m[i] = sum_{e: idx_i[e]=i} h[idx_j[e]] * Wij[e] * rcut[e], with all three gradients.  Wij / rcut arrive in the caller's
    edge order; the permutation to receiver-slot order is an index_select (data movement only)."""

    @staticmethod
    def forward(ctx, h, Wij, rcut, graph):
        hd = h.detach().contiguous()
        with ops.device_of(hd, Wij, rcut):
            eid = graph.slot_eid[:graph.n_edges].long()
            w_slot = Wij.detach().index_select(0, eid).contiguous()
            geo = torch.zeros((graph.n_edges, ops.GEO_STRIDE), dtype=torch.float32, device=hd.device)
            geo[:, 4] = rcut.detach().reshape(-1).index_select(0, eid)
            m = ops.cfconv_fwd(hd, w_slot, geo, graph, hd.shape[1])
        ctx.h = (hd, w_slot, geo, graph, eid, rcut.shape)
        return m

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_m):
        hd, w_slot, geo, graph, eid, rshape = ctx.h
        with ops.device_of(hd):
            g_h, g_w_slot, g_fc_slot = ops.cfconv_bwd(hd, w_slot, geo, g_m.contiguous(), graph, hd.shape[1])
            g_W = torch.empty_like(g_w_slot).index_copy_(0, eid, g_w_slot)
            g_rc = torch.empty_like(g_fc_slot).index_copy_(0, eid, g_fc_slot).view(rshape)
        return g_h, g_W, g_rc, None


# =====================================================================================================================
# Atomwise (atomistic/atomwise.py:69-88) and PairwiseDistances (atomistic/distances.py:14-26)
# =====================================================================================================================
class AtomwiseFunction(torch.autograd.Function):
    """q [N,F] -> (y [N], energy [B]) for outnet = Dense(F->H, silu) -> Dense(H->1)."""

    @staticmethod
    def forward(ctx, q, holder):
        pk, idx_m, n_mol, act = holder["pack"], holder["idx_m"], holder["n_mol"], holder["act"]
        qd = q.detach().contiguous()
        with ops.device_of(qd):
            hid, hpre = pk["l0"].fwd(qd, act, save_deriv=True)
            mol_ptr = ops.segment_ptr(idx_m, n_mol) if idx_m is not None else None
            y, energy = ops.atomwise_out(hid, pk["w1"], pk["b1"], mol_ptr, n_mol)
        ctx.holder = dict(pk=pk, hpre=hpre, idx_m=idx_m, act=act, N=q.shape[0])
        ctx.set_materialize_grads(False)
        if energy is None:
            energy = y.new_zeros((0,))
        return y, energy

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_y, g_e):
        h = ctx.holder
        pk = h["pk"]
        H = pk["w1"].shape[0]
        g_hid = None
        torch.cuda.set_device(pk["w1"].device)       # autograd worker thread: make the parameters' device current
        if h["idx_m"] is not None and g_e is not None and g_e.numel() > 0:
            g_hid = ops.atomwise_out_bwd(g_e.contiguous(), h["idx_m"], pk["w1"], h["N"], H)
        if g_y is not None:  # per-atom output used downstream (rare): g_hid += g_y (x) w1  -- plumbing-level torch op
            extra = g_y.contiguous()[:, None] * pk["w1"][None, :]
            g_hid = extra if g_hid is None else g_hid + extra
        if g_hid is None:
            return None, None
        g_q = pk["l0"].bwd(g_hid.contiguous(), a_pre=h["hpre"], a_act=ops.ACT_GIVEN)
        return g_q, None


class PairwiseDistancesFunction(torch.autograd.Function):
    """Rij = R[idx_j] - R[idx_i] + offsets; backward assembles dE/dR per atom from the CSR/CSC views (no atomics)."""

    @staticmethod
    def forward(ctx, R, offsets, holder):
        idx_i, idx_j = holder["idx_i"], holder["idx_j"]
        ctx.holder = holder
        ctx.off_grad = offsets is not None and offsets.requires_grad
        with ops.device_of(R, idx_i, idx_j):
            r_ij = ops.pairwise_fwd(R.detach().contiguous(), idx_i, idx_j,
                                    offsets.detach().contiguous() if offsets is not None else None)
        if holder.get("virial") is not None:
            # the virial contracts the edge gradient with r_ij itself: keep the output (no copy, no recompute launch)
            ctx.save_for_backward(r_ij)
        return r_ij

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_rij):
        g_rij = g_rij.contiguous()
        h = ctx.holder
        graph = h["graph"]
        with ops.device_of(g_rij):
            g_R = ops.pairwise_bwd(g_rij, graph, 1.0)
            if h.get("virial") is not None:
                (r_ij,) = ctx.saved_tensors
                ops.pairwise_virial(g_rij, r_ij, graph, h["sys_ptr"], h["virial"],
                                    accumulate=h.pop("virial_deposited", False))
        return g_R, (g_rij if ctx.off_grad else None), None


# =====================================================================================================================
# DipoleMoment / Polarizability (atomistic/atomwise.py:172-213, 267-293) with the gated equivariant MLP
# (nn/equivariant.py:57-71, nn/blocks.py:79-156)
# =====================================================================================================================
class HeadPack(ParamPack):
    """Kernel-ready weights of a head's outnet: hidden gated blocks as Lin triples, the last block as an
    ``spk_head_tail_t``; for the scalar dipole, the hidden Dense layers and the last layer's weight row."""

    def build(self, mod):
        from .nn import activation_code

        net = mod.outnet
        self.blocks = []
        if mod._vector:
            for blk in list(net)[:-1]:
                self.blocks.append(dict(mix=ops.Lin(blk.mix_vectors.weight), l0=ops.Lin(blk.scalar_net[0].weight,
                                        blk.scalar_net[0].bias), l1=ops.Lin(blk.scalar_net[1].weight, blk.scalar_net[1].bias),
                                        Fi=blk.n_sin, Fo=blk.n_vout, act=activation_code(blk.scalar_net[0].activation),
                                        sact=activation_code(blk.sactivation)))
            last = net[-1]
            self.tail, self._keep = ops.head_tail(last.mix_vectors.weight, last.scalar_net[0].weight,
                                                  last.scalar_net[0].bias, last.scalar_net[1].weight,
                                                  last.scalar_net[1].bias, activation_code(last.scalar_net[0].activation))
        else:
            for lin in list(net)[:-1]:
                self.blocks.append(dict(lin=ops.Lin(lin.weight, lin.bias), act=activation_code(lin.activation)))
            self.w1 = _c(net[-1].weight).reshape(-1)
            self.b1 = _c(net[-1].bias)
            self.tail = None


def _charges_grad(h, g_charges):
    """dE/dq of the tail's charges from dE/dcharges (the correction's reverse), or None when no charge gradient arrives."""
    if g_charges is None or not h.get("diff_charges") or g_charges.numel() == 0:
        return None
    return ops.head_charges_bwd(g_charges.contiguous(), h["idx_m"], h["sys_ptr"], h["n_sys"], h["correct"])


def _dipole_grad_out(h, g_out, like):
    if g_out is not None:
        return g_out.contiguous()
    shape = (h["n_sys"],) if h["magnitude"] else (h["n_sys"], 3)
    return torch.zeros(shape, dtype=torch.float32, device=like.device)


class GatedHeadFunction(torch.autograd.Function):
    """(s [N,Fi], V [N,3,Fi], R [N,3]) -> (dipole [B,3] / |dipole| [B] / polarizability [B,3,3], charges [N]).  The head
    output is differentiable with respect to s, V and R, the charges too when ``holder["diff_charges"]`` is set; a charge
    gradient takes the ``spk_head_bwd_q`` reverse, without one the reverse is exactly ``spk_head_bwd``."""

    @staticmethod
    def forward(ctx, s, V, R, holder):
        pk, kind = holder["pack"], holder["kind"]
        s, V, Rd = _c(s), _c(V), _c(R)
        N = s.shape[0]
        tape = []
        with ops.device_of(s, V, Rd):
            for b in pk.blocks:
                Fi, Fo = b["Fi"], b["Fo"]
                VW = b["mix"].fwd(V.view(3 * N, Fi)).view(N, 3, 2 * Fo)
                c = ops.geq_ctx(s, VW, Fi, Fo)
                h, d0 = b["l0"].fwd(c, b["act"], save_deriv=True)
                x = b["l1"].fwd(h)
                tape.append((VW, d0, x))
                s, V = ops.geq_gate(x, VW, Fo, b["sact"])
            out, q_atom, saved = ops.head_fwd(kind, pk.tail, s, V, None, Rd, holder["idx_m"], holder["sys_ptr"],
                                              holder["total_charge"], holder["n_sys"], holder["correct"],
                                              holder["magnitude"], holder["want_charges"])
            charges = ops.head_charges(q_atom, holder["idx_m"], saved) if q_atom is not None else s.new_zeros((0,))
        ctx.holder = dict(holder, tape=tape, s=s, V=V, R=Rd, saved=saved)
        if not holder.get("diff_charges"):
            ctx.mark_non_differentiable(charges)
        ctx.set_materialize_grads(False)
        return out, charges

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_out, g_charges):
        h = ctx.holder
        g_q = _charges_grad(h, g_charges)
        if g_out is None and g_q is None:
            return None, None, None, None
        pk = h["pack"]
        with ops.device_of(h["s"]):
            if g_q is None:
                g_s, g_V, g_R = ops.head_bwd(h["kind"], pk.tail, h["s"], h["V"], h["R"], h["idx_m"], h["saved"],
                                             g_out.contiguous(), h["correct"], h["magnitude"])
            else:
                g_s, g_V, g_R = ops.head_bwd_q(pk.tail, h["s"], h["V"], h["R"], h["idx_m"], h["saved"],
                                               _dipole_grad_out(h, g_out, g_q), g_q, h["correct"], h["magnitude"])
            N = g_s.shape[0]
            for b, (VW, d0, x) in zip(reversed(pk.blocks), reversed(h["tape"])):
                Fi, Fo = b["Fi"], b["Fo"]
                g_x, g_VW = ops.geq_gate_bwd(g_s, g_V, x, VW, Fo, b["sact"])
                g_h = b["l1"].bwd(g_x)
                g_c = b["l0"].bwd(g_h, a_pre=d0, a_act=ops.ACT_GIVEN)
                g_s = ops.geq_ctx_bwd(g_c, VW, g_VW, Fi, Fo)
                g_V = b["mix"].bwd(g_VW.view(3 * N, 2 * Fo)).view(N, 3, Fi)
        return g_s, g_V, g_R, None


class ScalarDipoleFunction(torch.autograd.Function):
    """(s [N,F], R [N,3]) -> (dipole [B,3] / |dipole| [B], charges [N]) for charges from a plain MLP (Lin layers, then
    ``spk_atomwise_out`` without aggregation for the last Dense H -> 1).  Differentiable as ``GatedHeadFunction``."""

    @staticmethod
    def forward(ctx, s, R, holder):
        pk = holder["pack"]
        h, Rd = _c(s), _c(R)
        tape = []
        with ops.device_of(h, Rd):
            for b in pk.blocks:
                h, d = b["lin"].fwd(h, b["act"], save_deriv=True)
                tape.append(d)
            q, _ = ops.atomwise_out(h, pk.w1, pk.b1, None, 0)
            out, _, saved = ops.head_fwd(ops.HEAD_DIPOLE, None, None, None, q, Rd, holder["idx_m"], holder["sys_ptr"],
                                         holder["total_charge"], holder["n_sys"], holder["correct"],
                                         holder["magnitude"], False)
            charges = ops.head_charges(q, holder["idx_m"], saved) if holder["want_charges"] else q.new_zeros((0,))
        ctx.holder = dict(holder, tape=tape, q=q, R=Rd, saved=saved)
        if not holder.get("diff_charges"):
            ctx.mark_non_differentiable(charges)
        ctx.set_materialize_grads(False)
        return out, charges

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_out, g_charges):
        h = ctx.holder
        g_q = _charges_grad(h, g_charges)
        if g_out is None and g_q is None:
            return None, None, None
        pk = h["pack"]
        with ops.device_of(h["q"]):
            if g_q is None:
                g_h, g_R = ops.head_scalar_bwd(h["q"], h["R"], h["idx_m"], h["saved"], g_out.contiguous(), h["correct"],
                                               h["magnitude"], pk.w1)
            else:
                g_h, g_R = ops.head_scalar_bwd_q(h["q"], h["R"], h["idx_m"], h["saved"], _dipole_grad_out(h, g_out, g_q),
                                                 g_q, h["correct"], h["magnitude"], pk.w1)
            for b, d in zip(reversed(pk.blocks), reversed(h["tape"])):
                g_h = b["lin"].bwd(g_h, a_pre=d, a_act=ops.ACT_GIVEN)
        return g_h, g_R, None


# =====================================================================================================================
# Pair energies: ZBL repulsion (atomistic/nuclear_repulsion.py:70-108) and Coulomb (atomistic/electrostatic.py:109-152)
# =====================================================================================================================
class PairEnergyFunction(torch.autograd.Function):
    """(r_ij [E,3], q [N] | None) -> energy [B] of one pair term on csrc/pair_energy.cu; backward gives dE/dr_ij and, for
    Coulomb, dE/dq (which reaches the charge head through its differentiable charges output)."""

    @staticmethod
    def forward(ctx, r_ij, q, holder):
        rd = r_ij.detach().contiguous()
        qd = q.detach().contiguous() if q is not None else None
        with ops.device_of(rd, qd):
            e = ops.pair_energy_fwd(holder["params"], rd, holder["idx_i"], holder["idx_j"], holder.get("Z"), qd,
                                    holder["idx_m"], holder["graph"], holder["sys_ptr"], holder["n_sys"])
        ctx.h = (holder, rd, qd)
        ctx.want_q = q is not None and ctx.needs_input_grad[1]
        ctx.set_materialize_grads(False)
        return e

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_E):
        if g_E is None:
            return None, None, None
        h, rd, qd = ctx.h
        with ops.device_of(rd):
            g_rij, g_q = ops.pair_energy_bwd(h["params"], rd, h["idx_i"], h["idx_j"], h.get("Z"), qd, h["idx_m"],
                                             g_E.contiguous(), h["graph"], ctx.want_q)
        return g_rij, g_q, None


# =====================================================================================================================
# Ewald summation (atomistic/electrostatic.py:155-375): real space on csrc/pair_energy.cu, reciprocal and self terms on
# csrc/ewald.cu
# =====================================================================================================================
class EwaldFunction(torch.autograd.Function):
    """(r_ij [E,3], R [N,3], q [N], cell [B,3,3]) -> energy [B] = E_real + E_rec - E_self.  Backward: dE/dr_ij (real
    space), dE/dR (reciprocal), dE/dq (all three terms) and dE/dcell (reciprocal, for the Strain path).  With a virial
    requested from PairwiseDistances (``holder["sink"]``) it also deposits the reciprocal virial there; this backward
    always runs before PairwiseDistances' (which needs dE/dr_ij from it), so the pairwise pass then adds to it."""

    @staticmethod
    def forward(ctx, r_ij, R, q, cell, holder):
        rd, Rd, qd = r_ij.detach().contiguous(), R.detach().contiguous(), q.detach().contiguous()
        cd = cell.detach().reshape(-1, 3, 3).contiguous()
        with ops.device_of(rd, Rd, qd, cd):
            e_real = ops.pair_energy_fwd(holder["params"], rd, holder["idx_i"], holder["idx_j"], None, qd, holder["idx_m"],
                                         holder["graph"], holder["sys_ptr"], holder["n_sys"])
            energy, ws = ops.ewald_fwd(Rd, qd, cd, holder["kvecs"], holder["idx_m"], holder["sys_ptr"], holder["n_sys"],
                                       holder["ke"], holder["alpha"], addend=e_real)
        ctx.h = (holder, rd, Rd, qd, cd, ws)
        ctx.cell_shape = cell.shape
        ctx.set_materialize_grads(False)
        return energy

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_E):
        if g_E is None:
            return None, None, None, None, None
        h, rd, Rd, qd, cd, ws = ctx.h
        _, want_R, want_q, want_cell, _ = ctx.needs_input_grad
        sink = h.get("sink")
        virial, acc = None, False
        if sink is not None:
            virial, acc = sink["virial"], sink.get("virial_deposited", False)
            sink["virial_deposited"] = True
        with ops.device_of(rd):
            g_E = g_E.contiguous()
            g_rij, g_q = ops.pair_energy_bwd(h["params"], rd, h["idx_i"], h["idx_j"], None, qd, h["idx_m"], g_E, h["graph"],
                                             want_q)
            g_R, g_cell = ops.ewald_bwd(Rd, qd, cd, h["kvecs"], h["idx_m"], h["sys_ptr"], h["n_sys"], h["ke"], h["alpha"],
                                        g_E, ws, want_R, g_q, want_cell, virial, acc)
        return g_rij, g_R, g_q, (g_cell.view(ctx.cell_shape) if g_cell is not None else None), None


class PMEFunction(torch.autograd.Function):
    """``EwaldFunction`` with the reciprocal term by smooth particle-mesh Ewald (csrc/pme.cu, fp64 FFTs between its
    launches): the same inputs, backward outputs and virial-sink protocol; ``holder["mesh"]`` and ``holder["order"]``
    replace the k-vectors."""

    @staticmethod
    def forward(ctx, r_ij, R, q, cell, holder):
        rd, Rd, qd = r_ij.detach().contiguous(), R.detach().contiguous(), q.detach().contiguous()
        cd = cell.detach().reshape(-1, 3, 3).contiguous()
        with ops.device_of(rd, Rd, qd, cd):
            e_real = ops.pair_energy_fwd(holder["params"], rd, holder["idx_i"], holder["idx_j"], None, qd, holder["idx_m"],
                                         holder["graph"], holder["sys_ptr"], holder["n_sys"])
            energy, conv, ws = ops.pme_fwd(Rd, qd, cd, holder["idx_m"], holder["sys_ptr"], holder["n_sys"],
                                           holder["mesh"], holder["order"], holder["ke"], holder["alpha"], addend=e_real)
        ctx.h = (holder, rd, Rd, qd, conv, ws)
        ctx.cell_shape = cell.shape
        ctx.set_materialize_grads(False)
        return energy

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_E):
        if g_E is None:
            return None, None, None, None, None
        h, rd, Rd, qd, conv, ws = ctx.h
        _, want_R, want_q, want_cell, _ = ctx.needs_input_grad
        sink = h.get("sink")
        virial, acc = None, False
        if sink is not None:
            virial, acc = sink["virial"], sink.get("virial_deposited", False)
            sink["virial_deposited"] = True
        with ops.device_of(rd):
            g_E = g_E.contiguous()
            g_rij, g_q = ops.pair_energy_bwd(h["params"], rd, h["idx_i"], h["idx_j"], None, qd, h["idx_m"], g_E, h["graph"],
                                             want_q)
            g_R, g_cell = ops.pme_bwd(Rd, qd, h["idx_m"], h["sys_ptr"], h["n_sys"], h["mesh"], h["order"], h["ke"],
                                      h["alpha"], g_E, conv, ws, want_R, g_q, want_cell, virial, acc)
        return g_rij, g_R, g_q, (g_cell.view(ctx.cell_shape) if g_cell is not None else None), None
