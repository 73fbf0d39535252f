"""Python-side plumbing over the C ABI: tensor checks, buffer allocation (torch owns device memory), stream handoff.

Every function here launches hand-written sm_90a kernels from ``csrc/`` through ``include/spk_b200.h``; there is no
torch arithmetic on the hot path and no CPU fallback (non-CUDA tensors raise).
"""
from __future__ import annotations

import ctypes
import os
import weakref
from ctypes import c_void_p
from typing import Optional

import torch

from . import _lib
from ._lib import ACT_GIVEN, ACT_NONE, ACT_SILU, ACT_SSP, GEO_STRIDE, RBF_BESSEL, RBF_GAUSSIAN, SAVE_DERIV  # noqa: F401

Tensor = torch.Tensor


def _p(t: Optional[Tensor]):
    return None if t is None else c_void_p(t.data_ptr())


def _stream():
    """Current stream of the CURRENT device; ``device_of`` makes the tensors' device current around every pipeline."""
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def device_of(*tensors):
    """Context manager that makes the (single) CUDA device of ``tensors`` current, so that the stream handed to the C ABI,
    the library's per-device launch caches and the memory all belong to the same GPU even when the caller never called
    ``torch.cuda.set_device`` (e.g. ``model.to('cuda:1')``).  Mixed devices raise."""
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError(f"schnetpack_b200: CUDA tensors only (no CPU fallback); got {t.device}")
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise RuntimeError(f"schnetpack_b200: tensors on different devices ({dev} and {t.device})")
    return torch.cuda.device(dev)


def on_tensor_device(fn):
    """Decorator for the public ``forward`` methods: run with the CUDA device of the first tensor argument (a tensor, or
    the first CUDA tensor of an ``inputs`` dict) current.  Everything below -- graph build, weight packing, streams handed
    to the C ABI, per-device launch caches -- then agrees with the tensors' device even when the caller never called
    ``torch.cuda.set_device`` (``model.to('cuda:1')``)."""
    import functools

    @functools.wraps(fn)
    def wrapped(self, *args, **kwargs):
        dev = None
        for a in args:
            if isinstance(a, Tensor):
                if a.is_cuda:
                    dev = a.device
                    break
            elif isinstance(a, dict):
                for v in a.values():
                    if isinstance(v, Tensor) and v.is_cuda:
                        dev = v.device
                        break
                if dev is not None:
                    break
        if dev is None or dev.index == torch.cuda.current_device():
            return fn(self, *args, **kwargs)
        with torch.cuda.device(dev):
            return fn(self, *args, **kwargs)

    return wrapped


def _chk(t: Tensor, dtype, name: str):
    if not t.is_cuda:
        raise RuntimeError(f"schnetpack_b200: '{name}' must be a CUDA tensor (no CPU fallback); got {t.device}")
    if t.dtype != dtype:
        raise TypeError(f"schnetpack_b200: '{name}' must be {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"schnetpack_b200: '{name}' must be contiguous")
    return t


def f32(t: Tensor, name: str = "tensor") -> Tensor:
    return _chk(t, torch.float32, name)


def i64(t: Tensor, name: str = "index") -> Tensor:
    return _chk(t, torch.int64, name)


def kp(n_rbf: int) -> int:
    return (n_rbf + 3) & ~3


# ------------------------------------------------------------------------------------------------------------ graph
VALIDATE_INDICES = os.environ.get("SPK_B200_VALIDATE", "1") != "0"   # host check of a NEW neighbour list (one sync per list)


class EdgeGraph:
    """Receiver-grouped (CSR) and sender-grouped views of an (idx_i, idx_j) edge list, built on device."""

    __slots__ = ("n_atoms", "n_edges", "rowptr", "slot_j", "slot_eid", "sptr", "pos_slot", "pos_i", "status",
                 "_ref_i", "_ref_j", "_ver", "__weakref__")

    def __init__(self, idx_i: Tensor, idx_j: Tensor, n_atoms: int, r_ij: Optional[Tensor] = None,
                 cutoff: Optional[float] = None):
        """With ``r_ij`` / ``cutoff`` the views cover the ACTIVE edges only (|r_ij| < cutoff, spk_graph_build_active):
        ``rowptr[-1]`` on the device is their number, ``n_edges`` stays the capacity of the slot arrays."""
        i64(idx_i, "_idx_i")
        i64(idx_j, "_idx_j")
        if idx_i.shape != idx_j.shape or idx_i.dim() != 1:
            raise ValueError("idx_i / idx_j must be 1-D and of equal length")
        dev = idx_i.device
        E = idx_i.shape[0]
        self.n_atoms, self.n_edges = int(n_atoms), int(E)
        i32 = dict(dtype=torch.int32, device=dev)
        self.rowptr = torch.empty(n_atoms + 1, **i32)
        self.sptr = torch.empty(n_atoms + 1, **i32)
        self.slot_j = torch.empty(max(E, 1), **i32)
        self.slot_eid = torch.empty(max(E, 1), **i32)
        self.pos_slot = torch.empty(max(E, 1), **i32)
        self.pos_i = torch.empty(max(E, 1), **i32)
        self.status = torch.empty(4, **i32)
        nbytes = _lib.lib().spk_graph_workspace_bytes(n_atoms, E)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        if r_ij is None:
            _lib.call("spk_graph_build", _p(idx_i), _p(idx_j), n_atoms, E, _p(self.rowptr), _p(self.slot_j),
                      _p(self.slot_eid), _p(self.sptr), _p(self.pos_slot), _p(self.pos_i), _p(self.status), _p(ws),
                      nbytes, _stream())
        else:
            _lib.call("spk_graph_build_active", _p(idx_i), _p(idx_j), _p(f32(r_ij, "_Rij")), float(cutoff), n_atoms, E,
                      _p(self.rowptr), _p(self.slot_j), _p(self.slot_eid), _p(self.sptr), _p(self.pos_slot),
                      _p(self.pos_i), _p(self.status), _p(ws), nbytes, _stream())
        self._ref_i = weakref.ref(idx_i)
        self._ref_j = weakref.ref(idx_j)
        self._ver = (idx_i._version, idx_j._version)
        if VALIDATE_INDICES and E > 0 and not torch.cuda.is_current_stream_capturing():
            # the reference raises IndexError from index_select on a bad neighbour index; here the check costs one host
            # read per NEW neighbour list (cached graphs and captured evaluations skip it; the kernels are safe either way:
            # a bad list is evaluated as an empty graph with NaN distances)
            n_bad = int(self.status[1])
            if n_bad:
                raise IndexError(f"{n_bad} neighbour indices out of range [0, {self.n_atoms})")

    def matches(self, idx_i: Tensor, idx_j: Tensor, n_atoms: int) -> bool:
        return (self._ref_i() is idx_i and self._ref_j() is idx_j and self.n_atoms == n_atoms
                and self._ver == (idx_i._version, idx_j._version))

    def validate(self):
        """Host-synchronising check of the device status word (bad indices) -- used by tests / debug only."""
        st = self.status.tolist()
        if st[1] != 0:
            raise IndexError(f"{st[1]} neighbour indices out of range [0, {self.n_atoms})")
        return dict(sorted=bool(st[0]), max_in_degree=st[2], max_out_degree=st[3])


_GRAPH_CACHE: "dict[int, EdgeGraph]" = {}
_GRAPH_CACHE_MAX = 8


def get_graph(idx_i: Tensor, idx_j: Tensor, n_atoms: int) -> EdgeGraph:
    """Graph for this exact pair of index tensors (identity + version checked), rebuilt when they change."""
    key = id(idx_i)
    g = _GRAPH_CACHE.get(key)
    if g is not None and g.matches(idx_i, idx_j, n_atoms):
        return g
    g = EdgeGraph(idx_i, idx_j, n_atoms)
    if len(_GRAPH_CACHE) >= _GRAPH_CACHE_MAX:
        _GRAPH_CACHE.pop(next(iter(_GRAPH_CACHE)))
    _GRAPH_CACHE[key] = g
    return g


def segment_ptr(idx_m: Tensor, n_mol: int) -> Tensor:
    i64(idx_m, "_idx_m")
    out = torch.empty(n_mol + 1, dtype=torch.int32, device=idx_m.device)
    _lib.call("spk_segment_ptr", _p(idx_m), idx_m.shape[0], n_mol, _p(out), _stream())
    return out


# ------------------------------------------------------------------------------------------------------------ geometry
def pairwise_fwd(R: Tensor, idx_i: Tensor, idx_j: Tensor, offsets: Optional[Tensor]) -> Tensor:
    f32(R, "_positions")
    E = idx_i.shape[0]
    out = torch.empty((E, 3), dtype=torch.float32, device=R.device)
    _lib.call("spk_pairwise_fwd", _p(R), _p(i64(idx_i)), _p(i64(idx_j)),
              _p(f32(offsets, "_offsets")) if offsets is not None else None, R.shape[0], E, _p(out), _stream())
    return out


def pairwise_bwd(g_rij: Tensor, graph: EdgeGraph, sign: float = 1.0) -> Tensor:
    f32(g_rij, "g_rij")
    out = torch.empty((graph.n_atoms, 3), dtype=torch.float32, device=g_rij.device)
    _lib.call("spk_pairwise_bwd", _p(g_rij), _p(graph.rowptr), _p(graph.slot_eid), _p(graph.sptr), _p(graph.pos_slot),
              graph.n_atoms, float(sign), _p(out), _stream())
    return out


def pairwise_virial(g_rij: Tensor, r_ij: Tensor, graph: EdgeGraph, sys_ptr: Tensor, virial: Tensor,
                    accumulate: bool = False):
    """virial[m] = sum over the edges received by the atoms of system m of g_rij (x) r_ij, fp64, in place (``accumulate``:
    added to what virial holds)."""
    f32(g_rij, "g_rij")
    f32(r_ij, "_Rij")
    n_sys = virial.shape[0]
    nbytes = int(_lib.lib().spk_pairwise_virial_workspace_bytes(graph.n_edges, n_sys))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=g_rij.device)
    _lib.call("spk_pairwise_virial_add" if accumulate else "spk_pairwise_virial", _p(g_rij), _p(r_ij), _p(graph.rowptr),
              _p(graph.slot_eid), _p(sys_ptr), graph.n_edges, n_sys, _p(virial), _p(ws), nbytes, _stream())


def edge_geometry(r_ij: Tensor, graph: Optional[EdgeGraph], rbf_kind: int, n_rbf: int, p0: Tensor, p1: Optional[Tensor],
                  cutoff: float, need_grad: bool = True, active_only: bool = False):
    """``active_only``: ``graph`` was built from the active edges (EdgeGraph(..., r_ij, cutoff)); only its
    ``rowptr[-1]`` slots are filled."""
    f32(r_ij, "_Rij")
    E = r_ij.shape[0]
    KP = kp(n_rbf)
    dev = r_ij.device
    phi = torch.empty((E, KP), dtype=torch.float32, device=dev)
    dphi = torch.empty((E, KP), dtype=torch.float32, device=dev) if need_grad else None
    geo = torch.empty((E, GEO_STRIDE), dtype=torch.float32, device=dev)
    _lib.call("spk_edge_geometry", _p(r_ij), _p(graph.slot_eid) if graph is not None else None, E, rbf_kind, n_rbf,
              _p(f32(p0)), _p(f32(p1)) if p1 is not None else None, float(cutoff),
              _p(graph.rowptr[graph.n_atoms:]) if active_only else None, _p(phi), _p(dphi), _p(geo), _stream())
    return phi, dphi, geo


def rbf(d: Tensor, rbf_kind: int, p0: Tensor, p1: Optional[Tensor], need_grad: bool = False):
    f32(d, "d")
    n_rbf = p0.shape[0]
    out = torch.empty(tuple(d.shape) + (n_rbf,), dtype=torch.float32, device=d.device)
    dout = torch.empty_like(out) if need_grad else None
    _lib.call("spk_rbf_fwd", _p(d), d.numel(), rbf_kind, n_rbf, _p(f32(p0)), _p(f32(p1)) if p1 is not None else None,
              _p(out), _p(dout), _stream())
    return out, dout


def cosine_cutoff(d: Tensor, cutoff: float, need_grad: bool = False):
    f32(d, "d")
    out = torch.empty_like(d)
    dout = torch.empty_like(d) if need_grad else None
    _lib.call("spk_cosine_cutoff_fwd", _p(d), d.numel(), float(cutoff), _p(out), _p(dout), _stream())
    return out, dout


def activation(x: Tensor, act: int, need_grad: bool = False):
    f32(x, "x")
    y = torch.empty_like(x)
    dy = torch.empty_like(x) if need_grad else None
    _lib.call("spk_act_fwd", _p(x), x.numel(), act, _p(y), _p(dy), _stream())
    return y, dy


def embedding(table: Tensor, Z: Tensor) -> Tensor:
    f32(table, "embedding.weight")
    i64(Z, "_atomic_numbers")
    out = torch.empty((Z.shape[0], table.shape[1]), dtype=torch.float32, device=table.device)
    _lib.call("spk_embedding", _p(table), _p(Z), Z.shape[0], table.shape[1], table.shape[0], _p(out), _stream())
    return out


def segment_sum(x: Tensor, rowptr: Tensor, slot_eid: Optional[Tensor], n_out: int) -> Tensor:
    f32(x, "x")
    C = 1
    for d in x.shape[1:]:
        C *= int(d)
    out = torch.empty((n_out,) + tuple(x.shape[1:]), dtype=torch.float32, device=x.device)
    _lib.call("spk_segment_sum", _p(x), _p(rowptr), _p(slot_eid), n_out, max(C, 1), _p(out), _stream())
    return out


def add(a: Tensor, b: Optional[Tensor], out: Optional[Tensor] = None) -> Tensor:
    f32(a)
    if out is None:
        out = torch.empty_like(a)
    _lib.call("spk_add", _p(a), _p(b), a.numel(), _p(out), _stream())
    return out


# ------------------------------------------------------------------------------------------------------------ dense
def dense(A: Tensor, B: Tensor, bias: Optional[Tensor] = None, act: int = ACT_NONE, a_pre: Optional[Tensor] = None,
          a_act: int = ACT_NONE, addend: Optional[Tensor] = None, save_pre: bool = False, k: Optional[int] = None,
          out: Optional[Tensor] = None):
    """Y = act((A .* act'(a_pre)) @ B + bias) + addend ; A [M,lda] (first k columns used), B [K,N] contiguous.
    ``out`` [M, ldy>=N] may be given (padded outputs).  Returns Y or (Y, pre)."""
    f32(A, "A")
    f32(B, "B")
    M, lda = A.shape
    K = lda if k is None else int(k)
    K2, N = B.shape
    if K2 != K:
        raise ValueError(f"dense: inner dimensions differ ({K} vs {K2})")
    if out is None:
        Y = torch.empty((M, N), dtype=torch.float32, device=A.device)
    else:
        Y = f32(out, "out")
        if Y.shape[0] != M or Y.shape[1] < N:
            raise ValueError("dense: bad output buffer")
    ldy = Y.shape[1]
    pre = torch.empty_like(Y) if save_pre else None
    if addend is not None and (addend.shape[0] != M or addend.shape[1] != N):
        raise ValueError("dense: addend shape mismatch")
    _lib.call("spk_dense", _p(A), M, K, lda, _p(a_pre), a_act, _p(B), N, _p(bias), act, _p(addend), N, _p(Y), ldy,
              _p(pre), _stream())
    return (Y, pre) if save_pre else Y


def tc_pack_weight(w: Tensor) -> Tensor:
    """Pack W [N,K] into the tensor-core kernel's operand tiles (hi|lo TF32 split, shared-memory layout)."""
    f32(w, "weight")
    N, K = w.shape
    out = torch.empty(_lib.lib().spk_tc_packed_floats(N, K), dtype=torch.float32, device=w.device)
    _lib.call("spk_tc_pack_weight", _p(w), N, K, _p(out), _stream())
    return out


def dense_tc(A: Tensor, w_packed: Tensor, n_out: int, bias: Optional[Tensor] = None, act: int = ACT_NONE,
             a_pre: Optional[Tensor] = None, a_act: int = ACT_NONE, addend: Optional[Tensor] = None,
             save_pre: bool = False, k: Optional[int] = None, out: Optional[Tensor] = None):
    """wgmma / 3xTF32 variant of ``dense``: Y = act((A .* act'(a_pre)) @ W^T + bias) + addend with W [n_out, K] given
    in packed form (``tc_pack_weight``)."""
    f32(A, "A")
    M, lda = A.shape
    K = lda if k is None else int(k)
    N = int(n_out)
    if out is None:
        Y = torch.empty((M, N), dtype=torch.float32, device=A.device)
    else:
        Y = f32(out, "out")
        if Y.shape[0] != M or Y.shape[1] < N:
            raise ValueError("dense_tc: bad output buffer")
    ldy = Y.shape[1]
    pre = torch.empty_like(Y) if save_pre else None
    if addend is not None and (addend.shape[0] != M or addend.shape[1] != N):
        raise ValueError("dense_tc: addend shape mismatch")
    _lib.call("spk_dense_tc", _p(A), M, K, lda, _p(a_pre), a_act, _p(f32(w_packed)), N, _p(bias), act, _p(addend), N,
              _p(Y), ldy, _p(pre), _stream())
    return (Y, pre) if save_pre else Y


def split_tf32(w: Tensor):
    """hi = round-to-nearest(ties away) TF32 of w (low 13 mantissa bits cleared), lo = w - hi (exact in fp32)."""
    bits = w.contiguous().view(torch.int32)
    hi = ((bits + 0x1000) & -8192).view(torch.float32)
    return hi.contiguous(), (w - hi).contiguous()


# dense-layer kernel (both meet the 1e-5 parity bar; r1: equal speed on cfg2 within run-to-run noise):
#   "tc"   (default) wgmma 3xTF32 tensor-core kernel csrc/gemm_tc.cu -- fresh accumulator per K-tile added in fp32 gives
#          fp32-grade error; shapes outside its vector fast path fall back to "ffma" per call
#   "ffma" fp32 CUDA-core kernel csrc/gemm.cu (packed FFMA2, IEEE fp32 accumulation like the reference SGEMM)
DENSE_IMPL = os.environ.get("SPK_B200_DENSE", "tc")


class Lin:
    """Kernel-ready copy of one Dense layer: W [N,K], W^T [K,N], bias, and their TF32 hi/lo splits."""

    __slots__ = ("w", "wt", "b", "w_pk", "wt_pk")

    def __init__(self, weight: Tensor, bias: Optional[Tensor] = None):
        self.w = weight.detach().contiguous()
        self.wt = weight.detach().t().contiguous()
        self.b = bias.detach().contiguous() if bias is not None else None
        self.w_pk = self.wt_pk = None
        if DENSE_IMPL == "tc" and self.w.is_cuda:
            self.w_pk = tc_pack_weight(self.w)
            self.wt_pk = tc_pack_weight(self.wt)

    @staticmethod
    def _tc_ok(A: Tensor, n_out: int, act: int, bias: Optional[Tensor], kw) -> bool:
        """calls the tensor-core kernel's vector fast path covers; spk_dense_tc refuses every other one, and the fp32
        kernel runs it: K, N, lda and ldy multiples of 4, 16 B-aligned base pointers, and not both a backward prologue
        (a_act) and a forward activation"""
        k = kw.get("k")
        K = A.shape[1] if k is None else int(k)
        out = kw.get("out")
        ldy = n_out if out is None else out.shape[1]
        if K % 4 or n_out % 4 or A.shape[1] % 4 or ldy % 4:
            return False
        a_pre = kw.get("a_pre")
        if a_pre is not None and kw.get("a_act", ACT_NONE) != ACT_NONE and (act & ~SAVE_DERIV) != ACT_NONE:
            return False
        return all(t.data_ptr() % 16 == 0 for t in (A, a_pre, bias, kw.get("addend"), out) if t is not None)

    def fwd(self, A: Tensor, act: int = ACT_NONE, save_deriv: bool = False, **kw):
        """act(A W^T + b) [+ addend].  ``save_deriv=True`` returns (Y, act'(pre)): the tensor the input-gradient layer
        multiplies by (``bwd(G, a_pre=deriv, a_act=ACT_GIVEN)``) without re-evaluating the activation."""
        if save_deriv:
            kw["save_pre"] = True
            act = act | SAVE_DERIV
        if self.w_pk is not None and self._tc_ok(A, self.w.shape[0], act, self.b, kw):
            return dense_tc(A, self.w_pk, self.w.shape[0], self.b, act, **kw)
        return dense(A, self.wt, self.b, act, **kw)

    def bwd(self, G: Tensor, **kw):
        """(G .* act'(a_pre)) W [+ addend]  -- input gradient of the layer"""
        if self.wt_pk is not None and self._tc_ok(G, self.wt.shape[0], ACT_NONE, None, kw):
            return dense_tc(G, self.wt_pk, self.wt.shape[0], None, ACT_NONE, **kw)
        return dense(G, self.w, None, ACT_NONE, **kw)


# bench.py reports this in impl_switches; there is no chain path, so it is always False.
CHAIN_IMPL = False


# ------------------------------------------------------------------------------------------------------------ PaiNN
# edge kernels: "tc" (default) = persistent kernels with the continuous filter on the tensor cores (csrc/painn_tc.cu:
# wgmma 3xTF32, channels on the M side) for F == 128, n_rbf <= 23 and >= EDGE_TC_MIN_EDGES edges; everything else, and
# SPK_B200_EDGE=ldg, runs the streaming kernels with the filter on the CUDA cores (csrc/painn.cu).
EDGE_IMPL = os.environ.get("SPK_B200_EDGE", "tc")
EDGE_TC_MIN_EDGES = 4096


def edge_tc_ok(F: int, n_rbf: int, n_edges: int) -> bool:
    """The tensor-core filter path (csrc/painn_tc.cu) covers F == 128, n_rbf <= 23 (its filter GEMM has K = n_rbf + 1 <=
    24); tiny edge lists stay on the streaming kernel (a persistent CTA per SM needs work for its 4 consumer groups)."""
    return EDGE_IMPL == "tc" and F == 128 and n_rbf <= 23 and n_edges >= EDGE_TC_MIN_EDGES


def painn_pack_filter(wf: Tensor, bf: Tensor, F: int, n_rbf: int) -> Tensor:
    out = torch.empty(_lib.lib().spk_painn_filter_packed_floats(), dtype=torch.float32, device=wf.device)
    _lib.call("spk_painn_pack_filter", _p(f32(wf, "wf")), _p(f32(bf, "bf")), F, n_rbf, _p(out), _stream())
    return out


def painn_edge_fwd(x, mu, q, phi, geo, graph: EdgeGraph, wf, bf, F: int, n_rbf: int, wf_packed=None,
                   n_rows: Optional[int] = None):
    """``n_rows``: number of RECEIVER rows (default: every atom of the graph).  A partition that appends read-only ghost
    senders after its owned atoms passes the owned count: the kernels then never walk the edge-free ghost rows (16 k empty
    rows at the end of the last CTA's range cost 2.5 ms at cfg5 / 2 GPUs) and ``q`` / the outputs have ``n_rows`` rows."""
    N = graph.n_atoms if n_rows is None else int(n_rows)
    q_out = torch.empty((N, F), dtype=torch.float32, device=x.device)
    mu_out = torch.empty((N, 3, F), dtype=torch.float32, device=x.device)
    if wf_packed is not None and edge_tc_ok(F, n_rbf, graph.n_edges):
        _lib.call("spk_painn_edge_fwd_tc", _p(x), _p(mu), _p(q), _p(phi), _p(geo), _p(graph.rowptr), _p(graph.slot_j),
                  _p(wf_packed), N, graph.n_edges, F, n_rbf, _p(q_out), _p(mu_out), _stream())
    else:
        _lib.call("spk_painn_edge_fwd", _p(x), _p(mu), _p(q), _p(phi), _p(geo), _p(graph.rowptr), _p(graph.slot_j),
                  _p(wf), _p(bf), N, graph.n_edges, F, n_rbf, _p(q_out), _p(mu_out), _stream())
    return q_out, mu_out


def painn_edge_bwd(x, mu, g_q, g_mu, phi, dphi, geo, graph: EdgeGraph, wf, bf, F: int, n_rbf: int, g_rij: Tensor,
                   accumulate: bool, wf_packed=None):
    N = graph.n_atoms
    g_x = torch.empty((N, 3 * F), dtype=torch.float32, device=x.device)
    g_mu_in = torch.empty((N, 3, F), dtype=torch.float32, device=x.device) if mu is not None else None
    if wf_packed is not None and edge_tc_ok(F, n_rbf, graph.n_edges):
        _lib.call("spk_painn_edge_bwd_tc", _p(x), _p(mu), _p(g_q), _p(g_mu), _p(phi), _p(dphi), _p(geo), _p(graph.sptr),
                  _p(graph.pos_slot), _p(graph.pos_i), _p(graph.slot_eid), _p(wf_packed), N, graph.n_edges, F, n_rbf,
                  _p(g_x), _p(g_mu_in), _p(g_rij), 1 if accumulate else 0, _stream())
    else:
        _lib.call("spk_painn_edge_bwd", _p(x), _p(mu), _p(g_q), _p(g_mu), _p(phi), _p(dphi), _p(geo), _p(graph.sptr), _p(graph.pos_slot), _p(graph.pos_i), _p(graph.slot_eid), _p(wf), _p(bf), N,
                  graph.n_edges, F, n_rbf, _p(g_x), _p(g_mu_in), _p(g_rij), 1 if accumulate else 0, _stream())
    return g_x, g_mu_in


def painn_edge_wij_fwd(x, mu, q, Wij, dir_ij, graph: EdgeGraph, F: int):
    """Block-level interaction with a materialised filter Wij [E,3F] / dir_ij [E,3] in the caller's edge order."""
    N = graph.n_atoms
    q_out = torch.empty((N, F), dtype=torch.float32, device=x.device)
    mu_out = torch.empty((N, 3, F), dtype=torch.float32, device=x.device)
    _lib.call("spk_painn_edge_wij_fwd", _p(f32(x)), _p(f32(mu)), _p(f32(q)), _p(f32(Wij, "Wij")), _p(f32(dir_ij, "dir_ij")),
              _p(graph.rowptr), _p(graph.slot_j), _p(graph.slot_eid), N, graph.n_edges, F, _p(q_out), _p(mu_out), _stream())
    return q_out, mu_out


def painn_edge_wij_bwd(x, mu, g_q, g_mu, Wij, dir_ij, graph: EdgeGraph, F: int):
    N, E = graph.n_atoms, graph.n_edges
    dev = x.device
    g_x = torch.empty((N, 3 * F), dtype=torch.float32, device=dev)
    g_mu_in = torch.empty((N, 3, F), dtype=torch.float32, device=dev)
    g_W = torch.empty((E, 3 * F), dtype=torch.float32, device=dev)
    g_dir = torch.empty((E, 3), dtype=torch.float32, device=dev)
    _lib.call("spk_painn_edge_wij_bwd", _p(f32(x)), _p(f32(mu)), _p(f32(g_q)), _p(f32(g_mu)), _p(f32(Wij)), _p(f32(dir_ij)),
              _p(graph.sptr), _p(graph.pos_slot), _p(graph.pos_i), _p(graph.slot_eid), N, E, F, _p(g_x), _p(g_mu_in),
              _p(g_W), _p(g_dir), _stream())
    return g_x, g_mu_in, g_W, g_dir


def painn_mix_ctx(q, VW, F: int, eps: float):
    N = q.shape[0]
    ctx = torch.empty((N, 2 * F), dtype=torch.float32, device=q.device)
    _lib.call("spk_painn_mix_ctx", _p(q), _p(VW), N, F, float(eps), _p(ctx), _stream())
    return ctx


def painn_mix_update(q, mu, s, VW, F: int):
    N = q.shape[0]
    q_out = torch.empty_like(q)
    mu_out = torch.empty_like(mu)
    _lib.call("spk_painn_mix_update", _p(q), _p(mu), _p(s), _p(VW), N, F, _p(q_out), _p(mu_out), _stream())
    return q_out, mu_out


def painn_mix_update_bwd(g_q, g_mu, s, VW, F: int):
    N = g_q.shape[0]
    g_s = torch.empty((N, 3 * F), dtype=torch.float32, device=g_q.device)
    g_VW = torch.empty((N, 3, 2 * F), dtype=torch.float32, device=g_q.device)
    _lib.call("spk_painn_mix_update_bwd", _p(g_q), _p(g_mu), _p(s), _p(VW), N, F, _p(g_s), _p(g_VW), _stream())
    return g_s, g_VW


def painn_mix_ctx_bwd(g_ctx, g_q, VW, g_VW, F: int, eps: float):
    N = g_q.shape[0]
    g_q_out = torch.empty_like(g_q)
    _lib.call("spk_painn_mix_ctx_bwd", _p(g_ctx), _p(g_q), _p(VW), N, F, float(eps), _p(g_q_out), _p(g_VW), _stream())
    return g_q_out


# ------------------------------------------------------------------------------------------------------------ SchNet
def cfconv_fwd(h, w_raw, geo, graph: EdgeGraph, F: int):
    N = graph.n_atoms
    m = torch.empty((N, F), dtype=torch.float32, device=h.device)
    _lib.call("spk_cfconv_fwd", _p(h), _p(w_raw), _p(geo), _p(graph.rowptr), _p(graph.slot_j), N, graph.n_edges, F,
              _p(m), _stream())
    return m


# fused forward block (csrc/schnet_tc.cu): filter network on wgmma inside the edge kernel; F == n_filters == 128, n_rbf <= 31.
# SPK_B200_CFCONV=mat restores the materialised-filter pipeline (two dense kernels over [E, .] + spk_cfconv_fwd).
CFCONV_IMPL = os.environ.get("SPK_B200_CFCONV", "tc")
CFCONV_TC_MIN_EDGES = 2048


def cfconv_tc_ok(F: int, n_filters: int, n_rbf: int, n_edges: int) -> bool:
    return CFCONV_IMPL == "tc" and F == 128 and n_filters == 128 and n_rbf <= 31 and n_edges >= CFCONV_TC_MIN_EDGES


# ------------------------------------------------------------------------------------------------------------ shapes
# Widths the per-channel edge kernels are compiled for: one thread per channel, F / 32 warps in {1, 2, 4, 8}
# (DISPATCH_F_NRB of csrc/painn.cu, k_cfconv_{fwd,bwd}<NW> of csrc/schnet.cu).  The radial-basis records of the PaiNN
# edge kernels and of spk_radial_bwd hold at most 32 functions.
EDGE_WIDTHS = (32, 64, 128, 256)
MAX_N_RBF = 32


def check_painn_shape(F: int, n_rbf: int):
    """Raise NotImplementedError, before anything is launched, for a PaiNN the edge kernels cannot evaluate."""
    if F not in EDGE_WIDTHS:
        raise NotImplementedError(f"PaiNN: n_atom_basis = {F} has no edge kernel (supported: {EDGE_WIDTHS})")
    if n_rbf > MAX_N_RBF:
        raise NotImplementedError(f"PaiNN: n_rbf = {n_rbf} has no edge kernel (supported: n_rbf <= {MAX_N_RBF})")


def check_schnet_shape(n_filters: int, n_rbf: int, need_grad: bool):
    """Raise NotImplementedError, before anything is launched, for a SchNet evaluation the kernels cannot run: the
    convolution needs one of EDGE_WIDTHS filters, and the radial reverse (forces) at most MAX_N_RBF basis functions.
    Energy-only evaluations with more basis functions run on the materialised-filter path."""
    if n_filters not in EDGE_WIDTHS:
        raise NotImplementedError(f"SchNet: n_filters = {n_filters} has no convolution kernel (supported: {EDGE_WIDTHS})")
    if need_grad and n_rbf > MAX_N_RBF:
        raise NotImplementedError(f"SchNet: n_rbf = {n_rbf} has no radial reverse kernel for forces "
                                  f"(supported: n_rbf <= {MAX_N_RBF}; energy-only evaluations take any n_rbf)")


def schnet_pack_filter(w0: Tensor, b0: Tensor, w1: Tensor, n_rbf: int) -> Tensor:
    out = torch.empty(_lib.lib().spk_schnet_filter_packed_floats(), dtype=torch.float32, device=w0.device)
    _lib.call("spk_schnet_pack_filter", _p(f32(w0)), _p(f32(b0)), _p(f32(w1)), w1.shape[0], n_rbf, _p(out), _stream())
    return out


def schnet_cfconv_fwd_tc(h, phi, geo, graph: EdgeGraph, filter_packed, b1, act: int, n_rbf: int):
    N, F = graph.n_atoms, h.shape[1]
    m = torch.empty((N, F), dtype=torch.float32, device=h.device)
    _lib.call("spk_schnet_cfconv_fwd_tc", _p(f32(h)), _p(phi), _p(geo), _p(graph.rowptr), _p(graph.slot_j),
              _p(filter_packed), _p(b1), act, N, graph.n_edges, F, n_rbf, _p(m), _stream())
    return m


def cfconv_bwd(h, w_raw, geo, g_m, graph: EdgeGraph, F: int):
    N, E = graph.n_atoms, graph.n_edges
    g_h = torch.empty((N, F), dtype=torch.float32, device=h.device)
    g_wraw = torch.empty((E, F), dtype=torch.float32, device=h.device)
    g_fc = torch.empty((E,), dtype=torch.float32, device=h.device)
    _lib.call("spk_cfconv_bwd", _p(h), _p(w_raw), _p(geo), _p(g_m), _p(graph.sptr), _p(graph.pos_slot),
              _p(graph.pos_i), N, E, F, _p(g_h), _p(g_wraw), _p(g_fc), _stream())
    return g_h, g_wraw, g_fc


def radial_bwd(g_phi, g_fc, dphi, geo, graph: Optional[EdgeGraph], n_rbf: int, g_rij: Tensor, accumulate: bool):
    E = geo.shape[0]
    _lib.call("spk_radial_bwd", _p(g_phi), _p(g_fc), _p(dphi), _p(geo),
              _p(graph.slot_eid) if graph is not None else None, E, n_rbf, _p(g_rij), 1 if accumulate else 0,
              _stream())
    return g_rij


# ------------------------------------------------------------------------------------------------------------ head
def atomwise_out(hid, w1, b1, mol_ptr: Optional[Tensor], n_mol: int):
    N, H = hid.shape
    y = torch.empty((N,), dtype=torch.float32, device=hid.device)
    energy = torch.empty((n_mol,), dtype=torch.float32, device=hid.device) if mol_ptr is not None else None
    _lib.call("spk_atomwise_out", _p(hid), _p(w1), _p(b1), _p(mol_ptr), N, n_mol if mol_ptr is not None else 0, H,
              _p(y), _p(energy), _stream())
    return y, energy


def atomwise_out_bwd(g_energy: Optional[Tensor], idx_m: Optional[Tensor], w1, n_atoms: int, H: int):
    g_hid = torch.empty((n_atoms, H), dtype=torch.float32, device=w1.device)
    _lib.call("spk_atomwise_out_bwd", _p(g_energy), _p(idx_m), _p(w1), n_atoms, H, _p(g_hid), _stream())
    return g_hid


# ------------------------------------------------------------------------------------------------------------ SO3net
def so3_conv_fwd(x, phi, geo, graph: EdgeGraph, wf, bf, lmax: int, F: int, n_rbf: int):
    """SO3Convolution of one interaction block: x [N,S,F] -> y [N,S,F], filter evaluated in-kernel."""
    N, S = graph.n_atoms, (lmax + 1) ** 2
    y = torch.empty((N, S, F), dtype=torch.float32, device=x.device)
    _lib.call("spk_so3_conv_fwd", _p(x), _p(phi), _p(geo), _p(graph.rowptr), _p(graph.slot_j), _p(wf), _p(bf), N,
              graph.n_edges, lmax, F, n_rbf, _p(y), _stream())
    return y


def so3_conv_bwd(x, g_y, phi, dphi, geo, graph: EdgeGraph, wf, bf, lmax: int, F: int, n_rbf: int,
                 g_res: Optional[Tensor], g_rij: Tensor, accumulate: bool, need_gx: bool = True):
    """(dE/dy, residual dE/dx) -> dE/dx_in [N,S,F] (None unless ``need_gx``); dE/dr_ij written or added to ``g_rij``."""
    N, S = graph.n_atoms, (lmax + 1) ** 2
    g_x = torch.empty((N, S, F), dtype=torch.float32, device=x.device) if need_gx else None
    _lib.call("spk_so3_conv_bwd", _p(x), _p(g_y), _p(phi), _p(dphi), _p(geo), _p(graph.sptr), _p(graph.pos_slot),
              _p(graph.pos_i), _p(graph.slot_eid), _p(wf), _p(bf), N, graph.n_edges, lmax, F, n_rbf, _p(g_res), _p(g_x),
              _p(g_rij), 1 if accumulate else 0, _stream())
    return g_x


def so3_tp_fwd(dx, ddx, lmax: int, F: int):
    out = torch.empty_like(dx)
    _lib.call("spk_so3_tp_fwd", _p(dx), _p(ddx), dx.shape[0], lmax, F, _p(out), _stream())
    return out


def so3_tp_bwd(g, dx, ddx, lmax: int, F: int):
    g_dx = torch.empty_like(dx)
    g_ddx = torch.empty_like(dx)
    _lib.call("spk_so3_tp_bwd", _p(g), _p(dx), _p(ddx), dx.shape[0], lmax, F, _p(g_dx), _p(g_ddx), _stream())
    return g_dx, g_ddx


def so3_gate_fwd(x, h, lmax: int, F: int):
    y = torch.empty_like(x)
    _lib.call("spk_so3_gate_fwd", _p(x), _p(h), x.shape[0], lmax, F, _p(y), _stream())
    return y


def so3_gate_bwd(g_y, x, h, lmax: int, F: int):
    """-> (dE/dx [N,S,F] with row 0 left for the caller, dE/dx row 0 through the gate [N,F], dE/dh [N,(lmax+1)F])"""
    N = x.shape[0]
    g_x = torch.empty_like(x)
    g_x0 = torch.empty((N, F), dtype=torch.float32, device=x.device)
    g_h = torch.empty_like(h)
    _lib.call("spk_so3_gate_bwd", _p(g_y), _p(x), _p(h), N, lmax, F, _p(g_x), _p(g_x0), _p(g_h), _stream())
    return g_x, g_x0, g_h


def so3_put_l0(src: Optional[Tensor], v: Optional[Tensor], n_atoms: int, lmax: int, F: int, device):
    out = torch.empty((n_atoms, (lmax + 1) ** 2, F), dtype=torch.float32, device=device)
    _lib.call("spk_so3_put_l0", _p(src), _p(v), n_atoms, lmax, F, _p(out), _stream())
    return out


def so3_take_l0(x, lmax: int, F: int):
    q = torch.empty((x.shape[0], F), dtype=torch.float32, device=x.device)
    _lib.call("spk_so3_take_l0", _p(x), x.shape[0], lmax, F, _p(q), _stream())
    return q


# ------------------------------------------------------------------------------------------------------------ output heads
HEAD_DIPOLE, HEAD_POLAR = _lib.CONSTANTS["SPK_HEAD_DIPOLE"], _lib.CONSTANTS["SPK_HEAD_POLAR"]


def geq_ctx(s: Tensor, VW: Tensor, Fi: int, Fo: int) -> Tensor:
    """[s | ||V||] of a GatedEquivariantBlock (VW = mix_vectors(V) [N,3,2Fo])."""
    N = s.shape[0]
    ctx = torch.empty((N, Fi + Fo), dtype=torch.float32, device=s.device)
    _lib.call("spk_geq_ctx", _p(f32(s, "s")), _p(f32(VW, "VW")), N, Fi, Fo, _p(ctx), _stream())
    return ctx


def geq_ctx_bwd(g_ctx: Tensor, VW: Tensor, g_VW: Tensor, Fi: int, Fo: int) -> Tensor:
    """-> g_s [N,Fi]; writes the V columns of g_VW"""
    N = g_ctx.shape[0]
    g_s = torch.empty((N, Fi), dtype=torch.float32, device=g_ctx.device)
    _lib.call("spk_geq_ctx_bwd", _p(f32(g_ctx, "g_ctx")), _p(VW), N, Fi, Fo, _p(g_s), _p(g_VW), _stream())
    return g_s


def geq_gate(x: Tensor, VW: Tensor, Fo: int, act: int):
    N = x.shape[0]
    s_out = torch.empty((N, Fo), dtype=torch.float32, device=x.device)
    v_out = torch.empty((N, 3, Fo), dtype=torch.float32, device=x.device)
    _lib.call("spk_geq_gate", _p(f32(x, "x")), _p(f32(VW, "VW")), N, Fo, act, _p(s_out), _p(v_out), _stream())
    return s_out, v_out


def geq_gate_bwd(g_s: Optional[Tensor], g_v: Optional[Tensor], x: Tensor, VW: Tensor, Fo: int, act: int):
    """-> (g_x [N,2Fo], g_VW [N,3,2Fo] with the W columns written)"""
    N = x.shape[0]
    g_x = torch.empty((N, 2 * Fo), dtype=torch.float32, device=x.device)
    g_VW = torch.empty((N, 3, 2 * Fo), dtype=torch.float32, device=x.device)
    _lib.call("spk_geq_gate_bwd", _p(g_s), _p(g_v), _p(x), _p(VW), N, Fo, act, _p(g_x), _p(g_VW), _stream())
    return g_x, g_VW


def head_tail(wmix: Tensor, w0: Tensor, b0: Tensor, w1: Tensor, b1: Tensor, act: int):
    """Kernel-ready weights of the last gated block (n_sout = n_vout = 1); returns (struct, tensors kept alive)."""
    keep = [f32(t.detach().contiguous(), "weight") for t in (wmix, w0, w0.t(), b0, w1, b1)]
    st = _lib.HeadTail()
    st.wmix, st.w0, st.w0t, st.b0, st.w1, st.b1 = (t.data_ptr() for t in keep)
    st.Fi, st.H, st.act = int(wmix.shape[1]), int(w0.shape[0]), int(act)
    return st, keep


def head_fwd(kind: int, tail, s: Optional[Tensor], V: Optional[Tensor], q: Optional[Tensor], R: Tensor, idx_m: Tensor,
             sys_ptr: Tensor, total_charge: Optional[Tensor], n_sys: int, correct: bool, magnitude: bool,
             want_q: bool):
    """-> (out [B,3] / [B] / [B,3,3], q_atom [N] or None, saved [B,8] fp64)"""
    N = R.shape[0]
    dev = R.device
    shape = (n_sys, 3, 3) if kind == HEAD_POLAR else ((n_sys,) if magnitude else (n_sys, 3))
    out = torch.empty(shape, dtype=torch.float32, device=dev)
    saved = torch.empty((n_sys, 8), dtype=torch.float64, device=dev)
    q_atom = torch.empty((N,), dtype=torch.float32, device=dev) if want_q and tail is not None else None
    nbytes = int(_lib.lib().spk_head_workspace_bytes(N, n_sys))
    ws = torch.empty(max(nbytes, 8), dtype=torch.uint8, device=dev)
    _lib.call("spk_head_fwd", kind, tail, _p(s), _p(V), _p(q), _p(f32(R, "_positions")), _p(i64(idx_m, "_idx_m")),
              _p(sys_ptr), _p(total_charge), N, n_sys, int(correct), int(magnitude), _p(out), _p(q_atom), _p(saved),
              _p(ws), nbytes, _stream(), launches=2 if N > 0 else 1)
    return out, q_atom, saved


def head_charges(q_atom: Tensor, idx_m: Tensor, saved: Tensor) -> Tensor:
    charges = torch.empty_like(q_atom)
    _lib.call("spk_head_charges", _p(q_atom), _p(idx_m), _p(saved), q_atom.shape[0], _p(charges), _stream())
    return charges


def head_bwd(kind: int, tail, s: Tensor, V: Tensor, R: Tensor, idx_m: Tensor, saved: Tensor, g_out: Tensor,
             correct: bool, magnitude: bool):
    N, Fi = s.shape
    dev = s.device
    g_s = torch.empty((N, Fi), dtype=torch.float32, device=dev)
    g_V = torch.empty((N, 3, Fi), dtype=torch.float32, device=dev)
    g_R = torch.empty((N, 3), dtype=torch.float32, device=dev)
    _lib.call("spk_head_bwd", kind, tail, _p(s), _p(V), _p(R), _p(idx_m), _p(saved), _p(f32(g_out, "g_out")), N,
              int(correct), int(magnitude), _p(g_s), _p(g_V), _p(g_R), _stream())
    return g_s, g_V, g_R


def head_scalar_bwd(q: Tensor, R: Tensor, idx_m: Tensor, saved: Tensor, g_out: Tensor, correct: bool, magnitude: bool,
                    w1: Tensor):
    N, H = q.shape[0], w1.numel()
    g_hid = torch.empty((N, H), dtype=torch.float32, device=q.device)
    g_R = torch.empty((N, 3), dtype=torch.float32, device=q.device)
    _lib.call("spk_head_scalar_bwd", _p(q), _p(R), _p(idx_m), _p(saved), _p(f32(g_out, "g_out")), int(correct),
              int(magnitude), _p(w1), N, H, _p(g_hid), _p(g_R), _stream())
    return g_hid, g_R


def head_charges_bwd(g_charges: Tensor, idx_m: Tensor, sys_ptr: Tensor, n_sys: int, correct: bool) -> Tensor:
    """Reverse of the charge correction: g_q = g_charges - per-system mean (fp64 sums) with ``correct``."""
    N = g_charges.shape[0]
    g_q = torch.empty_like(g_charges)
    nbytes = int(_lib.lib().spk_head_charges_bwd_workspace_bytes(N, n_sys))
    ws = torch.empty(max(nbytes, 8), dtype=torch.uint8, device=g_charges.device)
    _lib.call("spk_head_charges_bwd", _p(f32(g_charges, "g_charges")), _p(idx_m), _p(sys_ptr), N, n_sys, int(correct),
              _p(g_q), _p(ws), nbytes, _stream(), launches=3 if correct and n_sys > 0 else 1)
    return g_q


def head_bwd_q(tail, s: Tensor, V: Tensor, R: Tensor, idx_m: Tensor, saved: Tensor, g_out: Tensor, g_q: Tensor,
               correct: bool, magnitude: bool):
    """``head_bwd`` of the dipole with the charges' own gradient ``g_q`` [N] added."""
    N, Fi = s.shape
    dev = s.device
    g_s = torch.empty((N, Fi), dtype=torch.float32, device=dev)
    g_V = torch.empty((N, 3, Fi), dtype=torch.float32, device=dev)
    g_R = torch.empty((N, 3), dtype=torch.float32, device=dev)
    _lib.call("spk_head_bwd_q", HEAD_DIPOLE, tail, _p(s), _p(V), _p(R), _p(idx_m), _p(saved), _p(f32(g_out, "g_out")),
              _p(f32(g_q, "g_q")), N, int(correct), int(magnitude), _p(g_s), _p(g_V), _p(g_R), _stream())
    return g_s, g_V, g_R


def head_scalar_bwd_q(q: Tensor, R: Tensor, idx_m: Tensor, saved: Tensor, g_out: Tensor, g_q: Tensor, correct: bool,
                      magnitude: bool, w1: Tensor):
    """``head_scalar_bwd`` with the charges' own gradient ``g_q`` [N] added."""
    N, H = q.shape[0], w1.numel()
    g_hid = torch.empty((N, H), dtype=torch.float32, device=q.device)
    g_R = torch.empty((N, 3), dtype=torch.float32, device=q.device)
    _lib.call("spk_head_scalar_bwd_q", _p(q), _p(R), _p(idx_m), _p(saved), _p(f32(g_out, "g_out")), _p(f32(g_q, "g_q")),
              int(correct), int(magnitude), _p(w1), N, H, _p(g_hid), _p(g_R), _stream())
    return g_hid, g_R


# ------------------------------------------------------------------------------------------------------------ pair energies
PAIR_ZBL, PAIR_COULOMB, PAIR_DAMPED_COULOMB = _lib.PAIR_ZBL, _lib.PAIR_COULOMB, _lib.PAIR_DAMPED_COULOMB
PAIR_EWALD_REAL = _lib.PAIR_EWALD_REAL


def pair_params(kind: int, ke: float, cutoff: Optional[float] = None, shift: float = 0.0, switch_on: float = 0.0,
                switch_off: float = 0.0, d_max: Optional[float] = None, zbl=None, alpha: float = 0.0):
    """``spk_pair_t`` for a pair term; ``zbl`` = (a_pow, a_div, coefficients, exponents) device tensors, read by the kernels
    at every launch (a captured graph sees updated values).  Returns (struct, tensors kept alive)."""
    st = _lib.PairParams()
    st.kind = int(kind)
    keep = []
    if zbl is not None:
        keep = [f32(t.detach(), name) for t, name in zip(zbl, ("a_pow", "a_div", "coefficients", "exponents"))]
        if keep[2].numel() != keep[3].numel() or not 0 < keep[2].numel() <= _lib.PAIR_MAX_TERMS:
            raise ValueError(f"ZBL: coefficients and exponents must have equal length <= {_lib.PAIR_MAX_TERMS}")
        st.a_pow, st.a_div, st.coefficients, st.exponents = (t.data_ptr() for t in keep)
        st.n_terms = int(keep[2].numel())
    st.ke = float(ke)
    st.cutoff = float(cutoff) if cutoff is not None else 0.0
    st.shift = float(shift)
    st.switch_on, st.switch_off = float(switch_on), float(switch_off)
    st.d_max = float(d_max) if d_max is not None else 0.0
    st.alpha = float(alpha)
    return st, keep


def pair_energy_fwd(params, r_ij: Tensor, idx_i: Tensor, idx_j: Tensor, Z: Optional[Tensor], q: Optional[Tensor],
                    idx_m: Tensor, graph: EdgeGraph, sys_ptr: Tensor, n_sys: int) -> Tensor:
    """energy [n_sys] = 0.5 ke sum over the edges received by the atoms of each system (fp64, fixed order)."""
    dev = r_ij.device
    energy = torch.empty((n_sys,), dtype=torch.float32, device=dev)
    E = graph.n_edges
    nbytes = int(_lib.lib().spk_pair_energy_workspace_bytes(E, n_sys))
    ws = torch.empty(max(nbytes, 8), dtype=torch.uint8, device=dev)
    _lib.call("spk_pair_energy_fwd", params, _p(f32(r_ij, "_Rij")), _p(i64(idx_i)), _p(i64(idx_j)),
              _p(i64(Z, "_atomic_numbers")) if Z is not None else None, _p(f32(q, "charges")) if q is not None else None,
              _p(i64(idx_m, "_idx_m")), _p(graph.rowptr), _p(graph.slot_eid), _p(sys_ptr), E, n_sys, _p(energy), _p(ws),
              nbytes, _stream(), launches=2 if E > 0 else 1)
    return energy


def pair_energy_bwd(params, r_ij: Tensor, idx_i: Tensor, idx_j: Tensor, Z: Optional[Tensor], q: Optional[Tensor],
                    idx_m: Tensor, g_E: Tensor, graph: EdgeGraph, want_q: bool):
    """-> (g_rij [E,3] in edge order, g_q [N] or None)"""
    dev = r_ij.device
    E, N = graph.n_edges, graph.n_atoms
    g_rij = torch.empty((E, 3), dtype=torch.float32, device=dev)
    g_q = torch.empty((N,), dtype=torch.float32, device=dev) if want_q else None
    _lib.call("spk_pair_energy_bwd", params, _p(r_ij), _p(idx_i), _p(idx_j), _p(Z), _p(q), _p(idx_m),
              _p(f32(g_E, "g_E")), _p(graph.rowptr), _p(graph.slot_j), _p(graph.slot_eid), _p(graph.sptr),
              _p(graph.pos_slot), _p(graph.pos_i), N, E, _p(g_rij), _p(g_q), _stream(),
              launches=int(E > 0) + int(want_q and N > 0))
    return g_rij, g_q


# ------------------------------------------------------------------------------------------------------------ Ewald
def ewald_fwd(R: Tensor, q: Tensor, cell: Tensor, kvecs: Tensor, idx_m: Tensor, sys_ptr: Tensor, n_sys: int, ke: float,
              alpha: float, addend: Optional[Tensor] = None):
    """-> (energy [n_sys] = addend + E_rec - E_self, workspace the reverse reads)"""
    dev = R.device
    N, K = R.shape[0], kvecs.shape[0]
    energy = torch.empty((n_sys,), dtype=torch.float32, device=dev)
    nbytes = int(_lib.lib().spk_ewald_workspace_bytes(N, n_sys, K))
    ws = torch.empty(max(nbytes, 8), dtype=torch.uint8, device=dev)
    _lib.call("spk_ewald_fwd", _p(f32(R, "_positions")), _p(f32(q, "charges")), _p(f32(cell, "_cell")),
              _p(f32(kvecs, "kvecs")), _p(i64(idx_m, "_idx_m")), _p(sys_ptr), N, n_sys, K, float(ke), float(alpha),
              _p(f32(addend, "energy")) if addend is not None else None, _p(energy), _p(ws), nbytes, _stream(),
              launches=(2 if N > 0 else 1) + (1 if K > 0 else 0) + 1)
    return energy, ws


def ewald_bwd(R: Tensor, q: Tensor, cell: Tensor, kvecs: Tensor, idx_m: Tensor, sys_ptr: Tensor, n_sys: int, ke: float,
              alpha: float, g_E: Tensor, ws: Tensor, want_R: bool, g_q: Optional[Tensor], want_cell: bool,
              virial: Optional[Tensor] = None, accumulate_virial: bool = False):
    """-> (g_R [N,3] or None, g_cell [n_sys,3,3] or None); ``g_q`` [N] (the real-space charge gradient) gets the reciprocal
    and self terms added in place; ``virial`` [n_sys,3,3] fp64 gets the reciprocal virial (added with
    ``accumulate_virial``)."""
    dev = R.device
    N, K = R.shape[0], kvecs.shape[0]
    g_R = torch.empty((N, 3), dtype=torch.float32, device=dev) if want_R else None
    g_cell = torch.empty((n_sys, 3, 3), dtype=torch.float32, device=dev) if want_cell else None
    _lib.call("spk_ewald_bwd", _p(R), _p(q), _p(cell), _p(kvecs), _p(idx_m), _p(sys_ptr), N, n_sys, K, float(ke),
              float(alpha), _p(f32(g_E, "g_E")), _p(g_R), _p(g_q), 1, _p(g_cell), _p(virial), int(accumulate_virial),
              _p(ws), ws.numel(), _stream(),
              launches=(int(K > 0) + 1 if N > 0 else 0) + int(want_cell or virial is not None))
    return g_R, g_cell


# ------------------------------------------------------------------------------------------------------------ PME
PME_ORDERS = (4, 6, 8)


def pme_workspace(n_atoms: int, n_sys: int, mesh, order: int, device) -> Tensor:
    nbytes = int(_lib.lib().spk_pme_workspace_bytes(n_atoms, n_sys, *mesh, order))
    if nbytes == 0:
        raise ValueError(f"PME: invalid mesh {tuple(mesh)} or order {order}")
    return torch.empty(nbytes, dtype=torch.uint8, device=device)


def pme_fwd(R: Tensor, q: Tensor, cell: Tensor, idx_m: Tensor, sys_ptr: Tensor, n_sys: int, mesh, order: int, ke: float,
            alpha: float, addend: Optional[Tensor] = None):
    """-> (energy [n_sys] = addend + E_rec - E_self, conv [n_sys, n1, n2, n3 // 2 + 1] complex128, workspace): the charge
    mesh of csrc/pme.cu, its fp64 rfftn, and the influence pass; ``conv`` and the workspace are what the reverse reads."""
    dev = R.device
    N = R.shape[0]
    n1, n2, n3 = mesh
    ws = pme_workspace(N, n_sys, mesh, order, dev)
    Q = torch.empty((n_sys, n1, n2, n3), dtype=torch.float64, device=dev)
    R, q, cell, idx_m = f32(R, "_positions"), f32(q, "charges"), f32(cell, "_cell"), i64(idx_m, "_idx_m")
    _lib.call("spk_pme_spread", _p(R), _p(q), _p(cell), _p(idx_m), _p(sys_ptr), N, n_sys, n1, n2, n3, int(order), _p(Q),
              _p(ws), ws.numel(), _stream(), launches=8 if N > 0 else 4)
    spec = torch.fft.rfftn(Q, dim=(1, 2, 3)).contiguous()
    energy = torch.empty((n_sys,), dtype=torch.float32, device=dev)
    conv = torch.empty_like(spec)
    _lib.call("spk_pme_energy", _p(q), _p(sys_ptr), _p(spec), N, n_sys, n1, n2, n3, int(order), float(ke), float(alpha),
              _p(f32(addend, "energy")) if addend is not None else None, _p(energy), _p(conv), _p(ws), ws.numel(),
              _stream())
    return energy, conv, ws


def pme_bwd(R: Tensor, q: Tensor, idx_m: Tensor, sys_ptr: Tensor, n_sys: int, mesh, order: int, ke: float, alpha: float,
            g_E: Tensor, conv: Tensor, ws: Tensor, want_R: bool, g_q: Optional[Tensor], want_cell: bool,
            virial: Optional[Tensor] = None, accumulate_virial: bool = False):
    """The reverse of ``pme_fwd``: potential mesh = irfftn(conv), then the gather; outputs as ``ewald_bwd``."""
    dev = R.device
    N = R.shape[0]
    phi = torch.fft.irfftn(conv, s=tuple(mesh), dim=(1, 2, 3)).contiguous()
    g_R = torch.empty((N, 3), dtype=torch.float32, device=dev) if want_R else None
    g_cell = torch.empty((n_sys, 3, 3), dtype=torch.float32, device=dev) if want_cell else None
    _lib.call("spk_pme_bwd", _p(R), _p(q), _p(idx_m), _p(sys_ptr), _p(phi), N, n_sys, *mesh, int(order), float(ke),
              float(alpha), _p(f32(g_E, "g_E")), _p(g_R), _p(g_q), 1, _p(g_cell), _p(virial), int(accumulate_virial),
              _p(ws), ws.numel(), _stream(), launches=int(N > 0) + int(want_cell or virial is not None))
    return g_R, g_cell


# ------------------------------------------------------------------------------------------------------- vibrations
def vib_displace(params: "_lib.VibParams"):
    """replica positions and realised steps of the chunk the counter names (csrc/vibrations.cu)"""
    _lib.call("spk_vib_displace", ctypes.byref(params), _stream())


def vib_assemble(params: "_lib.VibParams"):
    """the chunk's Hessian columns and dipole / polarizability derivatives from the replica outputs"""
    _lib.call("spk_vib_assemble", ctypes.byref(params), _stream())


def vib_finish(params: "_lib.VibParams"):
    """symmetrised Hessian in the Response layout and its mass-weighted blocks, once after the last chunk"""
    _lib.call("spk_vib_finish", ctypes.byref(params), _stream())


# ------------------------------------------------------------------------------------------------------- phonons
def ph_force_constants(params: "_lib.PhononParams", rounds: int):
    """force constants in the block layout after ``rounds`` symmetrisation / sum-rule rounds (csrc/phonons.cu)"""
    _lib.call("spk_ph_force_constants", ctypes.byref(params), _stream(), launches=1 + rounds)


def ph_images(params: "_lib.PhononParams"):
    """the minimum-image table of every force-constant row"""
    _lib.call("spk_ph_images", ctypes.byref(params), _stream())


def ph_dynmat(params: "_lib.PhononParams", q: Tensor, dyn_ptr: Tensor, n_el: int) -> Tensor:
    """[Q, n_el] complex128 mass-weighted dynamical matrices at q [Q, 3] (reduced reciprocal coordinates); n_el =
    dyn_ptr[-1], system m at dyn_ptr[m] as [3 n_m, 3 n_m]"""
    q = q.to(torch.float64).contiguous()
    out = torch.empty(q.shape[0], n_el, dtype=torch.complex128, device=q.device)
    _lib.call("spk_ph_dynmat", ctypes.byref(params), _p(q), q.shape[0], _p(dyn_ptr), _p(out), _stream())
    return out


def ph_dos(freq: Tensor, prim_ptr: Tensor, grid: Tensor, width: float) -> Tensor:
    """[B, G] Gaussian density of states of the frequencies [Q, 3 N_prim] on ``grid`` [G] (same unit as freq)"""
    n_sys = prim_ptr.shape[0] - 1
    out = torch.empty(n_sys, grid.shape[0], dtype=torch.float64, device=freq.device)
    _lib.call("spk_ph_dos", _p(freq), freq.shape[0], freq.shape[1], _p(prim_ptr), n_sys, _p(grid), grid.shape[0],
              float(width), _p(out), _stream())
    return out


def ph_thermo(freq: Tensor, prim_ptr: Tensor, temperatures: Tensor, seg_ptr: Tensor, n_items: int, min_freq: float,
              ev_per_invcm: float, k_b: float) -> Tensor:
    """[T B, 6] per-cell harmonic thermodynamics of the frequencies [Q, 3 N_prim] in cm^-1 (csrc/phonons.cu)"""
    n_sys, n_t = prim_ptr.shape[0] - 1, temperatures.shape[0]
    nbytes = _lib.lib().spk_ph_thermo_workspace_bytes(n_items, n_sys * n_t)
    ws = torch.empty(-(-nbytes // 8), dtype=torch.float64, device=freq.device)
    out = torch.empty(n_t * n_sys, _lib.PH_THERMO_FIELDS, dtype=torch.float64, device=freq.device)
    _lib.call("spk_ph_thermo", _p(freq), freq.shape[0], freq.shape[1], _p(prim_ptr), n_sys, _p(temperatures), n_t,
              _p(seg_ptr), n_items, float(min_freq), float(ev_per_invcm), float(k_b), _p(out), _p(ws), nbytes,
              _stream())
    return out
