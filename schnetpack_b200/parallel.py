"""Multi-GPU plumbing for the hot path (SURVEY.md §8e).

Molecule batches shard by *system* with no data-path collective: every rank evaluates a contiguous slice of the systems
of a collated batch and only the (tiny) results are gathered.  ``shard_batch`` cuts the reference's flat-graph batch
(`data/loader.py:13-58` layout) at system boundaries and re-bases the neighbour indices; ``gather_results`` reassembles
per-system / per-atom outputs in the original order with one ``all_gather`` each (NCCL on GPUs, gloo in the CPU tests).
A single large periodic system does not shard this way (it needs spatial bricks + halo exchange, DESIGN.md §6).
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import properties


def system_slices(n_atoms: np.ndarray, world: int) -> List[Tuple[int, int]]:
    """Contiguous system ranges [m0, m1) per rank, balanced by atom count (a proxy for edge work)."""
    n_atoms = np.asarray(n_atoms, dtype=np.int64)
    B = n_atoms.shape[0]
    cum = np.concatenate([[0], np.cumsum(n_atoms)])
    total = int(cum[-1])
    cuts = [0]
    for r in range(1, world):
        target = total * r / world
        m = int(np.searchsorted(cum, target, side="left"))
        m = min(max(m, cuts[-1]), B)
        cuts.append(m)
    cuts.append(B)
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def shard_batch(batch: Dict[str, np.ndarray], rank: int, world: int) -> Dict[str, np.ndarray]:
    """Sub-batch of ``batch`` holding the systems assigned to ``rank`` (numpy in, numpy out; indices re-based)."""
    n_at = np.asarray(batch[properties.n_atoms], dtype=np.int64)
    m0, m1 = system_slices(n_at, world)[rank]
    cum = np.concatenate([[0], np.cumsum(n_at)])
    a0, a1 = int(cum[m0]), int(cum[m1])
    idx_i = np.asarray(batch[properties.idx_i])
    idx_j = np.asarray(batch[properties.idx_j])
    emask = (idx_i >= a0) & (idx_i < a1)          # edges never cross systems, so idx_j is in the same range
    out: Dict[str, np.ndarray] = {}
    for k, v in batch.items():
        v = np.asarray(v)
        if k in (properties.idx_i, properties.idx_j):
            out[k] = v[emask] - a0
        elif k in (properties.offsets, properties.Rij):
            out[k] = v[emask]
        elif k == properties.idx_m:
            out[k] = v[a0:a1] - m0
        elif k in (properties.n_atoms, properties.cell):
            out[k] = v[m0:m1]
        elif k == properties.pbc:
            out[k] = v[3 * m0:3 * m1]
        elif v.shape[:1] == (int(cum[-1]),):       # per-atom arrays (Z, R, ...)
            out[k] = v[a0:a1]
        else:
            out[k] = v
    return out


def gather_results(results: Dict[str, torch.Tensor], n_systems_total: int, n_atoms_total: int, n_atoms_local: int,
                   group=None) -> Dict[str, torch.Tensor]:
    """All-gather per-system ([B_local, ...]) and per-atom ([N_local, ...]) result tensors into full-batch tensors.
    Shards are contiguous and ordered by rank, so concatenation restores the original order."""
    import torch.distributed as dist

    world = dist.get_world_size(group)
    out = {}
    for k, v in results.items():
        per_atom = v.shape[0] == n_atoms_local and k != properties.energy
        sizes = [torch.zeros(1, dtype=torch.int64, device=v.device) for _ in range(world)]
        dist.all_gather(sizes, torch.tensor([v.shape[0]], dtype=torch.int64, device=v.device), group=group)
        sizes = [int(s) for s in sizes]
        mx = max(sizes)
        pad = torch.zeros((mx,) + tuple(v.shape[1:]), dtype=v.dtype, device=v.device)
        pad[: v.shape[0]] = v
        parts = [torch.empty_like(pad) for _ in range(world)]
        dist.all_gather(parts, pad, group=group)
        full = torch.cat([p[:s] for p, s in zip(parts, sizes)], dim=0)
        if full.shape[0] != (n_atoms_total if per_atom else n_systems_total):
            raise RuntimeError(f"gather_results: {k} has {full.shape[0]} rows after the gather")
        out[k] = full
    return out


# ----------------------------------------------------------------------------------------------------------------------
# One LARGE system over several ranks (SURVEY.md section 8e, cfg5): graph partition + halo exchange.
#
# The neighbour list already says who needs whom, so the halo is defined by the GRAPH, not by geometry: a rank owns a slab
# of atoms, evaluates the edges whose RECEIVER it owns, and needs the per-atom rows (positions, x = context(q), mu) of the
# senders it does not own -- its ghosts.  Per interaction block that is one exchange of x (and mu) rows forward and, for
# forces, the reverse exchange of their gradients; ``HaloExchange`` is that exchange as an autograd function over
# torch.distributed point-to-point calls (NCCL on GPUs, gloo in the CPU tests), so the chain rule through positions and
# features of ghost atoms reaches the owner's leaves without any rank seeing the whole system.
# ----------------------------------------------------------------------------------------------------------------------
class RankPlan:
    """What rank ``rank`` of ``world`` needs to evaluate its part of one big graph (all index arrays int64, numpy).

    owned      global ids of the atoms this rank owns (ascending)
    ghosts     global ids of the senders it needs from other ranks, grouped by owner rank (ascending rank, ascending id
               inside a group); local index = len(owned) + position
    edge_ids   positions in the global edge list of the edges with an owned receiver (global order preserved)
    idx_i, idx_j   those edges in LOCAL indices (receivers < len(owned); senders may be ghosts)
    send[p]    local (owned) indices of the rows peer p needs from this rank, in the order p stores them as ghosts
    recv[p]    (start, stop) slice of this rank's ghost block filled by peer p
    """

    def __init__(self, rank, world, owned, ghosts, edge_ids, idx_i, idx_j, send, recv, ghost_rank=None, ghost_row=None,
                 send_pos=None):
        self.rank, self.world = rank, world
        self.owned, self.ghosts, self.edge_ids, self.idx_i, self.idx_j = owned, ghosts, edge_ids, idx_i, idx_j
        self.send, self.recv = send, recv
        # for the peer-memory halo: owner rank of every ghost and its row index in the owner's local table; and, per peer
        # p, where in p's ghost block the rows of send[p] start
        self.ghost_rank, self.ghost_row, self.send_pos = ghost_rank, ghost_row, (send_pos or {})
        self._dev_send = {}

    def to_device(self, device):
        """Cache the per-peer send lists as index tensors on ``device`` (the exchange then never copies them again)."""
        self._dev_send = {p: torch.as_tensor(v).to(device) for p, v in self.send.items()}
        return self

    def send_index(self, p, device):
        t = self._dev_send.get(p)
        if t is None or t.device != torch.device(device):
            t = torch.as_tensor(self.send[p]).to(device)
            self._dev_send[p] = t
        return t

    @property
    def n_owned(self) -> int:
        return int(self.owned.shape[0])

    @property
    def n_ghost(self) -> int:
        return int(self.ghosts.shape[0])


def slab_owners(positions: np.ndarray, world: int, axis: int = None) -> np.ndarray:
    """Owner rank of every atom: ``world`` slabs of equal atom count along ``axis`` (default: the longest extent).
    Ties are broken by atom index, so every rank computes the same assignment."""
    R = np.asarray(positions, dtype=np.float64)
    if axis is None:
        axis = int(np.argmax(R.max(axis=0) - R.min(axis=0))) if R.shape[0] else 0
    order = np.lexsort((np.arange(R.shape[0]), R[:, axis]))
    owner = np.empty(R.shape[0], dtype=np.int64)
    bounds = [(R.shape[0] * r) // world for r in range(world + 1)]
    for r in range(world):
        owner[order[bounds[r]:bounds[r + 1]]] = r
    return owner


def partition_graph(owner: np.ndarray, idx_i: np.ndarray, idx_j: np.ndarray, rank: int, world: int) -> RankPlan:
    """Plan of ``rank`` for the graph (idx_i = receivers, idx_j = senders) under the atom -> rank map ``owner``."""
    owner = np.asarray(owner, dtype=np.int64)
    idx_i, idx_j = np.asarray(idx_i, dtype=np.int64), np.asarray(idx_j, dtype=np.int64)
    n = owner.shape[0]

    def ghosts_of(r):
        e = np.nonzero(owner[idx_i] == r)[0]
        s = np.unique(idx_j[e])
        return e, s[owner[s] != r]

    owned = np.nonzero(owner == rank)[0]
    edge_ids, ghosts = ghosts_of(rank)
    # ghosts grouped by owner rank (ascending rank, ascending id inside): the block peer p fills is contiguous
    ghosts = ghosts[np.lexsort((ghosts, owner[ghosts]))]
    local = np.full(n, -1, dtype=np.int64)
    local[owned] = np.arange(owned.shape[0])
    local[ghosts] = owned.shape[0] + np.arange(ghosts.shape[0])
    row_on_owner = np.empty(n, dtype=np.int64)         # index of every atom in its OWNER's local table (owned ids ascending)
    for p in range(world):
        sel = np.nonzero(owner == p)[0]
        row_on_owner[sel] = np.arange(sel.shape[0])
    recv, send, send_pos = {}, {}, {}
    for p in range(world):
        if p == rank:
            continue
        sel = np.nonzero(owner[ghosts] == p)[0]
        if sel.size:
            recv[p] = (int(sel[0]), int(sel[-1]) + 1)
        # what p needs from me: p's ghosts that I own, in p's storage order
        _, gp = ghosts_of(p)
        gp = gp[np.lexsort((gp, owner[gp]))]
        mine = gp[owner[gp] == rank]
        if mine.size:
            send[p] = local[mine]
            send_pos[p] = int(np.count_nonzero(owner[gp] < rank))      # p's ghost block is ordered by owner rank
    return RankPlan(rank, world, owned, ghosts, edge_ids, local[idx_i[edge_ids]], local[idx_j[edge_ids]], send, recv,
                    ghost_rank=owner[ghosts].astype(np.int32), ghost_row=row_on_owner[ghosts].astype(np.int32),
                    send_pos=send_pos)


class HaloExchange(torch.autograd.Function):
    """rows of the owned atoms [n_owned, ...]  ->  rows of this rank's ghost atoms [n_ghost, ...]  (autograd-aware).

    forward: every rank sends the rows its peers list as ghosts and receives its own ghost rows (isend/irecv);
    backward: the gradients of the ghost rows travel back to their owners and are accumulated onto the rows they came
    from (fixed peer order: deterministic).  All ranks must call it the same number of times in the same order.

    On GPUs the transport is NCCL point-to-point (grouped send/recv over NVLink; receives land directly in the ghost block,
    one index-gather kernel per peer packs the send rows).  With the gloo backend (CPU tests, or several ranks sharing one
    GPU in the single-GPU test of the CUDA engine) CUDA rows are staged through host memory, which gloo requires."""

    @staticmethod
    def _staged(rows, group):
        import torch.distributed as dist

        return rows.is_cuda and dist.get_backend(group) == "gloo"

    @staticmethod
    def forward(ctx, rows: torch.Tensor, plan: RankPlan, group=None):
        import torch.distributed as dist

        ctx.plan, ctx.group, ctx.n_owned = plan, group, rows.shape[0]
        tail = tuple(rows.shape[1:])
        staged = HaloExchange._staged(rows, group)
        ghost = rows.new_empty((plan.n_ghost,) + tail)
        ops, keep, late = [], [], []
        for p in sorted(set(plan.send) | set(plan.recv)):
            if p in plan.send:
                sb = rows.detach().index_select(0, plan.send_index(p, rows.device))
                if staged:
                    sb = sb.cpu()
                keep.append(sb)
                ops.append(dist.P2POp(dist.isend, sb, p, group))
            if p in plan.recv:
                a, b = plan.recv[p]
                if staged:
                    rb = torch.empty((b - a,) + tail, dtype=rows.dtype)
                    late.append((rb, a, b))
                else:
                    rb = ghost[a:b]                                      # contiguous block of the ghost rows: no unpack
                ops.append(dist.P2POp(dist.irecv, rb, p, group))
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()
        for rb, a, b in late:
            ghost[a:b] = rb.to(rows.device)
        return ghost

    @staticmethod
    def backward(ctx, g_ghost: torch.Tensor):
        import torch.distributed as dist

        plan, group = ctx.plan, ctx.group
        tail = tuple(g_ghost.shape[1:])
        staged = HaloExchange._staged(g_ghost, group)
        g_ghost = g_ghost.contiguous()
        g_rows = g_ghost.new_zeros((ctx.n_owned,) + tail)
        ops, recvs, keep = [], [], []
        for p in sorted(set(plan.send) | set(plan.recv)):
            if p in plan.recv:                               # my ghosts came from p: their gradients go back to p
                a, b = plan.recv[p]
                sb = g_ghost[a:b].cpu() if staged else g_ghost[a:b]
                keep.append(sb)
                ops.append(dist.P2POp(dist.isend, sb, p, group))
            if p in plan.send:                               # p holds ghosts of my rows: receive their gradients
                n = len(plan.send[p])
                rb = torch.empty((n,) + tail, dtype=g_ghost.dtype) if staged else g_ghost.new_empty((n,) + tail)
                recvs.append((p, rb))
                ops.append(dist.P2POp(dist.irecv, rb, p, group))
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()
        for p, rb in recvs:                                  # ascending peer order: deterministic accumulation
            g_rows.index_add_(0, plan.send_index(p, g_rows.device), rb.to(g_rows.device))
        return g_rows, None, None


# ----------------------------------------------------------------------------------------------------------------------
# Halo over NVLink peer memory (csrc/halo.cu): every rank READS the rows of its ghosts out of their owners' buffers -- the
# gather that a send-side pack would do, the transfer and the unpack are one hand-written kernel; NCCL is not involved.
# The buffers are torch symmetric memory (CUDA IPC mappings of every rank's allocation into every process); the only
# synchronisation is its device-side barrier between "owners have written" and "peers pull".
# ----------------------------------------------------------------------------------------------------------------------
class PeerHalo:
    """State of the peer-memory halo for one ``RankPlan``: two generations of a symmetric buffer (so that one barrier per
    exchange suffices: a buffer is rewritten only after the NEXT exchange's barrier, which every peer reaches after its
    pull from this one), the peer address tables and the index lists of the two kernels."""

    def __init__(self, plan: RankPlan, device, max_row_floats: int, group=None):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm

        self.plan, self.device, self.group = plan, torch.device(device), group if group is not None else dist.group.WORLD
        cap = torch.tensor([max(plan.n_owned, plan.n_ghost, 1)], dtype=torch.int64, device=device)
        dist.all_reduce(cap, op=dist.ReduceOp.MAX, group=group)
        self.cap_rows, self.row_floats = int(cap.item()), int(max_row_floats)
        self.bufs, self.hdls, self.ptrs = [], [], []
        try:
            symm.enable_symm_mem_for_group(self.group.group_name)      # idempotent; newer torch enables it implicitly
        except Exception:
            pass
        for _ in range(2):
            b = symm.empty(self.cap_rows * self.row_floats, dtype=torch.float32, device=self.device)
            h = symm.rendezvous(b, self.group)
            self.bufs.append(b)
            self.hdls.append(h)
            self.ptrs.append(torch.tensor([int(v) for v in h.buffer_ptrs], dtype=torch.int64, device=self.device))
        self.gen = 0
        i32 = dict(dtype=torch.int32, device=self.device)
        self.g_rank = torch.as_tensor(plan.ghost_rank, **i32)
        self.g_row = torch.as_tensor(plan.ghost_row, **i32)
        # reverse: entries (owned row, peer, position in the peer's ghost block), grouped by row, peers ascending
        rows, ranks, pos = [], [], []
        for p in sorted(plan.send):
            k = np.arange(len(plan.send[p]), dtype=np.int64)
            rows.append(np.asarray(plan.send[p], dtype=np.int64))
            ranks.append(np.full(k.shape[0], p, dtype=np.int64))
            pos.append(plan.send_pos[p] + k)
        if rows:
            rows, ranks, pos = np.concatenate(rows), np.concatenate(ranks), np.concatenate(pos)
            order = np.lexsort((ranks, rows))
            rows, ranks, pos = rows[order], ranks[order], pos[order]
            uniq, start = np.unique(rows, return_index=True)
            ptr = np.concatenate([start, [rows.shape[0]]])
        else:
            uniq, ptr, ranks, pos = (np.zeros(0, dtype=np.int64), np.zeros(1, dtype=np.int64), np.zeros(0, dtype=np.int64),
                                     np.zeros(0, dtype=np.int64))
        self.r_rows, self.r_ptr = torch.as_tensor(uniq, **i32), torch.as_tensor(ptr, **i32)
        self.r_rank, self.r_pos = torch.as_tensor(ranks, **i32), torch.as_tensor(pos, **i32)

    def publish(self, rows2d: torch.Tensor) -> int:
        """Copy ``rows2d`` [n, C] to the front of the next buffer generation and run the cross-rank barrier; returns the
        generation to pull from."""
        n, C = rows2d.shape
        if C > self.row_floats or n > self.cap_rows:
            raise ValueError("PeerHalo: rows exceed the symmetric buffer")
        g = self.gen
        self.gen ^= 1
        self.bufs[g][: n * C].copy_(rows2d.reshape(-1))
        self.hdls[g].barrier()
        return g


class PeerHaloExchange(torch.autograd.Function):
    """``HaloExchange`` over NVLink peer memory: same contract (owned rows -> ghost rows; backward sums the ghost-row
    gradients into their owners in ascending peer order), transport = ``spk_halo_pull`` / ``spk_halo_pull_add``."""

    @staticmethod
    def forward(ctx, rows: torch.Tensor, halo: PeerHalo):
        from . import _lib, ops

        ctx.halo, ctx.shape = halo, tuple(rows.shape)
        tail = tuple(rows.shape[1:])
        C = 1
        for d in tail:
            C *= int(d)
        plan = halo.plan
        with torch.cuda.device(halo.device):
            g = halo.publish(rows.detach().reshape(rows.shape[0], C))
            ghost = torch.empty((plan.n_ghost,) + tail, dtype=torch.float32, device=halo.device)
            _lib.call("spk_halo_pull", ops._p(ghost), ops._p(halo.ptrs[g]), ops._p(halo.g_rank), ops._p(halo.g_row),
                      plan.n_ghost, C, ops._stream())
        return ghost

    @staticmethod
    def backward(ctx, g_ghost: torch.Tensor):
        from . import _lib, ops

        halo = ctx.halo
        tail = ctx.shape[1:]
        C = 1
        for d in tail:
            C *= int(d)
        with torch.cuda.device(halo.device):
            g = halo.publish(g_ghost.contiguous().reshape(g_ghost.shape[0], C))
            g_rows = torch.zeros(ctx.shape, dtype=torch.float32, device=halo.device)
            _lib.call("spk_halo_pull_add", ops._p(g_rows), ops._p(halo.ptrs[g]), ops._p(halo.r_rows), ops._p(halo.r_ptr),
                      ops._p(halo.r_rank), ops._p(halo.r_pos), int(halo.r_rows.shape[0]), C, ops._stream())
        return g_rows, None


# ----------------------------------------------------------------------------------------------------------------------
# The CUDA engine on a partition: per-block kernel pipelines with a halo exchange in front of every edge kernel.
# ----------------------------------------------------------------------------------------------------------------------
def _halo(rows: torch.Tensor, plan: RankPlan, group, peer: Optional["PeerHalo"] = None):
    if plan.world == 1:
        return rows.new_zeros((0,) + tuple(rows.shape[1:]))
    if peer is not None:
        return PeerHaloExchange.apply(rows, peer)          # collective (barrier): every rank calls it, ghosts or not
    if plan.n_ghost == 0 and not plan.send:
        return rows.new_zeros((0,) + tuple(rows.shape[1:]))
    return HaloExchange.apply(rows, plan, group)


class PartitionedPotential:
    """Energy + forces of ONE large system evaluated by the ranks of a process group (SURVEY.md section 8e, cfg5), every
    rank running the sm_90a kernels on its part of the graph:

        owned atoms  -> context net (dense kernels)            x [n_owned, 3F]
        halo         -> ghost rows of (x, mu) from their owners  (HaloExchange: NCCL point-to-point, autograd-aware)
        local edges  -> fused edge kernel (receivers owned, senders owned or ghost)
        owned atoms  -> mixing (dense kernels + glue)

    per interaction block, then the Atomwise head on the owned atoms; forces come from ``torch.autograd.grad`` exactly as
    in the single-device model, the reverse halo (gradients of ghost rows summed into their owners, ghost position
    gradients returned with the first exchange's backward) being HaloExchange's backward.  Each directed edge is computed
    by exactly one rank, so owned-atom results are complete without a reduction; the only collective besides the halo is
    the all-reduce of the per-system partial energies.

    ``model`` is a ``schnetpack_b200.model.NeuralNetworkPotential`` with a PaiNN representation and an Atomwise head;
    ``batch`` is the GLOBAL system (numpy or tensors: Z, positions, idx_i, idx_j, offsets, idx_m, n_atoms) which every rank
    holds at set-up (only its part goes to the device).
    """

    def __init__(self, model, batch: Dict, plan: RankPlan, device, group=None):
        from . import functional as K
        from . import ops

        self.K, self.ops = K, ops
        self.model, self.plan, self.group, self.device = model, plan, group, torch.device(device)
        rep = model.representation
        if type(rep).__name__ != "PaiNN":
            raise NotImplementedError("PartitionedPotential: PaiNN representation (the named large-system configs)")
        if any(type(m).__name__ == "EnergyPME" for m in model.output_modules):
            raise NotImplementedError("PartitionedPotential: EnergyPME (its charge mesh spans the atoms of every rank); "
                                      "evaluate the model on one device")
        self.rep = rep
        self.head = [m for m in model.output_modules if type(m).__name__ == "Atomwise"][0]
        dev = self.device

        def take(key, sel):
            v = batch[key]
            v = v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
            return torch.as_tensor(v[sel]).to(dev)

        self.Z = take(properties.Z, plan.owned)
        self.R_own = take(properties.R, plan.owned).float().contiguous()
        self.offsets = take(properties.offsets, plan.edge_ids).float().contiguous()
        self.idx_m = take(properties.idx_m, plan.owned)
        self.idx_i = torch.as_tensor(plan.idx_i).to(dev)
        self.idx_j = torch.as_tensor(plan.idx_j).to(dev)
        self.n_sys = int(np.asarray(batch[properties.n_atoms].cpu() if isinstance(batch[properties.n_atoms], torch.Tensor)
                                    else batch[properties.n_atoms]).shape[0])
        self.n_local = plan.n_owned + plan.n_ghost
        plan.to_device(dev)
        with torch.cuda.device(dev):
            self.graph = ops.EdgeGraph(self.idx_i, self.idx_j, self.n_local)
        # transport of the halo: NVLink peer memory (hand-written pull kernels over torch symmetric memory) when the ranks
        # talk NCCL on one node, torch.distributed point-to-point otherwise (gloo tests) or with SPK_B200_HALO=nccl
        self.peer: Optional[PeerHalo] = None
        self.transport = "none" if plan.world == 1 else "p2p"
        if plan.world > 1 and os.environ.get("SPK_B200_HALO", "peer") == "peer":
            import torch.distributed as dist

            if dist.get_backend(group) == "nccl":
                # every rank must take the same branch: agree on success with an all-reduce
                ok = torch.ones(1, dtype=torch.int32, device=dev)
                try:
                    self.peer = PeerHalo(plan, dev, 6 * int(rep.n_atom_basis), group)
                except Exception as exc:          # symmetric memory unavailable (no P2P / IPC): NCCL point-to-point
                    self.peer_error = repr(exc)[:200]
                    ok.zero_()
                dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
                if int(ok.item()) == 1:
                    self.transport = "peer"
                else:
                    self.peer = None

    def set_positions(self, R_own: torch.Tensor):
        self.R_own = R_own.to(self.device, torch.float32).contiguous()

    def __call__(self):
        """Returns (energy [n_systems] summed over ranks, forces of the OWNED atoms [n_owned, 3])."""
        K, ops, plan, rep, group = self.K, self.ops, self.plan, self.rep, self.group
        n_o, n_g = plan.n_owned, plan.n_ghost
        dev = self.device
        with torch.cuda.device(dev), torch.enable_grad():
            pk = rep._pack()
            F, act = pk.F, rep._act
            R_own = self.R_own.detach().requires_grad_(True)                      # model/base.py:105-111
            R_loc = torch.cat([R_own, _halo(R_own, plan, group, self.peer)], dim=0)          # ghost positions (autograd-aware)
            r_ij = K.PairwiseDistancesFunction.apply(R_loc, self.offsets,        # atomistic/distances.py:14-26
                                                     dict(idx_i=self.idx_i, idx_j=self.idx_j, graph=self.graph))
            geom = K.EdgeGeometry(rep, r_ij, self.graph)                          # painn.py:227-230, shared by the blocks
            if isinstance(rep.embedding, torch.nn.Embedding) and len(rep.electronic_embeddings) == 0:
                q = ops.embedding(rep.embedding.weight.detach().contiguous(), self.Z)   # painn.py:239
            else:
                raise NotImplementedError("PartitionedPotential: plain nn.Embedding only")
            mu = None
            for t in range(pk.T):
                b = pk.blocks[t]
                x = K.PaiNNContextFunction.apply(q, b, act)                       # painn.py:54 on the owned atoms
                if mu is None:                                                    # first block: mu == 0 everywhere
                    x_loc = torch.cat([x, _halo(x, plan, group, self.peer)], dim=0)          # senders' rows incl. ghosts
                    mu_loc = None
                else:                                                             # ONE exchange of the 6F-float rows (x | mu)
                    gh = _halo(torch.cat([x, mu.reshape(n_o, 3 * F)], dim=1), plan, group, self.peer)
                    x_loc = torch.cat([x, gh[:, :3 * F]], dim=0)
                    mu_loc = torch.cat([mu, gh[:, 3 * F:].reshape(n_g, 3, F)], dim=0)
                # receivers = the n_o owned rows of q; senders = all local rows of x_loc / mu_loc (owned + ghosts)
                q1, mu1 = K.PaiNNEdgeFunction.apply(x_loc, mu_loc, q, r_ij, geom, pk, t)         # :55-65
                q, mu = K.PaiNNMixingFunction.apply(q1, mu1, b, F, pk.eps, act)                  # :103-116
            inputs = {"scalar_representation": q, properties.idx_m: self.idx_m,
                      properties.n_atoms: torch.empty(self.n_sys, dtype=torch.int64, device=dev)}
            agg = self.head.aggregation_mode
            if agg != "sum":
                raise NotImplementedError("PartitionedPotential: Atomwise(aggregation_mode='sum')")
            e_part = self.head(inputs)[self.head.output_key]                      # atomwise.py:69-88 on the owned atoms
            (g,) = torch.autograd.grad([e_part], [R_own], grad_outputs=[torch.ones_like(e_part)])   # response.py:62-68
            energy = e_part.detach().clone()
            if plan.world > 1:
                import torch.distributed as dist

                dist.all_reduce(energy, group=group)
        return energy, -g.detach()
