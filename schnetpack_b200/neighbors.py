"""Device-resident neighbour lists (SURVEY.md section 8, "next" row f1).

Mirrors the contract of the reference's neighbour-list transforms (/root/reference/src/schnetpack/transform/
neighborlist.py:159-286,428-553: ``forward(inputs)`` fills ``_idx_i``, ``_idx_j``, ``_offsets``) but works on a collated
batch that already lives on the GPU, so an MD driver never copies positions to the host to rebuild its list
(md/neighborlist_md.py:129,213-232 does, every rebuild).  The search is the linked-cell kernel of csrc/neighbors.cu.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import _lib, ops
from . import properties as P

__all__ = ["neighbor_list", "CellListNeighborList"]

Tensor = torch.Tensor


def _sys_ptr(n_atoms_per_system: Tensor) -> Tensor:
    ptr = torch.zeros(n_atoms_per_system.numel() + 1, dtype=torch.int32, device=n_atoms_per_system.device)
    ptr[1:] = torch.cumsum(n_atoms_per_system.to(torch.int64), 0).to(torch.int32)
    return ptr


def neighbor_list(positions: Tensor, cell: Optional[Tensor], pbc: Optional[Tensor], n_atoms: Tensor, cutoff: float,
                  capacity: Optional[int] = None, pad: bool = False, return_shifts: bool = False):
    """All pairs within ``cutoff`` of a collated batch on the GPU.

    positions [N,3] fp32 (cuda), cell [B,3,3] (or [3,3] / None for a non-periodic batch), pbc [B,3] bool (or [3] / None),
    n_atoms [B] atoms per system.  Returns ``idx_i, idx_j`` (int64), ``offsets`` [E,3] fp32 (and ``shifts`` int32).

    * ``capacity=None`` (default): exact size -- a counting pass, one host read of the pair count, then the fill pass;
    * ``capacity=E_max``: no host synchronisation; with ``pad=True`` the result always has ``E_max`` entries, the unused
      capacity being spread over the rows as self pairs at distance 2*cutoff (zero contribution to any cutoff-weighted
      model; ``idx_i`` stays sorted, no row grows long) -- the form to use under CUDA-graph capture; the returned ``n_pairs`` tensor (device, int64 [2]) holds the true count and an overflow flag;
    * ``capacity=0``: count only, ``n_pairs`` = (pairs, 1 if there are any).

    Positions may lie any number of cells away from the cell, and the rows of non-periodic axes may be zero.
    """
    if not positions.is_cuda:
        raise ValueError("schnetpack_b200.neighbors: positions must be a CUDA tensor (no CPU fallback)")
    dev = positions.device
    R = positions.detach().to(torch.float32).contiguous()
    N = R.shape[0]
    n_atoms = n_atoms.to(dev)
    B = int(n_atoms.numel())
    if cell is None:
        cell = torch.zeros((B, 3, 3), dtype=torch.float32, device=dev)
    cell = cell.detach().to(device=dev, dtype=torch.float32).reshape(-1, 3, 3)
    if cell.shape[0] == 1 and B > 1:
        cell = cell.expand(B, 3, 3)
    cell = cell.contiguous()
    if pbc is None:
        pbc = torch.zeros((B, 3), dtype=torch.bool, device=dev)
    pbc = pbc.to(dev).reshape(-1, 3)
    if pbc.shape[0] == 1 and B > 1:
        pbc = pbc.expand(B, 3)
    pbc = pbc.to(torch.uint8).contiguous()
    sys_ptr = _sys_ptr(n_atoms)
    ws = torch.empty(_lib.lib().spk_neighbor_list_workspace_bytes(N, B), dtype=torch.uint8, device=dev)
    n_pairs = torch.zeros(2, dtype=torch.int64, device=dev)
    p = ops._p

    def run(cap, idx_i, idx_j, off, sh, do_pad):
        _lib.call("spk_neighbor_list", p(R), p(cell), p(pbc), p(sys_ptr), N, B, float(cutoff), cap, 1 if do_pad else 0,
                  p(idx_i), p(idx_j), p(off), p(sh), p(n_pairs), p(ws), ws.numel(), ops._stream())

    exact = capacity is None
    if exact:
        run(0, None, None, None, None, False)            # count only
        capacity = int(n_pairs[0].item())                # the one host read of the exact-size mode
        pad = False
    idx_i = torch.empty(capacity, dtype=torch.int64, device=dev)
    idx_j = torch.empty(capacity, dtype=torch.int64, device=dev)
    off = torch.empty((capacity, 3), dtype=torch.float32, device=dev)
    sh = torch.empty((capacity, 3), dtype=torch.int32, device=dev) if return_shifts else None
    if capacity > 0 or not exact:                        # capacity=0 counts: n_pairs = (total, total > 0)
        run(capacity, idx_i, idx_j, off, sh, pad)
    out = (idx_i, idx_j, off) + ((sh,) if return_shifts else ())
    return out + (n_pairs,)


class CellListNeighborList(torch.nn.Module):
    """Batch-level, GPU-resident counterpart of ``NeighborListTransform`` (transform/neighborlist.py:159-210): reads
    ``_positions``, ``_cell``, ``_pbc``, ``_n_atoms`` of a collated batch and writes ``_idx_i``, ``_idx_j``, ``_offsets``.
    ``capacity`` / ``pad`` as in :func:`neighbor_list` (fixed-size, synchronisation-free lists for graph capture)."""

    is_preprocessor: bool = True
    is_postprocessor: bool = False

    def __init__(self, cutoff: float, capacity: Optional[int] = None, pad: bool = False):
        super().__init__()
        self._cutoff = float(cutoff)
        self.capacity = capacity
        self.pad = pad

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
        R = inputs[P.R]
        res = neighbor_list(R, inputs.get(P.cell), inputs.get(P.pbc), inputs[P.n_atoms], self._cutoff, self.capacity,
                            self.pad)
        inputs[P.idx_i], inputs[P.idx_j], inputs[P.offsets] = res[0], res[1], res[2]
        inputs["_n_pairs"] = res[-1]
        return inputs
