"""Batch layouts that stress the per-system reductions, their fp64 restatements and the error bounds the kernels are held
to.

Every per-system sum of the package (energy, kinetic energy and its tensor, the virial, the dipole and polarizability
heads, the ring-polymer and barostat sums) reduces items of consecutive systems in two passes (csrc/segscan.cuh): CTAs of
T consecutive items leave one fp64 partial per (system, CTA), and one 128-thread CTA per system adds a system's partials,
thread t taking partials t, t + 128, t + 256, ...  The layouts below are built around T, so that a system spans more
than 128 (or 256) partial blocks, starts exactly on a block boundary, ends one item before one, or sits among runs of
empty systems.

The restatements sum in float64 by explicit segment id (numpy's bincount), never in the kernels' order.  A kernel result
is held to ``bound = 4 (n_s + 20) 2^-53 sum|terms|`` per system and component; ``smallest_block_effect`` shows that this
bound would see a single partial block dropped or counted twice."""
import numpy as np

SEG_FIN_T = 128                  # threads of the per-system pass (csrc/segscan.cuh)
LAYOUTS = ("giant", "aligned", "empties", "many", "none")
EPS64 = 2.0 ** -53


def layout(name, T, n_many=70_000):
    """per-system item counts (int64) of layout ``name`` for T items per partial block"""
    if name == "giant":          # starts mid-block, spans more than 2 x 128 blocks
        c = [5, 2 * SEG_FIN_T * T + T // 2 + 1, 3]
    elif name == "aligned":      # the second system starts on a boundary and spans exactly 129 blocks
        c = [T, (SEG_FIN_T + 1) * T, T - 1, 1, 2 * T + 1]
    elif name == "empties":      # empties first, a run of 300, a giant, an empty, one item, an empty last
        c = [0, 0, 3, 7] + [0] * 300 + [SEG_FIN_T * T + T // 2 + 7, 0, 1, 0]
    elif name == "many":         # more than 65 535 systems of 1, 2, 3 items, a few of them empty
        c = np.tile([1, 2, 3], n_many // 3 + 1)[:n_many]
        c[[0, 17, n_many // 2, n_many // 2 + 1, n_many - 1]] = 0
    elif name == "none":
        c = [0, 0, 0]
    else:
        raise KeyError(name)
    return np.asarray(c, dtype=np.int64)


def seg_ptr(counts):
    return np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)


def seg_ids(counts):
    return np.repeat(np.arange(len(counts)), counts)


def seg_sum(terms, counts):
    """[n_sys, C] fp64 sums of ``terms`` [n, C] (or [n]) over the segments of ``counts``"""
    t = np.asarray(terms, dtype=np.float64)
    t2 = t.reshape(t.shape[0], int(np.prod(t.shape[1:])))
    ids = seg_ids(counts)
    out = np.stack([np.bincount(ids, weights=t2[:, c], minlength=len(counts)) for c in range(t2.shape[1])], axis=1)
    return out.reshape((len(counts),) + t.shape[1:])


def bound(terms, counts):
    """4 (n_s + 20) 2^-53 sum_s |terms|, per system and component"""
    a = seg_sum(np.abs(np.asarray(terms, dtype=np.float64)), counts)
    n = np.asarray(counts, dtype=np.float64).reshape((-1,) + (1,) * (a.ndim - 1))
    return 4.0 * (n + 20.0) * EPS64 * a


def smallest_block_effect(counts, T, terms):
    """[n_sys, C]: the smallest |sum of one partial block| of each system that spans more than SEG_FIN_T blocks of T
    items (the blocks of the global T grid cut at the system's ends), inf for every other system.  If this exceeds ten
    times ``bound``, a result that dropped or doubled one partial is outside the bound."""
    t = np.asarray(terms, dtype=np.float64)
    t2 = t.reshape(t.shape[0], int(np.prod(t.shape[1:])))
    ptr = seg_ptr(counts)
    out = np.full((len(counts), t2.shape[1]), np.inf)
    for s, (a, b) in enumerate(zip(ptr[:-1], ptr[1:])):
        if b <= a or (b - 1) // T - a // T + 1 <= SEG_FIN_T:
            continue
        cuts = np.concatenate([[a], np.arange((a // T + 1) * T, b, T)])
        out[s] = np.abs(np.add.reduceat(t2[a:b], cuts - a, axis=0)).min(axis=0)
    return out.reshape((len(counts),) + t.shape[1:])


def n_blocks(counts, T):
    """partial blocks each system spans (0 for an empty system)"""
    ptr = seg_ptr(counts)
    a, b = ptr[:-1], ptr[1:]
    return np.where(b > a, (b - 1) // T - a // T + 1, 0)
