"""Seeded synthetic inputs and weights for the five BASELINE.json configurations (numpy only, CPU).

Shared by ``bench.py``, ``tests/`` and ``tests/golden/make_golden.py`` so that the CUDA path, the oracle and
the live reference are always evaluated on byte-identical tensors.  Definitions follow SURVEY.md §8(d).

The layout of every batch is the reference's collate layout (``/root/reference/src/schnetpack/data/loader.py:13-58``):
atoms of all systems concatenated, ``_idx_m`` = system id per atom, ``_idx_i/_idx_j`` shifted by the cumulative
atom count, ``_offsets`` Cartesian periodic shifts, ``_cell [B,3,3]``, ``_pbc [B*3]``, ``_n_atoms [B]``.
Key names are the reference's (``/root/reference/src/schnetpack/properties.py:10-40``).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np

# --- reference dictionary keys (properties.py:10-40) -------------------------------------------------------------
Z = "_atomic_numbers"
R = "_positions"
idx_m = "_idx_m"
idx_i = "_idx_i"
idx_j = "_idx_j"
Rij = "_Rij"
offsets = "_offsets"
cell = "_cell"
pbc = "_pbc"
n_atoms = "_n_atoms"

# MD17 ethanol geometry of tests/testdata/md_ethanol.xyz (9 atoms, Angstrom), Z = C C H H H H H O H
ETHANOL_Z = np.array([6, 6, 1, 1, 1, 1, 1, 8, 1], dtype=np.int64)
ETHANOL_R = np.array(
    [
        [-4.92196480914482, 1.53680877549233, -0.06612792847094],
        [-3.41079303549336, 1.45138155063184, -0.14009009720834],
        [-5.22648850340463, 2.28202241947302, 0.66236410391492],
        [-5.34004680800574, 0.57895313793668, 0.22257334141131],
        [-5.33193076526251, 1.80898014947387, -1.03229511269262],
        [-3.00368348713509, 1.18933429199764, 0.83479697695625],
        [-2.99557504133053, 2.41817570143478, -0.41886385105291],
        [-3.07553304550781, 0.47652256654287, -1.09348059854212],
        [-2.13350450471551, 0.40432140701697, -1.15817683431555],
    ]
)

# aspirin geometry of interfaces/lammps/examples/aspirin/aspirin.data (21 atoms; LAMMPS types 1->C, 2->H, 3->O)
ASPIRIN_Z = np.array([6, 6, 6, 6, 6, 6, 6, 8, 8, 8, 6, 6, 8, 1, 1, 1, 1, 1, 1, 1, 1], dtype=np.int64)
ASPIRIN_R = np.array(
    [
        [7.13448882, 4.01563895, 4.80478211],
        [5.76264381, 5.95941395, 3.3200711],
        [7.66034484, 4.59207395, 3.69269609],
        [6.91031682, 5.39396596, 2.85298014],
        [1.96980977, 6.49540496, 5.71966213],
        [5.84942484, 4.44912893, 5.2843751],
        [5.23844682, 5.47350594, 4.5955781],
        [5.89789581, 2.72356796, 6.73006105],
        [2.61654782, 5.41777894, 3.53714311],
        [4.52379882, 4.47091293, 7.33925915],
        [5.39299181, 3.80976295, 6.53798211],
        [2.87701488, 5.95175993, 4.6022951],
        [4.19533384, 6.28624594, 5.1105091],
        [4.50619683, 3.81320798, 8.09597421],
        [7.55473471, 3.19750297, 5.39213109],
        [5.33068982, 6.85571098, 2.65473604],
        [8.80379391, 4.50628096, 3.54379714],
        [7.23114085, 5.55718595, 1.8758502],
        [2.29106975, 7.484658, 5.9269281],
        [0.86951685, 6.48216701, 5.4312661],
        [2.12585187, 6.00320899, 6.69948506],
    ]
)


# ------------------------------------------------------------------------------------------------------------------
# neighbour lists (CPU, numpy) -- input generators only; ordering = sorted by idx_i then idx_j (then shift)
# ------------------------------------------------------------------------------------------------------------------
def molecule_pairs(pos: np.ndarray, cutoff: float):
    """All ordered pairs (i, j), i != j, |R_j - R_i| < cutoff for an open (non-periodic) system."""
    n = pos.shape[0]
    d = np.linalg.norm(pos[None, :, :] - pos[:, None, :], axis=-1)
    mask = (d < cutoff) & ~np.eye(n, dtype=bool)
    ii, jj = np.nonzero(mask)  # row-major => sorted by i then j
    return ii.astype(np.int64), jj.astype(np.int64)


def periodic_cell_list(pos: np.ndarray, box: float, cutoff: float):
    """Full periodic neighbour list of a cubic box (minimum-image not assumed) via a linked-cell sweep.

    Returns idx_i, idx_j (int64, sorted by i then j then shift) and integer shifts S [E,3] such that
    r_ij = R[j] - R[i] + S*box with |r_ij| < cutoff.  Vectorised over the 27 stencil offsets.
    """
    n = pos.shape[0]
    nc = max(1, int(math.floor(box / cutoff)))
    if nc < 3:
        # small boxes: brute force over the required images
        nimg = int(math.ceil(cutoff / box))
        rng = np.arange(-nimg, nimg + 1)
        shifts = np.array([(a, b, c) for a in rng for b in rng for c in rng], dtype=np.int64)
        out_i, out_j, out_s = [], [], []
        for s in shifts:
            dvec = pos[None, :, :] + s[None, None, :] * box - pos[:, None, :]
            d = np.linalg.norm(dvec, axis=-1)
            mask = d < cutoff
            if not s.any():
                mask &= ~np.eye(n, dtype=bool)
            ii, jj = np.nonzero(mask)
            out_i.append(ii)
            out_j.append(jj)
            out_s.append(np.broadcast_to(s, (ii.shape[0], 3)))
        ii = np.concatenate(out_i)
        jj = np.concatenate(out_j)
        ss = np.concatenate(out_s)
    else:
        w = pos - np.floor(pos / box) * box  # wrapped copy for binning
        wrap_shift = -np.floor(pos / box).astype(np.int64)  # w = pos + wrap_shift*box
        cs = box / nc
        cidx = np.minimum((w / cs).astype(np.int64), nc - 1)
        lin = (cidx[:, 0] * nc + cidx[:, 1]) * nc + cidx[:, 2]
        order = np.argsort(lin, kind="stable")
        lin_sorted = lin[order]
        start = np.searchsorted(lin_sorted, np.arange(nc**3), side="left")
        end = np.searchsorted(lin_sorted, np.arange(nc**3), side="right")
        counts = end - start
        maxc = int(counts.max())
        # padded cell -> atom table
        table = -np.ones((nc**3, maxc), dtype=np.int64)
        rank = np.arange(n) - start[lin_sorted]
        table[lin_sorted, rank] = order
        out_i, out_j, out_s = [], [], []
        for dx in (-1, 0, 1):
            for dy in (-1, 0, 1):
                for dz in (-1, 0, 1):
                    nb = cidx + np.array([dx, dy, dz])
                    img = np.floor_divide(nb, nc)  # -1, 0, +1 image of the neighbour cell
                    nbw = nb - img * nc
                    nlin = (nbw[:, 0] * nc + nbw[:, 1]) * nc + nbw[:, 2]
                    cand = table[nlin]  # [n, maxc]
                    valid = cand >= 0
                    cj = np.where(valid, cand, 0)
                    dvec = w[cj] + (img * box)[:, None, :] - w[:, None, :]
                    d2 = np.einsum("ijk,ijk->ij", dvec, dvec)
                    mask = valid & (d2 < cutoff * cutoff)
                    mask &= ~((cj == np.arange(n)[:, None]) & (img == 0).all(axis=1)[:, None])
                    ai, slot = np.nonzero(mask)
                    aj = cj[ai, slot]
                    # shift relative to the *unwrapped* input positions
                    # w = pos + wrap_shift*box  =>  r_ij = pos[j]-pos[i] + (img + ws[j] - ws[i])*box
                    s = img[ai] + wrap_shift[aj] - wrap_shift[ai]
                    out_i.append(ai)
                    out_j.append(aj)
                    out_s.append(s)
        ii = np.concatenate(out_i)
        jj = np.concatenate(out_j)
        ss = np.concatenate(out_s)
    key = np.lexsort((ss[:, 2], ss[:, 1], ss[:, 0], jj, ii))
    return ii[key].astype(np.int64), jj[key].astype(np.int64), ss[key].astype(np.int64)


def _collate(systems):
    """Concatenate per-system dicts the way the reference's _atoms_collate_fn does (data/loader.py:13-58)."""
    out: Dict[str, np.ndarray] = {}
    nat = np.array([s[Z].shape[0] for s in systems], dtype=np.int64)
    seg = np.concatenate([[0], np.cumsum(nat)[:-1]])
    out[n_atoms] = nat
    out[idx_m] = np.repeat(np.arange(len(systems), dtype=np.int64), nat)
    out[Z] = np.concatenate([s[Z] for s in systems])
    out[R] = np.concatenate([s[R] for s in systems]).astype(np.float32)
    out[idx_i] = np.concatenate([s[idx_i] + o for s, o in zip(systems, seg)])
    out[idx_j] = np.concatenate([s[idx_j] + o for s, o in zip(systems, seg)])
    out[offsets] = np.concatenate([s[offsets] for s in systems]).astype(np.float32)
    out[cell] = np.stack([s[cell] for s in systems]).astype(np.float32)
    out[pbc] = np.concatenate([s[pbc] for s in systems])
    return out


def _open_system(zs, pos, cutoff):
    ii, jj = molecule_pairs(pos, cutoff)
    return {
        Z: zs.astype(np.int64),
        R: pos,
        idx_i: ii,
        idx_j: jj,
        offsets: np.zeros((ii.shape[0], 3)),
        cell: np.zeros((3, 3)),
        pbc: np.zeros(3, dtype=bool),
    }


# ------------------------------------------------------------------------------------------------------------------
# the five configurations
# ------------------------------------------------------------------------------------------------------------------
def ethanol_batch(batch: int = 1, cutoff: float = 5.0, jitter: float = 0.0, seed: int = 0):
    """cfg1: MD17 ethanol (9 atoms, 72 ordered pairs at rc=5), optional Gaussian jitter for batch>1."""
    rng = np.random.default_rng(seed)
    systems = []
    for b in range(batch):
        pos = ETHANOL_R + (rng.normal(0.0, jitter, ETHANOL_R.shape) if jitter > 0 else 0.0)
        systems.append(_open_system(ETHANOL_Z, pos, cutoff))
    return _collate(systems)


def aspirin_batch(batch: int = 256, cutoff: float = 5.0, jitter: float = 0.05, seed: int = 0):
    """cfg2: aspirin x batch with N(0, jitter) noise, ordered pairs d<rc (~306 per molecule), sorted by idx_i."""
    rng = np.random.default_rng(seed)
    systems = []
    for b in range(batch):
        pos = ASPIRIN_R + rng.normal(0.0, jitter, ASPIRIN_R.shape)
        systems.append(_open_system(ASPIRIN_Z, pos, cutoff))
    return _collate(systems)


def _compact_molecule(rng, n, min_dist=0.9, spread=1.25):
    """Random compact molecule: sequential placement near a random already-placed atom, min pair distance."""
    pos = np.zeros((n, 3))
    k = 1
    while k < n:
        anchor = pos[rng.integers(0, k)]
        v = rng.normal(size=3)
        v /= np.linalg.norm(v)
        cand = anchor + v * rng.uniform(min_dist * 1.05, min_dist * 1.05 + spread * 0.6)
        if np.min(np.linalg.norm(pos[:k] - cand, axis=1)) >= min_dist:
            pos[k] = cand
            k += 1
    return pos


def qm9like_batch(batch: int = 1024, cutoff: float = 5.0, seed: int = 0, padded: bool = False, max_atoms: int = 29):
    """cfg3: QM9-like molecules, n_atoms ~ clip(round(N(18,3)),3,29), Z in {1,6,7,8,9}.

    padded=True pads every molecule to max_atoms*(max_atoms-1) edge slots; padding slots point at valid atoms
    (atom 0 <- atom 1 of the molecule) but carry r_ij=(rc,0,0) so that the cosine cutoff zeroes them exactly
    (nn/cutoff.py:30-32).  Padded batches return ``_Rij`` directly (key ``Rij``) since offsets cannot encode it.
    """
    rng = np.random.default_rng(seed)
    systems = []
    zs_pool = np.array([1, 6, 7, 8, 9])
    for b in range(batch):
        n = int(np.clip(np.rint(rng.normal(18, 3)), 3, max_atoms))
        pos = _compact_molecule(rng, n)
        zs = zs_pool[rng.integers(0, 5, n)]
        s = _open_system(zs, pos, cutoff)
        if padded:
            slots = max_atoms * (max_atoms - 1)
            e = s[idx_i].shape[0]
            rij = pos[s[idx_j]] - pos[s[idx_i]]
            pad = slots - e
            # keep idx_i sorted: padding edges are appended to the LAST atom's row
            s[idx_i] = np.concatenate([s[idx_i], np.full(pad, n - 1, dtype=np.int64)])
            s[idx_j] = np.concatenate([s[idx_j], np.zeros(pad, dtype=np.int64)])
            s[offsets] = np.zeros((slots, 3))
            prij = np.zeros((pad, 3))
            prij[:, 0] = cutoff
            s["_rij_direct"] = np.concatenate([rij, prij])
        systems.append(s)
    out = _collate(systems)
    if padded:
        out[Rij] = np.concatenate([s["_rij_direct"] for s in systems]).astype(np.float32)
    return out


def periodic_box(n_atoms_total: int = 8192, density: float = 0.1002, cutoff: float = 5.0, seed: int = 0,
                 min_dist: float = 0.8, build_list: bool = True):
    """cfg4/cfg5: water-density periodic cubic box, Z pattern O,H,H, jittered-lattice positions.

    L = (N/density)^(1/3) (43.4 A at N=8192, 137.9 A at N=262144), ~52 neighbours/atom at rc=5.
    ``build_list=False`` leaves the neighbour list out (for large boxes the caller builds it on the device with
    ``schnetpack_b200.neighbors.neighbor_list``; the numpy sweep below needs minutes beyond ~50 k atoms).
    """
    rng = np.random.default_rng(seed)
    n = n_atoms_total
    box = (n / density) ** (1.0 / 3.0)
    m = int(math.ceil(n ** (1.0 / 3.0)))
    a = box / m
    grid = np.stack(np.meshgrid(np.arange(m), np.arange(m), np.arange(m), indexing="ij"), -1).reshape(-1, 3)
    sel = rng.permutation(grid.shape[0])[:n]
    sel.sort()
    amp = max(0.0, (a - min_dist) / 2.0) * 0.98
    pos = (grid[sel] + 0.5) * a + rng.uniform(-amp, amp, (n, 3))
    zs = np.tile(np.array([8, 1, 1], dtype=np.int64), n // 3 + 1)[:n]
    cellm = np.eye(3) * box
    if not build_list:
        return {n_atoms: np.array([n], dtype=np.int64), idx_m: np.zeros(n, dtype=np.int64), Z: zs,
                R: pos.astype(np.float32), cell: cellm[None].astype(np.float32), pbc: np.ones(3, dtype=bool)}
    ii, jj, ss = periodic_cell_list(pos, box, cutoff)
    out = {
        n_atoms: np.array([n], dtype=np.int64),
        idx_m: np.zeros(n, dtype=np.int64),
        Z: zs,
        R: pos.astype(np.float32),
        idx_i: ii,
        idx_j: jj,
        offsets: (ss @ cellm).astype(np.float32),
        cell: cellm[None].astype(np.float32),
        pbc: np.ones(3, dtype=bool),
    }
    return out


# ------------------------------------------------------------------------------------------------------------------
# model specs and seeded weights (keys = the reference state_dict keys, SURVEY.md §8b)
# ------------------------------------------------------------------------------------------------------------------
def model_spec(kind: str = "painn", n_atom_basis: int = 128, n_interactions: int = 3, n_rbf: int = 20,
               cutoff: float = 5.0, rbf: str = "gaussian", shared_interactions: bool = False,
               shared_filters: bool = False, epsilon: float = 1e-8, n_filters: Optional[int] = None,
               forces: bool = True, lmax: int = 2):
    spec = dict(kind=kind, n_atom_basis=n_atom_basis, n_interactions=n_interactions, n_rbf=n_rbf, cutoff=cutoff,
                rbf=rbf, shared_interactions=shared_interactions, shared_filters=shared_filters, epsilon=epsilon,
                n_filters=n_filters or n_atom_basis, forces=forces)
    if kind == "so3net":
        spec["lmax"] = lmax
    return spec


def _xavier(rng, out_f, in_f):
    a = math.sqrt(6.0 / (in_f + out_f))
    return rng.uniform(-a, a, (out_f, in_f)).astype(np.float32)


def init_params(spec: dict, seed: int = 0, bias_scale: float = 0.1) -> Dict[str, np.ndarray]:
    """Seeded weights with the reference's shapes/keys.  Weights: xavier-uniform like nn/base.py:27-28; biases are
    drawn U(-bias_scale, bias_scale) (instead of the reference's zeros) so that parity tests exercise the bias paths;
    embedding ~ N(0,1) like nn.Embedding."""
    rng = np.random.default_rng(seed)
    F = spec["n_atom_basis"]
    T = spec["n_interactions"]
    nr = spec["n_rbf"]
    p: Dict[str, np.ndarray] = {}

    def bias(n):
        return rng.uniform(-bias_scale, bias_scale, n).astype(np.float32)

    pre = "representation."
    p[pre + "cutoff_fn.cutoff"] = np.array([spec["cutoff"]], dtype=np.float32)
    if spec["rbf"] == "gaussian":
        off = np.linspace(0.0, spec["cutoff"], nr, dtype=np.float32)
        p[pre + "radial_basis.offsets"] = off
        p[pre + "radial_basis.widths"] = (np.abs(off[1] - off[0]) * np.ones_like(off)).astype(np.float32)
    else:
        p[pre + "radial_basis.freqs"] = (np.arange(1, nr + 1) * math.pi / spec["cutoff"]).astype(np.float32)
    p[pre + "embedding.weight"] = rng.normal(0, 1, (100, F)).astype(np.float32)
    nblocks = 1 if spec["shared_interactions"] else T
    if spec["kind"] == "painn":
        nf = 3 * F if spec["shared_filters"] else T * 3 * F
        p[pre + "filter_net.weight"] = _xavier(rng, nf, nr)
        p[pre + "filter_net.bias"] = bias(nf)
        for t in range(nblocks):
            b = f"{pre}interactions.{t}.interatomic_context_net."
            p[b + "0.weight"] = _xavier(rng, F, F)
            p[b + "0.bias"] = bias(F)
            p[b + "1.weight"] = _xavier(rng, 3 * F, F)
            p[b + "1.bias"] = bias(3 * F)
            m = f"{pre}mixing.{t}."
            p[m + "intraatomic_context_net.0.weight"] = _xavier(rng, F, 2 * F)
            p[m + "intraatomic_context_net.0.bias"] = bias(F)
            p[m + "intraatomic_context_net.1.weight"] = _xavier(rng, 3 * F, F)
            p[m + "intraatomic_context_net.1.bias"] = bias(3 * F)
            p[m + "mu_channel_mix.weight"] = _xavier(rng, 2 * F, F)
    elif spec["kind"] == "schnet":
        nfil = spec["n_filters"]
        for t in range(nblocks):
            b = f"{pre}interactions.{t}."
            p[b + "in2f.weight"] = _xavier(rng, nfil, F)
            p[b + "f2out.0.weight"] = _xavier(rng, F, nfil)
            p[b + "f2out.0.bias"] = bias(F)
            p[b + "f2out.1.weight"] = _xavier(rng, F, F)
            p[b + "f2out.1.bias"] = bias(F)
            p[b + "filter_network.0.weight"] = _xavier(rng, nfil, nr)
            p[b + "filter_network.0.bias"] = bias(nfil)
            p[b + "filter_network.1.weight"] = _xavier(rng, nfil, nfil)
            p[b + "filter_network.1.bias"] = bias(nfil)
    elif spec["kind"] == "so3net":
        L = spec["lmax"]
        from .nn.so3 import sh_indices, sparse_clebsch_gordan

        widx = sh_indices(L)[0][sparse_clebsch_gordan(L)[1]].numpy()     # SO3Convolution.Widx (a persistent buffer)
        for t in range(nblocks):
            c = f"{pre}so3convs.{t}."
            p[c + "Widx"] = widx
            p[c + "filternet.weight"] = _xavier(rng, (L + 1) * F, nr)
            p[c + "filternet.bias"] = bias((L + 1) * F)
            for k in ("mixings1", "mixings2", "mixings3"):
                p[f"{pre}{k}.{t}.weight"] = _xavier(rng, F, F)
            g = f"{pre}gatings.{t}.scaling."
            p[g + "weight"] = _xavier(rng, (L + 1) * F, F)
            p[g + "bias"] = bias((L + 1) * F)
    else:
        raise ValueError(spec["kind"])
    # Atomwise head F -> F//2 -> 1 (atomistic/atomwise.py:60-66, nn/blocks.py:38-76)
    h = max(1, F // 2)
    p["output_modules.0.outnet.0.weight"] = _xavier(rng, h, F)
    p["output_modules.0.outnet.0.bias"] = bias(h)
    p["output_modules.0.outnet.1.weight"] = _xavier(rng, 1, h)
    p["output_modules.0.outnet.1.bias"] = bias(1)
    return p


CONFIGS = {
    "cfg1": dict(desc="MD17 ethanol (9 atoms) SchNet 128x3 E+F, batch 1",
                 spec=dict(kind="schnet", n_interactions=3), data=("ethanol_batch", dict(batch=1))),
    "cfg2": dict(desc="MD17 aspirin (21 atoms) PaiNN 128x3 E+F, batch 256",
                 spec=dict(kind="painn", n_interactions=3), data=("aspirin_batch", dict(batch=256))),
    "cfg3": dict(desc="QM9-like SchNet 128x6 energy, batch 1024 padded neighbour list",
                 spec=dict(kind="schnet", n_interactions=6, forces=False),
                 data=("qm9like_batch", dict(batch=1024, padded=True))),
    "cfg4": dict(desc="bulk water 8192 atoms periodic PaiNN 128x3 E+F",
                 spec=dict(kind="painn", n_interactions=3), data=("periodic_box", dict(n_atoms_total=8192))),
    "cfg5": dict(desc="262144-atom periodic box PaiNN 128x3 E+F",
                 spec=dict(kind="painn", n_interactions=3), data=("periodic_box", dict(n_atoms_total=262144))),
}


def make_config(name: str, **overrides):
    c = CONFIGS[name]
    fn, kw = c["data"]
    kw = dict(kw)
    kw.update(overrides)
    return model_spec(**c["spec"]), globals()[fn](**kw)
