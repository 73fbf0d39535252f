"""GPU: every per-system reduction against an fp64 restatement on the batch layouts of tests/reduction_oracle.py -- a
system spanning more than 256 partial blocks, one starting exactly on a block boundary and spanning 129, runs of empty
systems, more than 65 535 systems, and a batch of empty systems only.  These are the layouts where the second pass of
csrc/segscan.cuh (thread t adds partials t, t + 128, t + 256, ...) loops more than once and where a partial is routed to
``sys_part`` or ``head``.

Every direct kernel call gets NaN-filled outputs and a NaN-filled workspace of exactly the advertised size followed by a
4 KiB sentinel that must come back unchanged, so a partial that nothing wrote, or a write past the workspace, shows.  Two
calls must agree bit for bit, and empty systems must give exact zeros.  An fp64 result is held to RO.bound per system
and component, and every such check also asserts that this bound would see one partial block dropped or doubled
(RO.smallest_block_effect)."""
import numpy as np
import pytest
import torch

import reduction_oracle as RO
from conftest import rel_err
from schnetpack_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NAN = float("nan")
SENTINEL = 4096
SENTINEL_VALUE = -1.25e300
BIG = ("giant", "aligned", "empties")        # layouts with a system of more than 128 partial blocks
layouts = pytest.mark.parametrize("name", RO.LAYOUTS)


def _np(t):
    return t.detach().cpu().numpy()


def _nan(shape, dtype=torch.float32):
    return torch.full(shape, NAN, dtype=dtype, device=DEV)


class _Workspace:
    """NaN-filled workspace of ``nbytes`` followed by a sentinel tail"""

    def __init__(self, nbytes):
        self.nbytes = int(nbytes)
        n8 = -(-self.nbytes // 8)
        self.buf = torch.full((n8 + SENTINEL // 8,), NAN, dtype=torch.float64, device=DEV)
        self.buf[n8:] = SENTINEL_VALUE
        self.n8 = n8

    @property
    def ptr(self):
        return ops._p(self.buf)

    def check(self):
        assert bool((self.buf[self.n8:] == SENTINEL_VALUE).all()), "write past the workspace"


def _batch(counts):
    idx = torch.as_tensor(RO.seg_ids(counts), dtype=torch.int64, device=DEV)
    return idx, ops.segment_ptr(idx, len(counts))


def _check_sum(got, ref, bnd, counts, T, terms, scale=1.0):
    """|got - ref| <= bound everywhere, exact zeros for empty systems, and the bound sees one block dropped"""
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    bnd = scale * np.asarray(bnd).reshape(got.shape)
    err = np.abs(got - ref)
    assert np.all(err <= bnd), (np.argmax((err - bnd).reshape(len(counts), -1).max(1)), float((err - bnd).max()))
    assert np.all(got[counts == 0] == 0.0)
    eff = scale * RO.smallest_block_effect(counts, T, terms).reshape(got.shape)
    fin = np.isfinite(eff)
    assert np.all(eff[fin] > 10.0 * bnd[fin])
    return int(fin.reshape(len(counts), -1).any(1).sum())


# ---- sys_ptr ------------------------------------------------------------------------------------------------------------
@layouts
@pytest.mark.parametrize("T", [8, 256])
def test_segment_ptr_equals_searchsorted(name, T):
    counts = RO.layout(name, T)
    ids = RO.seg_ids(counts)
    got = ops.segment_ptr(torch.as_tensor(ids, dtype=torch.int64, device=DEV), len(counts))
    assert np.array_equal(_np(got), np.searchsorted(ids, np.arange(len(counts) + 1), side="left"))


# ---- energy: spk_atomwise_out's k_mol_sum (fp32, one CTA per system) ------------------------------------------------------
def _atomwise(hid, w1, b1, ptr, n_mol):
    y, e = _nan((hid.shape[0],)), _nan((n_mol,))
    _lib.call("spk_atomwise_out", ops._p(hid), ops._p(w1), ops._p(b1), ops._p(ptr), hid.shape[0], n_mol, hid.shape[1],
              ops._p(y), ops._p(e), ops._stream())
    return y, e


@layouts
def test_energy_sum_against_fp64_and_alone(name):
    counts = RO.layout(name, 256)
    n_sys, N, H = len(counts), int(counts.sum()), 32
    g = torch.Generator().manual_seed(7)
    hid = torch.randn(N, H, generator=g).to(DEV)
    w1, b1 = torch.randn(H, generator=g).to(DEV), torch.tensor([0.3], device=DEV)
    _, ptr = _batch(counts)
    y, e = _atomwise(hid, w1, b1, ptr, n_sys)
    y2, e2 = _atomwise(hid, w1, b1, ptr, n_sys)
    torch.cuda.synchronize()
    assert torch.equal(y, y2) and torch.equal(e, e2)
    y64 = _np(y).astype(np.float64)
    ref, absum = RO.seg_sum(y64, counts), RO.seg_sum(np.abs(y64), counts)
    tol = (np.ceil(counts / 256) + 13) * 2.0 ** -24 * absum
    assert np.all(np.abs(_np(e) - ref) <= tol) and np.all(_np(e)[counts == 0] == 0.0)
    # each system's energy depends on its own atoms only, bit for bit
    rng = np.random.default_rng(1)
    pick = np.arange(n_sys) if n_sys <= 400 else np.r_[rng.choice(n_sys, 300, replace=False), np.flatnonzero(counts == 0)]
    hp = RO.seg_ptr(counts)
    for s in pick:
        one = torch.tensor([0, counts[s]], dtype=torch.int32, device=DEV)
        _, es = _atomwise(hid[hp[s]:hp[s + 1]].contiguous(), w1, b1, one, 1)
        assert _np(es)[0] == _np(e)[s], s


# ---- kinetic energy, temperature and kinetic-energy tensor ---------------------------------------------------------------
def _momenta(counts, seed):
    rng = np.random.default_rng(seed)
    N = int(counts.sum())
    m = rng.choice([1.008, 12.011, 15.999], size=N).astype(np.float32)
    p = (rng.normal(size=(N, 3)) * np.sqrt(m)[:, None]).astype(np.float32)
    return m, p


@layouts
def test_kinetic_energy_and_temperature(name):
    counts = RO.layout(name, 256)
    n_sys, N, kB = len(counts), int(counts.sum()), 2.0 ** -7
    m, p = _momenta(counts, 3)
    idx, ptr = _batch(counts)
    mt, pt = torch.as_tensor(m, device=DEV), torch.as_tensor(p, device=DEV)
    ws = _Workspace(_lib.lib().spk_md_thermostat_workspace_bytes(N, n_sys))
    res = []
    for _ in range(2):
        ke, temp = _nan((n_sys,), torch.float64), _nan((n_sys,), torch.float64)
        _lib.call("spk_md_kinetic_energy", ops._p(pt), ops._p(mt), ops._p(idx), ops._p(ptr), N, n_sys, kB, ops._p(ke),
                  ops._p(temp), ws.ptr, ws.nbytes, ops._stream())
        res.append((ke, temp))
    torch.cuda.synchronize()
    ws.check()
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    ke, temp = _np(res[0][0]), _np(res[0][1])
    p64, m64 = p.astype(np.float64), m.astype(np.float64)
    terms = (p64 ** 2).sum(1) / m64
    bnd = RO.bound(terms, counts)
    ref = 0.5 * RO.seg_sum(terms, counts)
    hit = _check_sum(ke, ref, bnd, counts, 256, terms, scale=0.5)
    assert hit > 0 or name not in BIG
    n = np.maximum(counts, 1).astype(np.float64)
    t_ref = 2.0 / (3.0 * n * kB) * ref
    assert np.all(np.abs(temp - t_ref) <= 2.0 / (3.0 * n * kB) * 0.5 * bnd + 4 * RO.EPS64 * np.abs(t_ref))
    assert np.all(temp[counts == 0] == 0.0)


@layouts
def test_kinetic_energy_tensor(name):
    counts = RO.layout(name, 256)
    n_sys, N = len(counts), int(counts.sum())
    m, p = _momenta(counts, 4)
    idx, ptr = _batch(counts)
    mt, pt = torch.as_tensor(m, device=DEV), torch.as_tensor(p, device=DEV)
    ws = _Workspace(_lib.lib().spk_md_barostat_workspace_bytes(N, n_sys))
    res = []
    for _ in range(2):
        K = _nan((n_sys, 3, 3), torch.float64)
        _lib.call("spk_md_kinetic_energy_tensor", ops._p(pt), ops._p(mt), ops._p(idx), ops._p(ptr), N, n_sys, ops._p(K),
                  ws.ptr, ws.nbytes, ops._stream())
        res.append(K)
    torch.cuda.synchronize()
    ws.check()
    assert torch.equal(res[0], res[1])
    p64, m64 = p.astype(np.float64), m.astype(np.float64)
    terms = p64[:, :, None] * p64[:, None, :] / m64[:, None, None]
    hit = _check_sum(_np(res[0]), 0.5 * RO.seg_sum(terms, counts), RO.bound(terms, counts), counts, 256, terms, 0.5)
    assert hit > 0 or name not in BIG


# ---- virial: spk_pairwise_virial over the receiver slots of each system --------------------------------------------------
def _edge_batch(counts, seed):
    """a synthetic edge list whose systems hold ``counts`` edge slots: a system with edges has n_recv receiver atoms plus
    one atom without edges in the middle; systems without edges have 0, 1 or 2 atoms"""
    rng = np.random.default_rng(seed)
    n_at, ii, jj, start = [], [], [], 0
    for s, e in enumerate(counts.tolist()):
        if e == 0:
            na = s % 3
        else:
            nr = min(e, 1 + e // 40)
            na = nr + 1
            recv = rng.integers(0, nr, e)
            recv = np.where(recv >= nr // 2, recv + 1, recv)          # atom nr // 2 receives nothing
            ii.append(start + recv)
            jj.append(start + rng.integers(0, na, e))
        n_at.append(na)
        start += na
    cat = (lambda x: np.concatenate(x) if x else np.zeros(0, dtype=np.int64))   # noqa: E731
    ii, jj = cat(ii), cat(jj)
    perm = rng.permutation(ii.shape[0])
    return np.asarray(n_at), ii[perm], jj[perm]


@layouts
def test_pairwise_virial(name):
    counts = RO.layout(name, 256)
    n_sys = len(counts)
    n_at, ii, jj = _edge_batch(counts, 5)
    N, E = int(n_at.sum()), ii.shape[0]
    rng = np.random.default_rng(6)
    g = rng.normal(size=(E, 3)).astype(np.float32)
    r = rng.normal(scale=2.0, size=(E, 3)).astype(np.float32)
    graph = ops.EdgeGraph(torch.as_tensor(ii, device=DEV), torch.as_tensor(jj, device=DEV), N)
    idx_m = torch.as_tensor(RO.seg_ids(n_at), dtype=torch.int64, device=DEV)
    sys_ptr = ops.segment_ptr(idx_m, n_sys)
    gt, rt = torch.as_tensor(g, device=DEV), torch.as_tensor(r, device=DEV)
    ws = _Workspace(_lib.lib().spk_pairwise_virial_workspace_bytes(E, n_sys))
    res = []
    for _ in range(2):
        W = _nan((n_sys, 3, 3), torch.float64)
        _lib.call("spk_pairwise_virial", ops._p(gt), ops._p(rt), ops._p(graph.rowptr), ops._p(graph.slot_eid),
                  ops._p(sys_ptr), E, n_sys, ops._p(W), ws.ptr, ws.nbytes, ops._stream())
        res.append(W)
    torch.cuda.synchronize()
    ws.check()
    assert torch.equal(res[0], res[1])
    rowptr = _np(graph.rowptr)
    assert np.array_equal(np.diff(rowptr[RO.seg_ptr(n_at)]), counts)          # the layout is the slot layout
    terms = g.astype(np.float64)[:, :, None] * r.astype(np.float64)[:, None, :]   # W[b][a] = g_b r_a
    slot_terms = terms[_np(graph.slot_eid)[:E]] if E else terms
    hit = _check_sum(_np(res[0]), RO.seg_sum(slot_terms, counts), RO.bound(slot_terms, counts), counts, 256, slot_terms)
    assert hit > 0 or name not in BIG
    # a system with atoms but no edges
    assert np.any((counts == 0) & (n_at > 0)) or name in ("giant", "aligned")


def test_virial_of_a_thousand_atom_box_equals_the_strain_path():
    """a cfg4-density box of 1000 atoms (about 52 k edges, some 200 partial blocks) and a second box in one batch: the
    kernel virial over the volume equals this package's Strain stress"""
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, from_spec
    from test_cuda_barostats import _collate, _eval

    parts = [S.periodic_box(1000, seed=12), S.periodic_box(128, seed=4)]
    batch = _collate(parts)
    assert batch["_idx_i"].shape[0] > 129 * 256
    spec = S.model_spec("painn", n_atom_basis=64, n_interactions=2)
    params = S.init_params(spec, seed=8)
    dev = torch.device(DEV)
    x = batch_to_device(batch, dev)
    model = from_spec(spec, params, dev)
    W1, W2 = _nan((2, 3, 3), torch.float64), _nan((2, 3, 3), torch.float64)
    _eval(model, x, W1)
    _eval(model, x, W2)
    out = from_spec(dict(spec, stress=True), params, dev)({k: v.clone() for k, v in x.items()})
    torch.cuda.synchronize()
    assert torch.equal(W1, W2)
    V = np.abs(np.linalg.det(batch["_cell"].astype(np.float64)))
    stress = _np(out["stress"]).reshape(2, 3, 3)
    for m in range(2):
        assert rel_err(_np(W1[m]) / V[m], stress[m]) < 1e-5, m


# ---- dipole / polarizability heads ----------------------------------------------------------------------------------------
HEAD_MANY = 5000          # systems of layout "many" for the heads (the ATen reference is slow beyond that)


def _head_inputs(counts, F, seed):
    g = torch.Generator().manual_seed(seed)
    N, B = int(counts.sum()), len(counts)
    idx = torch.as_tensor(RO.seg_ids(counts), dtype=torch.int64)
    return {"scalar_representation": torch.randn(N, F, generator=g).to(DEV),
            "vector_representation": torch.randn(N, 3, F, generator=g).to(DEV),
            "_positions": (3.0 * torch.randn(N, 3, generator=g)).to(DEV), "_idx_m": idx.to(DEV),
            "_n_atoms": torch.as_tensor(counts).to(DEV), "total_charge": torch.randn(B, generator=g).to(DEV)}


def _head_counts(name, T):
    return RO.layout(name, T, n_many=HEAD_MANY)


@layouts
@pytest.mark.parametrize("cfg", ["dipole", "dipole_magnitude", "polar", "scalar_dipole"])
def test_heads_match_aten_forward_and_backward(name, cfg):
    """the module path (spk_head_fwd / spk_head_bwd) against functional_torch in fp64, outputs and gradients"""
    import heads_oracle as HO
    from schnetpack_b200 import functional_torch as FT
    from test_cuda_heads import _head

    c = {"dipole": HO.dip(charges=True), "dipole_magnitude": HO.dip(magnitude=True), "polar": HO.pol(),
         "scalar_dipole": HO.dip(vector=False, charges=True, act="ssp")}[cfg]
    counts = _head_counts(name, 128 if cfg == "scalar_dipole" else 8)
    F = 32
    base = _head_inputs(counts, F, 11)
    torch.manual_seed(2)
    head = _head(c, F).to(DEV).eval()
    outs = []
    for kind in ("kernel", "aten"):
        x = {k: (v.clone().double() if kind == "aten" and v.is_floating_point() else v.clone()) for k, v in base.items()}
        leaves = [x[k].requires_grad_(True) for k in ("scalar_representation", "vector_representation", "_positions")]
        if kind == "aten":
            y = (FT.dipole_moment if c["kind"] == "dipole" else FT.polarizability)(head.double(), dict(x))
            head.float()
        else:
            y = head(dict(x))
        out = y[c["key"]]
        w = torch.randn(out.shape, generator=torch.Generator().manual_seed(1)).to(DEV, out.dtype)
        grads = torch.autograd.grad((out * w).sum(), leaves, allow_unused=True)
        res = [out] + [gg if gg is not None else torch.zeros_like(v) for gg, v in zip(grads, leaves)]
        if c.get("charges"):
            res.append(y[c["charges_key"]])
        outs.append([r.detach().double().cpu().numpy() for r in res])
        if kind == "kernel":
            assert torch.all(out.reshape(len(counts), -1)[torch.as_tensor(counts == 0, device=DEV)] == 0)
    # rel_err is max|a - b| / max|b| over the whole batch, so the small systems beside a giant are held to 1e-5 of the
    # giant's magnitude here; each system's sums are checked on their own by test_dipole_tail_sums_restated_from_kernel_outputs
    # and test_scalar_dipole_is_restated_exactly
    for i, (a, b) in enumerate(zip(*outs)):
        assert a.shape == b.shape and (a.size == 0 or rel_err(a, b) <= 1e-5), (i, a.size and rel_err(a, b))


def _tail_of(head):
    from schnetpack_b200.nn import activation_code

    last = head.outnet[-1]
    return ops.head_tail(last.mix_vectors.weight, last.scalar_net[0].weight, last.scalar_net[0].bias,
                         last.scalar_net[1].weight, last.scalar_net[1].bias, activation_code(last.scalar_net[0].activation))


def _head_fwd(kind, tail, s, V, q, R, idx, ptr, Q, n_sys, magnitude, ws):
    N = R.shape[0]
    shape = (n_sys, 3, 3) if kind == ops.HEAD_POLAR else ((n_sys,) if magnitude else (n_sys, 3))
    out, saved = _nan(shape), _nan((n_sys, 8), torch.float64)
    q_atom = _nan((N,)) if tail is not None else None
    _lib.call("spk_head_fwd", kind, tail, ops._p(s), ops._p(V), ops._p(q), ops._p(R), ops._p(idx), ops._p(ptr),
              ops._p(Q), N, n_sys, 1, int(magnitude), ops._p(out), ops._p(q_atom), ops._p(saved), ws.ptr, ws.nbytes,
              ops._stream(), launches=2 if N > 0 else 1)
    return out, q_atom, saved


@layouts
def test_dipole_tail_sums_restated_from_kernel_outputs(name):
    """the vector tail (8-atom tiles, warp scan): saved = (c, mean R, mu, n) and the corrected charges, restated from
    the kernel's own per-atom charges"""
    import heads_oracle as HO
    from test_cuda_heads import _head

    counts = _head_counts(name, 8)
    n_sys, N, F = len(counts), int(counts.sum()), 32
    x = _head_inputs(counts, F, 13)
    torch.manual_seed(3)
    head = _head(HO.dip(n_layers=1, charges=True), F).to(DEV).eval()
    tail, keep = _tail_of(head)
    idx, ptr = _batch(counts)
    ws = _Workspace(_lib.lib().spk_head_workspace_bytes(N, n_sys))
    args = (x["scalar_representation"], x["vector_representation"], None, x["_positions"], idx, ptr, x["total_charge"],
            n_sys, False, ws)
    o1, q1, s1 = _head_fwd(ops.HEAD_DIPOLE, tail, *args)
    o2, q2, s2 = _head_fwd(ops.HEAD_DIPOLE, tail, *args)
    charges = ops.head_charges(q1, idx, s1) if N else q1
    torch.cuda.synchronize()
    ws.check()
    assert torch.equal(o1, o2) and torch.equal(q1, q2) and torch.equal(s1, s2)
    sv, q = _np(s1), _np(q1).astype(np.float64)
    R, Q = _np(x["_positions"]).astype(np.float64), _np(x["total_charge"]).astype(np.float64)
    n = np.maximum(counts, 1).astype(np.float64)
    assert np.array_equal(sv[:, 7], counts.astype(np.float64))
    # mean positions: the sums of R
    hit = _check_sum(sv[:, 1:4] * n[:, None], RO.seg_sum(R, counts), RO.bound(R, counts) + 4 * RO.EPS64 *
                     np.abs(RO.seg_sum(R, counts)), counts, 8, R)
    # the charge correction c = (Q - sum q) / n from the kernel's own q_atom
    sq = RO.seg_sum(q, counts)
    c_ref = np.where(counts > 0, (Q - sq) / n, 0.0)
    assert np.all(np.abs(sv[:, 0] - c_ref) <= (RO.bound(q, counts) + 4 * RO.EPS64 * np.abs(Q)) / n + 4 * RO.EPS64 *
                  np.abs(c_ref))
    eff, bq = RO.smallest_block_effect(counts, 8, q), RO.bound(q, counts)
    assert np.all(eff[np.isfinite(eff)] > 10 * bq[np.isfinite(eff)])
    assert hit > 0 or name not in BIG
    if N:
        assert torch.equal(charges, (q1.double() + s1[idx, 0]).float())
    assert np.all(sv[counts == 0, :7] == 0.0) and np.all(_np(o1)[counts == 0] == 0.0)


@layouts
def test_scalar_dipole_is_restated_exactly(name):
    """the scalar-charge path (128-atom tiles, block scan) with given charges: mu = sum (q + c) R in fp64"""
    counts = _head_counts(name, 128)
    n_sys, N = len(counts), int(counts.sum())
    rng = np.random.default_rng(9)
    q = rng.normal(scale=0.3, size=N).astype(np.float32)
    R = rng.normal(scale=3.0, size=(N, 3)).astype(np.float32)
    Q = rng.normal(size=n_sys).astype(np.float32)
    idx, ptr = _batch(counts)
    ws = _Workspace(_lib.lib().spk_head_workspace_bytes(N, n_sys))
    qt, Rt, Qt = (torch.as_tensor(a, device=DEV) for a in (q, R, Q))
    o1, _, s1 = _head_fwd(ops.HEAD_DIPOLE, None, None, None, qt, Rt, idx, ptr, Qt, n_sys, False, ws)
    o2, _, s2 = _head_fwd(ops.HEAD_DIPOLE, None, None, None, qt, Rt, idx, ptr, Qt, n_sys, False, ws)
    torch.cuda.synchronize()
    ws.check()
    assert torch.equal(o1, o2) and torch.equal(s1, s2)
    q64, R64, Q64 = q.astype(np.float64), R.astype(np.float64), Q.astype(np.float64)
    n = np.maximum(counts, 1).astype(np.float64)
    c = np.where(counts > 0, (Q64 - RO.seg_sum(q64, counts)) / n, 0.0)
    qR = q64[:, None] * R64
    mu = RO.seg_sum(qR, counts) + c[:, None] * RO.seg_sum(R64, counts)
    absR = RO.seg_sum(np.abs(R64), counts)
    bnd = (RO.bound(qR, counts) + np.abs(c)[:, None] * RO.bound(R64, counts) +
           ((RO.bound(q64, counts) + 4 * RO.EPS64 * np.abs(Q64)) / n)[:, None] * absR)
    got = _np(o1).astype(np.float64)
    assert np.all(np.abs(got - mu) <= 2.0 ** -24 * np.abs(mu) + bnd)
    assert np.all(got[counts == 0] == 0.0)
    for t in (qR, R64, q64):
        eff, b = RO.smallest_block_effect(counts, 128, t), RO.bound(t, counts)
        assert np.all(eff[np.isfinite(eff)] > 10 * b[np.isfinite(eff)])
        assert np.isfinite(eff).any() or name not in BIG


# ---- ring-polymer centroid and barostat sums, NHC barostat steps ------------------------------------------------------
def _giant_batch():
    """layout "giant" for 256 atoms per partial block (a system of 65 665 atoms over 258 blocks, starting mid-block)
    between small systems; no empty system, which the ring-polymer and barostat oracles do not take"""
    return [1] + RO.layout("giant", 256).tolist() + [9]


@pytest.mark.parametrize("name", ["pile_g", "nhc_global"])
@pytest.mark.parametrize("P", [1, 4])
def test_rpmd_global_thermostats_on_a_giant_system(P, name):
    """the centroid sums of the global PILE and NHC thermostats (k_rpmd_centroid_partials + k_seg_finish) against
    tests/rpmd_oracle.py, as in tests/test_cuda_rpmd.py"""
    import test_cuda_rpmd as TR
    from schnetpack_b200 import md

    n_atoms, masses, x, p = TR._mixed_batch(P, n_atoms=_giant_batch())
    base, rp = TR._bind(P, n_atoms, masses)
    dev_th, ref_th = TR._thermostats(md)[name]
    dev_th.bind(base, TR.DT_EXACT, rp)
    ref_th.init(TR._rp_oracle(P), masses.astype(np.float64), n_atoms)
    pt = torch.as_tensor(p, device=DEV).reshape(-1, 3)
    pr = torch.as_tensor(p, dtype=torch.float64)
    for _ in range(4):
        dev_th.apply(pt)
        pr = ref_th.apply(pr)
    torch.cuda.synchronize()
    got, ref = _np(pt).reshape(p.shape), pr.numpy()
    assert np.isfinite(got).all()
    assert rel_err(got, ref) < 1e-5
    giant = slice(n_atoms[0] + n_atoms[1], n_atoms[0] + n_atoms[1] + n_atoms[2])
    assert rel_err(got[:, giant].mean(0), ref[:, giant].mean(0)) < 1e-5               # the giant's centroid
    assert np.abs(ref - p).max() / np.abs(p).max() > (1e-6 if name.startswith("nhc") else 1e-2)
    if name.startswith("nhc"):
        v, f, m = ref_th.chain_state()
        assert rel_err(_np(dev_th.masses), m) < 1e-12
        assert rel_err(_np(dev_th.velocities), v) < 1e-6
        assert rel_err(_np(dev_th.forces), f) < 1e-6


@pytest.mark.parametrize("P", [1, 4])
def test_rpmd_pile_barostat_on_a_giant_system(P):
    """the PILE barostat's sums (k_rpmd_baro_partials + k_rpmd_baro_finish) against tests/rpmd_npt_oracle.py with the
    checks of tests/test_cuda_rpmd_npt.py"""
    import test_cuda_rpmd_npt as TRN

    TRN.barostat_follows_the_oracle(P, TRN._mixed_batch(P, n_atoms=_giant_batch()))


@pytest.mark.parametrize("kind", ["iso", "aniso"])
def test_nhc_barostat_steps_on_a_giant_system(kind):
    """two NPT steps of the NHC barostats (thermostat, kick, half and main steps: the sums of k_ke7_partials, with the
    2 KE channel that drives the particle chain) against tests/npt_oracle.py, in the protocol of
    tests/golden/make_golden_md_barostats.py"""
    import npt_oracle as NPO
    from schnetpack_b200 import md as M

    n_atoms = _giant_batch()
    B, N = len(n_atoms), sum(n_atoms)
    rng = np.random.default_rng(31)
    kB, fs, bar, dt, tau = 2.0 ** -7, 2.0 ** -10, 2.0 ** -12, 2.0 ** -7, 128.0
    masses = rng.choice([1.0, 12.0, 16.0], size=N).astype(np.float32)
    p0 = (rng.normal(size=(N, 3)) * np.sqrt(masses * kB * 300.0)[:, None]).astype(np.float32)
    cells = np.stack([np.diag(rng.uniform(30.0, 40.0, 3)) for _ in range(B)])
    x0 = (rng.uniform(0.0, 1.0, size=(N, 3)) * 30.0).astype(np.float32)
    forces = (rng.normal(size=(2, N, 3)) * 5.0).astype(np.float32)
    stress = rng.normal(scale=0.05, size=(3, B, 3, 3))
    stress = 0.5 * (stress + stress.transpose(0, 1, 3, 2))
    kw = dict(anisotropic=kind == "aniso", massive=False, integration_order=7 if kind == "aniso" else 3)
    cls = M.NHCBarostatAnisotropic if kw.pop("anisotropic") else M.NHCBarostatIsotropic
    b = cls(40.0, 300.0, tau, time_constant_cell=0.5 * tau, time_constant_barostat=2.0 * tau, kB=kB, fs=fs, bar=bar, **kw)
    ref = NPO.NHCBarostat(40.0, 300.0, tau, kB, fs, bar, time_constant_cell=0.5 * tau, time_constant_barostat=2.0 * tau,
                          anisotropic=kind == "aniso", **kw)
    idx_m = torch.as_tensor(RO.seg_ids(np.asarray(n_atoms)), device=DEV)
    b.bind(M._Systems(torch.as_tensor(masses, device=DEV), idx_m, B), dt)
    ref.init(masses, np.asarray(n_atoms), dt)
    x, p = torch.as_tensor(x0, device=DEV), torch.as_tensor(p0, device=DEV)
    cell = torch.as_tensor(cells, device=DEV).contiguous()
    t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))  # noqa: E731
    xr, pr, cr = t(x0), t(p0), t(cells)

    def kick(s):
        b.kick(p, cell, (torch.as_tensor(s, device=DEV) * torch.linalg.det(cell)[:, None, None]).contiguous(), 1.0)

    f_dev, f_ref = torch.zeros_like(x), torch.zeros_like(xr)
    for k in range(2):
        b.apply_thermostat(p)
        kick(stress[k])
        b.half_step(p, f_dev)
        b.main_step(x, p, cell)
        f_dev = torch.as_tensor(forces[k], device=DEV)
        b.half_step(p, f_dev)
        kick(stress[k + 1])
        b.apply_thermostat(p)
        pr = ref.thermostat(pr)
        ref.kick(pr, cr, t(stress[k]))
        pr = ref.half_step(pr, f_ref)
        xr, cr = ref.main_step(xr, pr, cr)
        f_ref = t(forces[k])
        pr = ref.half_step(pr, f_ref)
        ref.kick(pr, cr, t(stress[k + 1]))
        pr = ref.thermostat(pr)
    torch.cuda.synchronize()
    assert rel_err(_np(x), xr.numpy()) < 1e-6
    assert rel_err(_np(p), pr.numpy()) < 1e-6
    assert rel_err(_np(cell), cr.numpy()) < 1e-6
    assert np.abs(cr.numpy() - cells).max() > 1e-6 * np.abs(cells).max()                # the cells moved
    st = ref.state()
    for k, dev in (("t_velocities", b.t_velocities), ("t_forces", b.t_forces), ("t_velocities_cell", b.t_velocities_cell),
                   ("t_forces_cell", b.t_forces_cell), ("b_velocities_cell", b.b_velocities),
                   ("b_forces_cell", b.b_forces)):
        r = st[k].numpy()
        assert rel_err(_np(dev).reshape(r.shape), r) < 1e-5, k


# ---- relaxation: warp / cluster boundary -------------------------------------------------------------------------------
def test_relaxation_on_the_warp_and_cluster_boundaries():
    """systems of 256 / 257 atoms (warp path / cluster path), around 8 x 512 = 4096 atoms, 9000 atoms, one atom and an
    empty system: 10 steps against the fp64 oracle; the empty system is converged with fmax 0"""
    from relax_oracle import LBFGSOracle
    from schnetpack_b200.relax import LBFGSState

    sizes = [256, 257, 1, 0, 4095, 4096, 4097, 9000]
    ptr = RO.seg_ptr(np.asarray(sizes))
    rng = np.random.default_rng(21)
    n = int(ptr[-1])
    r = rng.normal(scale=3.0, size=(n, 3))
    centre = r + rng.normal(scale=0.4, size=(n, 3))
    stiff = rng.uniform(0.5, 3.0, size=(n, 1))

    def forces(x):
        return (-(x - centre) * stiff + 0.2 * np.sin(2.0 * x)).astype(np.float32)

    idx_m = torch.as_tensor(RO.seg_ids(np.asarray(sizes)), device=DEV)
    kw = dict(memory=5, maxstep=0.15, damping=0.9, alpha=4.0)
    st = LBFGSState(torch.as_tensor(r, device=DEV), idx_m, len(sizes), fmax=1e-9, **kw)
    assert st.n_warp == 3 and sorted(st.order.tolist()[:3]) == [0, 2, 3]
    o = LBFGSOracle(r, ptr, **kw)
    for k in range(10):
        f = forces(o.r)
        ft = torch.as_tensor(f, device=DEV)
        st.check(ft)
        np.testing.assert_allclose(_np(st.fmax), o.fmax(f), rtol=1e-12)
        ref = np.array([np.sqrt((f[a:b].astype(np.float64) ** 2).sum(1).max()) if b > a else 0.0
                        for a, b in zip(ptr[:-1], ptr[1:])])
        np.testing.assert_allclose(_np(st.fmax), ref, rtol=1e-12)
        assert _np(st.fmax)[3] == 0.0 and int(st.converged[3]) == 1
        st.step(ft)
        o.step(f.astype(np.float64), 1e-9)
        assert rel_err(_np(st.r), o.r) <= 1e-9, k
        assert rel_err(_np(st.p), o.p) <= 1e-9, k
    assert _np(st.converged).tolist() == [0, 0, 0, 1, 0, 0, 0, 0]


# ---- neighbour list over more than 65 535 systems ------------------------------------------------------------------------
def test_neighbor_list_over_seventy_thousand_molecules():
    """layout "many" as molecules without PBC (empty systems included) plus two periodic boxes at the end"""
    from oracle import nl_oracle as NL
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.neighbors import neighbor_list

    counts = RO.layout("many", 256)
    rng = np.random.default_rng(4)
    mol = rng.normal(scale=1.5, size=(int(counts.sum()), 3))
    boxes = [S.periodic_box(150, seed=3), S.periodic_box(96, seed=8)]
    R = np.concatenate([mol] + [b["_positions"] for b in boxes]).astype(np.float32)
    cells = np.concatenate([np.zeros((len(counts), 3, 3))] +
                           [np.asarray(b["_cell"], dtype=np.float64).reshape(1, 3, 3) for b in boxes])
    pbc = np.concatenate([np.zeros((len(counts), 3), dtype=bool), np.ones((2, 3), dtype=bool)])
    n_atoms = np.r_[counts, [150, 96]]
    ref = NL.batch_neighbor_list(R.astype(np.float64), cells, pbc, n_atoms, 5.0)
    ii, jj, off, sh, n_pairs = neighbor_list(torch.as_tensor(R, device=DEV), torch.as_tensor(cells, device=DEV),
                                             torch.as_tensor(pbc, device=DEV), torch.as_tensor(n_atoms, device=DEV), 5.0,
                                             return_shifts=True)
    n = int(n_pairs[0])
    assert int(n_pairs[1]) == 0
    gi, gj, gs = NL.canonical(_np(ii[:n]), _np(jj[:n]), _np(sh[:n]).astype(np.int64))
    assert gi.shape == ref[0].shape
    assert (gi == ref[0]).all() and (gj == ref[1]).all() and (gs == ref[2]).all()
