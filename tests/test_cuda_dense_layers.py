"""GPU: the two dense-layer kernels -- k_dense_tc (csrc/gemm_tc.cu: wgmma with 3xTF32) and k_dense (csrc/gemm.cu: fp32
FFMA, which runs every shape the tensor-core path refuses) -- against fp64 torch on the device, element by element, at
the shapes their own tiling rules select.

* The GEMM is checked through the saved pre-activation with a per-element bound
      |pre - pre64| <= C * 2^-24 * s,     s = sum_k |a'_ik| |w_jk| + |b_j|,     a' = a * act'(a_pre),
  so a large error at a small output cannot hide under a matrix-wide maximum.  The epilogue is checked on its own,
  against the fp64 activation evaluated at the kernel's own fp32 pre-activation.
* All-positive operands show whether a K-sum is biased: the tensor core truncates when it accumulates, which is why
  k_dense_tc adds every K-tile's fresh accumulator to its fp32 sum with round-to-nearest.
* Bitwise invariants that follow from the code: row, column-tile and row-tile independence, launch chaining, nothing
  written outside [M, N], nothing read past K or past N of the addend, and a non-finite input stays in its row.

The calibrated constants carry the largest ratio measured on an H100 SXM (132 SMs, 700 W power limit) beside them;
``pytest -s`` prints the largest ratio of every bound this run measured."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
EPS = 2.0 ** -24
ACT_NONE, ACT_SILU, ACT_SSP, ACT_GIVEN, SAVE_DERIV = 0, 1, 2, 3, 0x10   # include/spk_b200.h
SENTINEL = 0x7FBADBAD                                                     # a NaN bit pattern no kernel produces


# Largest values measured on the H100 SXM (132 SMs, 700 W) over every case of this file.  The tensor-core ratio is
# largest at one K-tile (8.05) and falls with K (6.43 at 2 K-tiles, 2.87 at 9, 1.66 at 64), so one constant covers all K.
C_TC = 36           # k_dense_tc per-element GEMM error, units of 2^-24 * s; measured 8.05
C_FFMA = 36         # k_dense per-element GEMM error, units of 2^-24 * s; measured 8.11
C_EPI = 10          # epilogue (activation, saved act', addend), units of 2^-24 * (|value| + 1); measured 2.29
BIAS_TC = 5.0       # |mean((pre - pre64) / s)| on positive operands, units of 2^-24; measured 1.10, flat in K
BIAS_FFMA = 0.25    # the same for k_dense; measured 0.026

_WORST = {}


def _note(key, value):
    _WORST[key] = max(_WORST.get(key, 0.0), float(value))
    return float(value)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for key in sorted(_WORST):
        print(f"dense layers, largest measured {key}: {_WORST[key]:.3g}")


# ------------------------------------------------------------------------------------------- the kernels' own rules
def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cdiv(a, b):
    return -(-a // b)


def tc_tile_n(M, N):
    """gemm_tc.cu tile_n: 128-wide column tiles when N % 128 == 0 and either N >= 256 or 64-wide tiles would need more
    than one wave of CTAs"""
    if N % 128:
        return 64
    if N >= 256:
        return 128
    return 128 if _cdiv(M, 128) * (N // 64) > _nsm() else 64


def tc_last_narrow_rows(N):
    """largest M that k_dense_tc still runs with 64-wide column tiles (N == 128)"""
    M = (_nsm() // (N // 64)) * 128
    assert tc_tile_n(M, N) == 64 and tc_tile_n(M + 1, N) == 128
    return M


def ffma_bm(M, N):
    """gemm.cu spk_dense: the largest row tile that still gives every SM three CTAs"""
    want, nt = 3 * _nsm(), _cdiv(N, 64)
    return 128 if _cdiv(M, 128) * nt >= want else 64 if _cdiv(M, 64) * nt >= want else 32


def ffma_first_rows(bm, N):
    """smallest M for which spk_dense picks row tile bm (bm = 64 or 128)"""
    M = (_cdiv(3 * _nsm(), _cdiv(N, 64)) - 1) * bm + 1
    assert ffma_bm(M, N) == bm and ffma_bm(M - 1, N) == bm // 2
    return M


# ------------------------------------------------------------------------------------------------------ helpers
def act64(x, act):
    if act == ACT_SILU:
        return x * torch.sigmoid(x)
    if act == ACT_SSP:
        return torch.nn.functional.softplus(x) - math.log(2.0)
    return x


def dact64(x, act):
    if act == ACT_SILU:
        s = torch.sigmoid(x)
        return s * (1.0 + x * (1.0 - s))
    if act == ACT_SSP:
        return torch.sigmoid(x)
    if act == ACT_GIVEN:
        return x
    return torch.ones_like(x)


def _abi(kern, A, M, K, lda, a_pre, a_act, Wk, N, bias, act, addend, ld_add, Y, ldy, y_pre):
    """one call of spk_dense_tc / spk_dense with every argument explicit (the ops wrappers fix ld_add = N)"""
    from schnetpack_b200 import _lib, ops

    _lib.call("spk_dense_tc" if kern == "tc" else "spk_dense", ops._p(A), M, K, lda, ops._p(a_pre), a_act, ops._p(Wk),
              N, ops._p(bias), act, ops._p(addend), ld_add, ops._p(Y), ldy, ops._p(y_pre), ops._stream())


def _operand(kern, W):
    """W [N, K] in the form the kernel takes: packed hi|lo tiles, or W^T [K, N] for the FFMA kernel"""
    from schnetpack_b200 import ops

    return ops.tc_pack_weight(W) if kern == "tc" else W.t().contiguous()


def _place(x, off=0):
    """a contiguous copy of x whose first element sits `off` floats past a 16 B-aligned allocation"""
    buf = torch.empty(x.numel() + off, device=DEV)
    v = buf[off:].view(x.shape)
    v.copy_(x)
    return v


def _sentinel(rows, ld):
    return torch.full((rows, ld), SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)


def _untouched(buf, M, N, what):
    b = buf.view(torch.int32)
    assert bool((b[M:] == SENTINEL).all()) and bool((b[:M, N:] == SENTINEL).all()), f"{what} written outside [M, N]"


def _bits(t):
    return t.contiguous().view(torch.int32)


def _bitwise_equal(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _gen(seed):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return g


# ---------------------------------------------------------------------------------------------- per-element check
def _check_layer(kern, M, K, N, a_act, act, *, bias=True, addend=True, lda=None, ldy=None, ld_add=None, a_off=0,
                 seed=0):
    """Run one layer twice through the C ABI (saving pre, then act'(pre) with SPK_SAVE_DERIV) and check it.

    A and a_pre are [M, lda] rows `a_off` floats off 16 B alignment with NaN in columns [K, lda); the addend is
    [M, ld_add] with NaN past N; Y and y_pre are the first M rows of [M + 2, ldy] sentinel-filled buffers."""
    lda, ldy, ld_add = lda or K, ldy or N, ld_add or N
    g = _gen(seed)
    nan = float("nan")
    a = torch.randn(M, lda, generator=g, device=DEV)
    a[:, K:] = nan
    A = _place(a, a_off)
    a_pre = None
    if a_act != ACT_NONE:
        p = torch.randn(M, lda, generator=g, device=DEV) * (1.0 if a_act == ACT_GIVEN else 3.0)
        p[:, K:] = nan
        a_pre = _place(p, a_off)
    W = torch.randn(N, K, generator=g, device=DEV) / math.sqrt(K)
    Wk = _operand(kern, W)
    b = torch.randn(N, generator=g, device=DEV) if bias else None
    add = None
    if addend:
        add = torch.randn(M, ld_add, generator=g, device=DEV)
        add[:, N:] = nan
    tag = f"{kern} M={M} K={K} N={N} a_act={a_act} act={act}"

    # fp64 truth and the per-element scale s
    a64 = A[:, :K].double()
    if a_act != ACT_NONE:
        a64 = a64 * dact64(a_pre[:, :K].double(), a_act)
    w64 = W.double()
    pre64 = a64 @ w64.t()
    s = a64.abs() @ w64.abs().t()
    if b is not None:
        pre64 += b.double()
        s += b.double().abs()
    add64 = add[:, :N].double() if add is not None else torch.zeros_like(pre64)

    Y, P = _sentinel(M + 2, ldy), _sentinel(M + 2, ldy)
    _abi(kern, A, M, K, lda, a_pre, a_act, Wk, N, b, act, add, ld_add, Y, ldy, P)
    _untouched(Y, M, N, f"{tag}: Y")
    _untouched(P, M, N, f"{tag}: y_pre")
    pre, y = P[:M, :N].double(), Y[:M, :N].double()
    assert bool(torch.isfinite(pre).all()) and bool(torch.isfinite(y).all()), f"{tag}: non-finite output"

    r = (pre - pre64).abs() / (EPS * s.clamp_min(1e-30))
    if kern == "tc":
        c = C_TC
        r = _note(f"tc GEMM ratio, {_cdiv(K, 16)} K-tiles", r.max())
    else:
        c = C_FFMA
        r = _note("ffma GEMM ratio", r.max())
    assert r <= c, f"{tag}: GEMM error {r:.3g} x 2^-24 s > {c}"

    f = act64(pre, act)
    r = _note("epilogue Y ratio", ((y - (f + add64)).abs() / (EPS * (f.abs() + add64.abs() + 1.0))).max())
    assert r <= C_EPI, f"{tag}: epilogue error {r:.3g} x 2^-24 > {C_EPI}"

    Y2, D = _sentinel(M + 2, ldy), _sentinel(M + 2, ldy)
    _abi(kern, A, M, K, lda, a_pre, a_act, Wk, N, b, act | SAVE_DERIV, add, ld_add, Y2, ldy, D)
    _untouched(Y2, M, N, f"{tag}: Y (SAVE_DERIV)")
    _untouched(D, M, N, f"{tag}: y_pre (SAVE_DERIV)")
    if act == ACT_NONE:
        assert bool((D[:M, :N] == 1.0).all()), f"{tag}: SAVE_DERIV with ACT_NONE must store act' = 1"
        assert _bitwise_equal(Y2[:M, :N], Y[:M, :N]), f"{tag}: SAVE_DERIV changed Y"
    else:
        d64 = dact64(pre, act)
        r = _note("epilogue act' ratio", ((D[:M, :N].double() - d64).abs() / (EPS * (pre.abs() + 1.0))).max())
        assert r <= C_EPI, f"{tag}: saved act' error {r:.3g} x 2^-24 > {C_EPI}"
        r = _note("epilogue Y ratio", ((Y2[:M, :N].double() - (f + add64)).abs() /
                                       (EPS * (f.abs() + add64.abs() + 1.0))).max())
        assert r <= C_EPI, f"{tag}: epilogue error (SAVE_DERIV) {r:.3g} x 2^-24 > {C_EPI}"


# every (a_act, act) the tensor-core kernel accepts, with and without bias / addend, padded lda / ldy / ld_add
TC_VARIANTS = [  # a_act, act, bias, addend
    (ACT_NONE, ACT_NONE, True, True), (ACT_NONE, ACT_SILU, True, False), (ACT_NONE, ACT_SSP, False, True),
    (ACT_SILU, ACT_NONE, False, False), (ACT_SSP, ACT_NONE, True, True), (ACT_GIVEN, ACT_NONE, False, True)]

_TC_K = [4, 12, 16, 20, 48, 80, 132, 144, 1024]            # ceil(K/16) = 1, 1, 1, 2, 3, 5, 9, 9, 64
_TC_N = [4, 60, 64, 68, 128, 132, 192, 256, 260, 384]
_TC_M = [1, 63, 64, 65, 127, 129, 257]
TC_SHAPES = sorted(set(
    [(129, k, 64) for k in _TC_K]                  # one 64-wide column block: odd unit counts take the peeled else-tail
    + [(129, k, 256) for k in _TC_K]               # two 64-column blocks per consumer (TN = 128)
    + [(129, 80, n) for n in _TC_N]
    + [(m, 80, 132) for m in _TC_M]
    + [(1, 4, 4), (65, 1024, 384), (257, 12, 260), (63, 132, 192), (16128, 256, 128)]))   # last: the PaiNN mix^T layer


def _tc_variants(M, K, N, seed):
    for i, (a_act, act, bias, addend) in enumerate(TC_VARIANTS):
        _check_layer("tc", M, K, N, a_act, act, bias=bias, addend=addend, lda=K + 4 * (i % 3 == 0),
                     ldy=N + 4 * (i % 2), ld_add=N + 8 * (i % 4 == 1), seed=seed + i)


@pytest.mark.parametrize("M,K,N", TC_SHAPES)
def test_tc_elementwise(M, K, N):
    _tc_variants(M, K, N, seed=M + 7 * K + 31 * N)


def test_tc_elementwise_at_column_tile_threshold():
    """N = 128 switches from 64- to 128-wide column tiles when 64-wide tiles need more than one wave of CTAs"""
    m = tc_last_narrow_rows(128)
    for M in (m, m + 1):
        _tc_variants(M, 80, 128, seed=M)


FFMA_SHAPES = [  # M, K, N, lda, ldy, a_off (floats off 16 B alignment, A and a_pre)
    (129, 13, 64, 13, 64, 0),       # K % 4 != 0: every A load on the scalar path
    (77, 25, 68, 28, 68, 0),        # K % 4 != 0 with lda % 4 == 0: vector loads, scalar tail chunk
    (129, 64, 13, 64, 17, 0),       # N % 4 != 0, ldy % 4 != 0
    (200, 48, 70, 48, 70, 0),       # N % 4 != 0 across two column tiles
    (129, 32, 64, 32, 65, 0),       # ldy % 4 != 0 with N % 4 == 0: scalar stores
    (129, 64, 128, 64, 128, 1),     # contiguous A one float off 16 B alignment
    (65, 13, 20, 13, 20, 1),
    (333, 384, 128, 384, 132, 0),
    (100, 1024, 64, 1024, 64, 0),
]
FFMA_ACTS = [(a, f) for a in (ACT_NONE, ACT_SILU, ACT_SSP, ACT_GIVEN) for f in (ACT_NONE, ACT_SILU, ACT_SSP)]


@pytest.mark.parametrize("M,K,N,lda,ldy,a_off", FFMA_SHAPES)
def test_ffma_elementwise(M, K, N, lda, ldy, a_off):
    """every (a_act, act) pair the C ABI accepts, including the six with both a prologue and an activation"""
    for i, (a_act, act) in enumerate(FFMA_ACTS):
        _check_layer("ffma", M, K, N, a_act, act, bias=i % 3 != 1, addend=i % 2 == 0, lda=lda, ldy=ldy,
                     ld_add=N + 3 * (i % 4 == 2), a_off=a_off, seed=i)


@pytest.mark.parametrize("bm", [32, 64, 128])
def test_ffma_elementwise_each_row_tile(bm):
    """the M at which spk_dense switches to row tile bm, and the M just below the next switch"""
    N = 132
    lo = 1 if bm == 32 else ffma_first_rows(bm, N)
    hi = ffma_first_rows(2 * bm, N) - 1 if bm < 128 else lo + 1000
    for M in (lo, hi):
        assert ffma_bm(M, N) == bm
        for i, (a_act, act) in enumerate([(ACT_NONE, ACT_SILU), (ACT_SSP, ACT_NONE), (ACT_GIVEN, ACT_SSP)]):
            _check_layer("ffma", M, 37, N, a_act, act, seed=M + i)


# ------------------------------------------------------------------------------------------------ accumulation bias
@pytest.mark.parametrize("kern", ["tc", "ffma"])
@pytest.mark.parametrize("K", [64, 1024, 4096])
def test_positive_operands_unbiased(kern, K):
    """With A, W > 0 every rounding that leans one way adds up: a K-sum that truncates across K-tiles is biased by about
    ceil(K/16) * 2^-25 relative.  The mean relative error must stay below a constant that does not grow with K."""
    M, N = 2048, 128
    g = _gen(K)
    A = torch.rand(M, K, generator=g, device=DEV)
    W = torch.rand(N, K, generator=g, device=DEV)
    Y = torch.empty(M, N, device=DEV)
    _abi(kern, A, M, K, K, None, ACT_NONE, _operand(kern, W), N, None, ACT_NONE, None, N, Y, N, None)
    ref = A.double() @ W.double().t()
    mean = _note(f"{kern} |mean relative error| on positive operands, K={K}", ((Y.double() - ref) / ref).mean().abs() / EPS)
    c = BIAS_TC if kern == "tc" else BIAS_FFMA
    assert mean <= c, f"{kern} K={K}: mean relative error {mean:.3g} x 2^-24 > {c}"


# ----------------------------------------------------------------------------------------------- bitwise invariants
def _layer_pair(kern, A, Wk, N, b, add, P, M):
    """a forward layer (bias, ssp, addend) and a backward one (ACT_GIVEN prologue) on the first M rows"""
    K = A.shape[1]
    Y1, Y2 = torch.empty(M, N, device=DEV), torch.empty(M, N, device=DEV)
    _abi(kern, A, M, K, K, None, ACT_NONE, Wk, N, b, ACT_SSP, add, N, Y1, N, None)
    _abi(kern, A, M, K, K, P, ACT_GIVEN, Wk, N, None, ACT_NONE, None, N, Y2, N, None)
    return Y1, Y2


@pytest.mark.parametrize("kern", ["tc", "ffma"])
def test_rows_independent_bitwise(kern):
    """Y(A)[r0:r1] == Y(A[r0:r1]): a row's result does not depend on where its row tile starts"""
    M, K, N, r0, r1 = 300, 80, 256, 70, 250
    g = _gen(11)
    A, P = torch.randn(M, K, generator=g, device=DEV), torch.randn(M, K, generator=g, device=DEV)
    W = torch.randn(N, K, generator=g, device=DEV) / math.sqrt(K)
    b, add = torch.randn(N, generator=g, device=DEV), torch.randn(M, N, generator=g, device=DEV)
    Wk = _operand(kern, W)
    full = _layer_pair(kern, A, Wk, N, b, add, P, M)
    part = _layer_pair(kern, A[r0:r1].clone(), Wk, N, b, add[r0:r1].clone(), P[r0:r1].clone(), r1 - r0)
    for f, p in zip(full, part):
        assert _bitwise_equal(f[r0:r1], p)


def test_tc_column_tile_width_bitwise():
    """N = 128 below and above the wave threshold: 64- and 128-wide column tiles give every 64-column block the same
    m64n64k8 products in the same order, so the rows they share are bitwise equal"""
    from schnetpack_b200 import ops

    N, K = 128, 144
    m = tc_last_narrow_rows(N)
    g = _gen(12)
    A, P = torch.randn(m + 1, K, generator=g, device=DEV), torch.randn(m + 1, K, generator=g, device=DEV)
    W = torch.randn(N, K, generator=g, device=DEV) / math.sqrt(K)
    b, add = torch.randn(N, generator=g, device=DEV), torch.randn(m + 1, N, generator=g, device=DEV)
    wide = _layer_pair("tc", A, ops.tc_pack_weight(W), N, b, add, P, m + 1)
    narrow = _layer_pair("tc", A, ops.tc_pack_weight(W), N, b, add, P, m)
    for w, n in zip(wide, narrow):
        assert _bitwise_equal(w[:m], n)


@pytest.mark.parametrize("K", [37, 64])
def test_ffma_row_tile_bitwise(K):
    """k_dense at row tiles 32, 64 and 128: every output is the same FMA chain in K order"""
    N = 132
    m64, m128 = ffma_first_rows(64, N), ffma_first_rows(128, N)
    g = _gen(13)
    A, P = torch.randn(m128, K, generator=g, device=DEV), torch.randn(m128, K, generator=g, device=DEV)
    W = torch.randn(N, K, generator=g, device=DEV) / math.sqrt(K)
    b, add = torch.randn(N, generator=g, device=DEV), torch.randn(m128, N, generator=g, device=DEV)
    Wk = _operand("ffma", W)
    ref = _layer_pair("ffma", A, Wk, N, b, add, P, m128)
    for M in (m64 - 1, m64, m128 - 1):
        for r, y in zip(ref, _layer_pair("ffma", A, Wk, N, b, add, P, M)):
            assert _bitwise_equal(r[:M], y), f"rows {M} (row tile {ffma_bm(M, N)})"


def test_launch_chain_bitwise():
    """tc -> tc -> ffma -> tc (ACT_GIVEN prologue) enqueued back to back must equal the same chain synchronised after
    every layer, and a replay of its CUDA-graph capture with new inputs copied in.

    Every layer is launched with programmatic dependent launch: it may start while its predecessor runs.  k_dense_tc
    issues its weight TMAs before griddepcontrol.wait and loads A only after it; a load moved above the wait would read
    the NaN the output buffers are filled with.  Such an ordering bug shows up only when the timing lets it, so this
    test can catch it only probabilistically: a pass does not prove the ordering right."""
    from schnetpack_b200 import ops

    M, K0, N1, N2, N4 = 16128, 128, 256, 128, 128
    g = _gen(14)
    X = torch.randn(M, K0, generator=g, device=DEV)
    X2 = torch.randn(M, K0, generator=g, device=DEV)
    W1 = torch.randn(N1, K0, generator=g, device=DEV) / math.sqrt(K0)
    W2 = torch.randn(N2, N1, generator=g, device=DEV) / math.sqrt(N1)
    B3 = torch.randn(N2, N1, generator=g, device=DEV) / math.sqrt(N2)
    W4 = torch.randn(N4, N1, generator=g, device=DEV) / math.sqrt(N1)
    b1, b2, b3 = (torch.randn(n, generator=g, device=DEV) for n in (N1, N2, N1))
    w1p, w2p, w4p = ops.tc_pack_weight(W1), ops.tc_pack_weight(W2), ops.tc_pack_weight(W4)
    bufs = [torch.empty(M, n, device=DEV) for n in (N1, N1, N2, N1, N4)]    # Y1, act'(pre1), Y2, Y3, Y4

    def layers(x, sync):
        y1, d1, y2, y3, y4 = bufs
        _abi("tc", x, M, K0, K0, None, ACT_NONE, w1p, N1, b1, ACT_SILU | SAVE_DERIV, None, N1, y1, N1, d1)
        sync()
        _abi("tc", y1, M, N1, N1, None, ACT_NONE, w2p, N2, b2, ACT_SSP, None, N2, y2, N2, None)
        sync()
        _abi("ffma", y2, M, N2, N2, None, ACT_NONE, B3, N1, b3, ACT_NONE, None, N1, y3, N1, None)
        sync()
        _abi("tc", y3, M, N1, N1, d1, ACT_GIVEN, w4p, N4, None, ACT_NONE, None, N4, y4, N4, None)

    def run(x, sync):
        for t in bufs:
            t.fill_(float("nan"))
        layers(x, sync)
        torch.cuda.synchronize()
        return [t.clone() for t in bufs]

    serial = run(X, torch.cuda.synchronize)
    assert all(bool(torch.isfinite(t).all()) for t in serial)
    for _ in range(3):
        for s, c in zip(serial, run(X, lambda: None)):
            assert _bitwise_equal(c, s)

    x_static = X.clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        layers(x_static, lambda: None)
    serial2 = run(X2, torch.cuda.synchronize)
    for t in bufs:
        t.fill_(float("nan"))
    x_static.copy_(X2)
    graph.replay()
    torch.cuda.synchronize()
    for s, c in zip(serial2, bufs):
        assert _bitwise_equal(c, s)


# --------------------------------------------------------------------------------------------------------- guards
@pytest.mark.parametrize("kern,K,lda", [("tc", 20, 32), ("tc", 132, 136), ("ffma", 13, 16), ("ffma", 25, 27)])
def test_k_tail_never_read(kern, K, lda):
    """A and a_pre with NaN in columns [K, lda) give finite results, bitwise equal to a compact copy"""
    M, N = 257, 68
    g = _gen(15)
    A, P = torch.randn(M, lda, generator=g, device=DEV), torch.randn(M, lda, generator=g, device=DEV)
    A[:, K:] = float("nan")
    P[:, K:] = float("nan")
    W = torch.randn(N, K, generator=g, device=DEV) / math.sqrt(K)
    b = torch.randn(N, generator=g, device=DEV)
    Wk = _operand(kern, W)
    Ac, Pc = A[:, :K].contiguous(), P[:, :K].contiguous()
    for a_act, act in ((ACT_NONE, ACT_SILU | SAVE_DERIV), (ACT_SSP, ACT_NONE), (ACT_GIVEN, ACT_NONE)):
        out = []
        for a, p, ld in ((A, P, lda), (Ac, Pc, K)):
            Y, D = torch.empty(M, N, device=DEV), torch.empty(M, N, device=DEV)
            _abi(kern, a, M, K, ld, p, a_act, Wk, N, b, act, None, N, Y, N, D)
            out.append((Y, D))
        (y, d), (yc, dc) = out
        assert bool(torch.isfinite(y).all()) and bool(torch.isfinite(d).all())
        assert _bitwise_equal(y, yc) and _bitwise_equal(d, dc)


@pytest.mark.parametrize("kern", ["tc", "ffma"])
def test_nonfinite_input_stays_in_its_row(kern):
    """one +inf in row r of A makes row r non-finite and leaves every other row bitwise unchanged"""
    M, K, N, r = 200, 80, 132, 77
    g = _gen(16)
    A = torch.randn(M, K, generator=g, device=DEV)
    W = torch.randn(N, K, generator=g, device=DEV) / math.sqrt(K)
    b = torch.randn(N, generator=g, device=DEV)
    Wk = _operand(kern, W)
    A_hit = A.clone()
    A_hit[r, 5] = float("inf")
    outs = []
    for a in (A, A_hit):
        Y, P = torch.empty(M, N, device=DEV), torch.empty(M, N, device=DEV)
        _abi(kern, a, M, K, K, None, ACT_NONE, Wk, N, b, ACT_NONE, None, N, Y, N, P)
        outs.append((Y, P))
    keep = torch.arange(M, device=DEV) != r
    for clean, hit in zip(*outs):
        assert not bool(torch.isfinite(hit[r]).any())
        assert _bitwise_equal(clean[keep], hit[keep])


# ---------------------------------------------------------------------------------------------------- Lin dispatch
def test_lin_falls_back_where_tensor_core_path_refuses():
    """Lin sends every call spk_dense_tc would refuse -- a base pointer off 16 B alignment (A, a_pre, bias, out) or a
    backward prologue together with a forward activation -- to the FFMA kernel, bitwise equal to ops.dense"""
    from schnetpack_b200 import ops

    old = ops.DENSE_IMPL
    ops.DENSE_IMPL = "tc"
    try:
        M, K, N = 129, 64, 128
        g = _gen(17)
        A, P = torch.randn(M, K, generator=g, device=DEV), torch.randn(M, K, generator=g, device=DEV)
        G = torch.randn(M, N, generator=g, device=DEV)
        W = torch.randn(N, K, generator=g, device=DEV) / math.sqrt(K)
        b = torch.randn(N, generator=g, device=DEV)
        lin = ops.Lin(W, b)
        assert lin.w_pk is not None
        Am, Pm, Gm = _place(A, 1), _place(P, 1), _place(G, 1)
        assert Am.is_contiguous() and Am.data_ptr() % 16 == 4

        # aligned calls stay on the tensor-core kernel
        assert _bitwise_equal(lin.fwd(A, ACT_SILU), ops.dense_tc(A, lin.w_pk, N, lin.b, ACT_SILU))
        for act in (ACT_NONE, ACT_SILU, ACT_SSP):
            assert _bitwise_equal(lin.fwd(Am, act), ops.dense(Am, lin.wt, lin.b, act))
        y, d = lin.fwd(Am, ACT_SSP, save_deriv=True)
        y_ref, d_ref = ops.dense(Am, lin.wt, lin.b, ACT_SSP | SAVE_DERIV, save_pre=True)
        assert _bitwise_equal(y, y_ref) and _bitwise_equal(d, d_ref)
        assert _bitwise_equal(lin.bwd(Gm), ops.dense(Gm, lin.w, None))
        assert _bitwise_equal(lin.bwd(G, a_pre=_place(d, 1), a_act=ACT_GIVEN),
                              ops.dense(G, lin.w, None, a_pre=d, a_act=ACT_GIVEN))
        out = _place(torch.zeros(M, N, device=DEV), 1)
        assert lin.fwd(A, ACT_SILU, out=out).data_ptr() == out.data_ptr()
        assert _bitwise_equal(out, ops.dense(A, lin.wt, lin.b, ACT_SILU))
        assert _bitwise_equal(lin.fwd(A, ACT_SILU, a_pre=P, a_act=ACT_SSP),
                              ops.dense(A, lin.wt, lin.b, ACT_SILU, a_pre=P, a_act=ACT_SSP))
        lin_b = ops.Lin(W, _place(b, 1))
        assert _bitwise_equal(lin_b.fwd(A, ACT_SILU), ops.dense(A, lin.wt, lin.b, ACT_SILU))
    finally:
        ops.DENSE_IMPL = old
