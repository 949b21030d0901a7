"""The weighted pair identity of the shared-plan kernels (dks_shared.cuh: dm_quad_w, w2_quad, quad_acc_w), restated in
NumPy float32 with the kernels' order of operations, against float64 direct sums  sum_j w'_j / (1 + A Dm_j)  and
sum_j w'_j A Dm_j / (1 + A Dm_j)  over skewed k-means-like weights.  Pins the numerics of the four-floats-per-pair layout
(X and Y both stored) without a GPU, up to the largest A the packed path takes (1e18, just under 2^59.8) on backgrounds
whose weight sits on a few rows (W2 = w'a + w'b of a pair in the hundreds)."""
import numpy as np
import pytest

f32 = np.float32


def _fma(a, b, c):
    """float32 fused multiply-add (the product of two float32 values is exact in float64)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def _weighted_sums(A, dm, w):
    """(sum p1, sum p0) of one row as the weighted kernels form them: pairs (0,2) (1,3) of every quad of columns, columns
    past N with Dm = 0 and weight 0 (up to an even number of quads), two accumulator chains over the quads.  ``A``
    [rows], ``dm`` [rows, N] float32 (the normalised row of Dm), ``w`` [N] float32 (N w_j)."""
    rows, N = dm.shape
    nq = ((N + 3) // 4 + 1) & ~1
    d = np.zeros((rows, 4 * nq), f32)
    d[:, :N] = dm
    ww = np.zeros(4 * nq, f32)
    ww[:N] = w
    A = A.astype(f32)
    AA = A * A
    acc1 = [np.zeros((rows, 2), f32), np.zeros((rows, 2), f32)]
    acc0 = [np.zeros((rows, 2), f32), np.zeros((rows, 2), f32)]
    for q in range(nq):
        d0, d1, d2, d3 = (d[:, 4 * q + k] for k in range(4))
        w0, w1, w2, w3 = (ww[4 * q + k] for k in range(4))
        ds = np.stack([d0 + d2, d1 + d3], -1)
        dq = np.stack([d0 * d2, d1 * d3], -1)
        X = np.stack([w0 * d2 + w2 * d0, w1 * d3 + w3 * d1], -1)
        Y = np.stack([w0 * d0 + w2 * d2, w1 * d1 + w3 * d3], -1)
        W2 = np.array([w0 + w2, w1 + w3], f32)[None, :].repeat(rows, 0)
        A2, AA2 = np.stack([A, A], -1), np.stack([AA, AA], -1)
        sm = A2 * ds
        qq = AA2 * dq
        den = (sm + f32(1)) + qq
        r = (f32(1) / den).astype(f32)                         # rcp.approx: within 1 ulp of this
        acc1[q & 1] = _fma(r, _fma(A2, X, W2), acc1[q & 1])
        acc0[q & 1] = _fma(r * qq, W2, _fma(r, A2 * Y, acc0[q & 1]))       # (r q) W2: q W2 may pass the fp32 range
    s1 = acc1[0] + acc1[1]
    s0 = acc0[0] + acc0[1]
    return s1[:, 0] + s1[:, 1], s0[:, 0] + s0[:, 1]


def _direct(A, dm, w):
    u = A[:, None].astype(np.float64) * dm.astype(np.float64)
    p1 = 1.0 / (1.0 + u)
    return p1 @ w.astype(np.float64), (u * p1) @ w.astype(np.float64)


def _kmeans_weights(rng, N, concentrated=False):
    w = np.round(np.exp(rng.uniform(0.0, np.log(500.0), size=N)))
    w[0], w[-1] = 1.0, 400.0
    if N > 4:
        w[N // 2] = 0.0
    if concentrated:                       # most of the weight on the pair (0, 2): W2 close to N
        w[:] = 1.0
        w[0], w[2] = 20000.0, 5000.0
    return (N * w / w.sum()).astype(f32)


@pytest.mark.parametrize("N,concentrated", [(1, False), (2, False), (3, False), (5, False), (17, False), (100, False),
                                            (128, False), (128, True), (200, True), (300, True)])
@pytest.mark.parametrize("log2A", [-30.0, -8.0, 0.0, 8.0, 30.0, 55.0, 59.7])
def test_weighted_pair_formula_matches_float64(N, concentrated, log2A):
    rng = np.random.default_rng(N * 101 + int(log2A))
    rows = 64
    # normalised rows of Dm: entries 2^(d - rint(max d)) in (0, sqrt 2], down to 2^-40 (a spread of scores); the rows of
    # the largest A sit at the packed path's limit with every entry near sqrt 2, where q = A^2 Dma Dmb is largest
    d = -rng.uniform(0.0, 40.0, size=(rows, N))
    d -= np.rint(d.max(axis=1, keepdims=True))
    if log2A > 59:
        d[:] = rng.uniform(0.45, 0.5, size=(rows, N))
    dm = np.exp2(d).astype(f32)
    A = np.exp2(log2A + rng.uniform(-0.5, 0.5, size=rows))
    if log2A > 59:
        A = np.minimum(A, 1.0e18)
    w = _kmeans_weights(rng, N, concentrated)
    s1, s0 = _weighted_sums(A, dm, w)
    t1, t0 = _direct(A, dm, w)
    # each sum to a few float32 ulps of its own magnitude: p0 keeps its own sum, so it stays accurate where it is tiny
    assert np.all(np.abs(s1 - t1) <= 2e-6 * t1 + 1e-30), np.max(np.abs(s1 - t1) / t1)
    assert np.all(np.abs(s0 - t0) <= 2e-6 * t0 + 1e-30), np.max(np.abs(s0 - t0) / t0)


def test_pair_product_times_pair_weight_does_not_overflow():
    """200 rows, one of them carrying nearly all the weight (W2 = 192), every entry of Dm at sqrt 2 and A just under the
    clamped path's threshold: q W2 = 2e36 * 192 would pass the fp32 range; (r q) W2 does not."""
    N = 200
    w = np.ones(N)
    w[0] = 5000.0
    w = (N * w / w.sum()).astype(f32)
    dm = np.full((4, N), 1.41, f32)
    A = np.array([0.5e18, 0.9e18, 0.99e18, 1.0e18])
    assert float(A[2]) ** 2 * 1.41 ** 2 * float(w[0] + w[2]) > float(np.finfo(f32).max)
    s1, s0 = _weighted_sums(A, dm, w)
    t1, t0 = _direct(A, dm, w)
    assert np.all(np.isfinite(s0)) and np.all(np.isfinite(s1))
    np.testing.assert_allclose(s0, t0, rtol=2e-6)
    np.testing.assert_allclose(s1, t1, rtol=2e-6)


def test_zero_weight_columns_contribute_nothing():
    """A pair whose second column has weight 0 and Dm 0 (the padding past N) gives exactly the single-column terms."""
    rng = np.random.default_rng(5)
    dm = rng.uniform(0.1, 1.4, size=(16, 1)).astype(f32)
    A = np.exp2(rng.uniform(-4, 4, size=16))
    w = np.array([3.0], f32)
    s1, s0 = _weighted_sums(A, dm, w)
    u = (A.astype(f32) * dm[:, 0]).astype(f32)
    r = (f32(1) / (f32(1) + u)).astype(f32)
    np.testing.assert_array_equal(s1, (w[0] * r).astype(f32))
    t1, t0 = _direct(A, dm, w)
    np.testing.assert_allclose(s0, t0, rtol=2e-6)
