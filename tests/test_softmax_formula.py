"""NumPy float32 restatement of the softmax coalition kernel's per-element formula (csrc/dks_multi.cuh) and its clamp
rule, held to float64 direct sums  sum_j w'_j softmax_c(a + d_j).

Per row s and class c the plan holds Dm_c(s, j) = 2^(d_c - max_c' d_c') in fp32 and lo_c(s) = min_j log2 Dm_c(s, j); per
instance A_c = 2^(a_c - max_c' a_c') is formed as 2^n 2^f with f exact in fp32.  Then u_c = A_c Dm_c, den = sum_c u_c,
and each class accumulates u_c (w'_j / den).  Rows with lo_ca(s) < -60 (ca = argmax a) take the float64 clamped path."""
import numpy as np
import pytest

LO_MIN = -60.0


def _plan(d):
    """d [N, C] log2-unit background parts of one row -> Dm [N, C] fp32, lo [C]."""
    e = d - d.max(axis=1, keepdims=True)
    return np.exp2(e).astype(np.float32), e.min(axis=0)


def _factors(a):
    e = a - a.max()
    en = np.rint(e)
    A = np.exp2((e - en).astype(np.float32)) * np.exp2(np.maximum(en, -126)).astype(np.float32)
    return np.where(e < -125.0, np.float32(0), A).astype(np.float32)


def kernel_row(a, d, wn):
    """What the kernel accumulates for one (instance, row): [C] fp32 sums (clamped rows in float64)."""
    Dm, lo = _plan(d)
    if lo[int(np.argmax(a))] < LO_MIN:
        t = a[None, :] + d
        p = np.exp2(t - t.max(axis=1, keepdims=True))
        p /= p.sum(axis=1, keepdims=True)
        return (wn[:, None] * p).sum(0).astype(np.float32), True
    A = _factors(a)
    acc = np.zeros(len(a), dtype=np.float32)
    for j in range(d.shape[0]):
        u = A * Dm[j]
        den = np.float32(0)
        for c in range(len(a)):
            den = np.float32(den + u[c])
        rw = np.float32(np.float32(wn[j]) * np.float32(1.0 / den))
        acc = (acc + u * rw).astype(np.float32)
    return acc, False


def direct(a, d, wn):
    t = a[None, :] + d
    p = np.exp2(t - t.max(axis=1, keepdims=True))
    p /= p.sum(axis=1, keepdims=True)
    return (wn[:, None] * p).sum(0)


def _weights(rng, N, weighted):
    w = rng.uniform(0.05, 1.0, N) if weighted else np.ones(N)
    return (N * w / w.sum()).astype(np.float32).astype(np.float64)


@pytest.mark.parametrize("C", [2, 3, 4, 5, 8])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("gap", [0.0, 40.0, 58.0, 80.0])
def test_formula_against_float64(C, weighted, gap):
    """Score gaps (in nats) up to 80 between a dominant class and the others, in the instance part and the background
    part; every class sum resolved to 1e-5 of itself down to probabilities of 2^-60."""
    rng = np.random.default_rng(C * 100 + int(gap) + weighted)
    N = 37
    wn = _weights(rng, N, weighted)
    L2E = 1.4426950408889634
    for trial in range(20):
        a = rng.normal(0, 3, C) * L2E
        d = rng.normal(0, 3, (N, C)) * L2E
        a[trial % C] += gap * L2E * (1 if trial % 2 else -1)
        d[:, (trial + 1) % C] += gap * L2E * (1 if trial % 3 else -1)
        got, _ = kernel_row(a, d, wn)
        want = direct(a, d, wn)
        assert np.all(np.isfinite(got))
        keep = want / N > 2.0 ** -60
        np.testing.assert_allclose(got[keep], want[keep], rtol=1e-5)
        assert np.all(got[~keep] <= 2.0 ** -55 * N)


def test_clamp_rule_edges():
    """den is bounded by Dm_ca(s, j) >= 2^lo_ca: just inside the bound the fp32 path stays exact to 1e-5 for the small
    classes; just outside, the row goes to the clamped path, which never produces Inf or NaN."""
    C, N = 3, 5
    wn = np.ones(N)
    a = np.array([0.0, -10.0, -30.0])
    for lo_edge, clamped_expected in [(-59.5, False), (-60.5, True), (-125.0, True), (-200.0, True)]:
        d = np.zeros((N, C))
        d[:, 1] = 0.0
        d[0, 0] = lo_edge                  # class 0 (argmax a) sinks to lo_edge below the row's max in column 0
        got, clamped = kernel_row(a, d, wn)
        want = direct(a, d, wn)
        assert clamped == clamped_expected
        assert np.all(np.isfinite(got))
        keep = want / N > 2.0 ** -60
        np.testing.assert_allclose(got[keep], want[keep], rtol=1e-5)
    # largest and smallest fp32-range instance factors: A = 2^-125 and below flush to 0 without harm
    a = np.array([0.0, -124.9, -126.0, -300.0])
    A = _factors(a)
    assert A[0] == 1.0 and A[1] > 0 and A[2] == 0 and A[3] == 0
