"""The one-vs-rest head (normalised per-class sigmoids) on the host: the NumPy head against scikit-learn's
``_predict_proba_lr``, model extraction, a NumPy float32 restatement of the coalition kernel's per-element formula and
range rule (csrc/dks_multi.cuh), and the float64 reference (tests/ovr_reference.py) against the oracle and exact Shapley
values."""
import itertools
from math import factorial

import numpy as np
import pytest

from ovr_reference import OvrReference, ovr_probabilities


def _predict_proba_lr(z):
    """scikit-learn 0.23.2 ``LinearClassifierMixin._predict_proba_lr`` for C >= 3 classes, restated."""
    from scipy.special import expit
    prob = expit(z)
    prob /= prob.sum(axis=1).reshape((prob.shape[0], -1))
    return prob


def _model(seed, C=4, D=6):
    rng = np.random.default_rng(seed)
    return rng.normal(0, 1.0, (C, D)), rng.normal(0, 0.5, C), rng.standard_normal((40, D)) * 2.0


# ---------------------------------------------------------------------------------------------------------------------
# the head and model extraction
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [3, 4, 8])
def test_numpy_head_is_predict_proba_lr(C):
    from distributedkernelshap_b200.predictors import LinearModelSpec
    W, b, X = _model(C, C=C)
    spec = LinearModelSpec(W, b, "ovr")
    np.testing.assert_allclose(spec(X), _predict_proba_lr(X @ W.T + b), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(ovr_probabilities(X @ W.T + b), spec(X), rtol=1e-12, atol=1e-15)
    assert spec.n_outputs == C and spec.act_code == 3


def test_numpy_head_equals_installed_one_vs_rest_classifier():
    from sklearn.linear_model import LogisticRegression
    from sklearn.multiclass import OneVsRestClassifier
    from distributedkernelshap_b200.predictors import extract_linear_spec
    rng = np.random.default_rng(3)
    X = rng.standard_normal((300, 5))
    y = np.argmax(X[:, :4] + 0.5 * rng.standard_normal((300, 4)), axis=1)
    ovr = OneVsRestClassifier(LogisticRegression()).fit(X, y)
    spec = extract_linear_spec(ovr.predict_proba)
    assert spec.activation == "ovr" and spec.W.shape == (4, 5)
    np.testing.assert_allclose(spec(X), ovr.predict_proba(X), rtol=1e-12, atol=1e-12)


class _LogReg:
    """Stand-in for a fitted scikit-learn 0.23.2 LogisticRegression (attributes only)."""

    def __init__(self, coef, intercept, multi_class, solver):
        self.coef_, self.intercept_, self.multi_class, self.solver = coef, intercept, multi_class, solver
        self.classes_ = np.arange(coef.shape[0])

    def predict_proba(self, X):
        return _predict_proba_lr(X @ self.coef_.T + self.intercept_)

    def predict(self, X):
        return self.classes_[np.argmax(self.predict_proba(X), axis=1)]


@pytest.mark.parametrize("multi_class,solver,want", [("ovr", "lbfgs", "ovr"), ("warn", "liblinear", "ovr"),
                                                     ("auto", "liblinear", "ovr"), ("auto", "lbfgs", "softmax"),
                                                     ("multinomial", "saga", "softmax")])
def test_extract_follows_the_0_23_2_rule(multi_class, solver, want):
    from distributedkernelshap_b200.predictors import extract_linear_spec
    W, b, X = _model(1)
    spec = extract_linear_spec(_LogReg(W, b, multi_class, solver).predict_proba)
    assert spec.activation == want
    np.testing.assert_array_equal(spec.W, W)


def test_extract_hook_and_stand_in_classifier():
    from distributedkernelshap_b200.predictors import LinearSoftmaxClassifier, extract_linear_spec
    W, b, X = _model(2, C=5)
    clf = LinearSoftmaxClassifier(W, b, multi_class="ovr")
    spec = extract_linear_spec(clf.predict_proba)
    assert spec.activation == "ovr"
    np.testing.assert_allclose(clf.predict_proba(X), _predict_proba_lr(X @ W.T + b), rtol=1e-12)
    assert extract_linear_spec(clf).activation == "ovr"                       # the dks_linear_spec() hook
    assert LinearSoftmaxClassifier(W[:1], b[:1], multi_class="ovr").dks_linear_spec().activation == "binary_logistic"


def test_extract_still_refuses():
    from sklearn.linear_model import LogisticRegression
    from sklearn.multiclass import OneVsRestClassifier
    from distributedkernelshap_b200.predictors import LinearModelSpec, extract_linear_spec
    W, b, X = _model(4)
    with pytest.raises(TypeError):
        extract_linear_spec(lambda x: _predict_proba_lr(x @ W.T + b))        # opaque callable
    with pytest.raises(TypeError):
        extract_linear_spec(_LogReg(W, b, "ovr", "liblinear").predict)         # labels
    with pytest.raises(ValueError):
        LinearModelSpec(W, b, "ovr", kappa=2.0)                                # a multinomial-style kappa
    with pytest.raises(ValueError):
        LinearModelSpec(W[:2], b[:2], "ovr")                                   # fewer than three classes
    rng = np.random.default_rng(5)
    Xf = rng.standard_normal((200, 4))
    Y = (Xf[:, :3] + 0.3 * rng.standard_normal((200, 3)) > 0).astype(int)
    multilabel = OneVsRestClassifier(LogisticRegression()).fit(Xf, Y)
    with pytest.raises(NotImplementedError):
        extract_linear_spec(multilabel.predict_proba)
    y = np.argmax(Xf[:, :3], axis=1)
    single = OneVsRestClassifier(LogisticRegression()).fit(Xf, y)
    with pytest.raises(TypeError):
        extract_linear_spec(single.decision_function)


# ---------------------------------------------------------------------------------------------------------------------
# the kernel's per-element formula and range rule
# ---------------------------------------------------------------------------------------------------------------------
LO_MIN, K_MAX, ND_MAX = -60.0, 64.0, 1048576.0
TINY = np.float32(2.0 ** -126)


def _ftz(x):
    x = np.asarray(x, dtype=np.float32)
    return np.where(np.abs(x) < TINY, np.float32(0), x).astype(np.float32)


def _plan(d):
    """d [N, C] log2-unit background parts of one row -> Dm [N, C] fp32, nd [N], lo [C], hi."""
    mx = d.max(axis=1)
    nd = np.clip(np.ceil(mx), -ND_MAX, ND_MAX)
    e = d - nd[:, None]
    hi = np.max(np.where(mx > ND_MAX, 1e30, nd))
    with np.errstate(over="ignore"):                  # parts beyond the nd clamp: the rule sends those rows away
        Dm = _ftz(np.exp2(e))
    return Dm, nd.astype(np.int64), e.min(axis=0), hi


def _factors(a, na):
    e = a - na
    en = np.rint(e)
    A = np.exp2((e - en).astype(np.float32)) * np.exp2(np.maximum(en, -126)).astype(np.float32)
    return np.where(e < -125.0, np.float32(0), A).astype(np.float32)


def _pow2(k):
    return np.float32(0) if k <= -127 else np.float32(2.0 ** k)


def kernel_row(a, d, wn):
    """What the kernel accumulates for one (instance, row): [C] fp32 sums, and whether the row took the scalar path."""
    Dm, nd, lo, hi = _plan(d)
    na = np.ceil(a.max())
    if lo[int(np.argmax(a))] < LO_MIN or na + hi > K_MAX:
        return direct(a, d, wn).astype(np.float32), True
    A = _factors(a, na)
    ka = int(np.clip(na, -2 * ND_MAX, 2 * ND_MAX))
    acc = np.zeros(len(a), dtype=np.float32)
    for j in range(d.shape[0]):
        k = ka + int(nd[j])
        alpha, beta = _pow2(-max(k, 0)), _pow2(max(min(k, 0), -127))
        u = _ftz(A * Dm[j])
        r = _ftz(u * (np.float32(1) / (beta * u + alpha).astype(np.float32)))
        den = np.float32(0)
        for c in range(len(a)):
            den = np.float32(den + r[c])
        rw = np.float32(np.float32(wn[j]) * np.float32(1.0 / den))
        acc = (acc + r * rw).astype(np.float32)
    return acc, False


def direct(a, d, wn):
    """sum_j w'_j p_c(a + d_j) in float64 (t in log2 units)."""
    return (wn[:, None] * ovr_probabilities((a[None, :] + d) * np.log(2.0))).sum(0)


def _weights(rng, N, weighted):
    w = rng.uniform(0.05, 1.0, N) if weighted else np.ones(N)
    return (N * w / w.sum()).astype(np.float32).astype(np.float64)


def _check(got, want, N):
    """Relative 1e-5, except that each element's probability below 2^-60 may be lost (the range rule)."""
    assert np.all(np.isfinite(got))
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=N * 2.0 ** -60)


L2E = 1.4426950408889634


@pytest.mark.parametrize("C", [3, 4, 8])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("case", ["moderate", "all_below", "one_above", "mixed"])
def test_formula_against_float64(C, weighted, case):
    """Every class far below 0 (the head tends to a softmax), one class far above 0, and classes saturated on both
    sides: every class sum resolved to 1e-5 of itself down to probabilities of 2^-60."""
    rng = np.random.default_rng(C * 100 + weighted + len(case))
    N = 37
    wn = _weights(rng, N, weighted)
    paths = set()
    for trial in range(20):
        a = rng.normal(0, 3, C) * L2E
        d = rng.normal(0, 3, (N, C)) * L2E
        if case == "all_below":
            a -= (60.0 + 10 * trial) * L2E
        elif case == "one_above":
            a[trial % C] += (10.0 + 3 * trial) * L2E
        elif case == "mixed":
            a[trial % C] += 40.0 * L2E
            a[(trial + 1) % C] -= 40.0 * L2E
            d[:, (trial + 2) % C] += 30.0 * L2E * (1 if trial % 2 else -1)
        got, clamped = kernel_row(a, d, wn)
        paths.add(clamped)
        _check(got, direct(a, d, wn), N)
    if case in ("moderate", "all_below"):
        assert paths == {False}


def test_range_rule_edges():
    """The scalar path takes rows whose den bound lo_ca falls below -60 or whose k = na + nd can exceed 64; just inside
    both bounds the fp32 path holds 1e-5, and nothing produces Inf or NaN."""
    C, N = 3, 5
    wn = np.ones(N)
    for a0, lo_edge, clamped_expected in [(0.0, -59.5, False), (0.0, -60.5, True), (60.0, 0.0, False),
                                          (64.2, 0.0, True), (200.0, 0.0, True), (-300.0, 0.0, False),
                                          (-300.0, -59.0, False), (2.0e7, 0.0, True)]:
        a = np.array([a0, a0 - 10.0, a0 - 30.0])
        d = np.zeros((N, C))
        d[0, 0] = lo_edge                  # class 0 (argmax a) sinks lo_edge below the row's max in column 0
        got, clamped = kernel_row(a, d, wn)
        assert clamped == clamped_expected, (a0, lo_edge)
        _check(got, direct(a, d, wn), N)


def test_background_parts_beyond_the_nd_clamp_take_the_scalar_path():
    C, N = 3, 4
    d = np.zeros((N, C))
    d[1] = 3.0e6
    _, _, _, hi = _plan(d)
    assert hi == 1e30
    got, clamped = kernel_row(np.zeros(C), d, np.ones(N))
    assert clamped


# ---------------------------------------------------------------------------------------------------------------------
# the float64 reference
# ---------------------------------------------------------------------------------------------------------------------
def _problem(seed, C, widths, N=12, weights=False):
    rng = np.random.default_rng(seed)
    groups, start = [], 0
    for wd in widths:
        groups.append(list(range(start, start + wd)))
        start += wd
    W = rng.normal(0, 0.8, (C, start))
    b = rng.normal(0, 0.5, C)
    bg, X = rng.standard_normal((N, start)), rng.standard_normal((3, start))
    return W, b, bg, X, groups, rng.uniform(0.2, 1.0, N) if weights else None


@pytest.mark.parametrize("link,C,weights", [("logit", 3, False), ("identity", 5, True), ("logit", 8, True)])
def test_reference_matches_oracle(link, C, weights):
    from distributedkernelshap_b200.plan import build_plan
    from distributedkernelshap_b200.predictors import LinearModelSpec
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    W, b, bg, X, groups, wts = _problem(21 + C, C, (1, 2, 1, 1, 2, 1), weights=weights)
    ref = OvrReference(W, b, bg, groups, wts, link=link)
    orc = KernelExplainerOracle(LinearModelSpec(W, b, "ovr"),
                                DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, wts), link=link)
    np.random.seed(1)
    plan = build_plan(6, 40)
    for x in X:
        want = orc.explain(x[None, :], plan=(plan.dense(), plan.weights), nsamples=40, l1_reg=False)
        got = ref.explain(x, plan=(plan.dense(), plan.weights))
        np.testing.assert_allclose(got, want.reshape(got.shape), rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("link", ["logit", "identity"])
def test_reference_full_enumeration_is_exact_shapley(link):
    from distributedkernelshap_b200.plan import build_plan
    W, b, bg, X, groups, wts = _problem(5, 4, (1, 2, 1, 1), weights=True)
    ref = OvrReference(W, b, bg, groups, wts, link=link)
    M = len(groups)
    plan = build_plan(M, 10 ** 6)
    x = X[0]

    def value(S):
        rows = bg.copy()
        for k in S:
            rows[:, groups[k]] = x[groups[k]]
        return ref.link(np.einsum("jc,j->c", _predict_proba_lr(b + rows @ W.T), ref.weights))

    exact = np.zeros((M, W.shape[0]))
    for k in range(M):
        rest = [q for q in range(M) if q != k]
        for r in range(M):
            for S in itertools.combinations(rest, r):
                wgt = factorial(r) * factorial(M - r - 1) / factorial(M)
                exact[k] += wgt * (value(S + (k,)) - value(S))
    got = ref.explain(x, plan=(plan.dense(), plan.weights))
    np.testing.assert_allclose(got, exact, rtol=1e-10, atol=1e-12)
