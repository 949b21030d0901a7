"""The mixture head (averaging ensembles of linear classifiers) on the host: extraction from fitted scikit-learn
ensembles against their own predict_proba / predict / decision_function, the refusals, a NumPy float32 restatement of the
CUDA-core kernel's per-element mixture sums (csrc/dks_mixture.cuh), and the float64 reference
(tests/mixture_reference.py) against the oracle driven by the real estimator and against exact Shapley values."""
import itertools
import warnings
from math import factorial

import numpy as np
import pytest

from mixture_reference import MixtureReference, mixture_outputs

TOL = 1e-12


def _data(seed, C, n=240, D=6):
    D = max(D, C)
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, D))
    z = X[:, :C] + 0.8 * rng.standard_normal((n, C)) if C > 2 else X[:, :1] + 0.8 * rng.standard_normal((n, 1))
    y = np.argmax(z, axis=1) if C > 2 else (z[:, 0] > 0).astype(int)
    return X, y


def _fit(est, C, seed=0):
    X, y = _data(seed, C)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return est.fit(X, y), X


def _spec(bound):
    from distributedkernelshap_b200.predictors import extract_linear_spec
    return extract_linear_spec(bound)


def _calibrated(base, **kw):
    from sklearn.calibration import CalibratedClassifierCV
    return CalibratedClassifierCV(base, method="sigmoid", **kw)


def _bases():
    from sklearn.linear_model import LogisticRegression, RidgeClassifier, SGDClassifier
    from sklearn.svm import LinearSVC
    return {"svc": LinearSVC(), "sgd": SGDClassifier(random_state=0), "logreg": LogisticRegression(),
            "ridge": RidgeClassifier()}


# ---------------------------------------------------------------------------------------------------------------------
# extraction: every accepted estimator reproduces its own method to 1e-12
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [2, 3, 4])
@pytest.mark.parametrize("base", ["svc", "sgd", "logreg", "ridge"])
def test_calibrated_classifier(base, C):
    clf, X = _fit(_calibrated(_bases()[base]), C)
    spec = _spec(clf.predict_proba)
    assert spec.activation == "mixture" and spec.K == 5
    assert spec.member == ("binary_logistic" if C == 2 else "ovr") and spec.n_outputs == C
    np.testing.assert_allclose(spec(X), clf.predict_proba(X), rtol=TOL, atol=TOL)


@pytest.mark.parametrize("C", [2, 3])
def test_calibrated_without_ensemble_is_a_single_head(C):
    from sklearn.svm import LinearSVC
    clf, X = _fit(_calibrated(LinearSVC(), ensemble=False), C)
    spec = _spec(clf.predict_proba)
    assert spec.activation == ("binary_logistic" if C == 2 else "ovr")
    np.testing.assert_allclose(spec(X), clf.predict_proba(X), rtol=TOL, atol=TOL)


@pytest.mark.parametrize("C", [2, 3])
def test_soft_voting_with_weights_and_nested_calibration(C):
    from sklearn.ensemble import VotingClassifier
    from sklearn.linear_model import LogisticRegression
    from sklearn.svm import LinearSVC
    vote = VotingClassifier([("a", LogisticRegression(solver="liblinear" if C == 2 else "lbfgs")),
                             ("b", _calibrated(LinearSVC(), cv=3)), ("c", "drop"), ("d", LogisticRegression(C=0.1)),
                             ("e", LogisticRegression(C=10.0))],
                            voting="soft", weights=[2.0, 1.0, 5.0, 0.0, 0.5])
    if C > 2:   # multinomial members are softmax heads: calibrated one-vs-rest folds would mix heads
        vote.set_params(b="drop")
    clf, X = _fit(vote, C)
    spec = _spec(clf.predict_proba)
    assert spec.activation == "mixture"
    assert spec.K == (5 if C == 2 else 2)        # zero weight dropped; nested folds flattened
    np.testing.assert_allclose(spec(X), clf.predict_proba(X), rtol=TOL, atol=TOL)


@pytest.mark.parametrize("C", [2, 3])
@pytest.mark.parametrize("features", [dict(), dict(max_features=0.5), dict(max_features=4, bootstrap_features=True)])
def test_bagging_classifier(C, features):
    from sklearn.ensemble import BaggingClassifier
    from sklearn.linear_model import LogisticRegression
    clf, X = _fit(BaggingClassifier(LogisticRegression(), n_estimators=6, random_state=1, **features), C)
    spec = _spec(clf.predict_proba)
    assert spec.activation == "mixture" and spec.K == 6 and spec.W.shape[1] == X.shape[1]
    np.testing.assert_allclose(spec(X), clf.predict_proba(X), rtol=TOL, atol=TOL)
    lin = _spec(clf.decision_function)
    assert lin.activation == "identity"
    np.testing.assert_allclose(lin(X), clf.decision_function(X), rtol=TOL, atol=TOL)


def test_voting_of_bagging_of_calibrated():
    from sklearn.ensemble import BaggingClassifier, VotingClassifier
    from sklearn.linear_model import LogisticRegression
    from sklearn.svm import LinearSVC
    clf, X = _fit(VotingClassifier([("bag", BaggingClassifier(_calibrated(LinearSVC(), cv=2), n_estimators=3,
                                                              max_features=0.7, random_state=0)),
                                    ("lr", LogisticRegression())], voting="soft", weights=[3, 1]), 2)
    spec = _spec(clf.predict_proba)
    assert spec.K == 7
    np.testing.assert_allclose(spec(X), clf.predict_proba(X), rtol=TOL, atol=TOL)


def test_regressors_fold_into_one_identity_head():
    from sklearn.ensemble import BaggingRegressor, VotingRegressor
    from sklearn.linear_model import LinearRegression, Ridge
    rng = np.random.default_rng(4)
    X = rng.standard_normal((150, 5))
    y = X @ rng.standard_normal(5) + 0.1 * rng.standard_normal(150)
    vote = VotingRegressor([("a", Ridge()), ("b", LinearRegression()), ("c", "drop")], weights=[1.0, 3.0, 9.0]).fit(X, y)
    bag = BaggingRegressor(Ridge(), n_estimators=5, max_features=3, bootstrap_features=True, random_state=0).fit(X, y)
    for model in (vote, bag):
        spec = _spec(model.predict)
        assert spec.activation == "identity" and spec.scalar_out and spec.R == 1
        np.testing.assert_allclose(spec(X), model.predict(X), rtol=TOL, atol=TOL)


def test_pipeline_ending_in_calibrated_linear_svc():
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler
    from sklearn.svm import LinearSVC
    pipe, X = _fit(make_pipeline(StandardScaler(), _calibrated(LinearSVC())), 3)
    spec = _spec(pipe.predict_proba)
    assert spec.activation == "mixture" and spec.maps is not None and spec.member == "ovr"
    np.testing.assert_allclose(spec(X), pipe.predict_proba(X), rtol=TOL, atol=TOL)


def test_mixture_spec_codes_and_row_blocks():
    from distributedkernelshap_b200 import _cabi
    from distributedkernelshap_b200.engine import MAX_ROWS_PER_CALL, rows_per_call
    from distributedkernelshap_b200.predictors import LinearModelSpec
    spec = LinearModelSpec(np.ones((15, 3)), np.zeros(15), "mixture", pi=np.full(5, 0.2), member="ovr")
    assert spec.act_code == _cabi.ACT_MIX == 5 and spec.K == 5 and spec.n_outputs == 3
    assert rows_per_call(spec.act_code, 3, "shared", 12, spec.R) == MAX_ROWS_PER_CALL // 15
    assert rows_per_call(_cabi.ACT_MIX, 2, "shared", 12, 2) == MAX_ROWS_PER_CALL // 2


# ---------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_refusals():
    from sklearn.calibration import CalibratedClassifierCV
    from sklearn.ensemble import BaggingClassifier, VotingClassifier, VotingRegressor
    from sklearn.linear_model import LogisticRegression, PoissonRegressor
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler
    from sklearn.svm import LinearSVC
    from distributedkernelshap_b200.predictors import LinearModelSpec
    cases = [
        (CalibratedClassifierCV(LinearSVC(), method="isotonic"), 2, "predict_proba", "isotonic"),
        (VotingClassifier([("a", LogisticRegression()), ("b", LogisticRegression(C=0.1))], voting="hard"), 2,
         "predict", "hard"),
        (BaggingClassifier(LinearSVC(), n_estimators=3, random_state=0), 2, "predict_proba", "no predict_proba"),
        (VotingClassifier([("a", LogisticRegression()), ("b", _calibrated(LinearSVC(), cv=2))], voting="soft"), 3,
         "predict_proba", "different heads"),
        (VotingClassifier([("a", make_pipeline(StandardScaler(), LogisticRegression())), ("b", LogisticRegression())],
                          voting="soft"), 2, "predict_proba", "Pipeline inside"),
        (VotingClassifier([("a", LogisticRegression()), ("b", LogisticRegression(C=0.1))], voting="soft",
                          weights=[1.0, -1.0]), 2, "predict_proba", "non-negative"),
        (_calibrated(LinearSVC(), cv=5), 7, "predict_proba", "at most 32"),
    ]
    for est, C, method, msg in cases:
        clf, _ = _fit(est, C)
        with pytest.raises((NotImplementedError, TypeError), match=msg):
            _spec(getattr(clf, method))
    rng = np.random.default_rng(0)
    X = rng.standard_normal((80, 4))
    glm = VotingRegressor([("a", PoissonRegressor()), ("b", PoissonRegressor(alpha=2.0))]).fit(X, np.exp(X[:, 0]))
    with pytest.raises(NotImplementedError, match="not linear"):
        _spec(glm.predict)
    clf, _ = _fit(_calibrated(LinearSVC(), cv=2), 3)
    clf.calibrated_classifiers_[1].estimator.classes_ = np.array([0, 1, 5])
    with pytest.raises(NotImplementedError, match="other classes"):
        _spec(clf.predict_proba)
    with pytest.raises(ValueError, match="summing to 1"):
        LinearModelSpec(np.ones((2, 3)), np.zeros(2), "mixture", pi=[0.5, 0.6], member="binary_logistic")


# ---------------------------------------------------------------------------------------------------------------------
# the CUDA-core kernel's per-element sums, restated in float32
# ---------------------------------------------------------------------------------------------------------------------
def _kernel_sums_f32(t, pi, wj, member):
    """csrc/dks_mixture.cuh per element: t [K, R_m] = log2(e) z in fp32, pw = pi_k w_j; returns the fp32 sums (binary:
    [sum p0, sum p1])."""
    f = np.float32
    acc = np.zeros(2 if member == "binary_logistic" else t.shape[1], dtype=f)
    for k in range(t.shape[0]):
        pw = f(pi[k]) * f(wj)
        if member == "binary_logistic":
            tt = np.clip(t[k, 0], f(-120), f(120))
            e = f(np.exp2(-tt))
            r1 = f(1) / (f(1) + e)
            acc[1] = f(pw * r1 + acc[1])
            acc[0] = f(pw * (e * r1) + acc[0])
        else:
            mx = t[k].max()
            if member == "ovr":
                h = min(mx, f(0))
                with np.errstate(over="ignore"):      # classes 2^-128 below the leader: 1 / inf = 0, as on the device
                    s = f(1) / (f(np.exp2(h)) + np.exp2(h - t[k]).astype(f))
            else:
                s = np.exp2(t[k] - mx).astype(f)
            inv = pw * (f(1) / s.sum(dtype=f))
            acc = (s * inv + acc).astype(f)
    return acc


@pytest.mark.parametrize("member,Rm", [("binary_logistic", 1), ("ovr", 3), ("softmax", 4)])
def test_kernel_sums_against_float64(member, Rm):
    rng = np.random.default_rng(7 + Rm)
    K, N = 5, 50
    pi = rng.uniform(0.2, 1.0, K)
    pi /= pi.sum()
    w = rng.uniform(0.1, 1.0, N)
    w /= w.mean()
    for scale in (1.0, 8.0, 40.0):
        z = rng.normal(0, scale, (N, K * Rm))
        want = np.einsum("jc,j->c", mixture_outputs(z, pi, member), w) / N
        got = np.zeros(2 if member == "binary_logistic" else Rm, dtype=np.float32)
        for j in range(N):
            got += _kernel_sums_f32((np.log2(np.e) * z[j]).astype(np.float32).reshape(K, Rm), pi, w[j], member)
        got = got.astype(np.float64) / N
        np.testing.assert_allclose(got, want, rtol=2e-5, atol=1e-7)
        if member == "binary_logistic":
            assert got.sum() == pytest.approx(1.0, abs=1e-5)


# ---------------------------------------------------------------------------------------------------------------------
# the float64 reference against the oracle driven by the real estimator, and against exact Shapley values
# ---------------------------------------------------------------------------------------------------------------------
def _groups(widths):
    groups, start = [], 0
    for wd in widths:
        groups.append(list(range(start, start + wd)))
        start += wd
    return groups


@pytest.mark.parametrize("link", ["logit", "identity"])
@pytest.mark.parametrize("model", ["calibrated2", "calibrated3", "bagging3", "voting2"])
def test_reference_matches_oracle_on_the_real_estimator(model, link):
    from sklearn.ensemble import BaggingClassifier, VotingClassifier
    from sklearn.linear_model import LogisticRegression
    from sklearn.svm import LinearSVC
    from distributedkernelshap_b200.plan import build_plan
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    est = {"calibrated2": (_calibrated(LinearSVC()), 2), "calibrated3": (_calibrated(LinearSVC()), 3),
           "bagging3": (BaggingClassifier(LogisticRegression(), n_estimators=4, max_features=0.7, random_state=0), 3),
           "voting2": (VotingClassifier([("a", LogisticRegression()), ("b", _calibrated(LinearSVC(), cv=3))],
                                        voting="soft", weights=[1, 2]), 2)}[model]
    clf, X = _fit(*est)
    spec = _spec(clf.predict_proba)
    groups = _groups((1, 2, 1, 1, 1))
    rng = np.random.default_rng(3)
    bg, wts = X[:14], rng.uniform(0.2, 1.0, 14)
    ref = MixtureReference(spec.W, spec.b, spec.pi, spec.member, bg, groups, wts, link=link)
    orc = KernelExplainerOracle(clf.predict_proba, DenseData(bg, [f"g{i}" for i in range(5)], groups, wts), link=link)
    np.testing.assert_allclose(ref.fnull, orc.fnull, rtol=1e-12, atol=1e-14)
    np.random.seed(1)
    plan = build_plan(5, 24)
    for x in X[100:103]:
        want = orc.explain(x[None, :], plan=(plan.dense(), plan.weights), nsamples=24, l1_reg=False)
        got = ref.explain(x, plan=(plan.dense(), plan.weights))
        np.testing.assert_allclose(got, want.reshape(got.shape), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("member,Rm", [("binary_logistic", 1), ("ovr", 3), ("softmax", 3)])
def test_reference_full_enumeration_is_exact_shapley(member, Rm):
    from distributedkernelshap_b200.plan import build_plan
    rng = np.random.default_rng(11)
    groups = _groups((1, 2, 1, 1))
    K = 3
    W, b = rng.normal(0, 0.8, (K * Rm, 5)), rng.normal(0, 0.5, K * Rm)
    pi = np.array([0.5, 0.3, 0.2])
    bg, x, wts = rng.standard_normal((10, 5)), rng.standard_normal(5), rng.uniform(0.2, 1.0, 10)
    ref = MixtureReference(W, b, pi, member, bg, groups, wts, link="logit")
    M = len(groups)
    plan = build_plan(M, 10 ** 6)

    def value(S):
        rows = bg.copy()
        for k in S:
            rows[:, groups[k]] = x[groups[k]]
        return ref.link(np.einsum("jc,j->c", ref.predict(rows), ref.weights))

    exact = np.zeros((M, ref.C))
    for k in range(M):
        rest = [q for q in range(M) if q != k]
        for r in range(M):
            for S in itertools.combinations(rest, r):
                wgt = factorial(r) * factorial(M - r - 1) / factorial(M)
                exact[k] += wgt * (value(S + (k,)) - value(S))
    got = ref.explain(x, plan=(plan.dense(), plan.weights))
    np.testing.assert_allclose(got, exact, rtol=1e-10, atol=1e-12)
