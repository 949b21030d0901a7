"""IsolationForest and AdaBoostClassifier read into ``TreeEnsembleSpec`` (distributedkernelshap_b200/trees.py): every spec
reproduces the scikit-learn method it was read from on held-out rows, NaN included, and what the tree route does not cover
is refused by name.  The anomaly head is restated here on its own, from the definition of the isolation score."""
import warnings

import numpy as np
import pytest

sklearn = pytest.importorskip("sklearn")
from sklearn.calibration import CalibratedClassifierCV  # noqa: E402
from sklearn.ensemble import (AdaBoostClassifier, AdaBoostRegressor, BaggingClassifier, IsolationForest,  # noqa: E402
                              StackingClassifier)
from sklearn.linear_model import LogisticRegression  # noqa: E402
from sklearn.tree import DecisionTreeClassifier, ExtraTreeClassifier  # noqa: E402

from distributedkernelshap_b200.ensembles import extract_ensemble_spec  # noqa: E402
from distributedkernelshap_b200.trees import extract_tree_spec  # noqa: E402

RTOL = 1e-12
ATOL = 1e-14        # a decision_function near 0 is a difference of two numbers near -0.5


def _data(seed, n=300, P=6, nan=False):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P))
    if nan:
        X[rng.random(X.shape) < 0.05] = np.nan
    return X, rng


def _held_out(rng, P, nan=False, n=250):
    X = rng.normal(size=(n, P)) * 1.5
    X[:5] *= 10.0                                   # far outliers, isolated near the root
    if nan:
        X[rng.random(X.shape) < 0.05] = np.nan
    return X


def _check(fn, X):
    spec = extract_tree_spec(fn)
    got, want = spec(X), fn(X)
    assert got.shape == want.shape
    np.testing.assert_allclose(got, want, rtol=RTOL, atol=ATOL)
    return spec


def _c(n):
    """Average path length of an unsuccessful search in a binary search tree of n keys (Liu et al., 2008)."""
    if n <= 1:
        return 0.0
    if n == 2:
        return 1.0
    return 2.0 * (np.log(n - 1.0) + np.euler_gamma) - 2.0 * (n - 1.0) / n


def _isolation_scores(iso, X):
    """score_samples restated: each tree's path length to the leaf x reaches (edges walked + 1 at the root, the float32
    value compared) plus c(leaf size) - 1, averaged, then -2^(-mean / c(max_samples))."""
    X = np.asarray(X, dtype=np.float32).astype(np.float64)
    total = np.zeros(X.shape[0])
    for est, feats in zip(iso.estimators_, iso.estimators_features_):
        t = est.tree_
        Xs = X[:, feats] if len(feats) != X.shape[1] else X
        for i, x in enumerate(Xs):
            nd, depth = 0, 1
            while t.children_left[nd] >= 0:
                v = x[t.feature[nd]]
                left = t.missing_go_to_left[nd] if np.isnan(v) else v <= t.threshold[nd]
                nd = t.children_left[nd] if left else t.children_right[nd]
                depth += 1
            total[i] += depth + _c(t.n_node_samples[nd]) - 1.0
    d = len(iso.estimators_) * _c(iso.max_samples_)
    return -2.0 ** (-(total / d) if d > 0 else -1.0)


# ---- IsolationForest ---------------------------------------------------------------------------------------------------

IFOREST = {
    "defaults": dict(),
    "max_features_half": dict(max_features=0.5),
    "max_samples_int": dict(max_samples=64),
    "max_samples_float": dict(max_samples=0.3),
    "max_samples_1": dict(max_samples=1),
    "max_samples_2": dict(max_samples=2),
    "contamination": dict(contamination=0.1),
    "bootstrap": dict(bootstrap=True),
    "one_tree": dict(n_estimators=1),
    "300_trees": dict(n_estimators=300),
}


@pytest.mark.parametrize("case", sorted(IFOREST))
@pytest.mark.parametrize("method", ["decision_function", "score_samples"])
def test_iforest_spec_reproduces_sklearn(case, method):
    X, rng = _data(1)
    iso = IsolationForest(random_state=0, **IFOREST[case]).fit(X)
    spec = _check(getattr(iso, method), _held_out(rng, X.shape[1]))
    assert spec.head == "iforest" and spec.scalar_out and spec.n_outputs == 1 and spec.cmp == 0
    assert spec.offset == (iso.offset_ if method == "decision_function" else 0.0)


def test_iforest_nan_at_fit_and_predict():
    X, rng = _data(2, nan=True)
    iso = IsolationForest(n_estimators=50, random_state=0).fit(X)
    Xe = _held_out(rng, X.shape[1], nan=True)
    _check(iso.decision_function, Xe)
    _check(iso.score_samples, Xe)


@pytest.mark.parametrize("case", ["defaults", "max_features_half", "max_samples_1", "max_samples_2"])
def test_iforest_against_the_isolation_score(case):
    X, rng = _data(3, nan=True)
    iso = IsolationForest(n_estimators=20, random_state=0, **IFOREST[case]).fit(X)
    Xe = _held_out(rng, X.shape[1], nan=True, n=60)
    want = _isolation_scores(iso, Xe)
    np.testing.assert_allclose(extract_tree_spec(iso.score_samples)(Xe), want, rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(extract_tree_spec(iso.decision_function)(Xe), want - iso.offset_, rtol=RTOL, atol=ATOL)


def test_iforest_feature_subsets_read_original_columns():
    X, _ = _data(4, P=8)
    iso = IsolationForest(n_estimators=30, max_features=0.5, random_state=0).fit(X)
    spec = extract_tree_spec(iso.decision_function)
    used = set(spec.feature[spec.feature >= 0].tolist())
    assert spec.n_features == 8 and len(used) > 4          # each tree sees 4 columns, the forest more of them


# ---- AdaBoostClassifier ------------------------------------------------------------------------------------------------

def _labels(X, K, seed=0):
    s = X[:, 0] + 0.5 * X[:, 1] - 0.3 * X[:, 2] * X[:, 3]
    q = np.quantile(s, np.linspace(0, 1, K + 1)[1:-1])
    return np.digitize(s, q)


BASES = {"stump": lambda: None, "depth3": lambda: DecisionTreeClassifier(max_depth=3, random_state=0),
         "extra": lambda: ExtraTreeClassifier(max_depth=3, random_state=0)}


@pytest.mark.parametrize("K", [2, 3, 8])
@pytest.mark.parametrize("base", sorted(BASES))
@pytest.mark.parametrize("method", ["predict_proba", "decision_function"])
def test_adaboost_spec_reproduces_sklearn(K, base, method):
    X, rng = _data(5, n=400)
    ada = AdaBoostClassifier(estimator=BASES[base](), n_estimators=30, random_state=0).fit(X, _labels(X, K))
    spec = _check(getattr(ada, method), _held_out(rng, X.shape[1]))
    heads = {"predict_proba": "sigmoid" if K == 2 else "softmax", "decision_function": "identity"}
    assert spec.head == heads[method] and spec.R == (1 if K == 2 else K)
    assert spec.scalar_out == (K == 2 and method == "decision_function")


@pytest.mark.parametrize("method", ["predict_proba", "decision_function"])
def test_adaboost_non_contiguous_labels(method):
    X, rng = _data(6, n=400)
    y = np.array([-7, 3, 40])[_labels(X, 3)]
    ada = AdaBoostClassifier(estimator=DecisionTreeClassifier(max_depth=2), n_estimators=20, random_state=0).fit(X, y)
    _check(getattr(ada, method), _held_out(rng, X.shape[1]))


@pytest.mark.parametrize("method", ["predict_proba", "decision_function"])
def test_adaboost_early_stop_with_one_estimator(method):
    X, rng = _data(7)
    y = (X[:, 0] > 0).astype(int)                   # a perfect first tree: boosting stops after it
    ada = AdaBoostClassifier(estimator=DecisionTreeClassifier(max_depth=1), n_estimators=10, random_state=0).fit(X, y)
    assert len(ada.estimators_) == 1 and len(ada.estimator_weights_) == 10
    spec = _check(getattr(ada, method), _held_out(rng, X.shape[1]))
    assert spec.n_trees == 1


def test_adaboost_tie_goes_to_the_first_class():
    X = np.array([[0.0], [0.0], [1.0], [1.0]])
    y = np.array([0, 1, 0, 2])                       # the left leaf holds one sample of class 0 and one of class 1
    ada = AdaBoostClassifier(estimator=DecisionTreeClassifier(max_depth=1), n_estimators=1).fit(X, y)
    _check(ada.decision_function, np.array([[0.0], [1.0], [0.5]]))


def test_adaboost_is_a_soft_voting_member():
    from sklearn.ensemble import VotingClassifier
    from sklearn.neural_network import MLPClassifier
    X, rng = _data(8, n=300)
    y = _labels(X, 2)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        vote = VotingClassifier([("ada", AdaBoostClassifier(n_estimators=10, random_state=0)),
                                 ("mlp", MLPClassifier((8,), max_iter=50, random_state=0))], voting="soft").fit(X, y)
    spec = extract_ensemble_spec(vote.predict_proba)
    Xe = _held_out(rng, X.shape[1], n=50)
    np.testing.assert_allclose(spec(Xe), vote.predict_proba(Xe), rtol=1e-9, atol=1e-12)


# ---- refusals ----------------------------------------------------------------------------------------------------------

def _refused():
    X, _ = _data(9)
    y2, y9 = _labels(X, 2), _labels(X, 9)
    iso = IsolationForest(n_estimators=5, random_state=0).fit(X)
    ada = AdaBoostClassifier(n_estimators=5, random_state=0).fit(X, y2)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        one = AdaBoostClassifier(n_estimators=3).fit(X, np.zeros(len(X), dtype=int))
        stack = StackingClassifier([("ada", ada)], final_estimator=LogisticRegression()).fit(X, y2)
    return {
        "adaboost_regressor": (lambda: AdaBoostRegressor(n_estimators=5, random_state=0).fit(X, X[:, 0]).predict,
                               NotImplementedError, "AdaBoostRegressor.*weighted median"),
        "adaboost_linear_base": (lambda: AdaBoostClassifier(LogisticRegression(), n_estimators=3).fit(X, y2).predict_proba,
                                 NotImplementedError, "over LogisticRegression.*sklearn.tree"),
        "iforest_predict": (lambda: iso.predict, TypeError, "IsolationForest.predict.*labels"),
        "adaboost_predict": (lambda: ada.predict, TypeError, "AdaBoostClassifier.predict.*labels"),
        "adaboost_one_class": (lambda: one.predict_proba, NotImplementedError, "one class"),
        "adaboost_nine_classes": (lambda: AdaBoostClassifier(n_estimators=5, random_state=0).fit(X, y9).predict_proba,
                                  NotImplementedError, "9 classes"),
        "calibrated": (lambda: CalibratedClassifierCV(AdaBoostClassifier(n_estimators=3), cv=2).fit(X, y2).predict_proba,
                       NotImplementedError, "CalibratedClassifierCV holding a tree model"),
        "bagging": (lambda: BaggingClassifier(AdaBoostClassifier(n_estimators=3), n_estimators=2).fit(X, y2).predict_proba,
                    NotImplementedError, "BaggingClassifier holding a tree model"),
        "stacking": (lambda: stack.predict_proba, NotImplementedError, "Stacking"),
    }


REFUSED = ["adaboost_regressor", "adaboost_linear_base", "iforest_predict", "adaboost_predict", "adaboost_one_class",
           "adaboost_nine_classes", "calibrated", "bagging", "stacking"]


@pytest.mark.parametrize("name", REFUSED)
def test_refusals(name):
    make, exc, words = _refused()[name]
    fn = make()
    with pytest.raises(exc, match=words):
        if name == "stacking":
            extract_ensemble_spec(fn)
        extract_tree_spec(fn)
