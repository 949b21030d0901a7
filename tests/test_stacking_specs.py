"""CPU checks of ``stacking.extract_stacking_spec``: the spec restates scikit-learn's stacking methods in NumPy, an
all-linear ``StackingRegressor`` folds into one linear model, and what the route does not cover is refused by name."""
import warnings

import numpy as np
import pytest

from distributedkernelshap_b200.predictors import LinearModelSpec
from distributedkernelshap_b200.stacking import StackingSpec, extract_stacking_spec

sk = pytest.importorskip("sklearn")
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.ensemble import (GradientBoostingClassifier, RandomForestClassifier, RandomForestRegressor,  # noqa: E402
                              StackingClassifier, StackingRegressor, VotingClassifier)
from sklearn.linear_model import LinearRegression, LogisticRegression, PoissonRegressor, Ridge, RidgeCV  # noqa: E402
from sklearn.multiclass import OneVsRestClassifier  # noqa: E402
from sklearn.neighbors import KNeighborsClassifier, KNeighborsRegressor  # noqa: E402
from sklearn.neural_network import MLPClassifier  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import OneHotEncoder, StandardScaler  # noqa: E402
from sklearn.svm import SVC, SVR, LinearSVC  # noqa: E402
from sklearn.tree import DecisionTreeClassifier  # noqa: E402

RTOL = 1e-12


def _data(n=160, d=5, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d))
    return X, rng


def _close(got, want):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape
    np.testing.assert_allclose(got, want, rtol=RTOL, atol=RTOL * np.abs(want).max())


def _fit(est, X, y):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return est.fit(X, y)


def _families():
    return [("lr", LogisticRegression()), ("rf", RandomForestClassifier(12, max_depth=4, random_state=0)),
            ("svc", SVC(random_state=0)), ("mlp", MLPClassifier((8,), max_iter=400, random_state=0)),
            ("knn", KNeighborsClassifier(5)), ("lsvc", LinearSVC())]


@pytest.mark.parametrize("method", ["predict_proba", "decision_function"])
def test_binary_every_family(method):
    X, rng = _data()
    y = (X[:, 0] + X[:, 1] > 0).astype(int)
    st = _fit(StackingClassifier(_families(), final_estimator=LogisticRegression()), X, y)
    spec = extract_stacking_spec(getattr(st, method))
    assert isinstance(spec, StackingSpec) and len(spec.members) == 6
    Xt = rng.normal(size=(60, 5))
    _close(spec(Xt), getattr(st, method)(Xt))


@pytest.mark.parametrize("passthrough", [False, True])
def test_three_classes(passthrough):
    X, rng = _data(seed=1)
    y = np.digitize(X[:, 0] + 0.5 * X[:, 2], [-0.5, 0.5])
    st = _fit(StackingClassifier([("lr", LogisticRegression()), ("gb", GradientBoostingClassifier(n_estimators=10)),
                                  ("knn", KNeighborsClassifier(7))], passthrough=passthrough), X, y)
    for method in ("predict_proba", "decision_function"):
        spec = extract_stacking_spec(getattr(st, method))
        assert spec.meta(X[:3]).shape[1] == 9
        Xt = rng.normal(size=(60, 5))
        _close(spec(Xt), getattr(st, method)(Xt))


def test_regressor_passthrough():
    X, rng = _data(seed=2)
    y = X[:, 0] - 2 * X[:, 3] + np.sin(X[:, 1])
    st = _fit(StackingRegressor([("rf", RandomForestRegressor(10, max_depth=4, random_state=0)), ("svr", SVR()),
                                 ("knn", KNeighborsRegressor(4)), ("lin", Ridge())], final_estimator=RidgeCV(),
                                passthrough=True), X, y)
    spec = extract_stacking_spec(st.predict)
    assert isinstance(spec, StackingSpec) and spec.scalar_out and spec.W_pass.shape == (1, 5)
    Xt = rng.normal(size=(60, 5))
    _close(spec(Xt), st.predict(Xt))


def test_drop_member_and_explicit_stack_method():
    X, rng = _data(seed=3)
    y = (X[:, 1] > 0).astype(int)
    st = _fit(StackingClassifier([("a", "drop"), ("svc", SVC(random_state=0)), ("rf", DecisionTreeClassifier(max_depth=3))],
                                 stack_method="auto"), X, y)
    spec = extract_stacking_spec(st.predict_proba)
    assert len(spec.members) == 2
    Xt = rng.normal(size=(40, 5))
    _close(spec(Xt), st.predict_proba(Xt))
    st2 = _fit(StackingClassifier([("svc", SVC(probability=False, random_state=0))], stack_method="decision_function"),
               X, y)
    spec2 = extract_stacking_spec(st2.predict_proba)
    assert [cols for cols, _ in spec2.members] == [(0, 1)]
    _close(spec2(Xt), st2.predict_proba(Xt))


def test_outer_column_transformer():
    X, rng = _data(seed=4)
    X[:, 4] = rng.integers(0, 3, size=X.shape[0])
    y = (X[:, 0] + (X[:, 4] == 1) > 0.3).astype(int)
    ct = ColumnTransformer([("num", StandardScaler(), [0, 1, 2, 3]), ("cat", OneHotEncoder(), [4])])
    pipe = _fit(make_pipeline(ct, StackingClassifier([("lr", LogisticRegression()),
                                                      ("rf", RandomForestClassifier(8, max_depth=3, random_state=0))],
                                                     passthrough=True)), X, y)
    out = extract_stacking_spec(pipe.predict_proba)
    assert isinstance(out, tuple)
    spec, enc = out
    assert spec.n_features == 5 and enc.E == 7 and spec.W_pass.shape == (1, 7)
    Xt = X[:40]
    _close(spec(pipe[:-1].transform(Xt)), pipe.predict_proba(Xt))


def test_all_linear_regressor_folds():
    X, rng = _data(seed=5)
    y = X @ np.array([1.0, -2.0, 0.5, 0.0, 3.0]) + 0.1 * rng.normal(size=X.shape[0])
    for passthrough in (False, True):
        st = _fit(StackingRegressor([("a", Ridge(alpha=2.0)), ("b", LinearRegression())], final_estimator=LinearRegression(),
                                    passthrough=passthrough), X, y)
        spec = extract_stacking_spec(st.predict)
        assert isinstance(spec, LinearModelSpec) and spec.activation == "identity"
        Xt = rng.normal(size=(60, 5))
        _close(spec(Xt), st.predict(Xt))


def test_all_linear_classifier_takes_the_stacking_route():
    X, rng = _data(seed=6)
    y = (X[:, 0] - X[:, 2] > 0).astype(int)
    st = _fit(StackingClassifier([("a", LogisticRegression()), ("b", LinearSVC())]), X, y)
    spec = extract_stacking_spec(st.predict_proba)
    assert isinstance(spec, StackingSpec)
    Xt = rng.normal(size=(60, 5))
    _close(spec(Xt), st.predict_proba(Xt))


def test_not_stacking_is_none():
    X, _ = _data()
    lr = _fit(LogisticRegression(), X, (X[:, 0] > 0).astype(int))
    assert extract_stacking_spec(lr.predict_proba) is None
    assert extract_stacking_spec(lambda x: x) is None


def _refusal(case):
    X, rng = _data(seed=7)
    y = (X[:, 0] > 0).astype(int)
    y3 = np.digitize(X[:, 0], [-0.5, 0.5])
    base = [("lr", LogisticRegression()), ("rf", RandomForestClassifier(5, max_depth=3, random_state=0))]
    if case == "tree_final":
        return _fit(StackingClassifier(base, final_estimator=DecisionTreeClassifier()), X, y).predict_proba
    if case == "mlp_final":
        return _fit(StackingClassifier(base, final_estimator=MLPClassifier((4,), max_iter=50)), X, y).predict_proba
    if case == "ovr_final":
        ovr = OneVsRestClassifier(LogisticRegression())
        return _fit(StackingClassifier(base, final_estimator=ovr), X, y3).predict_proba
    if case == "exp_final":
        return _fit(StackingRegressor([("rf", RandomForestRegressor(5, random_state=0))], final_estimator=PoissonRegressor()),
                    X, np.abs(X[:, 0])).predict
    if case == "predict_member":
        return _fit(StackingClassifier(base, stack_method="predict"), X, y).predict_proba
    if case == "pipeline_member":
        return _fit(StackingClassifier([("p", make_pipeline(StandardScaler(), SVC()))]), X, y).predict_proba
    if case == "nested":
        inner = VotingClassifier(base, voting="soft")
        return _fit(StackingClassifier([("v", inner), ("lr", LogisticRegression())]), X, y).predict_proba
    if case == "multilabel":
        Y = np.c_[y, (X[:, 1] > 0).astype(int)]
        return _fit(StackingClassifier([("rf", RandomForestClassifier(5, random_state=0))],
                                       final_estimator=RandomForestClassifier(3)), X, Y).predict_proba
    if case == "members":
        return _fit(StackingClassifier([(f"t{k}", DecisionTreeClassifier(max_depth=2, random_state=k))
                                        for k in range(17)]), X, y).predict_proba
    if case == "predict_method":
        return _fit(StackingClassifier(base), X, y).predict
    raise AssertionError(case)


REFUSALS = {
    "tree_final": (NotImplementedError, "not a linear model"),
    "mlp_final": (NotImplementedError, "not a linear model"),
    "ovr_final": (NotImplementedError, "one-vs-rest"),
    "exp_final": (NotImplementedError, "exp-head"),
    "predict_member": (NotImplementedError, "predict, which returns labels"),
    "pipeline_member": (NotImplementedError, "put the preprocessing in front of the ensemble"),
    "nested": (NotImplementedError, "nested voting or stacking"),
    "multilabel": (NotImplementedError, "multilabel"),
    "members": (NotImplementedError, "at most 16"),
    "predict_method": (TypeError, "pass predict_proba or decision_function"),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_refusals(case):
    exc, words = REFUSALS[case]
    try:
        fn = _refusal(case)
    except (ValueError, TypeError) as e:        # scikit-learn itself refuses to fit this combination
        pytest.skip(f"scikit-learn does not fit it: {e}")
    with pytest.raises(exc, match=words):
        extract_stacking_spec(fn)


def test_meta_column_bound():
    # 17 members of 8 outputs each would be refused for their number first; 16 members with 8 classes is F = 128 (allowed)
    X, rng = _data(n=400, seed=8)
    y = rng.integers(0, 8, size=X.shape[0])
    st = _fit(StackingClassifier([(f"t{k}", DecisionTreeClassifier(max_depth=2, random_state=k)) for k in range(16)],
                                 final_estimator=LogisticRegression(max_iter=50)), X, y)
    spec = extract_stacking_spec(st.predict_proba)
    assert sum(nc for (_, nc), _ in spec.members) == 128
