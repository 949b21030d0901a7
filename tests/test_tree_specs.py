"""Tree ensembles read into ``TreeEnsembleSpec`` (distributedkernelshap_b200/trees.py): every spec reproduces the
scikit-learn method it was read from, on inputs with NaN, on split thresholds and next to their float32 rounding, and the
models the tree route does not cover are refused by name -- while the linear extraction keeps refusing trees as before."""
import numpy as np
import pytest

sklearn = pytest.importorskip("sklearn")
from sklearn.calibration import CalibratedClassifierCV  # noqa: E402
from sklearn.dummy import DummyRegressor  # noqa: E402
from sklearn.ensemble import (ExtraTreesClassifier, ExtraTreesRegressor, GradientBoostingClassifier,  # noqa: E402
                              GradientBoostingRegressor, HistGradientBoostingClassifier, HistGradientBoostingRegressor,
                              RandomForestClassifier, RandomForestRegressor, VotingClassifier)
from sklearn.linear_model import LinearRegression, LogisticRegression  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import StandardScaler  # noqa: E402
from sklearn.tree import DecisionTreeClassifier, DecisionTreeRegressor  # noqa: E402

from distributedkernelshap_b200.predictors import extract_linear_spec  # noqa: E402
from distributedkernelshap_b200.trees import TreeEnsembleSpec, extract_tree_spec  # noqa: E402


def _data(seed, n=300, P=6, nan=True):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P))
    if nan:
        X[rng.random(X.shape) < 0.05] = np.nan
    return X, rng


def _probe(spec, rng, nan=True, n=400):
    """Random rows plus rows placed exactly on split thresholds and on both sides of their float32 rounding."""
    X = rng.normal(size=(n, spec.n_features))
    if nan:
        X[rng.random(X.shape) < 0.05] = np.nan
    inner = np.nonzero((spec.feature >= 0) & np.isfinite(spec.threshold))[0]
    pick = inner[rng.permutation(len(inner))[: n // 4]]
    for q, nd in enumerate(pick):
        f, t = spec.feature[nd], spec.threshold[nd]
        X[q, f] = t
        t32 = np.float32(t)
        X[n // 4 + q, f] = float(np.nextafter(t32, np.float32(np.inf))) - 1e-13
        X[n // 2 + q, f] = float(np.nextafter(t32, np.float32(-np.inf))) + 1e-13
    return X


def _fit_cases():
    X, rng = _data(0)
    Xf = np.nan_to_num(X)
    yr = Xf[:, 1] + 0.3 * rng.normal(size=len(X))
    cases = []
    for C in (2, 3, 8):
        y = rng.integers(0, C, len(X))
        y[:C] = np.arange(C)
        cases += [(DecisionTreeClassifier(max_depth=6, random_state=0).fit(X, y), "predict_proba", True),
                  (RandomForestClassifier(12, max_depth=6, random_state=0).fit(X, y), "predict_proba", True),
                  (ExtraTreesClassifier(8, max_depth=5, random_state=0).fit(X, y), "predict_proba", True),
                  (GradientBoostingClassifier(n_estimators=10, max_depth=3, random_state=0).fit(Xf, y), "predict_proba", False),
                  (GradientBoostingClassifier(n_estimators=10, max_depth=2, random_state=0).fit(Xf, y),
                   "decision_function", False),
                  (HistGradientBoostingClassifier(max_iter=10, random_state=0).fit(X, y), "predict_proba", True),
                  (HistGradientBoostingClassifier(max_iter=10, random_state=0).fit(X, y), "decision_function", True)]
    cases += [(DecisionTreeRegressor(max_depth=7, random_state=0).fit(X, yr), "predict", True),
              (RandomForestRegressor(10, random_state=0).fit(X, yr), "predict", True),
              (ExtraTreesRegressor(10, max_depth=8, random_state=0).fit(X, yr), "predict", True),
              (GradientBoostingRegressor(n_estimators=15, random_state=0).fit(Xf, yr), "predict", False),
              (GradientBoostingRegressor(n_estimators=15, init="zero", random_state=0).fit(Xf, yr), "predict", False),
              (GradientBoostingClassifier(n_estimators=5, init="zero", random_state=0).fit(Xf, (yr > 0).astype(int)),
               "predict_proba", False),
              (HistGradientBoostingRegressor(max_iter=15, random_state=0).fit(X, yr), "predict", True),
              (HistGradientBoostingRegressor(max_iter=15, loss="poisson", random_state=0).fit(X, np.abs(yr)), "predict", True),
              (HistGradientBoostingRegressor(max_iter=15, loss="gamma", random_state=0).fit(X, np.abs(yr) + 0.1), "predict",
               True)]
    return cases


CASES = _fit_cases()


@pytest.mark.parametrize("k", range(len(CASES)))
def test_spec_reproduces_sklearn(k):
    model, method, nan = CASES[k]
    fn = getattr(model, method)
    spec = extract_tree_spec(fn)
    assert isinstance(spec, TreeEnsembleSpec)
    X = _probe(spec, np.random.default_rng(k), nan=nan)
    want = np.asarray(fn(X), dtype=np.float64)
    got = spec(X)
    assert got.shape == want.shape
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * max(1.0, np.max(np.abs(want))))
    assert spec.n_outputs == (1 if want.ndim == 1 else want.shape[1])
    assert spec.scalar_out == (want.ndim == 1)


def test_float32_cast_decides_the_side():
    # just above the threshold in float64, but equal to it once cast to float32: sklearn.tree sends it left
    X = np.array([[0.0], [1.0]])
    tree = DecisionTreeRegressor().fit(X, [0.0, 1.0])
    thr = tree.tree_.threshold[0]
    assert thr == 0.5
    spec = extract_tree_spec(tree.predict)
    x = np.nextafter(thr, np.inf)
    assert x > thr and np.float64(np.float32(x)) <= thr
    probe = np.array([[thr], [x], [float(np.nextafter(np.float32(thr), np.float32(1.0)))]])
    np.testing.assert_array_equal(tree.predict(probe), [0.0, 0.0, 1.0])
    np.testing.assert_array_equal(spec(probe), tree.predict(probe))


def test_hgb_compares_float64():
    X, rng = _data(3, nan=False)
    y = (X[:, 0] > 0.1).astype(int)
    m = HistGradientBoostingClassifier(max_iter=5).fit(X, y)
    spec = extract_tree_spec(m.predict_proba)
    assert spec.cmp == 1
    Xp = _probe(spec, rng, nan=True)
    np.testing.assert_allclose(spec(Xp), m.predict_proba(Xp), rtol=0, atol=1e-13)


def test_stump_and_single_leaf():
    X = np.arange(10.0).reshape(-1, 1)
    stump = DecisionTreeRegressor(max_depth=1).fit(X, (X[:, 0] > 4).astype(float))
    leaf = DecisionTreeRegressor().fit(X, np.ones(10))
    for m in (stump, leaf):
        spec = extract_tree_spec(m.predict)
        Xp = np.linspace(-2, 12, 57).reshape(-1, 1)
        np.testing.assert_array_equal(spec(Xp), m.predict(Xp))
    assert extract_tree_spec(leaf.predict).n_nodes == 1


def test_not_a_tree_gives_none():
    X, _ = _data(4, nan=False)
    lin = LogisticRegression().fit(X, (X[:, 0] > 0).astype(int))
    assert extract_tree_spec(lin.predict_proba) is None
    assert extract_tree_spec(lambda z: z) is None


def _refusals():
    X, rng = _data(5, nan=False)
    y2 = (X[:, 0] > 0).astype(int)
    y9 = np.arange(len(X)) % 9
    yr = X[:, 1]
    hgb_cat = HistGradientBoostingClassifier(max_iter=3, categorical_features=[0])
    Xc = X.copy()
    Xc[:, 0] = rng.integers(0, 4, len(X))
    hgb_cat.fit(Xc, y2)
    rf = RandomForestClassifier(5, max_depth=3, random_state=0).fit(X, y2)
    return {
        "hgb_categorical": (hgb_cat.predict_proba, NotImplementedError, "categorical"),
        "gb_custom_init": (GradientBoostingRegressor(n_estimators=3, init=LinearRegression()).fit(X, yr).predict,
                           NotImplementedError, "init"),
        "multi_output_regressor": (RandomForestRegressor(3).fit(X, np.stack([yr, yr], 1)).predict, NotImplementedError,
                                   "multi-output"),
        "more_than_8_classes": (DecisionTreeClassifier(max_depth=3).fit(X, y9).predict_proba, NotImplementedError,
                                "at most 8"),
        "gb_9_classes": (GradientBoostingClassifier(n_estimators=2, max_depth=1).fit(X, y9).predict_proba,
                         NotImplementedError, "at most 8"),
        "pipeline": (make_pipeline(StandardScaler(), DecisionTreeClassifier(max_depth=2)).fit(X, y2).predict_proba,
                     NotImplementedError, "Pipeline"),
        "voting": (VotingClassifier([("rf", rf), ("lr", LogisticRegression())], voting="soft").fit(X, y2).predict_proba,
                   NotImplementedError, "ensemble"),
        "calibrated": (CalibratedClassifierCV(DecisionTreeClassifier(max_depth=2), cv=2).fit(X, y2).predict_proba,
                       NotImplementedError, "ensemble"),
        "classifier_predict": (rf.predict, TypeError, "labels"),
        "regressor_proba": (DummyRegressor().fit(X, yr).predict, None, None),
    }


REFUSALS = _refusals()


@pytest.mark.parametrize("name", sorted(REFUSALS))
def test_refusals(name):
    fn, exc, words = REFUSALS[name]
    if exc is None:                    # not a tree model at all: left to the linear extraction
        assert extract_tree_spec(fn) is None
        return
    with pytest.raises(exc, match=words):
        extract_tree_spec(fn)


def test_linear_extraction_still_refuses_trees():
    X, _ = _data(6, nan=False)
    y = (X[:, 0] > 0).astype(int)
    rf = RandomForestClassifier(4, max_depth=3, random_state=0).fit(X, y)
    with pytest.raises((TypeError, NotImplementedError)):
        extract_linear_spec(rf.predict_proba)
    with pytest.raises((TypeError, NotImplementedError)):
        extract_linear_spec(HistGradientBoostingClassifier(max_iter=3).fit(X, y).predict_proba)
    vote = VotingClassifier([("rf", rf), ("lr", LogisticRegression())], voting="soft").fit(X, y)
    with pytest.raises((TypeError, NotImplementedError)):
        extract_linear_spec(vote.predict_proba)
