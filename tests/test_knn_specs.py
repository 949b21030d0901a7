"""Nearest-neighbour models read into ``KnnSpec`` (no GPU): extraction of every accepted estimator, metric, weighting and
scaler pipeline; the spec against scikit-learn on continuous data and against the independent reference
(tests/knn_reference.py) everywhere; the lower-index rule on tied integer data; the zero-distance rule; the refusals."""
import numpy as np
import pytest

sklearn = pytest.importorskip("sklearn")
from sklearn.ensemble import BaggingClassifier, VotingRegressor  # noqa: E402
from sklearn.neighbors import (KNeighborsClassifier, KNeighborsRegressor, RadiusNeighborsClassifier,  # noqa: E402
                               RadiusNeighborsRegressor)
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import (MaxAbsScaler, MinMaxScaler, PolynomialFeatures, RobustScaler,  # noqa: E402
                                   StandardScaler)

from distributedkernelshap_b200.neighbors import KnnSpec, extract_knn_spec  # noqa: E402
from knn_reference import neighbours, reference  # noqa: E402


def _data(seed=0, n=240, P=5, classes=3):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 3.0, P) + np.linspace(-1.0, 4.0, P)
    s = X[:, 0] - X[:, 0].mean() + (X[:, 1] - X[:, 1].mean()) * 0.7
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, classes + 1)[1:-1]))
    T = np.stack([s, X[:, 2] * 2 - X[:, 3]], axis=1)
    Q = rng.normal(size=(60, P)) * np.linspace(0.5, 3.0, P) + np.linspace(-1.0, 4.0, P)
    return X, y, T, Q


METRICS = [dict(), dict(metric="euclidean"), dict(metric="manhattan"), dict(metric="l1"), dict(metric="l2"),
           dict(metric="cityblock"), dict(metric="minkowski", p=3), dict(p=1.5), dict(metric="sqeuclidean"),
           dict(metric="minkowski", p=1)]
WANT_METRIC = ["euclidean", "euclidean", "manhattan", "manhattan", "euclidean", "manhattan", "minkowski", "minkowski",
               "sqeuclidean", "manhattan"]
SCALERS = [None, StandardScaler, MinMaxScaler, MaxAbsScaler, RobustScaler]


def _fit(est, X, target, scaler=None):
    return (make_pipeline(scaler(), est) if scaler else est).fit(X, target)


@pytest.mark.parametrize("mi", range(len(METRICS)))
@pytest.mark.parametrize("weights", ["uniform", "distance"])
def test_every_metric_and_weighting_matches_scikit_learn(mi, weights):
    X, y, T, Q = _data(mi)
    for est, target, method in ((KNeighborsClassifier(n_neighbors=6, weights=weights, **METRICS[mi]), y, "predict_proba"),
                                (KNeighborsRegressor(n_neighbors=4, weights=weights, **METRICS[mi]), T, "predict")):
        fn = getattr(_fit(est, X, target), method)
        spec = extract_knn_spec(fn)
        assert spec.metric == WANT_METRIC[mi] and spec.weights == weights
        np.testing.assert_allclose(spec(Q), fn(Q), rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(spec(Q[:12]), reference(spec)(Q[:12]), rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("scaler", SCALERS)
@pytest.mark.parametrize("algorithm", ["auto", "brute", "kd_tree", "ball_tree"])
def test_scaler_pipelines_and_algorithms(scaler, algorithm):
    X, y, T, Q = _data(3)
    clf = _fit(KNeighborsClassifier(algorithm=algorithm), X, y, scaler)
    reg = _fit(KNeighborsRegressor(algorithm=algorithm, weights="distance"), X, T[:, 0], scaler)
    for fn in (clf.predict_proba, reg.predict):
        spec = extract_knn_spec(fn)
        got = spec(Q)
        assert got.shape == fn(Q).shape
        np.testing.assert_allclose(got, fn(Q), rtol=1e-12, atol=1e-15)
    assert extract_knn_spec(reg.predict).scalar_out and not extract_knn_spec(clf.predict_proba).scalar_out


def test_uniform_probabilities_are_bit_identical():
    X, y, _, Q = _data(5, classes=8)
    fn = KNeighborsClassifier(n_neighbors=7).fit(X, y).predict_proba
    spec = extract_knn_spec(fn)
    assert spec.R == 8
    np.testing.assert_array_equal(spec(Q), fn(Q))                       # count / k, as scikit-learn divides


def test_eight_targets_and_k_edges():
    X, _, T, Q = _data(6)
    Y = np.concatenate([T, T ** 2, T[:, :1] - 1, T[:, 1:] * 3, T[:, :1] * T[:, 1:], T.sum(1, keepdims=True)], axis=1)
    assert Y.shape[1] == 8
    for k in (1, 32):
        fn = KNeighborsRegressor(n_neighbors=k, weights="distance").fit(X, Y).predict
        spec = extract_knn_spec(fn)
        np.testing.assert_allclose(spec(Q), fn(Q), rtol=1e-12, atol=1e-12)


def test_ties_on_integer_data_follow_the_lower_index_rule():
    rng = np.random.default_rng(1)
    X = rng.integers(0, 3, size=(300, 4)).astype(float)
    y = rng.integers(0, 2, 300)
    Q = rng.integers(0, 3, size=(200, 4)).astype(float)
    spec = extract_knn_spec(KNeighborsClassifier(n_neighbors=5, algorithm="brute").fit(X, y).predict_proba)
    idx, _, tie = spec.neighbors(Q)
    assert tie.sum() > 50                                               # the data really ties at the boundary
    for i in range(Q.shape[0]):
        d = ((X - Q[i]) ** 2).sum(1)
        want = np.lexsort((np.arange(300), d))[:5]                      # (distance, index), lexicographically
        np.testing.assert_array_equal(idx[i], want)
        if i < 30:
            assert [v for _, v in neighbours(spec, Q[i])] == list(want)
    np.testing.assert_array_equal(spec(Q[:30]), reference(spec)(Q[:30]))


def test_zero_distance_rule():
    X, y, T, _ = _data(8)
    clf = _fit(KNeighborsClassifier(weights="distance"), X, y)
    spec = extract_knn_spec(clf.predict_proba)
    Q = X[:20]                                                         # training rows: distance exactly 0 to themselves
    _, exact = spec.statistic(Q)
    idx, ts, _ = spec.neighbors(Q)
    got = spec(Q)
    for i in range(20):
        zero = exact[i][idx[i]]
        assert zero.any() and np.all(ts[i][zero] == 0.0)
        want = np.zeros(spec.R)
        for v in idx[i][zero]:
            want[int(spec.y[v])] += 1.0
        np.testing.assert_array_equal(got[i], want / want.sum())       # the zero-distance neighbours alone vote
    np.testing.assert_array_equal(got, reference(spec)(Q))
    # a duplicated training row: both copies sit at distance 0 and share the vote
    Xd = np.concatenate([X, X[:1]])
    yd = np.concatenate([y, [(y[0] + 1) % 3]])
    spec = extract_knn_spec(KNeighborsClassifier(weights="distance").fit(Xd, yd).predict_proba)
    np.testing.assert_array_equal(spec(X[:1])[0][[y[0], (y[0] + 1) % 3]], [0.5, 0.5])
    reg = extract_knn_spec(KNeighborsRegressor(weights="distance").fit(X, T).predict)
    np.testing.assert_array_equal(reg(X[3:4])[0], T[3])


def test_other_models_are_not_neighbour_models():
    from sklearn.linear_model import LogisticRegression
    X, y, _, _ = _data(2)
    assert extract_knn_spec(LogisticRegression().fit(X, y).predict_proba) is None
    assert extract_knn_spec(np.sum) is None
    spec = extract_knn_spec(KNeighborsClassifier().fit(X, y).predict_proba)
    assert extract_knn_spec(spec) is spec


def _refusal(fn, exc, words):
    with pytest.raises(exc) as e:
        extract_knn_spec(fn)
    assert words in str(e.value), str(e.value)


def test_refusals():
    X, y, T, _ = _data(4)
    Xs = X[:, :3]
    _refusal(KNeighborsClassifier().fit(X, y).predict, TypeError, "pass predict_proba (predict returns labels)")
    _refusal(KNeighborsRegressor().fit(X, T).kneighbors, TypeError, "pass predict")
    _refusal(KNeighborsClassifier().fit(X, np.stack([y, y], 1)).predict_proba, NotImplementedError, "multi-output")
    _refusal(KNeighborsClassifier(weights=lambda d: 1 / (1 + d)).fit(X, y).predict_proba, NotImplementedError,
             "weights=<callable>")
    _refusal(KNeighborsClassifier(metric="chebyshev").fit(X, y).predict_proba, NotImplementedError,
             "metric='chebyshev'")
    _refusal(KNeighborsClassifier(p=np.inf).fit(X, y).predict_proba, NotImplementedError, "metric='chebyshev'")
    _refusal(KNeighborsClassifier(metric="cosine").fit(X, y).predict_proba, NotImplementedError, "metric='cosine'")
    D = ((Xs[:, None] - Xs[None]) ** 2).sum(-1)
    _refusal(KNeighborsClassifier(metric="precomputed").fit(D, y).predict_proba, NotImplementedError,
             "metric='precomputed'")
    _refusal(KNeighborsClassifier(metric="minkowski", metric_params={"w": np.ones(5)}).fit(X, y).predict_proba,
             NotImplementedError, "metric_params")
    _refusal(KNeighborsClassifier(n_neighbors=33).fit(X, y).predict_proba, NotImplementedError, "up to 32")
    _refusal(KNeighborsRegressor().fit(X, np.tile(T, 5)).predict, NotImplementedError, "10 targets")
    _refusal(KNeighborsClassifier().fit(X, np.arange(240) % 9).predict_proba, NotImplementedError, "9 classes")
    _refusal(make_pipeline(PolynomialFeatures(), KNeighborsClassifier()).fit(X, y).predict_proba, NotImplementedError,
             "PolynomialFeatures")
    _refusal(make_pipeline(MinMaxScaler(clip=True), KNeighborsClassifier()).fit(X, y).predict_proba,
             NotImplementedError, "clip=True")
    _refusal(RadiusNeighborsClassifier(radius=5.0).fit(X, y).predict_proba, NotImplementedError,
             "RadiusNeighborsClassifier is not supported")
    _refusal(RadiusNeighborsRegressor(radius=5.0).fit(X, T).predict, NotImplementedError,
             "RadiusNeighborsRegressor is not supported")
    _refusal(BaggingClassifier(KNeighborsClassifier(), n_estimators=2).fit(X, y).predict_proba, NotImplementedError,
             "BaggingClassifier holding a neighbour model")
    _refusal(VotingRegressor([("a", KNeighborsRegressor()), ("b", KNeighborsRegressor(3))]).fit(X, T[:, 0]).predict,
             NotImplementedError, "VotingRegressor holding a neighbour model")
    with pytest.raises(TypeError, match="not fitted"):
        extract_knn_spec(KNeighborsClassifier().predict_proba)


def test_spec_refusals():
    X, y, _, _ = _data(7, n=20)
    with pytest.raises(NotImplementedError, match="at least n_neighbors training rows"):
        KnnSpec(X[:4], np.ones(5), np.zeros(5), 5, "euclidean", 2, "uniform", "classify", y[:4], 3, 5)
    with pytest.raises(NotImplementedError, match="finite p >= 1"):
        KnnSpec(X, np.ones(5), np.zeros(5), 5, "minkowski", 0.5, "uniform", "classify", y, 3, 5)
    spec = KnnSpec(X, np.ones(5), np.zeros(5), 5, "euclidean", 2, "uniform", "classify", y, 3, 5)
    Q = X[:2].copy()
    Q[1, 2] = np.nan
    with pytest.raises(ValueError, match="NaN or an infinity"):
        spec(Q)


def test_scaler_refusals_name_the_neighbour_model():
    X, y, _, _ = _data(9)
    for pipe, words in ((make_pipeline(PolynomialFeatures(), KNeighborsClassifier()), "in front of a neighbour model"),
                        (make_pipeline(MinMaxScaler(clip=True), KNeighborsClassifier()), "neighbour models fold"),
                        (make_pipeline(PolynomialFeatures(), KNeighborsClassifier()), "its column weights and origins")):
        with pytest.raises(NotImplementedError) as e:
            extract_knn_spec(pipe.fit(X, y).predict_proba)
        assert words in str(e.value) and "kernel machine" not in str(e.value), str(e.value)


def test_a_statistic_that_rounds_to_zero_is_not_a_zero_distance():
    fitX = np.array([[0.0, 0.0], [1e-170, 0.0], [5.0, 5.0]])       # row 1's squared difference underflows to 0
    spec = KnnSpec(fitX, np.ones(2), np.zeros(2), 2, "euclidean", 2, "distance", "classify", [0, 1, 1], 2, 2)
    t, exact = spec.statistic(np.array([[0.0, 0.0]]))
    assert t[0, 0] == 0.0 and exact[0, 0] and t[0, 1] == 2.0 ** -1000 and not exact[0, 1]
    np.testing.assert_array_equal(spec(np.array([[0.0, 0.0], [1e-170, 0.0]])), [[1.0, 0.0], [0.0, 1.0]])
    np.testing.assert_array_equal(spec(fitX[:2]), reference(spec)(fitX[:2]))
