"""CPU checks of the soft-voting ensemble reader (``ensembles.extract_ensemble_spec``): the NumPy ``EnsembleSpec`` against
scikit-learn for every member family, weights, dropped and nested members and an outer ColumnTransformer; all-linear
ensembles left to the mixture route; every refusal with its wording."""
import numpy as np
import pytest

sklearn = pytest.importorskip("sklearn")
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.calibration import CalibratedClassifierCV  # noqa: E402
from sklearn.ensemble import (BaggingClassifier, GradientBoostingClassifier, RandomForestClassifier,  # noqa: E402
                              RandomForestRegressor, StackingClassifier, VotingClassifier, VotingRegressor)
from sklearn.multiclass import OneVsRestClassifier  # noqa: E402
from sklearn.linear_model import LinearRegression, LogisticRegression, PoissonRegressor, Ridge  # noqa: E402
from sklearn.neighbors import KNeighborsClassifier, KNeighborsRegressor  # noqa: E402
from sklearn.neural_network import MLPClassifier, MLPRegressor  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import OneHotEncoder, StandardScaler  # noqa: E402
from sklearn.svm import SVC, SVR  # noqa: E402
from sklearn.tree import DecisionTreeClassifier  # noqa: E402

from distributedkernelshap_b200.ensembles import EnsembleSpec, extract_ensemble_spec  # noqa: E402
from distributedkernelshap_b200.mlp import MlpSpec  # noqa: E402


def _data(n=160, d=5, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d))
    y2 = (X[:, 0] + 0.5 * X[:, 1] > 0).astype(int)
    y3 = np.digitize(X[:, 0] + 0.3 * X[:, 2], [-0.4, 0.4])
    yr = X[:, 0] - 2 * X[:, 1] + 0.5 * X[:, 2] * X[:, 3]
    return X, y2, y3, yr


def _mlp(**kw):
    return MLPClassifier((8,), max_iter=300, random_state=0, **kw)


def _close(spec, want, X):
    got = spec(X)
    assert got.shape == np.asarray(want).shape
    np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-13)


@pytest.mark.parametrize("classes", [2, 3])
def test_every_member_family(classes):
    X, y2, y3, _ = _data()
    y = y2 if classes == 2 else y3
    members = [("lr", LogisticRegression()), ("rf", RandomForestClassifier(5, max_depth=4, random_state=0)),
               ("mlp", _mlp()), ("knn", KNeighborsClassifier(4))]
    if classes == 2:                        # the calibrated kernel machine is binary
        members.append(("svc", CalibratedClassifierCV(SVC(), cv=2, ensemble=False)))
    w = np.array([1, 2, 0.5, 1, 1.5])[:len(members)]
    vote = VotingClassifier(members, voting="soft", weights=w).fit(X, y)
    spec = extract_ensemble_spec(vote.predict_proba)
    assert isinstance(spec, EnsembleSpec) and spec.n_outputs == classes and len(spec.members) == len(members)
    np.testing.assert_allclose(spec.weights, w / w.sum())
    assert isinstance(spec.members[0][1], MlpSpec)            # the linear member, lowered
    _close(spec, vote.predict_proba(X), X)


def test_regressor_drop_and_nesting():
    X, _, _, yr = _data()
    inner = VotingRegressor([("ridge", Ridge()), ("knn", KNeighborsRegressor(3))], weights=[3, 1])
    vote = VotingRegressor([("lin", LinearRegression()), ("gone", "drop"), ("rf", RandomForestRegressor(4, random_state=0)),
                            ("mlp", MLPRegressor(hidden_layer_sizes=(6,), max_iter=200, random_state=0)), ("svr", SVR()), ("in", inner)],
                           weights=[1, 5, 2, 1, 1, 2]).fit(X, yr)
    spec = extract_ensemble_spec(vote.predict)
    assert spec.scalar_out and spec.n_outputs == 1 and len(spec.members) == 6
    np.testing.assert_allclose(spec.weights, np.array([1, 2, 1, 1, 2 * 0.75, 2 * 0.25]) / 7.0)
    _close(spec, vote.predict(X), X)


def test_nested_classifier_and_gradient_boosting():
    X, _, y3, _ = _data()
    inner = VotingClassifier([("gb", GradientBoostingClassifier(n_estimators=5, max_depth=2, random_state=0)),
                              ("lr", LogisticRegression())], voting="soft", weights=[1, 3])
    vote = VotingClassifier([("in", inner), ("dt", DecisionTreeClassifier(max_depth=3, random_state=0))],
                            voting="soft").fit(X, y3)
    spec = extract_ensemble_spec(vote.predict_proba)
    np.testing.assert_allclose(spec.weights, [0.125, 0.375, 0.5])
    _close(spec, vote.predict_proba(X), X)


def test_outer_column_transformer():
    X, y2, _, _ = _data()
    Xc = np.c_[X[:, :3], np.random.default_rng(1).integers(0, 3, size=(len(X), 2)).astype(float)]
    ct = ColumnTransformer([("num", StandardScaler(), [0, 1, 2]), ("cat", OneHotEncoder(handle_unknown="ignore"), [3, 4])],
                           sparse_threshold=0)
    pipe = make_pipeline(ct, VotingClassifier([("lr", LogisticRegression()), ("rf", RandomForestClassifier(5,
                                               random_state=0)), ("knn", KNeighborsClassifier(3))],
                                              voting="soft")).fit(Xc, y2)
    spec, enc = extract_ensemble_spec(pipe.predict_proba)
    assert spec.n_features == 5 and enc.E == 3 + 6
    _close(spec, pipe.predict_proba(Xc), pipe[:-1].transform(Xc))


def test_all_linear_ensembles_stay_on_the_mixture_route():
    X, y2, _, yr = _data()
    vote = VotingClassifier([("a", LogisticRegression()), ("b", LogisticRegression(C=0.1))], voting="soft").fit(X, y2)
    assert extract_ensemble_spec(vote.predict_proba) is None
    assert extract_ensemble_spec(VotingRegressor([("a", Ridge()), ("b", LinearRegression())]).fit(X, yr).predict) is None
    assert extract_ensemble_spec(LogisticRegression().fit(X, y2).predict_proba) is None
    assert extract_ensemble_spec(RandomForestClassifier(3).fit(X, y2).predict_proba) is None


def _refusals():
    X, y2, y3, yr = _data()
    rf = RandomForestClassifier(3, max_depth=3, random_state=0)
    yield "hard", VotingClassifier([("rf", rf), ("lr", LogisticRegression())]).fit(X, y2).predict, \
        NotImplementedError, "voting='hard'"
    yield "stacking", StackingClassifier([("rf", rf), ("lr", LogisticRegression())], cv=2).fit(X, y2).predict_proba, \
        NotImplementedError, "StackingClassifier is not supported"
    yield "pipeline_member", VotingClassifier([("p", make_pipeline(StandardScaler(), DecisionTreeClassifier())),
                                               ("lr", LogisticRegression())], voting="soft").fit(X, y2).predict_proba, \
        NotImplementedError, "put the preprocessing in front of the ensemble"
    yield "bagged_tree", VotingClassifier([("b", BaggingClassifier(DecisionTreeClassifier(), n_estimators=2)),
                                           ("m", _mlp())], voting="soft").fit(X, y2).predict_proba, \
        NotImplementedError, "ensemble"
    yield "ovr_member", VotingClassifier([("rf", rf), ("lr", OneVsRestClassifier(LogisticRegression()))],
                                         voting="soft").fit(X, y3).predict_proba, NotImplementedError, "one-vs-rest"
    yield "mixture_member", VotingClassifier([("rf", rf), ("cal", CalibratedClassifierCV(LogisticRegression(), cv=2))],
                                             voting="soft").fit(X, y2).predict_proba, NotImplementedError, "a mixture"
    yield "exp_member", VotingRegressor([("rf", RandomForestRegressor(3)), ("p", PoissonRegressor())]).fit(
        X, np.exp(yr / 4)).predict, NotImplementedError, "exp-head"
    yield "members", VotingRegressor([(f"m{k}", Ridge(alpha=k + 1.0)) for k in range(16)] +
                                     [("rf", RandomForestRegressor(2))]).fit(X, yr).predict, NotImplementedError, "at most 16"
    y9 = np.arange(len(X)) % 9
    yield "outputs", VotingClassifier([("dt", DecisionTreeClassifier(max_depth=2)), ("k", KNeighborsClassifier(2))],
                                      voting="soft").fit(X, y9).predict_proba, NotImplementedError, "8"
    yield "method", VotingRegressor([("rf", RandomForestRegressor(2)), ("r", Ridge())]).fit(X, yr).score, TypeError, \
        "pass predict"


REFUSALS = {name: rest for name, *rest in _refusals()}


@pytest.mark.parametrize("name", sorted(REFUSALS))
def test_refusals(name):
    fn, exc, words = REFUSALS[name]
    with pytest.raises(exc) as e:
        extract_ensemble_spec(fn)
    assert words in str(e.value), str(e.value)
