"""MLPs read into float64 layers in raw feature space (distributedkernelshap_b200/mlp.py): the spec reproduces every covered
scikit-learn method behind each affine scaler, every refusal names its reason, and the other model families keep their own
extractions (CPU only)."""
import warnings

import numpy as np
import pytest

sklearn = pytest.importorskip("sklearn")
from sklearn.exceptions import ConvergenceWarning  # noqa: E402
from sklearn.neural_network import MLPClassifier, MLPRegressor  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import MaxAbsScaler, MinMaxScaler, RobustScaler, StandardScaler  # noqa: E402

from distributedkernelshap_b200.mlp import MlpSpec, extract_mlp_spec  # noqa: E402

TOL = 1e-12

SCALERS = {"none": None, "standard": StandardScaler, "minmax": MinMaxScaler, "maxabs": MaxAbsScaler,
           "robust": RobustScaler}


def _data(seed, P=6, n=150):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 3.0, P) + np.linspace(-2.0, 4.0, P)
    s = X[:, 0] - X[:, 0].mean() + 0.3 * (X[:, 1] - X[:, 1].mean()) * (X[:, 2] - X[:, 2].mean())
    return X, s, rng


def _fit(est, scaler, X, y):
    model = est if SCALERS.get(scaler) is None else make_pipeline(SCALERS[scaler](), est)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return model.fit(X, y)


def _head_target(head, s):
    if head == "sigmoid":
        return (s > 0).astype(int)
    if head == "softmax":
        return np.digitize(s, np.quantile(s, [0.33, 0.66]))
    return s


def _rel(got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (got.shape, want.shape)
    return float(np.max(np.abs(got - want)) / max(np.max(np.abs(want)), 1e-300))


CASES = [(act, head, depth) for act in ("identity", "logistic", "tanh", "relu")
         for head in ("identity", "sigmoid", "softmax") for depth in (1, 2, 3, 4)]


@pytest.mark.parametrize("act,head,depth", CASES)
def test_spec_reproduces_every_activation_head_and_depth(act, head, depth):
    X, s, rng = _data(depth * 7 + len(act) + len(head))
    hidden = tuple(int(h) for h in rng.integers(3, 12, size=depth))
    cls = MLPRegressor if head == "identity" else MLPClassifier
    model = _fit(cls(hidden_layer_sizes=hidden, activation=act, max_iter=60, random_state=0), "standard", X, _head_target(head, s))
    fn = model.predict if head == "identity" else model.predict_proba
    spec = extract_mlp_spec(fn)
    assert isinstance(spec, MlpSpec) and spec.head == head and spec.n_hidden == depth
    Xt = X[:40] + rng.normal(size=(40, X.shape[1]))
    assert _rel(spec(Xt), fn(Xt)) < TOL


@pytest.mark.parametrize("scaler", list(SCALERS))
@pytest.mark.parametrize("kind", ["classifier2", "classifier3", "regressor1", "regressor3"])
def test_spec_reproduces_behind_each_scaler(scaler, kind):
    X, s, rng = _data(3)
    if kind.startswith("classifier"):
        y = _head_target("sigmoid" if kind == "classifier2" else "softmax", s)
        model = _fit(MLPClassifier(hidden_layer_sizes=(9, 5), activation="tanh", max_iter=80, random_state=1), scaler, X, y)
        fn = model.predict_proba
    else:
        y = s if kind == "regressor1" else np.stack([s, 2 * s + X[:, 3], X[:, 4] - s], axis=1)
        model = _fit(MLPRegressor(hidden_layer_sizes=(8,), activation="relu", max_iter=80, random_state=1), scaler, X, y)
        fn = model.predict
    spec = extract_mlp_spec(fn)
    Xt = X[50:90] * 1.3
    want = fn(Xt)
    got = spec(Xt)
    assert got.shape == want.shape                   # a 1-D array for one regression target
    assert _rel(got, want) < TOL


def test_spec_of_a_float32_fitted_model():
    X, s, _ = _data(5)
    model = _fit(MLPClassifier(hidden_layer_sizes=(10, 6), max_iter=60, random_state=0), "standard", X.astype(np.float32), (s > 0).astype(int))
    assert model[-1].coefs_[0].dtype == np.float32
    spec = extract_mlp_spec(model.predict_proba)
    assert spec.coefs[0].dtype == np.float64
    Xt = X[:30]                                      # float64 rows: scikit-learn computes in float64
    assert _rel(spec(Xt), model.predict_proba(Xt)) < TOL


def test_default_pipeline_spec():
    X, s, _ = _data(8)
    model = _fit(MLPClassifier(max_iter=30, random_state=0), "standard", X, (s > 0).astype(int))
    spec = extract_mlp_spec(model.predict_proba)
    assert spec.widths == [X.shape[1], 100, 1] and spec.hidden_activation == "relu" and spec.n_outputs == 2
    widths, W, b = spec.flat()
    assert list(widths) == spec.widths and W.size == X.shape[1] * 100 + 100 and b.size == 101


def test_refusals_name_their_reason():
    X, s, _ = _data(9)
    y2 = (s > 0).astype(int)
    clf = _fit(MLPClassifier(hidden_layer_sizes=(5,), max_iter=20, random_state=0), None, X, y2)
    with pytest.raises(TypeError, match="predict returns labels"):
        extract_mlp_spec(clf.predict)
    multilabel = _fit(MLPClassifier(hidden_layer_sizes=(5,), max_iter=20, random_state=0), None, X, np.stack([y2, 1 - y2, y2], axis=1))
    with pytest.raises(NotImplementedError, match="multilabel"):
        extract_mlp_spec(multilabel.predict_proba)
    deep = _fit(MLPRegressor(hidden_layer_sizes=(3,) * 5, max_iter=20, random_state=0), None, X, s)
    with pytest.raises(NotImplementedError, match="5 hidden layers"):
        extract_mlp_spec(deep.predict)
    wide = _fit(MLPRegressor(hidden_layer_sizes=(257,), max_iter=5, random_state=0), None, X, s)
    with pytest.raises(NotImplementedError, match="257 units"):
        extract_mlp_spec(wide.predict)
    many = _fit(MLPRegressor(hidden_layer_sizes=(4,), max_iter=5, random_state=0), None, X, np.tile(s[:, None], (1, 9)))
    with pytest.raises(NotImplementedError, match="9 outputs"):
        extract_mlp_spec(many.predict)
    reg = _fit(MLPRegressor(hidden_layer_sizes=(4,), max_iter=5, random_state=0), None, X, s)
    with pytest.raises(TypeError, match="pass predict"):
        extract_mlp_spec(reg.score)
    from sklearn.decomposition import PCA
    pca = _fit(make_pipeline(PCA(3), MLPRegressor(hidden_layer_sizes=(4,), max_iter=5, random_state=0)), None, X, s)
    with pytest.raises(NotImplementedError, match="pca"):
        extract_mlp_spec(pca.predict)
    clipped = _fit(make_pipeline(MinMaxScaler(clip=True), MLPRegressor(hidden_layer_sizes=(4,), max_iter=5, random_state=0)), None, X, s)
    with pytest.raises(NotImplementedError, match="clip"):
        extract_mlp_spec(clipped.predict)


def test_other_families_keep_their_extractions():
    from sklearn.ensemble import RandomForestRegressor
    from sklearn.linear_model import LogisticRegression
    from sklearn.svm import SVC

    from distributedkernelshap_b200.predictors import extract_linear_spec
    X, s, _ = _data(11)
    y = (s > 0).astype(int)
    for fn in (LogisticRegression().fit(X, y).predict_proba, RandomForestRegressor(n_estimators=3).fit(X, s).predict,
               SVC().fit(X, y).decision_function, make_pipeline(StandardScaler(), SVC()).fit(X, y).decision_function,
               lambda Z: Z.sum(1)):
        assert extract_mlp_spec(fn) is None
    mlp = _fit(MLPClassifier(hidden_layer_sizes=(4,), max_iter=10, random_state=0), "standard", X, y)
    with pytest.raises((TypeError, NotImplementedError)):
        extract_linear_spec(mlp.predict_proba)


def test_spec_passes_through_and_checks_its_shapes():
    W0, W1 = np.ones((3, 4)), np.ones((4, 1))
    spec = MlpSpec([W0, W1], [np.zeros(4), np.zeros(1)], "relu", "sigmoid", 3)
    assert extract_mlp_spec(spec) is spec
    with pytest.raises(ValueError, match="do not chain"):
        MlpSpec([W0, np.ones((5, 1))], [np.zeros(4), np.zeros(1)], "relu", "identity", 3)
    with pytest.raises(ValueError, match="sigmoid head"):
        MlpSpec([W0, np.ones((4, 2))], [np.zeros(4), np.zeros(2)], "relu", "sigmoid", 3)
