"""Kernel machines, MLPs and k-nearest-neighbour models behind per-column preprocessing
(``trees.extract_encoded_pipeline_spec``): the spec of the bare final estimator evaluated on the compiled column encoding
reproduces the pipeline's own method, scaler-only pipelines stay on the folded route, and the refusals raise with their
wording."""
import warnings

import numpy as np
import pytest

sklearn = pytest.importorskip("sklearn")
from sklearn.calibration import CalibratedClassifierCV  # noqa: E402
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.decomposition import PCA  # noqa: E402
from sklearn.impute import SimpleImputer  # noqa: E402
from sklearn.kernel_ridge import KernelRidge  # noqa: E402
from sklearn.neighbors import KNeighborsClassifier, KNeighborsRegressor  # noqa: E402
from sklearn.neural_network import MLPClassifier, MLPRegressor  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import (KBinsDiscretizer, MaxAbsScaler, MinMaxScaler, OneHotEncoder,  # noqa: E402
                                   OrdinalEncoder, PolynomialFeatures, RobustScaler, StandardScaler)
from sklearn.svm import SVC, SVR  # noqa: E402

from distributedkernelshap_b200.kernel_machines import extract_kernel_machine_spec  # noqa: E402
from distributedkernelshap_b200.mlp import extract_mlp_spec  # noqa: E402
from distributedkernelshap_b200.neighbors import extract_knn_spec  # noqa: E402
from distributedkernelshap_b200.trees import extract_encoded_pipeline_spec  # noqa: E402


def raw(seed, n, nan=False):
    rng = np.random.default_rng(seed)
    X = np.empty((n, 5))
    X[:, :3] = rng.normal(size=(n, 3)) * np.array([1.0, 2.0, 3.0]) + np.arange(3)
    if nan:
        X[rng.random(n) < 0.1, 2] = np.nan
    X[:, 3] = rng.choice([0.0, 1.0, 2.0, 5.0], n, p=[0.4, 0.3, 0.27, 0.03])
    X[:, 4] = rng.integers(0, 4, n).astype(float)
    s = X[:, 0] - 0.5 * X[:, 1] + (X[:, 3] == 1) + 0.3 * np.nan_to_num(X[:, 2]) + 0.2 * X[:, 4]
    return X, s


def ct(*parts, **kw):
    return ColumnTransformer(list(parts), **kw)


PRE = {   # (factory, NaN in column 2)
    "onehot_ignore": (lambda: ct(("n", StandardScaler(), [0, 1, 2]), ("c", OneHotEncoder(handle_unknown="ignore"),
                                                                      [3, 4])), False),
    "onehot_infrequent": (lambda: ct(("n", RobustScaler(), [0, 1]),
                                     ("c", OneHotEncoder(min_frequency=20, handle_unknown="infrequent_if_exist"), [3, 4]),
                                     remainder="passthrough"), False),
    "onehot_drop_first": (lambda: ct(("n", MaxAbsScaler(), [0, 1, 2]),
                                     ("c", OneHotEncoder(drop="first", handle_unknown="ignore"), [3, 4])), False),
    "ordinal_unknown": (lambda: ct(("c", OrdinalEncoder(handle_unknown="use_encoded_value", unknown_value=-1), [3, 4]),
                                   remainder="passthrough"), False),
    "kbins": (lambda: ct(("k", KBinsDiscretizer(5, encode="onehot-dense", strategy="quantile"), [0, 1]),
                         ("n", StandardScaler(), [2]), ("c", OneHotEncoder(handle_unknown="ignore"), [3])), False),
    "imputer_indicator": (lambda: ct(("i", make_pipeline(SimpleImputer(add_indicator=True), StandardScaler()), [0, 1, 2]),
                                     ("c", OneHotEncoder(handle_unknown="ignore"), [3, 4])), True),
    "minmax_clip": (lambda: make_pipeline(MinMaxScaler(clip=True)), False),
    "nested_drop": (lambda: ct(("n", make_pipeline(StandardScaler(), MinMaxScaler(clip=True)), [0, 1]),
                               ("c", OneHotEncoder(handle_unknown="ignore"), [4])), False),
    "sparse": (lambda: ct(("n", StandardScaler(), [0, 1, 2]), ("c", OneHotEncoder(handle_unknown="ignore"), [3, 4]),
                          sparse_threshold=1.0), False),
}
HEADS = {   # (estimator, method, target: classes (0: regression), rtol)
    "svc": (lambda: SVC(gamma=0.3), "decision_function", 2, 1e-10),
    "svr": (lambda: SVR(kernel="poly", degree=2, gamma=0.1), "predict", 0, 1e-10),
    "krr": (lambda: KernelRidge(kernel="laplacian", alpha=1.0, gamma=0.1), "predict", 0, 1e-10),
    "cal_svc": (lambda: CalibratedClassifierCV(SVC(kernel="sigmoid", gamma=0.01), cv=3), "predict_proba", 2, 1e-10),
    "mlp2": (lambda: MLPClassifier(hidden_layer_sizes=(10,), max_iter=200, random_state=0), "predict_proba", 2, 1e-12),
    "mlp3": (lambda: MLPClassifier(hidden_layer_sizes=(8, 6), activation="relu", max_iter=200, random_state=0), "predict_proba", 3, 1e-12),
    "mlp_reg": (lambda: MLPRegressor(hidden_layer_sizes=(8,), activation="logistic", max_iter=200, random_state=0), "predict", 0, 1e-12),
    "knn": (lambda: KNeighborsClassifier(5), "predict_proba", 2, 0.0),
    "knn_reg": (lambda: KNeighborsRegressor(4, weights="distance"), "predict", 0, 1e-12),
}


def fit(pre, head, n=250):
    make_pre, nan = PRE[pre]
    make, method, classes, rtol = HEADS[head]
    X, s = raw(0, n, nan=nan)
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, classes + 1)[1:-1])) if classes else s
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe = make_pipeline(make_pre(), make()).fit(X, y)
    return pipe, getattr(pipe, method), rtol, nan


@pytest.mark.parametrize("head", list(HEADS))
@pytest.mark.parametrize("pre", list(PRE))
def test_spec_on_the_encoding_reproduces_the_pipeline(pre, head):
    pipe, fn, rtol, nan = fit(pre, head)
    spec, enc = extract_encoded_pipeline_spec(fn)
    assert spec.n_features == enc.D == 5
    X, _ = raw(1, 60, nan=nan)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = np.asarray(fn(X), dtype=np.float64)
    got = np.asarray(spec(enc.transform(X)), dtype=np.float64)
    if head.startswith("knn"):
        tied = spec.boundary_ties(enc.transform(X))
        got, want = got[~tied], want[~tied]
    if rtol == 0.0:
        np.testing.assert_array_equal(got, want)
    else:
        np.testing.assert_allclose(got, want, rtol=rtol, atol=rtol * np.abs(want).max())


def test_colw_and_colo_are_the_identity():
    for head in ("svc", "knn"):
        spec, _ = extract_encoded_pipeline_spec(fit("onehot_ignore", head)[1])
        assert np.all(spec.colw == 1) and np.all(spec.colo == 0)


def test_calibrator_behind_the_preprocessing_and_a_single_fold():
    X, s = raw(0, 250)
    y = (s > np.median(s)).astype(int)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cal = CalibratedClassifierCV(make_pipeline(PRE["onehot_ignore"][0](), SVC()), ensemble=False).fit(X, y)
    spec, enc = extract_encoded_pipeline_spec(cal.predict_proba)
    assert spec.head == "calibrated" and spec.K == 1
    np.testing.assert_allclose(spec(enc.transform(X[:50])), cal.predict_proba(X[:50]), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("head", ["svc", "mlp2", "knn"])
def test_scaler_only_pipelines_keep_the_fold(head):
    make, method, classes, _ = HEADS[head]
    X, s = raw(0, 200)
    y = (s > np.median(s)).astype(int)
    pipe = make_pipeline(StandardScaler(), MinMaxScaler(), make()).fit(X, y)
    fn = getattr(pipe, method)
    assert extract_encoded_pipeline_spec(fn) is None
    extract = {"svc": extract_kernel_machine_spec, "mlp2": extract_mlp_spec, "knn": extract_knn_spec}[head]
    np.testing.assert_allclose(extract(fn)(X[:40]), fn(X[:40]), rtol=1e-9, atol=1e-12)   # the folded route
    assert extract_encoded_pipeline_spec(make().fit(X, y).__getattribute__(method)) is None


def test_existing_extractors_keep_their_refusals():
    pipe, fn, _, _ = fit("onehot_ignore", "svc")
    with pytest.raises(NotImplementedError, match="only StandardScaler, MinMaxScaler, MaxAbsScaler and RobustScaler"):
        extract_kernel_machine_spec(fn)
    X, s = raw(0, 200)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe = make_pipeline(MinMaxScaler(clip=True), MLPClassifier(hidden_layer_sizes=(4,), max_iter=20)).fit(X, s > 0)
    fn = pipe.predict_proba
    assert extract_encoded_pipeline_spec(fn) is not None
    with pytest.raises(NotImplementedError, match=r"MinMaxScaler\(clip=True\) is not affine"):
        extract_mlp_spec(fn)


@pytest.mark.parametrize("step,name", [(lambda: PolynomialFeatures(2), "PolynomialFeatures"), (lambda: PCA(2), "PCA")])
@pytest.mark.parametrize("head", ["svc", "mlp2", "knn"])
def test_refuses_steps_that_mix_columns(step, name, head):
    make, method, _, _ = HEADS[head]
    X, s = raw(0, 200)
    y = (s > np.median(s)).astype(int)
    pipe = make_pipeline(ct(("p", step(), [0, 1]), ("c", OneHotEncoder(handle_unknown="ignore"), [3])), make()).fit(X, y)
    family = {"svc": "a kernel machine", "mlp2": "an MLP", "knn": "a neighbour model"}[head]
    with pytest.raises(NotImplementedError, match=f"Pipeline in front of {family}: {name} is not supported.*encoders"):
        extract_encoded_pipeline_spec(getattr(pipe, method))


def test_refuses_string_categories_folds_and_dtypes():
    X, s = raw(0, 200)
    y = (s > np.median(s)).astype(int)
    Xs = X.astype(object)
    Xs[:, 3] = np.where(X[:, 3] > 0, "a", "b")
    strs = make_pipeline(ct(("c", OneHotEncoder(handle_unknown="ignore"), [3])), SVC()).fit(Xs, y)
    with pytest.raises(NotImplementedError, match="string categories are not supported"):
        extract_encoded_pipeline_spec(strs.decision_function)
    folds = CalibratedClassifierCV(make_pipeline(PRE["onehot_ignore"][0](), SVC()), cv=3).fit(X, y)
    with pytest.raises(NotImplementedError, match=r"3 folds, each with its own fitted preprocessing \(ColumnTransformer\)"
                                                  ".*move the preprocessing in front of the calibrator"):
        extract_encoded_pipeline_spec(folds.predict_proba)
    f32 = make_pipeline(ct(("c", OneHotEncoder(handle_unknown="ignore", dtype=np.float32), [3])),
                        MLPClassifier(hidden_layer_sizes=(4,), max_iter=50, random_state=0))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        f32.fit(X, y)
    with pytest.raises(NotImplementedError, match=r"dtype=float32\): only float64 encoder output is supported behind an MLP"):
        extract_encoded_pipeline_spec(f32.predict_proba)
