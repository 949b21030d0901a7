"""Kernel machines read into ``KernelMachineSpec`` (CPU): the spec and the independent reference reproduce every
scikit-learn method the kernel-machine route covers, behind each affine scaler; every refusal names its reason; linear SVMs
and trees keep their own extraction."""
import numpy as np
import pytest

sklearn = pytest.importorskip("sklearn")
from sklearn.calibration import CalibratedClassifierCV  # noqa: E402
from sklearn.ensemble import RandomForestClassifier  # noqa: E402
from sklearn.kernel_ridge import KernelRidge  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import (MaxAbsScaler, MinMaxScaler, PolynomialFeatures, RobustScaler,  # noqa: E402
                                   StandardScaler)
from sklearn.svm import SVC, SVR, LinearSVC, NuSVC, NuSVR  # noqa: E402

from distributedkernelshap_b200.kernel_machines import KernelMachineSpec, extract_kernel_machine_spec  # noqa: E402
from kernel_machine_reference import outputs  # noqa: E402

TOL = 1e-10
SCALERS = {"none": None, "standard": StandardScaler, "minmax": MinMaxScaler, "maxabs": MaxAbsScaler,
           "robust": RobustScaler}


def _data(seed=0, n=150, P=5):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 3.0, P) + np.linspace(-2.0, 4.0, P)
    s = (X[:, 0] - X[:, 0].mean()) + 0.3 * (X[:, 1] - X[:, 1].mean()) * (X[:, 2] - X[:, 2].mean())
    Xt = rng.normal(size=(40, P)) * np.linspace(0.5, 3.0, P) + np.linspace(-2.0, 4.0, P)
    return X, (s > 0).astype(int), s, Xt


def _wrap(est, scaler):
    return est if SCALERS[scaler] is None else make_pipeline(SCALERS[scaler](), est)


def _kw(kernel):
    return {"gamma": 0.02} if kernel == "sigmoid" else {}


def _check(fn, Xt):
    spec = extract_kernel_machine_spec(fn)
    assert isinstance(spec, KernelMachineSpec)
    want = np.asarray(fn(Xt), dtype=np.float64)
    scale = np.abs(want).max()
    for got in (spec(Xt), outputs(spec, Xt)):
        assert got.shape == want.shape
        assert np.abs(got - want).max() <= TOL * scale, np.abs(got - want).max() / scale
    return spec


@pytest.mark.parametrize("scaler", list(SCALERS))
@pytest.mark.parametrize("kernel", ["rbf", "poly", "sigmoid"])
@pytest.mark.parametrize("cls", [SVC, NuSVC])
def test_svc_decision_function(cls, kernel, scaler):
    X, y, _, Xt = _data()
    spec = _check(_wrap(cls(kernel=kernel, **_kw(kernel)), scaler).fit(X, y).decision_function, Xt)
    assert spec.head == "identity" and spec.scalar_out and spec.K == 1


@pytest.mark.parametrize("scaler", list(SCALERS))
@pytest.mark.parametrize("kernel", ["rbf", "poly", "sigmoid"])
@pytest.mark.parametrize("cls", [SVR, NuSVR])
def test_svr_predict(cls, kernel, scaler):
    X, _, s, Xt = _data(1)
    _check(_wrap(cls(kernel=kernel, **_kw(kernel)), scaler).fit(X, s).predict, Xt)


@pytest.mark.parametrize("scaler", list(SCALERS))
@pytest.mark.parametrize("kernel", ["rbf", "laplacian", "poly", "polynomial", "sigmoid"])
@pytest.mark.parametrize("targets", [1, 3, 8])
def test_kernel_ridge_predict(kernel, scaler, targets):
    X, y, s, Xt = _data(2)
    Y = s if targets == 1 else np.stack([s * (q + 1) + q * y for q in range(targets)], axis=1)
    spec = _check(_wrap(KernelRidge(kernel=kernel, alpha=0.5, **_kw(kernel)), scaler).fit(X, Y).predict, Xt)
    assert spec.scalar_out == (targets == 1) and spec.n_outputs == targets


def test_kernel_ridge_gamma_none_is_one_over_features():
    X, _, s, Xt = _data(3)
    spec = _check(KernelRidge(kernel="rbf").fit(X, s).predict, Xt)
    assert spec.gamma[0] == 1.0 / X.shape[1]


@pytest.mark.parametrize("scaler", list(SCALERS))
@pytest.mark.parametrize("kernel", ["rbf", "poly", "sigmoid"])
@pytest.mark.parametrize("ensemble", [True, False])
def test_calibrated_svc_predict_proba(kernel, scaler, ensemble):
    X, y, _, Xt = _data(4)
    est = CalibratedClassifierCV(_wrap(SVC(kernel=kernel, **_kw(kernel)), scaler), ensemble=ensemble, cv=3)
    spec = _check(est.fit(X, y).predict_proba, Xt)
    assert spec.head == "calibrated" and spec.K == (3 if ensemble else 1)


@pytest.mark.parametrize("kernel", ["rbf", "poly"])
def test_pipeline_around_calibrated_nusvc(kernel):
    X, y, _, Xt = _data(5)
    est = make_pipeline(MinMaxScaler(), CalibratedClassifierCV(make_pipeline(StandardScaler(), NuSVC(kernel=kernel)),
                                                               ensemble=True, cv=3))
    _check(est.fit(X, y).predict_proba, Xt)


def test_two_scalers_compose():
    X, _, s, Xt = _data(6)
    _check(make_pipeline(RobustScaler(), MaxAbsScaler(), SVR()).fit(X, s).predict, Xt)


def test_refusals():
    X, y, s, Xt = _data(7)
    y3 = np.digitize(s, [-1.0, 1.0])
    with pytest.raises(NotImplementedError, match="one-vs-one"):
        extract_kernel_machine_spec(SVC().fit(X, y3).decision_function)
    with pytest.raises(NotImplementedError, match=r"CalibratedClassifierCV\(SVC\(\), ensemble=False\)"):
        extract_kernel_machine_spec(SVC(probability=True).fit(X, y).predict_proba)
    with pytest.raises(NotImplementedError, match="precomputed"):
        extract_kernel_machine_spec(SVC(kernel="precomputed").fit(X @ X.T, y).decision_function)
    with pytest.raises(NotImplementedError, match="callable"):
        extract_kernel_machine_spec(SVR(kernel=lambda A, B: A @ B.T).fit(X, s).predict)
    with pytest.raises(NotImplementedError, match="chi2"):
        extract_kernel_machine_spec(KernelRidge(kernel="chi2", gamma=1.0).fit(np.abs(X), s).predict)
    for degree in (2.5, -1):
        bad = KernelRidge(kernel="poly", degree=2).fit(X, s)
        bad.degree = degree                  # scikit-learn's own fit fails on the NaN / inf such a degree gives
        with pytest.raises(NotImplementedError, match="integer"):
            extract_kernel_machine_spec(bad.predict)
    with pytest.raises(NotImplementedError, match="PolynomialFeatures"):
        extract_kernel_machine_spec(make_pipeline(PolynomialFeatures(2), SVR()).fit(X, s).predict)
    with pytest.raises(NotImplementedError, match="clip"):
        extract_kernel_machine_spec(make_pipeline(MinMaxScaler(clip=True), SVR()).fit(X, s).predict)
    with pytest.raises(NotImplementedError, match="isotonic"):
        extract_kernel_machine_spec(CalibratedClassifierCV(SVC(), method="isotonic", cv=3).fit(X, y).predict_proba)
    with pytest.raises(TypeError, match="decision_function"):
        extract_kernel_machine_spec(SVC().fit(X, y).predict)
    with pytest.raises(TypeError, match="predict"):
        extract_kernel_machine_spec(SVR().fit(X, s).score)


def test_other_models_keep_their_route():
    from distributedkernelshap_b200.predictors import extract_linear_spec
    from distributedkernelshap_b200.trees import extract_tree_spec
    X, y, s, _ = _data(8)
    for fn in (SVC(kernel="linear").fit(X, y).decision_function, LinearSVC().fit(X, y).decision_function,
               make_pipeline(StandardScaler(), SVC(kernel="linear")).fit(X, y).decision_function):
        assert extract_kernel_machine_spec(fn) is None
        assert extract_linear_spec(fn).activation == "identity"
    forest = RandomForestClassifier(5, max_depth=3, random_state=0).fit(X, y).predict_proba
    assert extract_kernel_machine_spec(forest) is None
    assert extract_tree_spec(forest) is not None
    assert extract_kernel_machine_spec(lambda Z: Z.sum(1)) is None
