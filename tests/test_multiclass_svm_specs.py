"""Multi-class SVMs read into ``MulticlassSvmSpec`` (CPU): the spec and the independent reference reproduce scikit-learn's
``decision_function_shape='ovo'`` pair values and ``CalibratedClassifierCV(SVC | NuSVC)`` probabilities over 3 to 8
classes, behind scalers inside the folds and around the calibrator; every refusal names its reason."""
import numpy as np
import pytest

sklearn = pytest.importorskip("sklearn")
from sklearn.calibration import CalibratedClassifierCV  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import MaxAbsScaler, MinMaxScaler, RobustScaler, StandardScaler  # noqa: E402
from sklearn.svm import SVC, NuSVC  # noqa: E402

from distributedkernelshap_b200.kernel_machines import (KernelMachineSpec, MulticlassSvmSpec,  # noqa: E402
                                                        extract_kernel_machine_spec)
from multiclass_svm_reference import outputs  # noqa: E402

TOL = 1e-10
SCALERS = {"none": None, "standard": StandardScaler, "minmax": MinMaxScaler, "maxabs": MaxAbsScaler,
           "robust": RobustScaler}


def _data(classes, seed=0, n=240, P=5):
    """Labels drawn from a softmax of a seeded random linear score."""
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 3.0, P) + np.linspace(-2.0, 4.0, P)
    Z = (X - X.mean(0)) / X.std(0) @ rng.normal(size=(P, classes)) * 2.0
    pr = np.exp(Z - Z.max(1, keepdims=True))
    pr /= pr.sum(1, keepdims=True)
    y = np.array([rng.choice(classes, p=p) for p in pr])
    y[:classes] = np.arange(classes)                    # every class present
    Xt = rng.normal(size=(30, P)) * np.linspace(0.5, 3.0, P) + np.linspace(-2.0, 4.0, P)
    return X, y, Xt


def _wrap(est, scaler):
    return est if SCALERS[scaler] is None else make_pipeline(SCALERS[scaler](), est)


def _svm(cls, kernel, **kw):
    kw = dict(kw)
    if kernel == "sigmoid":
        kw["gamma"] = 0.02
    if kernel == "poly":
        kw["degree"] = 2                                # degree 3 on unscaled columns: dec cancels to 1e-10 of its terms
    if cls is NuSVC:
        kw["nu"] = 0.05
    return cls(kernel=kernel, **kw)


def _check(fn, Xt):
    spec = extract_kernel_machine_spec(fn)
    assert isinstance(spec, MulticlassSvmSpec) and isinstance(spec, KernelMachineSpec)
    want = np.asarray(fn(Xt), dtype=np.float64)
    scale = np.abs(want).max()
    for got in (spec(Xt), outputs(spec, Xt)):
        assert got.shape == want.shape
        assert np.abs(got - want).max() <= TOL * scale, np.abs(got - want).max() / scale
    return spec


@pytest.mark.parametrize("scaler", ["none", "standard", "robust"])
@pytest.mark.parametrize("kernel", ["rbf", "poly", "sigmoid"])
@pytest.mark.parametrize("classes", [3, 4])
@pytest.mark.parametrize("cls", [SVC, NuSVC])
def test_ovo_decision_function(cls, classes, kernel, scaler):
    X, y, Xt = _data(classes, seed=classes)
    est = _wrap(_svm(cls, kernel, decision_function_shape="ovo"), scaler).fit(X, y)
    spec = _check(est.decision_function, Xt)
    P = classes * (classes - 1) // 2
    assert spec.head == "ovo" and spec.K == 1 and spec.n_outputs == P and spec.intercept.shape == (1, P)


@pytest.mark.parametrize("scaler", ["none", "standard", "minmax"])
@pytest.mark.parametrize("kernel", ["rbf", "poly", "sigmoid"])
@pytest.mark.parametrize("classes", [3, 5, 8])
@pytest.mark.parametrize("ensemble", [True, False])
@pytest.mark.parametrize("cls", [SVC, NuSVC])
def test_calibrated_predict_proba(cls, ensemble, classes, kernel, scaler):
    X, y, Xt = _data(classes, seed=10 + classes)
    est = CalibratedClassifierCV(_wrap(_svm(cls, kernel), scaler), ensemble=ensemble, cv=3).fit(X, y)
    spec = _check(est.predict_proba, Xt)
    assert spec.head == "ovo_proba" and spec.K == (3 if ensemble else 1) and spec.n_outputs == classes
    assert spec.cal_a.shape == (spec.K, classes)


@pytest.mark.parametrize("ensemble", [True, False])
def test_scalers_inside_and_around_the_calibrator(ensemble):
    X, y, Xt = _data(4, seed=3)
    inner = make_pipeline(StandardScaler(), MaxAbsScaler(), SVC(kernel="poly", degree=2))
    est = make_pipeline(MinMaxScaler(), RobustScaler(), CalibratedClassifierCV(inner, ensemble=ensemble, cv=3))
    _check(est.fit(X, y).predict_proba, Xt)


def test_four_classes_ovo_round_trip_of_class_blocks():
    X, y, _ = _data(4, seed=4)
    pipe = make_pipeline(StandardScaler(), SVC(decision_function_shape="ovo")).fit(X, y)
    spec = extract_kernel_machine_spec(pipe.decision_function)
    assert spec.cls_off.tolist() == [[0] + np.cumsum(pipe[-1].n_support_).tolist()]


def test_refusals():
    X, y3, _ = _data(3, seed=7)
    X9, y9, _ = _data(9, seed=8, n=400)
    _, y5, _ = _data(5, seed=9)
    with pytest.raises(NotImplementedError, match="one-vs-one") as e:
        extract_kernel_machine_spec(SVC().fit(X, y3).decision_function)
    assert "decision_function_shape='ovo'" in str(e.value)
    assert "CalibratedClassifierCV(SVC(), ensemble=False).predict_proba" in str(e.value)
    with pytest.raises(NotImplementedError, match="one-vs-one"):
        extract_kernel_machine_spec(make_pipeline(StandardScaler(), NuSVC(nu=0.05)).fit(X, y3).decision_function)
    with pytest.raises(NotImplementedError, match="10 pair values"):
        extract_kernel_machine_spec(SVC(decision_function_shape="ovo").fit(X, y5).decision_function)
    with pytest.raises(NotImplementedError, match="9 classes"):
        extract_kernel_machine_spec(SVC(decision_function_shape="ovo").fit(X9, y9).decision_function)
    with pytest.raises(NotImplementedError, match="9 classes"):
        extract_kernel_machine_spec(CalibratedClassifierCV(SVC(), ensemble=False).fit(X9, y9).predict_proba)
    with pytest.raises(NotImplementedError, match="isotonic"):
        extract_kernel_machine_spec(CalibratedClassifierCV(SVC(), method="isotonic", cv=3).fit(X, y3).predict_proba)
    with pytest.raises(NotImplementedError, match="temperature"):
        extract_kernel_machine_spec(CalibratedClassifierCV(SVC(), method="temperature", cv=3).fit(X, y3).predict_proba)
    with pytest.raises(NotImplementedError, match=r"CalibratedClassifierCV\(SVC\(\), ensemble=False\)"):
        extract_kernel_machine_spec(SVC(probability=True).fit(X, y3).predict_proba)
    # a fold whose estimator saw fewer classes than the calibrator: class 2 only in the last rows, unshuffled folds
    Xs = X[:90]
    ys = np.r_[np.zeros(40, int), np.ones(40, int), np.full(10, 2)]
    from sklearn.model_selection import KFold
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cal = CalibratedClassifierCV(SVC(), cv=KFold(3), ensemble=True).fit(Xs, ys)
    with pytest.raises(NotImplementedError, match="fold"):
        extract_kernel_machine_spec(cal.predict_proba)
    with pytest.raises(TypeError, match="decision_function"):
        extract_kernel_machine_spec(SVC().fit(X, y3).predict)


def test_linear_multiclass_svc_keeps_its_route():
    X, y, _ = _data(3, seed=11)
    assert extract_kernel_machine_spec(SVC(kernel="linear", decision_function_shape="ovo").fit(X, y)
                                       .decision_function) is None
