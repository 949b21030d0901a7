"""Gaussian-process regressors, KernelRidge with a scikit-learn kernel object and one-class SVMs read into
``KernelMachineSpec`` (CPU): the spec reproduces scikit-learn's own ``predict`` / ``decision_function`` /
``score_samples`` behind each affine scaler, the kernel algebra becomes at most four statistics and a postfix expression,
and every refusal names its reason."""
import warnings

import numpy as np
import pytest

sklearn = pytest.importorskip("sklearn")
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.ensemble import StackingRegressor, VotingRegressor  # noqa: E402
from sklearn.gaussian_process import GaussianProcessClassifier, GaussianProcessRegressor  # noqa: E402
from sklearn.gaussian_process.kernels import (RBF, CompoundKernel, ConstantKernel, DotProduct,  # noqa: E402
                                              ExpSineSquared, Matern, PairwiseKernel, RationalQuadratic, WhiteKernel)
from sklearn.kernel_ridge import KernelRidge  # noqa: E402
from sklearn.linear_model import Ridge  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import (MaxAbsScaler, MinMaxScaler, OneHotEncoder, RobustScaler,  # noqa: E402
                                   StandardScaler)
from sklearn.svm import SVC, SVR, OneClassSVM  # noqa: E402

from distributedkernelshap_b200.ensembles import extract_ensemble_spec  # noqa: E402
from distributedkernelshap_b200.kernel_machines import (MAX_STATS, KernelMachineSpec,  # noqa: E402
                                                        extract_kernel_machine_spec)
from distributedkernelshap_b200.stacking import extract_stacking_spec  # noqa: E402
from distributedkernelshap_b200.trees import extract_encoded_pipeline_spec  # noqa: E402

TOL = 1e-12
SCALERS = {"none": None, "standard": StandardScaler, "minmax": MinMaxScaler, "maxabs": MaxAbsScaler,
           "robust": RobustScaler}
P = 4

# every leaf of the kernel algebra, per-column and scalar length scales, and composites of sums, products and powers
KERNELS = {
    "rbf_scalar": lambda: RBF(1.5),
    "rbf_percol": lambda: RBF([0.8, 1.5, 2.5, 4.0]),
    "matern05": lambda: Matern(1.2, nu=0.5),
    "matern15": lambda: Matern([1.0, 2.0, 3.0, 1.5], nu=1.5),
    "matern25": lambda: Matern(2.0, nu=2.5),
    "matern_inf": lambda: Matern([1.0, 2.0, 3.0, 1.5], nu=np.inf),
    "rq": lambda: RationalQuadratic(length_scale=2.0, alpha=0.7),
    "expsine": lambda: ExpSineSquared(length_scale=3.0, periodicity=20.0),
    "dot": lambda: DotProduct(sigma_0=0.5),
    "const_rbf_white": lambda: ConstantKernel(2.0) * RBF(1.5) + WhiteKernel(0.1),
    "sum_product": lambda: RBF(2.0) * Matern(3.0, nu=1.5) + ConstantKernel(0.5),
    "power": lambda: (DotProduct(sigma_0=1.0) + ConstantKernel(0.3)) ** 2,
    "four_stats": lambda: (ConstantKernel(1.5) * RBF([0.8, 1.5, 2.5, 4.0]) + ConstantKernel(0.7) * Matern(2.0, nu=2.5)
                           + DotProduct(sigma_0=0.4) ** 2 + WhiteKernel(0.2)),
}


def _data(seed=0, n=80):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    y = np.sin(X[:, 0]) + 0.3 * X[:, 1] * X[:, 2] - 0.2 * X[:, 3]
    Xt = rng.normal(size=(30, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    return X, y, Xt


def _wrap(est, scaler):
    return est if SCALERS[scaler] is None else make_pipeline(SCALERS[scaler](), est)


def _fit(est, X, y):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return est.fit(X, y)


def _scale(spec, X, want):
    """The size of the sum the prediction is, sum_v |dual[v] K(x, v)| + |intercept| (a prediction can be far smaller
    than its terms), or of the prediction when larger."""
    if spec.program is not None:
        Kv = spec.program(spec.program.statistics(X, spec.sv))
    else:
        Kv = spec.kernel_values(spec.statistic(X, 0), 0)
    return max(np.abs(want).max(), (np.abs(Kv) @ np.abs(spec.dual)).max() + np.abs(spec.intercept).max())


def _check(fn, Xt):
    spec = extract_kernel_machine_spec(fn)
    assert isinstance(spec, KernelMachineSpec)
    want = np.asarray(fn(Xt), dtype=np.float64)
    got = spec(Xt)
    assert got.shape == want.shape
    scale = _scale(spec, Xt, want)
    assert np.abs(got - want).max() <= TOL * scale, np.abs(got - want).max() / scale
    return spec


def _gp(kernel, **kw):
    # ExpSineSquared is not positive definite over several columns: a larger noise term keeps the fit's Cholesky finite
    alpha = 1.0 if "ExpSineSquared" in repr(kernel) else 0.1
    return GaussianProcessRegressor(kernel, alpha=alpha, optimizer=None, **kw)


@pytest.mark.parametrize("scaler", list(SCALERS))
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_gp_predict(kernel, scaler):
    X, y, Xt = _data()
    spec = _check(_fit(_wrap(_gp(KERNELS[kernel]()), scaler), X, y).predict, Xt)
    assert spec.kernel == "program" and spec.head == "identity" and spec.scalar_out and spec.R == 1
    assert 1 <= spec.program.L <= MAX_STATS


@pytest.mark.parametrize("normalize_y", [False, True])
@pytest.mark.parametrize("targets", [1, 3])
def test_gp_targets_and_normalisation(targets, normalize_y):
    X, y, Xt = _data(1)
    Y = y if targets == 1 else np.c_[y, y ** 2, 3.0 - y]
    gp = _fit(_gp(ConstantKernel(1.2) * RBF([0.8, 1.5, 2.5, 4.0]), normalize_y=normalize_y), X, Y)
    spec = _check(gp.predict, Xt)
    assert spec.R == targets and spec.scalar_out == (targets == 1)


def test_gp_one_target_column_is_squeezed():
    X, y, Xt = _data(2)
    spec = _check(_fit(_gp(RBF(1.0), normalize_y=True), X, y[:, None]).predict, Xt)
    assert spec.scalar_out


def test_gp_optimised_kernel_is_read():
    """kernel_ (the fitted hyperparameters), not the kernel passed in"""
    X, y, Xt = _data(3)
    gp = _fit(GaussianProcessRegressor(ConstantKernel() * RBF(np.ones(P)) + WhiteKernel(), normalize_y=True), X, y)
    assert gp.kernel_ != gp.kernel
    _check(gp.predict, Xt)


def test_four_statistics_composite():
    X, y, Xt = _data(4)
    spec = _check(_fit(_gp(KERNELS["four_stats"]()), X, y).predict, Xt)
    assert spec.program.L == 3 and spec.program.kinds.count("dot") == 1
    k = (RBF(1.0) + RBF(2.0) * Matern(2.0, nu=0.5) + RationalQuadratic(1.0, 1.0) + DotProduct())
    spec = _check(_fit(_gp(k), X, y).predict, Xt)
    assert spec.program.L == 4


def test_shared_statistics():
    """leaves with the same length scales read one statistic"""
    X, y, Xt = _data(5)
    spec = _check(_fit(_gp(RBF(2.0) + Matern(2.0, nu=1.5) * Matern(2.0, nu=0.5)), X, y).predict, Xt)
    assert spec.program.L == 1


@pytest.mark.parametrize("scaler", ["none", "standard", "robust"])
def test_kernel_ridge_kernel_object(scaler):
    X, y, Xt = _data(6)
    for k in (RBF([0.8, 1.5, 2.5, 4.0]), Matern(2.0, nu=1.5) + DotProduct(0.3)):
        spec = _check(_fit(_wrap(KernelRidge(alpha=0.5, kernel=k), scaler), X, y).predict, Xt)
        assert spec.kernel == "program"
    spec = _check(_fit(KernelRidge(kernel=RBF(2.0)), X, np.c_[y, -y]).predict, Xt)
    assert spec.R == 2 and not spec.scalar_out


@pytest.mark.parametrize("scaler", list(SCALERS))
@pytest.mark.parametrize("kernel", ["rbf", "poly", "sigmoid"])
@pytest.mark.parametrize("method", ["decision_function", "score_samples"])
def test_one_class_svm(method, kernel, scaler):
    X, _, Xt = _data(7)
    kw = {"gamma": 0.05} if kernel == "sigmoid" else {}
    est = _fit(_wrap(OneClassSVM(kernel=kernel, nu=0.3, **kw), scaler), X, None)
    spec = _check(getattr(est, method), Xt)
    assert spec.kernel == kernel and spec.scalar_out and spec.program is None


def test_program_flat_form():
    X, y, _ = _data(8)
    spec = extract_kernel_machine_spec(_fit(_gp(KERNELS["four_stats"]()), X, y).predict)
    ops, args, a, b = spec.program.flat()
    assert ops.dtype == np.int32 and args.dtype == np.int32 and len(ops) == len(a) == len(b) == len(args)
    assert spec.program.depth() <= 4
    assert spec.program.colw.shape == (spec.program.L, P) and np.all(spec.program.colw > 0)


def test_is_kernel_machine_in_ensembles_and_pipelines():
    """GPs become soft-voting and stacking members, and sit behind encoded pipelines"""
    X, y, Xt = _data(9)
    vote = _fit(VotingRegressor([("gp", _gp(RBF(1.5))), ("ridge", Ridge())]), X, y)
    spec = extract_ensemble_spec(vote.predict)
    assert spec is not None
    assert np.abs(spec(Xt) - vote.predict(Xt)).max() <= 1e-12 * np.abs(vote.predict(Xt)).max()
    stack = _fit(StackingRegressor([("gp", _gp(Matern(2.0, nu=1.5))), ("svr", SVR())], final_estimator=Ridge(), cv=3),
                 X, y)
    sspec = extract_stacking_spec(stack.predict)
    sspec = sspec[0] if isinstance(sspec, tuple) else sspec
    assert np.abs(sspec(Xt) - stack.predict(Xt)).max() <= 1e-12 * np.abs(stack.predict(Xt)).max()
    rng = np.random.default_rng(0)
    Xc = np.c_[X, rng.integers(0, 3, size=len(X))]
    ct = ColumnTransformer([("num", StandardScaler(), [0, 1, 2, 3]), ("cat", OneHotEncoder(), [4])])
    for est, method in ((_gp(RBF(2.0)), "predict"), (OneClassSVM(nu=0.3), "decision_function")):
        pipe = _fit(make_pipeline(ct, est), Xc, y if method == "predict" else None)
        got = extract_encoded_pipeline_spec(getattr(pipe, method))
        assert got is not None and isinstance(got[0], KernelMachineSpec)


class MyRBF(RBF):
    pass


@pytest.mark.parametrize("make, match", [
    (lambda: _gp(Matern(1.0, nu=1.0)), "Bessel"),
    (lambda: _gp(PairwiseKernel(metric="laplacian")), "PairwiseKernel"),
    (lambda: _gp(MyRBF(1.0)), "user-defined"),
    (lambda: _gp(RBF(1.0) + RBF(2.0) + RBF(3.0) + RBF(4.0) + RBF(5.0)), "5 statistics"),
    (lambda: _gp(ConstantKernel(2.0) + WhiteKernel()), "constant"),
])
def test_kernel_refusals(make, match):
    X, y, _ = _data()
    est = _fit(make(), X, y)
    with pytest.raises(NotImplementedError, match=match):
        extract_kernel_machine_spec(est.predict)


def test_kernel_ridge_kernel_params_refused():
    X, y, _ = _data()
    est = _fit(KernelRidge(kernel=RBF(1.0)), X, y)
    est.kernel_params = {"length_scale": 2.0}
    with pytest.raises(NotImplementedError, match="kernel_params"):
        extract_kernel_machine_spec(est.predict)


def test_compound_kernel_refused():
    X, y, _ = _data()
    gp = _gp(RBF(1.0))
    _fit(gp, X, y)
    gp.kernel_ = CompoundKernel([RBF(1.0), RBF(2.0)])
    with pytest.raises(NotImplementedError, match="CompoundKernel"):
        extract_kernel_machine_spec(gp.predict)


def test_model_refusals():
    X, y, _ = _data()
    yc = (y > np.median(y)).astype(int)
    with pytest.raises(NotImplementedError, match="GaussianProcessClassifier"):
        extract_kernel_machine_spec(_fit(GaussianProcessClassifier(RBF(1.0)), X, yc).predict_proba)
    with pytest.raises(NotImplementedError, match="kernel objects"):
        extract_kernel_machine_spec(_fit(SVC(kernel=RBF(1.0)), X, yc).decision_function)
    with pytest.raises(NotImplementedError, match="kernel objects"):
        extract_kernel_machine_spec(_fit(SVR(kernel=RBF(1.0)), X, y).predict)
    for kernel in ("linear", "precomputed"):
        Xk = X @ X.T if kernel == "precomputed" else X
        with pytest.raises(NotImplementedError, match=kernel):
            extract_kernel_machine_spec(_fit(OneClassSVM(kernel=kernel), Xk, None).decision_function)
    with pytest.raises(TypeError, match="labels"):
        extract_kernel_machine_spec(_fit(OneClassSVM(), X, None).predict)
    with pytest.raises(TypeError, match="not fitted"):
        extract_kernel_machine_spec(GaussianProcessRegressor(RBF(1.0)).predict)
    with pytest.raises(TypeError, match="pass predict"):
        extract_kernel_machine_spec(_fit(_gp(RBF(1.0)), X, y).sample_y)
    with pytest.raises(NotImplementedError, match="9 targets"):
        extract_kernel_machine_spec(_fit(_gp(RBF(1.0)), X, np.repeat(y[:, None], 9, axis=1)).predict)
