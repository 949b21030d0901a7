"""Every device and pinned-host allocation the engine holds has one owner (dks_live_allocations counts them): constructing,
explaining and closing an explainer of every head and family gives back all it took; repeated calls, refits, plan
replacements and refused calls leave the count where it was; an ensemble owns and frees its members, and members it
refuses stay the caller's to free."""
import ctypes as C
import gc
import warnings

import numpy as np
import pytest

from distributedkernelshap_b200 import _cabi

pytestmark = pytest.mark.gpu
pytest.importorskip("sklearn")
from sklearn.calibration import CalibratedClassifierCV  # noqa: E402
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.ensemble import RandomForestClassifier, VotingClassifier  # noqa: E402
from sklearn.linear_model import LogisticRegression, PoissonRegressor, Ridge  # noqa: E402
from sklearn.multiclass import OneVsRestClassifier  # noqa: E402
from sklearn.neighbors import KNeighborsRegressor  # noqa: E402
from sklearn.neural_network import MLPClassifier  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import OneHotEncoder, StandardScaler  # noqa: E402
from sklearn.svm import SVR, LinearSVC  # noqa: E402
from sklearn.tree import DecisionTreeClassifier  # noqa: E402


def live():
    gc.collect()                       # explainers of earlier tests free their contexts when collected
    n = C.c_int64(-1)
    _cabi.check(_cabi.load().dks_live_allocations(C.byref(n)))
    return n.value


def raw(seed, n):
    """Six raw columns, 3 and 4 categorical (small integers), and binary / three-class / positive targets."""
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, 6))
    X[:, 3] = rng.integers(0, 3, n)
    X[:, 4] = rng.integers(0, 4, n)
    s = X[:, 0] - 0.7 * X[:, 1] + 0.5 * X[:, 2] * (X[:, 3] - 1) + 0.3 * X[:, 4]
    return X, (s > 0).astype(int), np.digitize(s, [-0.5, 0.5]), np.exp(0.3 * s)


def columns(unknown="ignore"):
    return ColumnTransformer([("n", StandardScaler(), [0, 1, 2]), ("c", OneHotEncoder(handle_unknown=unknown), [3, 4])],
                             remainder="passthrough")


def _mlp():
    return MLPClassifier((8,), max_iter=300, random_state=0)


MODELS = {   # name: fitted model's output function, given (X, binary y, three-class y, positive y)
    "binary": lambda X, y2, y3, yp: LogisticRegression().fit(X, y2).predict_proba,
    "softmax": lambda X, y2, y3, yp: LogisticRegression().fit(X, y3).predict_proba,
    "ovr": lambda X, y2, y3, yp: OneVsRestClassifier(LogisticRegression()).fit(X, y3).predict_proba,
    "identity": lambda X, y2, y3, yp: Ridge().fit(X, yp).predict,
    "glm": lambda X, y2, y3, yp: PoissonRegressor(alpha=0.01).fit(X, yp).predict,
    "mixture": lambda X, y2, y3, yp: CalibratedClassifierCV(LinearSVC(), method="sigmoid", cv=3).fit(X, y2).predict_proba,
    "tree": lambda X, y2, y3, yp: RandomForestClassifier(4, max_depth=3, random_state=0).fit(X, y2).predict_proba,
    "kmach": lambda X, y2, y3, yp: SVR(gamma=0.3).fit(X, yp).predict,
    "mlp": lambda X, y2, y3, yp: _mlp().fit(X, y3).predict_proba,
    "knn": lambda X, y2, y3, yp: KNeighborsRegressor(4).fit(X, yp).predict,
    "ensemble": lambda X, y2, y3, yp: VotingClassifier(
        [("lr", LogisticRegression()), ("dt", DecisionTreeClassifier(max_depth=3, random_state=0)), ("mlp", _mlp())],
        voting="soft").fit(X, y2).predict_proba,
    "tree_pipeline": lambda X, y2, y3, yp: make_pipeline(columns(), DecisionTreeClassifier(max_depth=4, random_state=0))
    .fit(X, y2).predict_proba,
    "mlp_pipeline": lambda X, y2, y3, yp: make_pipeline(columns(), _mlp()).fit(X, y2).predict_proba,
    "linear_pipeline": lambda X, y2, y3, yp: make_pipeline(columns(), LogisticRegression()).fit(X, y2).predict_proba,
}


def explainer(f, bg, **kw):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    return GpuKernelExplainer(f, bg, link="identity", seed=0, **kw)


def model(name):
    X, y2, y3, yp = raw(0, 300)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return MODELS[name](X, y2, y3, yp), X[:16], X[100:110]


@pytest.mark.parametrize("plan_mode,l1_reg", [("shared", False), ("shared", "aic"), ("per_instance", False)])
@pytest.mark.parametrize("name", list(MODELS))
def test_construct_explain_close_frees_everything(name, plan_mode, l1_reg):
    f, bg, X = model(name)
    base = live()
    eng = explainer(f, bg, plan_mode=plan_mode)
    try:
        assert live() > base
        eng.shap_values(X, l1_reg=l1_reg)
    except NotImplementedError:        # an l1 selection the head does not run: the construction is still checked
        assert l1_reg
    finally:
        eng.close()
    assert live() == base


def test_plans_of_more_than_128_groups_are_freed():
    from conftest import make_problem
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.predictors import LinearSoftmaxClassifier
    prob = make_problem(seed=3, n=4, N=20, widths=(1,) * 160)
    clf = LinearSoftmaxClassifier(prob["clf"].coef_ * (2.0 / np.sqrt(160)), prob["clf"].intercept_, multi_class="multinomial")
    base = live()
    eng = explainer(clf.predict_proba, DenseData(prob["bg"], prob["group_names"], prob["groups"]))
    try:
        eng.shap_values(prob["X"], nsamples=600, l1_reg=False)
    finally:
        eng.close()
    assert live() == base


@pytest.mark.parametrize("name", ["binary", "tree_pipeline", "ensemble"])
def test_steady_state_calls_allocate_nothing_new(name):
    f, bg, X = model(name)
    eng = explainer(f, bg)
    try:
        eng.shap_values(X[:6], l1_reg=False)
        after = live()
        eng.shap_values(X[:6], l1_reg=False)
        eng.shap_values(X[:3], l1_reg=False)
        eng.predict(X[:6])
        assert live() == after
        eng.shap_values(X, l1_reg=False)          # more rows: the workspace is replaced, not added to
        assert live() == after
    finally:
        eng.close()


@pytest.mark.parametrize("name", ["binary", "softmax", "mixture", "tree", "mlp_pipeline"])
def test_refit_and_plan_replacement_return_to_the_same_count(name):
    f, bg, X = model(name)
    eng = explainer(f, bg)
    try:
        eng.shap_values(X, nsamples=40, l1_reg=False)
        after_a = live()
        _cabi.check(eng.lib.dks_fit(eng._ctx))
        eng.shap_values(X, nsamples=40, l1_reg=False)
        assert live() == after_a
        eng.shap_values(X, nsamples=24, l1_reg=False)
        eng.shap_values(X, nsamples=40, l1_reg=False)
        assert live() == after_a
    finally:
        eng.close()


def test_refused_raw_values_leave_the_count_unchanged():
    X, y2, _, _ = raw(0, 300)
    pipe = make_pipeline(columns(unknown="error"), DecisionTreeClassifier(max_depth=4, random_state=0)).fit(X, y2)
    bg, Xi = X[:10], X[10:14].copy()
    eng = explainer(pipe.predict_proba, bg)
    try:
        eng.shap_values(Xi, l1_reg=False)
        eng.predict(Xi)
        eng.encode(Xi)
        after = live()
        Xi[2, 4] = 9.0                             # a category unseen at fit time under handle_unknown='error'
        for call in (eng.predict, eng.encode, lambda x: eng.shap_values(x, l1_reg=False)):
            with pytest.raises(ValueError, match="2"):
                call(Xi)
            assert live() == after
    finally:
        eng.close()


def _knn_context(lib, rng):
    """A context holding a neighbour regressor over three columns (one output)."""
    ctx = C.c_void_p()
    _cabi.check(lib.dks_create(C.byref(ctx), 0))
    bg = np.ascontiguousarray(rng.normal(size=(10, 3)))
    _cabi.check(lib.dks_set_background(ctx, _cabi.ptr(bg), 10, 3, None))
    fitX, y = np.ascontiguousarray(rng.normal(size=(12, 3))), np.ascontiguousarray(rng.normal(size=12))
    colw, colo = np.ones(3), np.zeros(3)
    _cabi.check(lib.dks_set_knn_model(ctx, 12, _cabi.ptr(fitX), _cabi.ptr(colw), _cabi.ptr(colo), 3, 0, 2.0, 0, 1,
                                      _cabi.ptr(y), 1, 1))     # euclidean, uniform weights, regression head
    return ctx, bg


def test_ensemble_owns_accepted_members_and_leaves_refused_ones_to_the_caller():
    lib = _cabi.load()
    rng = np.random.default_rng(5)
    base = live()
    parent, bg = _knn_context(lib, rng)
    members = [_knn_context(lib, rng)[0] for _ in range(2)]
    ptrs = (C.c_void_p * 2)(*[m.value for m in members])
    pi = np.array([0.5, 0.5])
    assert lib.dks_set_ensemble(parent, 2, ptrs, _cabi.ptr(pi), 2, 1) == _cabi.DKS_ERR_UNSUPPORTED   # members give 1 output
    for m in members:
        _cabi.check(lib.dks_destroy(m))
    _cabi.check(lib.dks_destroy(parent))
    assert live() == base

    parent, bg = _knn_context(lib, rng)
    members = [_knn_context(lib, rng)[0] for _ in range(2)]
    ptrs = (C.c_void_p * 2)(*[m.value for m in members])
    _cabi.check(lib.dks_set_ensemble(parent, 2, ptrs, _cabi.ptr(pi), 1, 1))
    _cabi.check(lib.dks_fit(parent))
    assert live() > base
    _cabi.check(lib.dks_destroy(parent))          # frees its members with it
    assert live() == base
