"""Stacking ensembles of tree, kernel-machine, MLP, neighbour and linear members with a linear final estimator, explained on
the device: parity with the oracle calling the ensemble's own method, every plan source and entry point, background
chunks, the raw values a member refuses, an outer pipeline, the all-linear regressor's linear route, the device memory
owner, and the refusals."""
import warnings

import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")
from sklearn.calibration import CalibratedClassifierCV  # noqa: E402
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.ensemble import (GradientBoostingClassifier, RandomForestClassifier, RandomForestRegressor,  # noqa: E402
                              StackingClassifier, StackingRegressor)
from sklearn.linear_model import LinearRegression, LogisticRegression, Ridge, RidgeCV  # noqa: E402
from sklearn.neighbors import KNeighborsClassifier, KNeighborsRegressor  # noqa: E402
from sklearn.neural_network import MLPClassifier, MLPRegressor  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import OneHotEncoder, StandardScaler  # noqa: E402
from sklearn.svm import SVC, SVR, LinearSVC  # noqa: E402
from sklearn.tree import DecisionTreeClassifier  # noqa: E402

TOL = 1e-9
KNN_TOL = 1e-8
L1_TOL = 1e-5           # the l1 moments go through the 2^-40 fixed point


def _mlp():
    return MLPClassifier((8,), max_iter=300, random_state=0)


def _svc():
    return CalibratedClassifierCV(SVC(gamma=0.3), cv=2, ensemble=False)


MODELS = {   # members, classes (0: regression), stacking keyword arguments
    "clf2_five": (lambda: [("lr", LogisticRegression()), ("rf", RandomForestClassifier(6, max_depth=4, random_state=0)),
                           ("mlp", _mlp()), ("knn", KNeighborsClassifier(5)), ("svc", _svc())], 2, {}),
    "clf2_svc_df": (lambda: [("svc", SVC(gamma=0.3)), ("lsvc", LinearSVC()),
                             ("rf", RandomForestClassifier(4, max_depth=3, random_state=0))], 2,
                    {"stack_method": "auto"}),
    "clf3_pass": (lambda: [("gb", GradientBoostingClassifier(n_estimators=8, max_depth=2, random_state=0)),
                           ("mlp", _mlp()), ("knn", KNeighborsClassifier(6, weights="distance"))], 3,
                  {"passthrough": True}),
    "reg_pass": (lambda: [("rf", RandomForestRegressor(5, max_depth=4, random_state=0)), ("svr", SVR(gamma=0.2)),
                          ("mlp", MLPRegressor(hidden_layer_sizes=(8,), max_iter=300, random_state=0)),
                          ("knn", KNeighborsRegressor(4))], 0, {"passthrough": True, "final_estimator": RidgeCV()}),
    "clf2_linear": (lambda: [("lr", LogisticRegression()), ("lsvc", LinearSVC()), ("lr2", LogisticRegression(C=0.1))],
                    2, {}),
}
LINKS = {"clf2_five": ("identity", "logit"), "clf2_svc_df": ("logit",), "clf3_pass": ("identity", "logit"),
         "reg_pass": ("identity",), "clf2_linear": ("logit",)}
CASES = [(m, link) for m in MODELS for link in LINKS[m]]


def raw(seed, n, d=5):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)) * np.linspace(1.0, 2.0, d)
    s = X[:, 0] - 0.5 * X[:, 1] + 0.3 * X[:, 2] * X[:, 3] + 0.2 * np.sin(X[:, 4 % d])
    return X, s


def fitted(kind, seed=0, n=300, d=5, method=None):
    members, classes, kw = MODELS[kind]
    X, s = raw(seed, n, d)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if classes:
            y = np.digitize(s, np.quantile(s, np.linspace(0, 1, classes + 1)[1:-1]))
            st = StackingClassifier(members(), **kw).fit(X, y)
            return st, getattr(st, method or "predict_proba")
        st = StackingRegressor(members(), **kw).fit(X, s)
        return st, st.predict


def problem(seed, N, n, d=5, partial=True, weights=False):
    bg, _ = raw(seed, N, d)
    X, _ = raw(seed + 1, n, d)
    if partial:                                  # x takes the background's constant value of column 1 on every other row
        bg[:, 1] = 0.75
        X[::2, 1] = 0.75
    w = None
    if weights:
        w = np.random.default_rng(seed).uniform(0.1, 1.0, N)
        w[1] = 0.0                               # a zero-weight row is skipped, not divided by
    return bg, X, w


def data(bg, w=None, groups=None):
    from distributedkernelshap_b200.data import DenseData
    groups = groups or [[k] for k in range(bg.shape[1])]
    return DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, w)


def engine(fn, bg, link, w=None, groups=None, **kw):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    return GpuKernelExplainer(fn, data(bg, w, groups), link=link, seed=7, **kw)


def oracle(fn, bg, link, w=None, groups=None):
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    groups = groups or [[k] for k in range(bg.shape[1])]
    return KernelExplainerOracle(fn, DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, w), link=link)


def as_list(phi):
    return phi if isinstance(phi, list) else [phi]


def own_plans(eng, X, ns="auto"):
    M, _ = eng.varying(X)
    return lambda i: None if M[i] < 2 else (eng.shared_plan(int(M[i]), ns).dense(), eng.shared_plan(int(M[i]), ns).weights)


def compare(got, orc, X, plans, tol, l1_reg=False, nsamples="auto"):
    got = as_list(got)
    worst = 0.0
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for i in range(X.shape[0]):
            want = orc.explain(X[i:i + 1], plan=plans(i), l1_reg=l1_reg, nsamples=nsamples)
            want = want.reshape(want.shape[0], -1)
            for c in range(want.shape[1]):
                e = rel_err(got[c][i], want[:, c])
                worst = max(worst, e)
                assert e < tol, (i, c, e)
    return worst


def tol(kind):
    return KNN_TOL if kind in ("clf2_five", "clf3_pass", "reg_pass") else TOL     # the ones with a neighbour member


@pytest.mark.parametrize("kind,link", CASES)
def test_parity_with_the_oracle(kind, link):
    st, fn = fitted(kind)
    bg, X, _ = problem(11, N=16, n=4)
    eng = engine(fn, bg, link)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "stacking"
    M, _ = eng.varying(X)
    assert {int(m) for m in M} == {4, 5}                     # full and partial varying sets in one call
    worst = compare(got, oracle(fn, bg, link), X, own_plans(eng, X), tol(kind))
    print(f"{kind} {link}: max|d|/max|phi| = {worst:.2e}")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want_fx = np.asarray(fn(X), dtype=np.float64).reshape(X.shape[0], -1)
    np.testing.assert_allclose(eng.predict(X), want_fx, rtol=1e-10, atol=1e-12)


def test_decision_function_identity_link():
    st, fn = fitted("clf3_pass", method="decision_function")
    bg, X, _ = problem(12, N=10, n=3)
    eng = engine(fn, bg, "identity")
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "stacking"
    compare(got, oracle(fn, bg, "identity"), X, own_plans(eng, X), KNN_TOL)


@pytest.mark.parametrize("plan_mode", ["per_instance", "caller"])
def test_plan_sources(plan_mode):
    st, fn = fitted("clf2_five")
    bg, X, _ = problem(5, N=12, n=3, partial=plan_mode == "per_instance")
    if plan_mode == "per_instance":
        eng = engine(fn, bg, "logit", plan_mode="per_instance")
        got = eng.shap_values(X, l1_reg=False)
        assert eng.last_path()["general"] == "stacking"
        zb, wts = eng.instance_plans()
        M, _ = eng.varying(X)
        from distributedkernelshap_b200.plan import resolve_nsamples

        def plans(i):
            S, _ = resolve_nsamples(int(M[i]), "auto")
            k = np.arange(int(M[i]))
            return ((zb[i, :S, None] >> k.astype(np.uint64)) & np.uint64(1)).astype(np.uint8), wts[i, :S]
        compare(got, oracle(fn, bg, "logit"), X, plans, KNN_TOL)
        return
    rng = np.random.default_rng(0)
    plans = []
    for i in range(3):
        Z = rng.integers(0, 2, size=(24, 5)).astype(np.uint8)
        Z[0], Z[1] = 0, 1
        Z[2:7] = np.eye(5, dtype=np.uint8)
        plans.append((Z, rng.uniform(0.1, 1.0, 24)))
    eng = engine(fn, bg, "logit")
    got = eng.shap_values(X, l1_reg=False, nsamples=24, plans=plans)
    assert eng.last_path()["general"] == "stacking"
    compare(got, oracle(fn, bg, "logit"), X, lambda i: plans[i], KNN_TOL, nsamples=24)


def test_weighted_background_and_grouped_columns():
    st, fn = fitted("clf3_pass")
    bg, X, w = problem(5, N=14, n=4, weights=True)
    groups = [[0, 3], [1], [2, 4]]
    eng = engine(fn, bg, "identity", w=w, groups=groups)
    got = eng.shap_values(X, l1_reg=False)
    compare(got, oracle(fn, bg, "identity", w=w, groups=groups), X, own_plans(eng, X), KNN_TOL)


@pytest.mark.parametrize("l1_reg", ["aic", "bic", "num_features(2)"])
def test_l1_selection(l1_reg):
    members = lambda: [("rf", RandomForestClassifier(4, max_depth=3, random_state=0)), ("mlp", _mlp()),  # noqa: E731
                       ("lr", LogisticRegression())]
    MODELS["wide"] = (members, 2, {"passthrough": True})
    try:
        st, fn = fitted("wide", d=14, n=400)
    finally:
        del MODELS["wide"]
    bg, X, _ = problem(8, N=8, n=3, d=14)
    eng = engine(fn, bg, "logit")
    got = eng.shap_values(X, l1_reg=l1_reg)
    path = eng.last_path()
    assert path["general"] in ("stacking", "simt") and path["general_l1"] == 1, path
    compare(got, oracle(fn, bg, "logit"), X, own_plans(eng, X), L1_TOL, l1_reg=l1_reg)


def test_zero_one_and_two_varying_groups():
    st, fn = fitted("clf3_pass")
    bg, _ = raw(4, 10)
    bg[:] = bg[0]                                # every column constant over the background
    X = np.repeat(bg[:1], 3, axis=0)
    X[1, 2] += 1.0                               # M = 1
    X[2, [0, 4]] -= 0.5                          # M = 2
    eng = engine(fn, bg, "identity")
    M, _ = eng.varying(X)
    assert list(M) == [0, 1, 2]
    got = eng.shap_values(X, l1_reg=False)
    assert np.all(np.stack(got)[:, 0] == 0)
    compare(got, oracle(fn, bg, "identity"), X, own_plans(eng, X), KNN_TOL)


def test_sixty_four_groups():
    rng = np.random.default_rng(1)
    Xt = rng.normal(size=(300, 64))
    y = (Xt[:, 1] - Xt[:, 62] > 0).astype(int)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        st = StackingClassifier([("dt", DecisionTreeClassifier(max_depth=5, random_state=0)), ("mlp", _mlp())],
                                passthrough=True).fit(Xt, y)
    bg = Xt[:6].copy()
    X = Xt[10:12].copy()
    eng = engine(st.predict_proba, bg, "identity")
    got = eng.shap_values(X, l1_reg=False, nsamples=200)
    assert list(eng.varying(X)[0]) == [64, 64]
    compare(got, oracle(st.predict_proba, bg, "identity"), X, own_plans(eng, X, 200), TOL, nsamples=200)


def test_batch_instances_bit_identical_to_the_instance_alone():
    st, fn = fitted("clf3_pass")
    bg, _ = raw(9, 8)
    X, _ = raw(10, 3000)                         # more than three instances per CTA of every launch
    eng = engine(fn, bg, "logit")
    got = np.stack(eng.shap_values(X, l1_reg=False, nsamples=32))
    for i in (0, 1777, 2999):
        alone = np.stack(eng.shap_values(X[i:i + 1], l1_reg=False, nsamples=32))
        np.testing.assert_array_equal(got[:, i:i + 1], alone)


def test_background_chunks_bit_identical(monkeypatch):
    from distributedkernelshap_b200 import engine as engine_mod
    st, fn = fitted("clf2_five")
    bg, X, w = problem(13, N=11, n=6, weights=True)
    want = np.stack(engine(fn, bg, "logit", w=w).shap_values(X, l1_reg=False, nsamples=40))
    # a budget below one background row's workspace: one chunk per background row
    monkeypatch.setattr(engine_mod, "MAX_STACKING_BYTES_PER_CALL", 1)
    eng = engine(fn, bg, "logit", w=w)
    eng.shap_values(X, l1_reg=False, nsamples=40)          # the shared plans are built on the first call
    before = eng.kernel_launches()
    got = np.stack(eng.shap_values(X, l1_reg=False, nsamples=40))
    K = len(eng.spec.members)
    # stage 1 (the varying groups, K member predictions, f(x)), then per chunk K members and a reduction, and the tail
    assert eng.kernel_launches() - before == (K + 2) + 11 * (K + 1) + 1
    np.testing.assert_array_equal(got, want)


def test_device_run_graph_replay_and_launch_count():
    import torch
    st, fn = fitted("clf2_svc_df")
    bg, X, _ = problem(41, N=20, n=16)
    eng = engine(fn, bg, "identity")
    want = np.stack(as_list(eng.shap_values(X, nsamples=24, l1_reg=False)))
    K = len(eng.spec.members)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(X).cuda()
        phi = torch.zeros((2, 16, 5), dtype=torch.float64, device="cuda")
        eng.explain_device(X_dev.data_ptr(), 16, phi.data_ptr(), nsamples=24)
        eng.check_status()
        before = eng.kernel_launches()
        eng.explain_device(X_dev.data_ptr(), 16, phi.data_ptr(), nsamples=24)
        # stage 1 (the varying groups, K member predictions, f(x)) and the explain (one chunk: K members and the
        # reduction, then the tail)
        assert eng.kernel_launches() - before == (K + 2) + (K + 1) + 1
        for _ in range(3):
            eng.explain_device(X_dev.data_ptr(), 16, phi.data_ptr(), nsamples=24)
        eng.check_status()
        assert eng.graph_launches() >= 1
        assert eng.last_path()["general"] == "stacking"
        np.testing.assert_array_equal(phi.cpu().numpy(), want)
    eng.set_stream(0)


def test_raw_values_members_refuse():
    st, fn = fitted("clf2_five")                  # a kernel-machine member refuses NaN
    bg, X, _ = problem(2, N=10, n=4)
    eng = engine(fn, bg, "identity")
    X[2, 3] = np.nan
    with pytest.raises(ValueError, match="instance 2"):
        eng.shap_values(X, l1_reg=False)
    with pytest.raises(ValueError, match="row 2"):
        eng.predict(X)


def _outer_pipeline():
    rng = np.random.default_rng(6)
    X = np.column_stack([rng.normal(size=(300, 3)), rng.integers(0, 3, (300, 2)).astype(float)])
    y = (X[:, 0] - X[:, 1] + (X[:, 3] == 1) > 0).astype(int)
    ct = ColumnTransformer([("n", StandardScaler(), [0, 1, 2]), ("c", OneHotEncoder(handle_unknown="ignore"), [3, 4])])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe = make_pipeline(ct, StackingClassifier([("lr", LogisticRegression()),
                                                     ("rf", RandomForestClassifier(5, max_depth=4, random_state=0)),
                                                     ("mlp", _mlp())], passthrough=True)).fit(X, y)
    return pipe, X


def test_outer_pipeline_bit_identical_to_the_encoded_reading():
    pipe, X = _outer_pipeline()
    bg, Xi = X[:12], X[200:206]
    eng = engine(pipe.predict_proba, bg, "logit")
    assert eng.encoding is not None and eng.spec.n_features == 5
    enc = eng.encoding
    groups = [[int(e) for e in np.nonzero(enc.sources == c)[0]] for c in range(enc.D)]
    dense = lambda A: np.asarray(pipe[:-1].transform(A), dtype=np.float64)   # noqa: E731
    ref = engine(pipe[-1].predict_proba, dense(bg), "logit", groups=groups)
    got = np.stack(eng.shap_values(Xi, l1_reg=False, nsamples=40))
    want = np.stack(ref.shap_values(dense(Xi), l1_reg=False, nsamples=40))
    assert eng.last_path()["general"] == ref.last_path()["general"] == "stacking"
    np.testing.assert_array_equal(got, want)
    compare(list(got), oracle(pipe.predict_proba, bg, "logit"), Xi, own_plans(eng, Xi, 40), TOL, nsamples=40)


def test_kernel_shap_default_kwargs():
    from distributedkernelshap_b200.data import convert_to_link
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    st, _ = fitted("clf2_five")
    bg, X, _ = problem(23, N=30, n=6, partial=False)
    ks = KernelShap(st.predict_proba, link="logit", seed=0)
    ks.fit(bg)
    exp = ks.explain(X, silent=True)
    assert ks._explainer.last_path()["general"] in ("stacking", "simt")
    sv = exp.shap_values
    assert len(sv) == 2 and sv[0].shape == (6, 5)
    fx = convert_to_link("logit").f(st.predict_proba(X))
    for c in range(2):
        np.testing.assert_allclose(sv[c].sum(1), fx[:, c] - exp.expected_value[c], rtol=1e-8, atol=1e-8)


def test_all_linear_regressor_takes_the_linear_route():
    from distributedkernelshap_b200.predictors import LinearModelSpec
    X, s = raw(3, 300)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        st = StackingRegressor([("a", Ridge(alpha=2.0)), ("b", LinearRegression())], final_estimator=LinearRegression(),
                               passthrough=True).fit(X, s)
    bg, Xi, _ = problem(4, N=12, n=4)
    eng = engine(st.predict, bg, "identity")
    assert isinstance(eng.spec, LinearModelSpec)
    got = eng.shap_values(Xi, l1_reg=False)
    assert eng.last_path()["general"] != "stacking"
    compare(got, oracle(st.predict, bg, "identity"), Xi, own_plans(eng, Xi), TOL)


def test_device_memory_returns_after_destroy_and_refit():
    from distributedkernelshap_b200 import _cabi
    import ctypes
    lib = _cabi.load()

    def live():
        n = ctypes.c_int64()
        _cabi.check(lib.dks_live_allocations(ctypes.byref(n)))
        return n.value
    st, fn = fitted("clf3_pass")
    bg, X, _ = problem(31, N=10, n=5)
    start = live()
    eng = engine(fn, bg, "logit")
    eng.shap_values(X, l1_reg=False)
    _cabi.check(lib.dks_fit(eng._ctx))           # a refit frees what the previous fit built
    eng.shap_values(X, l1_reg=False)
    eng.close()
    assert live() == start


def test_refusals():
    from distributedkernelshap_b200._cabi import DksError
    st, fn = fitted("clf3_pass")
    bg, X, _ = problem(1, N=8, n=2)
    for kernel in ("tcgen05", "shared"):
        eng = engine(fn, bg, "identity", kernel=kernel)
        with pytest.raises(DksError, match="stacking ensembles run on the stacking kernels only"):
            eng.shap_values(X, l1_reg=False)
    rng = np.random.default_rng(0)
    Xw = rng.normal(size=(100, 65))
    wide = StackingClassifier([("dt", DecisionTreeClassifier(max_depth=3)), ("lr", LogisticRegression())]).fit(
        Xw, (Xw[:, 0] > 0).astype(int))
    with pytest.raises(NotImplementedError, match="stacking ensembles are explained up to 64 groups"):
        engine(wide.predict_proba, Xw[:5], "identity")
