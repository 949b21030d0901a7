"""Kernel machines, MLPs and k-nearest-neighbour models behind per-column preprocessing pipelines, explained in raw
feature space (the device replays ``pipe[:-1].transform`` and the family's own kernels read the encoded rows): parity
with the oracle calling the real pipeline on the masked raw batches, phi bit-identical to the same fitted estimator
explained on the encoded columns, every plan source and entry point, the raw values the pipeline refuses, and the
refusals."""
import warnings

import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")
from sklearn.calibration import CalibratedClassifierCV  # noqa: E402
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.impute import SimpleImputer  # noqa: E402
from sklearn.kernel_ridge import KernelRidge  # noqa: E402
from sklearn.neighbors import KNeighborsClassifier, KNeighborsRegressor  # noqa: E402
from sklearn.neural_network import MLPClassifier, MLPRegressor  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import (KBinsDiscretizer, MinMaxScaler, OneHotEncoder, OrdinalEncoder,  # noqa: E402
                                   PolynomialFeatures, StandardScaler)
from sklearn.svm import SVC  # noqa: E402

TOL = 1e-9              # kernel machines and MLPs, float64 end to end
KNN_TOL = 1e-8
L1_TOL = 1e-5           # the l1 moments go through the 2^-40 fixed point


def raw(seed, n, nan=False):
    """Raw rows: three numeric columns (the third with NaN if asked), then two integer-coded categorical columns."""
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


PRE = {
    "std_onehot": lambda: ct(("n", StandardScaler(), [0, 1, 2]), ("c", OneHotEncoder(handle_unknown="ignore"), [3, 4])),
    "imputer_onehot_drop": lambda: ct(("i", make_pipeline(SimpleImputer(add_indicator=True), StandardScaler()),
                                       [0, 1, 2]),
                                      ("c", OneHotEncoder(drop="first", handle_unknown="ignore"), [3, 4])),
    "clip_ordinal_passthrough": lambda: ct(("n", MinMaxScaler(clip=True), [0, 1]),
                                           ("c", OrdinalEncoder(handle_unknown="use_encoded_value", unknown_value=-1),
                                            [3, 4]), remainder="passthrough"),
    "kbins_infrequent_sparse": lambda: ct(("n", StandardScaler(), [0, 2]),
                                          ("k", KBinsDiscretizer(4, encode="onehot", strategy="uniform"), [1]),
                                          ("c", OneHotEncoder(min_frequency=20, handle_unknown="infrequent_if_exist"), [3]),
                                          ("o", OneHotEncoder(handle_unknown="ignore"), [4]), sparse_threshold=1.0),
}
MODELS = {   # (estimator, method, pipeline, NaN in the data, classes (0: regression) or -targets, links, family)
    "svc": (lambda: SVC(gamma=0.3), "decision_function", "std_onehot", False, 2, ("identity",), "kmach"),
    "krr3": (lambda: KernelRidge(kernel="rbf", alpha=0.5, gamma=0.2), "predict", "clip_ordinal_passthrough", False, -3,
             ("identity",), "kmach"),
    "cal_svc": (lambda: CalibratedClassifierCV(SVC(gamma=0.2), cv=3), "predict_proba", "kbins_infrequent_sparse", False,
                2, ("identity", "logit"), "kmach"),
    "mlp2": (lambda: MLPClassifier(hidden_layer_sizes=(16,), max_iter=300, random_state=0), "predict_proba", "imputer_onehot_drop", True,
             2, ("identity", "logit"), "mlp"),
    "mlp3": (lambda: MLPClassifier(hidden_layer_sizes=(12, 8), activation="tanh", max_iter=300, random_state=0), "predict_proba",
             "std_onehot", False, 3, ("logit",), "mlp"),
    "mlp_reg": (lambda: MLPRegressor(hidden_layer_sizes=(16,), max_iter=300, random_state=0), "predict", "kbins_infrequent_sparse", False, 0,
                ("identity",), "mlp"),
    "knn_clf": (lambda: KNeighborsClassifier(5), "predict_proba", "std_onehot", False, 2, ("identity",), "knn"),
    "knn_clf_dist": (lambda: KNeighborsClassifier(6, weights="distance"), "predict_proba", "clip_ordinal_passthrough",
                     False, 3, ("identity",), "knn"),
    "knn_reg": (lambda: KNeighborsRegressor(4), "predict", "kbins_infrequent_sparse", False, 0, ("identity",), "knn"),
    "knn_reg_dist": (lambda: KNeighborsRegressor(5, weights="distance"), "predict", "imputer_onehot_drop", True, 0,
                     ("identity",), "knn"),
}
CASES = [(m, link) for m in MODELS for link in MODELS[m][5]]


def fitted(kind, seed=0, n=300):
    make, method, pre, nan, classes, _, _ = MODELS[kind]
    X, s = raw(seed, n, nan=nan)
    if classes > 0:
        target = np.digitize(s, np.quantile(s, np.linspace(0, 1, classes + 1)[1:-1]))
    elif classes < 0:
        target = np.stack([s, np.sin(s), 0.5 * s * s], axis=1)[:, :-classes]
    else:
        target = s
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe = make_pipeline(PRE[pre](), make()).fit(X, target)
    return pipe, getattr(pipe, method)


def problem(kind, seed, N, n, partial=True, weights=False):
    nan = MODELS[kind][3]
    bg, _ = raw(seed, N, nan=nan)
    X, _ = raw(seed + 1, n, nan=nan)
    if partial:                                  # x takes the background's constant value of column 1 on every other row
        bg[:, 1] = 0.75
        X[::2, 1] = 0.75
    w = None
    if weights:
        w = np.random.default_rng(seed).uniform(0.1, 1.0, N)
        w[1] = 0.0                               # a zero-weight row is skipped, not divided by
    return bg, X, w


def dense(pipe, X):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = pipe[:-1].transform(X)
    return np.asarray(out.toarray() if hasattr(out, "toarray") else out, dtype=np.float64)


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
    return KNN_TOL if MODELS[kind][6] == "knn" else TOL


@pytest.mark.parametrize("kind,link", CASES)
def test_parity_with_the_oracle(kind, link):
    pipe, fn = fitted(kind)
    bg, X, _ = problem(kind, 11, N=16, n=4)
    eng = engine(fn, bg, link)
    assert eng.encoding is not None and eng.spec.n_features == 5
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == MODELS[kind][6]
    M, _ = eng.varying(X)
    assert {int(m) for m in M} == {4, 5}                     # full and partial varying sets in one call
    worst = compare(got, oracle(fn, bg, link), X, own_plans(eng, X), tol(kind))
    print(f"{kind} {link}: max|d|/max|phi| = {worst:.2e}")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want_fx = np.asarray(fn(X), dtype=np.float64).reshape(X.shape[0], -1)
    np.testing.assert_allclose(eng.predict(X), want_fx, rtol=1e-10, atol=1e-12)


def test_calibrated_single_fold_with_its_own_preprocessing():
    X, s = raw(0, 300)
    y = (s > np.median(s)).astype(int)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cal = CalibratedClassifierCV(make_pipeline(PRE["std_onehot"](), SVC(gamma=0.3)), ensemble=False).fit(X, y)
    bg, Xe, _ = problem("svc", 3, N=14, n=4)
    eng = engine(cal.predict_proba, bg, "logit")
    assert eng.encoding is not None
    got = eng.shap_values(Xe, l1_reg=False)
    assert eng.last_path()["general"] == "kmach"
    compare(got, oracle(cal.predict_proba, bg, "logit"), Xe, own_plans(eng, Xe), TOL)


@pytest.mark.parametrize("kind", ["svc", "mlp2", "knn_reg_dist"])
def test_weighted_background_and_grouped_columns(kind):
    pipe, fn = fitted(kind)
    bg, X, w = problem(kind, 5, N=14, n=4, weights=True)
    link = MODELS[kind][5][-1]
    groups = [[0, 3], [1], [2, 4]]
    eng = engine(fn, bg, link, w=w, groups=groups)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == MODELS[kind][6]
    compare(got, oracle(fn, bg, link, w=w, groups=groups), X, own_plans(eng, X), tol(kind))


def _encoded_reading(pipe, method, enc, bg, X, link, **kw):
    """The pipeline's own fitted estimator explained on pipe[:-1].transform, one group per raw column's encoded block."""
    groups = [[int(e) for e in np.nonzero(enc.sources == c)[0]] for c in range(enc.D)]
    return engine(getattr(pipe[-1], method), dense(pipe, bg), link, groups=groups, **kw), dense(pipe, X)


@pytest.mark.parametrize("plan_mode", ["shared", "per_instance"])
@pytest.mark.parametrize("kind", ["svc", "cal_svc", "mlp2", "mlp_reg", "knn_clf", "knn_reg_dist"])
def test_same_phi_as_the_encoded_reading(kind, plan_mode):
    pipe, fn = fitted(kind)
    # binning can map x's raw column 1 into the bin of the background's constant 0.75: the raw reading sees that group
    # vary where the encoded one does not (DESIGN.md §5.0.16), so those pipelines take full varying sets here
    bg, X, _ = problem(kind, 13, N=12, n=6, partial=MODELS[kind][2] != "kbins_infrequent_sparse")
    link = MODELS[kind][5][-1]
    eng = engine(fn, bg, link, plan_mode=plan_mode)
    ref, Xe = _encoded_reading(pipe, MODELS[kind][1], eng.encoding, bg, X, link, plan_mode=plan_mode)
    np.testing.assert_array_equal(eng.varying(X)[0], ref.varying(Xe)[0])
    got = np.stack(as_list(eng.shap_values(X, l1_reg=False, nsamples=24)))
    want = np.stack(as_list(ref.shap_values(Xe, l1_reg=False, nsamples=24)))
    assert eng.last_path()["general"] == ref.last_path()["general"] == MODELS[kind][6]
    assert np.abs(got - want).max() == 0
    np.testing.assert_array_equal(np.atleast_1d(eng.expected_value), np.atleast_1d(ref.expected_value))


@pytest.mark.parametrize("kind", ["krr3", "mlp3", "knn_clf_dist"])
def test_caller_supplied_plans(kind):
    pipe, fn = fitted(kind)
    bg, X, _ = problem(kind, 8, N=10, n=3, partial=False)
    rng = np.random.default_rng(0)
    plans = []
    for i in range(3):
        Z = rng.integers(0, 2, size=(24, 5)).astype(np.uint8)
        Z[0], Z[1] = 0, 1
        Z[2:7] = np.eye(5, dtype=np.uint8)
        plans.append((Z, rng.uniform(0.1, 1.0, 24)))
    link = MODELS[kind][5][-1]
    eng = engine(fn, bg, link)
    got = eng.shap_values(X, l1_reg=False, nsamples=24, plans=plans)
    assert eng.last_path()["general"] == MODELS[kind][6]
    compare(got, oracle(fn, bg, link), X, lambda i: plans[i], tol(kind), nsamples=24)


def _wide(make, seed=0):
    """14 raw columns (12 numeric, 2 categorical): l1_reg='auto' selects at nsamples='auto'."""
    rng = np.random.default_rng(seed)
    X = np.column_stack([rng.normal(size=(420, 12)), rng.integers(0, 3, (420, 2)).astype(float)])
    y = (X[:, 0] - X[:, 3] + (X[:, 12] == 1) > 0).astype(int)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe = make_pipeline(ct(("n", StandardScaler(), list(range(12))),
                                ("c", OneHotEncoder(handle_unknown="ignore"), [12, 13])), make()).fit(X[:400], y[:400])
    return pipe, X[400:408], X[408:411]


@pytest.mark.parametrize("l1_reg", ["auto", "num_features(4)"])
@pytest.mark.parametrize("family", ["kmach", "mlp"])
def test_l1_selection(family, l1_reg):
    make = (lambda: SVC(gamma=0.1)) if family == "kmach" else (lambda: MLPClassifier(hidden_layer_sizes=(8,), max_iter=200, random_state=0))
    pipe, bg, X = _wide(make)
    fn = pipe.decision_function if family == "kmach" else pipe.predict_proba
    link = "identity" if family == "kmach" else "logit"
    eng = engine(fn, bg, link)
    got = eng.shap_values(X, l1_reg=l1_reg)
    path = eng.last_path()
    assert path["general"] in (family, "simt") and path["general_l1"] == 1, path
    compare(got, oracle(fn, bg, link), X, own_plans(eng, X), L1_TOL, l1_reg=l1_reg)


def test_row_blocks_give_the_same_phi(monkeypatch):
    from distributedkernelshap_b200 import engine as engine_mod
    pipe, fn = fitted("mlp2")
    bg, X, _ = problem("mlp2", 17, N=12, n=11)
    eng = engine(fn, bg, "logit")
    want = np.stack(eng.shap_values(X, l1_reg=False))
    monkeypatch.setattr(engine_mod, "MAX_ENCODED_BYTES_PER_CALL", 8 * eng.encoding.E * 3)   # 3 rows per call
    assert eng._rows_per_call() == 3
    got = np.stack(eng.shap_values(X, l1_reg=False))
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("kind", ["svc", "knn_clf"])
def test_graph_replay_is_bit_identical_to_the_host_path(kind):
    import torch
    pipe, fn = fitted(kind)
    bg, X, _ = problem(kind, 41, N=20, n=16)
    eng = engine(fn, bg, "identity")
    want = np.stack(as_list(eng.shap_values(X, nsamples=24, l1_reg=False)))
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(X).cuda()
        phi = torch.zeros((want.shape[0], 16, 5), dtype=torch.float64, device="cuda")
        for _ in range(4):
            eng.explain_device(X_dev.data_ptr(), 16, phi.data_ptr(), nsamples=24)
        eng.check_status()
        assert eng.graph_launches() >= 1
        assert eng.last_path()["general"] == MODELS[kind][6]
        np.testing.assert_array_equal(phi.cpu().numpy(), want)
    eng.set_stream(0)


def test_kernel_shap_default_kwargs():
    from distributedkernelshap_b200.data import convert_to_link
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    pipe, _ = fitted("mlp2")
    bg, X, _ = problem("mlp2", 23, N=30, n=6, partial=False)
    ks = KernelShap(pipe.predict_proba, link="logit", seed=0)
    ks.fit(bg)
    exp = ks.explain(X, silent=True)                     # default kwargs: nsamples='auto', l1_reg='auto'
    assert ks._explainer.last_path()["general"] in ("mlp", "simt")
    sv = exp.shap_values
    assert len(sv) == 2 and sv[0].shape == (6, 5)        # one value per raw column
    fx = convert_to_link("logit").f(pipe.predict_proba(X))
    for c in range(2):
        np.testing.assert_allclose(sv[c].sum(1), fx[:, c] - exp.expected_value[c], rtol=1e-8, atol=1e-8)


def test_raw_values_the_pipeline_refuses():
    # a NaN the imputer fills is explained (its parity is in test_parity_with_the_oracle[mlp2-*])
    pipe, fn = fitted("mlp2")
    bg, X, _ = problem("mlp2", 2, N=10, n=4)
    X[1, 2] = np.nan
    eng = engine(fn, bg, "logit")
    assert np.isfinite(np.stack(eng.shap_values(X, l1_reg=False))).all()
    # a NaN without an imputer, an unknown category under 'error', and +-inf anywhere a step or the estimator reads it
    Xr, s = raw(0, 300)
    y = (s > np.median(s)).astype(int)
    err = make_pipeline(ct(("n", StandardScaler(), [0, 1]), ("c", OneHotEncoder(handle_unknown="error"), [3, 4]),
                           remainder="passthrough"), SVC()).fit(Xr, y)
    drop = make_pipeline(ct(("n", StandardScaler(), [0, 1]), ("c", OneHotEncoder(handle_unknown="ignore"), [3, 4])),
                         KNeighborsClassifier()).fit(Xr, y)
    bg = Xr[:10].copy()
    for fn in (err.decision_function, drop.predict_proba):
        eng = engine(fn, bg, "identity")
        cases = [(2, np.inf), (0, -np.inf), (3, 9.0)] + ([(2, np.nan), (4, 7.0)] if fn == err.decision_function else [])
        for col, v in cases:
            Xi = Xr[10:14].copy()
            Xi[2, col] = v
            sk_raises = True
            try:
                fn(Xi)
                sk_raises = False
            except ValueError:
                pass
            if sk_raises:
                with pytest.raises(ValueError, match="instance 2"):
                    eng.shap_values(Xi, l1_reg=False)
                with pytest.raises(ValueError, match="row 2"):
                    eng.predict(Xi)
            else:
                assert np.isfinite(np.stack(as_list(eng.shap_values(Xi, l1_reg=False)))).all()
                np.testing.assert_allclose(eng.predict(Xi), np.asarray(fn(Xi)).reshape(4, -1), rtol=1e-10, atol=1e-12)
    bad_bg = bg.copy()
    bad_bg[4, 3] = 9.0
    with pytest.raises(ValueError, match="background row 4"):
        engine(err.decision_function, bad_bg, "identity")


def test_knn_background_from_the_training_rows():
    """A background row drawn from the training rows is at distance exactly 0 from its encoded training row (the
    encoding is bit-exact), and on mostly categorical data the fit check's tie warning fires."""
    import logging
    rng = np.random.default_rng(4)
    X = np.column_stack([rng.normal(size=200), rng.integers(0, 3, (200, 4)).astype(float)])
    y = (X[:, 0] + X[:, 1] > 1).astype(int)
    pipe = make_pipeline(ct(("n", StandardScaler(), [0]), ("c", OneHotEncoder(handle_unknown="ignore"), [1, 2, 3, 4])),
                         KNeighborsClassifier(5, weights="distance")).fit(X, y)
    eng = engine(pipe.predict_proba, X[:12], "identity")
    t, exact = eng.spec.statistic(eng.encode(X[:12]))
    assert exact[np.arange(12), np.arange(12)].all() and (t[np.arange(12), np.arange(12)] == 0).all()
    np.testing.assert_allclose(eng.predict(X[:12]), pipe.predict_proba(X[:12]), rtol=0, atol=1e-15)
    cat = make_pipeline(ct(("c", OneHotEncoder(handle_unknown="ignore"), [1, 2, 3, 4])), KNeighborsClassifier(5))
    cat.fit(X, y)
    logger = logging.getLogger("distributedkernelshap_b200.engine")
    seen = []
    handler = logging.Handler()
    handler.emit = lambda record: seen.append(record.getMessage())
    logger.addHandler(handler)
    try:
        engine(cat.predict_proba, X[20:60], "identity")
    finally:
        logger.removeHandler(handler)
    assert any("equidistant" in m for m in seen), seen


def test_refusals():
    Xr, s = raw(0, 300)
    y = (s > np.median(s)).astype(int)
    bg = Xr[:10]
    poly = make_pipeline(ct(("p", PolynomialFeatures(2), [0, 1])), SVC()).fit(Xr, y)
    with pytest.raises(NotImplementedError, match="PolynomialFeatures.*OneHotEncoder|PolynomialFeatures"):
        engine(poly.decision_function, bg, "identity")
    folds = CalibratedClassifierCV(make_pipeline(PRE["std_onehot"](), SVC()), cv=3).fit(Xr, y)
    with pytest.raises(NotImplementedError, match="in front of the calibrator"):
        engine(folds.predict_proba, bg, "identity")
    pipe, fn = fitted("mlp2")
    eng = engine(fn, bg, "logit", kernel="simt")
    from distributedkernelshap_b200._cabi import DksError
    for kernel in ("tcgen05", "shared"):
        eng.set_kernel(kernel)
        with pytest.raises(DksError, match="MLP"):
            eng.shap_values(Xr[10:12], l1_reg=False)
