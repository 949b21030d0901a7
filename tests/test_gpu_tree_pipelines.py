"""Tree models behind per-column preprocessing pipelines, explained in raw feature space on the tree route (the device
replays ``pipe[:-1].transform`` with ``encode_kernel``): parity with the oracle calling the real pipeline on the masked
raw batches, phi bit-identical to the same fitted trees explained on the encoded columns, the device encoding bit for
bit equal to scikit-learn's on adversarial values, every plan source and entry point, and the refusals."""
import warnings

import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.ensemble import (ExtraTreesRegressor, GradientBoostingClassifier, HistGradientBoostingClassifier,  # noqa: E402
                              HistGradientBoostingRegressor, RandomForestClassifier, VotingClassifier)
from sklearn.impute import SimpleImputer  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import (KBinsDiscretizer, MaxAbsScaler, MinMaxScaler, OneHotEncoder,  # noqa: E402
                                   OrdinalEncoder, PolynomialFeatures, RobustScaler, StandardScaler)
from sklearn.tree import DecisionTreeClassifier  # noqa: E402

TOL = 1e-9              # float64 end to end without selection
L1_TOL = 1e-5           # the l1 moments go through the 2^-40 fixed point


def raw(seed, n, P_num=3, nan=True, nan_cat=False, y_classes=2):
    """Raw rows: P_num numeric columns (the third with NaN), then two integer-coded categorical columns."""
    rng = np.random.default_rng(seed)
    X = np.empty((n, P_num + 2))
    X[:, :P_num] = rng.normal(size=(n, P_num)) * np.linspace(1.0, 4.0, P_num) + np.arange(P_num)
    if nan:
        X[rng.random(n) < 0.1, 2] = np.nan
    X[:, P_num] = rng.choice([0.0, 1.0, 2.0, 5.0], n, p=[0.4, 0.3, 0.27, 0.03])
    X[:, P_num + 1] = rng.integers(0, 4, n).astype(float)
    if nan_cat:
        X[rng.random(n) < 0.08, P_num + 1] = np.nan
    s = X[:, 0] - 0.5 * X[:, 1] + (X[:, P_num] == 1) + 0.3 * np.nan_to_num(X[:, 2])
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, y_classes + 1)[1:-1]))
    return X, y, s


def ct(*parts, remainder="drop"):
    return ColumnTransformer(list(parts), remainder=remainder)


PRE = {
    "standard_onehot": lambda: ct(("n", StandardScaler(), [0, 1]), ("c", OneHotEncoder(handle_unknown="ignore"), [3, 4]),
                                  remainder="passthrough"),
    "minmax_clip_ordinal": lambda: ct(("n", MinMaxScaler(clip=True), slice(0, 2)), ("c", OrdinalEncoder(), [3, 4]),
                                      ("p", "passthrough", [2])),
    "robust_maxabs_kbins": lambda: ct(("a", RobustScaler(), [0]), ("b", MaxAbsScaler(), [2]),
                                      ("k", KBinsDiscretizer(4, encode="onehot", strategy="uniform"), [1]),
                                      ("c", "passthrough", np.array([False, False, False, True, True]))),
    "imputer_onehot_drop": lambda: ct(("i", make_pipeline(SimpleImputer(add_indicator=True), StandardScaler()), [0, 1, 2]),
                                      ("c", OneHotEncoder(drop="first", handle_unknown="ignore"), [3, 4])),
    "infrequent_ordinal_missing": lambda: ct(("n", StandardScaler(), [0, 1, 2]),
                                             ("c", OneHotEncoder(min_frequency=20, handle_unknown="infrequent_if_exist"),
                                              [3]),
                                             ("o", OrdinalEncoder(handle_unknown="use_encoded_value", unknown_value=-1,
                                                                  encoded_missing_value=-2), [4])),
    "standard_no_mean_passthrough": lambda: ct(("n", StandardScaler(with_mean=False), [0, 1]),
                                               remainder="passthrough"),
}
MODELS = {   # (model, method, pipeline, data has NaN in numeric / categorical columns, classes, links)
    "dt": (lambda: DecisionTreeClassifier(max_depth=6, random_state=0), "predict_proba", "standard_onehot", True, False,
           2, ("identity",)),
    "rf": (lambda: RandomForestClassifier(12, max_depth=6, random_state=0), "predict_proba", "minmax_clip_ordinal", True,
           False, 3, ("identity",)),
    "et_reg": (lambda: ExtraTreesRegressor(10, max_depth=6, random_state=0), "predict", "robust_maxabs_kbins", True,
               False, 0, ("identity",)),
    "gb2": (lambda: GradientBoostingClassifier(n_estimators=25, max_depth=3, random_state=0), "predict_proba",
            "imputer_onehot_drop", True, False, 2, ("identity", "logit")),
    "gb4": (lambda: GradientBoostingClassifier(n_estimators=10, max_depth=2, random_state=0), "predict_proba",
            "robust_maxabs_kbins", False, False, 4, ("identity", "logit")),
    "hgb": (lambda: HistGradientBoostingClassifier(max_iter=20, random_state=0), "predict_proba",
            "infrequent_ordinal_missing", True, True, 2, ("identity", "logit")),
    "hgb_poisson": (lambda: HistGradientBoostingRegressor(max_iter=15, loss="poisson", random_state=0), "predict",
                    "standard_no_mean_passthrough", True, False, 0, ("identity",)),
}
CASES = [(m, link) for m in MODELS for link in MODELS[m][-1]]


def fitted(kind, seed=0, n=400):
    make, method, pre, nan, nan_cat, classes, _ = MODELS[kind]
    X, y, s = raw(seed, n, nan=nan, nan_cat=nan_cat, y_classes=max(classes, 2))
    target = y if classes else (np.exp(0.2 * s) if kind == "hgb_poisson" else s)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe = make_pipeline(PRE[pre](), make()).fit(X, target)
    return pipe, getattr(pipe, method), nan, nan_cat


def problem(kind, seed, N, n, partial=True, weights=False):
    _, _, _, nan, nan_cat, _, _ = MODELS[kind]
    bg, _, _ = raw(seed, N, nan=nan, nan_cat=nan_cat)
    X, _, _ = raw(seed + 1, n, nan=nan, nan_cat=nan_cat)
    if partial:                                  # x takes the background's constant value of column 1 on every other row
        bg[:, 1] = 0.75
        X[::2, 1] = 0.75
    w = np.random.default_rng(seed).uniform(0.1, 1.0, N) if weights else None
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


def oracle(fn, bg, link, w=None):
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    groups = [[k] for k in range(bg.shape[1])]
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


@pytest.mark.parametrize("kind,link", CASES)
def test_parity_with_the_oracle(kind, link):
    pipe, fn, _, _ = fitted(kind)
    bg, X, _ = problem(kind, 11, N=16, n=4)
    eng = engine(fn, bg, link)
    assert eng.encoding is not None and eng.spec.n_features == 5
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "trees"
    M, _ = eng.varying(X)
    assert {int(m) for m in M} == {4, 5}                     # full and partial varying sets in one call
    worst = compare(got, oracle(fn, bg, link), X, own_plans(eng, X), TOL)
    print(f"{kind} {link}: max|d|/max|phi| = {worst:.2e}")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want_fx = np.asarray(fn(X), dtype=np.float64).reshape(X.shape[0], -1)
    np.testing.assert_allclose(eng.predict(X), want_fx, rtol=1e-12, atol=1e-12)


def test_weighted_background():
    pipe, fn, _, _ = fitted("gb2")
    bg, X, w = problem("gb2", 5, N=14, n=4, weights=True)
    eng = engine(fn, bg, "logit", w=w)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "trees"
    compare(got, oracle(fn, bg, "logit", w=w), X, own_plans(eng, X), TOL)


def _encoded_reading(pipe, enc, bg, X, link, **kw):
    """The pipeline's own fitted trees explained on pipe[:-1].transform, one group per raw column's encoded block."""
    groups = [[int(e) for e in np.nonzero(enc.sources == c)[0]] for c in range(enc.D)]
    final = getattr(pipe[-1], "predict_proba" if hasattr(pipe[-1], "predict_proba") else "predict")
    return engine(final, dense(pipe, bg), link, groups=groups, **kw), dense(pipe, X)


@pytest.mark.parametrize("plan_mode", ["shared", "per_instance"])
@pytest.mark.parametrize("kind", ["dt", "gb2", "hgb"])
def test_same_phi_as_the_encoded_reading(kind, plan_mode):
    pipe, fn, _, _ = fitted(kind)
    bg, X, _ = problem(kind, 13, N=12, n=6)
    link = MODELS[kind][-1][-1]
    eng = engine(fn, bg, link, plan_mode=plan_mode)
    ref, Xe = _encoded_reading(pipe, eng.encoding, bg, X, link, plan_mode=plan_mode)
    np.testing.assert_array_equal(eng.varying(X)[0], ref.varying(Xe)[0])
    got = np.stack(as_list(eng.shap_values(X, l1_reg=False, nsamples=24)))
    want = np.stack(as_list(ref.shap_values(Xe, l1_reg=False, nsamples=24)))
    assert eng.last_path()["general"] == "trees" and ref.last_path()["general"] == "trees"
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(np.atleast_1d(eng.expected_value), np.atleast_1d(ref.expected_value))


def _adversarial(pipe, X):
    rows = []
    vals = {c: [np.nan, 0.0, -0.0, 7.0, 5.0, -1.0] for c in range(X.shape[1])}
    for _, t, cols in pipe[0].transformers_:
        idx = list(range(X.shape[1]))[cols] if isinstance(cols, slice) else \
            [i for i, b in enumerate(cols) if b] if np.asarray(cols).dtype == bool else [int(c) for c in cols]
        first = t.steps[0][1] if hasattr(t, "steps") else t
        for j, c in enumerate(idx):
            if isinstance(first, KBinsDiscretizer):
                vals[c] += [v for e in first.bin_edges_[j] for v in (e, np.nextafter(e, -np.inf), np.nextafter(e, np.inf))]
            if isinstance(first, MinMaxScaler):
                vals[c] += [v for b in (first.data_min_[j], first.data_max_[j])
                            for v in (b, np.nextafter(b, -np.inf), np.nextafter(b, np.inf), 3 * b + 1, -3 * b - 1)]
            if isinstance(first, (StandardScaler, RobustScaler, MaxAbsScaler)):
                vals[c] += list(np.random.default_rng(c).normal(size=40) * 10.0)
    tree = getattr(pipe[-1], "tree_", None)
    if tree is not None:      # raw values near the split thresholds: scan a fine grid around each
        for c in range(X.shape[1]):
            vals[c] += list(np.linspace(np.nanmin(X[:, c]), np.nanmax(X[:, c]), 400))
    for c, vs in vals.items():
        for v in vs:
            r = X[len(rows) % len(X)].copy()
            r[c] = v
            rows.append(r)
    rows = np.asarray(rows)
    ok = np.zeros(len(rows), dtype=bool)
    for i, r in enumerate(rows):
        try:
            dense(pipe, r[None, :])
            ok[i] = True
        except ValueError:
            pass
    return rows[ok]


@pytest.mark.parametrize("kind", ["dt", "rf", "et_reg", "gb2", "hgb", "hgb_poisson"])
def test_device_encoding_is_bit_exact(kind):
    pipe, fn, _, _ = fitted(kind)
    bg, X, _ = problem(kind, 3, N=10, n=8, partial=False)
    eng = engine(fn, bg, "identity")
    rows = _adversarial(pipe, X)
    got, want = eng.encode(rows), dense(pipe, rows)
    assert np.array_equal(got, want, equal_nan=True), np.argwhere(~((got == want) | (np.isnan(got) & np.isnan(want))))[:5]
    assert np.array_equal(got, eng.encoding.transform(rows), equal_nan=True)


def test_fma_and_nan_clip_on_the_device():
    """MinMaxScaler's x * s + o is two roundings (a fused multiply-add would round once) and its clip keeps NaN."""
    X, y, _ = raw(0, 300)
    pipe = make_pipeline(ct(("m", MinMaxScaler(clip=True), [0, 1, 2]), ("r", MinMaxScaler(), [0, 1, 2])),
                         HistGradientBoostingClassifier(max_iter=5)).fit(X, y)
    eng = engine(pipe.predict_proba, X[:10], "identity")
    rows = np.random.default_rng(1).normal(size=(4000, 5)) * 5.0
    rows[::7, 2] = np.nan
    got, want = eng.encode(rows), dense(pipe, rows)
    assert np.array_equal(got, want, equal_nan=True)
    assert np.isnan(got[::7, 2]).all() and np.isnan(got[::7, 5]).all()
    # the case is sensitive: one rounding instead of two changes some of these values
    s, o = pipe[0].transformers_[1][1].scale_, pipe[0].transformers_[1][1].min_
    x = rows[:, :3]
    two = x * s + o
    one = np.array([[float(np.longdouble(v) * np.longdouble(sc) + np.longdouble(oc)) for v, sc, oc in zip(r, s, o)]
                    for r in x[:400]])
    assert (np.nan_to_num(one) != np.nan_to_num(two[:400])).any()


def test_caller_supplied_plans():
    pipe, fn, _, _ = fitted("hgb")
    bg, X, _ = problem("hgb", 8, N=10, n=3, partial=False)
    rng = np.random.default_rng(0)
    plans = []
    for i in range(3):
        Z = rng.integers(0, 2, size=(24, 5)).astype(np.uint8)
        Z[0], Z[1] = 0, 1
        Z[2:7] = np.eye(5, dtype=np.uint8)
        plans.append((Z, rng.uniform(0.1, 1.0, 24)))
    eng = engine(fn, bg, "logit")
    got = eng.shap_values(X, l1_reg=False, nsamples=24, plans=plans)
    assert eng.last_path()["general"] == "trees"
    compare(got, oracle(fn, bg, "logit"), X, lambda i: plans[i], TOL, nsamples=24)


def _wide(seed=0):
    """14 raw groups (12 numeric, 2 categorical): l1_reg='auto' selects at nsamples='auto'."""
    X, y, _ = raw(seed, 400, P_num=12, nan=False)
    pipe = make_pipeline(ct(("n", StandardScaler(), list(range(12))), ("c", OneHotEncoder(handle_unknown="ignore"),
                                                                        [12, 13])),
                         GradientBoostingClassifier(n_estimators=20, max_depth=3, random_state=0)).fit(X, y)
    bg, _, _ = raw(seed + 1, 8, P_num=12, nan=False)
    Xe, _, _ = raw(seed + 2, 3, P_num=12, nan=False)
    return pipe, bg, Xe


@pytest.mark.parametrize("l1_reg", ["auto", "num_features(4)"])
def test_l1_selection(l1_reg):
    pipe, bg, X = _wide()
    fn = pipe.predict_proba
    eng = engine(fn, bg, "logit")
    got = eng.shap_values(X, l1_reg=l1_reg)
    path = eng.last_path()
    assert path["general"] in ("trees", "simt") and path["general_l1"] == 1, path
    compare(got, oracle(fn, bg, "logit"), X, own_plans(eng, X), L1_TOL, l1_reg=l1_reg)


def test_row_blocks_give_the_same_phi(monkeypatch):
    from distributedkernelshap_b200 import engine as engine_mod
    pipe, fn, _, _ = fitted("gb2")
    bg, X, _ = problem("gb2", 17, N=12, n=11)
    eng = engine(fn, bg, "logit")
    want = np.stack(eng.shap_values(X, l1_reg=False))
    monkeypatch.setattr(engine_mod, "MAX_ENCODED_BYTES_PER_CALL", 8 * eng.encoding.E * 3)   # 3 rows per call
    assert eng._rows_per_call() == 3
    got = np.stack(eng.shap_values(X, l1_reg=False))
    np.testing.assert_array_equal(got, want)


def test_graph_replay_is_bit_identical_to_the_host_path():
    import torch
    pipe, fn, _, _ = fitted("hgb")
    bg, X, _ = problem("hgb", 41, N=20, n=16)
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
        assert eng.last_path()["general"] == "trees"
        np.testing.assert_array_equal(phi.cpu().numpy(), want)
    eng.set_stream(0)


def test_kernel_shap_default_kwargs():
    from distributedkernelshap_b200.data import convert_to_link
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    pipe, fn, _, _ = fitted("gb2")
    bg, X, _ = problem("gb2", 23, N=30, n=6, partial=False)
    ks = KernelShap(pipe.predict_proba, link="logit", seed=0)
    ks.fit(bg)
    exp = ks.explain(X, silent=True)                     # default kwargs: nsamples='auto', l1_reg='auto'
    assert ks._explainer.last_path()["general"] in ("trees", "simt")
    sv = exp.shap_values
    assert len(sv) == 2 and sv[0].shape == (6, 5)        # one value per raw column
    fx = convert_to_link("logit").f(pipe.predict_proba(X))
    for c in range(2):
        np.testing.assert_allclose(sv[c].sum(1), fx[:, c] - exp.expected_value[c], rtol=1e-8, atol=1e-8)


def test_refusals():
    from distributedkernelshap_b200._cabi import DksError
    X, y, _ = raw(0, 300, nan=False)
    err = make_pipeline(ct(("n", "passthrough", [0, 1, 2]), ("c", OneHotEncoder(handle_unknown="error"), [3, 4])),
                        DecisionTreeClassifier(max_depth=4, random_state=0)).fit(X, y)
    bg, Xi = X[:10].copy(), X[10:14].copy()
    eng = engine(err.predict_proba, bg, "identity")
    Xi[2, 4] = 9.0                                       # unseen under handle_unknown='error'
    with pytest.raises(ValueError, match="instance 2"):
        eng.shap_values(Xi, l1_reg=False)
    with pytest.raises(ValueError, match="row 2"):
        eng.predict(Xi)
    bad_bg = bg.copy()
    bad_bg[4, 3] = 9.0
    with pytest.raises(ValueError, match="background row 4"):
        engine(err.predict_proba, bad_bg, "identity")
    poly = make_pipeline(ct(("p", PolynomialFeatures(2), [0, 1])), DecisionTreeClassifier()).fit(X, y)
    with pytest.raises(TypeError, match="PolynomialFeatures"):
        engine(poly.predict_proba, bg, "identity")
    for kernel in ("tcgen05", "shared"):
        e2 = engine(err.predict_proba, bg, "identity", kernel=kernel)
        with pytest.raises(DksError, match="tree"):
            e2.shap_values(X[10:12], l1_reg=False)
    Xw = np.random.default_rng(0).normal(size=(100, 65))
    wide = make_pipeline(StandardScaler(), DecisionTreeClassifier(max_depth=3)).fit(Xw, (Xw[:, 0] > 0).astype(int))
    with pytest.raises(NotImplementedError, match="64"):
        engine(wide.predict_proba, Xw[:5], "identity")
    vote = VotingClassifier([("a", make_pipeline(StandardScaler(), DecisionTreeClassifier())),
                             ("b", make_pipeline(StandardScaler(), DecisionTreeClassifier(max_depth=2)))],
                            voting="soft").fit(X, y)
    with pytest.raises(NotImplementedError, match="ensemble"):
        engine(vote.predict_proba, bg, "identity")
