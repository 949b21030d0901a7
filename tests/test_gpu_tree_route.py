"""Tree ensembles on the device (the tree route, ``last_path()['general'] == 'trees'``) against the oracle calling the
real scikit-learn model on the masked batch, fed the coalition plans the engine used: every family and head, both links,
full and partial varying sets, weighted backgrounds, per-instance device plans, caller-supplied plans, l1 selection,
shape edges, the device-resident entry and its graph replay, the public ``KernelShap`` API and the refusals."""
import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")
from sklearn.ensemble import (ExtraTreesClassifier, GradientBoostingClassifier, GradientBoostingRegressor,  # noqa: E402
                              HistGradientBoostingClassifier, HistGradientBoostingRegressor, RandomForestClassifier,
                              RandomForestRegressor)
from sklearn.tree import DecisionTreeClassifier, DecisionTreeRegressor  # noqa: E402

PLAIN_TOL = 1e-9        # float64 end to end without selection
L1_TOL = 1e-5           # the l1 moments go through the 2^-40 fixed point


def _xy(seed, n, P, nan=False):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P))
    if nan:
        X[rng.random(X.shape) < 0.04] = np.nan
    return X, rng


def _model(kind, P, seed=0):
    """(fitted model, method name, allows NaN)."""
    X, rng = _xy(seed, 400, P)
    s = X[:, 0] + 0.5 * X[:, 1] - 0.7 * X[:, 2] * X[:, 3 % P]
    y2 = (s > 0).astype(int)
    y4 = np.digitize(s, [-1.0, 0.0, 1.0])
    Xn = X.copy()
    Xn[rng.random(X.shape) < 0.04] = np.nan
    table = {
        "gb_binary": (lambda: GradientBoostingClassifier(n_estimators=30, max_depth=3, random_state=0).fit(X, y2),
                      "predict_proba", False),
        "gb_multi": (lambda: GradientBoostingClassifier(n_estimators=15, max_depth=2, random_state=0).fit(X, y4),
                     "predict_proba", False),
        "gb_decision": (lambda: GradientBoostingClassifier(n_estimators=15, max_depth=2, random_state=0).fit(X, y4),
                        "decision_function", False),
        "gb_regressor": (lambda: GradientBoostingRegressor(n_estimators=25, random_state=0).fit(X, s), "predict", False),
        "rf_binary": (lambda: RandomForestClassifier(20, max_depth=6, random_state=0).fit(Xn, y2), "predict_proba", True),
        "rf_multi": (lambda: RandomForestClassifier(10, max_depth=5, random_state=0).fit(Xn, y4), "predict_proba", True),
        "et_multi": (lambda: ExtraTreesClassifier(10, max_depth=5, random_state=0).fit(Xn, y4), "predict_proba", True),
        "rf_regressor": (lambda: RandomForestRegressor(10, max_depth=7, random_state=0).fit(Xn, s), "predict", True),
        "dt_classifier": (lambda: DecisionTreeClassifier(max_depth=6, random_state=0).fit(Xn, y4), "predict_proba", True),
        "hgb_binary": (lambda: HistGradientBoostingClassifier(max_iter=25, random_state=0).fit(Xn, y2), "predict_proba",
                       True),
        "hgb_multi": (lambda: HistGradientBoostingClassifier(max_iter=10, random_state=0).fit(Xn, y4), "predict_proba",
                      True),
        "hgb_decision": (lambda: HistGradientBoostingClassifier(max_iter=25, random_state=0).fit(Xn, y2),
                         "decision_function", True),
        "hgb_poisson": (lambda: HistGradientBoostingRegressor(max_iter=20, loss="poisson", random_state=0)
                        .fit(Xn, np.exp(0.5 * s)), "predict", True),
    }
    make, method, nan = table[kind]
    return make(), method, nan


LINKS = {"gb_binary": ("identity", "logit"), "gb_multi": ("identity", "logit"), "gb_decision": ("identity",),
         "gb_regressor": ("identity",), "rf_binary": ("identity", "logit"), "rf_multi": ("identity",),
         "et_multi": ("identity",), "rf_regressor": ("identity",), "dt_classifier": ("identity",),
         "hgb_binary": ("identity", "logit"), "hgb_multi": ("identity", "logit"), "hgb_decision": ("identity",),
         "hgb_poisson": ("identity",)}
CASES = [(k, link) for k in LINKS for link in LINKS[k]]


def _problem(seed, P, N, n, nan=False, constant_cols=(), weights=False):
    rng = np.random.default_rng(seed)
    bg = rng.normal(size=(N, P))
    X = rng.normal(size=(n, P))
    if nan:
        bg[rng.random(bg.shape) < 0.05] = np.nan
        X[rng.random(X.shape) < 0.05] = np.nan
    for c in constant_cols:              # partial varying sets: x equals the constant background column on some rows
        bg[:, c] = 0.25
        X[::2, c] = 0.25
    w = rng.uniform(0.1, 1.0, N) if weights else None
    return bg, X, w


def _data(bg, w=None, groups=None):
    from distributedkernelshap_b200.data import DenseData
    groups = groups or [[k] for k in range(bg.shape[1])]
    return DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, w)


def _engine(fn, bg, link, w=None, groups=None, **kw):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    return GpuKernelExplainer(fn, _data(bg, w, groups), link=link, seed=7, **kw)


def _oracle(fn, bg, link, w=None, groups=None):
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    groups = groups or [[k] for k in range(bg.shape[1])]
    return KernelExplainerOracle(fn, DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, w), link=link)


def _as_list(phi):
    return phi if isinstance(phi, list) else [phi]


def _compare(got, oracle, X, plans, tol, l1_reg=False, nsamples="auto"):
    """Oracle fed plans(i) per instance; returns the worst max|d| / max|phi| over instances and outputs."""
    got = _as_list(got)
    worst = 0.0
    for i in range(X.shape[0]):
        want = oracle.explain(X[i:i + 1], plan=plans(i), l1_reg=l1_reg, nsamples=nsamples)
        want = want.reshape(want.shape[0], -1)
        for c in range(want.shape[1]):
            e = rel_err(got[c][i], want[:, c])
            worst = max(worst, e)
            assert e < tol, (i, c, e)
    return worst


def _own_plans(eng, X, ns="auto"):
    M, _ = eng.varying(X)
    return lambda i: None if M[i] < 2 else (eng.shared_plan(int(M[i]), ns).dense(), eng.shared_plan(int(M[i]), ns).weights)


def _check_additivity(eng, fn, got, X, link):
    from distributedkernelshap_b200.data import convert_to_link
    lk = convert_to_link(link)
    fx = np.asarray(fn(X), dtype=np.float64).reshape(X.shape[0], -1)
    ev = np.atleast_1d(eng.expected_value)
    for c, ph in enumerate(_as_list(got)):
        np.testing.assert_allclose(ph.sum(1), lk.f(fx[:, c]) - ev[c], rtol=1e-8, atol=1e-8)


@pytest.mark.parametrize("kind,link", CASES)
def test_parity_every_family_and_head(kind, link):
    P = 7
    model, method, nan = _model(kind, P)
    fn = getattr(model, method)
    bg, X, _ = _problem(11, P, N=20, n=5, nan=nan, constant_cols=(6,))
    eng = _engine(fn, bg, link)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "trees" and eng.last_path()["shared"] == "none"
    M, _ = eng.varying(X)
    assert {int(m) for m in M} == {6, 7}                    # full and partial varying sets in one call
    worst = _compare(got, _oracle(fn, bg, link), X, _own_plans(eng, X), PLAIN_TOL)
    print(f"{kind} {link}: max|d|/max|phi| = {worst:.2e}")
    _check_additivity(eng, fn, got, X, link)
    out = _as_list(got)
    if len(out) == 2:
        np.testing.assert_array_equal(out[0], -out[1] + 0.0)    # class 0 is the exact negation of class 1


def test_weighted_background_and_kmeans():
    from distributedkernelshap_b200.data import kmeans
    P = 6
    model, method, _ = _model("gb_binary", P)
    fn = model.predict_proba
    rng = np.random.default_rng(3)
    summary = kmeans(rng.normal(size=(200, P)), 15, round_values=False)
    bg, w = np.asarray(summary.data, dtype=np.float64), np.asarray(summary.weights, dtype=np.float64)
    X = rng.normal(size=(4, P))
    eng = _engine(fn, bg, "logit", w=w)
    got = eng.shap_values(X, l1_reg=False)
    _compare(got, _oracle(fn, bg, "logit", w=w), X, _own_plans(eng, X), PLAIN_TOL)
    _check_additivity(eng, fn, got, X, "logit")


def test_grouped_columns():
    P = 8
    model, method, nan = _model("hgb_multi", P)
    fn = model.predict_proba
    groups = [[0, 1], [2], [3, 4, 5], [6], [7]]
    bg, X, _ = _problem(5, P, N=16, n=4, nan=True)
    eng = _engine(fn, bg, "identity", groups=groups)
    got = eng.shap_values(X, l1_reg=False, nsamples=20)
    _compare(got, _oracle(fn, bg, "identity", groups=groups), X, _own_plans(eng, X, 20), PLAIN_TOL, nsamples=20)


def test_per_instance_device_plans():
    P = 9
    model, method, _ = _model("rf_multi", P)
    fn = model.predict_proba
    bg, X, _ = _problem(21, P, N=12, n=6, constant_cols=(8,))
    eng = _engine(fn, bg, "identity", plan_mode="per_instance")
    got = eng.shap_values(X, l1_reg=False, nsamples=300)
    assert eng.last_path()["general"] == "trees"
    zb, w = eng.instance_plans()
    M, _ = eng.varying(X)
    from distributedkernelshap_b200.plan import resolve_nsamples

    def plans(i):
        S, _ = resolve_nsamples(int(M[i]), 300)
        k = np.arange(int(M[i]))
        Z = ((zb[i, :S, None] >> k.astype(np.uint64)) & np.uint64(1)).astype(np.uint8)
        return Z, w[i, :S]
    _compare(got, _oracle(fn, bg, "identity"), X, plans, PLAIN_TOL, nsamples=300)


def test_caller_supplied_plans():
    P = 6
    model, method, _ = _model("hgb_binary", P)
    fn = model.predict_proba
    bg, X, _ = _problem(8, P, N=10, n=3)
    rng = np.random.default_rng(0)
    plans = []
    for i in range(3):
        Z = rng.integers(0, 2, size=(40, P)).astype(np.uint8)
        Z[0] = 0
        Z[1] = 1
        Z[2:2 + P] = np.eye(P, dtype=np.uint8)
        plans.append((Z, rng.uniform(0.1, 1.0, 40)))
    eng = _engine(fn, bg, "logit")
    got = eng.shap_values(X, l1_reg=False, nsamples=40, plans=plans)
    assert eng.last_path()["general"] == "trees"
    _compare(got, _oracle(fn, bg, "logit"), X, lambda i: plans[i], PLAIN_TOL, nsamples=40)


@pytest.mark.parametrize("l1_reg", ["auto", "aic", "bic", "num_features(4)"])
def test_l1_selection(l1_reg):
    P = 14                                    # 'auto' selects: 2076 of 16382 coalitions evaluated
    model, method, _ = _model("gb_binary", P)
    fn = model.predict_proba
    bg, X, _ = _problem(31, P, N=8, n=4, constant_cols=(13,))
    eng = _engine(fn, bg, "logit")
    got = eng.shap_values(X, l1_reg=l1_reg)
    path = eng.last_path()
    assert path["general"] in ("trees", "simt") and path["general_l1"] == 1, path
    oracle = _oracle(fn, bg, "logit")
    _compare(got, oracle, X, _own_plans(eng, X), L1_TOL, l1_reg=l1_reg)
    plans = _own_plans(eng, X)
    selected = 0
    for i in range(X.shape[0]):              # the selected sets are the oracle's
        oracle.last_nonzero_inds = None
        oracle.explain(X[i:i + 1], plan=plans(i), l1_reg=l1_reg)
        if oracle.last_nonzero_inds is None:
            continue                         # 'auto' does not select for this instance's M
        selected += 1
        M, mask = eng.varying(X[i:i + 1])
        vary = [g for g in range(P) if (int(mask[0]) >> g) & 1]
        sel = {vary[k] for k in oracle.last_nonzero_inds}
        nz = {g for g in range(P) if got[1][i, g] != 0.0}
        assert nz <= sel, (i, nz, sel)
    assert selected >= 2


@pytest.mark.parametrize("shape", [("stump", 3, 10), ("leaf", 3, 10), ("m1", 4, 10), ("m2", 4, 10), ("g64", 64, 6),
                                   ("n_boundary", 6, 255), ("n_boundary", 6, 257)])
def test_shape_edges(shape):
    name, P, N = shape
    X_fit, rng = _xy(1, 200, P)
    yr = X_fit[:, 0] + X_fit[:, 1 % P]
    if name == "stump":
        model = DecisionTreeRegressor(max_depth=1).fit(X_fit, yr)
    elif name == "leaf":
        model = DecisionTreeRegressor().fit(X_fit, np.ones(200))
    elif name == "g64":
        model = GradientBoostingRegressor(n_estimators=10, max_depth=3, random_state=0).fit(X_fit, X_fit[:, :8].sum(1))
    else:
        model = GradientBoostingRegressor(n_estimators=10, random_state=0).fit(X_fit, yr)
    fn = model.predict
    bg = rng.normal(size=(N, P))
    X = rng.normal(size=(3, P))
    if name in ("m1", "m2"):                 # only one / two groups vary
        bg[:, 1:] = 0.5
        X[:, 1:] = 0.5
        if name == "m2":
            bg[:, 1] = rng.normal(size=N)
    eng = _engine(fn, bg, "identity")
    ns = 300 if name == "g64" else "auto"
    got = eng.shap_values(X, l1_reg=False, nsamples=ns)
    assert eng.last_path()["general"] == "trees"
    _compare(got, _oracle(fn, bg, "identity"), X, _own_plans(eng, X, ns), PLAIN_TOL, nsamples=ns)
    _check_additivity(eng, fn, got, X, "identity")


def test_graph_replay_is_bit_identical_to_the_host_path():
    import torch
    P = 8
    model, method, _ = _model("hgb_multi", P)
    bg, X, _ = _problem(41, P, N=20, n=16, constant_cols=(7,))
    eng = _engine(model.predict_proba, bg, "identity")
    want = np.stack(eng.shap_values(X, nsamples=200, l1_reg=False))
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(X).cuda()
        phi = torch.zeros((want.shape[0], 16, P), dtype=torch.float64, device="cuda")
        for _ in range(4):
            eng.explain_device(X_dev.data_ptr(), 16, phi.data_ptr(), nsamples=200)
        eng.check_status()
        assert eng.graph_launches() >= 1
        assert eng.last_path()["general"] == "trees"
        np.testing.assert_array_equal(phi.cpu().numpy(), want)
    eng.set_stream(0)


def test_kernel_shap_default_kwargs_on_an_adult_shaped_gbm():
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    d = adult_like(n_explain=40, n_background=60, seed=0)
    X_all = np.concatenate([d["background"], d["X_explain"]])
    y = d["predictor"].predict(X_all)
    gbm = GradientBoostingClassifier(n_estimators=40, max_depth=3, random_state=0).fit(X_all, y)
    ks = KernelShap(gbm.predict_proba, link="logit", feature_names=d["group_names"], seed=0)
    ks.fit(d["background"], group_names=d["group_names"], groups=d["groups"])
    exp = ks.explain(d["X_explain"][:6], silent=True)          # default kwargs: nsamples='auto', l1_reg='auto'
    assert ks._explainer.last_path()["general"] in ("trees", "simt")
    sv = exp.shap_values
    from distributedkernelshap_b200.data import convert_to_link
    fx = convert_to_link("logit").f(gbm.predict_proba(d["X_explain"][:6]))
    for c in range(2):
        np.testing.assert_allclose(sv[c].sum(1), fx[:, c] - exp.expected_value[c], rtol=1e-8, atol=1e-8)


def test_refusals():
    from distributedkernelshap_b200._cabi import DksError
    P = 5
    model, method, _ = _model("gb_binary", P)
    bg, X, _ = _problem(2, P, N=8, n=2)
    for kernel in ("tcgen05", "shared"):
        eng = _engine(model.predict_proba, bg, "identity", kernel=kernel)
        with pytest.raises(DksError, match="tree"):
            eng.shap_values(X, l1_reg=False)
    wide = GradientBoostingRegressor(n_estimators=3).fit(*_xy(0, 100, 65)[:1], np.arange(100.0))
    with pytest.raises(NotImplementedError, match="64"):
        _engine(wide.predict, np.zeros((4, 65)), "identity")
    pois, _, _ = _model("hgb_poisson", P)
    with pytest.raises(NotImplementedError, match="logit"):
        _engine(pois.predict, bg, "logit")
    # a pure leaf under the logit link: link(f(x)) is not finite -- reported, never written
    Xp, _ = _xy(0, 50, P)
    pure = DecisionTreeClassifier(max_depth=2).fit(Xp, (Xp[:, 0] > 0).astype(int))
    eng = _engine(pure.predict_proba, np.full((4, P), 5.0), "identity")
    Xo = np.full((1, P), -5.0)
    eng.shap_values(Xo, l1_reg=False)                           # identity link: fine
    with pytest.raises(DksError):
        _engine(pure.predict_proba, np.full((4, P), 5.0), "logit")
