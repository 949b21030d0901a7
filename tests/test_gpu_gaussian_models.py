"""Gaussian generative models on the device (the Gaussian route, ``last_path()['general'] == 'gauss'``) against the oracle
fed scikit-learn's own method and the coalition plans the engine used: QDA, GaussianNB, Gaussian mixtures and
EllipticEnvelope with every head, both links, full and partial varying sets, the varying-set edges, rows far from every
centre, weighted backgrounds, grouped columns, per-instance and caller-supplied plans, l1 selection, scaler and encoded
pipelines, graph replay, the shared-memory limit, the public ``KernelShap`` API and the refusals."""
import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.covariance import EllipticEnvelope  # noqa: E402
from sklearn.discriminant_analysis import QuadraticDiscriminantAnalysis  # noqa: E402
from sklearn.mixture import BayesianGaussianMixture, GaussianMixture  # noqa: E402
from sklearn.naive_bayes import GaussianNB  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import OneHotEncoder, StandardScaler  # noqa: E402

PLAIN_TOL = 1e-9        # float64 end to end without selection
L1_TOL = 1e-5           # the l1 moments go through the 2^-40 fixed point

MODELS = {
    "qda2": (lambda: QuadraticDiscriminantAnalysis(reg_param=0.1), 2),
    "qda5": (lambda: QuadraticDiscriminantAnalysis(reg_param=0.05), 5),
    "nb": (lambda: GaussianNB(priors=[0.2, 0.5, 0.3]), 3),
    "gmm_full": (lambda: GaussianMixture(3, random_state=0), 0),
    "gmm_tied": (lambda: GaussianMixture(3, covariance_type="tied", random_state=0), 0),
    "gmm_diag": (lambda: GaussianMixture(4, covariance_type="diag", random_state=0), 0),
    "gmm_spherical": (lambda: GaussianMixture(2, covariance_type="spherical", random_state=0), 0),
    # balanced weights: under the default Dirichlet-process prior one component takes 0.999 of the weight on this data,
    # and its probability's phi (about 1e-7) is then below the float64 rounding of predict_proba itself
    "bgmm": (lambda: BayesianGaussianMixture(n_components=3, weight_concentration_prior_type="dirichlet_distribution",
                                             weight_concentration_prior=100.0, random_state=0, max_iter=300), 0),
    "bgmm_dp": (lambda: BayesianGaussianMixture(n_components=3, random_state=0, max_iter=200), 0),
    "envelope": (lambda: EllipticEnvelope(random_state=0), 0),
}


def _fit_data(seed, P, n=300, classes=3):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    s = X[:, 0] - X[:, 0].mean() + 0.7 * (X[:, 1 % P] - X[:, 1 % P].mean())
    s = s + rng.normal(scale=2.0 * s.std(), size=n)         # overlapping classes: moderate posteriors
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, classes + 1)[1:-1]))
    return X, y, rng


def _model(key, method, P, seed=0, scaler=None, n=300):
    make, classes = MODELS[key]
    X, y, _ = _fit_data(seed, P, n, max(classes, 2))
    est = make()
    m = make_pipeline(scaler(), est) if scaler else est
    m.fit(X, y) if classes else m.fit(X)
    return getattr(m, method)


def _problem(seed, P, N, n, constant_cols=(), weights=False, zero_row=False):
    rng = np.random.default_rng(seed + 1000)
    bg = rng.normal(size=(N, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    for c in constant_cols:              # partial varying sets: x equals the constant background column on some rows
        bg[:, c] = 0.25
        X[::2, c] = 0.25
    w = rng.uniform(0.1, 1.0, N) if weights else None
    if zero_row:
        w[1] = 0.0
    return bg, X, w


def _data(bg, w=None, groups=None):
    from distributedkernelshap_b200.data import DenseData
    groups = groups or [[k] for k in range(bg.shape[1])]
    return DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, w)


def _engine(fn, bg, link="identity", w=None, groups=None, **kw):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    return GpuKernelExplainer(fn, _data(bg, w, groups), link=link, seed=7, **kw)


def _oracle(fn, bg, link="identity", w=None, groups=None):
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    groups = groups or [[k] for k in range(bg.shape[1])]
    return KernelExplainerOracle(fn, DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, w), link=link)


def _as_list(phi):
    return phi if isinstance(phi, list) else [phi]


def _compare(got, oracle, X, plans, tol=PLAIN_TOL, l1_reg=False, nsamples="auto"):
    got = _as_list(got)
    for i in range(X.shape[0]):
        want = oracle.explain(X[i:i + 1], plan=plans(i), l1_reg=l1_reg, nsamples=nsamples)
        want = want.reshape(want.shape[0], -1)
        assert want.shape[1] == len(got)
        for c in range(want.shape[1]):
            e = rel_err(got[c][i], want[:, c])
            assert e < tol, (i, c, e)


def _own_plans(eng, X, ns="auto"):
    M, _ = eng.varying(X)
    return lambda i: None if M[i] < 2 else (eng.shared_plan(int(M[i]), ns).dense(), eng.shared_plan(int(M[i]), ns).weights)


def _check_additivity(eng, fn, got, X, link="identity"):
    from distributedkernelshap_b200.data import convert_to_link
    fx = np.asarray(fn(X), dtype=np.float64).reshape(X.shape[0], -1)
    ev = np.atleast_1d(eng.expected_value)
    for c, ph in enumerate(_as_list(got)):
        want = convert_to_link(link).f(fx[:, c]) - ev[c]
        np.testing.assert_allclose(ph.sum(1), want, rtol=1e-8, atol=1e-8 * max(1.0, float(np.max(np.abs(want)))))


CASES = ([("qda2", "predict_proba", "identity"), ("qda2", "predict_proba", "logit"), ("qda2", "decision_function", "identity"),
          ("qda5", "predict_proba", "identity"), ("qda5", "predict_proba", "logit"), ("qda5", "decision_function", "identity"),
          ("nb", "predict_proba", "identity"), ("nb", "predict_proba", "logit"),
          ("envelope", "decision_function", "identity"), ("envelope", "score_samples", "identity")]
         + [(g, "score_samples", "identity") for g in ("gmm_full", "gmm_tied", "gmm_diag", "gmm_spherical", "bgmm", "bgmm_dp")]
         + [(g, "predict_proba", link) for g in ("gmm_full", "bgmm") for link in ("identity", "logit")]
         + [(g, "predict_proba", "identity") for g in ("gmm_tied", "gmm_diag", "gmm_spherical")])


@pytest.mark.parametrize("key,method,link", CASES)
def test_parity_every_model_method_and_link(key, method, link):
    P = 6
    fn = _model(key, method, P)
    bg, X, _ = _problem(11, P, N=10, n=4, constant_cols=(5,))
    eng = _engine(fn, bg, link)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "gauss" and eng.last_path()["shared"] == "none"
    M, _ = eng.varying(X)
    assert {int(m) for m in M} == {5, 6}                    # full and partial varying sets in one call
    _compare(got, _oracle(fn, bg, link), X, _own_plans(eng, X))
    _check_additivity(eng, fn, got, X, link)


@pytest.mark.parametrize("key,method", [("gmm_full", "score_samples"), ("qda2", "decision_function"),
                                        ("envelope", "score_samples"), ("nb", "predict_proba")])
def test_rows_far_from_every_centre(key, method):
    P = 6
    fn = _model(key, method, P)
    bg, X, _ = _problem(12, P, N=8, n=3)
    X = X * 20.0 + 60.0
    bg[:3] = bg[:3] * 20.0 - 60.0
    eng = _engine(fn, bg)
    got = eng.shap_values(X, l1_reg=False)
    _compare(got, _oracle(fn, bg), X, _own_plans(eng, X))
    _check_additivity(eng, fn, got, X)


def test_weighted_background_with_a_zero_weight_row():
    P = 6
    fn = _model("qda5", "predict_proba", P)
    bg, X, w = _problem(3, P, N=10, n=3, weights=True, zero_row=True)
    eng = _engine(fn, bg, w=w)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "gauss"
    _compare(got, _oracle(fn, bg, w=w), X, _own_plans(eng, X))


def test_grouped_columns():
    P = 8
    fn = _model("gmm_full", "score_samples", P)
    groups = [[0, 5], [2], [3, 4, 1], [6], [7]]
    bg, X, _ = _problem(5, P, N=9, n=3)
    eng = _engine(fn, bg, groups=groups)
    got = eng.shap_values(X, l1_reg=False, nsamples=20)
    _compare(got, _oracle(fn, bg, groups=groups), X, _own_plans(eng, X, 20), nsamples=20)


@pytest.mark.parametrize("shape", [("m0", 4), ("m1", 4), ("m2", 4), ("g64", 64)])
def test_varying_set_edges(shape):
    name, P = shape
    fn = _model("gmm_diag", "predict_proba", P)
    rng = np.random.default_rng(2)
    bg = rng.normal(size=(4, P))
    X = rng.normal(size=(3, P))
    if name != "g64":
        keep = {"m0": 0, "m1": 1, "m2": 2}[name]
        bg[:, keep:] = 0.5
        X[:, keep:] = 0.5
    eng = _engine(fn, bg)
    ns = 200 if P == 64 else "auto"
    got = eng.shap_values(X, l1_reg=False, nsamples=ns)
    M, _ = eng.varying(X)
    assert set(int(m) for m in M) == {"m0": {0}, "m1": {1}, "m2": {2}, "g64": {64}}[name]
    if name != "m0":
        assert eng.last_path()["general"] == "gauss"
    _compare(got, _oracle(fn, bg), X, _own_plans(eng, X, ns), nsamples=ns)
    _check_additivity(eng, fn, got, X)


def test_per_instance_device_plans():
    P = 9
    fn = _model("envelope", "decision_function", P)
    bg, X, _ = _problem(21, P, N=8, n=5, constant_cols=(8,))
    eng = _engine(fn, bg, plan_mode="per_instance")
    got = eng.shap_values(X, l1_reg=False, nsamples=300)
    assert eng.last_path()["general"] == "gauss"
    zb, w = eng.instance_plans()
    M, _ = eng.varying(X)
    from distributedkernelshap_b200.plan import resolve_nsamples

    def plans(i):
        S, _ = resolve_nsamples(int(M[i]), 300)
        k = np.arange(int(M[i]))
        Z = ((zb[i, :S, None] >> k.astype(np.uint64)) & np.uint64(1)).astype(np.uint8)
        return Z, w[i, :S]
    _compare(got, _oracle(fn, bg), X, plans, nsamples=300)


def test_caller_supplied_plans():
    P = 6
    fn = _model("nb", "predict_proba", P)
    bg, X, _ = _problem(8, P, N=7, n=3)
    rng = np.random.default_rng(0)
    plans = []
    for i in range(3):
        Z = rng.integers(0, 2, size=(40, P)).astype(np.uint8)
        Z[0] = 0
        Z[1] = 1
        Z[2:2 + P] = np.eye(P, dtype=np.uint8)
        plans.append((Z, rng.uniform(0.1, 1.0, 40)))
    eng = _engine(fn, bg)
    got = eng.shap_values(X, l1_reg=False, nsamples=40, plans=plans)
    assert eng.last_path()["general"] == "gauss"
    _compare(got, _oracle(fn, bg), X, lambda i: plans[i], nsamples=40)


@pytest.mark.parametrize("l1_reg", ["auto", "aic", "bic", "num_features(4)"])
def test_l1_selection(l1_reg):
    P = 14                                    # 'auto' selects: 2076 of 16382 coalitions evaluated
    fn = _model("qda2", "predict_proba", P)
    bg, X, _ = _problem(31, P, N=4, n=3, constant_cols=(13,))
    eng = _engine(fn, bg)
    got = eng.shap_values(X, l1_reg=l1_reg)
    path = eng.last_path()
    assert path["general"] in ("gauss", "simt", "none") and path["general_l1"] == 1, path
    _compare(got, _oracle(fn, bg), X, _own_plans(eng, X), L1_TOL, l1_reg=l1_reg)


def test_scaler_pipeline_matches_the_bare_model_on_scaled_columns():
    P = 7
    X, y, _ = _fit_data(4, P)
    pipe = make_pipeline(StandardScaler(), QuadraticDiscriminantAnalysis(reg_param=0.1)).fit(X, y)
    sc = pipe[0]
    bare = QuadraticDiscriminantAnalysis(reg_param=0.1).fit(sc.transform(X), y)
    bg, Xe, _ = _problem(9, P, N=8, n=3, constant_cols=(6,))
    got = _engine(pipe.predict_proba, bg).shap_values(Xe, l1_reg=False)
    want = _engine(bare.predict_proba, sc.transform(bg)).shap_values(sc.transform(Xe), l1_reg=False)
    for g, w in zip(got, want):
        assert rel_err(g, w) < PLAIN_TOL


def test_encoded_pipeline():
    P = 6
    X, y, rng = _fit_data(6, P)
    Xc = np.concatenate([X, rng.integers(0, 3, size=(X.shape[0], 1)).astype(np.float64)], axis=1)
    pre = ColumnTransformer([("num", StandardScaler(), list(range(P))), ("cat", OneHotEncoder(), [P])])
    pipe = make_pipeline(pre, GaussianMixture(3, random_state=0)).fit(Xc)
    bg, Xe, _ = _problem(10, P, N=8, n=3)
    bg = np.concatenate([bg, np.arange(8)[:, None] % 3.0], axis=1)
    Xe = np.concatenate([Xe, np.array([[0.0], [2.0], [1.0]])], axis=1)
    for method in ("score_samples", "predict_proba"):
        fn = getattr(pipe, method)
        eng = _engine(fn, bg)
        assert eng.encoding is not None
        got = eng.shap_values(Xe, l1_reg=False)
        assert eng.last_path()["general"] == "gauss"
        _compare(got, _oracle(fn, bg), Xe, _own_plans(eng, Xe))


def test_graph_replay_is_bit_identical_to_the_host_path():
    import torch
    P = 8
    fn = _model("gmm_full", "predict_proba", P)
    bg, X, _ = _problem(41, P, N=10, n=16, constant_cols=(7,))
    eng = _engine(fn, bg)
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
        assert eng.last_path()["general"] == "gauss"
        np.testing.assert_array_equal(phi.cpu().numpy(), want)
    eng.set_stream(0)


def test_shared_memory_limit():
    """Eight components at 64 groups need 8 (64^2 + 1) doubles of tables: more than an H100 CTA's shared memory."""
    from distributedkernelshap_b200._cabi import DksError
    P = 64
    rng = np.random.default_rng(3)
    fn = GaussianMixture(8, covariance_type="diag", random_state=0).fit(rng.normal(size=(400, P))).score_samples
    bg, X = rng.normal(size=(4, P)), rng.normal(size=(2, P))
    with pytest.raises(DksError, match="needs .* B of shared memory .* components too many"):
        _engine(fn, bg).shap_values(X, l1_reg=False, nsamples=200)
    fn2 = GaussianMixture(2, covariance_type="diag", random_state=0).fit(rng.normal(size=(400, P))).score_samples
    eng = _engine(fn2, bg)
    got = eng.shap_values(X, l1_reg=False, nsamples=200)
    _compare(got, _oracle(fn2, bg), X, _own_plans(eng, X, 200), nsamples=200)


def _adult():
    from distributedkernelshap_b200.datasets import adult_like
    d = adult_like(n_explain=600, n_background=40, seed=0)     # QDA needs more rows per class than its 49 columns
    X_all = np.concatenate([d["background"], d["X_explain"]])
    y = d["predictor"].predict(X_all)
    return d, X_all, y


@pytest.mark.parametrize("which", ["gmm_score_samples", "qda_logit"])
def test_kernel_shap_on_adult_with_default_kwargs(which):
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    d, X_all, y = _adult()
    if which == "gmm_score_samples":
        model = GaussianMixture(3, covariance_type="diag", random_state=0).fit(X_all)
        fn, link = model.score_samples, "identity"
    else:
        model = QuadraticDiscriminantAnalysis(reg_param=0.5).fit(X_all, y)
        fn, link = model.predict_proba, "logit"
    ks = KernelShap(fn, link=link, feature_names=d["group_names"], seed=0)
    ks.fit(d["background"], group_names=d["group_names"], groups=d["groups"])
    exp = ks.explain(d["X_explain"][:5], silent=True)          # default kwargs: nsamples='auto', l1_reg='auto'
    assert ks._explainer.last_path()["general"] in ("gauss", "none")
    fx = np.asarray(fn(d["X_explain"][:5])).reshape(5, -1)
    ev = np.atleast_1d(exp.expected_value)
    for c in range(fx.shape[1]):
        want = np.log(fx[:, c] / (1 - fx[:, c])) if link == "logit" else fx[:, c]
        np.testing.assert_allclose(np.asarray(exp.shap_values[c]).sum(1), want - ev[c], rtol=1e-8,
                                   atol=1e-8 * max(1.0, float(np.max(np.abs(want)))))


def test_refusals():
    from distributedkernelshap_b200._cabi import DksError
    P = 5
    fn = _model("qda2", "predict_proba", P)
    bg, X, _ = _problem(2, P, N=6, n=2)
    for kernel in ("tcgen05", "shared"):
        eng = _engine(fn, bg, kernel=kernel)
        with pytest.raises(DksError, match="Gaussian kernel"):
            eng.shap_values(X, l1_reg=False)
    wide = _model("nb", "predict_proba", 65, n=400)
    with pytest.raises(NotImplementedError, match="64"):
        _engine(wide, np.random.default_rng(0).normal(size=(4, 65)))
    with pytest.raises(NotImplementedError, match="link='identity' only"):
        _engine(_model("gmm_full", "score_samples", P), bg, link="logit")
    eng = _engine(fn, bg)
    Xn = X.copy()
    Xn[1, 2] = np.nan
    with pytest.raises(ValueError, match="instance 1"):
        eng.shap_values(Xn, l1_reg=False)
    bgi = bg.copy()
    bgi[3, 0] = np.inf
    from distributedkernelshap_b200.gaussian_models import extract_gaussian_spec
    with pytest.raises(ValueError, match="background row 3"):
        _engine(extract_gaussian_spec(fn), bgi)
