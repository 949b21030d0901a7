"""IsolationForest anomaly scores and AdaBoostClassifier on the tree route (``last_path()['general'] == 'trees'``) against
the oracle calling the real scikit-learn model on the masked batch, fed the coalition plans the engine used: both links
for AdaBoost, every plan source, weighted backgrounds, l1 selection, 0 / 1 / 2 varying groups, partial varying sets and 64
groups, outliers and NaN, batch against single rows, the device-resident entry and its graph replay, a ColumnTransformer
pipeline in raw feature space, AdaBoost as a soft-voting member, the public ``KernelShap`` API and the refusals."""
import warnings

import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")
from sklearn.ensemble import AdaBoostClassifier, IsolationForest, VotingClassifier  # noqa: E402
from sklearn.tree import DecisionTreeClassifier  # noqa: E402

PLAIN_TOL = 1e-9        # float64 end to end without selection
L1_TOL = 1e-5           # the l1 moments go through the 2^-40 fixed point


def _fit_rows(seed, n, P, nan=False):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P))
    if nan:
        X[rng.random(X.shape) < 0.04] = np.nan
    return X


def _labels(X, K):
    s = X[:, 0] + 0.5 * X[:, 1] - 0.7 * X[:, 2] * X[:, 3 % X.shape[1]]
    return np.digitize(s, np.quantile(s, np.linspace(0, 1, K + 1)[1:-1]))


def _model(kind, P, nan=False):
    X = _fit_rows(0, 400, P, nan=nan and kind.startswith("iso"))
    if kind == "iso_decision":
        return IsolationForest(n_estimators=40, random_state=0).fit(X).decision_function
    if kind == "iso_contamination":
        return IsolationForest(n_estimators=30, max_features=0.6, contamination=0.1, random_state=0).fit(X).decision_function
    if kind == "iso_score":
        return IsolationForest(n_estimators=30, max_samples=64, random_state=0).fit(X).score_samples
    K = {"ada2": 2, "ada3": 3, "ada3_decision": 3, "ada2_decision": 2}[kind]
    ada = AdaBoostClassifier(DecisionTreeClassifier(max_depth=2), n_estimators=25, random_state=0).fit(X, _labels(X, K))
    return ada.decision_function if kind.endswith("decision") else ada.predict_proba


def _problem(seed, P, N, n, nan=False, constant_cols=(), weights=False, outlier=False):
    rng = np.random.default_rng(seed)
    bg = rng.normal(size=(N, P))
    X = rng.normal(size=(n, P))
    if nan:
        bg[rng.random(bg.shape) < 0.05] = np.nan
        X[rng.random(X.shape) < 0.08] = np.nan
    if outlier:
        X[0, 0] = 40.0                       # isolated by the first split on column 0 of nearly every tree
    for c in constant_cols:                  # partial varying sets: x equals the constant background column on some rows
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


CASES = [("iso_decision", "identity"), ("iso_contamination", "identity"), ("iso_score", "identity"),
         ("ada2", "identity"), ("ada2", "logit"), ("ada3", "identity"), ("ada3", "logit"), ("ada2_decision", "identity"),
         ("ada3_decision", "identity")]


@pytest.mark.parametrize("kind,link", CASES)
def test_parity_with_the_oracle(kind, link):
    P = 7
    fn = _model(kind, P, nan=True)
    bg, X, _ = _problem(11, P, N=20, n=5, nan=kind.startswith("iso"), constant_cols=(6,), outlier=True)
    eng = _engine(fn, bg, link)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "trees" and eng.last_path()["shared"] == "none"
    M, _ = eng.varying(X)
    assert {int(m) for m in M} == {6, 7}                    # full and partial varying sets in one call
    want = fn(X)
    np.testing.assert_allclose(np.asarray(eng.predict(X)).reshape(want.shape), want, rtol=1e-12, atol=1e-14)
    worst = _compare(got, _oracle(fn, bg, link), X, _own_plans(eng, X), PLAIN_TOL)
    print(f"{kind} {link}: max|d|/max|phi| = {worst:.2e}")
    _check_additivity(eng, fn, got, X, link)
    out = _as_list(got)
    if len(out) == 2:
        np.testing.assert_array_equal(out[0], -out[1] + 0.0)    # class 0 is the exact negation of class 1


def test_outlier_isolated_at_the_root_takes_the_largest_share():
    P = 5
    fn = _model("iso_decision", P)
    bg, X, _ = _problem(12, P, N=16, n=3, outlier=True)
    eng = _engine(fn, bg, "identity")
    got = eng.shap_values(X, l1_reg=False)
    _compare(got, _oracle(fn, bg, "identity"), X, _own_plans(eng, X), PLAIN_TOL)
    assert np.argmin(got[0]) == 0 and got[0, 0] < 0          # the outlying column lowers the score most


def test_weighted_background():
    P = 6
    fn = _model("iso_decision", P)
    bg, X, w = _problem(3, P, N=15, n=4, weights=True)
    eng = _engine(fn, bg, "identity", w=w)
    got = eng.shap_values(X, l1_reg=False)
    _compare(got, _oracle(fn, bg, "identity", w=w), X, _own_plans(eng, X), PLAIN_TOL)
    _check_additivity(eng, fn, got, X, "identity")


@pytest.mark.parametrize("kind", ["iso_decision", "ada3"])
def test_per_instance_device_plans(kind):
    P = 8
    fn = _model(kind, P)
    bg, X, _ = _problem(21, P, N=12, n=5, constant_cols=(7,))
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


@pytest.mark.parametrize("kind,link", [("iso_score", "identity"), ("ada2", "logit")])
def test_caller_supplied_plans(kind, link):
    P = 6
    fn = _model(kind, P)
    bg, X, _ = _problem(8, P, N=10, n=3)
    rng = np.random.default_rng(0)
    plans = []
    for i in range(3):
        Z = rng.integers(0, 2, size=(40, P)).astype(np.uint8)
        Z[0] = 0
        Z[1] = 1
        Z[2:2 + P] = np.eye(P, dtype=np.uint8)
        plans.append((Z, rng.uniform(0.1, 1.0, 40)))
    eng = _engine(fn, bg, link)
    got = eng.shap_values(X, l1_reg=False, nsamples=40, plans=plans)
    assert eng.last_path()["general"] == "trees"
    _compare(got, _oracle(fn, bg, link), X, lambda i: plans[i], PLAIN_TOL, nsamples=40)


@pytest.mark.parametrize("kind,link,l1_reg", [("iso_decision", "identity", "auto"), ("iso_decision", "identity", "bic"),
                                              ("ada2", "logit", "auto"), ("ada3", "identity", "num_features(4)")])
def test_l1_selection(kind, link, l1_reg):
    P = 14                                    # 'auto' selects: 2076 of 16382 coalitions evaluated
    fn = _model(kind, P)
    bg, X, _ = _problem(31, P, N=8, n=4, constant_cols=(13,))
    eng = _engine(fn, bg, link)
    got = eng.shap_values(X, l1_reg=l1_reg)
    path = eng.last_path()
    assert path["general"] in ("trees", "simt") and path["general_l1"] == 1, path     # 'simt': every instance selected
    _compare(got, _oracle(fn, bg, link), X, _own_plans(eng, X), L1_TOL, l1_reg=l1_reg)


@pytest.mark.parametrize("vary", [0, 1, 2])
def test_zero_one_and_two_varying_groups(vary):
    P = 5
    fn = _model("iso_decision", P)
    rng = np.random.default_rng(4)
    bg = np.full((10, P), 0.5)
    X = np.full((3, P), 0.5)
    for c in range(vary):
        bg[:, c] = rng.normal(size=10)
        X[:, c] = rng.normal(size=3)
    eng = _engine(fn, bg, "identity")
    got = eng.shap_values(X, l1_reg=False)
    M, _ = eng.varying(X)
    assert set(M.tolist()) == {vary}
    _compare(got, _oracle(fn, bg, "identity"), X, _own_plans(eng, X), PLAIN_TOL)
    _check_additivity(eng, fn, got, X, "identity")
    if vary == 0:
        assert not np.any(got)


def test_sixty_four_groups():
    P = 64
    X_fit = _fit_rows(1, 300, P)
    fn = IsolationForest(n_estimators=20, random_state=0).fit(X_fit).decision_function
    bg, X, _ = _problem(6, P, N=6, n=2)
    eng = _engine(fn, bg, "identity")
    got = eng.shap_values(X, l1_reg=False, nsamples=300)
    assert eng.last_path()["general"] == "trees"
    _compare(got, _oracle(fn, bg, "identity"), X, _own_plans(eng, X, 300), PLAIN_TOL, nsamples=300)


def test_batch_and_single_rows_are_bit_identical():
    P = 6
    fn = _model("iso_decision", P, nan=True)
    bg, _, _ = _problem(9, P, N=8, n=1)
    _, X, _ = _problem(10, P, N=1, n=600, nan=True, constant_cols=(5,))
    eng = _engine(fn, bg, "identity")
    got = eng.shap_values(X, l1_reg=False, nsamples=32)
    for i in (0, 301, 599):
        np.testing.assert_array_equal(got[i:i + 1], eng.shap_values(X[i:i + 1], l1_reg=False, nsamples=32))


def test_graph_replay_is_bit_identical_to_the_host_path():
    import torch
    P = 8
    fn = _model("ada3", P)
    bg, X, _ = _problem(41, P, N=20, n=16, constant_cols=(7,))
    eng = _engine(fn, bg, "logit")
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


def test_column_transformer_pipeline_is_the_encoded_reading():
    from sklearn.compose import ColumnTransformer
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import OneHotEncoder, StandardScaler
    rng = np.random.default_rng(2)
    Xr = np.column_stack([rng.normal(size=400), rng.normal(size=400) * 3, rng.integers(0, 4, 400).astype(float)])
    pre = ColumnTransformer([("n", StandardScaler(), [0, 1]), ("c", OneHotEncoder(handle_unknown="ignore"), [2])])
    pipe = make_pipeline(pre, IsolationForest(n_estimators=30, random_state=0)).fit(Xr)
    bg, X = Xr[:12], np.column_stack([rng.normal(size=5), rng.normal(size=5), [0.0, 1.0, 2.0, 3.0, 7.0]])
    eng = _engine(pipe.decision_function, bg, "identity")
    got = eng.shap_values(X, l1_reg=False, nsamples=24)
    assert eng.last_path()["general"] == "trees"
    _compare(got, _oracle(pipe.decision_function, bg, "identity"), X, _own_plans(eng, X, 24), PLAIN_TOL, nsamples=24)
    enc = eng.encoding
    groups = [[int(e) for e in np.nonzero(enc.sources == c)[0]] for c in range(enc.D)]
    dense = lambda A: np.asarray(pipe[:-1].transform(A), dtype=np.float64)     # noqa: E731
    ref = _engine(pipe[-1].decision_function, dense(bg), "identity", groups=groups)
    want = ref.shap_values(dense(X), l1_reg=False, nsamples=24)
    np.testing.assert_array_equal(got, want)
    assert eng.expected_value == ref.expected_value


def test_soft_voting_member_is_the_members_phi_averaged():
    from sklearn.neural_network import MLPClassifier
    P = 6
    X_fit = _fit_rows(3, 300, P)
    y = _labels(X_fit, 2)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        vote = VotingClassifier([("ada", AdaBoostClassifier(n_estimators=15, random_state=0)),
                                 ("mlp", MLPClassifier((8,), max_iter=300, random_state=0))], voting="soft",
                                weights=[2.0, 1.0]).fit(X_fit, y)
    bg, X, _ = _problem(5, P, N=12, n=4)
    eng = _engine(vote.predict_proba, bg, "identity")
    got = np.stack(eng.shap_values(X, l1_reg=False))
    assert eng.last_path()["general"] == "ensemble"
    want = 0.0
    for est, wk in zip(vote.estimators_, (2.0 / 3.0, 1.0 / 3.0)):
        want = want + wk * np.stack(_engine(est.predict_proba, bg, "identity").shap_values(X, l1_reg=False))
    assert rel_err(got.reshape(-1), want.reshape(-1)) < 1e-12
    _compare(list(got), _oracle(vote.predict_proba, bg, "identity"), X, _own_plans(eng, X), PLAIN_TOL)


def test_kernel_shap_default_kwargs():
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    P = 8
    X_fit = _fit_rows(7, 500, P)
    iso = IsolationForest(random_state=0).fit(X_fit)
    bg, X, _ = _problem(17, P, N=30, n=6, outlier=True)
    ks = KernelShap(iso.decision_function, task="regression")
    ks.fit(bg)
    exp = ks.explain(X, silent=True)                            # nsamples='auto', l1_reg='auto'
    assert ks._explainer.last_path()["general"] == "trees"
    sv = exp.shap_values[0] if isinstance(exp.shap_values, list) else exp.shap_values
    ev = np.atleast_1d(exp.expected_value)[0]
    np.testing.assert_allclose(sv.sum(1), iso.decision_function(X) - ev, rtol=1e-8, atol=1e-8)
    ada = AdaBoostClassifier(random_state=0).fit(X_fit, _labels(X_fit, 2))
    ks = KernelShap(ada.predict_proba, link="logit")
    ks.fit(bg)
    exp = ks.explain(X, silent=True)
    assert ks._explainer.last_path()["general"] == "trees"
    from distributedkernelshap_b200.data import convert_to_link
    fx = convert_to_link("logit").f(ada.predict_proba(X))
    for c in range(2):
        np.testing.assert_allclose(exp.shap_values[c].sum(1), fx[:, c] - exp.expected_value[c], rtol=1e-8, atol=1e-8)


def test_refusals():
    from distributedkernelshap_b200._cabi import DksError
    P = 5
    bg, X, _ = _problem(2, P, N=8, n=2)
    for kind in ("iso_decision", "iso_score"):
        with pytest.raises(NotImplementedError, match="anomaly head.*logit"):
            _engine(_model(kind, P), bg, "logit")
    eng = _engine(_model("iso_decision", P), bg, "identity", kernel="tcgen05")
    with pytest.raises(DksError, match="tree"):
        eng.shap_values(X, l1_reg=False)
