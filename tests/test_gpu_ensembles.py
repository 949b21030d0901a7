"""Soft-voting ensembles mixing tree, kernel-machine, MLP, neighbour and linear members, explained on the device: parity
with the oracle calling the ensemble's own method, phi equal to the members' phi averaged (identity link), every plan
source and entry point, the raw values a member refuses, an outer pipeline, and the refusals."""
import logging
import warnings

import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")
from sklearn.calibration import CalibratedClassifierCV  # noqa: E402
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.ensemble import (GradientBoostingClassifier, RandomForestClassifier, RandomForestRegressor,  # noqa: E402
                              VotingClassifier, VotingRegressor)
from sklearn.linear_model import LogisticRegression, Ridge  # noqa: E402
from sklearn.neighbors import KNeighborsClassifier, KNeighborsRegressor  # noqa: E402
from sklearn.neural_network import MLPClassifier, MLPRegressor  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import OneHotEncoder, StandardScaler  # noqa: E402
from sklearn.svm import SVC, SVR  # noqa: E402
from sklearn.tree import DecisionTreeClassifier  # noqa: E402

TOL = 1e-9
KNN_TOL = 1e-8
L1_TOL = 1e-5           # the l1 moments go through the 2^-40 fixed point
SUM_TOL = 1e-12


def _mlp():
    return MLPClassifier((8,), max_iter=300, random_state=0)


def _svc():
    return CalibratedClassifierCV(SVC(gamma=0.3), cv=2, ensemble=False)


MODELS = {   # members, classes (0: regression), weights
    "clf2_five": (lambda: [("lr", LogisticRegression()), ("rf", RandomForestClassifier(6, max_depth=4, random_state=0)),
                           ("mlp", _mlp()), ("knn", KNeighborsClassifier(5)), ("svc", _svc())], 2, [1, 2, 1, 1, 0.5]),
    "clf3_gb_mlp": (lambda: [("gb", GradientBoostingClassifier(n_estimators=8, max_depth=2, random_state=0)),
                             ("mlp", _mlp())], 3, None),
    "clf3_lr_knn_dt": (lambda: [("lr", LogisticRegression()), ("knn", KNeighborsClassifier(6, weights="distance")),
                                ("dt", DecisionTreeClassifier(max_depth=4, random_state=0))], 3, [2, 1, 1]),
    "reg_four": (lambda: [("rf", RandomForestRegressor(5, max_depth=4, random_state=0)), ("svr", SVR(gamma=0.2)),
                          ("mlp", MLPRegressor(hidden_layer_sizes=(8,), max_iter=300, random_state=0)), ("ridge", Ridge())], 0, None),
    "reg_knn_tree": (lambda: [("knn", KNeighborsRegressor(4)), ("rf", RandomForestRegressor(3, random_state=0))], 0,
                     [1, 3]),
}
LINKS = {"clf2_five": ("identity", "logit"), "clf3_gb_mlp": ("logit",), "clf3_lr_knn_dt": ("identity",),
         "reg_four": ("identity",), "reg_knn_tree": ("identity",)}
CASES = [(m, link) for m in MODELS for link in LINKS[m]]


def raw(seed, n, d=5):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)) * np.linspace(1.0, 2.0, d)
    s = X[:, 0] - 0.5 * X[:, 1] + 0.3 * X[:, 2] * X[:, 3] + 0.2 * np.sin(X[:, 4 % d])
    return X, s


def fitted(kind, seed=0, n=300, d=5):
    members, classes, weights = MODELS[kind]
    X, s = raw(seed, n, d)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if classes:
            y = np.digitize(s, np.quantile(s, np.linspace(0, 1, classes + 1)[1:-1]))
            vote = VotingClassifier(members(), voting="soft", weights=weights).fit(X, y)
            return vote, vote.predict_proba
        vote = VotingRegressor(members(), weights=weights).fit(X, s)
        return vote, vote.predict


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
    return KNN_TOL if "knn" in kind or "five" in kind else TOL


@pytest.mark.parametrize("kind,link", CASES)
def test_parity_with_the_oracle(kind, link):
    vote, fn = fitted(kind)
    bg, X, _ = problem(11, N=16, n=4)
    eng = engine(fn, bg, link)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "ensemble"
    M, _ = eng.varying(X)
    assert {int(m) for m in M} == {4, 5}                     # full and partial varying sets in one call
    worst = compare(got, oracle(fn, bg, link), X, own_plans(eng, X), tol(kind))
    print(f"{kind} {link}: max|d|/max|phi| = {worst:.2e}")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want_fx = np.asarray(fn(X), dtype=np.float64).reshape(X.shape[0], -1)
    np.testing.assert_allclose(eng.predict(X), want_fx, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("kind", ["clf3_gb_mlp", "reg_four"])
def test_identity_link_phi_is_the_members_phi_averaged(kind):
    vote, fn = fitted(kind)
    bg, X, _ = problem(3, N=12, n=5)
    eng = engine(fn, bg, "identity")
    got = np.stack(as_list(eng.shap_values(X, l1_reg=False)))
    members = vote.estimators_
    w = np.ones(len(members)) if vote.weights is None else np.asarray(vote.weights, dtype=float)
    want = 0.0
    for est, wk in zip(members, w / w.sum()):
        if isinstance(est, Ridge):          # a linear member alone runs the linear route: its phi is added below
            continue
        alone = engine(est.predict_proba if hasattr(est, "predict_proba") else est.predict, bg, "identity")
        want = want + wk * np.stack(as_list(alone.shap_values(X, l1_reg=False)))
    if kind == "reg_four":                  # the ridge member's phi: exactly coef (x - mean bg) per column
        ridge = members[3]
        want = want + (w[3] / w.sum()) * (ridge.coef_ * (X - bg.mean(0)))[None]
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-10 * np.abs(want).max())
    else:
        assert rel_err(got.reshape(-1), want.reshape(-1)) < SUM_TOL


@pytest.mark.parametrize("plan_mode", ["per_instance", "caller"])
def test_plan_sources(plan_mode):
    vote, fn = fitted("clf2_five")
    bg, X, _ = problem(5, N=12, n=3, partial=plan_mode == "per_instance")
    if plan_mode == "per_instance":
        eng = engine(fn, bg, "logit", plan_mode="per_instance")
        got = eng.shap_values(X, l1_reg=False)
        assert eng.last_path()["general"] == "ensemble"
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
    assert eng.last_path()["general"] == "ensemble"
    compare(got, oracle(fn, bg, "logit"), X, lambda i: plans[i], KNN_TOL, nsamples=24)


def test_weighted_background_and_grouped_columns():
    vote, fn = fitted("clf3_lr_knn_dt")
    bg, X, w = problem(5, N=14, n=4, weights=True)
    groups = [[0, 3], [1], [2, 4]]
    eng = engine(fn, bg, "identity", w=w, groups=groups)
    got = eng.shap_values(X, l1_reg=False)
    compare(got, oracle(fn, bg, "identity", w=w, groups=groups), X, own_plans(eng, X), KNN_TOL)


@pytest.mark.parametrize("l1_reg", ["auto", "aic", "num_features(4)"])
def test_l1_selection(l1_reg):
    members = lambda: [("rf", RandomForestClassifier(4, max_depth=3, random_state=0)), ("mlp", _mlp()),  # noqa: E731
                       ("lr", LogisticRegression())]
    MODELS["wide"] = (members, 2, None)
    try:
        vote, fn = fitted("wide", d=14, n=400)
    finally:
        del MODELS["wide"]
    bg, X, _ = problem(8, N=8, n=3, d=14, partial=l1_reg != "auto")
    eng = engine(fn, bg, "logit")
    got = eng.shap_values(X, l1_reg=l1_reg)
    path = eng.last_path()
    assert path["general"] in ("ensemble", "simt") and path["general_l1"] == 1, path
    compare(got, oracle(fn, bg, "logit"), X, own_plans(eng, X), L1_TOL, l1_reg=l1_reg)


def test_zero_one_and_two_varying_groups():
    vote, fn = fitted("clf2_five")
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


@pytest.mark.parametrize("fixed", [0, 63])
def test_sixty_four_groups(fixed):
    rng = np.random.default_rng(1)
    Xt = rng.normal(size=(300, 64))
    y = (Xt[:, 1] - Xt[:, 62] > 0).astype(int)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        vote = VotingClassifier([("dt", DecisionTreeClassifier(max_depth=5, random_state=0)), ("mlp", _mlp())],
                                voting="soft").fit(Xt, y)
    bg = Xt[:6].copy()
    bg[:, fixed] = 0.25
    X = Xt[10:12].copy()
    X[:, fixed] = 0.25
    eng = engine(vote.predict_proba, bg, "identity")
    got = eng.shap_values(X, l1_reg=False, nsamples=200)
    assert list(eng.varying(X)[0]) == [63, 63]
    compare(got, oracle(vote.predict_proba, bg, "identity"), X, own_plans(eng, X, 200), TOL, nsamples=200)


def test_batch_instances_bit_identical_to_the_instance_alone():
    vote, fn = fitted("clf3_gb_mlp")
    bg, _ = raw(9, 8)
    X, _ = raw(10, 4000)                         # more than three instances per CTA of every launch
    eng = engine(fn, bg, "logit")
    got = np.stack(eng.shap_values(X, l1_reg=False, nsamples=32))
    for i in (0, 1777, 3999):
        alone = np.stack(eng.shap_values(X[i:i + 1], l1_reg=False, nsamples=32))
        np.testing.assert_array_equal(got[:, i:i + 1], alone)


def test_device_run_graph_replay_and_launch_count():
    import torch
    vote, fn = fitted("reg_four")
    bg, X, _ = problem(41, N=20, n=16)
    eng = engine(fn, bg, "identity")
    want = np.stack(as_list(eng.shap_values(X, nsamples=24, l1_reg=False)))
    K = len(eng.spec.members)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(X).cuda()
        phi = torch.zeros((1, 16, 5), dtype=torch.float64, device="cuda")
        eng.explain_device(X_dev.data_ptr(), 16, phi.data_ptr(), nsamples=24)
        eng.check_status()
        before = eng.kernel_launches()
        eng.explain_device(X_dev.data_ptr(), 16, phi.data_ptr(), nsamples=24)
        # stage 1 (the varying groups, K member predictions, f(x)) and the explain (K members, the tail)
        assert eng.kernel_launches() - before == 2 * K + 3
        for _ in range(3):
            eng.explain_device(X_dev.data_ptr(), 16, phi.data_ptr(), nsamples=24)
        eng.check_status()
        assert eng.graph_launches() >= 1
        assert eng.last_path()["general"] == "ensemble"
        np.testing.assert_array_equal(phi.cpu().numpy(), want)
    eng.set_stream(0)


def test_raw_values_members_refuse():
    vote, fn = fitted("clf2_five")                # a kernel-machine member refuses NaN
    bg, X, _ = problem(2, N=10, n=4)
    eng = engine(fn, bg, "identity")
    X[2, 3] = np.nan
    with pytest.raises(ValueError, match="instance 2"):
        eng.shap_values(X, l1_reg=False)
    with pytest.raises(ValueError, match="row 2"):
        eng.predict(X)
    Xt, s = raw(0, 300)
    Xt[::7, 2] = np.nan
    y = (s > 0).astype(int)
    trees = VotingClassifier([("dt", DecisionTreeClassifier(max_depth=4, random_state=0)),
                              ("rf", RandomForestClassifier(4, max_depth=3, random_state=0))], voting="soft").fit(Xt, y)
    teng = engine(trees.predict_proba, bg, "identity")
    got = teng.shap_values(X, l1_reg=False)
    compare(got, oracle(trees.predict_proba, bg, "identity"), X, own_plans(teng, X), TOL)


def test_knn_member_tie_warning_passes_through():
    rng = np.random.default_rng(4)
    X = rng.integers(0, 3, (200, 4)).astype(float)
    y = (X[:, 0] + X[:, 1] > 2).astype(int)
    vote = VotingClassifier([("knn", KNeighborsClassifier(5)), ("dt", DecisionTreeClassifier(max_depth=3))],
                            voting="soft").fit(X, y)
    logger = logging.getLogger("distributedkernelshap_b200.engine")
    seen = []
    handler = logging.Handler()
    handler.emit = lambda record: seen.append(record.getMessage())
    logger.addHandler(handler)
    try:
        engine(vote.predict_proba, X[20:60], "identity")
    finally:
        logger.removeHandler(handler)
    assert any("equidistant" in m for m in seen), seen


def _outer_pipeline():
    # no neighbour member: on these integer-coded columns its ties are broken by the engine's rule, not scikit-learn's
    rng = np.random.default_rng(6)
    X = np.column_stack([rng.normal(size=(300, 3)), rng.integers(0, 3, (300, 2)).astype(float)])
    y = (X[:, 0] - X[:, 1] + (X[:, 3] == 1) > 0).astype(int)
    ct = ColumnTransformer([("n", StandardScaler(), [0, 1, 2]), ("c", OneHotEncoder(handle_unknown="ignore"), [3, 4])])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe = make_pipeline(ct, VotingClassifier([("lr", LogisticRegression()),
                                                   ("rf", RandomForestClassifier(5, max_depth=4, random_state=0)),
                                                   ("mlp", _mlp())], voting="soft")).fit(X, y)
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
    assert eng.last_path()["general"] == ref.last_path()["general"] == "ensemble"
    np.testing.assert_array_equal(got, want)
    compare(list(got), oracle(pipe.predict_proba, bg, "logit"), Xi, own_plans(eng, Xi, 40), TOL, nsamples=40)


def test_kernel_shap_default_kwargs():
    from distributedkernelshap_b200.data import convert_to_link
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    vote, _ = fitted("clf2_five")
    bg, X, _ = problem(23, N=30, n=6, partial=False)
    ks = KernelShap(vote.predict_proba, link="logit", seed=0)
    ks.fit(bg)
    exp = ks.explain(X, silent=True)
    assert ks._explainer.last_path()["general"] in ("ensemble", "simt")
    sv = exp.shap_values
    assert len(sv) == 2 and sv[0].shape == (6, 5)
    fx = convert_to_link("logit").f(vote.predict_proba(X))
    for c in range(2):
        np.testing.assert_allclose(sv[c].sum(1), fx[:, c] - exp.expected_value[c], rtol=1e-8, atol=1e-8)


def test_refusals():
    from distributedkernelshap_b200._cabi import DksError
    vote, fn = fitted("clf3_gb_mlp")
    bg, X, _ = problem(1, N=8, n=2)
    for kernel in ("tcgen05", "shared"):
        eng = engine(fn, bg, "identity", kernel=kernel)
        with pytest.raises(DksError, match="soft-voting ensembles run on the ensemble kernels only"):
            eng.shap_values(X, l1_reg=False)
    rng = np.random.default_rng(0)
    Xw = rng.normal(size=(100, 65))
    wide = VotingClassifier([("dt", DecisionTreeClassifier(max_depth=3)), ("lr", LogisticRegression())],
                            voting="soft").fit(Xw, (Xw[:, 0] > 0).astype(int))
    with pytest.raises(NotImplementedError, match="soft-voting ensembles are explained up to 64 groups"):
        engine(wide.predict_proba, Xw[:5], "identity")
