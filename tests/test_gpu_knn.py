"""Nearest-neighbour models on the device (the neighbour route, ``last_path()['general'] == 'knn'``) against the oracle fed
scikit-learn's own method (or, where equidistant training rows make scikit-learn's choice of neighbours undefined, the
engine's rule in ``KnnSpec``) and the coalition plans the engine used: both heads, both weightings, every metric, full and
partial varying sets, weighted backgrounds, per-instance device plans, caller-supplied plans, l1 selection, zero
distances, ties, the kernel's shape edges, the tie-aware fit check, the logit link's numeric reporting, the public
``KernelShap`` API and the refusals."""
import logging

import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")
from sklearn.neighbors import KNeighborsClassifier, KNeighborsRegressor  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import MinMaxScaler, StandardScaler  # noqa: E402

from distributedkernelshap_b200.neighbors import KnnSpec, extract_knn_spec  # noqa: E402

TOL = 1e-8              # float64 end to end without selection
L1_TOL = 1e-5           # the l1 moments go through the 2^-40 fixed point


def _fit_data(seed, P, n=150, classes=3):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    s = X[:, 0] - X[:, 0].mean() + 0.5 * (X[:, 1 % P] - X[:, 1 % P].mean()) * (X[:, 2 % P] - X[:, 2 % P].mean())
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, classes + 1)[1:-1]))
    T = np.stack([s + 0.1 * c * X[:, c % P] for c in range(8)], axis=1)
    return X, y, T, rng


def _model(kind, P, weights="uniform", k=5, scaler=StandardScaler, seed=0, n=150, classes=3, targets=2, **kw):
    X, y, T, _ = _fit_data(seed, P, n, classes)
    if kind == "clf":
        est, target, method = KNeighborsClassifier(n_neighbors=k, weights=weights, **kw), y, "predict_proba"
    else:
        est, target, method = KNeighborsRegressor(n_neighbors=k, weights=weights, **kw), \
            (T[:, 0] if targets == 1 else T[:, :targets]), "predict"
    fitted = (make_pipeline(scaler(), est) if scaler else est).fit(X, target)
    return getattr(fitted, method), X


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


def _compare(got, oracle, X, plans, tol=TOL, l1_reg=False, nsamples="auto", rows=None):
    got = _as_list(got)
    for i in (range(X.shape[0]) if rows is None else rows):
        want = oracle.explain(X[i:i + 1], plan=plans(i), l1_reg=l1_reg, nsamples=nsamples)
        want = want.reshape(want.shape[0], -1)
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
        np.testing.assert_allclose(ph.sum(1), convert_to_link(link).f(fx[:, c]) - ev[c], rtol=1e-8, atol=1e-8)


CASES = [(kind, weights, metric) for kind in ("clf", "reg") for weights in ("uniform", "distance")
         for metric in ({}, {"metric": "manhattan"}, {"p": 3})]


@pytest.mark.parametrize("kind,weights,metric", CASES)
def test_parity_every_head_weighting_and_metric(kind, weights, metric):
    P = 7
    fn, _ = _model(kind, P, weights, **metric)
    bg, X, _ = _problem(11, P, N=10, n=4, constant_cols=(6,))
    eng = _engine(fn, bg)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "knn" and eng.last_path()["shared"] == "none"
    M, _ = eng.varying(X)
    assert {int(m) for m in M} == {6, 7}                    # full and partial varying sets in one call
    _compare(got, _oracle(fn, bg), X, _own_plans(eng, X))
    _check_additivity(eng, fn, got, X)
    if kind == "clf":
        assert len(got) == 3                                # every class solved on its own


def test_weighted_background_with_a_zero_weight_row():
    P = 6
    fn, _ = _model("clf", P, "distance", scaler=MinMaxScaler)
    bg, X, w = _problem(3, P, N=10, n=3, weights=True, zero_row=True)
    eng = _engine(fn, bg, w=w)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "knn"
    _compare(got, _oracle(fn, bg, w=w), X, _own_plans(eng, X))


def test_grouped_columns():
    P = 8
    fn, _ = _model("reg", P, "distance", targets=3)
    groups = [[0, 1], [2], [3, 4, 5], [6], [7]]
    bg, X, _ = _problem(5, P, N=9, n=3)
    eng = _engine(fn, bg, groups=groups)
    got = eng.shap_values(X, l1_reg=False, nsamples=20)
    _compare(got, _oracle(fn, bg, groups=groups), X, _own_plans(eng, X, 20), nsamples=20)


def test_per_instance_device_plans():
    P = 9
    fn, _ = _model("reg", P, targets=1)
    bg, X, _ = _problem(21, P, N=8, n=5, constant_cols=(8,))
    eng = _engine(fn, bg, plan_mode="per_instance")
    got = eng.shap_values(X, l1_reg=False, nsamples=300)
    assert eng.last_path()["general"] == "knn"
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
    fn, _ = _model("clf", P, "distance", metric="manhattan")
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
    assert eng.last_path()["general"] == "knn"
    _compare(got, _oracle(fn, bg), X, lambda i: plans[i], nsamples=40)


@pytest.mark.parametrize("l1_reg", ["auto", "aic", "num_features(4)"])
def test_l1_selection(l1_reg):
    P = 14                                    # 'auto' selects: 2076 of 16382 coalitions evaluated
    fn, _ = _model("reg", P, "distance", targets=2, n=80)
    bg, X, _ = _problem(31, P, N=4, n=3, constant_cols=(13,))
    eng = _engine(fn, bg)
    got = eng.shap_values(X, l1_reg=l1_reg)
    path = eng.last_path()
    assert path["general"] in ("knn", "simt", "none") and path["general_l1"] == 1, path
    _compare(got, _oracle(fn, bg), X, _own_plans(eng, X), L1_TOL, l1_reg=l1_reg)


@pytest.mark.parametrize("weights", ["uniform", "distance"])
def test_background_from_the_training_rows_hits_distance_zero(weights):
    """The empty coalition reproduces bg_j, a training row: distance exactly 0, decided from the equality masks."""
    P = 6
    fn, Xfit = _model("clf", P, weights, scaler=None, algorithm="kd_tree")   # kd_tree: scikit-learn's distances exact
    bg = Xfit[::15][:10].copy()
    _, X, _ = _problem(4, P, N=2, n=3)
    eng = _engine(fn, bg)
    np.testing.assert_array_equal(eng.predict(bg), fn(bg))
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "knn"
    _compare(got, _oracle(fn, bg), X, _own_plans(eng, X))
    _check_additivity(eng, fn, got, X)


def _tied_problem():
    rng = np.random.default_rng(1)
    Xfit = rng.integers(0, 3, size=(300, 4)).astype(float)
    y = rng.integers(0, 2, 300)
    bg = rng.integers(0, 3, size=(12, 4)).astype(float)
    X = rng.integers(0, 3, size=(4, 4)).astype(float)
    X[X == bg[0]] += 3.0                               # every group varies
    return KNeighborsClassifier(n_neighbors=5, algorithm="brute").fit(Xfit, y), bg, X


def test_integer_data_with_boundary_ties(caplog):
    clf, bg, X = _tied_problem()
    spec = extract_knn_spec(clf.predict_proba)
    assert spec.boundary_ties(bg).any() and not spec.boundary_ties(bg).all()
    with caplog.at_level(logging.WARNING):
        eng = _engine(clf.predict_proba, bg)             # the tie-aware fit check passes, with a warning
    assert any("equidistant" in r.getMessage() for r in caplog.records)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "knn"
    _compare(got, _oracle(spec, bg), X, _own_plans(eng, X))     # the engine's rule: the lower training index wins
    _check_additivity(eng, spec, got, X)


def test_the_fit_check_refuses_a_corrupted_spec(monkeypatch):
    import distributedkernelshap_b200.engine as engine
    fn, _ = _model("clf", 5)
    bg, _, _ = _problem(2, 5, N=8, n=1)
    good = extract_knn_spec(fn)
    bad = KnnSpec(good.fitX, good.colw, good.colo, good.k, good.metric, good.p, good.weights, good.head,
                  (good.y + 1) % good.R, good.R, good.n_features)
    monkeypatch.setattr(engine, "extract_knn_spec", lambda model: bad)
    with pytest.raises(ValueError, match="does not reproduce"):
        _engine(fn, bg)


def test_the_fit_check_never_passes_vacuously():
    rng = np.random.default_rng(3)
    A = rng.normal(size=(40, 3))
    clf = KNeighborsClassifier(n_neighbors=1).fit(np.concatenate([A, A]), np.r_[np.zeros(40), np.ones(40)])
    with pytest.raises(ValueError, match="every background row"):   # every nearest row is one of two copies
        _engine(clf.predict_proba, rng.normal(size=(6, 3)))


@pytest.mark.parametrize("k,n_fit", [(1, 50), (32, 70), (7, 33)])
def test_neighbour_counts_and_training_rows_around_the_tile(k, n_fit):
    P = 6
    fn, _ = _model("reg", P, "distance", k=k, n=n_fit, targets=2)
    bg, X, _ = _problem(4, P, N=6, n=3, constant_cols=(5,))
    eng = _engine(fn, bg)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "knn"
    _compare(got, _oracle(fn, bg), X, _own_plans(eng, X))
    _check_additivity(eng, fn, got, X)


@pytest.mark.parametrize("shape", [("m0", 4), ("m1", 4), ("m2", 4), ("g64", 64)])
def test_varying_set_edges(shape):
    name, P = shape
    fn, _ = _model("clf", P, "distance", n=60)
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
        assert eng.last_path()["general"] == "knn"
    _compare(got, _oracle(fn, bg), X, _own_plans(eng, X, ns), nsamples=ns)
    _check_additivity(eng, fn, got, X)


def test_coalition_chunks_and_eight_classes():
    """k = 32 at 4094 coalitions: three classes' sums take 98 KB of shared memory and the solve region 32 KB, which
    leaves room for about 260 neighbour lists of 32 x 12 B: the coalitions go in chunks.  Then 8 classes."""
    P = 12
    fn, _ = _model("clf", P, "uniform", k=32, n=120, classes=3)
    bg, X, _ = _problem(6, P, N=3, n=2)
    eng = _engine(fn, bg)
    got = eng.shap_values(X, l1_reg=False, nsamples=4094)
    assert eng.last_path()["general"] == "knn"
    _compare(got, _oracle(fn, bg), X, _own_plans(eng, X, 4094), nsamples=4094)
    fn8, _ = _model("clf", 5, "distance", k=9, classes=8)
    bg8, X8, _ = _problem(7, 5, N=6, n=3)
    eng8 = _engine(fn8, bg8)
    got8 = eng8.shap_values(X8, l1_reg=False)
    assert len(got8) == 8
    _compare(got8, _oracle(fn8, bg8), X8, _own_plans(eng8, X8))


def test_eight_targets():
    P = 5
    fn, _ = _model("reg", P, "uniform", targets=8)
    bg, X, _ = _problem(12, P, N=6, n=3)
    eng = _engine(fn, bg)
    got = eng.shap_values(X, l1_reg=False)
    assert len(got) == 8 and eng.last_path()["general"] == "knn"
    _compare(got, _oracle(fn, bg), X, _own_plans(eng, X))


def test_grid_stride_batches_are_bit_identical_to_each_instance_alone():
    P = 4
    fn, _ = _model("clf", P, "distance", n=40)
    rng = np.random.default_rng(9)
    bg = rng.normal(size=(3, P))
    n = 132 * 8 * 2 + 17                      # more instances than CTAs
    X = rng.normal(size=(n, P))
    eng = _engine(fn, bg)
    got = np.stack(eng.shap_values(X, l1_reg=False))
    assert eng.last_path()["general"] == "knn"
    for i in (0, 1, n // 2, n - 1):
        np.testing.assert_array_equal(np.stack(eng.shap_values(X[i:i + 1], l1_reg=False))[:, 0], got[:, i])
    _compare(list(got), _oracle(fn, bg), X, _own_plans(eng, X), rows=(0, n - 1))


def test_probabilities_of_zero_or_one_under_the_logit_link():
    from distributedkernelshap_b200 import _cabi
    P = 4
    fn, _ = _model("clf", P, "uniform", k=3, classes=2)
    bg, X, _ = _problem(1, P, N=8, n=40)
    assert 0 < fn(bg).mean(0)[1] < 1
    sure = np.flatnonzero(fn(X)[:, 1] == 1.0)[:1]           # an instance all of whose neighbours are class 1
    assert sure.size == 1
    eng = _engine(fn, bg, "logit")
    with pytest.raises(_cabi.DksError) as e:
        eng.shap_values(X[sure], l1_reg=False)
    assert e.value.code == _cabi.DKS_ERR_NUMERIC


def test_kernel_shap_on_a_scaled_classifier_with_default_kwargs():
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    P = 6
    X, y, _, rng = _fit_data(13, P, n=400)
    clf = make_pipeline(StandardScaler(), KNeighborsClassifier()).fit(X, y)
    names = [f"f{i}" for i in range(P)]
    ks = KernelShap(clf.predict_proba, feature_names=names, seed=0)
    ks.fit(X[:30], group_names=names, groups=[[i] for i in range(P)])
    Xe = rng.normal(size=(4, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    exp = ks.explain(Xe, silent=True)                          # default kwargs: nsamples='auto', l1_reg='auto'
    assert ks._explainer.last_path()["general"] in ("knn", "none")
    fx = clf.predict_proba(Xe)
    for c in range(3):
        np.testing.assert_allclose(exp.shap_values[c].sum(1), fx[:, c] - exp.expected_value[c], rtol=1e-8, atol=1e-8)


def test_refusals():
    from distributedkernelshap_b200._cabi import DksError
    P = 5
    fn, _ = _model("clf", P)
    bg, X, _ = _problem(2, P, N=6, n=2)
    for kernel in ("tcgen05", "shared"):
        eng = _engine(fn, bg, kernel=kernel)
        with pytest.raises(DksError, match="neighbour kernel"):
            eng.shap_values(X, l1_reg=False)
    wide, X65 = _model("reg", 65, targets=1)
    with pytest.raises(NotImplementedError, match="64"):
        _engine(wide, X65[:4])
    few = KNeighborsClassifier(n_neighbors=10).fit(X[:2].repeat(3, 0), [0, 1] * 3).predict_proba
    with pytest.raises(NotImplementedError, match="at least n_neighbors"):
        _engine(few, bg)
    eng = _engine(fn, bg)
    Xn = X.copy()
    Xn[1, 2] = np.nan
    with pytest.raises(ValueError, match="instance 1"):
        eng.shap_values(Xn, l1_reg=False)
    bgi = bg.copy()
    bgi[3, 0] = np.inf
    with pytest.raises(ValueError, match="background row 3"):
        _engine(KnnSpec(bg, np.ones(P), np.zeros(P), 2, "euclidean", 2, "uniform", "regress", bg[:, 0], 1, P), bgi)


def _level_rows(seed, P, n):
    """n distinct training rows whose column c takes one of three non-dyadic levels of its own: a masked row can equal a
    training row exactly, and the table sums are not exact."""
    rng = np.random.default_rng(seed)
    levels = rng.uniform(0.1, 0.9, size=(P, 3))
    codes = np.unique(rng.integers(0, 3, size=(4 * n, P)), axis=0)
    codes = codes[rng.permutation(len(codes))[:n]]
    return levels[np.arange(P), codes], codes, rng


@pytest.mark.parametrize("metric", [{}, {"metric": "manhattan"}])
def test_coalitions_that_reproduce_a_training_row_hit_distance_zero(metric):
    """Background rows and instances are training rows over a few levels per column, so masked rows of non-empty, non-full
    coalitions are often training rows too: their distance 0 comes from the equality masks alone (the nibble-table sum
    of non-dyadic levels does not round to 0).  A grouped pair of columns and a group that does not vary for half the
    instances exercise the per-group masks and the non-varying-group test."""
    P = 7
    Xfit, codes, rng = _level_rows(3, P, 220)
    y = rng.integers(0, 3, len(Xfit))
    # each row's near twin, 1e-4 away with another label: it is a neighbour of every masked row that reproduces the row,
    # and weighs nothing next to the row's exact 0 -- but about 1e-4 of the row's weight if that 0 were read from the
    # rounded sum (about 1e-17)
    Xfit = np.concatenate([Xfit, Xfit + np.eye(P)[2] * 1e-4])
    y = np.concatenate([y, (y + 1) % 3])
    fn = KNeighborsClassifier(weights="distance", algorithm="kd_tree", **metric).fit(Xfit, y).predict_proba
    same6 = np.flatnonzero(codes[:, 6] == 1)
    bg = Xfit[same6[:8]]                                     # column 6 constant over the background
    X = np.concatenate([Xfit[same6[8:10]], Xfit[np.flatnonzero(codes[:, 6] != 1)[:2]]])
    groups = [[0, 1], [2], [3], [4], [5], [6]]
    eng = _engine(fn, bg, groups=groups)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "knn"
    M, vmask = eng.varying(X)
    assert {int(m) for m in M} == {5, 6}
    train = {tuple(r) for r in Xfit}
    hits = 0
    for i in range(X.shape[0]):
        Z = eng.shared_plan(int(M[i]), "auto").dense()
        vary = [g for g in range(len(groups)) if (int(vmask[i]) >> g) & 1]
        for z in Z:
            if z.all() or not z.any():
                continue
            cols = [c for g, on in zip(vary, z) if on for c in groups[g]]
            for b in bg:
                row = b.copy()
                row[cols] = X[i, cols]
                hits += tuple(row) in train
    assert hits > 20, hits
    _compare(got, _oracle(fn, bg, groups=groups), X, _own_plans(eng, X))
    _check_additivity(eng, fn, got, X)


def test_a_statistic_that_rounds_to_zero_is_not_a_zero_distance():
    """A training row 1e-170 away from the query has a squared difference that underflows to 0; it is not at distance 0,
    so under distance weights the exactly equal training row alone counts."""
    fitX = np.array([[0.0, 0.0], [1e-170, 0.0], [5.0, 5.0], [6.0, 6.0]])
    spec = KnnSpec(fitX, np.ones(2), np.zeros(2), 2, "euclidean", 2, "distance", "classify", [0, 1, 1, 0], 2, 2)
    bg = np.array([[5.0, 5.0], [6.0, 5.0]])                 # no tie between the 2nd and 3rd neighbour
    eng = _engine(spec, bg)
    Q = np.array([[0.0, 0.0], [1e-170, 0.0]])
    np.testing.assert_array_equal(eng.predict(Q), [[1.0, 0.0], [0.0, 1.0]])
    np.testing.assert_array_equal(eng.predict(Q), spec(Q))
