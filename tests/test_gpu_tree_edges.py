"""The tree kernel (``explain_tree_kernel``, dks_trees.cuh) where its own code changes behaviour: CTAs that take several
instances, more trees than one divergence pass holds, values on split thresholds, NaN and infinity, eight outputs, the
shared-memory limit, 64 groups with a partial varying set, zero-weight background rows, a forest of 70 k nodes and a walk
300 levels deep.  The reference is the oracle fed the float64 walk of tests/tree_reference.py (hand-built ensembles) or the
scikit-learn model's own method (fitted ones), with the coalition plans the engine used."""
import numpy as np
import pytest

import tree_reference as ref

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")
from sklearn.ensemble import (GradientBoostingClassifier, HistGradientBoostingClassifier,  # noqa: E402
                              RandomForestClassifier)
from sklearn.tree import DecisionTreeRegressor  # noqa: E402

from distributedkernelshap_b200.trees import CMP_F32, CMP_F64, extract_tree_spec  # noqa: E402

PLAIN_TOL = 1e-9        # float64 end to end without selection
L1_TOL = 1e-5           # the l1 moments go through the 2^-40 fixed point


def rel_err(got, want):
    """max|got - want| / max|want| of one instance and output.  phi is of order 1 in every problem here, except for the
    instances that differ from the background only where no split looks: theirs is rounding noise around 0 (1e-15 under
    the logit link), and the floor holds it to tol * 1e-3 absolute."""
    return float(np.abs(np.asarray(got) - want).max() / max(np.abs(want).max(), 1e-3))


# ---- plumbing ---------------------------------------------------------------------------------------------------------
def _groups(P, groups):
    return groups or [[k] for k in range(P)]


def _engine(model, bg, link, w=None, groups=None, **kw):
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    groups = _groups(bg.shape[1], groups)
    return GpuKernelExplainer(model, DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, w), link=link, seed=7, **kw)


def _oracle(fn, bg, link, w=None, groups=None):
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    groups = _groups(bg.shape[1], groups)
    return KernelExplainerOracle(fn, DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, w), link=link)


def _as_list(phi):
    return phi if isinstance(phi, list) else [phi]


def _shared_plans(eng, X, ns="auto"):
    M, _ = eng.varying(X)
    return lambda i: None if M[i] < 2 else (eng.shared_plan(int(M[i]), ns).dense(), eng.shared_plan(int(M[i]), ns).weights)


def _worst(got, oracle, X, plans, tol, rows=None, l1_reg=False, nsamples="auto"):
    """Oracle fed plans(i) for the given rows (default all); the worst max|d| / max|phi| over them and the outputs."""
    got = _as_list(got)
    worst = 0.0
    for i in (range(X.shape[0]) if rows is None else rows):
        want = oracle.explain(X[i:i + 1], plan=plans(i), l1_reg=l1_reg, nsamples=nsamples)
        want = want.reshape(want.shape[0], -1)
        for c in range(want.shape[1]):
            e = rel_err(got[c][i], want[:, c])
            worst = max(worst, e)
            assert e < tol, (i, c, e)
    return worst


def _same_varying_sets(eng, oracle, X, rows=None):
    M, mask = eng.varying(X)
    for i in (range(X.shape[0]) if rows is None else rows):
        want = set(int(g) for g in oracle.varying_groups(X[i:i + 1]))
        assert {g for g in range(eng.data.groups_size) if (int(mask[i]) >> g) & 1} == want and M[i] == len(want), i
    return M


def _additive(eng, fn, got, X, link):
    from distributedkernelshap_b200.data import convert_to_link
    lk = convert_to_link(link)
    fx = np.asarray(fn(X), dtype=np.float64).reshape(X.shape[0], -1)
    ev = np.atleast_1d(eng.expected_value)
    for c, ph in enumerate(_as_list(got)):
        np.testing.assert_allclose(ph.sum(1), lk.f(fx[:, c]) - ev[c], rtol=1e-8, atol=1e-8)


def _negated(got):
    out = _as_list(got)
    if len(out) == 2:
        np.testing.assert_array_equal(out[0], -out[1] + 0.0)    # class 0 is the exact negation of class 1


def _run(case, model, fn, bg, X, link, w=None, groups=None, nsamples="auto", l1_reg=False, tol=PLAIN_TOL, rows=None):
    """Explains X with ``model`` (a spec or a scikit-learn method) on the tree kernel and compares with the oracle calling
    ``fn``: the varying sets, phi of ``rows`` (default all), additivity, the negation of a two-output model."""
    eng = _engine(model, bg, link, w=w, groups=groups)
    got = eng.shap_values(X, l1_reg=l1_reg, nsamples=nsamples)
    path = eng.last_path()
    assert path["general"] == "trees" and path["shared"] == "none", path
    oracle = _oracle(fn, bg, link, w=w, groups=groups)
    _same_varying_sets(eng, oracle, X, rows)
    worst = _worst(got, oracle, X, _shared_plans(eng, X, nsamples), tol, rows=rows, l1_reg=l1_reg, nsamples=nsamples)
    print(f"{case}: max|d|/max|phi| = {worst:.2e}")
    _additive(eng, fn, got, X, link)
    _negated(got)
    return eng, got


def _bit_identical_alone(eng, got, X, **kw):
    """phi of instance i in the batch is phi of X[i:i+1] explained alone: the sums do not depend on the grid, and a CTA
    carries nothing from one instance to its next."""
    got = _as_list(got)
    for i in range(X.shape[0]):
        call = dict(kw)
        if "plans" in call:
            call["plans"] = call["plans"][i:i + 1]
        alone = _as_list(eng.shap_values(X[i:i + 1], **call))
        for c in range(len(got)):
            assert np.array_equal(alone[c][0], got[c][i]), (i, c, alone[c][0], got[c][i])


# ---- 1. CTAs that take several instances ---------------------------------------------------------------------------------
def _batch_rows():
    import torch                      # at most 8 CTAs per SM: every CTA takes three or four instances
    return 3 * 8 * torch.cuda.get_device_properties(0).multi_processor_count + 37


def _mixed_background(rng, n, P, const_cols, N=6):
    """Some background columns constant; each row of X matches all, some or none of them, in no regular order."""
    bg = rng.normal(size=(N, P))
    bg[:, const_cols] = rng.normal(size=len(const_cols))
    X = rng.normal(size=(n, P))
    match = rng.random((n, len(const_cols))) < 0.5
    X[:, const_cols] = np.where(match, bg[0, const_cols], X[:, const_cols])
    return bg, X, P - match.sum(1)


def _background_from_zero(rng, n, P, N=6):
    """N identical background rows; row i of X differs from them in k_i columns, k shuffled over 0..P."""
    b = rng.normal(size=P)
    k = rng.permutation(np.arange(n) % (P + 1))
    X = np.tile(b, (n, 1))
    for i in range(n):
        cols = rng.permutation(P)[:k[i]]
        X[i, cols] += rng.choice([-1.0, 1.0], size=k[i]) * rng.uniform(0.5, 2.0, size=k[i])
    return np.tile(b, (N, 1)), X, k


@pytest.mark.parametrize("background", ["mixed", "from_zero"])
def test_grid_stride_shared_plans(background):
    rng = np.random.default_rng(17)
    n, P = _batch_rows(), 6
    spec = ref.random_trees(rng, 5, 3, P, head="sigmoid", cmp=CMP_F64, scale=1.0)
    bg, X, M_want = (_mixed_background(rng, n, P, [0, 1, 2]) if background == "mixed" else _background_from_zero(rng, n, P))
    eng, got = _run(f"grid stride, {background}, {n} instances", spec, ref.model(spec), bg, X, "logit")
    M, _ = eng.varying(X)
    np.testing.assert_array_equal(M, M_want)
    assert set(M.tolist()) == ({3, 4, 5, 6} if background == "mixed" else set(range(P + 1)))
    _bit_identical_alone(eng, got, X, l1_reg=False)


def _distinct_plan(rng, M, nsamples):
    """A plan of this instance's own: the singletons (the normal matrix has full rank), then other coalitions in a
    random order, random weights."""
    S = min(nsamples, 2 ** M - 2)
    single = 1 << np.arange(M)
    rest = [c for c in rng.permutation(np.arange(1, 2 ** M - 1)) if c & (c - 1)]
    codes = np.concatenate([single, rest])[:S].astype(np.int64)
    return ((codes[:, None] >> np.arange(M)) & 1).astype(np.uint8), rng.uniform(0.1, 1.0, S)


def test_grid_stride_caller_supplied_plans():
    rng = np.random.default_rng(18)
    n, P, ns = _batch_rows(), 6, 20
    spec = ref.random_trees(rng, 5, 3, P, head="sigmoid", cmp=CMP_F64, scale=1.0)
    bg, X, M_want = _mixed_background(rng, n, P, [0, 1, 2])
    plans = [_distinct_plan(rng, int(m), ns) for m in M_want]
    eng = _engine(spec, bg, "logit")
    got = eng.shap_values(X, l1_reg=False, nsamples=ns, plans=plans)
    assert eng.last_path()["general"] == "trees"
    rows = list(range(0, n, n // 30))
    worst = _worst(got, _oracle(ref.model(spec), bg, "logit"), X, lambda i: plans[i], PLAIN_TOL, rows=rows, nsamples=ns)
    print(f"grid stride, a plan per instance, {n} instances ({len(rows)} against the reference): max|d|/max|phi| = {worst:.2e}")
    _negated(got)
    _bit_identical_alone(eng, got, X, l1_reg=False, nsamples=ns, plans=plans)


def test_grid_stride_l1_selection():
    rng = np.random.default_rng(19)
    n, P = _batch_rows(), 14                  # 'auto' selects at M = 14 (2076 of 16382 coalitions), not at 12 or 13
    spec = ref.random_trees(rng, 8, 3, P, head="sigmoid", cmp=CMP_F64, scale=1.0)
    bg, X, M_want = _mixed_background(rng, n, P, [12, 13])
    eng = _engine(spec, bg, "logit")
    got = eng.shap_values(X, l1_reg="auto")
    path = eng.last_path()
    assert path["general"] == "trees" and path["general_l1"] == 1, path
    M, _ = eng.varying(X)
    np.testing.assert_array_equal(M, M_want)
    assert set(M.tolist()) == {12, 13, 14}
    rows = [int(i) for m in (12, 13, 14) for i in np.nonzero(M == m)[0][:8]]
    worst = _worst(got, _oracle(ref.model(spec), bg, "logit"), X, _shared_plans(eng, X), L1_TOL, rows=rows, l1_reg="auto")
    print(f"grid stride, l1_reg='auto', {n} instances ({len(rows)} against the reference): max|d|/max|phi| = {worst:.2e}")
    _additive(eng, ref.model(spec), got, X, "logit")
    _negated(got)
    _bit_identical_alone(eng, got, X, l1_reg="auto")


# ---- 2. more trees than one divergence pass ----------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 3])
@pytest.mark.parametrize("T", ref.CHUNK_T)
def test_tree_chunks(T, R):
    # tests/test_tree_reference.py shows that divergent and non-divergent trees occur in every chunk of 256
    spec, bg, X = ref.chunk_problem(T, R)
    _run(f"{T} trees, {R} raw scores", spec, ref.model(spec), bg, X, "logit")


@pytest.mark.parametrize("link", ["identity", "logit"])
def test_default_gradient_boosting_on_three_classes(link):
    rng = np.random.default_rng(2)
    Xf = rng.normal(size=(300, 6))
    y = np.digitize(Xf[:, 0] + 0.5 * Xf[:, 1] - 0.7 * Xf[:, 2] * Xf[:, 3], [-0.5, 0.5])
    gb = GradientBoostingClassifier(random_state=0).fit(Xf, y)
    assert extract_tree_spec(gb.predict_proba).n_trees == 300
    _run(f"GradientBoostingClassifier(), 300 trees, {link}", gb.predict_proba, gb.predict_proba, rng.normal(size=(10, 6)),
         rng.normal(size=(3, 6)), link)


# ---- 3. values on split thresholds ---------------------------------------------------------------------------------------
def _fitted(kind):
    rng = np.random.default_rng(4)
    Xf = rng.normal(size=(300, 6))
    s = Xf[:, 0] + 0.5 * Xf[:, 1] - 0.7 * Xf[:, 2] * Xf[:, 3]
    y = (s > 0).astype(int)
    return {"dt_regressor": lambda: (DecisionTreeRegressor(max_depth=5, random_state=0).fit(Xf, s).predict, "identity", CMP_F32),
            "rf_classifier": lambda: (RandomForestClassifier(8, max_depth=4, random_state=0).fit(Xf, y).predict_proba,
                                      "identity", CMP_F32),
            "gb_classifier": lambda: (GradientBoostingClassifier(n_estimators=20, random_state=0).fit(Xf, y).predict_proba,
                                      "logit", CMP_F32),
            "hgb_classifier": lambda: (HistGradientBoostingClassifier(max_iter=10, random_state=0).fit(Xf, y).predict_proba,
                                       "logit", CMP_F64)}[kind]()


def _check_fnull_and_predict(eng, fn, bg, X, link):
    from distributedkernelshap_b200.data import convert_to_link
    fnull = np.asarray(fn(bg), dtype=np.float64).reshape(len(bg), -1).mean(0)
    np.testing.assert_allclose(np.atleast_1d(eng.expected_value), convert_to_link(link).f(fnull), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(eng.predict(X), np.asarray(fn(X), dtype=np.float64).reshape(len(X), -1), rtol=0, atol=1e-12)


@pytest.mark.parametrize("kind", ["dt_regressor", "rf_classifier", "gb_classifier", "hgb_classifier"])
def test_split_ties_fitted(kind):
    fn, link, cmp = _fitted(kind)
    spec = extract_tree_spec(fn)
    assert spec.cmp == cmp
    rng = np.random.default_rng(6)
    bg, share_bg = ref.on_thresholds(spec, rng, 8)
    X, share_x = ref.on_thresholds(spec, rng, 6)
    assert min(share_bg, share_x) >= 1 / 3
    eng, _ = _run(f"split ties, {kind}", fn, fn, bg, X, link)
    _check_fnull_and_predict(eng, fn, bg, X, link)


@pytest.mark.parametrize("cmp", [CMP_F32, CMP_F64])
def test_split_ties_hand_built(cmp):
    # the same node arrays, background and instances under both codes: tests/test_tree_reference.py shows that their
    # Shapley values differ by more than 1e-3
    spec, bg, X, share = ref.tie_problem(cmp)
    assert share >= 1 / 3 and spec.cmp == cmp
    eng, _ = _run(f"split ties, hand-built, cmp {cmp}", spec, ref.model(spec), bg, X, "logit")
    _check_fnull_and_predict(eng, ref.model(spec), bg, X, "logit")


# ---- 4. NaN and infinity -------------------------------------------------------------------------------------------------
def _nan_case(name):
    rng = np.random.default_rng(12)
    bg, X = rng.normal(size=(6, 4)), rng.normal(size=(5, 4))
    nan, inf = np.nan, np.inf
    if name in ("x_nan", "both_nan"):
        X[0, 0], X[1, 1], X[2, [0, 2]], X[3, :] = nan, nan, nan, nan
    if name in ("bg_nan", "both_nan"):
        bg[0, 0], bg[1, 1], bg[2, :], bg[3, 2] = nan, nan, nan, nan
    if name == "bg_column_all_nan":              # column 0 varies for the rows of X that hold a number there
        bg[:, 0], bg[1, 2] = nan, nan
        X[0, 0], X[2, [0, 2]] = nan, nan
    if name == "inf":
        X[0, 0], X[1, 1], X[2, :] = inf, -inf, [inf, -inf, inf, nan]
        bg[0, 0], bg[1, 2], bg[2, 0], bg[3, 3] = inf, -inf, inf, nan
    if name == "bg_column_all_inf":              # +inf equals +inf: column 0 does not vary for row 0
        bg[:, 0] = inf
        X[0, 0], X[2, 0] = inf, -inf
    infinite = name in ("inf", "bg_column_all_inf")
    return ref.nan_spec(CMP_F64 if infinite else CMP_F32, inf_fraction=0.3 if infinite else 0.0), bg, X


@pytest.mark.parametrize("name", ["x_nan", "bg_nan", "both_nan", "bg_column_all_nan", "inf", "bg_column_all_inf"])
def test_nan_and_infinity_hand_built(name):
    spec, bg, X = _nan_case(name)
    if name.startswith("bg_column"):
        assert np.any(spec.feature == 0)
    eng, _ = _run(f"missing values, {name}", spec, ref.model(spec), bg, X, "identity")
    if name.startswith("bg_column"):
        M, _ = eng.varying(X)
        assert M[0] == 3 and M[1] == 4
    _check_fnull_and_predict(eng, ref.model(spec), bg, X, "identity")


def test_fitted_missing_versus_rest_splits():
    est, Xf = ref.hgb_with_missing_split()
    spec = extract_tree_spec(est.predict_proba)
    assert np.any(np.isposinf(spec.threshold[spec.feature >= 0]))
    bg = Xf[:10].copy()
    assert 0 < np.isnan(bg[:, 0]).sum() < 10
    X = Xf[10:16].copy()
    X[0, 0], X[1, 0], X[2, 0], X[3, 0], X[4, 1] = np.nan, np.inf, -np.inf, 0.3, np.inf
    eng, _ = _run("missing values, fitted HistGradientBoostingClassifier with +inf thresholds", est.predict_proba,
                  est.predict_proba, bg, X, "logit")
    _check_fnull_and_predict(eng, est.predict_proba, bg, X, "logit")


# ---- 5. eight outputs; two outputs with one varying group or none -----------------------------------------------------------
def _eight_classes(rng):
    Xf = rng.normal(size=(400, 6))
    return Xf, np.digitize(Xf[:, 0] + 0.5 * Xf[:, 1] - 0.7 * Xf[:, 2] * Xf[:, 3], [-1.5, -1.0, -0.5, 0.0, 0.5, 1.0, 1.5])


@pytest.mark.parametrize("kind,link", [("rf", "identity"), ("gb", "identity"), ("gb", "logit"), ("hand_40", "identity"),
                                       ("hand_3", "logit")])
def test_eight_outputs(kind, link):
    rng = np.random.default_rng(8)
    if kind == "rf":
        model = fn = RandomForestClassifier(10, max_depth=5, random_state=0).fit(*_eight_classes(rng)).predict_proba
    elif kind == "gb":
        model = fn = GradientBoostingClassifier(n_estimators=5, max_depth=2, random_state=0).fit(*_eight_classes(rng)).predict_proba
    else:       # leaf values of size 40: saturated probabilities, a softmax that must subtract the maximum; size 3 for the logit
        model = ref.random_trees(rng, 16, 2, 6, R=8, head="softmax", cmp=CMP_F32, scale=float(kind.split("_")[1]))
        fn = ref.model(model)
    bg, X = rng.normal(size=(8, 6)), rng.normal(size=(3, 6))
    eng, got = _run(f"eight outputs, {kind}, {link}", model, fn, bg, X, link)
    assert len(got) == 8
    if kind == "hand_40":
        assert np.max(np.asarray(fn(X))) > 1 - 1e-9


@pytest.mark.parametrize("link", ["identity", "logit"])
@pytest.mark.parametrize("kind", ["hand_sigmoid", "gb_binary", "rf_binary"])
def test_two_outputs_with_one_varying_group_or_none(kind, link):
    rng = np.random.default_rng(9)
    P = 5
    if kind == "hand_sigmoid":
        model = ref.stumps(7, rng.integers(0, P, 7), rng.normal(size=7), rng.normal(size=7), rng.normal(size=7), P,
                           base=0.3, head="sigmoid")
        fn = ref.model(model)
    else:
        Xf = rng.normal(size=(300, P))
        y = (Xf[:, 0] + Xf[:, 1] * Xf[:, 2] + rng.normal(size=300) > 0).astype(int)
        est = (GradientBoostingClassifier(n_estimators=20, random_state=0) if kind == "gb_binary" else
               RandomForestClassifier(10, max_depth=3, min_samples_leaf=20, random_state=0)).fit(Xf, y)
        model = fn = est.predict_proba
    b = rng.normal(size=P)
    X = np.tile(b, (3 * P + 1, 1))
    for k in range(P):                       # rows 0..P-1: column k differs (M = 1); then two columns (M = 2); then none
        X[k, k] += 1.5
        X[P + k, [k, (k + 1) % P]] -= 1.5
        X[2 * P + k, k] -= 0.7
    eng, got = _run(f"two outputs, M = 0, 1, 2, {kind}, {link}", model, fn, np.tile(b, (4, 1)), X, link)
    M, _ = eng.varying(X)
    assert M.tolist() == [1] * P + [2] * P + [1] * P + [0]
    assert np.any(got[1][:P] != 0.0) and not np.any(got[1][-1])


# ---- 6. the shared-memory limit --------------------------------------------------------------------------------------------
def _smem_bytes(C, S, R, T):
    return 8 * (C * S + 63 * 63 + 64 + 256 * R + 8) + 4 * (T + 72)


def _last_S_that_fits(C, R, T):
    import torch
    limit = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    S = ((limit - 4 * (T + 72)) // 8 - (63 * 63 + 64 + 256 * R + 8)) // C
    assert _smem_bytes(C, S, R, T) <= limit < _smem_bytes(C, S + 1, R, T)
    return S


def _refused_and_nothing_written(eng, X, C, **kw):
    from distributedkernelshap_b200 import _cabi
    with pytest.raises(_cabi.DksError, match="shared memory"):
        eng.shap_values(X, l1_reg=False, **kw)
    phi = np.full((C, X.shape[0], X.shape[1]), 7.0)          # the plans are uploaded by now: the call is refused whole
    rc = eng.lib.dks_explain_host(eng._ctx, _cabi.ptr(X), X.shape[0], _cabi.ptr(phi), None, None, 0)
    assert rc == _cabi.DKS_ERR_UNSUPPORTED and np.all(phi == 7.0)


@pytest.mark.parametrize("C", [8, 1])
def test_shared_memory_limit(C):
    rng = np.random.default_rng(10)
    P, T = (13, 4) if C == 8 else (15, 4)              # S stays below 2^P - 2
    spec = ref.random_trees(rng, T, 2, P, R=C, head="softmax" if C > 1 else "identity", cmp=CMP_F64, scale=1.0)
    fn = ref.model(spec)
    S = _last_S_that_fits(C, C, T)
    assert S + 1 < 2 ** P - 2
    bg, X = rng.normal(size=(3, P)), rng.normal(size=(2, P))
    eng, _ = _run(f"shared memory, C = {C}, the last S that fits ({S})", spec, fn, bg, X, "identity", nsamples=S)
    _refused_and_nothing_written(_engine(spec, bg, "identity"), X, C, nsamples=S + 1)
    # caller-supplied plans of that stride
    plan = eng.shared_plan(P, S)
    Z, w = plan.dense(), plan.weights
    mine = _engine(spec, bg, "identity")
    got = mine.shap_values(X, l1_reg=False, nsamples=S, plans=[(Z, w)] * 2)
    assert mine.last_path()["general"] == "trees"
    worst = _worst(got, _oracle(fn, bg, "identity"), X, lambda i: (Z, w), PLAIN_TOL, nsamples=S)
    print(f"shared memory, C = {C}, caller-supplied plans of stride {S}: max|d|/max|phi| = {worst:.2e}")
    from distributedkernelshap_b200 import _cabi
    longer = (np.vstack([Z, Z[:1]]), np.append(w, w[0]))
    with pytest.raises(_cabi.DksError, match="shared memory"):
        _engine(spec, bg, "identity").shap_values(X, l1_reg=False, nsamples=S + 1, plans=[longer] * 2)


# ---- 7. groups --------------------------------------------------------------------------------------------------------------
def test_64_groups_with_the_first_or_the_last_not_varying():
    rng = np.random.default_rng(13)
    P = 64
    spec = ref.random_trees(rng, 12, 3, P, cmp=CMP_F32, features=[0, 1, 31, 32, 62, 63], scale=1.0)
    bg, X = rng.normal(size=(6, P)), rng.normal(size=(4, P))
    bg[:, [0, 63]] = [0.25, -0.5]
    X[0, 63], X[1, 0], X[2, [0, 63]] = -0.5, 0.25, [0.25, -0.5]
    eng, _ = _run("64 groups, M = 63, 63, 62, 64", spec, ref.model(spec), bg, X, "identity", nsamples=300)
    M, mask = eng.varying(X)
    assert M.tolist() == [63, 63, 62, 64]
    assert [int(m) >> 63 for m in mask] == [0, 1, 0, 1] and [int(m) & 1 for m in mask] == [1, 0, 0, 1]


def test_groups_of_several_split_columns_and_of_an_unused_column():
    rng = np.random.default_rng(14)
    groups = [[0, 1, 2, 3, 4], [5], [6, 7], [8, 9, 10], [11], [12, 13], [14, 15, 16], [17, 18, 19]]
    used = [c for c in range(20) if c != 11]
    spec = ref.random_trees(rng, 30, 3, 20, R=3, head="softmax", cmp=CMP_F32, features=used)
    assert set(spec.feature[spec.feature >= 0]) == set(used)
    bg, X = rng.normal(size=(7, 20)), rng.normal(size=(4, 20))
    bg[:, 17:] = 0.5
    X[0, 17:] = 0.5
    eng, got = _run("8 groups over 20 columns", spec, ref.model(spec), bg, X, "logit", groups=groups)
    M, _ = eng.varying(X)
    assert M.tolist() == [7, 8, 8, 8]


# ---- 8. background weights ----------------------------------------------------------------------------------------------------
def test_zero_weight_background_rows():
    rng = np.random.default_rng(15)
    P = 5
    spec = ref.random_trees(rng, 10, 3, P, head="sigmoid", cmp=CMP_F32, scale=1.0)
    fn = ref.model(spec)
    bg, X = rng.normal(size=(6, P)), rng.normal(size=(3, P))
    bg[0, :] = np.nan                                   # weight 0: an all-NaN row
    bg[3, :] = -50.0                                    # weight 0: a row far from all others
    w = np.array([0.0, 0.9, 0.02, 0.0, 0.05, 0.03])     # row 1 carries 90 % of the weight
    assert all(np.any(fn(bg[[3]]) != fn(bg[[j]])) for j in (1, 2, 4, 5))
    eng, got = _run("zero-weight background rows", spec, fn, bg, X, "logit", w=w)
    keep = w > 0
    _, without = _run("the same without them", spec, fn, bg[keep], X, "logit", w=w[keep])
    for a, b in zip(got, without):
        np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-12)
    uniform = _oracle(fn, bg, "logit")                 # and the weights matter
    plan = _shared_plans(eng, X)(0)
    assert rel_err(uniform.explain(X[:1], plan=plan, l1_reg=False)[:, 1], got[1][0]) > 1e-3


# ---- 9. size ------------------------------------------------------------------------------------------------------------------
def test_unpruned_forest():
    rng = np.random.default_rng(16)
    Xf = rng.normal(size=(4000, 8))
    y = (Xf[:, 0] + Xf[:, 1] * Xf[:, 2] + 1.5 * rng.normal(size=4000) > 0).astype(int)
    rf = RandomForestClassifier(50, random_state=0, n_jobs=4).fit(Xf, y)
    spec = extract_tree_spec(rf.predict_proba)
    assert spec.n_nodes > 65535 and ref.max_depth(spec) > 16, (spec.n_nodes, ref.max_depth(spec))
    _run(f"unpruned forest, {spec.n_nodes} nodes, depth {ref.max_depth(spec)}", rf.predict_proba, rf.predict_proba,
         rng.normal(size=(8, 8)), rng.normal(size=(2, 8)), "identity", nsamples=60)


def test_chain_of_depth_300():
    rng = np.random.default_rng(20)
    spec = ref.chain(300, [0, 1], 4)
    bg = np.abs(rng.normal(size=(8, 4))) * 1.5           # rows leave the chain at different depths
    X = np.array([[10.0, 10.0, 0.0, 1.0], [2.2, 0.7, 1.0, 0.0]])
    leaves = {ref.leaf_of(spec, 0, r) for r in np.concatenate([bg, X])}
    assert len(leaves) >= 8 and ref.leaf_of(spec, 0, X[0]) == spec.n_nodes - 1
    _run("chain of depth 300", spec, ref.model(spec), bg, X, "identity")
