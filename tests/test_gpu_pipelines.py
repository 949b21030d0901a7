"""Pipelines with per-column preprocessing explained in raw feature space on the device (column maps evaluated by the
prep, fit and predict kernels): the raw-space Adult model against the encoded one, parity with the oracle (which calls
the pipeline itself) for every head, shared and per-instance plans, l1 selection and a k-means-weighted background, the
"error" policy, and the public API."""
import warnings

import numpy as np
import pytest

from conftest import rel_err

pytest.importorskip("sklearn")
pytestmark = pytest.mark.gpu
TOL = 1e-5


def _quiet(fn, *a, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **kw)


# ---- raw-space Adult -----------------------------------------------------------------------------------------------
def _adult_raw():
    """adult_like's one-hot blocks decoded into level codes and the raw-space pipeline with the encoded model's
    coefficients."""
    from distributedkernelshap_b200.datasets import (ADULT_ONEHOT_WIDTHS, adult_like, decode_onehot_blocks,
                                                     raw_space_pipeline)
    d = adult_like(n_explain=256)
    raw_bg, raw_X = (decode_onehot_blocks(A, 4, ADULT_ONEHOT_WIDTHS, True) for A in (d["background"], d["X_explain"]))
    pipe = raw_space_pipeline(d["predictor"], np.vstack([raw_bg, raw_X]), 4, ADULT_ONEHOT_WIDTHS, True)
    np.testing.assert_allclose(pipe.predict_proba(raw_X), d["predictor"].predict_proba(d["X_explain"]), rtol=1e-10)
    return d, pipe, raw_bg, raw_X


def test_raw_space_adult_matches_the_encoded_model():
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    d, pipe, raw_bg, raw_X = _adult_raw()
    enc = KernelShap(d["predictor"].predict_proba, link="logit", feature_names=d["group_names"], seed=0)
    enc.fit(d["background"], group_names=d["group_names"], groups=d["groups"])
    want = enc.explain(d["X_explain"], silent=True, nsamples=2048, l1_reg=False).shap_values
    assert enc._explainer.last_path()["shared"] == "fused"
    rawk = KernelShap(pipe.predict_proba, link="logit", feature_names=d["group_names"], seed=0)
    rawk.fit(raw_bg)
    got = rawk.explain(raw_X, silent=True, nsamples=2048, l1_reg=False).shap_values
    assert rawk._explainer.last_path()["shared"] == "fused"
    for c in range(2):
        assert np.abs(got[c] - want[c]).max() / np.abs(want[c]).max() < 1e-5
    M_raw, _ = rawk._explainer.varying(raw_X)
    M_enc, _ = enc._explainer.varying(d["X_explain"])
    np.testing.assert_array_equal(M_raw, M_enc)


# ---- parity with the oracle ----------------------------------------------------------------------------------------
def _raw(n, seed, nan_bg=True):
    """Ten raw columns: numeric (0, 1, 2), binned (3, 4), ordinal (5), one-hot with unseen levels in X (6, 7), numeric
    with NaN, imputed (8), one-hot after imputation (9)."""
    rng = np.random.default_rng(seed)
    A = np.c_[rng.normal(size=(n, 3)), rng.uniform(-2, 2, (n, 2)), rng.integers(0, 6, n), rng.integers(0, 4, n),
              rng.choice([1.5, 2.5, 4.0], n), rng.normal(size=n), rng.integers(0, 3, n).astype(float)]
    if nan_bg:
        A[rng.random(n) < 0.15, 8] = np.nan
        A[rng.random(n) < 0.15, 9] = np.nan
    return A


def _preprocessor():
    from sklearn.compose import ColumnTransformer
    from sklearn.impute import SimpleImputer
    from sklearn.pipeline import make_pipeline
    from sklearn import preprocessing as pp
    return ColumnTransformer([
        ("num", pp.StandardScaler(), [0, 1, 2]),
        ("bins", pp.KBinsDiscretizer(n_bins=4, encode="onehot", quantile_method="averaged_inverted_cdf"), [3, 4]),
        ("ord", pp.OrdinalEncoder(handle_unknown="use_encoded_value", unknown_value=-1), [5]),
        ("oh", pp.OneHotEncoder(handle_unknown="ignore"), [6, 7]),
        ("imp", make_pipeline(SimpleImputer(add_indicator=True), pp.MinMaxScaler()), [8]),
        ("impoh", make_pipeline(SimpleImputer(strategy="most_frequent"), pp.OneHotEncoder(drop="first")), [9]),
    ])


def _targets(kind, A, seed=5):
    rng = np.random.default_rng(seed)
    s = A[:, 0] - 0.5 * A[:, 3] + 0.3 * A[:, 5] - 0.4 * A[:, 6] + 0.3 * np.nan_to_num(A[:, 8]) + rng.normal(size=len(A))
    if kind == "binary":
        return (s > 0.5).astype(int)
    if kind == "multi":
        return np.digitize(s, [-0.5, 0.5, 1.5])
    if kind == "reg1":
        return s
    if kind == "reg3":
        return np.c_[s, A[:, 1] - s, A[:, 5] + s]
    return rng.poisson(np.exp(0.3 * np.clip(s, -3, 3)))


def _final(name):
    from sklearn.linear_model import LogisticRegression, PoissonRegressor, Ridge
    from sklearn.multiclass import OneVsRestClassifier
    return {"binary": (LogisticRegression(max_iter=1000), "binary", "predict_proba", "logit"),
            "softmax": (LogisticRegression(max_iter=1000), "multi", "predict_proba", "logit"),
            "ovr": (OneVsRestClassifier(LogisticRegression(max_iter=1000)), "multi", "predict_proba", "logit"),
            "ridge1": (Ridge(alpha=1.0), "reg1", "predict", "identity"),
            "ridge3": (Ridge(alpha=1.0), "reg3", "predict", "identity"),
            "poisson": (PoissonRegressor(alpha=0.05, max_iter=500), "count", "predict", "identity")}[name]


def _fitted(name, nan_bg=True):
    from sklearn.pipeline import make_pipeline
    est, kind, method, link = _final(name)
    A = _raw(600, 11, nan_bg)
    pipe = _quiet(make_pipeline(_preprocessor(), est).fit, A, _targets(kind, A))
    bg = A[:40]
    X = _raw(12, 12, True)
    X[0, 6], X[1, 7], X[2, 5] = 9.0, 3.25, 17.0        # unseen categories: 'ignore' and 'use_encoded_value'
    X[3, 3] = pipe[0].named_transformers_["bins"].bin_edges_[0][2]          # on a bin edge
    return pipe, getattr(pipe, method), link, bg, X


def _oracle_check(f, link, bg, X, got, plan_of, weights=None, l1_reg=False, nsamples="auto"):
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    G = X.shape[1]
    orc = KernelExplainerOracle(f, DenseData(bg, [f"c{k}" for k in range(G)], None, weights), link=link)
    got = np.stack(got, axis=-1) if isinstance(got, list) else got[..., None]      # [n, G, C]
    for i in range(X.shape[0]):
        want = _quiet(orc.explain, X[i:i + 1], plan=plan_of(i), nsamples=nsamples, l1_reg=l1_reg).reshape(G, -1)
        if l1_reg is not False:             # the same selected groups (without selection a group can vary and still
            np.testing.assert_array_equal(got[i] != 0, want != 0, err_msg=str(i))   # contribute nothing: phi ~ 0)
        for c in range(want.shape[1]):
            assert rel_err(got[i][:, c], want[:, c]) < TOL, (i, c, rel_err(got[i][:, c], want[:, c]))
    return orc


def _additive(eng, got, f, link, X):
    from distributedkernelshap_b200.data import convert_to_link
    fx = np.asarray(f(X), dtype=np.float64).reshape(X.shape[0], -1)
    lf = convert_to_link(link).f(fx)
    got = np.stack(got, axis=-1) if isinstance(got, list) else got[..., None]
    ev = np.atleast_1d(eng.expected_value)
    np.testing.assert_allclose(got.sum(1), lf - ev, rtol=1e-8, atol=1e-8)


@pytest.mark.parametrize("name", ["binary", "softmax", "ovr", "ridge1", "ridge3", "poisson"])
def test_oracle_parity_shared_plans(name):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    pipe, f, link, bg, X = _fitted(name)
    eng = GpuKernelExplainer(f, bg, link=link, seed=7)
    assert eng.spec.maps is not None
    got = eng.shap_values(X, l1_reg=False)
    M, _ = eng.varying(X)
    _oracle_check(f, link, bg, X, got, lambda i: (eng.shared_plan(int(M[i])).dense(), eng.shared_plan(int(M[i])).weights))
    _additive(eng, got, f, link, X)


@pytest.mark.parametrize("name", ["binary", "softmax", "ridge1"])
def test_oracle_parity_per_instance_plans(name):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.plan import resolve_nsamples
    pipe, f, link, bg, X = _fitted(name)
    eng = GpuKernelExplainer(f, bg, link=link, seed=7, plan_mode="per_instance")
    got = eng.shap_values(X, l1_reg=False)
    M, _ = eng.varying(X)
    zb, w = eng.instance_plans()

    def plan_of(i):
        S = resolve_nsamples(int(M[i]), "auto")[0]
        k = np.arange(int(M[i]), dtype=np.uint64)
        return ((zb[i, :S, None] >> k[None, :]) & np.uint64(1)).astype(np.uint8), w[i, :S]
    _oracle_check(f, link, bg, X, got, plan_of)
    _additive(eng, got, f, link, X)


@pytest.mark.parametrize("name", ["binary", "ridge1"])
def test_oracle_parity_l1_auto_selects(name):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    pipe, f, link, bg, X = _fitted(name)
    eng = GpuKernelExplainer(f, bg, link=link, seed=7)
    got = eng.shap_values(X, nsamples=100, l1_reg="auto")
    path = eng.last_path()
    assert path["solve"] == "l1" or path["general_l1"] == 1, path
    M, _ = eng.varying(X)
    _oracle_check(f, link, bg, X, got, lambda i: (eng.shared_plan(int(M[i]), 100).dense(),
                                                  eng.shared_plan(int(M[i]), 100).weights),
                  l1_reg="auto", nsamples=100)


def test_oracle_parity_kmeans_weighted_background():
    from distributedkernelshap_b200.data import kmeans
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    pipe, f, link, _, X = _fitted("softmax", nan_bg=False)
    summary = kmeans(_raw(600, 11, False)[:300], 12)
    eng = GpuKernelExplainer(f, summary, link=link, seed=7)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["bg_weights"] == "weighted" or eng.last_path()["shared"] == "none"
    M, _ = eng.varying(X)
    _oracle_check(f, link, summary.data, X, got,
                  lambda i: (eng.shared_plan(int(M[i])).dense(), eng.shared_plan(int(M[i])).weights),
                  weights=summary.weights)
    _additive(eng, got, f, link, X)


def test_error_policy_raises_value_error():
    from sklearn.compose import ColumnTransformer
    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import OneHotEncoder, StandardScaler
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    A = _raw(300, 3, nan_bg=False)
    pipe = _quiet(make_pipeline(ColumnTransformer([("s", StandardScaler(), [0, 1, 2, 8]),
                                                   ("o", OneHotEncoder(handle_unknown="error"), [5, 6])]),
                                LogisticRegression(max_iter=500)).fit, A, _targets("binary", A))
    eng = GpuKernelExplainer(pipe.predict_proba, A[:20], link="logit", seed=1)
    X = A[20:24].copy()
    eng.shap_values(X, l1_reg=False)
    X[2, 6] = 11.0                                     # unseen category, handle_unknown='error'
    with pytest.raises(ValueError, match="instance 2"):
        eng.shap_values(X, l1_reg=False)
    X = A[20:24].copy()
    X[1, 8] = np.nan                                   # NaN reaching the estimator
    with pytest.raises(ValueError, match="instance 1"):
        eng.shap_values(X, l1_reg=False)
    with pytest.raises(ValueError):
        eng.predict(X)
    bad = A[:20].copy()
    bad[4, 5] = 99.0
    with pytest.raises(ValueError, match="background row 4"):
        GpuKernelExplainer(pipe.predict_proba, bad, link="logit", seed=1)


def test_public_api_kernel_shap_on_a_pipeline():
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    from distributedkernelshap_b200.data import convert_to_link
    pipe, f, link, bg, X = _fitted("binary")
    ks = KernelShap(pipe.predict_proba, link="logit", seed=2)
    ks.fit(bg)
    exp = ks.explain(X, silent=True)
    want = convert_to_link("logit").f(pipe.predict_proba(X))
    np.testing.assert_allclose(np.asarray(exp.data["raw"]["raw_prediction"]), want, rtol=1e-10, atol=1e-12)
    sv = exp.shap_values
    np.testing.assert_allclose(np.asarray(sv[1]).sum(1), want[:, 1] - np.ravel(exp.expected_value)[1], rtol=1e-8,
                               atol=1e-8)
