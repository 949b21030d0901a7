"""The exp head (log-link GLM regressors: ``predict = exp(X w + b)``) on the host: model extraction, the float64 reference of
the factorised formula (tests/glm_reference.py) against the oracle's masked batch, and the CUDA-core kernels' fp32 range
rule (csrc/dks_kernels.cuh: exp_row_ey) restated in NumPy."""
import warnings

import numpy as np
import pytest

from glm_reference import ExpReference


def _glm_data(seed, n=300, d=5):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d))
    mu = np.exp(0.3 * X[:, 0] - 0.2 * X[:, 1] + 0.1)
    return X, rng, mu


def _fit(est, X, y):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return est.fit(X, y)


@pytest.mark.parametrize("kind", ["poisson", "gamma", "tweedie_log", "tweedie_auto"])
def test_log_link_glms_extract_the_exp_head(kind):
    from sklearn.linear_model import GammaRegressor, PoissonRegressor, TweedieRegressor
    from distributedkernelshap_b200.predictors import extract_linear_spec
    X, rng, mu = _glm_data(3)
    if kind == "poisson":
        est, y = PoissonRegressor(alpha=0.01), rng.poisson(mu).astype(float)
    elif kind == "gamma":
        est, y = GammaRegressor(alpha=0.01), rng.gamma(2.0, mu / 2.0)
    elif kind == "tweedie_log":
        est, y = TweedieRegressor(power=1.5, link="log", alpha=0.01), rng.gamma(2.0, mu / 2.0)
    else:
        est, y = TweedieRegressor(power=1.5, alpha=0.01), rng.gamma(2.0, mu / 2.0)      # link='auto', power > 0: log
    _fit(est, X, y)
    spec = extract_linear_spec(est.predict)
    assert spec.activation == "exp" and spec.scalar_out and spec.W.shape == (1, X.shape[1])
    want = est.predict(X)
    got = spec(X)
    assert got.shape == want.shape
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)


@pytest.mark.parametrize("params", [dict(power=0.0), dict(power=0.0, link="identity")])
def test_identity_link_tweedie_keeps_the_identity_head(params):
    from sklearn.linear_model import TweedieRegressor
    from distributedkernelshap_b200.predictors import extract_linear_spec
    X, rng, mu = _glm_data(4)
    est = _fit(TweedieRegressor(alpha=0.01, **params), X, mu + rng.normal(0, 0.1, len(mu)))
    spec = extract_linear_spec(est.predict)
    assert spec.activation == "identity"
    np.testing.assert_allclose(spec(X), est.predict(X), rtol=1e-12, atol=1e-12)


def test_exp_spec_shape_rules_and_hook():
    from distributedkernelshap_b200 import _cabi
    from distributedkernelshap_b200.predictors import LinearModelSpec, extract_linear_spec
    with pytest.raises(ValueError):
        LinearModelSpec(np.ones((2, 3)), np.zeros(2), "exp")
    spec = LinearModelSpec(np.array([[0.5, -1.0, 0.25]]), [0.1], "exp", scalar_out=True)
    assert spec.act_code == _cabi.ACT_EXP == 4 and spec.n_outputs == 1
    X = np.array([[1.0, 2.0, 3.0], [0.0, 0.0, 0.0]])
    np.testing.assert_allclose(spec(X), np.exp(X @ spec.W[0] + 0.1), rtol=1e-15)
    assert LinearModelSpec(spec.W, spec.b, "exp")(X).shape == (2, 1)

    class Glm:                                   # a model offering the dks_linear_spec() hook on its predict
        def dks_linear_spec(self):
            return spec

        def predict(self, X):
            return spec(X)

    m = Glm()
    assert extract_linear_spec(m.predict) is spec and extract_linear_spec(m) is spec


def _problem(seed, G, N, weights):
    rng = np.random.default_rng(seed)
    coef = rng.normal(0, 0.6, G)
    bg = rng.standard_normal((N, G))
    w = None
    if weights:
        w = rng.uniform(0.1, 1.0, N)
        w[0] = 0.0                               # a zero-weight row: skipped by the log-sum-exp
        bg[0, :] = 40.0                          # ... whatever its score
    return coef, float(rng.normal(0, 0.3)), bg, w


@pytest.mark.parametrize("weights", [False, True])
def test_reference_matches_the_oracle_including_partial_sets(weights):
    from distributedkernelshap_b200.plan import build_plan
    from distributedkernelshap_b200.predictors import LinearModelSpec
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    G, N = 7, 12
    coef, b, bg, w = _problem(11 + weights, G, N, weights)
    groups = [[k] for k in range(G)]
    bg[:, [1, 4]] = bg[1, [1, 4]]                # groups 1 and 4 constant over the background ...
    rng = np.random.default_rng(5)
    X = rng.standard_normal((6, G))
    X[2:4][:, [1, 4]] = bg[1, [1, 4]]            # ... and equal to it in rows 2 and 3: partial varying sets
    ref = ExpReference(coef, b, bg, groups, w)
    spec = LinearModelSpec(coef[None, :], [b], "exp", scalar_out=True)
    orc = KernelExplainerOracle(spec, DenseData(bg, [f"g{k}" for k in range(G)], groups, w))
    np.testing.assert_allclose(orc.expected_value, ref.expected_value, rtol=1e-13)
    seen_partial = False
    for i in range(X.shape[0]):
        v = ref.varying(X[i])
        seen_partial |= len(v) < G
        plan = build_plan(len(v), 40, rng=np.random.RandomState(i))
        want = orc.explain(X[i:i + 1], plan=(plan.dense(), plan.weights), nsamples=40, l1_reg=False).reshape(G)
        got = ref.explain(X[i], plan=(plan.dense(), plan.weights))
        assert np.max(np.abs(got - want)) <= 1e-10 * np.max(np.abs(want)), i
        np.testing.assert_allclose(got.sum(), ref.predict(X[i])[0] - ref.expected_value, rtol=1e-10)
    assert seen_partial


def test_log_e_depends_on_the_varying_set():
    coef, b, bg, w = _problem(2, 5, 9, True)
    ref = ExpReference(coef, b, bg, [[k] for k in range(5)], w)
    Z = np.array([[1, 0, 1], [0, 1, 1]], dtype=float)
    assert not np.allclose(ref.log_e(Z, np.array([0, 1, 2])), ref.log_e(Z, np.array([2, 3, 4])))
    # against the plain sum of the positive-weight rows
    d = ref.base[1:][None, :] - Z @ ref.BW[1:][:, [0, 1, 2]].T
    np.testing.assert_allclose(ref.log_e(Z, np.array([0, 1, 2])), np.log(np.exp(d) @ ref.weights[1:]), rtol=1e-14)


# ---- the CUDA-core kernels' range rule, restated in float32 ------------------------------------------------------------
T_LO, T_HI = -60.0, 100.0        # DKS_EXP_T_LO / DKS_EXP_T_HI


def _ex2_ftz(t):
    """ex2.approx.ftz.f32 up to its rounding: results below 2^-126 flush to zero."""
    with np.errstate(over="ignore"):
        u = np.exp2(np.asarray(t, dtype=np.float32))
    return np.where(u < np.float32(2.0 ** -126), np.float32(0), u).astype(np.float32)


def _row_fp32(a, tp):
    """(ey, took_float64) of one coalition row as exp_row_ey forms it: tp = the t'_j (log2 units, weights folded in)."""
    tp = np.asarray(tp, dtype=np.float32)
    s = np.float32(0)
    for u in _ex2_ftz(tp):
        s = np.float32(s + u)
    thi = float(np.max(tp))
    if T_LO <= thi <= T_HI:
        with np.errstate(over="ignore"):
            ey = float(np.exp2(np.float64(a))) * float(s)
        if np.isfinite(ey):
            return ey, False
    return _row_f64(a, tp), True


def _row_f64(a, tp):
    tp = np.asarray(tp, dtype=np.float64)
    m = tp[np.isfinite(tp)].max()
    return 2.0 ** (a + m + np.log2(np.sum(np.exp2(tp - m))))


@pytest.mark.parametrize("n", [1, 100, 4096])
def test_range_rule_edges(n):
    rng = np.random.default_rng(n)
    for thi in (T_HI, T_HI - 0.5, T_LO, T_LO + 0.5, 0.0):
        # every term at the top (largest possible sum), and one term at the top with the rest far below (flushed)
        for rest in (np.full(n - 1, thi), thi - rng.uniform(0, 300, n - 1)):
            tp = np.concatenate([[thi], rest]).astype(np.float32)
            ey, f64 = _row_fp32(3.0, tp)
            assert not f64 and np.isfinite(ey)
            # the rounding of n sequential fp32 additions, as for every head's background sum
            assert abs(ey - _row_f64(3.0, tp)) <= (2e-6 + n * 2.0 ** -24) * _row_f64(3.0, tp)
    # a zero background weight folds into t' = -inf: it adds exactly nothing and does not move the maximum
    ey, f64 = _row_fp32(0.0, np.array([-np.inf, 1.0, 2.0], dtype=np.float32))
    assert not f64 and ey == 6.0


def test_outside_the_rule_fp32_would_overflow_or_flush():
    # what the rule guards against: a top term at 2^128 overflows fp32, one below 2^-126 flushes to 0
    assert np.isinf(_ex2_ftz(np.float32(128.0)))
    assert _ex2_ftz(np.float32(-127.0)) == 0
    # 2^100 terms summed over 2^20 rows stay finite; at 2^108 they would not
    with np.errstate(over="ignore"):
        assert np.isfinite(np.float32(2.0 ** 100) * np.float32(2 ** 20))
        assert np.isinf(np.float32(2.0 ** 108) * np.float32(2 ** 20))
    # rows outside the rule take float64 and are exact, including sums whose every fp32 term would flush or overflow
    for shift in (-300.0, -61.0, 101.0, 300.0):
        tp = np.array([shift, shift - 1.0, shift - 40.0], dtype=np.float32)
        ey, f64 = _row_fp32(-shift, tp)
        assert f64
        np.testing.assert_allclose(ey, 1.0 + 0.5 + 2.0 ** -40, rtol=1e-14)
    # an instance part that overflows 2^a on its own while the product is finite also goes to float64
    ey, f64 = _row_fp32(1030.0, np.array([-20.0, -21.0], dtype=np.float32))
    assert f64 and np.isfinite(ey)
