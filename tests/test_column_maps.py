"""Column maps compiled from scikit-learn pipelines (distributedkernelshap_b200/column_maps.py), checked in NumPy against
the pipelines themselves: per raw column, on random values, on every breakpoint and its float neighbours, on every
category, on unseen values and on NaN.  No GPU here."""
import warnings

import numpy as np
import pytest

pytest.importorskip("sklearn")
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.decomposition import PCA  # noqa: E402
from sklearn.impute import SimpleImputer  # noqa: E402
from sklearn.linear_model import LinearRegression, LogisticRegression, PoissonRegressor, Ridge  # noqa: E402
from sklearn.multiclass import OneVsRestClassifier  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn import preprocessing as pp  # noqa: E402

from distributedkernelshap_b200.column_maps import CATEGORICAL  # noqa: E402
from distributedkernelshap_b200.predictors import extract_linear_spec  # noqa: E402


def raw_data(n=300, seed=0):
    """Six raw columns: two numeric, two small-integer categorical, one uniform, one numeric with NaN."""
    rng = np.random.default_rng(seed)
    X = np.c_[rng.normal(size=n), rng.normal(size=n) * 3 + 1, rng.integers(0, 5, n), rng.choice([1.5, 2.0, 7.0, 9.0], n),
              rng.uniform(-2, 2, n), rng.normal(size=n)]
    X[rng.random(n) < 0.1, 5] = np.nan
    y = (np.nan_to_num(X[:, 0]) + X[:, 2] + rng.normal(size=n) > 2).astype(int)
    return X, y


NUM, CAT, NANCOL = [0, 1, 4], [2, 3], [5]
BINS = dict(quantile_method="averaged_inverted_cdf")


def ct(num, cat, nan=None, **kw):
    parts = [("num", num, NUM), ("cat", cat, CAT)]
    parts.append(("nan", nan if nan is not None else SimpleImputer(), NANCOL))
    return ColumnTransformer(parts, **kw)


PIPELINES = {
    "standard_onehot_drop": lambda: ct(pp.StandardScaler(), pp.OneHotEncoder(drop="first")),
    "minmax_onehot_ignore": lambda: ct(pp.MinMaxScaler(), pp.OneHotEncoder(handle_unknown="ignore")),
    "minmax_clip_onehot_error": lambda: ct(pp.MinMaxScaler(clip=True), pp.OneHotEncoder(handle_unknown="error")),
    "maxabs_infrequent": lambda: ct(pp.MaxAbsScaler(),
                                    pp.OneHotEncoder(handle_unknown="infrequent_if_exist", min_frequency=70)),
    "robust_max_categories": lambda: ct(pp.RobustScaler(), pp.OneHotEncoder(max_categories=3, handle_unknown="ignore")),
    "kbins_onehot_ordinal": lambda: ct(pp.KBinsDiscretizer(n_bins=5, encode="onehot", **BINS),
                                       pp.OrdinalEncoder(handle_unknown="use_encoded_value", unknown_value=-1)),
    "kbins_dense_uniform": lambda: ct(pp.KBinsDiscretizer(n_bins=4, encode="onehot-dense", strategy="uniform"),
                                      pp.OneHotEncoder(drop="if_binary", handle_unknown="ignore")),
    "kbins_ordinal_scaled": lambda: ct(make_pipeline(pp.KBinsDiscretizer(n_bins=3, encode="ordinal", **BINS),
                                                     pp.StandardScaler()),
                                       make_pipeline(pp.OrdinalEncoder(handle_unknown="use_encoded_value",
                                                                       unknown_value=np.nan),
                                                     SimpleImputer(strategy="most_frequent"), pp.OneHotEncoder())),
    "imputer_indicator_nested": lambda: ct(pp.StandardScaler(), pp.OneHotEncoder(handle_unknown="ignore"),
                                           nan=make_pipeline(SimpleImputer(strategy="median", add_indicator=True),
                                                             pp.MinMaxScaler(clip=True))),
    "imputer_then_kbins": lambda: ct(pp.StandardScaler(), pp.OneHotEncoder(handle_unknown="ignore"),
                                     nan=make_pipeline(SimpleImputer(strategy="constant", fill_value=-9.0),
                                                       pp.KBinsDiscretizer(n_bins=3, **BINS))),
    "remainder_passthrough_mask": lambda: ColumnTransformer(
        [("a", pp.StandardScaler(), np.array([True, False, False, False, True, False])),
         ("b", pp.OneHotEncoder(handle_unknown="ignore"), slice(2, 4)), ("c", SimpleImputer(), [-1])],
        remainder="passthrough"),
    "remainder_drop_nested_ct": lambda: make_pipeline(
        ColumnTransformer([("inner", ColumnTransformer([("s", pp.StandardScaler(), [0]),
                                                        ("o", pp.OneHotEncoder(), [1])]), [1, 3]),
                           ("imp", SimpleImputer(add_indicator=True), [5])], remainder="drop"),
        pp.MaxAbsScaler()),
}


def fitted(name, final=None, X=None, y=None):
    if X is None:
        X, y = raw_data()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe = make_pipeline(PIPELINES[name](), final if final is not None else LogisticRegression(max_iter=1000))
        pipe.fit(X, y)
    return pipe, X


def encoded_scores(pipe, X):
    """``pipe[:-1].transform(X) @ coef.T + intercept`` per row, NaN in the rows where the pipeline raises (or hands NaN
    to the model)."""
    def transform(A):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            T = pipe[:-1].transform(A)
        return T.toarray() if hasattr(T, "toarray") else np.asarray(T, dtype=np.float64)
    try:
        T = transform(X)
    except ValueError:                  # isolate the rows that raise
        rows = []
        for i in range(X.shape[0]):
            try:
                rows.append(transform(X[i:i + 1])[0])
            except ValueError:
                rows.append(None)
        width = next(len(r) for r in rows if r is not None)
        T = np.stack([r if r is not None else np.full(width, np.nan) for r in rows])
    est = pipe[-1]
    z = T @ np.atleast_2d(est.coef_).T + est.intercept_
    z[np.isnan(T).any(axis=1)] = np.nan
    return z


def probe_values(spec, col, X):
    """Random values, every breakpoint and its neighbours, every key, unseen values, NaN."""
    flags, keys, _, _ = spec.maps.column(col)
    vals = [X[~np.isnan(X[:, col]), col]]
    vals.append(np.random.default_rng(col).normal(size=50) * 4)
    for t in keys:
        vals.append([t, np.nextafter(t, -np.inf), np.nextafter(t, np.inf)])
    if flags & CATEGORICAL:
        vals.append([keys.min() - 1.0, keys.max() + 1.0, 0.5 * (keys[0] + keys[-1]) + 0.25])
    return np.unique(np.concatenate([np.asarray(v, dtype=np.float64).ravel() for v in vals]))


def check_columns(pipe, X):
    spec = extract_linear_spec(pipe.predict_proba if hasattr(pipe, "predict_proba") else pipe.predict)
    base = X[np.all(~np.isnan(X), axis=1)][0]
    for col in range(X.shape[1]):
        values = np.r_[probe_values(spec, col, X), np.nan]
        rows = np.repeat(base[None, :], len(values), axis=0)
        rows[:, col] = values
        want = encoded_scores(pipe, rows)
        refused = np.isnan(want).any(axis=1)
        for row in rows[refused]:
            with pytest.raises(ValueError):
                spec.maps.contributions(row[None, :])
        got = spec.maps.contributions(rows[~refused]) + spec.b
        scale = np.maximum(1.0, np.abs(want[~refused]).max(axis=1, keepdims=True))
        assert np.all(np.abs(got - want[~refused]) <= 1e-12 * scale), col
    return spec


@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_maps_equal_transform_times_coef_per_column(name):
    pipe, X = fitted(name)
    check_columns(pipe, X)


@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_spec_equals_predict_proba(name):
    pipe, X = fitted(name)
    spec = extract_linear_spec(pipe.predict_proba)
    ok = ~np.isnan(encoded_scores(pipe, X)).any(axis=1)
    np.testing.assert_allclose(spec(X[ok]), pipe.predict_proba(X[ok]), rtol=1e-12, atol=1e-14)


def test_minmax_clip_has_three_pieces_and_kbins_uses_inner_edges():
    pipe, X = fitted("minmax_clip_onehot_error")
    spec = extract_linear_spec(pipe.predict_proba)
    flags, keys, rows, _ = spec.maps.column(0)
    assert not flags & CATEGORICAL and len(keys) == 2 and rows.shape[0] == 3
    assert rows[0, 0, 0] == 0.0 and rows[2, 0, 0] == 0.0
    pipe, X = fitted("kbins_onehot_ordinal")
    spec = extract_linear_spec(pipe.predict_proba)
    kb = pipe[0].named_transformers_["num"]
    for i, col in enumerate(NUM):
        _, keys, rows, _ = spec.maps.column(col)
        np.testing.assert_array_equal(keys, kb.bin_edges_[i][1:-1])
        assert np.all(rows[:, 0, :] == 0.0)      # piecewise constant


FINALS = {
    "binary_logistic": (lambda: LogisticRegression(max_iter=1000), "binary", "predict_proba"),
    "softmax": (lambda: LogisticRegression(max_iter=1000), "multi", "predict_proba"),
    "one_vs_rest": (lambda: OneVsRestClassifier(LogisticRegression(max_iter=1000)), "multi", "predict_proba"),
    "decision_function": (lambda: LogisticRegression(max_iter=1000), "multi", "decision_function"),
    "ridge_1": (lambda: Ridge(alpha=0.5), "reg1", "predict"),
    "ridge_3": (lambda: Ridge(alpha=0.5), "reg3", "predict"),
    "linear": (lambda: LinearRegression(), "reg1", "predict"),
    "poisson": (lambda: PoissonRegressor(alpha=0.1, max_iter=500), "count", "predict"),
}


def targets(kind, X, seed=1):
    rng = np.random.default_rng(seed)
    s = np.nan_to_num(X[:, 0]) + 0.3 * X[:, 2] - 0.2 * X[:, 3] + rng.normal(size=len(X))
    if kind == "binary":
        return (s > 1).astype(int)
    if kind == "multi":
        return np.digitize(s, [0.5, 1.5, 2.5])
    if kind == "reg1":
        return s
    if kind == "reg3":
        return np.c_[s, 2 * s - X[:, 3], np.nan_to_num(X[:, 5])]
    return rng.poisson(np.exp(0.3 * np.clip(s, -3, 3)))


@pytest.mark.parametrize("final", sorted(FINALS))
def test_spec_equals_final_method(final):
    make, kind, method = FINALS[final]
    X, _ = raw_data()
    y = targets(kind, X)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe = make_pipeline(PIPELINES["imputer_indicator_nested"](), make()).fit(X, y)
    spec = extract_linear_spec(getattr(pipe, method))
    want = getattr(pipe, method)(X)
    np.testing.assert_allclose(spec(X).reshape(want.shape), want, rtol=1e-11, atol=1e-12)


@pytest.mark.parametrize("step", [
    lambda: PCA(n_components=2), lambda: pp.PolynomialFeatures(), lambda: pp.Normalizer(),
    lambda: pp.SplineTransformer(), lambda: pp.QuantileTransformer(n_quantiles=20), lambda: pp.PowerTransformer(),
    lambda: pp.FunctionTransformer(np.log1p), lambda: pp.TargetEncoder(target_type="binary"),
])
def test_refused_steps_raise_type_error_naming_them(step):
    X, y = raw_data()
    X = np.abs(np.nan_to_num(X))
    s = step()
    cols = [0, 1] if not isinstance(s, pp.TargetEncoder) else [2]
    pipe = make_pipeline(ColumnTransformer([("s", s, cols)], remainder="passthrough"), LogisticRegression(max_iter=500))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe.fit(X, y)
    with pytest.raises(TypeError, match=type(s).__name__):
        extract_linear_spec(pipe.predict_proba)


def test_string_categories_are_refused():
    rng = np.random.default_rng(0)
    X = rng.choice(["a", "b", "c"], size=(60, 1)).astype(object)
    y = (X[:, 0] == "a").astype(int)
    pipe = make_pipeline(pp.OneHotEncoder(), LogisticRegression()).fit(X, y)
    with pytest.raises(TypeError, match="string categories"):
        extract_linear_spec(pipe.predict_proba)


def test_column_selection_by_name_is_refused():
    pd = pytest.importorskip("pandas")
    X, y = raw_data()
    df = pd.DataFrame(np.nan_to_num(X), columns=[f"c{i}" for i in range(X.shape[1])])
    pipe = make_pipeline(ColumnTransformer([("s", pp.StandardScaler(), ["c0", "c1"])]), LogisticRegression())
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe.fit(df, y)
    with pytest.raises(TypeError, match="by name"):
        extract_linear_spec(pipe.predict_proba)


def test_plain_linear_model_keeps_the_w_path():
    X, y = raw_data()
    clf = LogisticRegression(max_iter=500).fit(np.nan_to_num(X), y)
    spec = extract_linear_spec(clf.predict_proba)
    assert spec.maps is None and spec.W.shape == (1, X.shape[1])
