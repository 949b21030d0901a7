"""Tree models behind per-column preprocessing (``trees.extract_tree_pipeline_spec``): the compiled column encoding
replays ``pipe[:-1].transform`` bit for bit on adversarial raw values (bin edges and their float64 neighbours, values
landing on the fitted tree's split thresholds and one ulp either side, clip bounds, +-inf where the pipeline accepts it,
NaN, unseen and infrequent categories), the spec on the encoded rows reproduces the pipeline's method, and the refusals
raise with their messages.  CPU only."""
import warnings

import numpy as np
import pytest

sklearn = pytest.importorskip("sklearn")
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.ensemble import (GradientBoostingClassifier, HistGradientBoostingClassifier,  # noqa: E402
                              HistGradientBoostingRegressor, RandomForestClassifier, VotingClassifier)
from sklearn.impute import SimpleImputer  # noqa: E402
from sklearn.linear_model import LogisticRegression  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import (KBinsDiscretizer, MaxAbsScaler, MinMaxScaler, OneHotEncoder,  # noqa: E402
                                   OrdinalEncoder, PolynomialFeatures, RobustScaler, StandardScaler)
from sklearn.tree import DecisionTreeClassifier, DecisionTreeRegressor  # noqa: E402

from distributedkernelshap_b200 import column_maps as cm  # noqa: E402
from distributedkernelshap_b200.trees import extract_tree_pipeline_spec, extract_tree_spec  # noqa: E402

NUM, NANCOL, CAT = [0, 1], 2, [3, 4]       # raw layout: two numeric columns, one numeric with NaN, two categorical


def raw_data(seed, n, nan_cat=False, nan=True):
    rng = np.random.default_rng(seed)
    X = np.empty((n, 5))
    X[:, 0] = rng.normal(3.0, 2.0, n)
    X[:, 1] = rng.uniform(-5.0, 40.0, n)
    X[:, 2] = rng.normal(0.0, 1.0, n)
    if nan:
        X[rng.random(n) < 0.1, 2] = np.nan
    X[:, 3] = rng.choice([0.0, 1.0, 2.0, 5.0], n, p=[0.4, 0.3, 0.27, 0.03])   # 5: an infrequent level
    X[:, 4] = rng.integers(0, 4, n).astype(float)
    if nan_cat:
        X[rng.random(n) < 0.08, 4] = np.nan
    y = ((X[:, 0] > 3) ^ (X[:, 3] == 1) ^ (np.nan_to_num(X[:, 2]) > 0.3)).astype(int)
    return X, y


def ct(*parts, remainder="drop"):
    return ColumnTransformer(list(parts), remainder=remainder, sparse_threshold=0.0)


IMP = [NANCOL]
PIPES = {
    "standard_onehot": lambda: ct(("num", StandardScaler(), NUM), ("cat", OneHotEncoder(handle_unknown="ignore"), CAT),
                                  remainder="passthrough"),
    "standard_no_mean_no_std": lambda: ct(("a", StandardScaler(with_mean=False), [0]),
                                          ("b", StandardScaler(with_std=False), [1]), ("c", "passthrough", CAT)),
    "robust_maxabs": lambda: ct(("a", RobustScaler(), [0]), ("b", MaxAbsScaler(), [1]), ("c", "passthrough", [3])),
    "minmax_clip": lambda: ct(("a", MinMaxScaler(clip=True), NUM), ("b", MinMaxScaler(), [0]),
                              ("c", OrdinalEncoder(), CAT)),
    "imputer_indicator": lambda: ct(("i", make_pipeline(SimpleImputer(add_indicator=True), StandardScaler()), [2, 0]),
                                    ("c", "passthrough", CAT)),
    "onehot_drop_error": lambda: ct(("n", "passthrough", NUM),
                                    ("c", OneHotEncoder(drop="first", handle_unknown="error"), CAT)),
    "onehot_infrequent": lambda: ct(("n", "passthrough", NUM),
                                    ("c", OneHotEncoder(min_frequency=20, handle_unknown="infrequent_if_exist"), CAT)),
    "ordinal_unknown_missing": lambda: ct(("n", "passthrough", slice(0, 2)),
                                          ("c", OrdinalEncoder(handle_unknown="use_encoded_value", unknown_value=-1,
                                                               encoded_missing_value=-2), CAT)),
    "kbins_ordinal_onehot": lambda: ct(("o", KBinsDiscretizer(5, encode="ordinal", quantile_method="averaged_inverted_cdf"),
                                        [0]),
                                       ("h", KBinsDiscretizer(4, encode="onehot-dense", strategy="uniform"), [1]),
                                       ("c", "passthrough", CAT)),
    "kbins_then_onehot": lambda: ct(("k", make_pipeline(KBinsDiscretizer(4, encode="ordinal", strategy="uniform"),
                                                        OneHotEncoder(sparse_output=False)), [1]),
                                    ("n", StandardScaler(), [0])),
    "onehot_then_scaler": lambda: ct(("c", make_pipeline(OneHotEncoder(sparse_output=False), MaxAbsScaler()), [4]),
                                     ("n", "passthrough", [0])),
    "bool_selector_remainder": lambda: ct(("n", StandardScaler(), np.array([True, True, False, False, False])),
                                          ("c", OneHotEncoder(handle_unknown="ignore"), [-2, -1]),
                                          remainder=make_pipeline(SimpleImputer(), MinMaxScaler(clip=True))),
    "column_in_encoder_and_scaler": lambda: ct(("c", OneHotEncoder(handle_unknown="ignore"), [3]),
                                               ("n", StandardScaler(), [3, 0])),
}
NAN_CAT = {"ordinal_unknown_missing"}


def fitted(name, model=None, nan_cat=False, nan=True):
    X, y = raw_data(0, 300, nan_cat=nan_cat or name in NAN_CAT, nan=nan)
    model = model if model is not None else DecisionTreeClassifier(max_depth=7, random_state=0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe = make_pipeline(PIPES[name](), model).fit(X, y)
    return pipe, X


def dense_transform(pipe, X):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = pipe[:-1].transform(X)
    return np.asarray(out.toarray() if hasattr(out, "toarray") else out, dtype=np.float64)


def _invert(enc, e, v):
    """A raw value the scalar ops of encoded column e map near v (ops undone in reverse; lookups skipped)."""
    _, first, count = enc.hdr[e]
    for k in range(first + count - 1, first - 1, -1):
        code, c0 = enc.ops[k][0], enc.opvals[k][0]
        if code == cm.OP_SUB:
            v = v + c0
        elif code == cm.OP_DIV:
            v = v * c0
        elif code == cm.OP_MUL:
            v = v / c0
        elif code == cm.OP_ADD:
            v = v - c0
    return v


def adversarial_rows(pipe, enc, X):
    """Rows of X with one raw value replaced by an adversarial one."""
    base = X[:6]
    spec_tree = pipe[-1]
    vals = {c: [np.nan, np.inf, -np.inf, 99.0, 5.0, -1.0, 0.0, -0.0] for c in range(X.shape[1])}
    tree = getattr(spec_tree, "tree_", None)
    if tree is not None:
        for f, thr in zip(tree.feature, tree.threshold):
            if f < 0:
                continue
            r = _invert(enc, f, float(thr))
            vals[int(enc.hdr[f, 0])] += [r] + [np.nextafter(r, s * np.inf) for s in (-1, 1)] + \
                [np.nextafter(np.nextafter(r, s * np.inf), s * np.inf) for s in (-1, 1)]
    for step in pipe[:-1].named_steps.values():
        for name, t, cols in getattr(step, "transformers_", []):
            idx = list(range(X.shape[1]))[cols] if isinstance(cols, slice) else \
                [i for i, b in enumerate(cols) if b] if np.asarray(cols).dtype == bool else [int(c) % 5 for c in cols]
            last = t.steps[0][1] if hasattr(t, "steps") else t
            for j, c in enumerate(idx):
                if isinstance(last, KBinsDiscretizer):
                    for edge in last.bin_edges_[j]:
                        vals[c] += [edge, np.nextafter(edge, -np.inf), np.nextafter(edge, np.inf)]
                if isinstance(last, MinMaxScaler):
                    for b in (last.data_min_[j], last.data_max_[j]):
                        vals[c] += [b, np.nextafter(b, -np.inf), np.nextafter(b, np.inf), b * 3 + 1, -3 * b - 1]
    rows = []
    for c, vs in vals.items():
        for v in vs:
            r = base[len(rows) % len(base)].copy()
            r[c] = v
            rows.append(r)
    return np.asarray(rows)


def accepted(pipe, rows):
    ok = np.zeros(len(rows), dtype=bool)
    for i, r in enumerate(rows):
        try:
            dense_transform(pipe, r[None, :])
            ok[i] = True
        except ValueError:
            pass
    return ok


@pytest.mark.parametrize("name", sorted(PIPES))
def test_encoding_is_bit_exact(name):
    pipe, X = fitted(name)
    spec, enc = extract_tree_pipeline_spec(pipe.predict_proba)
    assert enc.D == 5 and spec.n_features == 5
    assert np.array_equal(enc.transform(X), dense_transform(pipe, X), equal_nan=True)
    rows = adversarial_rows(pipe, enc, X)
    ok = accepted(pipe, rows)
    assert ok.sum() > len(rows) // 3
    got, want = enc.transform(rows[ok]), dense_transform(pipe, rows[ok])
    assert np.array_equal(got, want, equal_nan=True), np.argwhere(~((got == want) | (np.isnan(got) & np.isnan(want))))
    # the spec on the encoded rows is the pipeline's method (on the rows this tree model itself accepts: finite ones)
    fin = np.isfinite(got).all(axis=1)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        np.testing.assert_allclose(spec(got[fin]), pipe.predict_proba(rows[ok][fin]), rtol=1e-12, atol=1e-12)
    # what the pipeline refuses, the evaluator refuses (unseen categories under 'error', NaN into an encoder without
    # a NaN category); +-inf is the exception: scikit-learn's input validation refuses it, the encoding computes on it
    for r in rows[~ok]:
        if np.isinf(r).any():
            continue
        with pytest.raises(ValueError, match="refuses"):
            enc.transform(r[None, :])


@pytest.mark.parametrize("model, method", [
    (HistGradientBoostingClassifier(max_iter=15, random_state=0), "predict_proba"),
    (HistGradientBoostingRegressor(max_iter=15, loss="poisson", random_state=0), "predict"),
    (GradientBoostingClassifier(n_estimators=10, max_depth=2, random_state=0), "decision_function"),
    (RandomForestClassifier(8, max_depth=5, random_state=0), "predict_proba"),
    (DecisionTreeRegressor(max_depth=5, random_state=0), "predict"),
])
def test_spec_on_encoded_rows_equals_pipeline(model, method):
    nan = not isinstance(model, GradientBoostingClassifier)       # the others split on NaN themselves
    pipe, X = fitted("standard_onehot", model=model, nan=nan)
    fn = getattr(pipe, method)
    spec, enc = extract_tree_pipeline_spec(fn)
    Xt, _ = raw_data(1, 80, nan=nan)
    Xt[0, 3] = 7.0                                      # unseen under handle_unknown='ignore'
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = fn(Xt)
    np.testing.assert_allclose(spec(enc.transform(Xt)), want, rtol=1e-12, atol=1e-12)


def test_not_a_tree_pipeline_is_none():
    X, y = raw_data(0, 100, nan=False)
    lin = make_pipeline(PIPES["standard_onehot"](), LogisticRegression()).fit(X, y)
    assert extract_tree_pipeline_spec(lin.predict_proba) is None
    tree = DecisionTreeClassifier(max_depth=2).fit(X[:, :2], y)
    assert extract_tree_pipeline_spec(tree.predict_proba) is None


def test_refusals():
    X, y = raw_data(0, 200, nan=False)
    with pytest.raises(NotImplementedError, match="Pipeline"):          # the bare-tree reader still refuses a Pipeline
        extract_tree_spec(make_pipeline(StandardScaler(), DecisionTreeClassifier()).fit(X, y).predict_proba)
    poly = make_pipeline(ct(("p", PolynomialFeatures(2), NUM)), DecisionTreeClassifier()).fit(X, y)
    with pytest.raises(TypeError, match="PolynomialFeatures"):
        extract_tree_pipeline_spec(poly.predict_proba)
    f32 = make_pipeline(ct(("c", OneHotEncoder(dtype=np.float32), CAT)), DecisionTreeClassifier()).fit(X, y)
    with pytest.raises(TypeError, match="float32"):
        extract_tree_pipeline_spec(f32.predict_proba)
    vote = make_pipeline(StandardScaler(), VotingClassifier([("a", DecisionTreeClassifier()), ("b", LogisticRegression())],
                                                            voting="soft")).fit(X[:, :3] * 0 + 1, y)
    assert extract_tree_pipeline_spec(vote.predict_proba) is None
    with pytest.raises(NotImplementedError, match="ensemble"):
        extract_tree_spec(vote.predict_proba)
    hgb_cat = make_pipeline(ct(("n", "passthrough", [0, 3])),
                            HistGradientBoostingClassifier(max_iter=3, categorical_features=[1])).fit(X, y)
    with pytest.raises(NotImplementedError, match="categorical"):
        extract_tree_pipeline_spec(hgb_cat.predict_proba)
    with pytest.raises(TypeError, match="predict_proba"):
        extract_tree_pipeline_spec(make_pipeline(StandardScaler(), DecisionTreeClassifier()).fit(X[:, :2], y).predict)


def test_linear_merge_rule_stays_for_column_maps():
    """A raw column feeding an encoder and a scaler: a tree reads it, the linear column maps still refuse it."""
    pipe, X = fitted("column_in_encoder_and_scaler")
    lin = make_pipeline(PIPES["column_in_encoder_and_scaler"](), LogisticRegression()).fit(*raw_data(0, 300, nan=False))
    pre, est = cm.pipeline_parts(lin)
    with pytest.raises(TypeError, match="feeds both"):
        cm.compile_maps(pre, 5, est.coef_)
    spec, enc = extract_tree_pipeline_spec(pipe.predict_proba)
    assert sorted(set(enc.sources.tolist())) == [0, 3]
