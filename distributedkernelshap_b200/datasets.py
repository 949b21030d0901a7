"""Synthetic stand-ins for the reference's datasets (no network here: the Adult pickles of
explainers/utils.py:14-19 are unreachable).  Shapes follow SURVEY.md §8(d).

``adult_like``: D = 49 encoded columns = 4 standardised numeric + 8 one-hot blocks (``drop='first'``) of widths
[8, 6, 3, 8, 5, 4, 1, 10] (scripts/process_adult_data.py:58-60, :77-122, :184-218), 12 groups, 2560 instances to
explain, first 100 "training" rows as background, a 2-class multinomial logistic-regression head
(scripts/fit_adult_model.py:27-32).  Everything is drawn from ``numpy.random.default_rng(seed)``.
"""
import numpy as np

from .predictors import LinearSoftmaxClassifier

ADULT_NUMERIC = ["Age", "Capital Gain", "Capital Loss", "Hours per week"]
ADULT_CATEGORICAL = ["Workclass", "Education", "Marital Status", "Occupation", "Relationship", "Race", "Sex", "Country"]
ADULT_ONEHOT_WIDTHS = [8, 6, 3, 8, 5, 4, 1, 10]


def _onehot_block(rng, n_rows, width, probs):
    """One categorical variable with width + 1 levels, first level dropped (all-zero row)."""
    levels = rng.choice(width + 1, size=n_rows, p=probs)
    block = np.zeros((n_rows, width))
    rows = np.nonzero(levels > 0)[0]
    block[rows, levels[rows] - 1] = 1.0
    return block


def adult_like(n_explain=2560, n_background=100, seed=0):
    """Returns ``{'data': <dict shaped like the reference's load_data()>, 'predictor': classifier, 'groups': ...,
    'group_names': ..., 'X_explain': [n, 49], 'background': [N, 49]}``."""
    rng = np.random.default_rng(seed)
    n_total = n_background + n_explain
    cols = [rng.standard_normal((n_total, len(ADULT_NUMERIC)))]
    for width in ADULT_ONEHOT_WIDTHS:
        probs = rng.dirichlet(np.ones(width + 1))
        cols.append(_onehot_block(rng, n_total, width, probs))
    X = np.concatenate(cols, axis=1)
    D = X.shape[1]

    groups, start = [], 0
    for _ in ADULT_NUMERIC:
        groups.append([start])
        start += 1
    for width in ADULT_ONEHOT_WIDTHS:
        groups.append(list(range(start, start + width)))
        start += width
    group_names = ADULT_NUMERIC + ADULT_CATEGORICAL

    coef = rng.normal(0.0, 0.5, size=(1, D))
    intercept = rng.normal(0.0, 1.0, size=(1,))
    predictor = LinearSoftmaxClassifier(coef, intercept, multi_class="multinomial")

    background = X[:n_background]
    X_explain = X[n_background:]
    y = predictor.predict(X_explain)
    from scipy import sparse
    data = {
        "all": {
            "X": {"raw": {"train": None, "test": None},
                  "processed": {"train": sparse.csr_matrix(background), "test": sparse.csr_matrix(X_explain)}},
            "y": {"train": predictor.predict(background), "test": y},
            "groups": groups,
            "group_names": group_names,
            "orig_feature_names": group_names,
        },
        "background": {"X": {"raw": None, "preprocessed": sparse.csr_matrix(background)},
                       "y": predictor.predict(background)},
    }
    return {"data": data, "predictor": predictor, "groups": groups, "group_names": group_names,
            "X_explain": X_explain, "background": background}


def dense_tabular(n, n_features, n_background, seed=0, dtype=np.float64):
    """Configs [2] and [4] of BASELINE.json: X, bg ~ N(0, 1), one group per column, 2-class multinomial LR."""
    rng = np.random.default_rng(seed)
    background = rng.standard_normal((n_background, n_features)).astype(dtype)
    X = rng.standard_normal((n, n_features)).astype(dtype)
    coef = rng.normal(0.0, 1.0 / np.sqrt(n_features), size=(1, n_features))
    intercept = rng.normal(0.0, 1.0, size=(1,))
    predictor = LinearSoftmaxClassifier(coef, intercept, multi_class="multinomial")
    return {"predictor": predictor, "X_explain": X, "background": background,
            "groups": [[i] for i in range(n_features)], "group_names": [f"f{i}" for i in range(n_features)]}


def wide_onehot(n, n_blocks=64, block_width=16, n_background=256, seed=0, singleton_groups=False):
    """Config [3] of BASELINE.json (SURVEY.md §8d): ``n_blocks`` categorical variables one-hot encoded without dropping a
    level (``n_blocks * block_width`` columns), 2-class LR.  Grouped reading (default): one group per variable, level
    probabilities ~ Dirichlet(1).  ``singleton_groups=True`` is the other reading -- every column its own group
    (M = D = 1024) -- with uniform level probabilities, so that every column takes both values in the background and
    all M groups vary for every instance (with skewed levels a column that is 0 in the whole background and in x does
    not vary, and the varying sets differ from instance to instance)."""
    rng = np.random.default_rng(seed)
    D = n_blocks * block_width

    def draw(rows):
        out = np.zeros((rows, D))
        for b in range(n_blocks):
            probs = np.full(block_width, 1.0 / block_width) if singleton_groups else rng.dirichlet(np.ones(block_width))
            levels = rng.choice(block_width, size=rows, p=probs)
            out[np.arange(rows), b * block_width + levels] = 1.0
        return out

    both = draw(n_background + n)
    coef = rng.normal(0.0, 0.5, size=(1, D))
    intercept = rng.normal(0.0, 1.0, size=(1,))
    predictor = LinearSoftmaxClassifier(coef, intercept, multi_class="multinomial")
    if singleton_groups:
        groups = [[c] for c in range(D)]
        names = [f"var{c // block_width}={c % block_width}" for c in range(D)]
    else:
        groups = [list(range(b * block_width, (b + 1) * block_width)) for b in range(n_blocks)]
        names = [f"var{b}" for b in range(n_blocks)]
    return {"predictor": predictor, "X_explain": both[n_background:], "background": both[:n_background],
            "groups": groups, "group_names": names}


def decode_onehot_blocks(A, n_numeric, widths, drop_first):
    """Raw columns of an encoded matrix: the ``n_numeric`` leading columns as they are, then one level code per one-hot
    block of ``widths`` (``drop_first``: an all-zero block is level 0 and column k is level k + 1; else column k is level
    k)."""
    cols, start = [A[:, :n_numeric]], n_numeric
    for w in widths:
        block = A[:, start:start + w]
        code = block.argmax(axis=1) + (1 if drop_first else 0)
        if drop_first:
            code = np.where(block.any(axis=1), code, 0)
        cols.append(code[:, None].astype(np.float64))
        start += w
    return np.hstack(cols)


def raw_space_pipeline(predictor, raw, n_numeric, widths, drop_first):
    """A fitted scikit-learn ``Pipeline(ColumnTransformer(StandardScaler, OneHotEncoder(drop='first' | None)),
    LogisticRegression)`` over the raw columns of ``decode_onehot_blocks`` that computes what the encoded two-class
    ``predictor`` (``LinearSoftmaxClassifier``, p1 = sigmoid(2 z)) computes: its coefficients, with the scaler folded
    back in.  This is how such a model ships (the reference's Adult model, scripts/process_adult_data.py)."""
    from sklearn.compose import ColumnTransformer
    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import OneHotEncoder, StandardScaler
    num = list(range(n_numeric))
    cats = [np.arange(w + (1.0 if drop_first else 0.0)) for w in widths]
    parts = [("cat", OneHotEncoder(drop="first" if drop_first else None, categories=cats),
              list(range(n_numeric, n_numeric + len(widths))))]
    if n_numeric:
        parts.insert(0, ("num", StandardScaler(), num))
    ct = ColumnTransformer(parts).fit(raw)
    lr = LogisticRegression().fit(ct.transform(raw)[:4], [0, 1, 0, 1])
    coef, b = predictor.coef_[0], float(predictor.intercept_[0])
    if n_numeric:
        sc = ct.named_transformers_["num"]
        coef = np.r_[coef[:n_numeric] * sc.scale_, coef[n_numeric:]]
        b += float(predictor.coef_[0, :n_numeric] @ sc.mean_)
    lr.coef_, lr.intercept_ = 2.0 * coef[None, :], np.array([2.0 * b])
    return Pipeline([("prep", ct), ("clf", lr)])
