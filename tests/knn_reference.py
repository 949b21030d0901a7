"""Float64 NumPy evaluation of a k-nearest-neighbour model, written apart from ``neighbors.KnnSpec`` for the tests to compare
both the spec and the device against.

Per query row: the row in the fitted space ``x' = colw * x + colo``, per training row the statistic summed over the columns
in order (0 where ``x'`` equals the training row column for column, at least 2^-1000 otherwise), the ``k`` training rows
of smallest ``(statistic, index)``, then scikit-learn's vote or mean of their labels or targets with ``uniform`` or
``distance`` weights (the neighbours at distance 0 alone count when there are any)."""
import numpy as np


def _stat(spec, xs, v):
    t = 0.0
    for c in range(v.shape[0]):
        d = xs[c] - v[c]
        if spec.metric in ("euclidean", "sqeuclidean"):
            t = t + d * d
        elif spec.metric == "manhattan":
            t = t + abs(d)
        else:
            t = t + abs(d) ** spec.p
    return 0.0 if np.array_equal(xs, v) else max(t, 2.0 ** -1000)


def _dist(spec, t):
    if spec.metric == "euclidean":
        return np.sqrt(t)
    if spec.metric == "minkowski":
        return t ** (1.0 / spec.p)
    return t


def neighbours(spec, x):
    """[(statistic, index)] of the k nearest training rows of one raw row, in rank order."""
    xs = np.asarray(x, dtype=np.float64) * spec.colw + spec.colo
    ranked = sorted((_stat(spec, xs, spec.fitX[v]), v) for v in range(spec.fitX.shape[0]))
    return ranked[:spec.k]


def predict_row(spec, x):
    nb = neighbours(spec, x)
    if spec.weights == "uniform":
        w = [1.0] * len(nb)
    else:
        d = [_dist(spec, t) for t, _ in nb]
        if any(di == 0.0 for di in d):
            w = [1.0 if di == 0.0 else 0.0 for di in d]
        else:
            w = [1.0 / di for di in d]
    if spec.head == "classify":
        s = np.zeros(spec.R)
        for wi, (_, v) in zip(w, nb):
            s[int(spec.y[v])] += wi
        return s / (float(spec.k) if spec.weights == "uniform" else sum(s[c] for c in range(spec.R)))
    num = np.zeros(spec.R)
    den = 0.0
    for wi, (_, v) in zip(w, nb):
        num = num + spec.y[v] * wi
        den += wi
    return num / (float(spec.k) if spec.weights == "uniform" else den)


def reference(spec):
    """The model as a callable of raw rows [n, D] -> [n, R] (1-D for a single-target regressor)."""
    def fn(X):
        X = np.atleast_2d(np.asarray(X, dtype=np.float64))
        out = np.stack([predict_row(spec, x) for x in X]) if X.shape[0] else np.zeros((0, spec.R))
        return out[:, 0] if spec.scalar_out else out
    return fn
