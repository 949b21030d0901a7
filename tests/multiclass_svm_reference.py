"""An independent float64 reference for multi-class SVMs under the one-vs-one head.

``reference(spec)`` restates the definition in include/dks.h (``dks_set_svc_multiclass``) from the spec's arrays alone:
per member and support vector, the kernel statistic added column by column with the member's column weight and origin;
``K = phi(t)``; for pair k = (i, j), ``dec_k = sum_{v in class i} dual[v][j - 1] K + sum_{v in class j} dual[v][i] K +
intercept[m][k]``, support vectors found through the class offsets one row at a time; then the head (pair values, or
votes, confidences, per-class sigmoids, normalisation and the clip).  Nothing here calls ``sklearn.metrics.pairwise`` or
``MulticlassSvmSpec.__call__`` / ``pair_values``: a mistake in the product's NumPy evaluation is not inherited.
"""
import numpy as np


def _term(kernel, m, v, w, o):
    if kernel == "rbf":
        return w * (m - v) * (m - v)
    return w * (m - o) * (v - o)


def _phi(kernel, t, gamma, degree, coef0):
    if kernel == "rbf":
        return np.exp(-gamma * t)
    u = gamma * t + coef0
    return np.power(u, degree) if kernel == "poly" else np.tanh(u)


def _class_of(spec, m, v):
    off = spec.cls_off[m]
    for c in range(spec.classes):
        if off[c] <= v < off[c + 1]:
            return c
    raise AssertionError(f"support vector {v} is in no class block of member {m}")


def pair_values(spec, X):
    """dec [n, K, P], one support vector and one column at a time (vectorised over rows only)."""
    X = np.atleast_2d(np.asarray(X, dtype=np.float64))
    n, D = X.shape
    nc = spec.classes
    pairs = [(i, j) for i in range(nc) for j in range(i + 1, nc)]
    dec = np.zeros((n, spec.K, len(pairs)))
    for m in range(spec.K):
        for v in range(int(spec.sv_off[m]), int(spec.sv_off[m + 1])):
            t = np.zeros(n)
            for c in range(D):
                t = t + _term(spec.kernel, X[:, c], spec.sv[v, c], spec.colw[m, c], spec.colo[m, c])
            kv = _phi(spec.kernel, t, spec.gamma[m], spec.degree, spec.coef0)
            c = _class_of(spec, m, v)
            for k, (i, j) in enumerate(pairs):
                if c == i:
                    dec[:, m, k] += spec.dual[v, j - 1] * kv
                elif c == j:
                    dec[:, m, k] += spec.dual[v, i] * kv
        for k in range(len(pairs)):
            dec[:, m, k] += spec.intercept[m, k]
    return dec


def outputs(spec, X):
    dec = pair_values(spec, X)
    n = dec.shape[0]
    nc = spec.classes
    if spec.head == "ovo":
        out = dec[:, 0, :]
        return out[:, 0] if spec.scalar_out else out
    out = np.zeros((n, nc))
    for m in range(spec.K):
        for r in range(n):
            votes = [0.0] * nc
            conf = [0.0] * nc
            k = 0
            for i in range(nc):
                for j in range(i + 1, nc):
                    d = dec[r, m, k]
                    if d >= 0:
                        votes[i] += 1.0
                    else:
                        votes[j] += 1.0
                    conf[i] += d
                    conf[j] -= d
                    k += 1
            e = []
            for c in range(nc):
                f = votes[c] + conf[c] / (3.0 * (abs(conf[c]) + 1.0))
                z = spec.cal_a[m, c] * f + spec.cal_b[m, c]
                e.append(1.0 / (1.0 + np.exp(z)) if z < 700 else 0.0)
            s = sum(e)
            for c in range(nc):
                p = e[c] / s if s != 0 else 1.0 / nc
                if 1.0 < p <= 1.0 + 1e-5:
                    p = 1.0
                out[r, c] += spec.pi[m] * p
    return out[:, 0] if spec.scalar_out else out


def min_abs_pair_value(spec, X):
    """min |dec| over every row of X and every member and pair: a vote flip cannot hide in rounding when it is large."""
    return float(np.abs(pair_values(spec, X)).min())


def reference(spec):
    """The model as a callable (for the oracle and for comparisons)."""
    return lambda X: outputs(spec, X)
