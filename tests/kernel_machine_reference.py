"""An independent float64 reference for kernel machines.

``reference(spec)`` restates the definition in include/dks.h (``dks_set_kernel_machine``) from the spec's arrays alone: per
member, support vector and column, the term ``h(x_c, v_c)`` with the member's column weight and origin, added column by
column into ``t``; ``K = phi(t)``; ``f_k = sum_v dual[v] K + intercept_k``; then the head.  Nothing here calls
``sklearn.metrics.pairwise`` or ``KernelMachineSpec.__call__`` / ``scores``: a mistake in the product's NumPy evaluation is
not inherited.  phi comes from the oracle (oracle/shap_kernel_oracle.py) fed ``reference(spec)`` and the engine's plan.
"""
import numpy as np


def _term(kernel, m, v, w, o):
    if kernel == "rbf":
        return w * (m - v) * (m - v)
    if kernel == "laplacian":
        return w * np.abs(m - v)
    return w * (m - o) * (v - o)


def _phi(kernel, t, gamma, degree, coef0):
    if kernel in ("rbf", "laplacian"):
        return np.exp(-gamma * t)
    u = gamma * t + coef0
    return np.power(u, degree) if kernel == "poly" else np.tanh(u)


def member_scores(spec, X):
    """f [n, K, R], one support vector and one column at a time (vectorised over rows only)."""
    X = np.atleast_2d(np.asarray(X, dtype=np.float64))
    n, D = X.shape
    f = np.zeros((n, spec.K, spec.R))
    for k in range(spec.K):
        for v in range(int(spec.sv_off[k]), int(spec.sv_off[k + 1])):
            t = np.zeros(n)
            for c in range(D):
                t = t + _term(spec.kernel, X[:, c], spec.sv[v, c], spec.colw[k, c], spec.colo[k, c])
            kv = _phi(spec.kernel, t, spec.gamma[k], spec.degree, spec.coef0)
            for q in range(spec.R):
                f[:, k, q] += spec.dual[v, q] * kv
        f[:, k, :] += spec.intercept[k]
    return f


def outputs(spec, X):
    f = member_scores(spec, X)
    if spec.head == "calibrated":
        p1 = np.zeros(f.shape[0])
        for k in range(spec.K):
            z = spec.cal_a[k] * f[:, k, 0] + spec.cal_b[k]
            with np.errstate(over="ignore"):
                p1 += spec.pi[k] / (1.0 + np.exp(z))
        out = np.stack([1.0 - p1, p1], axis=1)
    else:
        out = f[:, 0, :]
    return out[:, 0] if spec.scalar_out else out


def reference(spec):
    """The model as a callable (for the oracle and for comparisons)."""
    return lambda X: outputs(spec, X)
