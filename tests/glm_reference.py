"""Float64 reference for KernelSHAP on log-link GLM regressors (``predict = exp(x . coef + intercept)``) -- TEST
INFRASTRUCTURE.

Same semantics as ``oracle.shap_kernel_oracle.KernelExplainerOracle.explain(plan=...)`` with the identity link, without the
``S*N x D`` masked batch.  The masked score separates as for every linear model (``tests/linear_reference.py``),
``score(s, j) = a(s) + d(s, j)`` with ``a(s) = sum_{k in s} XW[v_k]`` and ``d(s, j) = base_j - sum_{k in s} BW[j, v_k]``, and the
exponential factorises:

    ey(s) = sum_j w_j exp(a(s) + d(s, j)) = exp(a(s) + l(s)),    l(s) = ln sum_j w_j exp(d(s, j)).

``l(s)`` is a max-shifted log-sum-exp over the background rows with positive weight.  With a partial varying set ``v`` the
columns subtracted in ``d`` are those of ``v``, so ``l`` depends on the instance's varying set, not only on the plan."""
import numpy as np

from linear_reference import LinearReference

BLOCK = 4096        # coalitions per block of the [S, N] exponent matrix


class ExpReference:
    """``coef`` [D], ``intercept`` scalar, ``background`` [N, D], ``groups`` list of column lists, ``weights`` [N] (None:
    uniform; normalised to sum 1).  One output, identity link."""

    def __init__(self, coef, intercept, background, groups, weights=None):
        self.coef = np.asarray(coef, dtype=np.float64).reshape(-1)
        self.intercept = float(np.asarray(intercept, dtype=np.float64).reshape(-1)[0])
        self.bg = np.asarray(background, dtype=np.float64)
        self.groups = [np.asarray(g, dtype=np.int64) for g in groups]
        w = np.ones(self.bg.shape[0]) if weights is None else np.asarray(weights, dtype=np.float64)
        self.weights = w / np.sum(w)
        self.BW = np.stack([self.bg[:, g] @ self.coef[g] for g in self.groups], axis=1)          # [N, G]
        self.base = self.intercept + self.bg @ self.coef                                         # [N]
        self.fnull = float(np.sum(self.weights * np.exp(self.base)))
        self.expected_value = self.fnull

    def predict(self, X):
        return np.exp(self.intercept + np.atleast_2d(np.asarray(X, dtype=np.float64)) @ self.coef)

    def varying(self, x):
        x = np.asarray(x, dtype=np.float64).reshape(-1)
        return np.asarray([k for k, g in enumerate(self.groups)
                           if np.any(~np.isclose(x[g][None, :], self.bg[:, g], equal_nan=True))], dtype=np.int64)

    def log_e(self, Z, v):
        """l(s) for the rows of ``Z`` [S, M] over the varying groups ``v``: zero-weight rows skipped, max-shifted."""
        pos = self.weights > 0
        wl = np.log(self.weights[pos])
        out = np.empty(Z.shape[0])
        for s0 in range(0, Z.shape[0], BLOCK):
            d = self.base[pos][None, :] - Z[s0:s0 + BLOCK] @ self.BW[pos][:, v].T + wl[None, :]      # [block, N+]
            m = d.max(axis=1)
            out[s0:s0 + BLOCK] = m + np.log(np.exp(d - m[:, None]).sum(axis=1))
        return out

    def explain(self, x, plan=None, varying=None):
        """phi [G] of one instance for the plan ``(Z [S, M], w [S])`` over its varying groups."""
        x = np.asarray(x, dtype=np.float64).reshape(-1)
        v = self.varying(x) if varying is None else np.asarray(varying, dtype=np.int64)
        M, G = len(v), len(self.groups)
        XW = np.array([x[g] @ self.coef[g] for g in self.groups])
        delta = float(np.exp(self.intercept + x @ self.coef)) - self.fnull
        phi = np.zeros(G)
        if M == 0:
            return phi
        if M == 1:
            phi[v[0]] = delta
            return phi
        Z, w = plan
        Z = np.asarray(Z).astype(np.float64)
        w = np.asarray(w, dtype=np.float64)
        assert Z.shape == (len(w), M), "plan must be [S, M] / [S] for this instance"
        ey = np.exp(Z @ XW[v] + self.log_e(Z, v))
        phi[v] = LinearReference._solve(Z, w, ey - self.fnull, delta)
        return phi
