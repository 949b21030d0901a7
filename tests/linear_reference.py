"""Fast float64 reference for KernelSHAP on linear-score models -- TEST INFRASTRUCTURE.

Same semantics as ``oracle.shap_kernel_oracle.KernelExplainerOracle.explain(plan=...)`` for a linear model followed by
the binary-logistic head (``predict_proba``) or the identity head (``decision_function``), without the ``S*N x D``
masked batch the oracle builds.  For a linear model the masked score separates:

    score(s, j) = base_j + sum_k Z[s, k] (XW[v_k] - BW[j, v_k]),    base_j = intercept + bg_j . coef,

where XW[g] / BW[j, g] are the grouped contributions of the instance / background row j and v the varying groups.
Everything after the score follows upstream's float64 formulas line by line: the probabilities through
``LinearModelSpec.__call__`` (softmax of [-t/2, t/2], t = kappa * score, with the max subtracted), ``ey`` as the
weighted background mean, the link ``log(x / (1 - x))`` (not a more accurate one: the engine computes delta with the
same formula, so the reference must too) and the constrained WLS of ``KernelExplainerOracle._solve`` (last varying group
eliminated, ``inv(E^T W E)``, |phi| < 1e-10 snapped to 0).  Cost per instance: one [S, M] x [M, N] product and 2 S N
exponentials, evaluated BLOCK coalitions at a time so that the temporaries stay a few MB whatever S is -- S = 65534,
N = 128 takes about a tenth of a second, where the oracle would need a 100 GB batch."""
import numpy as np

BLOCK = 4096        # coalitions per block of the score / probability evaluation


def _link_f(link):
    if link == "logit":
        return lambda p: np.log(p / (1 - p))
    if link == "identity":
        return lambda p: p
    raise ValueError(f"unknown link {link!r}")


class LinearReference:
    """``coef`` [D] or [1, D], ``intercept`` scalar, ``background`` [N, D], ``groups`` list of column lists, ``weights``
    [N] (None: uniform; normalised to sum 1 like ``DenseData``).  ``head``: 'logistic' (two outputs [p0, p1] with
    p1 = sigmoid(kappa * score); kappa = 2 is scikit-learn 0.23's binary multinomial model) or 'identity' (one output,
    the score itself: a scalar ``decision_function``).  ``link``: 'logit' or 'identity'."""

    def __init__(self, coef, intercept, background, groups, weights=None, head="logistic", kappa=2.0, link="logit"):
        self.coef = np.asarray(coef, dtype=np.float64).reshape(-1)
        self.intercept = float(np.asarray(intercept, dtype=np.float64).reshape(-1)[0])
        self.bg = np.asarray(background, dtype=np.float64)
        self.groups = [np.asarray(g, dtype=np.int64) for g in groups]
        w = np.ones(self.bg.shape[0]) if weights is None else np.asarray(weights, dtype=np.float64)
        self.weights = w / np.sum(w)
        if head not in ("logistic", "identity"):
            raise ValueError(f"unknown head {head!r}")
        self.head, self.kappa = head, float(kappa)
        self.link = _link_f(link)
        self.C = 2 if head == "logistic" else 1
        self.BW = np.stack([self.bg[:, g] @ self.coef[g] for g in self.groups], axis=1)          # [N, G]
        self.base = self.intercept + self.bg @ self.coef                                         # [N]
        f_bg = self._outputs(self.base[None, :])[0]                                             # [N, C]
        self.fnull = np.sum((f_bg.T * self.weights).T, 0)
        self.expected_value = self.link(self.fnull)

    def _outputs(self, score):
        """Model outputs [..., C] of linear scores [...], as ``LinearModelSpec.__call__`` computes them."""
        if self.head == "identity":
            return score[..., None]
        t = self.kappa * score
        a, b = -t / 2.0, t / 2.0
        m = np.maximum(a, b)
        e0, e1 = np.exp(a - m), np.exp(b - m)
        s = e0 + e1
        return np.stack([e0 / s, e1 / s], axis=-1)

    def varying(self, x):
        """Upstream's ``varying_groups``: groups where some background row differs from x (np.isclose, NaN == NaN)."""
        x = np.asarray(x, dtype=np.float64).reshape(-1)
        out = [k for k, g in enumerate(self.groups)
               if np.any(~np.isclose(x[g][None, :], self.bg[:, g], equal_nan=True))]
        return np.asarray(out, dtype=np.int64)

    def explain(self, x, plan=None, varying=None):
        """phi [G, C] of one instance for the coalition plan ``(Z [S, M], w [S])`` over the varying groups (``varying``:
        their indices, default upstream's rule).  M < 2 needs no plan."""
        x = np.asarray(x, dtype=np.float64).reshape(-1)
        v = self.varying(x) if varying is None else np.asarray(varying, dtype=np.int64)
        M, G = len(v), len(self.groups)
        XW = np.array([x[g] @ self.coef[g] for g in self.groups])
        fx = self._outputs(np.array([self.intercept + x @ self.coef]))[0]
        delta = self.link(fx) - self.link(self.fnull)
        phi = np.zeros((G, self.C))
        if M == 0:
            return phi
        if M == 1:
            phi[v[0]] = delta
            return phi
        Z, w = plan
        Z = np.asarray(Z).astype(np.float64)
        w = np.asarray(w, dtype=np.float64)
        assert Z.shape == (len(w), M), "plan must be [S, M] / [S] for this instance"
        DT = (XW[v][None, :] - self.BW[:, v]).T                                                 # [M, N]
        ey = np.empty((len(w), self.C))
        for s0 in range(0, len(w), BLOCK):
            score = self.base[None, :] + Z[s0:s0 + BLOCK] @ DT                                  # [block, N]
            # the oracle's reduction, term for term: with 70 groups the WLS turns a last-bit difference in ey into 1e-8
            ey[s0:s0 + BLOCK] = np.einsum("sjc,j->sc", self._outputs(score), self.weights)
        for c in range(self.C):
            phi[v, c] = self._solve(Z, w, self.link(ey[:, c]) - self.link(self.fnull[c]), delta[c])
        return phi

    @staticmethod
    def _solve(Z, w, eyAdj, delta):
        """``KernelExplainerOracle._solve`` without the l1 branch."""
        M = Z.shape[1]
        eyAdj2 = eyAdj - Z[:, -1] * delta
        etmp = Z[:, :-1] - Z[:, -1][:, None]
        tmp = etmp * w[:, None]
        wsol = np.linalg.inv(tmp.T @ etmp) @ (tmp.T @ eyAdj2)
        phi = np.zeros(M)
        phi[:-1] = wsol
        phi[-1] = delta - sum(wsol)
        phi[np.abs(phi) < 1e-10] = 0.0
        return phi

    def shap_values(self, X, plans):
        """phi [n, G, C] for rows X with one plan per row (``plans[i]``: ``(Z, w)``, or None for M < 2)."""
        X = np.atleast_2d(np.asarray(X, dtype=np.float64))
        return np.stack([self.explain(X[i], plans[i]) for i in range(X.shape[0])])
