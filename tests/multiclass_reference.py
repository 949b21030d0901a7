"""Float64 reference for KernelSHAP on linear models with C outputs -- TEST INFRASTRUCTURE.

``linear_reference.LinearReference`` covers the binary-logistic head and the scalar identity head.  This one covers the
softmax head over C = R linear scores (``LinearSoftmaxClassifier.predict_proba`` with C >= 3 classes) and the identity
head with R outputs (``decision_function`` of a multi-output linear model), with the same semantics as
``oracle.shap_kernel_oracle.KernelExplainerOracle.explain(plan=...)``: per coalition and background row the masked
scores ``base_j + sum_k Z[s, k] (XW[v_k] - BW[j, v_k])`` per output, the head, the weighted background mean, the link
``log(x / (1 - x))`` and the constrained WLS per output (last varying group eliminated, |phi| < 1e-10 snapped to 0)."""
import numpy as np

from linear_reference import BLOCK, LinearReference, _link_f


class MultiOutputReference:
    """``W`` [R, D], ``b`` [R], ``background`` [N, D], ``groups`` list of column lists, ``weights`` [N] or None.
    ``head``: 'softmax' (C = R >= 2 class probabilities) or 'identity' (the R scores).  ``link``: 'logit' / 'identity'."""

    def __init__(self, W, b, background, groups, weights=None, head="softmax", link="logit"):
        self.W = np.atleast_2d(np.asarray(W, dtype=np.float64))
        self.b = np.atleast_1d(np.asarray(b, dtype=np.float64))
        self.bg = np.asarray(background, dtype=np.float64)
        self.groups = [np.asarray(g, dtype=np.int64) for g in groups]
        w = np.ones(self.bg.shape[0]) if weights is None else np.asarray(weights, dtype=np.float64)
        self.weights = w / np.sum(w)
        if head not in ("softmax", "identity"):
            raise ValueError(f"unknown head {head!r}")
        self.head = head
        self.link = _link_f(link)
        self.C = self.W.shape[0]
        self.BW = np.stack([self.bg[:, g] @ self.W[:, g].T for g in self.groups], axis=1)      # [N, G, C]
        self.base = self.b + self.bg @ self.W.T                                                 # [N, C]
        self.fnull = np.einsum("jc,j->c", self._outputs(self.base), self.weights)
        self.expected_value = self.link(self.fnull)

    def _outputs(self, score):
        """Model outputs [..., C] of scores [..., C], as ``LinearModelSpec.__call__`` computes them."""
        if self.head == "identity":
            return score
        e = np.exp(score - score.max(axis=-1, keepdims=True))
        return e / e.sum(axis=-1, keepdims=True)

    def varying(self, x):
        x = np.asarray(x, dtype=np.float64).reshape(-1)
        return np.asarray([k for k, g in enumerate(self.groups)
                           if np.any(~np.isclose(x[g][None, :], self.bg[:, g], equal_nan=True))], dtype=np.int64)

    def explain(self, x, plan=None, varying=None):
        """phi [G, C] of one instance for the plan ``(Z [S, M], w [S])`` over its varying groups."""
        x = np.asarray(x, dtype=np.float64).reshape(-1)
        v = self.varying(x) if varying is None else np.asarray(varying, dtype=np.int64)
        M, G = len(v), len(self.groups)
        XW = np.stack([x[g] @ self.W[:, g].T for g in self.groups])                            # [G, C]
        delta = self.link(self._outputs(self.b + x @ self.W.T)) - self.link(self.fnull)
        phi = np.zeros((G, self.C))
        if M == 0:
            return phi
        if M == 1:
            phi[v[0]] = delta
            return phi
        Z, w = plan
        Z = np.asarray(Z).astype(np.float64)
        w = np.asarray(w, dtype=np.float64)
        D = XW[v][None, :, :] - self.BW[:, v, :]                                                # [N, M, C]
        ey = np.empty((len(w), self.C))
        for s0 in range(0, len(w), BLOCK):
            score = self.base[None, :, :] + np.einsum("sm,jmc->sjc", Z[s0:s0 + BLOCK], D)      # [block, N, C]
            ey[s0:s0 + BLOCK] = np.einsum("sjc,j->sc", self._outputs(score), self.weights)
        for c in range(self.C):
            phi[v, c] = LinearReference._solve(Z, w, self.link(ey[:, c]) - self.link(self.fnull[c]), delta[c])
        return phi
