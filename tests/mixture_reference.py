"""Float64 reference for KernelSHAP on the mixture head -- TEST INFRASTRUCTURE.

``multiclass_reference.MultiOutputReference`` with the head swapped for ``p = sum_k pi_k h(z_k)``: R = K R_m linear scores
stacked member-major, each member's head (binary ``[1 - expit(z), expit(z)]``, softmax, or one-vs-rest normalised
sigmoids) on its own R_m rows, the pi-weighted sum, then the same weighted background mean, link and constrained WLS per
output.  The masked scores keep the separable form ``base_j + sum_k Z[s, k] (XW[v_k] - BW[j, v_k])`` per score row."""
import numpy as np

from linear_reference import BLOCK, LinearReference, _link_f


def mixture_outputs(score, pi, member):
    """[..., K R_m] scores -> [..., C] mixture outputs (C = 2 for binary members, else R_m)."""
    pi = np.asarray(pi, dtype=np.float64)
    z = score.reshape(score.shape[:-1] + (len(pi), -1))
    if member == "binary_logistic":
        p1 = np.exp(-np.logaddexp(0.0, -z[..., 0]))
        out = np.stack([1.0 - p1, p1], axis=-1)
    elif member == "ovr":
        ls = -np.logaddexp(0.0, -z)
        e = np.exp(ls - ls.max(axis=-1, keepdims=True))
        out = e / e.sum(axis=-1, keepdims=True)
    else:
        e = np.exp(z - z.max(axis=-1, keepdims=True))
        out = e / e.sum(axis=-1, keepdims=True)
    return np.einsum("...kc,k->...c", out, pi)


class MixtureReference:
    """``W`` [K R_m, D], ``b`` [K R_m], ``pi`` [K], ``member`` head, ``background`` [N, D], ``groups`` list of column
    lists, ``weights`` [N] or None, ``link`` 'logit' / 'identity'."""

    def __init__(self, W, b, pi, member, background, groups, weights=None, link="logit"):
        self.W = np.atleast_2d(np.asarray(W, dtype=np.float64))
        self.b = np.atleast_1d(np.asarray(b, dtype=np.float64))
        self.pi, self.member = np.asarray(pi, dtype=np.float64), member
        self.bg = np.asarray(background, dtype=np.float64)
        self.groups = [np.asarray(g, dtype=np.int64) for g in groups]
        w = np.ones(self.bg.shape[0]) if weights is None else np.asarray(weights, dtype=np.float64)
        self.weights = w / np.sum(w)
        self.link = _link_f(link)
        self.BW = np.stack([self.bg[:, g] @ self.W[:, g].T for g in self.groups], axis=1)      # [N, G, R]
        self.base = self.b + self.bg @ self.W.T                                                 # [N, R]
        self.fnull = np.einsum("jc,j->c", self._outputs(self.base), self.weights)
        self.C = self.fnull.shape[0]
        self.expected_value = self.link(self.fnull)

    def _outputs(self, score):
        return mixture_outputs(score, self.pi, self.member)

    def predict(self, X):
        return self._outputs(self.b + np.asarray(X, dtype=np.float64) @ self.W.T)

    def varying(self, x):
        x = np.asarray(x, dtype=np.float64).reshape(-1)
        return np.asarray([k for k, g in enumerate(self.groups)
                           if np.any(~np.isclose(x[g][None, :], self.bg[:, g], equal_nan=True))], dtype=np.int64)

    def explain(self, x, plan=None, varying=None):
        """phi [G, C] of one instance for the plan ``(Z [S, M], w [S])`` over its varying groups."""
        x = np.asarray(x, dtype=np.float64).reshape(-1)
        v = self.varying(x) if varying is None else np.asarray(varying, dtype=np.int64)
        M, G = len(v), len(self.groups)
        XW = np.stack([x[g] @ self.W[:, g].T for g in self.groups])                            # [G, R]
        delta = self.link(self.predict(x[None, :])[0]) - self.link(self.fnull)
        phi = np.zeros((G, self.C))
        if M == 0:
            return phi
        if M == 1:
            phi[v[0]] = delta
            return phi
        Z, w = plan
        Z = np.asarray(Z).astype(np.float64)
        w = np.asarray(w, dtype=np.float64)
        D = XW[v][None, :, :] - self.BW[:, v, :]                                                # [N, M, R]
        ey = np.empty((len(w), self.C))
        for s0 in range(0, len(w), BLOCK):
            score = self.base[None, :, :] + np.einsum("sm,jmr->sjr", Z[s0:s0 + BLOCK], D)      # [block, N, R]
            ey[s0:s0 + BLOCK] = np.einsum("sjc,j->sc", self._outputs(score), self.weights)
        for c in range(self.C):
            phi[v, c] = LinearReference._solve(Z, w, self.link(ey[:, c]) - self.link(self.fnull[c]), delta[c])
        return phi
