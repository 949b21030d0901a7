"""Gaussian generative models of scikit-learn read into component scores (``GaussianModelSpec``) for the device's Gaussian
route.

A spec is what ``dks_set_gaussian_model`` takes (include/dks.h): K <= 8 components scored as

    l_k(x) = c_k - gamma_k ||L_k^T (x - mu_k)||^2          (L_k: D x r_k)

and a fixed head over the scores:

* ``softmax``: ``QuadraticDiscriminantAnalysis``, ``GaussianNB``, ``GaussianMixture`` and ``BayesianGaussianMixture``
  ``predict_proba``;
* ``logsumexp``: the mixtures' ``score_samples`` (the log density);
* ``identity``: multi-class QDA ``decision_function`` and ``EllipticEnvelope`` ``decision_function`` / ``score_samples``
  (one component, ``gamma = 1``: minus the Mahalanobis distance, less ``offset_`` for ``decision_function``);
* ``diff``: binary QDA ``decision_function``, ``l_1 - l_0``.

What each model contributes:

* QDA: ``L_k = rotations_[k] scalings_[k]^-1/2``, ``gamma = 1/2``, ``c_k = log priors_k - 1/2 sum log scalings_[k]``;
* GaussianNB: ``L_k = diag(var_[k]^-1/2)``, ``gamma = 1/2``, ``c_k = log class_prior_k - 1/2 sum log(2 pi var_[k])``;
* the mixtures, every ``covariance_type``: ``L_k`` from ``precisions_cholesky_`` (full: the matrix, tied: the shared
  one, diag: its diagonal, spherical: a multiple of the identity), ``gamma = 1/2`` and ``c_k = -D/2 log(2 pi) +
  log det L_k + log weights_k``; a ``BayesianGaussianMixture`` adds its degrees-of-freedom and digamma constants and takes
  the expected log weights of its weight prior in place of ``log weights_k``;
* EllipticEnvelope: ``L = V diag(w)^1/2`` from the eigendecomposition ``precision_ = V diag(w) V^T``.

A ``Pipeline`` of per-column affine scalers in front folds into ``mu`` and ``L`` (``x' = a x + b``:
``L^T (x' - mu) = (diag(a) L)^T (x - (mu - b) / a)``).  ``GaussianModelSpec.__call__`` evaluates the scores and the head
in NumPy, in float64, the softmax and logsumexp shifted by the largest score.
"""
import numpy as np

from .kernel_machines import _final, _names, _unwrap

MAX_COMPONENTS = 8
MAX_GROUPS = 64
HEADS = ("softmax", "logsumexp", "identity", "diff")     # DKS_GAUSS_HEAD_* codes 0..3
# a precision eigenvalue below -NEG_EIG_RTOL times the largest one is a real negative eigenvalue, not rounding
NEG_EIG_RTOL = 1e-10

_QDA = {"QuadraticDiscriminantAnalysis"}
_NB = {"GaussianNB"}
_GMM = {"GaussianMixture", "BayesianGaussianMixture"}
_EE = {"EllipticEnvelope"}
_GAUSSIAN = _QDA | _NB | _GMM | _EE
# estimators that hold other estimators: a Gaussian model inside one of them is refused by name
_CONTAINERS = {"VotingClassifier", "VotingRegressor", "BaggingClassifier", "BaggingRegressor", "CalibratedClassifierCV",
               "StackingClassifier", "StackingRegressor", "OneVsRestClassifier", "OneVsOneClassifier",
               "MultiOutputRegressor", "MultiOutputClassifier", "AdaBoostClassifier"}


class GaussianModelSpec:
    """K component scores ``l_k = c_k - gamma_k ||L_k^T (x - mu_k)||^2`` and a head in ``HEADS``.

    mu [K, D], L: a list of K arrays [D, r_k], gamma [K], c [K]."""

    activation = "gauss"
    act_code = 13         # DKS_ACT_GAUSS
    maps = None

    def __init__(self, mu, L, gamma, c, head, n_features, scalar_out=False):
        self.mu = np.ascontiguousarray(np.atleast_2d(np.asarray(mu, dtype=np.float64)))
        self.K, D = self.mu.shape
        self.L = [np.asarray(Lk, dtype=np.float64).reshape(D, -1) for Lk in L]
        self.gamma = np.ascontiguousarray(np.asarray(gamma, dtype=np.float64).reshape(self.K))
        self.c = np.ascontiguousarray(np.asarray(c, dtype=np.float64).reshape(self.K))
        self.head = head
        self.n_features = int(n_features)
        self.scalar_out = bool(scalar_out)
        if head not in HEADS:
            raise ValueError(f"unknown Gaussian head {head!r}")
        if not 1 <= self.K <= MAX_COMPONENTS:
            raise NotImplementedError(f"{self.K} components or classes: Gaussian models are explained with at most "
                                      f"{MAX_COMPONENTS}")
        if head == "diff" and self.K != 2:
            raise ValueError("the difference head needs two components")
        if len(self.L) != self.K or any(Lk.shape[1] < 1 for Lk in self.L):
            raise ValueError("one projection of rank >= 1 per component")
        if not (np.all(np.isfinite(self.mu)) and all(np.all(np.isfinite(Lk)) for Lk in self.L)
                and np.all(np.isfinite(self.c)) and np.all(np.isfinite(self.gamma)) and np.all(self.gamma > 0)):
            raise NotImplementedError("a Gaussian model with non-finite means, precisions or constants")
        self.n_outputs = self.K if head in ("softmax", "identity") else 1
        self.R = self.K       # score rows: the component scores the head reads

    @property
    def head_code(self):
        return HEADS.index(self.head)

    def flat(self):
        """(r_off [K + 1] int32, L [r_off[K], D]: the columns of every L_k as rows), as ``dks_set_gaussian_model`` takes
        them."""
        r_off = np.zeros(self.K + 1, dtype=np.int32)
        r_off[1:] = np.cumsum([Lk.shape[1] for Lk in self.L])
        return r_off, np.ascontiguousarray(np.concatenate([Lk.T for Lk in self.L], axis=0))

    def scores(self, X):
        """The component scores l [n, K]."""
        X = np.atleast_2d(np.asarray(X, dtype=np.float64))
        if not np.all(np.isfinite(X)):
            raise ValueError("a row holds NaN or an infinity: Gaussian models refuse it, as scikit-learn does")
        out = np.empty((X.shape[0], self.K))
        for k in range(self.K):
            u = (X - self.mu[k]) @ self.L[k]
            out[:, k] = self.c[k] - self.gamma[k] * np.sum(u * u, axis=1)
        return out

    def __call__(self, X):
        """The model's outputs [n, C] under the head (a 1-D array for one output)."""
        l = self.scores(X)
        if self.head == "identity":
            out = l
        elif self.head == "diff":
            out = l[:, 1:2] - l[:, 0:1]
        else:
            mx = l.max(axis=1, keepdims=True)
            e = np.exp(l - mx)
            s = e.sum(axis=1, keepdims=True)
            out = mx + np.log(s) if self.head == "logsumexp" else e / s
        return out[:, 0] if self.scalar_out else out


def _contains_gaussian(obj, depth=0):
    if depth > 6 or obj is None or isinstance(obj, str):
        return False
    if _names(obj) & _GAUSSIAN:
        return True
    for attr in ("steps", "estimators", "estimators_", "calibrated_classifiers_", "estimator", "base_estimator",
                 "estimator_", "final_estimator", "final_estimator_"):
        v = getattr(obj, attr, None)
        if v is None or isinstance(v, str):
            continue
        kids = list(np.ravel(np.asarray(v, dtype=object))) if isinstance(v, (list, tuple, np.ndarray)) else [v]
        for e in kids:
            if _contains_gaussian(e[-1] if isinstance(e, tuple) else e, depth + 1):
                return True
    return False


def refuse_gaussian_members(predictor):
    """Raises ``NotImplementedError`` when ``predictor`` is a method of an ensemble (possibly behind a ``Pipeline``) that
    holds a Gaussian model: those are explained on their own, not as members."""
    owner = getattr(predictor, "__self__", None)
    if owner is None:
        return
    est = _final(owner)
    if _names(est) & _CONTAINERS and _contains_gaussian(est):
        raise NotImplementedError(f"{type(est).__name__} holding a Gaussian model (QDA, GaussianNB, a Gaussian mixture or "
                                  "EllipticEnvelope): Gaussian models inside an ensemble are not supported; pass the "
                                  "Gaussian model's own method")


def _qda(est, method):
    K = len(est.classes_)
    if method == "predict_proba":
        head = "softmax"
    elif method == "decision_function":
        head = "diff" if K == 2 else "identity"
    else:
        raise TypeError(f"QuadraticDiscriminantAnalysis.{method} is not supported: pass predict_proba or "
                        "decision_function" + (" (predict returns labels)" if method == "predict" else ""))
    if K > MAX_COMPONENTS:
        raise NotImplementedError(f"QuadraticDiscriminantAnalysis with {K} classes: Gaussian models are explained with at "
                                  f"most {MAX_COMPONENTS}")
    L, c = [], []
    for k in range(K):
        S = np.asarray(est.scalings_[k], dtype=np.float64)
        if not (np.all(np.isfinite(S)) and np.all(S > 0)):
            raise NotImplementedError(f"QuadraticDiscriminantAnalysis: class {k} has a zero or non-finite scaling (its "
                                      "covariance is singular; scikit-learn's scores are not finite): set reg_param > 0")
        L.append(np.asarray(est.rotations_[k], dtype=np.float64) * S ** -0.5)
        c.append(np.log(est.priors_[k]) - 0.5 * np.sum(np.log(S)))
    return np.asarray(est.means_, dtype=np.float64), L, np.full(K, 0.5), np.asarray(c), head, head == "diff"


def _nb(est, method):
    if method != "predict_proba":
        raise TypeError(f"GaussianNB.{method} is not supported: pass predict_proba"
                        + (" (predict returns labels)" if method == "predict" else ""))
    K = len(est.classes_)
    if K > MAX_COMPONENTS:
        raise NotImplementedError(f"GaussianNB with {K} classes: Gaussian models are explained with at most "
                                  f"{MAX_COMPONENTS}")
    var = np.asarray(est.var_, dtype=np.float64)
    if not (np.all(np.isfinite(var)) and np.all(var > 0)):
        raise NotImplementedError("GaussianNB with a zero or non-finite variance is not supported")
    L = [np.diag(var[k] ** -0.5) for k in range(K)]
    c = np.log(est.class_prior_) - 0.5 * np.sum(np.log(2.0 * np.pi * var), axis=1)
    return np.asarray(est.theta_, dtype=np.float64), L, np.full(K, 0.5), c, "softmax", False


def _mixture(est, method):
    name = type(est).__name__
    if method not in ("predict_proba", "score_samples"):
        raise TypeError(f"{name}.{method} is not supported: pass predict_proba or score_samples"
                        + (" (predict returns labels)" if method == "predict" else ""))
    mu = np.asarray(est.means_, dtype=np.float64)
    K, D = mu.shape
    if K > MAX_COMPONENTS:
        raise NotImplementedError(f"{name} with {K} components: Gaussian models are explained with at most "
                                  f"{MAX_COMPONENTS}")
    P = np.asarray(est.precisions_cholesky_, dtype=np.float64)
    ct = est.covariance_type
    if ct == "full":
        L = [P[k] for k in range(K)]
        logdet = np.array([np.sum(np.log(np.diag(P[k]))) for k in range(K)])
    elif ct == "tied":
        L = [P] * K
        logdet = np.full(K, np.sum(np.log(np.diag(P))))
    elif ct == "diag":
        L = [np.diag(P[k]) for k in range(K)]
        logdet = np.sum(np.log(P), axis=1)
    else:
        L = [P[k] * np.eye(D) for k in range(K)]
        logdet = D * np.log(P)
    c = -0.5 * D * np.log(2 * np.pi) + logdet
    if "BayesianGaussianMixture" in _names(est):
        from scipy.special import digamma
        dof = np.asarray(est.degrees_of_freedom_, dtype=np.float64)
        log_lambda = D * np.log(2.0) + np.sum(digamma(0.5 * (dof - np.arange(0, D)[:, np.newaxis])), 0)
        c = c - 0.5 * D * np.log(dof) + 0.5 * (log_lambda - D / np.asarray(est.mean_precision_, dtype=np.float64))
        wc = est.weight_concentration_
        if est.weight_concentration_prior_type == "dirichlet_process":
            dsum = digamma(wc[0] + wc[1])
            logw = digamma(wc[0]) - dsum + np.hstack((0, np.cumsum(digamma(wc[1]) - dsum)[:-1]))
        else:
            logw = digamma(wc) - digamma(np.sum(wc))
    else:
        logw = np.log(est.weights_)
    c = c + logw
    head = "softmax" if method == "predict_proba" else "logsumexp"
    return mu, L, np.full(K, 0.5), c, head, head == "logsumexp"


def _envelope(est, method):
    if method not in ("decision_function", "score_samples"):
        raise TypeError(f"EllipticEnvelope.{method} is not supported: pass decision_function or score_samples"
                        + (" (predict returns labels)" if method == "predict" else ""))
    w, V = np.linalg.eigh(np.asarray(est.get_precision(), dtype=np.float64))
    if w.min() < -NEG_EIG_RTOL * max(np.abs(w).max(), np.finfo(np.float64).tiny):
        raise NotImplementedError(f"EllipticEnvelope: its precision has a negative eigenvalue ({w.min():.3g}), so its "
                                  "Mahalanobis distance is not a sum of squares")
    L = V * np.sqrt(np.maximum(w, 0.0))
    c = -float(est.offset_) if method == "decision_function" else 0.0
    return np.asarray(est.location_, dtype=np.float64)[None, :], [L], np.ones(1), np.array([c]), "identity", True


def extract_gaussian_spec(predictor):
    """``GaussianModelSpec`` of a bound method of a fitted Gaussian generative model -- ``QuadraticDiscriminantAnalysis``
    (``predict_proba``, ``decision_function``), ``GaussianNB`` (``predict_proba``), ``GaussianMixture`` and
    ``BayesianGaussianMixture`` (``predict_proba``, ``score_samples``), ``EllipticEnvelope`` (``decision_function``,
    ``score_samples``) -- each possibly behind a ``Pipeline`` of per-column affine scalers, and ``None`` for anything
    else.  A spec passes through.  Raises ``TypeError`` for the other methods (``predict`` returns labels;
    ``predict_log_proba``, ``score``) and ``NotImplementedError`` naming the reason for more than 8 classes or components,
    a singular QDA class, a precision with a negative eigenvalue, pipeline steps other than the four scalers and Gaussian
    models inside an ensemble."""
    if isinstance(predictor, GaussianModelSpec):
        return predictor
    owner = getattr(predictor, "__self__", None)
    method = getattr(predictor, "__name__", None)
    if owner is None:
        return None
    est = _final(owner)
    names = _names(est)
    if not names & _GAUSSIAN:
        refuse_gaussian_members(predictor)
        return None
    name = type(est).__name__
    if not hasattr(est, "n_features_in_"):
        raise TypeError(f"{name} is not fitted")
    P = int(owner.n_features_in_)
    try:
        _, a, b = _unwrap(owner, P, family="Gaussian model", target="its means and precisions")
    except NotImplementedError as e:
        raise NotImplementedError(f"{name}: {e}") from e
    read = _qda if names & _QDA else _nb if names & _NB else _mixture if names & _GMM else _envelope
    mu, L, gamma, c, head, scalar = read(est, method)
    mu = (mu - b) / a
    L = [a[:, None] * Lk for Lk in L]
    return GaussianModelSpec(mu, L, gamma, c, head, P, scalar_out=scalar)
