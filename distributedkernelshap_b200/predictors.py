"""The model side of the hot path: linear scores followed by a probability head.

The reference passes an opaque Python callable (``clf.predict_proba`` of a scikit-learn
``LogisticRegression(multi_class='multinomial')``, benchmarks/ray_pool.py:34, scripts/fit_adult_model.py:27-32).
CUDA kernels cannot call Python, so the engine needs the callable's parameters.  ``extract_linear_spec``
recovers them from the bound method's owner and ``GpuKernelExplainer`` checks the recovered model against the
callable on the background rows before trusting it; anything else raises (there is no CPU fallback)."""
import numpy as np

from . import _cabi


class LinearModelSpec:
    """``z = X W^T + b`` then a head.  ``W`` is [R, D], ``b`` [R].  With ``maps`` (a ``column_maps.ColumnMaps``; ``W`` is
    then None) the scores are ``z = b + sum_col f_col(X[:, col])``: a linear model behind per-column preprocessing.

    activation: 'identity' (outputs z), 'binary_logistic' (R == 1; outputs [1 - s, s], s = sigmoid(kappa z)),
    'softmax' (outputs softmax(z), R = C >= 2), 'ovr' (one-vs-rest, R = C >= 3: s_c = sigmoid(z_c), outputs
    s_c / sum_c' s_c', scikit-learn's ``_predict_proba_lr``; kappa 1), 'exp' (R = 1: outputs exp(z), the ``predict`` of
    scikit-learn's log-link GLM regressors).  ``scalar_out``: the callable returns a 1-D array."""

    def __init__(self, W, b, activation, kappa=1.0, scalar_out=False, maps=None):
        self.b = np.ascontiguousarray(np.atleast_1d(np.asarray(b, dtype=np.float64)))
        self.maps = maps
        if maps is None:
            self.W = np.ascontiguousarray(np.atleast_2d(np.asarray(W, dtype=np.float64)))
            R = self.W.shape[0]
        else:
            self.W = None           # the scores are b + maps.contributions(x) (column_maps.py)
            R = maps.R
        if R != self.b.shape[0]:
            raise ValueError(f"W has {R} rows but b has {self.b.shape[0]} entries")
        if activation not in ("identity", "binary_logistic", "softmax", "ovr", "exp"):
            raise ValueError(f"unknown activation {activation!r}")
        if activation == "binary_logistic" and R != 1:
            raise ValueError("binary_logistic needs a single score row")
        if activation == "exp" and R != 1:
            raise ValueError("the exp head needs a single score row (log-link models with several outputs are not supported)")
        if activation == "ovr" and (R < 3 or float(kappa) != 1.0):
            raise ValueError("the one-vs-rest head needs at least three score rows and kappa = 1")
        self.activation = activation
        self.kappa = float(kappa)
        self.scalar_out = bool(scalar_out)

    @property
    def R(self):
        """Score rows."""
        return self.b.shape[0]

    @property
    def n_features(self):
        """Raw input columns the model reads."""
        return self.maps.D if self.maps is not None else self.W.shape[1]

    @property
    def act_code(self):
        return {"identity": _cabi.ACT_IDENTITY, "binary_logistic": _cabi.ACT_BINARY_LOGISTIC,
                "softmax": _cabi.ACT_SOFTMAX, "ovr": _cabi.ACT_OVR, "exp": _cabi.ACT_EXP}[self.activation]

    @property
    def n_outputs(self):
        return 2 if self.activation == "binary_logistic" else self.R

    def __call__(self, X):
        """NumPy evaluation with scikit-learn's conventions (used on the host by build_explanation and tests)."""
        X = np.asarray(X, dtype=np.float64)
        if X.ndim == 1:
            X = X.reshape(1, -1)
        z = (self.maps.contributions(X) if self.maps is not None else X @ self.W.T) + self.b
        if self.activation == "identity":
            return z[:, 0] if self.scalar_out else z
        if self.activation == "exp":
            e = np.exp(z)
            return e[:, 0] if self.scalar_out else e
        if self.activation == "binary_logistic":
            t = self.kappa * z[:, 0]
            scores = np.c_[-t / 2.0, t / 2.0]
        elif self.activation == "ovr":
            # _predict_proba_lr (scikit-learn 0.23.2): expit of each score, then each row divided by its sum
            p = np.exp(-np.logaddexp(0.0, -z))
            return p / p.sum(axis=1, keepdims=True)
        else:
            scores = z
        scores = scores - scores.max(axis=1, keepdims=True)
        e = np.exp(scores)
        return e / e.sum(axis=1, keepdims=True)


class LinearSoftmaxClassifier:
    """Minimal stand-in for the fitted scikit-learn 0.23 ``LogisticRegression(multi_class='multinomial')`` the
    reference pickles (scripts/fit_adult_model.py:27-32): ``coef_`` [1, D] / ``intercept_`` [1] for two classes
    with ``predict_proba = softmax([-z, z])`` (so p1 = sigmoid(2 z)), or [C, D] / [C] with a plain softmax.
    ``multi_class='ovr'`` with C >= 3 classes: the one-vs-rest head (normalised per-class sigmoids)."""

    def __init__(self, coef, intercept, multi_class="multinomial"):
        self.coef_ = np.atleast_2d(np.asarray(coef, dtype=np.float64))
        self.intercept_ = np.atleast_1d(np.asarray(intercept, dtype=np.float64))
        self.multi_class = multi_class
        self.classes_ = np.arange(2 if self.coef_.shape[0] == 1 else self.coef_.shape[0])

    def dks_linear_spec(self):
        if self.coef_.shape[0] == 1:
            return LinearModelSpec(self.coef_, self.intercept_, "binary_logistic",
                                   kappa=2.0 if self.multi_class == "multinomial" else 1.0)
        if self.multi_class == "ovr":
            return LinearModelSpec(self.coef_, self.intercept_, "ovr")
        if self.multi_class != "multinomial":
            raise NotImplementedError(f"multi_class={self.multi_class!r} is not supported")
        return LinearModelSpec(self.coef_, self.intercept_, "softmax")

    def decision_function(self, X):
        z = np.asarray(X, dtype=np.float64) @ self.coef_.T + self.intercept_
        return z[:, 0] if z.shape[1] == 1 else z

    def predict_proba(self, X):
        return self.dks_linear_spec()(X)

    def predict(self, X):
        return self.classes_[np.argmax(self.predict_proba(X), axis=1)]


def extract_linear_spec(predictor):
    """Recover ``LinearModelSpec`` from what the reference hands to ``KernelShap`` (a callable).

    Accepts: a ``LinearModelSpec``; any object/bound method whose owner offers ``dks_linear_spec()``; bound
    ``predict_proba`` / ``decision_function`` / ``predict`` of scikit-learn linear models (``coef_``/``intercept_``);
    bound ``predict_proba`` of a single-label ``OneVsRestClassifier`` over at least three binary linear models; bound
    ``predict`` of the log-link GLM regressors (``_is_log_link_glm``), whose head is 'exp'; the same methods of a fitted
    scikit-learn ``Pipeline`` whose transformers act on one column at a time and whose final step is any of the above
    (``_pipeline_spec``: the model is read in raw feature space through column maps).
    Raises ``TypeError`` for everything else."""
    if isinstance(predictor, LinearModelSpec):
        return predictor
    owner = getattr(predictor, "__self__", None)
    method = getattr(predictor, "__name__", None)
    if owner is None and hasattr(predictor, "dks_linear_spec"):
        return predictor.dks_linear_spec()
    if owner is None:
        raise TypeError("predictor must be a bound method of a linear model (e.g. clf.predict_proba) or a "
                        "LinearModelSpec: the CUDA engine cannot call an opaque Python function and has no CPU fallback")
    if _is_sklearn_pipeline(owner):
        return _pipeline_spec(owner, method)
    if hasattr(owner, "dks_linear_spec") and (method == "predict_proba" or
                                              (method == "predict" and not hasattr(owner, "classes_"))):
        return owner.dks_linear_spec()     # a regressor's predict (e.g. a log-link GLM stand-in) takes the hook too
    if hasattr(owner, "estimators_") and not hasattr(owner, "coef_"):
        return _one_vs_rest_spec(owner, method)
    if not (hasattr(owner, "coef_") and hasattr(owner, "intercept_")):
        raise TypeError(f"{type(owner).__name__} exposes no coef_/intercept_: only linear models are supported")
    coef = np.atleast_2d(np.asarray(owner.coef_, dtype=np.float64))
    intercept = np.atleast_1d(np.asarray(owner.intercept_, dtype=np.float64))
    if method == "predict_proba":
        if coef.shape[0] == 1:
            mc = getattr(owner, "multi_class", "auto")
            # scikit-learn >= 1.5 binary problems: sigmoid(z); 0.23 'multinomial' binary: softmax([-z, z])
            kappa = 2.0 if mc == "multinomial" else 1.0
            return LinearModelSpec(coef, intercept, "binary_logistic", kappa=kappa)
        if _is_ovr_rule(owner):
            return LinearModelSpec(coef, intercept, "ovr")
        return LinearModelSpec(coef, intercept, "softmax")
    if method in ("decision_function", "predict", "_decision_function"):
        if method == "predict" and hasattr(owner, "classes_"):
            raise TypeError("classifier.predict returns labels, which KernelSHAP cannot explain; pass predict_proba")
        if method == "predict" and _is_log_link_glm(owner):
            return LinearModelSpec(coef, intercept, "exp", scalar_out=True)
        return LinearModelSpec(coef, intercept, "identity", scalar_out=coef.shape[0] == 1)
    raise TypeError(f"unsupported predictor method {method!r}")


def _is_sklearn_pipeline(owner):
    return any(c.__name__ == "Pipeline" and c.__module__.startswith("sklearn.") for c in type(owner).__mro__)


def _pipeline_spec(pipe, method):
    """A Pipeline's ``method`` as column maps over its raw columns (``column_maps.compile_maps``) followed by the head
    its final estimator's ``method`` has.  The final estimator's intercept becomes ``b``."""
    from .column_maps import compile_maps, pipeline_parts
    pre, final = pipeline_parts(pipe)
    bound = getattr(final, method, None)
    if bound is None:
        raise TypeError(f"{type(final).__name__} has no {method}")
    inner = extract_linear_spec(bound)
    n_raw = getattr(pipe, "n_features_in_", None)
    if n_raw is None:
        raise TypeError("the Pipeline is not fitted (no n_features_in_)")
    maps = compile_maps(pre, int(n_raw), inner.W)
    return LinearModelSpec(None, inner.b, inner.activation, kappa=inner.kappa, scalar_out=inner.scalar_out, maps=maps)


def _is_log_link_glm(owner):
    """scikit-learn's GLM regressors (0.23 and later) whose ``predict`` is ``exp(X coef_ + intercept_)``:
    ``PoissonRegressor``, ``GammaRegressor``, and ``TweedieRegressor`` with ``link='log'``, or ``link='auto'`` and
    ``power > 0`` (``power <= 0`` picks the identity link).  Decided from the class and its public parameters; the
    fit-time check against the callable has the last word."""
    names = {c.__name__ for c in type(owner).__mro__ if c.__module__.startswith("sklearn.")}
    if names & {"PoissonRegressor", "GammaRegressor"}:
        return True
    if "TweedieRegressor" in names:
        link = getattr(owner, "link", "auto")
        return link == "log" or (link == "auto" and float(getattr(owner, "power", 0.0)) > 0)
    return False


def _is_ovr_rule(owner):
    """scikit-learn 0.23.2 ``LogisticRegression.predict_proba`` with C >= 3 classes is one-vs-rest (``_predict_proba_lr``)
    when ``multi_class`` is 'ovr' or 'warn', or 'auto' with the liblinear solver; otherwise a softmax."""
    mc = getattr(owner, "multi_class", "multinomial")
    return mc in ("ovr", "warn") or (mc == "auto" and getattr(owner, "solver", None) == "liblinear")


def _one_vs_rest_spec(owner, method):
    """``OneVsRestClassifier.predict_proba`` over C >= 3 binary linear models: ``p_c = predict_proba_c[:, 1]`` normalised
    per row.  Each estimator's ``predict_proba[:, 1]`` must be ``sigmoid(coef_ x + intercept_)`` -- the fit-time check
    against the callable holds the stacked model to that."""
    if method != "predict_proba":
        raise TypeError(f"{type(owner).__name__}.{method} is not supported: pass predict_proba")
    if getattr(owner, "multilabel_", False):
        raise NotImplementedError("multilabel one-vs-rest outputs are not normalised per row: not supported")
    ests = list(owner.estimators_)
    if len(ests) < 3:
        raise NotImplementedError(f"one-vs-rest over {len(ests)} estimator(s): the one-vs-rest head needs at least three "
                                  "classes")
    rows, bias = [], []
    for e in ests:
        if not (hasattr(e, "coef_") and hasattr(e, "intercept_")):
            raise TypeError(f"{type(e).__name__} exposes no coef_/intercept_: only linear models are supported")
        coef = np.atleast_2d(np.asarray(e.coef_, dtype=np.float64))
        if coef.shape[0] != 1 or getattr(e, "multi_class", "auto") == "multinomial":
            raise NotImplementedError("one-vs-rest estimators must be binary models with predict_proba = sigmoid(z)")
        rows.append(coef[0])
        bias.append(float(np.atleast_1d(np.asarray(e.intercept_, dtype=np.float64))[0]))
    return LinearModelSpec(np.stack(rows), np.asarray(bias), "ovr")
