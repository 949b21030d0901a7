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
    scikit-learn's log-link GLM regressors), 'mixture' (outputs ``sum_k pi_k h(z_k)``: K >= 2 members with ``pi`` [K] > 0
    summing to 1 and the member head ``member`` -- 'binary_logistic' with kappa folded into the scores (R_m = 1, outputs
    [1 - p, p]), 'softmax' or 'ovr' (R_m = C) --, score rows stacked member-major, R = K R_m <= 32).
    ``scalar_out``: the callable returns a 1-D array."""

    def __init__(self, W, b, activation, kappa=1.0, scalar_out=False, maps=None, pi=None, member=None):
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
        if activation not in ("identity", "binary_logistic", "softmax", "ovr", "exp", "mixture"):
            raise ValueError(f"unknown activation {activation!r}")
        self.pi, self.member = None, None
        if activation == "mixture":
            pi = np.atleast_1d(np.asarray(pi, dtype=np.float64))
            if member not in MIXTURE_MEMBER_HEADS:
                raise ValueError(f"mixture member head {member!r}: one of {MIXTURE_MEMBER_HEADS}")
            if len(pi) < 2 or not np.all(np.isfinite(pi)) or np.any(pi <= 0) or abs(pi.sum() - 1.0) > 1e-12:
                raise ValueError("a mixture needs K >= 2 positive, finite weights pi summing to 1")
            if R % len(pi) or (member == "binary_logistic" and R != len(pi)) or (member != "binary_logistic" and R // len(pi) < 3):
                raise ValueError(f"{R} score rows do not split into {len(pi)} {member} members")
            if R > MIXTURE_MAX_ROWS:
                raise NotImplementedError(f"a mixture of {len(pi)} members with {R // len(pi)} score row(s) each has {R} "
                                          f"score rows; the engine evaluates at most {MIXTURE_MAX_ROWS}")
            self.pi, self.member = pi, member
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
                "softmax": _cabi.ACT_SOFTMAX, "ovr": _cabi.ACT_OVR, "exp": _cabi.ACT_EXP,
                "mixture": _cabi.ACT_MIX}[self.activation]

    @property
    def K(self):
        """Members of a mixture (1 for the other heads)."""
        return 1 if self.pi is None else len(self.pi)

    @property
    def n_outputs(self):
        if self.activation == "mixture":
            return 2 if self.member == "binary_logistic" else self.R // self.K
        return 2 if self.activation == "binary_logistic" else self.R

    def __call__(self, X):
        """NumPy evaluation with scikit-learn's conventions (used on the host by build_explanation and tests)."""
        X = np.asarray(X, dtype=np.float64)
        if X.ndim == 1:
            X = X.reshape(1, -1)
        z = (self.maps.contributions(X) if self.maps is not None else X @ self.W.T) + self.b
        if self.activation == "mixture":
            zk = z.reshape(z.shape[0], self.K, -1)
            if self.member == "binary_logistic":
                p1 = np.exp(-np.logaddexp(0.0, -zk[:, :, 0]))          # expit, as scikit-learn's members compute it
                out = np.stack([1.0 - p1, p1], axis=2)
            elif self.member == "ovr":
                p = np.exp(-np.logaddexp(0.0, -zk))
                out = p / p.sum(axis=2, keepdims=True)
            else:
                e = np.exp(zk - zk.max(axis=2, keepdims=True))
                out = e / e.sum(axis=2, keepdims=True)
            return np.einsum("nkc,k->nc", out, self.pi)
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


MIXTURE_MEMBER_HEADS = ("binary_logistic", "softmax", "ovr")
MIXTURE_MAX_ROWS = 32


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
    (``_pipeline_spec``: the model is read in raw feature space through column maps); the averaging ensembles of those
    (``_ENSEMBLES``: ``CalibratedClassifierCV`` with sigmoid calibration, soft ``VotingClassifier`` and
    ``BaggingClassifier`` give the 'mixture' head; ``VotingRegressor``, ``BaggingRegressor`` and
    ``BaggingClassifier.decision_function`` one identity head, as they are exactly linear).
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
    ensemble = _sklearn_names(owner) & set(_ENSEMBLES)
    if ensemble:
        return _ENSEMBLES[ensemble.pop()](owner, method)
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
    return LinearModelSpec(None, inner.b, inner.activation, kappa=inner.kappa, scalar_out=inner.scalar_out, maps=maps,
                           pi=inner.pi, member=inner.member)


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


# ---------------------------------------------------------------------------------------------------------------------
# averaging ensembles: mixtures of linear heads, and exact linear folds of identity heads
# ---------------------------------------------------------------------------------------------------------------------
def _sklearn_names(owner):
    return {c.__name__ for c in type(owner).__mro__ if c.__module__.startswith("sklearn.")}


def _members(spec):
    """``[(pi, W [R_m, D], b [R_m], member head)]`` of a classifier's ``predict_proba`` spec: one member for a plain head
    (kappa folded into the scores; a two-class softmax becomes the binary member ``z_1 - z_0``), the members of a mixture."""
    if spec.maps is not None:
        raise NotImplementedError("a Pipeline inside an ensemble member is not supported: the ensemble's members must be "
                                  "linear models on the ensemble's own columns")
    if spec.activation == "mixture":
        Rm = spec.R // spec.K
        return [(spec.pi[k], spec.W[k * Rm:(k + 1) * Rm], spec.b[k * Rm:(k + 1) * Rm], spec.member) for k in range(spec.K)]
    if spec.activation == "binary_logistic":
        return [(1.0, spec.kappa * spec.W, spec.kappa * spec.b, "binary_logistic")]
    if spec.activation == "softmax" and spec.R == 2:
        return [(1.0, spec.W[1:] - spec.W[:1], spec.b[1:] - spec.b[:1], "binary_logistic")]
    if spec.activation in ("softmax", "ovr"):
        return [(1.0, spec.W, spec.b, spec.activation)]
    if spec.activation == "exp":
        raise NotImplementedError("log-link GLM members (a mixture of exponentials) are not supported")
    raise NotImplementedError(f"members with the {spec.activation!r} head have no predict_proba the engine can average")


def _mixture_spec(members):
    """One spec from ``[(weight, W, b, head)]``: the weights are normalised; a single member is its own head."""
    heads = {m[3] for m in members}
    if len(heads) != 1:
        raise NotImplementedError(f"ensemble members with different heads ({sorted(heads)}) are not supported: every member "
                                  "of a mixture must have the same head")
    head = heads.pop()
    rows = {m[1].shape[0] for m in members}
    if len(rows) != 1:
        raise NotImplementedError("ensemble members with different numbers of classes are not supported")
    pi = np.asarray([m[0] for m in members], dtype=np.float64)
    pi = pi / pi.sum()
    W = np.concatenate([m[1] for m in members], axis=0)
    b = np.concatenate([m[2] for m in members])
    if len(members) == 1:
        return LinearModelSpec(W, b, head)
    return LinearModelSpec(W, b, "mixture", pi=pi, member=head)


def _member_of(est, method):
    """The spec of a fitted ensemble member's bound ``method``; pipelines inside members are refused."""
    if _is_sklearn_pipeline(est):
        raise NotImplementedError("a Pipeline inside an ensemble member is not supported: the ensemble's members must be "
                                  "linear models on the ensemble's own columns")
    bound = getattr(est, method, None)
    if bound is None:
        raise NotImplementedError(f"ensemble member {type(est).__name__} has no {method}")
    return extract_linear_spec(bound)


def _calibrated_spec(owner, method):
    """``CalibratedClassifierCV(method='sigmoid').predict_proba``: the mean over folds of the calibrated fold.  A fold's
    class-c probability is ``expit(-(a_c f_c(x) + b_c))`` with ``f`` its estimator's ``decision_function``: binary folds are
    a binary-logistic member with score ``-(a (w x + c) + b)``, multi-class folds a one-vs-rest member over those scores
    (scikit-learn divides each fold's row by its sum).  scikit-learn 0.23.2 spells the fold's parts ``base_estimator`` /
    ``calibrators_``."""
    if method != "predict_proba":
        raise TypeError(f"CalibratedClassifierCV.{method} is not supported: pass predict_proba")
    cal = getattr(owner, "method", "sigmoid")
    if cal != "sigmoid":
        raise NotImplementedError(f"CalibratedClassifierCV(method={cal!r}) is not supported: only the sigmoid calibration "
                                  "is a logistic function of the linear score ('isotonic' is piecewise constant in it)")
    classes = np.asarray(owner.classes_)
    members = []
    for fold in owner.calibrated_classifiers_:
        est = getattr(fold, "estimator", None)
        if est is None:
            est = getattr(fold, "base_estimator", None)
        cals = getattr(fold, "calibrators", None)
        if cals is None:
            cals = getattr(fold, "calibrators_", None)
        if _is_sklearn_pipeline(est):
            raise NotImplementedError("a Pipeline inside a calibrated fold is not supported: pass the Pipeline around the "
                                      "CalibratedClassifierCV instead")
        if not (hasattr(est, "coef_") and hasattr(est, "intercept_") and hasattr(est, "decision_function")):
            raise TypeError(f"calibrated fold estimator {type(est).__name__} exposes no decision_function with coef_ / "
                            "intercept_: only linear models are supported")
        if not np.array_equal(np.asarray(est.classes_), classes):
            raise NotImplementedError("a calibrated fold whose estimator saw other classes than the model is not supported")
        coef = np.atleast_2d(np.asarray(est.coef_, dtype=np.float64))
        icpt = np.atleast_1d(np.asarray(est.intercept_, dtype=np.float64))
        a = np.asarray([float(c.a_) for c in cals])
        bb = np.asarray([float(c.b_) for c in cals])
        if coef.shape[0] != len(cals):
            raise NotImplementedError("a calibrated fold with one calibrator per score row was expected")
        members.append((1.0, -a[:, None] * coef, -(a * icpt + bb), "binary_logistic" if len(classes) == 2 else "ovr"))
    return _mixture_spec(members)


def _voting_weights(owner):
    """Weights of the fitted (not dropped) members, as ``_weights_not_none`` gives them; ones when none are set."""
    ests = list(owner.estimators_)
    if owner.weights is None:
        return ests, np.ones(len(ests))
    w = [w for (_, e), w in zip(owner.estimators, owner.weights) if not (isinstance(e, str) and e == "drop")]
    return ests, np.asarray(w, dtype=np.float64)


def _voting_classifier_spec(owner, method):
    """Soft ``VotingClassifier.predict_proba``: ``np.average`` of the members' probabilities, pi = weights / sum.  Zero
    weights drop their member; nested calibrated, bagging or voting members are flattened with pi multiplied."""
    if getattr(owner, "voting", "hard") != "soft":
        raise NotImplementedError("VotingClassifier(voting='hard') averages labels, not probabilities: it is not supported")
    if method != "predict_proba":
        raise TypeError(f"VotingClassifier.{method} is not supported: pass predict_proba")
    ests, w = _voting_weights(owner)
    if np.any(w < 0) or not np.all(np.isfinite(w)) or not np.any(w > 0):
        raise NotImplementedError("VotingClassifier weights must be finite, non-negative and not all zero")
    members = []
    for est, wk in zip(ests, w / w.sum()):
        if wk > 0:
            members += [(wk * m[0],) + m[1:] for m in _members(_member_of(est, "predict_proba"))]
    return _mixture_spec(members)


def _bagging_scatter(spec, features, D):
    """W of a member trained on ``X[:, features]`` (repeats allowed) as a [R, D] matrix on the ensemble's columns."""
    W = np.zeros((spec.R, D))
    np.add.at(W.T, np.asarray(features), spec.W.T)
    return W


def _bagging_classifier_spec(owner, method):
    """``BaggingClassifier``: ``predict_proba`` is the mean of the members' probabilities on their feature subsets
    (``estimators_features_``), ``decision_function`` the mean of their decision functions -- one identity head."""
    D = int(owner.n_features_in_)
    ests, feats = list(owner.estimators_), list(owner.estimators_features_)
    if method == "decision_function":
        return _linear_fold([(1.0 / len(ests), _member_of(e, "decision_function"), f) for e, f in zip(ests, feats)], D)
    if method != "predict_proba":
        raise TypeError(f"BaggingClassifier.{method} is not supported: pass predict_proba or decision_function")
    members = []
    for est, f in zip(ests, feats):
        if not hasattr(est, "predict_proba"):
            raise NotImplementedError(f"bagging of {type(est).__name__}, which has no predict_proba (scikit-learn then "
                                      "averages hard votes), is not supported")
        if len(est.classes_) != int(owner.n_classes_):
            raise NotImplementedError("a bagging member that saw fewer classes than the ensemble is not supported")
        spec = _member_of(est, "predict_proba")
        scattered = LinearModelSpec(_bagging_scatter(spec, f, D), spec.b, spec.activation, kappa=spec.kappa,
                                    pi=spec.pi, member=spec.member)
        members += [(m[0] / len(ests),) + m[1:] for m in _members(scattered)]
    return _mixture_spec(members)


def _linear_fold(parts, D):
    """``[(weight, identity spec, features or None)]`` -> one identity spec ``W = sum_k w_k W_k``, ``b = sum_k w_k b_k``."""
    W, b, scalar = 0.0, 0.0, None
    for wk, spec, f in parts:
        if spec.activation != "identity" or spec.maps is not None:
            raise NotImplementedError(f"averaging members with the {spec.activation!r} head is not linear: only "
                                      "identity-head (linear regression / decision_function) members fold into one model")
        Wk = spec.W if f is None else _bagging_scatter(spec, f, D)
        W, b = W + wk * Wk, b + wk * spec.b
        scalar = spec.scalar_out if scalar is None else scalar
    return LinearModelSpec(W, b, "identity", scalar_out=bool(scalar))


def _voting_regressor_spec(owner, method):
    """``VotingRegressor.predict``: ``np.average`` of the members' predictions -- exactly linear."""
    if method != "predict":
        raise TypeError(f"VotingRegressor.{method} is not supported: pass predict")
    ests, w = _voting_weights(owner)
    if not np.all(np.isfinite(w)) or w.sum() == 0:
        raise NotImplementedError("VotingRegressor weights must be finite with a non-zero sum")
    return _linear_fold([(wk / w.sum(), _member_of(e, "predict"), None) for e, wk in zip(ests, w)], None)


def _bagging_regressor_spec(owner, method):
    """``BaggingRegressor.predict``: the mean of the members' predictions on their feature subsets -- exactly linear."""
    if method != "predict":
        raise TypeError(f"BaggingRegressor.{method} is not supported: pass predict")
    ests = list(owner.estimators_)
    return _linear_fold([(1.0 / len(ests), _member_of(e, "predict"), f)
                         for e, f in zip(ests, owner.estimators_features_)], int(owner.n_features_in_))


_ENSEMBLES = {"CalibratedClassifierCV": _calibrated_spec, "VotingClassifier": _voting_classifier_spec,
              "BaggingClassifier": _bagging_classifier_spec, "VotingRegressor": _voting_regressor_spec,
              "BaggingRegressor": _bagging_regressor_spec}
