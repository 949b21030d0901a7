"""Stacking ensembles of scikit-learn models from different families read into ``StackingSpec`` for the device's stacking
route (DESIGN.md §5.0.20).

``StackingClassifier.predict_proba`` / ``.decision_function`` and ``StackingRegressor.predict`` apply a final estimator to
the members' outputs of each row: ``f(x) = head(W m(x) + b (+ W_pass x))``, with ``m(x)`` the meta columns scikit-learn's
``_concatenate_predictions`` forms (a binary ``predict_proba`` keeps class 1, a 1-D output one column, anything else every
column; with ``passthrough=True`` the stacking's own input columns come last).  The final estimator is not linear in the
members, so the device evaluates it on every masked row before the background mean.  Members are read as the soft-voting
route reads them (``ensembles._member_spec``): tree models, kernel machines, MLPs and neighbour models through their
family extractors, linear members lowered exactly to one-identity-hidden-layer MLPs.  The final estimator must be linear
with a logistic, softmax or identity head (``predictors.extract_linear_spec``).  The stacking ensemble may be the last
step of a ``Pipeline`` of per-column steps (``column_maps.compile_encoding``).  An all-linear ``StackingRegressor`` is
exactly linear and folds into one identity-head ``LinearModelSpec`` instead.
"""
import numpy as np

from .ensembles import MAX_GROUPS, MAX_MEMBERS, MAX_OUTPUTS, _STACKING, _VOTING, _member_spec
from .kernel_machines import _names

MAX_META = MAX_MEMBERS * MAX_OUTPUTS      # DKS_STACK_MAX_F
_HEADS = {"binary_logistic": "sigmoid", "softmax": "softmax", "identity": "identity"}
_HEAD_CODES = {"identity": 0, "sigmoid": 1, "softmax": 2}      # DKS_STACK_HEAD_*
_PIPELINE_MEMBER = ("a Pipeline inside a stacking ensemble member is not supported: put the preprocessing in front of the "
                    "ensemble (make_pipeline(preprocessing, StackingClassifier(...)))")

__all__ = ["StackingSpec", "extract_stacking_spec", "MAX_GROUPS"]


class StackingSpec:
    """A stacking ensemble: ``members`` = ``[((col_first, col_count), member spec)]`` (members in order, each a
    ``TreeEnsembleSpec``, ``KernelMachineSpec``, ``MlpSpec`` or ``KnnSpec`` on the same ``n_features`` columns, outputs
    ``col_first .. col_first + col_count - 1`` kept as meta columns), and the final estimator ``W`` [R, F], ``b`` [R],
    ``W_pass`` [R, n_features] or None and ``head`` ('identity': C = R outputs; 'sigmoid': R = 1, outputs [1 - p, p];
    'softmax': C = R)."""

    activation = "stacking"
    act_code = 12         # DKS_ACT_STACKING
    maps = None
    R = 1                 # score rows of the zero linear model stage 1 evaluates

    def __init__(self, members, W, b, head, W_pass, n_features, scalar_out=False):
        self.members = [((int(c0), int(nc)), spec) for (c0, nc), spec in members]
        self.W = np.ascontiguousarray(W, dtype=np.float64)
        self.b = np.ascontiguousarray(np.atleast_1d(b), dtype=np.float64)
        self.W_pass = None if W_pass is None else np.ascontiguousarray(W_pass, dtype=np.float64)
        self.head = head
        self.n_outputs = 2 if head == "sigmoid" else self.W.shape[0]
        self._n_features = int(n_features)
        self.scalar_out = bool(scalar_out)

    @property
    def n_features(self):
        return self._n_features

    @n_features.setter
    def n_features(self, value):          # behind a column encoding: the raw columns (the members read the encoded ones)
        self._n_features = int(value)

    @property
    def head_code(self):
        return _HEAD_CODES[self.head]

    @property
    def col_first(self):
        return np.asarray([c0 for (c0, _), _ in self.members], dtype=np.int32)

    @property
    def col_count(self):
        return np.asarray([nc for (_, nc), _ in self.members], dtype=np.int32)

    def meta(self, X):
        """The meta columns ``[n, F]`` of the rows X (the columns the members read)."""
        X = np.atleast_2d(np.asarray(X, dtype=np.float64))
        cols = [np.asarray(spec(X), dtype=np.float64).reshape(X.shape[0], -1)[:, c0:c0 + nc]
                for (c0, nc), spec in self.members]
        return np.hstack(cols)

    def __call__(self, X):
        """The scikit-learn method the spec was read from, in NumPy, on the columns the members read."""
        from scipy.special import expit
        X = np.atleast_2d(np.asarray(X, dtype=np.float64))
        feats = self.meta(X)
        W = self.W
        if self.W_pass is not None:
            feats, W = np.hstack([feats, X]), np.hstack([self.W, self.W_pass])
        z = feats @ W.T + self.b
        if self.head == "sigmoid":
            p = expit(z[:, 0])
            return np.c_[1.0 - p, p]
        if self.head == "softmax":
            e = np.exp(z - z.max(axis=1, keepdims=True))
            return e / e.sum(axis=1, keepdims=True)
        return z[:, 0] if self.scalar_out else z


def _final_linear(final, method, name):
    """``(W, b, head, scalar_out)`` of the final estimator's ``method``: a logistic (kappa folded into W and b), softmax
    or identity head, else refused."""
    from .predictors import extract_linear_spec
    what = f"{name}: the final estimator {type(final).__name__}"
    if not hasattr(final, method):
        raise NotImplementedError(f"{what} has no {method}")
    try:
        spec = extract_linear_spec(getattr(final, method))
    except TypeError as e:
        raise NotImplementedError(f"{what} is not a linear model with a logistic, softmax or identity head, so it is not "
                                  f"supported ({e})") from e
    head = _HEADS.get(spec.activation)
    if head is None or spec.maps is not None:
        kind = {"ovr": "a one-vs-rest", "mixture": "a mixture", "exp": "an exp-head (log-link)"}.get(spec.activation,
                                                                                                 "a per-column pipeline")
        raise NotImplementedError(f"{what} is {kind} model: only a linear final estimator with a logistic, softmax or "
                                  "identity head is supported")
    W = np.asarray(spec.W, dtype=np.float64) * spec.kappa
    b = np.asarray(spec.b, dtype=np.float64).reshape(-1) * spec.kappa
    return W, b, head, spec.scalar_out


def _members(owner, name):
    """``[(member, stack method)]`` of the fitted members (``'drop'`` ones are in neither list)."""
    ests, methods = list(owner.estimators_), list(owner.stack_method_)
    if len(ests) != len(methods):
        raise NotImplementedError(f"{name}: {len(ests)} fitted members but {len(methods)} stack methods")
    if len(ests) > MAX_MEMBERS:
        raise NotImplementedError(f"a stacking ensemble of {len(ests)} members: at most {MAX_MEMBERS} are explained")
    return list(zip(ests, methods))


def _check_member(est, method, k, classifier):
    names = _names(est)
    if "Pipeline" in names:
        raise NotImplementedError(_PIPELINE_MEMBER)
    if names & (_VOTING | _STACKING):
        raise NotImplementedError(f"stacking ensemble member {k} ({type(est).__name__}): nested voting or stacking "
                                  "ensembles are not supported")
    if classifier and method == "predict":
        raise NotImplementedError(f"stacking ensemble member {k} ({type(est).__name__}) is stacked with predict, which "
                                  "returns labels: pass stack_method='predict_proba' or 'decision_function'")


def _linear_fold(owner, members, method):
    """An all-linear ``StackingRegressor.predict`` as one identity-head ``LinearModelSpec`` (``W = sum_k w_k W_k (+
    W_pass)``), or None when a member or the final estimator is not a plain linear regressor."""
    from .predictors import LinearModelSpec, extract_linear_spec
    specs = []
    for est, m in members:
        if m != "predict" or "Pipeline" in _names(est):
            return None
        try:
            s = extract_linear_spec(getattr(est, m))
        except (TypeError, NotImplementedError):
            return None
        if s.activation != "identity" or s.maps is not None or s.R != 1:
            return None
        specs.append(s)
    try:
        fin = extract_linear_spec(getattr(owner.final_estimator_, method))
    except (TypeError, NotImplementedError):
        return None
    if fin.activation != "identity" or fin.maps is not None or fin.R != 1:
        return None
    K = len(specs)
    wf = np.asarray(fin.W, dtype=np.float64)[0]
    if wf.shape[0] not in (K, K + specs[0].W.shape[1]):
        return None
    W = np.zeros_like(specs[0].W)
    b = np.asarray(fin.b, dtype=np.float64).copy()
    for wk, s in zip(wf[:K], specs):
        W = W + wk * s.W
        b = b + wk * s.b
    if wf.shape[0] > K:
        W = W + wf[K:][None, :]
    return LinearModelSpec(W, b, "identity", scalar_out=True)


def extract_stacking_spec(predictor):
    """``StackingSpec`` of a bound ``predict_proba`` / ``decision_function`` of a fitted ``StackingClassifier`` (2 to 8
    classes) or ``predict`` of a fitted ``StackingRegressor`` (one target); ``(StackingSpec, ColumnEncoding)`` when it is
    the last step of a ``Pipeline`` of per-column steps (the members and the passthrough read the encoded columns); an
    identity-head ``LinearModelSpec`` for a bare all-linear ``StackingRegressor`` (exactly linear); ``None`` for
    anything else.  Raises ``NotImplementedError`` / ``TypeError`` naming the reason for what the route does not cover: a
    final estimator that is not linear with a logistic, softmax or identity head, classifier members stacked with
    ``predict``, members that are pipelines or nested ensembles, multilabel targets, more than 16 members, 128 meta
    columns or 8 outputs, and whatever a member's own extractor refuses."""
    owner = getattr(predictor, "__self__", None)
    method = getattr(predictor, "__name__", None)
    if owner is None:
        return None
    pre, final = [], owner
    if "Pipeline" in _names(owner) and hasattr(owner, "steps"):
        from .column_maps import pipeline_parts
        pre, final = pipeline_parts(owner)
    names = _names(final)
    if not names & _STACKING:
        return None
    name = type(final).__name__
    classifier = "StackingClassifier" in names
    if not hasattr(final, "final_estimator_"):
        raise TypeError(f"{name} is not fitted")
    allowed = ("predict_proba", "decision_function") if classifier else ("predict",)
    if method not in allowed:
        raise TypeError(f"{name}.{method} is not supported: pass {' or '.join(allowed)}")
    if classifier and isinstance(getattr(final, "_label_encoder", None), list):
        raise NotImplementedError(f"{name} fitted on a multilabel target is not supported")
    if classifier and np.ndim(final.classes_) != 1:
        raise NotImplementedError(f"{name} fitted on a multilabel target is not supported")
    members = _members(final, name)
    for k, (est, m) in enumerate(members):
        _check_member(est, m, k, classifier)
    if not classifier and final is owner:
        folded = _linear_fold(final, members, method)
        if folded is not None:
            return folded
    W, b, head, scalar_out = _final_linear(final.final_estimator_, method, name)
    n_classes = len(final.classes_) if classifier else 0
    specs = []
    for k, (est, m) in enumerate(members):
        try:
            spec = _member_spec(est, m)
        except NotImplementedError as e:
            raise NotImplementedError(str(e).replace("a soft-voting ensemble", "a stacking ensemble")) from e
        C = spec.n_outputs
        if getattr(spec, "scalar_out", False) or C == 1:
            cols = (0, 1)
        elif m == "predict_proba" and n_classes == 2:
            cols = (1, C - 1)                 # the first column is dropped: the probabilities are collinear
        else:
            cols = (0, C)
        specs.append((cols, spec))
    F = sum(nc for (_, nc), _ in specs)
    if F > MAX_META:
        raise NotImplementedError(f"a stacking ensemble with {F} meta columns: at most {MAX_META} are explained")
    widths = {spec.n_features for _, spec in specs}
    if len(widths) != 1:
        raise NotImplementedError("stacking ensemble members reading different numbers of columns are not supported")
    D = widths.pop()
    passthrough = bool(getattr(final, "passthrough", False))
    if W.shape[1] != F + (D if passthrough else 0):
        raise NotImplementedError(f"{name}: the final estimator reads {W.shape[1]} columns, the members give {F} meta "
                                  f"columns{f' and the passthrough {D}' if passthrough else ''}")
    R = W.shape[0]
    C = 2 if head == "sigmoid" else R
    if C > MAX_OUTPUTS:
        raise NotImplementedError(f"a stacking ensemble with {C} outputs: at most {MAX_OUTPUTS} are explained")
    spec = StackingSpec(specs, W[:, :F], b, head, W[:, F:] if passthrough else None, D, scalar_out=scalar_out)
    if final is owner:
        return spec
    if not hasattr(owner, "n_features_in_"):
        raise TypeError("Pipeline is not fitted")
    from .column_maps import compile_encoding
    try:
        enc = compile_encoding(pre, int(owner.n_features_in_), spec.n_features, model="a stacking ensemble")
    except TypeError as e:
        raise NotImplementedError(f"Pipeline in front of a stacking ensemble: {e}") from e
    spec.n_features = enc.D
    return spec, enc
