"""Soft-voting ensembles of scikit-learn models from different families read into ``EnsembleSpec`` for the device's ensemble
route (DESIGN.md §5.0.17).

``VotingClassifier(voting='soft').predict_proba`` and ``VotingRegressor.predict`` are ``f = sum_k pi_k f_k`` with
``pi = weights / sum(weights)``: linear in the members, so the device explains the average by adding the members' masked
background means before one link and one solve.  A member is anything the family extractors read as a bare estimator
(``extract_tree_spec``, ``extract_kernel_machine_spec`` -- a sigmoid-calibrated SVC included --, ``extract_mlp_spec``,
``extract_knn_spec``), or a linear member lowered exactly to an ``MlpSpec`` with one identity hidden layer: a binary or
multinomial ``LogisticRegression`` (``z = x coef^T + intercept`` through ``W_1 = I``, then the sigmoid or softmax head), or
a regressor's ``coef_`` / ``intercept_`` (identity head).  Nested voting ensembles are flattened with their weights
multiplied.  The ensemble may be the last step of a ``Pipeline`` of per-column steps, compiled with
``column_maps.compile_encoding`` into the one column encoding every member reads.
"""
import numpy as np

from .kernel_machines import _is_kernel_machine, _names, extract_kernel_machine_spec
from .mlp import _MLPS, MlpSpec, extract_mlp_spec
from .neighbors import _KNN, extract_knn_spec
from .trees import _TREE_MODELS, extract_tree_spec

MAX_MEMBERS = 16
MAX_OUTPUTS = 8
MAX_GROUPS = 64

_VOTING = {"VotingClassifier", "VotingRegressor"}
_STACKING = {"StackingClassifier", "StackingRegressor"}
_PIPELINE_MEMBER = ("a Pipeline inside a soft-voting ensemble member is not supported: put the preprocessing in front of "
                    "the ensemble (make_pipeline(preprocessing, VotingClassifier(...)))")


class EnsembleSpec:
    """A soft-voting ensemble: ``members`` = ``[(pi_k, member spec)]`` (pi summing to 1, members in order), each member a
    ``TreeEnsembleSpec``, ``KernelMachineSpec``, ``MlpSpec`` or ``KnnSpec`` of ``n_outputs`` outputs on the same
    ``n_features`` columns."""

    activation = "ensemble"
    act_code = 10         # DKS_ACT_ENSEMBLE
    maps = None
    R = 1                 # score rows of the zero linear model stage 1 evaluates

    def __init__(self, members, n_outputs, n_features, scalar_out=False):
        self.members = [(float(pi), spec) for pi, spec in members]
        self.n_outputs = int(n_outputs)
        self._n_features = int(n_features)
        self.scalar_out = bool(scalar_out)

    @property
    def n_features(self):
        return self._n_features

    @n_features.setter
    def n_features(self, value):          # behind a column encoding: the raw columns (the members read the encoded ones)
        self._n_features = int(value)

    @property
    def weights(self):
        return np.asarray([pi for pi, _ in self.members])

    def __call__(self, X):
        """The scikit-learn method the spec was read from, in NumPy, on the columns the members read."""
        X = np.atleast_2d(np.asarray(X, dtype=np.float64))
        out = sum(pi * np.asarray(spec(X), dtype=np.float64).reshape(X.shape[0], self.n_outputs)
                  for pi, spec in self.members)
        return out[:, 0] if self.scalar_out else out


def _nonlinear(est):
    """A tree model, kernel machine (a calibrated SVC included), MLP or neighbour model, possibly behind a wrapper."""
    if est is None or isinstance(est, str):
        return False
    names = _names(est)
    if names & (_TREE_MODELS | _MLPS | _KNN) or _is_kernel_machine(est):
        return True
    kids = []
    for attr in ("steps", "estimators", "estimators_", "calibrated_classifiers_", "estimator", "base_estimator",
                 "final_estimator_"):
        v = getattr(est, attr, None)
        if isinstance(v, (list, tuple)):
            kids += [e[-1] if isinstance(e, tuple) else e for e in v]
        elif v is not None and not isinstance(v, str):
            kids.append(v)
    return any(_nonlinear(k) for k in kids)


def _voting_members(owner):
    """``[(member, weight)]`` of the fitted members (``'drop'`` ones left out), ones when no weights are set."""
    ests = list(owner.estimators_)
    if owner.weights is None:
        return [(e, 1.0) for e in ests]
    w = [w for (_, e), w in zip(owner.estimators, owner.weights) if not (isinstance(e, str) and e == "drop")]
    return list(zip(ests, [float(x) for x in w]))


def _linear_member(est, method, name):
    """The ``MlpSpec`` a linear member lowers to: one identity hidden layer of R units (``W_1 = I``)."""
    from .predictors import extract_linear_spec
    spec = extract_linear_spec(getattr(est, method))
    head = {"binary_logistic": "sigmoid", "softmax": "softmax", "identity": "identity"}.get(spec.activation)
    if head is None or spec.maps is not None:
        kind = {"ovr": "a one-vs-rest", "mixture": "a mixture", "exp": "an exp-head (log-link)"}.get(spec.activation,
                                                                                                 repr(spec.activation))
        raise NotImplementedError(f"ensemble member {name}: {kind} linear member is not supported in a soft-voting "
                                  "ensemble with tree, kernel-machine, MLP or neighbour members")
    W = np.asarray(spec.W, dtype=np.float64) * spec.kappa
    b = np.asarray(spec.b, dtype=np.float64).reshape(-1) * spec.kappa
    R = W.shape[0]
    return MlpSpec([W.T, np.eye(R)], [b, np.zeros(R)], "identity", head, W.shape[1], scalar_out=spec.scalar_out)


def _member_spec(est, method):
    name = type(est).__name__
    if "Pipeline" in _names(est):
        raise NotImplementedError(_PIPELINE_MEMBER)
    if not hasattr(est, method):
        raise NotImplementedError(f"ensemble member {name} has no {method}")
    bound = getattr(est, method)
    for extract in (extract_tree_spec, extract_kernel_machine_spec, extract_mlp_spec, extract_knn_spec):
        spec = extract(bound)
        if spec is not None:
            return spec
    return _linear_member(est, method, name)


def _flatten(owner, method, scale, out):
    """Appends ``(pi, spec)`` of every member of the voting ensemble ``owner`` (nested ones flattened) to ``out``."""
    members = _voting_members(owner)
    w = np.asarray([wk for _, wk in members], dtype=np.float64)
    name = type(owner).__name__
    if len(w) == 0 or not np.all(np.isfinite(w)) or np.any(w < 0) or not w.sum() > 0:
        raise NotImplementedError(f"{name} weights must be finite and non-negative with a positive sum")
    for (est, _), wk in zip(members, w / w.sum()):
        if _names(est) & _VOTING:
            _check_voting(est, method)
            _flatten(est, method, scale * wk, out)
        else:
            out.append((scale * wk, _member_spec(est, method)))


def _check_voting(owner, method):
    if "VotingClassifier" in _names(owner):
        if getattr(owner, "voting", "hard") != "soft":
            raise NotImplementedError("VotingClassifier(voting='hard') averages labels, not probabilities: it is not "
                                      "supported")
        if method != "predict_proba":
            raise TypeError(f"VotingClassifier.{method} is not supported: pass predict_proba")
    elif method != "predict":
        raise TypeError(f"VotingRegressor.{method} is not supported: pass predict")


def extract_ensemble_spec(predictor):
    """``EnsembleSpec`` of a bound ``predict_proba`` of a fitted soft ``VotingClassifier`` (2 to 8 classes) or ``predict``
    of a fitted ``VotingRegressor`` with at least one tree, kernel-machine, MLP or neighbour member; ``(EnsembleSpec,
    ColumnEncoding)`` when such an ensemble is the last step of a ``Pipeline`` of per-column steps (the members read the
    encoded columns); ``None`` for anything else, all-linear ensembles included (they keep the mixture route).  Raises
    ``NotImplementedError`` / ``TypeError`` naming the reason for what the route does not cover: hard voting, stacking,
    members that are pipelines, one-vs-rest, mixture and exp-head linear members, more than 16 members or 8 outputs, and
    whatever a member's own extractor refuses."""
    owner = getattr(predictor, "__self__", None)
    method = getattr(predictor, "__name__", None)
    if owner is None:
        return None
    pre, final = [], owner
    if "Pipeline" in _names(owner) and hasattr(owner, "steps"):
        from .column_maps import pipeline_parts
        pre, final = pipeline_parts(owner)
    names = _names(final)
    if names & _STACKING and _nonlinear(final):
        raise NotImplementedError(f"{type(final).__name__} is not supported: its final estimator is not linear in the "
                                  "members' outputs of each masked row, so the model is not an average of its members "
                                  "(a soft VotingClassifier or a VotingRegressor is)")
    if not (names & _VOTING) or not _nonlinear(final):
        return None
    _check_voting(final, method)
    members = []
    _flatten(final, method, 1.0, members)
    if len(members) > MAX_MEMBERS:
        raise NotImplementedError(f"a soft-voting ensemble of {len(members)} members: at most {MAX_MEMBERS} are explained")
    outs = {spec.n_outputs for _, spec in members}
    if len(outs) != 1:
        raise NotImplementedError(f"ensemble members with different numbers of outputs ({sorted(outs)}) are not supported")
    C = outs.pop()
    if C > MAX_OUTPUTS:
        raise NotImplementedError(f"a soft-voting ensemble with {C} outputs: at most {MAX_OUTPUTS} are explained")
    widths = {spec.n_features for _, spec in members}
    if len(widths) != 1:
        raise NotImplementedError("ensemble members reading different numbers of columns are not supported")
    spec = EnsembleSpec(members, C, widths.pop(), scalar_out=method == "predict")
    if final is owner:
        return spec
    if not hasattr(owner, "n_features_in_"):
        raise TypeError("Pipeline is not fitted")
    from .column_maps import compile_encoding
    try:
        enc = compile_encoding(pre, int(owner.n_features_in_), spec.n_features, model="a soft-voting ensemble")
    except TypeError as e:
        raise NotImplementedError(f"Pipeline in front of a soft-voting ensemble: {e}") from e
    spec.n_features = enc.D
    return spec, enc
