"""Multi-layer perceptrons of scikit-learn read into float64 layers in raw feature space (``MlpSpec``) for the device's MLP
route.

A spec is what ``dks_set_mlp`` takes (include/dks.h): hidden layers ``a_l = act(a_{l-1} W_l + b_l)`` with one activation
of scikit-learn's ``ACTIVATIONS`` (``identity``, ``logistic``, ``tanh``, ``relu``), then the output layer ``z = a W + b``
and a head:

* ``identity``: ``MLPRegressor.predict`` (1 to 8 targets; a 1-D array for one);
* ``sigmoid``: binary ``MLPClassifier.predict_proba``, ``p = expit(z)``, outputs ``[1 - p, p]``;
* ``softmax``: ``MLPClassifier.predict_proba`` over 3 to 8 classes.

A ``Pipeline`` of per-column affine scalers in front of the model, ``x'_c = a_c x_c + b_c``, folds into the first layer:
``W_0[c] <- a_c W_0[c]`` and ``b_0 <- b_0 + sum_c b_c W_0[c]``.  ``MlpSpec.__call__`` evaluates the scikit-learn method in
NumPy, on the folded layers.
"""
import numpy as np

from .kernel_machines import _final, _names, _unwrap

MAX_HIDDEN = 4
MAX_WIDTH = 256
MAX_OUTPUTS = 8
MAX_GROUPS = 64
ACTIVATIONS = ("identity", "logistic", "tanh", "relu")     # DKS_MLP_ACT_* codes 0..3
HEADS = ("identity", "sigmoid", "softmax")                 # DKS_MLP_HEAD_* codes 0..2

_MLPS = {"MLPClassifier", "MLPRegressor"}


def _act(name, a):
    if name == "logistic":
        return 1.0 / (1.0 + np.exp(-a))
    if name == "tanh":
        return np.tanh(a)
    if name == "relu":
        return np.maximum(a, 0)
    return a


class MlpSpec:
    """The layers of an MLP in raw feature space and its head.

    coefs: list of float64 [K_l, H_l] weight matrices (layer 0 reads the raw columns, its scalers folded in), intercepts:
    list of float64 [H_l]; activation in ``ACTIVATIONS``, head in ``HEADS``."""

    activation = "mlp"
    act_code = 8          # DKS_ACT_MLP
    maps = None
    R = 1                 # score rows of the zero linear model stage 1 evaluates

    def __init__(self, coefs, intercepts, activation, head, n_features, scalar_out=False):
        self.coefs = [np.ascontiguousarray(np.atleast_2d(np.asarray(W, dtype=np.float64))) for W in coefs]
        self.intercepts = [np.ascontiguousarray(np.asarray(b, dtype=np.float64).reshape(-1)) for b in intercepts]
        self.hidden_activation = activation
        self.head = head
        self.n_features = int(n_features)
        self.scalar_out = bool(scalar_out)
        if activation not in ACTIVATIONS:
            raise ValueError(f"unknown MLP activation {activation!r}")
        if head not in HEADS:
            raise ValueError(f"unknown MLP head {head!r}")
        if len(self.coefs) != len(self.intercepts) or len(self.coefs) < 2:
            raise ValueError("an MLP needs at least one hidden layer and one bias vector per layer")
        n_hidden = len(self.coefs) - 1
        if n_hidden > MAX_HIDDEN:
            raise NotImplementedError(f"{n_hidden} hidden layers: MLPs are explained up to {MAX_HIDDEN}")
        widths = self.widths
        if widths[0] != self.n_features:
            raise ValueError(f"the first layer reads {widths[0]} columns, the model {self.n_features}")
        for l, (W, b) in enumerate(zip(self.coefs, self.intercepts)):
            if W.shape != (widths[l], widths[l + 1]) or b.shape != (widths[l + 1],):
                raise ValueError(f"layer {l}: weights {W.shape} and biases {b.shape} do not chain")
        for l, h in enumerate(widths[1:-1], 1):
            if h > MAX_WIDTH:
                raise NotImplementedError(f"hidden layer {l} has {h} units: MLPs are explained up to {MAX_WIDTH} per layer")
        R = widths[-1]
        if R > MAX_OUTPUTS:
            raise NotImplementedError(f"{R} output units: MLPs are explained up to {MAX_OUTPUTS} outputs")
        if head == "sigmoid" and R != 1:
            raise ValueError("the sigmoid head takes one output unit")
        if head == "softmax" and R < 2:
            raise ValueError("the softmax head takes at least two output units")
        self.n_outputs = 2 if head == "sigmoid" else R

    @property
    def widths(self):
        return [self.coefs[0].shape[0]] + [W.shape[1] for W in self.coefs]

    @property
    def n_hidden(self):
        return len(self.coefs) - 1

    @property
    def act_code_hidden(self):
        return ACTIVATIONS.index(self.hidden_activation)

    @property
    def head_code(self):
        return HEADS.index(self.head)

    def flat(self):
        """(widths int32 [n_hidden + 2], weights, biases) concatenated as ``dks_set_mlp`` reads them."""
        return (np.ascontiguousarray(self.widths, dtype=np.int32),
                np.ascontiguousarray(np.concatenate([W.reshape(-1) for W in self.coefs])),
                np.ascontiguousarray(np.concatenate(self.intercepts)))

    def scores(self, X):
        """The output layer's values z [n, R]."""
        a = np.atleast_2d(np.asarray(X, dtype=np.float64))
        for l, (W, b) in enumerate(zip(self.coefs, self.intercepts)):
            a = a @ W + b
            if l < len(self.coefs) - 1:
                a = _act(self.hidden_activation, a)
        return a

    def __call__(self, X):
        """The scikit-learn method the spec was read from, in NumPy."""
        z = self.scores(X)
        if self.head == "sigmoid":
            p = 1.0 / (1.0 + np.exp(-z[:, 0]))
            return np.stack([1 - p, p], axis=1)
        if self.head == "softmax":
            e = np.exp(z - z.max(axis=1, keepdims=True))
            return e / e.sum(axis=1, keepdims=True)
        return z[:, 0] if self.scalar_out else z


def _is_mlp(est):
    return bool(_names(_final(est)) & _MLPS)


def extract_mlp_spec(predictor):
    """``MlpSpec`` of a bound method of a fitted scikit-learn MLP -- ``MLPClassifier.predict_proba`` (2 to 8 classes) or
    ``MLPRegressor.predict`` (1 to 8 targets), each possibly behind a ``Pipeline`` of per-column affine scalers
    (``StandardScaler``, ``MinMaxScaler`` without ``clip``, ``MaxAbsScaler``, ``RobustScaler``) -- and ``None`` for anything
    else.  A spec passes through.  Raises ``NotImplementedError`` / ``TypeError`` naming the reason for MLPs the route does
    not cover: a multilabel classifier, more than 4 hidden layers, more than 256 units in a layer, more than 8 outputs,
    ``predict`` of a classifier, pipeline steps other than the four scalers."""
    if isinstance(predictor, MlpSpec):
        return predictor
    owner = getattr(predictor, "__self__", None)
    method = getattr(predictor, "__name__", None)
    if owner is None or not _is_mlp(owner):
        return None
    est = _final(owner)
    name = type(est).__name__
    if not hasattr(est, "coefs_"):
        raise TypeError(f"{name} is not fitted")
    P = int(owner.n_features_in_)
    if "MLPClassifier" in _names(est):
        if est.out_activation_ == "logistic" and est.n_outputs_ > 1:
            raise NotImplementedError(f"multilabel {name} ({est.n_outputs_} independent logistic outputs) is not supported: "
                                      "its outputs are not one distribution over classes")
        if method != "predict_proba":
            raise TypeError(f"{name}.{method} is not supported: pass predict_proba (predict returns labels)")
        head = "sigmoid" if est.out_activation_ == "logistic" else "softmax"
        scalar = False
    else:
        if method != "predict":
            raise TypeError(f"{name}.{method} is not supported: pass predict")
        head = "identity"
        scalar = est.n_outputs_ == 1
    n_hidden = len(est.coefs_) - 1
    if n_hidden > MAX_HIDDEN:
        raise NotImplementedError(f"{name} with {n_hidden} hidden layers: MLPs are explained up to {MAX_HIDDEN}")
    widths = [int(W.shape[1]) for W in est.coefs_]
    if max(widths[:-1]) > MAX_WIDTH:
        raise NotImplementedError(f"{name} with a hidden layer of {max(widths[:-1])} units: MLPs are explained up to "
                                  f"{MAX_WIDTH} units per layer")
    if widths[-1] > MAX_OUTPUTS:
        raise NotImplementedError(f"{name} with {widths[-1]} outputs: MLPs are explained up to {MAX_OUTPUTS}")
    if est.activation not in ACTIVATIONS:
        raise NotImplementedError(f"{name}(activation={est.activation!r}) is not supported")
    try:
        _, a, b = _unwrap(owner, P)                     # the scalers composed into x' = a x + b (kernel_machines._affine)
    except NotImplementedError as e:
        raise NotImplementedError(f"{name}: {e}") from e
    coefs = [np.asarray(W, dtype=np.float64) for W in est.coefs_]
    intercepts = [np.asarray(c, dtype=np.float64) for c in est.intercepts_]
    intercepts[0] = intercepts[0] + b @ coefs[0]
    coefs[0] = a[:, None] * coefs[0]
    return MlpSpec(coefs, intercepts, est.activation, head, P, scalar_out=scalar)
