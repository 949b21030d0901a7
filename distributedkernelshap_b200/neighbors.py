"""Nearest-neighbour models of scikit-learn read into their training rows (``KnnSpec``) for the device's neighbour route.

A spec is what ``dks_set_knn_model`` takes (include/dks.h).  The distance between a row ``x`` and a training point ``v``
comes from a statistic that adds up over columns, ``t = sum_c h(x'_c - v_c)`` summed in column order, where
``x'_c = colw_c * x_c + colo_c`` is the row in the space the model was fitted in (a ``Pipeline`` of per-column affine
scalers folds into ``colw`` / ``colo``; ``v`` is the training row as scikit-learn stored it):

* ``euclidean``: ``h = d^2``, distance ``sqrt(t)``;
* ``sqeuclidean``: ``h = d^2``, distance ``t``;
* ``manhattan``: ``h = |d|``, distance ``t``;
* ``minkowski`` (finite ``p >= 1``): ``h = |d|^p``, distance ``t^(1/p)``.

The engine defines the function it explains where scikit-learn leaves it open:

* **Ties.** The ``k`` neighbours are the first ``k`` training points ranked by ``(t, training index)``: of several
  equidistant points the lower index wins.  scikit-learn's search structures do not promise any order among ties.
* **Zero distances.** A row equal to ``v`` column for column (``x'_c == v_c`` exactly) is at distance exactly 0, whatever
  the rounding of ``t``; every other ``t`` is raised to at least ``T_FLOOR`` (2^-1000), so a sum that rounds to 0 is
  never a zero distance.  Under ``weights='distance'`` the neighbours at distance 0 take weight 1 and the others weight
  0, as ``neighbors._base._get_weights`` does.  Behind a scaler, ``x * colw + colo`` need not reproduce the rounding of
  the scaler's own ``transform`` (``StandardScaler`` computes ``(x - mean) / scale``), so a raw training row is then
  usually not at distance exactly 0 but at a tiny one, and takes a very large finite weight instead of weight 1.
* **Outputs.** ``KNeighborsClassifier.predict_proba`` (2 to 8 classes): per-class sums of the neighbour weights in rank
  order, divided by their sum over classes (``uniform``: ``count / k``).  ``KNeighborsRegressor.predict`` (1 to 8
  targets): the rank-order sum of the targets over ``k`` (``uniform``) or of ``w y`` over the sum of ``w``.

``KnnSpec.__call__`` evaluates exactly these rules in NumPy.
"""
import numpy as np

from .kernel_machines import _dense, _final, _names, _unwrap

MAX_NEIGHBORS = 32
MAX_OUTPUTS = 8
MAX_GROUPS = 64
T_FLOOR = 2.0 ** -1000     # least t of a training row the row does not equal (dks_knn.cuh)
METRICS = ("euclidean", "manhattan", "minkowski", "sqeuclidean")   # DKS_KNN_METRIC_* codes 0..3
WEIGHTS = ("uniform", "distance")                                  # DKS_KNN_WEIGHTS_* codes 0..1
HEADS = ("classify", "regress")                                    # DKS_KNN_HEAD_* codes 0..1

_ALIASES = {"l1": "manhattan", "cityblock": "manhattan", "l2": "euclidean"}
_KNN = {"KNeighborsClassifier", "KNeighborsRegressor"}
_RADIUS = {"RadiusNeighborsClassifier", "RadiusNeighborsRegressor"}
# estimators that hold other estimators: a neighbour model inside one of them is refused by name
_CONTAINERS = {"VotingClassifier", "VotingRegressor", "BaggingClassifier", "BaggingRegressor", "CalibratedClassifierCV",
               "StackingClassifier", "StackingRegressor", "OneVsRestClassifier", "OneVsOneClassifier",
               "MultiOutputRegressor", "MultiOutputClassifier"}


class KnnSpec:
    """The training rows of a k-nearest-neighbour model, the column map into its fitted space and its rule.

    fitX [n_fit, D] float64 (the fitted space), colw / colo [D], k, metric in ``METRICS``, p (minkowski), weights in
    ``WEIGHTS``, head in ``HEADS``; y: class indices [n_fit] (classify, ``R`` classes) or targets [n_fit, R]."""

    activation = "knn"
    act_code = 9          # DKS_ACT_KNN
    maps = None

    def __init__(self, fitX, colw, colo, k, metric, p, weights, head, y, R, n_features, scalar_out=False):
        self.fitX = np.ascontiguousarray(np.atleast_2d(np.asarray(fitX, dtype=np.float64)))
        self.n_fit, D = self.fitX.shape
        self.colw = np.ascontiguousarray(np.asarray(colw, dtype=np.float64).reshape(D))
        self.colo = np.ascontiguousarray(np.asarray(colo, dtype=np.float64).reshape(D))
        self.k = int(k)
        self.metric = metric
        self.p = float(p)
        self.weights = weights
        self.head = head
        self.R = int(R)
        self.n_features = int(n_features)
        self.scalar_out = bool(scalar_out)
        if metric not in METRICS:
            raise ValueError(f"unknown neighbour metric {metric!r}")
        if weights not in WEIGHTS:
            raise ValueError(f"unknown neighbour weights {weights!r}")
        if head not in HEADS:
            raise ValueError(f"unknown neighbour head {head!r}")
        if metric == "minkowski" and not (np.isfinite(self.p) and self.p >= 1):
            raise NotImplementedError(f"minkowski p={p!r}: neighbour models are explained for a finite p >= 1")
        if not 1 <= self.k <= MAX_NEIGHBORS:
            raise NotImplementedError(f"n_neighbors={self.k}: neighbour models are explained up to {MAX_NEIGHBORS}")
        if self.n_fit < self.k:
            raise NotImplementedError(f"n_neighbors={self.k} with {self.n_fit} training rows: a neighbour model needs at "
                                      "least n_neighbors training rows")
        if not 1 <= self.R <= MAX_OUTPUTS or (head == "classify" and self.R < 2):
            raise NotImplementedError(f"{self.R} {'classes' if head == 'classify' else 'targets'}: neighbour models are "
                                      f"explained with {'2' if head == 'classify' else '1'} to {MAX_OUTPUTS}")
        if head == "classify":
            self.y = np.ascontiguousarray(np.asarray(y, dtype=np.float64).reshape(self.n_fit))
            if not np.all((self.y >= 0) & (self.y < self.R) & (self.y == np.floor(self.y))):
                raise ValueError("class indices must be integers in [0, R)")
        else:
            self.y = np.ascontiguousarray(np.asarray(y, dtype=np.float64).reshape(self.n_fit, self.R))
        if not (np.all(np.isfinite(self.fitX)) and np.all(np.isfinite(self.y)) and np.all(np.isfinite(self.colw))
                and np.all(np.isfinite(self.colo))):
            raise NotImplementedError("a neighbour model with non-finite training rows, targets or scaler parameters")
        self.n_outputs = self.R

    @property
    def metric_code(self):
        return METRICS.index(self.metric)

    @property
    def weights_code(self):
        return WEIGHTS.index(self.weights)

    @property
    def head_code(self):
        return HEADS.index(self.head)

    def _rows(self, X):
        X = np.atleast_2d(np.asarray(X, dtype=np.float64))
        if not np.all(np.isfinite(X)):
            raise ValueError("a row holds NaN or an infinity: neighbour models refuse it, as scikit-learn does")
        return X * self.colw + self.colo

    def statistic(self, X):
        """(t [n, n_fit] in column order, exact [n, n_fit]: the row equals the training point column for column)."""
        Xs = self._rows(X)
        t = np.zeros((Xs.shape[0], self.n_fit))
        exact = np.ones((Xs.shape[0], self.n_fit), dtype=bool)
        for c in range(self.fitX.shape[1]):
            d = Xs[:, c:c + 1] - self.fitX[None, :, c]
            if self.metric in ("euclidean", "sqeuclidean"):
                h = d * d
            elif self.metric == "manhattan":
                h = np.abs(d)
            else:
                h = np.abs(d) ** self.p
            t = t + h
            exact &= d == 0
        return np.where(exact, 0.0, np.maximum(t, T_FLOOR)), exact

    def distance(self, t):
        t = np.maximum(t, 0.0)
        if self.metric == "euclidean":
            return np.sqrt(t)
        if self.metric == "minkowski":
            return t ** (1.0 / self.p)
        return t

    def neighbors(self, X):
        """(indices [n, k] in rank order, t [n, k], boundary tie [n]: the k-th and (k+1)-th smallest t are equal)."""
        t, _ = self.statistic(X)
        idx = np.argsort(t, axis=1, kind="stable")            # stable: equal t keep the lower training index first
        ts = np.take_along_axis(t, idx, axis=1)
        tie = ts[:, self.k] == ts[:, self.k - 1] if self.n_fit > self.k else np.zeros(t.shape[0], dtype=bool)
        return idx[:, :self.k], ts[:, :self.k], tie

    def boundary_ties(self, X):
        return self.neighbors(X)[2]

    def _weights(self, ts):
        if self.weights == "uniform":
            return None
        with np.errstate(divide="ignore"):
            w = 1.0 / self.distance(ts)
        inf = np.isinf(w)
        rows = inf.any(axis=1)
        w[rows] = inf[rows]
        return w

    def __call__(self, X):
        """The model's outputs [n, R] under the rules above (a 1-D array for a single-target regressor)."""
        out = []
        for s in range(0, np.atleast_2d(X).shape[0], 2048):
            out.append(self._outputs(np.atleast_2d(X)[s:s + 2048]))
        out = np.concatenate(out) if out else np.zeros((0, self.R))
        return out[:, 0] if self.scalar_out else out

    def _outputs(self, X):
        idx, ts, _ = self.neighbors(X)
        w = self._weights(ts)
        n = idx.shape[0]
        rows = np.arange(n)
        if self.head == "classify":
            sums = np.zeros((n, self.R))
            lab = self.y[idx].astype(np.int64)
            for r in range(self.k):
                sums[rows, lab[:, r]] += 1.0 if w is None else w[:, r]
            if w is None:
                return sums / self.k
            norm = np.zeros(n)
            for c in range(self.R):
                norm = norm + sums[:, c]
            return sums / norm[:, None]
        Y = self.y[idx]                                        # [n, k, R]
        num = np.zeros((n, self.R))
        if w is None:
            for r in range(self.k):
                num = num + Y[:, r]
            return num / self.k
        den = np.zeros(n)
        for r in range(self.k):
            num = num + Y[:, r] * w[:, r:r + 1]
            den = den + w[:, r]
        return num / den[:, None]


def _contains_knn(obj, depth=0):
    if depth > 6 or obj is None:
        return False
    if _names(obj) & (_KNN | _RADIUS):
        return True
    for attr in ("steps", "estimators", "estimators_", "calibrated_classifiers_", "estimator", "base_estimator",
                 "estimator_", "final_estimator_"):
        v = getattr(obj, attr, None)
        if v is None or isinstance(v, str):
            continue
        kids = list(np.ravel(np.asarray(v, dtype=object))) if isinstance(v, (list, tuple, np.ndarray)) else [v]
        for e in kids:
            if _contains_knn(e[-1] if isinstance(e, tuple) else e, depth + 1):
                return True
    return False


def _metric(est, name):
    """(metric, p) of a fitted neighbour model as it measures distances."""
    if callable(est.weights):
        raise NotImplementedError(f"{name}(weights=<callable>) is not supported: weights 'uniform' or 'distance' only")
    if est.metric_params:
        raise NotImplementedError(f"{name}(metric_params={est.metric_params!r}) is not supported")
    metric = _ALIASES.get(est.effective_metric_, est.effective_metric_)
    params = {key: v for key, v in (est.effective_metric_params_ or {}).items() if not (key == "w" and v is None)}
    if callable(metric) or metric not in METRICS:
        shown = "a callable" if callable(metric) else repr(metric)
        raise NotImplementedError(f"{name}(metric={shown}) is not supported: metrics 'euclidean', 'manhattan', "
                                  "'minkowski' (finite p >= 1) and 'sqeuclidean' only")
    p = 2.0
    if metric == "minkowski":
        p = float(params.pop("p", 2))
        if not (np.isfinite(p) and p >= 1):
            raise NotImplementedError(f"{name}(metric='minkowski', p={p!r}) is not supported: a finite p >= 1 only")
        if p == 1:
            metric = "manhattan"
        elif p == 2:
            metric = "euclidean"
    if params:
        raise NotImplementedError(f"{name} with metric parameters {sorted(params)} is not supported")
    return metric, p


def extract_knn_spec(predictor):
    """``KnnSpec`` of a bound method of a fitted scikit-learn nearest-neighbour model --
    ``KNeighborsClassifier.predict_proba`` (2 to 8 classes) or ``KNeighborsRegressor.predict`` (1 to 8 targets), any
    ``algorithm``, each possibly behind a ``Pipeline`` of per-column affine scalers (``StandardScaler``,
    ``MinMaxScaler`` without ``clip``, ``MaxAbsScaler``, ``RobustScaler``) -- and ``None`` for anything else.  A spec
    passes through.  Raises ``NotImplementedError`` / ``TypeError`` naming the reason for neighbour models the route does
    not cover: ``predict`` of a classifier, multi-output classifiers, callable weights, metrics other than euclidean,
    manhattan, minkowski (finite ``p >= 1``) and sqeuclidean, ``metric_params``, more than 32 neighbours or 8 outputs,
    pipeline steps other than the four scalers, ``RadiusNeighbors*`` and neighbour models inside an ensemble."""
    if isinstance(predictor, KnnSpec):
        return predictor
    owner = getattr(predictor, "__self__", None)
    method = getattr(predictor, "__name__", None)
    if owner is None:
        return None
    est = _final(owner)
    names = _names(est)
    if names & _RADIUS:
        raise NotImplementedError(f"{type(est).__name__} is not supported: the neighbour route explains "
                                  "KNeighborsClassifier and KNeighborsRegressor only")
    if not names & _KNN:
        if names & _CONTAINERS and _contains_knn(est):
            raise NotImplementedError(f"{type(est).__name__} holding a neighbour model: neighbour models inside an "
                                      "ensemble are not supported; pass the neighbour model's own method")
        return None
    name = type(est).__name__
    if not hasattr(est, "_fit_X"):
        raise TypeError(f"{name} is not fitted")
    classify = "KNeighborsClassifier" in names
    if classify:
        if method != "predict_proba":
            raise TypeError(f"{name}.{method} is not supported: pass predict_proba (predict returns labels)")
        if est.outputs_2d_:
            raise NotImplementedError(f"multi-output {name} is not supported: its outputs are not one distribution "
                                      "over classes")
    elif method != "predict":
        raise TypeError(f"{name}.{method} is not supported: pass predict")
    metric, p = _metric(est, name)
    k = int(est.n_neighbors)
    if k > MAX_NEIGHBORS:
        raise NotImplementedError(f"{name}(n_neighbors={k}): neighbour models are explained up to {MAX_NEIGHBORS}")
    P = int(owner.n_features_in_)
    try:
        _, a, b = _unwrap(owner, P, family="neighbour model", target="its column weights and origins")
    except NotImplementedError as e:
        raise NotImplementedError(f"{name}: {e}") from e
    fitX = _dense(est._fit_X)
    if classify:
        y, R, scalar = np.asarray(est._y).reshape(-1), len(est.classes_), False
    else:
        y = np.asarray(est._y, dtype=np.float64)
        R, scalar = (1 if y.ndim == 1 else y.shape[1]), y.ndim == 1
    if R > MAX_OUTPUTS or (classify and R < 2):
        what = "classes" if classify else "targets"
        raise NotImplementedError(f"{name} with {R} {what}: neighbour models are explained with "
                                  f"{'2' if classify else '1'} to {MAX_OUTPUTS}")
    return KnnSpec(fitX, a, b, k, metric, p, est.weights, "classify" if classify else "regress", y, R, P,
                   scalar_out=scalar)
