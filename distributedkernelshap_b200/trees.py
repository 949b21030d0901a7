"""Tree ensembles of scikit-learn read into flat node arrays (``TreeEnsembleSpec``) for the device's tree route.

A spec is what ``dks_set_tree_model`` takes (include/dks.h): every tree's nodes concatenated, a raw score per model row
``r = base + sum_t leaf_t(x)`` and a head applied to it:

* ``DecisionTree*``, ``RandomForest*``, ``ExtraTrees*``: identity head over the mean of the trees' leaf outputs (class
  fractions of ``tree_.value`` for classifiers, the leaf value for regressors); ``1/T`` is folded into the leaves.
* ``GradientBoosting*``: the learning rate is folded into the leaves and ``base`` is the initial raw prediction
  (``init_`` a ``DummyClassifier`` / ``DummyRegressor`` or ``'zero'``).  ``predict_proba``: ``[1 - expit(r), expit(r)]``
  for two classes, a softmax over the K raw scores (K trees per stage) otherwise; ``decision_function`` / ``predict`` of
  the regressor: identity.
* ``HistGradientBoosting*``: as gradient boosting, ``base`` the baseline prediction; the regressor's ``predict`` is
  ``exp(r)`` under a log-link loss (``'poisson'``, ``'gamma'``).
* ``AdaBoostClassifier`` (SAMME) over ``sklearn.tree`` classifiers: tree t votes ``w_t`` for the class its leaf predicts
  (``argmax tree_.value``, the first class on a tie) and ``-w_t / (K - 1)`` for every other class; ``1 / sum w`` is folded
  into the leaves.  ``decision_function``: identity head, for two classes one score ``dec[1] - dec[0]``;
  ``predict_proba``: ``[1 - expit(r), expit(r)]`` on that score for two classes, a softmax of ``dec / (K - 1)`` (folded
  into the leaves) otherwise.
* ``IsolationForest``: tree t's leaf holds ``h = depth + c(n_node_samples) - 1`` (``compute_node_depths``, the root at 1;
  ``c`` the average path length of an unsuccessful search), times ``-1 / d`` with ``d = T c(max_samples)``, so that
  ``score_samples = -2^r`` (every score ``-0.5`` when ``d = 0``) and ``decision_function = -2^r - offset_``: the
  ``"iforest"`` head.  A tree fitted on a feature subset has its split features mapped back to the original columns.

A split sends x left when ``x <= threshold``: ``sklearn.tree`` compares the value cast to float32 (``DTYPE``), the
histogram-based estimators compare float64 values.  NaN goes where the node's ``missing_go_to_left`` says.
``TreeEnsembleSpec.__call__`` evaluates the same thing in NumPy.
"""
import numpy as np

MAX_OUTPUTS = 8
MAX_GROUPS = 64
HEADS = ("identity", "sigmoid", "softmax", "exp", "iforest")     # DKS_TREE_HEAD_* codes 0..4
CMP_F32, CMP_F64 = 0, 1                               # DKS_TREE_CMP_*

_SKTREE_FORESTS = {"DecisionTreeClassifier", "DecisionTreeRegressor", "ExtraTreeClassifier", "ExtraTreeRegressor",
                   "RandomForestClassifier", "RandomForestRegressor", "ExtraTreesClassifier", "ExtraTreesRegressor"}
_GB = {"GradientBoostingClassifier", "GradientBoostingRegressor"}
_HGB = {"HistGradientBoostingClassifier", "HistGradientBoostingRegressor"}
_ADABOOST = {"AdaBoostClassifier"}
_IFOREST = {"IsolationForest"}
_TREE_MODELS = _SKTREE_FORESTS | _GB | _HGB | _ADABOOST | _IFOREST
# the base estimators an AdaBoostClassifier is read with
_SKTREE_CLASSIFIERS = {"DecisionTreeClassifier", "ExtraTreeClassifier"}
# estimators that hold other estimators: a tree model inside one of them is refused by name
_CONTAINERS = {"Pipeline", "VotingClassifier", "VotingRegressor", "BaggingClassifier", "BaggingRegressor",
               "CalibratedClassifierCV", "StackingClassifier", "StackingRegressor", "OneVsRestClassifier",
               "OneVsOneClassifier", "MultiOutputRegressor", "MultiOutputClassifier"}


class TreeEnsembleSpec:
    """Flat node arrays of a tree ensemble and its head.

    feature [nodes] int32 (-1 at a leaf), threshold [nodes] float64, left / right [nodes] int32 (global node indices; -1 at
    a leaf), missing_left [nodes] uint8, value [nodes, R] float64 (leaf outputs, scaled), roots [T] int32, base [R],
    head in ``HEADS``, cmp ``CMP_F32`` / ``CMP_F64``; offset: what the ``"iforest"`` head subtracts."""

    activation = "trees"
    act_code = 6          # DKS_ACT_TREES
    maps = None

    def __init__(self, feature, threshold, left, right, missing_left, value, roots, base, head, cmp, n_features,
                 scalar_out=False, n_outputs=None, offset=0.0):
        self.feature = np.ascontiguousarray(feature, dtype=np.int32)
        self.threshold = np.ascontiguousarray(threshold, dtype=np.float64)
        self.left = np.ascontiguousarray(left, dtype=np.int32)
        self.right = np.ascontiguousarray(right, dtype=np.int32)
        self.missing_left = np.ascontiguousarray(missing_left, dtype=np.uint8)
        self.value = np.ascontiguousarray(np.atleast_2d(value), dtype=np.float64)
        self.roots = np.ascontiguousarray(roots, dtype=np.int32)
        self.base = np.ascontiguousarray(np.atleast_1d(base), dtype=np.float64)
        self.head = head
        self.cmp = int(cmp)
        self.n_features = int(n_features)
        self.scalar_out = bool(scalar_out)
        self.offset = float(offset)
        self.R = self.value.shape[1]
        self.n_outputs = int(n_outputs if n_outputs is not None else (2 if head == "sigmoid" else self.R))
        if head not in HEADS:
            raise ValueError(f"unknown tree head {head!r}")
        if self.n_outputs > MAX_OUTPUTS:
            raise NotImplementedError(f"{self.n_outputs} model outputs: the tree route covers at most {MAX_OUTPUTS}")

    @property
    def head_code(self):
        return HEADS.index(self.head)

    @property
    def n_nodes(self):
        return len(self.feature)

    @property
    def n_trees(self):
        return len(self.roots)

    def raw(self, X):
        """r = base + sum over trees of the leaf value [n, R], trees added in order."""
        X = np.atleast_2d(np.asarray(X, dtype=np.float64))
        Xc = X.astype(np.float32).astype(np.float64) if self.cmp == CMP_F32 else X
        n = X.shape[0]
        out = np.tile(self.base, (n, 1))
        rows = np.arange(n)
        for root in self.roots:
            node = np.full(n, root, dtype=np.int64)
            while True:
                f = self.feature[node]
                inner = f >= 0
                if not inner.any():
                    break
                v = Xc[rows[inner], f[inner]]
                nd = node[inner]
                go_left = np.where(np.isnan(v), self.missing_left[nd] != 0, v <= self.threshold[nd])
                node[inner] = np.where(go_left, self.left[nd], self.right[nd])
            out += self.value[node]
        return out

    def __call__(self, X):
        """The scikit-learn method the spec was read from, in NumPy."""
        r = self.raw(X)
        if self.head == "sigmoid":
            p1 = 1.0 / (1.0 + np.exp(-r[:, 0]))
            out = np.stack([1.0 - p1, p1], axis=1)
        elif self.head == "softmax":
            e = np.exp(r - r.max(axis=1, keepdims=True))
            out = e / e.sum(axis=1, keepdims=True)
        elif self.head == "exp":
            out = np.exp(r)
        elif self.head == "iforest":
            out = -np.exp2(r) - self.offset
        else:
            out = r
        return out[:, 0] if self.scalar_out else out


def _names(obj):
    return {c.__name__ for c in type(obj).__mro__ if c.__module__.startswith("sklearn.")}


def _contains_tree(obj, depth=0):
    if depth > 6 or obj is None:
        return False
    if _names(obj) & _TREE_MODELS:
        return True
    kids = []
    for attr in ("steps", "estimators", "estimators_", "calibrated_classifiers_", "estimator", "base_estimator",
                 "estimator_", "final_estimator_"):
        v = getattr(obj, attr, None)
        if v is None or isinstance(v, str):
            continue
        if isinstance(v, (list, tuple, np.ndarray)):
            for e in np.ravel(np.asarray(v, dtype=object)) if isinstance(v, np.ndarray) else v:
                kids.append(e[-1] if isinstance(e, tuple) else e)
        else:
            kids.append(v)
    for k in kids:
        if hasattr(k, "estimator") and not (_names(k) & (_CONTAINERS | _TREE_MODELS)):
            k = k.estimator                 # calibrated classifier wrappers
        if _contains_tree(k, depth + 1):
            return True
    return False


def _flatten(trees, n_features):
    """trees: list of (feature, threshold, left, right, missing_left, value [nodes, R]) with tree-local child indices."""
    feats, thrs, lefts, rights, miss, vals, roots = [], [], [], [], [], [], []
    off = 0
    for f, t, l, r, m, v in trees:
        f = np.asarray(f, dtype=np.int64)
        leaf = f < 0
        roots.append(off)
        feats.append(np.where(leaf, -1, f))
        thrs.append(np.where(leaf, 0.0, np.asarray(t, dtype=np.float64)))
        lefts.append(np.where(leaf, -1, np.asarray(l, dtype=np.int64) + off))
        rights.append(np.where(leaf, -1, np.asarray(r, dtype=np.int64) + off))
        miss.append(np.asarray(m, dtype=np.uint8))
        vals.append(np.where(leaf[:, None], np.asarray(v, dtype=np.float64), 0.0))
        off += len(f)
    if off >= 2 ** 31 - 1:
        raise NotImplementedError("tree ensemble with more than 2^31 nodes")
    out = [np.concatenate(a) for a in (feats, thrs, lefts, rights, miss, vals)]
    if (out[0] >= n_features).any():
        raise ValueError("a split refers to a feature the model does not have")
    return out + [np.asarray(roots)]


def _sk_tree(est, value):
    t = est.tree_
    feature = np.where(t.children_left < 0, -1, t.feature)
    miss = getattr(t, "missing_go_to_left", np.zeros(t.node_count, dtype=np.uint8))
    return feature, t.threshold, t.children_left, t.children_right, miss, value


def _classifier_fractions(est, n_classes):
    v = np.asarray(est.tree_.value[:, 0, :n_classes], dtype=np.float64)
    s = v.sum(axis=1, keepdims=True)
    s[s == 0.0] = 1.0
    return v / s


def _forest_spec(owner, method, names):
    ests = list(getattr(owner, "estimators_", [owner]))
    P = int(owner.n_features_in_)
    if getattr(owner, "n_outputs_", 1) != 1:
        raise NotImplementedError(f"{type(owner).__name__} with {owner.n_outputs_} outputs: multi-output trees are not "
                                  "supported")
    T = len(ests)
    if hasattr(owner, "classes_"):
        if method != "predict_proba":
            raise TypeError(f"{type(owner).__name__}.{method} is not supported: pass predict_proba (predict returns labels)")
        C = len(owner.classes_)
        if C > MAX_OUTPUTS:
            raise NotImplementedError(f"{C} classes: the tree route covers at most {MAX_OUTPUTS} outputs")
        trees = [_sk_tree(e, _classifier_fractions(e, C) / T) for e in ests]
        arrs = _flatten(trees, P)
        return TreeEnsembleSpec(*arrs[:6], arrs[6], np.zeros(C), "identity", CMP_F32, P)
    if method != "predict":
        raise TypeError(f"{type(owner).__name__}.{method} is not supported: pass predict")
    trees = [_sk_tree(e, np.asarray(e.tree_.value[:, 0, :1], dtype=np.float64) / T) for e in ests]
    arrs = _flatten(trees, P)
    return TreeEnsembleSpec(*arrs[:6], arrs[6], np.zeros(1), "identity", CMP_F32, P, scalar_out=True)


def _gb_spec(owner, method, names):
    P = int(owner.n_features_in_)
    init = owner.init_
    if not (isinstance(init, str) and init == "zero") and not (_names(init) & {"DummyClassifier", "DummyRegressor"}):
        raise NotImplementedError(f"{type(owner).__name__} with init={type(init).__name__}: only the default "
                                  "(DummyClassifier / DummyRegressor) or 'zero' initial estimator is supported")
    stages = owner.estimators_            # [n_stages, K] DecisionTreeRegressor
    K = stages.shape[1]
    base = np.asarray(owner._raw_predict_init(np.zeros((1, P))), dtype=np.float64).reshape(-1)
    lr = float(owner.learning_rate)
    trees = []
    for s in range(stages.shape[0]):
        for k in range(K):
            e = stages[s, k]
            v = np.zeros((e.tree_.node_count, K))
            v[:, k] = lr * e.tree_.value[:, 0, 0]
            trees.append(_sk_tree(e, v))
    arrs = _flatten(trees, P)
    return _boosted_head(owner, method, arrs, base, K, CMP_F32, P)


def _boosted_head(owner, method, arrs, base, K, cmp, P, link_exp=False):
    name = type(owner).__name__
    if hasattr(owner, "classes_"):
        C = len(owner.classes_)
        if C > MAX_OUTPUTS:
            raise NotImplementedError(f"{C} classes: the tree route covers at most {MAX_OUTPUTS} outputs")
        if method == "predict_proba":
            return TreeEnsembleSpec(*arrs[:6], arrs[6], base, "sigmoid" if K == 1 else "softmax", cmp, P)
        if method == "decision_function":
            return TreeEnsembleSpec(*arrs[:6], arrs[6], base, "identity", cmp, P, scalar_out=K == 1)
        raise TypeError(f"{name}.{method} is not supported: pass predict_proba or decision_function")
    if method != "predict":
        raise TypeError(f"{name}.{method} is not supported: pass predict")
    if K != 1:
        raise NotImplementedError(f"{name} with {K} outputs: multi-output regressors are not supported")
    return TreeEnsembleSpec(*arrs[:6], arrs[6], base, "exp" if link_exp else "identity", cmp, P, scalar_out=True)


def _hgb_spec(owner, method, names):
    P = int(owner.n_features_in_)
    if getattr(owner, "_preprocessor", None) is not None:
        raise NotImplementedError(f"{type(owner).__name__} with categorical features (a fitted _preprocessor): "
                                  "categorical splits are not supported")
    cat = getattr(owner, "is_categorical_", None)
    if cat is not None and np.any(cat):
        raise NotImplementedError(f"{type(owner).__name__} with categorical features: categorical splits are not supported")
    K = int(owner.n_trees_per_iteration_)
    base = np.asarray(owner._baseline_prediction, dtype=np.float64).reshape(-1)
    trees = []
    for it in owner._predictors:
        for k, pred in enumerate(it):
            nd = pred.nodes
            if np.any(nd["is_categorical"]):
                raise NotImplementedError("categorical splits are not supported")
            leaf = nd["is_leaf"].astype(bool)
            v = np.zeros((len(nd), K))
            v[:, k] = np.where(leaf, nd["value"], 0.0)
            f = np.where(leaf, -1, nd["feature_idx"].astype(np.int64))
            trees.append((f, nd["num_threshold"], nd["left"], nd["right"], nd["missing_go_to_left"], v))
    arrs = _flatten(trees, P)
    link_exp = False
    if not hasattr(owner, "classes_"):
        link = type(getattr(getattr(owner, "_loss", None), "link", None)).__name__
        if link not in ("IdentityLink", "LogLink"):
            raise NotImplementedError(f"{type(owner).__name__} with loss {owner.loss!r}: identity or log link only")
        link_exp = link == "LogLink"
    return _boosted_head(owner, method, arrs, base, K, CMP_F64, P, link_exp=link_exp)


def _average_path_length(n):
    """c(n) of ``sklearn.ensemble._iforest``: 0 for n <= 1, 1 for n = 2, else 2 (ln(n - 1) + gamma) - 2 (n - 1) / n."""
    n = np.asarray(n, dtype=np.float64)
    out = np.zeros(n.shape)
    big = n > 2
    out[n == 2] = 1.0
    out[big] = 2.0 * (np.log(n[big] - 1.0) + np.euler_gamma) - 2.0 * (n[big] - 1.0) / n[big]
    return out


def _iforest_spec(owner, method, names):
    if method not in ("score_samples", "decision_function"):
        raise TypeError(f"IsolationForest.{method} is not supported: pass decision_function or score_samples "
                        "(predict returns labels)")
    P = int(owner.n_features_in_)
    ests = list(owner.estimators_)
    d = len(ests) * float(_average_path_length([owner.max_samples_])[0])
    trees = []
    for e, feats in zip(ests, owner.estimators_features_):
        t = e.tree_
        h = t.compute_node_depths() + _average_path_length(t.n_node_samples) - 1.0
        feature, thr, left, right, miss, _ = _sk_tree(e, None)
        if len(feats) != P:                     # a feature subset: scikit-learn reads X[:, feats]
            feature = np.where(feature < 0, -1, np.asarray(feats)[np.maximum(feature, 0)])
        # d = 0 (max_samples = 1): scikit-learn takes the ratio as 1, so r = base = -1 and every score is -2^-1
        trees.append((feature, thr, left, right, miss, (-h / d if d != 0 else np.zeros_like(h))[:, None]))
    arrs = _flatten(trees, P)
    offset = float(owner.offset_) if method == "decision_function" else 0.0
    return TreeEnsembleSpec(*arrs[:6], arrs[6], np.array([0.0 if d != 0 else -1.0]), "iforest", CMP_F32, P,
                            scalar_out=True, offset=offset)


def _adaboost_spec(owner, method, names):
    name = type(owner).__name__
    if method not in ("predict_proba", "decision_function"):
        raise TypeError(f"{name}.{method} is not supported: pass predict_proba or decision_function (predict returns "
                        "labels)")
    P = int(owner.n_features_in_)
    classes = np.asarray(owner.classes_)
    K = len(classes)
    if K < 2:
        raise NotImplementedError(f"{name} with one class: its outputs are constant, there is nothing to explain")
    if K > MAX_OUTPUTS:
        raise NotImplementedError(f"{K} classes: the tree route covers at most {MAX_OUTPUTS} outputs")
    ests = list(owner.estimators_)
    for e in ests:
        if not (_names(e) & _SKTREE_CLASSIFIERS):
            raise NotImplementedError(f"{name} over {type(e).__name__}: only sklearn.tree classifiers "
                                      "(DecisionTreeClassifier, ExtraTreeClassifier) are supported as base estimators")
        if getattr(e, "n_outputs_", 1) != 1:
            raise NotImplementedError(f"{name} over multi-output trees is not supported")
    w = np.asarray(owner.estimator_weights_, dtype=np.float64)
    wsum = float(w.sum())
    # SAMME: K = 2 folds dec[1] - dec[0] into one score (+-2 w_t); more classes: K scores, over K - 1 for predict_proba
    scale = 1.0 / wsum if K == 2 or method == "decision_function" else 1.0 / (wsum * (K - 1))
    trees = []
    for e, wt in zip(ests, w):              # an early stop leaves fewer estimators than weights; the rest are 0
        pred = np.searchsorted(classes, e.classes_)[np.argmax(e.tree_.value[:, 0, :], axis=1)]    # ensemble indices
        if K == 2:
            v = np.where(pred == 1, 2.0 * wt, -2.0 * wt)[:, None] * scale
        else:
            v = np.full((e.tree_.node_count, K), -wt / (K - 1))
            v[np.arange(len(pred)), pred] = wt
            v *= scale
        trees.append(_sk_tree(e, v))
    arrs = _flatten(trees, P)
    R = 1 if K == 2 else K
    if method == "predict_proba":
        return TreeEnsembleSpec(*arrs[:6], arrs[6], np.zeros(R), "sigmoid" if K == 2 else "softmax", CMP_F32, P)
    return TreeEnsembleSpec(*arrs[:6], arrs[6], np.zeros(R), "identity", CMP_F32, P, scalar_out=K == 2)


def extract_tree_spec(predictor):
    """``TreeEnsembleSpec`` of a bound method of a fitted scikit-learn tree model, ``None`` for anything else (the engine
    then reads a linear model).  A spec passes through.  Raises ``NotImplementedError`` / ``TypeError`` naming the reason
    for tree models the route does not cover: categorical splits, custom boosting init estimators, multi-output
    regressors, more than 8 outputs, trees inside a Pipeline or an ensemble, ``AdaBoostRegressor``, AdaBoost over base
    estimators that are not ``sklearn.tree`` classifiers or with one class, and unsupported methods."""
    if isinstance(predictor, TreeEnsembleSpec):
        return predictor
    owner = getattr(predictor, "__self__", None)
    method = getattr(predictor, "__name__", None)
    if owner is None:
        return None
    names = _names(owner)
    if "AdaBoostRegressor" in names:
        raise NotImplementedError("AdaBoostRegressor: its prediction is the weighted median of its trees' predictions, "
                                  "not a sum of leaf values, so the tree route cannot read it")
    if names & _TREE_MODELS:
        if not hasattr(owner, "n_features_in_"):
            raise TypeError(f"{type(owner).__name__} is not fitted")
        if names & _IFOREST:
            return _iforest_spec(owner, method, names)
        if names & _ADABOOST:
            return _adaboost_spec(owner, method, names)
        if names & _HGB:
            return _hgb_spec(owner, method, names)
        if names & _GB:
            return _gb_spec(owner, method, names)
        return _forest_spec(owner, method, names)
    if names & _CONTAINERS and _contains_tree(owner):
        raise NotImplementedError(f"{type(owner).__name__} holding a tree model: trees inside an ensemble are not "
                                  "supported, and a Pipeline of per-column steps ending in a tree model is read by "
                                  "extract_tree_pipeline_spec; pass the tree model's own method")
    return None


def extract_tree_pipeline_spec(predictor):
    """``(TreeEnsembleSpec, ColumnEncoding)`` of a bound method of a fitted ``Pipeline`` of per-column steps ending in a
    tree model ``extract_tree_spec`` reads: the spec of the final estimator (its features index the encoded columns) and
    the exact programs of ``pipe[:-1].transform`` (``column_maps.compile_encoding``).  ``None`` for anything else.  The
    steps the column maps refuse raise ``TypeError`` naming the step; so do trees inside ensembles or calibrators behind
    the pipeline, and the final estimator's own refusals raise as in ``extract_tree_spec``."""
    from .column_maps import compile_encoding, pipeline_parts
    owner = getattr(predictor, "__self__", None)
    method = getattr(predictor, "__name__", None)
    if owner is None or "Pipeline" not in _names(owner) or not hasattr(owner, "steps"):
        return None
    pre, final = pipeline_parts(owner)
    if not (_names(final) & _TREE_MODELS):
        return None
    if not hasattr(owner, "n_features_in_") or not hasattr(final, "n_features_in_"):
        raise TypeError("Pipeline is not fitted")
    spec = extract_tree_spec(getattr(final, method))
    enc = compile_encoding(pre, int(owner.n_features_in_), spec.n_features)
    spec.n_features = enc.D
    return spec, enc


def _foldable(step):
    """A step ``kernel_machines._unwrap`` folds into the model: one of the four affine scalers (``MinMaxScaler``
    without ``clip``), or no step."""
    from .kernel_machines import _SCALERS
    if step is None or isinstance(step, str):
        return True
    return type(step).__name__ in _SCALERS and not (type(step).__name__ == "MinMaxScaler" and step.clip)


def extract_encoded_pipeline_spec(predictor):
    """``(spec, ColumnEncoding)`` of a bound method of a fitted ``Pipeline`` of per-column steps ending in a kernel
    machine (``extract_kernel_machine_spec``, the sigmoid-calibrated SVC included), an MLP (``extract_mlp_spec``) or a
    k-nearest-neighbour model (``extract_knn_spec``), when some step is not one of the four affine scalers those
    extractors fold: the spec of the bare final estimator (its columns are the encoded ones, ``colw = 1`` and
    ``colo = 0``) and the exact programs of the steps (``column_maps.compile_encoding``).  A
    ``CalibratedClassifierCV(ensemble=False)`` whose one fold is such a pipeline counts as one.  ``None`` for anything
    else, scaler-only pipelines included (the extractors fold those).  Raises ``NotImplementedError`` naming the step
    for steps the encoding refuses and for calibrated ensembles whose folds each hold their own fitted preprocessing; the
    final estimator's own refusals raise as in its extractor."""
    from .column_maps import compile_encoding, pipeline_parts
    from .kernel_machines import _calibrated_spec, _final, _is_kernel_machine, extract_kernel_machine_spec
    from .mlp import _MLPS, extract_mlp_spec
    from .neighbors import _KNN, extract_knn_spec
    owner = getattr(predictor, "__self__", None)
    method = getattr(predictor, "__name__", None)
    if owner is None:
        return None
    pre, final = pipeline_parts(owner) if "Pipeline" in _names(owner) and hasattr(owner, "steps") else ([], owner)
    names = _names(final)
    inner = False                   # the preprocessing of a single calibrated fold is compiled too
    if "CalibratedClassifierCV" in names:
        ccs = getattr(final, "calibrated_classifiers_", None)
        if not ccs or not any(_is_kernel_machine(cc.estimator) for cc in ccs):
            return None
        family, extract = "a kernel machine", extract_kernel_machine_spec
        folds = [pipeline_parts(cc.estimator)[0] if "Pipeline" in _names(cc.estimator) else [] for cc in ccs]
        steps = [type(s).__name__ for s in folds[0] if not _foldable(s)]
        if any(not _foldable(s) for f in folds for s in f):
            if len(ccs) > 1:
                raise NotImplementedError(
                    f"CalibratedClassifierCV with {len(ccs)} folds, each with its own fitted preprocessing "
                    f"({', '.join(steps)}): the device holds one column encoding; move the preprocessing in front of "
                    "the calibrator (make_pipeline(preprocessing, CalibratedClassifierCV(...))) or pass ensemble=False")
            pre, inner = pre + folds[0], True
    elif _is_kernel_machine(final):
        family, extract = "a kernel machine", extract_kernel_machine_spec
    elif names & _MLPS:
        family, extract = "an MLP", extract_mlp_spec
    elif names & _KNN:
        family, extract = "a neighbour model", extract_knn_spec
    else:
        return None
    if all(_foldable(s) for s in pre):
        return None
    if not hasattr(owner, "n_features_in_"):
        raise TypeError("Pipeline is not fitted")
    if inner:
        bare = _final(final.calibrated_classifiers_[0].estimator)
        if not hasattr(bare, "n_features_in_"):
            raise TypeError(f"{type(bare).__name__} is not fitted")
        spec = _calibrated_spec(final, method, int(bare.n_features_in_), bare=True)
    else:
        spec = extract(getattr(final, method))
    if spec is None:
        return None
    try:
        enc = compile_encoding(pre, int(owner.n_features_in_), spec.n_features, model=family)
    except TypeError as e:
        raise NotImplementedError(f"Pipeline in front of {family}: {e}") from e
    spec.n_features = enc.D
    return spec, enc
