"""An independent float64 reference for tree ensembles, and hand-built ensembles for the tree route's edge tests.

``walk`` and ``head`` restate the definition in include/dks.h (``dks_set_tree_model``) from the node arrays alone:
``r = base + sum over trees of the value of the leaf x reaches``, a split sends x left when ``x <= threshold`` (x cast to
float32 first under ``CMP_F32``), NaN goes left where ``missing_left`` is set, and the head maps r to the outputs.  Nothing
here calls ``TreeEnsembleSpec.raw`` / ``__call__``: ``distributedkernelshap_b200.trees`` is imported only for the container
the engine takes, so a mistake in the product's NumPy evaluation is not inherited.  phi comes from the oracle
(oracle/shap_kernel_oracle.py) fed ``model(arrays)`` and the engine's plan.

The builders return a ``TreeEnsembleSpec`` with every child after its parent, as ``dks_set_tree_model`` requires.
"""
import numpy as np
from scipy.special import expit, softmax

from distributedkernelshap_b200.trees import TreeEnsembleSpec

CMP_F32, CMP_F64 = 0, 1


# ---- the reference ------------------------------------------------------------------------------------------------
def goes_left(x, thr, miss, cmp):
    """One value at one node."""
    if x != x:
        return bool(miss)
    v = float(np.float32(x)) if cmp == CMP_F32 else float(x)
    return v <= thr


def leaf_of(a, k, x, cmp=None):
    """The leaf row x reaches in tree k, one node at a time."""
    cmp = a.cmp if cmp is None else cmp
    nd = int(a.roots[k])
    while a.feature[nd] >= 0:
        left = goes_left(x[a.feature[nd]], a.threshold[nd], a.missing_left[nd], cmp)
        nd = int(a.left[nd] if left else a.right[nd])
    return nd


def walk(a, X, cmp=None):
    """Raw scores [n, R] of the rows of X.  Each tree's rows are split node by node from the root down (the rows that
    reach a node are sent left or right together), which is the one-row loop of ``leaf_of`` applied to sets of rows."""
    cmp = a.cmp if cmp is None else cmp
    X = np.atleast_2d(np.asarray(X, dtype=np.float64))
    with np.errstate(over="ignore"):
        Xc = X.astype(np.float32).astype(np.float64) if cmp == CMP_F32 else X
    out = np.tile(np.asarray(a.base, dtype=np.float64), (X.shape[0], 1))
    for root in a.roots:
        todo = [(int(root), np.arange(X.shape[0]))]
        while todo:
            nd, rows = todo.pop()
            if len(rows) == 0:
                continue
            f = a.feature[nd]
            if f < 0:
                out[rows] += a.value[nd]
                continue
            v = Xc[rows, f]
            left = np.where(np.isnan(v), bool(a.missing_left[nd]), v <= a.threshold[nd])
            todo.append((int(a.left[nd]), rows[left]))
            todo.append((int(a.right[nd]), rows[~left]))
    return out


def head(a, r):
    """Outputs [n, C] of the raw scores [n, R]."""
    if a.head == "sigmoid":
        return np.stack([expit(-r[:, 0]), expit(r[:, 0])], axis=1)
    if a.head == "softmax":
        return softmax(r, axis=1)
    if a.head == "exp":
        return np.exp(r)
    assert a.head == "identity"
    return r


def model(a, cmp=None):
    """The callable the oracle explains: head(walk(X)), ``[n]`` for a scalar-output ensemble."""
    def fn(X):
        out = head(a, walk(a, X, cmp))
        return out[:, 0] if a.scalar_out else out
    return fn


def divergent_trees(a, x, b, varying_cols, cmp=None):
    """Per tree, whether x and background row b part ways at a node on a varying column before reaching a leaf, walking
    b's way everywhere else (the masked row keeps b's value on columns that do not vary)."""
    cmp = a.cmp if cmp is None else cmp
    out = np.zeros(len(a.roots), dtype=bool)
    for k in range(len(a.roots)):
        nd = int(a.roots[k])
        while a.feature[nd] >= 0:
            f = a.feature[nd]
            wb = goes_left(b[f], a.threshold[nd], a.missing_left[nd], cmp)
            if f in varying_cols and goes_left(x[f], a.threshold[nd], a.missing_left[nd], cmp) != wb:
                out[k] = True
                break
            nd = int(a.left[nd] if wb else a.right[nd])
    return out


def max_depth(a):
    depth = np.zeros(len(a.feature), dtype=np.int64)
    for nd in range(len(a.feature)):                    # children follow their parent
        if a.feature[nd] >= 0:
            depth[a.left[nd]] = depth[a.right[nd]] = depth[nd] + 1
    return int(depth.max())


# ---- hand-built ensembles -----------------------------------------------------------------------------------------
class _Nodes:
    def __init__(self, R):
        self.R = R
        self.feature, self.threshold, self.left, self.right, self.miss, self.value, self.roots = [], [], [], [], [], [], []

    def add(self, feature=-1, threshold=0.0, miss=0, value=None):
        self.feature.append(feature)
        self.threshold.append(threshold)
        self.left.append(-1)
        self.right.append(-1)
        self.miss.append(miss)
        self.value.append(np.zeros(self.R) if value is None else np.asarray(value, dtype=np.float64))
        return len(self.feature) - 1

    def spec(self, base, head, cmp, P):
        return TreeEnsembleSpec(self.feature, self.threshold, self.left, self.right, self.miss, np.array(self.value),
                                self.roots, base, head, cmp, P, scalar_out=(head in ("identity", "exp") and self.R == 1))


def _leaf_value(rng, k, R, scale):
    v = np.zeros(R)
    v[k % R] = scale * rng.normal()           # tree k feeds raw score k mod R, as a boosting stage's K trees do
    return v


def stumps(T, features, thresholds, left_values, right_values, P, base=0.0, head="identity", cmp=CMP_F64, missing_left=0):
    """T depth-1 trees: tree k splits ``features[k]`` at ``thresholds[k]``; values [T] or [T, R]."""
    lv, rv = np.asarray(left_values, dtype=np.float64).reshape(T, -1), np.asarray(right_values, dtype=np.float64).reshape(T, -1)
    nodes = _Nodes(lv.shape[1])
    miss = np.broadcast_to(missing_left, (T,))
    for k in range(T):
        root = nodes.add(int(features[k]), float(thresholds[k]), int(miss[k]))
        nodes.roots.append(root)
        nodes.left[root] = nodes.add(value=lv[k])
        nodes.right[root] = nodes.add(value=rv[k])
    return nodes.spec(np.broadcast_to(base, (nodes.R,)), head, cmp, P)


def chain(depth, features, P, step=0.01, cmp=CMP_F64):
    """One degenerate tree of the given depth: node k splits ``features[k % len]`` at ``k * step``, its left child a
    leaf worth ``sin(k)``, its right child node k + 1; a row goes down while its value exceeds the thresholds."""
    nodes = _Nodes(1)
    nd = nodes.add(int(features[0]), 0.0)
    nodes.roots.append(nd)
    for k in range(depth):
        nodes.left[nd] = nodes.add(value=[np.sin(k)])
        nxt = nodes.add(int(features[(k + 1) % len(features)]), (k + 1) * step) if k + 1 < depth else nodes.add(value=[2.0])
        nodes.right[nd] = nxt
        nd = nxt
    return nodes.spec([0.25], "identity", cmp, P)


def random_trees(rng, T, depth, P, R=1, head="identity", cmp=CMP_F64, missing="random", features=None, scale=None,
                 inf_fraction=0.0):
    """T trees of depth drawn from ``depth`` (an int or (lo, hi)), splits on ``features`` (default every column) at
    normal thresholds, a fraction ``inf_fraction`` of them +inf; ``missing``: 0, 1 or
    'random' per node.  Tree k's leaves feed raw score k mod R, of size ``scale`` (default 1 / sqrt(T / R))."""
    features = np.arange(P) if features is None else np.asarray(features)
    lo, hi = (depth, depth) if np.isscalar(depth) else depth
    scale = 1.0 / np.sqrt(max(T // R, 1)) if scale is None else scale
    nodes = _Nodes(R)

    def grow(k, d):
        if d == 0:
            return nodes.add(value=_leaf_value(rng, k, R, scale))
        thr = float(rng.normal())
        if rng.random() < inf_fraction:
            thr = np.inf
        miss = int(rng.integers(0, 2)) if missing == "random" else int(missing)
        nd = nodes.add(int(rng.choice(features)), thr, miss)
        nodes.left[nd] = grow(k, d - 1)
        nodes.right[nd] = grow(k, d - 1)
        return nd

    for k in range(T):
        nodes.roots.append(len(nodes.feature))
        grow(k, int(rng.integers(lo, hi + 1)))
    return nodes.spec(0.1 * rng.normal(size=R), head, cmp, P)


# ---- inputs on split thresholds -------------------------------------------------------------------------------------
def on_thresholds(spec, rng, rows, fraction=0.45):
    """Normal rows with ``fraction`` of the entries moved onto a finite threshold of their column: the threshold itself,
    its float64 neighbours, and just inside the float32 neighbours of its float32 rounding -- the values on which the
    float32 cast decides the side.  Returns (X, share of entries placed)."""
    X = rng.normal(size=(rows, spec.n_features))
    placed = 0
    for f in range(spec.n_features):
        thr = spec.threshold[(spec.feature == f) & np.isfinite(spec.threshold)]
        if len(thr) == 0:
            continue
        for i in range(rows):
            if rng.random() >= fraction:
                continue
            t = float(rng.choice(thr))
            t32 = np.float32(t)
            X[i, f] = (t, float(np.nextafter(t, np.inf)), float(np.nextafter(t, -np.inf)),
                       float(np.nextafter(t32, np.float32(np.inf))) - 1e-13,
                       float(np.nextafter(t32, np.float32(-np.inf))) + 1e-13)[int(rng.integers(0, 5))]
            placed += 1
    return X, placed / X.size


# ---- problems shared by the CPU and the GPU tests ---------------------------------------------------------------------
CHUNK_T = (1, 255, 256, 257, 512, 513, 700)     # tree counts around the 256 trees one divergence pass takes


def nan_spec(cmp, inf_fraction=0.0):
    """Eight depth-3 trees over 4 columns whose nodes send NaN either way: with so few columns a path splits one
    feature twice, with both values of ``missing_left``."""
    return random_trees(np.random.default_rng(11), 8, 3, 4, cmp=cmp, missing="random", inf_fraction=inf_fraction, scale=1.0)


def chunk_problem(T, R, seed=0):
    """Hand-built depth 1..3 trees over 6 columns, 2 instances and 5 background rows for the tree kernel's divergence
    pass, which takes the trees 256 at a time.  The heads are not linear: under an identity head and link a constant
    added to every coalition's value (a lost leaf of a non-divergent tree) cancels in the Shapley values."""
    rng = np.random.default_rng(1000 * R + T + seed)
    spec = random_trees(rng, T, (1, 3), 6, R=R, head="softmax" if R > 1 else "sigmoid", cmp=CMP_F32)
    return spec, rng.normal(size=(5, 6)), rng.normal(size=(2, 6))


def tie_problem(cmp, seed=5):
    """Hand-built trees with thresholds no float32 holds, and a background and instances that sit on them."""
    rng = np.random.default_rng(seed)
    spec = random_trees(rng, 12, (2, 3), 6, R=1, head="sigmoid", cmp=cmp, scale=1.0)
    bg, share_bg = on_thresholds(spec, rng, 8)
    X, share_x = on_thresholds(spec, rng, 6)
    return spec, bg, X, min(share_bg, share_x)


def hgb_with_missing_split(seed=0):
    """A fitted HistGradientBoostingClassifier on data whose column 0 is 30 % NaN and informative through its missingness,
    so that the trees hold missing-versus-rest splits (threshold +inf)."""
    from sklearn.ensemble import HistGradientBoostingClassifier
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(600, 5))
    gone = rng.random(600) < 0.3
    y = (np.where(gone, 1.5, -0.5) + 0.5 * X[:, 1] + 0.3 * rng.normal(size=600) > 0).astype(int)
    X[gone, 0] = np.nan
    return HistGradientBoostingClassifier(max_iter=12, max_depth=3, random_state=0).fit(X, y), X
