"""The float64 tree reference (tests/tree_reference.py) against scikit-learn's own methods and ``TreeEnsembleSpec.__call__``
on thresholds, their float32 neighbours, NaN and infinity; the hand-built ensembles and problems the GPU edge tests use
(tests/test_gpu_tree_edges.py) have the properties those tests rely on.  No GPU."""
import numpy as np
import pytest

sklearn = pytest.importorskip("sklearn")

import tree_reference as ref  # noqa: E402
from test_tree_specs import CASES, _probe  # noqa: E402

from distributedkernelshap_b200.trees import CMP_F32, CMP_F64, extract_tree_spec  # noqa: E402
from oracle.shap_kernel_oracle import KernelExplainerOracle, build_plan  # noqa: E402


def _agree(got, want):
    want = np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * max(1.0, np.max(np.abs(want))))


@pytest.mark.parametrize("k", range(len(CASES)))
def test_walk_reproduces_sklearn_and_the_spec(k):
    est, method, nan = CASES[k]
    fn = getattr(est, method)
    spec = extract_tree_spec(fn)
    rng = np.random.default_rng(100 + k)
    X = _probe(spec, rng, nan=nan)                       # thresholds, both float32 neighbours, NaN
    Xt, _ = ref.on_thresholds(spec, rng, 100)            # and the float64 neighbours
    X = np.concatenate([X, Xt])
    if spec.cmp == CMP_F64:                              # the histogram estimators take infinite inputs
        X[rng.random(X.shape) < 0.03] = np.inf
        X[rng.random(X.shape) < 0.03] = -np.inf
    got = ref.model(spec)(X)
    _agree(got, fn(X))
    _agree(got, spec(X))
    i = int(rng.integers(0, len(X)))                     # the one-row, one-node loop reaches the same leaves
    one = spec.base + sum(spec.value[ref.leaf_of(spec, t, X[i])] for t in range(spec.n_trees))
    np.testing.assert_allclose(ref.walk(spec, X[i:i + 1])[0], one, rtol=0, atol=1e-12)


def test_missing_versus_rest_split_has_an_infinite_threshold():
    est, X = ref.hgb_with_missing_split()
    spec = extract_tree_spec(est.predict_proba)
    inner = spec.feature >= 0
    assert np.any(np.isposinf(spec.threshold[inner])), "no +inf threshold: this scikit-learn encodes the split otherwise"
    assert not np.any(np.isnan(spec.threshold[inner]))
    rng = np.random.default_rng(0)
    P = rng.normal(size=(200, 5))
    for v, lo in ((np.nan, 0), (np.inf, 50), (-np.inf, 100)):
        P[lo:lo + 50, 0] = v
    P[150:170, 1] = np.inf
    got = ref.model(spec)(P)
    _agree(got, est.predict_proba(P))
    _agree(got, spec(P))
    # a hand-built node of the same kind: everything but NaN goes left
    stump = ref.stumps(1, [0], [np.inf], [1.0], [5.0], 1)
    np.testing.assert_array_equal(ref.model(stump)(np.array([[np.nan], [np.inf], [-np.inf], [0.0]])), [5.0, 1.0, 1.0, 1.0])
    np.testing.assert_array_equal(stump(np.array([[np.nan], [np.inf], [-np.inf], [0.0]])), [5.0, 1.0, 1.0, 1.0])


def test_hand_built_ensembles_are_well_formed():
    rng = np.random.default_rng(0)
    specs = [ref.stumps(3, [0, 1, 0], [0.1, 0.2, 0.3], [1, 2, 3], [4, 5, 6], 2),
             ref.chain(300, [0, 1], 2),
             ref.random_trees(rng, 7, (1, 3), 4, R=3, head="softmax", cmp=CMP_F32, inf_fraction=0.2)]
    for s in specs:
        inner = s.feature >= 0
        nd = np.arange(s.n_nodes)
        assert np.all(s.left[inner] > nd[inner]) and np.all(s.right[inner] > nd[inner])
        assert np.all(s.feature < s.n_features) and np.all(np.isfinite(s.value)) and not np.any(np.isnan(s.threshold))
        X = rng.normal(size=(50, s.n_features))
        _agree(ref.model(s)(X), s(X))
    assert ref.max_depth(specs[1]) == 300
    deep = ref.model(specs[1])(np.array([[10.0, 10.0], [1.505, 10.0], [10.0, -1.0]]))
    np.testing.assert_allclose(deep, [2.25, 0.25 + np.sin(152), 0.25 + np.sin(1)])


def test_both_kinds_of_tree_in_every_chunk_of_the_divergence_pass():
    for R in (1, 3):
        for T in ref.CHUNK_T:
            spec, bg, X = ref.chunk_problem(T, R)
            assert spec.n_trees == T and spec.R == R
            div = np.array([[ref.divergent_trees(spec, x, b, set(range(6))) for b in bg] for x in X])    # [n, N, T]
            for t0 in range(0, T, 256):
                c = div[:, :, t0:t0 + 256]
                if c.shape[2] > 1:
                    assert np.all(c.any(axis=2)) and not np.any(c.all(axis=2)), (T, R, t0)
                else:                                       # a chunk of one tree: both kinds over the (x, bg_j) pairs
                    assert c.any() and not c.all(), (T, R, t0)


def _phi(spec, bg, X, cmp):
    oracle = KernelExplainerOracle(ref.model(spec, cmp), bg, link="logit")
    M = bg.shape[1]
    Z, w, _ = build_plan(M, 2 ** M - 2)
    return np.stack([oracle.explain(X[i:i + 1], plan=(Z, w), l1_reg=False) for i in range(len(X))])


def test_the_comparison_code_changes_phi_on_the_tie_problem():
    # what gives the GPU test its teeth: on identical node arrays, background and instances the two comparison codes
    # have different Shapley values, so a kernel that ignored the code could not match both references
    spec, bg, X, share = ref.tie_problem(CMP_F32)
    assert share >= 1 / 3
    a, b = _phi(spec, bg, X, CMP_F32), _phi(spec, bg, X, CMP_F64)
    assert np.max(np.abs(a - b)) / np.max(np.abs(a)) > 1e-3
    per_instance = np.abs(a - b).max(axis=(1, 2)) / np.abs(a).max(axis=(1, 2))
    assert np.sum(per_instance > 1e-3) >= 3


def test_nan_problem_routes_one_feature_both_ways():
    spec = ref.nan_spec(CMP_F64)
    both = False
    for nd in np.nonzero(spec.feature >= 0)[0]:           # a node and a descendant on the same feature, NaN sent opposite ways
        todo = [spec.left[nd], spec.right[nd]]
        while todo:
            c = todo.pop()
            if spec.feature[c] < 0:
                continue
            both |= spec.feature[c] == spec.feature[nd] and spec.missing_left[c] != spec.missing_left[nd]
            todo += [spec.left[c], spec.right[c]]
    assert both
    assert set(spec.missing_left[spec.feature >= 0]) == {0, 1}
