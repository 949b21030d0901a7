"""The float64 multi-output reference (softmax head with C classes, identity head with R outputs) against the oracle and
against exact Shapley values."""
import itertools
from math import factorial

import numpy as np
import pytest

from multiclass_reference import MultiOutputReference


def _problem(seed, C, widths, N=12, weights=False, scale=1.0):
    rng = np.random.default_rng(seed)
    groups, start = [], 0
    for wd in widths:
        groups.append(list(range(start, start + wd)))
        start += wd
    D = start
    W = rng.normal(0, 0.8, (C, D)) * scale
    b = rng.normal(0, 0.5, C) * scale
    bg, X = rng.standard_normal((N, D)), rng.standard_normal((3, D))
    wts = rng.uniform(0.2, 1.0, N) if weights else None
    return W, b, bg, X, groups, wts


def _oracle(W, b, bg, groups, wts, head, link):
    from distributedkernelshap_b200.predictors import LinearModelSpec
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    spec = LinearModelSpec(W, b, "softmax" if head == "softmax" else "identity")
    return KernelExplainerOracle(spec, DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, wts), link=link)


@pytest.mark.parametrize("head,link,C,weights", [("softmax", "logit", 3, False), ("softmax", "identity", 5, True),
                                                 ("softmax", "logit", 8, True), ("identity", "identity", 3, False),
                                                 ("identity", "identity", 1, True)])
def test_reference_matches_oracle(head, link, C, weights):
    from distributedkernelshap_b200.plan import build_plan
    W, b, bg, X, groups, wts = _problem(11 + C, C, (1, 2, 1, 1, 2, 1), weights=weights)
    ref = MultiOutputReference(W, b, bg, groups, wts, head=head, link=link)
    orc = _oracle(W, b, bg, groups, wts, head, link)
    np.random.seed(1)
    plan = build_plan(6, 40)
    for x in X:
        want = orc.explain(x[None, :], plan=(plan.dense(), plan.weights), nsamples=40, l1_reg=False)
        got = ref.explain(x, plan=(plan.dense(), plan.weights))
        np.testing.assert_allclose(got, want.reshape(got.shape), rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("head,link", [("softmax", "logit"), ("softmax", "identity"), ("identity", "identity")])
def test_reference_full_enumeration_is_exact_shapley(head, link):
    """With every coalition enumerated KernelSHAP is exact: phi = Shapley values of v(S) = link(E_bg f(x_S, bg_rest))."""
    from distributedkernelshap_b200.plan import build_plan
    W, b, bg, X, groups, wts = _problem(5, 4, (1, 2, 1, 1), weights=True)
    ref = MultiOutputReference(W, b, bg, groups, wts, head=head, link=link)
    M = len(groups)
    plan = build_plan(M, 10 ** 6)
    x = X[0]

    def value(S):
        rows = bg.copy()
        for k in S:
            rows[:, groups[k]] = x[groups[k]]
        return ref.link(np.einsum("jc,j->c", ref._outputs(b + rows @ W.T), ref.weights))

    exact = np.zeros((M, W.shape[0]))
    for k in range(M):
        rest = [q for q in range(M) if q != k]
        for r in range(M):
            for S in itertools.combinations(rest, r):
                wgt = factorial(r) * factorial(M - r - 1) / factorial(M)
                exact[k] += wgt * (value(S + (k,)) - value(S))
    got = ref.explain(x, plan=(plan.dense(), plan.weights))
    np.testing.assert_allclose(got, exact, rtol=1e-10, atol=1e-12)
