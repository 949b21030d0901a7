"""Pins the fast float64 reference (tests/linear_reference.py) that the GPU kernel-path matrix compares against: it must
agree with the CPU oracle fed the same plan to 1e-12 relative, and with exact Shapley values under full enumeration."""
import time

import numpy as np
import pytest

from conftest import make_problem, rel_err
from linear_reference import LinearReference
from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle, build_plan, effective_nsamples, exact_shapley


def _pair(prob, link, head="logistic"):
    clf = prob["clf"]
    args = (prob["groups"],) + ((prob["weights"],) if prob["weights"] is not None else ())
    dd = DenseData(prob["bg"], prob["group_names"], *args)
    predict = clf.predict_proba if head == "logistic" else clf.decision_function
    orc = KernelExplainerOracle(predict, dd, link=link)
    kappa = 2.0 if clf.multi_class == "multinomial" else 1.0
    ref = LinearReference(clf.coef_, clf.intercept_, prob["bg"], prob["groups"], prob["weights"], head=head, kappa=kappa,
                          link=link)
    return orc, ref


def _check_against_oracle(prob, link, nsamples, head="logistic", seed=0):
    orc, ref = _pair(prob, link, head)
    np.testing.assert_allclose(ref.expected_value, np.atleast_1d(orc.expected_value), rtol=1e-13, atol=1e-15)
    worst = 0.0
    for i in range(prob["X"].shape[0]):
        x = prob["X"][i]
        v = ref.varying(x)
        np.testing.assert_array_equal(v, orc.varying_groups(x[None]))
        plan = None
        if len(v) >= 2:
            S, _ = effective_nsamples(len(v), nsamples)
            np.random.seed(seed + i)
            Z, w, _ = build_plan(len(v), S)
            plan = (Z, w)
        want = orc.explain(x[None], plan=plan, nsamples=nsamples, l1_reg=False).reshape(len(prob["groups"]), -1)
        got = ref.explain(x, plan)
        assert got.shape == want.shape
        for c in range(got.shape[1]):
            worst = max(worst, rel_err(got[:, c], want[:, c]))
    assert worst < 1e-12, worst
    return worst


@pytest.mark.parametrize("link", ["logit", "identity"])
@pytest.mark.parametrize("kappa", [1.0, 2.0])
def test_matches_oracle_sampled_plans_weights_and_partial_varying_sets(link, kappa):
    """Non-uniform weights, two constant groups (partial varying sets), a sampled plan of 9 groups."""
    prob = make_problem(seed=31, n=5, N=11, widths=(1, 2, 1, 1, 3, 1, 2, 1, 1, 1, 2), kappa=kappa, weights=True,
                        constant_groups=(3, 7))
    _check_against_oracle(prob, link, nsamples=150)


@pytest.mark.parametrize("link", ["logit", "identity"])
def test_matches_oracle_full_enumeration_m2_and_m16(link):
    """M = 2 (S = 2) and M = 16 with every one of the 65534 coalitions (exact Shapley values)."""
    _check_against_oracle(make_problem(seed=32, n=3, N=6, widths=(2, 1), kappa=1.0), link, nsamples=10 ** 6)
    _check_against_oracle(make_problem(seed=33, n=2, N=3, widths=(1,) * 16), link, nsamples=70000)


def test_matches_oracle_sampled_plan_70_groups():
    _check_against_oracle(make_problem(seed=34, n=2, N=5, widths=(1,) * 70, weights=True), "logit", nsamples=600)


def test_matches_oracle_identity_head():
    """decision_function (one output, the score itself) with the identity link: the affine case."""
    _check_against_oracle(make_problem(seed=35, n=4, N=9, widths=(1, 2, 1, 3, 1, 1), weights=True), "identity",
                          nsamples=40, head="identity")


@pytest.mark.parametrize("link", ["logit", "identity"])
def test_full_enumeration_equals_exact_shapley_values(link):
    prob = make_problem(seed=36, n=3, N=7, widths=(1, 2, 1, 1, 3, 1, 1, 2), weights=True)
    _, ref = _pair(prob, link)
    groups, wb, f = prob["groups"], ref.weights, prob["clf"].predict_proba
    for i in range(3):
        x = prob["X"][i]

        def value(mask):
            rows = prob["bg"].copy()
            for k, on in enumerate(mask):
                if on:
                    rows[:, groups[k]] = x[groups[k]]
            return ref.link((f(rows) * wb[:, None]).sum(0)) - ref.link(ref.fnull)
        want = exact_shapley(value, len(groups))
        S, _ = effective_nsamples(len(groups), 10 ** 6)
        Z, w, _ = build_plan(len(groups), S)
        got = ref.explain(x, (Z, w))
        np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-11)


def test_large_plan_is_fast():
    """S = 65534 coalitions x N = 128 background rows, the sizes of the GPU large-plan tests, cost a small multiple of one
    exponential over the [S, N] scores (about 20 of them): the reference never builds anything per background row and
    feature.  Timed against that exponential on the same machine, best of three, so that the bound holds on a slow or
    busy machine as well as on a fast one."""
    prob = make_problem(seed=37, n=1, N=128, widths=(1,) * 16)
    _, ref = _pair(prob, "logit")
    S, _ = effective_nsamples(16, 65534)
    Z, w, _ = build_plan(16, S)
    scores = np.random.default_rng(0).standard_normal((S, 128))
    t_ref, t_exp = [], []
    for _ in range(3):
        t = time.perf_counter()
        np.exp(scores)
        t_exp.append(time.perf_counter() - t)
        t = time.perf_counter()
        phi = ref.explain(prob["X"][0], (Z, w))
        t_ref.append(time.perf_counter() - t)
    assert min(t_ref) < 60 * min(t_exp), (min(t_ref), min(t_exp))
    np.testing.assert_allclose(phi[:, 1].sum(), ref.link(ref._outputs(np.array([ref.intercept + prob["X"][0] @ ref.coef]))[0, 1])
                               - ref.expected_value[1], rtol=1e-10)
