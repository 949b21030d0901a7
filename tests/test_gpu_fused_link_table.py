"""The fused kernel's per-row link table (dks_fused.cuh, DESIGN.md 5.0.1): y(i, s) read from a float64-fitted table
instead of summed over the background.  Against the float64 reference at the fused path's edges (uniform and weighted
backgrounds), no less accurate than the exact loop (``fused_table`` 0), the same bits under every layout, the exact loop
for passes outside a table's domain, and a plan whose table would be too large keeps the exact loop."""
import numpy as np
import pytest

from test_gpu_kernel_paths import _check, _engine, _expect, _problem, _reference
from test_gpu_weighted_background import _wproblem

pytestmark = pytest.mark.gpu


def _phi(eng, prob):
    return np.stack(eng.shap_values(prob["X"], nsamples=2048, l1_reg=False), axis=-1)


def _max_err(eng, prob, got):
    ref = _reference(prob)
    plans = []
    for x in prob["X"]:
        v = ref.varying(x)
        plan = eng.shared_plan(len(v), 2048) if len(v) >= 2 else None
        plans.append(None if plan is None else (plan.dense(), plan.weights))
    return float(np.abs(got[..., 1] - ref.shap_values(prob["X"], plans)[..., 1]).max())


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("G", [2, 13, 14, 16])
@pytest.mark.parametrize("N", [1, 17, 64, 100, 101, 128])
def test_table_path_matches_reference(N, G, weighted):
    make = _wproblem if weighted else _problem
    prob = make(9100 + 7 * N + G + 1000 * weighted, G=G, N=N, n=24)
    eng = _engine(prob)
    got = _phi(eng, prob)
    _expect(eng.last_path(), shared="fused", solve="fused", fused_table=1)
    assert eng.fused_table_info(G)["bytes"] > 0
    _check(eng, prob, got, 2048, "fused link table")
    eng.set_option("fused_table", 0)
    exact = _phi(eng, prob)
    _expect(eng.last_path(), shared="fused", fused_table=0)
    assert _max_err(eng, prob, got) <= _max_err(eng, prob, exact) + 1e-12


def test_passes_outside_the_domain_take_the_exact_loop():
    prob = _problem(9400, G=12, N=100, n=40)
    coef = prob["clf"].coef_.reshape(-1)
    prob["X"][0] = -14.0 * coef / (coef @ coef)            # linear score -14: 2^x Dm > 2^33 on whole rows
    eng = _engine(prob)
    before = eng.fused_table_info(12)["fallback_passes"]
    got = _phi(eng, prob)
    _expect(eng.last_path(), shared="fused", fused_table=1)
    assert eng.fused_table_info(12)["fallback_passes"] > before
    _check(eng, prob, got, 2048, "fused link table, exact-loop passes")


@pytest.mark.parametrize("weighted", [False, True])
def test_same_bits_under_every_layout(weighted):
    make = _wproblem if weighted else _problem
    prob = make(9500 + weighted, G=12, N=100, n=300)
    eng = _engine(prob)
    want = _phi(eng, prob)
    for opt, val in (("fused_warps", 1), ("fused_warps", 4), ("fused_batch", 8), ("fused_batch", 32)):
        eng.set_option(opt, val)
        got = _phi(eng, prob)
        _expect(eng.last_path(), shared="fused", fused_table=1)
        assert np.array_equal(got, want), (opt, val, np.abs(got - want).max())
        eng.set_option(opt, 0)


def test_plan_without_table_keeps_the_exact_loop():
    prob = _problem(9600, G=12, N=100, n=40)
    coef = prob["clf"].coef_.reshape(-1)
    prob["bg"][0] = 1000.0 * coef / (coef @ coef)          # one background row thousands of log2 units away: over budget
    eng = _engine(prob)
    got = _phi(eng, prob)
    _expect(eng.last_path(), shared="fused", fused_table=0)
    assert eng.fused_table_info(12)["bytes"] == 0
    eng.set_option("fused_table", 0)
    assert np.array_equal(_phi(eng, prob), got)
