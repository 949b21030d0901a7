"""l1 feature selection for instances whose varying set is partial (M < G <= 64 groups): the CUDA-core kernel forms their
moment vectors and l1_lars_kernel selects and solves on the shared plan of each instance's own M.  Every instance is
compared with the oracle fed ``eng.shared_plan(M_i, nsamples)`` and the same ``l1_reg``: identical non-zero pattern per
output, phi within 1e-5, additivity to 1e-8."""
import numpy as np
import pytest

from conftest import make_problem, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _problem(seed, G, N, n, head, C=1, kappa=1.0, weights=False, const_rows=None):
    """One column per group.  ``const_rows`` {group: rows}: the group is constant in the background and equal to it in
    those rows of X, which therefore have a partial varying set."""
    rng = np.random.default_rng(seed)
    R = 1 if head == "binary_logistic" else C
    bg, X = rng.standard_normal((N, G)), rng.standard_normal((n, G))
    for g, rows in (const_rows or {}).items():
        bg[:, g] = 0.5
        X[rows, g] = 0.5
    return dict(W=rng.normal(0, 2.0 / np.sqrt(G), (R, G)), b=rng.normal(0, 0.5, R), bg=bg, X=X, head=head, kappa=kappa,
                groups=[[k] for k in range(G)], wts=rng.uniform(0.2, 1.0, N) if weights else None)


def _pair(prob, link, **kw):
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.predictors import LinearModelSpec
    from oracle.shap_kernel_oracle import DenseData as ODenseData, KernelExplainerOracle
    spec = LinearModelSpec(prob["W"], prob["b"], prob["head"], kappa=prob["kappa"])
    names = [f"g{i}" for i in range(len(prob["groups"]))]
    eng = GpuKernelExplainer(spec, DenseData(prob["bg"], names, prob["groups"], prob["wts"]), link=link, seed=3, **kw)
    orc = KernelExplainerOracle(spec, ODenseData(prob["bg"], names, prob["groups"], prob["wts"]), link=link)
    return eng, orc


def _as_list(got):
    return got if isinstance(got, list) else [got]


def _check(eng, orc, X, nsamples, l1_reg, rows=None):
    """Explains X, checks the rows given (all by default) against the oracle and additivity; returns phi and M."""
    got = _as_list(eng.shap_values(X, nsamples=nsamples, l1_reg=l1_reg))
    lfx = eng.link_predictions().reshape(X.shape[0], -1)
    path = eng.last_path()
    M, _ = eng.varying(X)
    G = len(eng.data.groups)
    ev = np.atleast_1d(eng.expected_value)
    for i in (range(X.shape[0]) if rows is None else rows):
        plan = eng.shared_plan(int(M[i]), nsamples)
        want = np.asarray(orc.explain(X[i:i + 1], plan=(plan.dense(), plan.weights), nsamples=nsamples,
                                      l1_reg=l1_reg)).reshape(G, -1)
        for c in range(len(got)):
            np.testing.assert_array_equal(got[c][i] != 0, want[:, c] != 0, err_msg=f"instance {i} (M={M[i]}), output {c}")
            assert rel_err(got[c][i], want[:, c]) < TOL, (i, c, rel_err(got[c][i], want[:, c]))
    for c in range(len(got)):
        np.testing.assert_allclose(got[c].sum(1), lfx[:, c] - ev[c], rtol=1e-8, atol=1e-8)
    return got, M, path


# rows 0-3 lack group 3, rows 2-5 lack group 7: M in {14, 15, 16} of 16, full-set rows 6 and 7 share the call
MIXED = {3: [0, 1, 2, 3], 7: [2, 3, 4, 5]}


@pytest.mark.parametrize("head,C,kappa,link,weights,l1_reg", [
    ("binary_logistic", 1, 2.0, "logit", False, "auto"),
    ("binary_logistic", 1, 1.0, "identity", True, "aic"),
    ("binary_logistic", 1, 2.0, "logit", True, "num_features(15)"),
    ("softmax", 3, 1.0, "logit", False, "bic"),
    ("softmax", 3, 1.0, "identity", True, "num_features(4)"),
    ("ovr", 3, 1.0, "logit", True, "auto"),
    ("ovr", 4, 1.0, "identity", False, "num_features(20)"),
    ("identity", 1, 1.0, "identity", True, "auto"),
    ("identity", 2, 1.0, "identity", False, "aic"),
])
def test_partial_sets_select_like_upstream(head, C, kappa, link, weights, l1_reg):
    prob = _problem(11 + C + int(kappa), 16, 20, 8, head, C=C, kappa=kappa, weights=weights, const_rows=MIXED)
    eng, orc = _pair(prob, link)
    got, M, path = _check(eng, orc, prob["X"], 300, l1_reg)
    assert set(M.tolist()) == {14, 15, 16}
    assert path["general_l1"] == 1 and path["general"] == "simt" and path["solve"] == "l1", path
    if l1_reg.startswith("num_features"):
        k = int(l1_reg[13:-1])
        for i in range(8):
            assert np.count_nonzero(got[-1][i]) <= min(k, M[i])


def test_make_problem_and_dense_tabular_with_constant_columns():
    prob = make_problem(seed=21, n=6, N=15, widths=(1,) * 14 + (2,), kappa=1.0, weights=True, constant_groups=(2, 9))
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from oracle.shap_kernel_oracle import DenseData as ODenseData, KernelExplainerOracle
    eng = GpuKernelExplainer(prob["clf"].predict_proba, DenseData(prob["bg"], prob["group_names"], prob["groups"],
                                                                  prob["weights"]), link="logit", seed=1)
    orc = KernelExplainerOracle(prob["clf"].predict_proba, ODenseData(prob["bg"], prob["group_names"], prob["groups"],
                                                                      prob["weights"]), link="logit")
    _, M, _ = _check(eng, orc, prob["X"], 400, "auto")
    assert set(M.tolist()) == {13}
    from distributedkernelshap_b200.datasets import dense_tabular
    d = dense_tabular(n=6, n_features=30, n_background=40, seed=5)
    d["background"][:, [4, 9]] = 0.25
    d["X_explain"][:3, [4, 9]] = 0.25            # half the rows have M = 28, the rest all 30 groups
    eng = GpuKernelExplainer(d["predictor"].predict_proba, d["background"], link="logit", seed=2)
    orc = KernelExplainerOracle(d["predictor"].predict_proba, d["background"], link="logit")
    _, M, path = _check(eng, orc, d["X_explain"], "auto", "auto")
    assert set(M.tolist()) == {28, 30} and path["general_l1"] == 1 and path["solve"] == "l1"


def test_ungrouped_adult_like_through_the_public_api():
    """49 singleton groups, 100 background rows: every instance has 47 or 48 varying groups, none all 49."""
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    from oracle.shap_kernel_oracle import KernelExplainerOracle
    d = adult_like(2560, 100, seed=0)
    X = d["X_explain"][:200]
    ks = KernelShap(d["predictor"].predict_proba, link="logit", seed=4)
    ks.fit(d["background"])
    exp = ks.explain(X)
    eng = ks._explainer
    path = eng.last_path()
    assert path["general_l1"] == 1 and path["general"] == "simt", path
    t = eng.general_l1_timings_ms()
    assert t["general"] > 0 and t["lars"] > 0
    M, _ = eng.varying(X)
    assert M.max() < 49 and M.min() >= 47
    orc = KernelExplainerOracle(d["predictor"].predict_proba, d["background"], link="logit")
    for i in (0, 57, 199):
        plan = eng.shared_plan(int(M[i]), "auto")
        want = orc.explain(X[i:i + 1], plan=(plan.dense(), plan.weights)).reshape(49, 2)
        for c in range(2):
            np.testing.assert_array_equal(exp.shap_values[c][i] != 0, want[:, c] != 0)
            assert rel_err(exp.shap_values[c][i], want[:, c]) < TOL


def test_mixed_call_is_bit_identical_to_its_parts():
    prob = _problem(31, 16, 20, 8, "binary_logistic", kappa=2.0, const_rows=MIXED)
    eng, _ = _pair(prob, "logit")
    both = eng.shap_values(prob["X"], nsamples=300, l1_reg="auto")
    full = eng.shap_values(prob["X"][6:], nsamples=300, l1_reg="auto")
    assert eng.last_path()["general_l1"] == 0
    part = eng.shap_values(prob["X"][:6], nsamples=300, l1_reg="auto")
    for c in range(2):
        np.testing.assert_array_equal(both[c][6:], full[c])
        np.testing.assert_array_equal(both[c][:6], part[c])


def test_auto_selects_per_instance_m_at_the_20_percent_boundary():
    """G = 15, nsamples 'auto': M = 13 evaluates 2074 of 8190 coalitions (does not select), M = 14 2076 of 16382 (selects)."""
    prob = _problem(41, 15, 30, 6, "binary_logistic", kappa=2.0, const_rows={2: [0, 1], 5: [0, 1, 2, 3]})
    eng, orc = _pair(prob, "logit")
    plain = eng.shap_values(prob["X"], l1_reg=False)
    plain_general = eng.last_path()["general"]
    got, M, path = _check(eng, orc, prob["X"], "auto", "auto", rows=[2, 3])
    assert M.tolist() == [13, 13, 14, 14, 15, 15]
    assert path["general_l1"] == 1 and path["general"] == plain_general, (path, plain_general)
    for c in range(2):
        np.testing.assert_array_equal(got[c][:2], plain[c][:2])           # M = 13: the plain WLS, same kernel, same bits


def test_row_chunks_equal_one_call(monkeypatch):
    from distributedkernelshap_b200 import engine
    prob = _problem(51, 16, 20, 8, "ovr", C=3, const_rows=MIXED)
    eng, _ = _pair(prob, "logit")
    whole = eng.shap_values(prob["X"], nsamples=300, l1_reg="auto")
    monkeypatch.setattr(engine, "MAX_ROWS_PER_CALL", 3)        # row blocks of 3 * 2 // 3 = 2 for the three-class head
    chunked = eng.shap_values(prob["X"], nsamples=300, l1_reg="auto")
    for c in range(3):
        np.testing.assert_array_equal(whole[c], chunked[c])


def test_refusals():
    """A selecting instance whose CUDA-core staging does not fit shared memory, and forced kernels, raise status 3."""
    from distributedkernelshap_b200._cabi import DksError
    prob = _problem(61, 64, 512, 3, "softmax", C=3, const_rows={0: [0, 1, 2]})       # M = 63 everywhere
    eng, _ = _pair(prob, "logit")
    with pytest.raises(DksError) as ei:
        eng.shap_values(prob["X"], l1_reg="auto")
    assert ei.value.code == 3
    prob = _problem(62, 12, 20, 4, "binary_logistic", kappa=2.0, const_rows={3: [0, 1, 2, 3]})       # M = 11: tc covers it
    for kernel in ("simt", "tcgen05"):
        eng, _ = _pair(prob, "logit", kernel=kernel)
        with pytest.raises(DksError) as ei:
            eng.shap_values(prob["X"], nsamples=300, l1_reg="auto")
        assert ei.value.code == 3
        eng.shap_values(prob["X"], nsamples=300, l1_reg=False)
