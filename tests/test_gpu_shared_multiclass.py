"""Softmax (C classes) and identity (R outputs) heads on the shared-plan path: the softmax coalition kernel
(csrc/dks_multi.cuh), the identity head's tables, and the per-output solves and l1 selection, against the float64
reference (tests/multiclass_reference.py) and the oracle fed the engine's plan."""
import numpy as np
import pytest

from conftest import rel_err
from multiclass_reference import MultiOutputReference

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _problem(seed, G, N, n, C, scale=1.0, weights=False, width=1):
    rng = np.random.default_rng(seed)
    groups = [list(range(k * width, (k + 1) * width)) for k in range(G)]
    D = G * width
    W = rng.normal(0, 1.0 / np.sqrt(D), (C, D)) * 2.0 * scale
    b = rng.normal(0, 0.5, C) * scale
    return dict(W=W, b=b, bg=rng.standard_normal((N, D)), X=rng.standard_normal((n, D)), groups=groups,
                wts=rng.uniform(0.1, 1.0, N) if weights else None)


def _engine(prob, head, link, **kw):
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.predictors import LinearModelSpec
    spec = LinearModelSpec(prob["W"], prob["b"], head)
    names = [f"g{i}" for i in range(len(prob["groups"]))]
    return GpuKernelExplainer(spec, DenseData(prob["bg"], names, prob["groups"], prob["wts"]), link=link, seed=3, **kw)


def _reference(prob, head, link):
    return MultiOutputReference(prob["W"], prob["b"], prob["bg"], prob["groups"], prob["wts"], head=head, link=link)


def _as_list(got, C):
    return got if isinstance(got, list) else [got]


def _check(eng, prob, got, nsamples, head, link, tol=TOL):
    G = len(prob["groups"])
    ref = _reference(prob, head, link)
    plan = eng.shared_plan(G, nsamples)
    got = _as_list(got, ref.C)
    X = prob["X"]
    for i in range(X.shape[0]):
        want = ref.explain(X[i], plan=(plan.dense(), plan.weights))
        for c in range(ref.C):
            assert rel_err(got[c][i], want[:, c]) < tol, (i, c, rel_err(got[c][i], want[:, c]))
    fx = ref.link(ref._outputs(prob["b"] + X @ prob["W"].T))
    for c in range(ref.C):
        np.testing.assert_allclose(got[c].sum(1), fx[:, c] - ref.expected_value[c], rtol=1e-8, atol=1e-8)


# (G, N, n, nsamples): word and nibble-table edges of G, quad / chunk edges of N, instance counts around a warp and the
# SM count
SHAPES = [(2, 1, 1, "auto"), (5, 15, 31, "auto"), (16, 16, 32, 600), (17, 17, 33, 600), (64, 100, 4, 700),
          (65, 128, 3, 700), (128, 129, 2, 900), (12, 300, 132, "auto")]


@pytest.mark.parametrize("C", [3, 4, 8])
@pytest.mark.parametrize("shape", SHAPES)
def test_softmax_shared_path(shape, C):
    G, N, n, ns = shape
    link = "logit" if (G + C) % 2 else "identity"
    weights = N > 1 and (N + C) % 2 == 1     # (one background row has no weights to differ)
    prob = _problem(1000 * C + G + N, G, N, n, C, weights=weights)
    eng = _engine(prob, "softmax", link)
    got = eng.shap_values(prob["X"], nsamples=ns, l1_reg=False)
    path = eng.last_path()
    assert path["shared"] == "softmax" and path["solve"] == "wls_shared", path
    assert path["bg_weights"] == ("weighted" if weights else "uniform")
    _check(eng, prob, got, ns, "softmax", link)


@pytest.mark.parametrize("link", ["logit", "identity"])
def test_softmax_both_links_and_weights(link):
    for weights in (False, True):
        prob = _problem(77, 9, 23, 6, 4, weights=weights)
        eng = _engine(prob, "softmax", link)
        got = eng.shap_values(prob["X"], nsamples=300, l1_reg=False)
        assert eng.last_path()["shared"] == "softmax"
        _check(eng, prob, got, 300, "softmax", link)


def test_softmax_large_plan_beyond_the_simt_kernel():
    """S = 65534 at N = 128 (16 groups, full enumeration): the CUDA-core kernel cannot stage that plan."""
    prob = _problem(5, 16, 128, 2, 3)
    eng = _engine(prob, "softmax", "logit")
    got = eng.shap_values(prob["X"], nsamples=65534, l1_reg=False)
    assert eng.shared_plan(16, 65534).S == 65534 and eng.last_path()["shared"] == "softmax"
    _check(eng, prob, got, 65534, "softmax", "logit")


@pytest.mark.parametrize("C", [3, 8])
def test_softmax_saturated_rows_take_the_clamped_path(C):
    """Scores 30x larger: classes sit 100+ nats apart, so that many rows' den bound falls below 2^-60."""
    prob = _problem(9, 10, 40, 5, C, scale=30.0)
    eng = _engine(prob, "softmax", "identity")
    got = eng.shap_values(prob["X"], nsamples=400, l1_reg=False)
    for c in range(C):
        assert np.all(np.isfinite(got[c]))
    _check(eng, prob, got, 400, "softmax", "identity")


@pytest.mark.parametrize("R", [1, 3])
def test_identity_head_affine_path(R):
    """Closed form phi = XW - Bbar per group, an output scale of 2^30 and 2^-20 (the fixed point of the solve is scaled per
    output), and 65..128 groups."""
    for G, scale in [(8, 1.0), (8, 2.0 ** 30), (8, 2.0 ** -20), (80, 1.0)]:
        prob = _problem(31 + G + R, G, 20, 5, R, scale=scale, weights=True, width=2)
        eng = _engine(prob, "identity", "identity")
        got = _as_list(eng.shap_values(prob["X"], nsamples=300, l1_reg=False), R)
        assert eng.last_path()["shared"] == "affine", eng.last_path()
        wb = prob["wts"] / prob["wts"].sum()
        ref = _reference(prob, "identity", "identity")
        plan = eng.shared_plan(G, 300)
        for r in range(R):
            for g, cols in enumerate(prob["groups"]):
                closed = ((prob["X"][:, cols] - (wb[:, None] * prob["bg"][:, cols]).sum(0)) * prob["W"][r, cols]).sum(1)
                np.testing.assert_allclose(got[r][:, g], closed, rtol=1e-9, atol=1e-9 * scale)
            for i in range(5):
                want = ref.explain(prob["X"][i], plan=(plan.dense(), plan.weights))
                assert rel_err(got[r][i], want[:, r]) < 1e-9


def _oracle(prob, head, link):
    from distributedkernelshap_b200.predictors import LinearModelSpec
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    spec = LinearModelSpec(prob["W"], prob["b"], head)
    names = [f"g{i}" for i in range(len(prob["groups"]))]
    return KernelExplainerOracle(spec, DenseData(prob["bg"], names, prob["groups"], prob["wts"]), link=link)


L1_CASES = [(16, 300), (20, "auto"), (64, 1000), (80, 700)]


@pytest.mark.parametrize("head,C", [("softmax", 3), ("identity", 2)])
@pytest.mark.parametrize("G,ns", L1_CASES)
def test_l1_selection_per_output(head, C, G, ns):
    """The oracle fed the engine's shared plan runs upstream's selection for each output: same selected features, phi
    within 1e-5 -- for 'auto', 'aic', 'bic' and 'num_features(k)', weighted backgrounds included."""
    link = "logit" if head == "softmax" else "identity"
    prob = _problem(400 + G, G, 25, 3, C, weights=G % 2 == 0)
    eng = _engine(prob, head, link)
    orc = _oracle(prob, head, link)
    plan = eng.shared_plan(G, ns)
    for l1_reg in ["auto", "aic", "bic", "num_features(5)"]:
        got = _as_list(eng.shap_values(prob["X"], nsamples=ns, l1_reg=l1_reg), C)
        assert eng.last_path()["solve"] == "l1", (l1_reg, eng.last_path())
        for i in range(prob["X"].shape[0]):
            want = orc.explain(prob["X"][i:i + 1], plan=(plan.dense(), plan.weights), nsamples=ns, l1_reg=l1_reg)
            want = want.reshape(G, C)
            for c in range(C):
                np.testing.assert_array_equal(got[c][i] != 0, want[:, c] != 0, err_msg=f"{l1_reg} {i} {c}")
                assert rel_err(got[c][i], want[:, c]) < TOL, (l1_reg, i, c)


def test_public_api_defaults_regression_and_three_classes():
    """KernelShap(task='regression') on decision_function and a 3-class predict_proba, 20 features, default explain():
    l1_reg='auto' selects features there (2088 of 2^20 - 2 coalitions) and both used to raise."""
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    from distributedkernelshap_b200.predictors import LinearSoftmaxClassifier
    from oracle.shap_kernel_oracle import KernelExplainerOracle
    prob = _problem(12, 20, 30, 3, 3)
    clf = LinearSoftmaxClassifier(prob["W"], prob["b"])
    for predictor, task, link, C in [(clf.decision_function, "regression", "identity", 3),
                                     (clf.predict_proba, "classification", "logit", 3)]:
        ks = KernelShap(predictor, link=link, task=task, seed=4)
        ks.fit(prob["bg"])
        exp = ks.explain(prob["X"])
        plan = ks._explainer.shared_plan(20, "auto")
        orc = KernelExplainerOracle(predictor, prob["bg"], link=link)
        for i in range(3):
            want = orc.explain(prob["X"][i:i + 1], plan=(plan.dense(), plan.weights)).reshape(20, C)
            for c in range(C):
                np.testing.assert_array_equal(exp.shap_values[c][i] != 0, want[:, c] != 0)
                assert rel_err(exp.shap_values[c][i], want[:, c]) < TOL


def test_routing_determinism_and_refusals():
    import torch
    prob = _problem(21, 9, 40, 24, 4, weights=True)
    eng = _engine(prob, "softmax", "logit")
    auto = eng.shap_values(prob["X"], nsamples=300, l1_reg=False)
    assert eng.last_path()["shared"] == "softmax"
    eng.set_kernel("simt")
    simt = eng.shap_values(prob["X"], nsamples=300, l1_reg=False)
    assert eng.last_path()["shared"] == "none" and eng.last_path()["general"] == "simt"
    eng.set_kernel("auto")
    for c in range(4):
        assert rel_err(auto[c], simt[c]) < 2e-6
    # two halves give the bits of the whole
    a = eng.shap_values(prob["X"][:10], nsamples=300, l1_reg=False)
    b = eng.shap_values(prob["X"][10:], nsamples=300, l1_reg=False)
    for c in range(4):
        np.testing.assert_array_equal(np.concatenate([a[c], b[c]]), auto[c])
    # device-resident calls replayed as a CUDA graph: the bits of the host path
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(prob["X"]).cuda()
        phi = torch.zeros((4, 24, 9), dtype=torch.float64, device="cuda")
        for _ in range(4):
            eng.explain_device(X_dev.data_ptr(), 24, phi.data_ptr(), nsamples=300)
        eng.check_status()
        assert eng.graph_launches() >= 2 and eng.last_path()["shared"] == "softmax"
        for c in range(4):
            np.testing.assert_array_equal(phi[c].cpu().numpy(), auto[c])
    eng.set_stream(0)
    # identity head through a graph as well
    iprob = _problem(22, 9, 40, 24, 3, weights=True)
    ieng = _engine(iprob, "identity", "identity")
    ihost = ieng.shap_values(iprob["X"], nsamples=300, l1_reg=False)
    with torch.cuda.stream(stream):
        ieng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(iprob["X"]).cuda()
        phi = torch.zeros((3, 24, 9), dtype=torch.float64, device="cuda")
        for _ in range(4):
            ieng.explain_device(X_dev.data_ptr(), 24, phi.data_ptr(), nsamples=300)
        ieng.check_status()
        assert ieng.graph_launches() >= 2 and ieng.last_path()["shared"] == "affine"
        for c in range(3):
            np.testing.assert_array_equal(phi[c].cpu().numpy(), ihost[c])
    ieng.set_stream(0)


def test_mixed_batch_partial_varying_set_goes_to_the_general_kernel():
    prob = _problem(23, 8, 20, 10, 3)
    prob["bg"][:, 2] = 0.5
    prob["X"][:4, 2] = 0.5                    # group 2 does not vary for the first four rows
    eng = _engine(prob, "softmax", "logit")
    got = eng.shap_values(prob["X"], nsamples=200, l1_reg=False)
    path = eng.last_path()
    assert path["shared"] == "softmax" and path["general"] in ("simt", "tc"), path
    ref = _reference(prob, "softmax", "logit")
    M, _ = eng.varying(prob["X"])
    for i in range(10):
        plan = eng.shared_plan(int(M[i]), 200)
        want = ref.explain(prob["X"][i], plan=(plan.dense(), plan.weights))
        for c in range(3):
            assert rel_err(got[c][i], want[:, c]) < TOL


def test_refusals_beyond_the_new_path():
    prob = _problem(24, 130, 10, 2, 3)
    eng = _engine(prob, "softmax", "logit")
    with pytest.raises(Exception):
        eng.shap_values(prob["X"], nsamples=400, l1_reg=False)
    prob = _problem(25, 20, 10, 2, 3)
    eng = _engine(prob, "identity", "identity", plan_mode="per_instance")
    with pytest.raises(NotImplementedError):
        eng.shap_values(prob["X"], l1_reg="auto")
