"""One-vs-rest head (normalised per-class sigmoids, C = 3..8) on the device: the shared-plan class-sum kernel
(csrc/dks_multi.cuh) with the per-output solves and l1 selection, and the CUDA-core kernel for partial varying sets,
per-instance plans and kernel='simt' -- against the float64 reference (tests/ovr_reference.py) and the oracle."""
import numpy as np
import pytest

from conftest import rel_err
from ovr_reference import OvrReference

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _problem(seed, G, N, n, C, scale=1.0, weights=False):
    rng = np.random.default_rng(seed)
    W = rng.normal(0, 1.0 / np.sqrt(G), (C, G)) * 2.0 * scale
    b = rng.normal(0, 0.5, C) * scale
    return dict(W=W, b=b, bg=rng.standard_normal((N, G)), X=rng.standard_normal((n, G)),
                groups=[[k] for k in range(G)], wts=rng.uniform(0.1, 1.0, N) if weights else None)


def _data(prob):
    from distributedkernelshap_b200.data import DenseData
    return DenseData(prob["bg"], [f"g{i}" for i in range(len(prob["groups"]))], prob["groups"], prob["wts"])


def _engine(prob, link, **kw):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.predictors import LinearModelSpec
    return GpuKernelExplainer(LinearModelSpec(prob["W"], prob["b"], "ovr"), _data(prob), link=link, seed=3, **kw)


def _oracle(prob, link):
    from distributedkernelshap_b200.predictors import LinearModelSpec
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    names = [f"g{i}" for i in range(len(prob["groups"]))]
    return KernelExplainerOracle(LinearModelSpec(prob["W"], prob["b"], "ovr"),
                                 DenseData(prob["bg"], names, prob["groups"], prob["wts"]), link=link)


def _check(prob, got, link, plans, tol=TOL):
    """plans(i) -> (Z, w) of instance i; additivity to 1e-8."""
    ref = OvrReference(prob["W"], prob["b"], prob["bg"], prob["groups"], prob["wts"], link=link)
    X = prob["X"]
    for i in range(X.shape[0]):
        want = ref.explain(X[i], plan=plans(i))
        for c in range(ref.C):
            assert rel_err(got[c][i], want[:, c]) < tol, (i, c, rel_err(got[c][i], want[:, c]))
    fx = ref.link(ref._outputs(prob["b"] + X @ prob["W"].T))
    for c in range(ref.C):
        np.testing.assert_allclose(got[c].sum(1), fx[:, c] - ref.expected_value[c], rtol=1e-8, atol=1e-8)


def _shared(eng, G, ns):
    plan = eng.shared_plan(G, ns)
    return lambda i: (plan.dense(), plan.weights)


# (G, N, n, nsamples): word and nibble-table edges of G, background chunks below / at / above 128 columns
SHAPES = [(2, 1, 1, "auto"), (12, 100, 40, 2048), (16, 128, 32, 600), (17, 17, 33, 600), (64, 100, 4, 700),
          (65, 129, 3, 700), (80, 20, 5, 700), (128, 300, 2, 900)]


@pytest.mark.parametrize("C", [3, 4, 8])
@pytest.mark.parametrize("shape", SHAPES)
def test_ovr_shared_path(shape, C):
    G, N, n, ns = shape
    link = "logit" if (G + C) % 2 else "identity"
    weights = N > 1 and (N + C) % 2 == 1
    prob = _problem(2000 * C + G + N, G, N, n, C, weights=weights)
    eng = _engine(prob, link)
    got = eng.shap_values(prob["X"], nsamples=ns, l1_reg=False)
    path = eng.last_path()
    assert path["shared"] == "ovr" and path["solve"] == "wls_shared", path
    assert path["bg_weights"] == ("weighted" if weights else "uniform")
    assert path["chunks"] == (N + 127) // 128
    _check(prob, got, link, _shared(eng, G, ns))


@pytest.mark.parametrize("link", ["logit", "identity"])
def test_ovr_both_links_and_weights(link):
    for weights in (False, True):
        prob = _problem(77, 9, 23, 6, 4, weights=weights)
        eng = _engine(prob, link)
        got = eng.shap_values(prob["X"], nsamples=300, l1_reg=False)
        assert eng.last_path()["shared"] == "ovr"
        _check(prob, got, link, _shared(eng, 9, 300))


@pytest.mark.parametrize("C", [3, 8])
@pytest.mark.parametrize("shift", [0.0, -40.0, 40.0])
def test_ovr_saturated_rows(C, shift):
    """Scores 30x larger, shifted so that every class sits far below 0, or far above: many rows take the scalar path."""
    prob = _problem(9 + C, 10, 40, 5, C, scale=30.0)
    prob["b"] = prob["b"] + shift
    eng = _engine(prob, "identity")
    got = eng.shap_values(prob["X"], nsamples=400, l1_reg=False)
    assert eng.last_path()["shared"] == "ovr"
    for c in range(C):
        assert np.all(np.isfinite(got[c]))
    _check(prob, got, "identity", _shared(eng, 10, 400))


def test_general_path_partial_sets_simt_and_routing():
    import torch
    prob = _problem(23, 8, 20, 24, 3, weights=True)
    prob["bg"][:, 2] = 0.5
    prob["X"][:4, 2] = 0.5                    # group 2 does not vary for the first four rows
    eng = _engine(prob, "logit")
    auto = eng.shap_values(prob["X"], nsamples=200, l1_reg=False)
    path = eng.last_path()
    assert path["shared"] == "ovr" and path["general"] == "simt", path
    M, _ = eng.varying(prob["X"])
    _check(prob, auto, "logit", lambda i: (eng.shared_plan(int(M[i]), 200).dense(), eng.shared_plan(int(M[i]), 200).weights))
    eng.set_kernel("simt")
    simt = eng.shap_values(prob["X"], nsamples=200, l1_reg=False)
    assert eng.last_path()["shared"] == "none" and eng.last_path()["general"] == "simt"
    eng.set_kernel("auto")
    for c in range(3):
        assert rel_err(auto[c], simt[c]) < 2e-6
    # device-resident calls replayed as a CUDA graph: the bits of the host path
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(prob["X"]).cuda()
        phi = torch.zeros((3, 24, 8), dtype=torch.float64, device="cuda")
        for _ in range(4):
            eng.explain_device(X_dev.data_ptr(), 24, phi.data_ptr(), nsamples=200)
        eng.check_status()
        assert eng.graph_launches() >= 2 and eng.last_path()["shared"] == "ovr"
        for c in range(3):
            np.testing.assert_array_equal(phi[c].cpu().numpy(), auto[c])
    eng.set_stream(0)


def test_caller_plans_and_per_instance_plans():
    from distributedkernelshap_b200.plan import resolve_nsamples
    prob = _problem(31, 7, 12, 6, 4)
    orc = _oracle(prob, "logit")
    # caller-supplied plans
    from distributedkernelshap_b200.plan import build_plan
    eng = _engine(prob, "logit")
    plans = []
    for i in range(6):
        plan = build_plan(7, 60, rng=np.random.RandomState(100 + i))
        plans.append((plan.dense(), plan.weights))
    got = eng.shap_values(prob["X"], plans=plans, nsamples=60, l1_reg=False)
    assert eng.last_path()["general"] == "simt"
    for i in range(6):
        want = orc.explain(prob["X"][i:i + 1], plan=plans[i], nsamples=60, l1_reg=False).reshape(7, 4)
        for c in range(4):
            assert rel_err(got[c][i], want[:, c]) < TOL
    # plans drawn on the device, per instance: the plans the sampler twin says the device drew
    from test_gpu_sampler import _expected_plan
    eng = _engine(prob, "logit", plan_mode="per_instance")
    got = eng.shap_values(prob["X"], nsamples=60, l1_reg=False)
    zb, w = eng.instance_plans()
    Ms, _ = eng.varying(prob["X"])
    for i in range(6):
        M = int(Ms[i])
        S = resolve_nsamples(M, 60)[0]
        k = np.arange(M, dtype=np.uint64)
        twin_z, twin_w = _expected_plan(M, 60, 3, i)
        np.testing.assert_array_equal(zb[i, :S], twin_z)
        np.testing.assert_allclose(w[i, :S], twin_w, rtol=1e-13, atol=0)
        Z = ((twin_z[:, None] >> k[None, :]) & np.uint64(1)).astype(np.uint8)
        want = orc.explain(prob["X"][i:i + 1], plan=(Z, twin_w), nsamples=60, l1_reg=False).reshape(7, 4)
        for c in range(4):
            assert rel_err(got[c][i], want[:, c]) < TOL


@pytest.mark.parametrize("G,ns", [(16, 300), (20, "auto"), (64, 1000)])
def test_l1_selection_per_output(G, ns):
    """The oracle fed the engine's shared plan runs upstream's selection for each output: same selected features, phi
    within 1e-5."""
    prob = _problem(400 + G, G, 25, 3, 3, weights=G % 2 == 0)
    eng = _engine(prob, "logit")
    orc = _oracle(prob, "logit")
    plan = eng.shared_plan(G, ns)
    for l1_reg in ["auto", "aic", "bic", "num_features(5)"]:
        got = eng.shap_values(prob["X"], nsamples=ns, l1_reg=l1_reg)
        path = eng.last_path()
        assert path["solve"] == "l1" and path["shared"] == "ovr", (l1_reg, path)
        for i in range(prob["X"].shape[0]):
            want = orc.explain(prob["X"][i:i + 1], plan=(plan.dense(), plan.weights), nsamples=ns,
                               l1_reg=l1_reg).reshape(G, 3)
            for c in range(3):
                np.testing.assert_array_equal(got[c][i] != 0, want[:, c] != 0, err_msg=f"{l1_reg} {i} {c}")
                assert rel_err(got[c][i], want[:, c]) < TOL, (l1_reg, i, c)


def test_public_api_one_vs_rest_classifier_and_liblinear_rule():
    """KernelShap.fit/explain on an installed OneVsRestClassifier(LogisticRegression()) and on a liblinear-rule
    LogisticRegression stand-in, default arguments (20 features: l1_reg='auto' selects)."""
    from sklearn.linear_model import LogisticRegression
    from sklearn.multiclass import OneVsRestClassifier
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    from oracle.shap_kernel_oracle import KernelExplainerOracle
    rng = np.random.default_rng(12)
    G = 20
    Xt = rng.standard_normal((400, G))
    y = np.argmax(Xt[:, :4] + 0.5 * rng.standard_normal((400, 4)), axis=1)
    ovr = OneVsRestClassifier(LogisticRegression()).fit(Xt, y)

    class Liblinear:
        multi_class, solver = "auto", "liblinear"

        def __init__(self, W, b):
            self.coef_, self.intercept_ = W, b

        def predict_proba(self, X):
            p = 1.0 / (1.0 + np.exp(-(X @ self.coef_.T + self.intercept_)))
            return p / p.sum(axis=1, keepdims=True)

    lib = Liblinear(rng.normal(0, 0.5, (3, G)), rng.normal(0, 0.5, 3))
    bg, X = Xt[:30], rng.standard_normal((3, G))
    for predictor, C in [(ovr.predict_proba, 4), (lib.predict_proba, 3)]:
        ks = KernelShap(predictor, link="logit", task="classification", seed=4)
        ks.fit(bg)
        exp = ks.explain(X)
        assert ks._explainer.last_path()["shared"] == "ovr"
        plan = ks._explainer.shared_plan(G, "auto")
        orc = KernelExplainerOracle(predictor, bg, link="logit")
        for i in range(3):
            want = orc.explain(X[i:i + 1], plan=(plan.dense(), plan.weights)).reshape(G, C)
            for c in range(C):
                np.testing.assert_array_equal(exp.shap_values[c][i] != 0, want[:, c] != 0)
                assert rel_err(exp.shap_values[c][i], want[:, c]) < TOL


def test_refusals_beyond_128_groups():
    prob = _problem(24, 130, 10, 2, 3)
    eng = _engine(prob, "logit")
    with pytest.raises(NotImplementedError):
        eng.shap_values(prob["X"], nsamples=400, l1_reg="auto")
    with pytest.raises(Exception, match="softmax / one-vs-rest / identity head up to 128 groups"):
        eng.shap_values(prob["X"], nsamples=400, l1_reg=False)
