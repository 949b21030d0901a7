"""The mixture head (``sum_k pi_k h(z_k)``: calibrated, soft-voting and bagged linear classifiers) on the device: the
shared-plan route (one pass of the member head's coalition kernel per member, 2..128 groups, one- and two-word rows), the
CUDA-core kernel for partial varying sets, per-instance and caller-supplied plans, l1 selection on full and partial varying
sets, the device-resident entry, row blocks, the public API and the refusals -- against the float64 reference
(tests/mixture_reference.py) and the oracle calling the real estimator."""
import warnings

import numpy as np
import pytest

from conftest import rel_err
from mixture_reference import MixtureReference

pytestmark = pytest.mark.gpu
TOL = 1e-5

MODELS = {"binary2": ("binary_logistic", 1, 2), "binary5": ("binary_logistic", 1, 5), "binary32": ("binary_logistic", 1, 32),
          "ovr5x3": ("ovr", 3, 5), "softmax3x4": ("softmax", 4, 3)}


def _problem(seed, G, N, n, model, weights=False):
    """weights: False (uniform), True (random weights) or 'kmeans' (a k-means summary of 4 N rows into N weighted
    centroids, as ``KernelShap.fit(summarise_background=True)`` makes)."""
    member, Rm, K = MODELS[model]
    rng = np.random.default_rng(seed)
    R = K * Rm
    W = rng.normal(0, 2.0 / np.sqrt(G), (R, G))
    b = rng.normal(0, 0.5, R)
    pi = rng.uniform(0.2, 1.0, K)
    bg, wts = rng.standard_normal((N, G)), None
    if weights == "kmeans":
        from distributedkernelshap_b200.data import kmeans
        summary = kmeans(rng.standard_normal((4 * N, G)), N, round_values=False)
        bg, wts = np.asarray(summary.data, dtype=np.float64), np.asarray(summary.weights, dtype=np.float64)
    elif weights:
        wts = rng.uniform(0.1, 1.0, N)
    return dict(W=W, b=b, pi=pi / pi.sum(), member=member, bg=bg, X=rng.standard_normal((n, G)),
                groups=[[k] for k in range(G)], wts=wts)


def _spec(prob):
    from distributedkernelshap_b200.predictors import LinearModelSpec
    return LinearModelSpec(prob["W"], prob["b"], "mixture", pi=prob["pi"], member=prob["member"])


def _data(prob):
    from distributedkernelshap_b200.data import DenseData
    return DenseData(prob["bg"], [f"g{i}" for i in range(len(prob["groups"]))], prob["groups"], prob["wts"])


def _engine(prob, link, **kw):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    return GpuKernelExplainer(_spec(prob), _data(prob), link=link, seed=3, **kw)


def _ref(prob, link):
    return MixtureReference(prob["W"], prob["b"], prob["pi"], prob["member"], prob["bg"], prob["groups"], prob["wts"],
                            link=link)


def _oracle(prob, link):
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    names = [f"g{i}" for i in range(len(prob["groups"]))]
    return KernelExplainerOracle(_spec(prob), DenseData(prob["bg"], names, prob["groups"], prob["wts"]), link=link)


def _dense(zb, M):
    zb = zb.reshape(zb.shape[0], -1)
    k = np.arange(M)
    return ((zb[:, k // 64] >> (k % 64).astype(np.uint64)) & np.uint64(1)).astype(np.uint8)


def _check(prob, got, link, plans, tol=TOL):
    """plans(i) -> (Z, w) of instance i; additivity to 1e-8."""
    ref = _ref(prob, link)
    X = prob["X"]
    for i in range(X.shape[0]):
        want = ref.explain(X[i], plan=plans(i))
        for c in range(ref.C):
            assert rel_err(got[c][i], want[:, c]) < tol, (i, c, rel_err(got[c][i], want[:, c]))
    fx = ref.link(ref.predict(X))
    for c in range(ref.C):
        np.testing.assert_allclose(got[c].sum(1), fx[:, c] - ref.expected_value[c], rtol=1e-8, atol=1e-8)


def _own_plans(eng, ns, X):
    M, _ = eng.varying(X)
    return lambda i: (eng.shared_plan(int(M[i]), ns).dense(), eng.shared_plan(int(M[i]), ns).weights)


# (G, N, n, nsamples): one background chunk and three (N = 300); one-word rows of 12 and 20 groups, two-word rows of 80
@pytest.mark.parametrize("model", list(MODELS))
@pytest.mark.parametrize("shape", [(12, 100, 12, "auto"), (20, 300, 4, 1000), (80, 100, 3, 700)])
def test_shared_plan_route(model, shape):
    G, N, n, ns = shape
    member, Rm, K = MODELS[model]
    link = "logit" if (G + K) % 2 else "identity"
    weights = "kmeans" if (N + K) % 2 == 1 else False
    prob = _problem(100 * K + G + Rm, G, N, n, model, weights=weights)
    eng = _engine(prob, link)
    got = eng.shap_values(prob["X"], nsamples=ns, l1_reg=False)
    path = eng.last_path()
    assert path["shared"] == "mixture" and path["solve"] in ("pmat", "wls_shared"), path
    assert path["bg_weights"] == ("weighted" if weights else "uniform")
    assert path["chunks"] % K == 0 and path["chunks"] // K == (N + 127) // 128, path      # member x chunk launches
    _check(prob, got, link, _own_plans(eng, ns, prob["X"]))
    if G <= 64 and K * Rm * N * G * 4 < 150_000:
        # the CUDA-core kernel computes the same thing
        eng.set_kernel("simt")
        simt = eng.shap_values(prob["X"], nsamples=ns, l1_reg=False)
        assert eng.last_path()["shared"] == "none" and eng.last_path()["general"] == "simt"
        for c in range(len(got)):
            assert rel_err(simt[c], got[c]) < 2e-5


@pytest.mark.parametrize("link", ["logit", "identity"])
def test_oracle_on_plans_the_engine_used(link):
    prob = _problem(5, 9, 40, 5, "ovr5x3", weights=True)
    eng = _engine(prob, link)
    got = eng.shap_values(prob["X"], nsamples=200, l1_reg=False)
    orc = _oracle(prob, link)
    plan = eng.shared_plan(9, 200)
    for i in range(5):
        want = orc.explain(prob["X"][i:i + 1], plan=(plan.dense(), plan.weights), nsamples=200, l1_reg=False)
        want = np.asarray(want).reshape(9, 3)
        for c in range(3):
            assert rel_err(got[c][i], want[:, c]) < TOL


def test_partial_sets_per_instance_and_caller_plans():
    from distributedkernelshap_b200.plan import build_plan, resolve_nsamples
    prob = _problem(23, 8, 20, 12, "binary5", weights=True)
    prob["bg"][:, 2] = 0.5
    prob["X"][:4, 2] = 0.5                        # group 2 does not vary for the first four rows
    eng = _engine(prob, "logit")
    got = eng.shap_values(prob["X"], nsamples=200, l1_reg=False)
    assert eng.last_path()["general"] == "simt"
    _check(prob, got, "logit", _own_plans(eng, 200, prob["X"]))
    # device-drawn per-instance plans, and split calls that give the same bits
    pe = _engine(prob, "logit", plan_mode="per_instance")
    got = pe.shap_values(prob["X"], nsamples=60, l1_reg=False)
    assert pe.last_path()["general"] == "simt"
    zb, w = pe.instance_plans()
    M, _ = pe.varying(prob["X"])
    _check(prob, got, "logit", lambda i: (_dense(zb[i, :resolve_nsamples(int(M[i]), 60)[0]], int(M[i])),
                                          w[i, :resolve_nsamples(int(M[i]), 60)[0]]))
    a = pe.shap_values(prob["X"][:5], nsamples=60, l1_reg=False, row_offset=0)
    b = pe.shap_values(prob["X"][5:], nsamples=60, l1_reg=False, row_offset=5)
    for c in range(2):
        np.testing.assert_array_equal(np.concatenate([a[c], b[c]]), got[c])
    # caller-supplied plans
    plans = []
    for i in range(12):
        m = int(M[i])
        plan = build_plan(m, 50, rng=np.random.RandomState(100 + i))
        plans.append((plan.dense(), plan.weights))
    got = eng.shap_values(prob["X"], plans=plans, nsamples=50, l1_reg=False)
    _check(prob, got, "logit", lambda i: plans[i])


@pytest.mark.parametrize("model", ["binary5", "ovr5x3"])
def test_l1_selection_full_and_partial_sets(model):
    prob = _problem(77, 10, 15, 6, model, weights=True)
    eng = _engine(prob, "logit")
    orc = _oracle(prob, "logit")
    C = 2 if model.startswith("binary") else 3
    for partial in (False, True):
        if partial:
            prob["bg"][:, 7] = 1.0
            prob["X"][:3, 7] = 1.0                # group 7 does not vary for half of the rows
            eng, orc = _engine(prob, "logit"), _oracle(prob, "logit")
        M, _ = eng.varying(prob["X"])
        for l1_reg, ns in [("auto", 50), ("aic", 50), ("num_features(3)", 60)]:
            got = eng.shap_values(prob["X"], nsamples=ns, l1_reg=l1_reg)
            path = eng.last_path()
            assert path["shared"] == "mixture" and path["solve"] == "l1", (l1_reg, path)
            assert path["general_l1"] == (1 if partial else 0), (l1_reg, path)
            for i in range(6):
                plan = eng.shared_plan(int(M[i]), ns)
                want = orc.explain(prob["X"][i:i + 1], plan=(plan.dense(), plan.weights), nsamples=ns, l1_reg=l1_reg)
                want = np.asarray(want).reshape(10, C)
                for c in range(C):
                    np.testing.assert_array_equal(got[c][i] != 0, want[:, c] != 0, err_msg=f"{l1_reg} {i} {c}")
                    assert rel_err(got[c][i], want[:, c]) < TOL, (l1_reg, i, c)


def test_device_entry_graph_replay_and_row_blocks(monkeypatch):
    import torch
    from distributedkernelshap_b200 import engine as engine_mod
    prob = _problem(7, 12, 100, 64, "ovr5x3")
    eng = _engine(prob, "logit")
    host = eng.shap_values(prob["X"], nsamples=2048, l1_reg=False)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(prob["X"]).cuda()
        phi = torch.zeros((3, 64, 12), dtype=torch.float64, device="cuda")
        for _ in range(4):
            eng.explain_device(X_dev.data_ptr(), 64, phi.data_ptr(), nsamples=2048)
        eng.check_status()
        assert eng.graph_launches() >= 2 and eng.last_path()["shared"] == "mixture"
        for c in range(3):
            np.testing.assert_array_equal(phi[c].cpu().numpy(), host[c])
    eng.set_stream(0)
    monkeypatch.setattr(engine_mod, "MAX_ROWS_PER_CALL", 40)     # 40 // 15 = 2 rows per call
    assert eng._rows_per_call() == 2
    blocked = eng.shap_values(prob["X"], nsamples=2048, l1_reg=False)
    for c in range(3):
        np.testing.assert_array_equal(blocked[c], host[c])


@pytest.mark.parametrize("C", [2, 3])
def test_kernel_shap_on_calibrated_linear_svc(C):
    from sklearn.calibration import CalibratedClassifierCV
    from sklearn.svm import LinearSVC
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    from oracle.shap_kernel_oracle import KernelExplainerOracle
    rng = np.random.default_rng(12 + C)
    G = 10
    Xt = rng.standard_normal((400, G))
    y = np.argmax(Xt[:, :C] + 0.5 * rng.standard_normal((400, C)), axis=1) if C > 2 else (Xt[:, 0] > 0).astype(int)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        clf = CalibratedClassifierCV(LinearSVC(), method="sigmoid").fit(Xt, y)
    bg, X = Xt[:40], rng.standard_normal((5, G))
    ks = KernelShap(clf.predict_proba, link="logit", seed=4)
    ks.fit(bg)
    exp = ks.explain(X, l1_reg=False)
    assert ks._explainer.spec.activation == "mixture" and ks._explainer.last_path()["shared"] == "mixture"
    plan = ks._explainer.shared_plan(G, "auto")
    orc = KernelExplainerOracle(clf.predict_proba, bg, link="logit")
    for i in range(5):
        want = np.asarray(orc.explain(X[i:i + 1], plan=(plan.dense(), plan.weights), l1_reg=False)).reshape(G, C)
        for c in range(C):
            assert rel_err(np.asarray(exp.shap_values[c])[i], want[:, c]) < TOL
    ev = np.ravel(exp.expected_value)
    p = clf.predict_proba(X)
    for c in range(C):
        np.testing.assert_allclose(np.asarray(exp.shap_values[c]).sum(1), np.log(p[:, c] / (1 - p[:, c])) - ev[c],
                                   rtol=1e-8, atol=1e-8)


def test_refusals():
    from distributedkernelshap_b200 import _cabi
    prob = _problem(3, 8, 20, 4, "binary2")
    eng = _engine(prob, "logit", kernel="tcgen05")
    with pytest.raises(_cabi.DksError) as e:
        eng.shap_values(prob["X"], nsamples=100, l1_reg=False)
    assert e.value.code == _cabi.DKS_ERR_UNSUPPORTED
    wide = _problem(4, 80, 10, 2, "binary2")
    eng = _engine(wide, "logit", plan_mode="per_instance")           # per-instance plans of 65..128 groups
    with pytest.raises(_cabi.DksError) as e:
        eng.shap_values(wide["X"], nsamples=700, l1_reg=False)
    assert e.value.code == _cabi.DKS_ERR_UNSUPPORTED
    eng = _engine(wide, "logit", kernel="simt")                      # two-word rows exist on the shared-plan route only
    with pytest.raises(_cabi.DksError) as e:
        eng.shap_values(wide["X"], nsamples=700, l1_reg=False)
    assert e.value.code == _cabi.DKS_ERR_UNSUPPORTED
    beyond = _problem(5, 130, 4, 1, "binary2")
    eng = _engine(beyond, "logit")
    with pytest.raises(_cabi.DksError) as e:
        eng.shap_values(beyond["X"], nsamples=800, l1_reg=False)
    assert e.value.code == _cabi.DKS_ERR_UNSUPPORTED
    eng = _engine(prob, "logit")
    with pytest.raises(NotImplementedError, match="fixed Lasso"):
        eng.shap_values(prob["X"], nsamples=100, l1_reg=0.01)
