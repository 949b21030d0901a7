"""The exp head (log-link GLM regressors, ``predict = exp(X w + b)``) on the device: the shared-plan path, which reads
y = exp(a(s) + l(s)) - fnull from the instance's tables and the plan's l(s) with no coalition kernel, the CUDA-core kernels
(partial varying sets, per-instance and caller-supplied plans, 65..128-group per-instance plans) with their fp32 range rule,
l1 selection, the public API, the device-resident entry and the refusals -- against the float64 reference
(tests/glm_reference.py) and the oracle."""
import numpy as np
import pytest

from conftest import rel_err
from glm_reference import ExpReference

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _problem(seed, G, N, n, weights=False, shift=0.0, scale=1.0):
    rng = np.random.default_rng(seed)
    w = rng.normal(0, 0.8 / np.sqrt(G), G) * scale
    b = float(rng.normal(0, 0.3)) + shift
    wts = None
    if weights:
        wts = rng.uniform(0.1, 1.0, N)
        if N > 2:
            wts[1] = 0.0                          # zero-weight rows are skipped
    return dict(W=w[None, :], b=np.array([b]), bg=rng.standard_normal((N, G)), X=rng.standard_normal((n, G)),
                groups=[[k] for k in range(G)], wts=wts)


def _data(prob):
    from distributedkernelshap_b200.data import DenseData
    return DenseData(prob["bg"], [f"g{i}" for i in range(len(prob["groups"]))], prob["groups"], prob["wts"])


def _spec(prob):
    from distributedkernelshap_b200.predictors import LinearModelSpec
    return LinearModelSpec(prob["W"], prob["b"], "exp", scalar_out=True)


def _engine(prob, **kw):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    return GpuKernelExplainer(_spec(prob), _data(prob), seed=3, **kw)


def _oracle(prob):
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    names = [f"g{i}" for i in range(len(prob["groups"]))]
    return KernelExplainerOracle(_spec(prob), DenseData(prob["bg"], names, prob["groups"], prob["wts"]))


def _ref(prob):
    return ExpReference(prob["W"][0], prob["b"][0], prob["bg"], prob["groups"], prob["wts"])


def _dense(zb, M):
    """[S] or [S, 2] words -> [S, M] 0/1."""
    zb = zb.reshape(zb.shape[0], -1)
    k = np.arange(M)
    return ((zb[:, k // 64] >> (k % 64).astype(np.uint64)) & np.uint64(1)).astype(np.uint8)


def _check(prob, got, plans, tol):
    """plans(i) -> (Z, w) of instance i: phi per instance vs the reference, additivity to 1e-8 relative (up to upstream's
    snapping of |phi| < 1e-10 to zero)."""
    ref = _ref(prob)
    X = prob["X"]
    assert np.all(np.isfinite(got))
    for i in range(X.shape[0]):
        want = ref.explain(X[i], plan=plans(i))
        assert rel_err(got[i], want) < tol, (i, rel_err(got[i], want))
    fx = ref.predict(X)
    np.testing.assert_allclose(got.sum(1), fx - ref.expected_value, rtol=1e-8, atol=1e-10 * X.shape[1])


def _shared(eng, M, ns):
    plan = eng.shared_plan(M, ns)
    return lambda i: (plan.dense(), plan.weights)


def _own_plans(eng, prob, ns):
    M, _ = eng.varying(prob["X"])
    return lambda i: (eng.shared_plan(int(M[i]), ns).dense(), eng.shared_plan(int(M[i]), ns).weights)


# (G, N, n, nsamples): one- and two-word rows, nibble-table edges of G, single-row to a few hundred background rows
SHAPES = [(2, 1, 3, "auto"), (5, 7, 20, "auto"), (12, 100, 64, 2048), (16, 128, 30, 600), (17, 33, 17, 600),
          (64, 300, 6, 900), (65, 129, 4, 700), (80, 20, 5, 700), (128, 250, 3, 900)]
# uniform and weighted backgrounds (a weighted one needs several rows)
CASES = [(shape, weights) for shape in SHAPES for weights in (False, True) if not (weights and shape[1] < 3)]


@pytest.mark.parametrize("shape,weights", CASES)
def test_shared_path_all_groups_vary(shape, weights):
    G, N, n, ns = shape
    prob = _problem(100 * G + N, G, N, n, weights=weights)
    eng = _engine(prob)
    got = eng.shap_values(prob["X"], nsamples=ns, l1_reg=False)
    path = eng.last_path()
    assert path["shared"] == "exp" and path["solve"] == "wls_shared" and path["general"] in ("none", "simt", "flagged"), path
    _check(prob, got, _shared(eng, G, ns), 1e-9)
    np.testing.assert_allclose(eng.expected_value, _ref(prob).expected_value, rtol=1e-13)


def test_general_kernel_partial_sets_simt_and_device_entry():
    import torch
    prob = _problem(23, 8, 20, 24, weights=True)
    prob["bg"][:, [2, 5]] = 0.5
    prob["X"][:6, 2] = 0.5                        # group 2 does not vary for the first six rows
    prob["X"][3:9, 5] = 0.5
    eng = _engine(prob)
    auto = eng.shap_values(prob["X"], nsamples=200, l1_reg=False)
    path = eng.last_path()
    assert path["shared"] == "exp" and path["general"] == "simt", path
    _check(prob, auto, _own_plans(eng, prob, 200), TOL)
    eng.set_kernel("simt")
    simt = eng.shap_values(prob["X"], nsamples=200, l1_reg=False)
    assert eng.last_path()["shared"] == "none" and eng.last_path()["general"] == "simt"
    _check(prob, simt, _own_plans(eng, prob, 200), TOL)
    eng.set_kernel("auto")
    # device-resident calls replayed as a CUDA graph: the bits of the host path
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(prob["X"]).cuda()
        phi = torch.zeros((1, 24, 8), dtype=torch.float64, device="cuda")
        for _ in range(4):
            eng.explain_device(X_dev.data_ptr(), 24, phi.data_ptr(), nsamples=200)
        eng.check_status()
        assert eng.graph_launches() >= 2 and eng.last_path()["shared"] == "exp"
        np.testing.assert_array_equal(phi[0].cpu().numpy(), auto)
    eng.set_stream(0)


def test_device_entry_full_sets_bit_identical():
    import torch
    prob = _problem(7, 12, 100, 300)
    eng = _engine(prob)
    host = eng.shap_values(prob["X"], nsamples=2048, l1_reg=False)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(prob["X"]).cuda()
        phi = torch.zeros((1, 300, 12), dtype=torch.float64, device="cuda")
        for _ in range(4):
            eng.explain_device(X_dev.data_ptr(), 300, phi.data_ptr(), nsamples=2048)
        eng.check_status()
        assert eng.graph_launches() >= 2 and eng.last_path()["shared"] == "exp"
        np.testing.assert_array_equal(phi[0].cpu().numpy(), host)
    eng.set_stream(0)


@pytest.mark.parametrize("G,ns", [(7, 60), (80, 700)])
def test_per_instance_plans_and_row_offset_splits(G, ns):
    from distributedkernelshap_b200.plan import resolve_nsamples
    prob = _problem(31 + G, G, 12, 6, weights=G > 64)
    eng = _engine(prob, plan_mode="per_instance")
    got = eng.shap_values(prob["X"], nsamples=ns, l1_reg=False)
    assert eng.last_path()["general"] == ("simt_wide" if G > 64 else "simt")
    zb, w = eng.instance_plans()
    S = resolve_nsamples(G, ns)[0]
    _check(prob, got, lambda i: (_dense(zb[i, :S], G), w[i, :S]), TOL)
    a = eng.shap_values(prob["X"][:2], nsamples=ns, l1_reg=False, row_offset=0)
    b = eng.shap_values(prob["X"][2:], nsamples=ns, l1_reg=False, row_offset=2)
    np.testing.assert_array_equal(np.concatenate([a, b]), got)


def test_caller_supplied_oracle_plans():
    from distributedkernelshap_b200.plan import build_plan
    prob = _problem(41, 7, 12, 6)
    eng = _engine(prob)
    orc = _oracle(prob)
    plans = []
    for i in range(6):
        plan = build_plan(7, 60, rng=np.random.RandomState(100 + i))
        plans.append((plan.dense(), plan.weights))
    got = eng.shap_values(prob["X"], plans=plans, nsamples=60, l1_reg=False)
    assert eng.last_path()["general"] == "simt"
    for i in range(6):
        want = orc.explain(prob["X"][i:i + 1], plan=plans[i], nsamples=60, l1_reg=False).reshape(7)
        assert rel_err(got[i], want) < TOL
    _check(prob, got, lambda i: plans[i], TOL)


def _shifted(seed, G, N, n, shift, weights=False):
    """The background's scores shifted by `shift` nats and the instances' by -shift: f(x) stays O(1), while the background
    part of every masked score (the t' of the CUDA-core kernels) leaves the fp32 range rule."""
    prob = _problem(seed, G, N, n, weights=weights, shift=shift)
    w = prob["W"][0]
    prob["X"] = prob["X"] - shift * w / (w @ w)
    return prob


@pytest.mark.parametrize("shift", [-200.0, -80.0, 80.0, 200.0])
def test_range_rule_rows_leave_fp32(shift):
    """Scores shifted so far that every background term 2^t' of the CUDA-core kernels would overflow or flush in fp32:
    those rows are evaluated in float64 -- nothing is clamped.  The shared-plan path has no such limit."""
    prob = _shifted(9, 9, 40, 8, shift, weights=True)
    ns = 300
    for kernel in ("simt", "auto"):
        eng = _engine(prob, kernel=kernel)
        got = eng.shap_values(prob["X"], nsamples=ns, l1_reg=False)
        assert eng.last_path()["general" if kernel == "simt" else "shared"] == ("simt" if kernel == "simt" else "exp")
        _check(prob, got, _shared(eng, 9, ns), 1e-9 if kernel == "auto" else TOL)
    p80 = _shifted(10, 80, 20, 2, shift)
    eng = _engine(p80, plan_mode="per_instance")
    got = eng.shap_values(p80["X"], nsamples=700, l1_reg=False)
    assert eng.last_path()["general"] == "simt_wide"
    zb, w = eng.instance_plans()
    from distributedkernelshap_b200.plan import resolve_nsamples
    S = resolve_nsamples(80, 700)[0]
    _check(p80, got, lambda i: (_dense(zb[i, :S], 80), w[i, :S]), TOL)


@pytest.mark.parametrize("G,ns", [(16, 300), (20, "auto"), (64, 1000), (80, 900)])
def test_l1_selection_full_sets(G, ns):
    prob = _problem(400 + G, G, 25, 3, weights=G % 2 == 0)
    eng = _engine(prob)
    orc = _oracle(prob)
    plan = eng.shared_plan(G, ns)
    for l1_reg in ["auto", "aic", "bic", "num_features(5)"]:
        got = eng.shap_values(prob["X"], nsamples=ns, l1_reg=l1_reg)
        path = eng.last_path()
        assert path["solve"] == "l1" and path["shared"] == "exp", (l1_reg, path)
        for i in range(prob["X"].shape[0]):
            want = orc.explain(prob["X"][i:i + 1], plan=(plan.dense(), plan.weights), nsamples=ns, l1_reg=l1_reg).reshape(G)
            np.testing.assert_array_equal(got[i] != 0, want != 0, err_msg=f"{l1_reg} {i}")
            assert rel_err(got[i], want) < TOL, (l1_reg, i)


def test_l1_selection_partial_sets():
    prob = _problem(77, 10, 15, 6, weights=True)
    prob["bg"][:, [3, 7]] = 1.0
    prob["X"][:, 3] = 1.0                         # group 3 never varies; group 7 varies for half of the rows
    prob["X"][:3, 7] = 1.0
    eng = _engine(prob)
    orc = _oracle(prob)
    M, _ = eng.varying(prob["X"])
    assert set(M.tolist()) == {8, 9}
    for l1_reg, ns in [("auto", 50), ("aic", 50), ("bic", 60), ("num_features(3)", 60)]:
        got = eng.shap_values(prob["X"], nsamples=ns, l1_reg=l1_reg)
        assert eng.last_path()["general_l1"] == 1, l1_reg
        for i in range(6):
            plan = eng.shared_plan(int(M[i]), ns)
            want = orc.explain(prob["X"][i:i + 1], plan=(plan.dense(), plan.weights), nsamples=ns, l1_reg=l1_reg).reshape(10)
            np.testing.assert_array_equal(got[i] != 0, want != 0, err_msg=f"{l1_reg} {i}")
            assert rel_err(got[i], want) < TOL, (l1_reg, i)


def test_public_api_poisson_regressor():
    from sklearn.linear_model import PoissonRegressor
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    from oracle.shap_kernel_oracle import KernelExplainerOracle
    rng = np.random.default_rng(12)
    G = 12
    Xt = rng.standard_normal((500, G))
    y = rng.poisson(np.exp(0.4 * Xt[:, 0] - 0.3 * Xt[:, 1] + 0.2 * Xt[:, 2] + 0.5)).astype(float)
    glm = PoissonRegressor(alpha=0.01).fit(Xt, y)
    bg, X = Xt[:30], rng.standard_normal((4, G))
    ks = KernelShap(glm.predict, task="regression", seed=4)
    ks.fit(bg)
    exp = ks.explain(X)
    assert ks._explainer.last_path()["shared"] == "exp"
    sv = exp.shap_values[0] if isinstance(exp.shap_values, list) else exp.shap_values
    sv = np.asarray(sv).reshape(4, G)
    ev = float(np.ravel(exp.expected_value)[0])
    np.testing.assert_allclose(ev, glm.predict(bg).mean(), rtol=1e-12)
    np.testing.assert_allclose(sv.sum(1), glm.predict(X) - ev, rtol=1e-8)
    plan = ks._explainer.shared_plan(G, "auto")
    orc = KernelExplainerOracle(glm.predict, bg)
    for i in range(4):
        want = orc.explain(X[i:i + 1], plan=(plan.dense(), plan.weights)).reshape(G)
        assert rel_err(sv[i], want) < TOL


def test_non_finite_outputs_are_reported_not_written():
    from distributedkernelshap_b200 import _cabi
    prob = _problem(5, 6, 10, 4)
    eng = _engine(prob)
    X = prob["X"].copy()
    X[2, :] = 2000.0 / np.maximum(np.abs(prob["W"][0]), 1e-3) * np.sign(prob["W"][0])   # f(x) = exp(> 709) = inf
    with pytest.raises(_cabi.DksError) as e:
        eng.shap_values(X, nsamples=40, l1_reg=False)
    assert e.value.code == _cabi.DKS_ERR_NUMERIC
    ok = eng.shap_values(prob["X"], nsamples=40, l1_reg=False)       # the engine stays usable
    assert np.all(np.isfinite(ok))
    bad_bg = _problem(5, 6, 10, 4)
    bad_bg["bg"][0, :] = 5000.0 * np.sign(bad_bg["W"][0])
    with pytest.raises(_cabi.DksError) as e:
        _engine(bad_bg)
    assert e.value.code == _cabi.DKS_ERR_NUMERIC


def test_refusals():
    from distributedkernelshap_b200 import _cabi
    prob = _problem(24, 8, 10, 2)
    with pytest.raises(NotImplementedError, match="link='identity'"):
        _engine(prob, link="logit")
    eng = _engine(prob, kernel="tcgen05")
    with pytest.raises(_cabi.DksError) as e:
        eng.shap_values(prob["X"], nsamples=100, l1_reg=False)
    assert e.value.code == _cabi.DKS_ERR_UNSUPPORTED
    eng = _engine(prob, plan_mode="per_instance")
    with pytest.raises(NotImplementedError):
        eng.shap_values(prob["X"], nsamples=40, l1_reg="auto")       # 40 of 254 coalitions: 'auto' selects
    wide = _problem(25, 130, 10, 2)
    eng = _engine(wide)
    with pytest.raises(NotImplementedError):
        eng.shap_values(wide["X"], nsamples=400, l1_reg="auto")
    with pytest.raises(Exception, match="exp head up to 128 groups"):
        eng.shap_values(wide["X"], nsamples=400, l1_reg=False)
