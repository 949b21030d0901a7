"""Kernel machines on the device (the kernel-machine route, ``last_path()['general'] == 'kmach'``) against the oracle fed
the independent reference model (tests/kernel_machine_reference.py) and the coalition plans the engine used: every kernel
and head, both links, full and partial varying sets, weighted backgrounds, per-instance device plans, caller-supplied plans,
l1 selection, the kernel's own edges, the device-resident entry and its graph replay, the public ``KernelShap`` API and the
refusals."""
import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")
from sklearn.calibration import CalibratedClassifierCV  # noqa: E402
from sklearn.kernel_ridge import KernelRidge  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import MinMaxScaler, StandardScaler  # noqa: E402
from sklearn.svm import SVC, SVR, NuSVC  # noqa: E402

from distributedkernelshap_b200.kernel_machines import KernelMachineSpec, extract_kernel_machine_spec  # noqa: E402
from kernel_machine_reference import reference  # noqa: E402

PLAIN_TOL = 1e-9        # float64 end to end without selection
L1_TOL = 1e-5           # the l1 moments go through the 2^-40 fixed point


def _fit_data(seed, P, n=120):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    s = X[:, 0] - X[:, 0].mean() + 0.5 * (X[:, 1 % P] - X[:, 1 % P].mean()) * (X[:, 2 % P] - X[:, 2 % P].mean())
    return X, (s > 0).astype(int), s, rng


def _model(kind, kernel, P, seed=0):
    """(spec, sklearn method)."""
    X, y, s, _ = _fit_data(seed, P)
    kw = {"gamma": 0.05} if kernel == "sigmoid" else {}
    if kind == "svc":
        fn = make_pipeline(StandardScaler(), SVC(kernel=kernel, **kw)).fit(X, y).decision_function
    elif kind == "svr":
        fn = make_pipeline(MinMaxScaler(), SVR(kernel=kernel, **kw)).fit(X, s).predict
    elif kind == "krr3":
        Y = np.stack([s, 2 * s + y, y - s], axis=1)
        fn = make_pipeline(StandardScaler(), KernelRidge(kernel=kernel, alpha=0.5, **kw)).fit(X, Y).predict
    elif kind == "cal1":
        fn = CalibratedClassifierCV(make_pipeline(StandardScaler(), SVC(kernel=kernel, **kw)), ensemble=False,
                                    cv=3).fit(X, y).predict_proba
    else:   # cal3
        fn = CalibratedClassifierCV(make_pipeline(StandardScaler(), NuSVC(kernel=kernel, **kw)), ensemble=True,
                                    cv=3).fit(X, y).predict_proba
    return extract_kernel_machine_spec(fn), fn


def _problem(seed, P, N, n, constant_cols=(), weights=False, zero_row=False):
    _, _, _, rng = _fit_data(seed, P, 4)
    bg = rng.normal(size=(N, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    for c in constant_cols:              # partial varying sets: x equals the constant background column on some rows
        bg[:, c] = 0.25
        X[::2, c] = 0.25
    w = rng.uniform(0.1, 1.0, N) if weights else None
    if zero_row:
        w[1] = 0.0
    return bg, X, w


def _data(bg, w=None, groups=None):
    from distributedkernelshap_b200.data import DenseData
    groups = groups or [[k] for k in range(bg.shape[1])]
    return DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, w)


def _engine(fn, bg, link, w=None, groups=None, **kw):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    return GpuKernelExplainer(fn, _data(bg, w, groups), link=link, seed=7, **kw)


def _oracle(fn, bg, link, w=None, groups=None):
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    groups = groups or [[k] for k in range(bg.shape[1])]
    return KernelExplainerOracle(fn, DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, w), link=link)


def _as_list(phi):
    return phi if isinstance(phi, list) else [phi]


def _compare(got, oracle, X, plans, tol, l1_reg=False, nsamples="auto"):
    got = _as_list(got)
    worst = 0.0
    for i in range(X.shape[0]):
        want = oracle.explain(X[i:i + 1], plan=plans(i), l1_reg=l1_reg, nsamples=nsamples)
        want = want.reshape(want.shape[0], -1)
        for c in range(want.shape[1]):
            e = rel_err(got[c][i], want[:, c])
            worst = max(worst, e)
            assert e < tol, (i, c, e)
    return worst


def _own_plans(eng, X, ns="auto"):
    M, _ = eng.varying(X)
    return lambda i: None if M[i] < 2 else (eng.shared_plan(int(M[i]), ns).dense(), eng.shared_plan(int(M[i]), ns).weights)


def _check_additivity(eng, fn, got, X, link):
    from distributedkernelshap_b200.data import convert_to_link
    lk = convert_to_link(link)
    fx = np.asarray(fn(X), dtype=np.float64).reshape(X.shape[0], -1)
    ev = np.atleast_1d(eng.expected_value)
    for c, ph in enumerate(_as_list(got)):
        np.testing.assert_allclose(ph.sum(1), lk.f(fx[:, c]) - ev[c], rtol=1e-8, atol=1e-8)


CASES = [(kind, kernel, link) for kind in ("svc", "svr", "krr3", "cal1", "cal3")
         for kernel in (("rbf", "laplacian", "poly", "sigmoid") if kind == "krr3" else ("rbf", "poly", "sigmoid"))
         for link in (("identity", "logit") if kind.startswith("cal") else ("identity",))]


@pytest.mark.parametrize("kind,kernel,link", CASES)
def test_parity_every_kernel_and_head(kind, kernel, link):
    P = 7
    spec, _ = _model(kind, kernel, P)
    fn = reference(spec)
    bg, X, _ = _problem(11, P, N=12, n=4, constant_cols=(6,))
    eng = _engine(spec, bg, link)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "kmach" and eng.last_path()["shared"] == "none"
    M, _ = eng.varying(X)
    assert {int(m) for m in M} == {6, 7}                    # full and partial varying sets in one call
    worst = _compare(got, _oracle(fn, bg, link), X, _own_plans(eng, X), PLAIN_TOL)
    print(f"{kind} {kernel} {link}: max|d|/max|phi| = {worst:.2e}")
    _check_additivity(eng, fn, got, X, link)
    if kind.startswith("cal"):
        out = _as_list(got)
        np.testing.assert_array_equal(out[0], -out[1] + 0.0)    # class 0 is the exact negation of class 1


def test_weighted_background_with_a_zero_weight_row():
    P = 6
    spec, _ = _model("cal3", "rbf", P)
    bg, X, w = _problem(3, P, N=10, n=3, weights=True, zero_row=True)
    eng = _engine(spec, bg, "logit", w=w)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "kmach"
    _compare(got, _oracle(reference(spec), bg, "logit", w=w), X, _own_plans(eng, X), PLAIN_TOL)


def test_grouped_columns():
    P = 8
    spec, _ = _model("krr3", "laplacian", P)
    groups = [[0, 1], [2], [3, 4, 5], [6], [7]]
    bg, X, _ = _problem(5, P, N=9, n=3)
    eng = _engine(spec, bg, "identity", groups=groups)
    got = eng.shap_values(X, l1_reg=False, nsamples=20)
    _compare(got, _oracle(reference(spec), bg, "identity", groups=groups), X, _own_plans(eng, X, 20), PLAIN_TOL,
             nsamples=20)


def test_per_instance_device_plans():
    P = 9
    spec, _ = _model("svr", "rbf", P)
    bg, X, _ = _problem(21, P, N=8, n=5, constant_cols=(8,))
    eng = _engine(spec, bg, "identity", plan_mode="per_instance")
    got = eng.shap_values(X, l1_reg=False, nsamples=300)
    assert eng.last_path()["general"] == "kmach"
    zb, w = eng.instance_plans()
    M, _ = eng.varying(X)
    from distributedkernelshap_b200.plan import resolve_nsamples

    def plans(i):
        S, _ = resolve_nsamples(int(M[i]), 300)
        k = np.arange(int(M[i]))
        Z = ((zb[i, :S, None] >> k.astype(np.uint64)) & np.uint64(1)).astype(np.uint8)
        return Z, w[i, :S]
    _compare(got, _oracle(reference(spec), bg, "identity"), X, plans, PLAIN_TOL, nsamples=300)


def test_caller_supplied_plans():
    P = 6
    spec, _ = _model("cal1", "poly", P)
    bg, X, _ = _problem(8, P, N=7, n=3)
    rng = np.random.default_rng(0)
    plans = []
    for i in range(3):
        Z = rng.integers(0, 2, size=(40, P)).astype(np.uint8)
        Z[0] = 0
        Z[1] = 1
        Z[2:2 + P] = np.eye(P, dtype=np.uint8)
        plans.append((Z, rng.uniform(0.1, 1.0, 40)))
    eng = _engine(spec, bg, "logit")
    got = eng.shap_values(X, l1_reg=False, nsamples=40, plans=plans)
    assert eng.last_path()["general"] == "kmach"
    _compare(got, _oracle(reference(spec), bg, "logit"), X, lambda i: plans[i], PLAIN_TOL, nsamples=40)


@pytest.mark.parametrize("l1_reg", ["auto", "aic", "num_features(4)"])
def test_l1_selection(l1_reg):
    P = 14                                    # 'auto' selects: 2076 of 16382 coalitions evaluated
    spec, _ = _model("cal1", "rbf", P)
    bg, X, _ = _problem(31, P, N=5, n=3, constant_cols=(13,))
    eng = _engine(spec, bg, "logit")
    got = eng.shap_values(X, l1_reg=l1_reg)
    path = eng.last_path()
    assert path["general"] in ("kmach", "simt", "none") and path["general_l1"] == 1, path
    oracle = _oracle(reference(spec), bg, "logit")
    _compare(got, oracle, X, _own_plans(eng, X), L1_TOL, l1_reg=l1_reg)


def _hand_spec(n_sv, P, kernel="rbf", gamma=0.3, seed=0, R=1):
    rng = np.random.default_rng(seed)
    return KernelMachineSpec(rng.normal(size=(n_sv, P)), [0, n_sv], rng.normal(size=(n_sv, R)), rng.normal(size=(1, R)),
                             rng.uniform(0.5, 2.0, (1, P)), rng.normal(size=(1, P)) * 0.1, [gamma], kernel, 3, 0.5,
                             "identity", P, scalar_out=R == 1)


@pytest.mark.parametrize("n_sv", [1, 31, 32, 33, 65])
def test_support_vector_counts_around_the_tile(n_sv):
    P = 6
    spec = _hand_spec(n_sv, P, seed=n_sv)
    bg, X, _ = _problem(4, P, N=6, n=3, constant_cols=(5,))
    eng = _engine(spec, bg, "identity")
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "kmach"
    _compare(got, _oracle(reference(spec), bg, "identity"), X, _own_plans(eng, X), PLAIN_TOL)
    _check_additivity(eng, reference(spec), got, X, "identity")


@pytest.mark.parametrize("shape", [("m0", 4), ("m1", 4), ("m2", 4), ("g64_first", 64), ("g64_last", 64)])
def test_varying_set_edges(shape):
    name, P = shape
    spec = _hand_spec(40, P, kernel="poly", gamma=0.05)
    rng = np.random.default_rng(2)
    bg = rng.normal(size=(5, P))
    X = rng.normal(size=(3, P))
    if name in ("m0", "m1", "m2"):
        keep = {"m0": 0, "m1": 1, "m2": 2}[name]
        bg[:, keep:] = 0.5
        X[:, keep:] = 0.5
    else:
        c = 0 if name == "g64_first" else P - 1                 # group 0 or 63 does not vary
        bg[:, c] = 0.5
        X[:, c] = 0.5
    eng = _engine(spec, bg, "identity")
    ns = 300 if P == 64 else "auto"
    got = eng.shap_values(X, l1_reg=False, nsamples=ns)
    M, _ = eng.varying(X)
    assert set(int(m) for m in M) == ({"m0": {0}, "m1": {1}, "m2": {2}}.get(name) or {63})
    if name != "m0":
        assert eng.last_path()["general"] == "kmach"
    _compare(got, _oracle(reference(spec), bg, "identity"), X, _own_plans(eng, X, ns), PLAIN_TOL, nsamples=ns)
    _check_additivity(eng, reference(spec), got, X, "identity")


def test_grid_stride_batches_are_bit_identical_to_each_instance_alone():
    P = 5
    spec, _ = _model("cal3", "rbf", P)
    rng = np.random.default_rng(9)
    bg = rng.normal(size=(6, P))
    n = 132 * 8 * 3 + 17                      # more than three instances per CTA at the kernel's largest grid
    X = rng.normal(size=(n, P))
    X[::3, 4] = bg[0, 4]                      # mixed M between real instances
    bg[:, 4] = bg[0, 4]
    eng = _engine(spec, bg, "identity")
    got = np.stack(eng.shap_values(X, l1_reg=False, nsamples=60))
    assert eng.last_path()["general"] == "kmach"
    for i in (0, 1, 2, 500, n - 1):
        alone = np.stack(eng.shap_values(X[i:i + 1], l1_reg=False, nsamples=60))
        np.testing.assert_array_equal(got[:, i], alone[:, 0])


def test_rbf_kernel_underflow():
    P = 4
    spec = _hand_spec(20, P, gamma=400.0)     # gamma t > 745 for nearly every pair: exp underflows to 0
    bg, X, _ = _problem(6, P, N=5, n=3)
    eng = _engine(spec, bg, "identity")
    got = eng.shap_values(X, l1_reg=False)
    assert np.all(np.isfinite(got))
    _compare(got, _oracle(reference(spec), bg, "identity"), X, _own_plans(eng, X), PLAIN_TOL)
    _check_additivity(eng, reference(spec), got, X, "identity")


def _km_smem_bytes(C, S, R, G, cal):
    tile = 32 * (1 + R + G + 16 * ((G + 3) // 4))          # explain_kmach_kernel's layout (dks_kmach.cuh, smem_bytes)
    return 8 * ((C + cal) * S + max(tile, 63 * 63 + 64)) + 4 * 64


def test_shared_memory_limit():
    import torch
    from distributedkernelshap_b200._cabi import DksError
    P, R = 13, 8
    limit = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    S = ((limit - 4 * 64) // 8 - max(32 * (1 + R + P + 16 * 4), 63 * 63 + 64)) // R
    assert _km_smem_bytes(R, S, R, P, 0) <= limit < _km_smem_bytes(R, S + 1, R, P, 0) and S + 1 < 2 ** P - 2
    spec = _hand_spec(10, P, R=R)
    bg, X, _ = _problem(7, P, N=3, n=2)
    eng = _engine(spec, bg, "identity")
    got = eng.shap_values(X, l1_reg=False, nsamples=S)
    assert eng.last_path()["general"] == "kmach"
    _compare(got, _oracle(reference(spec), bg, "identity"), X, _own_plans(eng, X, S), PLAIN_TOL, nsamples=S)
    with pytest.raises(DksError, match="shared memory"):
        _engine(spec, bg, "identity").shap_values(X, l1_reg=False, nsamples=S + 1)


def test_graph_replay_is_bit_identical_to_the_host_path():
    import torch
    P = 8
    spec, _ = _model("krr3", "rbf", P)
    bg, X, _ = _problem(41, P, N=10, n=16, constant_cols=(7,))
    eng = _engine(spec, bg, "identity")
    want = np.stack(eng.shap_values(X, nsamples=200, l1_reg=False))
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(X).cuda()
        phi = torch.zeros((want.shape[0], 16, P), dtype=torch.float64, device="cuda")
        for _ in range(4):
            eng.explain_device(X_dev.data_ptr(), 16, phi.data_ptr(), nsamples=200)
        eng.check_status()
        assert eng.graph_launches() >= 1
        assert eng.last_path()["general"] == "kmach"
        np.testing.assert_array_equal(phi.cpu().numpy(), want)
    eng.set_stream(0)


def _adult():
    from distributedkernelshap_b200.datasets import adult_like
    d = adult_like(n_explain=20, n_background=40, seed=0)
    X_all = np.concatenate([d["background"], d["X_explain"]])
    y = d["predictor"].predict(X_all)
    return d, X_all, y


def test_kernel_shap_on_a_scaled_svc_decision_function():
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    d, X_all, y = _adult()
    svc = make_pipeline(StandardScaler(), SVC()).fit(X_all, y)
    ks = KernelShap(svc.decision_function, feature_names=d["group_names"], seed=0)
    ks.fit(d["background"], group_names=d["group_names"], groups=d["groups"])
    exp = ks.explain(d["X_explain"][:5], silent=True)          # default kwargs: nsamples='auto', l1_reg='auto'
    assert ks._explainer.last_path()["general"] in ("kmach", "none")
    fx = svc.decision_function(d["X_explain"][:5])
    np.testing.assert_allclose(np.asarray(exp.shap_values[0]).sum(1), fx - exp.expected_value[0], rtol=1e-8, atol=1e-8)


def test_kernel_shap_on_a_calibrated_svc_with_the_logit_link():
    from distributedkernelshap_b200.data import convert_to_link
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    d, X_all, y = _adult()
    cal = CalibratedClassifierCV(make_pipeline(StandardScaler(), SVC()), ensemble=False).fit(X_all, y)
    ks = KernelShap(cal.predict_proba, link="logit", feature_names=d["group_names"], seed=0)
    ks.fit(d["background"], group_names=d["group_names"], groups=d["groups"])
    exp = ks.explain(d["X_explain"][:5], silent=True)
    fx = convert_to_link("logit").f(cal.predict_proba(d["X_explain"][:5]))
    for c in range(2):
        np.testing.assert_allclose(exp.shap_values[c].sum(1), fx[:, c] - exp.expected_value[c], rtol=1e-8, atol=1e-8)


def test_refusals():
    from distributedkernelshap_b200._cabi import DksError
    P = 5
    spec, _ = _model("svc", "rbf", P)
    bg, X, _ = _problem(2, P, N=6, n=2)
    for kernel in ("tcgen05", "shared"):
        eng = _engine(spec, bg, "identity", kernel=kernel)
        with pytest.raises(DksError, match="kernel-machine"):
            eng.shap_values(X, l1_reg=False)
    X65, y65, _, _ = _fit_data(0, 65)
    wide = SVC().fit(X65, y65)
    with pytest.raises(NotImplementedError, match="64"):
        _engine(wide.decision_function, X65[:4], "identity")
    eng = _engine(spec, bg, "identity")
    Xn = X.copy()
    Xn[1, 2] = np.nan
    with pytest.raises(ValueError, match="instance 1"):
        eng.shap_values(Xn, l1_reg=False)
    bgn = bg.copy()
    bgn[3, 0] = np.nan
    with pytest.raises(ValueError, match="background row 3"):
        _engine(spec, bgn, "identity")
